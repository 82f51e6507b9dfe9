"""Per-launch timings of one eval feature pass / train forward+backward at the batch sizes of the
replay step (GPU box).  Uses the library's own CUDA-event profiler; every launch carries ~4 us of event
overhead, so compare rows, not absolute values.   usage: python tools/net_layers.py [out.csv]"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, 'gpurun_out', 'net_layers.csv')
os.environ['B200OCL_PROF_DUMP'] = out
from b200ocl import _native, engine  # noqa: E402
from b200ocl.engine import Engine  # noqa: E402


def main():
    lib = _native.lib()
    engine.set_graphs(False)      # the per-launch profiler records eager launches only
    torch.manual_seed(0)
    eng = Engine(32, 100)
    g = torch.Generator(device='cuda').manual_seed(1)
    eng.state.params.copy_(0.05 * torch.randn(eng.info.n_params, device='cuda', generator=g))
    eng.pack()
    if os.path.exists(out):
        os.remove(out)

    def mark(tag):
        with open(out, 'a') as fh:
            fh.write('# %s\n' % tag)

    for n in (210,):
        x = torch.randn(n, 3, 32, 32, device='cuda', generator=g)
        for _ in range(3):
            eng.features_eval(x)
        torch.cuda.synchronize()
        mark('features_eval N=%d' % n)
        lib.b200ocl_profile_begin()
        eng.features_eval(x)
        lib.b200ocl_profile_end()
    for n in (10, 20, 110):
        x = torch.randn(n, 3, 32, 32, device='cuda', generator=g)
        for _ in range(3):
            o, ws = eng.forward_train(x)
            eng.backward(x, torch.ones_like(o) / n, ws)
        torch.cuda.synchronize()
        mark('train fwd+bwd N=%d' % n)
        lib.b200ocl_profile_begin()
        o, ws = eng.forward_train(x)
        eng.backward(x, torch.ones_like(o) / n, ws)
        lib.b200ocl_profile_end()
    print(open(out).read())


if __name__ == '__main__':
    main()
