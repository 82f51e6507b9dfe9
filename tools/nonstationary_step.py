"""Time the float64 input path of the non-stationary tasks (--cl_type ni --ns_type noise|occlusion|blur: float64 NHWC
images in [0, 1]) against the uint8 path on the same images.

  * Task preparation, the host-to-device upload and the kernel reported separately, CUDA events around each: 4500
    images at 84x84 (NS-Mini-ImageNet with 10 factors) and 9000 at 32x32 (cifar100_noise.yml's 5 factors), float64 then
    uint8, alternating over --repeats runs; the upload from pageable memory (what StreamFeeder does) and, for
    comparison, from an already pinned host copy.  The kernel is timed over --launches back-to-back launches, and its
    achieved rate is the bytes it has to move (12 per value for float64, 5 for uint8) over that time.
  * ER steps (batch 10, a memory of 5000) over one call of the whole task, float64 against uint8 images: the call's
    time includes its stream preparation, so the difference is what the float64 input costs a task.

Prints the card and its power limit first and last, then one JSON line per result.

    python tools/nonstationary_step.py [--repeats R] [--launches L]
"""
import argparse
import contextlib
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from tricks_step import card  # noqa: E402

BATCH, MEM = 10, 5000
TASKS = {'mini_imagenet': (4500, 84), 'cifar100': (9000, 32)}


def _events():
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def prepare_times(x, launches):
    """(pageable upload ms, pinned upload ms, kernel ms per launch) for one task x (numpy NHWC)."""
    from b200ocl import ops
    host = torch.from_numpy(x)
    pinned = host.pin_memory()
    perm = torch.randperm(len(x)).cuda()
    torch.cuda.synchronize()
    a, b = _events()
    a.record()
    dev = host.to('cuda')
    b.record()
    torch.cuda.synchronize()
    up = a.elapsed_time(b)
    del dev
    a.record()
    dev = pinned.to('cuda', non_blocking=True)
    b.record()
    torch.cuda.synchronize()
    up_pinned = a.elapsed_time(b)
    ops.stream_prepare(dev, perm)                 # warm-up
    torch.cuda.synchronize()
    a.record()
    for _ in range(launches):
        ops.stream_prepare(dev, perm)
    b.record()
    torch.cuda.synchronize()
    return up, up_pinned, a.elapsed_time(b) / launches


def learner(data):
    from b200ocl import nets, registry
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick', 'kd_trick_star')}
    params = SimpleNamespace(data=data, cuda=True, epoch=1, batch=BATCH, verbose=False, mem_size=MEM, eps_mem_batch=10,
                             mem_iters=1, update='random', retrieve='random', agent='ER', k=3, aser_type='asvm',
                             n_smp_cls=1.5, num_tasks=10, buffer_tracker=False, optimizer='SGD', learning_rate=0.1,
                             weight_decay=0.0, temp=0.07, head='mlp', subsample=50, error_analysis=False, trick=trick)
    return registry.agents['ER'](nets.setup_architecture(params), None, params)


def er_call_ms(data, x, y):
    """ms of one ER train_learner call over the whole task (a fresh learner, warmed up on 20 steps of the same kind)."""
    hw = x.shape[1]
    with contextlib.redirect_stdout(sys.stderr):
        lrn = learner(data)
        lrn.buffer.update(torch.rand(MEM, 3, hw, hw, device='cuda'), torch.randint(0, 100, (MEM,), device='cuda'))
        lrn.train_learner(x[:20 * BATCH], y[:20 * BATCH])
    torch.cuda.synchronize()
    a, b = _events()
    a.record()
    with contextlib.redirect_stdout(sys.stderr):
        lrn.train_learner(x, y)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--launches', type=int, default=20)
    ap.add_argument('--no-er', action='store_true', help='time the preparation only')
    args = ap.parse_args()
    torch.cuda.set_device(0)
    torch.manual_seed(0)
    print('card:', card(), flush=True)
    rs = np.random.RandomState(7)
    images = {}
    for data, (n, hw) in TASKS.items():
        u8 = rs.randint(0, 256, (n, hw, hw, 3)).astype(np.uint8)
        f64 = np.clip(u8 / 255.0 + 0.12 * rs.standard_normal(u8.shape), 0.0, 1.0)      # a noise task, factor 1.2
        images[data] = {'float64': f64, 'uint8': u8, 'y': (np.arange(n) % 100)[rs.permutation(n)]}
    configs = [(d, k) for d in TASKS for k in ('float64', 'uint8')]
    prep = {c: [] for c in configs}
    er = {c: [] for c in configs}
    for _ in range(args.repeats):                     # the configurations alternate
        for c in configs:
            prep[c].append(prepare_times(images[c[0]][c[1]], args.launches))
            torch.cuda.empty_cache()
        if not args.no_er:
            for c in configs:
                er[c].append(er_call_ms(c[0], images[c[0]][c[1]], images[c[0]]['y']))
                torch.cuda.empty_cache()
    for (data, kind), r in prep.items():
        n, hw = TASKS[data]
        r = np.array(r)
        kernel = float(np.median(r[:, 2]))
        moved = n * hw * hw * 3 * (12 if kind == 'float64' else 5)
        print(json.dumps({'prepare': kind, 'data': data, 'images': n, 'hw': hw,
                          'host_mb': n * hw * hw * 3 * (8 if kind == 'float64' else 1) / 1e6,
                          'upload_ms': float(np.median(r[:, 0])), 'upload_pinned_ms': float(np.median(r[:, 1])),
                          'kernel_ms': kernel, 'kernel_gb_per_s': moved / kernel / 1e6, 'runs': r.tolist()}), flush=True)
    for (data, kind), r in er.items():
        if r:
            n, hw = TASKS[data]
            print(json.dumps({'er_call': kind, 'data': data, 'images': n, 'steps': n // BATCH, 'mem_size': MEM,
                              'call_ms': float(np.median(r)), 'ms_per_step': float(np.median(r)) / (n // BATCH),
                              'runs_ms': r}), flush=True)
    print('card:', card(), flush=True)


if __name__ == '__main__':
    main()
