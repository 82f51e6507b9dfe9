"""Time EWC++ at CIFAR-100 shapes (batch 10): CUDA events around a train_learner call of --steps batches with the penalty
live (the call after a first one) and the published fisher_update_after (50), after a warm-up call that captures the
graphs.  The EWC++ step (b200ocl_net_sgd_step_ewc) and the same learner with the plain SGD step in its place
alternate over --repeats runs; the median is reported, with kernel launches per step (the library's counter plus the
launches replayed inside CUDA graphs).  Then the fused kernel alone: CUDA events around --kernel-iters launches with the
penalty live, with and without the EMA, and its bytes/s over the arena passes it needs (8 fp32 arenas, 10 with the EMA),
next to the HBM3 lower bound at 3.35 TB/s (computed, not measured).  Prints the card and its power limit first.

    python tools/ewc_step.py [--steps S] [--repeats R] [--kernel-iters K]
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

BATCH, NUM_CLASSES, HBM_BYTES_PER_S = 10, 100, 3.35e12


def learner():
    from b200ocl import nets, registry
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick', 'kd_trick_star')}
    params = SimpleNamespace(data='cifar100', cuda=True, epoch=1, batch=BATCH, verbose=False, mem_size=0,
                             eps_mem_batch=10, mem_iters=1, update='random', retrieve='random', agent='EWC',
                             optimizer='SGD', learning_rate=0.1, weight_decay=0.0, lambda_=100.0, alpha=0.9,
                             fisher_update_after=50, error_analysis=False, trick=trick)
    return registry.extra_agents['EWC'](nets.setup_architecture(params), None, params)


def task(rs, n):
    return rs.randint(0, 256, (n, 32, 32, 3)).astype(np.uint8), (np.arange(n) % NUM_CLASSES)[rs.permutation(n)]


def time_config(fused, steps):
    from b200ocl import _native
    from b200ocl.engine import graph_launch_count
    rs = np.random.RandomState(7)
    with contextlib.redirect_stdout(sys.stderr):
        lrn = learner()
    eng = lrn.engine
    lrn.train_learner(*task(rs, 20 * BATCH))           # warm-up call: captures the graphs; the penalty is live after it
    if not fused:
        eng.sgd_step_ewc = lambda lr, wd, *a, **k: eng.sgd_step(lr, wd)
    x, y = task(rs, steps * BATCH)
    torch.cuda.synchronize()
    launches = _native.launch_count() + graph_launch_count()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    lrn.train_learner(x, y)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps, (_native.launch_count() + graph_launch_count() - launches) / steps


def time_kernel(iters):
    """The fused kernel on a CIFAR-100 engine with the penalty live: the library's per-launch CUDA events
    (b200ocl_profile_*) give the kernel alone; events around the whole loop give the entry point with its repack."""
    import ctypes
    from b200ocl import _native, nets
    lib = _native.lib()
    eng = nets.EngineModel(32, NUM_CLASSES).engine
    n = eng.state.params.numel()
    eng.state.grads.normal_(0, 1e-3)
    eng.ewc_state().normalized.uniform_()
    out = {}
    for ema in (False, True):
        for _ in range(10):
            eng.sgd_step_ewc(1e-6, 0.0, 100.0, True, ema, 0.1, 0.018)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            eng.sgd_step_ewc(1e-6, 0.0, 100.0, True, ema, 0.1, 0.018)
        b.record()
        torch.cuda.synchronize()
        ms_entry = a.elapsed_time(b) / iters
        lib.b200ocl_profile_begin()
        for _ in range(iters):
            eng.sgd_step_ewc(1e-6, 0.0, 100.0, True, ema, 0.1, 0.018)
        torch.cuda.synchronize()
        name, ms, cnt, work = ctypes.create_string_buffer(64), ctypes.c_double(), ctypes.c_int(), ctypes.c_double()
        kernel_ms = None
        for k in range(lib.b200ocl_profile_end()):
            lib.b200ocl_profile_get(k, name, 64, ctypes.byref(ms), ctypes.byref(cnt), ctypes.byref(work))
            if name.value.decode() == 'sgd_ewc':
                kernel_ms = ms.value / cnt.value
        nbytes = 4.0 * n * (10 if ema else 8)
        out['ema' if ema else 'no_ema'] = {'kernel_us': kernel_ms * 1e3, 'entry_with_repack_us': ms_entry * 1e3,
                                           'arena_bytes': nbytes, 'bytes_per_s': nbytes / (kernel_ms * 1e-3),
                                           'hbm_lower_bound_us': nbytes / HBM_BYTES_PER_S * 1e6}
    return n, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--kernel-iters', type=int, default=500)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    np.random.seed(0)
    torch.manual_seed(0)
    print('card:', card())
    res = {True: [], False: []}
    for _ in range(args.repeats):                    # the configurations alternate; each run builds a fresh learner
        for fused in (True, False):
            res[fused].append(time_config(fused, args.steps))
    for fused, r in res.items():
        print(json.dumps({'step': 'ewc' if fused else 'plain', 'ms_per_step': float(np.median([t[0] for t in r])),
                          'launches_per_step': float(np.median([t[1] for t in r])),
                          'runs_ms_per_step': [t[0] for t in r], 'steps': args.steps}), flush=True)
    n, k = time_kernel(args.kernel_iters)
    print(json.dumps({'kernel': 'net_sgd_ewc_kernel', 'n_params': n, **k}), flush=True)


if __name__ == '__main__':
    main()
