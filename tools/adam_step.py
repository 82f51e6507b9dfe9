"""Time Adam against SGD at CIFAR-100 shapes (batch 10): CUDA events around a train_learner call of --steps batches
after a warm-up call that captures the graphs, for ER (random retrieval, reservoir update, mem 5000) and SCR (mem
5000, 100 memory rows per step), each with params.optimizer 'Adam' (lr 0.001) and 'SGD' (lr 0.1).  The four
configurations alternate over --repeats runs; the median is reported, with kernel launches per step (the library's
counter plus the launches replayed inside CUDA graphs).  Then the Adam kernel alone (the library's per-launch CUDA
events over --kernel-iters launches of b200ocl_net_adam_step) with its bytes/s over the 28 B per parameter it must
move (read p, g, exp_avg, exp_avg_sq; write p, exp_avg, exp_avg_sq), next to the HBM3 lower bound at 3.35 TB/s
(computed, not measured).  Prints the card and its power limit first.

    python tools/adam_step.py [--steps S] [--repeats R] [--kernel-iters K]
"""
import argparse
import contextlib
import ctypes
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


def learner(agent, optimizer):
    from b200ocl import nets, registry
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick', 'kd_trick_star')}
    params = SimpleNamespace(data='cifar100', cuda=True, epoch=1, batch=BATCH, verbose=False, mem_size=5000,
                             eps_mem_batch=100 if agent == 'SCR' else 10, mem_iters=1, update='random',
                             retrieve='random', agent=agent, k=3, aser_type='asvm', n_smp_cls=1.5, num_tasks=10,
                             buffer_tracker=False, optimizer=optimizer,
                             learning_rate=0.001 if optimizer == 'Adam' else 0.1, weight_decay=0.0, temp=0.07,
                             head='mlp', subsample=50, error_analysis=False, trick=trick)
    return registry.agents[agent](nets.setup_architecture(params), None, params)


def task(rs, n):
    return rs.randint(0, 256, (n, 32, 32, 3)).astype(np.uint8), (np.arange(n) % NUM_CLASSES)[rs.permutation(n)]


def time_config(agent, optimizer, steps):
    from b200ocl import _native
    from b200ocl.engine import graph_launch_count
    rs = np.random.RandomState(7)
    with contextlib.redirect_stdout(sys.stderr):
        lrn = learner(agent, optimizer)
    lrn.buffer.update(torch.rand(5000, 3, 32, 32, device='cuda'), torch.randint(0, NUM_CLASSES, (5000,), device='cuda'))
    lrn.train_learner(*task(rs, 20 * BATCH))           # warm-up call: captures the graphs
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
    """b200ocl_net_adam_step on a CIFAR-100 classifier engine: the library's per-launch CUDA events give the kernel
    alone; events around the whole loop give the entry point with its repack."""
    from b200ocl import _native, nets
    lib = _native.lib()
    eng = nets.EngineModel(32, NUM_CLASSES).engine
    n = eng.state.params.numel()
    eng.state.grads.normal_(0, 1e-3)
    for _ in range(10):
        eng.adam_step(1e-6)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        eng.adam_step(1e-6)
    b.record()
    torch.cuda.synchronize()
    ms_entry = a.elapsed_time(b) / iters
    lib.b200ocl_profile_begin()
    for _ in range(iters):
        eng.adam_step(1e-6)
    torch.cuda.synchronize()
    name, ms, cnt, work = ctypes.create_string_buffer(64), ctypes.c_double(), ctypes.c_int(), ctypes.c_double()
    kernel_ms = None
    for k in range(lib.b200ocl_profile_end()):
        lib.b200ocl_profile_get(k, name, 64, ctypes.byref(ms), ctypes.byref(cnt), ctypes.byref(work))
        if name.value.decode() == 'adam':
            kernel_ms = ms.value / cnt.value
    nbytes = 28.0 * n
    return {'kernel': 'arena_step_kernel<Adam<true>>', 'n_params': n, 'kernel_us': kernel_ms * 1e3,
            'entry_with_repack_us': ms_entry * 1e3,
            'bytes': nbytes, 'bytes_per_s': nbytes / (kernel_ms * 1e-3),
            'hbm_lower_bound_us': nbytes / HBM_BYTES_PER_S * 1e6}


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
    configs = [(a, o) for a in ('ER', 'SCR') for o in ('Adam', 'SGD')]
    res = {c: [] for c in configs}
    for _ in range(args.repeats):                    # the configurations alternate; each run builds a fresh learner
        for c in configs:
            res[c].append(time_config(*c, args.steps))
    for (agent, opt), r in res.items():
        print(json.dumps({'agent': agent, 'optimizer': opt, 'ms_per_step': float(np.median([t[0] for t in r])),
                          'launches_per_step': float(np.median([t[1] for t in r])),
                          'runs_ms_per_step': [t[0] for t in r], 'steps': args.steps}), flush=True)
    print(json.dumps(time_kernel(args.kernel_iters)), flush=True)


if __name__ == '__main__':
    main()
