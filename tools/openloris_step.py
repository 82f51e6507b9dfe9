"""Time the engine's agents at OpenLORIS shapes (50x50 inputs, 69 classes, 160-wide features) against the same agents at
CIFAR-100 shapes: batch 10, a memory of 5000 images, CUDA events around a train_learner call of --steps replay steps
after one warm-up call of 20 steps.  ER (random retrieval, reservoir update), ER with ASER retrieval and update, and SCR
(mlp head, 100 memory rows per step); GDumb is timed over one train_mem epoch (re-initialisation included) of its full
memory.  Every call carries all the classes, as OpenLORIS's new-instance tasks do.  The configurations alternate over
--repeats runs and the median is reported.  Then one ER and one GDumb run at OpenLORIS shapes with CUDA graphs off and
the library's per-launch profiler on give the time per kernel class (the 50-wide layer-1 maps are too wide for the
halo-strip kernels and run the fp32 patch convolution and weight gradient), each with the card and its power limit
read right after the profiled call.  Prints the card and its power limit first, then one JSON line per result.

    python tools/openloris_step.py [--steps S] [--repeats R]
"""
import argparse
import contextlib
import ctypes
import json
import os
import random
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from core50_step import task  # noqa: E402
from tricks_step import card  # noqa: E402

BATCH, MEM = 10, 5000
SHAPES = {'openloris': (50, 69), 'cifar100': (32, 100)}


def learner(kind, data):
    from b200ocl import nets, registry
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick', 'kd_trick_star')}
    agent = {'er': 'ER', 'aser': 'ER', 'scr': 'SCR', 'gdumb': 'GDUMB'}[kind]
    plug = 'ASER' if kind == 'aser' else 'random'
    params = SimpleNamespace(data=data, cuda=True, epoch=1, batch=BATCH, verbose=False, mem_size=MEM,
                             eps_mem_batch=100 if kind == 'scr' else 10, mem_iters=1, update=plug, retrieve=plug,
                             agent=agent, k=3, aser_type='asvm', n_smp_cls=1.5, num_tasks=10, buffer_tracker=False,
                             optimizer='SGD', learning_rate=0.1, weight_decay=0.0, temp=0.07, head='mlp', subsample=50,
                             mem_epoch=1, clip=10.0, minlr=0.0005, error_analysis=False, trick=trick)
    return registry.agents[agent](nets.setup_architecture(params), None, params)


def build(kind, data):
    hw, ncls = SHAPES[data]
    rs = np.random.RandomState(7)
    random.seed(7)
    with contextlib.redirect_stdout(sys.stderr):
        lrn = learner(kind, data)
    if kind == 'gdumb':
        y = np.arange(MEM) % ncls
        lrn.before_train(None, y)
        slots, sources = lrn.memory.plan(y)
        lrn.memory.write(torch.from_numpy(rs.rand(MEM, 3, hw, hw).astype(np.float32)).cuda(), y, slots, sources)
    else:
        lrn.buffer.update(torch.rand(MEM, 3, hw, hw, device='cuda'), torch.randint(0, ncls, (MEM,), device='cuda'))
    return lrn, rs


def run(lrn, rs, kind, data, steps):
    """ms per replay step of one timed call (GDumb: per train_mem step)."""
    hw, ncls = SHAPES[data]
    if kind == 'gdumb':
        fn = lrn.train_mem
        steps = len(lrn.memory) // BATCH
    else:
        x, y = task(rs, steps * BATCH, hw, np.arange(ncls))
        fn = lambda: lrn.train_learner(x, y)    # noqa: E731
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    with contextlib.redirect_stdout(sys.stderr):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def time_config(kind, data, steps):
    lrn, rs = build(kind, data)
    hw, ncls = SHAPES[data]
    with contextlib.redirect_stdout(sys.stderr):
        if kind == 'gdumb':
            lrn.train_mem()                      # warm-up epoch: captures the graphs
        else:
            lrn.train_learner(*task(rs, 20 * BATCH, hw, np.arange(ncls)))
    return run(lrn, rs, kind, data, steps)


def profile(kind, steps):
    """Time per kernel class of the library's profiler over one OpenLORIS call (graphs off: eager launches)."""
    from b200ocl import _native, engine
    lib = _native.lib()
    engine.set_graphs(False)
    try:
        lrn, rs = build(kind, 'openloris')
        with contextlib.redirect_stdout(sys.stderr):
            if kind == 'gdumb':
                lrn.train_mem()
            else:
                lrn.train_learner(*task(rs, 20 * BATCH, 50, np.arange(69)))
        torch.cuda.synchronize()
        lib.b200ocl_profile_begin()
        run(lrn, rs, kind, 'openloris', steps)
        torch.cuda.synchronize()
        name, ms, cnt, work = ctypes.create_string_buffer(64), ctypes.c_double(), ctypes.c_int(), ctypes.c_double()
        split = {}
        for k in range(lib.b200ocl_profile_end()):
            lib.b200ocl_profile_get(k, name, 64, ctypes.byref(ms), ctypes.byref(cnt), ctypes.byref(work))
            split[name.value.decode()] = (ms.value, cnt.value)
    finally:
        engine.set_graphs(True)
    total = sum(v[0] for v in split.values())
    return {'profile': kind, 'card': card(), 'data': 'openloris', 'mem_size': MEM, 'kernel_ms_total': total,
            'classes': {k: {'ms': v[0], 'share': v[0] / total, 'launches': v[1]}
                        for k, v in sorted(split.items(), key=lambda kv: -kv[1][0])}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--profile-steps', type=int, default=50)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    np.random.seed(0)
    torch.manual_seed(0)
    print('card:', card(), flush=True)
    configs = [(k, d) for k in ('er', 'aser', 'scr', 'gdumb') for d in ('openloris', 'cifar100')]
    res = {c: [] for c in configs}
    for _ in range(args.repeats):                    # the configurations alternate; each run builds a fresh learner
        for c in configs:
            res[c].append(time_config(*c, args.steps))
            torch.cuda.empty_cache()
    for (kind, data), r in res.items():
        print(json.dumps({'agent': kind, 'data': data, 'mem_size': MEM, 'ms_per_step': float(np.median(r)),
                          'runs_ms_per_step': r, 'steps': args.steps if kind != 'gdumb' else MEM // BATCH}), flush=True)
    for kind in ('er', 'gdumb'):
        print(json.dumps(profile(kind, args.profile_steps)), flush=True)
    print('card:', card(), flush=True)


if __name__ == '__main__':
    main()
