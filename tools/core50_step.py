"""Time the engine's agents at CORe50 shapes (128x128 inputs, 50 classes, 2560-wide features) against the same agents at
CIFAR-100 shapes: batch 10, memories of 1000 and 5000 images (5000 at 128x128 is 983 MB of buffer), CUDA events around
a train_learner call of --steps replay steps after one warm-up call of 20 steps.  ER (random retrieval, reservoir
update), ER with ASER retrieval and update, and iCaRL; GDumb is timed over one train_mem epoch (re-initialisation
included) of its full memory.  The configurations alternate over --repeats runs and the median is reported.  Then one
ER and one GDumb run at CORe50 shapes with CUDA graphs off and the library's per-launch profiler on give the time per
kernel class, each with the card and its power limit read right after the profiled call.  Prints the card and its
power limit first, then one JSON line per result.

    python tools/core50_step.py [--steps S] [--repeats R]
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
from tricks_step import card  # noqa: E402

BATCH = 10
SHAPES = {'core50': (128, 50), 'cifar100': (32, 100)}


def learner(kind, data, mem_size):
    from b200ocl import nets, registry
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick', 'kd_trick_star')}
    agent = {'er': 'ER', 'aser': 'ER', 'icarl': 'ICARL', 'gdumb': 'GDUMB'}[kind]
    plug = 'ASER' if kind == 'aser' else 'random'
    params = SimpleNamespace(data=data, cuda=True, epoch=1, batch=BATCH, verbose=False, mem_size=mem_size,
                             eps_mem_batch=10, mem_iters=1, update=plug, retrieve=plug, agent=agent, k=3,
                             aser_type='asvm', n_smp_cls=1.5, num_tasks=10, buffer_tracker=False, optimizer='SGD',
                             learning_rate=0.1, weight_decay=0.0, temp=0.07, head='mlp', subsample=50, mem_epoch=1,
                             clip=10.0, minlr=0.0005, error_analysis=False, trick=trick)
    return registry.agents[agent](nets.setup_architecture(params), None, params)


def task(rs, n, hw, labels):
    labels = np.asarray(labels)
    return rs.randint(0, 256, (n, hw, hw, 3)).astype(np.uint8), labels[np.arange(n) % labels.size][rs.permutation(n)]


def labels(kind, ncls, timed):
    """The labels of a call.  iCaRL counts a label again in every task it recurs in (its logits must hold them all), so
    its warm-up and timed calls take 10 labels each, different ones; the other agents take every class."""
    if kind == 'icarl':
        return np.arange(10) + (10 if timed else 0)
    return np.arange(ncls)


def build(kind, data, mem_size):
    hw, ncls = SHAPES[data]
    rs = np.random.RandomState(7)
    random.seed(7)
    with contextlib.redirect_stdout(sys.stderr):
        lrn = learner(kind, data, mem_size)
    if kind == 'gdumb':
        y = np.arange(mem_size) % ncls
        lrn.before_train(None, y)
        slots, sources = lrn.memory.plan(y)
        lrn.memory.write(torch.from_numpy(rs.rand(mem_size, 3, hw, hw).astype(np.float32)).cuda(), y, slots, sources)
    else:
        lrn.buffer.update(torch.rand(mem_size, 3, hw, hw, device='cuda'), torch.randint(0, ncls, (mem_size,), device='cuda'))
    return lrn, rs


def run(lrn, rs, kind, data, steps):
    """ms per replay step of one timed call (GDumb: per train_mem step)."""
    hw, ncls = SHAPES[data]
    if kind == 'gdumb':
        fn = lrn.train_mem
        steps = len(lrn.memory) // BATCH
    else:
        x, y = task(rs, steps * BATCH, hw, labels(kind, ncls, True))
        fn = lambda: lrn.train_learner(x, y)    # noqa: E731
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    with contextlib.redirect_stdout(sys.stderr):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def time_config(kind, data, mem_size, steps):
    lrn, rs = build(kind, data, mem_size)
    hw, ncls = SHAPES[data]
    with contextlib.redirect_stdout(sys.stderr):
        if kind == 'gdumb':
            lrn.train_mem()                      # warm-up epoch: captures the graphs
        else:
            lrn.train_learner(*task(rs, 20 * BATCH, hw, labels(kind, ncls, False)))
    return run(lrn, rs, kind, data, steps)


def profile(kind, steps):
    """Time per kernel class of the library's profiler over one CORe50 call (graphs off: eager launches)."""
    from b200ocl import _native, engine
    lib = _native.lib()
    engine.set_graphs(False)
    try:
        lrn, rs = build(kind, 'core50', 5000)
        with contextlib.redirect_stdout(sys.stderr):
            if kind == 'gdumb':
                lrn.train_mem()
            else:
                lrn.train_learner(*task(rs, 20 * BATCH, 128, labels(kind, 50, False)))
        torch.cuda.synchronize()
        lib.b200ocl_profile_begin()
        run(lrn, rs, kind, 'core50', steps)
        torch.cuda.synchronize()
        name, ms, cnt, work = ctypes.create_string_buffer(64), ctypes.c_double(), ctypes.c_int(), ctypes.c_double()
        split = {}
        for k in range(lib.b200ocl_profile_end()):
            lib.b200ocl_profile_get(k, name, 64, ctypes.byref(ms), ctypes.byref(cnt), ctypes.byref(work))
            split[name.value.decode()] = (ms.value, cnt.value)
    finally:
        engine.set_graphs(True)
    total = sum(v[0] for v in split.values())
    return {'profile': kind, 'card': card(), 'data': 'core50', 'mem_size': 5000, 'kernel_ms_total': total,
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
    configs = [(k, d, m) for k in ('er', 'aser', 'icarl', 'gdumb') for m in (1000, 5000) for d in ('core50', 'cifar100')]
    res = {c: [] for c in configs}
    for _ in range(args.repeats):                    # the configurations alternate; each run builds a fresh learner
        for c in configs:
            res[c].append(time_config(*c, args.steps))
            torch.cuda.empty_cache()
    for (kind, data, mem), r in res.items():
        print(json.dumps({'agent': kind, 'data': data, 'mem_size': mem, 'ms_per_step': float(np.median(r)),
                          'runs_ms_per_step': r, 'steps': args.steps if kind != 'gdumb' else mem // BATCH}), flush=True)
    for kind in ('er', 'gdumb'):
        print(json.dumps(profile(kind, args.profile_steps)), flush=True)
    print('card:', card(), flush=True)


if __name__ == '__main__':
    main()
