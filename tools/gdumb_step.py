"""Time GDumb's train_mem at CIFAR-100 shapes (batch 10) over a full memory of 1000 and of 5000 images: CUDA events
around train_mem() running --epochs epochs (re-initialisation included), after one warm-up call of one epoch.  Each
memory size is timed with the clipped SGD step train_mem uses (b200ocl_net_sgd_step_clipped) and with the plain step
(b200ocl_net_sgd_step) in its place; the configurations alternate over --repeats runs and the median is reported.
Prints the card and its power limit, then one JSON line per configuration: ms per step and per epoch, and kernel
launches per step (the library's counter plus the launches replayed inside CUDA graphs).

    python tools/gdumb_step.py [--epochs E] [--repeats R]
"""
import argparse
import contextlib
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

BATCH, NUM_CLASSES = 10, 100


def learner(mem_size, seed):
    """A GDumb learner whose memory holds mem_size seeded images over the 100 classes, balanced by its own planner."""
    from b200ocl import nets, registry
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick', 'kd_trick_star')}
    params = SimpleNamespace(data='cifar100', cuda=True, epoch=1, batch=BATCH, verbose=False, mem_size=mem_size,
                             eps_mem_batch=10, mem_iters=1, update='random', retrieve='random', agent='GDUMB',
                             optimizer='SGD', learning_rate=0.1, weight_decay=0.0, mem_epoch=1, clip=10.0, minlr=0.0005,
                             error_analysis=False, trick=trick)
    lrn = registry.agents['GDUMB'](nets.setup_architecture(params), None, params)
    rs = np.random.RandomState(seed)
    random.seed(seed)
    y = np.arange(mem_size) % NUM_CLASSES
    lrn.before_train(None, y)
    x = torch.from_numpy(rs.rand(mem_size, 3, 32, 32).astype(np.float32)).cuda()
    slots, sources = lrn.memory.plan(y)
    lrn.memory.write(x, y, slots, sources)
    assert len(lrn.memory) == mem_size
    return lrn


def time_config(mem_size, clipped, epochs):
    from b200ocl import _native
    from b200ocl.engine import graph_launch_count
    with contextlib.redirect_stdout(sys.stderr):
        lrn = learner(mem_size, 7)
    eng = lrn.engine
    if not clipped:
        eng.sgd_step_clipped = lambda lr, wd, max_norm: eng.sgd_step(lr, wd)
    lrn.train_mem()                                  # warm-up epoch: captures the graphs of the forward and backward
    lrn.params.mem_epoch = epochs
    torch.cuda.synchronize()
    launches = _native.launch_count() + graph_launch_count()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    lrn.train_mem()
    b.record()
    torch.cuda.synchronize()
    steps = epochs * (mem_size // BATCH)
    ms = a.elapsed_time(b)
    return ms / steps, ms / epochs, (_native.launch_count() + graph_launch_count() - launches) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--epochs', type=int, default=3)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    np.random.seed(0)
    torch.manual_seed(0)
    print('card:', card())
    configs = [(mem, clipped) for mem in (1000, 5000) for clipped in (True, False)]
    res = {c: [] for c in configs}
    for _ in range(args.repeats):                    # the configurations alternate; each run builds a fresh learner
        for mem, clipped in configs:
            res[(mem, clipped)].append(time_config(mem, clipped, args.epochs))
    for (mem, clipped), r in res.items():
        step, epoch, launches = (float(np.median([t[i] for t in r])) for i in range(3))
        print(json.dumps({'mem_size': mem, 'step': 'clipped' if clipped else 'plain', 'ms_per_step': step,
                          'ms_per_epoch': epoch, 'launches_per_step': launches, 'runs_ms_per_step': [t[0] for t in r],
                          'epochs': args.epochs}), flush=True)


if __name__ == '__main__':
    main()
