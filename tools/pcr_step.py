"""Time PCR at CIFAR-100 shapes: memory 5000 prefilled, batch 10, eps_mem_batch 10.  CUDA events around a
train_learner call of --steps batches, after a warm-up call that captures the graphs, for three agents that alternate
over --repeats runs: PCR (pcr_temp 0.09), SCR (temp 0.07, mlp head) and ER, each with random retrieval and the reservoir
update.  The median is reported, with kernel launches per step (the library's counter plus the launches replayed inside
CUDA graphs).  Prints the card and its power limit first.

    python tools/pcr_step.py [--steps S] [--repeats R]
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

BATCH, MEM, NUM_CLASSES = 10, 5000, 100
CONFIGS = ('PCR', 'SCR', 'ER')


def learner(name):
    from b200ocl import nets, registry
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick', 'kd_trick_star')}
    params = SimpleNamespace(data='cifar100', cuda=True, epoch=1, batch=BATCH, verbose=False, mem_size=MEM,
                             eps_mem_batch=10, mem_iters=1, update='random', retrieve='random', agent=name,
                             optimizer='SGD', learning_rate=0.1, weight_decay=0.0, error_analysis=False,
                             pcr_temp=0.09, temp=0.07, head='mlp', buffer_tracker=False, trick=trick)
    cls = registry.agents.get(name) or registry.extra_agents[name]
    return cls(nets.setup_architecture(params), None, params)


def task(rs, n):
    return rs.randint(0, 256, (n, 32, 32, 3)).astype(np.uint8), (np.arange(n) % NUM_CLASSES)[rs.permutation(n)]


def time_config(name, steps):
    from b200ocl import _native
    from b200ocl.engine import graph_launch_count
    rs = np.random.RandomState(7)
    with contextlib.redirect_stdout(sys.stderr):
        lrn = learner(name)
        lrn.train_learner(*task(rs, MEM))              # warm-up call: fills the memory and captures the graphs
    x, y = task(rs, steps * BATCH)
    torch.cuda.synchronize()
    assert lrn.buffer.current_index == MEM
    launches = _native.launch_count() + graph_launch_count()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    lrn.train_learner(x, y)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps, (_native.launch_count() + graph_launch_count() - launches) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    np.random.seed(0)
    torch.manual_seed(0)
    print('card:', card())
    res = {k: [] for k in CONFIGS}
    for _ in range(args.repeats):                    # the configurations alternate; each run builds a fresh learner
        for name in CONFIGS:
            res[name].append(time_config(name, args.steps))
    for name, r in res.items():
        print(json.dumps({'agent': name, 'ms_per_step': float(np.median([t[0] for t in r])),
                          'launches_per_step': float(np.median([t[1] for t in r])),
                          'runs_ms_per_step': [t[0] for t in r], 'steps': args.steps}), flush=True)


if __name__ == '__main__':
    main()
