"""Time one iCaRL step against one ER step (random retrieval, reservoir update) at CIFAR-100 shapes: memory 5000, stream
batch 10.  The iCaRL step is timed from its second task on, with a previous model: 10 stream + 10 memory rows through
the student and the teacher, the fused BCE criterion, one backward pass, SGD and the reservoir update.  Each step is
timed with the teacher's forward issued beside the student's on a second stream (B200OCL_CONCURRENT=1) and after it
(=0).  CUDA events around K steps after W warm-up steps; prints the card and its power limit, then one JSON line per
configuration.

    python tools/icarl_step.py [--steps K] [--warmup W] [--repeats R]
"""
import argparse
import contextlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import bench  # noqa: E402
from tricks_step import card  # noqa: E402


def learner_for(agent, seed):
    """bench.py's learner (memory filled with seeded images and labels) for ER or iCaRL with random retrieval and the
    reservoir update.  iCaRL first trains one task over labels 0..49, so that its previous model exists."""
    from b200ocl import learners
    p = bench.params_for('aser')
    p.retrieve = p.update = 'random'
    p.agent = agent
    orig = bench.params_for
    bench.params_for = lambda k: p
    try:
        lrn = bench.build_learner('er', seed)
    finally:
        bench.params_for = orig
    if agent == 'ICARL':
        rs = np.random.RandomState(seed)
        lrn.train_learner(rs.randint(0, 256, (50, 32, 32, 3)).astype(np.uint8), np.arange(50))
        lrn.before_train(None, np.arange(50, 100))       # the second task: K = 100 positions
        assert lrn._prev_live and isinstance(lrn, learners.Icarl)
    else:
        lrn.before_train(None, np.arange(bench.NUM_CLASSES))
    return lrn


def time_config(agent, concurrent, steps, warmup):
    from b200ocl import learners
    learners.set_concurrent(concurrent)
    with contextlib.redirect_stdout(sys.stderr):
        lrn = learner_for(agent, 7)
    rs = np.random.RandomState(3)
    lo = 50 if agent == 'ICARL' else 0
    batches = []
    for _ in range(8):
        x = torch.rand(bench.BATCH, 3, 32, 32, device='cuda')
        y = rs.randint(lo, bench.NUM_CLASSES, bench.BATCH).astype(np.int64)
        batches.append((x, torch.from_numpy(y).cuda(), y))
    for i in range(warmup):
        lrn.replay_step(*batches[i % len(batches)])
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(steps):
        lrn.replay_step(*batches[i % len(batches)])
    b.record()
    torch.cuda.synchronize()
    learners.set_concurrent(True)
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    np.random.seed(0)
    torch.manual_seed(0)
    print('card:', card())
    configs = [(agent, conc) for agent in ('ER', 'ICARL') for conc in (True, False)]
    ms = {c: [] for c in configs}
    for _ in range(args.repeats):                # the configurations alternate; each run builds a fresh learner
        for agent, conc in configs:
            ms[(agent, conc)].append(time_config(agent, conc, args.steps, args.warmup))
    for (agent, conc), t in ms.items():
        print(json.dumps({'agent': agent, 'concurrent': int(conc), 'ms_per_step': t, 'median_ms': float(np.median(t)),
                          'steps': args.steps, 'warmup': args.warmup}), flush=True)


if __name__ == '__main__':
    main()
