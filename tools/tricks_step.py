"""Time one replay step at CIFAR-100 shapes (memory 5000, batch 10, 10 retrieved) with the training tricks:
ER, ER + labels_trick, ER + separated_softmax, ER + kd_trick with a live teacher, ER + ASER + kd_trick_star, and LwF
with a live teacher.  CUDA events around K steps after W warm-up steps; prints the card and its power limit, then one
JSON line per configuration.

    python tools/tricks_step.py [--steps K] [--warmup W]
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

CONFIGS = [  # name, bench kind, agent override, trick flags
    ('er', 'er', None, {}),
    ('er+labels_trick', 'er', None, {'labels_trick': True}),
    ('er+separated_softmax', 'er', None, {'separated_softmax': True}),
    ('er+kd_trick', 'er', None, {'kd_trick': True}),
    ('er+aser+kd_trick_star', 'aser', None, {'kd_trick_star': True}),
    ('lwf', 'er', 'LWF', {}),
]


def card():
    try:
        r = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def learner_for(kind, agent, trick, seed):
    """bench.py's learner (memory filled with seeded images and labels) for ER with random retrieval / reservoir
    update, or ER with the ASER plugins; LwF has no memory."""
    from b200ocl import nets, registry
    p = bench.params_for('aser')
    if kind == 'er':
        p.retrieve = p.update = 'random'
    p.agent = agent or 'ER'
    p.trick = dict(p.trick, **trick)
    if agent == 'LWF':
        lrn = registry.agents[agent](nets.setup_architecture(p), None, p)
        lrn.model.train()
        return lrn
    orig = bench.params_for
    bench.params_for = lambda k: p
    try:
        return bench.build_learner(kind, seed)
    finally:
        bench.params_for = orig


def time_config(name, kind, agent, trick, steps, warmup):
    with contextlib.redirect_stdout(sys.stderr):
        lrn = learner_for(kind, agent, trick, 7)
    rs = np.random.RandomState(3)
    y_task = np.arange(bench.NUM_CLASSES)
    lrn.before_train(None, y_task)           # the label tables of one task over every class
    if trick.get('kd_trick') or agent == 'LWF':
        lrn.after_train()                    # a teacher is live from the second task on
        lrn.before_train(None, y_task)
    batches = []
    for _ in range(8):
        x = torch.rand(bench.BATCH, 3, 32, 32, device='cuda')
        y = rs.randint(0, bench.NUM_CLASSES, bench.BATCH).astype(np.int64)
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
    return {'config': name, 'ms_per_step': a.elapsed_time(b) / steps, 'steps': steps, 'warmup': warmup,
            'teacher_live': bool(getattr(lrn, '_teacher_live', False))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--only', default='')
    args = ap.parse_args()
    torch.cuda.set_device(0)
    np.random.seed(0)
    torch.manual_seed(0)
    print('card:', card())
    for name, kind, agent, trick in CONFIGS:
        if args.only and name not in args.only.split(','):
            continue
        print(json.dumps(time_config(name, kind, agent, trick, args.steps, args.warmup)), flush=True)


if __name__ == '__main__':
    main()
