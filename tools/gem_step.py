"""Time GEM at CIFAR-100 shapes: num_tasks 20 and mem_size 5000 (M = 250 rows per task), batch 10, gem_margin 0.5.

For t = 0, 1, 4, 9 and 19 earlier tasks (their rings prefilled with random rows), CUDA events around a train_learner
call of --steps batches after a warm-up call that captures the graphs; each step is split by device events into the
memory passes (the t forward / backward passes over the earlier rings and the copies into G) and the Gram + QP +
projection launches (ops.gem_project).  A-GEM and ER (random retrieval, reservoir update, memory 5000 prefilled,
eps_mem_batch 10) are timed in the same call; all configurations alternate over --repeats runs and the median is
reported.  Then the Gram kernel alone (torch.profiler, CUDA activities, 50 calls) at each t with its achieved HBM
bandwidth from the (t + 1) n 4 bytes it must read.  Prints the card and its power limit first.

    python tools/gem_step.py [--steps S] [--repeats R]
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

BATCH, MEM, NUM_TASKS, NUM_CLASSES = 10, 5000, 20, 100
PAST = (0, 1, 4, 9, 19)


def learner(name):
    from b200ocl import nets, registry
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick', 'kd_trick_star')}
    params = SimpleNamespace(data='cifar100', cuda=True, epoch=1, batch=BATCH, verbose=False, mem_size=MEM,
                             eps_mem_batch=10, mem_iters=1, update='random', retrieve='random', agent=name,
                             optimizer='SGD', learning_rate=0.1, weight_decay=0.0, error_analysis=False,
                             num_tasks=NUM_TASKS, gem_margin=0.5, buffer_tracker=False, trick=trick)
    cls = registry.agents.get(name) or registry.extra_agents[name]
    return cls(nets.setup_architecture(params), None, params)


def task(rs, n):
    return rs.randint(0, 256, (n, 32, 32, 3)).astype(np.uint8), (np.arange(n) % NUM_CLASSES)[rs.permutation(n)]


def _timed_call(lrn, x, y, steps):
    from b200ocl import _native
    from b200ocl.engine import graph_launch_count
    torch.cuda.synchronize()
    launches = _native.launch_count() + graph_launch_count()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    lrn.train_learner(x, y)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps, (_native.launch_count() + graph_launch_count() - launches) / steps


def time_gem(t, steps):
    """(ms per step, launches per step, ms of memory passes per step, ms of gem_project per step)."""
    from b200ocl import learners, ops
    rs = np.random.RandomState(7)
    with contextlib.redirect_stdout(sys.stderr):
        lrn = learner('GEM')
    mem = lrn.rings
    for k in range(t):                                  # t earlier tasks, each ring full
        mem.begin_task(k)
        x = torch.from_numpy(rs.randint(0, 256, (mem.M, 3, 32, 32)).astype(np.float32) / 255).cuda()
        y = torch.from_numpy(rs.randint(0, NUM_CLASSES, mem.M)).cuda()
        mem.write(k, x, y, y.cpu().numpy())
    lrn.task_seen = t
    lrn.train_learner(*task(rs, 20 * BATCH))             # warm-up call: captures the graphs
    lrn.task_seen = t
    marks = []
    eng = lrn.engine
    fwd = eng.forward_train

    def forward_train(x, *a, slot=0, **k):
        if slot == lrn.MEM_SLOT and (not marks or marks[-1][0] != 'mem'):
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            marks.append(('mem', ev))
        elif slot == 0:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            marks.append(('stream', ev))
        return fwd(x, *a, slot=slot, **k)
    proj = ops.gem_project
    spans = []

    def gem_project(*a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = proj(*a, **k)
        e1.record()
        spans.append((e0, e1))
        return out
    eng.forward_train = forward_train
    learners.ops.gem_project = gem_project
    try:
        ms, launches = _timed_call(lrn, *task(rs, steps * BATCH), steps)
    finally:
        eng.forward_train = fwd
        learners.ops.gem_project = proj
    mem_ms = sum(a.elapsed_time(b) for (ka, a), (kb, b) in zip(marks, marks[1:]) if ka == 'mem' and kb == 'stream')
    proj_ms = sum(a.elapsed_time(b) for a, b in spans)
    return ms, launches, mem_ms / steps, proj_ms / steps


def time_baseline(name, steps):
    rs = np.random.RandomState(7)
    with contextlib.redirect_stdout(sys.stderr):
        lrn = learner(name)
        lrn.train_learner(*task(rs, MEM))              # warm-up call: fills the memory and captures the graphs
    assert lrn.buffer.current_index == MEM
    lrn.task_seen = 1                                  # A-GEM projects from the second task on
    ms, launches = _timed_call(lrn, *task(rs, steps * BATCH), steps)
    return ms, launches, 0.0, 0.0


def gram_bandwidth(t, n, calls=50):
    """(µs per Gram kernel, GB/s) from torch.profiler's CUDA activity of gem_gram_kernel."""
    from b200ocl import ops
    from torch.profiler import ProfilerActivity, profile
    rs = np.random.RandomState(t)
    G = torch.from_numpy(rs.standard_normal((t, n)).astype(np.float32)).cuda()
    g = torch.from_numpy(rs.standard_normal(n).astype(np.float32)).cuda()
    out = torch.empty_like(g)
    for _ in range(3):
        ops.gem_project(G, t, g, out=out)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            ops.gem_project(G, t, g, out=out)
        torch.cuda.synchronize()
    us = [e.device_time for e in prof.events() if 'gem_gram_kernel' in e.name]
    us = float(np.median(us))
    return us, (t + 1) * n * 4 / (us * 1e-6) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    np.random.seed(0)
    torch.manual_seed(0)
    print('card:', card())
    configs = [('GEM', t) for t in PAST] + [('AGEM', None), ('ER', None)]
    res = {c: [] for c in configs}
    for _ in range(args.repeats):                    # the configurations alternate; each run builds a fresh learner
        for c in configs:
            res[c].append(time_gem(c[1], args.steps) if c[0] == 'GEM' else time_baseline(c[0], args.steps))
    for (name, t), r in res.items():
        print(json.dumps({'agent': name, 'past_tasks': t, 'ms_per_step': float(np.median([x[0] for x in r])),
                          'memory_passes_ms': float(np.median([x[2] for x in r])),
                          'gem_project_ms': float(np.median([x[3] for x in r])),
                          'launches_per_step': float(np.median([x[1] for x in r])),
                          'runs_ms_per_step': [x[0] for x in r], 'steps': args.steps}), flush=True)
    from b200ocl import engine
    n = engine.describe(32, NUM_CLASSES)[1].n_params
    for t in PAST[1:] + (64,):
        us, gbs = gram_bandwidth(t, n)
        print(json.dumps({'gram_kernel': True, 't': t, 'n': n, 'us': us, 'GB_per_s': gbs}), flush=True)


if __name__ == '__main__':
    main()
