#!/usr/bin/env python
"""Stream images/s of R replay runs side by side on one GPU (multirun.run_group), R = 1, 2, 4, 8.

CIFAR-100 shapes, synthetic uint8 stream images, memory 5000 slots pre-filled (so ASER's kNN-SV retrieval and update
are active from the first step), batch 10 stream + 10 memory images.  Cases: ER + ASER (asvm, k=3, n_smp_cls 1.5),
SCR (mlp head, T=0.07) and ER with random retrieval / reservoir update.  Each R builds R fresh agents, warms them up
(every captured graph is recorded), then times STEPS rounds (one replay step of every run).  The R values are measured
in alternation, REPS times; the table gives the median.

Columns per (case, R):
  img/s      stream images per second over all runs (R x 10 x rounds / wall)
  wall/rnd   wall time of one round (one step of each of the R runs), ms
  host/rnd   host time spent issuing one round, ms: the steps' host time minus the time the learners' throttles and
             the deferred ASER decisions wait on the device.  host/rnd close to wall/rnd: the host is the bound.
  dev/step   mean time from a step's first to its last device work on its own stream (CUDA events), ms.  With the
             queue ahead of the device this is the step's device time, stretched by what shares the GPU with it.

    python tools/multirun_throughput.py [--steps 200] [--warmup 30] [--reps 3] [--out results/multirun.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MEM, BATCH, NCLS = 5000, 10, 100
CASES = {
    'er_aser': dict(agent='ER', retrieve='ASER', update='ASER'),
    'scr': dict(agent='SCR', retrieve='random', update='random'),
    'er_random': dict(agent='ER', retrieve='random', update='random'),
}


def params_for(case):
    base = dict(data='cifar100', cuda=True, epoch=1, batch=BATCH, verbose=False, mem_size=MEM, mem_iters=1,
                eps_mem_batch=BATCH, k=3, aser_type='asvm', n_smp_cls=1.5, num_tasks=10, buffer_tracker=False,
                optimizer='SGD', learning_rate=0.1, weight_decay=0, temp=0.07, head='mlp', subsample=50,
                error_analysis=False, trick={k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax',
                                                                'review_trick', 'ncm_trick', 'kd_trick_star')})
    base.update(CASES[case])
    return SimpleNamespace(**base)


def gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm,'
                            'driver_version', '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return 'nvidia-smi unavailable (%s)' % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--rs', default='1,2,4,8')
    ap.add_argument('--cases', default=','.join(CASES))
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this tool measures the GPU and has no CPU fallback')
    from b200ocl import learners, memory, multirun, nets, registry
    CB = memory.ClassBalancedRandomSampling

    # host time blocked on the device: the throttles and the deferred ASER decisions
    blocked = [0.0]
    throttle = learners.ContinualLearner._throttle
    flush = memory.flush_pending

    def timed(fn):
        def wrap(*args, **kw):
            t0 = time.perf_counter()
            try:
                return fn(*args, **kw)
            finally:
                blocked[0] += time.perf_counter() - t0
        return wrap
    learners.ContinualLearner._throttle = timed(throttle)
    memory.flush_pending = timed(flush)

    def make_agent_for(case, seed):
        params = params_for(case)

        def make(r):
            learner = registry.agents[params.agent](nets.setup_architecture(params), None, params)
            rs = np.random.RandomState(seed + r)
            buf = learner.buffer
            buf.buffer_img.copy_(torch.from_numpy(rs.rand(MEM, 3, 32, 32).astype(np.float32)).cuda())
            labels = rs.randint(0, NCLS, MEM).astype(np.int64)
            buf.buffer_label.copy_(torch.from_numpy(labels).cuda())
            buf.labels_host[:] = labels
            buf.current_index, buf.n_seen_so_far = MEM, MEM + BATCH
            if params.update == 'ASER':
                CB.reset()
                CB.update_cache(buf.buffer_label, NCLS, new_y=labels, ind=np.arange(MEM))
            return learner
        return make

    def measure(case, R, seed):
        n_steps = a.warmup + a.steps
        rs = np.random.RandomState(seed)
        tasks = [[(rs.randint(0, 256, (n_steps * BATCH, 32, 32, 3)).astype(np.uint8),
                   rs.randint(0, NCLS, n_steps * BATCH).astype(np.int64))] for _ in range(R)]
        make = make_agent_for(case, seed)
        stamps = {'t0': None, 'host': 0.0, 'blocked0': 0.0, 'spans': []}

        class Timed(object):
            """An agent whose evaluation is skipped: only its replay steps are measured."""

            def __init__(self, agent):
                self.agent = agent

            def _steps(self, x, y):
                for _ in self.agent._steps(x, y):
                    yield

            def evaluate(self, loaders):
                return np.zeros(0)

        agents = []

        def make_timed(r):
            ag = make(r)
            agents.append(ag)
            return Timed(ag)

        # one step of each run per round: drive run_group's round robin, timing from the first timed round
        orig_next = multirun._next_step
        state = {'calls': 0}

        def next_step(steps):
            k = state['calls']
            state['calls'] += 1
            rnd = k // R
            if rnd == a.warmup and k % R == 0:
                torch.cuda.synchronize()
                stamps['t0'] = time.perf_counter()
                stamps['blocked0'] = blocked[0]
            timing = a.warmup <= rnd < n_steps
            if timing:
                e0 = torch.cuda.Event(enable_timing=True)
                e1 = torch.cuda.Event(enable_timing=True)
                e0.record()
                h0 = time.perf_counter()
            ok = orig_next(steps)
            if timing:
                stamps['host'] += time.perf_counter() - h0
                e1.record()
                stamps['spans'].append((e0, e1))
            if rnd == n_steps - 1 and k % R == R - 1:
                torch.cuda.synchronize()
                stamps['t1'] = time.perf_counter()
                stamps['blocked1'] = blocked[0]
            return ok
        multirun._next_step = next_step
        try:
            multirun.run_group(tasks, [[]] * R, make_timed, R, seed=seed)
        finally:
            multirun._next_step = orig_next
        torch.cuda.synchronize()
        wall = stamps['t1'] - stamps['t0']
        host = stamps['host'] - (stamps['blocked1'] - stamps['blocked0'])
        dev = statistics.mean(e0.elapsed_time(e1) for e0, e1 in stamps['spans'])
        del agents[:]
        torch.cuda.empty_cache()
        return {'img_s': R * BATCH * a.steps / wall, 'wall_ms_round': 1e3 * wall / a.steps,
                'host_ms_round': 1e3 * host / a.steps, 'dev_ms_step': dev}

    rvals = [int(r) for r in a.rs.split(',')]
    info = gpu_info()
    print('GPU:', info, flush=True)
    results = {}
    for case in a.cases.split(','):
        for rep in range(a.reps):
            for R in rvals:                                  # alternate the R values within every repetition
                m = measure(case, R, seed=100 * rep + 7)
                results.setdefault(case, {}).setdefault(R, []).append(m)
                print(case, 'R=%d rep %d' % (R, rep), json.dumps({k: round(v, 3) for k, v in m.items()}), flush=True)
    table = {}
    print('\n| case | R | stream img/s | vs R=1 | wall ms/round | host ms/round | device ms/step |')
    print('|---|---|---|---|---|---|---|')
    for case, byr in results.items():
        base = statistics.median(m['img_s'] for m in byr[rvals[0]])
        for R in rvals:
            med = {k: statistics.median(m[k] for m in byr[R]) for k in byr[R][0]}
            table.setdefault(case, {})[R] = med
            print('| %s | %d | %.0f | x%.2f | %.2f | %.2f | %.2f |' % (case, R, med['img_s'], med['img_s'] / base,
                                                                       med['wall_ms_round'], med['host_ms_round'],
                                                                       med['dev_ms_step']))
    print('GPU:', gpu_info())
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump({'gpu': info, 'steps': a.steps, 'warmup': a.warmup, 'reps': a.reps, 'median': table,
                       'all': results}, f, indent=1)


if __name__ == '__main__':
    main()
