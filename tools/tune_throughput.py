#!/usr/bin/env python
"""Wall time of one tuning stage of main_tune.py's loop (multirun.multiple_run_tune_separate's stage 1) with R
trainings side by side on one GPU, R = 1, 2, 4, 8.

Synthetic CIFAR-100-shaped tasks: two tasks of --images uint8 images (500 per class, as in CIFAR-100), evaluated
after each task on one test loader per task of 100 images per class in batches of 128: --images 5000 is CIFAR-100 cut
into 10 tasks, --images 2500 into 20 (config/data/cifar100/cifar100_nc.yml of the reference).  An 8-point
grid (learning_rate 0.01, 0.03, 0.1, 0.3 x weight_decay 0, 1e-4), num_runs_val = 3: 24 trainings, each a fresh agent
seeded with multirun.tune_seed and run through multirun.run_group in groups of R, as the wrapper runs them.  Memory
1000 slots, batch 10 stream + 10 memory images.  Cases: ER with random retrieval / reservoir update, ER + ASER (asvm,
k=3, n_smp_cls 1.5) and SCR (mlp head, T=0.07).  Each case first runs two trainings that are not timed (module loading,
first allocations); then the R values alternate within every repetition, and the table gives the median over --reps
repetitions.

Columns per (case, R):
  s/training   stage wall time over the 24 trainings, s
  vs R=1       speedup of the stage over R = 1
  host/step    host time spent issuing one replay step, ms: the steps' host time minus the time the learners'
               throttles and the deferred ASER decisions wait on the device (as tools/multirun_throughput.py)
  dev/step     mean time from a step's first to its last device work on its own stream (CUDA events), ms
  setup        share of a training's wall time before its first step: its group's wall time from the first agent's
               construction to the first replay step, over the group's wall time
  eval         share of the stage's wall time spent in evaluate()

    python tools/tune_throughput.py [--images 5000] [--reps 3] [--rs 1,2,4,8] [--out results/tune.json]
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

MEM, BATCH, PER_CLASS, TEST_PER_CLASS = 1000, 10, 500, 100
GRID = {'learning_rate': [0.01, 0.03, 0.1, 0.3], 'weight_decay': [0.0, 1e-4]}
N_VAL_RUNS = 3
CASES = {
    'er_random': dict(agent='ER', retrieve='random', update='random'),
    'er_aser': dict(agent='ER', retrieve='ASER', update='ASER'),
    'scr': dict(agent='SCR', retrieve='random', update='random'),
}


def params_for(case):
    base = dict(data='cifar100', cuda=True, epoch=1, batch=BATCH, verbose=False, mem_size=MEM, mem_iters=1,
                eps_mem_batch=BATCH, k=3, aser_type='asvm', n_smp_cls=1.5, num_tasks=10, buffer_tracker=False,
                optimizer='SGD', learning_rate=0.1, weight_decay=0, temp=0.07, head='mlp', subsample=50,
                error_analysis=False, test_batch=128,
                trick={k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick',
                                          'ncm_trick', 'kd_trick_star')})
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
    ap.add_argument('--images', type=int, default=5000, help='stream images per task')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--rs', default='1,2,4,8')
    ap.add_argument('--cases', default=','.join(CASES))
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this tool measures the GPU and has no CPU fallback')
    from b200ocl import learners, memory, multirun, nets, registry

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

    def stage_data(seed):
        """One run's two tuning tasks and their test loaders (the tune data every training of the stage shares)."""
        rs = np.random.RandomState(seed)
        n_cls = max(1, a.images // PER_CLASS)
        n_test = n_cls * TEST_PER_CLASS
        tasks, loaders = [], []
        for t in range(2):
            labels = np.arange(n_cls * t, n_cls * (t + 1))
            tasks.append((rs.randint(0, 256, (a.images, 32, 32, 3)).astype(np.uint8),
                          labels[rs.randint(0, n_cls, a.images)]))
            x = torch.from_numpy(rs.rand(n_test, 3, 32, 32).astype(np.float32))
            y = torch.from_numpy(labels[np.arange(n_test) % n_cls])
            loaders.append([(x[i:i + 128], y[i:i + 128]) for i in range(0, n_test, 128)])
        return tasks, loaders

    def measure(case, R, seed, n_trainings=None):
        grid = multirun.param_grid(GRID)
        entries = [(g, v) for g in range(len(grid)) for v in range(N_VAL_RUNS)][:n_trainings]
        tasks, loaders = stage_data(seed)
        st = {'host': 0.0, 'spans': [], 'eval': 0.0, 'setup': [], 'group_t0': None, 'first_step': None}

        def make(i):
            params = params_for(case)
            vars(params).update(grid[entries[i][0]])
            model = nets.setup_architecture(params)
            opt = torch.optim.SGD(model.parameters(), lr=params.learning_rate, weight_decay=params.weight_decay)
            agent = registry.agents[params.agent](model, opt, params)
            inner = agent.evaluate

            def evaluate(ls):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = inner(ls)
                torch.cuda.synchronize()
                st['eval'] += time.perf_counter() - t0
                return out
            agent.evaluate = evaluate
            return agent

        def before_run(i):
            if i % R == 0:                                   # the group's first training
                torch.cuda.synchronize()
                st['group_t0'], st['first_step'] = time.perf_counter(), None

        def on_run_end(i, acc):
            if i % R == R - 1 or i == len(entries) - 1:      # the group's last training
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                st['setup'].append((st['first_step'] - st['group_t0']) / (t1 - st['group_t0']))

        orig_next = multirun._next_step

        def next_step(steps):
            if st['first_step'] is None:
                torch.cuda.synchronize()
                st['first_step'] = time.perf_counter()
            e0 = torch.cuda.Event(enable_timing=True)
            e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
            h0 = time.perf_counter()
            ok = orig_next(steps)
            st['host'] += time.perf_counter() - h0
            e1.record()
            if ok:
                st['spans'].append((e0, e1))
            return ok
        multirun._next_step = next_step
        torch.cuda.synchronize()
        b0, t0 = blocked[0], time.perf_counter()
        try:
            multirun.run_group([tasks] * len(entries), [loaders] * len(entries), make, R,
                               seeds=[multirun.tune_seed(seed, 0, g, v) for g, v in entries],
                               before_run=before_run, on_run_end=on_run_end)
        finally:
            multirun._next_step = orig_next
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        n_steps = len(st['spans'])
        host = st['host'] - (blocked[0] - b0)
        dev = statistics.mean(e0.elapsed_time(e1) for e0, e1 in st['spans'])
        torch.cuda.empty_cache()
        return {'s_training': wall / len(entries), 'wall_s': wall, 'host_ms_step': 1e3 * host / n_steps,
                'dev_ms_step': dev, 'setup_share': statistics.mean(st['setup']), 'eval_share': st['eval'] / wall,
                'steps': n_steps}

    rvals = [int(r) for r in a.rs.split(',')]
    info = gpu_info()
    print('GPU:', info, flush=True)
    results = {}
    for case in a.cases.split(','):
        measure(case, 2, seed=1, n_trainings=2)              # not timed: module loading, first allocations
    for rep in range(a.reps):
        for case in a.cases.split(','):
            for R in rvals:                                  # alternate the R values within every repetition
                m = measure(case, R, seed=100 * rep + 7)
                results.setdefault(case, {}).setdefault(R, []).append(m)
                print(case, 'R=%d rep %d' % (R, rep), json.dumps({k: round(v, 4) for k, v in m.items()}), flush=True)
    table = {}
    print('\n| case | R | s / training | vs R = 1 | host ms / step | device ms / step | before first step | eval |')
    print('|---|---|---|---|---|---|---|---|')
    for case, byr in results.items():
        base = statistics.median(m['s_training'] for m in byr[rvals[0]])
        for R in rvals:
            med = {k: statistics.median(m[k] for m in byr[R]) for k in byr[R][0]}
            table.setdefault(case, {})[R] = med
            print('| %s | %d | %.3f | x%.2f | %.2f | %.2f | %.1f %% | %.1f %% |'
                  % (case, R, med['s_training'], base / med['s_training'], med['host_ms_step'], med['dev_ms_step'],
                     100 * med['setup_share'], 100 * med['eval_share']))
    print('GPU:', gpu_info())
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump({'gpu': info, 'images': a.images, 'reps': a.reps, 'median': table, 'all': results}, f,
                      indent=1)


if __name__ == '__main__':
    main()
