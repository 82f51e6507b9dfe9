#!/usr/bin/env python
"""Wall time of one experiment (multirun.multiple_run, general_main.py's repetitions) of --runs CIFAR-100-shaped runs:
in process at R = 1 and R = 4 (B200OCL_CONCURRENT_RUNS), and on worker processes (B200OCL_RUN_DEVICES) 0, 0,0 and
0,0,0,0 at R = 1 per worker; and 0,1,...,n-1 when this machine has n > 1 devices.

Synthetic uint8 tasks behind a stub reference tree written to a temporary directory: --tasks tasks of --images images
of 5 classes each (500 per class, as CIFAR-100 cut into 20 tasks), each evaluated after every task on one test loader
per task of 500 images in batches of 128.  Memory 1000 slots, batch 10 stream + 10 memory images.  Cases: ER with
random retrieval / reservoir update, ER + ASER (asvm, k=3, n_smp_cls 1.5) and SCR (mlp head, T=0.07).  Every
configuration's wall time includes starting its workers (each imports torch and loads the engine) and building their
data.  One untimed in-process run loads the modules first; then the configurations alternate within each of --reps
repetitions, and the table gives the medians.  The card's name and power limit are read in the same call.

--startup splits a worker's fixed cost first: a fresh interpreter importing torch; one that also creates its CUDA
context; one that also imports the engine and loads libb200ocl.so; and a tiny experiment (one run, one task of 20
images) on worker 0 minus the same in process, which adds the spawn, the worker's setup and its first agent's
allocations and graph recordings.  --configs picks configurations by name (comma-separated: inproc, inproc4, 0, 00,
0000, all).  The stub reference lives in a temporary directory that is removed at the end.

    python tools/multidevice_throughput.py [--runs 8] [--tasks 3] [--images 2500] [--reps 2] [--startup]
                                           [--configs inproc,inproc4,0,00,0000,all] [--out results/md.json]
"""
import argparse
import contextlib
import io
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import textwrap
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = {
    'er_random': dict(agent='ER', retrieve='random', update='random'),
    'er_aser': dict(agent='ER', retrieve='ASER', update='ASER'),
    'scr': dict(agent='SCR', retrieve='random', update='random'),
}

# the stub reference: synthetic CIFAR-100-shaped runs, drawn from the run's random state like the reference's new_run
TREE = {
    'continuum/__init__.py': '',
    'continuum/continuum.py': '''
        import numpy as np
        import torch


        class DataObject(object):
            def __init__(self, params):
                self.task_nums = params.num_tasks


        class continuum(object):
            def __init__(self, data, scenario, params):
                self.params, self.data_object = params, DataObject(params)
                self.cur_run, self.cur_task = -1, 0

            def new_run(self):
                self.cur_run += 1
                self.cur_task = 0
                self.order = np.random.permutation(100)

            def __iter__(self):
                return self

            def __next__(self):
                p = self.params
                if self.cur_task == p.num_tasks:
                    raise StopIteration
                labels = self.order[5 * self.cur_task:5 * (self.cur_task + 1)]
                x = np.random.randint(0, 256, (p.images, 32, 32, 3)).astype(np.uint8)
                y = labels[np.random.randint(0, 5, p.images)]
                self.cur_task += 1
                return x, y, set(labels.tolist())

            def test_data(self):
                out = []
                for t in range(self.params.num_tasks):
                    labels = self.order[5 * t:5 * (t + 1)]
                    x = torch.from_numpy(np.random.rand(500, 3, 32, 32).astype(np.float32))
                    y = torch.from_numpy(labels[np.arange(500) % 5])
                    out.append([(x[i:i + 128], y[i:i + 128]) for i in range(0, 500, 128)])
                return out
    ''',
    'continuum/data_utils.py': '''
        def setup_test_loader(data, params):
            return list(data)
    ''',
    'experiment/__init__.py': '',
    'experiment/run.py': '''
        multiple_run = multiple_run_tune_separate = None
    ''',
    'experiment/metrics.py': '''
        def compute_performance(a):
            end = a[:, -1, :].mean(axis=1)
            return (end.mean(), 0.0), (0.0, 0.0), (0.0, 0.0), (0.0, 0.0), (0.0, 0.0)
    ''',
    'utils/__init__.py': '',
    'utils/io.py': '''
        def load_yaml(path, key=None):
            return {'result': 'result/'}
    ''',
    'utils/setup_elements.py': '''
        import torch
        from b200ocl.nets import setup_architecture


        def setup_opt(optimizer, model, lr, wd):
            return torch.optim.SGD(model.parameters(), lr=lr, weight_decay=wd)
    ''',
    'utils/utils.py': '''
        def maybe_cuda(model, cuda):
            return model
    ''',
    'utils/name_match.py': '''
        from b200ocl import registry

        agents = dict(registry.agents)
        retrieve_methods = {}
        update_methods = {}
    ''',
}


def params_for(case, a):
    base = dict(data='cifar100', cl_type='nc', cuda=True, epoch=1, batch=10, verbose=False, mem_size=1000, mem_iters=1,
                eps_mem_batch=10, k=3, aser_type='asvm', n_smp_cls=1.5, num_tasks=a.tasks, images=a.images,
                buffer_tracker=False, optimizer='SGD', learning_rate=0.1, weight_decay=0, temp=0.07, head='mlp',
                subsample=50, error_analysis=False, test_batch=128, num_runs=a.runs, seed=1, online=True,
                model_name='M', data_name='D',
                trick={k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick',
                                          'ncm_trick', 'kd_trick_star')})
    base.update(CASES[case])
    return SimpleNamespace(**base)


def gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=index,name,power.limit,clocks.max.sm,clocks.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return 'nvidia-smi unavailable (%s)' % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=8)
    ap.add_argument('--tasks', type=int, default=3)
    ap.add_argument('--images', type=int, default=2500, help='stream images per task')
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--cases', default=','.join(CASES))
    ap.add_argument('--configs', default='inproc,inproc4,0,00,0000,all')
    ap.add_argument('--startup', action='store_true')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    out = os.path.abspath(a.out) if a.out else None
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this tool measures the GPU and has no CPU fallback')
    from b200ocl import multirun, registry

    work = tempfile.mkdtemp(prefix='b200ocl-multidevice-')
    try:
        run(a, out, work, torch, multirun, registry)
    finally:
        os.chdir(ROOT)
        shutil.rmtree(work, ignore_errors=True)


def interpreter_wall(code):
    """Wall time of a fresh interpreter running `code` (from the repository root), s."""
    t0 = time.perf_counter()
    subprocess.run([sys.executable, '-c', code], cwd=ROOT, check=True)
    return time.perf_counter() - t0


def run(a, out, work, torch, multirun, registry):
    for rel, src in TREE.items():
        path = os.path.join(work, 'reference', rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, 'w') as f:
            f.write(textwrap.dedent(src))
    sys.path.insert(0, os.path.join(work, 'reference'))
    os.chdir(work)
    import utils.name_match as nm
    registry.install(nm)

    n_dev = torch.cuda.device_count()
    every = {'inproc': ('in process', (), 1), 'inproc4': ('in process, R = 4', (), 4), '0': ('0', (0,), 1),
             '00': ('0,0', (0, 0), 1), '0000': ('0,0,0,0', (0, 0, 0, 0), 1)}
    if n_dev > 1:
        every['all'] = (','.join(map(str, range(n_dev))), tuple(range(n_dev)), 1)
    picked = a.configs.split(',')
    configs = [every['inproc']] + [every[k] for k in picked if k in every and k != 'inproc']

    def measure(case, devices, R, runs=None):
        params = params_for(case, a)
        if runs is not None:
            params.num_runs = runs
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            multirun.multiple_run(params, n_concurrent=R, devices=devices)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    info = gpu_info()
    print('GPU:', info, flush=True)
    print('devices visible: %d' % n_dev, flush=True)
    startup = {}
    if a.startup:
        startup['import torch'] = interpreter_wall('import torch')
        startup['+ CUDA context'] = interpreter_wall('import torch; torch.zeros(1, device="cuda"); '
                                                     'torch.cuda.synchronize()')
        startup['+ engine import and library load'] = interpreter_wall(
            'import torch; torch.zeros(1, device="cuda"); from b200ocl import _native, registry; _native.lib()')
        tiny = SimpleNamespace(**vars(a))
        tiny.runs, tiny.tasks, tiny.images = 1, 1, 20

        def tiny_wall(devices):
            params = params_for('er_random', tiny)
            t0 = time.perf_counter()
            with contextlib.redirect_stdout(io.StringIO()):
                multirun.multiple_run(params, n_concurrent=1, devices=devices)
            return time.perf_counter() - t0
        tiny_wall(())                                          # not timed
        walls = [(tiny_wall(()), tiny_wall((0,))) for _ in range(3)]
        startup['1-run tiny experiment, in process'] = statistics.median(w[0] for w in walls)
        startup['1-run tiny experiment, worker 0'] = statistics.median(w[1] for w in walls)
        for k, v in startup.items():
            print('startup: %s: %.2f s' % (k, v), flush=True)
    for case in a.cases.split(','):
        measure(case, (), 1, runs=1)                              # not timed: module loading, first allocations
    results = {}
    for rep in range(a.reps):
        for case in a.cases.split(','):
            for name, devices, R in configs:                   # alternate the configurations within every repetition
                wall = measure(case, devices, R)
                results.setdefault(case, {}).setdefault(name, []).append(wall)
                print(case, name, 'rep %d' % rep, '%.2f s' % wall, flush=True)
    print('\n| case | workers | s / experiment | s / run | vs in process |')
    print('|---|---|---|---|---|')
    table = {}
    for case, byc in results.items():
        base = statistics.median(byc['in process'])
        for name, _, _ in configs:
            med = statistics.median(byc[name])
            table.setdefault(case, {})[name] = med
            print('| %s | %s | %.2f | %.2f | x%.2f |' % (case, name, med, med / a.runs, base / med))
    print('GPU:', gpu_info())
    if out:
        os.makedirs(os.path.dirname(out), exist_ok=True)
        with open(out, 'w') as f:
            json.dump({'gpu': info, 'devices': n_dev, 'runs': a.runs, 'tasks': a.tasks, 'images': a.images,
                       'reps': a.reps, 'startup': startup, 'median': table, 'all': results}, f, indent=1)


if __name__ == '__main__':
    main()
