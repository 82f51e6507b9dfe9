"""Time ContinualLearner.evaluate with and without --error_analysis at CIFAR-100 shapes: an ER learner whose label
bookkeeping has seen 10 tasks of 10 classes, 10 test loaders of 1000 images each (10 000 in all) in batches of 128 (the
reference's test_batch).  The two variants alternate over --reps rounds after --warmup rounds of each; every evaluate()
ends in a device -> host read, so a host clock around it covers the GPU work.  Prints one JSON line with the GPU's name
and power limit beside the medians.

    python tools/eval_error_analysis.py [--reps 10] [--warmup 2]
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def power_limit():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'this measurement needs the GPU'
    from b200ocl import nets, registry
    params = SimpleNamespace(data='cifar100', cuda=True, epoch=1, batch=10, verbose=False, mem_size=100, eps_mem_batch=10,
                             mem_iters=1, update='random', retrieve='random', agent='ER', k=3, aser_type='asvm',
                             n_smp_cls=1.5, num_tasks=10, buffer_tracker=False, optimizer='SGD', learning_rate=0.1,
                             weight_decay=0, temp=0.07, head='mlp', subsample=50, error_analysis=False, test_batch=128,
                             trick={'labels_trick': False, 'kd_trick': False, 'separated_softmax': False,
                                    'review_trick': False, 'ncm_trick': False, 'kd_trick_star': False})
    torch.manual_seed(0)
    agent = registry.agents['ER'](nets.setup_architecture(params), None, params)
    tasks = [list(range(t, t + 10)) for t in range(0, 100, 10)]
    for labels in tasks:
        agent.before_train(None, np.asarray(labels))
        agent.after_train()
    rs = np.random.RandomState(0)
    loaders = []
    for labels in tasks:
        x = torch.from_numpy(rs.rand(1000, 3, 32, 32).astype(np.float32))
        y = torch.from_numpy(rs.choice(labels, 1000).astype(np.int64))
        loaders.append([(x[i:i + 128].pin_memory(), y[i:i + 128].pin_memory()) for i in range(0, 1000, 128)])
    times = {False: [], True: []}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)                     # the analysis writes its confusion file to the working directory
        try:
            for r in range(a.warmup + a.reps):
                for ea in (False, True):
                    params.error_analysis = ea
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    with contextlib.redirect_stdout(io.StringIO()):
                        acc = agent.evaluate(loaders)
                    torch.cuda.synchronize()
                    if r >= a.warmup:
                        times[ea].append(time.perf_counter() - t0)
        finally:
            os.chdir(cwd)
    off, on = np.median(times[False]) * 1e3, np.median(times[True]) * 1e3
    print(json.dumps({'gpu': torch.cuda.get_device_name(0), 'power_limit': power_limit(), 'loaders': 10,
                      'test_images': 10000, 'test_batch': 128, 'reps': a.reps, 'evaluate_ms': round(off, 3),
                      'evaluate_error_analysis_ms': round(on, 3), 'overhead_ms': round(on - off, 3),
                      'min_ms': [round(min(times[False]) * 1e3, 3), round(min(times[True]) * 1e3, 3)],
                      'acc_mean': float(np.mean(acc))}))


if __name__ == '__main__':
    main()
