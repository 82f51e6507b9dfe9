"""What checkpointing costs a run with its snapshots written synchronously (B200OCL_CHECKPOINT_DIR) and behind the run
(B200OCL_CHECKPOINT_ASYNC=1), against no checkpoint at all: ER, memory 5000 (pre-filled with 8-bit rows, the largest
snapshot of a run), R runs side by side through multirun.run_group.

    python tools/checkpoint_async_cost.py [--data cifar100 core50] [--R 1 4] [--tasks 3] [--repeats 2] [--out f.json]

For each data shape and R the three modes run in turn, --repeats times (none, sync, async, none, ...).  Reported per
mode: wall time per task (the run_group call over --tasks tasks of --images stream images per run, host clock, ending
in a device synchronise, divided by --tasks), bytes per snapshot, the time run_group waited for a previous snapshot of
the same run (back-pressure, async only), and the host time per replay step (one step of one run, as run_group takes
it) while a write was in flight and while none was.  Snapshots go to a temporary directory (TMPDIR).  The card and its
power limit are printed with the numbers."""
import argparse
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

from b200ocl import checkpoint, memory, multirun, nets, ops, registry  # noqa: E402

SHAPES = {'cifar100': 32, 'core50': 128}
IMAGES = {'cifar100': 2500, 'core50': 1000}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = 'unknown'
    return {'name': name, 'power_limit': power}


def _params(data, mem):
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick',
                                'kd_trick_star')}
    return SimpleNamespace(data=data, cuda=True, epoch=1, batch=10, verbose=False, mem_size=mem, eps_mem_batch=10,
                           mem_iters=1, update='random', retrieve='random', agent='ER', k=3, aser_type='asvm',
                           n_smp_cls=1.5, num_tasks=10, buffer_tracker=False, optimizer='SGD', learning_rate=0.1,
                           weight_decay=0, temp=0.07, head='mlp', subsample=50, error_analysis=False, trick=trick)


def _make(params, hw):
    n_cls = memory.n_classes[params.data]

    def make(r):
        model = nets.setup_architecture(params)
        agent = registry.agents['ER'](model, torch.optim.SGD(model.parameters(), lr=params.learning_rate), params)
        buf, mem = agent.buffer, params.mem_size
        g = torch.Generator(device='cuda').manual_seed(r)
        for s in range(0, mem, 500):                             # 8-bit rows, as the stream writes them
            n = min(500, mem - s)
            u8 = torch.randint(0, 256, (n, hw, hw, 3), generator=g, device='cuda', dtype=torch.uint8)
            buf.buffer_img[s:s + n].copy_(ops.stream_prepare(u8))
        labels = np.arange(mem, dtype=np.int64) % n_cls
        buf.buffer_label.copy_(torch.from_numpy(labels))
        buf.labels_host = labels
        buf.current_index = buf.n_seen_so_far = mem
        return agent
    return make


def measure(data, R, mode, n_tasks, images, directory):
    hw, params = SHAPES[data], _params(data, 5000)
    n_cls = memory.n_classes[data]
    rs = np.random.RandomState(0)
    tasks = [[(rs.randint(0, 256, (images, hw, hw, 3)).astype(np.uint8), rs.randint(0, n_cls, images).astype(np.int64))
              for _ in range(n_tasks)] for _ in range(R)]
    ck = None if mode == 'none' else checkpoint.Checkpoint(os.path.join(directory, mode), 'runs', mode == 'async')
    sizes, busy, idle = [], [], []
    next_step, save = multirun._next_step, checkpoint.Checkpoint.save_snapshot

    def step(steps):
        w = checkpoint.writer()
        in_flight = bool(w.queue)
        t0 = time.perf_counter()
        out = next_step(steps)
        (busy if in_flight else idle).append(time.perf_counter() - t0)
        return out

    def saved(self, i, state):
        save(self, i, state)
        sizes.append(os.path.getsize(self._path(i, 'snapshot')))
    multirun._next_step, checkpoint.Checkpoint.save_snapshot = step, saved
    before = dict(checkpoint.stats)
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        multirun.run_group(tasks, [[]] * R, _make(params, hw), R, seed=1, checkpoint=ck)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    finally:
        multirun._next_step, checkpoint.Checkpoint.save_snapshot = next_step, save
    if mode == 'async':
        n = checkpoint.stats['snapshots'] - before['snapshots']
        sizes = [(checkpoint.stats['bytes'] - before['bytes']) / max(n, 1)] if n else []
    ms = lambda v: 1e3 * float(np.mean(v)) if v else None                # noqa: E731
    return {'data': data, 'R': R, 'mode': mode, 'wall_s_per_task': wall / n_tasks,
            'bytes_per_snapshot': float(np.mean(sizes)) if sizes else 0,
            'backpressure_s': checkpoint.stats['backpressure_s'] - before['backpressure_s'],
            'host_ms_per_step_write_in_flight': ms(busy), 'host_ms_per_step_no_write': ms(idle),
            'steps_with_write_in_flight': len(busy)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--data', nargs='+', default=['cifar100', 'core50'])
    ap.add_argument('--R', nargs='+', type=int, default=[1, 4])
    ap.add_argument('--tasks', type=int, default=3)
    ap.add_argument('--images', type=int, default=None, help='stream images per task (default 2500, CORe50 1000)')
    ap.add_argument('--repeats', type=int, default=2)
    ap.add_argument('--out', default=None, help='also write the results here as JSON')
    args = ap.parse_args()
    info = card()
    print(json.dumps({'card': info}), flush=True)
    results = []
    with tempfile.TemporaryDirectory() as d:
        for data in args.data:
            for R in args.R:
                for rep in range(args.repeats):
                    for mode in ('none', 'sync', 'async'):
                        res = measure(data, R, mode, args.tasks, args.images or IMAGES[data],
                                      os.path.join(d, '%s_R%d_%d' % (data, R, rep)))
                        res.update(repeat=rep, card=info['name'], power_limit=info['power_limit'])
                        results.append(res)
                        print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(results, f, indent=1)


if __name__ == '__main__':
    main()
