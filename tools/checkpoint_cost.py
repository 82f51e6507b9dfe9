"""What one snapshot of a run costs (B200OCL_CHECKPOINT_DIR): the time to take and write it, the time to read it and
restore it into a freshly built agent, and its size on disk, for ER with a full memory.

    python tools/checkpoint_cost.py [--data cifar100 core50] [--mem 5000] [--repeats 3] [--out checkpoint_cost.json]

run_group writes one snapshot per run per task (the last task writes the smaller record instead), so the bytes and the
write time below are per run per task.  The snapshot is written to a temporary directory (TMPDIR), as
checkpoint.write_atomic writes it: pickle, flush, fsync, os.replace.  Times are host wall clock (they include the
device-to-host copies, which synchronise the run's stream); median and range over --repeats."""
import argparse
import json
import os
import sys
import tempfile
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from b200ocl import checkpoint, memory, multirun, nets, registry  # noqa: E402


def _params(data, mem):
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick',
                                'kd_trick_star')}
    return SimpleNamespace(data=data, cuda=True, epoch=1, batch=10, verbose=False, mem_size=mem, eps_mem_batch=10,
                           mem_iters=1, update='random', retrieve='random', agent='ER', k=3, aser_type='asvm',
                           n_smp_cls=1.5, num_tasks=10, buffer_tracker=False, optimizer='SGD', learning_rate=0.1,
                           weight_decay=0, temp=0.07, head='mlp', subsample=50, error_analysis=False, trick=trick)


def _agent(params):
    model = nets.setup_architecture(params)
    return registry.agents['ER'](model, torch.optim.SGD(model.parameters(), lr=params.learning_rate), params)


def measure(data, mem, repeats, directory):
    params = _params(data, mem)
    agent = _agent(params)
    buf = agent.buffer
    n_cls = memory.n_classes[data]
    g = torch.Generator(device='cuda').manual_seed(0)
    buf.buffer_img.uniform_(0, 1, generator=g)                    # a full memory: the largest snapshot of the run
    labels = np.arange(mem, dtype=np.int64) % n_cls
    buf.buffer_label.copy_(torch.from_numpy(labels))
    buf.labels_host = labels
    buf.current_index = buf.n_seen_so_far = mem
    agent.old_labels = list(range(n_cls))
    torch.cuda.synchronize()
    ck = checkpoint.Checkpoint(directory, data)
    run = multirun._Run(0, 1)
    run.agent, run.acc = agent, [np.zeros(params.num_tasks)]
    write, read = [], []
    for _ in range(repeats):
        t0 = time.perf_counter()
        ck.save_snapshot(0, run.snapshot(0))
        write.append(time.perf_counter() - t0)
        size = os.path.getsize(ck._path(0, 'snapshot'))
        fresh = multirun._Run(0, 1)
        fresh.agent = fresh.call(_agent, params)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fresh.restore(ck.snapshot(0))
        torch.cuda.synchronize()
        read.append(time.perf_counter() - t0)
        assert torch.equal(fresh.agent.buffer.buffer_img, buf.buffer_img)
        assert torch.equal(fresh.agent.engine.state.params, agent.engine.state.params)
        del fresh
    stat = lambda v: {'median_s': float(np.median(v)), 'min_s': float(min(v)), 'max_s': float(max(v))}   # noqa: E731
    return {'data': data, 'mem_size': mem, 'bytes_per_run_per_task': size,
            'buffer_bytes': buf.buffer_img.numel() * 4 + buf.buffer_label.numel() * 8,
            'write': stat(write), 'restore': stat(read), 'repeats': repeats,
            'device': torch.cuda.get_device_name(0)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--data', nargs='+', default=['cifar100', 'core50'])
    ap.add_argument('--mem', type=int, default=5000)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the results here as JSON')
    args = ap.parse_args()
    results = []
    with tempfile.TemporaryDirectory() as d:
        for data in args.data:
            res = measure(data, args.mem, args.repeats, d)
            results.append(res)
            print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(results, f, indent=1)


if __name__ == '__main__':
    main()
