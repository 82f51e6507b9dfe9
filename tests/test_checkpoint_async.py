"""CPU: snapshots written behind the run (B200OCL_CHECKPOINT_ASYNC=1, checkpoint.py) with stub agents whose "device"
arrays are host tensors: the switch and its refusals in install(), the writer's order (a record is never overtaken by its
training's snapshot, the snapshot is deleted after it), draining when a hook raises, a failing write surfacing as
CheckpointError, an interrupted write leaving the previous file whole, and both file forms read by Checkpoint.snapshot()."""
import gc
import os
import threading
import weakref

import numpy as np
import pytest
import torch

from b200ocl import checkpoint, memory, multirun

from test_multirun import reference  # noqa: F401  (the stub reference tree, a fixture)
from test_checkpoint import Interrupt, N_RUNS, N_TASKS, SnapAgent


class PartsAgent(SnapAgent):
    """SnapAgent whose state also has "device" arrays: its draws as an int64 tensor and 8-bit rows."""

    def snapshot_parts(self):
        self.log.append(('snapshot', self.r))
        rows = torch.arange(12, dtype=torch.float32).reshape(3, 4) / 255
        return {'draws': list(self.draws), 'arr': torch.tensor(self.draws, dtype=torch.int64),
                'rows': memory.Rows8(rows)}

    def snapshot_capacity(self):
        return 1 << 10

    def restore(self, state):
        assert torch.equal(state['arr'], torch.tensor(state['draws'], dtype=torch.int64))
        super().restore(state)


def _experiment(directory, R, fail=None, seed=5):
    log, agents = [], {}

    def make(r):
        log.append(('build', r))
        agents[r] = PartsAgent(r, log)
        agents[r].device = 'cpu'
        return agents[r]

    def on_task(r, t, x, y):
        if fail == (r, t):
            raise Interrupt('run %d task %d' % (r, t))

    def on_run_end(r, acc):
        print('run %d end %r' % (r, acc[-1].tolist()))

    tasks = [[(np.zeros(2 + r), np.zeros(2 + r))] * N_TASKS for r in range(N_RUNS)]
    ck = None if directory is None else checkpoint.Checkpoint(str(directory), 'runs', async_write=True)
    res = multirun.run_group(tasks, [[None, None]] * N_RUNS, make, R, seed=seed, on_task=on_task,
                             on_run_end=on_run_end, checkpoint=ck)
    return log, agents, res


def test_switch_parsing_and_refusals(reference, monkeypatch, tmp_path):
    from b200ocl import registry
    d = {checkpoint.ENV: str(tmp_path)}
    assert checkpoint.checkpoint_async({}) is False
    assert checkpoint.checkpoint_async({checkpoint.ASYNC_ENV: '0'}) is False
    assert checkpoint.checkpoint_async({checkpoint.ASYNC_ENV: ''}) is False
    assert checkpoint.checkpoint_async(dict(d, **{checkpoint.ASYNC_ENV: ' 1 '})) is True
    assert checkpoint.checkpoint_async({checkpoint.ASYNC_ENV: '1'}, directory=str(tmp_path)) is True
    for bad in ('2', 'yes', 'true', '01'):
        with pytest.raises(ValueError, match=checkpoint.ASYNC_ENV):
            checkpoint.checkpoint_async(dict(d, **{checkpoint.ASYNC_ENV: bad}))
    with pytest.raises(ValueError, match=checkpoint.ENV):
        checkpoint.checkpoint_async({checkpoint.ASYNC_ENV: '1'})
    _, mods = reference
    nm, run = mods['utils.name_match'], mods['experiment.run']
    original = run.multiple_run
    for k in (multirun.ENV, multirun.DEVICES_ENV, checkpoint.ENV):
        monkeypatch.delenv(k, raising=False)
    for env in ({checkpoint.ASYNC_ENV: '1'}, {checkpoint.ASYNC_ENV: 'on', checkpoint.ENV: str(tmp_path / 'ck')}):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        with pytest.raises(ValueError, match=checkpoint.ASYNC_ENV):
            registry.install(nm)
        assert run.multiple_run is original                                  # nothing was replaced
    monkeypatch.setenv(checkpoint.ASYNC_ENV, '1')
    registry.install(nm)
    assert run.multiple_run is multirun.multiple_run
    registry.uninstall(nm)
    assert not (tmp_path / 'ck').exists()


def test_a_staged_run_resumes_like_a_synchronous_one(tmp_path, capsys):
    _, want_agents, want = _experiment(None, 1)
    want_out = capsys.readouterr().out
    d = tmp_path / 'ck'
    with pytest.raises(Interrupt):
        _experiment(d, 1, fail=(2, 1))                 # the hook raises: every queued write has ended before it leaves
    assert sorted(os.listdir(str(d / 'runs'))) == ['run0.record', 'run1.record', 'run2.snapshot']
    with open(str(d / 'runs' / 'run2.snapshot'), 'rb') as f:
        assert f.read(len(checkpoint.MAGIC)) == checkpoint.MAGIC
    snap = checkpoint.Checkpoint(str(d), 'runs').snapshot(2)
    assert snap['task'] == 0 and torch.equal(snap['agent']['rows'], torch.arange(12.).reshape(3, 4) / 255)
    capsys.readouterr()
    log, agents, got = _experiment(d, 1)
    assert [e[1] for e in log if e[0] == 'restore'] == [2]
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    assert all(agents[r].draws == want_agents[r].draws for r in agents)
    assert capsys.readouterr().out == want_out
    assert sorted(os.listdir(str(d / 'runs'))) == ['run%d.record' % r for r in range(N_RUNS)]


def test_a_record_is_never_overtaken_by_its_snapshot(tmp_path, monkeypatch):
    """The snapshot write is held until the record is queued: the record still lands after it and deletes it."""
    order, gate = [], threading.Event()
    write = checkpoint._Job.write

    def slow(job):
        gate.wait(10)
        write(job)
        order.append(('snapshot', os.path.basename(job.path)))
    save_record = checkpoint.Checkpoint._save_record

    def record(self, i, acc, text):
        order.append(('record', i, os.path.exists(self._path(i, 'snapshot'))))
        save_record(self, i, acc, text)
    monkeypatch.setattr(checkpoint._Job, 'write', slow)
    monkeypatch.setattr(checkpoint.Checkpoint, '_save_record', record)
    ck = checkpoint.Checkpoint(str(tmp_path), 'runs', async_write=True)
    staging = checkpoint.Staging(0, 'cpu')
    tree, job = staging.stage({'x': torch.ones(3)})
    ck.save_staged(0, {'task': 0, 'acc': [], 'rng': None, 'sampler': None, 'agent': tree}, job)
    ck.save_record(0, np.zeros(1), 'text')
    gate.set()
    checkpoint.writer().drain()
    assert order == [('snapshot', 'run0.snapshot'), ('record', 0, True)]
    assert os.listdir(str(tmp_path / 'runs')) == ['run0.record']


@pytest.mark.parametrize('where', ['replace', 'fsync'])
def test_a_failed_write_raises_checkpoint_error_and_keeps_the_previous_file(where, tmp_path, monkeypatch, capsys):
    d = tmp_path / 'ck'
    with pytest.raises(Interrupt):
        _experiment(d, 1, fail=(0, 2))                 # run 0's task-1 snapshot is on disk
    assert checkpoint.Checkpoint(str(d), 'runs').snapshot(0)['task'] == 1

    def boom(*args):
        raise OSError(28, 'No space left on device')
    monkeypatch.setattr(os, where, boom)
    ck = checkpoint.Checkpoint(str(d), 'runs', async_write=True)
    tree, job = checkpoint.Staging(0, 'cpu').stage({'x': torch.ones(3)})
    ck.save_staged(0, {'task': 2, 'acc': [1, 2, 3], 'rng': None, 'sampler': None, 'agent': tree}, job)
    with pytest.raises(checkpoint.CheckpointError, match='run0.snapshot') as e:
        checkpoint.writer().drain()
    assert isinstance(e.value.__cause__, OSError)
    monkeypatch.undo()
    assert checkpoint.Checkpoint(str(d), 'runs').snapshot(0)['task'] == 1   # the previous file is whole
    checkpoint.writer().check()                                             # raised once
    # a failure is also raised at the next boundary
    monkeypatch.setattr(os, where, boom)
    tree, job = checkpoint.Staging(0, 'cpu').stage({'x': torch.ones(3)})
    ck.save_staged(0, {'task': 2, 'acc': [1, 2, 3], 'rng': None, 'sampler': None, 'agent': tree}, job)
    job.done.wait(10)
    staging = checkpoint.Staging(0, 'cpu')
    with pytest.raises(checkpoint.CheckpointError, match='run0.snapshot'):
        staging.stage({'x': torch.ones(3)})
    assert staging.pending is None                                          # nothing was staged
    monkeypatch.undo()
    checkpoint.writer().drain()


def test_a_run_group_that_fails_leaves_no_write_error_behind(tmp_path, monkeypatch, capsys):
    """A write that fails while a hook raises is told with the hook's exception, and only there: the next run_group of
    the process does not meet it."""
    replace = os.replace

    def boom(src, dst):
        if dst.endswith('.snapshot'):
            raise OSError(28, 'No space left on device')
        return replace(src, dst)
    monkeypatch.setattr(os, 'replace', boom)
    with pytest.raises(Interrupt) as e:
        _experiment(tmp_path / 'a', 1, fail=(0, 1))        # run 0's task-0 snapshot fails, then the hook raises
    assert any('run0.snapshot' in n for n in getattr(e.value, '__notes__', []))
    monkeypatch.undo()
    _experiment(tmp_path / 'b', 1)                         # no stale CheckpointError
    assert sorted(os.listdir(str(tmp_path / 'b' / 'runs'))) == ['run%d.record' % r for r in range(N_RUNS)]


def test_a_job_that_cannot_be_queued_is_ended(tmp_path, monkeypatch):
    ck = checkpoint.Checkpoint(str(tmp_path), 'runs', async_write=True)
    staging = checkpoint.Staging(0, 'cpu')
    tree, job = staging.stage({'x': torch.ones(3)})

    def refuse(*args):
        raise RuntimeError('queue refused')
    monkeypatch.setattr(checkpoint.writer(), 'submit', refuse)
    with pytest.raises(RuntimeError, match='queue refused'):
        ck.save_staged(0, {'task': 0, 'acc': [], 'rng': None, 'sampler': None, 'agent': tree}, job)
    assert job.done.is_set() and job.staging is None
    staging.wait()                                         # returns: the next boundary does not hang


def test_a_finished_run_frees_its_staging_without_the_cyclic_collector(tmp_path, monkeypatch, capsys):
    made = []
    init = checkpoint.Staging.__init__

    def tracked(self, *args):
        init(self, *args)
        made.append(weakref.ref(self))
    monkeypatch.setattr(checkpoint.Staging, '__init__', tracked)
    gc.collect()
    gc.disable()
    try:
        _experiment(tmp_path / 'ck', 2)
        assert len(made) == N_RUNS
        assert [r() for r in made] == [None] * N_RUNS
    finally:
        gc.enable()


def test_a_plugin_with_only_snapshot_keeps_its_state():
    from types import SimpleNamespace
    from b200ocl.memory import Buffer

    class Plugin(object):
        def __init__(self, params):
            self.score = torch.arange(4.)

        def snapshot(self):
            return {'score': self.score.clone()}

        def restore(self, state):
            self.score.copy_(state['score'])
    params = SimpleNamespace(cuda=False, mem_size=4, data='cifar10', update='p', retrieve='r')
    buf = Buffer(None, params, update_methods={'p': Plugin}, retrieve_methods={'r': lambda p: None})
    snap = buf.snapshot()
    assert torch.equal(snap['update']['score'], torch.arange(4.))
    buf.update_method.score.zero_()
    buf.restore(snap)
    assert torch.equal(buf.update_method.score, torch.arange(4.))


def test_both_forms_are_read(tmp_path):
    ck = checkpoint.Checkpoint(str(tmp_path), 'runs')
    parts = {'p': torch.randn(5), 'n': torch.arange(4), 'rows': memory.Rows8(torch.tensor([0., 1., 128 / 255.]))}
    plain = memory.host_tree(parts)
    ck.save_snapshot(0, {'task': 0, 'acc': [], 'rng': None, 'sampler': 's', 'agent': plain})
    tree, job = checkpoint.Staging(0, 'cpu').stage(parts)
    ck.save_staged(1, {'task': 0, 'acc': [], 'rng': None, 'sampler': 's', 'agent': tree}, job)
    checkpoint.writer().drain()
    for i in (0, 1):
        got = ck.snapshot(i)['agent']
        assert set(got) == set(plain)
        for k in plain:
            assert got[k].dtype == plain[k].dtype and torch.equal(got[k], plain[k]), (i, k)
    with open(ck._path(1, 'snapshot'), 'r+b') as f:                         # a truncated payload is refused
        f.truncate(os.path.getsize(ck._path(1, 'snapshot')) - 1)
    with pytest.raises(checkpoint.CheckpointError, match='run1.snapshot'):
        ck.snapshot(1)
