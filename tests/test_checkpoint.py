"""CPU: resumable experiments (B200OCL_CHECKPOINT_DIR, checkpoint.py) with stub agents: the switch, install() /
uninstall(), the fingerprint check and the refusals before anything is built, the atomic snapshot write, and
run_group's bookkeeping -- which runs are skipped, which resume and at which task, the output order, the arrays and the
--store pickle of multiple_run -- against experiments that were never interrupted."""
import os
import pickle

import numpy as np
import pytest

from b200ocl import checkpoint, memory, multirun

import test_multirun as tm
from test_multirun import reference  # noqa: F401  (the stub reference tree, a fixture)


class Interrupt(Exception):
    pass


class SnapAgent(tm.StubAgent):
    """StubAgent with the snapshot / restore pair: its state is the list of draws it made."""

    def snapshot(self):
        self.log.append(('snapshot', self.r))
        return {'draws': list(self.draws)}

    def restore(self, state):
        self.log.append(('restore', self.r))
        self.draws = list(state['draws'])


N_RUNS, N_TASKS = 4, 3


def _experiment(directory, R, fail=None, seed=5):
    """run_group over N_RUNS runs of N_TASKS tasks (2 + r steps each) with on_task / on_run_end hooks that print; `fail`
    = (r, t) raises from on_task at run r, task t.  Returns (log, agents, results, stdout lines)."""
    log, agents = [], {}

    def make(r):
        log.append(('build', r))
        agents[r] = SnapAgent(r, log)
        return agents[r]

    def on_task(r, t, x, y):
        if fail == (r, t):
            raise Interrupt('run %d task %d' % (r, t))
        log.append(('task', r, t))

    def on_run_end(r, acc):
        print('run %d end %r' % (r, acc[-1].tolist()))

    tasks = [[(np.zeros(2 + r), np.zeros(2 + r))] * N_TASKS for r in range(N_RUNS)]
    ck = None if directory is None else checkpoint.Checkpoint(str(directory), 'runs')
    res = multirun.run_group(tasks, [[None, None]] * N_RUNS, make, R, seed=seed, on_task=on_task,
                             on_run_end=on_run_end, checkpoint=ck)
    return log, agents, res


def test_switch_parsing():
    assert checkpoint.checkpoint_dir({}) is None
    assert checkpoint.checkpoint_dir({checkpoint.ENV: ''}) is None
    assert checkpoint.checkpoint_dir({checkpoint.ENV: '   '}) is None
    assert checkpoint.checkpoint_dir({checkpoint.ENV: ' /tmp/ck '}) == '/tmp/ck'


def test_install_replaces_the_drivers_only_with_the_switch(reference, monkeypatch, tmp_path):
    from b200ocl import registry
    _, mods = reference
    nm, run = mods['utils.name_match'], mods['experiment.run']
    run.multiple_run_tune_separate = object()
    original, original_tune = run.multiple_run, run.multiple_run_tune_separate
    for k in (multirun.ENV, multirun.DEVICES_ENV, checkpoint.ENV):
        monkeypatch.delenv(k, raising=False)
    registry.install(nm)
    assert run.multiple_run is original and run.multiple_run_tune_separate is original_tune
    registry.uninstall(nm)
    monkeypatch.setenv(checkpoint.ENV, '')
    registry.install(nm)
    assert run.multiple_run is original
    registry.uninstall(nm)
    monkeypatch.setenv(checkpoint.ENV, str(tmp_path / 'ck'))
    registry.install(nm)
    assert run.multiple_run is multirun.multiple_run
    assert run.multiple_run_tune_separate is multirun.multiple_run_tune_separate
    registry.uninstall(nm)
    assert run.multiple_run is original and run.multiple_run_tune_separate is original_tune
    assert not (tmp_path / 'ck').exists()                                           # install() writes nothing


def test_parity_mode_and_data_parallel_sync_are_refused(reference, monkeypatch, tmp_path, capsys):
    from b200ocl import registry
    _, mods = reference
    nm, run = mods['utils.name_match'], mods['experiment.run']
    original = run.multiple_run
    monkeypatch.setenv(checkpoint.ENV, str(tmp_path / 'ck'))
    memory.set_mode(True)
    try:
        with pytest.raises(ValueError, match='parity'):
            registry.install(nm)
        assert run.multiple_run is original
        with pytest.raises(ValueError, match='parity'):
            multirun.multiple_run(tm._params(), n_concurrent=1)
        with pytest.raises(ValueError, match='parity'):
            multirun.run_group([[(np.zeros(1), None)]], [[None]], tm._never, 1,
                               checkpoint=checkpoint.Checkpoint(str(tmp_path / 'ck'), 'runs'))
    finally:
        memory.set_mode(False)
    with pytest.raises(ValueError, match='data-parallel'):
        checkpoint.check_checkpoint(str(tmp_path / 'ck'), grad_sync=True)
    monkeypatch.setattr(multirun, '_data_parallel', lambda: True)
    with pytest.raises(ValueError, match='data-parallel'):
        multirun.multiple_run(tm._params(), n_concurrent=1)
    with pytest.raises(ValueError, match='data-parallel'):
        registry.install(nm)
    assert capsys.readouterr().out == ''                                            # no data stream was set up
    assert not (tmp_path / 'ck').exists()
    checkpoint.check_checkpoint(None, grad_sync=True)                               # the switch off: no refusal


def test_a_fingerprint_mismatch_raises_before_anything_is_built(reference, tmp_path, capsys):
    d = str(tmp_path / 'ck')
    p = tm._params()
    checkpoint.open_dir(d, checkpoint.fingerprint(p))
    checkpoint.open_dir(d, checkpoint.fingerprint(tm._params()))                    # the same settings: accepted
    p.learning_rate = 0.05
    with pytest.raises(ValueError, match='learning_rate'):
        multirun.multiple_run(p, store=True, n_concurrent=1, checkpoint_dir=d)
    assert capsys.readouterr().out == ''
    for other in (dict(extra=('EWC',)), dict(grid={'learning_rate': [0.1]}), dict(build='another build')):
        with pytest.raises(ValueError):
            checkpoint.open_dir(d, checkpoint.fingerprint(tm._params(), **other))
    q = tm._params()
    q.seed = 1
    with pytest.raises(ValueError, match='seed'):
        checkpoint.open_dir(d, checkpoint.fingerprint(q))


def test_an_interrupted_write_leaves_the_previous_snapshot(tmp_path, monkeypatch):
    ck = checkpoint.Checkpoint(str(tmp_path), 'runs')
    ck.save_snapshot(3, {'task': 0, 'acc': [1], 'rng': None, 'sampler': None, 'agent': 'first'})

    def boom(src, dst):
        assert os.path.exists(src)
        raise Interrupt('between the write and the rename')
    monkeypatch.setattr(os, 'replace', boom)
    with pytest.raises(Interrupt):
        ck.save_snapshot(3, {'task': 1, 'acc': [1, 2], 'rng': None, 'sampler': None, 'agent': 'second'})
    monkeypatch.undo()
    assert ck.snapshot(3)['agent'] == 'first'
    assert ck.record(3) is None and ck.snapshot(2) is None


def test_an_unreadable_file_raises(tmp_path):
    ck = checkpoint.Checkpoint(str(tmp_path), 'runs')
    (tmp_path / 'runs').mkdir()
    (tmp_path / 'runs' / 'run0.snapshot').write_bytes(b'not a pickle')
    with pytest.raises(checkpoint.CheckpointError, match='run0.snapshot'):
        ck.snapshot(0)
    (tmp_path / 'runs' / 'run1.record').write_bytes(pickle.dumps([1, 2]))
    with pytest.raises(checkpoint.CheckpointError, match='not a record'):
        ck.record(1)
    (tmp_path / 'fingerprint.pkl').write_bytes(b'')
    with pytest.raises(checkpoint.CheckpointError, match='fingerprint'):
        checkpoint.open_dir(str(tmp_path), {'params': {}})


def _files(d):
    return sorted(os.listdir(os.path.join(str(d), 'runs')))


@pytest.mark.parametrize('R', [1, 3])
def test_run_group_skips_resumes_and_restarts(R, tmp_path, capsys):
    _, want_agents, want = _experiment(None, R)
    want_out = capsys.readouterr().out
    d = tmp_path / 'ck'
    with pytest.raises(Interrupt):
        _experiment(d, R, fail=(2, 1))
    first_out = capsys.readouterr().out
    if R == 1:
        # runs 0 and 1 ended (records), run 2 finished task 0 (snapshot), run 3 never started
        assert _files(d) == ['run0.record', 'run1.record', 'run2.snapshot']
        assert first_out == ''.join(l for l in want_out.splitlines(True) if l.startswith(('run 0', 'run 1')))
    else:
        # the first group (runs 0-2) finished task 0 and run 1 task 1 failed on run 2's hook: every run of the group has
        # its task-0 snapshot, run 0 and run 1 were not snapshot at task 1 (the group's evaluation never came)
        assert _files(d) == ['run0.snapshot', 'run1.snapshot', 'run2.snapshot']
        assert first_out == ''
    snaps = {r: checkpoint.Checkpoint(str(d), 'runs').snapshot(r) for r in range(N_RUNS)}
    assert snaps[2]['task'] == 0 and len(snaps[2]['acc']) == 1
    log, agents, got = _experiment(d, R)
    out = capsys.readouterr().out
    built = [e[1] for e in log if e[0] == 'build']
    assert built == ([2, 3] if R == 1 else [0, 1, 2, 3])
    assert [e[1] for e in log if e[0] == 'restore'] == ([2] if R == 1 else [0, 1, 2])
    tasks = [(e[1], e[2]) for e in log if e[0] == 'task']
    if R == 1:
        assert tasks == [(2, 1), (2, 2), (3, 0), (3, 1), (3, 2)]
    else:
        assert sorted(tasks) == sorted([(r, t) for r in range(3) for t in (1, 2)] + [(3, t) for t in range(3)])
    # the arrays, the draws of the resumed runs and the per-run lines are the uninterrupted ones, in run order
    assert len(got) == N_RUNS
    for r in range(N_RUNS):
        assert np.array_equal(got[r], want[r]), r
    for r in agents:
        assert agents[r].draws == want_agents[r].draws, r
    assert out == want_out                                          # the ended runs' lines come back from their records
    assert _files(d) == ['run%d.record' % r for r in range(N_RUNS)]
    # a third start trains nothing and gives the same arrays and lines
    log, _, again = _experiment(d, R)
    assert [e for e in log if e[0] == 'build'] == [] and capsys.readouterr().out == want_out
    assert all(np.array_equal(a, b) for a, b in zip(again, want))


def test_the_records_of_runs_before_a_group_come_first(tmp_path, capsys):
    """Run 1 has a record, run 0 and run 2 train: run 0's line, then run 1's, then run 2's."""
    _, _, want = _experiment(None, 2)
    want_out = capsys.readouterr().out
    d = tmp_path / 'ck'
    _experiment(d, 1)
    capsys.readouterr()
    for r in (0, 2, 3):
        os.remove(os.path.join(str(d), 'runs', 'run%d.record' % r))
    log, _, got = _experiment(d, 2)
    assert [e[1] for e in log if e[0] == 'build'] == [0, 2, 3]
    assert capsys.readouterr().out == want_out
    assert all(np.array_equal(a, b) for a, b in zip(got, want))


def test_multiple_run_resumes_with_the_same_store_and_summary(reference, monkeypatch, tmp_path, capsys):
    log, mods = reference

    class Agent(SnapAgent):
        def __init__(self, model, opt, params):
            super().__init__(model, log)
    mods['utils.name_match'].agents['ER'] = Agent

    def go(name, d, R):
        multirun.multiple_run(tm._params(), store=True, save_path=name, n_concurrent=R, checkpoint_dir=d)
        with open('result/cifar100/' + name, 'rb') as f:
            return pickle.load(f)['acc_array'], capsys.readouterr().out.splitlines()
    want, want_out = go('plain.pkl', '', 2)
    d = str(tmp_path / 'ck')
    on_task = multirun._Repetitions.on_task

    def failing(self, r, t, x, y):
        if (r, t) == (3, 2):
            raise Interrupt('run 3 task 2')
        return on_task(self, r, t, x, y)
    monkeypatch.setattr(multirun._Repetitions, 'on_task', failing)
    with pytest.raises(Interrupt):
        go('resumed.pkl', d, 2)
    assert not os.path.exists('result/cifar100/resumed.pkl')
    first = capsys.readouterr().out.splitlines()
    monkeypatch.setattr(multirun._Repetitions, 'on_task', on_task)
    got, out = go('resumed.pkl', d, 2)
    assert got.shape == (tm.N_RUNS, tm.N_TASKS, tm.N_TASKS) and np.array_equal(got, want)
    assert out[-1] == want_out[-1] and out[-1].startswith('----------- Avg_End_Acc')
    ends = lambda lines: [l.split('-----------train time')[0] for l in lines if 'avg_end_acc' in l]   # noqa: E731
    assert ends(out) == ends(want_out) and len(ends(want_out)) == tm.N_RUNS
    assert set(ends(first)) <= set(ends(want_out)) and len(ends(first)) == 2    # runs 0 and 1 ended in the first start
    assert sorted(os.listdir(os.path.join(d, 'runs'))) == ['run%d.record' % r for r in range(tm.N_RUNS)]
