"""GPU: an experiment interrupted by a Python exception and started again on the same checkpoint directory
(B200OCL_CHECKPOINT_DIR) ends with what an uninterrupted one gives, bit for bit: the --store acc_array, the summary line,
and every run's final state (agent_cases.final_state: parameters, BN statistics, the memory with DER++'s logits and
GEM's rings, Adam moments and step, EWC++ arenas).  Three runs of three synthetic CIFAR-shaped tasks
(test_gpu_multidevice.py's stub reference tree, written to tmp_path), at R = 1 and R = 3, interrupted from the on_task
hook at (run 1, task 2) or from inside step 2 of task 1 of run 2 (which resumes from the end of task 0), for
RESUME_CASES of agent_cases.CASES: ER (random, ASER, MIR, GSS update), SCR, A-GEM, LwF with kd_trick, ER with the review
trick and separated softmax, iCaRL, GDumb, EWC++, ER with torch.optim.Adam, DER++, PCR and GEM.  main_tune.py's loop
interrupted in its tuning stage chooses the same points, and runs on workers 0,0 resume like runs in process."""
import multiprocessing
import os
import pickle
import sys
import textwrap

import numpy as np
import pytest
import torch

from b200ocl import multirun

import agent_cases
import test_gpu_multidevice as md

pytestmark = pytest.mark.gpu

N_RUNS = 3
RESUME_CASES = ('er_random', 'er_aser', 'er_mir', 'er_gss', 'scr', 'agem', 'lwf_kd', 'er_review_sep', 'icarl', 'gdumb',
                'ewc', 'er_adam', 'derpp', 'pcr', 'gem')

TREE = dict(md.STUB_TREE)
TREE['utils/setup_elements.py'] = '''
    import torch
    from b200ocl.nets import setup_architecture


    def setup_opt(optimizer, model, lr, wd):
        if optimizer == 'Adam':
            return torch.optim.Adam(model.parameters(), lr=lr, weight_decay=wd)
        return torch.optim.SGD(model.parameters(), lr=lr, weight_decay=wd)
'''
TREE['utils/name_match.py'] = '''
    import os

    import torch
    from agent_cases import final_state
    from b200ocl import registry

    from continuum.continuum import LAST_RUN


    _recording = {}


    def recording(cls):
        """cls, saving its run's state to $CHECKPOINT_OUT/run<r>.pt after every evaluation, and raising RuntimeError
        after step k of task t of run r when $CHECKPOINT_FAIL_STEP is 'r,t,k'."""
        if cls not in _recording:
            class Recording(cls):
                def __init__(self, model, opt, params):
                    super().__init__(model, opt, params)
                    self.stub_run = LAST_RUN[0]

                def _steps(self, x, y):
                    fail = os.environ.get('CHECKPOINT_FAIL_STEP')
                    fail = tuple(int(v) for v in fail.split(',')) if fail else None
                    task, k = self.task_seen, 0
                    for _ in super()._steps(x, y):
                        yield
                        k += 1
                        if fail == (self.stub_run, task, k):
                            raise RuntimeError('injected failure in run %d, task %d, step %d' % fail)

                def evaluate(self, loaders):
                    acc = super().evaluate(loaders)
                    out = os.environ.get('CHECKPOINT_OUT')
                    if out:
                        torch.save(final_state(self), os.path.join(out, 'run%d.pt' % self.stub_run))
                    return acc
            _recording[cls] = Recording
        return _recording[cls]


    class Agents(dict):
        def __getitem__(self, key):
            return recording(dict.__getitem__(self, key))


    agents = Agents(registry.agents)
    retrieve_methods = {}
    update_methods = {}
'''


class Interrupt(Exception):
    pass


@pytest.fixture
def stub_tree(monkeypatch, tmp_path):
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    ref = tmp_path / 'reference'
    for rel, src in TREE.items():
        (ref / rel).parent.mkdir(parents=True, exist_ok=True)
        (ref / rel).write_text(textwrap.dedent(src))
    saved = {k: v for k, v in sys.modules.items() if k.split('.')[0] in md.PACKAGES}
    for k in saved:
        del sys.modules[k]
    monkeypatch.syspath_prepend(str(ref))
    monkeypatch.chdir(tmp_path)
    for k in (multirun.ENV, multirun.DEVICES_ENV, 'B200OCL_CHECKPOINT_DIR', 'CHECKPOINT_FAIL_STEP'):
        monkeypatch.delenv(k, raising=False)
    yield tmp_path
    for k in [k for k in sys.modules if k.split('.')[0] in md.PACKAGES]:
        del sys.modules[k]
    sys.modules.update(saved)
    assert multiprocessing.active_children() == []


def _params(case):
    p = md._params(case)
    p.num_runs = N_RUNS
    return p


def _experiment(case, R, name, d, monkeypatch, capsys, devices=()):
    """One multiple_run with checkpoint directory d ('' for none); returns (acc_array, summary line, final states)."""
    out = os.path.join(os.getcwd(), 'states_' + name)
    os.makedirs(out, exist_ok=True)
    monkeypatch.setenv('CHECKPOINT_OUT', out)
    multirun.multiple_run(_params(case), store=True, save_path=name + '.pkl', n_concurrent=R, devices=devices,
                          checkpoint_dir=d)
    torch.cuda.synchronize()
    lines = capsys.readouterr().out.splitlines()
    with open('result/cifar10/%s.pkl' % name, 'rb') as f:
        acc = pickle.load(f)['acc_array']
    return acc, lines[-1], [torch.load(os.path.join(out, 'run%d.pt' % r)) for r in range(N_RUNS)]


def _same(got, want, what):
    assert got[0].shape == (N_RUNS, 3, 3) and np.array_equal(got[0], want[0]), (what, got[0], want[0])
    assert got[1] == want[1] and got[1].startswith('----------- Avg_End_Acc'), (what, got[1], want[1])
    for r in range(N_RUNS):
        assert len(got[2][r]) == len(want[2][r]), (what, r)
        for i, (x, y) in enumerate(zip(got[2][r], want[2][r])):
            assert torch.equal(x, y), (what, r, i)
    assert not torch.equal(want[2][0][0], want[2][1][0])                           # the runs differ


_PLAIN = {}


def _install(case):
    from b200ocl import registry
    import utils.name_match as nm
    registry.install(nm, extra=agent_cases.extra(case))
    return lambda: registry.uninstall(nm)


@pytest.mark.parametrize('how', ['on_task', 'step'])
@pytest.mark.parametrize('R', [1, 3])
@pytest.mark.parametrize('case', sorted(RESUME_CASES))
def test_a_resumed_experiment_matches_an_uninterrupted_one(case, R, how, stub_tree, monkeypatch, capsys):
    uninstall = _install(case)
    try:
        if (case, R) not in _PLAIN:
            _PLAIN[case, R] = _experiment(case, R, 'plain', '', monkeypatch, capsys)
        d = str(stub_tree / 'ck')
        if how == 'on_task':
            on_task = multirun._Repetitions.on_task

            def failing(self, r, t, x, y):
                if (r, t) == (1, 2):
                    raise Interrupt('run 1, task 2')
                return on_task(self, r, t, x, y)
            monkeypatch.setattr(multirun._Repetitions, 'on_task', failing)
            with pytest.raises(Interrupt):
                _experiment(case, R, 'resumed', d, monkeypatch, capsys)
            monkeypatch.setattr(multirun._Repetitions, 'on_task', on_task)
            want_files = ['run0.record', 'run1.snapshot'] if R == 1 else ['run%d.snapshot' % r for r in range(3)]
        else:
            monkeypatch.setenv('CHECKPOINT_FAIL_STEP', '2,1,2')
            with pytest.raises(RuntimeError, match='injected failure'):
                _experiment(case, R, 'resumed', d, monkeypatch, capsys)
            monkeypatch.delenv('CHECKPOINT_FAIL_STEP')
            want_files = ['run0.record', 'run1.record', 'run2.snapshot'] if R == 1 else \
                ['run%d.snapshot' % r for r in range(3)]
        assert sorted(os.listdir(os.path.join(d, 'runs'))) == want_files
        got = _experiment(case, R, 'resumed', d, monkeypatch, capsys)
        assert sorted(os.listdir(os.path.join(d, 'runs'))) == ['run%d.record' % r for r in range(N_RUNS)]
    finally:
        uninstall()
    _same(got, _PLAIN[case, R], (case, R, how))


def test_runs_on_two_workers_resume_like_runs_in_process(stub_tree, monkeypatch, capsys):
    uninstall = _install('er_random')
    try:
        want = _experiment('er_random', 1, 'plain', '', monkeypatch, capsys)
        d = str(stub_tree / 'ck')
        monkeypatch.setenv('CHECKPOINT_FAIL_STEP', '2,1,2')
        with pytest.raises(RuntimeError, match='injected failure'):
            _experiment('er_random', 1, 'resumed', d, monkeypatch, capsys, devices=(0, 0))
        monkeypatch.delenv('CHECKPOINT_FAIL_STEP')
        assert 'run2.snapshot' in os.listdir(os.path.join(d, 'runs'))
        got = _experiment('er_random', 1, 'resumed', d, monkeypatch, capsys, devices=(0, 0))
    finally:
        uninstall()
    _same(got, want, 'workers 0,0')
    assert multiprocessing.active_children() == []


def test_tuning_resumed_in_its_tuning_stage_chooses_the_same_points(stub_tree, monkeypatch, capsys):
    """test_gpu_multidevice.py's tuning (2 x 2 grid, num_runs_val 2, two runs, num_val 2), interrupted at task 1 of
    tuning training 5, then started again."""
    def tune(name, d):
        params = md._params('er_random')
        vars(params).update(data='cifar100', num_runs=2, seed=3, num_val=2, num_runs_val=2, train_val=False,
                            stub_data='tune', weight_decay=0.0)
        multirun.multiple_run_tune_separate(params, md.TUNE_GRID, name, n_concurrent=1, checkpoint_dir=d)
        capsys.readouterr()
        with open('result/cifar100/nc/' + name, 'rb') as f:
            return pickle.load(f), vars(params)
    uninstall = _install('er_random')
    try:
        want, want_params = tune('plain.pkl', '')
        d = str(stub_tree / 'ck')
        tune_task = multirun._Tuning.tune_task

        def failing(self, i, t, x, y):
            if (i, t) == (5, 1):
                raise Interrupt('tuning training 5, task 1')
            return tune_task(self, i, t, x, y)
        monkeypatch.setattr(multirun._Tuning, 'tune_task', failing)
        with pytest.raises(Interrupt):
            tune('resumed.pkl', d)
        monkeypatch.setattr(multirun._Tuning, 'tune_task', tune_task)
        # trainings 0-4 ended, training 5 finished its task 0
        assert sorted(os.listdir(os.path.join(d, 'tune'))) == ['run%d.record' % i for i in range(5)] + ['run5.snapshot']
        got, got_params = tune('resumed.pkl', d)
    finally:
        uninstall()
    assert got['best_params'] == want['best_params'] and got_params == want_params
    assert np.array_equal(got['acc_array'], want['acc_array'])
    assert sorted(os.listdir(os.path.join(d, 'final'))) == ['run0.record', 'run1.record']
