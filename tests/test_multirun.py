"""CPU: the concurrent-runs driver (multirun.run_group / multiple_run) with stub agents: the fixed round-robin order,
one random state per run whatever the group, state swaps that leave other runs alone, the B200OCL_CONCURRENT_RUNS
switch and its refusals, and the reference's stdout lines and --store pickle from the wrapper."""
import os
import pickle
import random
import sys
import types

import numpy as np
import pytest
import torch

from b200ocl import memory, multirun


class StubAgent(object):
    """_steps draws from Python random, numpy and torch's CPU generator (and the CUDA generator when there is one) at
    every step; evaluate draws too.  Every event goes to the shared log."""

    def __init__(self, r, log):
        self.r, self.log = r, log
        self.init = (random.random(), float(np.random.rand()), float(torch.rand(1)))
        self.draws = []

    def _steps(self, x, y):
        for i in range(len(x)):
            d = (random.random(), float(np.random.rand()), float(torch.rand(1)), int(torch.randperm(7)[0]))
            if torch.cuda.is_available():
                d += (float(torch.rand(1, device='cuda')),)
            self.draws.append(d)
            self.log.append(('step', self.r, i))
            yield

    def evaluate(self, loaders):
        self.log.append(('eval', self.r))
        return np.array([np.random.rand() for _ in loaders])


def _tasks(n_steps_per_task):
    return [(np.zeros(n), np.zeros(n)) for n in n_steps_per_task]


def _run(runs, R, steps, first_run=0, seed=7):
    log, agents = [], {}

    def make_agent(r):
        agents[r] = StubAgent(r, log)
        return agents[r]
    tasks = [_tasks(steps(r)) for r in range(first_run, first_run + runs)]
    acc = multirun.run_group(tasks, [[None, None]] * runs, make_agent, R, seed=seed, first_run=first_run)
    return log, agents, acc


def test_round_robin_order_is_fixed():
    log, _, acc = _run(3, 3, lambda r: [2 + r, 1])
    # task 0: runs 0,1,2 step in turn; run 0 stops after 2 steps, run 1 after 3; then all evaluate in run order
    assert log == [('step', 0, 0), ('step', 1, 0), ('step', 2, 0),
                   ('step', 0, 1), ('step', 1, 1), ('step', 2, 1),
                   ('step', 1, 2), ('step', 2, 2),
                   ('step', 2, 3),
                   ('eval', 0), ('eval', 1), ('eval', 2),
                   ('step', 0, 0), ('step', 1, 0), ('step', 2, 0),
                   ('eval', 0), ('eval', 1), ('eval', 2)]
    assert [a.shape for a in acc] == [(2, 2)] * 3
    log2, _, _ = _run(3, 3, lambda r: [2 + r, 1])
    assert log2 == log
    # groups of 2: runs 0 and 1 finish before run 2 starts
    log3, _, acc3 = _run(3, 2, lambda r: [1, 1])
    assert [e for e in log3 if e[0] == 'step'][:4] == [('step', 0, 0), ('step', 1, 0), ('step', 0, 0), ('step', 1, 0)]
    assert len(acc3) == 3


@pytest.mark.parametrize('first_run', [5, 4, 3])
def test_a_run_draws_the_same_numbers_alone_or_in_a_group(first_run):
    """Run 5 alone and at position 0, 1 or 2 of a group of three: the same draws at construction, at every step and
    in evaluation."""
    steps = lambda r: [3, 2 + r % 2]                                                # noqa: E731
    _, solo, acc_solo = _run(1, 1, steps, first_run=5)
    _, grouped, acc_grp = _run(3, 3, steps, first_run=first_run)
    assert grouped[5].init == solo[5].init
    assert grouped[5].draws == solo[5].draws
    assert np.array_equal(acc_grp[5 - first_run], acc_solo[0])
    # R does not matter either
    _, seq, acc_seq = _run(3, 1, steps, first_run=first_run)
    assert seq[5].draws == solo[5].draws and np.array_equal(acc_seq[5 - first_run], acc_solo[0])
    # different runs draw differently
    other = [r for r in grouped if r != 5][0]
    assert grouped[other].draws != grouped[5].draws


def test_the_driver_restores_the_callers_state():
    random.seed(1), np.random.seed(1), torch.manual_seed(1)
    before = (random.getstate(), np.random.get_state()[1].copy(), torch.get_rng_state().clone())
    _run(2, 2, lambda r: [2])
    assert random.getstate() == before[0]
    assert np.array_equal(np.random.get_state()[1], before[1])
    assert torch.equal(torch.get_rng_state(), before[2])


def test_swapping_one_runs_states_leaves_the_others_unchanged():
    a, b = multirun.RunRng(multirun.run_seed(0, 0)), multirun.RunRng(multirun.run_seed(0, 1))
    snap = lambda s: (s.py, s.np[1].copy(), s.cpu.clone())                          # noqa: E731
    b0 = snap(b)
    a0 = snap(a)
    a.swap_in()
    x = (random.random(), np.random.rand(), float(torch.rand(1)))
    a.save()
    b1 = snap(b)
    assert b1[0] == b0[0] and np.array_equal(b1[1], b0[1]) and torch.equal(b1[2], b0[2])
    assert snap(a)[0] != a0[0] and not torch.equal(snap(a)[2], a0[2])
    # a run resumes where it stopped
    b.swap_in()
    random.random()
    b.save()
    a.swap_in()
    y = (random.random(), np.random.rand(), float(torch.rand(1)))
    a.save()
    r = multirun.RunRng(multirun.run_seed(0, 0))
    r.swap_in()
    ref = [(random.random(), np.random.rand(), float(torch.rand(1))) for _ in range(2)]
    assert [x, y] == ref


def test_host_state_is_per_run():
    """The class-level sampler state and the queued host-mirror updates travel with their run."""
    CB = memory.ClassBalancedRandomSampling
    CB.reset()
    s0, s1 = memory.RunHostState(), memory.RunHostState()
    s0.enter()
    CB.update_cache(np.zeros(4), 3, new_y=np.array([0, 1, 1, 2]), ind=np.arange(4))
    hits = []
    memory.defer(lambda: hits.append(0))
    s0.leave()
    assert CB.labels_host is None and not memory._pending
    s1.enter()
    assert CB.class_num_cache is None
    CB.update_cache(np.zeros(2), 2, new_y=np.array([1, 1]), ind=np.arange(2))      # flushes nothing of run 0
    assert hits == [] and CB.class_num_cache.tolist() == [0, 2]
    s1.leave()
    s0.enter()
    assert CB.class_num_cache.tolist() == [1, 2, 1]
    memory.flush_pending()
    assert hits == [0]
    s0.leave()
    CB.reset()


def test_run_seed_rule():
    assert multirun.run_seed(0, 0) == int(np.random.SeedSequence([0, 0]).generate_state(1, np.uint32)[0])
    assert len({multirun.run_seed(s, r) for s in range(4) for r in range(16)}) == 64
    with pytest.raises(ValueError):
        multirun.run_seed(-1, 0)


@pytest.mark.parametrize('raw,want', [(None, 1), ('', 1), ('1', 1), ('3', 3), (' 8 ', 8)])
def test_env_parsing(raw, want):
    env = {} if raw is None else {multirun.ENV: raw}
    assert multirun.concurrent_runs(env) == want


@pytest.mark.parametrize('raw', ['0', '-2', 'two', '2.5', '1e3'])
def test_env_parsing_rejects(raw):
    with pytest.raises(ValueError):
        multirun.concurrent_runs({multirun.ENV: raw})


def _never(r):
    raise AssertionError('nothing may be built')


def test_parity_mode_is_refused_before_anything_is_built():
    memory.set_mode(True)
    try:
        with pytest.raises(ValueError, match='parity'):
            multirun.run_group([_tasks([1])] * 2, [[None]] * 2, _never, 2)
        multirun.run_group([], [], _never, 1)                                       # R = 1 is allowed
    finally:
        memory.set_mode(False)


def test_data_parallel_sync_is_refused_before_anything_is_built(monkeypatch):
    with pytest.raises(ValueError, match='data-parallel'):
        multirun.check_concurrent(2, grad_sync=True)
    monkeypatch.setattr(multirun, '_data_parallel', lambda: True)
    with pytest.raises(ValueError, match='data-parallel'):
        multirun.run_group([_tasks([1])] * 2, [[None]] * 2, _never, 2)


def test_an_agent_with_gradient_sync_is_refused():
    def make(r):
        a = StubAgent(r, [])
        a.grad_sync = lambda eng: None
        return a
    with pytest.raises(ValueError, match='gradient sync'):
        multirun.run_group([_tasks([1])] * 2, [[None]] * 2, make, 2)


# --------------------------------------------------------------------------- the reference wrapper
N_TASKS, N_RUNS = 3, 5


def _stub_reference(log):
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        return m

    class Continuum(object):
        def __init__(self, data, scenario, params):
            self.cur_run, self.cur_task = -1, 0

        def new_run(self):
            self.cur_run += 1
            self.cur_task = 0
            self.order = np.random.permutation(N_TASKS)

        def __iter__(self):
            return self

        def __next__(self):
            if self.cur_task == N_TASKS:
                raise StopIteration
            self.cur_task += 1
            n = 2 + int(self.order[self.cur_task - 1])
            return np.zeros((n, 4, 4, 3), np.uint8), np.full(n, self.cur_run), None

        def test_data(self):
            return [(None, None)] * N_TASKS

    class Agent(StubAgent):
        def __init__(self, model, opt, params):
            super().__init__(model, log)

    def compute_performance(a):
        log.append(('perf', a.shape))
        return 0.5, 0.25, 0.125, 0.0625, 0.03125

    nm = mod('utils.name_match', agents={'ER': Agent}, retrieve_methods={}, update_methods={})
    return {'continuum': mod('continuum'), 'continuum.continuum': mod('continuum.continuum', continuum=Continuum),
            'continuum.data_utils': mod('continuum.data_utils', setup_test_loader=lambda data, params: list(data)),
            'experiment': mod('experiment'),
            'experiment.metrics': mod('experiment.metrics', compute_performance=compute_performance),
            'experiment.run': mod('experiment.run', agents=nm.agents, multiple_run=object()),
            'utils': mod('utils'), 'utils.name_match': nm,
            'utils.io': mod('utils.io', load_yaml=lambda path, key=None: {'result': 'result/'}),
            'utils.setup_elements': mod('utils.setup_elements',
                                        setup_architecture=lambda params: len(log),
                                        setup_opt=lambda *a: None),
            'utils.utils': mod('utils.utils', maybe_cuda=lambda m, cuda: m)}


@pytest.fixture
def reference(monkeypatch, tmp_path):
    log = []
    mods = _stub_reference(log)
    for k, v in mods.items():
        monkeypatch.setitem(sys.modules, k, v)
    monkeypatch.chdir(tmp_path)
    return log, mods


def _params(online=True):
    return types.SimpleNamespace(data='cifar100', cl_type='nc', num_runs=N_RUNS, seed=0, online=online, agent='ER',
                                 cuda=False, optimizer='SGD', learning_rate=0.1, weight_decay=0.0,
                                 model_name='ER', data_name='cifar100')


@pytest.mark.parametrize('R', [1, 2, 3])
def test_wrapper_prints_the_reference_lines_and_writes_its_pickle(reference, capsys, R):
    log, _ = reference
    multirun.multiple_run(_params(), store=True, n_concurrent=R)
    out = capsys.readouterr().out.splitlines()
    for r in range(N_RUNS):
        for t in range(N_TASKS):
            assert '-----------run {} training batch {}-------------'.format(r, t) in out
        assert sum(l.startswith('-----------run {}-----------avg_end_acc '.format(r)) and '-----------train time ' in l
                   for l in out) == 1
    assert out[0] == 'Setting up data stream' and out[1].startswith('data setup time: ')
    assert out[2] == 'result/cifar100'
    assert out[-2].startswith('----------- Total {} run: '.format(N_RUNS))
    assert out[-1] == ('----------- Avg_End_Acc 0.5 Avg_End_Fgt 0.25 Avg_Acc 0.125 Avg_Bwtp 0.0625 '
                       'Avg_Fwt 0.03125-----------')
    assert sum(l.startswith('size: ') for l in out) == N_RUNS * N_TASKS
    with open('result/cifar100/ER_cifar100.pkl', 'rb') as f:
        res = pickle.load(f)
    assert sorted(res) == ['acc_array', 'time'] and res['acc_array'].shape == (N_RUNS, N_TASKS, N_TASKS)
    assert ('perf', (N_RUNS, N_TASKS, N_TASKS)) in log
    # the numbers do not depend on R
    if R == 1:
        test_wrapper_prints_the_reference_lines_and_writes_its_pickle.acc = res['acc_array']
    else:
        assert np.array_equal(res['acc_array'], test_wrapper_prints_the_reference_lines_and_writes_its_pickle.acc)


def test_wrapper_offline_mode(reference, capsys):
    multirun.multiple_run(_params(online=False), store=True, save_path='off.pkl', n_concurrent=2)
    out = capsys.readouterr().out.splitlines()
    for r in range(N_RUNS):
        assert '----------run {} training-------------'.format(r) in out
    assert out.count('Training Start') == N_RUNS
    assert out[-1].startswith('avg_end_acc ')
    with open('result/cifar100/off.pkl', 'rb') as f:
        res = pickle.load(f)
    assert res['acc_array'].shape == (N_RUNS, N_TASKS)


def test_install_replaces_multiple_run_only_when_asked(reference, monkeypatch):
    from b200ocl import registry
    _, mods = reference
    run = mods['experiment.run']
    original = run.multiple_run
    monkeypatch.delenv(multirun.ENV, raising=False)
    registry.install(mods['utils.name_match'])
    assert run.multiple_run is original
    registry.uninstall(mods['utils.name_match'])
    monkeypatch.setenv(multirun.ENV, '1')
    registry.install(mods['utils.name_match'])
    assert run.multiple_run is original
    registry.uninstall(mods['utils.name_match'])
    monkeypatch.setenv(multirun.ENV, '4')
    registry.install(mods['utils.name_match'])
    assert run.multiple_run is multirun.multiple_run
    registry.uninstall(mods['utils.name_match'])
    assert run.multiple_run is original
    er = mods['utils.name_match'].agents['ER']
    for bad in ('0', 'x'):
        monkeypatch.setenv(multirun.ENV, bad)
        with pytest.raises(ValueError):
            registry.install(mods['utils.name_match'])
        assert run.multiple_run is original and mods['utils.name_match'].agents['ER'] is er
    monkeypatch.setenv(multirun.ENV, '2')
    memory.set_mode(True)
    try:
        with pytest.raises(ValueError, match='parity'):
            registry.install(mods['utils.name_match'])
        assert run.multiple_run is original and mods['utils.name_match'].agents['ER'] is er
    finally:
        memory.set_mode(False)
