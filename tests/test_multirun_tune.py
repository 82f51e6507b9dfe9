"""CPU: the concurrent tuning wrapper (multirun.multiple_run_tune_separate, main_tune.py's loop) with a stub reference
and stub agents: ParameterGrid's order, the chosen point and its ties, the reference's stdout lines and pickle for the
online, offline, num_val -1 and train_val branches at R = 1, 2 and 3, each agent's params and seed, what default_params
ends holding, the install switch for the second entry point, and run_group's seeding with and without a seed list."""
import gc
import pickle
import random
import re
import sys
import types
import weakref

import numpy as np
import pytest
import torch

from b200ocl import memory, multirun

N_TASKS, N_RUNS, N_VAL_RUNS = 4, 3, 2
GRID = {'weight_decay': [0.0, 0.5], 'learning_rate': [0.1, 0.01]}


def _score(params):
    """An agent's accuracy before noise: it depends on the grid point."""
    return 1.0 - params.weight_decay + (0.2 if params.learning_rate == 0.01 else 0.0)


class _Ref(object):
    """What the stub reference records: every agent built (its params and first draw), the live agents, the task shapes
    of every run."""

    def __init__(self):
        self.built, self.live, self.shapes, self.max_live = [], [], [], 0
        self.score = _score


def _stub_reference(ref, tune_entry=True):
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        return m

    class DataObject(object):
        task_nums = N_TASKS

    class Continuum(object):
        def __init__(self, data, scenario, params):
            self.data_object = DataObject()
            self.cur_run, self.cur_task = -1, 0

        def new_run(self):
            self.cur_run += 1
            self.cur_task = 0
            self.sizes = 2 + np.random.permutation(N_TASKS)
            ref.shapes.append([])

        def reset_run(self):
            self.cur_task = 0

        def __iter__(self):
            return self

        def __next__(self):
            if self.cur_task == N_TASKS:
                raise StopIteration
            n = int(self.sizes[self.cur_task])
            self.cur_task += 1
            ref.shapes[-1].append(n)
            return np.zeros((n, 4, 4, 3), np.uint8), np.full(n, self.cur_task), None

        def test_data(self):
            return [(None, None)] * N_TASKS

    class Agent(object):
        def __init__(self, model, opt, params):
            self.params = params
            self.first = random.random()
            ref.built.append((dict(vars(params)), self.first))
            ref.live = [w for w in ref.live if w() is not None] + [weakref.ref(self)]
            ref.max_live = max(ref.max_live, len(ref.live))

        def _steps(self, x, y):
            for _ in range(len(x)):
                np.random.rand(), torch.rand(1)
                yield

        def evaluate(self, loaders):
            return np.array([ref.score(self.params) + self.params.noise * np.random.rand() for _ in loaders])

    def compute_performance(a):
        """The reference's avg_end_acc; the other four are not read."""
        end = a[:, -1, :].mean(axis=1)
        return (end.mean(), 0.0), (0.0, 0.0), (0.0, 0.0), (0.0, 0.0), (0.0, 0.0)

    run = mod('experiment.run', multiple_run=object())
    if tune_entry:
        run.multiple_run_tune_separate = object()
    nm = mod('utils.name_match', agents={'ER': Agent}, retrieve_methods={}, update_methods={})
    return {'continuum': mod('continuum'), 'continuum.continuum': mod('continuum.continuum', continuum=Continuum),
            'continuum.data_utils': mod('continuum.data_utils', setup_test_loader=lambda data, params: list(data)),
            'experiment': mod('experiment'),
            'experiment.metrics': mod('experiment.metrics', compute_performance=compute_performance),
            'experiment.run': run, 'utils': mod('utils'), 'utils.name_match': nm,
            'utils.io': mod('utils.io', load_yaml=lambda path, key=None: {'result': 'result/', 'tables': 'tables/'},
                            check_ram_usage=lambda: 123.5),
            'utils.setup_elements': mod('utils.setup_elements', setup_architecture=lambda params: None,
                                        setup_opt=lambda *a: None),
            'utils.utils': mod('utils.utils', maybe_cuda=lambda m, cuda: m)}


@pytest.fixture
def reference(monkeypatch, tmp_path):
    ref = _Ref()
    mods = _stub_reference(ref)
    for k, v in mods.items():
        monkeypatch.setitem(sys.modules, k, v)
    monkeypatch.chdir(tmp_path)
    return ref, mods


def _params(online=True, train_val=False, num_val=2, trick=None):
    tricks = {'labels_trick': False, 'review_trick': False}
    tricks.update(trick or {})
    return types.SimpleNamespace(data='cifar100', cl_type='nc', num_runs=N_RUNS, seed=5, online=online, agent='ER',
                                 cuda=False, optimizer='SGD', learning_rate=0.3, weight_decay=0.25, num_val=num_val,
                                 num_runs_val=N_VAL_RUNS, train_val=train_val, trick=tricks, noise=0.05,
                                 model_name='ER', data_name='cifar100')


def _call(params, R, grid=GRID):
    np.random.seed(0)
    multirun.multiple_run_tune_separate(params, grid, None, n_concurrent=R)


# --------------------------------------------------------------------------- the grid and the choice
def test_grid_order_of_er_tune():
    lrs = [0.0001, 0.0003, 0.001, 0.003, 0.01, 0.03, 0.1]
    wds = [0.0001, 0.001, 0.01, 0.1]
    grid = multirun.param_grid({'learning_rate': lrs, 'weight_decay': wds})
    assert len(grid) == 28
    assert grid[:5] == [{'learning_rate': 0.0001, 'weight_decay': 0.0001},
                        {'learning_rate': 0.0001, 'weight_decay': 0.001},
                        {'learning_rate': 0.0001, 'weight_decay': 0.01},
                        {'learning_rate': 0.0001, 'weight_decay': 0.1},
                        {'learning_rate': 0.0003, 'weight_decay': 0.0001}]
    assert grid == [{'learning_rate': lr, 'weight_decay': wd} for lr in lrs for wd in wds]
    assert [list(p) for p in grid] == [['learning_rate', 'weight_decay']] * 28


def test_grid_order_of_aser_tune():
    grid = multirun.param_grid({'learning_rate': [0.01, 0.1], 'k': [3, 5, 7], 'n_smp_cls': [2.0, 5.0, 7.0]})
    want = [(3, 0.01, 2.0), (3, 0.01, 5.0), (3, 0.01, 7.0), (3, 0.1, 2.0), (3, 0.1, 5.0), (3, 0.1, 7.0),
            (5, 0.01, 2.0), (5, 0.01, 5.0), (5, 0.01, 7.0), (5, 0.1, 2.0), (5, 0.1, 5.0), (5, 0.1, 7.0),
            (7, 0.01, 2.0), (7, 0.01, 5.0), (7, 0.01, 7.0), (7, 0.1, 2.0), (7, 0.1, 5.0), (7, 0.1, 7.0)]
    assert grid == [{'k': k, 'learning_rate': lr, 'n_smp_cls': n} for k, lr, n in want]
    assert [list(p) for p in grid] == [['k', 'learning_rate', 'n_smp_cls']] * 18


def test_grid_edge_cases():
    assert multirun.param_grid({}) == [{}]
    with pytest.raises(TypeError):
        multirun.param_grid([{'learning_rate': [0.1]}])


def test_the_chosen_point_is_the_best_and_ties_go_to_the_earliest(reference):
    ref, _ = reference
    grid = multirun.param_grid(GRID)
    # (lr 0.1, wd 0.5) and (lr 0.01, wd 0.0) tie; the first of them in grid order is index 1
    assert grid[1] == {'learning_rate': 0.1, 'weight_decay': 0.5}
    assert grid[2] == {'learning_rate': 0.01, 'weight_decay': 0.0}
    ref.score = lambda p: 1.0 if (p.learning_rate, p.weight_decay) in ((0.1, 0.5), (0.01, 0.0)) else 0.5
    params = _params()
    params.noise = 0.0
    _call(params, 2)
    with open('result/cifar100/nc/ER_cifar100_5.pkl', 'rb') as f:
        res = pickle.load(f)
    assert res['best_params'] == [grid[1]] * N_RUNS


def test_the_chosen_point_has_the_best_mean_end_accuracy(reference, capsys):
    ref, _ = reference
    params = _params()
    _call(params, 3)
    out = capsys.readouterr().out.splitlines()
    grid = multirun.param_grid(GRID)
    ends = [float(l.split('avg_end_acc ')[1].rstrip('-')) for l in out if l.startswith('-----------tune run ')
            and 'avg_end_acc' in l]
    assert len(ends) == N_RUNS * len(grid) * N_VAL_RUNS
    ends = np.array(ends).reshape(N_RUNS, len(grid), N_VAL_RUNS).mean(axis=2)
    with open('result/cifar100/nc/ER_cifar100_5.pkl', 'rb') as f:
        res = pickle.load(f)
    assert res['best_params'] == [grid[int(np.argmax(np.round(e, 12)))] for e in ends]
    assert res['best_params'][0] == {'learning_rate': 0.01, 'weight_decay': 0.0}


# --------------------------------------------------------------------------- lines, pickle, params, seeds
BRANCHES = {'online': dict(), 'offline': dict(online=False), 'train_val': dict(train_val=True),
            'offline_train_val': dict(online=False, train_val=True),
            'num_val_all': dict(num_val=-1, train_val=True),
            'offline_num_val_all': dict(online=False, num_val=-1, train_val=True)}


def _normalize(line):
    line = re.sub(r'avg_end_acc [^-]+', 'avg_end_acc A', line)
    line = re.sub(r'train time .*$', 'train time T', line)
    line = re.sub(r'data setup time: .*$', 'data setup time: T', line)
    return re.sub(r'run: .*s -----------$', 'run: Ts -----------', line)


def _expected(params, shapes, best):
    """The reference's lines, run by run in its order, with the tuning blocks of all runs first."""
    grid = multirun.param_grid(GRID)
    nv = N_TASKS if params.num_val == -1 else params.num_val
    lines = ['Setting up data stream', 'data setup time: T', 'result/cifar100/nc']
    for r in range(N_RUNS):
        tune = [(s,) for s in shapes[r][:nv]] if params.online else [(sum(shapes[r][:nv]),)]
        lines.append(str(len(grid)))
        for p in grid:
            lines.append(str(p))
            for v in range(N_VAL_RUNS):
                for t, (n,) in enumerate(tune):
                    lines += ['-----------tune run {} task {}-------------'.format(v, t),
                              'size: {}, {}'.format((n, 4, 4, 3), (n,))]
                lines.append('-----------tune run {}-----------avg_end_acc A-----------'.format(v))
    for r in range(N_RUNS):
        lines += ['Tuning is done. Best hyper parameter set is {}'.format(best[r]), 'Training Start']
        first = 0 if params.train_val else nv
        if params.online:
            for i in range(first, N_TASKS):
                lines += ['----------run {} training batch {}-------------'.format(r, i),
                          'size: {}, {}'.format((shapes[r][i], 4, 4, 3), (shapes[r][i],))]
        else:
            n = sum(shapes[r][first:])
            lines += ['----------run {} training-------------'.format(r), 'size: {}, {}'.format((n, 4, 4, 3), (n,))]
        lines.append('-----------run {}-----------avg_end_acc A-----------train time T'.format(r))
    return lines + ['----------- Total {} run: Ts -----------'.format(N_RUNS), '----------- Seed 5 RAM: 123.5s -----------']


_SEEN = {}


@pytest.mark.parametrize('R', [1, 2, 3])
@pytest.mark.parametrize('branch', sorted(BRANCHES))
def test_lines_pickle_params_and_seeds(reference, capsys, branch, R):
    ref, _ = reference
    params = _params(**BRANCHES[branch])
    original = dict(vars(params))
    _call(params, R)
    out = capsys.readouterr().out.splitlines()
    with open('result/cifar100/nc/ER_cifar100_5.pkl', 'rb') as f:
        res = pickle.load(f)
    grid = multirun.param_grid(GRID)
    nv = N_TASKS if original['num_val'] == -1 else original['num_val']

    # stdout: every line of the reference, in its order, whatever R is
    assert [_normalize(l) for l in out] == _expected(params, ref.shapes, res['best_params'])
    # the final lines carry the final accuracies
    finals = [l for l in out if l.startswith('-----------run ')]
    for r, l in enumerate(finals):
        assert l.startswith('-----------run {}-----------avg_end_acc {}-----------train time '.format(
            r, np.mean(res['acc_array'][r][-1])))

    # the pickle
    assert sorted(res) == ['acc_array', 'best_params', 'ram', 'seed', 'time']
    assert res['seed'] == 5 and res['ram'] == 123.5 and res['time'] > 0
    n_final = N_TASKS if params.train_val else N_TASKS - nv
    n_loaders = N_TASKS if params.train_val else N_TASKS - nv
    want = (N_RUNS, n_final, n_loaders) if params.online else (N_RUNS, 1, n_loaders)
    assert res['acc_array'].shape == want
    assert len(res['best_params']) == N_RUNS and all(p in grid for p in res['best_params'])

    # every agent's params and seed: the tuning trainings in (run, point, repetition) order, then the final ones
    resolved = dict(original, num_val=nv)
    entries = [(r, g, v) for r in range(N_RUNS) for g in range(len(grid)) for v in range(N_VAL_RUNS)]
    assert len(ref.built) == len(entries) + N_RUNS
    for (r, g, v), (p, first) in zip(entries, ref.built):
        assert p == dict(resolved, **grid[g]), (r, g, v)
        assert first == random.Random(multirun.tune_seed(5, r, g, v)).random(), (r, g, v)
    for r, (p, first) in enumerate(ref.built[len(entries):]):
        assert p == dict(resolved, **res['best_params'][r])
        assert first == random.Random(multirun.run_seed(5, r)).random()
    # default_params ends as the reference leaves it: num_val resolved, the last run's point on top
    assert vars(params) == dict(resolved, **res['best_params'][-1])
    # no more than R agents alive at a time, none after the call
    assert ref.max_live <= R
    gc.collect()
    assert all(w() is None for w in ref.live)

    # the numbers do not depend on R
    key = branch
    if R == 1:
        _SEEN[key] = (res['acc_array'], res['best_params'])
    elif key in _SEEN:
        assert np.array_equal(res['acc_array'], _SEEN[key][0]) and res['best_params'] == _SEEN[key][1]


def test_the_trick_names_the_result_directory(reference, capsys):
    _call(_params(trick={'review_trick': True}), 2)
    out = capsys.readouterr().out.splitlines()
    assert out[2] == 'result/cifar100/nc/review_trick'
    with open('result/cifar100/nc/review_trick/ER_cifar100_5.pkl', 'rb') as f:
        assert sorted(pickle.load(f)) == ['acc_array', 'best_params', 'ram', 'seed', 'time']


def test_save_path_and_run_list(reference, capsys):
    ref, _ = reference
    params = _params()
    params.num_runs = [4, 7]
    np.random.seed(0)
    multirun.multiple_run_tune_separate(params, GRID, 'mine.pkl', n_concurrent=2)
    out = capsys.readouterr().out.splitlines()
    assert '----------run 7 training batch 3-------------' in out
    assert out[-2].startswith('----------- Total [4, 7] run: ')
    with open('result/cifar100/nc/mine.pkl', 'rb') as f:
        res = pickle.load(f)
    assert res['acc_array'].shape == (2, 2, 2)
    assert ref.built[0][1] == random.Random(multirun.tune_seed(5, 4, 0, 0)).random()
    assert ref.built[-1][1] == random.Random(multirun.run_seed(5, 7)).random()


def test_no_task_left_for_the_final_agents_is_refused_before_anything_is_built(reference, capsys):
    ref, _ = reference
    for online in (True, False):
        with pytest.raises(ValueError, match='train_val'):
            _call(_params(online=online, num_val=-1), 2)
    assert ref.built == []


def test_refusals_come_before_anything_is_built(reference, capsys, monkeypatch):
    ref, _ = reference
    memory.set_mode(True)
    try:
        with pytest.raises(ValueError, match='parity'):
            _call(_params(), 2)
    finally:
        memory.set_mode(False)
    monkeypatch.setattr(multirun, '_data_parallel', lambda: True)
    with pytest.raises(ValueError, match='data-parallel'):
        _call(_params(), 2)
    assert ref.built == [] and ref.shapes == [] and capsys.readouterr().out == ''


# --------------------------------------------------------------------------- the switch
def test_install_replaces_the_tuning_loop_only_when_asked(reference, monkeypatch):
    from b200ocl import registry
    _, mods = reference
    run, nm = mods['experiment.run'], mods['utils.name_match']
    original, original_mr = run.multiple_run_tune_separate, run.multiple_run
    for raw in (None, '1'):
        if raw is None:
            monkeypatch.delenv(multirun.ENV, raising=False)
        else:
            monkeypatch.setenv(multirun.ENV, raw)
        registry.install(nm)
        assert run.multiple_run_tune_separate is original
        registry.uninstall(nm)
    monkeypatch.setenv(multirun.ENV, '4')
    registry.install(nm)
    assert run.multiple_run_tune_separate is multirun.multiple_run_tune_separate
    assert run.multiple_run is multirun.multiple_run
    registry.uninstall(nm)
    assert run.multiple_run_tune_separate is original and run.multiple_run is original_mr
    for bad in ('0', 'x'):
        monkeypatch.setenv(multirun.ENV, bad)
        with pytest.raises(ValueError):
            registry.install(nm)
        assert run.multiple_run_tune_separate is original
    monkeypatch.setenv(multirun.ENV, '2')
    memory.set_mode(True)
    try:
        with pytest.raises(ValueError, match='parity'):
            registry.install(nm)
        assert run.multiple_run_tune_separate is original
    finally:
        memory.set_mode(False)
    monkeypatch.setattr(multirun, '_data_parallel', lambda: True)
    with pytest.raises(ValueError, match='data-parallel'):
        registry.install(nm)
    assert run.multiple_run_tune_separate is original and run.multiple_run is original_mr


def test_an_absent_tuning_loop_stays_absent(monkeypatch, tmp_path):
    from b200ocl import registry
    mods = _stub_reference(_Ref(), tune_entry=False)
    for k, v in mods.items():
        monkeypatch.setitem(sys.modules, k, v)
    run, nm = mods['experiment.run'], mods['utils.name_match']
    monkeypatch.setenv(multirun.ENV, '3')
    registry.install(nm)
    assert run.multiple_run is multirun.multiple_run
    assert not hasattr(run, 'multiple_run_tune_separate')
    registry.uninstall(nm)
    assert not hasattr(run, 'multiple_run_tune_separate')


# --------------------------------------------------------------------------- run_group's seeds
class _Drawing(object):
    def __init__(self):
        self.init = (random.random(), float(np.random.rand()), float(torch.rand(1)))
        self.draws = []

    def _steps(self, x, y):
        for _ in range(len(x)):
            self.draws.append((random.random(), float(np.random.rand()), float(torch.rand(1))))
            yield

    def evaluate(self, loaders):
        return np.array([np.random.rand() for _ in loaders])


def _group(n, R, first_run=0, seed=7, seeds=None):
    made = {}

    def make(r):
        made[r] = _Drawing()
        return made[r]
    acc = multirun.run_group([[(np.zeros(3), None), (np.zeros(2), None)]] * n, [[None]] * n, make, R, seed=seed,
                             first_run=first_run, seeds=seeds)
    return made, acc


def test_run_group_without_seeds_keeps_the_run_seed_rule():
    made, acc = _group(3, 2, first_run=4)
    for i, r in enumerate(range(4, 7)):
        want = multirun.RunRng(multirun.run_seed(7, r))
        keep = multirun.RunRng.capture()
        want.swap_in()
        init = (random.random(), float(np.random.rand()), float(torch.rand(1)))
        keep.swap_in()
        assert made[r].init == init
    same, acc2 = _group(3, 3, first_run=4, seeds=[multirun.run_seed(7, r) for r in range(4, 7)])
    assert all(same[r].draws == made[r].draws for r in range(4, 7))
    assert all(np.array_equal(a, b) for a, b in zip(acc, acc2))


def test_run_group_with_seeds_draws_by_seed_not_by_position():
    seeds = [multirun.tune_seed(1, 0, g, 0) for g in range(3)]
    grouped, acc = _group(3, 3, seeds=seeds)
    for i in range(3):
        solo, acc_solo = _group(1, 1, first_run=i, seeds=[seeds[i]])
        assert solo[i].init == grouped[i].init and solo[i].draws == grouped[i].draws
        assert np.array_equal(acc_solo[0], acc[i])
    with pytest.raises(ValueError, match='seeds'):
        _group(3, 3, seeds=seeds[:2])


def test_tune_seed_rule():
    assert multirun.tune_seed(0, 1, 2, 3) == int(np.random.SeedSequence([0, 1, 2, 3]).generate_state(1, np.uint32)[0])
    seeds = {multirun.tune_seed(s, r, g, v) for s in range(2) for r in range(3) for g in range(4) for v in range(3)}
    assert len(seeds) == 72
    with pytest.raises(ValueError):
        multirun.tune_seed(0, 0, -1, 0)
