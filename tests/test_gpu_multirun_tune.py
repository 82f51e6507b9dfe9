"""GPU: main_tune.py's loop through the concurrent wrapper (multirun.multiple_run_tune_separate) on real engine agents,
with a stub reference around them (synthetic CIFAR-100-shaped tasks, the same as test_gpu_multirun.py's but with 100
classes).  A 2 x 2 grid (learning_rate, weight_decay), num_runs_val = 2, two runs, ER with random retrieval and ER with
ASER retrieve / update.  Every tuning training's accuracy arrays and final state (parameter arena, BN statistics, memory)
are bit-identical at R = 1 and R = 4, and bit-identical to a solo train_learner / evaluate loop seeded with that
training's tune_seed; each run's final agent is built with the point of best mean end accuracy."""
import gc
import pickle
import sys
import types
import weakref

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SEED, N_RUNS, N_VAL_RUNS, NUM_VAL = 3, 2, 2, 2
N_TASKS, PER_TASK, N_TEST, CLS_PER_TASK = 3, 30, 40, 5
GRID = {'learning_rate': [0.05, 0.1], 'weight_decay': [0.0, 1e-3]}
CASES = {'er_random': dict(), 'er_aser': dict(update='ASER', retrieve='ASER')}


def _params(case):
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick',
                                'kd_trick_star')}
    base = dict(data='cifar100', cl_type='nc', cuda=True, epoch=1, batch=10, verbose=False, mem_size=20,
                eps_mem_batch=10, mem_iters=1, update='random', retrieve='random', agent='ER', k=3, aser_type='asvm',
                n_smp_cls=1.5, num_tasks=N_TASKS, buffer_tracker=False, optimizer='SGD', learning_rate=0.1,
                weight_decay=0.0, temp=0.07, head='mlp', subsample=20, error_analysis=False, test_batch=128,
                trick=trick, num_runs=N_RUNS, seed=SEED, num_val=NUM_VAL, num_runs_val=N_VAL_RUNS, online=True,
                train_val=False, model_name='ER', data_name='cifar100')
    base.update(CASES[case])
    return types.SimpleNamespace(**base)


def _data(r):
    """Run r's tasks (five of the 100 classes each) and test loaders, from a generator of its own."""
    rs = np.random.RandomState(2000 + r)
    tasks, loaders = [], []
    for t in range(N_TASKS):
        labels = np.arange(CLS_PER_TASK * t, CLS_PER_TASK * (t + 1))
        tasks.append((rs.randint(0, 256, (PER_TASK, 32, 32, 3)).astype(np.uint8),
                      labels[rs.permutation(PER_TASK) % CLS_PER_TASK]))
        x = torch.from_numpy(rs.rand(N_TEST, 3, 32, 32).astype(np.float32))
        loaders.append([(x[:25], torch.from_numpy(labels[np.arange(25) % CLS_PER_TASK])),
                        (x[25:], torch.from_numpy(labels[np.arange(15) % CLS_PER_TASK]))])
    return tasks, loaders


def _final(agent):
    eng = agent.engine
    out = [eng.state.params, eng.state.bn_stats, eng.state.bn_tracked, agent.buffer.buffer_img,
           agent.buffer.buffer_label]
    return [t.detach().clone() for t in out]


def _build(params):
    from b200ocl import nets, registry
    model = nets.setup_architecture(params)
    opt = torch.optim.SGD(model.parameters(), lr=params.learning_rate, weight_decay=params.weight_decay)
    return registry.agents[params.agent](model, opt, params)


def _stub_reference(records, live):
    from b200ocl import nets, registry

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
            self.tasks, self.loaders = _data(self.cur_run)

        def reset_run(self):
            self.cur_task = 0

        def __iter__(self):
            return self

        def __next__(self):
            if self.cur_task == N_TASKS:
                raise StopIteration
            x, y = self.tasks[self.cur_task]
            self.cur_task += 1
            return x, y, set(y.tolist())

        def test_data(self):
            return self.loaders

    class Recording(registry.agents['ER']):
        """Records the params it was built with, its accuracies and its state after every evaluation."""

        def __init__(self, model, opt, params):
            super().__init__(model, opt, params)
            self.rec = {'lr': params.learning_rate, 'wd': params.weight_decay, 'acc': [], 'final': None}
            records.append(self.rec)
            live.append(weakref.ref(self))

        def evaluate(self, loaders):
            acc = super().evaluate(loaders)
            self.rec['acc'].append(acc)
            self.rec['final'] = _final(self)
            return acc

    def compute_performance(a):
        end = a[:, -1, :].mean(axis=1)
        return (end.mean(), 0.0), (0.0, 0.0), (0.0, 0.0), (0.0, 0.0), (0.0, 0.0)

    def setup_opt(optimizer, model, lr, wd):
        return torch.optim.SGD(model.parameters(), lr=lr, weight_decay=wd)

    nm = mod('utils.name_match', agents={'ER': Recording}, retrieve_methods={}, update_methods={})
    return {'continuum': mod('continuum'), 'continuum.continuum': mod('continuum.continuum', continuum=Continuum),
            'continuum.data_utils': mod('continuum.data_utils', setup_test_loader=lambda data, params: list(data)),
            'experiment': mod('experiment'),
            'experiment.metrics': mod('experiment.metrics', compute_performance=compute_performance),
            'experiment.run': mod('experiment.run', multiple_run=object(), multiple_run_tune_separate=object()),
            'utils': mod('utils'), 'utils.name_match': nm,
            'utils.io': mod('utils.io', load_yaml=lambda path, key=None: {'result': 'result/'},
                            check_ram_usage=lambda: 0.0),
            'utils.setup_elements': mod('utils.setup_elements', setup_architecture=nets.setup_architecture,
                                        setup_opt=setup_opt),
            'utils.utils': mod('utils.utils', maybe_cuda=lambda m, cuda: m)}


def _tune(case, R, monkeypatch, tmp_path):
    from b200ocl import multirun
    records, live = [], []
    for k, v in _stub_reference(records, live).items():
        monkeypatch.setitem(sys.modules, k, v)
    monkeypatch.chdir(tmp_path)
    multirun.multiple_run_tune_separate(_params(case), GRID, 'R%d.pkl' % R, n_concurrent=R)
    torch.cuda.synchronize()
    with open('result/cifar100/nc/R%d.pkl' % R, 'rb') as f:
        res = pickle.load(f)
    gc.collect()
    assert all(w() is None for w in live), 'an agent outlived its training'
    return records, res


def _same(a, b, what):
    assert len(a['acc']) == len(b['acc']), what
    for x, y in zip(a['acc'], b['acc']):
        assert np.array_equal(x, y), (what, x, y)
    for i, (x, y) in enumerate(zip(a['final'], b['final'])):
        assert torch.equal(x, y), (what, i)


@pytest.mark.parametrize('case', sorted(CASES))
def test_tuning_trainings_match_across_R_and_solo_loops(case, monkeypatch, tmp_path):
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import memory, multirun
    grid = multirun.param_grid(GRID)
    entries = [(r, g, v) for r in range(N_RUNS) for g in range(len(grid)) for v in range(N_VAL_RUNS)]
    rec1, res1 = _tune(case, 1, monkeypatch, tmp_path)
    rec4, res4 = _tune(case, 4, monkeypatch, tmp_path)
    assert len(rec1) == len(rec4) == len(entries) + N_RUNS
    for i, e in enumerate(entries + [('final', r) for r in range(N_RUNS)]):
        _same(rec1[i], rec4[i], (case, e))
    assert np.array_equal(res1['acc_array'], res4['acc_array']) and res1['best_params'] == res4['best_params']
    assert res1['acc_array'].shape == (N_RUNS, N_TASKS - NUM_VAL, N_TASKS - NUM_VAL)

    # each training alone: train_learner / evaluate from its own seed on the default stream
    for i, (r, g, v) in enumerate(entries):
        assert (rec1[i]['lr'], rec1[i]['wd']) == (grid[g]['learning_rate'], grid[g]['weight_decay'])
        memory.flush_pending()
        multirun.RunRng(multirun.tune_seed(SEED, r, g, v)).swap_in()
        params = _params(case)
        vars(params).update(grid[g])
        agent = _build(params)
        tasks, loaders = _data(r)
        acc = []
        for x, y in tasks[:NUM_VAL]:
            agent.train_learner(x, y)
            acc.append(agent.evaluate(loaders[:NUM_VAL]))
        torch.cuda.synchronize()
        _same(rec1[i], {'acc': acc, 'final': _final(agent)}, (case, r, g, v, 'solo'))
        del agent

    # the chosen point: the best mean end accuracy over the repetitions, the earliest on a tie
    for r in range(N_RUNS):
        means = [np.mean([np.mean(rec1[entries.index((r, g, v))]['acc'][-1]) for v in range(N_VAL_RUNS)])
                 for g in range(len(grid))]
        best = grid[means.index(max(means))]
        assert res1['best_params'][r] == best
        final = rec1[len(entries) + r]
        assert (final['lr'], final['wd']) == (best['learning_rate'], best['weight_decay'])
        assert np.array_equal(np.array(final['acc']), res1['acc_array'][r])
    # the trainings differ from each other
    assert not torch.equal(rec1[0]['final'][0], rec1[1]['final'][0])
