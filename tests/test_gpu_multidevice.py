"""GPU: the experiment drivers on worker processes (B200OCL_RUN_DEVICES) against the in-process wrapper, on real engine
agents behind a stub reference tree written to tmp_path (spawned workers import it, and agent_cases.py, from the
sys.path they inherit).  Six runs of ER (random), ER + ASER, SCR with the review trick and GDumb (WORKER_CASES of
agent_cases.CASES) on workers 0,0 at R = 1 and R = 2 per worker: every run's accuracy arrays and final state
(agent_cases.final_state) are bit-identical to the in-process run_group at R = 1 with the same (seed, r).
main_tune.py's loop on the same 2 x 2 grid and data as test_gpu_multirun_tune.py gives the same chosen points and arrays
on workers as in process.  Workers 0,1 run only with two devices."""
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

pytestmark = pytest.mark.gpu

SEED, N_RUNS = 11, 6
WORKER_CASES = ('er_random', 'er_aser', 'scr_review', 'gdumb')
TUNE_GRID = {'learning_rate': [0.05, 0.1], 'weight_decay': [0.0, 1e-3]}

STUB_TREE = {
    'continuum/__init__.py': '',
    'continuum/continuum.py': '''
        import numpy as np
        import torch

        LAST_RUN = [None]          # the run of the last new_run(): an agent built next belongs to it


        def _runs_data(r):
            """test_gpu_multirun.py's tasks: three tasks of two classes, 30 images each, two test loaders per task."""
            rs = np.random.RandomState(1000 + r)
            tasks, loaders = [], []
            for t in range(3):
                labels = np.array([2 * t, 2 * t + 1])
                tasks.append((rs.randint(0, 256, (30, 32, 32, 3)).astype(np.uint8), labels[rs.permutation(30) % 2]))
                x = torch.from_numpy(rs.rand(40, 3, 32, 32).astype(np.float32))
                loaders.append([(x[:25], torch.from_numpy(labels[np.arange(25) % 2])),
                                (x[25:], torch.from_numpy(labels[np.arange(15) % 2]))])
            return tasks, loaders


        def _tune_data(r):
            """test_gpu_multirun_tune.py's tasks: three tasks of five of the 100 classes."""
            rs = np.random.RandomState(2000 + r)
            tasks, loaders = [], []
            for t in range(3):
                labels = np.arange(5 * t, 5 * (t + 1))
                tasks.append((rs.randint(0, 256, (30, 32, 32, 3)).astype(np.uint8), labels[rs.permutation(30) % 5]))
                x = torch.from_numpy(rs.rand(40, 3, 32, 32).astype(np.float32))
                loaders.append([(x[:25], torch.from_numpy(labels[np.arange(25) % 5])),
                                (x[25:], torch.from_numpy(labels[np.arange(15) % 5]))])
            return tasks, loaders


        class DataObject(object):
            task_nums = 3


        class continuum(object):
            def __init__(self, data, scenario, params):
                self.data_object = DataObject()
                self.cur_run, self.cur_task = -1, 0
                self.make = _tune_data if params.stub_data == 'tune' else _runs_data

            def new_run(self):
                self.cur_run += 1
                self.cur_task = 0
                LAST_RUN[0] = self.cur_run
                self.tasks, self.loaders = self.make(self.cur_run)

            def __iter__(self):
                return self

            def __next__(self):
                if self.cur_task == len(self.tasks):
                    raise StopIteration
                x, y = self.tasks[self.cur_task]
                self.cur_task += 1
                return x, y, set(y.tolist())

            def test_data(self):
                return self.loaders
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


        def check_ram_usage():
            return 0.0
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
        import os

        import torch
        from agent_cases import final_state
        from b200ocl import registry

        from continuum.continuum import LAST_RUN


        _recording = {}


        def recording(cls):
            """cls, saving its run's state to $MULTIDEVICE_OUT/run<r>.pt after every evaluation."""
            if cls not in _recording:
                class Recording(cls):
                    def __init__(self, model, opt, params):
                        super().__init__(model, opt, params)
                        self.stub_run = LAST_RUN[0]

                    def evaluate(self, loaders):
                        acc = super().evaluate(loaders)
                        out = os.environ.get('MULTIDEVICE_OUT')
                        if out:
                            torch.save(final_state(self), os.path.join(out, 'run%d.pt' % self.stub_run))
                        return acc
                _recording[cls] = Recording
            return _recording[cls]


        class Agents(dict):
            """install() puts the engine's classes in; a lookup hands out their recording subclass."""
            def __getitem__(self, key):
                return recording(dict.__getitem__(self, key))


        agents = Agents(registry.agents)
        retrieve_methods = {}
        update_methods = {}
    ''',
}
PACKAGES = ('continuum', 'experiment', 'utils')


@pytest.fixture
def stub_tree(monkeypatch, tmp_path):
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    ref = tmp_path / 'reference'
    for rel, src in STUB_TREE.items():
        (ref / rel).parent.mkdir(parents=True, exist_ok=True)
        (ref / rel).write_text(textwrap.dedent(src))
    saved = {k: v for k, v in sys.modules.items() if k.split('.')[0] in PACKAGES}
    for k in saved:
        del sys.modules[k]
    monkeypatch.syspath_prepend(str(ref))
    monkeypatch.chdir(tmp_path)
    for k in (multirun.ENV, multirun.DEVICES_ENV):
        monkeypatch.delenv(k, raising=False)
    yield tmp_path
    for k in [k for k in sys.modules if k.split('.')[0] in PACKAGES]:
        del sys.modules[k]
    sys.modules.update(saved)
    assert multiprocessing.active_children() == []


def _params(case):
    """agent_cases.params(case) with the fields of a multiple_run experiment on the stub tree."""
    p = agent_cases.params(case)
    vars(p).update(cl_type='nc', num_runs=N_RUNS, seed=SEED, online=True, model_name='M', data_name='D',
                   stub_data='runs')
    return p


def _experiment(case, devices, R, out, monkeypatch):
    """One multiple_run; returns its acc_array and every run's final state."""
    out.mkdir()
    monkeypatch.setenv('MULTIDEVICE_OUT', str(out))
    multirun.multiple_run(_params(case), store=True, save_path='%s.pkl' % out.name, n_concurrent=R, devices=devices)
    torch.cuda.synchronize()
    with open('result/cifar10/%s.pkl' % out.name, 'rb') as f:
        acc = pickle.load(f)['acc_array']
    return acc, [torch.load(str(out / ('run%d.pt' % r))) for r in range(N_RUNS)]


_SOLO = {}


def _check(case, devices, R, tmp_path, monkeypatch):
    from b200ocl import registry
    import utils.name_match as nm
    registry.install(nm, extra=agent_cases.extra(case))
    try:
        if case not in _SOLO:
            _SOLO[case] = _experiment(case, (), 1, tmp_path / 'solo', monkeypatch)
        acc, states = _experiment(case, devices, R, tmp_path / 'workers', monkeypatch)
    finally:
        registry.uninstall(nm)
    want_acc, want_states = _SOLO[case]
    assert acc.shape == (N_RUNS, 3, 3) and np.array_equal(acc, want_acc), (case, acc, want_acc)
    for r in range(N_RUNS):
        assert len(states[r]) == len(want_states[r])
        for i, (x, y) in enumerate(zip(states[r], want_states[r])):
            assert torch.equal(x, y), (case, devices, R, r, i)
    assert not torch.equal(states[0][0], states[1][0])                           # the runs differ
    assert multiprocessing.active_children() == []


@pytest.mark.parametrize('R', [1, 2])
@pytest.mark.parametrize('case', sorted(WORKER_CASES))
def test_runs_on_two_workers_match_in_process_runs_bit_for_bit(case, R, stub_tree, monkeypatch, capsys):
    _check(case, (0, 0), R, stub_tree, monkeypatch)


def test_runs_on_two_devices_match_in_process_runs_bit_for_bit(stub_tree, monkeypatch, capsys):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two CUDA devices')
    _check('er_random', (0, 1), 1, stub_tree, monkeypatch)


def test_tuning_on_two_workers_matches_in_process_tuning(stub_tree, monkeypatch, capsys):
    """test_gpu_multirun_tune.py's ER (random) tuning: 2 x 2 grid, num_runs_val 2, two runs, num_val 2."""
    from b200ocl import registry
    import utils.name_match as nm
    monkeypatch.delenv('MULTIDEVICE_OUT', raising=False)

    def tune(devices, R, name):
        params = _params('er_random')
        vars(params).update(data='cifar100', num_runs=2, seed=3, num_val=2, num_runs_val=2, train_val=False,
                            stub_data='tune', weight_decay=0.0)
        multirun.multiple_run_tune_separate(params, TUNE_GRID, name, n_concurrent=R, devices=devices)
        with open('result/cifar100/nc/' + name, 'rb') as f:
            return pickle.load(f), vars(params)
    registry.install(nm)
    try:
        solo, solo_params = tune((), 1, 'solo.pkl')
        pooled, pooled_params = tune((0, 0), 2, 'workers.pkl')
    finally:
        registry.uninstall(nm)
    assert solo['acc_array'].shape == (2, 1, 1)
    assert np.array_equal(pooled['acc_array'], solo['acc_array'])
    assert pooled['best_params'] == solo['best_params'] and pooled_params == solo_params
    assert multiprocessing.active_children() == []
