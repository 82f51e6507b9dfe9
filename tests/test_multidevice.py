"""CPU: B200OCL_RUN_DEVICES, the experiment drivers' worker processes (multirun.WorkerPool).  The switch's parsing and
refusals, directly and through install(); and real spawned workers running stub agents from a stub reference tree
written to tmp_path (a spawned worker imports what is on sys.path, not the sys.modules patches test_multirun.py's stubs
use).  With 1, 2 and 3 workers the accuracy arrays, the stdout lines and the pickle equal the in-process wrapper's at
R = 1, for repetitions and for main_tune.py's loop (single_tune and train_val), online and offline.  A training that
raises in a worker raises the same exception type here, naming the training, and no worker outlives a driver call."""
import multiprocessing
import os
import pickle
import re
import sys
import textwrap
from types import SimpleNamespace

import numpy as np
import pytest

from b200ocl import memory, multirun

N_RUNS = 5
GRID = {'weight_decay': [0.0, 0.5], 'learning_rate': [0.1, 0.01]}

STUB_TREE = {
    'continuum/__init__.py': '',
    'continuum/continuum.py': '''
        import numpy as np

        N_TASKS = 4
        LAST_RUN = [None]          # the run of the last new_run(): an agent built next belongs to it


        class DataObject(object):
            task_nums = N_TASKS


        class continuum(object):
            def __init__(self, data, scenario, params):
                self.data_object = DataObject()
                self.cur_run, self.cur_task = -1, 0
                self.base = int(np.random.randint(0, 3))       # the build draws too
                print('Loading data... base {}'.format(self.base))

            def new_run(self):
                self.cur_run += 1
                self.cur_task = 0
                LAST_RUN[0] = self.cur_run
                self.sizes = 2 + self.base + self.cur_run % 3 + np.random.permutation(N_TASKS)
                print('Task sizes of run {}: {}'.format(self.cur_run, self.sizes.tolist()))

            def reset_run(self):
                self.cur_task = 0

            def __iter__(self):
                return self

            def __next__(self):
                if self.cur_task == N_TASKS:
                    raise StopIteration
                n = int(self.sizes[self.cur_task])
                self.cur_task += 1
                print('Task: {}, Labels:[{}]'.format(self.cur_task - 1, self.cur_task))
                x = (np.arange(n * 48).reshape(n, 4, 4, 3) * (self.cur_run + 1) + self.cur_task) % 251
                return x.astype(np.uint8), np.full(n, self.cur_task), None

            def test_data(self):
                return [(self.cur_run, t) for t in range(N_TASKS)]
    ''',
    'continuum/data_utils.py': '''
        def setup_test_loader(data, params):
            return list(data)
    ''',
    'experiment/__init__.py': '',
    'experiment/run.py': '''
        def multiple_run(params, store=False, save_path=None):
            raise AssertionError('the reference loop ran')


        def multiple_run_tune_separate(default_params, tune_params, save_path):
            raise AssertionError('the reference loop ran')
    ''',
    'experiment/metrics.py': '''
        def compute_performance(a):
            end = a[:, -1, :].mean(axis=1)
            return (end.mean(), end.std()), (0.0, 0.0), (a.mean(), 0.0), (0.0, 0.0), (0.0, 0.0)
    ''',
    'utils/__init__.py': '',
    'utils/io.py': '''
        def load_yaml(path, key=None):
            return {'result': 'result/', 'tables': 'tables/'}


        def check_ram_usage():
            return 123.5
    ''',
    'utils/setup_elements.py': '''
        def setup_architecture(params):
            return None


        def setup_opt(*args):
            return None
    ''',
    'utils/utils.py': '''
        def maybe_cuda(model, cuda):
            return model
    ''',
    'utils/name_match.py': '''
        import random

        import numpy as np
        import torch

        from continuum.continuum import LAST_RUN


        class StubFailure(Exception):
            pass


        class Stub(object):
            """Draws from all three host generators, learns from its images, prints a line when built."""

            def __init__(self, model, opt, params):
                self.params, self.run = params, LAST_RUN[0]
                self.w = random.random() + params.learning_rate - params.weight_decay
                print('stub built: lr {} wd {}'.format(params.learning_rate, params.weight_decay))

            def _steps(self, x, y):
                for i in range(len(x)):
                    if self.params.fail_run == self.run and i == 1:
                        raise StubFailure('stub failed on purpose')
                    self.w += float(np.random.rand()) * float(torch.rand(1)) * float(x[i].mean()) / 255
                    yield

            def evaluate(self, loaders):
                return np.array([self.w + 0.01 * np.random.rand() for _ in loaders])


        agents = {'STUB': Stub}
        retrieve_methods = {}
        update_methods = {}
    ''',
}
PACKAGES = ('continuum', 'experiment', 'utils')
_REAL_CHECK_DEVICE_COUNT = multirun.check_device_count


@pytest.fixture
def stub_tree(monkeypatch, tmp_path):
    """The stub reference on sys.path (where spawned workers find it too), cwd in tmp_path, device counts unchecked."""
    ref = tmp_path / 'reference'
    for rel, src in STUB_TREE.items():
        (ref / rel).parent.mkdir(parents=True, exist_ok=True)
        (ref / rel).write_text(textwrap.dedent(src))
    saved = {k: v for k, v in sys.modules.items() if k.split('.')[0] in PACKAGES}
    for k in saved:
        del sys.modules[k]
    monkeypatch.syspath_prepend(str(ref))
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(multirun, 'check_device_count', lambda devices: None)
    for k in (multirun.ENV, multirun.DEVICES_ENV):
        monkeypatch.delenv(k, raising=False)
    yield ref
    for k in [k for k in sys.modules if k.split('.')[0] in PACKAGES]:
        del sys.modules[k]
    sys.modules.update(saved)
    assert multiprocessing.active_children() == []


def _params(**over):
    tricks = {'labels_trick': False, 'review_trick': False}
    p = dict(data='cifar100', cl_type='nc', num_runs=N_RUNS, seed=5, online=True, agent='STUB', cuda=False,
             optimizer='SGD', learning_rate=0.3, weight_decay=0.25, num_val=2, num_runs_val=2, train_val=False,
             trick=tricks, model_name='STUB', data_name='cifar100', fail_run=None)
    p.update(over)
    return SimpleNamespace(**p)


def _normalize(text):
    out = []
    for line in text.splitlines():
        line = re.sub(r'train time .*$', 'train time T', line)
        line = re.sub(r'data setup time: .*$', 'data setup time: T', line)
        out.append(re.sub(r'run: .*s -----------$', 'run: Ts -----------', line))
    return out


def _repetitions(capsys, devices, R, online):
    np.random.seed(0)
    multirun.multiple_run(_params(online=online), store=True, n_concurrent=R, devices=devices)
    after = np.random.rand()                     # the caller's random state after the call
    with open('result/cifar100/STUB_cifar100.pkl', 'rb') as f:
        res = pickle.load(f)
    return _normalize(capsys.readouterr().out), res['acc_array'], after


def _tuning(capsys, devices, R, online, train_val):
    np.random.seed(0)
    params = _params(online=online, train_val=train_val)
    multirun.multiple_run_tune_separate(params, GRID, None, n_concurrent=R, devices=devices)
    after = np.random.rand()                     # the caller's random state after the call
    with open('result/cifar100/nc/STUB_cifar100_5.pkl', 'rb') as f:
        res = pickle.load(f)
    return _normalize(capsys.readouterr().out), res['acc_array'], res['best_params'], vars(params), after


WORKERS = {1: ((0,), 1), 2: ((0, 0), 1), 3: ((0, 1, 0), 2)}       # devices, R per worker


# --------------------------------------------------------------------------- the switch
def test_run_devices_parsing():
    assert multirun.run_devices({}) == ()
    assert multirun.run_devices({multirun.DEVICES_ENV: ''}) == ()
    assert multirun.run_devices({multirun.DEVICES_ENV: '  '}) == ()
    assert multirun.run_devices({multirun.DEVICES_ENV: '0'}) == (0,)
    assert multirun.run_devices({multirun.DEVICES_ENV: '0,1,2,3'}) == (0, 1, 2, 3)
    assert multirun.run_devices({multirun.DEVICES_ENV: ' 0, 0 ,7'}) == (0, 0, 7)
    for bad, why in (('x', 'integer'), ('0,a', 'integer'), ('1.5', 'integer'), ('-1', '>= 0'), ('0,-2', '>= 0'),
                     ('0,,1', 'empty'), ('0,', 'empty'), (',0', 'empty')):
        with pytest.raises(ValueError, match=why):
            multirun.run_devices({multirun.DEVICES_ENV: bad})


def test_install_replaces_the_drivers_only_when_asked(stub_tree, monkeypatch):
    from b200ocl import registry
    import experiment.run as run
    import utils.name_match as nm
    original = run.multiple_run, run.multiple_run_tune_separate
    for raw in (None, ''):
        if raw is not None:
            monkeypatch.setenv(multirun.DEVICES_ENV, raw)
        registry.install(nm)
        assert (run.multiple_run, run.multiple_run_tune_separate) == original
        registry.uninstall(nm)
    monkeypatch.setenv(multirun.DEVICES_ENV, '0,0')
    registry.install(nm, extra=('EWC',))
    assert run.multiple_run is multirun.multiple_run
    assert run.multiple_run_tune_separate is multirun.multiple_run_tune_separate
    assert registry.installed_extra == ('EWC',)
    registry.uninstall(nm)
    assert (run.multiple_run, run.multiple_run_tune_separate) == original and registry.installed_extra == ()
    for bad in ('x', '-1', '0,,1'):
        monkeypatch.setenv(multirun.DEVICES_ENV, bad)
        with pytest.raises(ValueError, match=multirun.DEVICES_ENV):
            registry.install(nm)
        assert (run.multiple_run, run.multiple_run_tune_separate) == original
    monkeypatch.setenv(multirun.DEVICES_ENV, '0')
    memory.set_mode(True)
    try:
        with pytest.raises(ValueError, match='parity'):
            registry.install(nm)
    finally:
        memory.set_mode(False)
    monkeypatch.setattr(multirun, '_data_parallel', lambda: True)
    with pytest.raises(ValueError, match='data-parallel'):
        registry.install(nm)
    assert (run.multiple_run, run.multiple_run_tune_separate) == original


def test_the_drivers_refuse_before_starting_a_worker(stub_tree, monkeypatch, capsys):
    monkeypatch.setattr(multirun, 'check_device_count', _REAL_CHECK_DEVICE_COUNT)
    monkeypatch.setattr(multirun.torch.cuda, 'device_count', lambda: 2)
    with pytest.raises(ValueError, match='device.s. 2, 5'):
        multirun.multiple_run(_params(), devices=(0, 5, 2))
    with pytest.raises(ValueError, match='device.s. 2'):
        multirun.multiple_run_tune_separate(_params(), GRID, None, devices=(1, 2))
    memory.set_mode(True)
    try:
        with pytest.raises(ValueError, match='parity'):
            multirun.multiple_run(_params(), devices=(0,))
    finally:
        memory.set_mode(False)
    monkeypatch.setattr(multirun, '_data_parallel', lambda: True)
    with pytest.raises(ValueError, match='data-parallel'):
        multirun.multiple_run_tune_separate(_params(), GRID, None, devices=(0,))
    assert capsys.readouterr().out == '' and multiprocessing.active_children() == []


def test_a_worker_sees_one_device_and_not_the_switch(monkeypatch):
    monkeypatch.setenv(multirun.DEVICES_ENV, '3,1')
    monkeypatch.delenv('CUDA_VISIBLE_DEVICES', raising=False)
    with multirun._worker_environ(3):
        assert os.environ['CUDA_VISIBLE_DEVICES'] == '3' and multirun.DEVICES_ENV not in os.environ
    assert os.environ[multirun.DEVICES_ENV] == '3,1' and 'CUDA_VISIBLE_DEVICES' not in os.environ
    monkeypatch.setenv('CUDA_VISIBLE_DEVICES', '4, 6,GPU-abc')
    with multirun._worker_environ(2):
        assert os.environ['CUDA_VISIBLE_DEVICES'] == 'GPU-abc'
    assert os.environ['CUDA_VISIBLE_DEVICES'] == '4, 6,GPU-abc'
    with pytest.raises(ValueError, match='CUDA_VISIBLE_DEVICES'):
        with multirun._worker_environ(3):
            pass


# --------------------------------------------------------------------------- workers against the in-process wrapper
_BASE = {}


def _baseline(key, fn):
    if key not in _BASE:
        _BASE[key] = fn()
    return _BASE[key]


@pytest.mark.parametrize('online', [True, False], ids=['online', 'offline'])
@pytest.mark.parametrize('n_workers', sorted(WORKERS))
def test_repetitions_on_workers_match_the_in_process_wrapper(stub_tree, capsys, n_workers, online):
    devices, R = WORKERS[n_workers]
    want = _baseline(('rep', online), lambda: _repetitions(capsys, (), 1, online))
    got = _repetitions(capsys, devices, R, online)
    assert got[0] == want[0]
    assert np.array_equal(got[1], want[1])
    assert got[1].shape == ((N_RUNS, 4, 4) if online else (N_RUNS, 4))
    assert len(set(np.round(got[1][:, -1].ravel(), 9))) > 1                      # the runs differ
    assert sum(l.startswith('stub built') for l in got[0]) == N_RUNS
    # the continuum's build and every run's draws print once, where the in-process driver prints them
    assert sum(l.startswith('Loading data') for l in got[0]) == 1
    assert [l for l in got[0] if l.startswith('Task sizes of run')] == [
        l for l in want[0] if l.startswith('Task sizes of run')] and len(
        [l for l in got[0] if l.startswith('Task sizes of run')]) == N_RUNS
    assert got[2] == want[2]
    assert multiprocessing.active_children() == []


@pytest.mark.parametrize('train_val', [False, True], ids=['single_tune', 'train_val'])
@pytest.mark.parametrize('online', [True, False], ids=['online', 'offline'])
@pytest.mark.parametrize('n_workers', sorted(WORKERS))
def test_tuning_on_workers_matches_the_in_process_wrapper(stub_tree, capsys, n_workers, online, train_val):
    devices, R = WORKERS[n_workers]
    want = _baseline(('tune', online, train_val), lambda: _tuning(capsys, (), 1, online, train_val))
    got = _tuning(capsys, devices, R, online, train_val)
    assert got[0] == want[0]
    assert np.array_equal(got[1], want[1])
    assert got[2] == want[2] and got[3] == want[3]
    grid = multirun.param_grid(GRID)
    n_trainings = N_RUNS * (len(grid) * 2 + 1)
    assert sum(l.startswith('stub built') for l in got[0]) == n_trainings
    assert sum(l.startswith('Loading data') for l in got[0]) == 1
    assert sum(l.startswith('Task sizes of run') for l in got[0]) == N_RUNS
    assert got[4] == want[4]
    assert multiprocessing.active_children() == []


def test_a_worker_that_raises_names_the_training(stub_tree, capsys):
    import utils.name_match as nm
    for devices, R in (((0, 0), 1), ((0,), 2)):
        with pytest.raises(nm.StubFailure, match=r'run 2\b.*stub failed on purpose') as info:
            multirun.multiple_run(_params(fail_run=2), n_concurrent=R, devices=devices)
        assert any('worker traceback' in n for n in getattr(info.value, '__notes__', []))
        assert multiprocessing.active_children() == []
        out = capsys.readouterr().out
        assert '-----------run 3-----------' not in out


def test_a_worker_exits_when_its_pipe_closes(stub_tree):
    """The parent closing its end (as its death would) ends an idle worker: it sees EOF."""
    recipe = multirun._Repetitions(_params(), multirun.RunRng.capture())
    pool = multirun.WorkerPool((0,), recipe, 1)
    pool.__enter__()
    try:
        w = pool.workers[0]
        w.conn.close()
        w.proc.join(120)
        assert w.proc.exitcode == 0
    finally:
        pool.workers[0].proc.join(1)
        if pool.workers[0].proc.is_alive():
            pool.workers[0].proc.terminate()
            pool.workers[0].proc.join()
    assert multiprocessing.active_children() == []


LAUNCHED_SCRIPT = '''
import os
from types import SimpleNamespace

with open(os.environ['LAUNCH_LOG'], 'a') as f:      # the top level: run by the parent and, as __mp_main__, by workers
    f.write('%s\\n' % __name__)

if __name__ == "__main__":
    from b200ocl import multirun
    multirun.check_device_count = lambda devices: None     # the stub machine has no CUDA device
    from experiment.run import multiple_run
    multiple_run(SimpleNamespace(**PARAMS))
'''


def test_workers_through_the_launcher_run_the_experiment_once(stub_tree, tmp_path):
    """python -m b200ocl.launch <script>: the launcher makes the script __main__, so every spawned worker re-executes
    its top level as __mp_main__; its `if __name__ == "__main__"` guard keeps the experiment to the parent."""
    import subprocess
    script = stub_tree / 'general_main.py'
    script.write_text(LAUNCHED_SCRIPT.replace('PARAMS', repr(vars(_params()))))
    log = tmp_path / 'launch.log'
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, LAUNCH_LOG=str(log), PYTHONPATH=root, **{multirun.DEVICES_ENV: '0,0'})
    flags = ['-s'] if sys.flags.no_user_site else []
    out = subprocess.run([sys.executable] + flags + ['-m', 'b200ocl.launch', str(script)], env=env, cwd=str(tmp_path),
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.splitlines()
    assert lines.count('Setting up data stream') == 1
    assert sum(l.startswith('stub built') for l in lines) == N_RUNS
    ends = [re.match(r'-----------run (\d+)-----------avg_end_acc', l) for l in lines]
    assert [int(m.group(1)) for m in ends if m] == list(range(N_RUNS))
    assert sorted(log.read_text().split()) == ['__main__', '__mp_main__', '__mp_main__']


def test_a_tuning_worker_holds_only_the_runs_of_its_batch(stub_tree, capsys):
    """A worker's copy of the tuning recipe, given every third batch of both stages as one worker of three would be:
    it holds the lists of at most the runs its current batch trains, and trains them on the in-process data."""
    import io
    import time
    params = _params()
    np.random.seed(0)                                     # the caller's state on entry, which the worker replays
    recipe = multirun._Tuning(dict(vars(params)), multirun.param_grid(GRID), list(range(N_RUNS)), time.time(),
                              multirun.RunRng.capture())
    worker = pickle.loads(pickle.dumps(recipe))
    n = len(recipe.entries)
    held, accs = [], {}
    for i0 in range(0, n, 3 * 3):                         # this worker's batches of 3: every third one
        i1 = min(i0 + 3, n)
        for i, a in zip(range(i0, i1), worker.tune(i0, i1, 3, [io.StringIO() for _ in range(i0, i1)])):
            accs[i] = a
        held.append(set(worker.runs))
    keep = [multirun.param_grid(GRID)[0]] * N_RUNS
    for r0 in (1, 4):
        worker.final(r0, r0 + 1, 1, [io.StringIO()], params_keep=keep)
        held.append(set(worker.runs))
    assert max(len(h) for h in held) <= 2 and held[-1] == {4}
    np.random.seed(0)
    in_process = multirun._Tuning(dict(vars(params)), multirun.param_grid(GRID), list(range(N_RUNS)), time.time(),
                                  multirun.RunRng.capture())
    np.random.seed(0)
    from continuum.continuum import continuum
    in_process.data_all(continuum('cifar100', 'nc', params))
    want = in_process.tune(0, n, 1)
    assert all(np.array_equal(a, want[i]) for i, a in accs.items())
