"""Several repetitions of an experiment at once on one GPU (B200OCL_CONCURRENT_RUNS=R, R > 1).

The reference's multiple_run (experiment/run.py:17-87) trains num_runs repetitions of the stream one after another.
One replay step of a batch of 10 stream and 10 memory images launches kernels of a handful of CTAs each, so a single run
leaves most of the SMs idle.  Here up to R runs train side by side: each has its own agent, built and stepped under its
own CUDA stream, and the driver takes one replay step of each run in turn (a fixed round-robin order) through the
learners' step generators (learners.ContinualLearner._steps).  After each task every run is evaluated, in the same order.

Every run draws from its own random state (RunRng): the process-global generators the replay path reads (Python's
`random`, numpy's global RandomState, torch's CPU generator, the CUDA generator of the current device) are swapped in
before each of the run's steps and saved after it, together with the module-level host state of its buffers
(memory.RunHostState).  Run r is seeded from (params.seed, r) by run_seed(); its results therefore do not depend on R or
on how the runs are interleaved.  They are statistically equivalent to the reference's sequential runs, not the same
draws: the reference chains one global state through all runs.

multiple_run_tune_separate does the same for main_tune.py: every tuning training (run, grid point, repetition) and
every run's final training is one entry of run_group, seeded by tune_seed() and run_seed() respectively.
"""
import itertools
import os
import pickle
import random
import time
from types import SimpleNamespace

import numpy as np
import torch

from . import memory

ENV = 'B200OCL_CONCURRENT_RUNS'


def concurrent_runs(environ=None):
    """R from B200OCL_CONCURRENT_RUNS: 1 when unset or empty; anything but an integer >= 1 raises ValueError."""
    raw = (os.environ if environ is None else environ).get(ENV, '').strip()
    if raw == '':
        return 1
    if not raw.isdigit() or int(raw) < 1:
        raise ValueError('%s must be an integer >= 1, got %r' % (ENV, raw))
    return int(raw)


def _data_parallel():
    d = getattr(torch, 'distributed', None)
    return d is not None and d.is_available() and d.is_initialized() and d.get_world_size() > 1


def check_concurrent(n_concurrent, grad_sync=None):
    """The refusals of R > 1, raised before anything is built: parity mode replays the reference's one chain of global
    draws, which separate run states cannot; data-parallel gradient sync (a torch.distributed group of more than one
    rank, or grad_sync=True) makes every step a collective over ranks, which interleaved runs would mismatch."""
    if n_concurrent <= 1:
        return
    grad_sync = _data_parallel() if grad_sync is None else grad_sync
    if memory.parity():
        raise ValueError('B200OCL_MODE=parity replays the reference\'s single random stream; it cannot run %d runs at '
                         'once (%s=%d)' % (n_concurrent, ENV, n_concurrent))
    if grad_sync:
        raise ValueError('data-parallel gradient sync cannot be combined with %d concurrent runs (%s=%d)'
                         % (n_concurrent, ENV, n_concurrent))


def run_seed(seed, run):
    """The seed of run `run` of an experiment seeded with `seed`: the first 32-bit word numpy's SeedSequence derives from
    the entropy [seed, run].  It seeds all four generators of the run.  In the tuning wrapper
    (multiple_run_tune_separate) it is also the seed of run `run`'s final training, the one with the chosen point."""
    if int(seed) < 0 or int(run) < 0:
        raise ValueError('seed and run index must be >= 0, got (%d, %d)' % (seed, run))
    return int(np.random.SeedSequence([int(seed), int(run)]).generate_state(1, np.uint32)[0])


def tune_seed(seed, run, point, rep):
    """The seed of tuning training (run, point, rep) of multiple_run_tune_separate: the first 32-bit word of
    SeedSequence([seed, run, point, rep]), `point` the grid point's index in param_grid order and `rep` its repetition
    (0 .. num_runs_val - 1).  It depends on nothing else, so a training draws the same numbers whatever R is and
    wherever it sits in its group."""
    ids = [int(seed), int(run), int(point), int(rep)]
    if min(ids) < 0:
        raise ValueError('seed, run, point and repetition must be >= 0, got %s' % (tuple(ids),))
    return int(np.random.SeedSequence(ids).generate_state(1, np.uint32)[0])


def _cuda_rng():
    return torch.cuda.is_available()


class RunRng(object):
    """The four process-global random states of one run: Python `random`, numpy's global RandomState, torch's CPU
    generator and, when CUDA is in use, the CUDA generator of the current device.  swap_in() installs them, save()
    reads them back.  All four are host-side get_state / set_state calls; the CUDA generator's state is its seed and
    Philox offset, kept on the host, so neither call waits for the device."""
    __slots__ = ('py', 'np', 'cpu', 'cuda')

    def __init__(self, seed):
        seed = int(seed)
        self.py = random.Random(seed).getstate()
        self.np = np.random.RandomState(seed).get_state()
        self.cpu = torch.Generator().manual_seed(seed).get_state()
        self.cuda = torch.Generator(device='cuda').manual_seed(seed).get_state() if _cuda_rng() else None

    @classmethod
    def capture(cls):
        """The current global states (to put back after a group of runs)."""
        self = cls.__new__(cls)
        self.save()
        return self

    def swap_in(self):
        random.setstate(self.py)
        np.random.set_state(self.np)
        torch.set_rng_state(self.cpu)
        if self.cuda is not None:
            torch.cuda.set_rng_state(self.cuda)

    def save(self):
        self.py = random.getstate()
        self.np = np.random.get_state()
        self.cpu = torch.get_rng_state()
        self.cuda = torch.cuda.get_rng_state() if _cuda_rng() else None


class _Run(object):
    """One run of a group: its random state, its host state, its stream, its agent."""

    def __init__(self, index, rng_seed):
        self.index = index
        self.rng = RunRng(rng_seed)
        self.host = memory.RunHostState()
        self.stream = torch.cuda.Stream() if torch.cuda.is_available() else None
        self.agent = None
        self.steps = None
        self.acc = []

    def call(self, fn, *args):
        """fn(*args) with this run's random state, host state and stream current."""
        self.rng.swap_in()
        self.host.enter()
        try:
            if self.stream is None:
                return fn(*args)
            with torch.cuda.stream(self.stream):
                return fn(*args)
        finally:
            self.host.leave()
            self.rng.save()


def _next_step(steps):
    try:
        next(steps)
        return True
    except StopIteration:
        return False


def run_group(tasks_per_run, test_loaders_per_run, make_agent, n_concurrent, seed=0, first_run=0,
              on_task=None, on_run_end=None, before_run=None, seeds=None):
    """Train and evaluate len(tasks_per_run) runs, n_concurrent at a time, and return each run's accuracy array
    (np.array of the per-task evaluate() results, [n_tasks, n_test_loaders]).

    tasks_per_run[i]: the (x_train, y_train) tasks of run first_run + i (callables returning that list are accepted, and
    called under the run's random state when its group starts); test_loaders_per_run[i]: its test loaders (or callable).
    make_agent(r) builds the agent of run r; it is called with run r's random state current and under run r's stream.
    Run first_run + i is seeded with seeds[i] when a seed list is given, else with run_seed(seed, first_run + i).
    Runs are cut into groups of n_concurrent.  Inside a group each task is trained by taking one step of each run in
    turn, in run order, until all runs have finished the task; then every run is evaluated, in run order.  A run's
    agent is dropped once its last evaluation is done.
    Optional hooks, all called with the run's state current: before_run(r), on_task(r, t, x_train, y_train) before the
    run starts task t, on_run_end(r, acc) after the run's last evaluation."""
    n_concurrent = int(n_concurrent)
    if n_concurrent < 1:
        raise ValueError('n_concurrent must be >= 1, got %d' % n_concurrent)
    check_concurrent(n_concurrent)
    n_runs = len(tasks_per_run)
    if len(test_loaders_per_run) != n_runs:
        raise ValueError('%d task lists for %d sets of test loaders' % (n_runs, len(test_loaders_per_run)))
    if seeds is None:
        seeds = [run_seed(seed, first_run + i) for i in range(n_runs)]
    elif len(seeds) != n_runs:
        raise ValueError('%d seeds for %d runs' % (len(seeds), n_runs))
    memory.flush_pending()
    outer_rng, outer_host = RunRng.capture(), memory.RunHostState()
    outer_host.leave()
    results = []
    try:
        for g0 in range(0, n_runs, n_concurrent):
            group = [_Run(first_run + i, seeds[i]) for i in range(g0, min(g0 + n_concurrent, n_runs))]
            tasks, loaders = [], []
            for run in group:
                i = run.index - first_run
                if before_run is not None:
                    run.call(before_run, run.index)
                t, l = tasks_per_run[i], test_loaders_per_run[i]
                tasks.append(run.call(t) if callable(t) else t)
                loaders.append(run.call(l) if callable(l) else l)
                run.agent = run.call(make_agent, run.index)
                if n_concurrent > 1 and getattr(run.agent, 'grad_sync', None) is not None:
                    raise ValueError('run %d: an agent with data-parallel gradient sync cannot share the GPU with other '
                                     'runs' % run.index)
            for t in range(max(len(ts) for ts in tasks)):
                live = []
                for run, ts in zip(group, tasks):
                    if t < len(ts):
                        x, y = ts[t][0], ts[t][1]
                        if on_task is not None:
                            run.call(on_task, run.index, t, x, y)
                        run.steps = run.agent._steps(x, y)
                        live.append(run)
                while live:                                                 # one step per run, in run order
                    live = [run for run in live if run.call(_next_step, run.steps)]
                for run, ts, ls in zip(group, tasks, loaders):
                    if t < len(ts):
                        run.acc.append(run.call(run.agent.evaluate, ls))
            for run in group:
                acc = np.array(run.acc)
                if on_run_end is not None:
                    run.call(on_run_end, run.index, acc)
                results.append(acc)
                run.agent = run.steps = None                                # its engine arenas and graphs go with it
            del group, tasks, loaders
    finally:
        outer_host.enter()
        outer_rng.swap_in()
    return results


# --------------------------------------------------------------------------- the reference's multiple_run
def multiple_run(params, store=False, save_path=None, n_concurrent=None):
    """experiment/run.py:multiple_run with up to R = B200OCL_CONCURRENT_RUNS runs at once.  Same stdout lines (the per-run
    line of each run once it ends, then the compute_performance summary), same --store pickle ({'time', 'acc_array'} in
    config/global.yml's result path) and the offline mode (online: False) of the reference.  Each run of a group keeps
    its own task list and test loaders: one copy of the training set in host memory per concurrent run."""
    from continuum.continuum import continuum
    from continuum.data_utils import setup_test_loader
    from experiment.metrics import compute_performance
    from utils.io import load_yaml
    from utils.name_match import agents
    from utils.setup_elements import setup_opt, setup_architecture
    from utils.utils import maybe_cuda

    R = concurrent_runs() if n_concurrent is None else int(n_concurrent)
    check_concurrent(R)
    start = time.time()
    print('Setting up data stream')
    data_continuum = continuum(params.data, params.cl_type, params)
    data_end = time.time()
    print('data setup time: {}'.format(data_end - start))
    if store:
        result_path = load_yaml('config/global.yml', key='path')['result']
        table_path = result_path + params.data
        print(table_path)
        os.makedirs(table_path, exist_ok=True)
        if not save_path:
            save_path = params.model_name + '_' + params.data_name + '.pkl'

    online = params.online
    run_start = {}

    def new_run(r):
        run_start[r] = time.time()
        data_continuum.new_run()

    def task_list():
        tasks = [(x, y) for x, y, _ in data_continuum]
        if online:
            return tasks
        return [(np.concatenate([x for x, _ in tasks], axis=0), np.concatenate([y for _, y in tasks], axis=0))]

    def test_loaders():
        return setup_test_loader(data_continuum.test_data(), params)

    def make_agent(r):
        model = maybe_cuda(setup_architecture(params), params.cuda)
        opt = setup_opt(params.optimizer, model, params.learning_rate, params.weight_decay)
        return agents[params.agent](model, opt, params)

    def on_task(r, t, x, y):
        if online:
            print("-----------run {} training batch {}-------------".format(r, t))
        else:
            print('Training Start')
            print("----------run {} training-------------".format(r))
        print('size: {}, {}'.format(x.shape, y.shape))

    def on_run_end(r, acc):
        if online:
            print("-----------run {}-----------avg_end_acc {}-----------train time {}".format(
                r, np.mean(acc[-1]), time.time() - run_start[r]))

    # The continuum is one object: each run's new_run() and task list are taken before the next run's new_run(), so
    # the runs of a group get their own lists (callables, evaluated under the run's random state in run order).
    accuracy_list = []
    for g0 in range(0, params.num_runs, R):
        runs = range(g0, min(g0 + R, params.num_runs))
        accs = run_group([task_list] * len(runs), [test_loaders] * len(runs), make_agent, R, seed=params.seed,
                         first_run=g0, before_run=new_run, on_task=on_task, on_run_end=on_run_end)
        accuracy_list += accs if online else [a[0] for a in accs]
    accuracy_array = np.array(accuracy_list)
    end = time.time()
    if store:
        result = {'time': end - start}
        result['acc_array'] = accuracy_array
        with open(table_path + '/' + save_path, 'wb') as f:
            pickle.dump(result, f)
    if online:
        avg_end_acc, avg_end_fgt, avg_acc, avg_bwtp, avg_fwt = compute_performance(accuracy_array)
        print('----------- Total {} run: {}s -----------'.format(params.num_runs, end - start))
        print('----------- Avg_End_Acc {} Avg_End_Fgt {} Avg_Acc {} Avg_Bwtp {} Avg_Fwt {}-----------'
              .format(avg_end_acc, avg_end_fgt, avg_acc, avg_bwtp, avg_fwt))
    else:
        print('----------- Total {} run: {}s -----------'.format(params.num_runs, end - start))
        print("avg_end_acc {}".format(np.mean(accuracy_list)))


# --------------------------------------------------------------------------- the reference's multiple_run_tune_separate
def param_grid(tune_params):
    """The points of sklearn's ParameterGrid(tune_params) for a dict of value lists, in its order: the keys sorted,
    itertools.product over their value lists, the last key varying fastest.  A dict with no keys gives one empty point.
    Every point sets every key, which is what lets each training's params be built from the defaults alone."""
    if not isinstance(tune_params, dict):
        raise TypeError('the tuning grid must be a dict of value lists, got %s' % type(tune_params).__name__)
    keys = sorted(tune_params)
    return [dict(zip(keys, values)) for values in itertools.product(*(tune_params[k] for k in keys))]


def multiple_run_tune_separate(default_params, tune_params, save_path, n_concurrent=None):
    """experiment/run.py:multiple_run_tune_separate (main_tune.py) with up to R = B200OCL_CONCURRENT_RUNS trainings at
    once, for both of its branches (single_tune, and single_tune_train_val with train_val), online and offline.

    Every run's task list and test loaders are taken first: data_continuum.new_run() once per run, in run order, from the
    caller's random state.  A training is a (run r, grid point g, repetition v) triple.  Stage 1 trains every tuning
    training of every run through run_group, R at a time in (r, g, v) order, on run r's first num_val tasks (offline:
    their concatenation), evaluated on run r's first num_val test loaders after each task; training (r, g, v) is seeded
    with tune_seed(seed, r, g, v).  Stage 2 picks each run's point with the best compute_performance end accuracy (the
    earliest on a tie) and trains the runs' final agents, R at a time, seeded with run_seed(seed, r): on tasks num_val..
    evaluated on the remaining loaders, or with train_val on every task evaluated on every loader (offline: on the
    concatenation).  Each training's stdout lines are the reference's and are printed when it ends; the pickle is the
    reference's, at its path.  default_params ends holding what the reference leaves in it: num_val resolved, and the
    last run's chosen point."""
    from continuum.continuum import continuum
    from continuum.data_utils import setup_test_loader
    from experiment.metrics import compute_performance
    from utils.io import check_ram_usage, load_yaml
    from utils.name_match import agents
    from utils.setup_elements import setup_opt, setup_architecture
    from utils.utils import maybe_cuda

    R = concurrent_runs() if n_concurrent is None else int(n_concurrent)
    check_concurrent(R)
    start = time.time()
    print('Setting up data stream')
    data_continuum = continuum(default_params.data, default_params.cl_type, default_params)
    data_end = time.time()
    print('data setup time: {}'.format(data_end - start))
    if default_params.num_val == -1:
        default_params.num_val = data_continuum.data_object.task_nums
    num_val, online, train_val = default_params.num_val, default_params.online, default_params.train_val
    if not train_val and num_val >= data_continuum.data_object.task_nums:
        raise ValueError('num_val %d leaves none of the %d tasks for the final agents; use train_val to train them on '
                         'every task' % (num_val, data_continuum.data_object.task_nums))
    result_path = load_yaml('config/global.yml', key='path')['result']
    table_path = result_path + default_params.data + '/' + default_params.cl_type
    for i in default_params.trick:
        if default_params.trick[i]:
            table_path = result_path + default_params.data + '/' + default_params.cl_type + '/' + i
            break
    print(table_path)
    os.makedirs(table_path, exist_ok=True)
    if not save_path:
        save_path = default_params.model_name + '_' + default_params.data_name + '_' + str(default_params.seed) + '.pkl'
    run_list = list(range(default_params.num_runs) if isinstance(default_params.num_runs, int)
                    else default_params.num_runs)
    grid = param_grid(tune_params)
    defaults = dict(vars(default_params))

    def concat(tasks):
        return [(np.concatenate([x for x, _ in tasks], axis=0), np.concatenate([y for _, y in tasks], axis=0))]

    # every run's data, before any training: (tune tasks, tune loaders, final tasks, final loaders)
    data = []
    for run in run_list:
        data_continuum.new_run()
        loaders = setup_test_loader(data_continuum.test_data(), default_params)
        tasks = [(x, y) for x, y, _ in data_continuum]
        final = tasks if train_val else tasks[num_val:]
        if online:
            data.append((tasks[:num_val], loaders[:num_val], final, loaders if train_val else loaders[num_val:]))
        else:   # the final concatenation is made when its training starts
            data.append((concat(tasks[:num_val]), loaders[:num_val], (lambda f=final: concat(f)),
                         loaders if train_val else loaders[num_val:]))

    def build(params):
        model = maybe_cuda(setup_architecture(params), params.cuda)
        opt = setup_opt(params.optimizer, model, params.learning_rate, params.weight_decay)
        return agents[params.agent](model, opt, params)

    out = {}            # a training's stdout lines, printed when it ends
    run_start = {}

    # stage 1: every (run, point, repetition), in that order
    point_params = [SimpleNamespace(**dict(defaults, **point)) for point in grid]
    entries = [(ri, g, v) for ri in range(len(run_list)) for g in range(len(grid))
               for v in range(point_params[g].num_runs_val)]

    def tune_begin(i):
        ri, g, v = entries[i]
        run_start.setdefault(ri, time.time())
        out[i] = ([str(len(grid))] if g == 0 and v == 0 else []) + ([str(grid[g])] if v == 0 else [])

    def tune_task(i, t, x, y):
        out[i] += ['-----------tune run {} task {}-------------'.format(entries[i][2], t),
                   'size: {}, {}'.format(x.shape, y.shape)]

    def tune_end(i, acc):
        out[i].append('-----------tune run {}-----------avg_end_acc {}-----------'.format(entries[i][2],
                                                                                         np.mean(acc[-1])))
        print('\n'.join(out.pop(i)))

    tune_acc = run_group([data[ri][0] for ri, _, _ in entries], [data[ri][1] for ri, _, _ in entries],
                         lambda i: build(point_params[entries[i][1]]), R,
                         seeds=[tune_seed(default_params.seed, run_list[ri], g, v) for ri, g, v in entries],
                         before_run=tune_begin, on_task=tune_task, on_run_end=tune_end)

    # the chosen points, as tune_hyper chooses them
    params_keep = []
    for ri in range(len(run_list)):
        tune_accs = []
        for g in range(len(grid)):
            accs = np.array([a for (rj, gj, _), a in zip(entries, tune_acc) if (rj, gj) == (ri, g)])
            tune_accs.append(compute_performance(accs)[0][0])
        params_keep.append(grid[tune_accs.index(max(tune_accs))])

    # stage 2: each run's final agent, with the reference's in-place update of default_params
    def final_begin(ri):
        out[ri] = ['Tuning is done. Best hyper parameter set is {}'.format(params_keep[ri]), 'Training Start']

    def final_agent(ri):
        vars(default_params).update(params_keep[ri])
        return build(SimpleNamespace(**vars(default_params)))

    def final_task(ri, t, x, y):
        if online:
            out[ri] += ['----------run {} training batch {}-------------'.format(
                run_list[ri], t if train_val else t + num_val)]
        else:
            out[ri] += ['----------run {} training-------------'.format(run_list[ri])]
        out[ri] += ['size: {}, {}'.format(x.shape, y.shape)]

    def final_end(ri, acc):
        out[ri].append('-----------run {}-----------avg_end_acc {}-----------train time {}'.format(
            run_list[ri], np.mean(acc[-1]), time.time() - run_start.get(ri, start)))
        print('\n'.join(out.pop(ri)))

    accuracy_list = run_group([d[2] for d in data], [d[3] for d in data], final_agent, R,
                              seeds=[run_seed(default_params.seed, run) for run in run_list],
                              before_run=final_begin, on_task=final_task, on_run_end=final_end)
    end = time.time()
    result = {'seed': default_params.seed, 'time': end - start, 'acc_array': np.array(accuracy_list),
              'ram': check_ram_usage(), 'best_params': params_keep}
    with open(table_path + '/' + save_path, 'wb') as f:
        pickle.dump(result, f)
    print('----------- Total {} run: {}s -----------'.format(default_params.num_runs, end - start))
    print('----------- Seed {} RAM: {}s -----------'.format(default_params.seed, result['ram']))
