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

With B200OCL_RUN_DEVICES (a list of CUDA ordinals) both drivers hand their trainings to worker processes instead, one per
list entry (WorkerPool); each worker runs them through run_group, R at a time, on its own device.  A training's seed does
not depend on where it runs, so its numbers are the same as in one process.

With B200OCL_CHECKPOINT_DIR run_group writes each training's snapshot after every task and its record once it ends, and
both drivers resume an interrupted experiment from them (checkpoint.py).  With B200OCL_CHECKPOINT_ASYNC=1 as well the
snapshots are staged on the device and written by a background thread while the next task trains.
"""
import contextlib
import io
import itertools
import multiprocessing
import multiprocessing.connection
import os
import pickle
import random
import re
import sys
import time
import traceback
from types import SimpleNamespace

import numpy as np
import torch

from . import memory

ENV = 'B200OCL_CONCURRENT_RUNS'
DEVICES_ENV = 'B200OCL_RUN_DEVICES'


def concurrent_runs(environ=None):
    """R from B200OCL_CONCURRENT_RUNS: 1 when unset or empty; anything but an integer >= 1 raises ValueError."""
    raw = (os.environ if environ is None else environ).get(ENV, '').strip()
    if raw == '':
        return 1
    if not raw.isdigit() or int(raw) < 1:
        raise ValueError('%s must be an integer >= 1, got %r' % (ENV, raw))
    return int(raw)


def run_devices(environ=None):
    """The worker devices from B200OCL_RUN_DEVICES, a comma-separated list of CUDA ordinals (repeats allowed: '0,0' is
    two workers on device 0): () when unset or empty.  A non-integer, a negative ordinal or an empty entry raises
    ValueError.  Whether the ordinals exist is checked by the drivers (check_device_count), not here."""
    raw = (os.environ if environ is None else environ).get(DEVICES_ENV, '').strip()
    if raw == '':
        return ()
    devices = []
    for entry in raw.split(','):
        entry = entry.strip()
        if entry == '':
            raise ValueError('%s has an empty entry: %r' % (DEVICES_ENV, raw))
        if not re.fullmatch(r'[+-]?[0-9]+', entry):
            raise ValueError('%s entries must be integer CUDA ordinals, got %r in %r' % (DEVICES_ENV, entry, raw))
        if int(entry) < 0:
            raise ValueError('%s entries must be >= 0, got %r in %r' % (DEVICES_ENV, entry, raw))
        devices.append(int(entry))
    return tuple(devices)


def check_device_count(devices):
    """Every ordinal of `devices` must be a CUDA device of this process (torch.cuda.device_count())."""
    n = torch.cuda.device_count()
    missing = sorted(set(d for d in devices if d >= n))
    if missing:
        raise ValueError('%s names device(s) %s, but %d CUDA device(s) are visible'
                         % (DEVICES_ENV, ', '.join(map(str, missing)), n))


def _data_parallel():
    d = getattr(torch, 'distributed', None)
    return d is not None and d.is_available() and d.is_initialized() and d.get_world_size() > 1


def check_concurrent(n_concurrent, grad_sync=None, devices=()):
    """The refusals of R > 1 and of worker devices, raised before anything is built: parity mode replays the
    reference's one chain of global draws, which separate run states cannot; data-parallel gradient sync (a
    torch.distributed group of more than one rank, or grad_sync=True) makes every step a collective over ranks, which
    interleaved runs, or runs in other processes, would mismatch."""
    if n_concurrent <= 1 and not devices:
        return
    grad_sync = _data_parallel() if grad_sync is None else grad_sync
    if devices:
        where = 'worker processes (%s=%s)' % (DEVICES_ENV, ','.join(map(str, devices)))
        parity_msg, sync_msg = 'split its runs over ' + where, 'be combined with runs in ' + where
    else:
        parity_msg = 'run %d runs at once (%s=%d)' % (n_concurrent, ENV, n_concurrent)
        sync_msg = 'be combined with %d concurrent runs (%s=%d)' % (n_concurrent, ENV, n_concurrent)
    if memory.parity():
        raise ValueError('B200OCL_MODE=parity replays the reference\'s single random stream; it cannot ' + parity_msg)
    if grad_sync:
        raise ValueError('data-parallel gradient sync cannot ' + sync_msg)


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

    def snapshot(self):
        """The four states as a picklable tuple (restore() takes it back)."""
        return (self.py, self.np, self.cpu.clone(), None if self.cuda is None else self.cuda.clone())

    def restore(self, state):
        self.py, self.np, self.cpu, self.cuda = state
        if self.cuda is None and _cuda_rng():
            raise ValueError('a snapshot taken without CUDA cannot resume a run that uses the CUDA generator')


class _Tee(object):
    """A stdout that writes to two streams (a run's per-run line to its output and to its record)."""

    def __init__(self, out, copy):
        self.out, self.copy = out, copy

    def write(self, s):
        self.copy.write(s)
        return self.out.write(s)

    def flush(self):
        self.out.flush()


def _teed(fn, copy):
    def call(*args):
        out = sys.stdout
        sys.stdout = _Tee(out, copy)
        try:
            return fn(*args)
        finally:
            sys.stdout = out
    return call


class _Run(object):
    """One run of a group: its random state, its host state, its stream, its agent, and where its prints go (None: the
    current sys.stdout)."""

    def __init__(self, index, rng_seed, out=None):
        self.index = index
        self.rng = RunRng(rng_seed)
        self.host = memory.RunHostState()
        self.stream = torch.cuda.Stream() if torch.cuda.is_available() else None
        self.out = out
        self.agent = None
        self.steps = None
        self.staging = None     # its checkpoint.Staging when snapshots are written behind the run
        self.acc = []
        self.start = 0          # the first task this run trains (after a restored snapshot: the task after it)

    def snapshot(self, task):
        """The run's state at the end of `task`, after its evaluation: the deferred host-mirror updates are drained,
        then its agent's snapshot() is taken under its stream; the random and host states are the ones run.call left."""
        def take():
            memory.flush_pending()
            return self.agent.snapshot()
        agent = self.call(take)
        return {'task': task, 'acc': [np.array(a) for a in self.acc], 'rng': self.rng.snapshot(),
                'sampler': self.host.sampler, 'agent': agent}

    def stage(self, task):
        """snapshot(task), staged: the host state is captured as snapshot() captures it, the agent's device arrays
        (snapshot_parts()) are packed into the run's staging arena under its stream.  Returns (the snapshot with
        placeholders for those arrays, the job that writes them)."""
        def take():
            memory.flush_pending()
            return self.staging.stage(self.agent.snapshot_parts())
        agent, job = self.call(take)
        return {'task': task, 'acc': [np.array(a) for a in self.acc], 'rng': self.rng.snapshot(),
                'sampler': self.host.sampler, 'agent': agent}, job

    def restore(self, snap):
        """Continue from a snapshot of this run: its agent (built as usual) takes the snapshot's state, then the
        random state, the sampler state and the accuracy rows; training restarts at the task after the snapshot's."""
        if len(snap['acc']) != snap['task'] + 1:
            raise ValueError('run %d: a snapshot of task %d holds %d accuracy rows'
                             % (self.index, snap['task'], len(snap['acc'])))
        self.call(self.agent.restore, snap['agent'])
        self.rng.restore(snap['rng'])
        self.host.sampler, self.host.pending = snap['sampler'], []
        self.acc = [np.array(a) for a in snap['acc']]
        self.start = snap['task'] + 1

    def call(self, fn, *args):
        """fn(*args) with this run's random state, host state, stream and stdout current.  An exception leaves with
        the run's index in its `run_index` attribute (the innermost run's, when calls nest)."""
        self.rng.swap_in()
        self.host.enter()
        stdout = sys.stdout
        if self.out is not None:
            sys.stdout = self.out
        try:
            if self.stream is None:
                return fn(*args)
            with torch.cuda.stream(self.stream):
                return fn(*args)
        except Exception as e:
            if getattr(e, 'run_index', None) is None:
                e.run_index = self.index
            raise
        finally:
            if self.out is not None:
                sys.stdout = stdout
            self.host.leave()
            self.rng.save()


def _next_step(steps):
    try:
        next(steps)
        return True
    except StopIteration:
        return False


def run_group(tasks_per_run, test_loaders_per_run, make_agent, n_concurrent, seed=0, first_run=0,
              on_task=None, on_run_end=None, before_run=None, seeds=None, stdout=None, checkpoint=None):
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
    run starts task t, on_run_end(r, acc) after the run's last evaluation.  stdout[i], when given, receives everything
    run first_run + i prints (its hooks, its agent's construction, steps and evaluations).

    checkpoint (a checkpoint.Checkpoint, default None: nothing is read or written): run first_run + i is its training
    first_run + i.  A run with a record is not trained: its array is returned and its text printed in run order, before
    the next group if that group's runs all follow it, else just before the next run's on_run_end.  The others are cut
    into groups as above; a run with a snapshot is
    built as usual, then restored, and trains from the task after the snapshot's.  After its evaluation of every task
    but its last a run's snapshot is written; after on_run_end its record (what on_run_end printed).  With
    checkpoint.async_write each run gets a staging arena when it is built, snapshots are staged and they and the records
    are written by the writer thread; every write has ended when run_group returns or raises, and a failed write raises
    CheckpointError there or at the next task boundary."""
    n_concurrent = int(n_concurrent)
    if n_concurrent < 1:
        raise ValueError('n_concurrent must be >= 1, got %d' % n_concurrent)
    check_concurrent(n_concurrent)
    staged = checkpoint is not None and checkpoint.async_write
    if checkpoint is not None:
        from . import checkpoint as ckpt
        ckpt.check_checkpoint(checkpoint.directory)
    n_runs = len(tasks_per_run)
    if len(test_loaders_per_run) != n_runs:
        raise ValueError('%d task lists for %d sets of test loaders' % (n_runs, len(test_loaders_per_run)))
    if seeds is None:
        seeds = [run_seed(seed, first_run + i) for i in range(n_runs)]
    elif len(seeds) != n_runs:
        raise ValueError('%d seeds for %d runs' % (len(seeds), n_runs))
    if stdout is not None and len(stdout) != n_runs:
        raise ValueError('%d outputs for %d runs' % (len(stdout), n_runs))
    done = {}
    if checkpoint is not None:
        for i in range(n_runs):
            rec = checkpoint.record(first_run + i)
            if rec is not None:
                done[i] = rec
    results = [done[i][0] if i in done else None for i in range(n_runs)]
    replayed = []

    def replay(upto):
        """Print the records of the runs before position `upto`, in run order."""
        for i in sorted(done):
            if i < upto and i not in replayed:
                (sys.stdout if stdout is None else stdout[i]).write(done[i][1])
                replayed.append(i)
    memory.flush_pending()
    outer_rng, outer_host = RunRng.capture(), memory.RunHostState()
    outer_host.leave()
    todo = [i for i in range(n_runs) if i not in done]
    try:
        for g0 in range(0, len(todo), n_concurrent):
            group = [_Run(first_run + i, seeds[i], None if stdout is None else stdout[i])
                     for i in todo[g0:g0 + n_concurrent]]
            replay(group[0].index - first_run)
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
                if staged:
                    run.staging = run.call(lambda: ckpt.Staging(run.agent.snapshot_capacity(), run.agent.device))
                snap = None if checkpoint is None else run.call(checkpoint.snapshot, run.index, run.staging)
                if snap is not None:
                    run.restore(snap)
            for t in range(max(len(ts) for ts in tasks)):
                live = []
                for run, ts in zip(group, tasks):
                    if run.start <= t < len(ts):
                        x, y = ts[t][0], ts[t][1]
                        if on_task is not None:
                            run.call(on_task, run.index, t, x, y)
                        run.steps = run.agent._steps(x, y)
                        live.append(run)
                trained = list(live)
                while live:                                                 # one step per run, in run order
                    live = [run for run in live if run.call(_next_step, run.steps)]
                for run, ts, ls in zip(group, tasks, loaders):
                    if run in trained:
                        run.acc.append(run.call(run.agent.evaluate, ls))
                if checkpoint is not None:
                    for run, ts in zip(group, tasks):
                        if run in trained and t < len(ts) - 1:
                            if staged:
                                checkpoint.save_staged(run.index, *run.stage(t))
                            else:
                                checkpoint.save_snapshot(run.index, run.snapshot(t))
            for run in group:
                replay(run.index - first_run)
                acc = np.array(run.acc)
                if checkpoint is None:
                    if on_run_end is not None:
                        run.call(on_run_end, run.index, acc)
                else:
                    text = io.StringIO()
                    if on_run_end is not None:
                        run.call(_teed(on_run_end, text), run.index, acc)
                    checkpoint.save_record(run.index, acc, text.getvalue())
                results[run.index - first_run] = acc
                if run.staging is not None:
                    run.staging.release()
                run.agent = run.steps = run.staging = None                  # its engine arenas and graphs go with it
            del group, tasks, loaders
        replay(n_runs)
        if staged:
            ckpt.writer().drain()
    except BaseException as e:
        if staged:                     # every write ends; a failed one is told with the exception that is leaving
            failed = ckpt.writer().drain(check=False)
            if failed is not None:
                e.add_note('and a snapshot write failed meanwhile: %s' % failed)
        raise
    finally:
        outer_host.enter()
        outer_rng.swap_in()
    return results


# --------------------------------------------------------------------------- worker processes (B200OCL_RUN_DEVICES)
def _child_visible_device(ordinal):
    """The CUDA_VISIBLE_DEVICES of a worker on this process's device `ordinal`: that entry of our own list when we have
    one (ordinals count the devices we see), else the ordinal itself."""
    visible = os.environ.get('CUDA_VISIBLE_DEVICES')
    if visible is None or visible.strip() == '':
        return str(ordinal)
    ids = [v.strip() for v in visible.split(',')]
    if ordinal >= len(ids):
        raise ValueError('device %d is not in CUDA_VISIBLE_DEVICES=%r' % (ordinal, visible))
    return ids[ordinal]


@contextlib.contextmanager
def _worker_environ(ordinal):
    """The environment a spawned worker starts with: ours, with CUDA_VISIBLE_DEVICES naming its one device and without
    B200OCL_RUN_DEVICES (a worker trains in process).  A spawned child copies the environment when it starts, so this
    is in place before its interpreter, and torch, start."""
    keys = ('CUDA_VISIBLE_DEVICES', DEVICES_ENV)
    saved = {k: os.environ.get(k) for k in keys}
    visible = _child_visible_device(ordinal)
    try:
        os.environ['CUDA_VISIBLE_DEVICES'] = visible
        os.environ.pop(DEVICES_ENV, None)
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _worker_main(conn):
    """A worker: receives its setup (sys.path, extra agents, R, the recipe), installs the engine, then trains the
    batches it is sent until its pipe closes.  A batch is (method, i0, i1, args): recipe.method(i0, i1, R, outs, *args)
    trains entries i0..i1-1 and returns their accuracy arrays; the reply carries each array and what the training
    printed, or the exception of the first training that failed.  EOF on the pipe (the parent closed it, or died)
    ends the worker.  Whatever the worker prints outside a training (its continuum build, its replays of the data
    draws) goes to os.devnull: the parent prints those lines itself, where the in-process driver prints them."""
    sink = open(os.devnull, 'w')
    sys.stdout = sink
    try:
        setup = pickle.loads(conn.recv_bytes())
        sys.path[:] = setup['path']
        from . import registry
        registry.install(extra=setup['extra'])
        recipe, R = setup['recipe'], setup['R']
        while True:
            method, i0, i1, args = pickle.loads(conn.recv_bytes())
            outs = [io.StringIO() for _ in range(i0, i1)]
            try:
                accs = getattr(recipe, method)(i0, i1, R, outs, *args)
                reply = ('ok', [(a, o.getvalue()) for a, o in zip(accs, outs)])
            except Exception as e:
                i = getattr(e, 'run_index', None)
                where = recipe.describe(method, i) if i is not None else ', '.join(
                    recipe.describe(method, j) for j in range(i0, i1))
                try:
                    etype = pickle.dumps(type(e))
                except Exception:
                    etype = pickle.dumps(RuntimeError)
                reply = ('error', etype, '%s: %s' % (type(e).__name__, e), where, traceback.format_exc())
            conn.send_bytes(pickle.dumps(reply))
            if reply[0] == 'error':
                return
    except EOFError:
        return
    finally:
        conn.close()
        sys.stdout = sys.__stdout__
        sink.close()


class _Worker(object):
    __slots__ = ('device', 'proc', 'conn', 'batch')

    def __init__(self, device, proc, conn):
        self.device, self.proc, self.conn, self.batch = device, proc, conn, None


class WorkerPool(object):
    """One worker process per entry of `devices`, for the length of a `with` block.  Workers are spawned (the parent
    may hold a CUDA context, which fork would copy), each sees one device, as device 0.  map() hands the trainings of a
    recipe to idle workers, up to n_concurrent consecutive ones at a time (one run_group call in the worker), and
    prints what each training printed in training order, whatever order they finish in.  Leaving the block closes
    every pipe and joins every worker; on an exception (a worker's, re-raised here, or the caller's, KeyboardInterrupt
    included) the workers still running are terminated first.  The pool does not check that the devices exist.

    Two things a spawned worker does before _worker_main runs: it re-executes the top level of the parent's __main__
    script as __mp_main__ (under b200ocl.launch that is the reference's general_main.py or main_tune.py, whose
    `if __name__ == "__main__"` guard keeps it from starting another experiment), and multiprocessing starts its
    resource tracker in the parent, a helper that exits with the parent's interpreter, not with the pool."""

    def __init__(self, devices, recipe, n_concurrent, extra=()):
        self.devices, self.recipe, self.R, self.extra = tuple(devices), recipe, int(n_concurrent), tuple(extra)
        self.workers = []

    def __enter__(self):
        ctx = multiprocessing.get_context('spawn')
        setup = pickle.dumps({'path': list(sys.path), 'extra': self.extra, 'recipe': self.recipe, 'R': self.R})
        try:
            for d in self.devices:
                mine, theirs = ctx.Pipe()
                proc = ctx.Process(target=_worker_main, args=(theirs,), name='b200ocl-run-worker-dev%d' % d)
                with _worker_environ(d):
                    proc.start()
                theirs.close()                     # ours only: EOF reaches each side when the other end goes
                self.workers.append(_Worker(d, proc, mine))
                mine.send_bytes(setup)
        except BaseException:
            self.close(failed=True)
            raise
        return self

    def __exit__(self, exc_type, exc, tb):
        self.close(failed=exc_type is not None)
        return False

    def close(self, failed=False):
        for w in self.workers:
            if failed and w.proc.is_alive():
                w.proc.terminate()
            w.conn.close()                         # an idle worker sees EOF and exits
        for w in self.workers:
            w.proc.join(None if failed else 60)
            if w.proc.is_alive():
                w.proc.terminate()
                w.proc.join()
        self.workers = []

    def map(self, method, n, args=()):
        """recipe.method over entries 0..n-1 on the workers; returns their accuracy arrays in entry order."""
        pending = [(i0, min(i0 + self.R, n)) for i0 in range(0, n, self.R)][::-1]
        results, printed = [None] * n, 0
        while printed < n:
            for w in self.workers:
                if w.batch is None and pending:
                    w.batch = pending.pop()
                    w.conn.send_bytes(pickle.dumps((method, w.batch[0], w.batch[1], tuple(args))))
            busy = [w for w in self.workers if w.batch is not None]
            for conn in multiprocessing.connection.wait([w.conn for w in busy]):
                w = next(w for w in busy if w.conn is conn)
                reply = self._receive(w, method)
                if reply[0] == 'error':
                    self._raise(w, reply)
                for i, r in zip(range(*w.batch), reply[1]):
                    results[i] = r
                w.batch = None
            while printed < n and results[printed] is not None:
                sys.stdout.write(results[printed][1])
                printed += 1
            sys.stdout.flush()
        return [r[0] for r in results]

    def _receive(self, w, method):
        try:
            return pickle.loads(w.conn.recv_bytes())
        except EOFError:
            w.proc.join(5)
            raise RuntimeError('the worker on device %d exited (code %s) during %s'
                               % (w.device, w.proc.exitcode, ', '.join(self.recipe.describe(method, i)
                                                                       for i in range(*w.batch))))

    def _raise(self, w, reply):
        _, etype, message, where, tb = reply
        try:
            etype = pickle.loads(etype)
            exc = etype('%s, on the worker of device %d: %s' % (where, w.device, message))
        except Exception:
            exc = RuntimeError('%s, on the worker of device %d: %s' % (where, w.device, message))
        exc.add_note('worker traceback:\n' + tb.rstrip())
        raise exc


class _Recipe(object):
    """What a driver's trainings need, sent to every worker: picklable descriptions (params, seeds, the caller's random
    state) only.  Attributes named in LOCAL (the data continuum, task lists, hook state) are rebuilt where it runs."""
    LOCAL = ()
    checkpoint_dir = None         # B200OCL_CHECKPOINT_DIR of the driver (None: no checkpoints)
    checkpoint_async = False      # B200OCL_CHECKPOINT_ASYNC of the driver

    def _checkpoint(self, stage):
        if self.checkpoint_dir is None:
            return None
        from .checkpoint import Checkpoint
        return Checkpoint(self.checkpoint_dir, stage, self.checkpoint_async)

    def __getstate__(self):
        return {k: v for k, v in self.__dict__.items() if k not in self.LOCAL}

    def __setstate__(self, state):
        self.__dict__.update(state)
        self._local()

    def _continuum(self, params):
        """A continuum built from the caller's random state on entry, as the driver built its own, and the random
        state after the build.  The state of the process is left as it was."""
        from continuum.continuum import continuum
        keep = RunRng.capture()
        try:
            self.entry_rng.swap_in()
            return continuum(params.data, params.cl_type, params), RunRng.capture()
        finally:
            keep.swap_in()


def _open_checkpoint(checkpoint_dir, params, grid=None):
    """A driver's checkpoint directory (None: none) and whether its snapshots are written behind the runs
    (B200OCL_CHECKPOINT_ASYNC), with the refusals and the fingerprint checked before anything is built.  The switch is
    not part of the fingerprint: both forms of snapshot resume either way."""
    from . import checkpoint
    directory = checkpoint.checkpoint_dir() if checkpoint_dir is None else (checkpoint_dir or None)
    if directory is None:
        return None, False
    async_write = checkpoint.checkpoint_async(directory=directory)
    checkpoint.check_checkpoint(directory)
    from . import registry
    checkpoint.open_dir(directory, checkpoint.fingerprint(params, registry.installed_extra, grid=grid))
    return directory, async_write


# --------------------------------------------------------------------------- the reference's multiple_run
class _Repetitions(_Recipe):
    """The runs of multiple_run.  Run r draws its data under its own random state: new_run() with cur_run = r - 1, then
    its task list and test loaders, so any process with its own continuum gives run r the same data."""
    LOCAL = ('cont', 'run_start')

    def __init__(self, params, entry_rng, cont=None):
        self.params, self.entry_rng = params, entry_rng
        self._local()
        self.cont = cont

    def _local(self):
        self.cont, self.run_start = None, {}

    def describe(self, method, r):
        return 'run %d' % r

    def new_run(self, r):
        self.run_start[r] = time.time()
        self.cont.cur_run = r - 1
        self.cont.new_run()

    def task_list(self):
        tasks = [(x, y) for x, y, _ in self.cont]
        if self.params.online:
            return tasks
        return [(np.concatenate([x for x, _ in tasks], axis=0), np.concatenate([y for _, y in tasks], axis=0))]

    def test_loaders(self):
        from continuum.data_utils import setup_test_loader
        return setup_test_loader(self.cont.test_data(), self.params)

    def make_agent(self, r):
        from utils.name_match import agents
        from utils.setup_elements import setup_opt, setup_architecture
        from utils.utils import maybe_cuda
        params = self.params
        model = maybe_cuda(setup_architecture(params), params.cuda)
        opt = setup_opt(params.optimizer, model, params.learning_rate, params.weight_decay)
        return agents[params.agent](model, opt, params)

    def on_task(self, r, t, x, y):
        if self.params.online:
            print("-----------run {} training batch {}-------------".format(r, t))
        else:
            print('Training Start')
            print("----------run {} training-------------".format(r))
        print('size: {}, {}'.format(x.shape, y.shape))

    def on_run_end(self, r, acc):
        if self.params.online:
            print("-----------run {}-----------avg_end_acc {}-----------train time {}".format(
                r, np.mean(acc[-1]), time.time() - self.run_start[r]))

    def train(self, r0, r1, R, outs=None):
        """Runs r0..r1-1 through one run_group call, R at a time."""
        if self.cont is None:
            self.cont = self._continuum(self.params)[0]
        n = r1 - r0
        return run_group([self.task_list] * n, [self.test_loaders] * n, self.make_agent, R, seed=self.params.seed,
                         first_run=r0, before_run=self.new_run, on_task=self.on_task, on_run_end=self.on_run_end,
                         stdout=outs, checkpoint=self._checkpoint('runs'))


def multiple_run(params, store=False, save_path=None, n_concurrent=None, devices=None, checkpoint_dir=None):
    """experiment/run.py:multiple_run with up to R = B200OCL_CONCURRENT_RUNS runs at once.  Same stdout lines (the per-run
    line of each run once it ends, then the compute_performance summary), same --store pickle ({'time', 'acc_array'} in
    config/global.yml's result path) and the offline mode (online: False) of the reference.  Each run of a group keeps
    its own task list and test loaders: one copy of the training set in host memory per concurrent run.

    With worker devices (B200OCL_RUN_DEVICES, or `devices`) the runs are trained by a WorkerPool, R at a time in each
    worker, and each run's lines are printed in run order once it and every run before it have ended.  This process
    still builds the continuum, so its lines (and the caller's random state after it) are the in-process ones; it
    drops it before the workers start, and each worker builds its own, silently.

    With a checkpoint directory (B200OCL_CHECKPOINT_DIR, or `checkpoint_dir`; '' turns it off) the runs resume from it
    (checkpoint.py): its fingerprint is checked before anything is built."""
    from continuum.continuum import continuum
    from experiment.metrics import compute_performance
    from utils.io import load_yaml

    R = concurrent_runs() if n_concurrent is None else int(n_concurrent)
    devices = run_devices() if devices is None else tuple(devices)
    check_concurrent(R, devices=devices)
    if devices:
        check_device_count(devices)
    directory, async_write = _open_checkpoint(checkpoint_dir, params)
    entry_rng = RunRng.capture()
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
    recipe = _Repetitions(params, entry_rng, None if devices else data_continuum)
    recipe.checkpoint_dir, recipe.checkpoint_async = directory, async_write
    if devices:
        from . import registry
        del data_continuum
        with WorkerPool(devices, recipe, R, registry.installed_extra) as pool:
            accs = pool.map('train', params.num_runs)
    else:
        # The continuum is one object: each run's new_run() and task list are taken before the next run's new_run(),
        # so the runs of a group get their own lists (evaluated under the run's random state in run order).
        accs = []
        for g0 in range(0, params.num_runs, R):
            accs += recipe.train(g0, min(g0 + R, params.num_runs), R)
    accuracy_list = accs if online else [a[0] for a in accs]
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


class _Tuning(_Recipe):
    """The trainings of multiple_run_tune_separate.  Entry i of stage 1 ('tune') is the (run index, point, repetition)
    entries[i]; entry ri of stage 2 ('final') is run run_list[ri]'s final training.  Every run's data comes from one
    chain of the caller's random state, run after run: the driver draws them all up front (data_all); a worker replays
    the chain from the state on entry and keeps only the runs of the batch it trains (data, _keep_only).  Batches reach
    a worker in run order within each stage, so it replays the chain at most once per stage."""
    LOCAL = ('cont', 'runs', 'chain', 'after_build', 'next_run', 'out', 'run_start')

    def __init__(self, defaults, grid, run_list, start, entry_rng):
        self.defaults, self.grid, self.run_list, self.start, self.entry_rng = defaults, grid, run_list, start, entry_rng
        self.point_params = [SimpleNamespace(**dict(defaults, **point)) for point in grid]
        self.entries = [(ri, g, v) for ri in range(len(run_list)) for g in range(len(grid))
                        for v in range(self.point_params[g].num_runs_val)]
        self._local()

    def _local(self):
        self.cont = self.chain = self.after_build = None
        self.runs, self.out, self.run_start, self.next_run = {}, {}, {}, 0

    def describe(self, method, i):
        if method == 'final':
            return 'the final training of run %s' % self.run_list[i]
        ri, g, v = self.entries[i]
        return 'tuning training (run %s, point %d %s, repetition %d)' % (self.run_list[ri], g, self.grid[g], v)

    def _draw(self):
        """The next run's data from the current random state: (tune tasks, tune loaders, final tasks, final loaders)."""
        from continuum.data_utils import setup_test_loader
        p = self.defaults
        num_val, train_val = p['num_val'], p['train_val']
        self.cont.new_run()
        loaders = setup_test_loader(self.cont.test_data(), SimpleNamespace(**p))
        tasks = [(x, y) for x, y, _ in self.cont]
        final = tasks if train_val else tasks[num_val:]
        final_loaders = loaders if train_val else loaders[num_val:]
        if p['online']:
            return tasks[:num_val], loaders[:num_val], final, final_loaders
        # the final concatenation is made when its training starts
        return _concat(tasks[:num_val]), loaders[:num_val], (lambda f=final: _concat(f)), final_loaders

    def data_all(self, cont, keep=True):
        """Every run's data, in run order, from the caller's random state, as the in-process driver draws them (and
        prints what the draws print).  keep=False drops each run's lists once drawn: the driver does that when workers
        train, so that its output and the caller's random state afterwards are the in-process ones."""
        self.cont = cont
        for ri in range(len(self.run_list)):
            d = self._draw()
            if keep:
                self.runs[ri] = d
            del d
        if not keep:
            self.cont = None

    def _keep_only(self, ris):
        """Drop the lists of every run but `ris` (all of them in process, where one call trains every run)."""
        self.runs = {ri: d for ri, d in self.runs.items() if ri in ris}

    def data(self, ri):
        if ri not in self.runs:
            keep = RunRng.capture()
            try:
                if self.cont is None:
                    self.cont, self.chain = self._continuum(SimpleNamespace(**self.defaults))
                    self.after_build, self.next_run = self.chain, 0
                elif self.next_run > ri:                         # a run already passed: restart the chain
                    self.cont.cur_run, self.next_run, self.chain = -1, 0, self.after_build
                self.chain.swap_in()
                while self.next_run <= ri:                       # runs before ri are drawn and dropped
                    d = self._draw()
                    if self.next_run == ri:
                        self.runs[ri] = d
                    self.next_run += 1
                self.chain = RunRng.capture()
            finally:
                keep.swap_in()
        return self.runs[ri]

    def build(self, params):
        from utils.name_match import agents
        from utils.setup_elements import setup_opt, setup_architecture
        from utils.utils import maybe_cuda
        model = maybe_cuda(setup_architecture(params), params.cuda)
        opt = setup_opt(params.optimizer, model, params.learning_rate, params.weight_decay)
        return agents[params.agent](model, opt, params)

    # stage 1: every (run, point, repetition), in that order
    def tune_begin(self, i):
        ri, g, v = self.entries[i]
        self.run_start.setdefault(ri, time.time())
        self.out[i] = ([str(len(self.grid))] if g == 0 and v == 0 else []) + ([str(self.grid[g])] if v == 0 else [])

    def tune_task(self, i, t, x, y):
        self.out[i] += ['-----------tune run {} task {}-------------'.format(self.entries[i][2], t),
                        'size: {}, {}'.format(x.shape, y.shape)]

    def tune_end(self, i, acc):
        self.out[i].append('-----------tune run {}-----------avg_end_acc {}-----------'.format(
            self.entries[i][2], np.mean(acc[-1])))
        print('\n'.join(self.out.pop(i)))

    def tune(self, i0, i1, R, outs=None):
        ents = self.entries[i0:i1]
        self._keep_only(set(ri for ri, _, _ in ents))
        return run_group([self.data(ri)[0] for ri, _, _ in ents], [self.data(ri)[1] for ri, _, _ in ents],
                         lambda i: self.build(self.point_params[self.entries[i][1]]), R, first_run=i0,
                         seeds=[tune_seed(self.defaults['seed'], self.run_list[ri], g, v) for ri, g, v in ents],
                         before_run=self.tune_begin, on_task=self.tune_task, on_run_end=self.tune_end, stdout=outs,
                         checkpoint=self._checkpoint('tune'))

    # stage 2: each run's final agent, with its chosen point
    def final(self, r0, r1, R, outs=None, params_keep=(), default_params=None):
        """Stage 2 for runs r0..r1-1.  default_params, when given (in process), gets each run's point written into it
        before that run's final agent is built, as the reference does."""
        num_val, online, train_val = self.defaults['num_val'], self.defaults['online'], self.defaults['train_val']

        def begin(ri):
            self.out[ri] = ['Tuning is done. Best hyper parameter set is {}'.format(params_keep[ri]), 'Training Start']

        def task(ri, t, x, y):
            if online:
                self.out[ri] += ['----------run {} training batch {}-------------'.format(
                    self.run_list[ri], t if train_val else t + num_val)]
            else:
                self.out[ri] += ['----------run {} training-------------'.format(self.run_list[ri])]
            self.out[ri] += ['size: {}, {}'.format(x.shape, y.shape)]

        def end(ri, acc):
            self.out[ri].append('-----------run {}-----------avg_end_acc {}-----------train time {}'.format(
                self.run_list[ri], np.mean(acc[-1]), time.time() - self.run_start.get(ri, self.start)))
            print('\n'.join(self.out.pop(ri)))

        def make(ri):
            if default_params is not None:
                vars(default_params).update(params_keep[ri])
            return self.build(SimpleNamespace(**dict(self.defaults, **params_keep[ri])))

        ris = range(r0, r1)
        self._keep_only(set(ris))
        return run_group([self.data(ri)[2] for ri in ris], [self.data(ri)[3] for ri in ris], make, R,
                         first_run=r0, seeds=[run_seed(self.defaults['seed'], self.run_list[ri]) for ri in ris],
                         before_run=begin, on_task=task, on_run_end=end, stdout=outs,
                         checkpoint=self._checkpoint('final'))


def _concat(tasks):
    return [(np.concatenate([x for x, _ in tasks], axis=0), np.concatenate([y for _, y in tasks], axis=0))]


def multiple_run_tune_separate(default_params, tune_params, save_path, n_concurrent=None, devices=None,
                               checkpoint_dir=None):
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
    last run's chosen point.

    With worker devices (B200OCL_RUN_DEVICES, or `devices`) both stages are trained by one WorkerPool, R at a time in
    each worker, and each training's lines are printed in training order.  This process still draws every run's data,
    in run order, printing what the draws print, but keeps no run's lists; each worker replays the chain of draws from
    the caller's random state on entry, silently, and keeps the runs it is given.  default_params gets the last run's
    point once every final training has ended.

    With a checkpoint directory (B200OCL_CHECKPOINT_DIR, or `checkpoint_dir`; '' turns it off) both stages resume from
    it (checkpoint.py): its fingerprint, the grid included, is checked before anything is built."""
    from continuum.continuum import continuum
    from experiment.metrics import compute_performance
    from utils.io import check_ram_usage, load_yaml

    R = concurrent_runs() if n_concurrent is None else int(n_concurrent)
    devices = run_devices() if devices is None else tuple(devices)
    check_concurrent(R, devices=devices)
    if devices:
        check_device_count(devices)
    directory, async_write = _open_checkpoint(checkpoint_dir, default_params, grid=tune_params)
    entry_rng = RunRng.capture()
    start = time.time()
    print('Setting up data stream')
    data_continuum = continuum(default_params.data, default_params.cl_type, default_params)
    data_end = time.time()
    print('data setup time: {}'.format(data_end - start))
    if default_params.num_val == -1:
        default_params.num_val = data_continuum.data_object.task_nums
    num_val, train_val = default_params.num_val, default_params.train_val
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
    recipe = _Tuning(dict(vars(default_params)), grid, run_list, start, entry_rng)
    recipe.checkpoint_dir, recipe.checkpoint_async = directory, async_write

    def choose(tune_acc):
        """The chosen points, as tune_hyper chooses them."""
        params_keep = []
        for ri in range(len(run_list)):
            tune_accs = []
            for g in range(len(grid)):
                accs = np.array([a for (rj, gj, _), a in zip(recipe.entries, tune_acc) if (rj, gj) == (ri, g)])
                tune_accs.append(compute_performance(accs)[0][0])
            params_keep.append(grid[tune_accs.index(max(tune_accs))])
        return params_keep

    if devices:
        from . import registry
        recipe.data_all(data_continuum, keep=False)
        del data_continuum
        with WorkerPool(devices, recipe, R, registry.installed_extra) as pool:
            params_keep = choose(pool.map('tune', len(recipe.entries)))
            accuracy_list = pool.map('final', len(run_list), (params_keep,))
        vars(default_params).update(params_keep[-1])  # the final agents were built in the workers
    else:
        recipe.data_all(data_continuum)
        params_keep = choose(recipe.tune(0, len(recipe.entries), R))
        accuracy_list = recipe.final(0, len(run_list), R, params_keep=params_keep, default_params=default_params)
        if directory is not None:
            vars(default_params).update(params_keep[-1])    # the last run's final agent may come from a record
    end = time.time()
    result = {'seed': default_params.seed, 'time': end - start, 'acc_array': np.array(accuracy_list),
              'ram': check_ram_usage(), 'best_params': params_keep}
    with open(table_path + '/' + save_path, 'wb') as f:
        pickle.dump(result, f)
    print('----------- Total {} run: {}s -----------'.format(default_params.num_runs, end - start))
    print('----------- Seed {} RAM: {}s -----------'.format(default_params.seed, result['ram']))
