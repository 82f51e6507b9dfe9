"""Resume an interrupted experiment from its last finished task (B200OCL_CHECKPOINT_DIR=<dir>).

multirun.run_group, the loop every driver and every worker goes through, writes into the directory as it trains:
  * after the evaluation of task t of a training (a run, or a tuning training), that training's snapshot: its random
    state and host state (multirun.RunRng, memory.RunHostState) at the task boundary, its agent's snapshot() (engine
    arenas, optimizer and regulariser arenas, teacher, memory, label bookkeeping) and its accuracy rows so far.  Only the
    latest snapshot of a training is kept;
  * once its last evaluation is done, its record: the accuracy array and the text its per-run line printed.  Its
    snapshot is then deleted.
A driver started again on the same directory does not train the trainings that have a record (their arrays and lines
come back in training order), restarts those that have a snapshot at the task after it, and starts the rest from
scratch.  Every training draws from its own seeded random state and its own data, so the results are those of an
experiment that was never interrupted, bit for bit.

Layout: <dir>/fingerprint.pkl, then one directory per stage ('runs' for multiple_run, 'tune' and 'final' for
multiple_run_tune_separate) holding run<i>.snapshot and run<i>.record, i the training's index in its stage.  Every file
is written to a temporary name and moved into place with os.replace, so an interruption leaves the previous file whole.
"""
import hashlib
import os
import pickle

from . import _native, memory

ENV = 'B200OCL_CHECKPOINT_DIR'
FINGERPRINT = 'fingerprint.pkl'


class CheckpointError(RuntimeError):
    """A file of the checkpoint directory that cannot be read."""


def checkpoint_dir(environ=None):
    """The directory of B200OCL_CHECKPOINT_DIR, or None when it is unset or empty (surrounding blanks are dropped)."""
    raw = (os.environ if environ is None else environ).get(ENV, '').strip()
    return raw or None


def check_checkpoint(directory, grad_sync=None):
    """The refusals of checkpointing, raised before anything is built, for the reasons multirun.check_concurrent gives:
    parity mode replays the reference's one chain of global draws across all runs, which a run resumed from its own
    state cannot continue; data-parallel gradient sync makes every step a collective over ranks."""
    if not directory:
        return
    from . import multirun
    grad_sync = multirun._data_parallel() if grad_sync is None else grad_sync
    if memory.parity():
        raise ValueError('B200OCL_MODE=parity replays the reference\'s single random stream across all runs; a run '
                         'cannot resume from its own state (%s=%s)' % (ENV, directory))
    if grad_sync:
        raise ValueError('data-parallel gradient sync cannot be combined with resumable runs (%s=%s)' % (ENV, directory))


def engine_build():
    """The engine build a directory's results come from: the SHA-256 of libb200ocl.so."""
    if not os.path.exists(_native.LIB_PATH):
        raise _native.NativeError('%s is missing: build it with `python __graft_entry__.py`' % _native.LIB_PATH)
    h = hashlib.sha256()
    with open(_native.LIB_PATH, 'rb') as f:
        for block in iter(lambda: f.read(1 << 20), b''):
            h.update(block)
    return h.hexdigest()


def fingerprint(params, extra=(), grid=None, build=None):
    """What fixes an experiment's results: the params namespace (agent, plugins and seed included), the extra agents
    installed, the tuning grid (multiple_run_tune_separate) and the engine build.  Values are compared by repr()."""
    return {'params': {k: repr(v) for k, v in sorted(vars(params).items())},
            'agent': repr(getattr(params, 'agent', None)),
            'plugins': (repr(getattr(params, 'retrieve', None)), repr(getattr(params, 'update', None))),
            'extra': tuple(extra), 'seed': repr(getattr(params, 'seed', None)), 'grid': repr(grid),
            'engine': engine_build() if build is None else build}


def write_atomic(path, obj):
    """pickle obj to path + '.tmp', flush it to disk, then os.replace it onto path."""
    tmp = path + '.tmp'
    with open(tmp, 'wb') as f:
        pickle.dump(obj, f, protocol=pickle.HIGHEST_PROTOCOL)
        f.flush()
        os.fsync(f.fileno())
    os.replace(tmp, path)


def read(path, what):
    try:
        with open(path, 'rb') as f:
            return pickle.load(f)
    except Exception as e:
        raise CheckpointError('cannot read the %s %s: %s: %s' % (what, path, type(e).__name__, e)) from e


def open_dir(directory, fp):
    """Create `directory` holding fingerprint fp, or check the fingerprint it holds: any difference raises ValueError
    naming the entries that differ."""
    os.makedirs(directory, exist_ok=True)
    path = os.path.join(directory, FINGERPRINT)
    if not os.path.exists(path):
        write_atomic(path, fp)
        return
    old = read(path, 'fingerprint')
    if old != fp:
        keys = sorted(set(old) | set(fp)) if isinstance(old, dict) else ['fingerprint']
        diff = []
        for k in keys:
            a, b = (old.get(k), fp.get(k)) if isinstance(old, dict) else (old, fp)
            if k == 'params' and isinstance(a, dict) and isinstance(b, dict):
                diff += ['params.%s: %s -> %s' % (n, a.get(n), b.get(n)) for n in sorted(set(a) | set(b))
                         if a.get(n) != b.get(n)]
            elif a != b:
                diff.append('%s: %s -> %s' % (k, a, b))
        raise ValueError('%s=%s holds an experiment with other settings (%s); use another directory or empty this one'
                         % (ENV, directory, '; '.join(diff)))


class Checkpoint(object):
    """The files of one stage of a checkpoint directory.  Picklable (two strings): it travels to worker processes."""

    def __init__(self, directory, stage):
        self.directory, self.stage = directory, stage

    def _path(self, i, kind):
        return os.path.join(self.directory, self.stage, 'run%d.%s' % (i, kind))

    def _load(self, i, kind):
        path = self._path(i, kind)
        return read(path, kind) if os.path.exists(path) else None

    def record(self, i):
        """(accuracy array, printed text) of training i once it has ended, else None."""
        rec = self._load(i, 'record')
        if rec is not None and (not isinstance(rec, dict) or not {'acc', 'text'} <= set(rec)):
            raise CheckpointError('%s is not a record' % self._path(i, 'record'))
        return None if rec is None else (rec['acc'], rec['text'])

    def snapshot(self, i):
        """Training i's latest snapshot (a dict, 'task' the last task it finished), else None."""
        snap = self._load(i, 'snapshot')
        if snap is not None and (not isinstance(snap, dict) or not {'task', 'acc', 'rng', 'sampler', 'agent'} <= set(snap)):
            raise CheckpointError('%s is not a snapshot' % self._path(i, 'snapshot'))
        return snap

    def save_snapshot(self, i, state):
        os.makedirs(os.path.join(self.directory, self.stage), exist_ok=True)
        write_atomic(self._path(i, 'snapshot'), state)

    def save_record(self, i, acc, text):
        os.makedirs(os.path.join(self.directory, self.stage), exist_ok=True)
        write_atomic(self._path(i, 'record'), {'acc': acc, 'text': text})
        try:
            os.remove(self._path(i, 'snapshot'))
        except FileNotFoundError:
            pass
