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

With B200OCL_CHECKPOINT_ASYNC=1 as well, snapshots and records are written behind the run (Staging, _Writer).  At a task
boundary the host state is captured as above and the agent's device arrays (snapshot_parts()) are packed into the run's
staging arena by one kernel on the run's stream (b200ocl_snapshot_pack); training goes on at once.  A background thread
waits for the pack, moves the arena to the host through a small pinned ring and writes the file: a magic line, a small
pickled header, then the raw arrays.  Replay-memory rows whose every value is u / 255 for a byte u are stored at one
byte per value; any other value keeps the segment fp32.  Records go through the same queue, so a training's record is
never overtaken by its earlier snapshot.  The files hold the same state as synchronous ones (Checkpoint.snapshot()
reads both, and a directory resumes with the switch on or off).
"""
import collections
import hashlib
import os
import pickle
import threading
import time
import traceback

import numpy as np
import torch

from . import _native, memory

ENV = 'B200OCL_CHECKPOINT_DIR'
ASYNC_ENV = 'B200OCL_CHECKPOINT_ASYNC'
FINGERPRINT = 'fingerprint.pkl'
MAGIC = b'B200OCL staged snapshot 1\n'   # first bytes of a staged snapshot file; a synchronous one is a pickle
MAX_SEGMENTS = 64                         # device arrays of one snapshot (an agent has at most 17)
CHUNK = 8 << 20                           # bytes per device-to-host copy of the writer's pinned ring
PAD = 256                                 # a staged file's segments start at multiples of PAD in its payload (and in
                                          # the staging arena, so that a restore's single copy keeps them aligned)


def _padded(n):
    return (n + PAD - 1) // PAD * PAD


class CheckpointError(RuntimeError):
    """A file of the checkpoint directory that cannot be read."""


def checkpoint_dir(environ=None):
    """The directory of B200OCL_CHECKPOINT_DIR, or None when it is unset or empty (surrounding blanks are dropped)."""
    raw = (os.environ if environ is None else environ).get(ENV, '').strip()
    return raw or None


def checkpoint_async(environ=None, directory=None):
    """B200OCL_CHECKPOINT_ASYNC: False when unset, empty or '0', True for '1'.  Any other value raises ValueError, and
    so does '1' without a checkpoint directory (`directory`, else B200OCL_CHECKPOINT_DIR)."""
    env = os.environ if environ is None else environ
    raw = env.get(ASYNC_ENV, '').strip()
    if raw in ('', '0'):
        return False
    if raw != '1':
        raise ValueError('%s must be 0 or 1, got %r' % (ASYNC_ENV, raw))
    if (directory or checkpoint_dir(env)) is None:
        raise ValueError('%s=1 writes the snapshots of %s behind the run, but %s is not set' % (ASYNC_ENV, ENV, ENV))
    return True


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
    """The files of one stage of a checkpoint directory.  Picklable (two strings and a flag): it travels to worker
    processes.  async_write: snapshots are staged (Staging) and they and the records are written by the process's
    writer thread."""

    def __init__(self, directory, stage, async_write=False):
        self.directory, self.stage, self.async_write = directory, stage, bool(async_write)

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

    def snapshot(self, i, staging=None):
        """Training i's latest snapshot (a dict, 'task' the last task it finished), else None.  Both forms are read: a
        pickle (synchronous writes) and a staged file.  A staged file's arrays are host tensors, decoded here, or, with
        a `staging` that has a device arena, device tensors decoded by b200ocl_snapshot_unpack on the current stream."""
        path = self._path(i, 'snapshot')
        if not os.path.exists(path):
            return None
        try:
            with open(path, 'rb') as f:
                staged = f.read(len(MAGIC)) == MAGIC
        except OSError as e:
            raise CheckpointError('cannot read the snapshot %s: %s: %s' % (path, type(e).__name__, e)) from e
        if staged:
            try:
                snap = _read_staged(path, staging)
            except CheckpointError:
                raise
            except Exception as e:
                raise CheckpointError('cannot read the snapshot %s: %s: %s' % (path, type(e).__name__, e)) from e
        else:
            snap = read(path, 'snapshot')
        if not isinstance(snap, dict) or not {'task', 'acc', 'rng', 'sampler', 'agent'} <= set(snap):
            raise CheckpointError('%s is not a snapshot' % path)
        return snap

    def save_snapshot(self, i, state):
        os.makedirs(os.path.join(self.directory, self.stage), exist_ok=True)
        write_atomic(self._path(i, 'snapshot'), state)

    def save_staged(self, i, state, job):
        """Queue the write of a staged snapshot: `state` is the run's snapshot with the agent's device arrays replaced
        by placeholders, `job` what Staging.stage() returned for them.  If it cannot be queued the job is ended, so
        that nothing waits for it."""
        try:
            os.makedirs(os.path.join(self.directory, self.stage), exist_ok=True)
            job.path, job.state = self._path(i, 'snapshot'), pickle.dumps(state, protocol=pickle.HIGHEST_PROTOCOL)
            writer().submit(job.run, job.path, job.done)
        except BaseException:
            job.release()
            job.done.set()
            raise

    def save_record(self, i, acc, text):
        if self.async_write:
            writer().check()
            writer().submit(lambda: self._save_record(i, acc, text), self._path(i, 'record'))
        else:
            self._save_record(i, acc, text)

    def _save_record(self, i, acc, text):
        os.makedirs(os.path.join(self.directory, self.stage), exist_ok=True)
        write_atomic(self._path(i, 'record'), {'acc': acc, 'text': text})
        try:
            os.remove(self._path(i, 'snapshot'))
        except FileNotFoundError:
            pass


# --------------------------------------------------------------------------- staged snapshots (B200OCL_CHECKPOINT_ASYNC)
class _Segment(object):
    """The place of the index-th device array in a staged snapshot's state."""
    __slots__ = ('index',)

    def __init__(self, index):
        self.index = index

    def __getstate__(self):
        return self.index

    def __setstate__(self, index):
        self.index = index


def _split(tree, segs, device=None):
    """`tree` (a snapshot_parts() tree) with every tensor replaced by a _Segment; segs gets (tensor, 8-bit candidate).
    With a device, tensors elsewhere (host state of a plugin that only has snapshot()) stay in the tree as copies."""
    if isinstance(tree, dict):
        return {k: _split(v, segs, device) for k, v in tree.items()}
    if isinstance(tree, (memory.Rows8, torch.Tensor)):
        t = (tree.tensor if isinstance(tree, memory.Rows8) else tree).detach()
        if device is not None and t.device != device:
            return t.clone()
        segs.append((t, isinstance(tree, memory.Rows8) and t.dtype == torch.float32))
        return _Segment(len(segs) - 1)
    return tree


def _fill(tree, arrays):
    if isinstance(tree, dict):
        return {k: _fill(v, arrays) for k, v in tree.items()}
    if isinstance(tree, _Segment):
        return arrays[tree.index]
    return tree


def _dtype(name):
    return getattr(torch, name)


def _read_staged(path, staging=None):
    """A staged snapshot file as the dict the run wrote, its arrays decoded (u / 255 for 8-bit segments)."""
    with open(path, 'rb') as f:
        f.read(len(MAGIC))
        header = pickle.loads(f.read(int.from_bytes(f.read(8), 'little')))
        payload = f.read()
    segs = header['segments']                                        # [(dtype, shape, bytes, stored at 8 bits)]
    sizes = [n // 4 if u8 else n for _, _, n, u8 in segs]
    if len(payload) != sum(_padded(n) for n in sizes):
        raise CheckpointError('%s holds %d payload bytes, its header %d' % (path, len(payload),
                                                                           sum(_padded(n) for n in sizes)))
    state = pickle.loads(header['state'])
    arrays, off = [], 0
    if staging is not None and staging.arena is not None:
        from . import ops
        if len(payload) > staging.arena.numel() or len(segs) > MAX_SEGMENTS:
            raise CheckpointError('%s does not fit the run\'s staging arena' % path)
        dev = staging.arena.device
        staging.arena[:len(payload)].copy_(torch.frombuffer(bytearray(payload), dtype=torch.uint8))
        table = np.zeros(len(segs), ops.SNAP_SEGMENT)
        for k, ((dtype, shape, n, u8), size) in enumerate(zip(segs, sizes)):
            arrays.append(torch.empty(shape, dtype=_dtype(dtype), device=dev))
            table[k] = (arrays[-1].data_ptr(), n, off, ops.SNAP_U8 if u8 else ops.SNAP_COPY, 0)
            off += _padded(size)
        ops.snapshot_unpack(memory.to_device(table.view(np.uint8), dev), len(segs), staging.arena, staging.ws)
        if int(staging.ws[:4 * (len(segs) + 1)].view(torch.int32)[-1]) != 0:
            raise CheckpointError('%s: the staging arena refused a segment' % path)
    else:
        for (dtype, shape, n, u8), size in zip(segs, sizes):
            raw = np.frombuffer(payload, dtype=np.uint8, count=size, offset=off)
            if u8:
                arrays.append(torch.from_numpy(raw.astype(np.float32) / np.float32(255)).reshape(shape))
            else:
                arrays.append(torch.frombuffer(bytearray(raw), dtype=_dtype(dtype)).reshape(shape))
            off += _padded(size)
    state['agent'] = _fill(state['agent'], arrays)
    return state


class _Job(object):
    """One staged snapshot on its way to its file."""

    def __init__(self, staging, layout, keep, event):
        """keep: the host copies of the arrays (no device arena), else the device segment table the pack reads."""
        self.staging, self.layout, self.keep, self.event = staging, layout, keep, event
        self.path = self.state = None
        self.done = threading.Event()

    def run(self):
        """What the writer runs: write(), then drop the links to the staging arena and the arrays, whether or not the
        write succeeded, so that the arena goes as soon as its run lets go of it."""
        try:
            self.write()
        finally:
            self.release()

    def release(self):
        self.staging = self.keep = self.event = None

    def write(self):
        """The writer's part: wait for the pack, learn each 8-bit segment's form from its counter, then write the file
        chunk by chunk as the chunks land in the pinned ring."""
        st = self.staging
        n = len(self.layout)
        u8 = [False] * n
        if st.arena is not None:
            from .engine import capture_lock
            while True:                                 # the pack; see _Writer._put
                with capture_lock:
                    if self.event.query():
                        break
                time.sleep(2e-4)
            with capture_lock, torch.cuda.stream(writer().stream(st.arena.device)):
                counters = st.ws[:4 * (n + 1)].view(torch.int32).to('cpu').numpy()
            if counters[n] != 0:
                raise CheckpointError('%d segment(s) did not fit the staging arena' % counters[n])
            u8 = [seg['u8'] and counters[k] == 0 for k, seg in enumerate(self.layout)]
        sizes = [seg['bytes'] // 4 if e else seg['bytes'] for seg, e in zip(self.layout, u8)]
        header = pickle.dumps({'state': self.state, 'segments': [(seg['dtype'], seg['shape'], seg['bytes'], e)
                                                                 for seg, e in zip(self.layout, u8)]},
                              protocol=pickle.HIGHEST_PROTOCOL)
        tmp = self.path + '.tmp'
        with open(tmp, 'wb') as f:
            f.write(MAGIC)
            f.write(len(header).to_bytes(8, 'little'))
            f.write(header)
            if st.arena is None:
                for t, size in zip(self.keep, sizes):
                    f.write(memoryview(t.reshape(-1).view(torch.uint8).numpy()))
                    f.write(bytes(_padded(size) - size))
            else:
                writer().copy_out(f, st.arena, [(seg['offset'], size) for seg, size in zip(self.layout, sizes)])
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, self.path)
        stats['snapshots'] += 1
        stats['bytes'] += len(MAGIC) + 8 + len(header) + sum(_padded(n) for n in sizes)


stats = {'snapshots': 0, 'bytes': 0, 'backpressure_s': 0.0}   # staged snapshots written, their bytes, time waited


class Staging(object):
    """A run's staging arena on its device: capacity bytes plus room to align every segment, and the pack workspace.
    Built with the run, before its first step, so that a device without room for it fails there.  A run whose
    snapshot_parts() tensors are host tensors (no device) stages copies of them instead."""

    def __init__(self, capacity, device):
        self.arena = self.ws = None
        self.pending = None             # the last job staged here, until the writer is done with the arena
        device = torch.device(device)
        if device.type == 'cuda':
            from . import ops
            nbytes = int(capacity) + MAX_SEGMENTS * PAD
            try:
                self.arena = torch.empty(nbytes, dtype=torch.uint8, device=device)
                self.ws = ops.snapshot_workspace(MAX_SEGMENTS, device)
            except torch.OutOfMemoryError as e:
                raise torch.OutOfMemoryError('%s=1: no room on %s for a run\'s %d-byte snapshot staging arena; unset it '
                                             'to write snapshots synchronously' % (ASYNC_ENV, device, nbytes)) from e

    def wait(self):
        """Back-pressure: wait until the writer is done with the previous snapshot staged here (counted in stats)."""
        if self.pending is not None:
            if not self.pending.done.is_set():
                t0 = time.perf_counter()
                self.pending.done.wait()
                stats['backpressure_s'] += time.perf_counter() - t0
            self.pending = None

    def release(self):
        """At the end of the run: wait for its last snapshot's write, then free the arena."""
        self.wait()
        self.arena = self.ws = None

    def stage(self, parts):
        """Under the run's stream, at a task boundary: pack the device arrays of `parts` (a snapshot_parts() tree) into
        the arena and record an event after the pack.  Returns (the tree with placeholders, the job to write).  A
        failed earlier write raises here, before anything is packed."""
        self.wait()
        writer().check()
        segs = []
        tree = _split(parts, segs, None if self.arena is None else self.arena.device)
        layout, off = [], 0
        for t, u8 in segs:
            if not t.is_contiguous():
                raise ValueError('a snapshot array must be contiguous, got shape %s strides %s' % (tuple(t.shape),
                                                                                                  t.stride()))
            n = t.numel() * t.element_size()
            layout.append({'dtype': str(t.dtype).replace('torch.', ''), 'shape': tuple(t.shape), 'bytes': n,
                           'offset': off, 'u8': u8})
            off += _padded(n)
        if self.arena is None:
            job = _Job(self, layout, [t.clone() for t, _ in segs], None)
        else:
            from . import ops
            if len(segs) > MAX_SEGMENTS or off > self.arena.numel():
                raise ValueError('a snapshot of %d arrays and %d bytes does not fit the staging arena (%d arrays, %d '
                                 'bytes)' % (len(segs), off, MAX_SEGMENTS, self.arena.numel()))
            table = np.zeros(len(segs), ops.SNAP_SEGMENT)
            for k, ((t, _), seg) in enumerate(zip(segs, layout)):
                if t.device != self.arena.device:
                    raise ValueError('snapshot array on %s, staging arena on %s' % (t.device, self.arena.device))
                table[k] = (t.data_ptr(), seg['bytes'], seg['offset'], ops.SNAP_U8 if seg['u8'] else ops.SNAP_COPY, 0)
            dev_table = memory.to_device(table.view(np.uint8), self.arena.device)
            ops.snapshot_pack(dev_table, len(segs), self.arena, self.ws)
            event = torch.cuda.Event()
            event.record()
            job = _Job(self, layout, dev_table, event)
        self.pending = job
        return tree, job


class _Writer(object):
    """The process's one writer thread: a FIFO of writes (staged snapshots and records, of every training), done in
    submission order, so a training's record always follows its earlier snapshots.  The first failure is kept and
    raised by check() (at the next boundary or drain) as CheckpointError naming the file."""

    def __init__(self):
        self.queue = collections.deque()
        self.cv = threading.Condition()
        self.thread = None
        self.error = None
        self.streams, self.rings = {}, {}

    def submit(self, fn, path, done=None):
        with self.cv:
            self.queue.append((fn, path, done))
            if self.thread is None or not self.thread.is_alive():
                self.thread = threading.Thread(target=self._loop, name='b200ocl-checkpoint-writer', daemon=True)
                self.thread.start()
            self.cv.notify_all()

    def _loop(self):
        while True:
            with self.cv:
                while not self.queue:
                    self.cv.wait()
                fn, path, done = self.queue[0]
            try:
                fn()
            except BaseException as e:                 # kept for check(); the queue goes on
                traceback.clear_frames(e.__traceback__)  # its frames' locals would keep the staging arena alive
                with self.cv:
                    if self.error is None:
                        self.error = (path, e)
            finally:
                fn = None                              # nothing of a finished write outlives it here
                if done is not None:
                    done.set()
                with self.cv:
                    self.queue.popleft()
                    self.cv.notify_all()

    def drain(self, check=True):
        """Wait until every queued write has ended.  Then the first failure, if any, is taken: raised with check,
        else returned (None when there was none)."""
        with self.cv:
            while self.queue:
                self.cv.wait()
        err = self._take_error()
        if check and err is not None:
            raise err
        return err

    def check(self):
        """Raise the first failed write, if any, once."""
        err = self._take_error()
        if err is not None:
            raise err

    def _take_error(self):
        with self.cv:
            err, self.error = self.error, None
        if err is None:
            return None
        path, e = err
        out = CheckpointError('cannot write %s: %s: %s' % (path, type(e).__name__, e))
        out.__cause__ = e
        return out

    def stream(self, device):
        if device not in self.streams:
            self.streams[device] = torch.cuda.Stream(device)
        return self.streams[device]

    def copy_out(self, f, arena, regions):
        """Write arena[offset:offset + size] for each region to f, through two pinned CHUNK-byte buffers on the
        writer's stream: a chunk is written while the next one is being copied."""
        from .engine import capture_lock
        dev = arena.device
        with capture_lock:
            if dev not in self.rings:
                self.rings[dev] = [(torch.empty(CHUNK, dtype=torch.uint8).pin_memory(), torch.cuda.Event())
                                   for _ in range(2)]
            ring, stream = self.rings[dev], self.stream(dev)
        # (offset, bytes, zero bytes after them): a region's last piece is followed by its padding to PAD
        pieces = [(a + c, min(CHUNK, size - c), _padded(size) - size if c + CHUNK >= size else 0)
                  for a, size in regions for c in range(0, size, CHUNK)]
        prev = None
        for k, (a, m, pad) in enumerate(pieces):
            buf, ev = ring[k % 2]
            with capture_lock, torch.cuda.stream(stream):
                buf[:m].copy_(arena[a:a + m], non_blocking=True)
                ev.record(stream)
            if prev is not None:
                self._put(f, *prev)
            prev = (buf, ev, m, pad)
        if prev is not None:
            self._put(f, *prev)

    @staticmethod
    def _put(f, buf, ev, m, pad):
        """Wait for a chunk (an event query loop: a synchronise could start while a graph is being captured) and write
        it, then `pad` zero bytes."""
        from .engine import capture_lock
        while True:
            with capture_lock:
                if ev.query():
                    break
            time.sleep(2e-4)
        f.write(memoryview(buf.numpy())[:m])
        f.write(bytes(pad))


_writer = None
_writer_lock = threading.Lock()


def writer():
    """The writer of this process (created on first use)."""
    global _writer
    with _writer_lock:
        if _writer is None:
            _writer = _Writer()
        return _writer
