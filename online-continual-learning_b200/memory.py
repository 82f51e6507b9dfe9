"""Replay memory: the Buffer tensor store, uniform retrieval and class-balanced sampling, and GDumb's greedy
class-balanced memory (GreedyBalancedMemory, agents/gdumb.py:19-31).

Mirrors the reference surface (utils/buffer/buffer.py:8-41; utils/buffer/buffer_utils.py:9-26,
74-160) with a different split of work:
  * images and labels live on the GPU as in the reference ([mem,3,H,W] fp32, [mem] int64);
  * every *decision* about indices is taken on the host from a numpy mirror of the labels
    (no .item()/.tolist() round trips per sample: the reference does ~5000 of them to rebuild
    its class cache, buffer_utils.py:156-160);
  * rows move with the gather/scatter kernels of csrc/misc.cu.
"""
import os
import random
from collections import defaultdict

import numpy as np
import torch

from . import ops

# --------------------------------------------------------------------------- parity mode
# B200OCL_MODE=parity (or set_mode(True)) makes every random decision of the replay path consume the SAME
# generators, with the same calls in the same order, as the reference: per-class torch.randperm on the
# sampler's device in dict insertion order over Python sets built by the same add/remove history
# (buffer_utils.py:105-113), the reservoir's float32 uniform_ on x's device (reservoir_update.py:35) and a
# real DataLoader(shuffle=True) for the stream order.  A seeded reference run and a seeded b200ocl run then
# retrieve and evict the same slots without injected choices.  It costs what the reference's version costs
# (Python loops, device->host syncs), so it is a verification mode; the default mode draws from vectorised
# host generators (statistically identical, not stream-identical).
# B200OCL_PARITY_RNG=cpu pins the generators to the CPU (to replay a reference run that was recorded on a
# machine without a GPU); default: the device the reference would use (cuda when available).
_mode = {'parity': os.environ.get('B200OCL_MODE', '').lower() == 'parity',
         'rng': os.environ.get('B200OCL_PARITY_RNG', '').lower()}


def set_mode(parity, rng_device=None):
    _mode['parity'] = bool(parity)
    _mode['rng'] = (rng_device or '').lower()


def parity():
    return _mode['parity']


def parity_rng_device(natural=None):
    """Device of the reference's generator for a draw it makes on `natural` (default: its self.device)."""
    if _mode['rng'] == 'cpu':
        return torch.device('cpu')
    if natural is not None:
        return torch.device(natural)
    return torch.device('cuda' if torch.cuda.is_available() else 'cpu')

input_size_match = {      # utils/setup_elements.py:11-17
    'cifar100': [3, 32, 32], 'cifar10': [3, 32, 32], 'core50': [3, 128, 128],
    'mini_imagenet': [3, 84, 84], 'openloris': [3, 50, 50],
}
n_classes = {             # utils/setup_elements.py:20-26
    'cifar100': 100, 'cifar10': 10, 'core50': 50, 'mini_imagenet': 100, 'openloris': 69,
}


# --------------------------------------------------------------------------- host index logic
def class_balanced_indices(labels, n_valid, n_smp_cls, excl_mask=None, rng=None):
    """Up to n_smp_cls uniformly random slots of every class present in labels[:n_valid],
    skipping slots flagged in excl_mask.  Vectorised restatement of
    ClassBalancedRandomSampling.sample (buffer_utils.py:81-121): one random key per slot, sort
    by (class, key), keep the first n of every class.  Output is class-major (ascending class
    id), random inside a class."""
    rng = np.random if rng is None else rng
    if n_smp_cls <= 0 or n_valid <= 0:
        return np.zeros(0, dtype=np.int64)
    valid = np.arange(n_valid) if excl_mask is None else np.flatnonzero(~excl_mask[:n_valid])
    if valid.size == 0:
        return np.zeros(0, dtype=np.int64)
    lab = labels[valid]
    order = np.argsort(lab + rng.random(valid.size), kind='stable')
    lab_sorted = lab[order]
    first = np.flatnonzero(np.r_[True, lab_sorted[1:] != lab_sorted[:-1]])
    counts = np.diff(np.r_[first, lab_sorted.size])
    rank = np.arange(lab_sorted.size) - np.repeat(first, counts)
    return valid[order[rank < n_smp_cls]].astype(np.int64)


def uniform_indices(n_filled, num_retrieve, excl_indices=None):
    """np.random.choice without replacement over the filled slots minus excl_indices -- the same
    draw, on the same population, as random_retrieve (buffer_utils.py:9-17), so a seeded numpy
    stream yields the reference's indices.  (The population is built with a boolean mask instead of
    np.setdiff1d: same sorted result, 40x cheaper on the host.)"""
    keep = np.ones(n_filled, dtype=bool)
    if excl_indices is not None and len(excl_indices) > 0:
        ex = np.asarray(list(excl_indices) if not isinstance(excl_indices, np.ndarray) else excl_indices, dtype=np.int64)
        keep[ex[(ex >= 0) & (ex < n_filled)]] = False
    valid = np.flatnonzero(keep)
    num_retrieve = min(num_retrieve, valid.shape[0])
    return np.random.choice(valid, num_retrieve, replace=False).astype(np.int64)


# --------------------------------------------------------------------------- host <-> device plumbing
_TORCH_DTYPE = {np.int64: torch.int64, np.int32: torch.int32, np.float32: torch.float32, np.float64: torch.float64,
                np.uint8: torch.uint8, np.bool_: torch.bool}


class _PinnedRing:
    """Pinned staging ring for small host -> device uploads (indices, labels, augmentation parameters).
    torch's pageable .to(device) synchronises the stream on every call; uploads from this ring are truly
    asynchronous, so the host keeps running ahead of the GPU.  The ring has two halves; before a half is
    reused the event recorded when it was last left is waited on (long past in practice)."""

    def __init__(self, nbytes=1 << 20):
        self.nbytes = nbytes
        self.half = nbytes // 2
        self.buf = None
        self.cur = 0                  # half being filled (tracked explicitly, never derived from an offset)
        self.used = 0                 # bytes used in that half, 0..half
        self.events = [None, None]

    def _ensure(self):
        if self.buf is None:
            self.buf = torch.empty(self.nbytes, dtype=torch.uint8).pin_memory()

    # the three hooks tests replace to drive the ring without a GPU
    def _alloc(self, shape, dtype, device):
        return torch.empty(shape, dtype=dtype, device=device)

    class _Events(list):
        def synchronize(self):
            for ev in self:
                ev.synchronize()

    def _record(self):
        """One event per stream that issued a copy out of the half being left (the learners issue work on two streams)."""
        evs = self._Events()
        for st in self.__dict__.pop('_streams', None) or [torch.cuda.current_stream()]:
            ev = torch.cuda.Event()
            ev.record(st)
            evs.append(ev)
        return evs

    def _copy(self, out, view):
        streams = self.__dict__.setdefault('_streams', [])
        cur = torch.cuda.current_stream()
        if cur not in streams:
            streams.append(cur)
        out.view(torch.uint8).reshape(-1).copy_(view, non_blocking=True)

    def reserve(self, n):
        """Byte offset of an n-byte slot (n <= half).  Leaving a half always records its event, entering
        a half always waits for the event recorded when it was last left -- including when the
        previous uploads ended exactly on the half boundary."""
        need = (n + 15) // 16 * 16
        if self.used + need > self.half:
            self.events[self.cur] = self._record()
            self.cur ^= 1
            self.used = 0
            if self.events[self.cur] is not None:
                self.events[self.cur].synchronize()
                self.events[self.cur] = None
        off = self.cur * self.half + self.used
        self.used += need
        return off

    def upload(self, arr, device):
        arr = np.ascontiguousarray(arr)
        n = arr.nbytes
        out = self._alloc(arr.shape, _TORCH_DTYPE[arr.dtype.type], device)
        if n == 0:
            return out
        self._ensure()
        if n > self.half:      # large arrays bypass the ring
            out.copy_(torch.from_numpy(arr))
            return out
        off = self.reserve(n)
        view = self.buf[off:off + n]
        view.numpy()[:] = arr.reshape(-1).view(np.uint8)
        self._copy(out, view)
        return out


_ring = _PinnedRing()


def to_device(arr, device):
    """Small host array -> device tensor of the same dtype, without a stream synchronisation."""
    arr = np.ascontiguousarray(arr)
    if torch.device(device).type != 'cuda':
        return torch.from_numpy(arr.copy())
    return _ring.upload(arr, torch.device(device))


def to_device_i64(arr, device):
    """Small host int64 array -> device tensor."""
    return to_device(np.ascontiguousarray(arr, dtype=np.int64), device)


# Host-mirror updates that depend on device results (ASER's replacement decision) are deferred: the
# decision is copied to pinned memory asynchronously and applied here, the next time any host-side
# index logic runs -- by then the copy has long completed, so nothing waits on the GPU.
_pending = []        # [(owner id or None, fn)] in submission order
_pinned_pool = []


def defer(fn, owner=None):
    """Queue a host-mirror update.  `owner` (a Buffer) scopes it: reading another buffer's mirror does not wait for it."""
    _pending.append((None if owner is None else id(owner), fn))


def flush_pending(owner=None):
    """Apply queued updates in submission order: all of them (owner=None: the class-level sampler state is shared by
    every buffer, as in the reference) or only those of one buffer."""
    if owner is None:
        while _pending:
            _pending.pop(0)[1]()
        return
    oid = id(owner)
    keep = []
    while _pending:
        o, fn = _pending.pop(0)
        if o == oid:
            fn()
        else:
            keep.append((o, fn))
    _pending.extend(keep)


class Rows8(object):
    """A replay-memory image tensor in a snapshot_parts() tree: fp32 rows that, for 8-bit streams, all hold u / 255 for
    a byte u, so a staged snapshot may store them at one byte per value (checkpoint.py)."""
    __slots__ = ('tensor',)

    def __init__(self, tensor):
        self.tensor = tensor


def host_tree(tree):
    """A snapshot_parts() tree with every tensor on the host: one synchronise of the current stream when a leaf is on
    a CUDA device, then one device-to-host copy per tensor (a host tensor is kept as it is, as .to('cpu') does)."""
    def leaves(t):
        if isinstance(t, dict):
            return [x for v in t.values() for x in leaves(v)]
        if isinstance(t, (list, tuple)):
            return [x for v in t for x in leaves(v)]
        return [t.tensor if isinstance(t, Rows8) else t]

    def host(t):
        if isinstance(t, dict):
            return {k: host(v) for k, v in t.items()}
        if isinstance(t, Rows8):
            return t.tensor.to('cpu')
        if isinstance(t, torch.Tensor):
            return t.to('cpu')
        return t
    cuda = [t for t in leaves(tree) if isinstance(t, torch.Tensor) and t.is_cuda]
    if cuda:
        torch.cuda.current_stream(cuda[0].device).synchronize()
    return host(tree)


class RunHostState(object):
    """The module-level host state of the replay path that belongs to one run when several runs share the process
    (multirun.run_group): the class-level state of ClassBalancedRandomSampling, which the buffers of one run share as
    the reference's do, and the queued host-mirror updates of that run's buffers.  enter() makes it current, leave()
    takes it back; between the two nothing else may enter.  Swapping moves references only: no copy, no device wait
    (queued updates stay queued until their own run flushes them)."""
    __slots__ = ('sampler', 'pending')

    def __init__(self):
        self.sampler = None
        self.pending = []

    def enter(self):
        if _pending:
            raise RuntimeError('host-mirror updates of another run are still queued')
        ClassBalancedRandomSampling.load_state(self.sampler)
        _pending.extend(self.pending)
        self.pending = []

    def leave(self):
        self.sampler = ClassBalancedRandomSampling.export_state()
        self.pending = list(_pending)
        del _pending[:]
        ClassBalancedRandomSampling.load_state(None)


def pinned_i64(n):
    for i, t in enumerate(_pinned_pool):
        if t.numel() >= n:
            return _pinned_pool.pop(i)
    return torch.empty(max(64, n), dtype=torch.int64).pin_memory()


def release_pinned(t):
    if len(_pinned_pool) < 8:
        _pinned_pool.append(t)


# --------------------------------------------------------------------------- class-balanced sampler
class ClassBalancedRandomSampling:
    """Class-level state like the reference (buffer_utils.py:74-79): two buffers in one process
    share it and the ASER plugin constructors reset it (aser_retrieve.py:19, aser_update.py:20).

    Besides the reference's caches the sampler keeps a slot table tab[class, position] with counts and
    each slot's position, maintained incrementally; a class-balanced draw is then one block of uniform
    keys over the table and an argmin / argpartition per row (~80 us for 5000 slots x 100 classes,
    against ~400 us for the sort-based class_balanced_indices and ~5000 .item() calls in the reference)."""
    class_index_cache = None     # dict class -> set(slot)   (kept for parity with the reference's API)
    class_num_cache = None       # np.int64 [num_class]
    labels_host = None           # np.int64 [mem] mirror the sampler draws from
    n_valid = 0
    _member = None               # bool [mem]: slot registered through update_cache
    _tab = None                  # int64 [num_class, cap]
    _cnt = None                  # int64 [num_class]
    _pos = None                  # int64 [mem]

    _STATE = ('class_index_cache', 'class_num_cache', 'labels_host', 'n_valid', '_member', '_tab', '_cnt', '_pos')

    @classmethod
    def export_state(cls):
        """The class-level state as a dict (references, no copies): load_state(export_state()) restores it."""
        return {k: getattr(cls, k) for k in cls._STATE}

    @classmethod
    def load_state(cls, state):
        """Replace the class-level state (None: the state of a sampler that was never filled)."""
        for k in cls._STATE:
            setattr(cls, k, 0 if k == 'n_valid' else None) if state is None else setattr(cls, k, state[k])

    @classmethod
    def reset(cls):
        flush_pending()
        cls.class_index_cache = None
        cls.class_num_cache = None
        cls.labels_host = None
        cls.n_valid = 0
        cls._member = None
        cls._tab = None
        cls._cnt = None
        cls._pos = None

    # ---- slot table
    @classmethod
    def _tab_add(cls, slot, c):
        if c >= cls._tab.shape[0]:
            rows = max(c + 1, 2 * cls._tab.shape[0])
            cls._tab = np.vstack([cls._tab, np.full((rows - cls._tab.shape[0], cls._tab.shape[1]), -1, dtype=np.int64)])
            cls._cnt = np.concatenate([cls._cnt, np.zeros(rows - cls._cnt.shape[0], dtype=np.int64)])
        k = int(cls._cnt[c])
        if k >= cls._tab.shape[1]:
            cls._tab = np.hstack([cls._tab, np.full((cls._tab.shape[0], max(8, cls._tab.shape[1])), -1, dtype=np.int64)])
        cls._tab[c, k] = slot
        cls._pos[slot] = k
        cls._cnt[c] = k + 1

    @classmethod
    def _tab_remove(cls, slot, c):
        k, last = int(cls._pos[slot]), int(cls._cnt[c]) - 1
        moved = cls._tab[c, last]
        cls._tab[c, k] = moved
        cls._pos[moved] = k
        cls._tab[c, last] = -1
        cls._cnt[c] = last

    @classmethod
    def sample_indices(cls, n_smp_cls, excl_indices=None, rng=None):
        """Up to n_smp_cls uniformly random registered slots of every class, minus excl_indices
        (ClassBalancedRandomSampling.sample, buffer_utils.py:81-121).  Class-major output (ascending
        class id), random inside a class."""
        flush_pending()
        if cls.labels_host is None:
            raise RuntimeError('ClassBalancedRandomSampling.update_cache has not been called')
        if parity() and rng is None:
            return cls._sample_indices_parity(int(n_smp_cls), excl_indices)
        rng = np.random if rng is None else rng
        n = int(n_smp_cls)
        cap = int(cls._cnt.max()) if cls._cnt.size else 0
        if n <= 0 or cap == 0:
            return np.zeros(0, dtype=np.int64)
        C = cls._tab.shape[0]
        u = rng.random((C, cap))
        u[np.arange(cap)[None, :] >= cls._cnt[:, None]] = 2.0
        if excl_indices is not None and len(excl_indices) > 0:
            ex = np.asarray(list(excl_indices) if not isinstance(excl_indices, np.ndarray) else excl_indices, dtype=np.int64)
            ex = ex[cls._member[ex]]
            u[cls.labels_host[ex], cls._pos[ex]] = 2.0
        if n == 1:
            j = u.argmin(axis=1)
            rows = np.flatnonzero(u[np.arange(C), j] < 2.0)
            return cls._tab[rows, j[rows]].astype(np.int64)
        n_eff = min(n, cap)
        part = np.argpartition(u, n_eff - 1, axis=1)[:, :n_eff] if n_eff < cap else np.tile(np.arange(cap), (C, 1))
        keys = np.take_along_axis(u, part, axis=1)
        o = np.argsort(keys, axis=1, kind='stable')
        part, keys = np.take_along_axis(part, o, axis=1), np.take_along_axis(keys, o, axis=1)
        return cls._tab[np.arange(C)[:, None], part][keys < 2.0].astype(np.int64)

    @classmethod
    def _sample_indices_parity(cls, n, excl_indices):
        """The reference's own loop (buffer_utils.py:100-113): classes in dict insertion order, the set
        difference iterated in CPython set order, one torch.randperm per non-empty class on the sampler's
        device.  One device -> host copy at the end."""
        dev = parity_rng_device()
        excl = set() if excl_indices is None else set(int(i) for i in np.asarray(list(excl_indices)).tolist())
        parts = [torch.tensor([], device=dev, dtype=torch.long)]
        for ind_set in cls.class_index_cache.values():
            if ind_set:
                valid_ind = ind_set - excl
                perm_ind = torch.randperm(len(valid_ind), device=dev)
                parts.append(torch.tensor(list(valid_ind), device=dev, dtype=torch.long)[perm_ind][:n])
        return torch.cat(parts).cpu().numpy().astype(np.int64)

    @classmethod
    def sample(cls, buffer_x, buffer_y, n_smp_cls, excl_indices=None, device='cpu'):
        """Reference signature (buffer_utils.py:81): returns (x, y, sample_ind)."""
        ind = cls.sample_indices(n_smp_cls, excl_indices)
        ind_t = to_device_i64(ind, buffer_x.device)
        if buffer_x.is_cuda:
            return ops.gather_rows(buffer_x, ind_t), ops.gather_rows(buffer_y, ind_t), ind_t
        return buffer_x[ind_t], buffer_y[ind_t], ind_t

    @classmethod
    def update_cache(cls, buffer_y, num_class, new_y=None, ind=None, device='cpu', labels_host=None):
        """Incremental update (new_y/ind given, buffer_utils.py:140-154) or full rebuild from the
        label buffer (buffer_utils.py:155-160).  Accepts host arrays; device tensors are copied
        once (a sync) only when no host mirror is supplied."""
        flush_pending()
        cls._update_cache_now(buffer_y, num_class, new_y, ind, labels_host)

    @classmethod
    def _update_cache_now(cls, buffer_y, num_class, new_y=None, ind=None, labels_host=None):
        def host(a):
            if a is None:
                return None
            if isinstance(a, torch.Tensor):
                return a.detach().cpu().numpy().astype(np.int64)
            return np.asarray(a, dtype=np.int64)
        if cls.class_index_cache is None:
            n = buffer_y.shape[0]
            cls.class_index_cache = {}
            cls.class_num_cache = np.zeros(num_class, dtype=np.int64)
            cls.labels_host = np.zeros(n, dtype=np.int64)
            cls._member = np.zeros(n, dtype=bool)
            cls._tab = np.full((max(1, num_class), 8), -1, dtype=np.int64)
            cls._cnt = np.zeros(max(1, num_class), dtype=np.int64)
            cls._pos = np.zeros(n, dtype=np.int64)
        if new_y is not None:
            new_y, ind = host(new_y), host(ind)
            for i, ny in zip(ind.tolist(), new_y.tolist()):
                if cls._member[i]:
                    oy = int(cls.labels_host[i])
                    cls.class_index_cache[oy].discard(i)
                    cls.class_num_cache[oy] -= 1
                    cls._tab_remove(i, oy)
                cls.class_index_cache.setdefault(ny, set()).add(i)
                cls.class_num_cache[ny] += 1
                cls.labels_host[i] = ny
                cls._member[i] = True
                cls._tab_add(i, ny)
        else:
            lab = host(labels_host) if labels_host is not None else host(buffer_y)
            cls.labels_host = lab.copy()
            n = lab.shape[0]
            cls._member = np.ones(n, dtype=bool)
            cache = {}
            C = max(int(lab.max()) + 1 if n else 1, num_class, 1)
            counts = np.bincount(lab, minlength=C)
            cls._tab = np.full((C, max(8, int(counts.max()) if n else 8)), -1, dtype=np.int64)
            cls._cnt = counts.astype(np.int64)
            cls._pos = np.zeros(n, dtype=np.int64)
            order = np.argsort(lab, kind='stable')
            start = 0
            for c in range(C):
                k = int(counts[c])
                if k:
                    members = order[start:start + k]
                    cls._tab[c, :k] = members
                    cls._pos[members] = np.arange(k)
                    cache[c] = set(members.tolist())
                    start += k
            if parity():
                # the reference's rebuild (buffer_utils.py:156-160): classes keyed in order of first appearance,
                # slots added in ascending order -- the dict / set iteration orders the parity sampler relies on
                cache = defaultdict(set)
                for i, c in enumerate(lab.tolist()):
                    cache[c].add(i)
            cls.class_index_cache = cache
            # the reference leaves class_num_cache untouched on this path (buffer_utils.py:155-160)


# --------------------------------------------------------------------------- GDumb's memory
class GreedyBalancedMemory(object):
    """GDumb's greedy class-balanced memory (agents/gdumb.py:19-31) as a device pool of `mem_size` slots.

    The reference keeps per-class Python lists of image tensors and counts; here the lists hold slot ids into a
    [mem_size,3,H,W] fp32 image pool and a [mem_size] int64 label pool, and a stack keeps the free slots.  Every
    decision is taken on the host by plan() with the reference's rule and its draws on Python's global `random`; write()
    then moves the rows with one gather and one scatter."""

    def __init__(self, mem_size, in_hw, device):
        if int(mem_size) < 1:
            raise ValueError('GDumb needs mem_size >= 1, got %d' % int(mem_size))
        self.mem_size = int(mem_size)
        self.device = torch.device(device)
        self.images = torch.zeros((self.mem_size, 3, in_hw, in_hw), dtype=torch.float32, device=self.device)
        self.labels = torch.zeros(self.mem_size, dtype=torch.int64, device=self.device)
        self.mem_c = {}                   # label -> count, in the insertion order of the reference's mem_c / mem_img
        self.slots = {}                   # label -> slot ids in the order of the reference's mem_img[label] list
        self._free = list(range(self.mem_size - 1, -1, -1))    # stack of free slots (slot 0 on top)
        self._labels_host = np.zeros(self.mem_size, dtype=np.int64)
        self._size = 0

    def __len__(self):
        return self._size

    def plan(self, labels):
        """greedy_balancing_update (gdumb.py:19-31) for each label in order: (slots, sources), the slots this pass
        writes and, for each, the position in `labels` of the sample that ends up there (a slot freed and refilled
        within the pass keeps only its last source).  Updates mem_c and the slot lists."""
        src_of = {}
        for j, y in enumerate(np.asarray(labels, dtype=np.int64).tolist()):
            k_c = self.mem_size // max(1, len(self.mem_c))
            if y not in self.mem_c or self.mem_c[y] < k_c:
                if self._size >= self.mem_size:
                    cls_max = max(self.mem_c.items(), key=lambda kv: kv[1])[0]     # the first class of maximal count
                    idx = random.randrange(self.mem_c[cls_max])
                    self._free.append(self.slots[cls_max].pop(idx))
                    self.mem_c[cls_max] -= 1
                    self._size -= 1
                if y not in self.mem_c:
                    self.mem_c[y] = 0
                    self.slots[y] = []
                slot = self._free.pop()
                self.slots[y].append(slot)
                self.mem_c[y] += 1
                self._size += 1
                src_of[slot] = j
        slots = np.fromiter(src_of.keys(), dtype=np.int64, count=len(src_of))
        return slots, np.fromiter(src_of.values(), dtype=np.int64, count=len(src_of))

    def write(self, x, y_host, slots, sources):
        """images[slots] = x[sources] (one gather, one scatter) and labels[slots] = y_host[sources]."""
        if slots.size == 0:
            return
        src_t = to_device_i64(sources, self.device)
        ops.scatter_rows(self.images, to_device_i64(slots, self.device), ops.gather_rows(x, src_t))
        self._labels_host[slots] = np.asarray(y_host, dtype=np.int64)[sources]
        self.labels = to_device_i64(self._labels_host, self.device)

    def order(self):
        """Slot ids in train_mem's order (gdumb.py:53-58): classes in insertion order, each in its list order."""
        parts = [np.asarray(self.slots[c], dtype=np.int64) for c in self.mem_c]
        return np.concatenate(parts) if parts else np.zeros(0, dtype=np.int64)

    def snapshot_parts(self):
        """snapshot() with the pool left on the device (marked as 8-bit rows) and the decision state copied: counts and
        slot lists in their insertion order, the free-slot stack, the label mirror."""
        return {'images': Rows8(self.images), 'labels': self._labels_host.copy(), 'mem_c': dict(self.mem_c),
                'slots': {c: list(v) for c, v in self.slots.items()}, 'free': list(self._free), 'size': self._size}

    def snapshot(self):
        """The pool on the host (one device-to-host copy of the images after a synchronise of the current stream) and
        the decision state."""
        return host_tree(self.snapshot_parts())

    def snapshot_capacity(self):
        """Bytes of the largest snapshot_parts() device tree."""
        return self.images.numel() * self.images.element_size()

    def restore(self, state):
        if tuple(state['images'].shape) != tuple(self.images.shape):
            raise ValueError('snapshot memory %s does not fit %s' % (tuple(state['images'].shape), tuple(self.images.shape)))
        self.images.copy_(state['images'])
        self._labels_host = np.asarray(state['labels'], dtype=np.int64).copy()
        self.labels = torch.from_numpy(self._labels_host.copy()).to(self.device)
        self.mem_c = dict(state['mem_c'])
        self.slots = {c: list(v) for c, v in state['slots'].items()}
        self._free = list(state['free'])
        self._size = int(state['size'])


class TaskRingMemory(object):
    """GEM's episodic memory: one ring of M rows per task (images fp32 [M,3,H,W] and labels int64 [M] on the device, a
    host mirror of the labels), allocated when its task begins, so the memory grows one task at a time.  write() follows
    the authors' release: rows [cnt, endcnt) take the batch's first endcnt - cnt rows with endcnt = min(cnt + bsz, M)
    (truncated at the ring's end, not wrapped) and the counter returns to 0 when it reaches M; begin_task() restarts the
    counter of its task at 0.  A task's filled row count is min(rows written, M)."""

    def __init__(self, M, in_hw, device):
        if int(M) < 1:
            raise ValueError('GEM needs at least one memory row per task (mem_size // num_tasks >= 1), got %d' % int(M))
        self.M = int(M)
        self.in_hw = int(in_hw)
        self.device = torch.device(device)
        self.images, self.labels, self.labels_host = [], [], []
        self.filled, self.cnt = [], []

    def __len__(self):
        return len(self.images)

    def begin_task(self, task):
        """Rings up to task `task` exist (a task never written keeps an empty one); its counter restarts at 0."""
        while len(self.images) <= task:
            self.images.append(torch.zeros((self.M, 3, self.in_hw, self.in_hw), dtype=torch.float32, device=self.device))
            self.labels.append(torch.zeros(self.M, dtype=torch.int64, device=self.device))
            self.labels_host.append(np.zeros(self.M, dtype=np.int64))
            self.filled.append(0)
            self.cnt.append(0)
        self.cnt[task] = 0

    def write(self, task, x, y, y_host):
        """The ring write of one batch into task `task`'s ring; returns (start, rows written)."""
        cnt = self.cnt[task]
        end = min(cnt + x.size(0), self.M)
        k = end - cnt
        self.images[task][cnt:end].copy_(x[:k])
        self.labels[task][cnt:end].copy_(y[:k])
        self.labels_host[task][cnt:end] = np.asarray(y_host, dtype=np.int64)[:k]
        self.filled[task] = max(self.filled[task], end)
        self.cnt[task] = 0 if end == self.M else end
        return cnt, k

    def rows(self, task):
        """(images, labels) of task `task`'s filled rows: views of its ring."""
        n = self.filled[task]
        return self.images[task][:n], self.labels[task][:n]

    def snapshot_parts(self):
        """The filled rows of every ring on the device (images marked as 8-bit rows, one array per task), the label
        mirrors, counters and filled counts on the host."""
        return {'M': self.M, 'filled': list(self.filled), 'cnt': list(self.cnt),
                'labels': [lab[:n].copy() for lab, n in zip(self.labels_host, self.filled)],
                'images': {k: Rows8(img[:n]) for k, (img, n) in enumerate(zip(self.images, self.filled)) if n}}

    def snapshot(self):
        return host_tree(self.snapshot_parts())

    def snapshot_capacity(self, n_tasks):
        """Bytes of the snapshot_parts() device tree of n_tasks full rings."""
        return int(n_tasks) * self.M * 3 * self.in_hw * self.in_hw * 4

    def restore(self, state):
        if int(state['M']) != self.M:
            raise ValueError('snapshot memory of %d rows per task does not fit %d' % (int(state['M']), self.M))
        filled = [int(n) for n in state['filled']]
        self.images, self.labels, self.labels_host, self.filled, self.cnt = [], [], [], [], []
        if filled:
            self.begin_task(len(filled) - 1)
        for k, n in enumerate(filled):
            if n:
                self.images[k][:n].copy_(state['images'][k])
                self.labels_host[k][:n] = np.asarray(state['labels'][k], dtype=np.int64)
                self.labels[k].copy_(torch.from_numpy(self.labels_host[k]))
        self.filled = filled
        self.cnt = [int(c) for c in state['cnt']]


# --------------------------------------------------------------------------- buffer
def random_retrieve(buffer, num_retrieve, excl_indices=None, return_indices=False):
    """buffer_utils.py:9-26."""
    idx = uniform_indices(buffer.current_index, num_retrieve, excl_indices)
    buffer.last_random_idx = idx          # host record of the draw (tests replay it)
    x, y, idx_t = buffer.gather(idx)
    if return_indices:
        return x, y, idx_t
    return x, y


class Buffer(torch.nn.Module):
    """Same attributes as the reference Buffer (buffer.py:8-41): buffer_img, buffer_label
    (registered buffers), current_index, n_seen_so_far, model, params, device; plus labels_host,
    the numpy mirror every index decision reads."""

    def __init__(self, model, params, update_methods=None, retrieve_methods=None):
        super().__init__()
        self.params = params
        self.model = model
        self.cuda = self.params.cuda
        self.current_index = 0
        self.n_seen_so_far = 0
        use_cuda = torch.cuda.is_available()     # the reference ignores params.cuda here (buffer.py:22-23)
        self.device = 'cuda' if use_cuda else 'cpu'
        buffer_size = params.mem_size
        print('buffer has %d slots' % buffer_size)
        input_size = input_size_match[params.data]
        dev = torch.device(self.device)
        self.register_buffer('buffer_img', torch.zeros((buffer_size, *input_size), dtype=torch.float32, device=dev))
        self.register_buffer('buffer_label', torch.zeros(buffer_size, dtype=torch.int64, device=dev))
        self._labels_host = np.zeros(buffer_size, dtype=np.int64)
        if update_methods is None or retrieve_methods is None:
            from . import registry
            update_methods = update_methods or registry.update_methods
            retrieve_methods = retrieve_methods or registry.retrieve_methods
        self.update_method = update_methods[params.update](params)
        self.retrieve_method = retrieve_methods[params.retrieve](params)
        if getattr(self.params, 'buffer_tracker', False):
            raise NotImplementedError('buffer_tracker belongs to the match/mem_match retrievals, outside the replay path')

    @property
    def labels_host(self):
        """numpy mirror of buffer_label; this buffer's deferred device-decided updates are applied before it is read."""
        flush_pending(self)
        return self._labels_host

    @labels_host.setter
    def labels_host(self, value):
        flush_pending(self)
        self._labels_host = np.asarray(value, dtype=np.int64)

    def update(self, x, y, **kwargs):
        return self.update_method.update(buffer=self, x=x, y=y, **kwargs)

    def snapshot_parts(self):
        """snapshot() with the filled slots left on the device (the images marked as 8-bit rows) and the host values
        copied.  This buffer's deferred label-mirror updates are applied first.  The update plugin's state is its
        snapshot_parts(), or its snapshot() when it has only that."""
        flush_pending(self)
        n = self.current_index
        out = {'images': Rows8(self.buffer_img[:n]), 'labels': self.buffer_label[:n],
               'labels_host': self._labels_host.copy(), 'current_index': n, 'n_seen_so_far': self.n_seen_so_far}
        if hasattr(self.update_method, 'snapshot_parts'):
            out['update'] = self.update_method.snapshot_parts()
        elif hasattr(self.update_method, 'snapshot'):
            out['update'] = self.update_method.snapshot()
        return out

    def snapshot(self):
        """The filled slots on the host (rows current_index.. are never written before the rows below them), the
        counters, the label mirror with this buffer's deferred updates applied, and the update plugin's own state when
        it keeps one (GSS's scores).  The current stream is synchronised once, then one device-to-host copy per tensor."""
        return host_tree(self.snapshot_parts())

    def snapshot_capacity(self):
        """Bytes of the largest snapshot_parts() device tree (every slot filled)."""
        n = sum(t.numel() * t.element_size() for t in (self.buffer_img, self.buffer_label))
        if hasattr(self.update_method, 'snapshot_parts'):
            n += sum(t.numel() * t.element_size() for t in self.update_method.snapshot_parts().values())
        return n

    def restore(self, state):
        n = int(state['current_index'])
        if n > self.buffer_img.shape[0] or tuple(state['images'].shape[1:]) != tuple(self.buffer_img.shape[1:]):
            raise ValueError('snapshot buffer %s does not fit %s' % (tuple(state['images'].shape),
                                                                    tuple(self.buffer_img.shape)))
        flush_pending(self)
        self.buffer_img[:n].copy_(state['images'])
        self.buffer_label[:n].copy_(state['labels'])
        self._labels_host = np.asarray(state['labels_host'], dtype=np.int64).copy()
        self.current_index, self.n_seen_so_far = n, int(state['n_seen_so_far'])
        if 'update' in state:
            self.update_method.restore(state['update'])

    def retrieve(self, **kwargs):
        return self.retrieve_method.retrieve(buffer=self, **kwargs)

    # ---- row movement
    def gather(self, idx_host):
        """(x [n,3,H,W], y [n], idx device tensor) for host slot indices."""
        idx_t = to_device_i64(idx_host, self.buffer_img.device)
        if self.buffer_img.is_cuda:
            return ops.gather_rows(self.buffer_img, idx_t), ops.gather_rows(self.buffer_label, idx_t), idx_t
        return self.buffer_img[idx_t], self.buffer_label[idx_t], idx_t

    def write(self, slots_host, x_rows, y_rows, y_host):
        """buffer_img[slots] = x_rows; buffer_label[slots] = y_rows (+ host mirror)."""
        slots_host = np.asarray(slots_host, dtype=np.int64)
        if slots_host.size == 0:
            return
        idx_t = to_device_i64(slots_host, self.buffer_img.device)
        if self.buffer_img.is_cuda:
            ops.scatter_rows(self.buffer_img, idx_t, x_rows)
            ops.scatter_rows(self.buffer_label, idx_t, y_rows)
        else:
            self.buffer_img[idx_t] = x_rows
            self.buffer_label[idx_t] = y_rows
        self.labels_host[slots_host] = np.asarray(y_host, dtype=np.int64)


class LogitBuffer(Buffer):
    """DER++'s memory: a Buffer whose slots also keep buffer_logits [mem_size, out_dim] fp32, the logits the network gave
    each stored sample.  update(x, y, logits=...) is the reservoir update of Reservoir_update, with the same
    update.reservoir_draws / reservoir_plan calls, and writes each chosen stream row's logits beside its image and label.
    Retrieval is the inherited random one; the learner reads the logits of the slots it drew."""

    def __init__(self, model, params, out_dim, update_methods=None, retrieve_methods=None):
        super().__init__(model, params, update_methods, retrieve_methods)
        self.register_buffer('buffer_logits', torch.zeros((params.mem_size, int(out_dim)), dtype=torch.float32,
                                                          device=self.buffer_img.device))

    def update(self, x, y, logits=None, **kwargs):
        """The reservoir update of (x, y) (Reservoir_update.update) with buffer_logits[slot] = logits[row] for every row
        it stores.  Returns the slots written by the reservoir draws, as Reservoir_update does."""
        from . import update as _update
        if logits is None or logits.shape != (x.size(0), self.buffer_logits.shape[1]):
            raise ValueError('LogitBuffer.update needs the [%d, %d] logits of the stream rows'
                             % (x.size(0), self.buffer_logits.shape[1]))
        y_host = _update._host_labels(y, kwargs)
        batch_size = x.size(0)
        mem = self.buffer_img.size(0)
        place_left = max(0, mem - self.current_index)
        if place_left:
            offset = min(place_left, batch_size)
            s, e = self.current_index, self.current_index + offset
            self.buffer_img[s:e].copy_(x[:offset])
            self.buffer_label[s:e].copy_(y[:offset])
            self.buffer_logits[s:e].copy_(logits[:offset])
            self.labels_host[s:e] = y_host[:offset]
            self.current_index += offset
            self.n_seen_so_far += offset
            if offset == batch_size:
                return list(range(s, e))
        x, y, y_host, logits = x[place_left:], y[place_left:], y_host[place_left:], logits[place_left:]
        draws = _update.reservoir_draws(x.size(0), self.n_seen_so_far, x.device)
        self.last_draws = draws
        self.n_seen_so_far += x.size(0)
        slots, src = _update.reservoir_plan(draws, mem)
        if not slots:
            return []
        src_t = to_device_i64(src, x.device)
        if x.is_cuda:
            self.write(slots, ops.gather_rows(x, src_t), ops.gather_rows(y, src_t), y_host[src])
            ops.scatter_rows(self.buffer_logits, to_device_i64(slots, x.device), ops.gather_rows(logits, src_t))
        else:
            self.write(slots, x[src_t], y[src_t], y_host[src])
            self.buffer_logits[torch.as_tensor(slots)] = logits[src_t]
        return slots

    def snapshot_parts(self):
        """Buffer.snapshot_parts() plus the filled logit rows, on the device, kept as fp32."""
        out = super().snapshot_parts()
        out['logits'] = self.buffer_logits[:self.current_index]
        return out

    def snapshot_capacity(self):
        return super().snapshot_capacity() + self.buffer_logits.numel() * self.buffer_logits.element_size()

    def restore(self, state):
        super().restore(state)
        n = int(state['current_index'])
        if tuple(state['logits'].shape) != (n, self.buffer_logits.shape[1]):
            raise ValueError('snapshot logits %s do not fit %s' % (tuple(state['logits'].shape),
                                                                    tuple(self.buffer_logits.shape)))
        self.buffer_logits[:n].copy_(state['logits'])
