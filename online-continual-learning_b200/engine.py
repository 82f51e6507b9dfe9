"""Host handle of the Reduced-ResNet18 / SupConResNet engine (C ABI: b200ocl_net_*).

Owns the flat device arenas (parameters, gradients, packed weights, BN running
statistics) as torch tensors and hands raw pointers to libb200ocl.so.  The layer
plan, arena layout and every kernel live on the C side (csrc/net_*.cu*, conv.cu);
this file is plumbing.  Mirrors what the reference gets from nn.Module +
torch.optim.SGD (models/resnet.py, utils/setup_elements.py:46-82).
"""
import ctypes
from ctypes import c_int, c_int64, c_size_t, c_void_p
from types import SimpleNamespace

import torch

from . import _native, ops
from .ops import _stream, _workspace, _need_cuda

HEAD_CODES = {None: 0, 'classifier': 0, 'linear': 1, 'mlp': 2, 'None': 3}


class NetDesc(ctypes.Structure):
    _fields_ = [('in_h', c_int), ('in_w', c_int), ('nf', c_int), ('num_classes', c_int), ('head', c_int),
                ('feat_dim', c_int)]


class NetState(ctypes.Structure):
    _fields_ = [('params', c_void_p), ('grads', c_void_p), ('packed', c_void_p), ('bn_stats', c_void_p),
                ('bn_tracked', c_void_p)]


class EwcState(ctypes.Structure):
    _fields_ = [('running', c_void_p), ('tmp', c_void_p), ('normalized', c_void_p), ('prev', c_void_p)]


class AdamState(ctypes.Structure):
    _fields_ = [('exp_avg', c_void_p), ('exp_avg_sq', c_void_p)]


class NetInfo(ctypes.Structure):
    _fields_ = [('n_params', c_size_t), ('n_packed', c_size_t), ('n_bn_stats', c_size_t), ('n_bn', c_int),
                ('n_tensors', c_int), ('dim_in', c_int), ('out_dim', c_int)]


class NetWsLayout(ctypes.Structure):
    """b200ocl_net_ws_layout: byte offsets of one conv layer's tensors in a train workspace and its backward launches."""
    _fields_ = [('bytes', c_size_t), ('z', c_size_t), ('a', c_size_t), ('mean', c_size_t), ('invstd', c_size_t),
                ('feat', c_size_t), ('hid', c_size_t), ('proj', c_size_t), ('wg_part', c_size_t), ('wg_layer', c_size_t),
                ('cin', c_int), ('cout', c_int), ('ks', c_int), ('stride', c_int), ('hout', c_int), ('wout', c_int),
                ('bn_fused', c_int), ('bn_grid', c_int), ('wgrad_kernel', c_int), ('wgrad_splits', c_int), ('sms', c_int)]


class ConvGeom(ctypes.Structure):
    """b200ocl_conv_geom: the convolution kernel one launch runs, its template parameters and grid, the statistics
    partials it writes against the workspace region kept for them, and the halo-strip kernel's pipeline depths."""
    _fields_ = [('kernel', c_int), ('nt', c_int), ('bn', c_int), ('pt', c_int), ('kwarps', c_int), ('grid_x', c_int),
                ('grid_y', c_int), ('th', c_int), ('tw', c_int), ('ti', c_int), ('stat_bytes', c_size_t),
                ('stat_region', c_size_t), ('sms', c_int), ('tp_ps', c_int), ('tp_bs', c_int)]

    KERNELS = ('stem', 'tcp', 'tc', 'patch', 'tiled', 'ksplit')

    @property
    def name(self):
        return self.KERNELS[self.kernel] if self.kernel >= 0 else 'none'

    @property
    def template(self):
        """(kernel name, template parameters) of the instantiation that runs."""
        return {'stem': ('stem',), 'tcp': ('tcp', self.nt), 'tc': ('tc', self.nt), 'patch': ('patch', self.bn, self.pt),
                'tiled': ('tiled', self.bn, self.pt), 'ksplit': ('ksplit', self.pt, self.kwarps),
                'none': ('none',)}[self.name]


CONV_PASSES = {'train': 0, 'eval': 1, 'dgrad': 2}


def _lib():
    return _native.lib()


def train_ws_layout(desc, n, layer):
    """Host-only test hook (b200ocl_net_train_ws_layout) for conv layer `layer` of a train workspace of n images."""
    out = NetWsLayout()
    _native.check(_lib().b200ocl_net_train_ws_layout(ctypes.byref(desc), int(n), int(layer), ctypes.byref(out)),
                  'b200ocl_net_train_ws_layout')
    return out


def conv_geom(desc, n, layer, pass_, sms=0):
    """Host-only test hook (b200ocl_net_conv_geom): the convolution launch of conv layer `layer` over n images in pass
    'train', 'eval' or 'dgrad' on a GPU with sms SMs (0: the current device)."""
    out = ConvGeom()
    _native.check(_lib().b200ocl_net_conv_geom(ctypes.byref(desc), int(n), int(layer), CONV_PASSES[pass_], int(sms),
                                               ctypes.byref(out)), 'b200ocl_net_conv_geom')
    return out


def conv_selftest_geom(n, h, w, cin, cout, ks, stride, dgrad, path, mode, sms=0):
    """Host-only test hook (b200ocl_conv_selftest_geom): the launch b200ocl_conv_selftest makes for these arguments."""
    out = ConvGeom()
    _native.check(_lib().b200ocl_conv_selftest_geom(int(n), int(h), int(w), int(cin), int(cout), int(ks), int(stride),
                                                    int(dgrad), int(path), int(mode), int(sms), ctypes.byref(out)),
                  'b200ocl_conv_selftest_geom')
    return out


class WgradTcGeom(ctypes.Structure):
    """b200ocl_wgrad_tc_geom: the grid of the wgmma weight gradient and how it splits the strip's tiles into chains."""
    _fields_ = [('eligible', c_int), ('slices', c_int), ('cout_blocks', c_int), ('bn', c_int), ('tiles', c_int),
                ('tpc', c_int), ('chains', c_int), ('chains_per_cta', c_int), ('ctas_x', c_int), ('sm_share', c_int),
                ('sms', c_int)]


def wgrad_tc_selftest_geom(n, h, w, cin, cout, sms=0):
    """Host-only test hook (b200ocl_wgrad_tc_selftest_geom): the launch b200ocl_wgrad_tc_selftest makes."""
    out = WgradTcGeom()
    _native.check(_lib().b200ocl_wgrad_tc_selftest_geom(int(n), int(h), int(w), int(cin), int(cout), int(sms),
                                                        ctypes.byref(out)), 'b200ocl_wgrad_tc_selftest_geom')
    return out


def describe(in_hw, num_classes, head=None, feat_dim=128, nf=20):
    """Host-only: arena sizes and tensor table for a network description (no GPU needed)."""
    desc = NetDesc(int(in_hw), int(in_hw), int(nf), int(num_classes), HEAD_CODES[head], int(feat_dim))
    info = NetInfo()
    lib = _lib()
    _native.check(lib.b200ocl_net_query(ctypes.byref(desc), ctypes.byref(info)), 'b200ocl_net_query')
    table = []
    off, num, hg = c_size_t(), c_size_t(), c_int()
    for i in range(info.n_tensors):
        _native.check(lib.b200ocl_net_tensor(ctypes.byref(desc), i, ctypes.byref(off), ctypes.byref(num),
                                             ctypes.byref(hg)), 'b200ocl_net_tensor')
        table.append((off.value, num.value, bool(hg.value)))
    return desc, info, table


class ArenaState:
    """One set of arenas (the live model, or MIR's virtual copy)."""

    def __init__(self, info, device, with_grads=True):
        self.params = torch.zeros(info.n_params, dtype=torch.float32, device=device)
        self.grads = torch.zeros(info.n_params, dtype=torch.float32, device=device) if with_grads else None
        self.packed = torch.zeros(info.n_packed, dtype=torch.float32, device=device)
        self.bn_stats = torch.zeros(info.n_bn_stats, dtype=torch.float32, device=device)
        self.bn_tracked = torch.zeros(info.n_bn, dtype=torch.int64, device=device)
        self.c = NetState(self.params.data_ptr(), self.grads.data_ptr() if with_grads else None,
                          self.packed.data_ptr(), self.bn_stats.data_ptr(), self.bn_tracked.data_ptr())


# CUDA graphs for the network-level calls (40-120 kernel launches each): after two eager calls of a given
# (call, batch size, workspace) the launch sequence is captured once and replayed.  Replays read their inputs from
# static buffers (one device-to-device copy per call).  B200OCL_GRAPHS=0 or set_graphs(False) turns this off
# (the per-launch profiler needs eager launches).
import os as _os
_GRAPHS = _os.environ.get('B200OCL_GRAPHS', '1') != '0'


def set_graphs(on):
    global _GRAPHS
    _GRAPHS = bool(on)


_replayed = [0]      # kernel launches issued through graph replays (the library's own counter only sees eager ones)
# Held while a graph is captured.  A capture fails when another thread of the process makes a CUDA call that may
# synchronise meanwhile, so a thread that copies from the device beside training (checkpoint.py's writer) takes it
# around each of its CUDA calls.
import threading as _threading
capture_lock = _threading.Lock()


def graph_launch_count():
    return _replayed[0]


class _Graphed:
    """One captured call: static inputs / outputs, the graphs, and the number of eager warm-up calls so far.
    The same launch sequence is captured into N_EXEC executable graphs used round-robin, so that a replay never
    has to wait for the previous launch of the same executable when the host runs several steps ahead."""
    __slots__ = ('inputs', 'outputs', 'graphs', 'calls', 'kernels', 'turn')
    N_EXEC = 3

    def __init__(self, inputs, outputs):
        self.inputs, self.outputs, self.graphs, self.calls, self.kernels, self.turn = inputs, outputs, [], 0, 0, 0

    def run(self, launch):
        if self.calls < 1:                       # eager once: lets every launcher configure its kernel
            launch()
            self.calls += 1
            return
        if not self.graphs:                      # second call: capture all executables, run the first
            with capture_lock:
                for _ in range(self.N_EXEC):
                    before = _native.launch_count()
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        launch()
                    self.kernels = int(_native.launch_count() - before)
                    self.graphs.append(g)
        self.graphs[self.turn].replay()
        self.turn = (self.turn + 1) % self.N_EXEC
        _replayed[0] += self.kernels


class Engine:
    def __init__(self, in_hw, num_classes, head=None, feat_dim=128, device='cuda'):
        self.desc, self.info, self.table = describe(in_hw, num_classes, head, feat_dim)
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise _native.NativeError('the b200ocl engine runs on CUDA only; there is no CPU fallback')
        self.head = head
        self.in_hw = in_hw
        self.dim_in, self.out_dim = self.info.dim_in, self.info.out_dim
        self.state = ArenaState(self.info, self.device)
        self._virtual = None
        self._teacher = None
        self._eval_ws = {}
        self._train_ws = {}
        self._graphs = {}
        self._feat_off = {}

    # ------------------------------------------------------------------ state
    def param_views(self, shapes=None):
        """Views of the parameter arena, one per tensor in parameters() order."""
        return [self.state.params[o:o + n] for (o, n, _) in self.table]

    def grad_views(self):
        return [self.state.grads[o:o + n] for (o, n, _) in self.table]

    def load(self, params, bn_state=None):
        """params: iterable of tensors in parameters() order (any device); bn_state: iterable of
        (running_mean, running_var[, num_batches_tracked]) per BatchNorm2d in module order."""
        params = list(params)
        if len(params) != len(self.table):
            raise ValueError('expected %d parameter tensors, got %d' % (len(self.table), len(params)))
        for (o, n, _), t in zip(self.table, params):
            if t.numel() != n:
                raise ValueError('parameter size mismatch: %d vs %d' % (t.numel(), n))
            self.state.params[o:o + n].copy_(t.detach().reshape(-1).to(torch.float32))
        if bn_state is not None:
            off = 0
            for i, entry in enumerate(bn_state):
                rm, rv = entry[0], entry[1]
                c = rm.numel()
                self.state.bn_stats[off:off + c].copy_(rm.detach().reshape(-1))
                self.state.bn_stats[off + c:off + 2 * c].copy_(rv.detach().reshape(-1))
                if len(entry) > 2:
                    self.state.bn_tracked[i] = int(entry[2])
                off += 2 * c
            if off != self.info.n_bn_stats:
                raise ValueError('BN statistics do not cover the network')
        self.pack()

    def bn_views(self):
        """[(running_mean, running_var)] views per BatchNorm2d in module order."""
        out, off = [], 0
        sizes = [n for (o, n, _) in self.table[1:3 * self.info.n_bn:3]]
        for c in sizes:
            out.append((self.state.bn_stats[off:off + c], self.state.bn_stats[off + c:off + 2 * c]))
            off += 2 * c
        return out

    def pack(self, state=None):
        st = state or self.state
        _native.check(_lib().b200ocl_net_pack(ctypes.byref(self.desc), ctypes.byref(st.c), _stream()),
                      'b200ocl_net_pack')

    # ------------------------------------------------------------------ snapshot / restore (checkpoint.py)
    def snapshot_parts(self):
        """The arenas a resumed run reads, on the device: parameters, BN running statistics and bn_tracked, and when they
        exist the teacher's (parameters, statistics, bn_tracked), EWC++'s running / tmp / normalized Fisher and previous
        parameters, and Adam's moments and step count (a host int).  Packed weights, gradients, workspaces and MIR's
        virtual copy are rebuilt or overwritten before they are read, so they are not kept."""
        out = {'params': self.state.params, 'bn_stats': self.state.bn_stats, 'bn_tracked': self.state.bn_tracked}
        if self._teacher is not None:
            t = self._teacher
            out['teacher'] = {'params': t.params, 'bn_stats': t.bn_stats, 'bn_tracked': t.bn_tracked}
        if getattr(self, '_ewc', None) is not None:
            out['ewc'] = {k: getattr(self._ewc, k) for k in ('running', 'tmp', 'normalized', 'prev')}
        if getattr(self, '_adam', None) is not None:
            out['adam'] = {'exp_avg': self._adam.exp_avg, 'exp_avg_sq': self._adam.exp_avg_sq, 'step': self._adam.step}
        return out

    def snapshot(self):
        """snapshot_parts() on the host: the current stream is synchronised once, then each arena is one device-to-host
        copy."""
        from .memory import host_tree
        return host_tree(self.snapshot_parts())

    def snapshot_capacity(self):
        """Bytes of the largest snapshot_parts() this engine can give: its arenas plus the teacher, EWC++ and Adam arenas
        it may allocate later."""
        arena = self.info.n_params * 4 + self.info.n_bn_stats * 4 + self.info.n_bn * 8
        return 2 * arena + 6 * self.info.n_params * 4

    def restore(self, state):
        """Copy a snapshot() back into the arenas, in place (the Parameters, EWC++ views and optimizer state that alias
        them stay valid), allocating the teacher, EWC++ and Adam arenas it holds, then rebuild the packed weights with
        pack().  One host-to-device copy per arena on the current stream."""
        def put(dst, src):
            if dst.shape != src.shape or dst.dtype != src.dtype:
                raise ValueError('snapshot arena %s %s does not fit %s %s' % (tuple(src.shape), src.dtype,
                                                                          tuple(dst.shape), dst.dtype))
            dst.copy_(src)
        for k in ('params', 'bn_stats', 'bn_tracked'):
            put(getattr(self.state, k), state[k])
        if 'teacher' in state:
            if self._teacher is None:
                self._teacher = ArenaState(self.info, self.device, with_grads=False)
            for k in ('params', 'bn_stats', 'bn_tracked'):
                put(getattr(self._teacher, k), state['teacher'][k])
            self.pack(self._teacher)
        if 'ewc' in state:
            st = self.ewc_state()
            for k in ('running', 'tmp', 'normalized', 'prev'):
                put(getattr(st, k), state['ewc'][k])
        if 'adam' in state:
            st = self.adam_state()
            put(st.exp_avg, state['adam']['exp_avg'])
            put(st.exp_avg_sq, state['adam']['exp_avg_sq'])
            st.step = int(state['adam']['step'])
        self.pack()

    def virtual_state(self):
        if self._virtual is None:
            self._virtual = ArenaState(self.info, self.device, with_grads=False)
        return self._virtual

    # ------------------------------------------------------------------ distillation teacher
    TEACHER_SLOT = 6

    def update_teacher(self):
        """copy.deepcopy(model) of KdManager.update_teacher (utils/kd_manager.py:18-19): parameters, BN running
        statistics and num_batches_tracked copied into one persistent arena set.  Every call writes the same buffers, so
        the pointers a captured teacher forward holds stay valid."""
        t = self._teacher
        if t is None:
            t = self._teacher = ArenaState(self.info, self.device, with_grads=False)
        t.params.copy_(self.state.params)
        t.bn_stats.copy_(self.state.bn_stats)
        t.bn_tracked.copy_(self.state.bn_tracked)
        self.pack(t)

    @property
    def teacher(self):
        """The teacher's arenas, None until update_teacher() has run."""
        return self._teacher

    def teacher_forward(self, x, slot=TEACHER_SLOT):
        """teacher_model.forward(x) under no_grad (kd_manager.py:24-25).  The copy was taken from a model in train
        mode and never switched, so this is a train-mode forward: batch statistics, and the teacher's own running
        statistics move (they never feed anything).  Graphed like the live forward, under its own key."""
        if self._teacher is None:
            raise RuntimeError('no teacher: call update_teacher() first')
        return self.forward_train(x, state=self._teacher, slot=slot, _tag='teacher')[0]

    # ------------------------------------------------------------------ passes
    def _x(self, x):
        _need_cuda(x)
        x = x.detach().to(torch.float32).contiguous()
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[2] != self.in_hw or x.shape[3] != self.in_hw:
            raise ValueError('expected images [N,3,%d,%d], got %s' % (self.in_hw, self.in_hw, tuple(x.shape)))
        return x

    def features_eval(self, x, state=None):
        """model.eval(); model.features(x) under no_grad -> [N, dim_in]."""
        x = self._x(x)
        n = x.shape[0]
        if n == 0:
            return torch.empty((0, self.dim_in), dtype=torch.float32, device=x.device)
        lib = _lib()
        ws = self._eval_ws.get(n)
        if ws is None:
            ws = _workspace(lib.b200ocl_net_eval_workspace_bytes(ctypes.byref(self.desc), n), x.device)
            if len(self._eval_ws) < 8:
                self._eval_ws[n] = ws
        st = state or self.state

        def launch(xin, feat):
            rc = lib.b200ocl_net_features_eval(ctypes.byref(self.desc), ctypes.byref(st.c), xin.data_ptr(), n,
                                               feat.data_ptr(), ws.data_ptr(), ws.numel(), _stream())
            _native.check(rc, 'b200ocl_net_features_eval')

        if _GRAPHS and state is None and self._eval_ws.get(n) is ws:
            key = ('eval', n)
            e = self._graphs.get(key)
            if e is None:
                e = self._graphs[key] = _Graphed([torch.empty_like(x)],
                                                 [torch.empty((n, self.dim_in), dtype=torch.float32, device=x.device)])
            e.inputs[0].copy_(x)
            e.run(lambda: launch(e.inputs[0], e.outputs[0]))
            return e.outputs[0].clone()          # the static buffer is overwritten by the next call
        feat = torch.empty((n, self.dim_in), dtype=torch.float32, device=x.device)
        launch(x, feat)
        return feat

    def new_train_workspace(self, n):
        return _workspace(_lib().b200ocl_net_train_workspace_bytes(ctypes.byref(self.desc), n), self.device)

    def train_workspace(self, n, slot=0):
        key = (n, slot)
        ws = self._train_ws.get(key)
        if ws is None:
            ws = self.new_train_workspace(n)
            if len(self._train_ws) < 8:
                self._train_ws[key] = ws
        return ws

    def train_features(self, ws, n):
        """The encoder features [n, dim_in] the train-mode forward over n images left in its workspace ws
        (b200ocl_net_train_ws_layout's `feat`): a view, overwritten by the next forward into ws."""
        off = self._feat_off.get(n)
        if off is None:
            off = self._feat_off[n] = train_ws_layout(self.desc, n, 0).feat
        return ws[off:off + n * self.dim_in * 4].view(torch.float32).view(n, self.dim_in)

    def forward_train(self, x, ws=None, state=None, slot=0, eval_stats=False, defer_stats=False, features=False,
                      _tag='fwd'):
        """model.train(); model.forward(x).  Returns (out [N,out_dim], workspace kept for backward).
        eval_stats=True: model.eval() forward that can be differentiated (running statistics, nothing updated).
        defer_stats=True: the BN running statistics are left alone; apply_running_stats(ws, N) moves them later (so that
        the train-mode passes of one step can run concurrently on different streams and still update the statistics in
        the reference's order).  features=True: the same launches, returning the encoder features [N, dim_in] in place of
        out, as train_features(ws, N) gives them (a view of the workspace; backward(..., features=True) starts from
        their gradient).  _tag: the graph key of a forward over another persistent state (the teacher's); other
        forwards over a state= run eagerly."""
        x = self._x(x)
        n = x.shape[0]
        graphed = (_GRAPHS and ws is None and (state is None) == (_tag == 'fwd') and (n, slot) in self._train_ws
                   and not eval_stats)
        if ws is None:
            ws = self.train_workspace(n, slot)
        st = state or self.state
        name = ('b200ocl_net_forward_evalgrad' if eval_stats else
                'b200ocl_net_forward_train_deferred' if defer_stats else 'b200ocl_net_forward_train')

        def launch(xin, out):
            rc = getattr(_lib(), name)(ctypes.byref(self.desc), ctypes.byref(st.c), xin.data_ptr(), n, out.data_ptr(),
                                       ws.data_ptr(), ws.numel(), _stream())
            _native.check(rc, name)

        if graphed:
            key = (_tag, n, slot, bool(defer_stats))
            e = self._graphs.get(key)
            if e is None:
                other = self._graphs.get((_tag, n, slot, not defer_stats))      # one static input per (n, slot)
                e = self._graphs[key] = _Graphed([other.inputs[0] if other is not None else torch.empty_like(x)],
                                                 [torch.empty((n, self.out_dim), dtype=torch.float32, device=x.device)])
            e.inputs[0].copy_(x)
            e.run(lambda: launch(e.inputs[0], e.outputs[0]))
            if features:
                return self.train_features(ws, n), ws
            return e.outputs[0].clone(), ws      # the static buffer is overwritten by the next call
        out = torch.empty((n, self.out_dim), dtype=torch.float32, device=x.device)
        launch(x, out)
        return (self.train_features(ws, n) if features else out), ws

    def apply_running_stats(self, ws, n):
        """The running-statistics update of a forward_train(..., defer_stats=True) over n images kept in ws."""
        rc = _lib().b200ocl_net_apply_running_stats(ctypes.byref(self.desc), ctypes.byref(self.state.c), int(n), ws.data_ptr(),
                                                    ws.numel(), _stream())
        _native.check(rc, 'b200ocl_net_apply_running_stats')

    def alt_grads(self):
        """A second gradient arena (same layout): a backward pass that runs concurrently with another one writes here,
        add_alt_grads() folds it into the arena the optimizer reads."""
        if getattr(self, '_alt', None) is None:
            g = torch.zeros_like(self.state.grads)
            c = NetState(self.state.params.data_ptr(), g.data_ptr(), self.state.packed.data_ptr(),
                         self.state.bn_stats.data_ptr(), self.state.bn_tracked.data_ptr())
            self._alt = (g, c)
        return self._alt[0]

    def add_alt_grads(self):
        """grads += alt (one rounding per element: the same sum an accumulating backward pass forms)."""
        g, alt = self.state.grads, self.alt_grads()
        rc = _lib().b200ocl_sgd_step(g.data_ptr(), alt.data_ptr(), g.data_ptr(), g.numel(), -1.0, 0.0, _stream())
        _native.check(rc, 'b200ocl_sgd_step')

    def backward(self, x, dout, ws, accumulate=False, eval_stats=False, alt=False, features=False):
        """loss.backward() for the forward of the same x kept in ws; fills (or adds to) the grad arena.
        eval_stats=True: the forward was forward_train(..., eval_stats=True).  alt=True: into the second arena.
        features=True: dout is the gradient of the encoder features [N, dim_in]; the head's backward is skipped and its
        gradient entries (linear.* for the classifier network) are left as they are."""
        _need_cuda(dout)
        x = self._x(x)
        dout = dout.detach().to(torch.float32).contiguous()
        n = dout.shape[0]
        width = self.dim_in if features else self.out_dim
        if x.shape[0] != n or dout.dim() != 2 or dout.shape[1] != width:
            raise ValueError('dout must be [N, %s] for the same N as x' % ('dim_in' if features else 'out_dim'))
        if alt:
            self.alt_grads()
        st_c = self._alt[1] if alt else self.state.c

        def launch(xin, din):
            rc = _lib().b200ocl_net_backward(ctypes.byref(self.desc), ctypes.byref(st_c), xin.data_ptr(),
                                             din.data_ptr(), n, ws.data_ptr(), ws.numel(),
                                             (1 if accumulate else 0) | (2 if eval_stats else 0) |
                                             (4 if features else 0), _stream())
            _native.check(rc, 'b200ocl_net_backward')

        slot = next((k[1] for k, w in self._train_ws.items() if w is ws and k[0] == n), None) if (_GRAPHS and not eval_stats) else None
        fwd = (self._graphs.get(('fwd', n, slot, False)) or self._graphs.get(('fwd', n, slot, True))) if slot is not None else None
        if fwd is not None:
            # the images are the static copy the graphed forward read (same data as x)
            key = ('bwd_feat' if features else 'bwd', n, slot, bool(accumulate), bool(alt))
            e = self._graphs.get(key)
            if e is None:
                e = self._graphs[key] = _Graphed([fwd.inputs[0], torch.empty_like(dout)], [])
            e.inputs[1].copy_(dout)
            e.run(lambda: launch(e.inputs[0], e.inputs[1]))
            return
        launch(x, dout)

    def sgd_step(self, lr, weight_decay=0.0, dst=None):
        rc = _lib().b200ocl_net_sgd_step(ctypes.byref(self.desc), ctypes.byref(self.state.c), float(lr),
                                         float(weight_decay), ctypes.byref(dst.c) if dst is not None else None,
                                         _stream())
        _native.check(rc, 'b200ocl_net_sgd_step')

    def sgd_step_clipped(self, lr, weight_decay, max_norm):
        """torch.nn.utils.clip_grad_norm_(parameters, max_norm) then opt.step() (agents/gdumb.py:82-83): the gradient
        arena is scaled in place by min(max_norm / (norm + 1e-6), 1) and the SGD step uses it.  Returns the norm before
        clipping as a device tensor [1]; the next call overwrites it.  Nothing is read back to the host."""
        if getattr(self, '_clip', None) is None:
            lib = _lib()
            ws = _workspace(lib.b200ocl_net_sgd_step_clipped_workspace_bytes(ctypes.byref(self.desc)), self.device)
            self._clip = (ws, torch.zeros(1, dtype=torch.float32, device=self.device))
        ws, norm = self._clip
        rc = _lib().b200ocl_net_sgd_step_clipped(ctypes.byref(self.desc), ctypes.byref(self.state.c), float(lr),
                                                 float(weight_decay), float(max_norm), norm.data_ptr(), ws.data_ptr(),
                                                 ws.numel(), _stream())
        _native.check(rc, 'b200ocl_net_sgd_step_clipped')
        return norm

    # ------------------------------------------------------------------ EWC++ (agents/ewc_pp.py)
    def ewc_state(self):
        """The EWC++ arenas, allocated once per engine and zero at first (ewc_pp.py:16-18 init_fisher): an object with
        running, tmp, normalized and prev, each an fp32 tensor in the parameter arena's layout."""
        if getattr(self, '_ewc', None) is None:
            n = self.info.n_params
            st = SimpleNamespace(**{name: torch.zeros(n, dtype=torch.float32, device=self.device)
                                    for name in ('running', 'tmp', 'normalized', 'prev')})
            st.c = EwcState(st.running.data_ptr(), st.tmp.data_ptr(), st.normalized.data_ptr(), st.prev.data_ptr())
            lib = _lib()
            st.ws = _workspace(max(lib.b200ocl_net_sgd_step_ewc_workspace_bytes(ctypes.byref(self.desc)),
                                   lib.b200ocl_ewc_consolidate_workspace_bytes(ctypes.byref(self.desc))), self.device)
            st.penalty = torch.zeros(1, dtype=torch.float32, device=self.device)
            self._ewc = st
        return self._ewc

    def sgd_step_ewc(self, lr, weight_decay, up, penalty, ema, ema_keep=0.0, ema_add=0.0, want_penalty=False):
        """One EWC++ step after backward (b200ocl_net_sgd_step_ewc): with ema, update_running_fisher first
        (running = ema_keep * running + ema_add * tmp, tmp = 0); with penalty, the gradient of up * sum F * (p - prev)^2
        added to the gradient arena; tmp += g * g; then opt.step().  want_penalty: returns sum F * (p - prev)^2 over the
        pre-step weights as a device tensor [1] (the next call overwrites it), else None.  Nothing is read back."""
        st = self.ewc_state()
        flags = (1 if penalty else 0) | (2 if ema else 0)
        rc = _lib().b200ocl_net_sgd_step_ewc(ctypes.byref(self.desc), ctypes.byref(self.state.c), ctypes.byref(st.c),
                                             float(lr), float(weight_decay), float(up), flags, float(ema_keep),
                                             float(ema_add), st.penalty.data_ptr() if want_penalty else None,
                                             st.ws.data_ptr(), st.ws.numel(), _stream())
        _native.check(rc, 'b200ocl_net_sgd_step_ewc')
        return st.penalty if want_penalty else None

    def ewc_consolidate(self):
        """The end of an EWC++ call (b200ocl_ewc_consolidate, ewc_pp.py:71-78): prev = params, normalized = running
        min-max normalised over every tensor."""
        st = self.ewc_state()
        rc = _lib().b200ocl_ewc_consolidate(ctypes.byref(self.desc), ctypes.byref(self.state.c), ctypes.byref(st.c),
                                            st.ws.data_ptr(), st.ws.numel(), _stream())
        _native.check(rc, 'b200ocl_ewc_consolidate')

    # ------------------------------------------------------------------ torch.optim.Adam
    def adam_state(self):
        """Adam's state, allocated once per engine: exp_avg and exp_avg_sq (fp32, the parameter arena's layout, zero at
        first) and `step`, the host-side step count shared by every tensor that has a gradient."""
        if getattr(self, '_adam', None) is None:
            n = self.info.n_params
            st = SimpleNamespace(exp_avg=torch.zeros(n, dtype=torch.float32, device=self.device),
                                 exp_avg_sq=torch.zeros(n, dtype=torch.float32, device=self.device), step=0)
            st.c = AdamState(st.exp_avg.data_ptr(), st.exp_avg_sq.data_ptr())
            self._adam = st
        return self._adam

    def adam_step(self, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, foreach=True, grad_div=None):
        """opt.step() of torch.optim.Adam (b200ocl_net_adam_step): the step count advances, the scalars are formed on
        the host as torch forms them, one launch updates params / exp_avg / exp_avg_sq, then the packed weights are
        refreshed.  grad_div: the gradient arena is divided by it first (the review trick's p.grad.clone() / 10.)."""
        st = self.adam_state()
        st.step += 1
        s = ops.adam_scalars(lr, betas, eps, weight_decay, st.step, grad_div)
        flags = (ops.ADAM_FOREACH if foreach else 0) | (ops.ADAM_GRAD_SCALE if grad_div is not None else 0)
        rc = _lib().b200ocl_net_adam_step(ctypes.byref(self.desc), ctypes.byref(self.state.c), ctypes.byref(st.c),
                                          ctypes.byref(s), flags, _stream())
        _native.check(rc, 'b200ocl_net_adam_step')

    def adam_step_ewc(self, lr, betas, eps, weight_decay, foreach, up, penalty, ema, ema_keep=0.0, ema_add=0.0,
                      want_penalty=False):
        """sgd_step_ewc with torch.optim.Adam's update in place of SGD's (b200ocl_net_adam_step_ewc), one launch."""
        ewc, st = self.ewc_state(), self.adam_state()
        st.step += 1
        s = ops.adam_scalars(lr, betas, eps, weight_decay, st.step)
        flags = (1 if penalty else 0) | (2 if ema else 0)
        rc = _lib().b200ocl_net_adam_step_ewc(ctypes.byref(self.desc), ctypes.byref(self.state.c), ctypes.byref(ewc.c),
                                              ctypes.byref(st.c), ctypes.byref(s), ops.ADAM_FOREACH if foreach else 0,
                                              float(up), flags, float(ema_keep), float(ema_add),
                                              ewc.penalty.data_ptr() if want_penalty else None, ewc.ws.data_ptr(),
                                              ewc.ws.numel(), _stream())
        _native.check(rc, 'b200ocl_net_adam_step_ewc')
        return ewc.penalty if want_penalty else None


def _check_labels(logits, labels):
    """One label per row: the kernels read labels[0..N-1] and nothing else tells them the length."""
    if labels.dim() != 1 or labels.shape[0] != logits.shape[0]:
        raise ValueError('labels must be 1-D with one entry per logits row: got %s for logits %s'
                         % (tuple(labels.shape), tuple(logits.shape)))


def ce_loss(logits, labels, want_grad=True, want_per_sample=False, want_correct=False, err=None):
    """Mean cross-entropy (b200ocl_ce_loss) of logits [N,C] at labels [N]; returns dict(loss[1], dlogits,
    per_sample, n_correct[1]).  err: int32 device flag [1] set to 1 by a label outside [0,C); such a row has zero
    dlogits and a NaN per_sample and adds nothing to loss (still divided by N) or n_correct."""
    _need_cuda(logits, labels, err)
    _check_labels(logits, labels)
    logits = logits.detach().to(torch.float32).contiguous()
    labels = labels.detach().to(torch.int64).contiguous()
    n, c = logits.shape
    dev = logits.device
    out = {'loss': torch.empty(1, dtype=torch.float32, device=dev)}
    out['dlogits'] = torch.empty_like(logits) if want_grad else None
    out['per_sample'] = torch.empty(n, dtype=torch.float32, device=dev) if want_per_sample else None
    out['n_correct'] = torch.empty(1, dtype=torch.int64, device=dev) if want_correct else None
    ptr = lambda t: 0 if t is None else t.data_ptr()
    rc = _lib().b200ocl_ce_loss(logits.data_ptr(), labels.data_ptr(), n, c, out['loss'].data_ptr(),
                                ptr(out['per_sample']), ptr(out['dlogits']), ptr(out['n_correct']), ptr(err), _stream())
    _native.check(rc, 'b200ocl_ce_loss')
    return out


def logit_mse(logits, memory, idx, alpha, err=None):
    """DER++'s logit term (b200ocl_logit_mse): alpha * F.mse_loss(logits, memory[idx]) for logits [n,C], the logit
    memory [mem,C] and int64 slot indices idx [n] (read in place, no gather); returns dict(loss[1], dlogits).  err: int32
    device flag [1] set to 1 by a slot outside the memory; such a row has zero dlogits and adds nothing to loss."""
    _need_cuda(logits, memory, idx, err)
    logits = logits.detach().to(torch.float32).contiguous()
    idx = idx.detach().to(torch.int64).contiguous().reshape(-1)
    n, c = logits.shape
    if memory.dtype != torch.float32 or not memory.is_contiguous() or memory.dim() != 2 or memory.shape[1] != c:
        raise ValueError('the logit memory must be a contiguous fp32 [mem, %d] tensor, got %s %s'
                         % (c, memory.dtype, tuple(memory.shape)))
    if idx.numel() != n:
        raise ValueError('idx must hold one slot per logits row: got %d for %d rows' % (idx.numel(), n))
    out = {'loss': torch.empty(1, dtype=torch.float32, device=logits.device), 'dlogits': torch.empty_like(logits)}
    rc = _lib().b200ocl_logit_mse(logits.data_ptr(), memory.data_ptr(), memory.shape[0], idx.data_ptr(), n, c,
                                  float(alpha), out['loss'].data_ptr(), out['dlogits'].data_ptr(),
                                  0 if err is None else err.data_ptr(), _stream())
    _native.check(rc, 'b200ocl_logit_mse')
    return out


def pcr_loss(feats, labels, proxies, temperature, dproxies=None, dbias=None, err=None):
    """PCR's proxy-contrastive loss (b200ocl_pcr_loss) of features [R,d] at labels [R] against the proxies, the
    classifier weight [C,d]; returns dict(loss[1], dfeats [R,d], dproxies [C,d], dbias [C] (zeros)).  dproxies / dbias:
    where to write those two gradients (the classifier's slices of the gradient arena), fresh tensors when None.  err:
    int32 device flag [1] set to 1 by a label outside [0, C); such a row adds nothing to the loss and has zero dfeats."""
    _need_cuda(feats, labels, proxies, dproxies, dbias, err)
    feats = feats.detach().to(torch.float32).contiguous()
    labels = labels.detach().to(torch.int64).contiguous()
    proxies = proxies.detach().to(torch.float32).contiguous()
    if feats.dim() != 2 or proxies.dim() != 2 or proxies.shape[1] != feats.shape[1]:
        raise ValueError('feats [R,d] and proxies [C,d] must share d: got %s and %s'
                         % (tuple(feats.shape), tuple(proxies.shape)))
    _check_labels(feats, labels)
    r, d = feats.shape
    c = proxies.shape[0]
    dev = feats.device
    for name, t, shape in (('dproxies', dproxies, (c, d)), ('dbias', dbias, (c,))):
        if t is not None and (t.dtype != torch.float32 or not t.is_contiguous() or tuple(t.shape) != shape):
            raise ValueError('%s must be a contiguous fp32 %s tensor' % (name, shape))
    out = {'loss': torch.empty(1, dtype=torch.float32, device=dev), 'dfeats': torch.empty_like(feats),
           'dproxies': torch.empty((c, d), dtype=torch.float32, device=dev) if dproxies is None else dproxies,
           'dbias': torch.empty(c, dtype=torch.float32, device=dev) if dbias is None else dbias}
    lib = _lib()
    ws = _workspace(lib.b200ocl_pcr_loss_workspace_bytes(r, c), dev)
    rc = lib.b200ocl_pcr_loss(feats.data_ptr(), labels.data_ptr(), r, d, proxies.data_ptr(), c, float(temperature),
                              out['loss'].data_ptr(), out['dfeats'].data_ptr(), out['dproxies'].data_ptr(),
                              out['dbias'].data_ptr(), 0 if err is None else err.data_ptr(), ws.data_ptr(), ws.numel(),
                              _stream())
    _native.check(rc, 'b200ocl_pcr_loss')
    return out


CLS_MODES = {'ce': 0, 'labels_trick': 1, 'separated_softmax': 2}


def cls_loss(logits, labels, mode='ce', cols=None, n_old=0, pos_table=None, teacher=None, w_ce=1.0, w_kd=0.0,
             err=None, want_grad=True, want_correct=False):
    """w_ce * criterion + w_kd * distillation (b200ocl_cls_loss); returns dict(loss[1], dlogits, n_correct[1]).
    mode 'labels_trick' | 'separated_softmax' | 'ce'; separated softmax takes cols = old_labels ++ new_labels (int64
    device tensor), the boundary n_old and pos_table (label -> position, -1 unmapped).  teacher: teacher logits or None
    (no distillation term).  err: int32 device flag [1] set to 1 by an unmapped label."""
    _need_cuda(logits, labels, cols, pos_table, teacher, err)
    _check_labels(logits, labels)
    logits = logits.detach().to(torch.float32).contiguous()
    labels = labels.detach().to(torch.int64).contiguous()
    n, c = logits.shape
    if teacher is not None:
        teacher = teacher.detach().to(torch.float32).contiguous()
        if teacher.shape != logits.shape:
            raise ValueError('teacher logits must match the logits in shape')
    m = CLS_MODES[mode]
    if m == 2:
        cols, pos_table = cols.to(torch.int64).contiguous(), pos_table.to(torch.int64).contiguous()
    dev = logits.device
    out = {'loss': torch.empty(1, dtype=torch.float32, device=dev)}
    out['dlogits'] = torch.empty_like(logits) if want_grad else None
    out['n_correct'] = torch.empty(1, dtype=torch.int64, device=dev) if want_correct else None
    ptr = lambda t: 0 if t is None else t.data_ptr()
    rc = _lib().b200ocl_cls_loss(logits.data_ptr(), labels.data_ptr(), n, c, m, ptr(cols) if m == 2 else 0,
                                 cols.numel() if m == 2 else 0, int(n_old), ptr(pos_table) if m == 2 else 0,
                                 pos_table.numel() if m == 2 else 0, ptr(teacher), float(w_ce), float(w_kd),
                                 out['loss'].data_ptr(), ptr(out['dlogits']), ptr(out['n_correct']), ptr(err), _stream())
    _native.check(rc, 'b200ocl_cls_loss')
    return out


def icarl_loss(logits, labels, pos_table, K, n_old, teacher=None, err=None, want_grad=True):
    """iCaRL's criterion (b200ocl_icarl_loss, agents/icarl.py:42-62): BCE with logits over the first K columns, summed
    over the columns and averaged over the N rows; returns dict(loss[1], dlogits).  The first labels.numel() rows are the
    stream batch (one-hot at pos_table[label], the int64 device table of lbl_inv_map, -1 unmapped), the rest are memory
    rows (zero target).  teacher: the previous model's logits; their sigmoids are the targets of the first n_old columns
    (None needs n_old == 0).  err: int32 device flag [1] set to 1 by a label whose position is not in [n_old, K)."""
    _need_cuda(logits, labels, pos_table, teacher, err)
    logits = logits.detach().to(torch.float32).contiguous()
    labels = labels.detach().to(torch.int64).contiguous()
    pos_table = pos_table.to(torch.int64).contiguous()
    n, c = logits.shape
    if teacher is not None:
        teacher = teacher.detach().to(torch.float32).contiguous()
        if teacher.shape != logits.shape:
            raise ValueError('teacher logits must match the logits in shape')
    out = {'loss': torch.empty(1, dtype=torch.float32, device=logits.device)}
    out['dlogits'] = torch.empty_like(logits) if want_grad else None
    ptr = lambda t: 0 if t is None else t.data_ptr()
    rc = _lib().b200ocl_icarl_loss(logits.data_ptr(), ptr(teacher), labels.data_ptr(), pos_table.data_ptr(),
                                   pos_table.numel(), n, labels.numel(), c, int(K), int(n_old), out['loss'].data_ptr(),
                                   ptr(out['dlogits']), ptr(err), _stream())
    _native.check(rc, 'b200ocl_icarl_loss')
    return out
