"""GPU: the engine's CUDA-graph replays against its eager launches, bit for bit, with new inputs on every call.

Every network-level call of the engine runs as a CUDA graph by default (engine._Graphed): the first call of a key runs
eagerly, the second captures N_EXEC executables and later calls copy their inputs into static buffers and replay the
executables in turn.  The fp64 pins (test_gpu_forward_fp64, test_gpu_backward_fp64, test_gpu_core50,
test_gpu_openloris) pass their own workspaces, so they never reach a replay.  Here two engines loaded with the same
state run the same calls, one with graphs on and one with graphs off, and after every call the outputs, the parameter,
packed, gradient and second-gradient arenas, the BN running statistics and counters, the teacher's arenas and the
tensors every cached train workspace saves for the backward must be the same bits.  The engine has no float atomics and reduces in a fixed order, so nothing
less than equality is expected.
  * every call kind (features_eval, forward_train, backward with accumulate / alt) at every batch size of the fp64 pins
    and of the agents' evaluation, five calls per key: the eager call, the capture, the three executables, wrap-around;
  * deferred and plain forwards interleaved on one (N, slot); weight steps (SGD, Adam, clipped SGD, load) and
    update_teacher between replays; replays on a side stream and SCR's two-stream step; a ninth batch size past the
    workspace caches and the return to a cached one;
  * launch accounting: a replay stands for exactly the launches of the eager call (graph_launch_count, bench.py);
  * the backward's weight gradients on the side stream, serially (B200OCL_WG_ASYNC=0), under the per-launch profiler
    and from a fifth caller stream that gets no side-stream slot, each in a fresh process, bit for bit;
  * whole agents (test_gpu_multirun.RUN_CASES and ER with the GSS update) over a short seeded stream with graphs on and
    off."""
import json
import os
import subprocess
import sys
from collections import defaultdict

import numpy as np
import pytest
import torch

import agent_cases
import test_gpu_backward_fp64 as bwd
import test_gpu_core50 as core50
import test_gpu_forward_fp64 as fwd
import test_gpu_multirun as mr
import test_gpu_openloris as openloris
from oracle import resnet as oresnet

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = 5                                                   # eager, capture + first executable, second, third, first
COMBOS = [(False, False), (True, False), (False, True), (True, True)]       # backward (accumulate, alt)

# The batch sizes of the agents' evaluation that the pins do not hold: test_batch = 128, the last batch of a CIFAR-100
# task's 1000 test images (7 x 128 + 104), and the nearest-class-mean pass over the buffer in chunks of 500 (mlp head).
# The ASER eval batches are in test_gpu_forward_fp64.CASES.
EVAL_SIZES = [(32, None, 128), (32, None, 104), (32, 'mlp', 500)]


def _shapes():
    out = set(fwd.CASES + bwd.CASES + bwd.EVAL_CASES + EVAL_SIZES)
    out |= {(core50.HW, None, n) for n in core50.FWD_BATCHES + core50.BWD_BATCHES}
    out |= {(openloris.HW, None, n) for n in openloris.FWD_BATCHES + openloris.BWD_BATCHES}
    return sorted(out, key=lambda c: (c[0], str(c[1]), c[2]))


SHAPES = _shapes()
SEEN = defaultdict(set)        # (hw, head) -> graph keys created by the engines of this file
CALLED = defaultdict(int)      # (hw, head, key) -> calls made through it
RAN = set()                    # the tests (and parameters) that finished, for the coverage check


@pytest.fixture(scope='module')
def engine():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import engine
    return engine


@pytest.fixture(autouse=True)
def graphs_restored():
    """Every test switches engine._GRAPHS back and forth; the next test finds it as it was."""
    if not torch.cuda.is_available():
        yield
        return
    from b200ocl import engine
    was = engine._GRAPHS
    yield
    engine.set_graphs(was)


def _same_bits(a, b):
    """Equal bit patterns (so -0.0 is not 0.0, and NaN left in the same places matches)."""
    if a.dtype == torch.float32 and b.dtype == torch.float32:
        a, b = a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)
    return torch.equal(a, b)


def _diff(a, b):
    if a.dtype.is_floating_point and a.shape == b.shape:
        d = (a.double() - b.double()).abs()
        d[torch.isnan(d)] = float('inf')
        return 'max |diff| %.3g at %d of %d elements' % (float(d.max()), int((d != 0).sum()), d.numel())
    if a.shape == b.shape:
        bad = torch.nonzero(a.reshape(-1) != b.reshape(-1)).reshape(-1)
        return '%d of %d elements, the first at %d' % (bad.numel(), a.numel(), int(bad[0]) if bad.numel() else -1)
    return 'shapes %s / %s' % (tuple(a.shape), tuple(b.shape))


class Pair:
    """Two engines loaded with the same weights and statistics: `g` runs with graphs on, `e` with graphs off."""

    def __init__(self, engine, hw, head, seed):
        self.engine, self.hw, self.head = engine, hw, head
        self.spec = oresnet.Spec(hw, 20, 100, head=head)
        self.g, self.e = self._make(seed), self._make(seed)
        self.layouts = {}
        self.gen = torch.Generator().manual_seed(1000 * hw + seed)

    def _make(self, seed):
        eng = self.engine.Engine(self.hw, 100, head=self.head)
        eng.load(*self.weights(seed))
        return eng

    def weights(self, seed):
        params, bn = oresnet.seeded_state(self.spec, seed)
        return list(params.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(self.spec)]

    def images(self, n):
        return torch.rand(n, 3, self.hw, self.hw, generator=self.gen).cuda()

    def dout(self, n):
        return torch.randn(n, self.g.out_dim, generator=self.gen).cuda()

    def cache_ws(self, n, slot=0):
        """The (n, slot) train workspace of both engines, zeroed, so that unwritten entries compare equal."""
        for eng in (self.g, self.e):
            eng.train_workspace(n, slot).zero_()

    def state(self):
        g, e = self.g, self.e
        out = [(name, getattr(g.state, name), getattr(e.state, name))
               for name in ('params', 'grads', 'packed', 'bn_stats', 'bn_tracked')]
        if getattr(g, '_alt', None) is not None or getattr(e, '_alt', None) is not None:
            out.append(('alt grads', g.alt_grads(), e.alt_grads()))
        if g.teacher is not None or e.teacher is not None:
            assert g.teacher is not None and e.teacher is not None
            out += [('teacher ' + name, getattr(g.teacher, name), getattr(e.teacher, name))
                    for name in ('params', 'packed', 'bn_stats', 'bn_tracked')]
        assert set(g._train_ws) == set(e._train_ws)
        for k, w in g._train_ws.items():
            out += [('train workspace %s %s' % (k, name), a, b) for name, a, b in self.saved(k[0], w, e._train_ws[k])]
        return out

    def saved(self, n, wg, we):
        """The tensors a forward saves in a train workspace for the backward (train_ws_layout): per conv layer the raw and
        activated outputs and the batch statistics, and feat / hid / proj.  The rest of the workspace is the backward's
        scratch, whose layout depends on whether the weight gradients ran on a side stream or serially: a process gets
        four side-stream slots, so which form a call takes depends on the streams that came before it."""
        layout = self.layouts.get(n)
        if layout is None:
            layout = self.layouts[n] = [self.engine.train_ws_layout(self.g.desc, n, i) for i in range(self.g.info.n_bn)]
        out = []
        for i, L in enumerate(layout):
            act = 4 * n * L.hout * L.wout * L.cout
            out += [('layer %d %s' % (i, name), off, nbytes) for name, off, nbytes in
                    (('z', L.z, act), ('a', L.a, act), ('mean', L.mean, 4 * L.cout), ('invstd', L.invstd, 4 * L.cout))]
        L0 = layout[0]
        out.append(('feat', L0.feat, 4 * n * self.g.dim_in))
        if self.head == 'mlp':
            out.append(('hid', L0.hid, 4 * n * self.g.dim_in))
        if self.head in ('mlp', 'linear'):
            out.append(('proj', L0.proj, 4 * n * self.g.out_dim))
        return [(name, wg[off:off + nbytes], we[off:off + nbytes]) for name, off, nbytes in out]

    def call(self, what, fn):
        """fn(engine) on the eager engine with graphs off, then on the other with graphs on; the results and the whole
        state must be the same bits.  Launch accounting: a graph's per-replay count (_Graphed.kernels) stands for the
        launches the eager call made.  Returns the graph keys the call went through."""
        from b200ocl import _native
        engine = self.engine
        engine.set_graphs(False)
        before = _native.launch_count()
        ref = fn(self.e)
        eager = _native.launch_count() - before
        engine.set_graphs(True)
        phase = {k: len(v.graphs) for k, v in self.g._graphs.items()}
        turns = {k: (v.calls, v.turn) for k, v in self.g._graphs.items()}
        before, replayed = _native.launch_count(), engine.graph_launch_count()
        got = fn(self.g)
        launched, replayed = _native.launch_count() - before, engine.graph_launch_count() - replayed
        engine.set_graphs(False)
        used = [k for k, v in self.g._graphs.items() if turns.get(k) != (v.calls, v.turn) or phase.get(k) != len(v.graphs)]
        where = '%s (%dx%d, head %s; graph keys %s)' % (what, self.hw, self.hw, self.head, used or 'none: eager')
        SEEN[(self.hw, self.head)].update(self.g._graphs)
        for k in used:
            CALLED[(self.hw, self.head, k)] += 1
        # expected launches on the graphed engine: the eager ones, plus N_EXEC captures of a key captured now, minus the
        # launches a replay stands for
        N_EXEC = engine._Graphed.N_EXEC
        captured = sum(self.g._graphs[k].kernels for k in used if not phase.get(k) and self.g._graphs[k].graphs)
        replays = sum(self.g._graphs[k].kernels for k in used if self.g._graphs[k].graphs)
        assert replayed == replays, (where, 'graph_launch_count moved by', replayed, 'for replays of', replays)
        assert launched == eager + N_EXEC * captured - replays, (where, 'launches', launched, 'eager call', eager,
                                                                 'per-replay counts', [self.g._graphs[k].kernels for k in used])
        torch.cuda.synchronize()
        got = got if isinstance(got, (tuple, list)) else (got,)
        ref = ref if isinstance(ref, (tuple, list)) else (ref,)
        for i, (a, b) in enumerate(zip(got, ref)):
            if a is not None or b is not None:
                assert _same_bits(a, b), '%s: output %d differs from the eager call: %s' % (where, i, _diff(a, b))
        for name, a, b in self.state():
            assert _same_bits(a, b), '%s: %s differs from the eager call: %s' % (where, name, _diff(a, b))
        return used

    def replayed(self, key, calls=CALLS):
        """The key went through its eager call, the capture and replays of every executable, wrapping around."""
        e = self.g._graphs.get(key)
        assert e is not None, 'no graph under the key %s after %d calls (%dx%d, head %s; keys %s)' % (
            key, calls, self.hw, self.hw, self.head, sorted(self.g._graphs, key=str))
        N_EXEC = self.engine._Graphed.N_EXEC
        assert len(e.graphs) == N_EXEC and e.turn == (calls - 1) % N_EXEC and calls - 1 > N_EXEC, (key, e.turn)
        assert CALLED[(self.hw, self.head, key)] >= calls, (key, CALLED[(self.hw, self.head, key)])


def _round(pair, n, i, slot=0, defer=False, combos=COMBOS, label=''):
    """One round of new images: features_eval, forward_train, and a backward with new dout per (accumulate, alt)."""
    x = pair.images(n)
    pair.call('%sfeatures_eval(N=%d) call %d' % (label, n, i), lambda eng: eng.features_eval(x))
    pair.call('%sforward_train(N=%d, slot=%d, defer_stats=%s) call %d' % (label, n, slot, defer, i),
              lambda eng: eng.forward_train(x, slot=slot, defer_stats=defer)[0])
    if defer:
        pair.call('%sapply_running_stats(N=%d) call %d' % (label, n, i),
                  lambda eng: eng.apply_running_stats(eng.train_workspace(n, slot), n))
    for acc, alt in combos:
        d = pair.dout(n)
        pair.call('%sbackward(N=%d, slot=%d, accumulate=%s, alt=%s) call %d' % (label, n, slot, acc, alt, i),
                  lambda eng: eng.backward(x, d, eng.train_workspace(n, slot), accumulate=acc, alt=alt))


def _keys(n, slot=0, defer=False, combos=COMBOS):
    return [('eval', n), ('fwd', n, slot, defer)] + [('bwd', n, slot, a, b) for a, b in combos]


# ----------------------------------------------------------------------------- every call kind at every pinned size
@pytest.mark.parametrize('hw,head,N', SHAPES)
def test_replays_match_eager_calls(engine, hw, head, N):
    """Five calls per key, new images and gradients on each, at every batch size of the fp64 pins (CIFAR, the mlp,
    linear and None heads, Mini-ImageNet, CORe50, OpenLORIS) and of the agents' evaluation."""
    pair = Pair(engine, hw, head, N)
    pair.cache_ws(N)
    for i in range(CALLS):
        _round(pair, N, i)
    for key in _keys(N):
        pair.replayed(key)
    RAN.add(('shape', hw, head, N))


# ----------------------------------------------------------------------------- the hazards of the key logic
@pytest.mark.parametrize('hw,head,N', [(32, None, 20), (32, 'mlp', 110), (84, None, 22)])
def test_deferred_and_plain_forwards_interleaved(engine, hw, head, N):
    """Deferred and plain forwards of one (N, slot) share the static input but not the graph: alternating them with
    different images, each followed by its backward, must neither replay the other form nor read its images."""
    pair = Pair(engine, hw, head, 3 + N)
    pair.cache_ws(N)
    for i in range(2 * CALLS):
        _round(pair, N, i // 2, defer=(i % 2 == 0), combos=[(False, False)])
    for defer in (True, False):
        pair.replayed(('fwd', N, 0, defer))
    pair.replayed(('bwd', N, 0, False, False), 2 * CALLS)
    RAN.add('deferred')


@pytest.mark.parametrize('hw,head,N', [(32, None, 20), (84, None, 10)])
def test_replays_follow_weight_updates(engine, hw, head, N):
    """SGD, Adam, clipped SGD and load() between replays: the captured graphs must read the new arenas."""
    pair = Pair(engine, hw, head, 11 + N)
    pair.cache_ws(N)
    steps = ('sgd_step', 'adam_step', 'sgd_step_clipped', 'load')

    def step(eng, name, i):
        if name == 'sgd_step':
            eng.sgd_step(0.05, 1e-4)
        elif name == 'adam_step':
            eng.adam_step(1e-3, weight_decay=1e-4)
        elif name == 'sgd_step_clipped':
            return eng.sgd_step_clipped(0.1, 0.0, 0.5)
        else:
            eng.load(*pair.weights(100 + i))
    for i in range(2 * len(steps)):
        _round(pair, N, i, combos=[(False, False)])
        name = steps[i % len(steps)]
        pair.call('%s after round %d' % (name, i), lambda eng: step(eng, name, i))
    for key in _keys(N, combos=[(False, False)]):
        pair.replayed(key, 2 * len(steps))
    RAN.add('weights')


def test_teacher_replays_follow_update_teacher(engine):
    """LwF / iCaRL / the kd tricks: update_teacher() between teacher forwards, the student trained in between.  The
    teacher graph must read the teacher's arenas as they are now."""
    N = 10
    pair = Pair(engine, 32, None, 61)
    slot = engine.Engine.TEACHER_SLOT
    pair.cache_ws(N)
    pair.cache_ws(N, slot)
    for i in range(CALLS + 1):
        pair.call('update_teacher() before round %d' % i, lambda eng: eng.update_teacher())
        for j in range(2):                  # two teacher forwards per teacher, new images each
            x = pair.images(N)
            pair.call('teacher_forward(N=%d) round %d call %d' % (N, i, j), lambda eng: eng.teacher_forward(x))
        _round(pair, N, i, combos=[(False, False)], label='student ')
        pair.call('sgd_step after round %d' % i, lambda eng: eng.sgd_step(0.1))
    pair.replayed(('teacher', N, slot, False), 2 * (CALLS + 1))
    RAN.add('teacher')


def _scr_step(side, x1, x2, d1, d2, concurrent):
    """learners.SupContrastReplay.replay_step's network calls with given dout per view (the SupCon gradient's
    place), two-stream form (concurrent) or one-stream form; then the SGD step."""
    def step(eng):
        n = x1.shape[0]
        if concurrent:
            main = torch.cuda.current_stream()
            side.wait_stream(main)
            with torch.cuda.stream(side):
                f2, ws2 = eng.forward_train(x2, slot=1, defer_stats=True)
            f1, ws1 = eng.forward_train(x1, slot=0, defer_stats=True)
            main.wait_stream(side)
            eng.apply_running_stats(ws1, n)
            eng.apply_running_stats(ws2, n)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                eng.backward(x2, d2, ws2, alt=True)
            eng.backward(x1, d1, ws1)
            main.wait_stream(side)
            eng.add_alt_grads()
        else:
            f1, ws1 = eng.forward_train(x1, slot=0)
            f2, ws2 = eng.forward_train(x2, slot=1)
            eng.backward(x1, d1, ws1)
            eng.backward(x2, d2, ws2, accumulate=True)
        eng.sgd_step(0.1)
        return f1, f2
    return step


def test_replays_on_side_streams(engine):
    """Every call kind replayed on a non-default stream, then SCR's two-stream step (each view's forward and backward
    on its own stream, the second backward into the second arena) and its one-stream form, against the eager calls on
    the same streams."""
    N = 20
    pair = Pair(engine, 32, 'mlp', 23)
    pair.cache_ws(N)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for i in range(CALLS):
            _round(pair, N, i, label='side stream: ')
    torch.cuda.current_stream().wait_stream(s)
    for key in _keys(N):
        pair.replayed(key)
    n = 110
    pair.cache_ws(n, 0)
    pair.cache_ws(n, 1)
    side = torch.cuda.Stream()
    for concurrent in (True, False):
        for i in range(CALLS):
            x1, x2, d1, d2 = pair.images(n), pair.images(n), pair.dout(n), pair.dout(n)
            pair.call('SCR step (N=%d, two streams=%s) call %d' % (n, concurrent, i),
                      _scr_step(side, x1, x2, d1, d2, concurrent))
    for key in [('fwd', n, 0, True), ('fwd', n, 1, True), ('bwd', n, 1, False, True), ('fwd', n, 0, False),
                ('fwd', n, 1, False), ('bwd', n, 1, True, False)]:
        pair.replayed(key)
    pair.replayed(('bwd', n, 0, False, False), 2 * CALLS)          # the first view's backward in both forms
    RAN.add('streams')


def test_a_ninth_batch_size_runs_eagerly(engine):
    """Eight batch sizes fill the eval and train workspace caches; a ninth runs eagerly on workspaces of its own (no
    graph key), and the cached sizes keep replaying afterwards."""
    pair = Pair(engine, 32, None, 9)
    sizes = list(range(1, 9))
    for n in sizes:
        pair.cache_ws(n)
        for i in range(2):
            _round(pair, n, i, combos=[(False, False)])
    assert len(pair.g._eval_ws) == 8 and len(pair.g._train_ws) == 8
    n = 9
    for i in range(CALLS):
        x, d = pair.images(n), pair.dout(n)
        ws = {}

        def forward(eng):
            out, ws[id(eng)] = eng.forward_train(x)
            return out
        assert pair.call('features_eval(N=%d) call %d' % (n, i), lambda eng: eng.features_eval(x)) == []
        assert pair.call('forward_train(N=%d) call %d' % (n, i), forward) == []
        assert pair.call('backward(N=%d) call %d' % (n, i), lambda eng: eng.backward(x, d, ws[id(eng)])) == []
    assert not any(k[1] == n for k in pair.g._graphs) and n not in pair.g._eval_ws
    for i in range(2, CALLS):
        _round(pair, 3, i, combos=[(False, False)])
    for key in _keys(3, combos=[(False, False)]):
        pair.replayed(key)
    RAN.add('ninth')


# ----------------------------------------------------------------------------- serial and side-stream weight gradients
_WG_SCRIPT = r'''
import json, os, sys
import torch
from b200ocl import _native, engine
from oracle import resnet as oresnet

form, out_dir, cases = sys.argv[1], sys.argv[2], [tuple(c) for c in json.loads(sys.argv[3])]
engine.set_graphs(False)
lib = _native.lib()


def case(hw, head, N):
    spec = oresnet.Spec(hw, 20, 100, head=head)
    params, bn = oresnet.seeded_state(spec, 7 + N)
    eng = engine.Engine(hw, 100, head=head)
    eng.load(list(params.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
    gen = torch.Generator().manual_seed(1000 * hw + N)
    x = torch.rand(N, 3, hw, hw, generator=gen).cuda()
    dout = torch.randn(N, eng.out_dim, generator=gen).cuda()
    ws = eng.new_train_workspace(N)
    eng.forward_train(x, ws=ws)
    return eng, x, dout, ws


others = []
if form == 'fifth':                 # four other caller streams take the four side-stream slots first
    for _ in range(4):
        others.append(torch.cuda.Stream())
        with torch.cuda.stream(others[-1]):
            eng, x, dout, ws = case(32, None, 2)
            eng.backward(x, dout, ws)
        torch.cuda.synchronize()
if form == 'profiled':
    lib.b200ocl_profile_begin()
grads = {}
for hw, head, N in cases:
    eng, x, dout, ws = case(hw, head, N)
    eng.state.grads.fill_(float('nan'))
    eng.backward(x, dout, ws)
    grads['%d/%r/%d' % (hw, head, N)] = eng.state.grads.view(torch.int32).cpu()     # bits: unwritten entries stay NaN
# the streams one backward's kernels ran on, from the CUDA trace
eng, x, dout, ws = case(*cases[-1])
torch.cuda.synchronize()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    eng.backward(x, dout, ws)
    torch.cuda.synchronize()
trace = os.path.join(out_dir, form + '.trace.json')
prof.export_chrome_trace(trace)
with open(trace) as fh:
    events = json.load(fh)['traceEvents']
streams = sorted({ev['args']['stream'] for ev in events if ev.get('cat') == 'kernel'})
records = lib.b200ocl_profile_end() if form == 'profiled' else 0
torch.save({'grads': grads, 'streams': streams, 'records': records}, os.path.join(out_dir, form + '.pt'))
'''

WG_FORMS = {'side': {}, 'serial': {'B200OCL_WG_ASYNC': '0'}, 'profiled': {}, 'fifth': {}}


def test_weight_gradients_serial_and_side_stream_are_the_same_bits(engine, tmp_path):
    """The backward at every test_gpu_backward_fp64 shape with its weight gradients on the side stream (the default),
    serially (B200OCL_WG_ASYNC=0), with the per-launch profiler on (bench.py's profiled step) and from a fifth caller
    stream, which finds the four side-stream slots taken.  Each form runs in a process of its own (the slots and the
    switch are process-wide and read once); the CUDA trace of one backward shows which form ran."""
    script = tmp_path / 'wg_form.py'
    script.write_text(_WG_SCRIPT)
    cases = json.dumps([list(c) for c in bwd.CASES])
    out = {}
    for form, extra in WG_FORMS.items():
        env = {k: v for k, v in os.environ.items() if k != 'B200OCL_WG_ASYNC'}
        env.update(extra)
        env['PYTHONPATH'] = os.pathsep.join([ROOT] + [p for p in env.get('PYTHONPATH', '').split(os.pathsep) if p])
        cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [str(script), form, str(tmp_path), cases]
        r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, (form, r.returncode, r.stderr[-3000:])
        out[form] = torch.load(str(tmp_path / (form + '.pt')))
    streams = {form: len(o['streams']) for form, o in out.items()}
    assert streams == {'side': 2, 'serial': 1, 'profiled': 1, 'fifth': 1}, streams
    assert out['profiled']['records'] > 0
    ref = out['side']['grads']
    assert len(ref) == len(bwd.CASES)
    for form, o in out.items():
        for name, g in ref.items():
            assert torch.equal(o['grads'][name], g), (form, name, _diff(o['grads'][name], g))
    RAN.add('wgrad')


# ----------------------------------------------------------------------------- whole agents
AGENT_CASES = sorted(mr.RUN_CASES + ('er_gss',))
AGENT_KEYS = set()


def _agent_run(engine, case, graphs, r=2):
    from b200ocl import memory, multirun
    engine.set_graphs(graphs)
    memory.flush_pending()
    memory.ClassBalancedRandomSampling.reset()
    multirun.RunRng(multirun.run_seed(mr.SEED, r)).swap_in()
    agent = mr._maker(agent_cases.params(case), {})(r)
    tasks, loaders = mr._data(r)
    acc = []
    for x, y in tasks:
        agent.train_learner(x, y)
        acc.append(agent.evaluate(loaders))
    torch.cuda.synchronize()
    memory.flush_pending()
    return np.array(acc), agent_cases.final_state(agent), agent.engine._graphs


@pytest.mark.parametrize('case', AGENT_CASES)
def test_agents_with_and_without_graphs(engine, case):
    """A short seeded stream (three tasks of three calls) with graphs on and off: accuracies and final state
    (agent_cases.final_state), bit for bit."""
    acc_g, final_g, graphs = _agent_run(engine, case, True)
    acc_e, final_e, eager = _agent_run(engine, case, False)
    assert not eager
    assert any(len(e.graphs) for e in graphs.values()), (case, 'no call was replayed')
    AGENT_KEYS.update(graphs)
    assert np.array_equal(acc_g, acc_e), (case, acc_g, acc_e)
    assert len(final_g) == len(final_e)
    for i, (a, b) in enumerate(zip(final_g, final_e)):     # params, bn_stats, bn_tracked, then the rest of final_state
        assert _same_bits(a, b), (case, i, _diff(a, b))
    RAN.add(('agent', case))


# ----------------------------------------------------------------------------- coverage
def test_graph_keys_cover_every_form_and_pinned_size(engine):
    """Over this file, graphs were captured and replayed for every batch size of the fp64 pins and of the agents'
    evaluation in every call kind, and for every key form: eval, plain and deferred forwards on slots 0 and 1, the
    teacher's forward, and backward with each (accumulate, alt)."""
    wanted = {('shape',) + c for c in SHAPES} | {('agent', c) for c in AGENT_CASES}
    wanted |= {'deferred', 'weights', 'teacher', 'streams', 'ninth', 'wgrad'}
    if not wanted <= RAN:
        pytest.skip('needs the whole file: %d tests that create graph keys did not run here' % len(wanted - RAN))
    for hw, head, N in SHAPES:
        missing = [k for k in _keys(N) if CALLED[(hw, head, k)] < CALLS or k not in SEEN[(hw, head)]]
        assert not missing, (hw, head, N, missing)
    every = set().union(*SEEN.values()) | AGENT_KEYS
    forms = {k[:1] + tuple(x for x in k[2:]) for k in every}
    want = {('eval',), ('fwd', 0, False), ('fwd', 0, True), ('fwd', 1, False), ('fwd', 1, True),
            ('teacher', engine.Engine.TEACHER_SLOT, False), ('bwd', 1, False, True), ('bwd', 1, True, False)}
    want |= {('bwd', 0, a, b) for a, b in COMBOS}
    assert want <= forms, sorted(want - forms, key=str)
    agent_forms = {k[:1] + tuple(x for x in k[2:]) for k in AGENT_KEYS}
    assert {('eval',), ('fwd', 0, False), ('fwd', 1, True), ('bwd', 1, False, True), ('teacher', 6, False)} <= agent_forms, \
        sorted(agent_forms, key=str)
