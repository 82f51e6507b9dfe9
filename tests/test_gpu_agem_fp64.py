"""GPU: A-GEM against fp64 on the four networks it runs on, CIFAR-100 (32x32, 100 classes), Mini-ImageNet (84x84, 100),
OpenLORIS (50x50, 69, new-instance tasks) and CORe50 (128x128, 50, the 2560-input classifier).

  * The projection kernel (b200ocl_agem_project through ops.agem_project) at the four gradient-arena lengths and at the
    edge lengths of its launch (grid = min(2 SMs, 296) CTAs of 256 threads striding over the arena): 1, 31, 255, 256,
    257, grid*256 - 1, grid*256, grid*256 + 1 and a length that leaves CTAs without an element.  Rows: the engine's own
    stream and memory gradients, inner products far negative and far positive, g_ref = 0, disjoint supports (prod
    exactly 0), one planted product of -1e-30, g = -g_ref and subnormal entries.  Checked against fp64 with the
    kernel's rounding bound (project_bound, itself checked against an fp32 emulation in tests/test_agem_bound.py): the
    output, both dot products, the decision (fp64's prod < 0), every element written into a NaN-filled output between
    guard bands, the same bits with the output separate or aliasing either input and on a repeat, and the refusals.
  * learners.AGEM.replay_step against oracle.agem.step in float64 on every network, from the same weights and with the
    reference's random streams: the projected arena against the fp64 projection of the very arenas the kernel was
    given (within 2x project_bound), parameters, the update (Adam's against the fp64 Adam step of the engine's own
    gradients) and BN running statistics after every step, the memory bit for bit,
    and the decision on every step, both decisions occurring on every network.  Variants at CIFAR-100: mem_iters = 2, a
    memory smaller than eps_mem_batch, Adam, kd_trick with labels_trick; at CORe50 the memory draw's forward takes
    other convolution templates than the stream batch's.
  * The reference's own A-GEM runs at 84x84 and 128x128 (tests/golden/agem_maps.npz, written by
    tests/golden/make_golden_agem_maps.py) with the drop-in comparison and bars of test_gpu_dropin.py.

Measured on an H100 80GB HBM3 (SXM, 132 SMs, 700 W power limit), largest value over all cases of this file: see the
bars below.  The file runs in 46-55 s there (pytest's count), most of it the fp64 oracle on the CPU.

Mutations, each made on a scratch copy and never kept: the learner projecting before the memory backward fails every
learner test (the decision: g_ref is then the stream gradient, prod > 0 where fp64 has prod < 0).  On the CPU
(tests/test_agem_bound.py) the bit-exact check refuses the emulated kernel with `prod <= 0`, with a coefficient from
fp32-rounded dots and with a re-reduction that drops the last partial.  A grid-stride loop that skips the last element
leaves a NaN in run_guarded's output; that mutation was not built.
"""
import copy
import hashlib
import json
import os
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import adam as oadam
from oracle import agem as oagem
from oracle import replay_step as ors
from oracle import resnet as oresnet

pytestmark = pytest.mark.gpu

NETS = {'cifar100': (32, 100), 'mini_imagenet': (84, 100), 'openloris': (50, 69), 'core50': (128, 50)}
U32, U64 = 2.0 ** -24, 2.0 ** -53
U80 = float(np.finfo(np.longdouble).eps) / 2   # x87 extended precision on x86-64 (2^-64); u64 where there is none
TINY = 2.0 ** -150        # half the spacing of fp32 subnormals: the absolute error of one rounding there

# |kernel - fp64| <= BOUND_FACTOR x project_bound, the factor of test_gpu_loss_fp64.py.  Largest measured
# |kernel - fp64| / (2 project_bound): 0.498 (CIFAR-100 learner, Adam and kd_trick variants), 0.496 (CORe50 arena
# rows), 0.473 (edge lengths): the kernel uses just under the whole single bound, as a bound of that tightness should.
BOUND_FACTOR = 2.0
# whole step, |engine - oracle| / |oracle| (L2, _rel) over the parameters and over the BN running statistics: the
# step tolerance of test_gpu_replay.py.  Measured maximum: parameters 1.0e-4 (CORe50, first task-1 step), BN running
# statistics 1.2e-5 (mem_iters = 2, first step: its second forward runs from the first iteration's fp32 weights).
STEP_TOL = 2e-4
# the SGD update itself, |(p_after - p_before) engine - oracle| / |oracle's| (L2).  About 3x the largest measured,
# 1.6e-2 (mem_iters = 2, first step, whose second iteration runs from the first one's weights); single-iteration steps
# reach 4.6e-3, where a ReLU flip moves a few weights.
UPDATE_TOL = 5e-2
# the Adam update against the fp64 Adam step of the engine's own gradient arena (same L2 measure), about 3x the
# largest measured, 1.6e-4 (fourth step)
ADAM_UPDATE_TOL = 5e-4
# every |prod| / (|g| |g_ref|) of the learner runs sits at least this far from 0 (10x STEP_TOL), so that the fp64
# decision cannot turn on the engine's fp32 gradients; the smallest measured is 5.6e-3 (kd_trick + labels_trick)
COS_MARGIN = 10 * STEP_TOL
GUARD = 64                # guard elements on either side of the output
GUARD_BYTE = 0x5A


def spec_of(data):
    hw, ncls = NETS[data]
    return oresnet.Spec(hw, 20, ncls)


def arena_len(data):
    return sum(int(np.prod(s)) for s in oresnet.param_shapes(spec_of(data)).values())


@pytest.fixture(scope='module')
def b():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import _native, engine, learners, memory, nets, ops, registry
    return SimpleNamespace(native=_native, engine=engine, learners=learners, memory=memory, nets=nets, ops=ops,
                           registry=registry)


def grid_of():
    return min(2 * torch.cuda.get_device_properties(0).multi_processor_count, 296)


def edge_lengths():
    G = grid_of() * 256
    return [1, 31, 255, 256, 257, G // 2 + 7, G - 1, G, G + 1]


# ------------------------------------------------------------------------------------------------ the bound
def project_bound(g, r):
    """fp64 facts and the rounding bound of the kernel on fp32 vectors g, r: dict(P, R, eP, eR, project, ref, bound).
    P and R are the dots of products that are exact in float64, summed in extended precision and rounded once; eP / eR
    bound the kernel's own fp64 summation error plus that sum's, n (u64 + u80) sum |g_i r_i| and n (u64 + u80) R.  With c = P / R the kernel forms the fp32
    rounding of its fp64 quotient, multiplies by r_i (fused or not) and subtracts:
        |out~ - out| <= 2 u |c r_i| + u |out_i| + |c r_i| (eP / |P| + eR / R + 2 u64) + TINY (|r_i| + 2).
    Without a projection the output is g bit for bit (bound 0)."""
    g64, r64 = np.asarray(g, np.float32).astype(np.float64), np.asarray(r, np.float32).astype(np.float64)
    gr = g64 * r64
    n = g64.size
    P, R = float(gr.astype(np.longdouble).sum()), float((r64 * r64).astype(np.longdouble).sum())
    eP, eR = n * (U64 + U80) * float(np.abs(gr).sum()), n * (U64 + U80) * R
    project = P < 0
    if not project:
        return dict(P=P, R=R, eP=eP, eR=eR, project=False, ref=g64, bound=np.zeros_like(g64))
    c = P / R
    ref = g64 - c * r64
    cr = np.abs(c * r64)
    bound = 2 * U32 * cr + U32 * np.abs(ref) + cr * (eP / abs(P) + eR / R + 2 * U64) + TINY * (np.abs(r64) + 2)
    return dict(P=P, R=R, eP=eP, eR=eR, project=True, ref=ref, bound=bound)


def emulate(g, r, c32, fused):
    """The kernel's per-element arithmetic in fp32 for the coefficient c32: fma(-c, r_i, g_i) when the compiler
    contracts g_i - c * r_i, else the product and the difference each rounded."""
    g, r, c32 = np.asarray(g, np.float32), np.asarray(r, np.float32), np.float32(c32)
    if fused:
        return oadam.fma(-c32, r, g)
    return (g - (c32 * r).astype(np.float32)).astype(np.float32)


def coefficients(f):
    """The fp32 coefficients the kernel may form: fl32 of its fp64 quotient P~ / R~, which lies within
    (eP / |P| + eR / R + 2 u64) of P / R; both neighbours when that interval holds an fp32 rounding boundary."""
    q = f['P'] / f['R']
    d = abs(q) * (f['eP'] / abs(f['P']) + f['eR'] / f['R'] + 2 * U64)
    return sorted({float(np.float32(q - d)), float(np.float32(q)), float(np.float32(q + d))})


def check_projection(g, r, out, dots=None, where=''):
    """Kernel output (and dots) against project_bound, and bit for bit against the fp32 emulation of its arithmetic
    with a coefficient coefficients() allows, fused or unfused alike over the whole row.  Returns the largest
    |out - ref| / (BOUND_FACTOR * bound)."""
    f = project_bound(g, r)
    assert f['P'] == 0.0 or abs(f['P']) > f['eP'], (where, 'the decision turns on the summation order', f['P'], f['eP'])
    out = np.asarray(out, np.float32)
    assert np.all(np.isfinite(out)), where
    if dots is not None:
        d = np.asarray(dots, np.float64)
        assert abs(d[0] - f['P']) <= U32 * abs(f['P']) + f['eP'] + TINY, (where, 'prod', d[0], f['P'])
        assert abs(d[1] - f['R']) <= U32 * f['R'] + f['eR'] + TINY, (where, 'prod_ref', d[1], f['R'])
        assert (d[0] < 0) == f['project'], (where, 'decision', d[0], f['P'])
    if not f['project']:
        assert np.array_equal(out.view(np.int32), np.asarray(g, np.float32).view(np.int32)), (where, 'no projection: g')
        return 0.0
    err = np.abs(out.astype(np.float64) - f['ref'])
    ratio = err / (BOUND_FACTOR * f['bound'])
    k = int(np.argmax(ratio))
    assert ratio[k] <= 1.0, (where, 'element', k, float(out[k]), f['ref'][k], f['bound'][k])
    bits = out.view(np.int32)
    assert any(np.array_equal(emulate(g, r, c, fused).view(np.int32), bits)
               for c in coefficients(f) for fused in (True, False)), (where, 'not the fp32 arithmetic of fl32(P / R)')
    return float(ratio.max())


# ------------------------------------------------------------------------------------------------ rows
def synthetic_rows(n, seed):
    """(name, g, r) fp32 rows of length n."""
    rs = np.random.RandomState(seed)
    base = rs.standard_normal(n).astype(np.float32)
    noise = rs.standard_normal(n).astype(np.float32)
    rows = [('far_negative', (-3 * base + noise).astype(np.float32), base),
            ('far_positive', (3 * base + noise).astype(np.float32), base),
            ('zero_ref', noise, np.zeros(n, np.float32))]
    even = (np.arange(n) % 2 == 0)
    rows.append(('disjoint', np.where(even, noise, 0).astype(np.float32), np.where(even, 0, base).astype(np.float32)))
    g, r = np.where(even, noise, 0).astype(np.float32), np.where(even, 0, base).astype(np.float32)
    j = n - 1                                      # the planted product sits on the last element
    g[j], r[j] = np.float32(-1e-15), np.float32(1e-15)
    rows.append(('tiny_negative', g, r))
    rows.append(('opposite', (-base).astype(np.float32), base))
    rows.append(('subnormal_g', (-1e-40 * (base + 1e-3 * noise)).astype(np.float32), base))
    sub = np.where(even & (np.arange(n) > 0), base * np.float32(1e-41), base).astype(np.float32)   # entry 0 normal
    rows.append(('subnormal_ref', (-3 * sub + noise).astype(np.float32), sub))
    return rows


def real_rows(b, data, seed=3):
    """The engine's stream gradient and memory gradient from one train-mode backward each on the network, and the pair
    with the memory gradient negated (so that both decisions are taken on real gradients)."""
    spec = spec_of(data)
    hw, ncls = NETS[data]
    p, bn = oresnet.seeded_state(spec, seed)
    model = b.nets.Reduced_ResNet18(ncls, in_hw=hw)
    eng = model.engine
    eng.load(list(p.values()), [(bn[k + '.running_mean'], bn[k + '.running_var']) for k in oresnet.bn_names(spec)])
    rs = np.random.RandomState(seed + 1)
    out = []
    for _ in range(2):
        x = torch.from_numpy(rs.rand(10, 3, hw, hw).astype(np.float32)).cuda()
        y = torch.from_numpy(rs.randint(0, 4, 10)).cuda()
        logits, ws = eng.forward_train(x)
        eng.backward(x, b.engine.ce_loss(logits, y)['dlogits'], ws)
        out.append(eng.state.grads.cpu().numpy().copy())
    g, r = out
    return [('real', g, r), ('real_flipped', g, (-r).astype(np.float32))]


def run_guarded(b, g, r):
    """ops.agem_project into a NaN-filled output between guard bands: (out, dots), after checking the guards and that
    every element was written."""
    n = g.size
    buf = torch.empty(n + 2 * GUARD, dtype=torch.float32, device='cuda')
    buf.view(torch.uint8).fill_(GUARD_BYTE)
    buf[GUARD:GUARD + n] = float('nan')
    gd, rd = torch.from_numpy(g).cuda(), torch.from_numpy(r).cuda()
    out, dots = b.ops.agem_project(gd, rd, out=buf[GUARD:GUARD + n], want_dots=True)
    torch.cuda.synchronize()
    host = buf.cpu()
    raw = host.view(torch.uint8).numpy()
    assert np.all(raw[:GUARD * 4] == GUARD_BYTE) and np.all(raw[(GUARD + n) * 4:] == GUARD_BYTE), 'guard band written'
    o = host[GUARD:GUARD + n].numpy()
    assert not np.isnan(o).any(), ('elements left unwritten', np.flatnonzero(np.isnan(o))[:8])
    return o, dots.cpu().numpy(), gd, rd


def check_aliasing(b, gd, rd, want):
    """out aliasing g, out aliasing g_ref (the learner's call) and a repeat give the bits of the separate output."""
    a = gd.clone()
    b.ops.agem_project(a, rd, out=a)
    c = rd.clone()
    b.ops.agem_project(gd, c, out=c)
    again = b.ops.agem_project(gd, rd)
    w = torch.from_numpy(want).cuda()
    for name, t in (('out is g', a), ('out is g_ref', c), ('repeat', again)):
        assert torch.equal(t.view(torch.int32), w.view(torch.int32)), name


def test_edge_lengths_reach_the_launch_edges(b):
    """On this card: some edge length leaves CTAs without an element, one ends its tail one element into a grid
    stride, and every real arena length spans several grid strides."""
    G = grid_of()
    lens = edge_lengths()
    assert any(256 < n < G * 256 and (n + 255) // 256 < G for n in lens), (G, lens)      # busy and idle CTAs
    assert any(n > G * 256 and n % (G * 256) == 1 for n in lens), (G, lens)
    assert any(n % 256 not in (0, 1) and n < G * 256 for n in lens)         # a partial warp-block inside the first stride
    for data in NETS:
        assert arena_len(data) > 4 * G * 256


def test_arena_lengths_are_the_engines(b):
    for data, (hw, ncls) in NETS.items():
        assert (b.memory.input_size_match[data][1], b.memory.n_classes[data]) == (hw, ncls)
        eng = b.nets.Reduced_ResNet18(ncls, in_hw=hw).engine
        assert eng.state.grads.numel() == arena_len(data), data
    assert [arena_len(d) for d in NETS] == [1109240, 1157240, 1104249, 1221190]


@pytest.mark.parametrize('data', list(NETS))
def test_projection_at_arena_lengths(b, data):
    n = arena_len(data)
    worst = 0.0
    decisions = set()
    for name, g, r in real_rows(b, data) + synthetic_rows(n, 11):
        out, dots, gd, rd = run_guarded(b, g, r)
        worst = max(worst, check_projection(g, r, out, dots, (data, name)))
        decisions.add(bool(dots[0] < 0))
        if name in ('real', 'real_flipped', 'far_negative', 'tiny_negative'):
            check_aliasing(b, gd, rd, out)
    assert decisions == {True, False}
    print('agem projection %s n=%d worst %.3g of the bound' % (data, n, worst))


def test_projection_at_edge_lengths(b):
    worst = 0.0
    for n in edge_lengths():
        for name, g, r in synthetic_rows(n, 100 + n % 97):
            out, dots, gd, rd = run_guarded(b, g, r)
            worst = max(worst, check_projection(g, r, out, dots, (n, name)))
            check_aliasing(b, gd, rd, out)
    print('agem projection edge lengths worst %.3g of the bound' % worst)


def test_projection_refusals(b):
    """A workspace one byte short is refused before anything launches and leaves the output alone; n = 0 launches
    nothing."""
    lib, ops = b.native.lib(), b.ops
    g = torch.randn(1000, device='cuda')
    r = -g
    out = torch.full_like(g, float('nan'))
    need = lib.b200ocl_agem_project_workspace_bytes()
    ws = torch.empty(need, dtype=torch.uint8, device='cuda')
    torch.cuda.synchronize()
    before = b.native.launch_count()
    rc = lib.b200ocl_agem_project(ops._ptr(g), ops._ptr(r), ops._ptr(out), g.numel(), None, ops._ptr(ws), need - 1,
                                  ops._stream())
    assert rc == 3 and b'workspace' in lib.b200ocl_last_error().lower()      # B200OCL_EWORKSPACE
    rc = lib.b200ocl_agem_project(ops._ptr(g), ops._ptr(r), ops._ptr(out), 0, None, ops._ptr(ws), need, ops._stream())
    assert rc == 0
    empty = torch.empty(0, device='cuda')
    assert ops.agem_project(empty, empty).numel() == 0
    torch.cuda.synchronize()
    assert b.native.launch_count() == before
    assert torch.isnan(out).all()
    rc = lib.b200ocl_agem_project(ops._ptr(g), ops._ptr(r), ops._ptr(out), g.numel(), None, ops._ptr(ws), need,
                                  ops._stream())
    assert rc == 0 and b.native.launch_count() == before + 2


# ------------------------------------------------------------------------------------------------ the learner
def make_params(data, **kw):
    base = dict(data=data, cuda=True, epoch=1, batch=10, verbose=False, mem_size=10, eps_mem_batch=10, mem_iters=1,
                update='random', retrieve='random', agent='AGEM', num_tasks=5, buffer_tracker=False, optimizer='SGD',
                learning_rate=0.1, weight_decay=0, error_analysis=False,
                trick={'labels_trick': False, 'kd_trick': False, 'separated_softmax': False, 'review_trick': False,
                       'ncm_trick': False, 'kd_trick_star': False})
    trick = kw.pop('trick', {})
    base.update(kw)
    base['trick'] = dict(base['trick'], **trick)
    return SimpleNamespace(**base)


def _round_state(st):
    """The oracle's state rounded to the fp32 values the engine holds, so that each step starts from the same values."""
    for d in (st.params, st.bn):
        for k, v in d.items():
            if v.is_floating_point():
                d[k] = v.float().double()


def _sync(agent, st):
    agent.engine.load([v.float() for v in st.params.values()],
                      [(st.bn[n + '.running_mean'].float(), st.bn[n + '.running_var'].float())
                       for n in oresnet.bn_names(st.spec)])


def _rel(got, want):
    """|got - want| / |want| in the L2 norm.  A pre-activation within fp32 rounding of zero can flip its ReLU against
    fp64 and move a few weights by up to ~1e-3 of the largest (1.5e-3 of max |p| measured at lr 0.1 with
    mem_iters = 2), so the whole step is held in the norm, where such a flip weighs what it moves."""
    want = np.asarray(want, np.float64)
    return float(np.linalg.norm(np.asarray(got, np.float64) - want) / np.linalg.norm(want))


def _bn_flat(agent):
    return np.concatenate([torch.cat([rm, rv]).cpu().numpy() for rm, rv in agent.engine.bn_views()])


def _bn_flat_oracle(st):
    return np.concatenate([torch.cat([st.bn[n + '.running_mean'], st.bn[n + '.running_var']]).numpy()
                           for n in oresnet.bn_names(st.spec)])


def _batch(rs, st, kind, hw, draw, n=10):
    """'fill' / 'pos': fresh images of the memory's classes 0-3.  'neg', 'new', 'swap': the images of the memory draw
    this step makes (`draw`, its slots) under other labels, all class 4 ('neg'), classes 4-7 ('new') or the next of
    the memory's classes 0-3 ('swap'), so that the stream gradient and the memory gradient can point apart."""
    if kind in ('neg', 'new', 'swap'):
        idx = draw[np.arange(n) % draw.size]
        y = st.buffer_label[idx]
        y = {'neg': torch.full_like(y, 4), 'new': y % 4 + 4, 'swap': (y + 1) % 4}[kind]
        return st.buffer_img[idx].clone(), y.clone()
    x = torch.from_numpy(rs.rand(n, 3, hw, hw).astype(np.float32))
    return x, torch.from_numpy(rs.randint(0, 4, n).astype(np.int64))


def run_learner(b, monkeypatch, data, seed, task1=('neg', 'pos', 'neg'), n_task0=2, optimizer='SGD', lr=0.1,
                geometry=None, **kw):
    """Task 0 (n_task0 steps, no projection), then task 1 with a memory; every step of the engine against
    oracle.agem.step in float64.  Returns per task-1 memory iteration (decision, cosine, bound ratio)."""
    hw, ncls = NETS[data]
    spec = spec_of(data)
    params = make_params(data, optimizer=optimizer, learning_rate=lr, **kw)
    p0, bn0 = oresnet.seeded_state(spec, seed, dtype=torch.float64)
    agent = b.registry.agents['AGEM'](b.nets.setup_architecture(params), None, params)
    st = ors.ReplayState(spec, p0, bn0, params.mem_size, (3, hw, hw), ncls, lr=lr)
    _sync(agent, st)
    agent.model.train()
    calls = []
    orig = b.ops.agem_project

    def recorded(g, g_ref, out=None, want_dots=False):
        gh, rh = g.cpu().numpy().copy(), g_ref.cpu().numpy().copy()
        res, dots = orig(g, g_ref, out=out, want_dots=True)
        calls.append((gh, rh, res.cpu().numpy().copy(), dots.cpu().numpy()))
        return (res, dots) if want_dots else res
    monkeypatch.setattr(b.ops, 'agem_project', recorded)
    opt = oagem.AdamState(lr) if optimizer == 'Adam' else None
    shadow = oagem.AdamState(lr) if optimizer == 'Adam' else None     # fed the engine's gradients
    trick = params.trick
    mode = 'labels_trick' if trick['labels_trick'] else 'ce'
    teacher = None
    rs = np.random.RandomState(seed + 1)
    out, step_no = [], 0
    for task, kinds in ((0, ('fill',) * n_task0), (1, task1)):
        agent.before_train(None, np.arange(8) if data == 'openloris' else np.arange(4 * task, 4 * task + 4))
        for kind in kinds:
            np.random.seed(700 + step_no)
            x, y = _batch(rs, st, kind, hw, ors._random_indices(st, params.eps_mem_batch) if task else None)
            if geometry is not None and task == 1:
                geometry(min(params.eps_mem_batch, st.current_index), x.shape[0])
            where = (data, task, step_no, kind)
            n_calls = len(calls)
            p_before = oagem.flat(st.params)
            np.random.seed(700 + step_no); torch.manual_seed(700 + step_no)
            agent.replay_step(x.cuda(), y.cuda(), y.numpy())
            torch.cuda.synchronize()
            np.random.seed(700 + step_no); torch.manual_seed(700 + step_no)
            logs = oagem.step(st, x, y, task, eps_mem_batch=params.eps_mem_batch, mem_iters=params.mem_iters,
                              mode=mode, teacher=teacher, kd_trick=trick['kd_trick'], adam=opt)
            mine = calls[n_calls:]
            assert len(mine) == sum(lg['project'] is not None for lg in logs), where
            for (gh, rh, res, dots), lg in zip(mine, [lg for lg in logs if lg['project'] is not None]):
                cos = lg['prod'] / (np.linalg.norm(lg['g']) * np.linalg.norm(lg['g_ref']))
                assert abs(cos) >= COS_MARGIN, (where, 'cosine too close to 0 for the test to decide', cos)
                assert bool(dots[0] < 0) == lg['project'], (where, 'decision', dots[0], lg['prod'])
                ratio = check_projection(gh, rh, res, dots, where)
                out.append((lg['project'], cos, ratio, lg['ret_idx'].size))
            p_engine = agent.engine.state.params.cpu().numpy()
            ep = _rel(p_engine, oagem.flat(st.params))
            if optimizer == 'Adam':
                # Adam's early steps are lr * g / (|g| + eps): an element whose gradient lies within a ReLU flip's reach
                # of 0 may flip its whole step against fp64, so the update is checked against the fp64 Adam step of the
                # engine's own gradient arena (the gradient itself is checked above and by the projection check)
                p_dict = oagem._unflat(st, p_before)
                shadow.step(p_dict, oagem._unflat(st, agent.engine.state.grads.cpu().numpy().astype(np.float64)))
                eu = _rel(p_engine - p_before, oagem.flat(p_dict) - p_before)
                assert eu < ADAM_UPDATE_TOL, (where, 'Adam update', eu)
            else:
                eu = _rel(p_engine - p_before, oagem.flat(st.params) - p_before)
                assert eu < UPDATE_TOL, (where, 'update', eu)
            eb = _rel(_bn_flat(agent), _bn_flat_oracle(st))
            assert ep < STEP_TOL and eb < STEP_TOL, (where, 'step', ep, eb)
            buf = agent.buffer
            assert buf.current_index == st.current_index and buf.n_seen_so_far == st.n_seen_so_far, where
            np.testing.assert_array_equal(buf.buffer_label.cpu().numpy(), st.buffer_label.numpy())
            assert torch.equal(buf.buffer_img.cpu(), st.buffer_img), where
            print('agem step %s: params %.3g update %.3g bn %.3g' % (where, ep, eu, eb))
            _round_state(st)
            _sync(agent, st)
            step_no += 1
        if task == 0:
            agent.after_train()
            teacher = (copy.deepcopy(st.params), copy.deepcopy(st.bn)) if trick['kd_trick'] else None
    return out


# per network: (seed, task-1 batches, task-0 steps, eps_mem_batch), chosen so that both decisions occur with every
# |cosine| >= COS_MARGIN (the measured cosines are printed)
SCHEDULES = {'cifar100': (41, ('neg', 'pos', 'neg'), 2, 10),
             'mini_imagenet': (46, ('swap', 'pos', 'pos'), 1, 4),
             'openloris': (47, ('swap', 'pos', 'pos'), 1, 4),
             'core50': (45, ('swap', 'pos', 'pos'), 1, 4)}


@pytest.mark.parametrize('data', list(NETS))
def test_learner_matches_fp64(b, monkeypatch, data):
    """At CORe50 the memory draw of 4 rows also takes other convolution templates in its forward than the stream
    batch of 10."""
    seed, task1, n_task0, eps = SCHEDULES[data]
    hw, ncls = NETS[data]
    desc, info, _ = b.engine.describe(hw, ncls)
    other = []

    def geometry(n_mem, n_stream):
        other.append([i for i in range(info.n_bn) if b.engine.conv_geom(desc, n_mem, i, 'train').template !=
                      b.engine.conv_geom(desc, n_stream, i, 'train').template])
    res = run_learner(b, monkeypatch, data, seed, task1=task1, n_task0=n_task0, eps_mem_batch=eps, geometry=geometry)
    print('agem learner %s: %s; layers whose templates differ between the memory and the stream batch %s'
          % (data, [(p, round(c, 4), round(r, 3)) for p, c, r, _ in res], other))
    assert {p for p, _, _, _ in res} == {True, False}, res
    assert all(n == min(eps, 10) for _, _, _, n in res)
    if data == 'core50':
        assert other and all(other), other


@pytest.mark.parametrize('variant', ['mem_iters2', 'small_memory', 'adam', 'kd_labels'])
def test_learner_variants(b, monkeypatch, variant):
    # mem_iters = 2 at lr 0.01: the second iteration runs from the first one's weights without a resync, and at
    # lr 0.1 a ReLU flip of the first iteration moved its update by 5 % (7.6e-4 of |p|)
    kw = {'mem_iters2': dict(mem_iters=2, lr=0.01, task1=('neg', 'pos')),
          'small_memory': dict(mem_size=4, task1=('neg', 'pos')),
          'adam': dict(optimizer='Adam', lr=2e-5, task1=('new', 'pos')),
          'kd_labels': dict(trick={'kd_trick': True, 'labels_trick': True}, task1=('swap', 'pos'))}[variant]
    res = run_learner(b, monkeypatch, 'cifar100', 51, **kw)
    print('agem learner %s: %s' % (variant, [(p, round(c, 4), round(r, 3)) for p, c, r, _ in res]))
    assert {p for p, _, _, _ in res} == {True, False}, res
    if variant == 'small_memory':
        assert all(n == 4 for _, _, _, n in res)


# ------------------------------------------------------------------------------------------------ reference runs
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'agem_maps.npz')


@pytest.mark.parametrize('data', ['mini_imagenet', 'core50'])
def test_dropin_matches_reference_run(b, data):
    """The reference's own A-GEM runs at 84x84 and 128x128 (tests/golden/agem_maps.npz) with test_gpu_dropin.py's
    comparison and bars: index, seen, labels and image digest of the memory exactly, the sampled weight update and the
    BN statistics within the larger of the fp32 bar and 10x the reference's one-ulp spread, the accuracies."""
    import test_gpu_dropin as dropin
    g = np.load(GOLDEN)
    tag = data + '_'
    _, n_calls, wseed, seed, dseed = json.loads(str(g[tag + 'case']))
    params = SimpleNamespace(**json.loads(str(g[tag + 'params'])))
    params.cuda = True
    hw, ncls = NETS[data]
    spec = spec_of(data)
    b.memory.set_mode(True, 'cpu')                  # the reference ran on the CPU: its draws came from CPU generators
    try:
        agent = b.registry.agents['AGEM'](b.nets.setup_architecture(params), None, params)
        p, bn = oresnet.seeded_state(spec, wseed)
        agent.engine.load(list(p.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
        w0 = torch.cat([t.reshape(-1) for t in p.values()]).numpy()
        pick = dropin.dropin_sample(w0.size)
        w0 = w0[pick].astype(np.float64)
        np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
        x, y, calls, tests = oagem.dropin_inputs(np.random.RandomState(dseed), params.mem_size, hw, params.batch, n_calls)
        buf = agent.buffer
        buf.update(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda())
        for c, (xt, yt) in enumerate(calls):
            where = (data, 'call', c)
            agent.train_learner(xt, yt)
            torch.cuda.synchronize()
            assert buf.current_index == int(g[tag + 'index%d' % c]) and buf.n_seen_so_far == int(g[tag + 'seen%d' % c]), where
            np.testing.assert_array_equal(buf.buffer_label.cpu().numpy(), g[tag + 'label%d' % c])
            assert hashlib.sha1(buf.buffer_img.cpu().numpy().tobytes()).hexdigest() == str(g[tag + 'img%d' % c]), where
            w = agent.engine.state.params.cpu().numpy()[pick]
            err = dropin._rel(w - w0, g[tag + 'w%d' % c].astype(np.float64) - w0)
            print('agem dropin %s call %d weight update rel %.3g (spread %.3g)' % (data, c, err, g[tag + 'spread_w'][c]))
            assert err <= max(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_w'][c]), (where, 'weight update', err)
            err = dropin._rel(agent.engine.state.bn_stats.cpu().numpy(), g[tag + 'bn%d' % c].astype(np.float64))
            assert err <= max(dropin.BN_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_bn'][c]), (where, 'BN statistics', err)
        loaders = [[(torch.from_numpy(tx).permute(0, 3, 1, 2).float().div(255), torch.from_numpy(ty))] for tx, ty in tests]
        acc = np.asarray(agent.evaluate(loaders))
        assert np.abs(acc - g[tag + 'acc']).max() <= 3.1 / 96, (data, acc, g[tag + 'acc'])
    finally:
        b.memory.set_mode(False)
