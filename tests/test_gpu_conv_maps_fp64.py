"""The halo-strip convolution (csrc/conv_tcp.cu), its eval epilogues and the wgmma weight gradient (csrc/wgrad_tc.cu)
against fp64 at every map the four datasets' networks send them, and the eval epilogues of conv_tc and the CUDA-core
kernels at the maps too wide for the strip.

TABLE, the (channels, map) pairs of the strip kernels, is derived from oracle.resnet.block_plan for CIFAR-100 (32x32),
Mini-ImageNet (84x84), OpenLORIS (50x50) and CORe50 (128x128) inputs: every 3x3 stride-1 layer whose map is at most
STRIP_MAX_W wide.  The CPU test proves that it is exactly what the planner routes to conv_tcp (eval forward, data
gradient) and to wgrad_tc, for every network and SCR head, at 114, 132 and 148 SMs and every batch up to 512; so a new
dataset or width cannot join the strip kernels untested.  The GPU coverage tests prove that the batches below reach
every launch those networks make on the card in use: each (template, patch stages, weight ring depth), CTAs walking one,
two and three or more 128-position tiles, a last tile that ends inside the last image and one that runs into the zero
tail past it, and weight-gradient grids with one chain per CTA, chains rounded up to an even count, and CTAs capped
by the SM count.

Every output is NaN-filled (or holds the tensor accumulated into) and lies between two 1 MB guard bands of a fixed byte
pattern: every element must be written and the guards must come back untouched.  Every launch is repeated and must
give the same bits.  The eval forms are the network's three: folded BN alone (a shortcut), BN + ReLU (a block's conv1)
and BN + a residual in its own buffer + ReLU (a block's conv2).  Their BN parameters are like a trained network's:
output channels whose scales span decades (their weights scaled by 10^[-2, 0.5]) with running variances to match, so
that some fall to ~1e-5 and eps matters; running means on the scale of each channel's spread, three channels at 10x;
gamma of both signs with two channels near zero; residuals of both signs, so that ReLU clips on both sides.

Bars (max |got - ref| / max |ref| per tensor): 5e-6 for the convolutions, 5e-6 max and 2e-6 rms for the weight
gradient, as in test_gpu_conv_strip.py and test_gpu_wgrad_tc.py.  Largest values measured over every case of this file
on an H100 80GB HBM3 (SXM, 132 SMs, 700 W power limit):
  conv_tcp  forward raw 6.5e-7 (160 @ 4x4, N = 20), accumulate 6.1e-7 (160 @ 4x4, N = 20); data gradient raw 5.8e-7
            (80 @ 8x8, N = 220), accumulate 6.0e-7 (80 @ 8x8, N = 220); eval BN 4.9e-7 (40 @ 25x25, N = 210),
            BN + ReLU 6.6e-7 (160 @ 7x7, N = 10), BN + residual + ReLU 6.0e-7 (80 @ 32x32, N = 260)
  wide maps eval BN 4.8e-7 (20 @ 50x50, N = 24, patch<20, 2>), BN + ReLU 4.0e-7 and BN + residual + ReLU 3.7e-7
            (20 @ 128x128, N = 7, patch<20, 4>)
  wgrad_tc  max 2.4e-6 (40 @ 16x16, N = 1), rms 1.8e-6 (20 @ 32x32, N = 220): the weight gradient's 3xTF32 chains of
            256 positions, as test_gpu_wgrad_tc.py measures at CIFAR's maps
The whole file, CPU tests included, ran in 26 s there (pytest's count; 31 s with start-up).

tests/golden/conv_maps.npz (make_golden_conv_maps.py) holds the bits of conv_tcp's eval and data-gradient launches and
of wgrad_tc at the seven pairs CIFAR's network does not have, at N = 20 and 110; the kernels must reproduce them."""
import hashlib
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import bench
from oracle import resnet as oresnet

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import make_golden_conv_maps as mg  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'conv_maps.npz')

DATASETS = {'cifar100': 32, 'mini_imagenet': 84, 'openloris': 50, 'core50': 128}   # input_size_match
SMS = (114, 132, 148)
MAX_N = 512
# conv_tcp and wgrad_tc stage a strip of 128 + 2 * (W + 2) + 2 rows, 16 per loader pass, 13 passes at most
STRIP_MAX_W = 37
PATHS = {'cuda_core': 1, 'tc': 2, 'tcp': 3}
GUARD = 1 << 20
PATTERN = 0xA5
TOL, WG_MAX, WG_RMS = 5e-6, 5e-6, 2e-6


def conv_layers(hw):
    """(C, map) of every 3x3 stride-1 convolution of the reduced ResNet-18 (nf = 20) on hw x hw inputs, layer order.
    Every stride-1 block keeps its width, so C is both the input and the output channels."""
    out = []
    for _, cin, cout, stride, _ in oresnet.block_plan(oresnet.Spec(hw)):
        ho = (hw - 1) // stride + 1
        if stride == 1:
            assert cin == cout
            out.append((cout, ho))          # conv1
        out.append((cout, ho))              # conv2
        hw = ho
    return out


STRIP = {d: list(dict.fromkeys(p for p in conv_layers(hw) if p[1] <= STRIP_MAX_W)) for d, hw in DATASETS.items()}
WIDE_BY = {d: list(dict.fromkeys(p for p in conv_layers(hw) if p[1] > STRIP_MAX_W)) for d, hw in DATASETS.items()}
TABLE = [p for d in DATASETS for p in STRIP[d]]
WIDE = [p for d in DATASETS for p in WIDE_BY[d]]
assert len(set(TABLE)) == len(TABLE) and len(set(WIDE)) == len(WIDE)


def aser_eval_batches():
    """Batch sizes of ASER's eval-mode feature passes in the benchmark (as test_gpu_forward_fp64.aser_eval_batches)."""
    p, C = bench.params_for('aser'), bench.NUM_CLASSES
    return (p.batch + 2 * int(p.n_smp_cls) * C, int(p.n_smp_cls) * C + int(p.n_smp_cls * C) + p.batch)


# one and two images, ER's 10 and 20, SCR's 110 and 220, ASER's eval batches; then per pair the batches the coverage
# tests need on 114-, 132- and 148-SM cards: a last tile inside the last image at (80, 8), (40, 16) and (160, 11),
# two tiles per CTA at (160, 11), (40, 25) and (80, 13), three or more at (160, 4)
AGENT_BATCHES = (1, 2, 10, 20, 110, 220) + aser_eval_batches()
EXTRA = {(40, 16): (51,), (80, 8): (8,), (160, 4): (399,), (160, 11): (40,), (40, 25): (29,), (80, 13): (49,)}


def batches(C, H):
    return sorted(set(AGENT_BATCHES + EXTRA.get((C, H), ())))


CASES = [(C, H, N) for C, H in TABLE for N in batches(C, H)]


def case_id(c):
    return 'C%d-%dx%d-N%d' % (c[0], c[1], c[1], c[2])


def strip_tiles(N, H):
    """conv_tcp's 128-position tiles over N images of H x H (strip pitch H + 1, one zero row per image) and how far the
    last tile runs past the last image (<= 0: it ends inside that image)."""
    pitch = (H + 1) * (H + 1)
    last = (N - 1) * pitch + (H - 1) * (H + 1) + (H - 1)
    tiles = last // 128 + 1
    return tiles, tiles * 128 - N * pitch


def wgrad_classes(g):
    """The weight-gradient grid's classes: one chain per CTA, a chain count rounded up to even (one fewer would still
    have covered every chain with the CTAs the SM count allows), CTAs capped by the SM count."""
    out = set()
    if g.chains_per_cta == 1:
        out.add('one')
    if g.chains_per_cta > 1 and (g.chains_per_cta - 1) * min(g.sm_share, g.chains) >= g.chains:
        out.add('even')
    if g.ctas_x < g.chains:
        out.add('cut')
    return out


# ----------------------------------------------------------------------------------------------------------- CPU
class _Built(object):
    """Stands in for nets.EngineModel: records what setup_architecture asks for without allocating on a GPU."""
    def __init__(self, in_hw, num_classes, head=None, feat_dim=128, device='cuda'):
        self.in_hw, self.num_classes, self.head, self.feat_dim = in_hw, num_classes, head, feat_dim


def networks(monkeypatch):
    """[(dataset, head, desc, conv layers)]: each dataset's classifier network, and SupConResNet with each head SCR
    allows there."""
    from b200ocl import engine, memory, nets
    monkeypatch.setattr(nets, 'EngineModel', _Built)
    out = []
    for data, hw in DATASETS.items():
        assert memory.input_size_match[data][1:] == [hw, hw]
        m = nets.setup_architecture(SimpleNamespace(data=data, agent='ER', head='mlp'))
        desc, info, _ = engine.describe(m.in_hw, m.num_classes)
        out.append((data, None, desc, info.n_bn))
        for head in ('mlp', 'linear', 'None'):
            try:
                m = nets.setup_architecture(SimpleNamespace(data=data, agent='SCR', head=head))
            except (ValueError, NotImplementedError):
                continue
            desc, info, _ = engine.describe(m.in_hw, m.num_classes, head=m.head, feat_dim=m.feat_dim)
            out.append((data, head, desc, info.n_bn))
    return out


def test_conv_maps_table_is_the_planners_strip_routing(monkeypatch):
    """For every network, SCR head, SM count and batch up to 512: the layers whose eval forward and data gradient the
    planner sends to conv_tcp, and those whose weight gradient it sends to wgrad_tc, are exactly the table's."""
    from b200ocl import engine
    nets = networks(monkeypatch)
    assert {d for d, _, _, _ in nets} == set(DATASETS)
    assert {(d, h) for d, h, _, _ in nets if h} >= {('cifar100', 'mlp'), ('openloris', 'None')}
    assert TABLE == [(20, 32), (40, 16), (80, 8), (160, 4), (80, 21), (160, 11), (40, 25), (80, 13), (160, 7),
                     (80, 32), (160, 16)]
    for data, head, desc, n_conv in nets:
        L = [engine.train_ws_layout(desc, 1, i) for i in range(n_conv)]
        want = {i for i, l in enumerate(L) if i > 0 and l.ks == 3 and l.stride == 1 and (l.cout, l.hout) in STRIP[data]}
        assert {(L[i].cout, L[i].hout) for i in want} == set(STRIP[data]), (data, head)
        for N in range(1, MAX_N + 1):
            wg = {i for i in range(len(L)) if engine.train_ws_layout(desc, N, i).wgrad_kernel == 1}
            assert wg == want, (data, head, N, sorted(wg ^ want))
            for sms in SMS:
                for pass_ in ('eval', 'dgrad'):
                    got = {i for i in range(1, len(L)) if engine.conv_geom(desc, N, i, pass_, sms).name == 'tcp'}
                    assert got == want, (data, head, N, sms, pass_, sorted(got ^ want))


def test_conv_maps_wide_layers_and_golden_pairs():
    """The wide maps are the ones the eval tests below run on the other kernels, and the bit record covers every pair of
    the table that CIFAR's own record does not."""
    assert WIDE == [(20, 84), (40, 42), (20, 50), (20, 128), (40, 64)]
    assert sorted(mg.PAIRS) == sorted(set(TABLE) - set(STRIP['cifar100']))


def test_conv_maps_golden_records_every_case():
    rec = np.load(GOLDEN)
    assert len(mg.CASES) == 56 and len(rec.files) == len(mg.CASES) + len(mg.KEEP)
    for c in mg.CASES:
        sha = str(rec[mg.key(c) + '_sha256'])
        assert len(sha) == 64
        if c in mg.KEEP:
            y = rec[mg.key(c) + '_out']
            kind, N, C, H = c
            assert y.shape == ((C, C, 3, 3) if kind == 'wgrad' else (N, H, H, C)) and y.dtype == np.float32
            assert hashlib.sha256(y.astype('<f4').tobytes()).hexdigest() == sha


# ----------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope='module')
def engine():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import engine
    return engine


def network_layer(engine, C, H, wide=False):
    """(desc, conv layer index) of a network layer with this (C, map)."""
    for data, hw in DATASETS.items():
        if (C, H) in (WIDE_BY if wide else STRIP)[data]:
            desc, info, _ = engine.describe(hw, 100)
            for i in range(1, info.n_bn):
                L = engine.train_ws_layout(desc, 1, i)
                if (L.ks, L.stride, L.cout, L.hout) == (3, 1, C, H):
                    return desc, i
    raise AssertionError((C, H))


@pytest.mark.gpu
def test_conv_maps_cases_reach_every_strip_launch(engine):
    """On this card the cases reach every (pair, pass, template, patch stages, weight ring depth) that the networks'
    eval and data-gradient passes give conv_tcp at N <= 512, each with CTAs that walk 1, 2 and >= 3 tiles and with a
    last tile inside the last image and one past it; and every case's launch is the network's launch at that batch.
    The thresholds move with the SM count, so they are read through the hooks."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    every = set()
    for hw in DATASETS.values():
        desc, info, _ = engine.describe(hw, 100)
        for i in range(1, info.n_bn):
            L = engine.train_ws_layout(desc, 1, i)
            for pass_ in ('eval', 'dgrad'):
                for N in range(1, MAX_N + 1):
                    g = engine.conv_geom(desc, N, i, pass_)
                    assert g.sms == sms
                    if g.name == 'tcp':
                        every.add(((L.cout, L.hout), pass_, g.template, g.tp_ps, g.tp_bs))
    reached, rounds, tails = set(), {}, {}
    for C, H, N in CASES:
        desc, i = network_layer(engine, C, H)
        for pass_, dgrad, mode in (('eval', 0, 3), ('dgrad', 1, 0)):
            g = engine.conv_selftest_geom(N, H, H, C, C, 3, 1, dgrad, PATHS['tcp'], mode)
            net = engine.conv_geom(desc, N, i, pass_)
            assert (g.template, g.grid_x, g.grid_y, g.tp_ps, g.tp_bs) == \
                (net.template, net.grid_x, net.grid_y, net.tp_ps, net.tp_bs), (C, H, N, pass_)
            reached.add(((C, H), pass_, g.template, g.tp_ps, g.tp_bs))
            tiles, past = strip_tiles(N, H)
            rounds.setdefault((C, H, pass_), set()).add(min(3, -(-tiles // g.grid_x)))
            tails.setdefault((C, H, pass_), set()).add(past > 0)
    assert reached == every, sorted(every ^ reached)
    for k in rounds:
        assert rounds[k] == {1, 2, 3}, (k, rounds[k])
        assert tails[k] == {False, True}, (k, tails[k])


@pytest.mark.gpu
def test_conv_maps_cases_reach_every_weight_gradient_grid(engine):
    """On this card each pair's batches give wgrad_tc one chain per CTA, a chain count rounded up to even, and CTAs
    capped by the SM count; and wgrad_tc is the kernel the network runs there."""
    for C, H in TABLE:
        desc, i = network_layer(engine, C, H)
        got = set()
        for N in batches(C, H):
            g = engine.wgrad_tc_selftest_geom(N, H, H, C, C)
            assert g.eligible and engine.train_ws_layout(desc, N, i).wgrad_kernel == 1
            got |= wgrad_classes(g)
        assert got == {'one', 'even', 'cut'}, (C, H, got)


class Guarded(object):
    """An fp32 tensor of `shape` in the middle of a device buffer, between two GUARD-byte bands of PATTERN; it starts
    NaN-filled, or as a copy of `init`."""

    def __init__(self, shape, init=None):
        n = int(np.prod(shape))
        self.buf = torch.full((2 * GUARD + 4 * n,), PATTERN, dtype=torch.uint8, device='cuda')
        self.t = self.buf[GUARD:GUARD + 4 * n].view(torch.float32).view(shape)
        if init is None:
            self.t.fill_(float('nan'))
        else:
            self.t.copy_(init)

    def result(self, what):
        torch.cuda.synchronize()
        assert bool((self.buf[:GUARD] == PATTERN).all()), (what, 'guard band before the output overwritten')
        assert bool((self.buf[-GUARD:] == PATTERN).all()), (what, 'guard band after the output overwritten')
        nan = torch.isnan(self.t)
        assert not bool(nan.any()), (what, 'elements left unwritten', int(nan.sum()), nan.nonzero()[:4].tolist())
        return self.t


def _workspace(lib, N, C, H):
    nbytes = lib.b200ocl_conv_selftest_workspace_bytes(N, C, C, H, H, 3, 1)
    ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
    ws.view(torch.float32).fill_(float('nan'))          # nothing may be read before it is written
    return ws, nbytes


def launch_conv(x, w, dgrad, path, init=None):
    """Forward (dgrad = 0) or data gradient of a 3x3 stride-1 C -> C convolution, raw or accumulating into `init`."""
    from b200ocl import _native
    from b200ocl.ops import _stream
    lib = _native.lib()
    N, H, W, C = x.shape
    out = Guarded((N, H, W, C), init)
    ws, nbytes = _workspace(lib, N, C, H)
    rc = lib.b200ocl_conv_selftest(x.data_ptr(), w.data_ptr(), out.t.data_ptr(), N, H, W, C, C, 3, 1, dgrad, path,
                                   0 if init is None else 1, None, ws.data_ptr(), nbytes, _stream())
    _native.check(rc, 'b200ocl_conv_selftest')
    return out.result(('dgrad' if dgrad else 'forward', 'raw' if init is None else 'accumulate'))


def launch_eval(x, w, bn, residual, relu, path):
    from b200ocl import _native
    from b200ocl.ops import _stream
    lib = _native.lib()
    N, H, W, C = x.shape
    out = Guarded((N, H, W, C))
    ws, nbytes = _workspace(lib, N, C, H)
    rc = lib.b200ocl_conv_selftest_eval(x.data_ptr(), w.data_ptr(), bn.data_ptr(),
                                        None if residual is None else residual.data_ptr(), int(relu), out.t.data_ptr(),
                                        N, H, W, C, path, ws.data_ptr(), nbytes, _stream())
    _native.check(rc, 'b200ocl_conv_selftest_eval')
    return out.result(('eval', residual is not None, relu))


def launch_wgrad(x, dz):
    from b200ocl import _native
    from b200ocl.ops import _stream
    lib = _native.lib()
    N, H, W, C = x.shape
    nbytes = lib.b200ocl_wgrad_tc_selftest_workspace_bytes(N, H, W, C, C)
    ws = torch.full((nbytes // 4,), float('nan'), device='cuda')
    out = Guarded((C, C, 3, 3))
    rc = lib.b200ocl_wgrad_tc_selftest(x.data_ptr(), dz.data_ptr(), out.t.data_ptr(), N, H, W, C, C, ws.data_ptr(),
                                       nbytes, _stream())
    _native.check(rc, 'b200ocl_wgrad_tc_selftest')
    return out.result('wgrad')


def twice(fn, *args):
    """fn(*args), launched twice on fresh buffers: both launches must give the same bits."""
    a = fn(*args)
    b = fn(*args)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), ('repeat launch differs', fn.__name__)
    return a


def nchw(t):
    return t.permute(0, 3, 1, 2).double()


def reference(x, w, dgrad):
    f = F.conv_transpose2d if dgrad else F.conv2d
    return f(nchw(x), w.double(), padding=1).permute(0, 2, 3, 1)


def rel(got, ref, H):
    """max |got - ref| / max |ref|, and where the worst element lies: (image, row, column, channel, strip tile)."""
    d = (got.double() - ref).abs()
    k = int(d.argmax())
    n, y, x, c = np.unravel_index(k, tuple(d.shape))
    tile = ((n * (H + 1) + y) * (H + 1) + x) // 128
    return float(d.max() / ref.abs().max()), (int(n), int(y), int(x), int(c), int(tile))


def eval_inputs(x, w, g):
    """Scaled weights, BN block [mean | var | gamma | beta] and a residual like a trained network's (module docstring),
    and the fp64 convolution of x with the scaled weights."""
    C = w.shape[0]
    ch = 10 ** (2.5 * torch.rand(C, device='cuda', generator=g) - 2)
    ch[5] = 1e-2                                        # one channel of the smallest scale, its variance below 1e-4
    ws = (w * ch[:, None, None, None]).contiguous()
    conv = reference(x, ws, 0)
    spread = conv.reshape(-1, C).std(0)
    mean = spread * torch.randn(C, device='cuda', generator=g, dtype=torch.float64)
    mean[:3] *= 10
    var = spread ** 2 * 10 ** (torch.rand(C, device='cuda', generator=g, dtype=torch.float64) - 0.5)
    var[5] = 0.5 * spread[5] ** 2
    gamma = torch.randn(C, device='cuda', generator=g)
    gamma[3], gamma[4] = 1e-3, -2e-3
    beta = 0.5 * torch.randn(C, device='cuda', generator=g)
    bn = torch.cat([mean.float(), var.float(), gamma, beta]).contiguous()
    residual = torch.randn(x.shape, device='cuda', generator=g)
    return ws, bn, residual, conv


def eval_forms(x, ws, bn, residual, conv, path, H, errs):
    """The network's three eval forms through `path` against fp64 from the same fp32 parameters."""
    C = ws.shape[0]
    mean, var, gamma, beta = (t.double() for t in bn.reshape(4, C))
    y = (conv - mean) * (gamma / torch.sqrt(var + oresnet.BN_EPS)) + beta
    assert float(var.min()) < 1e-4 and float(gamma.min()) < 0
    errs['eval_bn'] = rel(twice(launch_eval, x, ws, bn, None, 0, path), y, H)
    errs['eval_bn_relu'] = rel(twice(launch_eval, x, ws, bn, None, 1, path), torch.relu(y), H)
    ref = torch.relu(y + residual.double())
    assert 0.2 < float((ref == 0).double().mean()) < 0.8       # ReLU clips a good share, both signs reach it
    errs['eval_bn_res_relu'] = rel(twice(launch_eval, x, ws, bn, residual, 1, path), ref, H)


def report(errs, where, tol=TOL):
    for k, (e, at) in sorted(errs.items()):
        print('MAXERR %s %s %.2e at %s' % (k, where, e, at))
    bad = sorted((e, k, at) for k, (e, at) in errs.items() if not e < tol)
    assert not bad, (where, bad)


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=case_id)
def test_conv_tcp_matches_fp64(engine, case):
    """Forward raw and accumulate, data gradient raw and accumulate, the three eval forms: forced onto conv_tcp."""
    C, H, N = case
    g = torch.Generator(device='cuda').manual_seed(1009 * N + 31 * C + H)
    w = torch.randn(C, C, 3, 3, device='cuda', generator=g) / np.sqrt(9 * C)
    x = torch.relu(torch.randn(N, H, H, C, device='cuda', generator=g))
    dz = torch.randn(N, H, H, C, device='cuda', generator=g)
    base = torch.randn(N, H, H, C, device='cuda', generator=g)
    errs, tcp = {}, PATHS['tcp']
    conv = reference(x, w, 0)
    scale = float(conv.abs().max())
    errs['fwd'] = rel(twice(launch_conv, x, w, 0, tcp), conv, H)
    e, at = rel(twice(launch_conv, x, w, 0, tcp, base), conv + base.double(), H)
    errs['fwd_acc'] = (e * float((conv + base.double()).abs().max()) / scale, at)
    dx = reference(dz, w, 1)
    scale = float(dx.abs().max())
    errs['dgrad'] = rel(twice(launch_conv, dz, w, 1, tcp), dx, H)
    e, at = rel(twice(launch_conv, dz, w, 1, tcp, base), dx + base.double(), H)
    errs['dgrad_acc'] = (e * float((dx + base.double()).abs().max()) / scale, at)
    del conv, dx
    eval_forms(x, *eval_inputs(x, w, g), tcp, H, errs)
    report(errs, case_id(case))


@pytest.mark.gpu
@pytest.mark.parametrize('C,H', WIDE)
def test_wide_map_eval_forms_match_fp64(engine, C, H):
    """The three eval forms at a map wider than the strip, at the smallest batch of each kernel instantiation the
    network's eval pass takes there (N <= 512) on this card, forced onto that kernel family."""
    desc, i = network_layer(engine, C, H, wide=True)
    first = {}
    for N in range(1, MAX_N + 1):
        first.setdefault(engine.conv_geom(desc, N, i, 'eval').template, N)
    assert 'tcp' not in {t[0] for t in first} and ('tc', 32 if C == 20 else 48) in first, first
    for template, N in sorted(first.items(), key=lambda kv: kv[1]):
        path = PATHS['tc'] if template[0] == 'tc' else PATHS['cuda_core']
        assert engine.conv_selftest_geom(N, H, H, C, C, 3, 1, 0, path, 3).template == template, (template, N)
        g = torch.Generator(device='cuda').manual_seed(1013 * N + 37 * C + H)
        w = torch.randn(C, C, 3, 3, device='cuda', generator=g) / np.sqrt(9 * C)
        x = torch.relu(torch.randn(N, H, H, C, device='cuda', generator=g))
        errs = {}
        eval_forms(x, *eval_inputs(x, w, g), path, H, errs)
        report(errs, 'C%d-%dx%d-N%d-%s' % (C, H, H, N, '-'.join(map(str, template))))


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=case_id)
def test_wgrad_tc_matches_fp64(engine, case):
    C, H, N = case
    g = torch.Generator(device='cuda').manual_seed(1019 * N + 41 * C + H)
    x = torch.relu(torch.randn(N, H, H, C, device='cuda', generator=g))
    dz = torch.randn(N, H, H, C, device='cuda', generator=g) / (N * H * H) ** 0.5
    ref = torch.nn.grad.conv2d_weight(nchw(x), (C, C, 3, 3), nchw(dz), padding=1)
    got = twice(launch_wgrad, x, dz).double()
    err = float((got - ref).abs().max() / ref.abs().max())
    rms = float(((got - ref) ** 2).mean().sqrt() / (ref ** 2).mean().sqrt())
    k = np.unravel_index(int((got - ref).abs().argmax()), tuple(ref.shape))
    print('MAXERR wgrad %s %.2e rms %.2e at %s' % (case_id(case), err, rms, tuple(int(v) for v in k)))
    assert err < WG_MAX and rms < WG_RMS, (case_id(case), err, rms, k)


@pytest.mark.gpu
@pytest.mark.parametrize('case', mg.CASES, ids=mg.key)
def test_conv_maps_bit_identical_to_recorded(engine, case):
    rec = np.load(GOLDEN)
    y = mg.run(case)
    k = mg.key(case)
    if k + '_out' in rec:
        want = rec[k + '_out']
        diff = np.flatnonzero(y.view(np.uint32) != want.view(np.uint32))
        assert diff.size == 0, (k, diff.size, diff[:8])
    assert mg.sha(y) == str(rec[k + '_sha256']), k
