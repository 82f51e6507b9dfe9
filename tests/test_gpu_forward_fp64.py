"""GPU: the network forward (b200ocl_net_forward_train and its eval-statistics and deferred forms, and
b200ocl_net_features_eval) against fp64, layer by layer from the engine's own tensors and end to end from the images,
at batch sizes that reach every convolution kernel instantiation the networks can take.

The train workspace is filled with NaN first, so every tensor checked must have been written.  Each layer is rebuilt in
float64 from what the engine left in the workspace (train_ws_layout offsets): its convolution from the engine's input to
that layer, its batch statistics from the engine's own raw output, its BN-apply from the engine's saved statistics.  So an
error cannot hide behind an error in an earlier layer, and the tolerances can be tight.  The end-to-end comparison with a
forward from the images alone catches what the per-layer checks cannot: a kernel that reads the wrong buffer, or one
that is not yet written."""
import pytest
import torch
import torch.nn.functional as F

import bench
from oracle import resnet as oresnet

pytestmark = pytest.mark.gpu


def aser_eval_batches():
    """Batch sizes of the ASER eval-mode feature passes of the benchmark (retrieve.py, update.py): retrieval runs the
    current batch, the cooperative samples and the candidates (n_smp_cls per class each); the update runs the eval
    samples (n_smp_cls per class), the candidates (n_smp_cls * classes) and the current batch."""
    p, C = bench.params_for('aser'), bench.NUM_CLASSES
    return (p.batch + 2 * int(p.n_smp_cls) * C, int(p.n_smp_cls) * C + int(p.n_smp_cls * C) + p.batch)


# The benchmark's forwards (ER at 10 and 20 images, SCR's mlp head at 110), the ASER eval batches, one image, the
# Mini-ImageNet sizes of the backward test, and the batch sizes the coverage test below needs to reach every
# (kernel, template) pair of the train and eval forwards on a 132-SM H100.
CASES = ([(32, None, n) for n in (1, 10, 20, 66) + aser_eval_batches()] + [(32, 'mlp', 110)] +
         [(84, None, n) for n in (1, 2, 6, 10, 20, 22, 42, 110, 160)])

# max |got - ref| / max |ref| per tensor, by kind, about 3x the largest value measured over all cases of this file on an
# H100 80GB HBM3 (SXM, 132 SMs, 700 W power limit):
#   z (conv outputs) 8.6e-7 (layer4.0.conv1, Mini-ImageNet N = 160), mean 2.2e-8 (layer4.0.bn1, Mini-ImageNet N = 22),
#   invstd 5.9e-8 (layer2.0.shortcut.1, Mini-ImageNet N = 2), a (activations) 1.4e-7 (layer3.0.bn2, SCR mlp N = 110,
#   eval statistics), feat 1.9e-7, head 1.9e-7 (out, Mini-ImageNet N = 20, eval statistics),
#   e2e (out from the images alone) 1.3e-6 (Mini-ImageNet N = 110), eval (features_eval) 2.0e-6 (CIFAR N = 260).
# run (running statistics, against running_ref): measured 0 (the same bits) in every case; set to two fp32 ulps of the
# largest statistic, since fp64 sums in another order could round a batch statistic the other way.
# The smallest last-image share measured is 1.9e-5 (mean, bn1, Mini-ImageNet N = 160), 9.5e-5 (invstd) and 2.9e-6
# (running_var, bn1, Mini-ImageNet N = 160), each more than 10 x TOL.
TOL = {'z': 2.6e-6, 'mean': 6.6e-8, 'invstd': 1.8e-7, 'a': 4.1e-7, 'feat': 5.6e-7, 'head': 5.7e-7, 'run': 2.4e-7,
       'e2e': 3.8e-6, 'eval': 6.1e-6}
STATS = ('mean', 'invstd', 'run')   # kinds whose tolerance must stay 10x below the last image's effect


@pytest.fixture(scope='module')
def engine():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import engine
    return engine


def make_engine(engine, spec, seed):
    params, bn = oresnet.seeded_state(spec, seed)
    eng = engine.Engine(spec.in_hw, spec.num_classes, head=spec.head)
    eng.load(list(params.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
    return eng


def images(spec, N):
    gen = torch.Generator().manual_seed(3000 * spec.in_hw + N)
    return torch.rand(N, 3, spec.in_hw, spec.in_hw, generator=gen).cuda()


def nan_workspace(eng, N):
    ws = eng.new_train_workspace(N)
    ws.view(torch.float32).fill_(float('nan'))
    return ws


def blocks(spec):
    """[(c1, c2, sc or -1)] conv layer indices of the 8 BasicBlocks (BatchNorm2d module order)."""
    out, i = [], 1
    for _, _, _, _, sc in oresnet.block_plan(spec):
        out.append((i, i + 1, i + 2 if sc else -1))
        i += 3 if sc else 2
    return out


class Workspace:
    """fp64 views of the tensors a forward left in a train workspace."""

    def __init__(self, engine, eng, ws, N):
        self.ws, self.N = ws, N
        self.L = [engine.train_ws_layout(eng.desc, N, i) for i in range(eng.info.n_bn)]

    def raw(self, off, shape):
        n = 1
        for s in shape:
            n *= s
        return self.ws[off:off + 4 * n].view(torch.float32).reshape(shape)

    def f64(self, off, shape):
        return self.raw(off, shape).double()

    def act(self, i, which):   # NHWC -> NCHW
        L = self.L[i]
        return self.f64(getattr(L, which), (self.N, L.hout, L.wout, L.cout)).permute(0, 3, 1, 2)

    def stats(self, i):
        L = self.L[i]
        return self.f64(L.mean, (L.cout,)), self.f64(L.invstd, (L.cout,))


def rel(got, ref, scale=None):
    scale = float(ref.abs().max()) if scale is None else scale
    assert scale > 0
    err = float((got.double() - ref).abs().max()) / scale
    return err if err == err else float('inf')


def chan(t):
    return t[None, :, None, None]


def running_ref(run, s):
    """The running-statistic update of the kernels (bn_running_update) from the fp64 batch statistic s, with their fp32
    roundings: fma(1 - 0.1f, run, fl(0.1f * fl(s))).  Leaves the fp32 result within an ulp of the engine's, so the
    tolerance can sit far below the last image's share of the update, a few ulps of a fp32 running statistic."""
    m = torch.tensor(oresnet.BN_MOMENTUM, dtype=torch.float32, device=s.device)
    return ((1 - m).double() * run.double() + (m * s.float()).double()).float().double()


def batch_stats(z):
    """fp64 mean, biased variance, unbiased variance per channel of NCHW z."""
    M = z.shape[0] * z.shape[2] * z.shape[3]
    mean = z.mean((0, 2, 3))
    var = ((z - chan(mean)) ** 2).sum((0, 2, 3)) / M
    return mean, var, var * M / max(M - 1, 1)


def check_layers(spec, eng, P, W, x, run_before, eval_stats=False):
    """Per-layer rows (kind, name, err, share): conv outputs, batch statistics, activations, head tensors and running
    statistics, each from the engine's own inputs.  share: how much dropping the last image moves a statistic (same
    scale as err), None where not applicable."""
    N, rows = W.N, []
    bns = oresnet.bn_names(spec)
    conv_w = [spec.prefix + 'conv1.weight']
    for name, _, _, _, sc in oresnet.block_plan(spec):
        conv_w += [spec.prefix + name + '.conv1.weight', spec.prefix + name + '.conv2.weight']
        if sc:
            conv_w.append(spec.prefix + name + '.shortcut.0.weight')
    inputs = {0: x.double()}
    for b, (c1, c2, sc) in enumerate(blocks(spec)):
        x_in = W.act(blocks(spec)[b - 1][1] if b else 0, 'a')
        inputs[c1] = x_in
        inputs[c2] = W.act(c1, 'a')
        if sc >= 0:
            inputs[sc] = x_in
    run_after = eng.bn_views()

    def bn(i):
        mean, invstd = W.stats(i)
        return (W.act(i, 'z') - chan(mean)) * chan(invstd * P[bns[i] + '.weight']) + chan(P[bns[i] + '.bias'])

    for i, name in enumerate(bns):
        L = W.L[i]
        z = W.act(i, 'z')
        ref = F.conv2d(inputs[i], P[conv_w[i]], stride=L.stride, padding=(L.ks - 1) // 2)
        rows.append(('z', name, rel(z, ref), None))
        mean, invstd = W.stats(i)
        rm0, rv0 = (t.double() for t in run_before[i])
        rm1, rv1 = (t.double() for t in run_after[i])
        if eval_stats:
            # GSS-greedy's eval-mode pass normalises with the running statistics: bit for bit what the kernel computes
            assert torch.equal(W.raw(L.mean, (L.cout,)), run_before[i][0]), name
            assert torch.equal(W.raw(L.invstd, (L.cout,)), 1.0 / torch.sqrt(run_before[i][1] + oresnet.BN_EPS)), name
        else:
            m, v, vu = batch_stats(z)
            zscale = float(z.abs().max())
            inv = 1.0 / torch.sqrt(v + oresnet.BN_EPS)
            share = (None,) * 4
            if N >= 2:
                m_, v_, vu_ = batch_stats(z[:-1])
                share = (rel(m_, m, zscale), rel(1.0 / torch.sqrt(v_ + oresnet.BN_EPS), inv),
                         rel(0.1 * m_, 0.1 * m, float(rm1.abs().max())), rel(0.1 * vu_, 0.1 * vu, float(rv1.abs().max())))
            rows.append(('mean', name, rel(mean, m, zscale), share[0]))
            rows.append(('invstd', name, rel(invstd, inv), share[1]))
            rows.append(('run', name + '.running_mean', rel(rm1, running_ref(rm0, m)), share[2]))
            rows.append(('run', name + '.running_var', rel(rv1, running_ref(rv0, vu)), share[3]))
    for i in [0] + [c1 for c1, _, _ in blocks(spec)]:
        rows.append(('a', bns[i], rel(W.act(i, 'a'), torch.relu(bn(i))), None))
    for b, (c1, c2, sc) in enumerate(blocks(spec)):
        res = bn(sc) if sc >= 0 else inputs[c1]
        rows.append(('a', bns[c2], rel(W.act(c2, 'a'), torch.relu(bn(c2) + res)), None))
        if sc >= 0:   # the forward never writes a shortcut's activation slot
            assert torch.isnan(W.raw(W.L[sc].a, (N, W.L[sc].hout, W.L[sc].wout, W.L[sc].cout))).all(), bns[sc]
    # head: avg_pool2d(., 4) of the top-left 4 * PH square (11 -> 8 on Mini-ImageNet), NCHW flatten
    PH = spec.pooled_hw
    last = W.act(blocks(spec)[-1][1], 'a')
    L0 = W.L[0]
    feat = W.f64(L0.feat, (N, spec.dim_in))
    rows.append(('feat', 'feat', rel(feat, F.avg_pool2d(last[:, :, :4 * PH, :4 * PH], 4).reshape(N, -1)), None))
    return rows, feat


def check_head(spec, eng, P, W, feat, out):
    rows, N = [], W.N
    if spec.head is None:
        rows.append(('head', 'out', rel(out, F.linear(feat, P['linear.weight'], P['linear.bias'])), None))
        return rows
    pre = feat
    if spec.head == 'mlp':
        hid = W.f64(W.L[0].hid, (N, spec.dim_in))
        proj = W.f64(W.L[0].proj, (N, eng.out_dim))
        rows.append(('head', 'hid', rel(hid, torch.relu(F.linear(feat, P['head.0.weight'], P['head.0.bias']))), None))
        rows.append(('head', 'proj', rel(proj, F.linear(hid, P['head.2.weight'], P['head.2.bias'])), None))
        pre = proj
    elif spec.head == 'linear':
        proj = W.f64(W.L[0].proj, (N, eng.out_dim))
        rows.append(('head', 'proj', rel(proj, F.linear(feat, P['head.weight'], P['head.bias'])), None))
        pre = proj
    rows.append(('head', 'out', rel(out, F.normalize(pre, dim=1)), None))
    return rows


def fp64_state(spec, eng):
    P = {k: v.double().reshape(s) for (k, s), v in zip(oresnet.param_shapes(spec).items(), eng.param_views())}
    bn = {}
    for name, (rm, rv) in zip(oresnet.bn_names(spec), eng.bn_views()):
        bn[name + '.running_mean'] = rm.double().clone()
        bn[name + '.running_var'] = rv.double().clone()
        bn[name + '.num_batches_tracked'] = torch.zeros((), dtype=torch.long)
    return P, bn


def run_case(engine, hw, head, N):
    """Train forward over a NaN-filled workspace, checked layer by layer, end to end and in eval mode.
    Returns [(kind, name, err, share)]."""
    spec = oresnet.Spec(hw, 20, 100, head=head)
    eng = make_engine(engine, spec, 40 + N)
    x = images(spec, N)
    P, bn_before = fp64_state(spec, eng)
    run_before = [(rm.clone(), rv.clone()) for rm, rv in eng.bn_views()]
    tracked = eng.state.bn_tracked.clone()
    ws = nan_workspace(eng, N)
    out, _ = eng.forward_train(x, ws=ws)
    assert torch.equal(eng.state.bn_tracked, tracked + 1)
    W = Workspace(engine, eng, ws, N)
    rows, feat = check_layers(spec, eng, P, W, x, run_before)
    rows += check_head(spec, eng, P, W, feat, out)
    with torch.no_grad():
        ref = oresnet.forward(spec, P, bn_before, x.double(), train=True)
    rows.append(('e2e', 'out', rel(out, ref), None))
    _, bn_after = fp64_state(spec, eng)
    with torch.no_grad():
        ref_eval = oresnet.features(spec, P, bn_after, x.double(), train=False)
    rows.append(('eval', 'features_eval', rel(eng.features_eval(x), ref_eval), None))
    return rows


def check(rows, N):
    # worst offenders first: a wrong layer spreads into every layer after it in the end-to-end rows
    bad = sorted(((err / TOL[k], k, name, err) for k, name, err, _ in rows if not err <= TOL[k]), reverse=True)
    assert not bad, bad[:4]
    if N >= 2:
        # a statistics tolerance that could hide a dropped image would be useless
        for k, name, _, share in rows:
            if k in STATS:
                assert 10 * TOL[k] <= share, (k, name, share, TOL[k])


@pytest.mark.parametrize('hw,head,N', CASES)
def test_forward_matches_fp64(engine, hw, head, N):
    check(run_case(engine, hw, head, N), N)


@pytest.mark.parametrize('hw,head,N', [(32, None, 10), (32, 'mlp', 110), (84, None, 20)])
def test_evalgrad_forward(engine, hw, head, N):
    """GSS-greedy's eval-statistics forward: the saved statistics are the running ones (mean bit for bit, invstd =
    1 / sqrtf(running_var + eps)), nothing moves, and every layer matches fp64 from the engine's own inputs."""
    spec = oresnet.Spec(hw, 20, 100, head=head)
    eng = make_engine(engine, spec, 60 + N)
    x = images(spec, N)
    P, _ = fp64_state(spec, eng)
    stats, tracked = eng.state.bn_stats.clone(), eng.state.bn_tracked.clone()
    run_before = [(rm.clone(), rv.clone()) for rm, rv in eng.bn_views()]
    ws = nan_workspace(eng, N)
    out, _ = eng.forward_train(x, ws=ws, eval_stats=True)
    assert torch.equal(eng.state.bn_stats, stats) and torch.equal(eng.state.bn_tracked, tracked)
    W = Workspace(engine, eng, ws, N)
    rows, feat = check_layers(spec, eng, P, W, x, run_before, eval_stats=True)
    rows += check_head(spec, eng, P, W, feat, out)
    _, bn = fp64_state(spec, eng)
    with torch.no_grad():
        ref = oresnet.forward(spec, P, bn, x.double(), train=False)
    rows.append(('eval', 'out', rel(out, ref), None))
    check(rows, 1)


@pytest.mark.parametrize('hw,head,N', [(32, None, 10), (32, 'mlp', 110), (84, None, 22)])
def test_deferred_forward_is_bit_identical(engine, hw, head, N):
    """The deferred-statistics forward leaves the running statistics alone and writes the same bits as the plain
    forward; applying its statistics afterwards moves the running statistics to the plain forward's bits."""
    spec = oresnet.Spec(hw, 20, 100, head=head)
    eng = make_engine(engine, spec, 80 + N)
    x = images(spec, N)
    stats, tracked = eng.state.bn_stats.clone(), eng.state.bn_tracked.clone()
    ws_d, ws_p = nan_workspace(eng, N), nan_workspace(eng, N)
    out_d, _ = eng.forward_train(x, ws=ws_d, defer_stats=True)
    assert torch.equal(eng.state.bn_stats, stats) and torch.equal(eng.state.bn_tracked, tracked)
    out_p, _ = eng.forward_train(x, ws=ws_p)
    assert torch.equal(out_d, out_p)
    Wd, Wp = Workspace(engine, eng, ws_d, N), Workspace(engine, eng, ws_p, N)
    for L in Wp.L:
        shape = (N, L.hout, L.wout, L.cout)
        for off, shp in ((L.z, shape), (L.mean, (L.cout,)), (L.invstd, (L.cout,))):
            assert torch.equal(Wd.raw(off, shp), Wp.raw(off, shp))
        assert torch.equal(Wd.raw(L.a, shape), Wp.raw(L.a, shape)) or torch.isnan(Wp.raw(L.a, shape)).all()
    L0 = Wp.L[0]
    for off, n in ((L0.feat, spec.dim_in), (L0.hid, spec.dim_in), (L0.proj, eng.out_dim)):
        if head == 'mlp' or off == L0.feat:
            assert torch.equal(Wd.raw(off, (N, n)), Wp.raw(off, (N, n)))
    plain, plain_tracked = eng.state.bn_stats.clone(), eng.state.bn_tracked.clone()
    eng.state.bn_stats.copy_(stats)
    eng.state.bn_tracked.copy_(tracked)
    eng.apply_running_stats(ws_d, N)
    assert torch.equal(eng.state.bn_stats, plain) and torch.equal(eng.state.bn_tracked, plain_tracked)


def test_cases_reach_every_forward_kernel(engine):
    """On this card, CASES reach every (kernel, template) pair the three networks can take at N <= 512 in the train
    and the eval forward, and the backward test's cases every pair of the data-gradient launches.  The thresholds move
    with the SM count, so they are read through the hook rather than written down."""
    import test_gpu_backward_fp64 as bwd
    nets = [(32, None), (32, 'mlp'), (84, None)]
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    def reach(cases, pass_):
        got = set()
        for hw, head, N in cases:
            desc, info, _ = engine.describe(hw, 100, head)
            for i in range(1 if pass_ == 'dgrad' else 0, info.n_bn):
                g = engine.conv_geom(desc, N, i, pass_)
                assert g.sms == sms
                got.add(g.template)
        return got

    for pass_, cases in (('train', CASES), ('eval', CASES), ('dgrad', bwd.CASES + bwd.EVAL_CASES)):
        every = reach([(hw, head, N) for hw, head in nets for N in range(1, 513)], pass_)
        assert reach(cases, pass_) == every, (pass_, sorted(every - reach(cases, pass_)))


def test_selftest_partials_stay_in_the_workspace(engine):
    """A train-mode 21x21 80 -> 80 convolution on the CUDA-core path at a batch size the planner sends to patch<80, 1>
    (16 images on 132 SMs: 22 tiles per image) against fp64, with a guard region after the workspace that must come
    back untouched."""
    from b200ocl import _native
    from b200ocl.ops import _stream
    S, C = 21, 80                                          # 21x21 map, 80 -> 80 channels, train mode on path 1
    N = next(n for n in range(1, 129) if engine.conv_selftest_geom(n, S, S, C, C, 3, 1, 0, 1, 2).template == ('patch', 80, 1))
    g = engine.conv_selftest_geom(N, S, S, C, C, 3, 1, 0, 1, 2)
    assert g.grid_x > (N * S * S + 31) // 32           # more CTAs than one per 32 pixels
    lib = _native.lib()
    nbytes = lib.b200ocl_conv_selftest_workspace_bytes(N, C, C, S, S, 3, 1)
    guard = 1 << 20
    buf = torch.empty(nbytes + guard, dtype=torch.uint8, device='cuda')
    buf[:nbytes].view(torch.float32).fill_(float('nan'))
    buf[nbytes:].fill_(0xA5)
    gen = torch.Generator(device='cuda').manual_seed(N)
    w = torch.randn(C, C, 3, 3, device='cuda', generator=gen) / (9 * C) ** 0.5
    x = torch.relu(torch.randn(N, S, S, C, device='cuda', generator=gen))
    out = torch.full((N, S, S, C), float('nan'), device='cuda')
    stats = torch.full((4 * C,), float('nan'), device='cuda')
    rc = lib.b200ocl_conv_selftest(x.data_ptr(), w.data_ptr(), out.data_ptr(), N, S, S, C, C, 3, 1, 0, 1, 2,
                                   stats.data_ptr(), buf.data_ptr(), nbytes, _stream())
    _native.check(rc, 'b200ocl_conv_selftest')
    torch.cuda.synchronize()
    assert bool((buf[nbytes:] == 0xA5).all())
    z = out.permute(0, 3, 1, 2).double()
    m, v, vu = batch_stats(z)
    st = stats.double().reshape(4, C)
    check([('z', 'out', rel(z, F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), padding=1)), None),
           ('mean', 'mean', rel(st[0], m, float(z.abs().max())), None),
           ('invstd', 'invstd', rel(st[1], 1.0 / torch.sqrt(v + oresnet.BN_EPS)), None),
           ('run', 'running_mean', rel(st[2], running_ref(torch.zeros_like(m), m)), None),
           ('run', 'running_var', rel(st[3], running_ref(torch.zeros_like(vu), vu)), None)], 1)
