"""GPU: the network backward (b200ocl_net_backward) against an fp64 restatement of it built from the engine's own
forward, at the batch sizes that take each BN-backward and weight-gradient launch geometry.

Given the tensors the forward leaves in the train workspace (raw and activated conv outputs, the saved BN batch
statistics, feat / hid / proj), the backward is a linear map of dout: the ReLU masks and batch statistics are the
engine's own, so no branch can flip between the engine and the reference and the tolerance can be tight.  The
reference follows net_bwd.cu step by step in float64 with torch ops on the GPU."""
import pytest
import torch
import torch.nn.grad as tgrad

from oracle import resnet as oresnet

pytestmark = pytest.mark.gpu

# batch sizes that cross the planner's thresholds (the coverage test below checks what they reach on this card)
CASES = ([(32, None, n) for n in (1, 2, 10, 20, 37, 110, 160, 210)] + [(32, 'mlp', n) for n in (2, 20, 110, 220)] +
         [(32, 'linear', 20), (32, 'None', 20)] + [(84, None, n) for n in (2, 6, 10, 20, 22, 110, 160)] + [(84, 'mlp', 110)])
EVAL_CASES = [(32, None, n) for n in (1, 10, 110)]

# max |got - ref| / max |ref| per parameter tensor, by kind, about 3x the largest value measured over all cases on an
# H100 80GB HBM3 (SXM, 132 SMs, 700 W power limit):
#   conv weights 9.6e-6 (encoder.layer1.0.conv1.weight, CIFAR mlp N = 220),
#   BN gamma / beta 1.2e-5 (layer2.0.bn1.bias, Mini-ImageNet N = 160),
#   head linears 5.4e-7 (linear.weight, CIFAR N = 160).
# The smallest last-image share measured is 2.5e-2 (BN), 4.9e-2 (conv) and 6.7e-2 (head), far above 10 x TOL.
TOL = {'conv': 3e-5, 'bn': 4e-5, 'head': 2e-6}


@pytest.fixture(scope='module')
def engine():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import engine
    return engine


def conv_name(bn):
    """Weight of the convolution a BatchNorm2d follows: bn1 -> conv1, shortcut.1 -> shortcut.0."""
    if bn.endswith('shortcut.1'):
        return bn[:-1] + '0.weight'
    return bn[:-3] + 'conv' + bn[-1] + '.weight'


def kind(name, shape):
    if len(shape) == 4:
        return 'conv'
    if name.startswith(('linear.', 'head.')):
        return 'head'
    return 'bn'


def make_engine(engine, spec, seed):
    params, bn = oresnet.seeded_state(spec, seed)
    eng = engine.Engine(spec.in_hw, spec.num_classes, head=spec.head)
    eng.load(list(params.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
    return eng


def inputs(spec, eng, N):
    gen = torch.Generator().manual_seed(1000 * spec.in_hw + N)
    x = torch.rand(N, 3, spec.in_hw, spec.in_hw, generator=gen)
    dout = torch.randn(N, eng.out_dim, generator=gen)
    return x.cuda(), dout.cuda()


def reference(engine, eng, spec, ws, N, x, dout, eval_stats):
    """fp64 backward from the engine's parameters and the tensors its forward left in ws.
    Returns name -> (gradient, the last image's share of it)."""
    P = {k: v.double().reshape(s) for (k, s), v in zip(oresnet.param_shapes(spec).items(), eng.param_views())}
    bns = oresnet.bn_names(spec)
    L = [engine.train_ws_layout(eng.desc, N, i) for i in range(len(bns))]

    def f32(off, shape):
        n = 1
        for s in shape:
            n *= s
        return ws[off:off + 4 * n].view(torch.float32).reshape(shape).double()

    def act(i, which):   # NHWC in the workspace -> NCHW
        return f32(getattr(L[i], which), (N, L[i].hout, L[i].wout, L[i].cout)).permute(0, 3, 1, 2)

    def chan(t):
        return t[None, :, None, None]

    R = {}

    def linear(w, b, dY, X):
        R[w] = (dY.t() @ X, torch.outer(dY[-1], X[-1]))
        R[b] = (dY.sum(0), dY[-1])
        return dY @ P[w]

    def l2norm_bwd(pre, d):
        nrm = pre.norm(dim=1, keepdim=True).clamp_min(1e-12)
        y = pre / nrm
        return (d - y * (y * d).sum(1, keepdim=True)) / nrm

    def bn_bwd(i, g):
        z = act(i, 'z')
        mean, invstd = f32(L[i].mean, (L[i].cout,)), f32(L[i].invstd, (L[i].cout,))
        xh = (z - chan(mean)) * chan(invstd)
        db, dg = g.sum((0, 2, 3)), (g * xh).sum((0, 2, 3))
        R[bns[i] + '.weight'] = (dg, (g[-1] * xh[-1]).sum((1, 2)))
        R[bns[i] + '.bias'] = (db, g[-1].sum((1, 2)))
        k = chan(P[bns[i] + '.weight'] * invstd)
        if eval_stats:
            return k * g
        M = g.shape[0] * g.shape[2] * g.shape[3]
        return k * (g - chan(db / M) - xh * chan(dg / M))

    def conv_bwd(i, xin, dz):
        name = conv_name(bns[i])
        w, s, p = P[name], L[i].stride, (L[i].ks - 1) // 2
        R[name] = (tgrad.conv2d_weight(xin, w.shape, dz, stride=s, padding=p),
                   tgrad.conv2d_weight(xin[-1:], w.shape, dz[-1:], stride=s, padding=p))
        return tgrad.conv2d_input(xin.shape, w, dz, stride=s, padding=p)

    feat = f32(L[0].feat, (N, spec.dim_in))
    d = dout.double()
    if spec.head is None:
        dfeat = linear('linear.weight', 'linear.bias', d, feat)
    elif spec.head == 'None':
        dfeat = l2norm_bwd(feat, d)
    else:
        dp = l2norm_bwd(f32(L[0].proj, (N, eng.out_dim)), d)
        if spec.head == 'linear':
            dfeat = linear('head.weight', 'head.bias', dp, feat)
        else:
            hid = f32(L[0].hid, (N, spec.dim_in))
            dhid = linear('head.2.weight', 'head.2.bias', dp, hid) * (hid > 0)
            dfeat = linear('head.0.weight', 'head.0.bias', dhid, feat)
    # avg_pool2d(., 4) + NCHW flatten; rows / columns past 4 * pooled get nothing (11 -> 8 on Mini-ImageNet)
    last = L[-1]
    PH = spec.pooled_hw
    dA = torch.zeros(N, last.cout, last.hout, last.wout, dtype=torch.float64, device=d.device)
    dA[:, :, :4 * PH, :4 * PH] = dfeat.reshape(N, last.cout, PH, PH).repeat_interleave(4, 2).repeat_interleave(4, 3) / 16
    blocks, i = [], 1
    for _, _, _, _, sc in oresnet.block_plan(spec):
        blocks.append((i, i + 1, i + 2 if sc else -1))
        i += 3 if sc else 2
    for b in reversed(range(len(blocks))):
        c1, c2, sc = blocks[b]
        x_in = act(blocks[b - 1][1] if b else 0, 'a')
        a1 = act(c1, 'a')
        g = dA * (act(c2, 'a') > 0)
        g3 = conv_bwd(c2, a1, bn_bwd(c2, g))
        g_in = conv_bwd(sc, x_in, bn_bwd(sc, g)) if sc >= 0 else g
        dA = g_in + conv_bwd(c1, x_in, bn_bwd(c1, g3 * (a1 > 0)))
    conv_bwd(0, x.double(), bn_bwd(0, dA * (act(0, 'a') > 0)))
    return R


def run_case(engine, hw, head, N, eval_stats=False):
    """Engine forward + backward over a NaN-filled gradient arena, and the fp64 reference.
    Returns the engine, its gradient arena and [(name, kind, rel error, rel size of the last image's share)]."""
    spec = oresnet.Spec(hw, 20, 100, head=head)
    eng = make_engine(engine, spec, 7 + N)
    x, dout = inputs(spec, eng, N)
    ws = eng.new_train_workspace(N)
    eng.forward_train(x, ws=ws, eval_stats=eval_stats)
    eng.state.grads.fill_(float('nan'))          # every element with a gradient must be written
    eng.backward(x, dout, ws, eval_stats=eval_stats)
    got = eng.state.grads.clone()
    R = reference(engine, eng, spec, ws, N, x, dout, eval_stats)
    rows = []
    for (name, shape), (o, n, has_grad) in zip(oresnet.param_shapes(spec).items(), eng.table):
        g = got[o:o + n]
        if not has_grad:                          # SupConResNet's encoder classifier: never touched
            assert torch.isnan(g).all(), name
            continue
        assert name in R, name
        ref, share = R[name]
        scale = float(ref.abs().max())
        assert scale > 0, name
        err = float((g.double() - ref.reshape(-1)).abs().max()) / scale
        rows.append((name, kind(name, shape), err if err == err else float('inf'), float(share.abs().max()) / scale))
    return eng, got, rows


def check(rows, N):
    # worst offenders first: an error in one layer spreads to every layer below it
    bad = sorted(((err / TOL[k], name, err) for name, k, err, _ in rows if not err <= TOL[k]), reverse=True)
    assert not bad, bad[:4]
    if N >= 2:
        # a tolerance that could hide a dropped image (or tile) would be useless
        for name, k, _, share in rows:
            assert 10 * TOL[k] <= share, (name, share, TOL[k])


@pytest.mark.parametrize('hw,head,N', CASES)
def test_backward_matches_fp64(engine, hw, head, N):
    _, _, rows = run_case(engine, hw, head, N)
    check(rows, N)


@pytest.mark.parametrize('hw,head,N', EVAL_CASES)
def test_evalgrad_backward_matches_fp64(engine, hw, head, N):
    """GSS-greedy's eval-mode backward: BN statistics are constants, dz = gamma * invstd * g."""
    _, _, rows = run_case(engine, hw, head, N, eval_stats=True)
    check(rows, N)


@pytest.mark.parametrize('hw,head,N', [(32, 'mlp', 110), (32, None, 160), (84, None, 22)])
def test_backward_bit_properties(engine, hw, head, N):
    """No float atomics and fixed-order reductions: repeated calls give the same bits; an accumulating call over the
    same batch gives exactly twice the gradient (g + g is exact in fp32); the second arena gets the same bits; the
    graphed replay over the engine's own slot workspace equals the eager call."""
    spec = oresnet.Spec(hw, 20, 100, head=head)
    eng = make_engine(engine, spec, 3)
    x, dout = inputs(spec, eng, N)
    ws = eng.new_train_workspace(N)
    eng.forward_train(x, ws=ws)
    eng.backward(x, dout, ws)
    first = eng.state.grads.clone()
    eng.backward(x, dout, ws)
    assert torch.equal(eng.state.grads, first)
    eng.backward(x, dout, ws, accumulate=True)
    assert torch.equal(eng.state.grads, 2 * first)
    eng.alt_grads().fill_(float('nan'))
    eng.backward(x, dout, ws, alt=True)
    has = [(o, n) for (o, n, h) in eng.table if h]
    for o, n in has:
        assert torch.equal(eng.alt_grads()[o:o + n], first[o:o + n])
    for rep in range(4):                          # eager, graph warm-up, capture + replay, replay
        _, ws_slot = eng.forward_train(x)
        eng.backward(x, dout, ws_slot)
        assert torch.equal(eng.state.grads, first), rep
    assert ('bwd', N, 0, False, False) in eng._graphs


def test_cases_reach_every_backward_geometry(engine):
    """The case list reaches, on this card: both BN-backward paths at C = 20 and the two-phase path at every width, all
    three weight-gradient kernels, and a fused BN backward over more than half the SMs.  The thresholds move with the
    SM count, so they are read through the hook rather than written down."""
    two_phase, fused, kernels, wide_fused, sms = set(), set(), set(), False, None
    for hw, head, N in CASES + EVAL_CASES:
        desc, info, _ = engine.describe(hw, 100, head)
        for i in range(info.n_bn):
            L = engine.train_ws_layout(desc, N, i)
            sms = L.sms
            (fused if L.bn_fused else two_phase).add(L.cout)
            kernels.add(L.wgrad_kernel)
            wide_fused |= bool(L.bn_fused) and 2 * L.bn_grid > L.sms
    assert sms == torch.cuda.get_device_properties(0).multi_processor_count
    assert 20 in fused and two_phase >= {20, 40, 80, 160}, (fused, two_phase)
    assert kernels == {0, 1, 2}
    assert wide_fused
