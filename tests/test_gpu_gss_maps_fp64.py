"""GPU: GSS-greedy's eval-statistics pass (b200ocl_net_forward_evalgrad, then b200ocl_net_backward with bit 1 of
`accumulate`), its gradient cosine (b200ocl_grad_cosine) and the update rule against fp64, on the four networks GSS
runs on: CIFAR-100 (32x32, 100 classes), Mini-ImageNet (84x84, 100), OpenLORIS (50x50, 69) and CORe50 (128x128, 50, the
2560-input classifier), at the batch sizes GSS feeds them.  Those are N = 1 (every per-sample score), the memory
sub-batches min(gss_batch_size, current_index) = 1...10 while the memory fills, and the stream batch (10 by default).

  * Forward and backward layer by layer, each layer rebuilt in fp64 from the engine's own tensors
    (test_gpu_forward_fp64.check_layers / test_gpu_backward_fp64.reference with eval_stats=True), with those files'
    bars and the backward's 10x last-image-share rule for N >= 2.  BATCHES is the smallest list per network whose
    launches are those of every N in 1...10 at 114, 132 and 148 SMs; the coverage test proves it on the card in use.
  * The whole GSS gradient (GSSGreedyUpdate._gradient) against oracle.gss.eval_grad_vector run in float64.
  * b200ocl_grad_cosine at the four arena lengths and K = 1 ... 64 against fp64 with the kernel's rounding bound
    (cos_bound), over real eval-mode gradients of the engine plus edge rows.
  * GSSGreedyUpdate driven through a Buffer against oracle.gss.update on a float64 state holding the engine's own
    parameters, with the same random draws: identical slot writes, labels and image rows.
  * tests/golden/gss_maps.npz: the reference's own GSS run at 128x128 and 50x50, replayed.

Measured on an H100 80GB HBM3 (SXM, 132 SMs, 700 W power limit), largest value over all cases of this file:
  forward (max |got - ref| / max |ref| per tensor): z 6.7e-7 (mini_imagenet layer1.1.conv1, N = 10), a 1.5e-7
    (mini_imagenet N = 5), feat 1.5e-7, head 3.1e-7 and eval (out against oresnet.forward(train=False)) 1.4e-6 (all
    core50 N = 10): the bars of test_gpu_forward_fp64 hold, 3.9x or more above them.
  backward (per parameter tensor): conv 4.3e-6 (cifar100 layer2.1.conv1.weight, N = 1), BN 3.7e-6 (mini_imagenet
    layer1.1.bn1.weight, N = 9), head 1.4e-7 (mini_imagenet linear.bias, N = 10): the bars of test_gpu_backward_fp64
    hold; the smallest last-image share is 9.3e-2 (core50 N = 10), far above 10x every bar.
  GSS gradient: see GRAD_TOL and VEC_TOL.  Cosine: at most 0.50 of cos_bound (cifar100), a bound derived, not measured.
  Update rule: see SIM_TOL.  Replay of the reference's run: see REPLAY_TOL.
The whole file runs in about 45 s there.
"""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import test_gpu_backward_fp64 as bwd
import test_gpu_forward_fp64 as fwd
from oracle import gss as ogss
from oracle import resnet as oresnet

pytestmark = pytest.mark.gpu

DATASETS = ('cifar100', 'mini_imagenet', 'openloris', 'core50')
# per network, the smallest list of N in 1...10 (N = 1 always: GSS's per-sample passes) whose convolution templates,
# BN-backward forms per width and weight-gradient kernels are those of every N in 1...10 at 114, 132 and 148 SMs
BATCHES = {'cifar100': (1, 5), 'mini_imagenet': (1, 5, 9, 10), 'openloris': (1, 8), 'core50': (1, 4, 5, 6, 10)}
CASES = [(d, n) for d in DATASETS for n in BATCHES[d]]
GSS_NMAX = 10          # gss_batch_size and the stream batch of the reference's defaults and GSS configs

# the GSS gradient, about 3x the largest measured.  GRAD_TOL, per tensor against the fp64 gradient through the engine's
# own ReLU masks (max |got - ref| / max |ref|): conv 3.9e-6 (cifar100 layer1.0.conv1.weight, N = 1), BN 2.7e-6 (core50
# layer1.0.bn1.bias, N = 1), head 1.9e-7 (mini_imagenet linear.weight, N = 10).  VEC_TOL, |got - ref| / |ref| over the
# whole vector against eval_grad_vector in float64 from the images: 1.5e-5 (mini_imagenet N = 5).
GRAD_TOL = {'conv': 1.2e-5, 'bn': 8e-6, 'head': 6e-7}
VEC_TOL = 4.5e-5
# |score - fp64 score| and |batch_sim - fp64 batch_sim| of the update rule, about 3x the largest measured: 1.2e-7 (one
# fp32 ulp at 1, every network).  The fp64 rule's cosines come from fp64 gradients, so this bar also carries the
# gradients' own fp32 error on top of the cosine kernel's rounding (cos_bound, 3.6e-7 at |cos| = 1).
SIM_TOL = 4e-7
# scores and batch_sim of the replay against the reference's fp32 CPU run, about 3x the largest measured: 1.7e-5
# (core50)
REPLAY_TOL = 5e-5
MARGIN = 10            # every batch_sim of the update runs must sit at least MARGIN x SIM_TOL away from 0

U32, U64 = 2.0 ** -24, 2.0 ** -53


def net(data):
    from b200ocl import memory
    return memory.input_size_match[data][1], memory.n_classes[data]


def spec_of(data):
    hw, ncls = net(data)
    return oresnet.Spec(hw, 20, ncls)


@pytest.fixture(scope='module')
def engine():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import engine
    return engine


# ----------------------------------------------------------------------------------------------------- coverage
def launches(engine, data, N):
    """What one eval-statistics pass of N images takes on this card: the forward's convolution templates, the data
    gradient's, the BN-backward form per width and the weight-gradient kernels."""
    hw, ncls = net(data)
    desc, info, _ = engine.describe(hw, ncls)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = set()
    for i in range(info.n_bn):
        g = engine.conv_geom(desc, N, i, 'train')
        assert g.sms == sms
        out.add(('train',) + g.template)
        if i:
            out.add(('dgrad',) + engine.conv_geom(desc, N, i, 'dgrad').template)
        L = engine.train_ws_layout(desc, N, i)
        assert L.sms == sms
        out.add(('bn', L.cout, 'fused' if L.bn_fused else 'two-phase'))
        out.add(('wgrad', L.wgrad_kernel))
    return out


@pytest.mark.parametrize('data', DATASETS)
def test_cases_reach_every_gss_launch(engine, data):
    """The eval-statistics cases alone reach, on this card, every train-convolution template, data-gradient template,
    BN-backward form at every width and weight-gradient kernel that N in 1...10 takes on this network.  The
    thresholds move with the SM count, so they are read through the hooks rather than written down."""
    every = set().union(*[launches(engine, data, N) for N in range(1, GSS_NMAX + 1)])
    reached = set().union(*[launches(engine, data, N) for N in BATCHES[data]])
    assert reached == every, sorted(every - reached)
    assert {('bn', c, 'fused') for c in (20, 40, 80, 160)} <= reached


# ------------------------------------------------------------------------------------------ forward, layer by layer
@pytest.mark.parametrize('data,N', CASES)
def test_evalgrad_forward_maps(engine, data, N):
    """Over a NaN-filled workspace: the saved mean is running_mean bit for bit, the saved invstd is
    1 / sqrtf(running_var + eps) bit for bit, nothing moves, every layer matches fp64 from the engine's own inputs and
    the output matches oresnet.forward(train=False) from the images."""
    spec = spec_of(data)
    eng = fwd.make_engine(engine, spec, 60 + N)
    x = fwd.images(spec, N)
    P, _ = fwd.fp64_state(spec, eng)
    stats, tracked = eng.state.bn_stats.clone(), eng.state.bn_tracked.clone()
    run_before = [(rm.clone(), rv.clone()) for rm, rv in eng.bn_views()]
    ws = fwd.nan_workspace(eng, N)
    out, _ = eng.forward_train(x, ws=ws, eval_stats=True)
    assert torch.equal(eng.state.bn_stats, stats) and torch.equal(eng.state.bn_tracked, tracked)
    W = fwd.Workspace(engine, eng, ws, N)
    rows, feat = fwd.check_layers(spec, eng, P, W, x, run_before, eval_stats=True)
    rows += fwd.check_head(spec, eng, P, W, feat, out)
    _, bn = fwd.fp64_state(spec, eng)
    with torch.no_grad():
        ref = oresnet.forward(spec, P, bn, x.double(), train=False)
    rows.append(('eval', 'out', fwd.rel(out, ref), None))
    worst = {}
    for k, name, err, _ in rows:
        worst[k] = max(worst.get(k, (0, '')), (err, name))
    print('gss fwd %s N=%d %s' % (data, N, worst))
    fwd.check(rows, 1)


# ----------------------------------------------------------------------------------------- backward, layer by layer
@pytest.mark.parametrize('data,N', CASES)
def test_evalgrad_backward_maps(engine, data, N):
    """dz = gamma * invstd * g with the running statistics, every parameter gradient written (NaN-filled arena) and
    within test_gpu_backward_fp64's bars of its fp64 restatement; for N >= 2 each bar sits 10x under the last image's
    share of its tensor."""
    spec = spec_of(data)
    eng = bwd.make_engine(engine, spec, 7 + N)
    x, dout = bwd.inputs(spec, eng, N)
    stats = eng.state.bn_stats.clone()
    ws = eng.new_train_workspace(N)
    eng.forward_train(x, ws=ws, eval_stats=True)
    eng.state.grads.fill_(float('nan'))
    eng.backward(x, dout, ws, eval_stats=True)
    assert torch.equal(eng.state.bn_stats, stats)
    got = eng.state.grads.clone()
    R = bwd.reference(engine, eng, spec, ws, N, x, dout, True)
    rows = []
    for (name, shape), (o, n, has_grad) in zip(oresnet.param_shapes(spec).items(), eng.table):
        assert has_grad and name in R, name
        ref, share = R[name]
        scale = float(ref.abs().max())
        assert scale > 0, name
        err = float((got[o:o + n].double() - ref.reshape(-1)).abs().max()) / scale
        rows.append((name, bwd.kind(name, shape), err if err == err else float('inf'), float(share.abs().max()) / scale))
    worst = {}
    for name, k, err, sh in rows:
        worst[k] = max(worst.get(k, (0, '')), (err, name))
    print('gss bwd %s N=%d %s min share %.3g' % (data, N, worst, min(r[3] for r in rows)))
    bwd.check(rows, N)


# ------------------------------------------------------------------------------------------ the GSS gradient, e2e
def gss_update(mem_size=1, strength=10, gbs=10):
    from b200ocl import update
    return update.GSSGreedyUpdate(SimpleNamespace(gss_mem_strength=strength, gss_batch_size=gbs, mem_size=mem_size))


def fp64_cuda(spec, eng):
    P, bn = fwd.fp64_state(spec, eng)
    return ({k: v.cuda() for k, v in P.items()},
            {k: (v.cuda() if v.is_floating_point() else v) for k, v in bn.items()})


def batch(spec, N, seed):
    rs = np.random.RandomState(seed)
    x = torch.from_numpy(rs.rand(N, 3, spec.in_hw, spec.in_hw).astype(np.float32)).cuda()
    y = torch.from_numpy(rs.randint(0, spec.num_classes, N).astype(np.int64)).cuda()
    return x, y


@pytest.mark.parametrize('data,N', CASES)
def test_gss_gradient_matches_fp64(engine, data, N):
    """GSSGreedyUpdate._gradient (eval-statistics forward, cross-entropy, eval-statistics backward, on the engine's
    slot workspace), with a NaN-filled arena and the running statistics left alone:
      * tensor by tensor within GRAD_TOL of the fp64 gradient of the mean cross-entropy of the logits the engine's own
        features give, back through the engine's own ReLU masks (test_gpu_backward_fp64.reference);
      * as a whole within VEC_TOL of oracle.gss.eval_grad_vector run in float64 from the images.  There the fp64
        forward decides its own ReLU masks: a pre-activation within fp32 rounding of 0 that falls the other way moves
        the few weights it feeds by up to a few 1e-3 of their tensor's largest entry (measured), so that comparison is
        made on the whole vector, the quantity the cosine reads."""
    spec = spec_of(data)
    p, bn0 = small_head_state(spec, 90 + N)
    eng = engine.Engine(spec.in_hw, spec.num_classes)
    eng.load(list(p.values()), [(bn0[n + '.running_mean'], bn0[n + '.running_var']) for n in oresnet.bn_names(spec)])
    x, y = batch(spec, N, 500 + N)
    stats, tracked = eng.state.bn_stats.clone(), eng.state.bn_tracked.clone()
    eng.state.grads.fill_(float('nan'))
    got = gss_update()._gradient(eng, x, y).clone()
    assert torch.equal(eng.state.bn_stats, stats) and torch.equal(eng.state.bn_tracked, tracked)
    P, bn = fp64_cuda(spec, eng)
    ws = eng.train_workspace(N, slot=gss_update().SLOT)
    L0 = engine.train_ws_layout(eng.desc, N, 0)
    feat = ws[L0.feat:L0.feat + 4 * N * spec.dim_in].view(torch.float32).reshape(N, spec.dim_in).double()
    logits = feat @ P['linear.weight'].t() + P['linear.bias']
    dlogits = (torch.softmax(logits, 1) - torch.nn.functional.one_hot(y, spec.num_classes).double()) / N
    R = bwd.reference(engine, eng, spec, ws, N, x, dlogits, True)
    bad, worst = [], {}
    for (name, shape), (o, n, _) in zip(oresnet.param_shapes(spec).items(), eng.table):
        r = R[name][0].reshape(-1)
        scale = float(r.abs().max())
        assert scale > 0, name
        err = float((got[o:o + n].double() - r).abs().max()) / scale
        err = err if err == err else float('inf')
        k = bwd.kind(name, shape)
        worst[k] = max(worst.get(k, (0, '')), (err, name))
        if not err <= GRAD_TOL[k]:
            bad.append((err / GRAD_TOL[k], name, err))
    ref = ogss.eval_grad_vector(spec, P, bn, x.double(), y)
    assert ref.dtype == torch.float64 and ref.numel() == got.numel()
    vec = float((got.double() - ref).norm() / ref.norm())
    print('gss grad %s N=%d %s vector %.3g' % (data, N, worst, vec))
    assert not bad, sorted(bad, reverse=True)[:4]
    assert vec <= VEC_TOL, vec


# -------------------------------------------------------------------------------------------- gradient cosine
def cos_bound(cos64, n):
    """|cos32 - cos64| bound of b200ocl_grad_cosine given fp32 inputs of length n.  The kernel sums the exact fp32
    products in fp64 (error <= n u64 sum |a_i b_i| <= n u64 |a| |b|, as does the fp64 reference), then rounds the dot,
    |m|^2 and |g|^2 to fp32 (u32 each), takes two sqrtf (u32 each, halving the input's error: 1.5 u32 per norm), one
    product (u32), the clamp fmaxf(den, fl32(1e-8)) (exact; fl32(1e-8) is within u32 / 2 of 1e-8, and a max is off by
    no more than its worst argument) and one division (u32): 6 u32 relative to cos, plus second-order terms."""
    return (6 * U32 + 64 * U32 * U32) * cos64.abs() + 4 * n * U64


@pytest.fixture(scope='module')
def gradient_pool(engine):
    """Per dataset: (g, pool [64, n]).  g is a real stream-batch gradient (N = 10); the pool holds edge rows, then real
    eval-mode gradients of memory sub-batches and single samples (N = 1...10), whose tensors span many decades."""
    out = {}
    for data in DATASETS:
        spec = spec_of(data)
        eng = bwd.make_engine(engine, spec, 300)
        upd = gss_update()
        x, y = batch(spec, GSS_NMAX, 1)
        g = upd._gradient(eng, x, y).clone()
        real = []
        for i in range(60):
            xi, yi = batch(spec, 1 + i % GSS_NMAX, 1000 + i)
            real.append(upd._gradient(eng, xi, yi).clone())
        g64 = g.double()
        ng = float(g64.norm())
        r = real.pop().double()
        perp = r - (r @ g64) / (g64 @ g64) * g64                # cosine ~0 after the fp32 rounding
        t = 1e-5                                                 # cosine +-1e-5: the sign batch_sim < 0 reads
        near = [(perp / perp.norm() * (1 - t * t) ** 0.5 + s * t * g64 / ng) * float(r.norm()) for s in (1, -1)]
        h = real.pop().double()
        clamp = [h * (1e-8 * f / (float(h.norm()) * ng)) for f in (1 - 2 ** -10, 1 + 2 ** -10)]
        edge = [torch.zeros_like(g64), g64, -g64, perp] + near + clamp
        rows = [e.float() for e in edge] + real
        pool = torch.stack(rows[:64]).contiguous()
        assert pool.shape == (64, eng.info.n_params)
        out[data] = (g, pool)
    return out


ARENA = {'cifar100': 1109240, 'mini_imagenet': 1157240, 'openloris': 1104249, 'core50': 1221190}


@pytest.mark.parametrize('K', (1, 2, 10, 20, 50, 63, 64))
@pytest.mark.parametrize('data', DATASETS)
def test_grad_cosine_real_shapes(engine, gradient_pool, data, K):
    """b200ocl_grad_cosine over every row of the pool, K rows per call: within cos_bound of fp64 with no row excused,
    the sign of fp64 wherever |cos64| exceeds the bound, and max_out the maximum of cos_out bit for bit, also when
    written into one element of a larger tensor (the per-sample scores of update.py)."""
    from b200ocl import ops
    g, pool = gradient_pool[data]
    n = pool.shape[1]
    assert n == ARENA[data]
    g64 = g.double()
    ng = g64.norm()
    worst = 0.0
    for start in range(0, 64, K):
        idx = torch.arange(start, start + K) % 64
        mem = pool[idx.cuda()].contiguous()
        m64 = mem.double()
        ref = (m64 @ g64) / (m64.norm(dim=1) * ng).clamp(min=1e-8)
        bound = cos_bound(ref, n)
        scores = torch.full((K + 2,), float('nan'), device='cuda')
        j = start % (K + 2)
        cos, mx = ops.grad_cosine(mem, g, max_out=scores[j:j + 1])
        err = (cos.double() - ref).abs()
        worst = max(worst, float((err / bound).max()))
        bad = (~(err <= bound)).nonzero().flatten().tolist()
        assert not bad, [(int(idx[i]), float(cos[i]), float(ref[i]), float(bound[i])) for i in bad[:4]]
        sure = ref.abs() > bound
        assert torch.equal(torch.sign(cos.double())[sure], torch.sign(ref)[sure])
        assert torch.equal(mx, cos.max().reshape(1)) and torch.equal(scores[j:j + 1], mx)
        others = torch.ones(K + 2, dtype=torch.bool, device='cuda')
        others[j] = False
        assert torch.isnan(scores[others]).all()
        cos2, _ = ops.grad_cosine(mem, g)
        assert torch.equal(cos, cos2)
    # the edge rows do what they are there for
    cos, _ = ops.grad_cosine(pool[:8].contiguous(), g)
    c = cos.tolist()
    assert c[0] == 0.0 and abs(c[1] - 1) <= 8 * U32 and abs(c[2] + 1) <= 8 * U32
    assert 0 < c[4] and c[5] < 0
    print('gss cosine %s K=%d worst err / bound %.3g' % (data, K, worst))


# ----------------------------------------------------------------------------------------------- the update rule
def small_head_state(spec, seed):
    """Seeded weights with a small classifier (as test_gss_update_golden): softmax outputs near uniform, so the sign
    of a batch's gradient cosine with the memory follows its label overlap with the memory."""
    p, bn = oresnet.seeded_state(spec, seed)
    p['linear.weight'] = p['linear.weight'] * 0.02
    p['linear.bias'] = torch.zeros_like(p['linear.bias'])
    return p, bn


def gss_model(data, p, bn, mem_size, strength, gbs):
    from b200ocl import memory, nets
    spec = spec_of(data)
    params = SimpleNamespace(data=data, agent='ER', head=None, cuda=True, mem_size=mem_size, update='GSS',
                             retrieve='random', gss_mem_strength=strength, gss_batch_size=gbs, buffer_tracker=False,
                             eps_mem_batch=10)
    model = nets.setup_architecture(params)
    model.engine.load(list(p.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
    buf = memory.Buffer(model, params)
    model.train()
    return model, buf


def cpu_multinomial():
    """torch.multinomial with CUDA probabilities drawn on the CPU generator (the reference's scores live on the CPU)."""
    orig = torch.multinomial

    def multinomial(probs, *a, **k):
        if probs.is_cuda:
            return orig(probs.cpu(), *a, **k).to(probs.device)
        return orig(probs, *a, **k)
    return orig, multinomial


# (data, gss_mem_strength, gss_batch_size, mem_size, seed): K = 10 on every network, K = 50 on CORe50 (the largest
# gss_mem_strength gss_tune_core50.yml sweeps) with two-image memory sub-batches
UPDATE_CASES = [(d, 10, 10, 100, 7) for d in DATASETS] + [('core50', 50, 2, 100, 7)]


def update_plan(mem_size, gbs):
    """(n images, label set) per update: a first insertion of gss_batch_size - 1 (so the next fill draws one memory
    sub-batch of current_index < gss_batch_size), fills of 10, one that only partly fits, then full-memory updates
    with unseen classes (batch_sim < 0: the replacement lottery) and with seen classes (batch_sim >= 0)."""
    plan = [(gbs - 1, 'seen')]
    left = mem_size - (gbs - 1)
    while left > 0:
        plan.append((10, 'seen'))
        left -= 10
    return plan + [(10, 'unseen'), (10, 'seen'), (10, 'unseen'), (10, 'seen')]


@pytest.mark.parametrize('data,strength,gbs,mem_size,seed', UPDATE_CASES)
def test_gss_update_matches_fp64(engine, data, strength, gbs, mem_size, seed):
    """GSSGreedyUpdate through a Buffer against oracle.gss.update on a float64 state holding the engine's parameters,
    with the same draws (CPU generator for randperm and both multinomials): the same slots written, the same labels,
    the same image rows bit for bit, scores and batch_sim within SIM_TOL, and every batch_sim at least MARGIN x SIM_TOL
    from the decision at 0.  After each update the fp64 state continues from the engine's scores, so the lotteries
    draw from the same probabilities."""
    spec = spec_of(data)
    p, bn = small_head_state(spec, seed)
    model, buf = gss_model(data, p, bn, mem_size, strength, gbs)
    upd = buf.update_method
    P, bn64 = fp64_cuda(spec, model.engine)
    st = ogss.GSSState(spec, P, bn64, mem_size, (3, spec.in_hw, spec.in_hw), mem_strength=strength, gss_batch_size=gbs)
    st.buffer_img = st.buffer_img.double().cuda()
    st.buffer_label = st.buffer_label.cuda()
    rs = np.random.RandomState(seed)
    sims, worst, k_max = [], 0.0, 0
    for u, (n, which) in enumerate(update_plan(mem_size, gbs)):
        x = torch.from_numpy(rs.rand(n, 3, spec.in_hw, spec.in_hw).astype(np.float32))
        lab = rs.randint(0, 3, n) + (3 + 3 * (u % 2) if which == 'unseen' else 0)
        y = torch.from_numpy(lab.astype(np.int64))
        full = buf.current_index >= mem_size
        k_max = max(k_max, min(strength, buf.current_index // max(min(gbs, buf.current_index), 1)))
        img0, score0 = buf.buffer_img.clone(), upd.buffer_score.clone()
        orig, multinomial = cpu_multinomial()
        torch.manual_seed(100 * seed + u)
        torch.multinomial = multinomial
        try:
            buf.update(x.cuda(), y.cuda(), y_host=lab)
        finally:
            torch.multinomial = orig
        torch.manual_seed(100 * seed + u)
        written = ogss.update(st, x.double().cuda(), y.cuda())
        assert model.training
        changed = (buf.buffer_img != img0).flatten(1).any(1).nonzero().flatten().tolist()
        assert changed == sorted(s for _, s in written), (u, changed, written)
        if full:
            src, slots = upd.last_replaced if upd.last_replaced is not None else ([], [])
            assert sorted(zip(np.asarray(slots).tolist(), np.asarray(src).tolist())) == sorted((s, i) for i, s in written)
            d = abs(upd.last_batch_sim - st.last_batch_sim)
            worst = max(worst, d)
            assert d <= SIM_TOL, (u, upd.last_batch_sim, st.last_batch_sim)
            sims.append(upd.last_batch_sim)
        assert buf.current_index == st.current_index
        assert torch.equal(buf.buffer_img.double(), st.buffer_img)
        assert torch.equal(buf.buffer_label, st.buffer_label)
        np.testing.assert_array_equal(buf.labels_host, st.buffer_label.cpu().numpy())
        score = upd.buffer_score.cpu()
        d = float((score.double() - st.buffer_score.double()).abs().max())
        worst = max(worst, d)
        assert d <= SIM_TOL, (u, d)
        moved = (score != score0.cpu()).nonzero().flatten().tolist()
        assert set(moved) <= {s for _, s in written}
        st.buffer_score.copy_(score)
    print('gss update %s K=%d batch_sim %s worst |d| %.3g' % (data, strength, ['%.4g' % s for s in sims], worst))
    assert k_max == strength
    assert any(s < 0 for s in sims) and any(s >= 0 for s in sims)
    for s in sims:
        assert abs(s) >= MARGIN * SIM_TOL, (s, sims)


# ------------------------------------------------------------------------------------- the reference's own run
@pytest.mark.parametrize('data', ('openloris', 'core50'))
def test_gss_maps_golden(engine, golden_dir, data):
    """The plugin replays the reference's GSS run of gss_maps.npz (make_golden_gss_maps.py) at 50x50 and 128x128:
    the same slots replaced with the same samples, the same labels, scores and batch_sim within the reference run's
    fp32 spread (REPLAY_TOL)."""
    g = np.load(os.path.join(golden_dir, 'gss_maps.npz'))
    pre = data + '_'
    mem, n, seed = int(g[pre + 'mem']), int(g[pre + 'batch']), int(g[pre + 'data_seed'])
    spec = spec_of(data)
    p, bn = small_head_state(spec, int(g[pre + 'model_seed']))
    model, buf = gss_model(data, p, bn, mem, 10, 10)
    upd = buf.update_method
    rs = np.random.RandomState(seed)
    src = np.full((mem, 2), -1, dtype=np.int64)
    ys = g[pre + 'y']
    worst = 0.0
    for u in range(ys.shape[0]):
        x = torch.from_numpy(rs.rand(n, 3, spec.in_hw, spec.in_hw).astype(np.float32))
        rs.randint(0, 3, n)
        before = buf.buffer_img.clone()
        orig, multinomial = cpu_multinomial()
        torch.manual_seed(int(g[pre + 'torch_seed0']) + u)
        torch.multinomial = multinomial
        try:
            buf.update(x.cuda(), torch.from_numpy(ys[u]).cuda(), y_host=ys[u])
        finally:
            torch.multinomial = orig
        for sl in (buf.buffer_img != before).flatten(1).any(1).nonzero().flatten().tolist():
            pos = [i for i in range(n) if torch.equal(buf.buffer_img[sl].cpu(), x[i])]
            assert len(pos) == 1
            src[sl] = (u, pos[0])
        ref_sim = float(g[pre + 'batch_sim'][u])
        worst = max(worst, float(np.abs(upd.buffer_score.cpu().numpy() - g[pre + 'scores'][u]).max()))
        if ref_sim == ref_sim:
            worst = max(worst, abs(upd.last_batch_sim - ref_sim))
            assert abs(upd.last_batch_sim - ref_sim) <= REPLAY_TOL, (u, upd.last_batch_sim, ref_sim)
        np.testing.assert_array_equal(buf.buffer_label.cpu().numpy(), g[pre + 'labels'][u], err_msg='update %d' % u)
        np.testing.assert_array_equal(src, g[pre + 'src'][u], err_msg='update %d' % u)
        np.testing.assert_allclose(upd.buffer_score.cpu().numpy(), g[pre + 'scores'][u], rtol=0, atol=REPLAY_TOL)
        upd.buffer_score.copy_(torch.from_numpy(g[pre + 'scores'][u]))
    print('gss golden %s worst |d| %.3g' % (data, worst))
    assert buf.current_index == mem

