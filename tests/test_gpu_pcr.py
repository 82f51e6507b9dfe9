"""GPU: PCR (learners.PCR, opt-in as agents['PCR']).

  * b200ocl_pcr_loss against oracle/pcr.py in fp64 over R in {2, 3, 40, 220, 4096}, d in {160, 640, 2560}, C in {10,
    50, 69, 100} and tau in {0.07, 0.09, 1}; labels in pairs as the agent makes them, a single class, and a class that
    occurs once (NaN loss, finite gradient); feature rows of zero norm, of norm near eps and of norm 1e4.  Each bar is
    the smaller of a bound derived from the fp32 roundings and 1e-4 of the tensor's largest element.  Exact: absent-class
    rows of dW and the bias slice are 0, a repeated call gives the same bits, an out-of-range label raises the flag.
  * b200ocl_cosine_argmax: fp64's arg-max on rows without near ties, the lowest index among duplicate proxy rows, and
    n_correct exact for B from 1 to 257 at the three widths.
  * The backward pass from the features on all four maps: the encoder gradient within test_gpu_backward_fp64.py's bars
    of its fp64 restatement (which runs through the engine's own ReLU masks, so no branch can flip), within a looser
    bar of oracle.resnet.features autograd in fp64, and the linear.* gradient entries left untouched.
  * Whole steps against oracle/pcr.py (fp64) on CIFAR-100, Mini-ImageNet, OpenLORIS and CORe50 with the identity
    transform, and once with the engine's own augmented images; mem_iters = 2, an empty memory, a memory smaller than
    eps_mem_batch, Adam and weight decay.
  * Two-task runs whose accuracies are the fp64 cosine arg-max of the engine's own features.
Checkpoint resume, staged snapshots, concurrent runs and graphs against eager launches are checked with the other
agents, as agent_cases.CASES['pcr'] (test_gpu_checkpoint.py, test_gpu_checkpoint_async.py, test_gpu_multirun.py,
test_gpu_graphs.py)."""
from collections import OrderedDict
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from agent_cases import HW, NCLS, _learner, _load
from oracle import agem as oagem
from oracle import pcr as opcr
from oracle import resnet as oresnet

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24


@pytest.fixture(scope='module')
def b():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    import b200ocl
    from b200ocl import _native, engine, learners, memory, nets, ops, registry
    return SimpleNamespace(native=_native, engine=engine, learners=learners, memory=memory, nets=nets, ops=ops,
                           registry=registry)


# ----------------------------------------------------------------------------- the loss kernel
def _labels(rs, R, C, pattern):
    if pattern == 'pairs':                 # [y_m; y_m; y; y]: every row comes with its copy
        half = rs.randint(0, C, (R + 1) // 2)
        y = np.concatenate((half, half))[:R]
        if R % 2:
            y[R // 2] = y[0]
    elif pattern == 'single':
        y = np.full(R, rs.randint(0, C))
    else:                                  # 'once': pairs, with one class carried by one row only
        y = _labels(rs, R, C, 'pairs')
        y[-1] = C - 1
        y[:-1][y[:-1] == C - 1] = 0
    return y.astype(np.int64)


def _features(rs, R, d, norms):
    F = (np.maximum(rs.standard_normal((R, d)), 0) * rs.uniform(0.5, 3, (R, 1))).astype(np.float32)
    if norms:
        F[0] = 0.0
        F[1] *= np.float32(1e-6 / np.linalg.norm(F[1]))
        F[2] *= np.float32(1e4 / np.linalg.norm(F[2]))
    return F


def _bars(want, mag, d, C, tau):
    """Element bars: the fp32 roundings of the logits (a dot of length d, two norms, a division by tau), carried through
    exp and the sums of length C and R, bounded by u32 (4 d / tau + 2 C + 4 d + 32) times the magnitude the element's
    sums run over; capped at 1e-4 of the tensor's largest element."""
    derived = U32 * (4.0 * d / tau + 2.0 * C + 4.0 * d + 32.0) * mag
    return np.minimum(derived, 1e-4 * np.abs(want).max())


def _magnitudes(F, y, W, tau):
    """|.|-sums of the gradient formulas: what the roundings of each element scale with."""
    F, W = torch.tensor(F, dtype=torch.float64), torch.tensor(W, dtype=torch.float64)
    R, C = F.shape[0], W.shape[0]
    nf, nw = F.norm(dim=1), W.norm(dim=1)
    u, v = F / (nf + 1e-6)[:, None], W / (nw + 1e-6)[:, None]
    onehot = torch.zeros((R, C), dtype=torch.float64)
    onehot[torch.arange(R), torch.tensor(y)] = 1
    g = u @ v.T / tau
    n = onehot.sum(0)
    m = n[None] - onehot
    e = m * torch.exp(g - g.max(1, keepdim=True).values)
    p = e / e.sum(1, keepdim=True)
    a = p + onehot
    du = a @ v.abs() / (tau * R)
    dv = a.T @ u.abs() / (tau * R)
    def through_norm(x, n, g):      # |g| / (n + eps) + |x| <|x|, |g|> / (n (n + eps)^2)
        t = torch.where(n > 0, (x.abs() * g).sum(1) / (n.clamp_min(1e-300) * (n + 1e-6) ** 2), torch.zeros_like(n))
        return 3 * (g / (n + 1e-6)[:, None] + x.abs() * t[:, None])
    return through_norm(F, nf, du).numpy(), through_norm(W, nw, dv).numpy()


CASES = [(2, 160, 10, 0.09, 'pairs', False), (3, 160, 10, 0.07, 'pairs', False), (40, 160, 100, 0.09, 'pairs', True),
         (40, 640, 100, 0.07, 'pairs', False), (40, 2560, 50, 0.09, 'pairs', True), (220, 160, 100, 0.09, 'pairs', True),
         (220, 640, 69, 1.0, 'pairs', False), (220, 2560, 50, 0.07, 'pairs', False),
         (4096, 160, 100, 0.09, 'pairs', True), (4096, 2560, 50, 1.0, 'pairs', False),
         (40, 160, 69, 1.0, 'single', False), (3, 640, 10, 0.09, 'single', False), (220, 2560, 10, 0.07, 'single', True),
         (40, 160, 100, 0.09, 'once', False), (220, 640, 69, 0.07, 'once', True), (2, 2560, 50, 0.09, 'once', False)]


def _call(b, F, y, W, tau, err=None, fill=float('nan')):
    C, d = W.shape
    dW = torch.full((C, d), fill, device='cuda')
    db = torch.full((C,), fill, device='cuda')
    out = b.engine.pcr_loss(torch.tensor(F).cuda(), torch.tensor(y).cuda(), torch.tensor(W).cuda(), tau, dproxies=dW,
                            dbias=db, err=err)
    return out


@pytest.mark.parametrize('R,d,C,tau,pattern,norms', CASES)
def test_pcr_loss_against_fp64(b, R, d, C, tau, pattern, norms):
    rs = np.random.RandomState(R * 7 + d + C)
    F = _features(rs, R, d, norms)
    W = (rs.standard_normal((C, d)) / np.sqrt(d)).astype(np.float32)
    y = _labels(rs, R, C, pattern)
    out = _call(b, F, y, W, tau)
    again = _call(b, F, y, W, tau)
    loss, dF, dW = opcr.loss_and_grads(torch.tensor(F, dtype=torch.float64), torch.tensor(y),
                                       torch.tensor(W, dtype=torch.float64), tau)
    dF, dW = dF.numpy(), dW.numpy()
    got_dF, got_dW = out['dfeats'].cpu().double().numpy(), out['dproxies'].cpu().double().numpy()
    mf, mw = _magnitudes(F, y, W, tau)
    for name, got, want, mag in (('dF', got_dF, dF, mf), ('dW', got_dW, dW, mw)):
        assert np.isfinite(got).all(), name
        bar = _bars(want, mag, d, C, tau)
        worst = float(np.max(np.abs(got - want) / np.maximum(bar, 1e-300)))
        assert worst <= 1.0, (name, worst, float(np.abs(want).max()))
    if pattern == 'once':
        assert torch.isnan(out['loss']).all() and np.isnan(float(loss))
    else:
        bar = min(U32 * (4.0 * d / tau + 64) * float(abs(loss)) + U32 * 8 / tau, 1e-4 * abs(float(loss)))
        assert abs(float(out['loss']) - float(loss)) <= bar, (float(out['loss']), float(loss))
    present = np.zeros(C, bool)
    present[y] = True
    assert torch.equal(out['dproxies'][torch.tensor(~present).cuda()], torch.zeros_like(out['dproxies'][torch.tensor(~present).cuda()]))
    assert torch.equal(out['dbias'], torch.zeros(C, device='cuda'))
    for k in ('loss', 'dfeats', 'dproxies', 'dbias'):
        assert torch.equal(out[k], again[k]) or (k == 'loss' and torch.isnan(out[k]).all() and torch.isnan(again[k]).all()), k


def test_pcr_loss_flags_labels_outside_the_classifier(b):
    rs = np.random.RandomState(3)
    F = _features(rs, 12, 160, False)
    W = (rs.standard_normal((10, 160)) / 13).astype(np.float32)
    y = _labels(rs, 12, 10, 'pairs')
    err = torch.zeros(1, dtype=torch.int32, device='cuda')
    good = _call(b, F, y, W, 0.09, err=err)
    assert int(err) == 0
    bad_y = y.copy()
    bad_y[3] = 10
    bad_y[5] = -1
    out = _call(b, F, bad_y, W, 0.09, err=err)
    torch.cuda.synchronize()
    assert int(err) == 1
    assert torch.equal(out['dfeats'][3], torch.zeros(160, device='cuda'))
    assert torch.equal(out['dfeats'][5], torch.zeros(160, device='cuda'))
    assert torch.isfinite(out['dfeats']).all() and torch.isfinite(out['dproxies']).all()
    assert torch.isfinite(good['loss']).all()


def test_pcr_loss_refusals(b):
    lib = b.native.lib()
    F = torch.ones((4, 160), device='cuda')
    y = torch.zeros(4, dtype=torch.int64, device='cuda')
    W = torch.ones((10, 160), device='cuda')
    loss, dF, dW, db = (torch.empty(1, device='cuda'), torch.empty_like(F), torch.empty_like(W),
                        torch.empty(10, device='cuda'))
    ws = torch.empty(lib.b200ocl_pcr_loss_workspace_bytes(4, 10), dtype=torch.uint8, device='cuda')
    s = torch.cuda.current_stream().cuda_stream
    args = [F.data_ptr(), y.data_ptr(), 4, 160, W.data_ptr(), 10, 0.09, loss.data_ptr(), dF.data_ptr(), dW.data_ptr(),
            db.data_ptr(), None, ws.data_ptr(), ws.numel(), s]
    assert lib.b200ocl_pcr_loss(*args) == 0
    for k in (0, 1, 4, 7, 8, 9, 10):
        bad = list(args)
        bad[k] = None
        assert lib.b200ocl_pcr_loss(*bad) == 1, k                       # B200OCL_EINVAL
    for k, v in ((2, 1), (2, 0), (3, 0), (5, 0), (6, 0.0), (6, -0.1), (6, float('inf')), (6, float('nan'))):
        bad = list(args)
        bad[k] = v
        assert lib.b200ocl_pcr_loss(*bad) == 1, (k, v)
    for k, v in ((2, 4097), (3, 2561), (5, 1025)):
        bad = list(args)
        bad[k] = v
        assert lib.b200ocl_pcr_loss(*bad) == 2, (k, v)                  # B200OCL_EUNSUPPORTED
    bad = list(args)
    bad[13] = ws.numel() - 256
    assert lib.b200ocl_pcr_loss(*bad) == 3                                # B200OCL_EWORKSPACE
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------- the cosine arg-max
@pytest.mark.parametrize('d', [160, 640, 2560])
def test_cosine_argmax_against_fp64(b, d):
    rs = np.random.RandomState(d)
    C = 100
    W = rs.standard_normal((C, d)).astype(np.float32) * rs.uniform(0.1, 10, (C, 1)).astype(np.float32)
    f = np.maximum(rs.standard_normal((600, d)), 0).astype(np.float32)
    f[:200] += 3 * W[rs.randint(0, C, 200)] / np.linalg.norm(W[:1])     # rows with a clear winner
    u = f / (np.linalg.norm(f.astype(np.float64), axis=1, keepdims=True) + 1e-6)
    v = W / (np.linalg.norm(W.astype(np.float64), axis=1, keepdims=True) + 1e-6)
    cos = u @ v.T
    top2 = np.sort(cos, axis=1)[:, -2:]
    keep = (top2[:, 1] - top2[:, 0]) > 1e-5                               # no near ties
    assert keep.sum() >= 500
    f = f[keep]
    want = opcr.cosine_argmax(f, W)
    pred = b.ops.cosine_argmax(torch.tensor(f).cuda(), torch.tensor(W).cuda())
    np.testing.assert_array_equal(pred.cpu().numpy(), want)
    # planted duplicate rows: the lowest index wins
    W2 = W.copy()
    W2[7] = W2[40] = W2[90] = W2[20]
    f2 = np.repeat(W2[20:21], 5, 0) + np.float32(0.01) * rs.standard_normal((5, d)).astype(np.float32)
    pred2 = b.ops.cosine_argmax(torch.tensor(f2).cuda(), torch.tensor(W2).cuda())
    assert pred2.cpu().tolist() == [7] * 5


@pytest.mark.parametrize('d', [160, 640, 2560])
def test_cosine_argmax_counts_hits_exactly(b, d):
    rs = np.random.RandomState(d + 1)
    W = rs.standard_normal((50, d)).astype(np.float32)
    for B in (1, 2, 7, 8, 9, 31, 32, 33, 100, 255, 256, 257):
        f = rs.standard_normal((B, d)).astype(np.float32)
        pred = b.ops.cosine_argmax(torch.tensor(f).cuda(), torch.tensor(W).cuda()).cpu().numpy()
        truth = pred.copy()
        flip = rs.rand(B) < 0.4
        truth[flip] = (truth[flip] + 1) % 50
        hits = torch.full((1,), 5, dtype=torch.int64, device='cuda')
        b.ops.cosine_argmax(torch.tensor(f).cuda(), torch.tensor(W).cuda(), truth=torch.tensor(truth).cuda(),
                            n_correct=hits)
        assert int(hits) == 5 + int((~flip).sum()), (d, B)


# ----------------------------------------------------------------------------- backward from the features
MAPS = [(32, 20), (84, 10), (50, 20), (128, 4)]


@pytest.mark.parametrize('hw,N', MAPS)
def test_backward_from_features_matches_fp64(b, hw, N):
    import test_gpu_backward_fp64 as bw
    probe = oresnet.Spec(hw, 20, 10)
    dim = probe.dim_in
    # a classifier of width dim_in set to the identity: the existing fp64 restatement's dout @ W is then dF itself
    spec = oresnet.Spec(hw, 20, dim)
    params, bn = oresnet.seeded_state(spec, 5 + hw)
    params['linear.weight'] = torch.eye(dim)
    params['linear.bias'] = torch.zeros(dim)
    eng = b.engine.Engine(hw, dim)
    eng.load(list(params.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
    gen = torch.Generator().manual_seed(hw * 100 + N)
    x = torch.rand(N, 3, hw, hw, generator=gen).cuda()
    dF = (torch.randn(N, dim, generator=gen) * 0.1).cuda()
    ws = eng.new_train_workspace(N)
    feat, _ = eng.forward_train(x, ws=ws, features=True)
    assert feat.shape == (N, dim)
    (wo, wn, _), (bo, bn_, _) = eng.table[-2], eng.table[-1]
    for accumulate in (False, True):
        eng.state.grads.fill_(float('nan') if not accumulate else 0.0)
        eng.state.grads[wo:bo + bn_] = 1.5                                 # the linear.* entries: left as they are
        eng.backward(x, dF, ws, accumulate=accumulate, features=True)
        got = eng.state.grads.clone()
        assert torch.equal(got[wo:bo + bn_], torch.full((wn + bn_,), 1.5, device='cuda')), accumulate
    R = bw.reference(b.engine, eng, spec, ws, N, x, dF, False)
    rows = []
    leaves = OrderedDict((k, v.double().requires_grad_(True)) for k, v in params.items())
    bn64 = OrderedDict((k, v.double() if v.is_floating_point() else v.clone()) for k, v in bn.items())
    f64 = oresnet.features(spec, leaves, bn64, x.cpu().double(), train=True)
    f64.backward(dF.cpu().double())
    worst_auto = 0.0
    for (name, shape), (o, n, _) in list(zip(oresnet.param_shapes(spec).items(), eng.table))[:-2]:
        g = got[o:o + n].double().cpu()
        ref, share = R[name]
        scale = float(ref.abs().max())
        err = float((g - ref.reshape(-1).cpu()).abs().max()) / scale
        rows.append((name, bw.kind(name, shape), err, float(share.abs().max()) / scale))
        auto = leaves[name].grad.reshape(-1)
        worst_auto = max(worst_auto, float((g - auto).abs().max() / auto.abs().max()))
    bw.check(rows, N)
    # independent fp64 autograd: a pre-activation within fp32 rounding of zero may take the other ReLU branch there,
    # which moves single weights by a few percent of their tensor's largest entry (5.8e-2 measured at 84x84, N = 10,
    # on an H100 80GB HBM3 at 700 W) while the restatement above, through the engine's own masks, holds the 3e-5 bars
    assert worst_auto < 0.2, worst_auto
    # the features the forward exposed are the fp64 forward's
    assert float((feat.double().cpu() - f64.detach()).abs().max() / f64.detach().abs().max()) < 1e-4


# ----------------------------------------------------------------------------- the learner
def make_params(**kw):
    base = dict(data='cifar100', cuda=True, epoch=1, batch=10, verbose=False, mem_size=30, eps_mem_batch=10,
                mem_iters=1, update='random', retrieve='random', agent='PCR', k=3, aser_type='asvm', n_smp_cls=1.5,
                num_tasks=5, buffer_tracker=False, optimizer='SGD', learning_rate=0.05, weight_decay=0, temp=0.07,
                head='mlp', subsample=20, error_analysis=False, pcr_temp=0.09,
                trick={'labels_trick': False, 'kd_trick': False, 'separated_softmax': False, 'review_trick': False,
                       'ncm_trick': False, 'kd_trick_star': False})
    base.update(kw)
    return SimpleNamespace(**base)


class _Transform(torch.nn.Module):
    def __init__(self, fn):
        super().__init__()
        self.fn = fn

    def forward(self, x):
        return self.fn(x)


def _identity(agent):
    agent.transform = _Transform(lambda t: t.detach().to(torch.float32).clone())


def _recording(agent):
    """Keep every augmented view the engine's transform returns, in call order."""
    seen = []
    tf = agent.transform

    def wrapped(t):
        out = tf(t)
        seen.append(out.cpu().double())
        return out
    agent.transform = _Transform(wrapped)
    return seen


def _steps_against_oracle(b, data, n_steps, seed, own_aug=False, adam=False, **kw):
    params = make_params(data=data, **kw)
    opt = (lambda m: torch.optim.Adam(m.parameters(), lr=params.learning_rate,
                                      weight_decay=params.weight_decay)) if adam else None
    agent, spec = _learner(params, seed, opt=opt)
    if own_aug:
        seen = _recording(agent)
    else:
        _identity(agent)
    hw, ncls = HW[data], NCLS[data]
    p64, bn64 = oresnet.seeded_state(spec, seed, dtype=torch.float64)
    st = opcr.ors.ReplayState(spec, p64, bn64, params.mem_size, (3, hw, hw), ncls, lr=params.learning_rate,
                              weight_decay=params.weight_decay)
    ad = oagem.AdamState(params.learning_rate, weight_decay=params.weight_decay) if adam else None
    agent.model.train()
    rs = np.random.RandomState(seed + 1)
    stepped = 0
    for i in range(n_steps):
        x = torch.tensor(rs.randint(0, 256, (10, 3, hw, hw)).astype(np.float32) / 255.0)
        y = torch.tensor(rs.randint(0, 5, 10))
        before = agent.engine.state.params.clone()
        agent.last_loss = None
        if own_aug:
            seen.clear()
        np.random.seed(100 + i); torch.manual_seed(100 + i)
        agent.replay_step(x.cuda(), y.cuda(), y.numpy())
        torch.cuda.synchronize()
        views = iter(list(seen)) if own_aug else None
        np.random.seed(100 + i); torch.manual_seed(100 + i)
        logs = opcr.step(st, x, y, eps_mem_batch=params.eps_mem_batch, mem_iters=params.mem_iters,
                         temperature=params.pcr_temp, transform=(lambda t: next(views)) if own_aug else None,
                         adam=ad)
        where = (data, i, kw)
        ran = [lg for lg in logs if lg['loss'] is not None]
        if not ran:                                                     # an empty memory: nothing ran, nothing moved
            assert agent.last_loss is None and torch.equal(agent.engine.state.params, before), where
        else:
            stepped += 1
            assert abs(float(agent.last_loss) - ran[-1]['loss']) < 2e-4 * abs(ran[-1]['loss']), \
                (where, float(agent.last_loss), ran[-1]['loss'])
        flat = torch.cat([v.reshape(-1) for v in st.params.values()])
        got = agent.engine.state.params.cpu().double()
        if adam and ran:
            # Adam's first step moves every element by about lr whatever the gradient's size, so an element whose
            # gradient is near zero is ill-conditioned there: the gradient is held through exp_avg = (1 - beta1) g,
            # and the step only to its bound lr.  Against the independent fp64 forward a ReLU can flip, so the
            # gradient's bar is on the whole arena's largest entry (6.6e-4 measured, H100 80GB HBM3, 700 W)
            g_want = torch.cat([v.reshape(-1) for v in ran[-1]['grads'].values()])
            g_got = agent.engine.adam_state().exp_avg.cpu().double() / 0.1
            err = float((g_got - g_want).abs().max() / g_want.abs().max())
            assert err < 2e-3, (where, err)
            assert float((got - flat).abs().max()) <= 2.001 * params.learning_rate, where
        elif not adam:
            err = float((got - flat).abs().max() / flat.abs().max())
            assert err < 2e-4, (where, err)
        bn_got = agent.engine.state.bn_stats.cpu().double()
        bn_want = torch.cat([torch.cat((st.bn[n + '.running_mean'], st.bn[n + '.running_var']))
                             for n in oresnet.bn_names(spec)])
        assert float((bn_got - bn_want).abs().max() / bn_want.abs().max()) < 1e-4, where
        np.testing.assert_array_equal(agent.buffer.buffer_label.cpu().numpy(), st.buffer_label.numpy())
        assert torch.equal(agent.buffer.buffer_img.cpu(), st.buffer_img), where
        if not adam:
            _load(agent, st.params, st.bn, spec)                       # the next step starts from the oracle's state
    assert agent.buffer.n_seen_so_far == st.n_seen_so_far == 10 * n_steps
    return stepped


@pytest.mark.parametrize('data', ['cifar100', 'mini_imagenet', 'openloris', 'core50'])
def test_steps_against_oracle(b, data):
    assert _steps_against_oracle(b, data, 4 if data != 'core50' else 3, 301) >= 2


def test_steps_against_oracle_with_the_engines_augmented_images(b):
    assert _steps_against_oracle(b, 'cifar100', 4, 302, own_aug=True) == 3


@pytest.mark.parametrize('kw', [dict(mem_iters=2), dict(eps_mem_batch=25), dict(weight_decay=1e-2),
                                dict(adam=True, optimizer='Adam', learning_rate=1e-3)],
                         ids=['mem_iters2', 'small_memory', 'weight_decay', 'adam'])
def test_step_variants_against_oracle(b, kw):
    kw = dict(kw)
    adam = kw.pop('adam', False)
    assert _steps_against_oracle(b, 'cifar100', 2 if adam else 4, 303, adam=adam, **kw) == (1 if adam else 3)


def _task(rs, n, labels, hw):
    x = rs.randint(0, 256, (n, hw, hw, 3)).astype(np.uint8)
    return x, rs.choice(np.asarray(list(labels)), n)


@pytest.mark.parametrize('data', ['cifar100', 'core50'])
def test_two_task_run_accuracy_is_the_fp64_cosine_argmax(b, data):
    params = make_params(data=data, mem_size=40)
    agent, _ = _learner(params, 9)
    hw = HW[data]
    rs = np.random.RandomState(3)
    labels = [range(0, 5), range(5, 10)]
    loaders = []
    for labs in labels:
        x, y = _task(rs, 50, labs, hw)
        loaders.append([(torch.from_numpy(x).permute(0, 3, 1, 2).float().div(255), torch.from_numpy(y))])
    for labs in labels:
        agent.train_learner(*_task(rs, 42, labs, hw))
        acc = agent.evaluate(loaders)
    torch.cuda.synchronize()
    eng = agent.engine
    (wo, wn, _), (_, bn_, _) = eng.table[-2], eng.table[-1]
    W = eng.state.params[wo:wo + wn].view(bn_, -1).cpu().double().numpy()
    for t, loader in enumerate(loaders):
        (x, y), = loader
        f = eng.features_eval(x.cuda()).cpu().double().numpy()
        pred = opcr.cosine_argmax(f, W)
        u = f / (np.linalg.norm(f, axis=1, keepdims=True) + 1e-6)
        v = W / (np.linalg.norm(W, axis=1, keepdims=True) + 1e-6)
        top2 = np.sort(u @ v.T, axis=1)[:, -2:]
        near = int(((top2[:, 1] - top2[:, 0]) < 1e-6).sum())
        hits = int((pred == y.numpy()).sum())
        assert abs(round(acc[t] * len(y)) - hits) <= near, (t, acc[t], hits, near)
        assert near == 0 or data == 'core50', (t, near)
    assert agent.buffer.current_index == 40 and agent.buffer.n_seen_so_far == 80       # full batches only


def test_error_analysis_is_refused_before_anything_launches(b):
    agent, _ = _learner(make_params(error_analysis=True), 9)
    before = b.native.launch_count()
    with pytest.raises(b.learners.ErrorAnalysisUnsupported):
        agent.evaluate([[(torch.zeros(2, 3, 32, 32), torch.zeros(2, dtype=torch.int64))]])
    assert b.native.launch_count() == before
