"""GPU: b200ocl_supcon against the float64 oracle (oracle/supcon.py) at every launch it can take on the card in use.

b200ocl_supcon picks one of 16 kernel instantiations (csrc/supcon.cu, supcon_plan): the fused kernel with the whole
contrast set resident, with a two-slot ring of 16-anchor units or of 64-anchor units (each with NC = 1..4 float4
columns per thread), or the stats + grad<DCH> fallback (DCH = 4/8/16/32).  Which one a shape reaches depends on the SM
count, so the cases are built from the device's SM count and test_cases_reach_every_launch checks, through the
host-only hook b200ocl_supcon_plan, that they reach every (family, NC / DCH) pair the hook reports for A <= 10 000 and
d <= 1024 on this card.

Bars, about 3x the largest error measured on an H100 80GB HBM3 (SXM, 132 SMs, 700 W power limit) over these cases:
  loss      |loss - loss64| / max(|loss64|, Lmax)                  LOSS_TOL  [measured in brackets]
  gradient  max |grad - grad64| / max(max |grad64|, Cmax / (A T))  GRAD_TOL
Lmax = max |c|^2 / T and Cmax / (A T) = max |c| / (A T) are the scales fp32 rounding is relative to (see scales()): a
loss or gradient that nearly cancels, as SCR's pairs layout does once its views agree, would otherwise turn a rounding
of the logits into a large relative error.  Each case also checks that its bars could see a dropped contrast row: the
fp64 loss and gradient with the last anchor left out of every contrast set (oracle drop_last_contrast) move by at least
10x the bar, in the same units."""
import numpy as np
import pytest
import torch

from oracle import supcon as osup

pytestmark = pytest.mark.gpu

LOSS_TOL = 4e-8        # [1.2e-8, fallback DCH = 32 at A = 3; the fused kernels <= 5.4e-9]
GRAD_TOL = 5e-5        # [1.5e-5, ring64 NC = 3 at A = 8449; resident <= 1.0e-6, fallback <= 4.6e-6]
A_MAX, D_MAX = 10000, 1024


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import ops as _ops
    return _ops


def device_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def reachable(ops, sms):
    """Every (family, NC / DCH) the hook reports for A <= A_MAX, d <= D_MAX, aligned or not."""
    out = set()
    for d in range(4, 257, 4):
        for A in list(range(1, 16 * sms + 2)) + [64 * sms + 1, A_MAX]:
            out.add(ops.supcon_plan(A, 1, d, True, sms).kernel)
    for d in range(1, D_MAX + 1):
        out.add(ops.supcon_plan(1, 1, d, False, sms).kernel)
    return out


def labels_for(kind, B, rs):
    if kind == 'pairs':                 # each anchor's only positive is its other view(s)
        return np.arange(B)
    if kind == 'one':
        return np.zeros(B, dtype=np.int64)
    per = 2 if kind == 'many' else 8    # at least two ('many') or eight ('few') samples per class, shuffled
    return rs.permutation(np.arange(B) % max(1, B // per))


def case_list(sms):
    """(tag, B, V, d, T, label kind, feature norm, misaligned)."""
    cases = [
        # SCR's own calls: the mlp head (d = 128), head 'None' at 32x32 (160) and 84x84 (640), batches of 10 / 100
        ('scr-mlp', 110, 2, 128, 0.07, 'few', 1.0, False),
        ('scr-mlp-small', 11, 2, 128, 0.07, 'pairs', 1.0, False),
        ('scr-none-32', 110, 2, 160, 0.07, 'few', 1.0, False),
        ('scr-none-84', 110, 2, 640, 0.07, 'few', 1.0, False),
        # the fallback at every DCH, V = 1 / 2 / 3, ragged d
        ('fb4', 40, 2, 33, 0.1, 'many', 1.0, False),
        ('fb8', 43, 3, 201, 0.05, 'few', 3.0, False),
        ('fb16', 65, 1, 300, 0.05, 'one', 3.0, False),
        ('fb32', 3, 1, 1024, 1.0, 'one', 1.0, False),
        # a float32 view one element into its storage: not 16-byte aligned, so the fallback takes a fused shape
        ('misaligned-128', 110, 2, 128, 0.07, 'few', 1.0, True),
        ('misaligned-256', 33, 3, 256, 0.05, 'pairs', 3.0, True),
    ]
    for nc in (1, 2, 3, 4):
        d_full, d_ragged = 64 * nc, 64 * nc - 4
        # resident: A = 65 and 129 (ragged against the 16-anchor unit and the 64-row tile)
        cases.append(('res-nc%d' % nc, 65, 1, d_ragged, 0.05, 'many', 3.0, False))
        cases.append(('res-nc%d-v3' % nc, 43, 3, d_full, 0.07, 'pairs', 1.0, False))
        # ring of 16-anchor units: the largest A that still takes it, A = 1 mod 16
        cases.append(('ring16-nc%d' % nc, 16 * sms - 15, 1, d_full, 0.05, 'few', 3.0, False))
        # ring of 64-anchor units with a second unit on CTA 0, A = 1 mod 64
        cases.append(('ring64-nc%d' % nc, 64 * sms + 1, 1, d_ragged, 0.05, 'few', 3.0, False))
    cases.append(('ring64-v2-pairs', 32 * sms + 1, 2, 128, 0.07, 'pairs', 1.0, False))
    return cases


def make_inputs(case, seed):
    tag, B, V, d, T, kind, norm, misaligned = case
    rs = np.random.RandomState(seed)
    y = labels_for(kind, B, rs)
    if V == 1 and kind == 'few':
        y[0] = y[-1] = y.max() + 1       # a class of two: the last contrast row is the first anchor's only positive
    # a cluster per class, as trained SupCon features are: at |c| = 3 and T = 0.05 the diagonal logit is ~180 and the
    # positives sit within ~40 of it, so exp(l - max) stays in fp32 range (random directions would underflow it)
    centers = rs.standard_normal((int(y.max()) + 1, d))
    centers /= np.linalg.norm(centers, axis=1, keepdims=True)
    f = centers[y][:, None, :] + 0.3 * rs.standard_normal((B, V, d)) / np.sqrt(d)
    f = norm * f / np.linalg.norm(f, axis=2, keepdims=True) * rs.uniform(0.97, 1.03, (B, V, 1))
    f = f.astype(np.float32)
    if misaligned:
        store = torch.empty(B * V * d + 1, dtype=torch.float32, device='cuda')
        ft = store[1:].view(B, V, d)
        ft.copy_(torch.from_numpy(f))
    else:
        ft = torch.from_numpy(f).cuda()
    return f, y, ft, torch.from_numpy(y).cuda()


def plan_of(ops, case, ft):
    tag, B, V, d = case[:4]
    return ops.supcon_plan(B, V, d, ft.data_ptr() % 16 == 0, 0)


def scales(f, T):
    """The sizes fp32 rounding is relative to: the loss is a mean of lse_i - mean_P l_ij, differences of logits up to
    Lmax = max |c|^2 / T; each gradient row is (1 / (A T)) sum_j W_ij c_j with sum_j |W_ij| <= 4."""
    B, V = f.shape[:2]
    c2 = float((f.astype(np.float64) ** 2).sum(2).max())
    return c2 / T, np.sqrt(c2) / (B * V * T)


def errors(loss, grad, ref_loss, ref_grad, lscale, gscale):
    le = abs(float(loss) - ref_loss) / max(abs(ref_loss), lscale)
    ge = float((grad.double() - ref_grad).abs().max()) / max(float(ref_grad.abs().max()), gscale)
    return le, ge


def test_cases_reach_every_launch(ops):
    sms = device_sms()
    want = reachable(ops, sms)
    got = {}
    for i, case in enumerate(case_list(sms)):
        _, _, ft, _ = make_inputs(case, i)
        got.setdefault(plan_of(ops, case, ft).kernel, []).append(case[0])
    print('sms %d: %s' % (sms, sorted(got.items())))
    assert want <= set(got), sorted(want - set(got))
    for case in case_list(sms):
        if case[0].startswith('ring64'):
            assert ops.supcon_plan(*case[1:4], True, sms).units_per_cta >= 2, case
    for tag, want_kernel in [('scr-mlp', ('resident', 2)), ('scr-mlp-small', ('resident', 2)),
                             ('scr-none-32', ('resident', 3)), ('scr-none-84', ('fallback', 32)),
                             ('misaligned-128', ('fallback', 4)), ('misaligned-256', ('fallback', 8))]:
        assert tag in got.get(want_kernel, []), (tag, want_kernel)


@pytest.mark.parametrize('idx', range(len(case_list(132))))        # the same number of cases on every SM count
def test_supcon_against_fp64(ops, idx):
    case = case_list(device_sms())[idx]
    tag, B, V, d, T = case[:5]
    f, y, ft, yt = make_inputs(case, idx)
    L = plan_of(ops, case, ft)
    loss, grad = ops.supcon(ft, yt, T)
    loss2, grad2 = ops.supcon(ft, yt, T)
    loss3, none = ops.supcon(ft, yt, T, need_grad=False)
    f64 = torch.from_numpy(f).cuda()
    ref_loss, ref_grad = osup.supcon_loss_and_grad_torch(f64, yt, T)
    drop_loss, drop_grad = osup.supcon_loss_and_grad_torch(f64, yt, T, drop_last_contrast=True)
    lscale, gscale = scales(f, T)
    le, ge = errors(loss, grad, ref_loss, ref_grad, lscale, gscale)
    dl, dg = errors(torch.tensor(drop_loss), drop_grad, ref_loss, ref_grad, lscale, gscale)
    dl = dl if np.isfinite(dl) else np.inf
    dg = dg if np.isfinite(dg) else np.inf
    print('supcon %-16s A=%5d d=%4d %-14s loss %.3g grad %.3g | drop-last moves loss %.3g grad %.3g'
          % (tag, B * V, d, '%s/%d' % L.kernel, le, ge, dl, dg))
    # bits: repeated calls, and the loss without the gradient pass (another barrier placement in the fused kernel)
    bits = lambda t: t.view(torch.int32)
    assert torch.equal(bits(loss), bits(loss2)) and torch.equal(bits(grad), bits(grad2)), tag
    assert none is None and torch.equal(bits(loss), bits(loss3)), tag
    assert le <= LOSS_TOL, (tag, le)
    assert ge <= GRAD_TOL, (tag, ge)
    # the bars would see a missing contrast row
    assert dl >= 10 * LOSS_TOL, (tag, dl)
    assert dg >= 10 * GRAD_TOL, (tag, dg)


def test_anchor_without_positives(ops):
    """V = 1 with a class of one sample: the loss is NaN (loss.py:90) and the gradient is finite, with that anchor's
    positive term taken as 0 (the contract in supcon.cu / b200ocl.h), on every family."""
    sms = device_sms()
    seen = set()
    for i, (B, d, misaligned) in enumerate([(40, 128, False), (16 * sms - 15, 64, False), (64 * sms + 1, 128, False),
                                            (40, 128, True), (40, 640, False)]):
        case = ('singleton', B, 1, d, 0.1, 'few', 1.0, misaligned)
        f, y, ft, yt = make_inputs(case, 100 + i)
        y[B // 2] = 10 ** 6                       # a class nobody else has
        yt = torch.from_numpy(y).cuda()
        seen.add(plan_of(ops, case, ft).name)
        loss, grad = ops.supcon(ft, yt, 0.1)
        assert torch.isnan(loss).all(), B
        assert bool(torch.isfinite(grad).all()), (B, d, misaligned)
        _, ref = osup.supcon_loss_and_grad_torch(torch.from_numpy(f).cuda(), yt, 0.1, finite_grad=True)
        _, nan_ref = osup.supcon_loss_and_grad_torch(torch.from_numpy(f).cuda(), yt, 0.1)
        assert bool(torch.isnan(nan_ref).all())    # what autograd on the reference gives
        _, err = errors(0.0, grad, 1.0, ref, 1.0, scales(f, 0.1)[1])
        assert err <= GRAD_TOL, (B, d, misaligned, err)
    assert seen == {'resident', 'ring16', 'ring64', 'fallback'}, seen
