"""GPU: the classification-loss kernels against fp64 at every shape the agents feed them, every row compared.

b200ocl_ce_loss (ce_kernel, csrc/net_fwd.cu) is the criterion of ER, MIR, ASER, A-GEM, GSS and GDumb whenever no trick
and no teacher is in force, and MIR orders its memory subsample by the difference of two of its per-sample vectors.  It
runs one CTA of 8 warps: row n is taken by warp n % 8, whose lanes stride the C columns by 32 and reduce the maximum,
the arg-max (ties to the lowest index, across lanes by a butterfly) and z = sum exp(x - mx) through 5 shuffle levels.
The sweep crosses N in {1, 7, 8, 9, 63, 64, 65, 110, 220, 1000, 4096} (warps with no row, one row and several; MIR
subsamples up to ops.RANK_MAX) with C in {1, 2, 10, 31, 32, 33, 50, 64, 100, 1000, 1024, 1025} (lanes with no column, a
partial last stride, CORe50's 50 classes, the 100-class heads), at logit scales 0.01, 1, 30 and 100, with one dominant
logit per row and with planted arg-max ties, labels at columns 0 and C - 1 included.  Output buffers start as NaN, so an
element the kernel leaves unwritten fails.

Bounds (u = 2^-24, gamma_n = n u / (1 - n u), K = ceil(C / 32)).  The library is built without fast-math: expf is within
2 ulp and logf within 1 ulp.  Per row, with mx the row maximum, x_y the target logit, lz = log z, lse = mx + lz and
l = (mx - x_y) + lz, all in fp64 from the same fp32 logits:
  z        a term carries the rounding of x - mx (relative u |x - mx| after exp, and sum_c t_c |log t_c| <= z ln C) and
           of expf (4u); the sum has depth K + 5 (K strided terms per lane, 5 butterfly levels).  So z~ = z (1 + t) with
           |t| <= theta = gamma_(K+5) + (4 + ln C) u;
  loss     per_sample = fl(fl(mx - x_y) + logf(z~)):  |l~ - l| <= u |mx - x_y| + theta + 2u |lz| + u |l|;
  dlogits  fl(fl(expf(fl(x_c - lse~)) - [c = y]) * fl(1/N)), lse~ = fl(mx + logf(z~)) within E = u (|mx| + 3 |lz|) + theta
           of lse:  |d~ - d| <= (p_c (E + u |x_c - lse| + 4u) + 3u |p_c - [c = y]|) / N, plus 2^-146 for results below
           the normal range;
  mean     |L~ - L| <= mean_n (bound of l_n) + (gamma_(ceil(N/8)+8) + u) L (the rows of a warp, the 8 warps, 1/N);
  sum      each dlogits row sums to 0 within the sum of its element bounds.
These are first-order bounds; the tests hold twice them (SLACK), which covers the second-order terms many times over.

The per-sample bound has no |mx| or |x_y| term.  The kernel used to form fl(fl(mx + lz) - x_y), which rounds lse first:
on rows whose target is the maximum at mx = 30..100 (losses down to 1e-10) that costs up to ulp(mx) / 2 = 3.8e-6
absolute, and on an H100 it missed this bound by up to 3.0x (rows like those of
test_ce_per_sample_keeps_small_losses_at_large_logits; 3.9e-6 absolute at mx = 100).  (mx - x_y) + lz keeps them within
0.16 of it [0.163, C = 50; 8.1e-7 absolute at most, C = 1025].

Every error is also held to a bar about 3x the largest value measured on an H100 80GB HBM3 (SXM, 700 W power limit)
over these cases [in brackets], in units of u times the row's magnitudes:
  per_sample  |l~ - l| / (u (1 + |mx - x_y| + |lz| + |l|))
  dlogits     |d~ - d| / max(u (p_c (1 + |lse| + |x_c - lse|) + |p_c - [c = y]|) / N, 2^-140)
  loss        |L~ - L| / (u (mean_n (1 + |mx - x_y| + |lz| + |l|) + (ceil(N/8) + 8) L))
  row sum     |sum_c d~_c| / (u sum_c (p_c (1 + |lse| + |x_c - lse|) + |p_c - [c = y]|) / N)
n_correct must equal numpy's first-maximum count exactly, and ce_loss and cls_loss(mode='ce', w_ce=1, no teacher) give
the same bits, as they perform the same operations.

The siblings cls_loss (labels trick, separated softmax, distillation) and icarl_loss are run at the same N / C edges
against oracle.tricks.criterion and oracle.icarl.icarl_loss with the tolerances of test_gpu_tricks.py and
test_gpu_icarl.py, plus separated-softmax segments of length 1, 32 and 33 and the labels trick at B200OCL_CLS_MAX_C."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import test_gpu_icarl as gicarl
import test_gpu_tricks as gtricks

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SLACK = 2.0
TINY = 2.0 ** -140
CLS_MAX_C = 12288                 # B200OCL_CLS_MAX_C

PS_BAR = 40.0          # per_sample, units above       [13.6, cancellation rows C = 1025; sweep 8.44, N = 110, C = 1024]
DL_BAR = 7.0           # dlogits                       [2.34, N = 63, C = 1024]
LOSS_BAR = 4.0         # mean loss                     [1.32, cancellation rows C = 1025; sweep 0.378, N = 1, C = 2]
SUM_BAR = 3.5          # dlogits row sum               [1.14, cancellation rows C = 1025; sweep 1.11, N = 4096]

N_SET = [1, 7, 8, 9, 63, 64, 65, 110, 220, 1000, 4096]
C_SET = [1, 2, 10, 31, 32, 33, 50, 64, 100, 1000, 1024, 1025]
REGIMES = ['0.01', '1', '30', '100', 'dominant', 'ties']


@pytest.fixture(scope='module')
def native():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import _native
    return _native


def gamma(n):
    return n * U / (1 - n * U)


def bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def make_case(N, C, regime, seed):
    """fp32 logits [N,C] and int64 labels [N]; labels 0 and C - 1 at the first and last rows."""
    rs = np.random.RandomState(seed)
    rows = np.arange(N)
    if regime == 'dominant':
        x = rs.standard_normal((N, C)) * 3
        dom = rs.randint(0, C, N)
        x[rows, dom] += rs.uniform(20, 60, N)
        y = np.where(rs.rand(N) < 0.5, dom, rs.randint(0, C, N))
    elif regime == 'ties':
        x = np.round(rs.standard_normal((N, C)) * 4) / 4            # quarter steps: natural ties as well
        y = rs.randint(0, C, N)
        if C >= 2:
            for n in range(N):
                if n % 3 == 1 and C > 32:                            # c and c + 32k: the same lane
                    c = rs.randint(0, C - 32)
                    partner = c + 32 * rs.randint(1, (C - 1 - c) // 32 + 1)
                else:                                                # c and c + 1: neighbouring lanes
                    c = rs.randint(0, C - 1)
                    partner = c + 1
                x[n, c] = x[n, partner] = x[n].max() + 1
                y[n] = (c, partner, y[n])[(n // 3) % 3]
    else:
        x = rs.standard_normal((N, C)) * float(regime)
        y = rs.randint(0, C, N)
    y[0], y[-1] = 0, C - 1
    return x.astype(np.float32), y.astype(np.int64)


def reference(x, y, n_div=None):
    """fp64 values and per-element bounds (module docstring) of the rows of x at labels y; n_div: the N of the mean."""
    x64 = x.astype(np.float64)
    N, C = x.shape
    n_div = N if n_div is None else n_div
    rows = np.arange(N)
    mx = x64.max(1)
    e = np.exp(x64 - mx[:, None])
    z = e.sum(1)
    lz = np.log(z)
    lse = mx + lz
    xy = x64[rows, y]
    l = (mx - xy) + lz
    p = e / z[:, None]
    delta = np.zeros_like(p)
    delta[rows, y] = 1.0
    d = (p - delta) / n_div
    theta = gamma(-(-C // 32) + 5) + (4 + math.log(C)) * U
    bl = SLACK * (U * np.abs(mx - xy) + theta + 2 * U * np.abs(lz) + U * np.abs(l))
    E = U * (np.abs(mx) + 3 * np.abs(lz)) + theta
    dist = np.abs(x64 - lse[:, None])
    bd = SLACK * (p * (E[:, None] + U * dist + 4 * U) + 3 * U * np.abs(p - delta)) / n_div + 2.0 ** -146
    ml = 1 + np.abs(mx - xy) + np.abs(lz) + np.abs(l)
    md = (p * (1 + np.abs(lse)[:, None] + dist) + np.abs(p - delta)) / n_div
    return SimpleNamespace(l=l, d=d, bl=bl, bd=bd, ml=ml, md=md, mx=mx, lz=lz)


def loss_bound(ref, n_div):
    L = ref.l.sum() / n_div
    return ref.bl.sum() / n_div + SLACK * (gamma(-(-n_div // 8) + 8) + U) * L, L


def raw_ce(native, xt, yt, loss=True, per_sample=True, dlogits=True, n_correct=True, err=None):
    """b200ocl_ce_loss into NaN-filled (n_correct: -1) outputs; a False output is passed as NULL."""
    N, C = xt.shape
    nan = float('nan')
    out = {'loss': torch.full((1,), nan, device='cuda') if loss else None,
           'per_sample': torch.full((N,), nan, device='cuda') if per_sample else None,
           'dlogits': torch.full((N, C), nan, device='cuda') if dlogits else None,
           'n_correct': torch.full((1,), -1, dtype=torch.int64, device='cuda') if n_correct else None}
    p = lambda t: 0 if t is None else t.data_ptr()
    rc = native.lib().b200ocl_ce_loss(p(xt), p(yt), N, C, p(out['loss']), p(out['per_sample']), p(out['dlogits']),
                                      p(out['n_correct']), p(err), torch.cuda.current_stream().cuda_stream)
    native.check(rc, 'b200ocl_ce_loss')
    return out


def same_bits(a, b, where):
    for k in a:
        if a[k] is not None and b.get(k) is not None:
            assert torch.equal(bits(a[k]), bits(b[k])), (where, k)


def measure(out, x, y, ref, where):
    """Check every output of one launch against fp64; returns the errors in bar units."""
    N = x.shape[0]
    ps = out['per_sample'].cpu().numpy().astype(np.float64)
    el = np.abs(ps - ref.l)
    assert bool((el <= ref.bl).all()), (where, 'per_sample', np.flatnonzero(~(el <= ref.bl))[:8].tolist())
    dl = out['dlogits'].cpu().numpy().astype(np.float64)
    ed = np.abs(dl - ref.d)
    assert bool((ed <= ref.bd).all()), (where, 'dlogits', np.argwhere(~(ed <= ref.bd))[:8].tolist())
    rsum = np.abs(dl.sum(1))
    assert bool((rsum <= ref.bd.sum(1) + x.shape[1] * 2.0 ** -53 * np.abs(dl).sum(1)).all()), (where, 'row sum')
    bL, L = loss_bound(ref, N)
    eL = abs(float(out['loss']) - L)
    assert eL <= bL, (where, 'loss', float(out['loss']), L, bL)
    want_hits = int((np.argmax(x, axis=1) == y).sum())             # numpy: the first maximum
    assert int(out['n_correct']) == want_hits, (where, int(out['n_correct']), want_hits)
    r = dict(ps=float((el / (U * ref.ml)).max()),
             dl=float((ed / np.maximum(U * ref.md, TINY)).max()),
             loss=eL / (U * (ref.ml.mean() + (-(-N // 8) + 8) * L)),
             sum=float((rsum / np.maximum(U * ref.md.sum(1), TINY)).max()))
    assert r['ps'] <= PS_BAR and r['dl'] <= DL_BAR and r['loss'] <= LOSS_BAR and r['sum'] <= SUM_BAR, (where, r)
    return r


@pytest.mark.parametrize('C', C_SET)
@pytest.mark.parametrize('N', N_SET)
def test_ce_loss_against_fp64(native, N, C):
    from b200ocl.engine import ce_loss, cls_loss
    worst = {}
    for k, regime in enumerate(REGIMES):
        where = (N, C, regime)
        x, y = make_case(N, C, regime, 1000 * N + 10 * C + k)
        xt, yt = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
        err = torch.zeros(1, dtype=torch.int32, device='cuda')
        full = raw_ce(native, xt, yt, err=err)
        r = measure(full, x, y, reference(x, y), where)
        worst = {q: max(worst.get(q, 0.0), v) for q, v in r.items()}
        assert int(err) == 0, where
        # repeat launches, the Python wrapper and cls_loss(mode='ce'): the same bits
        same_bits(raw_ce(native, xt, yt), full, where + ('repeat',))
        api = ce_loss(xt, yt, want_per_sample=True, want_correct=True, err=err)
        same_bits(api, full, where + ('ce_loss',))
        cls = cls_loss(xt, yt, 'ce', teacher=None, w_ce=1.0, w_kd=0.0, err=err, want_correct=True)
        same_bits(cls, full, where + ('cls_loss ce',))
        assert int(err) == 0, where
        if regime == '1':
            # every combination of requested and NULL outputs: requesting one does not change the bits of another
            for mask in range(16):
                want = dict(loss=bool(mask & 1), per_sample=bool(mask & 2), dlogits=bool(mask & 4),
                            n_correct=bool(mask & 8))
                same_bits(raw_ce(native, xt, yt, **want), full, where + (want,))
    torch.cuda.synchronize()
    print('ce N=%5d C=%5d  per_sample %.3g  dlogits %.3g  loss %.3g  row sum %.3g'
          % (N, C, worst['ps'], worst['dl'], worst['loss'], worst['sum']))


@pytest.mark.parametrize('C', [2, 10, 50, 100, 1025])
def test_ce_per_sample_keeps_small_losses_at_large_logits(native, C):
    """Rows whose target is the maximum at mx = 30..100, the others 5..12 + ln C below it: losses from about 1e-10 to 1e-2,
    where fl(lse) - x_y would lose up to ulp(mx) / 2 to cancellation.  Held to the per-sample bound, which has no |mx|
    term: a few u relative to the loss plus the summation floor gamma_(K+5)."""
    N = 1000
    rs = np.random.RandomState(C)
    mx0 = rs.uniform(30, 100, N)
    x = mx0[:, None] - (rs.uniform(5, 12, N) + math.log(C))[:, None] - rs.exponential(2.0, (N, C))
    y = rs.randint(0, C, N)
    x[np.arange(N), y] = mx0
    x = x.astype(np.float32)
    xt, yt = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    out = raw_ce(native, xt, yt)
    ref = reference(x, y)
    assert bool((ref.mx == x[np.arange(N), y]).all()) and ref.l.max() < 0.05 and ref.l.min() < 1e-4
    ps = out['per_sample'].cpu().numpy().astype(np.float64)
    e = np.abs(ps - ref.l)
    print('cancellation C=%4d: max |l~ - l| %.3g, max |l~ - l| / bound %.3g, max relative %.3g (at loss %.3g)'
          % (C, e.max(), (e / ref.bl).max(), (e / ref.l).max(), ref.l[np.argmax(e / ref.l)]))
    assert bool((e <= ref.bl).all()), (np.flatnonzero(e > ref.bl)[:8].tolist(), float((e / ref.bl).max()))
    measure(out, x, y, ref, ('cancellation', C))


@pytest.mark.parametrize('N,C', [(20, 10), (110, 100), (1000, 50), (4096, 100)])
def test_mir_scores_rank_as_fp32_and_agree_with_fp64(native, N, C):
    """MIR's ranking (retrieve.py): rank_desc(post - pre) of the kernel's own per-sample vectors before and after a
    virtual step."""
    from b200ocl import ops
    from b200ocl.engine import ce_loss
    rs = np.random.RandomState(N + C)
    pre = (rs.standard_normal((N, C)) * 2).astype(np.float32)
    post = (pre + rs.standard_normal((N, C)) * 0.2).astype(np.float32)
    y = rs.randint(0, C, N).astype(np.int64)
    yt = torch.from_numpy(y).cuda()
    a = ce_loss(torch.from_numpy(pre).cuda(), yt, want_grad=False, want_per_sample=True)['per_sample']
    b = ce_loss(torch.from_numpy(post).cuda(), yt, want_grad=False, want_per_sample=True)['per_sample']
    top = ops.rank_desc(b, N, sa=1.0, b=a, sb=-1.0).cpu().numpy()
    s32 = b.cpu().numpy() - a.cpu().numpy()                         # fp32 subtraction
    np.testing.assert_array_equal(top, np.argsort(-s32, kind='stable'))   # descending, ties lowest index first
    ra, rb = reference(pre, y), reference(post, y)
    s64 = rb.l - ra.l
    B = float((ra.bl + rb.bl + U * np.abs(s64)).max())             # a score's bound, its fp32 rounding included
    o64 = np.argsort(-s64, kind='stable')
    srt = s64[o64]
    cuts = np.flatnonzero(srt[:-1] - srt[1:] > 2 * B) + 1           # the top k is decided wherever the gap exceeds 2B
    pos64 = np.empty(N, dtype=np.int64)
    pos64[o64] = np.arange(N)
    prefix_max = np.maximum.accumulate(pos64[top])
    bad = [int(k) for k in cuts if prefix_max[k - 1] != k - 1]
    print('mir N=%d C=%d: %d of %d cuts decided (2B = %.3g)' % (N, C, len(cuts), N - 1, 2 * B))
    assert not bad, bad[:10]
    assert len(cuts) >= (N - 1) // 3


@pytest.mark.parametrize('N,C', [(9, 1), (110, 100), (220, 10), (1000, 1025)])
def test_ce_flags_labels_outside_the_classifier(native, N, C):
    from b200ocl.engine import ce_loss, cls_loss
    rs = np.random.RandomState(N * C)
    x = (rs.standard_normal((N, C)) * 3).astype(np.float32)
    y = rs.randint(0, C, N).astype(np.int64)
    bad = np.array([1, N // 2, N - 1])
    y[bad] = [-1, C, C + 40]
    ok = np.setdiff1d(np.arange(N), bad)
    xt, yt = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    err = torch.zeros(1, dtype=torch.int32, device='cuda')
    out = raw_ce(native, xt, yt, err=err)
    assert int(err) == 1
    dl = out['dlogits'].cpu().numpy()
    assert np.array_equal(dl[bad], np.zeros((len(bad), C), np.float32))
    ps = out['per_sample'].cpu().numpy()
    assert np.isnan(ps[bad]).all() and not np.isnan(ps[ok]).any()
    ref = reference(x[ok], y[ok], n_div=N)
    assert bool((np.abs(ps[ok] - ref.l) <= ref.bl).all())
    assert bool((np.abs(dl[ok] - ref.d) <= ref.bd).all())
    bL, L = loss_bound(ref, N)                                       # the valid rows' sum over N
    assert abs(float(out['loss']) - L) <= bL, (float(out['loss']), L, bL)
    assert int(out['n_correct']) == int((np.argmax(x[ok], axis=1) == y[ok]).sum())
    # without a flag: the same bits; the wrapper passes its flag; cls_loss(mode='ce') treats the rows alike
    same_bits(raw_ce(native, xt, yt), out, 'no flag')
    err.zero_()
    same_bits(ce_loss(xt, yt, want_per_sample=True, want_correct=True, err=err), out, 'ce_loss')
    assert int(err) == 1
    err.zero_()
    same_bits(cls_loss(xt, yt, 'ce', err=err, want_correct=True), out, 'cls_loss ce')
    assert int(err) == 1


def test_loss_wrappers_refuse_labels_that_do_not_match_the_rows(native):
    from b200ocl.engine import ce_loss, cls_loss
    x = torch.zeros(10, 5, device='cuda')
    for y in (torch.zeros(9, dtype=torch.int64), torch.zeros(11, dtype=torch.int64),
              torch.zeros(10, 1, dtype=torch.int64), torch.zeros((), dtype=torch.int64)):
        y = y.cuda()
        torch.cuda.synchronize()
        before = native.launch_count()
        with pytest.raises(ValueError):
            ce_loss(x, y)
        with pytest.raises(ValueError):
            cls_loss(x, y, 'labels_trick')
        assert native.launch_count() == before, tuple(y.shape)


def _er_params(trick):
    flags = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick',
                                'kd_trick_star')}
    if trick:
        flags[trick] = True
    return SimpleNamespace(data='cifar10', cuda=True, epoch=1, batch=10, verbose=False, mem_size=40, eps_mem_batch=10,
                           mem_iters=1, update='random', retrieve='random', agent='ER', k=3, aser_type='asvm',
                           n_smp_cls=1.5, num_tasks=5, buffer_tracker=False, optimizer='SGD', learning_rate=0.1,
                           weight_decay=0, temp=0.07, head='mlp', subsample=20, error_analysis=False, trick=flags)


@pytest.mark.parametrize('trick', [None, 'labels_trick'])
def test_er_raises_on_a_label_outside_the_classifier(native, trick):
    """A 10-class ER learner trained on label 10: plain CE (b200ocl_ce_loss) and the labels trick (b200ocl_cls_loss)
    both flag the row, and train_learner raises at its per-task check."""
    from b200ocl import nets, registry
    params = _er_params(trick)
    agent = registry.agents['ER'](nets.setup_architecture(params), None, params)
    rs = np.random.RandomState(3)
    x = rs.randint(0, 256, (30, 32, 32, 3)).astype(np.uint8)
    y = rs.randint(0, 5, 30).astype(np.int64)
    y[7] = 10
    with pytest.raises(KeyError):
        agent.train_learner(x, y)
    assert int(agent._err) == 0                                      # read and cleared once


# ------------------------------------------------------------------------------------------------- the siblings

def _sep_tables(rs, C):
    """old_labels (the first half of a permutation, one repeat) ++ new_labels (the rest) and lbl_inv_map."""
    perm = rs.permutation(C).tolist()
    old, new = perm[:C // 2], perm[C // 2:]
    if len(old) >= 2:
        old = old + [old[0]]                                         # a column held at two positions
    inv = {}
    for c in sorted(set(old)):
        inv[c] = old.index(c)
    for i, c in enumerate(new):
        inv[c] = len(old) + i
    return old, new, inv


@pytest.mark.parametrize('C', C_SET)
@pytest.mark.parametrize('N', N_SET)
def test_cls_loss_at_the_edges(native, N, C):
    rs = np.random.RandomState(7 * N + C)
    logits = (rs.standard_normal((N, C)) * rs.choice([0.01, 1, 30])).astype(np.float32)
    labels = rs.randint(0, C, N).astype(np.int64)
    labels[0], labels[-1] = 0, C - 1
    teacher = (rs.standard_normal((N, C)) * 3).astype(np.float32)
    old, new, inv = _sep_tables(rs, C)
    for kw in (dict(mode='ce', teacher=teacher, w_ce=0.4, w_kd=0.6),
               dict(mode='labels_trick', teacher=None, w_ce=1.0, w_kd=0.0),
               dict(mode='labels_trick', teacher=teacher, w_ce=0.25, w_kd=0.75),
               dict(mode='separated_softmax', teacher=None, w_ce=1.0, w_kd=0.0, old_labels=old, new_labels=new,
                    lbl_inv_map=inv)):
        gtricks._check(logits, labels, kw, (N, C, kw['mode'], kw['teacher'] is not None))


@pytest.mark.parametrize('n_old,n_new', [(1, 1), (1, 33), (32, 1), (32, 33), (33, 32), (33, 33), (0, 32), (32, 0)])
def test_separated_softmax_segments_of_1_32_and_33(native, n_old, n_new):
    C = 100
    for N in (9, 110):
        rs = np.random.RandomState(100 * n_old + n_new + N)
        perm = rs.permutation(C).tolist()
        old, new = perm[:n_old], perm[n_old:n_old + n_new]
        inv = {c: i for i, c in enumerate(old)}
        inv.update({c: n_old + i for i, c in enumerate(new)})
        logits = (rs.standard_normal((N, C)) * 4).astype(np.float32)
        labels = np.asarray(sorted(inv))[rs.randint(0, len(inv), N)].astype(np.int64)
        kw = dict(mode='separated_softmax', teacher=None, w_ce=1.0, w_kd=0.0, old_labels=old, new_labels=new,
                  lbl_inv_map=inv)
        gtricks._check(logits, labels, kw, (N, n_old, n_new))


def test_labels_trick_at_the_class_limit_and_its_refusal_beyond(native):
    from b200ocl.engine import cls_loss
    N, C = 110, CLS_MAX_C
    rs = np.random.RandomState(12288)
    logits = (rs.standard_normal((N, C)) * 3).astype(np.float32)
    labels = rs.randint(0, C, N).astype(np.int64)
    labels[0], labels[-1] = 0, C - 1
    gtricks._check(logits, labels, dict(mode='labels_trick', teacher=None, w_ce=1.0, w_kd=0.0), 'C = max')
    x = torch.zeros(N, C + 1, device='cuda')
    y = torch.zeros(N, dtype=torch.int64, device='cuda')
    torch.cuda.synchronize()
    before = native.launch_count()
    with pytest.raises(native.NativeError):
        cls_loss(x, y, 'labels_trick')
    assert native.launch_count() == before


@pytest.mark.parametrize('C', C_SET)
@pytest.mark.parametrize('N', N_SET)
def test_icarl_loss_at_the_edges(native, N, C):
    for with_old in (False, True):
        K_eq_C = C < 4 or with_old
        case = gicarl._sweep_case(N, C, with_old, K_eq_C, 500 + 11 * N + C + with_old)
        gicarl._check(*case, (N, C, with_old, K_eq_C))
