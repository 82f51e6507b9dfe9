"""GPU: the evaluation kernels of csrc/ncm.cu against the float64 restatement of evaluate() (oracle/evaluate.py).

Every accuracy evaluate() returns is a hit count from classify_kernel: b200ocl_ncm_classify (nearest class mean: SCR,
iCaRL, ncm_trick) or b200ocl_linear_argmax (every other agent).  Both run one warp per sample, 8 per CTA.

Predictions must equal the fp64 arg-min / arg-max except on near-ties.  The kernel's pick p is excused against the
fp64 winner b only when score64[p] - score64[b] is within the fp32 rounding of the two scores (EPS = 2^-24,
n = ceil(d / 32) + 5 additions per score: ceil(d / 32) per lane, then 5 shuffle levels; gamma_n = n EPS / (1 - n EPS)):
  nearest mean  |s - s64| <= gamma_{n+2} s + 2 (n + 3) EPS sqrt(s)   (the sum of squares, plus the rounding of the
                normalised feature, whose norm is itself an n-term sum, entering through 2 (f - mu) df)
  arg-max       |s - s64| <= gamma_{n+1} (sum_i |f_i w_i| + |b|)
and the bound used is twice the sum of the two scores' bounds.  Excused rows must be at most 1 % of a call (at least 1).

Class means (b200ocl_ncm_class_means) at the widths CIFAR (160) and Mini-ImageNet (640) features have: absolute error
of the unit-norm means, NCM_TOL, about 3x the largest measured on an H100 80GB HBM3 (SXM, 132 SMs, 700 W power limit)
[in brackets]."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import evaluate as oev

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24
NCM_TOL = 1e-7           # [3.4e-8 at d = 160, 1.8e-8 at d = 640]
DS = (1, 31, 33, 160, 640, 2560)
KS = (1, 2, 10, 50, 100)
BS = (0, 1, 7, 8, 9, 128, 1000)


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import ops as _ops
    return _ops


def gamma(n):
    return n * EPS / (1 - n * EPS)


def ncm_bound(s, d):
    n = math.ceil(d / 32) + 5
    return gamma(n + 2) * s + 2 * (n + 3) * EPS * np.sqrt(s)


def linear_bound(f, w, b):
    n = math.ceil(f.shape[1] / 32) + 5
    mag = np.abs(f.astype(np.float64)) @ np.abs(w.astype(np.float64)).T + np.abs(b.astype(np.float64))[None, :]
    return gamma(n + 1) * mag


def check_picks(pick, scores, bounds, tag):
    """pick[b]: the kernel's index; scores [B,K] fp64 (smaller wins); bounds [B,K] the fp32 error bound of each score.
    Returns the number of excused rows."""
    B = scores.shape[0]
    if B == 0:
        return 0
    best = oev.first_argmin(scores)
    bad = np.nonzero(pick != best)[0]
    for r in bad:
        gap = scores[r, pick[r]] - scores[r, best[r]]
        assert np.isfinite(gap) and gap <= 2 * (bounds[r, pick[r]] + bounds[r, best[r]]), \
            '%s row %d: picked %d (%.17g) over %d (%.17g), not a near-tie' % (tag, r, pick[r], scores[r, pick[r]], best[r],
                                                                              scores[r, best[r]])
    assert len(bad) <= max(1, B // 100), (tag, len(bad))
    return len(bad)


def class_ids_for(rs, K):
    return (rs.permutation(1000)[:K] * 3 + 7).astype(np.int64)       # unsorted, non-contiguous, as old_labels


def unit_rows(x):
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def truth_for(rs, pred64, class_ids, B):
    """Mostly the fp64 prediction, some other class, some label outside class_ids."""
    t = pred64.copy()
    flip = rs.rand(B) < 0.3
    t[flip] = class_ids[rs.randint(0, len(class_ids), B)][flip]
    out = rs.rand(B) < 0.1
    t[out] = 10 ** 6 + rs.randint(0, 5, B)[out]
    return t


def hits_tensor(start=0):
    return torch.full((1,), start, dtype=torch.int64, device='cuda')


@pytest.mark.parametrize('d', DS)
def test_ncm_classify_against_fp64(ops, d):
    rs = np.random.RandomState(d)
    excused = 0
    for K in KS:
        ids = class_ids_for(rs, K)
        means = unit_rows(rs.standard_normal((K, d))).astype(np.float32)
        for B in BS:
            # features near the means (as test features are) plus noise, then encoder-like ReLU
            f = np.maximum(means[rs.randint(0, K, B)] * 3 + rs.standard_normal((B, d)), 0).astype(np.float32)
            f[np.abs(f).sum(1) == 0, 0] = 1.0                        # zero rows are pinned separately
            f64s = oev.ncm_distances(f, means)
            pred64 = ids[oev.first_argmin(f64s)] if B else np.zeros(0, np.int64)
            truth = truth_for(rs, pred64, ids, B)
            hits = hits_tensor(5)
            pred = ops.ncm_classify(torch.from_numpy(f).cuda(), torch.from_numpy(means).cuda(), torch.from_numpy(ids).cuda(),
                                    truth=torch.from_numpy(truth).cuda(), n_correct=hits).cpu().numpy()
            assert pred.shape == (B,)
            assert np.isin(pred, ids).all()
            pick = np.array([int(np.nonzero(ids == p)[0][0]) for p in pred], dtype=np.int64)
            excused += check_picks(pick, f64s, ncm_bound(f64s, d), 'ncm d=%d K=%d B=%d' % (d, K, B))
            assert int(hits) == 5 + int((pred == truth).sum()), (d, K, B)
    print('ncm_classify d=%d: %d near-tie rows excused' % (d, excused))


@pytest.mark.parametrize('d', DS)
def test_linear_argmax_against_fp64(ops, d):
    rs = np.random.RandomState(1000 + d)
    excused = 0
    for C in KS:
        w = (rs.standard_normal((C, d)) / np.sqrt(d)).astype(np.float32)
        b = (0.1 * rs.standard_normal(C)).astype(np.float32)
        for B in BS:
            f = np.maximum(rs.standard_normal((B, d)), 0).astype(np.float32)
            neg = -oev.linear_logits(f, w, b)
            pred64 = oev.first_argmin(neg) if B else np.zeros(0, np.int64)
            truth = truth_for(rs, pred64, np.arange(C), B)
            hits = hits_tensor(3)
            pred = ops.linear_argmax(torch.from_numpy(f).cuda(), torch.from_numpy(w).cuda(), torch.from_numpy(b).cuda(),
                                     truth=torch.from_numpy(truth).cuda(), n_correct=hits).cpu().numpy()
            assert pred.shape == (B,) and ((pred >= 0) & (pred < C)).all()
            excused += check_picks(pred, neg, linear_bound(f, w, b) if B else neg, 'linear d=%d C=%d B=%d' % (d, C, B))
            assert int(hits) == 3 + int((pred == truth).sum()), (d, C, B)
    print('linear_argmax d=%d: %d near-tie rows excused' % (d, excused))


@pytest.mark.parametrize('d', [33, 160, 640, 2560])
def test_exact_ties_go_to_the_first_index(ops, d):
    """Duplicated class-mean rows / weight rows with equal biases: the fp32 scores are bit-equal, and the first index
    wins on the device as in the fp64 restatement (dists.min(1) / torch.max(logits, 1))."""
    rs = np.random.RandomState(d + 7)
    K = 12
    base = unit_rows(rs.standard_normal((K, d))).astype(np.float32)
    dup = np.concatenate([base, base[[3, 0, 7]]])               # rows 12, 13, 14 repeat rows 3, 0, 7
    dup = dup[[12, 1, 2, 3, 4, 5, 6, 13, 8, 9, 10, 11, 0, 14, 7]]   # copies: rows 0 = 3, 7 = 12, 13 = 14
    ids = class_ids_for(rs, dup.shape[0])
    f = np.maximum(dup[rs.randint(0, dup.shape[0], 300)] * 4 + 0.05 * rs.standard_normal((300, d)), 0).astype(np.float32)
    pred = ops.ncm_classify(torch.from_numpy(f).cuda(), torch.from_numpy(dup).cuda(), torch.from_numpy(ids).cuda()).cpu().numpy()
    first = oev.first_argmin(oev.ncm_distances(f, dup))
    np.testing.assert_array_equal(pred, ids[first])
    # every duplicated mean was some row's winner, and the first of its copies took it
    for a, b in [(0, 3), (7, 12), (13, 14)]:
        assert (first == a).any() and not (first == b).any(), (a, b)
    bias = np.zeros(dup.shape[0], np.float32)
    bias[[7, 12]] = 0.25                                         # the copies keep equal biases
    predl = ops.linear_argmax(torch.from_numpy(f).cuda(), torch.from_numpy(dup).cuda(), torch.from_numpy(bias).cuda()).cpu().numpy()
    firstl = oev.first_argmin(-oev.linear_logits(f, dup, bias))
    np.testing.assert_array_equal(predl, firstl)
    for a, b in [(0, 3), (7, 12), (13, 14)]:
        assert (firstl == a).any() and not (firstl == b).any(), (a, b)


def test_zero_feature_row_follows_torch(ops):
    """A zero feature: f / ||f|| is NaN, every distance is NaN, and torch's dists.min(1) returns index 0, so the
    prediction is class_ids[0]."""
    rs = np.random.RandomState(9)
    d, K = 160, 10
    means = unit_rows(rs.standard_normal((K, d))).astype(np.float32)
    ids = class_ids_for(rs, K)
    f = np.maximum(rs.standard_normal((9, d)), 0).astype(np.float32)
    f[[0, 4, 8]] = 0
    ft = torch.from_numpy(f)
    fn = ft / ft.norm(dim=1, keepdim=True)
    _, torch_pick = (fn[:, :, None] - torch.from_numpy(means).T[None]).pow(2).sum(1).min(1)
    assert (torch_pick[[0, 4, 8]] == 0).all()
    hits = hits_tensor()
    pred = ops.ncm_classify(ft.cuda(), torch.from_numpy(means).cuda(), torch.from_numpy(ids).cuda(),
                            truth=torch.from_numpy(ids[torch_pick.numpy()]).cuda(), n_correct=hits).cpu().numpy()
    np.testing.assert_array_equal(pred, ids[torch_pick.numpy()])
    np.testing.assert_array_equal(pred, oev.ncm_predict(f, means, ids))
    assert int(hits) == 9


def test_hit_count_accumulates(ops):
    rs = np.random.RandomState(10)
    d, K, B = 640, 50, 77
    means = unit_rows(rs.standard_normal((K, d))).astype(np.float32)
    ids = torch.from_numpy(class_ids_for(rs, K)).cuda()
    f = torch.from_numpy(np.maximum(rs.standard_normal((B, d)), 0).astype(np.float32)).cuda()
    m = torch.from_numpy(means).cuda()
    pred = ops.ncm_classify(f, m, ids)
    truth = pred.clone()
    truth[::3] = -5                                              # never a class id: never a hit
    want = int((pred == truth).sum())
    hits = hits_tensor(11)
    ops.ncm_classify(f, m, ids, truth=truth, n_correct=hits)
    ops.ncm_classify(f, m, ids, truth=truth, n_correct=hits)       # adds, never overwrites
    assert int(hits) == 11 + 2 * want
    ops.ncm_classify(f, m, ids, n_correct=hits)                     # no truth: untouched
    ops.ncm_classify(f[:0], m, ids, truth=truth[:0], n_correct=hits)   # B = 0: untouched
    assert int(hits) == 11 + 2 * want
    w, b = m[:20].contiguous(), torch.zeros(20, device='cuda')
    lp = ops.linear_argmax(f, w, b)
    lt = lp.clone()
    lt[1::2] = 20                                                  # outside [0, C)
    h2 = hits_tensor(2)
    ops.linear_argmax(f, w, b, truth=lt, n_correct=h2)
    ops.linear_argmax(f, w, b, truth=lt, n_correct=h2)
    ops.linear_argmax(f, w, b, n_correct=h2)
    ops.linear_argmax(f[:0], w, b, truth=lt[:0], n_correct=h2)
    assert int(h2) == 2 + 2 * int((lp == lt).sum())


def test_refusals(ops):
    f = torch.zeros(4, 16, device='cuda')
    ids = torch.arange(3, device='cuda')
    with pytest.raises(ValueError):
        ops.ncm_classify(f, torch.zeros(3, 15, device='cuda'), ids)
    with pytest.raises(ValueError):
        ops.ncm_classify(f, torch.zeros(3, 16, device='cuda'), torch.arange(2, device='cuda'))
    with pytest.raises(ValueError):
        ops.ncm_classify(f, torch.zeros(3, 16, device='cuda'), ids, truth=torch.zeros(5, dtype=torch.int64, device='cuda'))
    with pytest.raises(ValueError):
        ops.linear_argmax(f, torch.zeros(3, 17, device='cuda'), torch.zeros(3, device='cuda'))
    with pytest.raises(ValueError):
        ops.linear_argmax(f, torch.zeros(3, 16, device='cuda'), torch.zeros(4, device='cuda'))
    with pytest.raises(ValueError):
        ops.linear_argmax(f, torch.zeros(3, 16, device='cuda'), torch.zeros(3, device='cuda'),
                          truth=torch.zeros(3, dtype=torch.int64, device='cuda'))


@pytest.mark.parametrize('d', [160, 640])
def test_ncm_class_means_against_fp64(ops, d):
    """Classes with 0, 1 and many samples, a class listed twice, labels absent from class_ids."""
    rs = np.random.RandomState(d + 3)
    n = 1001
    f = np.maximum(rs.standard_normal((n, d)), 0).astype(np.float32)
    lab = rs.randint(0, 12, n) * 5 + 1                           # 1, 6, ..., 56
    lab[17] = 500                                                # one sample
    lab[lab == 56] = 999                                         # not in class_ids
    ids = np.array([31, 500, 6, 77, 1, 31, 46, 21, 16, 11, 51, 41, 36, 26], dtype=np.int64)   # 77: none; 31 twice
    means, counts = ops.ncm_class_means(torch.from_numpy(f).cuda(), torch.from_numpy(lab).cuda(), torch.from_numpy(ids).cuda())
    mu64, c64 = oev.class_means(f, lab, ids)
    np.testing.assert_array_equal(counts.cpu().numpy(), c64)
    assert c64[1] == 1 and c64[3] == 0 and c64[0] == c64[5] > 50
    m = means.cpu().numpy()
    assert (m[3] == 0).all()                                     # left for the caller's random mean
    assert np.array_equal(m[0], m[5])
    worst = float(np.abs(m - mu64).max())
    print('ncm_class_means d=%d abs %.3g' % (d, worst))
    assert worst <= NCM_TOL, (d, worst)


# ---------------------------------------------------------------------------------------------------------- evaluate()
def _agent(agent, hw, mem):
    from b200ocl import nets, registry
    from oracle import resnet as oresnet
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick', 'kd_trick_star')}
    data = 'cifar100' if hw == 32 else 'mini_imagenet'
    params = SimpleNamespace(data=data, cuda=True, epoch=1, batch=10, verbose=False, mem_size=mem, eps_mem_batch=10,
                             mem_iters=1, update='random', retrieve='random', agent=agent, k=3, aser_type='asvm',
                             n_smp_cls=1.5, num_tasks=5, buffer_tracker=False, optimizer='SGD', learning_rate=0.1,
                             weight_decay=0, temp=0.07, head='mlp', subsample=20, error_analysis=False, trick=trick)
    a = registry.agents[agent](nets.setup_architecture(params), None, params)
    head = 'mlp' if agent == 'SCR' else None
    spec = oresnet.Spec(hw, 20, 100, head=head)
    p, bn = oresnet.seeded_state(spec, 3)
    a.model.engine.load(list(p.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
    return a


@pytest.mark.parametrize('agent,hw', [('SCR', 32), ('ER', 32), ('ER', 84)])
def test_evaluate_matches_fp64_restatement(agent, hw):
    """evaluate() end to end on a seeded network: a full 1001-image buffer (features from three 500-image chunks) whose
    labels cover every seen class but one (that class gets the random mean), two test loaders of two batches each.
    The per-task accuracies equal the fp64 restatement applied to the engine's own features_eval outputs, up to the
    counted near-ties; the empty class's random mean is the same CPU draw on both sides."""
    rs = np.random.RandomState(hw)
    a = _agent(agent, hw, 1001)
    eng = a.engine
    seen = [int(c) for c in rs.permutation(100)[:15]]
    a.old_labels = list(seen)
    n = 1001
    buf_lab = np.array(seen[:14])[rs.randint(0, 14, n)]             # seen[14] has no exemplar
    a.buffer.buffer_img.copy_(torch.from_numpy(rs.rand(n, 3, hw, hw).astype(np.float32)))
    a.buffer.buffer_label.copy_(torch.from_numpy(buf_lab))
    a.buffer._labels_host[:] = buf_lab
    a.buffer.current_index = n
    loaders = []
    for t in range(2):
        loaders.append([(torch.from_numpy(rs.rand(bs, 3, hw, hw).astype(np.float32)),
                         torch.from_numpy(np.array(seen)[rs.randint(0, 15, bs)])) for bs in (37, 64)])
    torch.manual_seed(123)
    acc = np.asarray(a.evaluate(loaders))

    # the fp64 restatement on the engine's own features
    with torch.no_grad():
        if agent == 'SCR':
            bf = torch.cat([eng.features_eval(a.buffer.buffer_img[s:s + 500]) for s in range(0, n, 500)]).cpu().numpy()
            torch.manual_seed(123)
            draw = torch.normal(0, 1, size=(1, eng.dim_in)).squeeze().numpy()
            means, counts = oev.class_means(bf, buf_lab, seen, draws=[draw])
            assert counts[14] == 0 and (counts[:14] > 0).all()
        else:
            lin = (a.model.linear__weight, a.model.linear__bias) if hasattr(a.model, 'linear__weight') else \
                (a.model.linear.weight, a.model.linear.bias)
            W, b = (t.detach().cpu().numpy() for t in lin)
        for task, loader in enumerate(loaders):
            hits64, total, slack = 0, 0, 0
            for x, y in loader:
                f = eng.features_eval(x.cuda()).cpu().numpy()
                if agent == 'SCR':
                    s = oev.ncm_distances(f, means)
                    bound = ncm_bound(s, f.shape[1])
                    pred = np.asarray(seen)[oev.first_argmin(s)]
                else:
                    s = -oev.linear_logits(f, W, b)
                    bound = linear_bound(f, W, b)
                    pred = oev.first_argmin(s)
                best = oev.first_argmin(s)
                srt = np.sort(s, axis=1)
                # rows whose winner is within the rounding bound of the runner-up could go either way
                gap = srt[:, 1] - srt[:, 0] if s.shape[1] > 1 else np.full(len(s), np.inf)
                slack += int((gap <= 4 * bound[np.arange(len(s)), best]).sum())
                hits64 += int((pred == y.numpy()).sum())
                total += len(y)
            got = int(round(acc[task] * total))
            print('evaluate %s %dx%d task %d: %d / %d hits, fp64 %d, %d near-tie rows' % (agent, hw, hw, task, got, total,
                                                                                          hits64, slack))
            assert abs(got - hits64) <= slack, (agent, hw, task, got, hits64, slack)
            assert slack <= max(1, total // 100)
