"""GPU parity: CUDA kernels (through the C ABI) vs the CPU oracle and the reference-recorded
golden vectors.  Run on an H100:  python -m pytest tests -m gpu"""
import os

import numpy as np
import pytest
import torch

from oracle import aser as oaser
from oracle import knn_sv as oknn
from oracle import supcon as osup

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import ops as _ops
    return _ops


def dev(a, dtype=None):
    t = torch.as_tensor(np.asarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.cuda()


def relu_feats(rs, n, d):
    return np.maximum(rs.standard_normal((n, d)), 0).astype(np.float32)


def check_sv_against_oracle(ops, ef, ey, cf, cy, k, tag=''):
    """Every row against the fp64 recurrence on the kernel's own fp32 distance order (oracle.knn_sv.kernel_order), within
    3e-6 and the rounding bound derived in test_gpu_knn_sv_fp64.py; no row is excused."""
    eft, cft, eyt, cyt = dev(ef), dev(cf), dev(ey), dev(cy)
    out = ops.knn_sv(eft, eyt, cft, cyt, k, want_matrix=True, want_sum=True, want_max=True, want_min=True)
    L = ops.knn_sv_plan(eft.shape[0], cft.shape[0], eft.shape[1], True, True, 0)
    order, _ = oknn.kernel_order(eft, cft, large=L.name == 'large')
    sv64, abs_sum = oknn.knn_sv_torch(order, eyt, cyt, k)
    err = (out['sv'].double() - sv64).abs().max(1).values
    bad = torch.nonzero(err > torch.clamp(oknn.sv_row_bound(abs_sum, L, cft.shape[0]), max=3e-6)).flatten()
    assert bad.numel() == 0, (tag, bad[:10].tolist(), err[bad[:10]].tolist())
    sv = out['sv'].cpu().numpy()
    # reductions are reductions of the kernel's own matrix
    np.testing.assert_allclose(out['sum'].cpu().numpy(), sv.astype(np.float64).sum(0), rtol=0, atol=2e-5)
    np.testing.assert_array_equal(out['max'].cpu().numpy(), sv.max(0))
    np.testing.assert_array_equal(out['min'].cpu().numpy(), sv.min(0))
    return sv


def test_knn_sv_golden(ops, golden_dir):
    g = np.load(os.path.join(golden_dir, 'knn_sv.npz'))
    for i in range(int(g['n_cases'])):
        ef, cf, ey, cy, k = (g['c%d_%s' % (i, n)] for n in ('ef', 'cf', 'ey', 'cy', 'k'))
        sv = check_sv_against_oracle(ops, ef, ey, cf, cy, int(k), 'golden%d' % i)
        ref = g['c%d_sv' % i]
        rows_ok = np.abs(sv - ref).max(1) <= 3e-6
        assert rows_ok.mean() >= 0.98, (i, rows_ok.mean())


@pytest.mark.parametrize('C', [1, 2, 3, 4, 31, 32, 33, 64, 100, 128, 160, 257, 512, 600, 1000, 1024])
def test_knn_sv_candidate_sizes(ops, C):
    rs = np.random.RandomState(C)
    E, d, ncls = 19, 40, 7
    ef, cf = relu_feats(rs, E, d), relu_feats(rs, C, d)
    ey, cy = rs.randint(0, ncls, E), rs.randint(0, ncls, C)
    check_sv_against_oracle(ops, ef, ey, cf, cy, 3, 'C%d' % C)


@pytest.mark.parametrize('E,C,d,k', [(1500, 100, 64, 3), (1300, 600, 32, 5), (2000, 1000, 16, 3), (1, 50, 7, 1),
                                     (8, 160, 160, 3), (9, 160, 161, 3), (257, 37, 5, 10)])
def test_knn_sv_row_tilings(ops, E, C, d, k):
    rs = np.random.RandomState(E + C)
    ef, cf = relu_feats(rs, E, d), relu_feats(rs, C, d)
    ey, cy = rs.randint(0, 10, E), rs.randint(0, 10, C)
    check_sv_against_oracle(ops, ef, ey, cf, cy, k, 'E%d' % E)


@pytest.mark.parametrize('E,C,d,k', [(300, 1025, 16, 3), (40, 1500, 40, 3), (7, 3000, 64, 5), (3, 20000, 32, 3),
                                     (150, 2048, 24, 1)])
def test_knn_sv_large_candidate_sets(ops, E, C, d, k):
    """C > 1024: the scratch-line kernel (knn_sv_large.cu) -- same results as the fused kernel's contract."""
    rs = np.random.RandomState(E + C)
    ef, cf = relu_feats(rs, E, d), relu_feats(rs, C, d)
    ey, cy = rs.randint(0, 10, E), rs.randint(0, 10, C)
    check_sv_against_oracle(ops, ef, ey, cf, cy, k, 'large E%d C%d' % (E, C))


def test_knn_sv_large_ties(ops):
    rs = np.random.RandomState(6)
    cf = rs.randint(0, 3, (1300, 6)).astype(np.float32)    # integer features: many exact ties, lowest index first
    ef = np.concatenate([cf[:10], rs.randint(0, 3, (10, 6)).astype(np.float32)])
    cy, ey = rs.randint(0, 3, 1300), rs.randint(0, 3, 20)
    out = ops.knn_sv(dev(ef), dev(ey), dev(cf), dev(cy), 3, want_matrix=True)
    sv64, _, _ = oknn.knn_sv_matrix(ef, ey, cf, cy, 3)
    np.testing.assert_allclose(out['sv'].cpu().numpy(), sv64, atol=3e-6)


def test_knn_sv_ties_and_duplicates(ops):
    """Equal distances rank lowest candidate index first; a candidate equal to the eval point has
    distance exactly 0 (direct-difference form)."""
    rs = np.random.RandomState(5)
    cf = rs.randint(0, 3, (64, 6)).astype(np.float32)       # integer features: many exact ties
    ef = np.concatenate([cf[:10], rs.randint(0, 3, (10, 6)).astype(np.float32)])
    cy, ey = rs.randint(0, 3, 64), rs.randint(0, 3, 20)
    out = ops.knn_sv(dev(ef), dev(ey), dev(cf), dev(cy), 3, want_matrix=True)
    sv64, _, _ = oknn.knn_sv_matrix(ef, ey, cf, cy, 3)
    np.testing.assert_allclose(out['sv'].cpu().numpy(), sv64, atol=3e-6)


def test_knn_sv_deterministic_and_limits(ops):
    rs = np.random.RandomState(1)
    ef, cf = dev(relu_feats(rs, 3000, 48)), dev(relu_feats(rs, 200, 48))
    ey, cy = dev(rs.randint(0, 20, 3000)), dev(rs.randint(0, 20, 200))
    a = ops.knn_sv(ef, ey, cf, cy, 3, want_max=True, want_min=True)
    b = ops.knn_sv(ef, ey, cf, cy, 3, want_max=True, want_min=True)
    for key in ('sum', 'max', 'min'):
        assert torch.equal(a[key], b[key])
    big = ops.knn_sv(ef[:50], ey[:50], dev(relu_feats(rs, 1025, 48)), dev(rs.randint(0, 20, 1025)), 3)   # scratch-line kernel
    assert big['sum'].shape == (1025,) and bool(torch.isfinite(big['sum']).all())
    empty = ops.knn_sv(ef[:0], ey[:0], cf, cy, 3)
    assert float(empty['sum'].abs().sum()) == 0.0


def test_knn_sv_sweep_properties(ops):
    """BASELINE config 5 at full size (50k x 512 eval, 1k candidates): size-independent properties.
    Shapley efficiency: each row of SVs sums to the kNN utility of the full candidate set,
    (1/k) * #label matches among the k nearest; column sums are equivariant to candidate permutation;
    a sample of rows equals the fp64 oracle."""
    g = torch.Generator(device='cuda').manual_seed(0)
    E, C, d, k = 50000, 1000, 512, 3
    ef = torch.relu(torch.randn(E, d, device='cuda', generator=g))
    cf = torch.relu(torch.randn(C, d, device='cuda', generator=g))
    ey = torch.randint(0, 100, (E,), device='cuda', generator=g)
    cy = torch.randint(0, 100, (C,), device='cuda', generator=g)
    out = ops.knn_sv(ef, ey, cf, cy, k, want_sum=True, want_max=True, want_min=True)
    # independent utility: direct-difference distances in fp64 on chunks, torch.topk
    util = torch.zeros((), dtype=torch.float64, device='cuda')
    for s in range(0, E, 500):
        diff = ef[s:s + 500, None, :].double() - cf[None, :, :].double()
        dist = (diff * diff).sum(2)
        nn = dist.topk(k, dim=1, largest=False).indices
        util += (cy[nn] == ey[s:s + 500, None]).double().sum() / k
    total = out['sum'].double().sum()
    assert abs(float(total - util)) < 2e-3 * max(1.0, float(util)), (float(total), float(util))
    perm = torch.randperm(C, device='cuda', generator=g)
    out_p = ops.knn_sv(ef, ey, cf[perm], cy[perm], k, want_sum=True)
    # equivariant up to the tie-break: ~1e-4 of the fp32 distance pairs of a row collide exactly at this
    # size and ties are broken by candidate index, which the permutation changes
    dsum = (out_p['sum'] - out['sum'][perm]).abs()
    assert float((dsum <= 2e-4).float().mean()) >= 0.98 and float(dsum.max()) < 5e-3, float(dsum.max())
    rows = torch.arange(0, E, 997, device='cuda')
    check_sv_against_oracle(ops, ef[rows].cpu().numpy(), ey[rows].cpu().numpy(), cf.cpu().numpy(),
                            cy.cpu().numpy(), k, 'sweep-sample')


def test_rank_desc(ops):
    rs = np.random.RandomState(2)
    for n in [1, 2, 5, 100, 160, 1000, 1024, 1025, 4096]:
        v = rs.standard_normal(n).astype(np.float32)
        v[rs.randint(0, n, n // 3)] = 0.5       # ties
        v[rs.randint(0, n, max(1, n // 7))] = -0.0
        ref = oaser.argsort_desc_stable(np.where(v == 0, 0.0, v))
        got = ops.rank_desc(dev(v)).cpu().numpy()
        np.testing.assert_array_equal(got, ref)
        top = ops.rank_desc(dev(v), n_out=min(10, n)).cpu().numpy()
        np.testing.assert_array_equal(top, ref[:min(10, n)])
    a, b = rs.standard_normal(160).astype(np.float32), rs.standard_normal(160).astype(np.float32)
    idx, sc = ops.rank_desc(dev(a), 10, sa=1 / 100., b=dev(b), sb=-1 / 10., return_scores=True)
    score = a * np.float32(1 / 100.) + b * np.float32(-1 / 10.)
    np.testing.assert_allclose(sc.cpu().numpy(), score, rtol=1e-6, atol=1e-7)
    np.testing.assert_array_equal(idx.cpu().numpy(), oaser.argsort_desc_stable(sc.cpu().numpy())[:10])


def test_supcon_golden_and_oracle(ops, golden_dir):
    g = np.load(os.path.join(golden_dir, 'supcon.npz'))
    for i in range(int(g['n_cases'])):
        f, y, T = g['c%d_f' % i], g['c%d_y' % i], float(g['c%d_T' % i])
        loss, grad = ops.supcon(dev(f), dev(y), T)
        ref_loss, ref_grad = float(g['c%d_loss' % i]), g['c%d_grad' % i]
        if np.isnan(ref_loss):
            assert np.isnan(float(loss))
            continue
        # tolerance stated by north_star: 1e-3 relative in fp32
        assert abs(float(loss) - ref_loss) <= 1e-4 * abs(ref_loss), (i, float(loss), ref_loss)
        np.testing.assert_allclose(grad.cpu().numpy(), ref_grad, rtol=1e-3, atol=1e-3 * np.abs(ref_grad).max())
        o_loss, o_grad = osup.supcon_loss_and_grad(f, y, T)
        np.testing.assert_allclose(grad.cpu().numpy(), o_grad, rtol=1e-3, atol=2e-5 * np.abs(o_grad).max())


@pytest.mark.parametrize('B,V,d,T', [(110, 2, 128, 0.07), (7, 2, 33, 0.1), (1024, 2, 128, 0.07), (40, 3, 200, 0.5),
                                     (16, 2, 600, 0.07), (3, 1, 1024, 1.0),
                                     # the fused single-launch kernel: every tile configuration (TM 16 / 32 / 64),
                                     # every d chunk count, ragged last tiles, a unit count above the SM count
                                     (110, 2, 160, 0.07), (50, 2, 256, 0.1), (9, 1, 4, 0.2), (33, 3, 64, 0.07),
                                     (1300, 2, 128, 0.07), (1250, 2, 160, 0.1), (2500, 2, 128, 0.07),
                                     (2400, 2, 256, 0.07), (4801, 2, 64, 0.07)])
def test_supcon_shapes(ops, B, V, d, T):
    rs = np.random.RandomState(B + d)
    f = rs.standard_normal((B, V, d)).astype(np.float32)
    f /= np.linalg.norm(f, axis=2, keepdims=True)
    y = rs.randint(0, max(2, B // 4), B)
    if V == 1:
        y = np.arange(B) // 2 * 0        # all one class: every anchor has positives
    loss, grad = ops.supcon(dev(f), dev(y), T)
    o_loss, o_grad = osup.supcon_loss_and_grad(f, y, T)
    assert abs(float(loss) - o_loss) <= 1e-4 * abs(o_loss)
    np.testing.assert_allclose(grad.cpu().numpy(), o_grad, rtol=1e-3, atol=1e-4 * np.abs(o_grad).max())
    loss2, none = ops.supcon(dev(f), dev(y), T, need_grad=False)
    assert none is None and float(loss2) == float(loss)
    # invariance to sample permutation (SURVEY.md section 4)
    perm = rs.permutation(B)
    loss_p, _ = ops.supcon(dev(f[perm]), dev(y[perm]), T, need_grad=False)
    assert abs(float(loss_p) - float(loss)) <= 1e-5 * abs(float(loss))


def test_supcon_errors(ops):
    with pytest.raises(ValueError):
        ops.supcon(torch.zeros(4, 8, device='cuda'), torch.zeros(4, dtype=torch.long, device='cuda'), 0.07)
    with pytest.raises(ValueError):
        ops.supcon(torch.zeros(4, 2, 8, device='cuda'), torch.zeros(5, dtype=torch.long, device='cuda'), 0.07)


def test_rows_and_sgd(ops):
    rs = np.random.RandomState(3)
    src = dev(rs.standard_normal((500, 3, 32, 32)).astype(np.float32))
    lab = dev(rs.randint(0, 100, 500))
    idx = dev(rs.choice(500, 110, replace=False))
    torch.testing.assert_close(ops.gather_rows(src, idx), src[idx], rtol=0, atol=0)
    torch.testing.assert_close(ops.gather_rows(lab, idx), lab[idx], rtol=0, atol=0)
    odd = dev(rs.standard_normal((50, 7)).astype(np.float32))          # 28-byte rows: 4-byte path
    torch.testing.assert_close(ops.gather_rows(odd, idx[:20] % 50), odd[idx[:20] % 50], rtol=0, atol=0)
    dst = src.clone()
    new = dev(rs.standard_normal((110, 3, 32, 32)).astype(np.float32))
    ops.scatter_rows(dst, idx, new)
    ref = src.clone()
    ref[idx] = new
    torch.testing.assert_close(dst, ref, rtol=0, atol=0)
    p, gr = dev(rs.standard_normal(1109240).astype(np.float32)), dev(rs.standard_normal(1109240).astype(np.float32))
    out = torch.empty_like(p)
    ops.sgd_step(p, gr, 0.1, 0.0, out=out)
    torch.testing.assert_close(out, p - 0.1 * gr, rtol=1e-6, atol=1e-7)
    ops.sgd_step(p, gr, 0.05, 1e-4, out=out)
    torch.testing.assert_close(out, p - 0.05 * (gr + 1e-4 * p), rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize('n,hw', [(57, 32), (9, 84), (3, 50)])
def test_stream_prepare_matches_totensor(ops, n, hw):
    """uint8 HWC -> fp32 CHW /255 + shuffle, bit-identical to torchvision's ToTensor on the CPU
    (continuum/data_utils.py:38-54; utils/setup_elements.py:29-43)."""
    from torchvision import transforms
    rs = np.random.RandomState(n)
    x = rs.randint(0, 256, (n, hw, hw, 3)).astype(np.uint8)
    x[0] = 255; x[1] = 0
    perm = rs.permutation(n)[: n - 2]
    got = ops.stream_prepare(torch.from_numpy(x).cuda(), torch.from_numpy(perm).cuda()).cpu()
    tt = transforms.ToTensor()
    ref = torch.stack([tt(x[i]) for i in perm])
    assert torch.equal(got, ref)
    ident = ops.stream_prepare(torch.from_numpy(x).cuda()).cpu()
    assert torch.equal(ident, torch.stack([tt(x[i]) for i in range(n)]))


@pytest.mark.parametrize('flip', [False, True])
def test_agem_projection(ops, flip):
    """agents/agem.py:73-80 on flat gradient vectors: projection iff the inner product is negative."""
    rs = np.random.RandomState(11)
    g = rs.standard_normal(1109240).astype(np.float32)
    r = rs.standard_normal(1109240).astype(np.float32)
    if (np.dot(g.astype(np.float64), r.astype(np.float64)) < 0) != flip:
        r = -r
    out, dots = ops.agem_project(dev(g), dev(r), want_dots=True)
    prod, prod_ref = np.dot(g.astype(np.float64), r.astype(np.float64)), np.dot(r.astype(np.float64), r.astype(np.float64))
    ref = g - (prod / prod_ref) * r if prod < 0 else g
    np.testing.assert_allclose(dots.cpu().numpy(), [prod, prod_ref], rtol=1e-5)
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-5, atol=1e-6)
    # in place on the reference-gradient arena, and deterministic
    arena = dev(r).clone()
    ops.agem_project(dev(g), arena, out=arena)
    assert torch.equal(arena, out)
