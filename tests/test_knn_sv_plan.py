"""CPU: b200ocl_knn_sv_plan, the host-only hook that reports which kNN-SV kernel a call launches (the same function
b200ocl_knn_sv launches through), over the SM counts of the H100 PCIe (114), H100 SXM (132) and a 148-SM part: every C
from 1 to 1024 and every power-of-two edge (+-1) up to 262 144, E across 8 * SMs and multiples of the grid, d from 1 to
4096, aligned and misaligned pointers (no GPU needed: nothing is launched).  Also pins the oracle pieces the GPU tests
rest on: the fp32 fmaf emulation against exact rational arithmetic, the emulated distance chains of both kernels, and
the blocked torch fp64 form against the numpy form and the per-row loop."""
import math
from fractions import Fraction

import numpy as np
import pytest

SMS = (114, 132, 148)
C_MAX, D_MAX_LARGE, FUSED_MAX = 262144, 4096, 1024
SMEM_HW = 227 * 1024


def row_counts(sms):
    return sorted({1, 2, 7, 8, 9, 31, 32, 33, 8 * sms - 1, 8 * sms, 8 * sms + 1, 16 * sms - 1, 16 * sms, 16 * sms + 1,
                   32 * sms, 32 * sms + 1, 64 * sms + 5, 50000})


def large_counts():
    out = set()
    for e in range(10, 19):
        out.update({(1 << e) - 1, 1 << e, (1 << e) + 1})
    return sorted(c for c in out if FUSED_MAX < c <= C_MAX)


def check_fused(L, E, C, d, aligned, want_red, sms):
    where = (sms, E, C, d, aligned, want_red)
    kpl = next(p for p in (1, 2, 4, 8, 16, 32) if 32 * p >= C)
    te = 8 if E <= 8 * sms else (16 if kpl == 32 else 32)
    assert L.name == 'fused' and L.sms == sms, where
    assert (L.kpl, L.te, L.cpad) == (kpl, te, 32 * kpl), where
    assert L.wide == (kpl == 32 and te == 16 and d % 8 == 0 and aligned), where
    assert L.smem_bytes <= L.smem_limit <= SMEM_HW, where
    assert L.n_tiles == -(-E // te), where
    assert 1 <= L.grid <= sms and L.grid == min(L.n_tiles, sms), where
    assert L.tiles_per_cta == -(-L.n_tiles // L.grid), where
    assert L.part_bytes == (L.grid * 3 * C * 4 if want_red else 0), where
    assert 256 + L.part_bytes <= L.workspace_bytes, where
    assert L.key_bytes == 0 and L.far_stages == 0, where


def check_large(L, E, C, d, want_red, sms):
    where = (sms, E, C, d, want_red)
    cpad = 1 << max(10, math.ceil(math.log2(C)))
    S = min(cpad, 16384)
    m, s = int(math.log2(cpad)), int(math.log2(S))
    assert L.name == 'large' and L.sms == sms, where
    assert (L.cpad, L.block_keys) == (cpad, S) and L.cpad >= C, where
    assert L.far_stages == (m - s) * (m - s + 1) // 2, where
    assert L.grid == min(E, sms) and L.tiles_per_cta == -(-E // L.grid), where
    assert L.smem_bytes == S * 8 + (d + 1024) * 4 and L.smem_bytes <= L.smem_limit <= SMEM_HW, where
    assert L.part_bytes == (L.grid * 3 * C * 4 if want_red else 0), where
    assert 256 + L.part_bytes <= L.key_offset and L.key_offset % 256 == 0, where
    assert L.key_bytes == L.grid * cpad * 8 and L.key_offset + L.key_bytes <= L.workspace_bytes, where


@pytest.mark.parametrize('sms', SMS)
def test_fused_plans_fit(sms):
    """C <= 1024: KPL from C, TE from E against 8 * SMs, the wide phase 1 only for KPL = 32 / TE = 16 with d % 8 == 0
    and aligned pointers; shared memory within the limit the launcher sets, grid <= SMs, partials in the workspace."""
    from b200ocl import ops
    seen = set()
    for C in range(1, FUSED_MAX + 1):
        for E in row_counts(sms):
            for d, aligned in [(8, True), (12, True), (8, False)]:
                for want_red in (True, False):
                    L = ops.knn_sv_plan(E, C, d, aligned, want_red, sms)
                    check_fused(L, E, C, d, aligned, want_red, sms)
                    seen.add(L.kernel)
    want = {(p, 8, 'rows') for p in (1, 2, 4, 8, 16, 32)} | {(p, 32, 'rows') for p in (1, 2, 4, 8, 16)}
    want |= {(32, 16, 'rows'), (32, 16, 'wide')}
    assert seen == want, sorted(seen ^ want)
    for d in range(1, D_MAX_LARGE + 1):              # d only moves the phase-1 form
        for aligned in (True, False):
            check_fused(ops.knn_sv_plan(8 * sms + 1, 1000, d, aligned, True, sms), 8 * sms + 1, 1000, d, aligned, True,
                        sms)


@pytest.mark.parametrize('sms', SMS)
def test_large_plans_fit(sms):
    """C > 1024: the scratch-line kernel; key lines and partials inside the workspace the query gives at that SM count,
    shared memory within the 200 KB the launcher raises, d up to 4096."""
    from b200ocl import ops
    seen = set()
    for C in large_counts():
        for E in row_counts(sms):
            for d in (1, 33, 1024, 1025, 4096):
                for want_red in (True, False):
                    L = ops.knn_sv_plan(E, C, d, True, want_red, sms)
                    check_large(L, E, C, d, want_red, sms)
                    seen.add(L.far_stages)
    assert seen == {0, 1, 3, 6, 10}, sorted(seen)


def test_plan_matches_the_workspace_query():
    """sms = 0 plans for the device in use, and its workspace is what b200ocl_knn_sv_workspace_bytes returns."""
    from b200ocl import _native, ops
    lib = _native.lib()
    for E, C, d in [(1, 1, 1), (110, 160, 160), (51, 1000, 512), (3, 1025, 16), (2, C_MAX, 8)]:
        L = ops.knn_sv_plan(E, C, d)
        assert L.sms >= 1 and L.workspace_bytes == lib.b200ocl_knn_sv_workspace_bytes(E, C, d), (E, C, d)


def test_plan_refuses_bad_arguments():
    from b200ocl import _native, ops
    for args in [(0, 10, 8), (10, 0, 8), (10, 10, 0), (10, C_MAX + 1, 8), (10, FUSED_MAX + 1, D_MAX_LARGE + 1)]:
        with pytest.raises(_native.NativeError):
            ops.knn_sv_plan(*args, sms=132)
    with pytest.raises(_native.NativeError):
        ops.knn_sv_plan(10, 10, 8, sms=-1)
    assert ops.knn_sv_plan(10, FUSED_MAX, D_MAX_LARGE + 1, sms=132).name == 'fused'   # the fused kernel takes any d
    assert ops.knn_sv_plan(10, C_MAX, D_MAX_LARGE, sms=132).name == 'large'


# ----------------------------------------------------------------------------------------------- oracle pieces

def fp32_of(x):
    """Correctly rounded (ties to even) fp32 of a Fraction."""
    c = np.float32(float(x))
    cands = [np.nextafter(c, np.float32(-np.inf)), c, np.nextafter(c, np.float32(np.inf))]
    best = min(abs(Fraction(float(v)) - x) for v in cands)
    near = [v for v in cands if abs(Fraction(float(v)) - x) == best]
    if len(near) == 1:
        return near[0]
    return next(v for v in near if v.view(np.uint32) % 2 == 0)


def fmaf_exact(df, acc):
    return fp32_of(Fraction(float(df)) ** 2 + Fraction(float(acc)))


def test_fmaf_emulation_random():
    import torch
    from oracle import knn_sv as oknn
    rs = np.random.RandomState(0)
    n = 4000
    df = (rs.standard_normal(n) * np.exp2(rs.randint(-20, 20, n))).astype(np.float32)
    acc = (np.abs(rs.standard_normal(n)) * np.exp2(rs.randint(-40, 40, n))).astype(np.float32)
    acc[::7] = 0
    got = oknn.fmaf_sq(torch.from_numpy(df), torch.from_numpy(acc)).numpy()
    want = np.array([fmaf_exact(a, b) for a, b in zip(df, acc)], dtype=np.float32)
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))


def test_fmaf_emulation_midpoints():
    """df = m 2^j with m odd in [4097, 5792]: df^2 is a 25-bit odd multiple of 2^(2j), exactly halfway between two fp32
    values.  acc = 0 rounds it to even; a tiny acc of either sign (below fp64's half ulp of df^2, so that the fp64 sum
    is the midpoint itself and only TwoSum's error term sees it) decides the direction.  A plain fp64 rounding gets
    those wrong."""
    import torch
    from oracle import knn_sv as oknn
    dfs, accs = [], []
    for m in range(4097, 5793, 34):
        m += (m + 1) % 2                               # odd
        for j in (-30, -12, 0, 7):
            df = np.float32(m * 2.0 ** j)
            tiny = np.float32(2.0 ** (2 * j + 24 - 60))
            for acc in (np.float32(0), tiny, -tiny):
                dfs.append(df)
                accs.append(acc)
    df, acc = np.array(dfs, dtype=np.float32), np.array(accs, dtype=np.float32)
    got = oknn.fmaf_sq(torch.from_numpy(df), torch.from_numpy(acc)).numpy()
    want = np.array([fmaf_exact(a, b) for a, b in zip(df, acc)], dtype=np.float32)
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    naive = (df.astype(np.float64) ** 2 + acc.astype(np.float64)).astype(np.float32)
    assert (naive != want).sum() >= len(want) // 3     # the cases do reach the midpoint rule


def test_distance_chains():
    """The fused chain and the large kernel's 32 lane chains + xor butterfly, written out with exact fmaf and numpy fp32
    adds, against the vectorised emulations."""
    import torch
    from oracle import knn_sv as oknn
    rs = np.random.RandomState(1)
    for d in (1, 31, 40, 70):
        ef = np.maximum(rs.standard_normal((2, d)), 0).astype(np.float32)
        cf = np.maximum(rs.standard_normal((3, d)), 0).astype(np.float32)
        fused = oknn.dist_fp32_fused(torch.from_numpy(ef), torch.from_numpy(cf)).numpy()
        large = oknn.dist_fp32_large(torch.from_numpy(ef), torch.from_numpy(cf)).numpy()
        for e in range(2):
            for c in range(3):
                acc = np.float32(0)
                for f in range(d):
                    acc = fmaf_exact(ef[e, f] - cf[c, f], acc)
                assert fused[e, c].view(np.uint32) == acc.view(np.uint32), (d, e, c)
                lanes = []
                for ln in range(32):
                    a = np.float32(0)
                    for f in range(ln, d, 32):
                        a = fmaf_exact(ef[e, f] - cf[c, f], a)
                    lanes.append(a)
                lanes = np.array(lanes, dtype=np.float32)
                for o in (16, 8, 4, 2, 1):
                    lanes = lanes + lanes[np.arange(32) ^ o]
                assert large[e, c].view(np.uint32) == lanes[0].view(np.uint32), (d, e, c)


def test_kernel_order_breaks_ties_by_index():
    import torch
    from oracle import knn_sv as oknn
    cf = torch.tensor([[1.0], [0.0], [1.0], [2.0], [0.0]])
    ef = torch.tensor([[0.0], [1.0]])
    for large in (False, True):
        order, _ = oknn.kernel_order(ef, cf, large=large)
        assert order.tolist() == [[1, 4, 0, 2, 3], [0, 2, 1, 3, 4]]


def test_torch_form_matches_numpy_and_row_loop():
    import torch
    from oracle import knn_sv as oknn
    rs = np.random.RandomState(2)
    for E, C, d, k, block in [(7, 1, 3, 1, 3), (9, 40, 5, 3, 4), (5, 33, 2, 50, 64), (12, 200, 8, 5, 5)]:
        ef = rs.randint(0, 3, (E, d)).astype(np.float32)       # integer features: exact ties
        cf = rs.randint(0, 3, (C, d)).astype(np.float32)
        ey, cy = rs.randint(0, 4, E), rs.randint(0, 4, C)
        sv_np, order, dist = oknn.knn_sv_matrix(ef, ey, cf, cy, k)
        sv_t, abs_sum = oknn.knn_sv_torch(torch.from_numpy(order), torch.from_numpy(ey), torch.from_numpy(cy), k,
                                          block=block)
        np.testing.assert_allclose(sv_t.numpy(), sv_np, rtol=0, atol=1e-15)
        for r in range(E):
            np.testing.assert_allclose(sv_t[r].numpy(), oknn.knn_sv_row_loop(dist[r], ey[r], cy, k), rtol=0, atol=1e-15)
        assert (abs_sum.numpy() >= np.abs(sv_np).max(1) - 1e-15).all()
        korder, _ = oknn.kernel_order(torch.from_numpy(ef), torch.from_numpy(cf))
        assert np.array_equal(korder.numpy(), order)          # exact fp32 distances: the kernel order is the fp64 one
