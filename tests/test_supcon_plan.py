"""CPU: b200ocl_supcon_plan, the host-only hook that reports which SupCon kernels a call launches (the same function
b200ocl_supcon launches through), over the SM counts of the H100 PCIe (114), H100 SXM (132) and a 148-SM part, every
d from 1 to 1024, aligned and misaligned pointers, and anchor counts A = B * V up to 10 000 (no GPU needed: nothing
is launched).  Also pins the blocked torch form of the fp64 SupCon oracle to the dense numpy one."""
import numpy as np
import pytest

SMS = (114, 132, 148)
A_MAX = 10000
MBAR_TX_MAX = (1 << 20) - 1          # an mbarrier's transaction count is a 20-bit field


def anchor_counts(sms):
    """Every A up to one past the 16-anchor-unit bound (where the resident / ring-16 choice moves) and past one full
    wave of 64-anchor units, then a stride up to A_MAX."""
    dense = list(range(1, 64 * sms + 66))
    return dense + list(range(dense[-1] + 1, A_MAX, 37)) + [A_MAX]


def fused_widths():
    return [d for d in range(4, 257, 4)]


def partial_entries(B, V, d):
    from b200ocl import _native
    A = B * V
    ws = _native.lib().b200ocl_supcon_workspace_bytes(B, V, d)
    return (ws - 256) // 4 - 2 * A          # floats after lse [A] and npos [A]


@pytest.mark.parametrize('sms', SMS)
def test_fused_plans_fit(sms):
    """Every fused plan: shared memory within the limit the launcher raises the kernel to, grid <= SMs (the grid-wide
    wait needs every CTA resident), units spread over the grid, n_units within the workspace's loss partials, every
    mbarrier transaction below the hardware limit; the resident family only up to its 200 KB bound."""
    from b200ocl import ops
    seen = set()
    for d in fused_widths():
        for A in anchor_counts(sms):
            L = ops.supcon_plan(A, 1, d, True, sms)
            where = (sms, A, d, L.name)
            assert L.sms == sms and L.name != 'fallback', where
            assert L.nc == (d + 63) // 64 and L.dch == 0, where
            assert L.smem_bytes <= L.smem_limit == 227 * 1024, where
            assert 1 <= L.grid <= sms and L.grid == min(L.n_units, sms), where
            assert L.n_units == -(-A // (16 * L.rm)), where
            assert L.units_per_cta == -(-L.n_units // L.grid), where
            assert 0 < L.tx_bytes <= MBAR_TX_MAX, where
            if L.name == 'resident':
                assert (L.rm, L.rn) == (1, 4) and A <= 16 * sms and L.smem_bytes <= 200 * 1024, where
                assert L.tx_bytes == A * d * 4, where
            elif L.name == 'ring16':
                assert (L.rm, L.rn) == (1, 2) and A <= 16 * sms, where
            else:
                assert (L.rm, L.rn) == (4, 4) and A > 16 * sms, where
            seen.add(L.kernel)
        for V in (1, 2, 3):                          # only A matters
            B = 4001 // V
            assert ops.supcon_plan(B, V, d, True, sms).kernel == ops.supcon_plan(B * V, 1, d, True, sms).kernel
    assert seen == {(f, nc) for f in ('resident', 'ring16', 'ring64') for nc in (1, 2, 3, 4)}, sorted(seen)
    # partials: the largest n_units of each width is at the largest A
    for d in fused_widths():
        for B, V in [(A_MAX, 1), (A_MAX // 2, 2), (3333, 3), (16 * sms, 1), (16 * sms + 1, 1)]:
            assert ops.supcon_plan(B, V, d, True, sms).n_units <= partial_entries(B, V, d), (sms, B, V, d)


@pytest.mark.parametrize('sms', SMS)
def test_fallback_plans_fit(sms):
    """d not a multiple of 4, d > 256 or a misaligned pointer: the two-kernel fallback, one 8-anchor block per CTA, with
    DCH = 4 / 8 / 16 / 32 columns per lane covering d (32 * DCH >= d), in the shared memory it asks for."""
    from b200ocl import ops
    seen = set()
    for d in range(1, 1025):
        for aligned in (True, False):
            fused = aligned and d % 4 == 0 and d <= 256
            for A in (1, 7, 8, 9, 16 * sms + 1, A_MAX):
                L = ops.supcon_plan(A, 1, d, aligned, sms)
                where = (sms, A, d, aligned, L.name)
                if fused:
                    assert L.name != 'fallback', where
                    continue
                assert L.name == 'fallback' and L.nc == 0 and L.tx_bytes == 0, where
                assert L.dch in (4, 8, 16, 32) and 32 * L.dch >= d and (L.dch == 4 or 16 * L.dch < d), where
                assert L.grid == L.n_units == -(-A // 8) and L.units_per_cta == 1, where
                assert L.n_units <= partial_entries(A, 1, d), where
                assert L.smem_bytes <= L.smem_limit == 200 * 1024, where
                seen.add(L.kernel)
    assert seen == {('fallback', c) for c in (4, 8, 16, 32)}


@pytest.mark.parametrize('sms', SMS)
def test_production_shapes(sms):
    """Where SCR's own SupCon calls land: batches of 11..110 two-view pairs (A = 22..220) at d = 128 (mlp head) on the
    resident kernel with NC = 2; head 'None' at 32x32 (d = 160) on the resident kernel with NC = 3; head 'None' at
    84x84 (d = 640) on the fallback with DCH = 32."""
    from b200ocl import ops
    for B in range(11, 111):
        assert ops.supcon_plan(B, 2, 128, True, sms).kernel == ('resident', 2), B
        assert ops.supcon_plan(B, 2, 160, True, sms).kernel == ('resident', 3), B
        assert ops.supcon_plan(B, 2, 640, True, sms).kernel == ('fallback', 32), B


def test_plan_refuses_bad_arguments():
    from b200ocl import _native, ops
    for args in [(0, 2, 128), (10, 0, 128), (10, 2, 0), (10, 2, 1025)]:
        with pytest.raises(_native.NativeError):
            ops.supcon_plan(*args, sms=132)
    with pytest.raises(_native.NativeError):
        ops.supcon_plan(10, 2, 128, True, -1)


@pytest.mark.parametrize('finite_grad', [False, True])
def test_blocked_oracle_matches_dense(finite_grad):
    """oracle.supcon's blocked torch form (used on the GPU for large anchor sets) against its dense numpy form, with a
    singleton class at V = 1 (an anchor without positives) among the cases."""
    import torch
    from oracle import supcon as osup
    rs = np.random.RandomState(3)
    for B, V, d, T, blk in [(37, 2, 20, 0.07, 16), (50, 1, 9, 0.5, 7), (13, 3, 64, 0.05, 1000)]:
        f = rs.standard_normal((B, V, d))
        f = (3 * f / np.linalg.norm(f, axis=2, keepdims=True)).astype(np.float32)
        y = rs.randint(0, 6, B)
        if V == 1:
            y[0] = 99
        loss, grad = osup.supcon_loss_and_grad(f, y, T, finite_grad=finite_grad)
        tl, tg = osup.supcon_loss_and_grad_torch(torch.from_numpy(f), torch.from_numpy(y), T, finite_grad=finite_grad,
                                                 block=blk)
        if V == 1:
            assert np.isnan(loss) and np.isnan(tl)
            assert np.isfinite(grad).all() == finite_grad
        else:
            assert abs(tl - loss) <= 1e-12 * abs(loss)
        np.testing.assert_allclose(tg.numpy(), grad, rtol=1e-10, atol=1e-13)


def test_blocked_oracle_drop_last_contrast():
    """drop_last_contrast is the fp64 loss and gradient with the last anchor out of every contrast set: the dense
    oracle on that problem written out by hand (numerical derivative of the loss it defines)."""
    import torch
    from oracle import supcon as osup
    rs = np.random.RandomState(4)
    B, V, d, T = 6, 2, 5, 0.3
    f = rs.standard_normal((B, V, d))
    y = rs.randint(0, 2, B)

    def loss_of(x):
        return osup.supcon_loss_and_grad_torch(torch.from_numpy(x), torch.from_numpy(y), T, drop_last_contrast=True)[0]

    loss, grad = osup.supcon_loss_and_grad_torch(torch.from_numpy(f), torch.from_numpy(y), T, drop_last_contrast=True)
    num = np.zeros_like(f)
    h = 1e-6
    for idx in np.ndindex(f.shape):
        fp, fm = f.copy(), f.copy()
        fp[idx] += h
        fm[idx] -= h
        num[idx] = (loss_of(fp) - loss_of(fm)) / (2 * h)
    np.testing.assert_allclose(grad.numpy(), num, rtol=1e-6, atol=1e-8)
    full, _ = osup.supcon_loss_and_grad(f, y, T)
    assert abs(loss - full) > 1e-3
