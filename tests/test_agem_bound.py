"""CPU: the rounding bound tests/test_gpu_agem_fp64.py holds the A-GEM projection kernel to (project_bound), and its
bit-exact check (the fp32 arithmetic of fl32(P / R), fused or not), against a numpy emulation of the kernel:
per-CTA fp64 partials over a grid-stride loop, re-reduced in CTA order, the fp64 quotient rounded to fp32, then
g_i - c r_i with or without a fused multiply-add.  The bound must hold for both forms without the GPU test's factor 2,
and the check must refuse the arithmetic of three faults: the decision taken with <=, a coefficient formed from
fp32-rounded dots, and a re-reduction that drops the last partial."""
import numpy as np
import pytest

import test_gpu_agem_fp64 as t

GRID = 264                     # 2 x 132 SMs (H100 SXM); any grid gives another fp64 summation order


def kernel_dots(g, r, grid=GRID, drop_last=False):
    """agem_dots_kernel + the re-reduction of agem_apply_kernel: (prod, prod_ref) in fp64."""
    g64, r64 = g.astype(np.float64), r.astype(np.float64)
    n = g.size
    stride = grid * 256
    pad = (-n) % stride
    a = np.concatenate([g64 * r64, np.zeros(pad)]).reshape(-1, grid, 256).sum(axis=0)     # per thread, loop order
    b = np.concatenate([r64 * r64, np.zeros(pad)]).reshape(-1, grid, 256).sum(axis=0)
    pa, pb = a.sum(axis=1), b.sum(axis=1)                                                  # per CTA
    last = grid - 1 if drop_last else grid
    P = R = 0.0
    for k in range(last):
        P += pa[k]
        R += pb[k]
    return P, R


def kernel(g, r, fused, le=False, fp32_dots=False, drop_last=False):
    P, R = kernel_dots(g, r, drop_last=drop_last)
    project = P <= 0 if le else P < 0
    if not project:
        return g.copy()
    with np.errstate(invalid='ignore', divide='ignore'):
        c = np.float32(np.float32(P) / np.float32(R)) if fp32_dots else np.float32(P / R)
    return t.emulate(g, r, c, fused)


LENGTHS = [1, 31, 257, GRID * 256 - 1, GRID * 256 + 1, 300007]


def rows():
    for n in LENGTHS:
        yield from ((n, name, g, r) for name, g, r in t.synthetic_rows(n, 100 + n % 97))


@pytest.mark.parametrize('fused', [True, False])
def test_bound_holds_for_the_emulated_kernel(fused):
    worst = 0.0
    for n, name, g, r in rows():
        out = kernel(g, r, fused)
        f = t.project_bound(g, r)
        assert f['P'] == 0.0 or abs(f['P']) > f['eP'], (n, name)
        if not f['project']:
            assert np.array_equal(out.view(np.int32), g.view(np.int32)), (n, name)
            continue
        ratio = np.abs(out.astype(np.float64) - f['ref']) / f['bound']
        assert ratio.max() <= 1.0, (n, name, ratio.max())
        worst = max(worst, float(ratio.max()))
        t.check_projection(g, r, out, None, (n, name))
    assert worst > 0.05            # the bound is not vacuous


def test_check_refuses_faulty_arithmetic():
    caught = {'le': 0, 'fp32_dots': 0, 'drop_last': 0}
    for n, name, g, r in rows():
        f = t.project_bound(g, r)
        for fault in caught:
            out = kernel(g, r, True, **{fault: True})
            P, R = kernel_dots(g, r, drop_last=fault == 'drop_last')
            try:
                t.check_projection(g, r, out, np.array([P, R], np.float32), (n, name))
            except AssertionError:
                caught[fault] += 1
    assert all(v > 0 for v in caught.values()), caught
