"""GPU: b200ocl_knn_sv against the float64 oracle (oracle/knn_sv.py) at every launch it can take on the card in use,
every row compared, none excused.

b200ocl_knn_sv picks (csrc/knn_sv.cu, knn_plan) the fused kernel with KPL = 1..32 keys per lane and TE = 8 eval rows
per tile when E <= 8 * SMs, else TE = 32 (16 for KPL = 32, with the wide phase 1 when d % 8 == 0 and both feature
pointers are 16-byte aligned, the row-tiled one otherwise); or, for C > 1024, the scratch-line kernel, which sorts in
one shared-memory block up to Cpad = 16384 and needs far-partner stages through global memory beyond.  The cases are
built from the device's SM count and test_cases_reach_every_launch checks through the host-only hook
b200ocl_knn_sv_plan that they reach every one of those forms.

Ordering.  The kernels rank candidates by their fp32 distances, ties lowest index first.  oracle.knn_sv.kernel_order
reproduces those fp32 distances bit for bit (the fused kernel's sequential fmaf chain, the large kernel's 32
lane-strided chains and xor butterfly), so its stable sort is the kernel's order; the fp64 recurrence on that order
leaves only the rounding of the recurrence between kernel and oracle, and no row needs excusing.  The rank probes check
the order exactly: with k = 1 and one matching candidate per row at rank q, the kernel's SV of that candidate is the
single term fl32(1 / q) plus exact zeros, so it must equal np.float32(1) / np.float32(q) bit for bit.

Per-row bound (EPS = 2^-24, gamma_n = n EPS / (1 - n EPS)).  Each SV entry is a suffix sum of the terms
t_i = +-min(i, k) / (i k).  The kernel forms each term with two roundings (fl32(rank * k), then the division; the sign
is exact) and adds it in at most n fp32 additions:
  fused  n = KPL + 6: KPL in-lane additions (the run starts at 0), 5 levels of the shuffle suffix scan over the lane
         totals, and the addition of the lanes above;
  large  n = 2 L + 38, L = Cpad / 1024: the per-thread run of pass 1 (L), the 5-level block scan, its exclusive
         subtraction incl - v, the carry chain over the 32 blocks (<= 31), the carry's addition, and the run of pass 2
         (L).
Every term then carries at most n + 2 factors (1 + delta), |delta| <= EPS, so |SV - SV64| <= gamma_(n+2) sum_i |t_i|;
the fp64 oracle's cumsum adds C 2^-52 sum_i |t_i|.  Column sums: each partial adds at most R rows in fp32 (fused: the
TM = TE / 8 rows of each tile a warp takes times the tiles per CTA, then the 8-warp combine; large: the rows of one
CTA), the partials are added in fp64 and rounded once, so |sum - sum64| <= sum_r bound_r + gamma_(R+2) sum_r |SV64|.

The derived bound is 10-100x looser than what the kernels do, so every row is also held to ROW_TOL, about 3x the
largest error measured on an H100 80GB HBM3 (SXM, 132 SMs, 700 W power limit) over these cases [in brackets]."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import aser as oaser
from oracle import knn_sv as oknn

pytestmark = pytest.mark.gpu

ROW_TOL = 3e-7          # max |SV - SV64| over a row       [1.0e-7, L-far-multi; the fused kernel <= 5.9e-8]
SUM_TOL = 1.5e-6        # |sum - sum64| / max(1, |sum64|)  [4.9e-7, f2-32]


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import ops as _ops
    return _ops


def device_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def case_list(sms):
    """(tag, E, C, d, k, regime, misaligned).  Regimes: 'dense' integer features in {0,1,2} (many exact ties),
    'sparse' integers in 0..63 (a few ties; d * 63^2 < 2^24, so fp32 distances are exact), 'relu' ReLU(N(0,1)),
    'probe' ReLU features with one matching candidate per row at a chosen rank and k = 1."""
    E8, E32 = 8 * sms + 1, 64 * sms + 5
    return [
        # TE = 8, every KPL
        ('f1-8', 40, 20, 6, 3, 'dense', False),
        ('f2-8', 19, 50, 40, 1, 'relu', False),
        ('f4-8', 33, 128, 9, 127, 'sparse', False),
        ('f8-8', 19, 160, 40, 3, 'relu', False),
        ('f16-8', 19, 300, 33, 299, 'relu', False),
        ('f32-8', 19, 1000, 40, 2000, 'relu', False),
        ('f32-8-dense', 60, 1024, 5, 1, 'dense', False),
        # TE = 32 (16 for KPL = 32): one tile per CTA
        ('f1-32', E8, 32, 16, 3, 'sparse', False),
        ('f2-32', E8, 64, 24, 1, 'relu', False),
        ('f4-32', E8, 100, 7, 99, 'dense', False),
        ('f8-32', E8, 256, 12, 3, 'relu', False),
        ('f16-32', E8, 512, 16, 600, 'relu', False),
        ('f32-16-wide', E8, 1000, 16, 3, 'relu', False),
        ('f32-16-rows-d', E8, 1000, 20, 3, 'relu', False),
        ('f32-16-rows-mis', E8, 1000, 16, 3, 'relu', True),
        # several tiles per CTA, ragged last tile
        ('f8-32-multi', E32, 200, 8, 3, 'dense', False),
        ('f32-16-multi', 32 * sms + 3, 700, 24, 5, 'relu', False),
        ('f32-16-multi-mis', 32 * sms + 3, 700, 24, 5, 'sparse', True),
        # the scratch-line kernel
        ('L-one-block', 7, 3000, 64, 5, 'relu', False),
        ('L-one-block-multi', sms + 9, 1500, 40, 1500, 'dense', False),
        ('L-far', 3, 20000, 32, 3, 'relu', False),
        ('L-far-multi', sms + 2, 17000, 8, 1, 'sparse', False),
        ('L-wide-d', 5, 2048, 1100, 3, 'relu', False),
        ('L-max', 3, 262144, 8, 3, 'relu', False),
        # rank probes
        ('probe-fused', 40, 1000, 16, 1, 'probe', False),
        ('probe-one-block', 12, 16384, 8, 1, 'probe', False),
        ('probe-max', 10, 262144, 8, 1, 'probe', False),
    ]


def storage(x, misaligned):
    """x (fp32, [n, d]) on the device; misaligned: one element into its storage, so not 16-byte aligned."""
    if not misaligned:
        return x.contiguous()
    store = torch.empty(x.numel() + 1, dtype=torch.float32, device=x.device)
    v = store[1:].view(x.shape)
    v.copy_(x)
    return v


def probe_ranks(C, E):
    base = [1, 2, 3, C // 2, C - 2, C - 1, C]
    rs = np.random.RandomState(C)
    return (base + sorted(rs.randint(1, C + 1, max(0, E - len(base))).tolist()))[:E]


def make_inputs(case, seed):
    tag, E, C, d, k, regime, misaligned = case
    g = torch.Generator(device='cuda').manual_seed(seed)
    if regime == 'dense':
        ef, cf = (torch.randint(0, 3, (n, d), device='cuda', generator=g).float() for n in (E, C))
    elif regime == 'sparse':
        ef, cf = (torch.randint(0, 64, (n, d), device='cuda', generator=g).float() for n in (E, C))
    else:
        ef, cf = (torch.relu(torch.randn(n, d, device='cuda', generator=g)) for n in (E, C))
    if regime == 'probe':
        cy = torch.arange(C, device='cuda')                      # every label once
        order, _ = oknn.kernel_order(ef, cf)
        q = torch.tensor(probe_ranks(C, E), device='cuda')
        ey = order[torch.arange(E, device='cuda'), q - 1]        # row r matches the candidate at rank q_r only
    else:
        ncls = 3 if regime == 'dense' else 7
        ey = torch.randint(0, ncls, (E,), device='cuda', generator=g)
        cy = torch.randint(0, ncls, (C,), device='cuda', generator=g)
    return storage(ef, misaligned), ey, storage(cf, misaligned), cy


def plan_of(ops, ef, cf, want_red=True):
    aligned = ef.data_ptr() % 16 == 0 and cf.data_ptr() % 16 == 0
    return ops.knn_sv_plan(ef.shape[0], cf.shape[0], ef.shape[1], aligned, want_red, 0)


def reachable(ops, sms):
    """Every kernel form the hook reports on this card."""
    out = set()
    for C in (1, 33, 65, 129, 257, 513):
        for E in (1, 8 * sms + 1):
            out.add(ops.knn_sv_plan(E, C, 8, True, True, sms).kernel)
    for d, aligned in [(8, True), (12, True), (8, False)]:
        out.add(ops.knn_sv_plan(8 * sms + 1, 1000, d, aligned, True, sms).kernel)
        out.add(ops.knn_sv_plan(1, 1000, d, aligned, True, sms).kernel)
    return out


def test_cases_reach_every_launch(ops):
    sms = device_sms()
    want = reachable(ops, sms)
    got = {}
    plans = []
    for case in case_list(sms):
        tag, E, C, d = case[:4]
        ef = storage(torch.zeros(E, d, device='cuda'), case[6])
        cf = storage(torch.zeros(C, d, device='cuda'), case[6])
        L = plan_of(ops, ef, cf)
        plans.append((tag, L))
        got.setdefault(L.kernel, []).append(tag)
    print('sms %d: %s' % (sms, sorted(got.items(), key=str)))
    fused = {kern for kern in got if kern[0] != 'large'}
    assert want <= fused, sorted(want - fused)
    assert len(want) == 13
    # CTAs that walk several tiles, the last one ragged, with the column reductions on
    multi = [(L, case[1]) for (_, L), case in zip(plans, case_list(sms))
             if L.name == 'fused' and L.tiles_per_cta >= 2 and L.te > 8]
    assert any(L.kpl == 32 for L, _ in multi) and any(L.kpl < 32 for L, _ in multi)
    assert all(E % L.te != 0 for L, E in multi)
    large = [L for _, L in plans if L.name == 'large']
    assert any(L.far_stages == 0 for L in large) and any(L.far_stages >= 1 for L in large)
    assert any(L.far_stages == 10 and L.cpad == 262144 for L in large)
    assert any(L.tiles_per_cta == 1 and L.grid < sms for L in large)
    assert any(L.tiles_per_cta >= 2 for L in large)
    assert any(L.tiles_per_cta >= 2 and L.far_stages >= 1 for L in large)
    assert any(case[3] > 1024 for case, (_, L) in zip(case_list(sms), plans) if L.name == 'large')


def reference(ops, ef, ey, cf, cy, k, L):
    order, _ = oknn.kernel_order(ef, cf, large=L.name == 'large')
    sv64, abs_sum = oknn.knn_sv_torch(order, ey, cy, k)
    return order, sv64, oknn.sv_row_bound(abs_sum, L, cf.shape[0])


def sum_bound(sv64, bound, L):
    R = L.tiles_per_cta * (L.te // 8) + 8 if L.name == 'fused' else L.tiles_per_cta
    return bound.sum() + oknn.gamma(R + 2) * sv64.abs().sum(0)


bits = lambda t: t.contiguous().view(torch.int32)


@pytest.mark.parametrize('idx', range(len(case_list(132))))        # the same number of cases on every SM count
def test_knn_sv_against_fp64(ops, idx):
    case = case_list(device_sms())[idx]
    tag, E, C, d, k, regime = case[:6]
    ef, ey, cf, cy = make_inputs(case, idx)
    L = plan_of(ops, ef, cf)
    full = ops.knn_sv(ef, ey, cf, cy, k, want_matrix=True, want_sum=True, want_max=True, want_min=True)
    sv = full['sv']
    order, sv64, bound = reference(ops, ef, ey, cf, cy, k, L)
    err = (sv.double() - sv64).abs().max(1).values
    worst = int(err.argmax())
    s64 = sv64.sum(0)
    serr = float(((full['sum'].double() - s64).abs() / s64.abs().clamp(min=1)).max())
    print('knn %-18s E=%5d C=%6d d=%4d k=%6d %-22s row err %.3g (bound %.3g) sum err %.3g'
          % (tag, E, C, d, k, L.kernel, float(err.max()), float(bound[worst]), serr))
    bad = torch.nonzero(err > bound).flatten()
    assert bad.numel() == 0, (tag, bad[:10].tolist(), err[bad[:10]].tolist())
    assert float(err.max()) <= ROW_TOL, (tag, worst, float(err.max()))
    if regime == 'probe':
        q = torch.tensor(probe_ranks(C, E), device='cuda')
        got = sv[torch.arange(E, device='cuda'), ey]
        want = (torch.ones(E) / q.float().cpu()).cuda()                     # fp32 division: fl32(1 / q)
        assert torch.equal(bits(got), bits(want)), (tag, q.tolist(), got.tolist())
    # column reductions: max / min are those of the kernel's own matrix, bit for bit, and within the bar of fp64
    assert torch.equal(bits(full['max']), bits(sv.max(0).values)), tag
    assert torch.equal(bits(full['min']), bits(sv.min(0).values)), tag
    bmax = float(bound.max())
    assert float((full['max'].double() - sv64.max(0).values).abs().max()) <= bmax, tag
    assert float((full['min'].double() - sv64.min(0).values).abs().max()) <= bmax, tag
    assert bool(((full['sum'].double() - s64).abs() <= sum_bound(sv64, bound, L)).all()), tag
    assert serr <= SUM_TOL, (tag, serr)
    # every output combination, repeat launches: the same bits
    for want_matrix in (False, True):
        for ws in (False, True):
            for wx in (False, True):
                for wn in (False, True):
                    if not (want_matrix or ws or wx or wn):
                        continue
                    o = ops.knn_sv(ef, ey, cf, cy, k, want_matrix=want_matrix, want_sum=ws, want_max=wx, want_min=wn)
                    for key, val in o.items():
                        assert torch.equal(bits(val), bits(full[key])), (tag, key, want_matrix, ws, wx, wn)
    # the other phase-1 form on the same data: the wide and row-tiled forms give the same bits
    if L.name == 'fused' and L.kpl == 32 and L.te == 16:
        mis = ef.data_ptr() % 16 != 0
        ef2, cf2 = (storage(ef.clone(), not mis), storage(cf.clone(), not mis))
        L2 = plan_of(ops, ef2, cf2)
        assert L2.wide != L.wide or d % 8
        o = ops.knn_sv(ef2, ey, cf2, cy, k, want_matrix=True, want_sum=True, want_max=True, want_min=True)
        for key, val in o.items():
            assert torch.equal(bits(val), bits(full[key])), (tag, 'other phase-1 form', key)


def test_bench_shape_sampled(ops):
    """The benchmarked sweep call (50 000 x 1000 x 512, k = 3: the wide phase 1, several tiles per CTA): every 97th
    row against fp64 on the kernel's order; reductions against the kernel's full matrix."""
    E, C, d, k = 50000, 1000, 512, 3
    g = torch.Generator(device='cuda').manual_seed(0)
    ef = torch.relu(torch.randn(E, d, device='cuda', generator=g))
    cf = torch.relu(torch.randn(C, d, device='cuda', generator=g))
    ey = torch.randint(0, 100, (E,), device='cuda', generator=g)
    cy = torch.randint(0, 100, (C,), device='cuda', generator=g)
    L = plan_of(ops, ef, cf)
    assert L.kernel == (32, 16, 'wide') and L.tiles_per_cta >= 2
    full = ops.knn_sv(ef, ey, cf, cy, k, want_matrix=True, want_sum=True, want_max=True, want_min=True)
    rows = torch.arange(0, E, 97, device='cuda')
    _, sv64, bound = reference(ops, ef[rows], ey[rows], cf, cy, k, L)
    err = (full['sv'][rows].double() - sv64).abs().max(1).values
    print('bench sample: %d rows, row err %.3g' % (rows.numel(), float(err.max())))
    assert bool((err <= bound).all()) and float(err.max()) <= ROW_TOL
    sv = full['sv']
    assert torch.equal(bits(full['max']), bits(sv.max(0).values))
    assert torch.equal(bits(full['min']), bits(sv.min(0).values))
    s = sv.double().sum(0)
    R = L.tiles_per_cta * 2 + 8
    assert bool(((full['sum'].double() - s).abs() <= oknn.gamma(R + 2) * sv.double().abs().sum(0)).all())


def test_refusals(ops):
    from b200ocl import _native
    ef, cf = torch.rand(4, 8, device='cuda'), torch.rand(10, 8, device='cuda')
    ey, cy = torch.zeros(4, dtype=torch.long, device='cuda'), torch.zeros(10, dtype=torch.long, device='cuda')
    for kw in ({'want_max': True}, {'want_min': True}):
        with pytest.raises(_native.NativeError):
            ops.knn_sv(ef[:0], ey[:0], cf, cy, 3, **kw)
    assert float(ops.knn_sv(ef[:0], ey[:0], cf, cy, 3)['sum'].abs().sum()) == 0.0
    big = torch.zeros(262145, 1, device='cuda')
    with pytest.raises(_native.NativeError):
        ops.knn_sv(ef[:, :1], ey, big, torch.zeros(262145, dtype=torch.long, device='cuda'), 3)
    wide = torch.zeros(1025, 4097, device='cuda')
    with pytest.raises(_native.NativeError):
        ops.knn_sv(torch.zeros(2, 4097, device='cuda'), ey[:2], wide, torch.zeros(1025, dtype=torch.long, device='cuda'),
                   3)
    # a workspace one 256-byte line short of the query: refused before any launch
    lib = _native.lib()
    for C in (10, 1025):
        cfc = torch.rand(C, 8, device='cuda')
        cyc = torch.zeros(C, dtype=torch.long, device='cuda')
        need = lib.b200ocl_knn_sv_workspace_bytes(4, C, 8)
        ws = torch.empty(need, dtype=torch.uint8, device='cuda')
        out = torch.empty(C, device='cuda')
        p = lambda t: ctypes.c_void_p(t.data_ptr())
        rc = lib.b200ocl_knn_sv(p(ef), p(ey), p(cfc), p(cyc), 4, C, 8, 3, None, p(out), None, None, p(ws), need - 256,
                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 3, (C, rc)           # B200OCL_EWORKSPACE
        rc = lib.b200ocl_knn_sv(p(ef), p(ey), p(cfc), p(cyc), 4, C, 8, 3, None, p(out), None, None, p(ws), need,
                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, (C, rc)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------- ASER replacement

def aser_case(rs, n_cand_buf, n_cur, mem, layout):
    n = n_cand_buf + n_cur
    if layout == 'ties':
        sv_sum = rs.randint(0, 4, n).astype(np.float32) / 4          # many equal sums: ties lowest index first
    else:
        sv_sum = rs.standard_normal(n).astype(np.float32)
    if layout == 'none':                                            # current samples at the bottom: no pairs
        sv_sum[n_cand_buf:] = -10 - np.arange(n_cur)
    elif layout == 'all':                                           # current samples at the top: all inserted
        sv_sum[n_cand_buf:] = 10 + np.arange(n_cur)
    cand_slot = rs.choice(mem, n_cand_buf, replace=False).astype(np.int64)
    return sv_sum, cand_slot


@pytest.mark.parametrize('n_cand_buf,n_cur,layout', [(0, 10, 'random'), (10, 10, 'none'), (50, 10, 'all'),
                                                     (100, 10, 'random'), (150, 10, 'ties'), (4086, 10, 'random'),
                                                     (3000, 1096, 'ties'), (37, 30, 'random'), (5, 64, 'all')])
def test_aser_replace_against_oracle(ops, n_cand_buf, n_cur, layout):
    rs = np.random.RandomState(n_cand_buf + n_cur)
    mem = max(n_cand_buf + 5, 64)
    sv_sum, cand_slot = aser_case(rs, n_cand_buf, n_cur, mem, layout)
    order = oaser.argsort_desc_stable(sv_sum)
    ind_cur, ind_buffer = oaser.update_partition(sv_sum, n_cand_buf, cand_slot)
    if layout == 'none':
        assert len(ind_cur) == 0
    if layout == 'all':
        assert len(ind_cur) == min(n_cur, n_cand_buf)
    row = (3, 4, 4)
    img = rs.standard_normal((mem,) + row).astype(np.float32)
    lab = rs.randint(0, 100, mem).astype(np.int64)
    cur_x = rs.standard_normal((n_cur,) + row).astype(np.float32)
    cur_y = rs.randint(100, 200, n_cur).astype(np.int64)
    bimg, blab = torch.from_numpy(img).cuda(), torch.from_numpy(lab).cuda()
    pairs = ops.aser_replace(torch.from_numpy(order).cuda(), n_cand_buf, torch.from_numpy(cand_slot).cuda(),
                             torch.from_numpy(cur_x).cuda(), torch.from_numpy(cur_y).cuda(), bimg, blab).cpu().numpy()
    cnt = len(ind_cur)
    want_pairs = np.full(1 + 2 * n_cur, -1, dtype=np.int64)
    want_pairs[0] = cnt
    want_pairs[1:1 + cnt] = ind_cur
    want_pairs[1 + n_cur:1 + n_cur + cnt] = ind_buffer
    np.testing.assert_array_equal(pairs, want_pairs)
    img[ind_buffer] = cur_x[ind_cur]
    lab[ind_buffer] = cur_y[ind_cur]
    assert np.array_equal(bimg.cpu().numpy().view(np.int32), img.view(np.int32))   # no other slot touched
    np.testing.assert_array_equal(blab.cpu().numpy(), lab)
