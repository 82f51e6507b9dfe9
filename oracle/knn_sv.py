"""Oracle: exact kNN Shapley values of candidates w.r.t. evaluation points.

Restates ``compute_knn_sv`` (reference utils/buffer/aser_utils.py:7-61) on
*feature matrices* (the network forward of aser_utils.py:27 is covered by
oracle/resnet.py).  Test infrastructure only -- see oracle/__init__.py.

Conventions shared with the CUDA kernel (csrc/knn_sv.cu):
  * distance  = squared L2, direct-difference form sum((u-v)^2)
                (utils/utils.py:93-95), never |u|^2+|v|^2-2uv;
  * ordering  = ascending distance, ties broken lowest candidate index first
                (the reference's argsort at aser_utils.py:115 is unstable, so the
                tie order is ours to define -- SURVEY.md section 7.3-2);
  * recurrence (aser_utils.py:38-52), ranks i = 1..N over the sorted list,
                m_i = 1[label(cand_i) == label(eval)]:
                    s_N = m_N / N
                    s_i = s_{i+1} + (m_i - m_{i+1}) * min(i, k) / (i * k)
"""
import numpy as np


def sq_dist_matrix(eval_f, cand_f, dtype=np.float64, chunk=256):
    """[E,d],[C,d] -> [E,C] squared L2, direct-difference (utils/utils.py:93-95)."""
    eval_f = np.asarray(eval_f, dtype=dtype)
    cand_f = np.asarray(cand_f, dtype=dtype)
    E, C = eval_f.shape[0], cand_f.shape[0]
    out = np.empty((E, C), dtype=dtype)
    for s in range(0, E, chunk):
        diff = eval_f[s:s + chunk, None, :] - cand_f[None, :, :]
        out[s:s + chunk] = np.einsum('ecd,ecd->ec', diff, diff)
    return out


def sorted_cand_ind(eval_f, cand_f, dtype=np.float64):
    """Candidate indices by ascending distance per eval row, stable
    (aser_utils.py:94-116)."""
    dist = sq_dist_matrix(eval_f, cand_f, dtype=dtype)
    return np.argsort(dist, axis=1, kind='stable'), dist


def sv_factor(n_cand, k, dtype=np.float64):
    """factor[j] for 0-based sorted position j (rank i=j+1), aser_utils.py:43-49:
    min(i,k)/(i*k) for i < N, and 1/N for i == N."""
    i = np.arange(1, n_cand + 1, dtype=dtype)
    numer = i.copy()
    denom = i.copy()
    denom[:n_cand - 1] *= k
    numer[k:n_cand - 1] = k
    numer[n_cand - 1] = 1
    return numer / denom


def knn_sv_from_sorted(sorted_ind, eval_y, cand_y, k, dtype=np.float64):
    """SV matrix [E,C] in *candidate order* from per-row sorted candidate indices
    (aser_utils.py:32-59)."""
    sorted_ind = np.asarray(sorted_ind)
    eval_y = np.asarray(eval_y)
    cand_y = np.asarray(cand_y)
    E, C = sorted_ind.shape
    match = (cand_y[sorted_ind] == eval_y[:, None]).astype(dtype)          # :35-38
    nxt = np.zeros_like(match)
    nxt[:, :C - 1] = match[:, 1:]                                          # :39-40
    term = (match - nxt) * sv_factor(C, k, dtype)[None, :]                 # :41-51
    sv_sorted = np.cumsum(term[:, ::-1], axis=1, dtype=dtype)[:, ::-1]     # :52
    sv = np.zeros((E, C), dtype=dtype)
    np.put_along_axis(sv, sorted_ind, sv_sorted, axis=1)                   # :55-59
    return sv


def knn_sv_matrix(eval_f, eval_y, cand_f, cand_y, k, dtype=np.float64):
    """Full restatement on features.  Returns (sv [E,C], sorted_ind [E,C], dist [E,C])."""
    sorted_ind, dist = sorted_cand_ind(eval_f, cand_f, dtype=dtype)
    return knn_sv_from_sorted(sorted_ind, eval_y, cand_y, k, dtype=dtype), sorted_ind, dist


def knn_sv_row_loop(dist_row, eval_label, cand_y, k):
    """Pure-python per-row recurrence (Jia et al. 2019), fp64 -- small cases only.
    Independent of the vectorised form above; used to cross-check it."""
    C = len(dist_row)
    order = sorted(range(C), key=lambda j: (dist_row[j], j))
    m = [1.0 if cand_y[j] == eval_label else 0.0 for j in order]
    s = [0.0] * C
    s[C - 1] = m[C - 1] / C
    for pos in range(C - 2, -1, -1):
        i = pos + 1
        s[pos] = s[pos + 1] + (m[pos] - m[pos + 1]) * min(i, k) / (i * k)
    out = [0.0] * C
    for pos, j in enumerate(order):
        out[j] = s[pos]
    return out


def column_reductions(sv):
    """The three row-reductions the ASER plugins consume
    (aser_retrieve.py:79,82,86; aser_update.py:80)."""
    return sv.sum(0), sv.max(0), sv.min(0)


def order_mismatch_explained(sorted_a, sorted_b, dist64, rel_tol=4e-6):
    """Compare two per-row orderings.  A difference is *explained* when every
    position where they differ lies inside a run of candidates whose fp64
    distances agree to rel_tol (an fp32 summation-order near-tie).  Returns
    (n_rows_different, n_rows_unexplained)."""
    n_diff = n_bad = 0
    for r in range(sorted_a.shape[0]):
        a, b = sorted_a[r], sorted_b[r]
        if np.array_equal(a, b):
            continue
        n_diff += 1
        da, db = dist64[r][a], dist64[r][b]
        scale = np.maximum(np.abs(da), np.abs(db)) + 1e-30
        pos = np.nonzero(a != b)[0]
        if np.any(np.abs(da[pos] - db[pos]) > rel_tol * scale[pos]):
            n_bad += 1
    return n_diff, n_bad


# --------------------------------------------------------------------------- the kernel's own fp32 ordering
# The kernels (csrc/knn_sv.cu, csrc/knn_sv_large.cu) rank candidates by their fp32 distances, ties lowest index first.
# Where two fp64 distances are closer than fp32 rounding, the fp32 order is the kernel's own choice.  The functions
# below reproduce those fp32 distances bit for bit with float64 torch ops, so that the stable sort of them *is* the
# kernel's order and the fp64 recurrence on it differs from the kernel by rounding only.
#   fused kernel  acc = 0; for f in 0..d-1: df = u_f - v_f (fp32); acc = fmaf(df, df, acc)      (both phase-1 forms)
#   large kernel  lane l in 0..31: the same chain over f = l, l+32, ...; then warp_sum's xor butterfly,
#                 v_l <- fl32(v_l + v_(l^o)) for o = 16, 8, 4, 2, 1, and lane 0's value
# fmaf is emulated without contraction, one torch op per step: df^2 is exact in fp64 (a 24-bit significand squared);
# TwoSum gives df^2 + acc = s + e exactly; fl32(s + e) is fl32(s), except when s is exactly halfway between two fp32
# values, where the sign of e decides (e = 0: ties to even, which fl32(s) already did).

def _round_fp32(s, e):
    """fl32(s + e) for fp64 tensors s, e with |e| <= ulp64(s) / 2 (s + e exact, e.g. from TwoSum)."""
    import torch
    r = s.to(torch.float32)
    r64 = r.to(torch.float64)
    toward = torch.where(s > r64, torch.full_like(r, float('inf')), torch.full_like(r, float('-inf')))
    other = torch.nextafter(r, toward)
    other64 = other.to(torch.float64)
    mid = (r64 + other64) * 0.5                       # exact: two neighbouring fp32 values
    flip = (s == mid) & (e != 0) & ((e > 0) == (other64 > r64))
    return torch.where(flip, other, r)


def fmaf_sq(df, acc):
    """fmaf(df, df, acc) for fp32 tensors, correctly rounded, from fp64 torch ops."""
    import torch
    p = df.to(torch.float64) * df.to(torch.float64)   # exact
    a = acc.to(torch.float64)
    s = p + a                                         # TwoSum(p, a): s + e == p + a exactly
    bb = s - a
    e = (a - (s - bb)) + (p - bb)
    return _round_fp32(s, e)


def dist_fp32_fused(ef, cf):
    """[E,C] fp32 distances of the fused kernel: one sequential fmaf chain over the features.  fp32 torch tensors."""
    import torch
    acc = torch.zeros((ef.shape[0], cf.shape[0]), dtype=torch.float32, device=ef.device)
    for f in range(ef.shape[1]):
        acc = fmaf_sq(ef[:, f, None] - cf[None, :, f], acc)
    return acc


def dist_fp32_large(ef, cf, lanes=32):
    """[E,C] fp32 distances of the scratch-line kernel: 32 lane-strided fmaf chains, then the xor butterfly."""
    import torch
    E, d = ef.shape
    C = cf.shape[0]
    steps = -(-d // lanes)
    pad = steps * lanes - d                           # fmaf(0, 0, acc) == acc: idle lanes add nothing
    ep = torch.nn.functional.pad(ef, (0, pad))
    cp = torch.nn.functional.pad(cf, (0, pad))
    out = torch.empty((E, C), dtype=torch.float32, device=ef.device)
    idx = torch.arange(lanes, device=ef.device)
    for r in range(E):
        acc = torch.zeros((C, lanes), dtype=torch.float32, device=ef.device)
        for t in range(steps):
            sl = slice(t * lanes, (t + 1) * lanes)
            acc = fmaf_sq(ep[r, None, sl] - cp[:, sl], acc)
        for o in (16, 8, 4, 2, 1):
            acc = acc + acc[:, idx ^ o]
        out[r] = acc[:, 0]
    return out


def kernel_order(ef, cf, large=None):
    """The kernels' per-row candidate order [E,C] (int64) and fp32 distances: the stable sort of the emulated fp32
    distances.  large: the scratch-line kernel's distances (default: when C > 1024, as b200ocl_knn_sv picks)."""
    import torch
    if large is None:
        large = cf.shape[0] > 1024
    dist = dist_fp32_large(ef, cf) if large else dist_fp32_fused(ef, cf)
    return torch.sort(dist, dim=1, stable=True).indices, dist


def knn_sv_torch(order, eval_y, cand_y, k, block=64):
    """fp64 SV matrix [E,C] in candidate order from an explicit per-row order [E,C] (torch, any device), in blocks of
    rows so that C = 262 144 fits.  Also returns each row's sum of |terms| of the recurrence (the scale its fp32
    rounding is relative to)."""
    import torch
    E, C = order.shape
    dev = order.device
    factor = torch.from_numpy(sv_factor(C, k)).to(dev)
    sv = torch.empty((E, C), dtype=torch.float64, device=dev)
    abs_sum = torch.empty(E, dtype=torch.float64, device=dev)
    for s in range(0, E, block):
        o = order[s:s + block]
        match = (cand_y[o] == eval_y[s:s + block, None]).to(torch.float64)
        nxt = torch.zeros_like(match)
        nxt[:, :C - 1] = match[:, 1:]
        term = (match - nxt) * factor
        sv[s:s + block].scatter_(1, o, term.flip(1).cumsum(1).flip(1))
        abs_sum[s:s + block] = term.abs().sum(1)
    return sv, abs_sum


EPS32 = 2.0 ** -24


def gamma(n):
    return n * EPS32 / (1 - n * EPS32)


def kernel_add_depth(plan):
    """Additions an exact term passes through before it reaches an SV entry (see tests/test_gpu_knn_sv_fp64.py):
    fused: KPL in-lane + 5 shuffle levels + 1 (the lanes above); large: the per-thread run L = Cpad / 1024 twice, the
    5-level block scan, its exclusive subtraction, the 31-block carry chain and the carry's addition."""
    if plan.name == 'large':
        return 2 * (plan.cpad // 1024) + 5 + 1 + 31 + 1
    return plan.kpl + 6


def sv_row_bound(abs_sum, plan, C):
    """Per-row bound on |SV_kernel - SV_fp64| on the kernel's own order: gamma_(n+2) * sum |terms| (n additions and
    the two roundings of the factor, fl32(rank * k) and the division) plus the fp64 oracle's own cumsum rounding."""
    return (gamma(kernel_add_depth(plan) + 2) + C * 2.0 ** -52) * abs_sum
