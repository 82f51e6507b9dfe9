"""torch.optim.Adam (torch/optim/adam.py; amsgrad, maximize and decoupled weight decay off) restated in numpy: the host
scalars in float64 as Python forms them, then one fp32 rounding per torch op, with fma where torch's CUDA kernels
contract (ATen/native/Lerp.h, cuda/DeviceAddCmulCdiv.cuh).  foreach selects how sqrt(v) is divided by bc2_sqrt: an
IEEE division (the multi-tensor path, _foreach_div_ by a scalar list) or a multiplication by the fp32 rounding of the
reciprocal formed in double (the single-tensor path: a CUDA Tensor / Python float)."""
import numpy as np

F32 = np.float32


def host_scalars(lr, beta1, beta2, step):
    """(step_size, bc2_sqrt) of step number `step` as torch/optim/adam.py forms them in double."""
    bias_correction1 = 1 - beta1 ** float(step)
    bias_correction2 = 1 - beta2 ** float(step)
    return (lr / bias_correction1) * -1, bias_correction2 ** 0.5


def fma(a, b, c):
    """fp32 fma(a, b, c) with a single rounding: the product is exact in float64; the float64 sum is corrected by its
    rounding error where it lands on an fp32 rounding boundary (the only place the double rounding could differ)."""
    a, b, c = (np.asarray(t, dtype=np.float64) for t in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)                       # two-sum: p + c == s + err exactly
    r = s.astype(F32)
    other = np.nextafter(r, np.where(s > r.astype(np.float64), F32(np.inf), F32(-np.inf)).astype(F32))
    mid = (r.astype(np.float64) + other.astype(np.float64)) / 2
    tie = (s == mid) & (err != 0) & (other != r)
    toward_other = np.sign(err) == np.sign(other.astype(np.float64) - r.astype(np.float64))
    return np.where(tie & toward_other, other, r).astype(F32)


def step(p, g, m, v, step_no, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, foreach=True, grad_div=None):
    """One Adam step on fp32 arrays; returns new (p, g, m, v) (g changes only with grad_div, the review trick's
    p.grad.clone() / 10.: on CUDA a multiplication by fp32(1 / div), the reciprocal formed in double)."""
    p, g, m, v = (np.asarray(t, dtype=F32) for t in (p, g, m, v))
    beta1, beta2 = float(betas[0]), float(betas[1])
    step_size, bc2_sqrt = host_scalars(float(lr), beta1, beta2, step_no)
    if grad_div is not None:
        g = (g * F32(1 / float(grad_div))).astype(F32)
    gi = fma(F32(weight_decay), p, g) if weight_decay != 0 else g
    w1 = F32(1 - beta1)
    diff = (gi - m).astype(F32)
    if abs(w1) < 0.5:
        m2 = fma(w1, diff, m)
    else:
        m2 = fma(-diff, F32(F32(1) - w1), gi)
    c2 = F32(1 - beta2)
    vb = (v * F32(beta2)).astype(F32)
    v2 = fma(gi, gi, vb) if c2 == 1 else fma(c2, (gi * gi).astype(F32), vb)
    s = np.sqrt(v2).astype(F32)
    s = (s / F32(bc2_sqrt)).astype(F32) if foreach else (s * F32(1 / bc2_sqrt)).astype(F32)
    d = (s + F32(eps)).astype(F32)
    p2 = fma(F32(step_size), (m2 / d).astype(F32), p)
    return p2, g, m2, v2


def ulp_distance(a, b):
    """Per-element distance in fp32 ulps (units in the last place, counted over the ordered fp32 bit patterns)."""
    def key(x):
        i = np.asarray(x, dtype=F32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(key(a) - key(b))
