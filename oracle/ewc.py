"""EWC++ (agents/ewc_pp.py) restated in numpy: the running-Fisher EMA, the penalty and its autograd gradient, the Fisher
accumulation, the end-of-call normalisation and one whole step, each fp32 rounding of the reference's separate torch
ops spelled out (numpy never fuses a product into a sum), and the penalty value in fp64.  Arrays are fp32; dicts map
parameter names to arrays, as the reference's dicts do."""
import numpy as np

F32 = np.float32


def ema_schedule(n_batches, epochs, fisher_update_after):
    """ewc_pp.py:40-41: per step of one call, whether update_running_fisher fires before it."""
    return [(ep * n_batches + i + 1) % fisher_update_after == 0 for ep in range(epochs) for i in range(n_batches)]


def ema_coefficients(alpha, fisher_update_after):
    """(1 - alpha) and 1/fua * alpha, formed in double as Python forms them, rounded to fp32 where torch multiplies."""
    return F32(1. - alpha), F32(1. / fisher_update_after * alpha)


def update_running_fisher(running, tmp, alpha, fisher_update_after):
    """ewc_pp.py:103-108: (new running, new tmp = 0)."""
    keep, add = ema_coefficients(alpha, fisher_update_after)
    return ({n: F32(keep) * r + F32(add) * tmp[n] for n, r in running.items()},
            {n: np.zeros_like(t) for n, t in tmp.items()})


def penalty_up(lambda_, task_seen, kd_trick=False, kd_trick_star=False):
    """The gradient autograd delivers to the regulariser: fp32(lambda) times the mixing weights of ewc_pp.py:46-51,
    multiplied in fp32 from the outermost weight (kd_trick_star's) inward."""
    up = F32(1.0)
    if kd_trick_star:
        up = F32(up * F32(1 / ((task_seen + 1) ** 0.5)))
    if kd_trick:
        up = F32(up * F32(1 / (task_seen + 1)))
    return F32(up * F32(lambda_))


def penalty_grad(params, prev, fisher, up):
    """d(up * sum F * (p - prev)**2)/dp as autograd forms it: (up * F) * (2 * (p - prev))."""
    return {n: (F32(up) * fisher[n]) * (F32(2) * (p - prev[n])) for n, p in params.items()}


def penalty_value(params, prev, fisher):
    """sum_n (F_n * (p_n - prev_n)**2).sum() in fp64 (the difference is the fp32 difference the gradient uses)."""
    total = 0.0
    for n, p in params.items():
        d = (p - prev[n]).astype(np.float64)
        total += float(np.sum(fisher[n].astype(np.float64) * d * d))
    return total


def accum_fisher(tmp, grads):
    """ewc_pp.py:110-112: tmp += grad ** 2 (torch's pow 2 is grad * grad)."""
    return {n: t + grads[n] * grads[n] for n, t in tmp.items()}


def normalize(running):
    """ewc_pp.py:74-77: (running - mn) / ((mx - mn) + 1e-32) with the global min / max, fp32 with an IEEE division."""
    mx = max(F32(r.max()) for r in running.values())
    mn = min(F32(r.min()) for r in running.values())
    den = F32(F32(mx - mn) + F32(1e-32))
    return {n: ((r - mn) / den).astype(np.float32) for n, r in running.items()}


def step(params, grads, state, lr, wd, up, penalty, ema, alpha, fisher_update_after):
    """One step after backward: EMA (when it fires before this batch), the penalty gradient (from the second call on),
    tmp += g * g, then SGD as the engine applies it (p - lr * (g + wd * p), torch.optim.SGD without momentum).
    state: dict(running, tmp, normalized, prev) of dicts.  Returns (params, grads, state, penalty value or None)."""
    state = dict(state)
    if ema:
        state['running'], state['tmp'] = update_running_fisher(state['running'], state['tmp'], alpha,
                                                               fisher_update_after)
    pen = None
    if penalty:
        pen = penalty_value(params, state['prev'], state['normalized'])
        pg = penalty_grad(params, state['prev'], state['normalized'], up)
        grads = {n: g + pg[n] for n, g in grads.items()}
    state['tmp'] = accum_fisher(state['tmp'], grads)
    out = {}
    for n, p in params.items():
        g = grads[n].astype(np.float64) + wd * p.astype(np.float64)
        out[n] = (p.astype(np.float64) - lr * g).astype(np.float32)
    return out, grads, state, pen


def consolidate(params, state):
    """ewc_pp.py:70-77: prev = params, normalized from running."""
    state = dict(state)
    state['prev'] = {n: p.copy() for n, p in params.items()}
    state['normalized'] = normalize(state['running'])
    return state


def element_case_inputs(seed, shapes, scale, zero_running):
    """Seeded inputs of one element-level golden case (tests/golden/make_golden_ewc.py and tests/test_oracle_ewc.py
    both draw them from here): params, prev, running (times `scale`), tmp, the logits and labels of the detached stub.
    zero_running: running and tmp all zero, so that the normalisation meets an all-zero running."""
    rs = np.random.RandomState(seed)
    names = list(shapes)
    draw = lambda s: {n: (rs.standard_normal(shapes[n]) * s).astype(np.float32) for n in names}
    params = draw(0.1)
    prev = {n: (p + rs.standard_normal(p.shape).astype(np.float32) * F32(0.01)).astype(np.float32)
            for n, p in params.items()}
    running = {n: np.zeros(shapes[n], np.float32) if zero_running else
               (np.abs(rs.standard_normal(shapes[n])) * scale).astype(np.float32) for n in names}
    tmp = {n: np.abs(v) * F32(not zero_running) for n, v in draw(0.05).items()}
    logits = (rs.standard_normal((10, 5)) * 2).astype(np.float32)
    labels = rs.randint(0, 5, 10).astype(np.int64)
    return params, prev, running, tmp, logits, labels
