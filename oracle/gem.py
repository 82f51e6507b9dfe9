"""Oracle: GEM (Lopez-Paz & Ranzato, "Gradient Episodic Memory for Continual Learning", NeurIPS 2017) as
learners.GEM runs it, in float64 (or the ReplayState's parameter dtype).

  * Rings: one memory of M rows per task; a batch is written at the task's counter and truncated at the ring's end
    (endcnt = min(cnt + bsz, M), x[:endcnt - cnt]), the counter returns to 0 at M and restarts at 0 with every task;
    a task's filled row count is min(rows written, M).
  * gram: P = G G^T and q = G g.
  * solve_qp: min_v 1/2 v^T (P + eps I) v + q^T v subject to v >= margin, exactly: an active-set search on
    w = v - margin >= 0 whose final free set is solved once more by a direct solve, then checked against the KKT
    conditions.  solve_qp_enumerate tries every free set (t <= 10) for the tests.
  * step: one GEM step on replay_step.ReplayState with the rings.
Test infrastructure only -- see oracle/__init__.py.
"""
import itertools
from collections import OrderedDict

import numpy as np
import torch

from . import agem as oagem
from . import replay_step as ors
from . import resnet as oresnet

EPS = 1e-3


class Rings(object):
    """Per-task ring memories: images [M, ...] and labels [M] per task, with counters and filled counts."""

    def __init__(self, M, in_shape):
        if M < 1:
            raise ValueError('GEM needs at least one row per task')
        self.M = int(M)
        self.in_shape = tuple(in_shape)
        self.images, self.labels, self.filled, self.cnt = [], [], [], []

    def begin_task(self, task):
        """Make task `task` the current one: its ring exists (earlier tasks without one get empty rings) and its
        counter restarts at 0."""
        while len(self.images) <= task:
            self.images.append(torch.zeros((self.M,) + self.in_shape, dtype=torch.float32))
            self.labels.append(torch.zeros(self.M, dtype=torch.long))
            self.filled.append(0)
            self.cnt.append(0)
        self.cnt[task] = 0

    def write(self, task, x, y):
        """The authors' ring write: rows [cnt, endcnt) take x[:endcnt - cnt]; returns (start, count)."""
        cnt = self.cnt[task]
        end = min(cnt + x.shape[0], self.M)
        k = end - cnt
        self.images[task][cnt:end] = x[:k].to(torch.float32)
        self.labels[task][cnt:end] = y[:k]
        self.filled[task] = max(self.filled[task], end)
        self.cnt[task] = 0 if end == self.M else end
        return cnt, k


def ring_positions(M, batch_sizes):
    """Plain restatement of the ring rule for one task: per batch the (start, count) it writes, and the filled count."""
    cnt, written, out = 0, 0, []
    for b in batch_sizes:
        end = min(cnt + b, M)
        out.append((cnt, end - cnt))
        written += end - cnt
        cnt = 0 if end == M else end
    return out, min(written, M)


def gram(G, g):
    """(P [t,t], q [t]) in float64."""
    G = np.asarray(G, dtype=np.float64)
    g = np.asarray(g, dtype=np.float64)
    return G @ G.T, G @ g


def _free_solve(H, c, free):
    w = np.zeros(len(c))
    if free:
        f = list(free)
        w[f] = np.linalg.solve(H[np.ix_(f, f)], -c[f])
    return w


def kkt_residuals(H, c, w):
    """(primal, dual, complementarity) residuals of w for min 1/2 w^T H w + c^T w, w >= 0: max(0, -w); on the bound
    max(0, -lam), off it |lam|; max |w lam|; lam = H w + c."""
    lam = H @ w + c
    primal = float(np.max(np.maximum(0.0, -w))) if w.size else 0.0
    dual = float(np.max(np.where(w == 0, np.maximum(0.0, -lam), np.abs(lam)))) if w.size else 0.0
    comp = float(np.max(np.abs(w * lam))) if w.size else 0.0
    return primal, dual, comp


def _shifted(P, q, margin, eps):
    H = np.asarray(P, np.float64) + eps * np.eye(len(q))
    c = np.asarray(q, np.float64) + margin * H.sum(axis=1)
    return H, c


def solve_qp(P, q, margin=0.5, eps=EPS):
    """v minimising 1/2 v^T (P + eps I) v + q^T v subject to v >= margin (float64).  Lawson & Hanson's active-set loop
    on w = v - margin; the final free set is solved directly, so v_k == margin exactly on the bound."""
    H, c = _shifted(P, q, margin, eps)
    t = len(c)
    free = set()
    w = np.zeros(t)
    for _ in range(10 * t + 10):
        lam = H @ w + c
        tol = 1e-12 * (np.max(np.abs(c)) + np.max(np.diag(H)) * (w.max() if t else 0.0))
        cand = [k for k in range(t) if k not in free and lam[k] < -tol]
        if not cand:
            break
        free.add(min(cand, key=lambda k: (lam[k], k)))
        while True:
            z = _free_solve(H, c, sorted(free))
            f = sorted(free)
            if all(z[k] > 0 for k in f):
                w = z
                break
            ratios = [(w[k] / (w[k] - z[k]), k) for k in f if z[k] <= 0]
            alpha = min(r for r, _ in ratios)
            w = w + alpha * (z - w)
            for r, k in ratios:
                if r <= alpha:
                    w[k] = 0.0
                    free.discard(k)
            for k in list(free):
                if w[k] <= 0:
                    w[k] = 0.0
                    free.discard(k)
    else:
        raise RuntimeError('active-set QP did not converge')
    return w + margin


def solve_qp_enumerate(P, q, margin=0.5, eps=EPS):
    """The same QP by trying every free set (t <= 10): the unique KKT point of the strictly convex problem."""
    H, c = _shifted(P, q, margin, eps)
    t = len(c)
    if t > 10:
        raise ValueError('enumeration is for t <= 10')
    best = None
    for r in range(t + 1):
        for free in itertools.combinations(range(t), r):
            w = _free_solve(H, c, free)
            if free and w[list(free)].min() < 0:
                continue
            lam = H @ w + c
            act = [k for k in range(t) if k not in free]
            scale = np.abs(c).max() + np.abs(H).max() * max(w.max(), 1.0)
            if act and lam[act].min() < -1e-9 * scale:
                continue
            obj = 0.5 * w @ H @ w + c @ w
            if best is None or obj < best[0]:
                best = (obj, w)
    return best[1] + margin


def objective(P, q, v, eps=EPS):
    v = np.asarray(v, np.float64)
    return float(0.5 * v @ (np.asarray(P) + eps * np.eye(len(v))) @ v + np.asarray(q) @ v)


def project(G, g, margin=0.5, eps=EPS):
    """(out, v, flag): g + G^T v when min(G g) < 0, else g (flag False, v zeros)."""
    G = np.asarray(G, dtype=np.float64)
    g = np.asarray(g, dtype=np.float64)
    P, q = gram(G, g)
    if q.size == 0 or q.min() >= 0:
        return g.copy(), np.zeros(q.size), False
    v = solve_qp(P, q, margin, eps)
    return g + G.T @ v, v, True


def step(st, rings, task, batch_x, batch_y, margin=0.5, mem_iters=1, adam=None):
    """One GEM step on the ReplayState st with Rings `rings`, `task` being the current task (its ring already begun).
    Per iteration: the earlier tasks with a non-empty ring, in task order, each a train-mode forward over its filled
    rows, mean CE and backward (their BN statistics move first); then the stream batch's; the projection in float64;
    one SGD (st.lr, st.wd) or Adam step.  Then the ring write.  Returns one log per iteration: G, g, flag, v, out
    (float64 flat vectors) and the stream loss."""
    dtype = next(iter(st.params.values())).dtype
    logs = []
    for _ in range(mem_iters):
        rows = []
        for k in range(task):
            n = rings.filled[k]
            if n:
                _, _, gk = ors._train_fwd_bwd(st, rings.images[k][:n].to(dtype), rings.labels[k][:n])
                rows.append(oagem.flat(gk))
        loss, _, grads = ors._train_fwd_bwd(st, batch_x.to(dtype), batch_y)
        g = oagem.flat(grads)
        log = dict(loss=float(loss), g=g, flag=False, v=None, out=g)
        if rows:
            G = np.stack(rows)
            out, v, flag = project(G, g, margin)
            log.update(G=G, flag=flag, v=v, out=out)
            grads = oagem._unflat(st, out)
        if adam is None:
            oresnet.sgd_step(st.params, grads, st.lr, st.wd)
        else:
            adam.step(st.params, grads)
        logs.append(log)
    rings.write(task, batch_x, batch_y)
    return logs
