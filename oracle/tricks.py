"""fp64 numpy restatement of the training-trick criteria (agents/base.py:93-107), the distillation loss
(utils/kd_manager.py:6-11) and their mixing (exp_replay.py:41-47, agem.py:40-46, lwf.py:38-40): loss and d loss / d logits.
"""
import numpy as np

KD_T = 2.0


def _log_softmax(z):
    z = z - z.max(axis=1, keepdims=True)
    return z - np.log(np.exp(z).sum(axis=1, keepdims=True))


def ce(logits, labels):
    """Mean cross-entropy over all columns: (loss, dlogits)."""
    z = np.asarray(logits, np.float64)
    n = z.shape[0]
    ls = _log_softmax(z)
    g = np.exp(ls)
    g[np.arange(n), labels] -= 1.0
    return -ls[np.arange(n), labels].mean(), g / n


def labels_trick(logits, labels):
    """CE over the columns of the classes present in the batch, labels remapped to their rank among them."""
    z = np.asarray(logits, np.float64)
    unq = np.unique(labels)
    rank = np.searchsorted(unq, labels)
    loss, g_sub = ce(z[:, unq], rank)
    g = np.zeros_like(z)
    g[:, unq] = g_sub
    return loss, g


def separated_softmax(logits, labels, old_labels, new_labels, lbl_inv_map):
    """cat(log_softmax(z[:, old]), log_softmax(z[:, new])) and NLL at lbl_inv_map[label]; a column held at several
    positions gathers the gradient of each.  A label without an entry raises KeyError, as the reference does."""
    z = np.asarray(logits, np.float64)
    n = z.shape[0]
    old, new = list(old_labels), list(new_labels)
    pos = np.array([lbl_inv_map[int(y)] for y in labels], dtype=np.int64)
    segs = [ls for ls in (_log_softmax(z[:, old]) if old else None, _log_softmax(z[:, new]) if new else None)
            if ls is not None]
    ss = np.concatenate(segs, axis=1)
    loss = -ss[np.arange(n), pos].mean()
    cols = np.array(old + new, dtype=np.int64)
    g = np.zeros_like(z)
    for i in range(n):
        lo, hi = (0, len(old)) if pos[i] < len(old) else (len(old), len(cols))
        d = np.exp(ss[i, lo:hi])
        d[pos[i] - lo] -= 1.0
        np.add.at(g[i], cols[lo:hi], d / n)
    return loss, g


def kd(logits, teacher, T=KD_T):
    """T^2 * mean_i sum_j -softmax(t/T) * log_softmax(s/T): (loss, dlogits)."""
    s = np.asarray(logits, np.float64) / T
    t = np.asarray(teacher, np.float64) / T
    n = s.shape[0]
    p = np.exp(_log_softmax(t))
    ls = _log_softmax(s)
    loss = (-(p * ls).sum(axis=1)).mean() * T * T
    g = (np.exp(ls) * p.sum(axis=1, keepdims=True) - p) * T / n
    return loss, g


def mix(task_seen, kd_trick=False, kd_trick_star=False, lwf=False):
    """(w_ce, w_kd) with loss = w_ce * criterion + w_kd * kd."""
    w_ce, w_kd = 1.0, 0.0
    if kd_trick or lwf:
        a = 1.0 / (task_seen + 1)
        w_ce, w_kd = a, 1.0 - a
    if kd_trick_star and not lwf:
        b = 1.0 / np.sqrt(task_seen + 1)
        w_ce, w_kd = b * w_ce, b * w_kd + (1.0 - b)
    return w_ce, w_kd


def criterion(logits, labels, mode='ce', old_labels=(), new_labels=(), lbl_inv_map=None, teacher=None, w_ce=1.0,
              w_kd=0.0):
    """w_ce * criterion(mode) + w_kd * kd(teacher) (kd = 0 without a teacher): (loss, dlogits)."""
    if mode == 'labels_trick':
        loss, g = labels_trick(logits, labels)
    elif mode == 'separated_softmax':
        loss, g = separated_softmax(logits, labels, old_labels, new_labels, lbl_inv_map)
    else:
        loss, g = ce(logits, labels)
    loss, g = w_ce * loss, w_ce * g
    if teacher is not None:
        lk, gk = kd(logits, teacher)
        loss, g = loss + w_kd * lk, g + w_kd * gk
    return loss, g
