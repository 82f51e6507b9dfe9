"""fp64 numpy restatement of iCaRL's criterion (agents/icarl.py:42-62): the target construction, the loss
F.binary_cross_entropy_with_logits(logits[:, :K], target, reduction='none').sum(1).mean() and d loss / d logits.
"""
import numpy as np

LOSS_SEED = 7000     # loss-level golden case k of tests/golden/icarl.npz draws its logits from RandomState(LOSS_SEED + k)


def case_logits(seed, rows, C, scale, teacher):
    """Logits [rows,C] (and teacher logits when asked) of one loss-level golden case: the generator
    (tests/golden/make_golden_icarl.py) and the tests regenerate them from here instead of storing them."""
    rs = np.random.RandomState(seed)
    logits = (rs.standard_normal((rows, C)) * scale).astype(np.float32)
    return logits, ((rs.standard_normal((rows, C)) * scale).astype(np.float32) if teacher else None)


def sigmoid(z):
    return 0.5 * (1.0 + np.tanh(0.5 * np.asarray(z, np.float64)))


def targets(n_rows, labels, old_labels, new_labels, teacher=None):
    """[n_rows, K] target, K = len(old_labels) + len(new_labels): one-hot at len(old_labels) + new_labels.index(y) for
    the len(labels) stream rows, zero for the memory rows after them; with the previous model's logits (teacher), their
    sigmoids in the columns k < len(old_labels) of every row."""
    n_old = len(old_labels)
    K = n_old + len(new_labels)
    t = np.zeros((n_rows, K))
    for i, y in enumerate(labels):
        t[i, n_old + list(new_labels).index(int(y))] = 1.0
    if teacher is not None:
        t[:, :n_old] = sigmoid(np.asarray(teacher, np.float64)[:, :n_old])
    return t


def icarl_loss(logits, labels, old_labels, new_labels, teacher=None):
    """(loss, dlogits [N,C]); the columns at or beyond K get no gradient."""
    z_all = np.asarray(logits, np.float64)
    n = z_all.shape[0]
    t = targets(n, labels, old_labels, new_labels, teacher)
    K = t.shape[1]
    if K > z_all.shape[1]:
        raise ValueError('K = %d positions exceed the %d logits' % (K, z_all.shape[1]))
    z = z_all[:, :K]
    loss = (np.maximum(z, 0.0) - z * t + np.log1p(np.exp(-np.abs(z)))).sum(axis=1).mean()
    g = np.zeros_like(z_all)
    g[:, :K] = (sigmoid(z) - t) / n
    return loss, g
