"""CPU: the fp64 oracle of the training-trick criteria and the distillation mixing (oracle/tricks.py) against the
reference's own ContinualLearner.criterion and loss_fn_kd (tests/golden/tricks.npz, written by
tests/golden/make_golden_tricks.py), and the learners' host bookkeeping -- the separated-softmax position table and
the mixing coefficients -- against the reference's."""
import os

import numpy as np
import pytest

from oracle import tricks as otr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'tricks.npz')
LOSS_SEED = 5000          # tests/golden/make_golden_tricks.py: case k draws its logits from RandomState(LOSS_SEED + k)


def case_logits(seed, N, C, teacher):
    """tests/golden/make_golden_tricks.py case_logits(): logits [N,C] and, when asked, teacher logits."""
    rs = np.random.RandomState(seed)
    logits = (rs.standard_normal((N, C)) * 3).astype(np.float32)
    return logits, ((rs.standard_normal((N, C)) * 3).astype(np.float32) if teacher else None)


def loss_case(g, k):
    """The arguments of one loss-level golden case: (logits, labels, kwargs of oracle.tricks.criterion)."""
    from b200ocl.learners import kd_mix
    tag = 'l%d_' % k
    kdt, kds, alone = (bool(v) for v in g[tag + 'flags'])
    t = int(g[tag + 'task_seen'])
    mode = str(g[tag + 'mode'])
    N, C = (int(v) for v in g[tag + 'shape'])
    logits, teacher = case_logits(LOSS_SEED + k, N, C, bool(g[tag + 'teacher']))
    w_ce, w_kd = (0.0, 1.0) if alone else kd_mix(t, kdt, kds)
    kw = dict(mode=mode, teacher=teacher, w_ce=w_ce, w_kd=w_kd)
    if str(g[tag + 'hist']):
        kw.update(old_labels=g[tag + 'old'].tolist(), new_labels=g[tag + 'new'].tolist(),
                  lbl_inv_map={int(a): int(b) for a, b in g[tag + 'inv']})
    return logits, g[tag + 'labels'].astype(np.int64), kw


def _n_loss_cases():
    return int(np.load(GOLDEN)['n_loss_cases'])


@pytest.mark.parametrize('k', range(_n_loss_cases()))
def test_oracle_matches_reference_criterion(k):
    g = np.load(GOLDEN)
    logits, labels, kw = loss_case(g, k)
    loss, grad = otr.criterion(logits, labels, **kw)
    want = float(g['l%d_loss' % k])
    assert abs(loss - want) <= 1e-5 * max(abs(want), 1e-30), (k, kw['mode'], loss, want)
    assert np.abs(grad - g['l%d_dlogits' % k]).max() <= 1e-6, (k, kw['mode'])


def test_golden_covers_the_cases():
    g = np.load(GOLDEN)
    modes = [str(g['l%d_mode' % k]) for k in range(_n_loss_cases())]
    assert {'ce', 'labels_trick', 'separated_softmax'} <= set(modes)
    flags = np.stack([g['l%d_flags' % k] for k in range(_n_loss_cases())])
    assert flags[:, 0].any() and flags[:, 1].any() and flags[:, 2].any() and (flags[:, 0] & flags[:, 1]).any()
    # a separated-softmax case whose target lies in an old segment holding duplicate columns
    found = False
    for k in range(_n_loss_cases()):
        if modes[k] != 'separated_softmax' or 'l%d_old' % k not in g:
            continue
        old = g['l%d_old' % k]
        inv = dict(g['l%d_inv' % k].tolist())
        if len(set(old.tolist())) < len(old) and any(inv[int(y)] < len(old) for y in g['l%d_labels' % k]):
            found = True
    assert found


class _Bookkeeping(object):
    """The label bookkeeping of learners.ContinualLearner without an engine or a device."""

    def __init__(self):
        from b200ocl import learners
        self.old_labels, self.new_labels, self.lbl_inv_map, self.class_task_map = [], [], {}, {}
        self.task_seen = 0
        self.params = type('P', (), {'trick': {}})()
        self._takes_teacher = False
        self.before_train = learners.ContinualLearner.before_train.__get__(self)
        self.after_train = learners.ContinualLearner.after_train.__get__(self)

    def _task_tables(self):
        pass


@pytest.mark.parametrize('name', ['first10', 'first100', 'recur10', 'overlap100'])
def test_position_table_follows_the_reference_bookkeeping(name):
    """Recurring label sets: old_labels keeps every occurrence, lbl_inv_map points into the segment of the latest task,
    and the device table sends each label to the position the reference's NLL reads."""
    from b200ocl.learners import separated_softmax_table
    g = np.load(GOLDEN)
    book = _Bookkeeping()
    n = int(g['hist_%s_n' % name])
    for t in range(n):
        new = g['hist_%s_new%d' % (name, t)]
        book.before_train(new, new)
        assert book.old_labels == g['hist_%s_old%d' % (name, t)].tolist(), (name, t)
        assert sorted(book.new_labels) == sorted(new.tolist())
        inv = {int(a): int(b) for a, b in g['hist_%s_inv%d' % (name, t)]}
        assert book.lbl_inv_map == inv, (name, t)
        cols, n_old, pos = separated_softmax_table(book.old_labels, book.new_labels, book.lbl_inv_map)
        assert n_old == len(book.old_labels) and cols.tolist() == book.old_labels + book.new_labels
        for lbl, p in inv.items():
            assert pos[lbl] == p and cols[p] == lbl
        assert all(pos[c] == -1 for c in range(pos.size) if c not in inv)
        if t < n - 1:
            book.after_train()


def test_mixing_coefficients_follow_the_reference_formulas():
    """exp_replay.py:41-47 applied in order: kd_trick, then kd_trick_star on the result; LwF mixes as kd_trick."""
    from b200ocl.learners import kd_mix
    for t in range(6):
        a, b = 1 / (t + 1), 1 / ((t + 1) ** 0.5)
        assert kd_mix(t) == (1.0, 0.0)
        assert kd_mix(t, kd_trick=True) == pytest.approx((a, 1 - a), rel=1e-15)
        assert kd_mix(t, kd_trick_star=True) == pytest.approx((b, 1 - b), rel=1e-15)
        # b * (a * ce + (1 - a) * kd) + (1 - b) * kd
        assert kd_mix(t, True, True) == pytest.approx((b * a, b * (1 - a) + 1 - b), rel=1e-15)
        assert kd_mix(t, lwf=True) == kd_mix(t, kd_trick=True)
        assert kd_mix(t, True, True, lwf=True) == kd_mix(t, kd_trick=True)
