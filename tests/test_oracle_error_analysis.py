"""CPU: the error analysis of evaluate() (agents/base.py:144-226, --error_analysis) against the reference's own runs
(tests/golden/error_analysis.npz, recorded by tests/golden/make_golden_error_analysis.py):
  * oracle/error_analysis.py from the logits the reference's network produced: the four counts and the confusion lists
    exactly, the two logit means and the four weight / bias means to 1e-6 of their scale, NaN where the reference has
    NaN, KeyError where it raised;
  * the per-class tables the learner uploads (learners.error_analysis_tables) for class-incremental and new-instance
    label histories;
  * the learner's host side (ContinualLearner._error_analysis) fed what b200ocl_linear_argmax_ea and b200ocl_rows_mean
    return, restated here in numpy from the same logits: the appended attributes, the printed lines and the confusion
    file."""
import contextlib
import io
import os
import pickle

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'error_analysis.npz')
# The reference takes each mean in fp32 (torch's mean of a [B, |S|] slice, of weight[rows], of bias[rows]); the oracle
# in fp64.  Bar: 1e-6 of the mean absolute value of the averaged elements -- a mean of mixed signs near zero carries
# the fp32 error of its elements' scale, not of its own.
MEAN_TOL = 1e-6


def _g():
    return np.load(GOLDEN)


def _case(g, k):
    tag = 'e%d_' % k
    ctm = {int(a): int(b) for a, b in g[tag + 'class_task_map']}
    rows, tasks = g[tag + 'n_rows'], g[tag + 'batch_task']
    logits, labels = g[tag + 'logits'], g[tag + 'labels']
    batches, lo = [], 0
    for t, n in zip(tasks, rows):
        batches.append((int(t), logits[lo:lo + n], labels[lo:lo + n]))
        lo += n
    return tag, ctm, batches


def _scale(g, tag, batches):
    """The mean absolute value of the elements each of the six means averages (1 where a set is empty)."""
    from oracle.error_analysis import _mean
    zombie = g[tag + 'zombie'].tolist()
    old = sorted(set(g[tag + 'old_labels'].tolist()) - set(zombie))
    ts = int(g[tag + 'task_seen'])
    W, b = g[tag + 'W'].astype(np.float64), g[tag + 'b'].astype(np.float64)
    new_l = [np.abs(l[:, zombie]) for t, l, _ in batches if t == ts - 1]
    old_l = [np.abs(l[:, old]) for t, l, _ in batches if t < ts - 1]
    out = [max((_mean(a) for a in new_l), default=1.0), max((_mean(a) for a in old_l), default=1.0),
           _mean(np.abs(W[zombie])), _mean(np.abs(W[old])), _mean(np.abs(b[zombie])), _mean(np.abs(b[old]))]
    return np.nan_to_num(np.array(out), nan=1.0)


def _same_means(got, want, scale):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (got, want)
    ok = ~np.isnan(want)
    assert (np.abs(got[ok] - want[ok]) <= MEAN_TOL * scale[ok]).all(), (got, want, scale)


@pytest.mark.parametrize('k', range(int(np.load(GOLDEN)['n_eval'])))
def test_oracle_matches_reference_evaluate(k):
    from oracle.error_analysis import error_analysis
    g = _g()
    tag, ctm, batches = _case(g, k)
    args = (batches, int(g[tag + 'task_seen']), g[tag + 'old_labels'].tolist(), g[tag + 'zombie'].tolist(), ctm,
            g[tag + 'W'], g[tag + 'b'])
    if str(g[tag + 'raised']):
        assert str(g[tag + 'raised']) == 'KeyError'
        with pytest.raises(KeyError):
            error_analysis(*args)
        return
    r = error_analysis(*args)
    assert r['error'] == tuple(g[tag + 'error'].tolist())
    assert r['correct_lb'] == g[tag + 'correct_lb'].tolist()
    assert r['predict_lb'] == g[tag + 'predict_lb'].tolist()
    got = [r[n] for n in ('new_score', 'old_score', 'fc_new', 'fc_old', 'bias_new', 'bias_old')]
    _same_means(got, g[tag + 'scores'], _scale(g, tag, batches))


def test_golden_covers_the_edge_cases():
    """Class-incremental and new-instance states, NaN means, an empty meter (0) and the KeyError state are recorded."""
    g = _g()
    names = [str(g['e%d_name' % k]) for k in range(int(g['n_eval']))]
    raised = [str(g['e%d_raised' % k]) for k in range(int(g['n_eval']))]
    assert raised.count('KeyError') == 1 and raised.count('') == len(names) - 1
    scores = np.stack([g['e%d_scores' % k] for k in range(int(g['n_eval'])) if not raised[k]])
    assert np.isnan(scores).any() and (scores[:, 1] == 0).any()
    errors = np.stack([g['e%d_error' % k] for k in range(int(g['n_eval'])) if not raised[k]])
    assert (errors > 0).any(0).all()                       # each of no, nn, oo, on occurs somewhere


def _history(tasks):
    """The label bookkeeping of agents/base.py:43-61 after training on `tasks` (label lists)."""
    old, ctm, zombie = [], {}, []
    for t, labels in enumerate(tasks):
        new = list(set(labels))
        for c in new:
            ctm[c] = t
        old += new
        zombie = list(new)
    return old, zombie, ctm


@pytest.mark.parametrize('tasks,C', [([[0, 1], [2, 3], [4, 5]], 10), ([list(range(69))] * 3, 69),
                                     ([[5, 9], [1, 7, 3]], 12), ([], 4)])
def test_tables_follow_the_label_history(tasks, C):
    from b200ocl.learners import error_analysis_tables
    old, zombie, ctm = _history(tasks)
    sets, task = error_analysis_tables(old, zombie, ctm, C)
    assert sets.dtype == np.uint8 and task.dtype == np.int64 and sets.shape == task.shape == (C,)
    for c in range(C):
        assert bool(sets[c] & 1) == (c in zombie)
        assert bool(sets[c] & 2) == (c in old and c not in zombie)
        assert task[c] == ctm.get(c, -1)
    if tasks and len(set(map(tuple, tasks))) == 1:
        assert not (sets & 2).any()                       # new-instance: no old class outside the last task's


def test_tables_match_the_golden_bookkeeping():
    from b200ocl.learners import error_analysis_tables
    g = _g()
    for k in range(int(g['n_eval'])):
        tag, ctm, _ = _case(g, k)
        zombie, old = g[tag + 'zombie'].tolist(), g[tag + 'old_labels'].tolist()
        sets, task = error_analysis_tables(old, zombie, ctm, g[tag + 'W'].shape[0])
        assert sorted(np.flatnonzero(sets & 1).tolist()) == sorted(set(zombie))
        assert sorted(np.flatnonzero(sets & 2).tolist()) == sorted(set(old) - set(zombie))
        assert all(task[c] == ctm[c] for c in ctm) and (task[[c for c in range(len(task)) if c not in ctm]] == -1).all()


def test_tables_refuse_labels_outside_the_classifier():
    from b200ocl.learners import error_analysis_tables
    with pytest.raises(IndexError):
        error_analysis_tables([0, 12], [12], {0: 0, 12: 1}, 10)


def kernel_outputs(batches, sets, task_of, n_loaders, W, b, zombie, old):
    """What evaluate() reads back after its launches, restated in numpy: per loader the counts of
    b200ocl_linear_argmax_ea, the two b200ocl_rows_mean results, then per batch the predicted tasks and the rows'
    fp64 logit sums (one int64 buffer, as evaluate concatenates it)."""
    counts = np.zeros((n_loaders, 4), dtype=np.int64)
    recs = []
    for t, logits, labels in batches:
        pred = np.argmax(logits, axis=1)                   # first maximum
        pt = task_of[pred]
        sums = np.stack([(logits.astype(np.float64) * ((sets & bit) != 0)).sum(1) for bit in (1, 2)], 1)
        wrong = pred != labels
        m = sets[pred]
        counts[t, 0] += int((wrong & ((m & 1) != 0)).sum())
        counts[t, 1] += int((wrong & ((m & 1) == 0) & ((m & 2) != 0)).sum())
        counts[t, 2] += int((wrong & ((m & 3) == 0)).sum())
        counts[t, 3] += int((pt < 0).sum())
        recs += [pt.astype(np.int64), np.ascontiguousarray(sums).view(np.int64).reshape(-1)]
    with np.errstate(invalid='ignore', divide='ignore'):
        wb = np.array([W[zombie].astype(np.float64).mean() if zombie else np.nan,
                       b[zombie].astype(np.float64).mean() if zombie else np.nan,
                       W[old].astype(np.float64).mean() if old else np.nan,
                       b[old].astype(np.float64).mean() if old else np.nan], dtype=np.float32)
    return np.concatenate([counts.reshape(-1), wb.view(np.int64)] + recs)


class _Learner(object):
    """The attributes ContinualLearner._error_analysis reads and appends to."""

    def __init__(self, task_seen):
        self.task_seen = task_seen
        for n in ('error_list', 'new_class_score', 'old_class_score', 'fc_norm_new', 'fc_norm_old', 'bias_norm_new',
                  'bias_norm_old'):
            setattr(self, n, [])


@pytest.mark.parametrize('k', range(int(np.load(GOLDEN)['n_eval'])))
def test_host_side_reproduces_the_reference(k, tmp_path, monkeypatch):
    from b200ocl.learners import ContinualLearner, error_analysis_tables
    g = _g()
    tag, ctm, batches = _case(g, k)
    zombie = g[tag + 'zombie'].tolist()
    old = sorted(set(g[tag + 'old_labels'].tolist()) - set(zombie))
    W, b = g[tag + 'W'], g[tag + 'b']
    sets, task_of = error_analysis_tables(g[tag + 'old_labels'].tolist(), zombie, ctm, W.shape[0])
    n_loaders = int(g[tag + 'batch_task'].max()) + 1
    if str(g[tag + 'raised']):
        assert len(batches) == 1                          # the reference stopped in its first batch
    host = kernel_outputs(batches, sets, task_of, n_loaders, W, b, zombie, old)
    learner = _Learner(int(g[tag + 'task_seen']))
    monkeypatch.chdir(tmp_path)
    out = io.StringIO()
    acc = np.zeros(n_loaders)
    call = lambda: ContinualLearner._error_analysis(learner, host, n_loaders, [(t, l.shape[0]) for t, l, _ in batches],
                                                    int((sets & 1).astype(bool).sum()),
                                                    int((sets & 2).astype(bool).sum()), acc)
    if str(g[tag + 'raised']):
        with pytest.raises(KeyError):
            call()
        assert not learner.error_list and not os.path.exists('confusion')
        return
    with contextlib.redirect_stdout(out):
        call()
    assert learner.error_list == [tuple(g[tag + 'error'].tolist())]
    got = [learner.new_class_score[0], learner.old_class_score[0], learner.fc_norm_new[0], learner.fc_norm_old[0],
           learner.bias_norm_new[0], learner.bias_norm_old[0]]
    _same_means(got, g[tag + 'scores'], _scale(g, tag, batches))
    with open('confusion', 'rb') as fp:
        correct_lb, predict_lb = pickle.load(fp)
    assert correct_lb == g[tag + 'correct_lb'].tolist() and predict_lb == g[tag + 'predict_lb'].tolist()
    assert all(type(v) is int for v in correct_lb + predict_lb)
    # the printed lines after the accuracies: the ratios and the lists, in the reference's order and format
    want = str(g[tag + 'printed']).splitlines()[1:]
    got_lines = out.getvalue().splitlines()[1:]
    assert len(got_lines) == len(want)
    assert got_lines[:2] == want[:2] and got_lines[2] == want[2]
