"""Oracle: the error analysis of ``ContinualLearner.evaluate`` (reference agents/base.py:144-226, ``--error_analysis``) in
float64, from the logits of every test batch, its labels and the learner's label bookkeeping.

Per batch of loader ``task``: pred = first arg-max of the logits; correct_lb gets [task] * B and predict_lb the
class_task_map entry of every prediction (KeyError where there is none, in any loader).  Old test (task <
task_seen - 1): a wrong prediction into new_labels_zombie counts as on, any other wrong one as oo, and the batch mean of
the logits over the columns set(old_labels) - set(zombie) goes into the old-class meter with weight B.  New test (task
== task_seen - 1): a wrong prediction into set(old_labels) - set(zombie) counts as no, any other as nn; the mean over the
zombie columns goes into the new-class meter.  Later loaders only add to the two lists.  A meter's average is 0 when it
saw no batch; a mean over an empty column set is NaN.  Finally the means of weight[zombie], weight[old - zombie],
bias[zombie] and bias[old - zombie].
Test infrastructure only -- see oracle/__init__.py."""
import numpy as np

from .evaluate import first_argmin


def _mean(a):
    a = np.asarray(a, dtype=np.float64)
    return float(a.sum() / a.size) if a.size else float('nan')


def error_analysis(batches, task_seen, old_labels, zombie, class_task_map, weight, bias):
    """batches: [(task, logits [B,C], labels [B])] in evaluation order.  Returns a dict with error = (no, nn, oo, on),
    new_score, old_score, fc_new, fc_old, bias_new, bias_old, correct_lb and predict_lb; raises KeyError on a
    prediction class_task_map has no entry for."""
    zombie = list(dict.fromkeys(int(c) for c in zombie))
    z = set(zombie)
    old = sorted(set(int(c) for c in old_labels) - z)
    no = nn = oo = on = 0
    meters = {'new': [0.0, 0], 'old': [0.0, 0]}
    correct_lb, predict_lb = [], []
    for task, logits, labels in batches:
        logits = np.asarray(logits, dtype=np.float64)
        labels = np.asarray(labels).reshape(-1)
        pred = first_argmin(-logits)
        n = labels.size
        correct_lb += [int(task)] * n
        predict_lb += [class_task_map[int(p)] for p in pred]
        wrong = pred[pred != labels]
        if task < task_seen - 1:
            on_tmp = int(np.isin(wrong, zombie).sum())
            oo += wrong.size - on_tmp
            on += on_tmp
            meters['old'][0] += _mean(logits[:, old]) * n
            meters['old'][1] += n
        elif task == task_seen - 1:
            no_tmp = int(np.isin(wrong, old).sum())
            no += no_tmp
            nn += wrong.size - no_tmp
            meters['new'][0] += _mean(logits[:, zombie]) * n
            meters['new'][1] += n
    avg = {k: (s / c if c else 0) for k, (s, c) in meters.items()}
    w, b = np.asarray(weight, dtype=np.float64), np.asarray(bias, dtype=np.float64).reshape(-1)
    return dict(error=(no, nn, oo, on), new_score=avg['new'], old_score=avg['old'],
                fc_new=_mean(w[zombie]), fc_old=_mean(w[old]), bias_new=_mean(b[zombie]), bias_old=_mean(b[old]),
                correct_lb=correct_lb, predict_lb=predict_lb)
