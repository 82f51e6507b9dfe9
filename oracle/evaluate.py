"""Oracle: the classification inside ``ContinualLearner.evaluate`` (reference agents/base.py:118-175) in float64.

Nearest class mean (SCR, iCaRL, ncm_trick):
    feature f / ||f|| per buffered exemplar; mu_y = mean of those over the exemplars of class y, then mu_y / ||mu_y||;
    a class without exemplars gets a standard-normal draw of the feature's size, normalised (base.py:135-137);
    prediction for a test feature: the class whose mean is nearest to f / ||f|| in squared distance, first on ties
    (dists.min(1), base.py:170-171), mapped through old_labels.
Arg-max (everything else): the first largest logit f . w_c + b_c (torch.max(logits, 1), base.py:178-179).
Test infrastructure only -- see oracle/__init__.py."""
import numpy as np


def class_means(feats, labels, class_ids, draws=None):
    """(means [K,d], counts [K]) in float64.  draws: one vector per class without exemplars, in class order (the
    random mean before its normalisation); without draws those rows are left zero."""
    f = np.asarray(feats, dtype=np.float64)
    labels = np.asarray(labels).reshape(-1)
    K, d = len(class_ids), f.shape[1]
    means, counts = np.zeros((K, d)), np.zeros(K, dtype=np.int64)
    draws = list(draws) if draws is not None else None
    for k, cls in enumerate(class_ids):
        rows = f[labels == cls]
        counts[k] = rows.shape[0]
        if rows.shape[0]:
            mu = (rows / np.linalg.norm(rows, axis=1, keepdims=True)).mean(0)
        elif draws is not None:
            mu = np.asarray(draws.pop(0), dtype=np.float64).reshape(d)
        else:
            continue
        means[k] = mu / np.linalg.norm(mu)
    return means, counts


def ncm_distances(feats, means):
    """[B,K] squared distances between each normalised feature and each class mean, in float64."""
    f = np.asarray(feats, dtype=np.float64)
    with np.errstate(invalid='ignore', divide='ignore'):
        fn = f / np.linalg.norm(f, axis=1, keepdims=True)
    diff = fn[:, None, :] - np.asarray(means, dtype=np.float64)[None, :, :]
    return (diff * diff).sum(2)


def linear_logits(feats, weight, bias):
    return np.asarray(feats, np.float64) @ np.asarray(weight, np.float64).T + np.asarray(bias, np.float64)[None, :]


def first_argmin(scores):
    """Index of the first minimum of each row; a row holding NaN gives its first NaN, as torch's min does."""
    s = np.asarray(scores)
    nan = np.isnan(s)
    return np.where(nan.any(1), nan.argmax(1), np.argmin(np.where(nan, np.inf, s), axis=1))


def margins(scores, pick):
    """scores[b, pick[b]] minus the smallest score of row b: 0 where pick is an arg-min."""
    s = np.asarray(scores, dtype=np.float64)
    return s[np.arange(s.shape[0]), pick] - s.min(1)


def ncm_predict(feats, means, class_ids):
    return np.asarray(class_ids)[first_argmin(ncm_distances(feats, means))]


def linear_predict(feats, weight, bias):
    return first_argmin(-linear_logits(feats, weight, bias))
