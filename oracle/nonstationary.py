"""The non-stationary new-instance tasks (--cl_type ni --ns_type noise|occlusion) in numpy: Original, Noisy and
Occlusion `.next_task(factor)` of continuum/non_stationary.py:9-124 (each built with color=True) and the task loop of
construct_ns_multiple (:182-206), with the same RNG calls in the same order -- per task train, then val, then test;
np.random.normal for the noise, random.randint for the occlusion centre.  Every array comes out float64 NHWC in
[0, 1].  Blur (skimage's gaussian) is not restated: a blurred task is just another float64 array in [0, 1].
"""
import random

import numpy as np


def original(x):
    """Original(color=True).next_task(): x / 255 as float64."""
    return x / 255.0


def noisy(x, factor, sig=0.1):
    """Noisy(color=True).next_task(factor): Gaussian noise of scale sig times factor, clipped to [0, 1]."""
    x = x / 255.0
    return np.clip(x + factor * np.random.normal(loc=0.0, scale=sig, size=x.shape), 0.0, 1.0)


def occlusion(x, factor):
    """Occlusion(color=True).next_task(factor): one square of side int(factor * H), set to 1.0 in every image of the
    task, its centre drawn with random.randint (rows first, then columns)."""
    x = x / 255.0
    size = x.shape[1]
    half = int(factor * size) // 2
    lo, hi = min(half, size - half), max(half, size - half)
    cr = random.randint(lo, hi)
    cc = random.randint(lo, hi)
    x[:, max(cr - half, 0):min(cr + half, size), max(cc - half, 0):min(cc + half, size)] = 1
    return x


def next_task(x, ns_type, factor):
    """One task's images: factor 0 gives the original task, whatever ns_type is."""
    if factor == 0:
        return original(x)
    if ns_type == 'noise':
        return noisy(x, factor)
    if ns_type == 'occlusion':
        return occlusion(x, factor)
    raise NotImplementedError('ns_type %r is not restated (blur needs skimage)' % (ns_type,))


def construct_ns_multiple(train_x, train_y, val_x, val_y, test_x, test_y, ns_type, factors):
    """(train, val, test) lists of (images, labels), one entry per factor; labels pass through unchanged."""
    train, val, test = [], [], []
    for i, factor in enumerate(factors):
        train.append((next_task(train_x[i], ns_type, factor), train_y[i]))
        val.append((next_task(val_x[i], ns_type, factor), val_y[i]))
        test.append((next_task(test_x[i], ns_type, factor), test_y[i]))
    return train, val, test
