"""fp64 restatement of GDumb's step (agents/gdumb.py:75-83): mean cross-entropy, backward,
torch.nn.utils.clip_grad_norm_(parameters, clip) and one torch.optim.SGD step.
"""
import numpy as np
import torch

from . import resnet as oresnet


def dropin_inputs(rs, hw, n_label, n_per_call, n_calls):
    """Seeded inputs of a GDumb drop-in golden run (tests/golden/make_golden_gdumb.py and tests/test_gpu_gdumb.py both
    draw them from here): per call n_per_call uint8 NHWC images whose labels come from that call's share of the
    n_label classes, and two test sets of 96 images over all the classes."""
    k = n_label // n_calls
    calls = []
    for c in range(n_calls):
        y = (c * k + np.arange(n_per_call) % k)[rs.permutation(n_per_call)].astype(np.int64)
        calls.append((rs.randint(0, 256, (n_per_call, hw, hw, 3)).astype(np.uint8), y))
    tests = [(rs.randint(0, 256, (96, hw, hw, 3)).astype(np.uint8), rs.permutation(np.arange(96) % n_label).astype(np.int64))
             for _ in range(2)]
    return calls, tests


def clip_norm(grads):
    """(total L2 norm in fp64, coefficient min(max_norm / (norm + 1e-6), 1) as a function of max_norm) over the
    gradients that exist (torch/nn/utils/clip_grad.py skips parameters whose .grad is None)."""
    sq = sum(float(np.sum(np.asarray(g, np.float64) ** 2)) for g in grads if g is not None)
    norm = float(np.sqrt(sq))
    return norm, lambda max_norm: min(float(max_norm) / (norm + 1e-6), 1.0)


def clip_grads(grads, max_norm):
    """clip_grad_norm_ on fp64 copies: (scaled gradients, norm before clipping)."""
    norm, coef = clip_norm(grads)
    c = coef(max_norm)
    return [None if g is None else np.asarray(g, np.float64) * c for g in grads], norm


def train_mem_step(spec, params, bn, x, y, lr, weight_decay, max_norm):
    """One inner step of train_mem (gdumb.py:75-83) on the CPU: train-mode forward (running statistics move), mean CE,
    backward, clip_grad_norm_, SGD.  params / bn are updated in place; returns (loss, norm before clipping)."""
    loss, _, grads = oresnet.ce_loss_and_grads(spec, params, bn, x, y)
    names = list(grads)
    clipped, norm = clip_grads([None if grads[k] is None else grads[k].double().numpy() for k in names], max_norm)
    scaled = {k: None if g is None else torch.from_numpy(g).to(params[k].dtype) for k, g in zip(names, clipped)}
    oresnet.sgd_step(params, scaled, lr, weight_decay)
    return float(loss), norm
