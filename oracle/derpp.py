"""Oracle: one DER++ step (learners.DERPP) on the CPU, in the dtype of the ReplayState's parameters (fp64 with
oresnet.seeded_state(..., dtype=torch.float64)), with a logit memory beside the replay memory.

The stream half, the memory cross-entropy, the SGD step and the reservoir update are replay_step's own (er_step); the
draws are the ones er_step makes (numpy for the retrievals, the torch CPU generator for the reservoir), so with
der_alpha = 0 and der_beta = 1 a step equals er_step(retrieve='random', update='random') exactly.  The logit term's
gradient is written out (logit_mse) and fed to the network's backward pass.  Test infrastructure only -- see
oracle/__init__.py.
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

from . import aser as oaser
from . import replay_step as ors
from . import resnet as oresnet


def logit_mse(z, target, alpha):
    """(loss, dz) of alpha * F.mse_loss(z, target) (reduction 'mean' over all n*C entries), written out:
    loss = alpha * sum (z - t)^2 / (n*C), dz = alpha * 2 (z - t) / (n*C)."""
    z = np.asarray(z, dtype=np.float64)
    d = z - np.asarray(target, dtype=np.float64)
    m = float(d.size)
    return float(alpha) * float(np.sum(d * d)) / m, (2.0 * float(alpha) / m) * d


class DerState(ors.ReplayState):
    """ReplayState plus the logit memory [mem_size, num_classes], in the parameters' dtype."""

    def __init__(self, spec, params, bn, mem_size, in_shape, num_classes, lr=0.1, weight_decay=0.0):
        super().__init__(spec, params, bn, mem_size, in_shape, num_classes, lr, weight_decay)
        dtype = next(iter(params.values())).dtype
        self.buffer_logits = torch.zeros((mem_size, num_classes), dtype=dtype)


def _dtype(st):
    return next(iter(st.params.values())).dtype


def _logit_fwd_bwd(st, x, target, alpha):
    """One train-mode forward, the logit term against target and its backward.  Returns (loss, grads)."""
    leaves = OrderedDict((k, v.detach().clone().requires_grad_(True)) for k, v in st.params.items())
    z = oresnet.forward(st.spec, leaves, st.bn, x, train=True)
    loss, dz = logit_mse(z.detach().numpy(), target.numpy(), alpha)
    z.backward(torch.tensor(dz, dtype=z.dtype))
    return loss, OrderedDict((k, v.grad) for k, v in leaves.items())


def _ce_fwd_bwd(st, x, y, w):
    """One train-mode forward, w * mean CE at y and its backward.  Returns (loss, logits, grads)."""
    if w == 1.0:
        return ors._train_fwd_bwd(st, x, y)
    leaves = OrderedDict((k, v.detach().clone().requires_grad_(True)) for k, v in st.params.items())
    z = oresnet.forward(st.spec, leaves, st.bn, x, train=True)
    loss = w * F.cross_entropy(z, y)
    loss.backward()
    return loss.detach(), z.detach(), OrderedDict((k, v.grad) for k, v in leaves.items())


def _add(grads, more):
    for key in grads:
        if grads[key] is not None and more[key] is not None:
            grads[key] = grads[key] + more[key]


def _reservoir_update(st, x, y, logits):
    """replay_step's reservoir update of (x, y), with the logit row of every stored stream row written beside it."""
    place_left = max(0, st.mem_size - st.current_index)
    s = st.current_index
    written = ors._reservoir_update(st, x, y, None)
    if place_left:
        off = min(place_left, x.shape[0])
        st.buffer_logits[s:s + off] = logits[:off]
        if off == x.shape[0]:
            return written
    src = oaser.reservoir_slots(st.log['reservoir_draws'], st.mem_size)[1]
    if written:
        st.buffer_logits[written] = logits[place_left:][src]
    return written


def derpp_step(st, batch_x, batch_y, der_alpha, der_beta, eps_mem_batch=10):
    """One DER++ step (mem_iters = 1): the stream CE, the logit term on a first draw when der_alpha != 0, der_beta times
    the CE of a second draw when der_beta != 0, one SGD step, then the reservoir update with the stream logits.
    Returns (stream loss, logit-term loss or None, memory CE term or None); st.log holds the draws."""
    dtype = _dtype(st)
    x = batch_x.to(dtype)
    loss, logits, grads = ors._train_fwd_bwd(st, x, batch_y)
    loss1 = loss2 = None
    if der_alpha != 0:
        idx1 = ors._random_indices(st, eps_mem_batch)
        st.log['idx1'] = idx1
        if idx1.size:
            loss1, g1 = _logit_fwd_bwd(st, st.buffer_img[idx1].to(dtype), st.buffer_logits[idx1], der_alpha)
            _add(grads, g1)
    if der_beta != 0:
        idx2 = ors._random_indices(st, eps_mem_batch)
        st.log['idx2'] = idx2
        if idx2.size:
            loss2, _, g2 = _ce_fwd_bwd(st, st.buffer_img[idx2].to(dtype), st.buffer_label[idx2], der_beta)
            _add(grads, g2)
            loss2 = float(loss2)
    oresnet.sgd_step(st.params, grads, st.lr, st.wd)
    st.log['written'] = _reservoir_update(st, batch_x, batch_y, logits)
    return float(loss), loss1, loss2
