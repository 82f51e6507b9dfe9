"""Oracle: one A-GEM step (agents/agem.py:36-84, learners.AGEM.replay_step) on the CPU, in the dtype of the
ReplayState's parameters (float64 with oresnet.seeded_state(..., dtype=torch.float64)).

Per memory iteration: the train-mode forward and backward of the stream batch with the trick / distillation mixing of
agem.py:40-46; once a task has been seen and the memory is not empty, a random retrieve on the reference's random
streams (numpy, ors._random_indices), the train-mode forward of the memory batch (its BN running statistics move too)
and the backward of its criterion without the distillation term; then the projection of :71-80 and one SGD or Adam
step.  After the iterations, the reservoir update of replay_step.  Test infrastructure only -- see oracle/__init__.py.
"""
import math
from collections import OrderedDict

import numpy as np
import torch

from . import replay_step as ors
from . import resnet as oresnet
from . import tricks as otricks


def dropin_inputs(rs, mem, hw, batch, n_calls):
    """Seeded inputs of an A-GEM drop-in golden run (tests/golden/make_golden_agem_maps.py and
    tests/test_gpu_agem_fp64.py both draw them from here): the draws of make_golden.py dropin_inputs over 10 labels,
    with the memory's labels folded onto classes 0-4 and every call's onto classes 5-9, so that the calls' gradients
    can point away from the memory's (the projection branch).  Returns (x, y, calls, tests)."""
    x = rs.rand(mem, 3, hw, hw).astype(np.float32)
    y = rs.randint(0, 10, mem).astype(np.int64) % 5
    calls = []
    for _ in range(n_calls):
        n = batch + 3
        calls.append((rs.randint(0, 256, (n, hw, hw, 3)).astype(np.uint8), rs.permutation(np.arange(n) % 10) % 5 + 5))
    tests = [(rs.randint(0, 256, (96, hw, hw, 3)).astype(np.uint8), rs.permutation(np.arange(96) % 10).astype(np.int64))
             for _ in range(2)]
    return x, y, calls, tests


def flat(grads):
    """The flat gradient vector in model.parameters() order (the engine's gradient arena), as float64 numpy."""
    return np.concatenate([g.detach().double().reshape(-1).numpy() for g in grads.values()])


def project(g, g_ref):
    """agem.py:71-80 on flat float64 vectors: (projected g, prod, prod_ref, projected?).  prod_ref is formed whatever
    the decision (the kernel reports both dots)."""
    g, g_ref = np.asarray(g, np.float64), np.asarray(g_ref, np.float64)
    prod = float(np.dot(g, g_ref))
    prod_ref = float(np.dot(g_ref, g_ref))
    if prod < 0:
        return g - (prod / prod_ref) * g_ref, prod, prod_ref, True
    return g.copy(), prod, prod_ref, False


def _unflat(st, v):
    out, o = OrderedDict(), 0
    for k, p in st.params.items():
        out[k] = torch.from_numpy(v[o:o + p.numel()].reshape(p.shape).copy()).to(p.dtype)
        o += p.numel()
    return out


def _fwd_bwd(st, x, y, mode, teacher, w_ce, w_kd, old_labels=(), new_labels=(), lbl_inv_map=None):
    """Train-mode forward, w_ce * criterion(mode) + w_kd * kd(teacher logits) and its backward: (loss, logits, grads).
    Plain CE without distillation is replay_step's own _train_fwd_bwd."""
    x = x.to(next(iter(st.params.values())).dtype)
    if mode == 'ce' and teacher is None and w_ce == 1.0:
        return ors._train_fwd_bwd(st, x, y)
    t = None
    if teacher is not None and w_kd != 0.0:
        tp, tbn = teacher
        with torch.no_grad():                          # kd_manager.py:24-25: a train-mode copy, its statistics move
            t = oresnet.forward(st.spec, tp, tbn, x, train=True).numpy()
    leaves = OrderedDict((k, v.detach().clone().requires_grad_(True)) for k, v in st.params.items())
    z = oresnet.forward(st.spec, leaves, st.bn, x, train=True)
    loss, dz = otricks.criterion(z.detach().numpy(), y.numpy(), mode, old_labels, new_labels, lbl_inv_map, t, w_ce,
                                 w_kd if t is not None else 0.0)
    z.backward(torch.tensor(dz, dtype=z.dtype))
    return loss, z.detach(), OrderedDict((k, v.grad) for k, v in leaves.items())


class AdamState:
    """torch.optim.Adam's per-parameter state (amsgrad and decoupled weight decay off), in float64."""

    def __init__(self, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        self.m, self.v, self.t = None, None, 0

    def step(self, params, grads):
        b1, b2 = self.betas
        if self.m is None:
            self.m = OrderedDict((k, torch.zeros_like(p)) for k, p in params.items())
            self.v = OrderedDict((k, torch.zeros_like(p)) for k, p in params.items())
        self.t += 1
        bc1, bc2 = 1 - b1 ** self.t, 1 - b2 ** self.t
        for k, p in params.items():
            g = grads[k] + self.wd * p if self.wd else grads[k]
            self.m[k] = b1 * self.m[k] + (1 - b1) * g
            self.v[k] = b2 * self.v[k] + (1 - b2) * g * g
            p.sub_((self.lr / bc1) * self.m[k] / (self.v[k].sqrt() / math.sqrt(bc2) + self.eps))


def step(st, batch_x, batch_y, task_seen, eps_mem_batch=10, mem_iters=1, mode='ce', teacher=None, kd_trick=False,
         kd_trick_star=False, adam=None, old_labels=(), new_labels=(), lbl_inv_map=None, ret_idx=None):
    """One A-GEM step on the ReplayState st (params / bn updated in place).  teacher: (params, bn) of the distillation
    teacher or None; adam: an AdamState or None (SGD at st.lr, st.wd); ret_idx: the memory slots each iteration's
    retrieve returns, replayed instead of drawn (a recorded run).  Returns a list with one log per memory
    iteration: loss, ret_idx, step_grad (the flat gradient the optimizer step applies), and when a memory batch was
    replayed g, g_ref (flat float64), prod, prod_ref, project."""
    w_ce, w_kd = otricks.mix(task_seen, kd_trick, kd_trick_star)
    logs = []
    for it in range(mem_iters):
        loss, _, grads = _fwd_bwd(st, batch_x, batch_y, mode, teacher, w_ce, w_kd, old_labels, new_labels,
                                  lbl_inv_map)                                                   # :39-54
        log = dict(loss=float(loss), ret_idx=None, project=None)
        if task_seen > 0:
            idx = ors._random_indices(st, eps_mem_batch) if ret_idx is None else np.asarray(ret_idx[it])  # :58
            log['ret_idx'] = idx
            if idx.size:
                _, _, grads_ref = _fwd_bwd(st, st.buffer_img[idx], st.buffer_label[idx], mode, None, 1.0, 0.0,
                                           old_labels, new_labels, lbl_inv_map)                  # :62-70
                g, g_ref = flat(grads), flat(grads_ref)
                out, prod, prod_ref, proj = project(g, g_ref)                                    # :72-77
                log.update(g=g, g_ref=g_ref, prod=prod, prod_ref=prod_ref, project=proj, out=out)
                grads = _unflat(st, out)                                                         # :79-80
        log['step_grad'] = flat(grads)
        if adam is None:
            oresnet.sgd_step(st.params, grads, st.lr, st.wd)                                     # :81
        else:
            adam.step(st.params, grads)
        logs.append(log)
    st.log['written'] = ors._reservoir_update(st, batch_x, batch_y, None)                        # :83
    return logs
