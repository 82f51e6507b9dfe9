"""Oracle: PCR (Lin et al., "PCR: Proxy-based Contrastive Replay for Online Class-Incremental Continual Learning",
CVPR 2023) as learners.PCR runs it, in the dtype of the tensors it is given (fp64 in the GPU tests).

The proxies are the rows of the classifier weight linear.weight [C, d]; eps = 1e-6, tau the temperature:
    u_i = F_i / (||F_i|| + eps),  v_c = W_c / (||W_c|| + eps),  g_ic = <u_i, v_c> / tau
    n_c = #rows labelled c,  m_ic = n_c - [c = y_i],  Z_i = sum_c m_ic exp(g_ic)
    l_i = log Z_i - g_{i,y_i},  L = (1/R) sum_i l_i
With p_ic = m_ic exp(g_ic) / Z_i:
    dL/du_i = (sum_c p_ic v_c - v_{y_i}) / (tau R),   dL/dv_c = sum_i (p_ic - [y_i = c]) u_i / (tau R)
and through each normalisation dx = g / (n + eps) - x <x, g> / (n (n + eps)^2), the second term 0 at n = 0.  An anchor
whose class occurs once has no positive: its l_i is NaN and its gradients keep the log Z_i part only.

`step` is one learners.PCR.replay_step on replay_step.ReplayState: random retrieval on numpy's stream (as ER's), x' =
transform(x) then m' = transform(m), the train-mode forwards of [x; x'] and [m; m'] in that order, the loss of
[F_m; F_m'; F_x; F_x'], the backward, SGD (st.lr, st.wd) or an agem.AdamState step, then the reservoir update.
Test infrastructure only -- see oracle/__init__.py.
"""
from collections import OrderedDict

import numpy as np
import torch

from . import replay_step as ors
from . import resnet as oresnet

EPS = 1e-6


def _norm_backward(x, n, den, g):
    """d/dx of x / (||x|| + eps) applied to g, rowwise: g / den - x <x, g> / (n den^2), the second term 0 at n = 0."""
    dot = (x * g).sum(1)
    safe = torch.where(n > 0, n, torch.ones_like(n))
    t = torch.where(n > 0, dot / (safe * den * den), torch.zeros_like(n))
    return g / den[:, None] - x * t[:, None]


def loss_and_grads(feats, labels, proxies, temperature):
    """(loss, dfeats [R,d], dproxies [C,d]) of the proxy-contrastive loss, written out, in the dtype of feats.  The bias
    gradient is zero.  Labels must lie in [0, C)."""
    F = torch.as_tensor(feats)
    W = torch.as_tensor(proxies).to(F.dtype)
    y = torch.as_tensor(labels).to(torch.int64).reshape(-1)
    R, C = F.shape[0], W.shape[0]
    tau = float(temperature)
    nf = F.norm(dim=1)
    fden = nf + EPS
    u = F / fden[:, None]
    nw = W.norm(dim=1)
    wden = nw + EPS
    v = W / wden[:, None]
    g = (u @ v.T) / tau
    onehot = torch.zeros((R, C), dtype=F.dtype)
    onehot[torch.arange(R), y] = 1
    n = onehot.sum(0)
    m = n[None, :] - onehot
    gmax = torch.where(m > 0, g, torch.full_like(g, -float('inf'))).max(1, keepdim=True).values
    e = m * torch.exp(g - gmax)
    Z = e.sum(1, keepdim=True)
    p = e / Z
    pos = (n[y] > 1).to(F.dtype)
    lse = torch.log(Z[:, 0]) + gmax[:, 0]
    li = lse - g[torch.arange(R), y]
    li = torch.where(pos > 0, li, torch.full_like(li, float('nan')))
    loss = li.mean()
    coef = p - onehot * pos[:, None]
    du = (coef @ v) / (tau * R)
    dv = (coef.T @ u) / (tau * R)
    return loss, _norm_backward(F, nf, fden, du), _norm_backward(W, nw, wden, dv)


def cosine_argmax(feats, proxies):
    """arg-max_c <f / (||f|| + eps), w_c / (||w_c|| + eps)> per row, the first maximum on ties (numpy, fp64)."""
    f = np.asarray(feats, dtype=np.float64)
    w = np.asarray(proxies, dtype=np.float64)
    u = f / (np.linalg.norm(f, axis=1, keepdims=True) + EPS)
    v = w / (np.linalg.norm(w, axis=1, keepdims=True) + EPS)
    return np.argmax(u @ v.T, axis=1)


def step(st, batch_x, batch_y, eps_mem_batch=10, mem_iters=1, temperature=0.09, transform=None, adam=None,
         ret_idx=None):
    """One PCR step on the ReplayState st (params / bn updated in place).  transform: the augmentation T, called as
    transform(x) on the stream batch first and on the memory batch second (identity when None).  adam: an
    agem.AdamState or None (SGD at st.lr, st.wd).  ret_idx: the memory slots each iteration's retrieve returns,
    replayed instead of drawn.  Returns one log per memory iteration: ret_idx, and when a memory batch was drawn the
    loss, the features F and the gradient each parameter's step applied."""
    dtype = next(iter(st.params.values())).dtype
    x = batch_x.to(dtype)
    logs = []
    for it in range(mem_iters):
        idx = ors._random_indices(st, eps_mem_batch) if ret_idx is None else np.asarray(ret_idx[it])
        log = dict(ret_idx=idx, loss=None)
        logs.append(log)
        if idx.size == 0:
            continue
        mem_x, mem_y = st.buffer_img[idx].to(dtype), st.buffer_label[idx]
        x_aug = x if transform is None else transform(batch_x).to(dtype)
        m_aug = mem_x if transform is None else transform(st.buffer_img[idx]).to(dtype)
        leaves = OrderedDict((k, v.detach().clone().requires_grad_(True)) for k, v in st.params.items())
        fx = oresnet.features(st.spec, leaves, st.bn, torch.cat((x, x_aug)), train=True)
        fm = oresnet.features(st.spec, leaves, st.bn, torch.cat((mem_x, m_aug)), train=True)
        feats = torch.cat((fm, fx)).detach()
        labels = torch.cat((mem_y, mem_y, batch_y, batch_y))
        loss, dF, dW = loss_and_grads(feats, labels, st.params['linear.weight'], temperature)
        M = idx.size
        torch.autograd.backward([fm, fx], [dF[:2 * M], dF[2 * M:]])
        grads = OrderedDict((k, v.grad) for k, v in leaves.items())
        grads['linear.weight'] = dW
        grads['linear.bias'] = torch.zeros_like(st.params['linear.bias'])
        if adam is None:
            oresnet.sgd_step(st.params, grads, st.lr, st.wd)
        else:
            adam.step(st.params, grads)
        log.update(loss=float(loss), feats=feats, grads=grads)
    st.log['written'] = ors._reservoir_update(st, batch_x, batch_y, None)
    return logs
