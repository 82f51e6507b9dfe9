"""Oracle: supervised-contrastive loss and its gradient, all-views-anchor mode.

Restates ``SupConLoss.forward`` (reference utils/loss.py:19-96) in numpy, with
the analytic gradient the fused CUDA kernel produces (csrc/supcon.cu).  Test
infrastructure only -- see oracle/__init__.py.

With A = V*B anchors in *view-major* order (loss.py:56: cat(unbind(features,1))):
    l_ij   = c_i . c_j / T                                   (loss.py:67-69)
    mx_i   = max_j l_ij   (diagonal included, detached)      (loss.py:71-72)
    Z_i    = sum_{j != i} exp(l_ij - mx_i)                   (loss.py:77-86)
    P(i)   = { j != i : label_j == label_i }                 (loss.py:51,75,83)
    loss   = -(1/A) sum_i [ sum_{j in P(i)} (l_ij - mx_i - log Z_i) ] / |P(i)|   (loss.py:87-94)
No base_temperature factor (loss.py:93 differs from upstream SupContrast).
Gradient:  G_ij = (exp(l_ij - mx_i)/Z_i - 1[j in P(i)]/|P(i)|) / A  for j != i, 0 on the diagonal;
           dL/dc = (G + G^T) c / T.
"""
import numpy as np


def supcon_loss_and_grad(features, labels, temperature=0.07, dtype=np.float64, finite_grad=False):
    """features [B,V,...] float, labels [B] int -> (loss scalar, dfeatures [B,V,d]).
    finite_grad: an anchor without positives takes 0 as its positive term 1[j in P(i)]/|P(i)| (the kernels'
    gradient, csrc/supcon.cu) instead of 0/0; the loss is NaN either way."""
    f = np.asarray(features, dtype=dtype)
    if f.ndim < 3:
        raise ValueError('`features` needs to be [bsz, n_views, ...]')   # loss.py:36-38
    B, V = f.shape[0], f.shape[1]
    f = f.reshape(B, V, -1)
    labels = np.asarray(labels).reshape(-1)
    if labels.shape[0] != B:
        raise ValueError('Num of labels does not match num of features')  # loss.py:49-50
    d = f.shape[2]
    A = V * B
    c = f.transpose(1, 0, 2).reshape(A, d)            # view-major, loss.py:56
    lab = np.tile(labels, V)
    logits = (c @ c.T) / dtype(temperature)
    mx = logits.max(axis=1, keepdims=True)
    sh = logits - mx
    off = 1.0 - np.eye(A, dtype=dtype)
    pos = (lab[:, None] == lab[None, :]).astype(dtype) * off
    e = np.exp(sh) * off
    Z = e.sum(1, keepdims=True)
    log_prob = sh - np.log(Z)
    npos = pos.sum(1)
    with np.errstate(invalid='ignore', divide='ignore'):
        mean_lp = (pos * log_prob).sum(1) / npos       # 0/0 -> nan, as loss.py:90
        loss = -mean_lp.mean()
        inv_np = np.where(npos > 0, 1.0 / npos, 0.0) if finite_grad else 1.0 / npos
        G = (e / Z - pos * inv_np[:, None]) / A
    G = G * off
    dc = ((G + G.T) @ c) / dtype(temperature)
    dfeat = dc.reshape(V, B, d).transpose(1, 0, 2)
    return dtype(loss), dfeat


def supcon_loss_only(features, labels, temperature=0.07, dtype=np.float64):
    return supcon_loss_and_grad(features, labels, temperature, dtype)[0]


def supcon_loss_and_grad_torch(features, labels, temperature=0.07, finite_grad=False, drop_last_contrast=False,
                               block=2048):
    """The same in float64 with torch on the features' device, one block of anchor rows at a time (memory
    O(block * A) instead of O(A^2)), for anchor sets too large for the dense form above.
    drop_last_contrast: the last anchor (view-major order) is left out of every contrast set and gives no gradient
    term, i.e. the loss and gradient of a kernel that missed that contrast row."""
    import torch
    f = torch.as_tensor(features).to(torch.float64)
    B, V = f.shape[0], f.shape[1]
    f = f.reshape(B, V, -1)
    lab = torch.as_tensor(labels, device=f.device).reshape(-1)
    if lab.shape[0] != B:
        raise ValueError('Num of labels does not match num of features')
    d, A, T = f.shape[2], B * V, float(temperature)
    c = f.transpose(0, 1).reshape(A, d)
    lab = lab.repeat(V)
    keep = torch.ones(A, dtype=torch.float64, device=f.device)
    if drop_last_contrast:
        keep[A - 1] = 0
    lse = torch.empty(A, dtype=torch.float64, device=f.device)
    npos = torch.empty_like(lse)
    mean_lp = torch.empty_like(lse)

    def rows(s, e):
        logits = (c[s:e] @ c.T) / T
        off = keep[None, :].repeat(e - s, 1)
        off[torch.arange(e - s), torch.arange(s, e)] = 0
        pos = (lab[s:e, None] == lab[None, :]).to(torch.float64) * off
        return logits, off, pos

    for s in range(0, A, block):
        e = min(A, s + block)
        logits, off, pos = rows(s, e)
        mx = logits.max(1, keepdim=True).values
        Z = (torch.exp(logits - mx) * off).sum(1, keepdim=True)
        lse[s:e] = (mx + torch.log(Z)).squeeze(1)
        npos[s:e] = pos.sum(1)
        mean_lp[s:e] = (pos * (logits - mx - torch.log(Z))).sum(1) / npos[s:e]
    loss = -mean_lp.mean()
    inv_np = torch.where(npos > 0, 1.0 / npos, torch.zeros_like(npos)) if finite_grad else 1.0 / npos
    dc = torch.empty_like(c)
    for s in range(0, A, block):
        e = min(A, s + block)
        logits, off, pos = rows(s, e)
        # G_ij + G_ji (l and the same-label test are symmetric); G_ji needs i in anchor j's contrast set
        same = (lab[s:e, None] == lab[None, :]).to(torch.float64)
        off_t = (1.0 - (torch.arange(s, e, device=f.device)[:, None] == torch.arange(A, device=f.device)[None, :])
                 .to(torch.float64)) * keep[s:e, None]
        W = (torch.exp(logits - lse[s:e, None]) - pos * inv_np[s:e, None]) * off \
            + (torch.exp(logits - lse[None, :]) - same * off_t * inv_np[None, :]) * off_t
        dc[s:e] = (W @ c) / (A * T)
    return float(loss), dc.reshape(V, B, d).transpose(0, 1)
