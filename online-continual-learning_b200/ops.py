"""Tensor-level wrappers over the C ABI (include/b200ocl.h).

Every function takes CUDA torch tensors, hands raw device pointers and the current
CUDA stream to libb200ocl.so and returns torch tensors.  torch is used for memory and
streams only.  Non-CUDA inputs raise: there is no CPU path.
"""
import ctypes

import numpy as np
import torch

from . import _native

KNN_MAX_CAND = 262144    # B200OCL_KNN_MAX_CAND_LARGE (include/b200ocl.h)
RANK_MAX = 4096          # b200ocl_rank_desc limit


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _need_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise _native.NativeError('b200ocl ops need CUDA tensors (got a %s tensor); there is no CPU fallback'
                                      % t.device.type)


def _f32(t):
    return t.detach().to(torch.float32).contiguous()


def _i64(t):
    return t.detach().to(torch.int64).contiguous()


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _workspace(nbytes, device):
    return torch.empty((max(int(nbytes), 256) + 255) // 256 * 256, dtype=torch.uint8, device=device)


def knn_sv(eval_f, eval_y, cand_f, cand_y, k, want_matrix=False, want_sum=True, want_max=False, want_min=False):
    """Fused kNN Shapley values on feature matrices.

    Mirrors compute_knn_sv + its callers' row reductions
    (reference utils/buffer/aser_utils.py:29-59; aser_retrieve.py:79-86; aser_update.py:80).
    Returns dict with any of 'sv' [E,C], 'sum' [C], 'max' [C], 'min' [C]."""
    _need_cuda(eval_f, eval_y, cand_f, cand_y)
    eval_f, cand_f, eval_y, cand_y = _f32(eval_f), _f32(cand_f), _i64(eval_y), _i64(cand_y)
    if eval_f.dim() != 2 or cand_f.dim() != 2 or eval_f.shape[1] != cand_f.shape[1]:
        raise ValueError('eval_f [E,d] and cand_f [C,d] must share d')
    E, d = eval_f.shape
    C = cand_f.shape[0]
    if eval_y.numel() != E or cand_y.numel() != C:
        raise ValueError('label count does not match feature count')
    dev = eval_f.device
    out = {}
    sv = torch.empty((E, C), dtype=torch.float32, device=dev) if want_matrix else None
    cs = torch.empty(C, dtype=torch.float32, device=dev) if want_sum else None
    cx = torch.empty(C, dtype=torch.float32, device=dev) if want_max else None
    cn = torch.empty(C, dtype=torch.float32, device=dev) if want_min else None
    L = _native.lib()
    ws_bytes = L.b200ocl_knn_sv_workspace_bytes(E, C, d)
    ws = _workspace(ws_bytes, dev)
    rc = L.b200ocl_knn_sv(_ptr(eval_f), _ptr(eval_y), _ptr(cand_f), _ptr(cand_y), E, C, d, int(k),
                          _ptr(sv), _ptr(cs), _ptr(cx), _ptr(cn), _ptr(ws), ws.numel(), _stream())
    _native.check(rc, 'b200ocl_knn_sv')
    if want_matrix:
        out['sv'] = sv
    if want_sum:
        out['sum'] = cs
    if want_max:
        out['max'] = cx
    if want_min:
        out['min'] = cn
    return out


class KnnLaunch(ctypes.Structure):
    """b200ocl_knn_launch: the kernel one b200ocl_knn_sv call runs."""
    _fields_ = [('family', ctypes.c_int), ('kpl', ctypes.c_int), ('te', ctypes.c_int), ('wide', ctypes.c_int),
                ('cpad', ctypes.c_int), ('block_keys', ctypes.c_int), ('far_stages', ctypes.c_int),
                ('grid', ctypes.c_int), ('n_tiles', ctypes.c_int), ('tiles_per_cta', ctypes.c_int),
                ('smem_bytes', ctypes.c_size_t), ('smem_limit', ctypes.c_size_t), ('part_bytes', ctypes.c_size_t),
                ('key_offset', ctypes.c_size_t), ('key_bytes', ctypes.c_size_t), ('workspace_bytes', ctypes.c_size_t),
                ('sms', ctypes.c_int)]

    FAMILIES = ('fused', 'large')

    @property
    def name(self):
        return self.FAMILIES[self.family]

    @property
    def kernel(self):
        """(KPL, TE, 'wide' | 'rows') of a fused launch, ('large', block keys, far stages) of a scratch-line one."""
        if self.name == 'large':
            return ('large', self.block_keys, self.far_stages)
        return (self.kpl, self.te, 'wide' if self.wide else 'rows')


def knn_sv_plan(E, C, d, aligned=True, want_red=True, sms=0):
    """Host-only test hook (b200ocl_knn_sv_plan): the launch knn_sv() makes for E eval rows, C candidates of width d on
    a GPU with sms SMs (0: the current device); aligned: both feature pointers are 16-byte aligned; want_red: any of
    the column reductions is asked for."""
    out = KnnLaunch()
    _native.check(_native.lib().b200ocl_knn_sv_plan(int(E), int(C), int(d), 1 if aligned else 0, 1 if want_red else 0,
                                                    int(sms), ctypes.byref(out)), 'b200ocl_knn_sv_plan')
    return out


def rank_desc(a, n_out=None, sa=1.0, b=None, sb=0.0, return_scores=False):
    """Indices of the n_out largest entries of a*sa + b*sb, descending, ties lowest index
    first (sv.argsort(descending=True)[:n], aser_retrieve.py:88-91)."""
    _need_cuda(a, b)
    a = _f32(a).reshape(-1)
    n = a.numel()
    if b is not None:
        b = _f32(b).reshape(-1)
        if b.numel() != n:
            raise ValueError('a and b differ in length')
    n_out = n if n_out is None else min(int(n_out), n)
    idx = torch.empty(n_out, dtype=torch.int64, device=a.device)
    sc = torch.empty(n, dtype=torch.float32, device=a.device) if return_scores else None
    rc = _native.lib().b200ocl_rank_desc(_ptr(a), float(sa), _ptr(b), float(sb), n, _ptr(idx), n_out, _ptr(sc),
                                         _stream())
    _native.check(rc, 'b200ocl_rank_desc')
    return (idx, sc) if return_scores else idx


def supcon(features, labels, temperature, need_grad=True):
    """Fused SupCon loss (+ gradient w.r.t. features).  features [B,V,...], labels [B].
    Returns (loss[1] tensor, dfeatures or None).  utils/loss.py:19-96."""
    _need_cuda(features, labels)
    if features.dim() < 3:
        raise ValueError('`features` needs to be [bsz, n_views, ...],at least 3 dimensions are required')
    B, V = features.shape[0], features.shape[1]
    f = _f32(features).reshape(B, V, -1)
    labels = _i64(labels).reshape(-1)
    if labels.shape[0] != B:
        raise ValueError('Num of labels does not match num of features')
    d = f.shape[2]
    loss = torch.empty(1, dtype=torch.float32, device=f.device)
    grad = torch.empty_like(f) if need_grad else None
    L = _native.lib()
    ws = _workspace(L.b200ocl_supcon_workspace_bytes(B, V, d), f.device)
    rc = L.b200ocl_supcon(_ptr(f), _ptr(labels), B, V, d, float(temperature), _ptr(loss), _ptr(grad), _ptr(ws),
                          ws.numel(), _stream())
    _native.check(rc, 'b200ocl_supcon')
    return loss, grad


class SupconLaunch(ctypes.Structure):
    """b200ocl_supcon_launch: the kernels one b200ocl_supcon call runs."""
    _fields_ = [('family', ctypes.c_int), ('rm', ctypes.c_int), ('rn', ctypes.c_int), ('nc', ctypes.c_int),
                ('dch', ctypes.c_int), ('grid', ctypes.c_int), ('n_units', ctypes.c_int),
                ('units_per_cta', ctypes.c_int), ('smem_bytes', ctypes.c_size_t), ('smem_limit', ctypes.c_size_t),
                ('tx_bytes', ctypes.c_size_t), ('sms', ctypes.c_int)]

    FAMILIES = ('resident', 'ring16', 'ring64', 'fallback')

    @property
    def name(self):
        return self.FAMILIES[self.family]

    @property
    def kernel(self):
        """(family, NC) of a fused launch, ('fallback', DCH) of the two-kernel one."""
        return (self.name, self.dch if self.name == 'fallback' else self.nc)


def supcon_plan(B, V, d, aligned=True, sms=0):
    """Host-only test hook (b200ocl_supcon_plan): the launch supcon() makes for features [B,V,d] on a GPU with sms
    SMs (0: the current device); aligned: the feature and gradient pointers are 16-byte aligned."""
    out = SupconLaunch()
    _native.check(_native.lib().b200ocl_supcon_plan(int(B), int(V), int(d), 1 if aligned else 0, int(sms),
                                                    ctypes.byref(out)), 'b200ocl_supcon_plan')
    return out


def gather_rows(src, idx, out=None):
    """out[i] = src[idx[i]] over the first dimension (buffer_img[indices])."""
    _need_cuda(src, idx, out)
    if not src.is_contiguous():
        raise ValueError('src must be contiguous')
    idx = _i64(idx).reshape(-1)
    n = idx.numel()
    row_bytes = src[0].numel() * src.element_size() if src.shape[0] > 0 else 0
    if out is None:
        out = torch.empty((n,) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device)
    elif not out.is_contiguous() or out.dtype != src.dtype or out.shape[0] < n:
        raise ValueError('bad out tensor')
    if n == 0 or row_bytes == 0:
        return out
    rc = _native.lib().b200ocl_gather_rows(_ptr(src), _ptr(idx), n, row_bytes, _ptr(out), _stream())
    _native.check(rc, 'b200ocl_gather_rows')
    return out


def stream_prepare(x_u8_nhwc, perm=None):
    """uint8 [n,H,W,3] (device) -> fp32 [n,3,H,W] in [0,1], rows taken in `perm` order (ToTensor + shuffle).
    float64 [n,H,W,3] in [0,1] (the non-stationary tasks) -> fp32 [n,3,H,W] rounded to nearest even, bit-identical to
    the CPU's x.permute(0,3,1,2).float()."""
    _need_cuda(x_u8_nhwc, perm)
    if x_u8_nhwc.dtype not in (torch.uint8, torch.float64) or x_u8_nhwc.dim() != 4 or x_u8_nhwc.shape[3] != 3:
        raise ValueError('expected uint8 or float64 images [n,H,W,3]')
    x = x_u8_nhwc.contiguous()
    n, h, w = (perm.numel() if perm is not None else x.shape[0]), x.shape[1], x.shape[2]
    out = torch.empty((n, 3, h, w), dtype=torch.float32, device=x.device)
    if perm is not None:
        perm = _i64(perm).reshape(-1)
    name = 'b200ocl_stream_prepare' if x.dtype == torch.uint8 else 'b200ocl_stream_prepare_f64'
    rc = getattr(_native.lib(), name)(_ptr(x), _ptr(perm), n, h, w, _ptr(out), _stream())
    _native.check(rc, name)
    return out


def ncm_class_means(feats, labels, class_ids):
    """(means [K,d], counts [K] int32): normalised class means of normalised features (agents/base.py:121-141)."""
    _need_cuda(feats, labels, class_ids)
    feats, labels, class_ids = _f32(feats), _i64(labels).reshape(-1), _i64(class_ids).reshape(-1)
    n, d = feats.shape
    K = class_ids.numel()
    means = torch.zeros((K, d), dtype=torch.float32, device=feats.device)
    counts = torch.zeros(K, dtype=torch.int32, device=feats.device)
    rc = _native.lib().b200ocl_ncm_class_means(_ptr(feats), _ptr(labels), n, d, _ptr(class_ids), K, _ptr(means),
                                               _ptr(counts), _stream())
    _native.check(rc, 'b200ocl_ncm_class_means')
    return means, counts


def _check_truth(truth, B):
    if truth is None:
        return None
    truth = _i64(truth).reshape(-1)
    if truth.numel() != B:
        raise ValueError('truth must hold one label per feature row')
    return truth


def ncm_classify(feats, means, class_ids, truth=None, n_correct=None):
    """Nearest normalised class mean (agents/base.py:155-170).  Returns pred [B]; adds the number of hits to
    n_correct (uint64 tensor [1], as int64 storage) when truth is given."""
    _need_cuda(feats, means, class_ids, truth, n_correct)
    feats, means, class_ids = _f32(feats), _f32(means), _i64(class_ids).reshape(-1)
    B, d = feats.shape
    if means.dim() != 2 or means.shape[1] != d:
        raise ValueError('means [K,d] must have the features\' width d=%d' % d)
    if class_ids.numel() != means.shape[0]:
        raise ValueError('class_ids must hold one label per class mean')
    truth = _check_truth(truth, B)
    pred = torch.empty(B, dtype=torch.int64, device=feats.device)
    rc = _native.lib().b200ocl_ncm_classify(_ptr(feats), B, d, _ptr(means), means.shape[0], _ptr(class_ids), _ptr(truth),
                                            _ptr(pred), _ptr(n_correct), _stream())
    _native.check(rc, 'b200ocl_ncm_classify')
    return pred


def linear_argmax(feats, weight, bias, truth=None, n_correct=None):
    """arg-max of feats @ weight.T + bias (agents/base.py:172-175)."""
    _need_cuda(feats, weight, bias, truth, n_correct)
    feats, weight, bias = _f32(feats), _f32(weight), _f32(bias).reshape(-1)
    B, d = feats.shape
    if weight.dim() != 2 or weight.shape[1] != d:
        raise ValueError('weight [C,d] must have the features\' width d=%d' % d)
    if bias.numel() != weight.shape[0]:
        raise ValueError('bias must hold one entry per weight row')
    truth = _check_truth(truth, B)
    pred = torch.empty(B, dtype=torch.int64, device=feats.device)
    rc = _native.lib().b200ocl_linear_argmax(_ptr(feats), B, d, _ptr(weight), _ptr(bias), weight.shape[0], _ptr(truth),
                                             _ptr(pred), _ptr(n_correct), _stream())
    _native.check(rc, 'b200ocl_linear_argmax')
    return pred


def linear_argmax_ea(feats, weight, bias, truth, class_sets, class_task, counts, n_correct=None, pred=None):
    """linear_argmax with the error analysis of agents/base.py:177-205 in the same launch (b200ocl_linear_argmax_ea):
    the prediction written to pred and the hits added to n_correct are linear_argmax's, bit for bit.  class_sets
    (uint8 [C]: bit 0 for the last task's labels, bit 1 for the older labels without them) and class_task (int64 [C],
    -1 where unmapped) are the tables of learners.error_analysis_tables on the device; counts (int64 [4]) gains the
    wrong rows predicted into a bit-0 / bit-1 / neither class and the rows predicted into an unmapped class.
    Returns (pred_task [B] int64, set_sums [B,2] float64: each row's logits summed over the bit-0 / bit-1 classes)."""
    _need_cuda(feats, weight, bias, truth, class_sets, class_task, counts, n_correct, pred)
    feats, weight, bias = _f32(feats), _f32(weight), _f32(bias).reshape(-1)
    B, d = feats.shape
    C = weight.shape[0]
    if weight.dim() != 2 or weight.shape[1] != d:
        raise ValueError('weight [C,d] must have the features\' width d=%d' % d)
    if bias.numel() != C:
        raise ValueError('bias must hold one entry per weight row')
    truth = _check_truth(truth, B)
    if class_sets.dtype != torch.uint8 or class_sets.numel() != C or not class_sets.is_contiguous():
        raise ValueError('class_sets must be a contiguous uint8 tensor with one entry per class')
    if class_task.dtype != torch.int64 or class_task.numel() != C or not class_task.is_contiguous():
        raise ValueError('class_task must be a contiguous int64 tensor with one entry per class')
    if counts.dtype != torch.int64 or counts.numel() != 4 or not counts.is_contiguous():
        raise ValueError('counts must be a contiguous int64 tensor of 4')
    if pred is not None and (pred.dtype != torch.int64 or pred.numel() != B or not pred.is_contiguous()):
        raise ValueError('pred must be a contiguous int64 tensor with one entry per row')
    out = torch.empty(3 * B, dtype=torch.int64, device=feats.device)
    pred_task, set_sums = out[:B], out[B:].view(torch.float64).view(B, 2)
    rc = _native.lib().b200ocl_linear_argmax_ea(_ptr(feats), B, d, _ptr(weight), _ptr(bias), C, _ptr(truth),
                                                _ptr(class_sets), _ptr(class_task), _ptr(pred), _ptr(n_correct),
                                                _ptr(pred_task), _ptr(set_sums), _ptr(counts), _stream())
    _native.check(rc, 'b200ocl_linear_argmax_ea')
    return pred_task, set_sums


def rows_mean(weight, bias, rows, out=None):
    """(mean of weight[rows], mean of bias[rows]) as a float32 tensor [2] on the device, each summed in fp64 and
    rounded once (b200ocl_rows_mean); an empty row list gives NaN.  rows: a sequence of ints in [0, C)."""
    _need_cuda(weight, bias, out)
    weight, bias = _f32(weight), _f32(bias).reshape(-1)
    C, d = weight.shape
    if bias.numel() != C:
        raise ValueError('bias must hold one entry per weight row')
    rows = [int(r) for r in rows]
    if any(r < 0 or r >= C for r in rows):
        raise IndexError('rows %s lie outside the %d classifier rows' % (sorted(r for r in rows if r < 0 or r >= C), C))
    if out is None:
        out = torch.empty(2, dtype=torch.float32, device=weight.device)
    elif out.dtype != torch.float32 or out.numel() != 2 or not out.is_contiguous():
        raise ValueError('out must be a contiguous float32 tensor of 2')
    idx = torch.tensor(rows, dtype=torch.int64).to(weight.device) if rows else None
    rc = _native.lib().b200ocl_rows_mean(_ptr(weight), _ptr(bias), C, d, _ptr(idx), len(rows), _ptr(out), _stream())
    _native.check(rc, 'b200ocl_rows_mean')
    return out


def linear_fwd(x, weight, bias, relu=False):
    """x @ weight.T + bias (then ReLU when relu) with the network heads' kernel: y [N, out] for x [N, in], in <= 4096."""
    _need_cuda(x, weight, bias)
    x, weight, bias = _f32(x), _f32(weight), _f32(bias)
    N, d = x.shape
    y = torch.empty((N, weight.shape[0]), dtype=torch.float32, device=x.device)
    rc = _native.lib().b200ocl_linear_fwd(_ptr(x), _ptr(weight), _ptr(bias), _ptr(y), N, d, weight.shape[0],
                                          1 if relu else 0, _stream())
    _native.check(rc, 'b200ocl_linear_fwd')
    return y


def agem_project(g, g_ref, out=None, want_dots=False):
    """A-GEM projection of the flat gradient g against g_ref (agents/agem.py:60-80); out may alias either input."""
    _need_cuda(g, g_ref, out)
    g, g_ref = _f32(g).reshape(-1), _f32(g_ref).reshape(-1)
    if g.numel() != g_ref.numel():
        raise ValueError('g and g_ref must have the same length')
    if out is None:
        out = torch.empty_like(g)
    dots = torch.empty(2, dtype=torch.float32, device=g.device) if want_dots else None
    lib = _native.lib()
    ws = _workspace(lib.b200ocl_agem_project_workspace_bytes(), g.device)
    rc = lib.b200ocl_agem_project(_ptr(g), _ptr(g_ref), _ptr(out), g.numel(), _ptr(dots), _ptr(ws), ws.numel(), _stream())
    _native.check(rc, 'b200ocl_agem_project')
    return (out, dots) if want_dots else out


GRAD_COSINE_MAX_K = 64


def grad_cosine(mem_grads, g, max_out=None):
    """(cos [K], max [1]): cosine similarity of the flat gradient g with each stored gradient and their maximum
    (gss_greedy_update.py:84,120 with buffer_utils.py:50-55).  max_out: a one-element fp32 device tensor (view) to
    write the maximum into."""
    _need_cuda(mem_grads, g)
    mem_grads, g = _f32(mem_grads), _f32(g).reshape(-1)
    K, n = mem_grads.shape
    if g.numel() != n:
        raise ValueError('gradient length mismatch')
    cos = torch.empty(K, dtype=torch.float32, device=g.device)
    if max_out is None:
        max_out = torch.empty(1, dtype=torch.float32, device=g.device)
    elif max_out.numel() != 1 or max_out.dtype != torch.float32 or not max_out.is_cuda:
        raise ValueError('max_out must be a one-element fp32 CUDA tensor')
    lib = _native.lib()
    ws = _workspace(lib.b200ocl_grad_cosine_workspace_bytes(K), g.device)
    rc = lib.b200ocl_grad_cosine(_ptr(mem_grads), _ptr(g), K, n, _ptr(cos), _ptr(max_out), _ptr(ws), ws.numel(), _stream())
    _native.check(rc, 'b200ocl_grad_cosine')
    return cos, max_out


def scatter_rows(dst, idx, src):
    """dst[idx[i]] = src[i] over the first dimension (buffer_img[idx] = x)."""
    _need_cuda(dst, idx, src)
    if not dst.is_contiguous():
        raise ValueError('dst must be contiguous')
    idx = _i64(idx).reshape(-1)
    n = idx.numel()
    if n == 0:
        return dst
    src = src.detach().to(dst.dtype).contiguous()
    row_bytes = dst[0].numel() * dst.element_size()
    if src.numel() * src.element_size() != n * row_bytes:
        raise ValueError('src does not hold len(idx) rows of dst')
    rc = _native.lib().b200ocl_scatter_rows(_ptr(src), _ptr(idx), n, row_bytes, _ptr(dst), _stream())
    _native.check(rc, 'b200ocl_scatter_rows')
    return dst


def aser_replace(order, n_cand_buf, cand_slot, cur_x, cur_y, buffer_img, buffer_label):
    """ASER's memory replacement taken on the device (aser_update.py:88-112): moves the winning rows of
    the current batch into the losing candidates' slots and returns the decision as a device int64
    tensor [1 + 2*n_cur] = (count, positions in the current batch, buffer slots), -1 padded."""
    _need_cuda(order, cand_slot, cur_x, cur_y, buffer_img, buffer_label)
    order, cand_slot, cur_y = _i64(order).reshape(-1), _i64(cand_slot).reshape(-1), _i64(cur_y).reshape(-1)
    n_cur = cur_y.numel()
    if order.numel() != n_cand_buf + n_cur or cand_slot.numel() != n_cand_buf:
        raise ValueError('order must rank n_cand_buf + n_cur candidates')
    if not (cur_x.is_contiguous() and buffer_img.is_contiguous()) or cur_x.dtype != buffer_img.dtype:
        raise ValueError('cur_x / buffer_img must be contiguous and of one dtype')
    pairs = torch.empty(1 + 2 * n_cur, dtype=torch.int64, device=order.device)
    if n_cur == 0:
        return pairs.fill_(0)
    row_bytes = buffer_img[0].numel() * buffer_img.element_size()
    rc = _native.lib().b200ocl_aser_replace(_ptr(order), n_cand_buf + n_cur, n_cand_buf, _ptr(cand_slot), _ptr(cur_x),
                                            _ptr(cur_y), n_cur, row_bytes, _ptr(buffer_img), _ptr(buffer_label),
                                            _ptr(pairs), _stream())
    _native.check(rc, 'b200ocl_aser_replace')
    return pairs


def sgd_step(param, grad, lr, weight_decay=0.0, out=None):
    """out = param - lr*(grad + wd*param) over flat fp32 arenas; out defaults to param (in place)."""
    _need_cuda(param, grad, out)
    if out is None:
        out = param
    for t in (param, grad, out):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError('sgd_step needs contiguous fp32 tensors')
    if grad.numel() != param.numel() or out.numel() != param.numel():
        raise ValueError('size mismatch')
    rc = _native.lib().b200ocl_sgd_step(_ptr(param), _ptr(grad), _ptr(out), param.numel(), float(lr),
                                        float(weight_decay), _stream())
    _native.check(rc, 'b200ocl_sgd_step')
    return out


class AdamScalars(ctypes.Structure):
    """b200ocl_adam_scalars."""
    _fields_ = [(n, ctypes.c_float) for n in ('step_size', 'bc2_sqrt', 'bc2_sqrt_inv', 'eps', 'beta1_c', 'beta2',
                                              'beta2_c', 'weight_decay', 'grad_scale')]


ADAM_FOREACH, ADAM_GRAD_SCALE = 1, 2


def adam_scalars(lr, betas, eps, weight_decay, step, grad_div=None):
    """The scalars of Adam step number `step` (1-based), formed in double exactly as torch/optim/adam.py forms them
    for a float step counter (the foreach and single-tensor paths give the same doubles), then rounded to fp32 by
    ctypes as torch converts them to the kernels' op-math type.  A CUDA tensor divided by a Python float is multiplied
    by the reciprocal formed in double: bc2_sqrt_inv (foreach=False) and grad_scale = 1 / grad_div."""
    beta1, beta2 = float(betas[0]), float(betas[1])
    step = float(step)
    bias_correction1 = 1 - beta1 ** step
    bias_correction2 = 1 - beta2 ** step
    step_size = (float(lr) / bias_correction1) * -1
    bias_correction2_sqrt = bias_correction2 ** 0.5
    return AdamScalars(step_size, bias_correction2_sqrt, 1 / bias_correction2_sqrt, float(eps), 1 - beta1, beta2,
                       1 - beta2, float(weight_decay), 1 / float(grad_div) if grad_div is not None else 1.0)


def adam_step(param, grad, exp_avg, exp_avg_sq, step, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0,
              foreach=True, grad_div=None):
    """One torch.optim.Adam step (step = the state's step count after it, 1 for the first) over flat fp32 buffers, all
    updated in place; bit-identical to torch's multi-tensor path (foreach=True, its default on CUDA) or its
    single-tensor path (foreach=False).  grad_div: grad /= grad_div first (written back), as the review trick does."""
    _need_cuda(param, grad, exp_avg, exp_avg_sq)
    for t in (param, grad, exp_avg, exp_avg_sq):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError('adam_step needs contiguous fp32 tensors')
        if t.numel() != param.numel():
            raise ValueError('size mismatch')
    s = adam_scalars(lr, betas, eps, weight_decay, step, grad_div)
    flags = (ADAM_FOREACH if foreach else 0) | (ADAM_GRAD_SCALE if grad_div is not None else 0)
    rc = _native.lib().b200ocl_adam_step(_ptr(param), _ptr(grad), _ptr(exp_avg), _ptr(exp_avg_sq), param.numel(),
                                         ctypes.byref(s), flags, _stream())
    _native.check(rc, 'b200ocl_adam_step')
    return param


# --------------------------------------------------------------------------- task snapshots (checkpoint.py)
SNAP_COPY, SNAP_U8 = 0, 1           # B200OCL_SNAP_* (include/b200ocl.h)
SNAP_SEGMENT = np.dtype([('ptr', '<u8'), ('bytes', '<u8'), ('offset', '<u8'), ('kind', '<i4'), ('reserved', '<i4')])


def snapshot_workspace(n_segments, device):
    """Workspace of snapshot_pack / snapshot_unpack over n_segments segments: its first n_segments + 1 int32 are the
    counters (include/b200ocl.h)."""
    return _workspace(_native.lib().b200ocl_snapshot_workspace_bytes(int(n_segments)), device)


def _snapshot_call(name, table, n, staging, workspace):
    _need_cuda(table, staging, workspace)
    if table.dtype != torch.uint8 or table.numel() != n * SNAP_SEGMENT.itemsize:
        raise ValueError('the segment table must be %d uint8 records of %d bytes' % (n, SNAP_SEGMENT.itemsize))
    rc = getattr(_native.lib(), name)(_ptr(table), int(n), _ptr(staging), staging.numel() * staging.element_size(),
                                      _ptr(workspace), workspace.numel(), _stream())
    _native.check(rc, name)


def snapshot_pack(table, n, staging, workspace):
    """Copy (B200OCL_SNAP_COPY) or encode (B200OCL_SNAP_U8) the n segments of `table` (a device uint8 tensor of
    SNAP_SEGMENT records) into `staging`, on the current stream; workspace[:4 * (n + 1)] gets the counters.  Nothing
    is read back."""
    _snapshot_call('b200ocl_snapshot_pack', table, n, staging, workspace)


def snapshot_unpack(table, n, staging, workspace):
    """The inverse of snapshot_pack: each segment's region of `staging`, in the form its kind names, to its ptr."""
    _snapshot_call('b200ocl_snapshot_unpack', table, n, staging, workspace)
