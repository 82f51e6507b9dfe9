"""Generate tests/golden/conv_maps.npz (GPU box): what the halo-strip convolution (csrc/conv_tcp.cu) and the wgmma
weight gradient (csrc/wgrad_tc.cu) compute on seeded inputs at the strip-kernel layers of the Mini-ImageNet, OpenLORIS and
CORe50 networks -- the maps CIFAR's network does not have -- so that a later change of either kernel's schedule can be
held to the same bits there (tests/test_gpu_conv_maps_fp64.py).  conv_tcp_parent.npz and wgrad_tc_parent.npz hold
CIFAR's maps.

    python tests/golden/make_golden_conv_maps.py [REPO_ROOT [OUT.npz]]

REPO_ROOT (default: this checkout) is the built tree whose kernels are recorded.  Every case is one launch at N = 20 or
110 images: the eval forward with folded BN, a residual that is not the input, and ReLU (b200ocl_conv_selftest_eval);
the data gradient, raw and accumulating into a seeded tensor (b200ocl_conv_selftest); and the weight gradient
(b200ocl_wgrad_tc_selftest).  The record is the SHA-256 of the fp32 output (NHWC, dW in OIHW); the case of KEEP also
keeps the output itself, so that a mismatch of the eval epilogue shows where it lies.  No input is stored: inputs()
draws every input from a seed.
"""
import hashlib
import os
import sys

import numpy as np
import torch

# (channels, map) of the 3x3 stride-1 layers the strip kernels take at 84x84, 50x50 and 128x128 inputs
PAIRS = [(80, 21), (160, 11), (40, 25), (80, 13), (160, 7), (80, 32), (160, 16)]
KINDS = ('eval', 'dgrad', 'dgrad_acc', 'wgrad')
CASES = [(kind, N, C, H) for N in (20, 110) for C, H in PAIRS for kind in KINDS]
KEEP = {('eval', 20, 160, 7)}
TC_PATCH = 3


def key(case):
    return '%s_n%d_c%d_%dx%d' % (case[0], case[1], case[2], case[3], case[3])


def inputs(case):
    """Seeded CPU tensors: conv cases give (x NHWC, w OIHW, bn = [mean | var | gamma | beta], residual, starting
    output); the weight gradient gives (x NHWC, dz NHWC)."""
    kind, N, C, H = case
    g = torch.Generator().manual_seed(7919 * N + 131 * C + 7 * H + len(kind))
    if kind == 'wgrad':
        x = torch.relu(torch.randn(N, H, H, C, generator=g))
        return x, torch.randn(N, H, H, C, generator=g) / (N * H * H) ** 0.5
    w = torch.randn(C, C, 3, 3, generator=g) / np.sqrt(9 * C)
    x = torch.randn(N, H, H, C, generator=g)
    if kind == 'eval':
        x = torch.relu(x)
    bn = torch.cat([0.5 * torch.randn(C, generator=g), 10 ** (4 * torch.rand(C, generator=g) - 3),
                    torch.randn(C, generator=g), 0.5 * torch.randn(C, generator=g)])
    residual = torch.randn(N, H, H, C, generator=g)
    out = torch.randn(N, H, H, C, generator=g) if kind == 'dgrad_acc' else torch.full((N, H, H, C), float('nan'))
    return x, w, bn, residual, out


def run(case):
    """The kernel's output for one case on the current device, as a numpy array."""
    from b200ocl import _native
    from b200ocl.ops import _stream
    lib = _native.lib()
    kind, N, C, H = case
    if kind == 'wgrad':
        x, dz = (t.cuda() for t in inputs(case))
        nbytes = lib.b200ocl_wgrad_tc_selftest_workspace_bytes(N, H, H, C, C)
        ws = torch.full((nbytes // 4,), float('nan'), device='cuda')
        dw = torch.full((C, C, 3, 3), float('nan'), device='cuda')
        rc = lib.b200ocl_wgrad_tc_selftest(x.data_ptr(), dz.data_ptr(), dw.data_ptr(), N, H, H, C, C, ws.data_ptr(),
                                           nbytes, _stream())
        _native.check(rc, 'b200ocl_wgrad_tc_selftest')
        torch.cuda.synchronize()
        return dw.cpu().numpy()
    x, w, bn, residual, out = (t.cuda() for t in inputs(case))
    nbytes = lib.b200ocl_conv_selftest_workspace_bytes(N, C, C, H, H, 3, 1)
    ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
    ws.view(torch.float32).fill_(float('nan'))
    if kind == 'eval':
        rc = lib.b200ocl_conv_selftest_eval(x.data_ptr(), w.data_ptr(), bn.data_ptr(), residual.data_ptr(), 1,
                                            out.data_ptr(), N, H, H, C, TC_PATCH, ws.data_ptr(), nbytes, _stream())
        _native.check(rc, 'b200ocl_conv_selftest_eval')
    else:
        rc = lib.b200ocl_conv_selftest(x.data_ptr(), w.data_ptr(), out.data_ptr(), N, H, H, C, C, 3, 1, 1, TC_PATCH,
                                       int(kind == 'dgrad_acc'), None, ws.data_ptr(), nbytes, _stream())
        _native.check(rc, 'b200ocl_conv_selftest')
    torch.cuda.synchronize()
    return out.cpu().numpy()


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype='<f4').tobytes()).hexdigest()


def main():
    root = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else \
        os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    out = sys.argv[2] if len(sys.argv) > 2 else \
        os.path.join(os.path.dirname(os.path.abspath(__file__)), 'conv_maps.npz')
    sys.path.insert(0, root)
    rec = {}
    for c in CASES:
        y = run(c)
        assert np.isfinite(y).all(), c
        assert sha(run(c)) == sha(y), c       # a record of bits that move between launches would be useless
        rec[key(c) + '_sha256'] = np.array(sha(y))
        if c in KEEP:
            rec[key(c) + '_out'] = y
        print(key(c), sha(y))
    np.savez_compressed(out, **rec)
    print('wrote', out)


if __name__ == '__main__':
    main()
