"""Generate tests/golden/conv_tcp_parent.npz (GPU box): what the halo-strip convolution (csrc/conv_tcp.cu) computes on
seeded inputs at the launches of the benchmark's step, recorded from the build that added the kernel's timeline
(B200OCL_TCP_TRACE), so that later changes of its schedule can be held to the same bits.

    python tests/golden/make_golden_conv_tcp.py [REPO_ROOT [OUT.npz]]

REPO_ROOT (default: this checkout) is the built tree whose kernel is recorded.  For every case of CASES the record is
the SHA-256 of the fp32 NHWC output as b200ocl_conv_selftest writes it; the cases of KEEP also keep the output itself,
so that a mismatch shows where it lies.  No input is stored: every input is drawn from a seed by inputs().
"""
import hashlib
import os
import sys

import numpy as np
import torch

LAYERS = [(20, 32), (40, 16), (80, 8), (160, 4)]   # (channels, map) of the network's 3x3 stride-1 convolutions
# (kind, N, C, H): eval forward at the ASER batch (folded BN + residual + ReLU), data gradient at SCR's and ASER's
# backward batches, raw and accumulating into a seeded tensor
CASES = ([('eval', 210, C, H) for C, H in LAYERS] +
         [(kind, N, C, H) for N in (110, 20) for kind in ('dgrad', 'dgrad_acc') for C, H in LAYERS])
KEEP = {('dgrad_acc', 20, 160, 4)}
TC_PATCH = 3


def key(case):
    return '%s_n%d_c%d_%dx%d' % (case[0], case[1], case[2], case[3], case[3])


def inputs(case):
    """Seeded NHWC input, OIHW weights, eval BN statistics (mean, var, gamma, beta) and starting output, on the CPU."""
    kind, N, C, H = case
    g = torch.Generator().manual_seed(7907 * N + 131 * C + 7 * H + len(kind))
    w = torch.randn(C, C, 3, 3, generator=g) / np.sqrt(9 * C)
    x = torch.randn(N, H, H, C, generator=g)
    if kind == 'eval':
        x = torch.relu(x)
    stats = torch.cat([0.1 * torch.randn(C, generator=g), 0.5 + torch.rand(C, generator=g),
                       1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)])
    out = torch.randn(N, H, H, C, generator=g) if kind == 'dgrad_acc' else torch.full((N, H, H, C), float('nan'))
    return x, w, stats, out


def run(case):
    """The NHWC output of the strip kernel for one case on the current device."""
    from b200ocl import _native
    from b200ocl.ops import _stream
    lib = _native.lib()
    kind, N, C, H = case
    x, w, stats, out = (t.cuda() for t in inputs(case))
    dgrad = int(kind != 'eval')
    mode = {'eval': 4, 'dgrad': 0, 'dgrad_acc': 1}[kind]
    nbytes = lib.b200ocl_conv_selftest_workspace_bytes(N, C, C, H, H, 3, 1)
    ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
    ws.view(torch.float32).fill_(float('nan'))
    rc = lib.b200ocl_conv_selftest(x.data_ptr(), w.data_ptr(), out.data_ptr(), N, H, H, C, C, 3, 1, dgrad, TC_PATCH,
                                   mode, stats.data_ptr() if mode == 4 else None, ws.data_ptr(), nbytes, _stream())
    _native.check(rc, 'b200ocl_conv_selftest')
    torch.cuda.synchronize()
    return out.cpu().numpy()


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype='<f4').tobytes()).hexdigest()


def main():
    root = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else \
        os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    out = sys.argv[2] if len(sys.argv) > 2 else os.path.join(os.path.dirname(os.path.abspath(__file__)), 'conv_tcp_parent.npz')
    sys.path.insert(0, root)
    rec = {}
    for c in CASES:
        y = run(c)
        assert np.isfinite(y).all(), c
        rec[key(c) + '_sha256'] = np.array(sha(y))
        if c in KEEP:
            rec[key(c) + '_out'] = y
        print(key(c), sha(y))
    np.savez_compressed(out, **rec)
    print('wrote', out)


if __name__ == '__main__':
    main()
