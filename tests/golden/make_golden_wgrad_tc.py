"""Generate tests/golden/wgrad_tc_parent.npz (GPU box): what the wgmma weight-gradient kernel (csrc/wgrad_tc.cu)
computes on seeded inputs, recorded from the build the tile-fitting rewrite started from, so that the rewritten kernel
can be held to the same bits.

    python tests/golden/make_golden_wgrad_tc.py [REPO_ROOT [OUT.npz]]

REPO_ROOT (default: this checkout) is the built tree whose kernel is recorded.  For every shape of SHAPES the record
is the SHA-256 of the fp32 bytes of dW [cout, cin, 3, 3] as b200ocl_wgrad_tc_selftest returns it; the two smallest
shapes also keep dW itself, so that a mismatch shows where it lies.  No input is stored: every input is drawn from a
seed by inputs().
"""
import hashlib
import os
import sys

import numpy as np
import torch

# (N, H, W, cin, cout): the four CIFAR layer shapes of Reduced_ResNet18 at the stream and the replay batch size, an odd
# shape with a partial last channel slice and block, and the narrowest / widest strips the kernel takes
SHAPES = [
    (20, 32, 32, 20, 20), (20, 16, 16, 40, 40), (20, 8, 8, 80, 80), (20, 4, 4, 160, 160),
    (110, 32, 32, 20, 20), (110, 16, 16, 40, 40), (110, 8, 8, 80, 80), (110, 4, 4, 160, 160),
    (7, 11, 11, 36, 44), (2, 37, 5, 8, 12), (5, 9, 9, 44, 52),
]
KEEP = {(7, 11, 11, 36, 44), (2, 37, 5, 8, 12)}


def key(shape):
    return 'n%d_%dx%d_%d_%d' % shape


def inputs(shape):
    """Seeded NHWC activation (post-ReLU) and output gradient of one shape, on the CPU."""
    N, H, W, cin, cout = shape
    g = torch.Generator().manual_seed(7919 * N + 97 * H + 13 * W + 3 * cin + cout)
    x = torch.relu(torch.randn(N, H, W, cin, generator=g))
    dz = torch.randn(N, H, W, cout, generator=g) / (N * H * W) ** 0.5
    return x, dz


def run(shape, x=None, dz=None):
    """dW [cout, cin, 3, 3] of the wgmma kernel on the current device; NHWC x / dz default to inputs(shape)."""
    from b200ocl import _native
    from b200ocl.ops import _stream, _workspace
    lib = _native.lib()
    N, H, W, cin, cout = shape
    if x is None:
        x, dz = inputs(shape)
    x, dz = x.cuda(), dz.cuda()
    nbytes = lib.b200ocl_wgrad_tc_selftest_workspace_bytes(N, H, W, cin, cout)
    assert nbytes > 0
    ws = _workspace(nbytes, x.device)
    dw = torch.full((cout, cin, 3, 3), float('nan'), device=x.device)
    rc = lib.b200ocl_wgrad_tc_selftest(x.data_ptr(), dz.data_ptr(), dw.data_ptr(), N, H, W, cin, cout, ws.data_ptr(),
                                       ws.numel(), _stream())
    _native.check(rc, 'b200ocl_wgrad_tc_selftest')
    torch.cuda.synchronize()
    return dw.cpu().numpy()


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype='<f4').tobytes()).hexdigest()


def main():
    root = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else \
        os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    out = sys.argv[2] if len(sys.argv) > 2 else os.path.join(os.path.dirname(os.path.abspath(__file__)), 'wgrad_tc_parent.npz')
    sys.path.insert(0, root)
    rec = {}
    for s in SHAPES:
        dw = run(s)
        assert np.isfinite(dw).all(), s
        rec[key(s) + '_sha256'] = np.array(sha(dw))
        if s in KEEP:
            rec[key(s) + '_dw'] = dw
        print(key(s), sha(dw))
    np.savez_compressed(out, **rec)
    print('wrote', out)


if __name__ == '__main__':
    main()
