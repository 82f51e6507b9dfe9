"""GPU: the wgmma weight gradient with tiles fitted to the channel counts (csrc/wgrad_tc.cu: 3 kernel columns x 20
input channels per warpgroup, the output block at its real width rounded up to 8, one K step in flight).

The rewrite keeps every tensor-core accumulation chain (tiles, K steps, hi / lo products) in its order and only moves
rows and trims padded columns, so it must reproduce the kernel it replaced bit for bit: tests/golden/wgrad_tc_parent.npz
holds what that kernel computed on seeded inputs (make_golden_wgrad_tc.py).  Shapes whose last channel slice or output
block is partial are checked against fp64 with the bars of test_gpu_wgrad_tc.py."""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import make_golden_wgrad_tc as mg  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'wgrad_tc_parent.npz')


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')


@pytest.mark.gpu
@pytest.mark.parametrize('shape', mg.SHAPES, ids=mg.key)
def test_wgrad_tc_bit_identical_to_recorded(shape):
    _need_cuda()
    rec = np.load(GOLDEN)
    dw = mg.run(shape)
    k = mg.key(shape)
    if k + '_dw' in rec:
        want = rec[k + '_dw']
        diff = np.flatnonzero(dw.view(np.uint32) != want.view(np.uint32))
        assert diff.size == 0, (k, diff.size, diff[:8])
    assert mg.sha(dw) == str(rec[k + '_sha256']), k


# (N, H, W, cin, cout): partial last slice (cin % 20 != 0) and / or partial last block (cout not a multiple of the
# block width), single-slice / single-block shapes below 20 channels, the widest strip
@pytest.mark.gpu
@pytest.mark.parametrize('N,H,W,cin,cout', [
    (3, 11, 11, 44, 52), (2, 9, 9, 4, 4), (5, 6, 6, 60, 124), (2, 37, 5, 28, 20), (4, 7, 7, 100, 84),
    (6, 5, 5, 24, 164), (1, 3, 3, 16, 8),
])
def test_wgrad_tc_partial_slices_and_blocks_match_fp64(N, H, W, cin, cout):
    _need_cuda()
    g = torch.Generator().manual_seed(N * 1000 + H * 10 + cin + 7 * cout)
    x = torch.relu(torch.randn(N, cin, H, W, generator=g))
    dz = torch.randn(N, cout, H, W, generator=g) / (N * H * W) ** 0.5
    w = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, requires_grad=True)
    F.conv2d(x.double(), w, padding=1).backward(dz.double())
    ref = w.grad
    got = torch.from_numpy(mg.run((N, H, W, cin, cout), x.permute(0, 2, 3, 1).contiguous(),
                                  dz.permute(0, 2, 3, 1).contiguous())).double()
    assert torch.isfinite(got).all()
    err = float((got - ref).abs().max() / ref.abs().max())
    rms = float(((got - ref) ** 2).mean().sqrt() / (ref ** 2).mean().sqrt())
    print('N=%d %dx%d %d->%d  max %.2e  rms %.2e' % (N, H, W, cin, cout, err, rms))
    assert err < 5e-6 and rms < 2e-6, (err, rms)


def test_golden_records_every_shape():
    rec = np.load(GOLDEN)
    for s in mg.SHAPES:
        sha = str(rec[mg.key(s) + '_sha256'])
        assert len(sha) == 64
        if s in mg.KEEP:
            dw = rec[mg.key(s) + '_dw']
            assert dw.shape == (s[4], s[3], 3, 3) and dw.dtype == np.float32
            assert hashlib.sha256(dw.astype('<f4').tobytes()).hexdigest() == sha
