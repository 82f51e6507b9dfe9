"""GPU: every 3x3 convolution kernel family against an fp64 reference convolution, one layer at a time
(b200ocl_conv_selftest forces the path): CUDA-core kernels, wgmma with im2col tiles (conv_tc.cu), wgmma
fed from a halo patch (conv_tcp.cu); forward and data gradient, raw and accumulate.  Train-mode statistics,
stride 2 and 1x1 run on the kernels that cover them; the halo-patch kernel refuses those launches."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

PATHS = {'cuda_core': 1, 'tc_im2col': 2, 'tc_patch': 3}
EUNSUPPORTED = 2   # B200OCL_EUNSUPPORTED (include/b200ocl.h)


def run_conv(x_nhwc, w, dgrad, path, accumulate=None, train=False, stride=1, expect_rc=0):
    from b200ocl import _native
    from b200ocl.ops import _stream
    lib = _native.lib()
    N, H, W, _ = x_nhwc.shape
    cout, cin, ks = w.shape[0], w.shape[1], w.shape[2]
    pad = 1 if ks == 3 else 0
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    out = torch.zeros(N, Ho, Wo, cin if dgrad else cout, device='cuda') if accumulate is None else accumulate.clone()
    stats = torch.full((4 * cout,), float('nan'), device='cuda')
    nbytes = lib.b200ocl_conv_selftest_workspace_bytes(N, cin, cout, H, W, ks, stride)
    ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
    ws.view(torch.float32).fill_(float('nan'))        # nothing may be read before it is written
    mode = 2 if train else (0 if accumulate is None else 1)
    rc = lib.b200ocl_conv_selftest(x_nhwc.data_ptr(), w.data_ptr(), out.data_ptr(), N, H, W, cin, cout, ks, stride, int(dgrad),
                                   path, mode, stats.data_ptr() if train else None, ws.data_ptr(), nbytes, _stream())
    if expect_rc:
        assert rc == expect_rc, rc
        return None
    _native.check(rc, 'b200ocl_conv_selftest')
    torch.cuda.synchronize()
    return (out, stats) if train else out


def reference(x_nhwc, w, dgrad, stride=1):
    x = x_nhwc.permute(0, 3, 1, 2).double()
    pad = 1 if w.shape[2] == 3 else 0
    if dgrad:
        y = torch.nn.functional.conv_transpose2d(x, w.double(), padding=pad)
    else:
        y = torch.nn.functional.conv2d(x, w.double(), padding=pad, stride=stride)
    return y.permute(0, 2, 3, 1).contiguous()


SHAPES = [  # N, H, W, cin, cout
    (10, 32, 32, 20, 20), (110, 32, 32, 20, 20), (7, 16, 16, 40, 40), (110, 16, 16, 40, 40),
    (10, 8, 8, 80, 80), (7, 8, 8, 80, 80), (110, 8, 8, 80, 80), (3, 16, 16, 20, 40), (5, 8, 8, 40, 80),
    (1, 8, 8, 80, 80), (2, 32, 32, 20, 20), (64, 16, 16, 160, 160), (8, 8, 8, 80, 80), (8, 16, 16, 40, 40), (8, 32, 32, 20, 20),
    (10, 4, 4, 160, 160), (110, 4, 4, 160, 160), (7, 4, 4, 160, 160), (5, 21, 21, 40, 40), (3, 11, 11, 80, 80), (2, 6, 6, 160, 160),
]


@pytest.mark.parametrize('path', sorted(PATHS))
@pytest.mark.parametrize('dgrad', [0, 1])
@pytest.mark.parametrize('shape', SHAPES)
def test_conv3x3_matches_fp64(shape, dgrad, path):
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    N, H, W, cin, cout = shape
    g = torch.Generator(device='cuda').manual_seed(N * 1000 + H + cin + dgrad)
    w = torch.randn(cout, cin, 3, 3, device='cuda', generator=g) / np.sqrt(9 * cin)
    x = torch.randn(N, H, W, cout if dgrad else cin, device='cuda', generator=g)
    if not dgrad:
        x = torch.relu(x)
    ref = reference(x, w, dgrad)
    got = run_conv(x, w, dgrad, PATHS[path])
    err = float((got.double() - ref).abs().max() / ref.abs().max())
    assert err < 5e-6, err
    # accumulate mode adds onto an existing tensor
    base = torch.randn(got.shape, device='cuda', generator=g)
    got2 = run_conv(x, w, dgrad, PATHS[path], accumulate=base)
    err2 = float((got2.double() - (ref + base.double())).abs().max() / ref.abs().max())
    assert err2 < 5e-6, err2


@pytest.mark.parametrize('path', ['cuda_core', 'tc_im2col'])
@pytest.mark.parametrize('shape', SHAPES)
def test_conv3x3_train_statistics(shape, path):
    """Train-mode epilogue: raw output + batch mean / invstd / running statistics (fp64 sums in the kernels)."""
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    N, H, W, cin, cout = shape
    g = torch.Generator(device='cuda').manual_seed(N * 77 + H + cin)
    w = torch.randn(cout, cin, 3, 3, device='cuda', generator=g) / np.sqrt(9 * cin)
    x = torch.relu(torch.randn(N, H, W, cin, device='cuda', generator=g))
    ref = reference(x, w, 0)
    got, stats = run_conv(x, w, 0, PATHS[path], train=True)
    assert float((got.double() - ref).abs().max() / ref.abs().max()) < 5e-6
    z = ref.reshape(-1, cout)
    mean, var = z.mean(0), z.var(0, unbiased=False)
    st = stats.double().reshape(4, cout)
    scale = float(z.abs().max())
    assert float((st[0] - mean).abs().max()) < 2e-6 * scale
    assert float((st[1] - 1.0 / torch.sqrt(var + 1e-5)).abs().max() / (1.0 / torch.sqrt(var + 1e-5)).abs().max()) < 1e-5
    assert float((st[2] - 0.1 * mean).abs().max()) < 2e-6 * scale
    n = z.shape[0]
    unb = var * n / max(n - 1, 1)
    assert float((st[3] - 0.1 * unb).abs().max() / (0.1 * unb).abs().max()) < 1e-5


STRIDED = [  # N, H, W, cin, cout, ks, stride  (the network's down-sampling convolutions and shortcuts)
    (110, 32, 32, 20, 40, 3, 2), (10, 32, 32, 20, 40, 3, 2), (210, 16, 16, 40, 80, 3, 2), (7, 16, 16, 40, 80, 3, 2),
    (110, 8, 8, 80, 160, 3, 2), (10, 8, 8, 80, 160, 3, 2), (110, 32, 32, 20, 40, 1, 2), (10, 16, 16, 40, 80, 1, 2),
    (210, 8, 8, 80, 160, 1, 2), (5, 22, 22, 40, 40, 3, 2), (3, 8, 8, 80, 80, 1, 1),
]


@pytest.mark.parametrize('path', ['cuda_core'])
@pytest.mark.parametrize('shape', STRIDED)
def test_strided_and_pointwise_convolutions(shape, path):
    """3x3 stride-2 and 1x1 convolutions: raw output and train-mode statistics against fp64."""
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    N, H, W, cin, cout, ks, stride = shape
    g = torch.Generator(device='cuda').manual_seed(N * 31 + H + cin + ks)
    w = torch.randn(cout, cin, ks, ks, device='cuda', generator=g) / np.sqrt(ks * ks * cin)
    x = torch.relu(torch.randn(N, H, W, cin, device='cuda', generator=g))
    ref = reference(x, w, 0, stride)
    got = run_conv(x, w, 0, PATHS[path], stride=stride)
    assert got.shape == ref.shape
    assert float((got.double() - ref).abs().max() / ref.abs().max()) < 5e-6
    got2, stats = run_conv(x, w, 0, PATHS[path], train=True, stride=stride)
    assert float((got2.double() - ref).abs().max() / ref.abs().max()) < 5e-6
    z = ref.reshape(-1, cout)
    mean, var = z.mean(0), z.var(0, unbiased=False)
    st = stats.double().reshape(4, cout)
    assert float((st[0] - mean).abs().max()) < 2e-6 * float(z.abs().max())
    assert float((st[1] - 1.0 / torch.sqrt(var + 1e-5)).abs().max() / (1.0 / torch.sqrt(var + 1e-5)).abs().max()) < 1e-5


# The halo-patch kernel (path 3) covers 3x3 stride-1 eval / raw / accumulate launches only; every shape the two tests
# above run is refused with B200OCL_EUNSUPPORTED instead of launching.  Train mode on a 3x3 stride-1 layer reaches the
# mode check of conv_tcp_eligible; stride-2 and 1x1 layers get no strip weight image from the network plan, so they
# are refused for the missing image before the geometry checks.

@pytest.mark.parametrize('shape', SHAPES)
def test_tc_patch_refuses_train_mode(shape):
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    N, H, W, cin, cout = shape
    w = torch.randn(cout, cin, 3, 3, device='cuda')
    x = torch.relu(torch.randn(N, H, W, cin, device='cuda'))
    run_conv(x, w, 0, PATHS['tc_patch'], train=True, expect_rc=EUNSUPPORTED)


@pytest.mark.parametrize('shape', STRIDED)
def test_tc_patch_refuses_strided_and_pointwise(shape):
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    N, H, W, cin, cout, ks, stride = shape
    w = torch.randn(cout, cin, ks, ks, device='cuda')
    x = torch.relu(torch.randn(N, H, W, cin, device='cuda'))
    run_conv(x, w, 0, PATHS['tc_patch'], stride=stride, expect_rc=EUNSUPPORTED)
    run_conv(x, w, 0, PATHS['tc_patch'], train=True, stride=stride, expect_rc=EUNSUPPORTED)
