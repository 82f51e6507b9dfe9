"""GPU: the halo-strip convolution (conv_tcp.cu) at every strip shape the network runs, forced onto that kernel, in
eval (folded BatchNorm, with and without residual and ReLU), raw and accumulate modes, forward and data gradient,
against fp64.  The strip shares a one-position zero halo between neighbouring columns, rows and images, so the batch
sizes include ones whose last 128-row tile ends inside an image and ones whose tiles run into the zero tail past the
last image."""
import numpy as np
import pytest
import torch

from test_gpu_conv import reference, run_conv

pytestmark = pytest.mark.gpu

TC_PATCH = 3
# (channels, map): the 3x3 stride-1 layers of the reduced ResNet-18 whose maps the strip holds
LAYERS = [(20, 32), (40, 16), (80, 8), (160, 4)]
BATCHES = [1, 2, 20, 110, 210]


def strip_tiles(N, H, W):
    """Tiles of 128 strip positions and where the last one ends inside its image (0 = on an image boundary)."""
    pitch = (H + 1) * (W + 1)
    last = (N - 1) * pitch + (H - 1) * (W + 1) + (W - 1)
    tiles = last // 128 + 1
    return tiles, (tiles * 128) % pitch


def test_batches_cover_tiles_ending_inside_an_image():
    ends = [strip_tiles(N, H, H)[1] for _, H in LAYERS for N in BATCHES]
    assert any(e != 0 for e in ends)


def run_eval(x, w, bn, residual_relu):
    """Eval-mode forward through the strip kernel: folded BatchNorm, optionally + x as the residual and ReLU."""
    from b200ocl import _native
    from b200ocl.ops import _stream
    lib = _native.lib()
    N, H, W, cin = x.shape
    cout = w.shape[0]
    out = torch.full((N, H, W, cout), float('nan'), device='cuda')
    nbytes = lib.b200ocl_conv_selftest_workspace_bytes(N, cin, cout, H, W, 3, 1)
    ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
    ws.view(torch.float32).fill_(float('nan'))
    rc = lib.b200ocl_conv_selftest(x.data_ptr(), w.data_ptr(), out.data_ptr(), N, H, W, cin, cout, 3, 1, 0, TC_PATCH,
                                   4 if residual_relu else 3, bn.data_ptr(), ws.data_ptr(), nbytes, _stream())
    _native.check(rc, 'b200ocl_conv_selftest')
    torch.cuda.synchronize()
    return out


def rel_err(got, ref):
    assert not torch.isnan(got).any()
    return float((got.double() - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize('N', BATCHES)
@pytest.mark.parametrize('C,H', LAYERS)
def test_strip_conv_data_gradient(C, H, N):
    g = torch.Generator(device='cuda').manual_seed(C * 1000 + N)
    w = torch.randn(C, C, 3, 3, device='cuda', generator=g) / np.sqrt(9 * C)
    dz = torch.randn(N, H, H, C, device='cuda', generator=g)
    ref = reference(dz, w, 1)
    got = run_conv(dz, w, 1, TC_PATCH)
    assert rel_err(got, ref) < 5e-6
    assert torch.equal(run_conv(dz, w, 1, TC_PATCH), got)          # repeat launches give the same bits
    base = torch.randn(got.shape, device='cuda', generator=g)
    got2 = run_conv(dz, w, 1, TC_PATCH, accumulate=base)
    assert float((got2.double() - (ref + base.double())).abs().max() / ref.abs().max()) < 5e-6


@pytest.mark.parametrize('N', BATCHES)
@pytest.mark.parametrize('C,H', LAYERS)
def test_strip_conv_forward(C, H, N):
    g = torch.Generator(device='cuda').manual_seed(C * 7 + N)
    w = torch.randn(C, C, 3, 3, device='cuda', generator=g) / np.sqrt(9 * C)
    x = torch.relu(torch.randn(N, H, H, C, device='cuda', generator=g))
    conv = reference(x, w, 0)
    got = run_conv(x, w, 0, TC_PATCH)
    assert rel_err(got, conv) < 5e-6
    assert torch.equal(run_conv(x, w, 0, TC_PATCH), got)
    base = torch.randn(got.shape, device='cuda', generator=g)
    got2 = run_conv(x, w, 0, TC_PATCH, accumulate=base)
    assert float((got2.double() - (conv + base.double())).abs().max() / conv.abs().max()) < 5e-6
    # eval: (conv - mean) * gamma / sqrt(var + eps) + beta, then (+ x, ReLU)
    mean = 0.1 * torch.randn(C, device='cuda', generator=g)
    var = 0.5 + torch.rand(C, device='cuda', generator=g)
    gamma = 1.0 + 0.1 * torch.randn(C, device='cuda', generator=g)
    beta = 0.1 * torch.randn(C, device='cuda', generator=g)
    bn = torch.cat([mean, var, gamma, beta]).contiguous()
    scale = gamma.double() / torch.sqrt(var.double() + 1e-5)
    y = (conv - mean.double()) * scale + beta.double()
    got3 = run_eval(x, w, bn, False)
    assert rel_err(got3, y) < 5e-6
    got4 = run_eval(x, w, bn, True)
    assert rel_err(got4, torch.relu(y + x.double())) < 5e-6
    assert torch.equal(run_eval(x, w, bn, True), got4)
