"""GPU: the schedule of the halo-strip convolution (conv_tcp.cu) -- two taps in flight per consumer warpgroup, and the
epilogue warpgroup reading finished tiles from two shared-memory buffers -- at the launches that exercise it: CTAs that
walk one, two and three or more tiles (so both buffers are reused), the one-slice launch with all nine weight blocks
resident and the five-slice launch that streams them through the ring, and both patch-stage depths the launcher fits.
Eval with residual and ReLU (NaN-filled output) and the accumulating data gradient, each against fp64 with the bars of
test_gpu_conv_strip.py and repeated for identical bits."""
import numpy as np
import pytest
import torch

from test_gpu_conv import reference, run_conv
from test_gpu_conv_strip import TC_PATCH, rel_err, run_eval, strip_tiles

pytestmark = pytest.mark.gpu

# (channels, map): 20 @ 32x32 is one slice with resident weights; 40 @ 16x16 two slices through the ring; 160 @ 4x4
# five slices through the ring.  The first two fit 2 patch stages, the last 3.
LAYERS = [(20, 32), (40, 16), (160, 4)]
ROUNDS = [1, 2, 3]   # tiles per CTA; 3 stands for three or more


def slices(C):
    return (C + 31) // 32


def geom(N, C, H, dgrad, mode):
    from b200ocl import engine
    g = engine.conv_selftest_geom(N, H, H, C, C, 3, 1, dgrad, TC_PATCH, mode)
    assert g.kernel == 1   # conv_tcp
    return g


@pytest.mark.parametrize('dgrad,mode', [(0, 4), (1, 1)])
def test_layers_cover_both_stage_depths_and_weight_modes(dgrad, mode):
    """The depths are the ones the launcher fits (reported by the geometry hook), at the batches the tests run."""
    depths = {geom(batch_for(C, H, r, dgrad, mode), C, H, dgrad, mode).tp_ps for C, H in LAYERS for r in ROUNDS}
    assert depths == {2, 3}
    assert {slices(C) for C, _ in LAYERS} >= {1, 5}


def rounds(N, C, H, dgrad, mode):
    tiles = strip_tiles(N, H, H)[0]
    grid_x = geom(N, C, H, dgrad, mode).grid_x
    return (tiles + grid_x - 1) // grid_x


def batch_for(C, H, r, dgrad, mode):
    """The smallest batch whose CTAs walk r tiles (r = 3: three or more) on the card in use."""
    for N in range(1, 2000):
        k = rounds(N, C, H, dgrad, mode)
        if k == r or (r == 3 and k >= 3):
            return N
    raise AssertionError('no batch reaches %d rounds' % r)


@pytest.mark.parametrize('r', ROUNDS)
@pytest.mark.parametrize('C,H', LAYERS)
def test_pipeline_eval_residual(C, H, r):
    N = batch_for(C, H, r, 0, 4)
    g = torch.Generator(device='cuda').manual_seed(C * 31 + r)
    w = torch.randn(C, C, 3, 3, device='cuda', generator=g) / np.sqrt(9 * C)
    x = torch.relu(torch.randn(N, H, H, C, device='cuda', generator=g))
    mean = 0.1 * torch.randn(C, device='cuda', generator=g)
    var = 0.5 + torch.rand(C, device='cuda', generator=g)
    gamma = 1.0 + 0.1 * torch.randn(C, device='cuda', generator=g)
    beta = 0.1 * torch.randn(C, device='cuda', generator=g)
    bn = torch.cat([mean, var, gamma, beta]).contiguous()
    scale = gamma.double() / torch.sqrt(var.double() + 1e-5)
    y = (reference(x, w, 0) - mean.double()) * scale + beta.double()
    got = run_eval(x, w, bn, True)              # the output starts NaN-filled: rel_err checks none is left
    assert rel_err(got, torch.relu(y + x.double())) < 5e-6
    assert torch.equal(run_eval(x, w, bn, True), got)


@pytest.mark.parametrize('r', ROUNDS)
@pytest.mark.parametrize('C,H', LAYERS)
def test_pipeline_data_gradient_accumulate(C, H, r):
    N = batch_for(C, H, r, 1, 1)
    g = torch.Generator(device='cuda').manual_seed(C * 37 + r)
    w = torch.randn(C, C, 3, 3, device='cuda', generator=g) / np.sqrt(9 * C)
    dz = torch.randn(N, H, H, C, device='cuda', generator=g)
    ref = reference(dz, w, 1)
    base = torch.randn(ref.shape, device='cuda', generator=g)
    got = run_conv(dz, w, 1, TC_PATCH, accumulate=base)
    assert not torch.isnan(got).any()
    assert float((got.double() - (ref + base.double())).abs().max() / ref.abs().max()) < 5e-6
    assert torch.equal(run_conv(dz, w, 1, TC_PATCH, accumulate=base), got)
