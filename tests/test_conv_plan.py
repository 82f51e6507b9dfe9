"""CPU: b200ocl_net_conv_geom and b200ocl_conv_selftest_geom, the host-only hooks that report which convolution kernel
(and template instantiation, and grid) a launch runs.  The launch planner's thresholds move with the SM count, so the
sweep below runs it for the SM counts of the H100 PCIe (114), H100 SXM (132) and a 148-SM part, over every layer of
the three networks the replay step runs and every batch size up to 512 (no GPU needed: nothing is launched)."""
import pytest

from oracle import resnet as oresnet

SMS = (114, 132, 148)
NETS = [(32, None), (32, 'mlp'), (84, None)]      # CIFAR classifier, SCR's SupCon mlp head, Mini-ImageNet classifier
N_MAX = 512


def layer_shapes(spec):
    """[(ks, stride)] per conv layer in BatchNorm2d module order."""
    out = [(3, 1)]
    for _, cin, cout, stride, sc in oresnet.block_plan(spec):
        out += [(3, stride), (3, 1)] + ([(1, stride)] if sc else [])
    return out


@pytest.mark.parametrize('sms', SMS)
@pytest.mark.parametrize('hw,head', NETS)
def test_every_launch_fits_its_workspace(hw, head, sms):
    """Train-mode partials fit the statistics region; the halo-strip kernel (which has no statistics epilogue) never
    takes a train-mode launch; only layer 0 is the stem; the im2col wgmma kernel only takes 3x3 stride-1 layers."""
    from b200ocl import engine
    spec = oresnet.Spec(hw, 20, 100, head=head)
    desc, info, _ = engine.describe(hw, 100, head)
    shapes = layer_shapes(spec)
    assert len(shapes) == info.n_bn
    for N in range(1, N_MAX + 1):
        region = None
        for layer, (ks, stride) in enumerate(shapes):
            for pass_ in ('train', 'eval', 'dgrad'):
                if pass_ == 'dgrad' and layer == 0:
                    continue
                g = engine.conv_geom(desc, N, layer, pass_, sms)
                where = (N, layer, pass_, g.template, g.grid_x, g.grid_y)
                assert g.sms == sms and g.kernel >= 0, where
                assert (g.kernel == 0) == (layer == 0), where
                if g.name == 'tc':
                    assert ks == 3 and stride == 1, where
                if pass_ == 'train':
                    assert g.name != 'tcp', where
                    assert 0 < g.stat_bytes <= g.stat_region, where
                    region = region or g.stat_region
                    assert g.stat_region == region, where      # one region per workspace
                else:
                    assert g.stat_bytes == 0, where


@pytest.mark.parametrize('sms', SMS)
def test_reported_grids_follow_the_tilings(sms):
    """The grid the hook reports is the one each kernel family's tiling gives (so stat_bytes is what the launch
    writes): 128-pixel tiles for the stem and the im2col kernel, BM = (80 / bn) * 32 * pt pixels for the tiled kernel,
    32 * pt for the k-split kernel, and the patch kernel's spatial tiles."""
    from b200ocl import engine
    for hw, head in NETS:
        spec = oresnet.Spec(hw, 20, 100, head=head)
        desc, _, _ = engine.describe(hw, 100, head)
        for N in (1, 2, 10, 20, 22, 110, 160, 210, 260, 512):
            for layer in range(len(layer_shapes(spec))):
                L = engine.train_ws_layout(desc, N, layer)
                g = engine.conv_geom(desc, N, layer, 'train', sms)
                M, C = N * L.hout * L.wout, L.cout
                bm = {'stem': 128, 'tc': 128, 'tiled': (80 // max(g.bn, 1)) * 32 * g.pt, 'ksplit': 32 * g.pt}.get(g.name)
                if bm is not None:
                    assert g.grid_x == (M + bm - 1) // bm, (hw, N, layer, g.template)
                else:
                    assert g.name == 'patch'
                    assert g.th * g.tw * g.ti == (80 // g.bn) * 32 * g.pt
                    tiles = -(-N // g.ti) * -(-L.hout // g.th) * -(-L.wout // g.tw)
                    assert g.grid_x == tiles, (hw, N, layer, g.template)
                assert g.stat_bytes == g.grid_x * C * 16


def test_patch_tiles_can_exceed_one_cta_per_32_pixels():
    """The sizing bound the statistics region used to have, one CTA per 32 output pixels, does not hold for the patch
    kernel on maps that are not a power of two wide: Mini-ImageNet layer3.0.conv1 (42 -> 21, 40 -> 80 channels) at
    N = 20 on 132 SMs runs patch<80, 1> with 16 x 2 tiles, 22 per 441-pixel image."""
    from b200ocl import engine
    desc, _, _ = engine.describe(84, 100, None)
    layer = 10                                    # stem, layer1 (4), layer2 (5): layer3.0.conv1 is the 11th
    L = engine.train_ws_layout(desc, 20, layer)
    assert (L.cin, L.cout, L.stride, L.hout) == (40, 80, 2, 21)
    g = engine.conv_geom(desc, 20, layer, 'train', 132)
    assert g.template == ('patch', 80, 1) and (g.th, g.tw, g.ti) == (2, 16, 1)
    assert g.grid_x == 22 * 20 > (20 * 21 * 21 + 31) // 32
    assert g.stat_bytes <= g.stat_region


@pytest.mark.parametrize('sms', SMS)
def test_selftest_workspace_covers_its_launch(sms):
    """b200ocl_conv_selftest's workspace keeps room for the partials of the launch it makes.  On 132 SMs a train-mode
    21x21 80 -> 80 convolution of 16 images on the CUDA-core path runs patch<80, 1> on 352 CTAs."""
    from b200ocl import engine
    g = engine.conv_selftest_geom(16, 21, 21, 80, 80, 3, 1, 0, 1, 2, 132)
    assert g.template == ('patch', 80, 1) and g.grid_x * g.grid_y == 352
    assert g.stat_bytes == 352 * 80 * 16 <= g.stat_region
    for N in (1, 2, 5, 10, 16, 20, 64, 110, 210):
        for (H, cin, cout, ks, stride) in [(21, 80, 80, 3, 1), (21, 40, 80, 3, 2), (32, 20, 20, 3, 1), (11, 80, 80, 3, 1),
                                           (8, 80, 160, 1, 2), (16, 40, 40, 3, 1)]:
            for path in (0, 1, 2):
                g = engine.conv_selftest_geom(N, H, H, cin, cout, ks, stride, 0, path, 2, sms)
                if g.kernel < 0:
                    continue                      # the forced path does not cover this shape
                assert g.name != 'tcp'
                assert g.stat_bytes <= g.stat_region, (N, H, cin, cout, ks, stride, path, g.template)


def test_hooks_refuse_bad_arguments():
    from b200ocl import _native, engine
    desc, info, _ = engine.describe(32, 100, None)
    engine.conv_geom(desc, 1, info.n_bn - 1, 'dgrad', 132)
    for n, layer, pass_, sms in [(0, 1, 'train', 132), (10, -1, 'train', 132), (10, info.n_bn, 'eval', 132),
                                 (10, 0, 'dgrad', 132), (10, 1, 'train', -1)]:
        with pytest.raises(_native.NativeError):
            engine.conv_geom(desc, n, layer, pass_, sms)
    with pytest.raises(_native.NativeError):
        engine.conv_geom(engine.NetDesc(32, 32, 16, 100, 0, 128), 10, 0, 'train', 132)
    with pytest.raises(_native.NativeError):
        engine.conv_selftest_geom(4, 8, 8, 30, 20, 3, 1, 0, 0, 2, 132)
    # a forced path that does not cover the launch is reported, not refused: the halo strip has no train mode
    assert engine.conv_selftest_geom(4, 8, 8, 20, 20, 3, 1, 0, 3, 2, 132).kernel == -1
