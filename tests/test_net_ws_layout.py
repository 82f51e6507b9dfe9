"""CPU: b200ocl_net_train_ws_layout, the host-only hook that tells tests where a train workspace keeps each conv layer's
tensors and which backward launches a batch size gets (no GPU needed: it launches nothing)."""
import ctypes

import pytest

from oracle import resnet as oresnet


def conv_geometry(spec):
    """[(cin, cout, ks, stride, hout)] per conv layer in BatchNorm2d module order (stem, then conv1, conv2[, shortcut])."""
    hw = spec.in_hw
    out = [(3, spec.nf, 3, 1, hw)]
    for _, cin, cout, stride, sc in oresnet.block_plan(spec):
        ho = (hw + 2 - 3) // stride + 1
        out += [(cin, cout, 3, stride, ho), (cout, cout, 3, 1, ho)]
        if sc:
            out.append((cin, cout, 1, stride, (hw - 1) // stride + 1))
        hw = ho
    return out


def align(n):
    return (n + 255) // 256 * 256


@pytest.mark.parametrize('hw,head', [(32, None), (32, 'mlp'), (32, 'linear'), (84, None)])
@pytest.mark.parametrize('N', [1, 20, 110, 220])
def test_layout_regions(hw, head, N):
    from b200ocl import _native, engine
    spec = oresnet.Spec(hw, 20, 100, head=head)
    desc, info, _ = engine.describe(hw, 100, head)
    total = _native.lib().b200ocl_net_train_workspace_bytes(ctypes.byref(desc), N)
    geo = conv_geometry(spec)
    assert info.n_bn == len(geo)
    layouts = [engine.train_ws_layout(desc, N, i) for i in range(len(geo))]
    first = layouts[0]
    regions, wg_expect = [], 0
    for i, ((cin, cout, ks, stride, ho), L) in enumerate(zip(geo, layouts)):
        assert L.bytes == total
        for f in ('feat', 'hid', 'proj', 'wg_part', 'sms'):
            assert getattr(L, f) == getattr(first, f), (i, f)
        assert (L.cin, L.cout, L.ks, L.stride, L.hout, L.wout) == (cin, cout, ks, stride, ho, ho), i
        act = N * ho * ho * cout * 4
        regions += [('z%d' % i, L.z, act), ('a%d' % i, L.a, act), ('mean%d' % i, L.mean, cout * 4),
                    ('invstd%d' % i, L.invstd, cout * 4)]
        # the partials of every layer follow each other in layer order
        assert L.wg_layer == L.wg_part + wg_expect, i
        wg_expect += L.wgrad_splits * ks * ks * cin * cout * 4
        assert L.wgrad_splits >= 1 and L.bn_grid >= 1
        assert L.wgrad_kernel == 0 if i == 0 else L.wgrad_kernel in (1, 2)
        if ks == 1 or stride == 2:
            assert L.wgrad_kernel == 2, i
        if L.bn_fused:
            assert L.bn_grid <= L.sms
    # the split counts of all layers fill the partial region, which ends the workspace
    assert align(wg_expect) == total - first.wg_part
    regions += [('feat', first.feat, N * spec.dim_in * 4), ('hid', first.hid, N * spec.dim_in * 4),
                ('proj', first.proj, N * info.out_dim * 4), ('wg_part', first.wg_part, wg_expect)]
    regions.sort(key=lambda r: r[1])
    for (n0, o0, s0), (n1, o1, s1) in zip(regions, regions[1:]):
        assert s0 > 0 and o0 + s0 <= o1, (n0, o0, s0, n1, o1)
    assert regions[0][1] > 0 and regions[-1][1] + regions[-1][2] <= total


def test_layout_refuses_bad_arguments():
    from b200ocl import _native, engine
    desc, info, _ = engine.describe(32, 100, None)
    engine.train_ws_layout(desc, 1, info.n_bn - 1)
    for n, layer in [(0, 0), (-1, 0), (10, -1), (10, info.n_bn)]:
        with pytest.raises(_native.NativeError):
            engine.train_ws_layout(desc, n, layer)
    bad = engine.NetDesc(32, 32, 16, 100, 0, 128)      # nf != 20
    with pytest.raises(_native.NativeError):
        engine.train_ws_layout(bad, 10, 0)
