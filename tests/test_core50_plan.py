"""CPU: the network of CORe50 (128x128 inputs, Reduced_ResNet18(50) with the 2560-input classifier of
utils/setup_elements.py:59-62) on the engine's host-side plan -- its description, the convolution launch of every layer
and batch size, the train workspace, the batch limit, the 4096-feature cap, SCR's refusals, reference_init -- and the
oracle against the reference's forward and backward (tests/golden/core50.npz).  No GPU needed: nothing is launched."""
import ctypes
import hashlib
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import resnet as oresnet

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'core50.npz')
HW, NCLS = 128, 50
SMS = (114, 132, 148)


def _spec():
    return oresnet.Spec(HW, 20, NCLS)


def _geometry(spec):
    """[(cin, cout, ks, stride, hout)] per conv layer in BatchNorm2d module order."""
    hw = spec.in_hw
    out = [(3, spec.nf, 3, 1, hw)]
    for _, cin, cout, stride, sc in oresnet.block_plan(spec):
        ho = (hw + 2 - 3) // stride + 1
        out += [(cin, cout, 3, stride, ho), (cout, cout, 3, 1, ho)]
        if sc:
            out.append((cin, cout, 1, stride, (hw - 1) // stride + 1))
        hw = ho
    return out


def test_describe_matches_the_reference_module():
    """dim_in 2560 and a tensor table equal, shape for shape, to the reference module's parameters()."""
    from b200ocl import engine, nets
    _, info, table = engine.describe(HW, NCLS)
    assert info.dim_in == 2560 and info.out_dim == NCLS and _spec().dim_in == 2560
    shapes = list(oresnet.param_shapes(_spec()).values())
    assert [n for _, n, _ in table] == [int(np.prod(s)) for s in shapes]
    assert [tuple(s) for _, s in nets.param_layout(info.dim_in, NCLS)] == [tuple(s) for s in shapes]
    assert nets.reduced_resnet_dim_in(HW) == 2560
    assert all(hg for _, _, hg in table)


def test_feature_cap():
    """Descriptions up to 4096 features are planned, wider ones refused."""
    from b200ocl import _native, engine
    engine.describe(HW, 4096)                                  # out_dim 4096
    with pytest.raises(_native.NativeError):
        engine.describe(HW, 4097)
    with pytest.raises(_native.NativeError):
        engine.describe(200, 10)                               # 200 -> 25, pooled 6x6: 5760 features
    _, info, _ = engine.describe(HW, 10, head='mlp')           # a 2560 x 2560 hidden layer is within the cap
    assert info.dim_in == 2560 and info.out_dim == 128


@pytest.mark.parametrize('sms', SMS)
def test_every_launch_fits_its_workspace(sms):
    """test_conv_plan.py's sweep for the 128x128 classifier network: every layer, pass and batch size 1..512."""
    from b200ocl import engine
    desc, info, _ = engine.describe(HW, NCLS)
    geo = _geometry(_spec())
    assert len(geo) == info.n_bn
    for N in range(1, 513):
        region = None
        for layer, (_, _, ks, stride, _) in enumerate(geo):
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
                    assert g.stat_region == region, where
                else:
                    assert g.stat_bytes == 0, where


def test_wide_maps_take_the_wide_map_kernels():
    """The 128x128 and 64x64 layers never take the halo-strip kernels (conv_tcp, wgrad_tc: maps up to 37 wide); the
    32x32 and 16x16 layers do in the eval pass and the weight gradient of their 3x3 stride-1 convolutions."""
    from b200ocl import engine
    desc, _, _ = engine.describe(HW, NCLS)
    geo = _geometry(_spec())
    for N in (1, 10, 20, 64, 110):
        for layer, (cin, cout, ks, stride, ho) in enumerate(geo):
            L = engine.train_ws_layout(desc, N, layer)
            g = engine.conv_geom(desc, N, layer, 'eval', 132)
            if ho >= 64:
                assert g.name != 'tcp' and L.wgrad_kernel in (0, 2), (N, layer, g.template, L.wgrad_kernel)
            elif layer > 0 and ks == 3 and stride == 1:
                assert g.name == 'tcp' and L.wgrad_kernel == 1, (N, layer, g.template, L.wgrad_kernel)


@pytest.mark.parametrize('N', [1, 10, 20, 110])
def test_train_workspace_layout(N):
    """test_net_ws_layout.py's region checks for the 128x128 network."""
    from b200ocl import _native, engine
    desc, info, _ = engine.describe(HW, NCLS)
    total = _native.lib().b200ocl_net_train_workspace_bytes(ctypes.byref(desc), N)
    geo = _geometry(_spec())
    layouts = [engine.train_ws_layout(desc, N, i) for i in range(len(geo))]
    first = layouts[0]
    regions, wg = [], 0
    for i, ((cin, cout, ks, stride, ho), L) in enumerate(zip(geo, layouts)):
        assert L.bytes == total
        assert (L.cin, L.cout, L.ks, L.stride, L.hout, L.wout) == (cin, cout, ks, stride, ho, ho), i
        act = N * ho * ho * cout * 4
        regions += [('z%d' % i, L.z, act), ('a%d' % i, L.a, act), ('mean%d' % i, L.mean, cout * 4),
                    ('invstd%d' % i, L.invstd, cout * 4)]
        assert L.wg_layer == L.wg_part + wg, i
        wg += L.wgrad_splits * ks * ks * cin * cout * 4
        if L.bn_fused:
            assert L.bn_grid <= L.sms
    assert (wg + 255) // 256 * 256 == total - first.wg_part
    regions += [('feat', first.feat, N * 2560 * 4), ('hid', first.hid, N * 2560 * 4),
                ('proj', first.proj, N * info.out_dim * 4), ('wg_part', first.wg_part, wg)]
    regions.sort(key=lambda r: r[1])
    for (n0, o0, s0), (n1, o1, s1) in zip(regions, regions[1:]):
        assert s0 > 0 and o0 + s0 <= o1, (n0, o0, s0, n1, o1)
    assert regions[-1][1] + regions[-1][2] <= total


def test_scr_refusals():
    """SCR on CORe50: the reference's SupConResNet(dim_in=160) head cannot take 2560 features (ValueError, the
    reference fails at its first forward); without a head the SupCon loss would run at d = 2560 (NotImplementedError)."""
    from b200ocl import nets
    for head in ('mlp', 'linear'):
        with pytest.raises(ValueError, match='2560'):
            nets.setup_architecture(SimpleNamespace(data='core50', agent='SCR', head=head))
    with pytest.raises(NotImplementedError, match='2560'):
        nets.setup_architecture(SimpleNamespace(data='core50', agent='SCR', head='None'))
    with pytest.raises(NotImplementedError):
        nets.check_supcon(HW, 'None')
    nets.check_supcon(32, 'None')
    nets.check_supcon(84, 'mlp', 640)


def test_adopt_checks_the_classifier_width_first():
    """adopt() compares the module's classifier (or head) input width with the plan's dim_in and raises before it
    allocates anything (the module stays on the CPU here: the device check comes after)."""
    from b200ocl import nets
    m = torch.nn.Module()
    m.linear = torch.nn.Linear(160, NCLS)                      # Reduced_ResNet18(50) without the CORe50 classifier
    with pytest.raises(ValueError, match='2560'):
        nets.adopt(m, HW)
    m.linear = torch.nn.Linear(2560, NCLS)
    m.w = torch.nn.Parameter(torch.zeros(1))
    with pytest.raises(RuntimeError, match='CUDA'):           # the width passes; the CPU module is refused next
        nets.adopt(m, HW)


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip('core50.npz not generated')
    return np.load(GOLDEN)


@pytest.mark.parametrize('k', [0, 1])
def test_reference_init_matches_setup_architecture(k):
    """reference_init('core50') draws what the reference's setup_architecture draws: the 160-input classifier, then
    the 2560-input one that replaces it; the generator stands where the reference leaves it."""
    from b200ocl import nets
    g = _golden()
    tag = 'init%d_' % k
    torch.manual_seed(int(g[tag + 'seed']))
    flat = torch.cat([t.reshape(-1) for t in nets.reference_init('core50', NCLS, HW)]).numpy()
    assert hashlib.sha1(flat.tobytes()).hexdigest() == str(g[tag + 'sha1'])
    pick = np.sort(np.random.RandomState(7).choice(flat.size, 2048, replace=False))
    assert np.array_equal(flat[pick], g[tag + 'sample'])
    assert np.array_equal(torch.rand(4).numpy(), g[tag + 'after'])


def _net_inputs():
    """make_golden_core50.net_inputs()."""
    rs = np.random.RandomState(8)
    return rs.rand(6, 3, HW, HW).astype(np.float32), rs.randint(0, NCLS, 6).astype(np.int64)


def test_oracle_matches_reference_forward_and_backward():
    """The fp32 oracle network at 128x128 against the reference module from the same seeded weights: logits, loss, a
    gradient sample of every tensor and the running statistics after the train-mode forward."""
    g = _golden()
    spec = _spec()
    p, bn = oresnet.seeded_state(spec, 7)
    x, y = _net_inputs()
    loss, logits, grads = oresnet.ce_loss_and_grads(spec, p, bn, torch.from_numpy(x), torch.from_numpy(y))
    assert np.allclose(logits.numpy(), g['net_logits'], rtol=1e-4, atol=1e-4 * np.abs(g['net_logits']).max())
    assert abs(float(loss) - float(g['net_loss'])) <= 1e-5 * abs(float(g['net_loss']))
    assert len(grads) == int(g['net_n_tensors'])
    for i, gr in enumerate(grads.values()):
        flat = gr.reshape(-1).numpy()
        ref = g['net_grad%d' % i]
        sel = flat[np.random.RandomState(i).choice(flat.size, min(flat.size, 64), replace=False)]
        scale = max(np.abs(ref).max(), 1e-30)
        assert np.abs(sel - ref).max() <= 1e-3 * scale, (i, np.abs(sel - ref).max(), scale)
    run = np.concatenate([np.concatenate([bn[n + '.running_mean'].numpy(), bn[n + '.running_var'].numpy()])
                          for n in oresnet.bn_names(spec)])
    assert np.allclose(run, g['net_bn'], rtol=1e-5, atol=1e-6)
