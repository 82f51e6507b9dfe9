"""CPU: OpenLORIS on the engine's host side -- 50x50 inputs, plain Reduced_ResNet18(69) with its 160-input classifier
(utils/setup_elements.py:67-68; the maps go 50 -> 25 -> 13 -> 7 and avg_pool2d(4) floors 7x7 to 1x1): the description,
the convolution launch of every layer and batch size, which layers take the halo-strip kernels, the train workspace,
setup_architecture for every agent and SCR head, reference_init and the oracle against the reference's forward and
backward (tests/golden/openloris.npz), and nearest-class-mean evaluation's one mean and one random direction per
distinct class when new-instance streams repeat labels in old_labels.  No GPU needed: nothing is launched."""
import ctypes
import hashlib
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import resnet as oresnet

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'openloris.npz')
HW, NCLS = 50, 69
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
    """dim_in 160 and a tensor table equal, shape for shape, to the reference module's parameters()."""
    from b200ocl import engine, nets
    _, info, table = engine.describe(HW, NCLS)
    assert info.dim_in == 160 and info.out_dim == NCLS and _spec().dim_in == 160
    shapes = list(oresnet.param_shapes(_spec()).values())
    assert [n for _, n, _ in table] == [int(np.prod(s)) for s in shapes]
    assert [tuple(s) for _, s in nets.param_layout(info.dim_in, NCLS)] == [tuple(s) for s in shapes]
    assert nets.reduced_resnet_dim_in(HW) == 160
    assert [ho for _, _, _, _, ho in _geometry(_spec())][::5] == [50, 25, 13, 7]
    assert all(hg for _, _, hg in table)


@pytest.mark.parametrize('sms', SMS)
def test_every_launch_fits_its_workspace(sms):
    """test_conv_plan.py's sweep for the 50x50 network: every layer, pass and batch size 1..512 finds a kernel, the
    train pass's statistics partials fit their region, and the halo-strip convolution never takes a train pass."""
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


def test_which_layers_take_the_strip_kernels():
    """The 50x50 layers are wider than the halo-strip kernels take (conv_tcp, wgrad_tc: maps up to 37 wide): their
    eval pass runs conv_tc at N = 10 and the fp32 patch kernel from N = 20, their weight gradient the fp32 kernel.  The
    3x3 stride-1 convolutions of the 25x25, 13x13 and 7x7 layers take conv_tcp (eval, data gradient) and wgrad_tc."""
    from b200ocl import engine
    desc, _, _ = engine.describe(HW, NCLS)
    geo = _geometry(_spec())
    for sms in SMS:
        for N in (1, 10, 20, 64, 110):
            for layer, (cin, cout, ks, stride, ho) in enumerate(geo):
                L = engine.train_ws_layout(desc, N, layer)
                g = engine.conv_geom(desc, N, layer, 'eval', sms)
                where = (sms, N, layer, g.name, L.wgrad_kernel)
                if layer == 0:
                    assert g.name == 'stem' and L.wgrad_kernel == 0, where
                elif ho == HW:
                    assert g.name != 'tcp' and L.wgrad_kernel == 2, where
                elif ks == 3 and stride == 1:
                    assert g.name == 'tcp' and L.wgrad_kernel == 1, where
                    assert engine.conv_geom(desc, N, layer, 'dgrad', sms).name == 'tcp', where
                else:
                    assert g.name != 'tcp' and L.wgrad_kernel == 2, where
    for N, name in ((10, 'tc'), (20, 'patch'), (110, 'patch')):
        assert engine.conv_geom(desc, N, 1, 'eval', 132).name == name, N


@pytest.mark.parametrize('N', [1, 10, 20, 110])
def test_train_workspace_layout(N):
    """test_net_ws_layout.py's region checks for the 50x50 network."""
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
    regions += [('feat', first.feat, N * 160 * 4), ('hid', first.hid, N * 160 * 4),
                ('proj', first.proj, N * info.out_dim * 4), ('wg_part', first.wg_part, wg)]
    regions.sort(key=lambda r: r[1])
    for (n0, o0, s0), (n1, o1, s1) in zip(regions, regions[1:]):
        assert s0 > 0 and o0 + s0 <= o1, (n0, o0, s0, n1, o1)
    assert regions[-1][1] + regions[-1][2] <= total


class _Built(object):
    """Stands in for nets.EngineModel: records what the network constructors ask for without allocating on a GPU."""
    def __init__(self, in_hw, num_classes, head=None, feat_dim=128, device='cuda'):
        self.in_hw, self.num_classes, self.head, self.feat_dim = in_hw, num_classes, head, feat_dim


@pytest.mark.parametrize('agent', ['ER', 'AGEM', 'LWF', 'EWC', 'ICARL', 'GDUMB', 'SCR', 'SCP'])
def test_setup_architecture(agent, monkeypatch):
    """Every agent's network at 50x50: Reduced_ResNet18(69) for the classifier agents, and for SCR a SupConResNet built
    at 50x50 (not the 32x32 that its 160 features would select) whose mlp, linear and None heads all see 160 features."""
    from b200ocl import engine, nets
    monkeypatch.setattr(nets, 'EngineModel', _Built)
    heads = ('mlp', 'linear', 'None') if agent in ('SCR', 'SCP') else ('mlp',)
    for head in heads:
        m = nets.setup_architecture(SimpleNamespace(data='openloris', agent=agent, head=head))
        if agent in ('SCR', 'SCP'):
            assert (m.in_hw, m.num_classes, m.head, m.feat_dim) == (HW, 100, head, 128), head
            _, info, _ = engine.describe(HW, 100, head=head)
            assert info.dim_in == 160 and info.out_dim == (160 if head == 'None' else 128), head
        else:
            assert (m.in_hw, m.num_classes, m.head) == (HW, NCLS, None)
    nets.check_supcon(HW, 'None')                    # 160 features are within the SupCon kernel's 1024


def test_supconresnet_keeps_its_dim_in_fallback(monkeypatch):
    """Callers that give SupConResNet no in_hw still get the network dim_in selects."""
    from b200ocl import nets
    monkeypatch.setattr(nets, 'EngineModel', _Built)
    assert nets.SupConResNet(160).in_hw == 32 and nets.SupConResNet(640).in_hw == 84
    assert nets.SupConResNet(160, in_hw=HW).in_hw == HW


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip('openloris.npz not generated')
    return np.load(GOLDEN)


@pytest.mark.parametrize('k', [0, 1])
def test_reference_init_matches_setup_architecture(k):
    """reference_init('openloris') draws what the reference's setup_architecture draws: the 160-input classifier and no
    replacement; the generator stands where the reference leaves it."""
    from b200ocl import nets
    g = _golden()
    tag = 'init%d_' % k
    torch.manual_seed(int(g[tag + 'seed']))
    ps = nets.reference_init('openloris', NCLS, HW)
    assert tuple(ps[-2].shape) == (NCLS, 160) and tuple(ps[-1].shape) == (NCLS,)
    flat = torch.cat([t.reshape(-1) for t in ps]).numpy()
    assert hashlib.sha1(flat.tobytes()).hexdigest() == str(g[tag + 'sha1'])
    pick = np.sort(np.random.RandomState(7).choice(flat.size, 2048, replace=False))
    assert np.array_equal(flat[pick], g[tag + 'sample'])
    assert np.array_equal(torch.rand(4).numpy(), g[tag + 'after'])


def _net_inputs():
    """make_golden_openloris.net_inputs()."""
    rs = np.random.RandomState(10)
    return rs.rand(6, 3, HW, HW).astype(np.float32), rs.randint(0, NCLS, 6).astype(np.int64)


def test_oracle_matches_reference_forward_and_backward():
    """The fp32 oracle network at 50x50 against the reference module from the same seeded weights: logits, loss, a
    gradient sample of every tensor and the running statistics after the train-mode forward."""
    g = _golden()
    spec = _spec()
    p, bn = oresnet.seeded_state(spec, 9)
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


# ----------------------------------------------------------------------------- NCM over repeated old_labels
def _reference_means(old_labels, feats, labels, d):
    """A restatement of agents/base.py:124-141 over precomputed features: a dict keyed by old_labels (one entry per
    distinct class, in first-occurrence order), the normalised mean of the normalised features of each class's
    exemplars, and for a class without exemplars one torch.normal direction of the feature size, normalised."""
    cls_exemplar = {cls: [] for cls in old_labels}
    for f, y in zip(feats, labels):
        cls_exemplar[int(y)].append(f)
    means = {}
    for cls, exemplar in cls_exemplar.items():
        fs = [f / f.norm() for f in exemplar]
        if len(fs) == 0:
            mu = torch.normal(0, 1, size=(1, d)).squeeze()
        else:
            mu = torch.stack(fs).mean(0).squeeze()
        means[cls] = mu / mu.norm()
    return means


def _engine_means(old_labels, feats, labels, d):
    """evaluate()'s host side: learners.ncm_class_ids, the class means b200ocl_ncm_class_means computes (restated on
    the CPU in float64), then learners.ncm_fill_empty."""
    from b200ocl import learners
    ids = learners.ncm_class_ids(old_labels)
    means = torch.zeros(len(ids), d)
    counts = torch.zeros(len(ids), dtype=torch.int32)
    for k, c in enumerate(ids):
        rows = feats[labels == c].double()
        counts[k] = rows.shape[0]
        if rows.shape[0]:
            mu = (rows / rows.norm(dim=1, keepdim=True)).mean(0)
            means[k] = (mu / mu.norm()).float()
    return ids, learners.ncm_fill_empty(means, counts)


@pytest.mark.parametrize('tasks', [1, 2, 5])
def test_ncm_draws_one_direction_per_distinct_class(tasks):
    """old_labels as a new-instance stream leaves it after `tasks` tasks (every task holds every class, in a different
    set order): the engine keeps one mean per distinct class in first-occurrence order, draws one direction per empty
    class in the reference's order (the generator ends where the reference's does), and its nearest mean predicts the
    label the reference predicts over the repeated old_labels."""
    rs = np.random.RandomState(tasks)
    C, d = 12, 160
    order = list(rs.permutation(C))
    old = []
    for _ in range(tasks):
        old += order                      # set(y_train) has the same order every task: the labels repeat as a block
    labels = torch.from_numpy(rs.choice([0, 1, 3, 4, 7, 8, 11], 30)).long()     # 2, 5, 6, 9 and 10 stay empty
    feats = torch.from_numpy(np.maximum(rs.standard_normal((30, d)), 0).astype(np.float32) + 0.01)
    torch.manual_seed(17)
    ref = _reference_means(old, feats, labels, d)
    after_ref = torch.rand(3)
    torch.manual_seed(17)
    ids, means = _engine_means(old, feats, labels, d)
    after = torch.rand(3)
    assert ids == list(ref.keys()) == order
    assert torch.equal(after, after_ref)
    for k, c in enumerate(ids):
        assert torch.allclose(means[k], ref[c], atol=1e-6), c
    q = torch.from_numpy(rs.standard_normal((40, d)).astype(np.float32))
    q = q / q.norm(dim=1, keepdim=True)
    ref_stack = torch.stack([ref[c] for c in old])                               # base.py:164, repeats included
    ref_pred = np.array(old)[((q[:, None, :] - ref_stack[None]) ** 2).sum(2).argmin(1).numpy()]
    pred = np.array(ids)[((q[:, None, :] - means[None]) ** 2).sum(2).argmin(1).numpy()]
    assert np.array_equal(pred, ref_pred)


def test_ncm_class_ids_keep_distinct_streams_unchanged():
    """Without repeated labels (class-incremental streams) the class list is old_labels itself, so the draws and the
    results stay what they were."""
    from b200ocl import learners
    old = [7, 3, 9, 0, 12, 5]
    assert learners.ncm_class_ids(old) == old
    assert learners.ncm_class_ids(old + [3, 7, 1]) == old + [1]
