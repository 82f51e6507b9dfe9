"""OpenLORIS's network on the engine (50x50 inputs, Reduced_ResNet18(69) with the 160-input classifier):
  * the train-mode forward over a NaN-filled workspace, layer by layer from the engine's own tensors, end to end from
    the images and in eval mode (test_gpu_forward_fp64.run_case at 50x50), at batch sizes that reach every
    (kernel, template) pair the convolution planner picks at 50x50 on the card in use;
  * the backward against the fp64 restatement built from the tensors the engine's forward left in the workspace
    (test_gpu_backward_fp64.run_case at 50x50), at batch sizes that reach every BN-backward form and weight-gradient
    kernel at 50x50 on the card in use;
  * SupCon at SCR's 50x50 shapes (d = 128 with the mlp or linear head, d = 160 without a head) against oracle/supcon.py;
    the augmentation kernel at 50x50 against oracle/augment.py; stream preparation of 50x50x3 uint8 rows against
    torchvision's ToTensor;
  * drop-in runs on new-instance streams (every call carries all 69 classes) of ER, ER + ASER, ER + MIR, A-GEM, LwF,
    EWC++, SCR, ER with the separated softmax, ER with the NCM trick, iCaRL's first call and GDumb against the
    reference's own runs (tests/golden/openloris.npz) with the bars of test_gpu_dropin.py;
  * iCaRL's refusal at the second new-instance call, before anything launches.
Tolerances are about 3x the largest error measured on an H100 80GB HBM3 (132 SMs, 700 W power limit); the measured
maxima are printed by each test."""
import hashlib
import json
import os
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import test_gpu_backward_fp64 as bwd
import test_gpu_dropin as dropin
import test_gpu_forward_fp64 as fwd
import test_gpu_supcon_fp64 as sup

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'openloris.npz')
HW, NCLS = 50, 69
FWD_BATCHES = (2, 10, 14, 24, 83, 161)     # the coverage tests below check what they reach on the card in use
BWD_BATCHES = (1, 2, 14, 24, 37, 72, 108, 200, 300, 435)

# bars: about 3x the largest error measured on an H100 80GB HBM3 (in brackets)
# The fp64 forward and backward keep the bars of test_gpu_forward_fp64 / test_gpu_backward_fp64 and those files'
# last-image-share guards: over the batches below the 50x50 maxima stay 2.7-4.7x under them.  Forward (max |got - ref| /
# max |ref| per tensor): z 8.4e-7 (layer4.0.bn1, N = 161), mean 1.9e-8, invstd 5.6e-8, a 1.3e-7, feat 1.3e-7, head 1.5e-7,
# running statistics 2.3e-9, e2e 1.2e-6 (N = 83), eval 2.3e-6 (N = 10).  Backward (per parameter tensor): conv 6.4e-6
# (layer2.1.conv1.weight, N = 435), BN 1.3e-5 (bn1.bias, N = 300), head 6.7e-7 (linear.weight, N = 435).
FWD_TOL = dict(fwd.TOL)
BWD_TOL = dict(bwd.TOL)
SUPCON_LOSS_TOL = 1.5e-8   # SupCon loss, in test_gpu_supcon_fp64.py's units [4.2e-9, A = 220, d = 160]
SUPCON_GRAD_TOL = 2e-6     # SupCon gradient, in test_gpu_supcon_fp64.py's units [5.8e-7, A = 344, d = 128]
AUG_MAX = 2.5e-5           # augmentation, largest absolute pixel error [7.4e-6]
AUG_MEAN = 7e-7            # augmentation, mean absolute pixel error [2.3e-7, n = 220]


@pytest.fixture(scope='module')
def engine():
    from b200ocl import engine
    return engine


def _report(what, N, rows, share_kinds):
    """Print the worst error per kind (the numbers the bars come from) and the smallest last-image share."""
    worst, share = {}, {}
    for r in rows:
        k, name, err, sh = (r[1], r[0], r[2], r[3]) if what == 'bwd' else r
        if err > worst.get(k, (-1, ''))[0]:
            worst[k] = (err, name)
        if sh is not None and k in share_kinds and sh < share.get(k, (2, ''))[0]:
            share[k] = (sh, name)
    print('openloris %s N=%d worst %s; smallest share %s' % (
        what, N, ', '.join('%s %.3g (%s)' % (k, e, n) for k, (e, n) in sorted(worst.items())),
        ', '.join('%s %.3g (%s)' % (k, e, n) for k, (e, n) in sorted(share.items()))))


def _check(rows, N, tol, share_kinds, key):
    """test_gpu_forward_fp64.check / test_gpu_backward_fp64.check with the bars of this file."""
    bad = sorted(((err / tol[k], k, name, err) for k, name, err, _ in map(key, rows) if not err <= tol[k]), reverse=True)
    assert not bad, bad[:4]
    if N >= 2:
        # a tolerance that could hide a dropped image (or tile) would be useless
        for k, name, _, sh in map(key, rows):
            if k in share_kinds:
                assert 10 * tol[k] <= sh, (k, name, sh, tol[k])


def _conv_templates(engine, N, pass_):
    desc, info, _ = engine.describe(HW, 100)
    return {engine.conv_geom(desc, N, i, pass_).template for i in range(1 if pass_ == 'dgrad' else 0, info.n_bn)}


def _cover(per):
    """A small set of batch sizes reaching everything in per (N -> set): printed when a coverage test fails."""
    every, got, pick = set().union(*per.values()), set(), []
    while got != every:
        N = max(per, key=lambda n: (len(per[n] - got), -n))
        pick.append(N)
        got |= per[N]
    return sorted(pick)


def test_cases_reach_every_forward_kernel(engine):
    """FWD_BATCHES reach every (kernel, template) pair of the train and eval forwards at N <= 512 on this card, and
    BWD_BATCHES every pair of the data-gradient launches."""
    for pass_, batches in (('train', FWD_BATCHES), ('eval', FWD_BATCHES), ('dgrad', BWD_BATCHES)):
        per = {N: _conv_templates(engine, N, pass_) for N in range(1, 513)}
        every = set().union(*per.values())
        reached = set().union(*[per[N] for N in batches])
        assert reached == every, (pass_, sorted(every - reached), 'a cover', _cover(per))


def _bwd_geometry(engine, N):
    """(layer, BN backward fused or two-phase, wide fused grid, weight-gradient kernel) per conv layer."""
    desc, info, _ = engine.describe(HW, 100)
    out = set()
    for i in range(info.n_bn):
        L = engine.train_ws_layout(desc, N, i)
        assert L.sms == torch.cuda.get_device_properties(0).multi_processor_count
        out.add((i, bool(L.bn_fused), bool(L.bn_fused) and 2 * L.bn_grid > L.sms, L.wgrad_kernel))
    return out


def test_cases_reach_every_backward_geometry(engine):
    """BWD_BATCHES reach, on this card, every BN-backward form and weight-gradient kernel each layer of the 50x50
    network takes at N <= 512 (the thresholds move with the SM count, so they are read through the hook)."""
    per = {N: _bwd_geometry(engine, N) for N in range(1, 513)}
    every = set().union(*per.values())
    reached = set().union(*[per[N] for N in BWD_BATCHES])
    assert reached == every, (sorted(every - reached), 'a cover', _cover(per))
    assert {k for _, _, _, k in every} == {0, 1, 2}


@pytest.mark.parametrize('N', FWD_BATCHES)
def test_forward_matches_fp64(engine, N):
    rows = fwd.run_case(engine, HW, None, N)
    _report('fwd', N, rows, fwd.STATS)
    _check(rows, N, FWD_TOL, fwd.STATS, lambda r: r)


@pytest.mark.parametrize('N', BWD_BATCHES)
def test_backward_matches_fp64(engine, N):
    _, _, rows = bwd.run_case(engine, HW, None, N)
    _report('bwd', N, rows, ('conv', 'bn', 'head'))
    _check(rows, N, BWD_TOL, ('conv', 'bn', 'head'), lambda r: (r[1], r[0], r[2], r[3]))


# ----------------------------------------------------------------------------- SCR's kernels at 50x50
@pytest.mark.parametrize('B,d', [(110, 128), (110, 160), (172, 128), (172, 160)])
def test_supcon_at_scr_shapes(B, d):
    """The SupCon loss over SCR's two views of 100 memory + 10 stream rows (and + 72, the drop-in runs' batch): d = 128
    behind the mlp / linear head, d = 160 for head None, against the fp64 oracle in test_gpu_supcon_fp64.py's units."""
    from b200ocl import ops
    from oracle import supcon as osup
    case = ('openloris', B, 2, d, 0.07, 'few', 1.0, False)
    f, y, ft, yt = sup.make_inputs(case, B + d)
    loss, grad = ops.supcon(ft, yt, 0.07)
    ref_loss, ref_grad = osup.supcon_loss_and_grad_torch(torch.from_numpy(f).cuda(), yt, 0.07)
    le, ge = sup.errors(loss, grad, ref_loss, ref_grad, *sup.scales(f, 0.07))
    print('openloris supcon A=%d d=%d loss %.3g grad %.3g' % (2 * B, d, le, ge))
    assert le <= SUPCON_LOSS_TOL and ge <= SUPCON_GRAD_TOL, (le, ge)


@pytest.mark.parametrize('n,seed', [(110, 0), (220, 1)])
def test_augment_kernel_at_50(n, seed):
    """csrc/augment.cu at 50x50 with drawn parameters (crop boxes, flips, the four colour operations in every order,
    grayscale) against oracle/augment.py in float64."""
    from b200ocl.augment import SCRTransform, draw_params
    from oracle import augment as oaug
    rs = np.random.RandomState(50 + seed)
    x = rs.rand(n, 3, HW, HW).astype(np.float32)
    x[0, :, :4, :4] = 0.5
    x[1, :, :4, :4] = 0.0
    p = draw_params(n, HW, HW, rng=rs)
    p[:, 5] = 1
    for i in range(n):
        order = rs.permutation(4)
        p[i, 10] = float(sum(int(op) << (2 * k) for k, op in enumerate(order)))
    p[::3, 5] = rs.rand(len(p[::3])) < 0.5
    out = SCRTransform((HW, HW))(torch.from_numpy(x).cuda(), params=p).cpu().numpy()
    ref = oaug.scr_view(x, p)
    err = np.abs(out - ref)
    print('openloris augment n=%d max %.3g mean %.3g' % (n, err.max(), err.mean()))
    assert err.max() <= AUG_MAX, (err.max(), np.unravel_index(err.argmax(), err.shape))
    assert err.mean() <= AUG_MEAN
    assert (p[:, 2] < HW).any() and (p[:, 4] > 0.5).any() and (p[:, 11] > 0.5).any()


@pytest.mark.parametrize('n', [1, 75, 172])
def test_stream_prepare_50x50_rows(n):
    """uint8 HWC rows of 50 x 50 x 3 = 7500 bytes -> fp32 CHW / 255, in a shuffled order, bit-identical to torchvision's
    ToTensor (utils/setup_elements.py:41-42)."""
    from torchvision import transforms
    from b200ocl import ops
    rs = np.random.RandomState(n)
    x = rs.randint(0, 256, (n, HW, HW, 3)).astype(np.uint8)
    x[0, 0, 0] = 255
    x[-1, -1, -1] = 0
    perm = rs.permutation(n)
    got = ops.stream_prepare(torch.from_numpy(x).cuda(), torch.from_numpy(perm).cuda()).cpu()
    tt = transforms.ToTensor()
    assert torch.equal(got, torch.stack([tt(x[i]) for i in perm]))


# ----------------------------------------------------------------------------- drop-in runs against the reference
def ni_inputs(rs, mem, hw, n_label, per_call, n_calls):
    """tests/golden/make_golden_openloris.py ni_inputs()."""
    x = rs.rand(mem, 3, hw, hw).astype(np.float32)
    y = rs.randint(0, n_label, mem).astype(np.int64)
    calls = [(rs.randint(0, 256, (per_call, hw, hw, 3)).astype(np.uint8),
              rs.permutation(np.arange(per_call) % n_label).astype(np.int64)) for _ in range(n_calls)]
    tests = [(rs.randint(0, 256, (96, hw, hw, 3)).astype(np.uint8), rs.permutation(np.arange(96) % n_label).astype(np.int64))
             for _ in range(2)]
    return x, y, calls, tests


def _golden():
    return np.load(GOLDEN)


def _agent(params):
    from b200ocl import nets, registry
    name = params.agent
    cls = registry.agents.get(name) or registry.extra_agents[name]
    return cls(nets.setup_architecture(params), None, params)


def _loaders(tests):
    return [[(torch.from_numpy(tx).permute(0, 3, 1, 2).float().div(255), torch.from_numpy(ty))] for tx, ty in tests]


@pytest.mark.parametrize('case', range(int(np.load(GOLDEN)['n_dropin'])))
def test_dropin_matches_reference_run(case):
    """test_gpu_dropin.py's comparison at 50x50 and 69 classes on new-instance calls (agents with and without a memory):
    the memory, the weight update, the BN statistics, old_labels with its repeats and the accuracies."""
    from b200ocl import memory
    from b200ocl.augment import Identity
    from oracle import resnet as oresnet
    g = _golden()
    tag = 'c%d_' % case
    kind, n_calls, per_call, wseed, seed, dseed = json.loads(str(g[tag + 'case']))
    params = SimpleNamespace(**json.loads(str(g[tag + 'params'])))
    params.cuda = True
    spec = oresnet.Spec(HW, 20, 100, head='mlp') if params.agent == 'SCR' else oresnet.Spec(HW, 20, NCLS)
    memory.set_mode(True, 'cpu')                    # the reference ran on the CPU: its draws came from CPU generators
    memory.ClassBalancedRandomSampling.reset()
    try:
        agent = _agent(params)
        assert agent.engine.in_hw == HW
        if hasattr(agent, 'transform'):
            agent.transform = Identity()            # the reference side ran kornia stubbed to the identity
        p, bn = oresnet.seeded_state(spec, wseed)
        agent.engine.load(list(p.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
        w0 = torch.cat([t.reshape(-1) for t in p.values()]).numpy()
        pick = dropin.dropin_sample(w0.size)
        w0 = w0[pick].astype(np.float64)
        np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
        rs = np.random.RandomState(dseed)
        x, y, calls, tests = ni_inputs(rs, params.mem_size, HW, NCLS, per_call, n_calls)
        buf = getattr(agent, 'buffer', None)
        if buf is not None:
            dev = buf.buffer_img.device
            buf.update(torch.from_numpy(x).to(dev), torch.from_numpy(y).to(dev))
        for c, (xt, yt) in enumerate(calls):
            where = '%s case %d call %d' % (kind, case, c)
            agent.train_learner(xt, yt)
            torch.cuda.synchronize()
            if buf is not None:
                assert buf.current_index == int(g[tag + 'index%d' % c]) and buf.n_seen_so_far == int(g[tag + 'seen%d' % c]), where
                labels = buf.buffer_label.cpu().numpy()
                diff = np.flatnonzero(labels != g[tag + 'label%d' % c])
                if diff.size:
                    # ASER's near-tied keep / evict decisions, as in test_gpu_dropin.py: the case ends there
                    upd = buf.update_method
                    assert hasattr(upd, 'last_sv_sum'), (where, 'different slots written by a non-ASER update', diff[:10])
                    cand = upd.last_choices['upd_cand_ind'].tolist()
                    sv = torch.as_tensor(upd.last_sv_sum).cpu().numpy()
                    assert all(int(sl) in cand for sl in diff), (where, 'written slots outside the candidate draw', diff)
                    scores = np.array([sv[cand.index(int(sl))] for sl in diff])
                    near_tie = scores.max() - scores.min() <= dropin.NEAR_TIE * float(np.abs(sv).max())
                    assert diff.size <= int(g[tag + 'spread_slots'][c]) or near_tie, (where, diff, scores)
                    return
                assert hashlib.sha1(buf.buffer_img.cpu().numpy().tobytes()).hexdigest() == str(g[tag + 'img%d' % c]), where
            w = agent.engine.state.params.cpu().numpy()[pick]
            err = dropin._rel(w - w0, g[tag + 'w%d' % c].astype(np.float64) - w0)
            print('openloris dropin %s case %d call %d weight update rel %.3g (spread %.3g)'
                  % (kind, case, c, err, g[tag + 'spread_w'][c]))
            assert err <= max(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_w'][c]), (where, 'sampled weight update', err)
            err = dropin._rel(agent.engine.state.bn_stats.cpu().numpy(), g[tag + 'bn%d' % c].astype(np.float64))
            assert err <= max(dropin.BN_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_bn'][c]), (where, 'BN running statistics', err)
        assert agent.old_labels == g[tag + 'old_labels'].tolist()
        acc = np.asarray(agent.evaluate(_loaders(tests)))
        assert np.abs(acc - g[tag + 'acc']).max() <= 3.1 / 96, (kind, case, acc, g[tag + 'acc'])
    finally:
        memory.set_mode(False)
        memory.ClassBalancedRandomSampling.reset()


@pytest.mark.parametrize('case', range(int(np.load(GOLDEN)['n_gdumb'])))
def test_gdumb_dropin_matches_reference_run(case, monkeypatch):
    """test_gpu_gdumb.py's drop-in comparison at 50x50 on new-instance calls: the re-initialisation drawn as the
    reference's setup_architecture('openloris') draws it, the greedy memory balanced over 69 classes, the trained
    weights and the accuracies."""
    from b200ocl import learners, memory, nets
    g = _golden()
    tag = 'g%d_' % case
    n_calls, per_call, seed, dseed = json.loads(str(g[tag + 'case']))
    params = SimpleNamespace(**json.loads(str(g[tag + 'params'])))
    params.cuda = True
    inits = []
    orig = nets.reference_init

    def reference_init(*a):
        ps = orig(*a)
        inits.append(torch.cat([t.reshape(-1) for t in ps]).numpy())
        return ps
    monkeypatch.setattr(learners.nets, 'reference_init', reference_init)
    memory.set_mode(True, 'cpu')
    try:
        agent = _agent(params)
        np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
        _, _, calls, tests = ni_inputs(np.random.RandomState(dseed), 0, HW, NCLS, per_call, n_calls)
        pick = None
        for c, (xt, yt) in enumerate(calls):
            where = 'case %d call %d' % (case, c)
            agent.train_learner(xt, yt)
            torch.cuda.synchronize()
            mem_c = np.array(list(agent.mem_c.items()), dtype=np.int64).reshape(-1, 2)
            assert np.array_equal(mem_c, g[tag + 'mem_c%d' % c]), where
            rows = agent.memory.images[torch.from_numpy(agent.memory.order()).cuda()].cpu().numpy()
            assert hashlib.sha1(rows.tobytes()).hexdigest() == str(g[tag + 'mem%d' % c]), where
            pick = dropin.dropin_sample(inits[-1].size) if pick is None else pick
            w0 = g[tag + 'w_init%d' % c]
            assert np.array_equal(inits[-1][pick], w0), (where, 're-initialisation')
            w0 = w0.astype(np.float64)
            w = agent.engine.state.params.cpu().numpy()[pick]
            err = dropin._rel(w - w0, g[tag + 'w%d' % c].astype(np.float64) - w0)
            print('openloris gdumb call %d weight update rel %.3g (spread %.3g)' % (c, err, g[tag + 'spread_w'][c]))
            assert err <= max(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_w'][c]), (where, err)
            err = dropin._rel(agent.engine.state.bn_stats.cpu().numpy(), g[tag + 'bn%d' % c].astype(np.float64))
            assert err <= max(dropin.BN_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_bn'][c]), (where, 'BN statistics', err)
        acc = np.asarray(agent.evaluate(_loaders(tests)))
        assert np.abs(acc - g[tag + 'acc']).max() <= 3.1 / 96, (case, acc, g[tag + 'acc'])
    finally:
        memory.set_mode(False)


def test_icarl_refuses_the_second_new_instance_call():
    """iCaRL trains its first new-instance call; at the second, old_labels ++ new_labels holds 2 x 69 = 138 label
    positions for 69 logits (the reference fails at icarl.py:62).  The ValueError comes before anything launches."""
    from b200ocl import _native, memory
    g = _golden()
    case = [k for k in range(int(g['n_dropin'])) if json.loads(str(g['c%d_case' % k]))[0] == 'icarl'][0]
    params = SimpleNamespace(**json.loads(str(g['c%d_params' % case])))
    params.cuda = True
    memory.set_mode(True, 'cpu')
    try:
        agent = _agent(params)
        rs = np.random.RandomState(3)
        x, y, calls, _ = ni_inputs(rs, params.mem_size, HW, NCLS, params.batch + 3, 2)
        agent.buffer.update(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda())
        agent.train_learner(*calls[0])
        torch.cuda.synchronize()
        before = _native.launch_count()
        with pytest.raises(ValueError, match='138 label positions exceed the 69 logits'):
            agent.train_learner(*calls[1])
        torch.cuda.synchronize()
        assert _native.launch_count() == before
    finally:
        memory.set_mode(False)
