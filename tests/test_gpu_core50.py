"""CORe50's network on the engine (128x128 inputs, Reduced_ResNet18 with the 2560-input classifier):
  * the train-mode forward over a NaN-filled workspace, layer by layer from the engine's own tensors, end to end from
    the images and in eval mode (test_gpu_forward_fp64.run_case at 128x128), at batch sizes that reach every
    (kernel, template) pair the convolution planner picks at 128x128 on the card in use;
  * the backward against the fp64 restatement built from the tensors the engine's forward left in the workspace
    (test_gpu_backward_fp64.run_case at 128x128), at batch sizes that reach every BN-backward and weight-gradient
    geometry at 128x128 on the card in use;
  * the wide linear forward and the NCM class means against fp64 at d = 2560 and d = 4096; kNN-SV at d = 2560 against
    oracle/knn_sv.py;
  * the batch limit: a pass whose activations would leave 32-bit indexing is refused before it launches;
  * drop-in runs of ER, ER + ASER, ER + MIR, iCaRL (NCM evaluation at d = 2560), EWC++ and GDumb against the reference's
    own runs (tests/golden/core50.npz) with the bars of test_gpu_dropin.py.
Tolerances are about 3x the largest error measured on an H100 80GB HBM3 (132 SMs, 700 W power limit); the measured
maxima are given beside each bar."""
import ctypes
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

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'core50.npz')
HW, NCLS = 128, 50
FWD_BATCHES = (1, 5, 6, 20, 42)      # the coverage tests below check what they reach on the card in use
BWD_BATCHES = (1, 3, 6, 10, 42, 110)

# bars: about 3x the largest error measured on an H100 80GB HBM3 (in brackets)
# The fp64 forward and backward keep the bars of test_gpu_forward_fp64 / test_gpu_backward_fp64: over the batches
# below, the 128x128 maxima stay 2.2-4.6x under them.  Forward (max |got - ref| / max |ref| per tensor): z 9.5e-7
# (layer4.0.bn1, N = 42), mean 2.1e-8, invstd 4.8e-8, a 1.2e-7, feat 1.5e-7, head 2.6e-7, running statistics 0 (the same
# bits), e2e 1.3e-6 (N = 20), eval 2.0e-6.  Backward (per parameter tensor): conv 6.6e-6 (layer1.1.conv2.weight,
# N = 110), BN 1.4e-5 (layer1.0.bn2.bias, N = 110), head 5.1e-7.  The smallest last-image share is 2.9e-5 (mean),
# 2.0e-4 (invstd), 8.3e-6 (running_var) in the forward and 7.7e-2 (BN), 8.4e-2 (conv), 0.11 (head) in the backward, each
# more than 10x its bar.
FWD_TOL = dict(fwd.TOL)
BWD_TOL = dict(bwd.TOL)
LIN_TOL = 2e-7           # linear forward, relative to sum |x||w| [3.6e-8 in the last case of each d]
NCM_TOL = 5e-8           # class means, absolute (unit-norm vectors) [1.5e-8]
KNN_TOL = 1e-7           # kNN-SV, absolute per entry [2.4e-8]


@pytest.fixture(scope='module')
def engine():
    from b200ocl import engine
    return engine


def _spec():
    from oracle import resnet as oresnet
    return oresnet.Spec(HW, 20, NCLS)


def _model(seed=7):
    from b200ocl import nets
    from oracle import resnet as oresnet
    spec = _spec()
    p, bn = oresnet.seeded_state(spec, seed)
    model = nets.Reduced_ResNet18(NCLS, in_hw=HW)
    model.engine.load(list(p.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
    return model.engine, p, bn


def _report(what, N, rows, share_kinds):
    """Print the worst error per kind (the numbers the bars come from) and the smallest last-image share."""
    worst, share = {}, {}
    for r in rows:
        k, name, err, sh = (r[1], r[0], r[2], r[3]) if what == 'bwd' else r
        if err > worst.get(k, (-1, ''))[0]:
            worst[k] = (err, name)
        if sh is not None and k in share_kinds and sh < share.get(k, (2, ''))[0]:
            share[k] = (sh, name)
    print('core50 %s N=%d worst %s; smallest share %s' % (
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


def test_cases_reach_every_forward_kernel(engine):
    """FWD_BATCHES reach every (kernel, template) pair of the train and eval forwards at N <= 512 on this card, and
    BWD_BATCHES every pair of the data-gradient launches."""
    for pass_, batches in (('train', FWD_BATCHES), ('eval', FWD_BATCHES), ('dgrad', BWD_BATCHES)):
        every = set().union(*[_conv_templates(engine, N, pass_) for N in range(1, 513)])
        reached = set().union(*[_conv_templates(engine, N, pass_) for N in batches])
        assert reached == every, (pass_, sorted(every - reached))


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
    """BWD_BATCHES reach, on this card, every BN-backward form and weight-gradient kernel each layer of the 128x128
    network takes at N <= 512 (the thresholds move with the SM count, so they are read through the hook)."""
    every = set().union(*[_bwd_geometry(engine, N) for N in range(1, 513)])
    reached = set().union(*[_bwd_geometry(engine, N) for N in BWD_BATCHES])
    assert reached == every, sorted(every - reached)
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


@pytest.mark.parametrize('d', [160, 1024, 1025, 2560, 4096])
def test_linear_forward_against_fp64(d):
    from b200ocl import ops
    rs = np.random.RandomState(d)
    for N, out, relu in [(1, 50, False), (20, 50, False), (37, 100, True), (110, 3, False)]:
        x = torch.from_numpy(rs.standard_normal((N, d)).astype(np.float32)).cuda()
        w = torch.from_numpy((rs.standard_normal((out, d)) / np.sqrt(d)).astype(np.float32)).cuda()
        b = torch.from_numpy(rs.standard_normal(out).astype(np.float32)).cuda()
        y = ops.linear_fwd(x, w, b, relu=relu)
        y64 = x.double() @ w.double().T + b.double()
        if relu:
            y64 = y64.clamp_min(0)
        scale = (x.double().abs() @ w.double().abs().T + b.double().abs())
        err = float(((y.double() - y64).abs() / scale).max())
        assert err <= LIN_TOL, (d, N, out, err)
        assert torch.equal(y, ops.linear_fwd(x, w, b, relu=relu))          # deterministic
    print('core50 linear d=%d rel %.3g' % (d, err))


def test_linear_forward_refuses_wider_rows():
    from b200ocl import _native, ops
    x = torch.zeros(2, 4097, device='cuda')
    with pytest.raises(_native.NativeError, match='4096'):
        ops.linear_fwd(x, torch.zeros(3, 4097, device='cuda'), torch.zeros(3, device='cuda'))


@pytest.mark.parametrize('d', [1024, 1025, 2560, 4096])
def test_ncm_class_means_against_fp64(d):
    from b200ocl import ops
    rs = np.random.RandomState(d)
    n, K = 700, 13
    f = np.maximum(rs.standard_normal((n, d)), 0).astype(np.float32)
    lab = rs.randint(0, K + 2, n)
    ids = np.arange(K + 1)                                        # class K + 1 never occurs; class K may
    means, counts = ops.ncm_class_means(torch.from_numpy(f).cuda(), torch.from_numpy(lab).cuda(), torch.from_numpy(ids).cuda())
    worst = 0.0
    for k in ids:
        rows = f[lab == k].astype(np.float64)
        assert int(counts[k]) == rows.shape[0]
        if rows.shape[0] == 0:
            continue
        mu = (rows / np.linalg.norm(rows, axis=1, keepdims=True)).mean(0)
        mu /= np.linalg.norm(mu)
        worst = max(worst, float(np.abs(means[k].cpu().numpy() - mu).max()))
    print('core50 ncm d=%d abs %.3g' % (d, worst))
    assert worst <= NCM_TOL, (d, worst)


def test_ncm_class_means_refuses_wider_features():
    from b200ocl import _native, ops
    with pytest.raises(_native.NativeError):
        ops.ncm_class_means(torch.zeros(2, 4097, device='cuda'), torch.zeros(2, dtype=torch.int64, device='cuda'),
                            torch.zeros(1, dtype=torch.int64, device='cuda'))


def test_knn_sv_at_2560_against_oracle():
    from b200ocl import ops
    from oracle import knn_sv as oknn
    rs = np.random.RandomState(2560)
    for E, C, k in [(10, 100, 3), (110, 160, 3), (30, 600, 5)]:
        ef = np.maximum(rs.standard_normal((E, 2560)), 0).astype(np.float32)
        cf = np.maximum(rs.standard_normal((C, 2560)), 0).astype(np.float32)
        ey, cy = rs.randint(0, 50, E), rs.randint(0, 50, C)
        out = ops.knn_sv(torch.tensor(ef).cuda(), torch.tensor(ey).cuda(), torch.tensor(cf).cuda(), torch.tensor(cy).cuda(),
                         k, want_matrix=True, want_sum=True)
        sv64, _, _ = oknn.knn_sv_matrix(ef, ey, cf, cy, k)
        err = np.abs(out['sv'].cpu().numpy() - sv64).max(1)
        print('core50 knn_sv E=%d C=%d max %.3g, share within bar %.3f' % (E, C, err.max(), (err <= KNN_TOL).mean()))
        assert (err <= KNN_TOL).mean() >= 0.98, err.max()


def test_batch_limit_is_refused_before_launch():
    """6554 images of 128x128 would put the stem output past INT_MAX elements: refused before the workspace is even
    looked at (the tiny workspace would otherwise be the error), and nothing launches."""
    from b200ocl import _native
    eng, _, _ = _model()
    lib = _native.lib()
    x = torch.zeros(1, device='cuda')
    ws = torch.zeros(256, dtype=torch.uint8, device='cuda')
    torch.cuda.synchronize()
    before = _native.launch_count()
    for name in ('b200ocl_net_features_eval', 'b200ocl_net_forward_train'):
        rc = getattr(lib, name)(ctypes.byref(eng.desc), ctypes.byref(eng.state.c), x.data_ptr(), 6554, x.data_ptr(),
                                ws.data_ptr(), ws.numel(), None)
        assert rc != 0 and b'batch limit of 6553' in lib.b200ocl_last_error(), name
    rc = lib.b200ocl_net_backward(ctypes.byref(eng.desc), ctypes.byref(eng.state.c), x.data_ptr(), x.data_ptr(), 6554,
                                  ws.data_ptr(), ws.numel(), 0, None)
    assert rc != 0 and b'batch limit' in lib.b200ocl_last_error()
    assert _native.launch_count() == before


# ----------------------------------------------------------------------------- drop-in runs against the reference
def _golden():
    return np.load(GOLDEN)


def _agent(params):
    from b200ocl import nets, registry
    name = params.agent
    cls = registry.agents.get(name) or registry.extra_agents[name]
    return cls(nets.setup_architecture(params), None, params)


@pytest.mark.parametrize('case', range(int(np.load(GOLDEN)['n_dropin'])))
def test_dropin_matches_reference_run(case):
    """test_gpu_dropin.py's comparison at 128x128 and 50 classes (agents with and without a memory)."""
    from b200ocl import memory
    from oracle import resnet as oresnet
    g = _golden()
    tag = 'c%d_' % case
    kind, n_calls, n_label, wseed, seed, dseed = json.loads(str(g[tag + 'case']))
    params = SimpleNamespace(**json.loads(str(g[tag + 'params'])))
    params.cuda = True
    spec = _spec()
    memory.set_mode(True, 'cpu')                    # the reference ran on the CPU: its draws came from CPU generators
    memory.ClassBalancedRandomSampling.reset()
    try:
        agent = _agent(params)
        p, bn = oresnet.seeded_state(spec, wseed)
        agent.engine.load(list(p.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
        w0 = torch.cat([t.reshape(-1) for t in p.values()]).numpy()
        pick = dropin.dropin_sample(w0.size)
        w0 = w0[pick].astype(np.float64)
        np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
        rs = np.random.RandomState(dseed)
        x, y, calls, tests = dropin.dropin_inputs(rs, params.mem_size, HW, n_label, params.batch, n_calls)
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
            print('core50 dropin %s call %d weight update rel %.3g (spread %.3g)' % (kind, c, err, g[tag + 'spread_w'][c]))
            assert err <= max(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_w'][c]), (where, 'sampled weight update', err)
            err = dropin._rel(agent.engine.state.bn_stats.cpu().numpy(), g[tag + 'bn%d' % c].astype(np.float64))
            assert err <= max(dropin.BN_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_bn'][c]), (where, 'BN running statistics', err)
        loaders = [[(torch.from_numpy(tx).permute(0, 3, 1, 2).float().div(255), torch.from_numpy(ty))] for tx, ty in tests]
        acc = np.asarray(agent.evaluate(loaders))
        assert np.abs(acc - g[tag + 'acc']).max() <= 3.1 / 96, (kind, case, acc, g[tag + 'acc'])
    finally:
        memory.set_mode(False)
        memory.ClassBalancedRandomSampling.reset()


@pytest.mark.parametrize('case', range(int(np.load(GOLDEN)['n_gdumb'])))
def test_gdumb_dropin_matches_reference_run(case, monkeypatch):
    """test_gpu_gdumb.py's drop-in comparison at 128x128: the re-initialisation drawn as the reference's
    setup_architecture('core50') draws it, the greedy memory, the trained weights and the accuracies."""
    from b200ocl import learners, memory, nets
    from oracle import gdumb as ogd
    g = _golden()
    tag = 'g%d_' % case
    n_calls, n_label, n_per_call, seed, dseed = json.loads(str(g[tag + 'case']))
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
        calls, tests = ogd.dropin_inputs(np.random.RandomState(dseed), HW, n_label, n_per_call, n_calls)
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
            print('core50 gdumb call %d weight update rel %.3g (spread %.3g)' % (c, err, g[tag + 'spread_w'][c]))
            assert err <= max(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_w'][c]), (where, err)
            err = dropin._rel(agent.engine.state.bn_stats.cpu().numpy(), g[tag + 'bn%d' % c].astype(np.float64))
            assert err <= max(dropin.BN_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_bn'][c]), (where, 'BN statistics', err)
        loaders = [[(torch.from_numpy(tx).permute(0, 3, 1, 2).float().div(255), torch.from_numpy(ty))] for tx, ty in tests]
        acc = np.asarray(agent.evaluate(loaders))
        assert np.abs(acc - g[tag + 'acc']).max() <= 3.1 / 96, (case, acc, g[tag + 'acc'])
    finally:
        memory.set_mode(False)
