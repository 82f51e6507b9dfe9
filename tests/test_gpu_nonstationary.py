"""The non-stationary new-instance tasks on the engine (--cl_type ni --ns_type noise|occlusion): float64 NHWC images in
[0, 1] (continuum/non_stationary.py:9-124) fed through b200ocl_stream_prepare_f64.
  * the kernel against the CPU's x[perm].transpose(0,3,1,2).float(), bit for bit (int32 views, so NaN payloads count):
    at 32x32, 84x84 and odd non-square sizes that would catch an H/W swap, n = 1 and a few hundred, with and without
    perm; every k / 255.0, signed zeros, infinities, NaNs, values past FLT_MAX, doubles that round to fp32 subnormals
    or to zero, and round-to-even ties;
  * one launch over more than 2^31 source bytes (12 700 images at 84x84), first, middle and last rows;
  * drop-in runs of ER, ER + MIR, ER + ASER, A-GEM, LwF, EWC++, SCR, iCaRL's first call (32x32) and ER, ER + ASER, SCR
    (84x84, float64 labels), and GDumb at both sizes, on streams oracle/nonstationary.py builds, against the
    reference's own runs (tests/golden/nonstationary.npz) with the bars of test_gpu_openloris.py;
  * iCaRL's refusal at the second call, before anything launches."""
import hashlib
import json
import os
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import test_gpu_dropin as dropin

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'nonstationary.npz')
NCLS = 100
N_TEST = 100


def _cpu(x, perm=None):
    t = torch.from_numpy(x if perm is None else x[perm])
    return t.permute(0, 3, 1, 2).float().contiguous()


def _same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ----------------------------------------------------------------------------- the kernel
@pytest.mark.parametrize('h,w', [(32, 32), (84, 84), (37, 19), (5, 83), (1, 1)])
@pytest.mark.parametrize('n,use_perm', [(1, False), (1, True), (301, False), (301, True), (64, True)])
def test_kernel_matches_cpu_conversion(h, w, n, use_perm):
    from b200ocl import ops
    rs = np.random.RandomState(h * 1000 + w * 10 + n)
    x = rs.rand(n, h, w, 3)
    x[rs.rand(n, h, w, 3) < 0.05] = 1.0
    perm = None
    if use_perm:
        perm = rs.randint(0, n, n) if n == 64 else rs.permutation(n)    # n = 64: repeats, as a gather may
    got = ops.stream_prepare(torch.from_numpy(x).cuda(), None if perm is None else torch.from_numpy(perm).cuda()).cpu()
    assert got.shape == (n, 3, h, w)
    assert _same_bits(got, _cpu(x, perm))


def _special_values():
    f32 = np.finfo(np.float32)
    v = [k / 255.0 for k in range(256)]
    v += [0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 1e39, -1e39, float(f32.max), 3.4028235677973366e38,
          3.4028234663852886e38 * (1 + 2.0 ** -25), 1.0 + 2.0 ** -24, 1.0 + 3 * 2.0 ** -24, -(1.0 + 2.0 ** -24),
          float(f32.tiny), float(f32.tiny) * (1 - 2.0 ** -30), 2.0 ** -140, -2.0 ** -140, 2.0 ** -149, 1.5 * 2.0 ** -149,
          2.0 ** -150, 1.0000001 * 2.0 ** -150, 2.5 * 2.0 ** -149, 5e-324, -5e-324, 1e-300, 1e300, 1.0 / 3.0]
    bits = np.array(v, dtype=np.float64).view(np.uint64)
    # NaNs with payloads: quiet and signalling, both signs, a payload only in the low bits
    nans = np.array([0x7ff8000000000001, 0xfff4000000000000, 0x7ff0000020000000, 0x7ff0000000000001,
                     0xfffabcdef1234567], dtype=np.uint64)
    return np.concatenate([bits, nans]).view(np.float64)


def test_kernel_special_values():
    """Every k / 255.0 and the special values, at every position of a pixel and of a 16-byte load."""
    from b200ocl import ops
    v = _special_values()
    n_px = 3 * len(v) + 1                      # odd pixel count: chunks start on both parities of a double2
    flat = np.resize(np.concatenate([v, np.roll(v, 1), np.roll(v, 2)]), 5 * n_px * 3)
    x = flat.reshape(5, n_px, 1, 3)
    got = ops.stream_prepare(torch.from_numpy(x).cuda()).cpu()
    ref = _cpu(x)
    assert _same_bits(got, ref)
    g = got.numpy()
    assert np.isnan(g).sum() == np.isnan(x).sum() and np.isinf(g).sum() > np.isinf(x).sum()
    assert ((g != 0) & (np.abs(g) < np.finfo(np.float32).tiny)).any()          # subnormals were kept
    for k in range(256):
        assert (g == np.float32(k / 255.0)).any()


def test_kernel_over_2gb_of_source():
    """12 700 images at 84x84: 2.15e9 source bytes, with a reversing perm so the last image is read first."""
    from b200ocl import ops
    n, hw = 12700, 84
    assert n * hw * hw * 3 * 8 > 2 ** 31
    gen = torch.Generator(device='cuda').manual_seed(7)
    x = torch.rand((n, hw, hw, 3), dtype=torch.float64, device='cuda', generator=gen)
    perm = torch.arange(n - 1, -1, -1, device='cuda')
    got = ops.stream_prepare(x, perm)
    ident = ops.stream_prepare(x)
    torch.cuda.synchronize()
    for i in (0, 1, n // 2, n - 2, n - 1):
        src = x[n - 1 - i:n - i].cpu().numpy()
        assert _same_bits(got[i:i + 1].cpu(), _cpu(src)), i
        assert _same_bits(ident[n - 1 - i:n - i].cpu(), _cpu(src)), i
    del x, got, ident
    torch.cuda.empty_cache()


def test_feeder_uploads_and_converts_on_the_device():
    """StreamFeeder on CUDA: one launch of the float64 kernel for the task, the same tensors as the CPU path."""
    from b200ocl import _native, memory
    from b200ocl.learners import StreamFeeder
    from oracle import nonstationary as ons
    rs = np.random.RandomState(4)
    np.random.seed(4)
    x = ons.noisy(rs.randint(0, 256, (53, 84, 84, 3)).astype(np.uint8), 1.2)
    y = rs.randint(0, 100, 53).astype(np.float64)
    memory.set_mode(True)
    try:
        torch.manual_seed(9)
        cpu = list(StreamFeeder(x, y, 10, 'cpu'))
        torch.manual_seed(9)
        before = _native.launch_count()
        dev = StreamFeeder(x, y, 10, 'cuda')
        torch.cuda.synchronize()
        assert _native.launch_count() == before + 1
    finally:
        memory.set_mode(False)
    for (cx, cy, _), (gx, gy, _) in zip(cpu, dev):
        assert _same_bits(gx.cpu(), cx) and torch.equal(gy.cpu(), cy)


def test_feeder_refuses_before_uploading():
    from b200ocl import _native
    from b200ocl.learners import StreamFeeder
    before = _native.launch_count()
    mem = torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match='float64'):
        StreamFeeder(np.zeros((4, 32, 32, 3), dtype=np.float32), np.arange(4), 2, 'cuda')
    assert _native.launch_count() == before and torch.cuda.memory_allocated() == mem


# ----------------------------------------------------------------------------- drop-in runs against the reference
def ns_inputs(rs, mem, hw, per_call, ns_type, factors, label_dtype):
    """tests/golden/make_golden_nonstationary.py ns_inputs() with oracle/nonstationary.py as the builder."""
    from oracle import nonstationary as ons
    x = rs.rand(mem, 3, hw, hw).astype(np.float32)
    y = rs.randint(0, NCLS, mem).astype(np.int64)
    n = len(factors)
    tr_x = [rs.randint(0, 256, (per_call, hw, hw, 3)).astype(np.uint8) for _ in range(n)]
    tr_y = [rs.permutation(np.arange(per_call) % NCLS).astype(label_dtype) for _ in range(n)]
    va_x = [rs.randint(0, 256, (1, hw, hw, 3)).astype(np.uint8) for _ in range(n)]
    va_y = [np.zeros(1, dtype=label_dtype) for _ in range(n)]
    te_x = [rs.randint(0, 256, (N_TEST, hw, hw, 3)).astype(np.uint8) for _ in range(n)]
    te_y = [rs.permutation(np.arange(N_TEST) % NCLS).astype(label_dtype) for _ in range(n)]
    train, _, test = ons.construct_ns_multiple(tr_x, tr_y, va_x, va_y, te_x, te_y, ns_type, factors)
    return x, y, train, test


def _inputs(params, hw, mem, per_call, ns_type, factors, dseed):
    np.random.seed(dseed); random.seed(dseed)
    return ns_inputs(np.random.RandomState(dseed), mem, hw, per_call, ns_type, factors,
                     np.float64 if params.data == 'mini_imagenet' else np.int64)


def _golden():
    return np.load(GOLDEN)


def _agent(params):
    from b200ocl import nets, registry
    name = params.agent
    cls = registry.agents.get(name) or registry.extra_agents[name]
    return cls(nets.setup_architecture(params), None, params)


def _loaders(tests):
    """setup_test_loader's batches: ToTensor on float64 HWC is a transpose, then .float()."""
    return [[(torch.from_numpy(tx).permute(0, 3, 1, 2).float(), torch.from_numpy(ty).long())] for tx, ty in tests]


@pytest.mark.parametrize('case', range(int(np.load(GOLDEN)['n_dropin'])))
def test_dropin_matches_reference_run(case):
    """test_gpu_openloris.py's comparison on float64 non-stationary calls with all 100 classes in each: the memory, the
    weight update, the BN statistics, old_labels with its repeats and the accuracies."""
    from b200ocl import memory
    from b200ocl.augment import Identity
    from oracle import resnet as oresnet
    g = _golden()
    tag = 'c%d_' % case
    kind, hw, ns_type, factors, per_call, wseed, seed, dseed = json.loads(str(g[tag + 'case']))
    n_calls = len(factors)
    params = SimpleNamespace(**json.loads(str(g[tag + 'params'])))
    params.cuda = True
    spec = oresnet.Spec(hw, 20, 100, head='mlp') if params.agent == 'SCR' else oresnet.Spec(hw, 20, NCLS)
    memory.set_mode(True, 'cpu')                    # the reference ran on the CPU: its draws came from CPU generators
    memory.ClassBalancedRandomSampling.reset()
    try:
        agent = _agent(params)
        assert agent.engine.in_hw == hw
        if hasattr(agent, 'transform'):
            agent.transform = Identity()            # the reference side ran kornia stubbed to the identity
        p, bn = oresnet.seeded_state(spec, wseed)
        agent.engine.load(list(p.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
        w0 = torch.cat([t.reshape(-1) for t in p.values()]).numpy()
        pick = dropin.dropin_sample(w0.size)
        w0 = w0[pick].astype(np.float64)
        x, y, calls, tests = _inputs(params, hw, params.mem_size, per_call, ns_type, factors, dseed)
        np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
        buf = getattr(agent, 'buffer', None)
        if buf is not None:
            dev = buf.buffer_img.device
            buf.update(torch.from_numpy(x).to(dev), torch.from_numpy(y).to(dev))
        for c, (xt, yt) in enumerate(calls):
            assert xt.dtype == np.float64 and c < n_calls
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
            print('nonstationary dropin %s %dx%d case %d call %d weight update rel %.3g (spread %.3g)'
                  % (kind, hw, hw, case, c, err, g[tag + 'spread_w'][c]))
            assert err <= max(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_w'][c]), (where, 'sampled weight update', err)
            err = dropin._rel(agent.engine.state.bn_stats.cpu().numpy(), g[tag + 'bn%d' % c].astype(np.float64))
            assert err <= max(dropin.BN_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_bn'][c]), (where, 'BN running statistics', err)
        assert agent.old_labels == g[tag + 'old_labels'].tolist()
        acc = np.asarray(agent.evaluate(_loaders(tests)))
        assert np.abs(acc - g[tag + 'acc']).max() <= 3.1 / N_TEST, (kind, case, acc, g[tag + 'acc'])
    finally:
        memory.set_mode(False)
        memory.ClassBalancedRandomSampling.reset()


@pytest.mark.parametrize('case', range(int(np.load(GOLDEN)['n_gdumb'])))
def test_gdumb_dropin_matches_reference_run(case, monkeypatch):
    """test_gpu_openloris.py's GDumb comparison on float64 non-stationary calls: the re-initialisation, the greedy
    memory balanced over 100 classes, the trained weights and the accuracies."""
    from b200ocl import learners, memory, nets
    g = _golden()
    tag = 'g%d_' % case
    hw, ns_type, factors, per_call, seed, dseed = json.loads(str(g[tag + 'case']))
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
        assert agent.engine.in_hw == hw
        _, _, calls, tests = _inputs(params, hw, 0, per_call, ns_type, factors, dseed)
        np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
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
            print('nonstationary gdumb %dx%d call %d weight update rel %.3g (spread %.3g)' % (hw, hw, c, err, g[tag + 'spread_w'][c]))
            assert err <= max(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_w'][c]), (where, err)
            err = dropin._rel(agent.engine.state.bn_stats.cpu().numpy(), g[tag + 'bn%d' % c].astype(np.float64))
            assert err <= max(dropin.BN_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_bn'][c]), (where, 'BN statistics', err)
        acc = np.asarray(agent.evaluate(_loaders(tests)))
        assert np.abs(acc - g[tag + 'acc']).max() <= 3.1 / N_TEST, (case, acc, g[tag + 'acc'])
    finally:
        memory.set_mode(False)


def test_icarl_refuses_the_second_call():
    """iCaRL trains its first non-stationary call; at the second, old_labels ++ new_labels holds 2 x 100 = 200 label
    positions for 100 logits (the reference fails at icarl.py:62).  The ValueError comes before anything launches."""
    from b200ocl import _native, memory
    g = _golden()
    case = [k for k in range(int(g['n_dropin'])) if json.loads(str(g['c%d_case' % k]))[0] == 'icarl'][0]
    params = SimpleNamespace(**json.loads(str(g['c%d_params' % case])))
    params.cuda = True
    memory.set_mode(True, 'cpu')
    try:
        agent = _agent(params)
        x, y, calls, _ = _inputs(params, 32, params.mem_size, params.batch + 3, 'noise', [0.6, 1.4], 3)
        agent.buffer.update(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda())
        agent.train_learner(*calls[0])
        torch.cuda.synchronize()
        before = _native.launch_count()
        with pytest.raises(ValueError, match='200 label positions exceed the 100 logits'):
            agent.train_learner(*calls[1])
        torch.cuda.synchronize()
        assert _native.launch_count() == before
    finally:
        memory.set_mode(False)
