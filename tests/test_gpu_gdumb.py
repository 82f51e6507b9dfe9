"""GPU: the GDumb agent on the engine.
  * b200ocl_net_sgd_step_clipped: the norm within 1e-6 of an fp64 norm; clipped gradients and weights within a few ulp
    of torch.nn.utils.clip_grad_norm_ followed by torch.optim.SGD on copies; below the threshold the arenas are
    bit-identical to b200ocl_net_sgd_step; a zero gradient stays zero; the tensors without a gradient (the unused
    classifier of the SupCon network) are left out of the norm and untouched; repeat launches are bit-identical;
  * the clipped gradient is g times torch's own coefficient bit for bit, given the kernel's norm;
  * steps of the inner loop from a common state, and train_mem() itself step by step (its re-initialisation, the
    cumulative permutation, the batch rows, step size, weight decay and clip), against the CPU oracle (oracle/gdumb.py)
    within the replay path's 1e-3 bar (train_mem's weight update: 1e-3 at most steps, 3e-2 at every step);
  * drop-in runs against the reference's (tests/golden/gdumb.npz): mem_c and the memory rows in train_mem's order
    exactly, the re-initialised weights bit for bit, the weight update and BN statistics within the larger of the fp32
    bar and 10x the reference's own one-ulp spread, the accuracies within 3 of 96 test samples;
  * two seeded train_learner sequences are bit-identical; an empty memory and data-parallel gradient sync are refused."""
import hashlib
import json
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import gdumb as ogd
from oracle import resnet as oresnet

import test_gpu_dropin as dropin
from test_oracle_gdumb import GOLDEN, _params

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -23


def _engine(head=None, seed=5):
    from b200ocl import nets
    model = nets.EngineModel(32, 100, head=head)
    eng = model.engine
    rs = np.random.RandomState(seed)
    eng.state.params.copy_(torch.from_numpy(rs.standard_normal(eng.state.params.numel()).astype(np.float32) * 0.1))
    eng.state.grads.copy_(torch.from_numpy(rs.standard_normal(eng.state.grads.numel()).astype(np.float32) * 0.01))
    eng.pack()
    return model, eng


def _torch_step(eng, lr, wd, max_norm):
    """clip_grad_norm_ + torch.optim.SGD on copies of the arenas: (norm, grads, params) as flat arrays."""
    ps = []
    for (o, n, has_grad), pv, gv in zip(eng.table, eng.param_views(), eng.grad_views()):
        p = torch.nn.Parameter(pv.clone())
        p.grad = gv.clone() if has_grad else None
        ps.append(p)
    norm = torch.nn.utils.clip_grad_norm_(ps, max_norm)
    torch.optim.SGD(ps, lr=lr, weight_decay=wd).step()
    g = torch.cat([p.grad if p.grad is not None else gv for p, gv in zip(ps, eng.grad_views())])
    return float(norm), g.cpu().numpy(), torch.cat([p.detach() for p in ps]).cpu().numpy()


@pytest.mark.parametrize('head', [None, 'mlp'])
@pytest.mark.parametrize('max_norm', [0.05, 1.0])
def test_clipped_step_matches_clip_grad_norm_and_sgd(head, max_norm):
    _, eng = _engine(head)
    lr, wd = 0.1, 1e-4
    g0, p0 = eng.state.grads.cpu().numpy(), eng.state.params.cpu().numpy()
    has = np.zeros(g0.size, dtype=bool)
    for o, n, hg in eng.table:
        has[o:o + n] = hg
    t_norm, t_g, t_p = _torch_step(eng, lr, wd, max_norm)
    norm = float(eng.sgd_step_clipped(lr, wd, max_norm))
    g, p = eng.state.grads.cpu().numpy(), eng.state.params.cpu().numpy()
    exact = float(np.sqrt(np.sum(g0[has].astype(np.float64) ** 2)))
    assert abs(norm - exact) <= 1e-6 * exact, (norm, exact)
    assert abs(norm - t_norm) <= 1e-5 * exact
    assert max_norm < exact                                       # both cases clip
    assert np.abs(g - t_g).max() <= 8 * EPS32 * np.abs(t_g).max()
    scale = np.abs(p0) + lr * np.abs(t_g) + lr * wd * np.abs(p0)
    assert (np.abs(p - t_p) <= 4 * EPS32 * scale + 1e-30).all(), np.abs(p - t_p).max()
    if head is not None:                                          # the unused classifier: no gradient, not in the norm
        assert np.array_equal(g[~has], g0[~has]) and np.array_equal(p[~has], p0[~has])
    packed = eng.state.packed.clone()
    eng.pack()
    assert torch.equal(packed, eng.state.packed)                  # the step refreshed the packed weights


@pytest.mark.parametrize('max_norm', [0.05, 0.3, 1.0, 3.0, 10.0])
def test_clipped_gradient_uses_torchs_coefficient_exactly(max_norm):
    """Given the kernel's norm, the clipped gradient is g * coef bit for bit, with coef formed by torch's own expression
    clamp(max_norm / (norm + 1e-6), max=1) (the division is a reciprocal and a product: two roundings)."""
    _, eng = _engine(seed=9)
    eng.state.grads.mul_(100.0)                                   # norm ~ 1000: every max_norm here clips
    g0 = eng.state.grads.cpu()
    norm = eng.sgd_step_clipped(0.1, 0.0, max_norm).cpu()
    coef = torch.clamp(max_norm / (norm + 1e-6), max=1.0)
    assert float(coef) < 1.0
    assert torch.equal(eng.state.grads.cpu(), g0 * coef)


def test_clipped_step_below_the_threshold_is_the_plain_step():
    _, a = _engine(seed=6)
    _, b = _engine(seed=6)
    a.sgd_step_clipped(0.1, 1e-4, 1e6)
    b.sgd_step(0.1, 1e-4)
    for name in ('params', 'grads', 'packed', 'bn_stats'):
        assert torch.equal(getattr(a.state, name), getattr(b.state, name)), name


def test_clipped_step_with_a_zero_gradient():
    _, eng = _engine(seed=7)
    eng.state.grads.zero_()
    p0 = eng.state.params.clone()
    norm = eng.sgd_step_clipped(0.1, 0.0, 1.0)
    assert float(norm) == 0.0
    assert not eng.state.grads.any()
    assert torch.equal(eng.state.params, p0)


def test_clipped_step_repeat_launches_are_bit_identical():
    out = []
    for _ in range(2):
        _, eng = _engine(seed=8)
        norms = [eng.sgd_step_clipped(0.1, 1e-4, 0.5).clone() for _ in range(3)]
        out.append((torch.cat(norms), eng.state.params.clone(), eng.state.grads.clone()))
    for u, v in zip(*out):
        assert torch.equal(u, v)


def test_clipped_step_refuses_a_state_without_gradients():
    import ctypes
    from b200ocl import _native
    from b200ocl.engine import ArenaState
    _, eng = _engine()
    st = ArenaState(eng.info, eng.device, with_grads=False)
    ws = torch.empty(1 << 16, dtype=torch.uint8, device='cuda')
    lib = _native.lib()
    rc = lib.b200ocl_net_sgd_step_clipped(ctypes.byref(eng.desc), ctypes.byref(st.c), 0.1, 0.0, 1.0, None,
                                          ws.data_ptr(), ws.numel(), None)
    assert rc != 0
    rc = lib.b200ocl_net_sgd_step_clipped(ctypes.byref(eng.desc), ctypes.byref(eng.state.c), 0.1, 0.0, 1.0, None,
                                          ws.data_ptr(), 8, None)
    assert rc != 0                                                # workspace too small


def test_train_mem_steps_match_the_oracle():
    """Steps of train_mem's inner loop (forward, CE, backward, clip, SGD) from a common state: every step starts from the
    oracle's weights and statistics, as test_gpu_replay does."""
    from b200ocl import nets
    from b200ocl.engine import ce_loss
    spec = oresnet.Spec(32, 20, 100)
    p, bn = oresnet.seeded_state(spec, 21)
    eng = nets.Reduced_ResNet18(100).engine
    rs = np.random.RandomState(22)
    clipped = 0
    for i in range(4):
        eng.load(list(p.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
        x = torch.from_numpy(rs.randint(0, 256, (10, 3, 32, 32)).astype(np.float32) / 255.0)
        y = torch.from_numpy(rs.randint(0, 100, 10))
        logits, ws = eng.forward_train(x.cuda())
        out = ce_loss(logits, y.cuda())
        eng.backward(x.cuda(), out['dlogits'], ws)
        norm = float(eng.sgd_step_clipped(0.05, 1e-4, 2.0))
        loss, o_norm = ogd.train_mem_step(spec, p, bn, x, y, 0.05, 1e-4, 2.0)
        clipped += o_norm > 2.0
        assert abs(float(out['loss']) - loss) <= 1e-3 * abs(loss), (i, float(out['loss']), loss)
        assert abs(norm - o_norm) <= 1e-3 * o_norm, (i, norm, o_norm)
        flat = torch.cat([v.reshape(-1) for v in p.values()])
        assert float((eng.state.params.cpu() - flat).abs().max() / flat.abs().max()) < 1e-3, i
        stats = torch.cat([torch.cat([bn[n + '.running_mean'], bn[n + '.running_var']]) for n in oresnet.bn_names(spec)])
        assert float((eng.state.bn_stats.cpu() - stats).abs().max() / stats.abs().max()) < 1e-3, i
    assert clipped > 0


def _gdumb(params):
    from b200ocl import nets, registry
    return registry.agents['GDUMB'](nets.setup_architecture(params), None, params)


def test_train_mem_follows_the_oracle_step_by_step(monkeypatch):
    """train_mem() itself against the oracle (gdumb.py:52-83 restated on oracle.resnet): the re-initialisation drawn from
    the same torch seed, the memory rows in the same cumulative np.random.permutation order (45 rows: 4 batches of 10
    per epoch, the last 5 rows dropped), step size, weight decay and clip from params.  After every step of the learner
    the oracle takes the same step and the engine is then loaded with the oracle's state, so that each step is compared
    from a common state.  The norm and the BN statistics must agree within 1e-3 at every step.  The weight update must
    agree within 1e-3 at most steps and within 3e-2 at every step: with batches of 10 through a from-scratch network,
    a step now and then has pre-activations at a ReLU's kink, where the last bits decide the gradient path; at such
    steps fp32 results land up to ~1e-2 apart (the fp32 oracle lands 5e-3 from the same step in fp64).  Dropping the
    weight decay (1e-3 here) moves every update by 9e-2; a wrong batch, order, step size or clip moves it by 1 or more."""
    from b200ocl import nets
    lr, wd, clip, n_epoch = 0.05, 1e-3, 0.5, 2
    agent = _gdumb(_params(mem_size=45, mem_epoch=n_epoch, learning_rate=lr, weight_decay=wd, clip=clip))
    eng = agent.engine
    rs = np.random.RandomState(31)
    y = rs.permutation(np.arange(60) % 5)                          # 12 per class: 9 of each stay, 15 are evicted
    agent.before_train(None, y)
    random.seed(32)
    slots, sources = agent.memory.plan(y)
    agent.memory.write(torch.from_numpy(rs.rand(60, 3, 32, 32).astype(np.float32)).cuda(), y, slots, sources)
    order = torch.from_numpy(agent.memory.order()).cuda()
    rows, labels = agent.memory.images[order].cpu(), agent.memory.labels[order].cpu()
    n = rows.shape[0]
    assert n == 45 and len(set(labels.tolist())) == 5

    spec = oresnet.Spec(32, 20, 100)
    np.random.seed(33)
    perms = [np.random.permutation(n) for _ in range(n_epoch)]
    torch.manual_seed(34)
    P = dict(zip(oresnet.param_shapes(spec), nets.reference_init('cifar100', 100, 32)))
    BN = {}
    for name in oresnet.bn_names(spec):
        c = P[name + '.weight'].shape[0]
        BN.update({name + '.running_mean': torch.zeros(c), name + '.running_var': torch.ones(c),
                   name + '.num_batches_tracked': torch.zeros((), dtype=torch.long)})

    def flat_p():
        return torch.cat([v.reshape(-1) for v in P.values()]).double().numpy()

    def flat_bn():
        return torch.cat([torch.cat([BN[m + '.running_mean'], BN[m + '.running_var']]) for m in oresnet.bn_names(spec)])

    steps = n // agent.batch
    state = {'k': 0, 'rows': rows, 'labels': labels, 'clipped': 0, 'errs': []}
    learner_step = eng.sgd_step_clipped

    def step(lr_, wd_, max_norm):
        w0 = flat_p()
        assert np.array_equal(eng.state.params.cpu().double().numpy(), w0), state['k']   # the same state before the step
        norm = float(learner_step(lr_, wd_, max_norm))
        e, j = divmod(state['k'], steps)
        if j == 0:                                                    # gdumb.py:67-69, once per epoch, cumulative
            state['rows'], state['labels'] = state['rows'][perms[e]], state['labels'][perms[e]]
        bx, by = state['rows'][j * 10:(j + 1) * 10], state['labels'][j * 10:(j + 1) * 10]
        _, o_norm = ogd.train_mem_step(spec, P, BN, bx, by, lr, wd, clip)
        where = 'epoch %d step %d' % (e, j)
        assert abs(norm - o_norm) <= 1e-3 * o_norm, (where, norm, o_norm)
        err = dropin._rel(eng.state.params.cpu().numpy() - w0, flat_p() - w0)
        state['errs'].append(err)
        assert err <= 3e-2, (where, 'weight update', err)
        stats = flat_bn()
        assert float((eng.state.bn_stats.cpu() - stats).abs().max() / stats.abs().max()) <= 1e-3, where
        state['clipped'] += o_norm > clip
        state['k'] += 1
        eng.load(list(P.values()), [(BN[m + '.running_mean'], BN[m + '.running_var']) for m in oresnet.bn_names(spec)])
        return norm

    monkeypatch.setattr(eng, 'sgd_step_clipped', step)
    np.random.seed(33)
    torch.manual_seed(34)
    agent.train_mem()
    torch.cuda.synchronize()
    assert state['k'] == n_epoch * steps
    assert state['clipped'] > 0
    assert sum(e <= 1e-3 for e in state['errs']) > len(state['errs']) // 2, state['errs']   # most steps within 1e-3


def _task(rs, n, labels):
    return rs.randint(0, 256, (n, 32, 32, 3)).astype(np.uint8), np.asarray(labels, dtype=np.int64)[rs.permutation(n) % len(labels)]


def test_gdumb_whole_calls_are_deterministic():
    def run():
        agent = _gdumb(_params(mem_size=60, mem_epoch=2))
        np.random.seed(1); random.seed(1); torch.manual_seed(1)
        rs = np.random.RandomState(2)
        for t in range(2):
            agent.train_learner(*_task(rs, 45, range(5 * t, 5 * t + 5)))
        torch.cuda.synchronize()
        eng = agent.engine
        order = torch.from_numpy(agent.memory.order()).cuda()
        return (list(agent.mem_c.items()), [eng.state.params.clone(), eng.state.grads.clone(), eng.state.bn_stats.clone(),
                                            eng.state.bn_tracked.clone(), agent.memory.images[order].clone(),
                                            agent.memory.labels[order].clone(), agent.last_loss.clone()])
    a, ta = run()
    b, tb = run()
    assert a == b
    for u, v in zip(ta, tb):
        assert torch.equal(u, v)


def test_gdumb_refuses_an_empty_memory_and_grad_sync():
    agent = _gdumb(_params())
    rs = np.random.RandomState(3)
    with pytest.raises(RuntimeError, match='empty'):
        agent.train_learner(*_task(rs, 7, range(3)))            # fewer samples than one batch: nothing enters
    agent = _gdumb(_params())
    agent.grad_sync = lambda eng: None
    with pytest.raises(NotImplementedError, match='data-parallel'):
        agent.train_learner(*_task(rs, 20, range(3)))


@pytest.mark.parametrize('case', range(int(np.load(GOLDEN)['n_dropin'])))
def test_gdumb_dropin_matches_reference_run(case, monkeypatch):
    from b200ocl import learners, memory, nets
    g = np.load(GOLDEN)
    tag = 'c%d_' % case
    n_calls, n_label, n_per_call, seed, dseed = json.loads(str(g[tag + 'case']))
    params = SimpleNamespace(**json.loads(str(g[tag + 'params'])))
    params.cuda = True
    hw = 84 if params.data == 'mini_imagenet' else 32
    inits = []
    orig = nets.reference_init

    def reference_init(*a):
        ps = orig(*a)
        inits.append(torch.cat([t.reshape(-1) for t in ps]).numpy())
        return ps
    monkeypatch.setattr(learners.nets, 'reference_init', reference_init)
    memory.set_mode(True, 'cpu')                    # the reference ran on the CPU: its draws came from CPU generators
    try:
        agent = _gdumb(params)
        np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
        calls, tests = ogd.dropin_inputs(np.random.RandomState(dseed), hw, n_label, n_per_call, n_calls)
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
            assert err <= max(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_w'][c]), \
                (where, 'sampled weight update', err, 'one-ulp spread', g[tag + 'spread_w'][c])
            err = dropin._rel(agent.engine.state.bn_stats.cpu().numpy(), g[tag + 'bn%d' % c].astype(np.float64))
            assert err <= max(dropin.BN_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_bn'][c]), (where, 'BN statistics', err)
        loaders = [[(torch.from_numpy(tx).permute(0, 3, 1, 2).float().div(255), torch.from_numpy(ty))] for tx, ty in tests]
        acc = np.asarray(agent.evaluate(loaders))
        assert np.abs(acc - g[tag + 'acc']).max() <= 3.1 / 96, (case, acc, g[tag + 'acc'])   # <= 3 of 96 samples
    finally:
        memory.set_mode(False)
