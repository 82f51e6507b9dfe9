"""GPU: torch.optim.Adam on the engine.
  * b200ocl_adam_step against torch.optim.Adam on the same device, bit for bit, for torch's default multi-tensor path
    and for foreach=False: n in {1, 255, 257, 1 000 003}, weight decay 0 / 5e-4, several lr / betas / eps, up to 50
    consecutive steps with state carried, gradients with zeros, subnormals and values near 1e30; the review trick's
    p.grad.clone() / 10. before the step;
  * b200ocl_net_adam_step against torch's Adam over the network's own tensors (the SupCon network: the unused
    classifier untouched in all four arenas), the packed weights (eval features equal a fresh engine's loaded with the
    stepped weights), and the EWC++ step under Adam against the reference's op sequence in torch;
  * drop-in runs of the agents with optimizer='Adam' against the reference's (tests/golden/adam.npz) under the
    comparison of test_gpu_dropin.py;
  * opt.state after train_learner (torch's keys, shapes, dtypes and step) and a state_dict round trip into a fresh
    optimizer and engine, bit-identical to running straight through; determinism; launches per step."""
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

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'adam.npz')


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _grad(gen, n, dev='cuda'):
    """A gradient with zeros, subnormals and values near +-1e30 among normal ones."""
    g = torch.randn(n, generator=gen, device=dev) * 0.05
    g[::13] = 0.0
    g[5::17] = torch.rand(g[5::17].shape, generator=gen, device=dev) * 1e-40        # subnormal
    g[7::101] = (torch.rand(g[7::101].shape, generator=gen, device=dev) - 0.5) * 4e30
    return g


HYPER = [   # (lr, betas, eps)
    (1e-3, (0.9, 0.999), 1e-8),
    (3e-4, (0.8, 0.99), 1e-6),
    (1e-2, (0.5, 0.9), 1e-3),      # lerp weight 0.5: Lerp.h's second branch
]


@pytest.mark.parametrize('foreach', [None, False])
@pytest.mark.parametrize('wd', [0.0, 5e-4])
@pytest.mark.parametrize('n', [1, 255, 257, 1000003])
def test_flat_step_matches_torch(n, wd, foreach):
    from b200ocl import ops
    steps = 50 if n < 1000 else 4
    for h, (lr, betas, eps) in enumerate(HYPER):
        gen = torch.Generator(device='cuda').manual_seed(1000 * h + n)
        p0 = torch.randn(n, generator=gen, device='cuda') * 0.1
        ref = torch.nn.Parameter(p0.clone())
        opt = torch.optim.Adam([ref], lr=lr, betas=betas, eps=eps, weight_decay=wd, foreach=foreach)
        p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
        for s in range(1, steps + 1):
            g = _grad(gen, n)
            ref.grad = g.clone()
            opt.step()
            ops.adam_step(p, g, m, v, s, lr, betas, eps, wd, foreach=foreach is not False)
            st = opt.state[ref]
            where = (n, wd, foreach, h, s)
            assert _same(p, ref.detach()), where
            assert _same(m, st['exp_avg']), where
            assert _same(v, st['exp_avg_sq']), where


@pytest.mark.parametrize('foreach', [None, False])
def test_flat_review_prescale_matches_torch(foreach):
    """agents/base.py:84-87: grad = p.grad.clone() / 10., p.grad.data.copy_(grad), opt.step()."""
    from b200ocl import ops
    n = 4099
    gen = torch.Generator(device='cuda').manual_seed(3)
    p0 = torch.randn(n, generator=gen, device='cuda') * 0.1
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([ref], lr=1e-3, weight_decay=5e-4, foreach=foreach)
    p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    for s in range(1, 8):
        g = _grad(gen, n)
        ref.grad = g.clone()
        ref.grad.data.copy_(ref.grad.clone() / 10.)
        opt.step()
        ops.adam_step(p, g, m, v, s, 1e-3, weight_decay=5e-4, foreach=foreach is not False, grad_div=10.0)
        assert _same(g, ref.grad), s                      # the scaled gradient is written back
        assert _same(p, ref.detach()) and _same(m, opt.state[ref]['exp_avg']), s
        assert _same(v, opt.state[ref]['exp_avg_sq']), s


def _engine(head=None, seed=5):
    from b200ocl import nets
    eng = nets.EngineModel(32, 100, head=head).engine
    rs = np.random.RandomState(seed)
    n = eng.state.params.numel()
    eng.state.params.copy_(torch.from_numpy((rs.standard_normal(n) * 0.1).astype(np.float32)).cuda())
    eng.pack()
    return eng


def _has_grad(eng):
    has = torch.zeros(eng.state.params.numel(), dtype=torch.bool, device='cuda')
    for o, n, hg in eng.table:
        has[o:o + n] = hg
    return has


@pytest.mark.parametrize('head', [None, 'mlp'])
@pytest.mark.parametrize('foreach', [None, False])
def test_net_step_matches_torch_over_the_network_tensors(head, foreach):
    """torch.optim.Adam over the network's tensors that have a gradient (the others have .grad None, so torch makes no
    state for them) against b200ocl_net_adam_step, three steps with new gradients, weight decay on."""
    eng = _engine(head)
    has = _has_grad(eng)
    st = eng.adam_state()
    before = {'params': eng.state.params.clone(), 'm': st.exp_avg.clone(), 'v': st.exp_avg_sq.clone()}
    sentinel = torch.full_like(st.exp_avg, 7.0)
    st.exp_avg.copy_(sentinel), st.exp_avg_sq.copy_(sentinel)    # the skip range must keep whatever it holds
    for o, n, hg in eng.table:
        if hg:
            st.exp_avg[o:o + n].zero_(), st.exp_avg_sq[o:o + n].zero_()
    ref = [torch.nn.Parameter(eng.state.params[o:o + n].clone()) for o, n, hg in eng.table if hg]
    opt = torch.optim.Adam(ref, lr=1e-3, weight_decay=5e-4, foreach=foreach)
    gen = torch.Generator(device='cuda').manual_seed(11)
    for s in range(3):
        g = torch.randn(eng.state.grads.shape, generator=gen, device='cuda') * 0.01
        g[~has] = 123.0
        eng.state.grads.copy_(g)
        for q, (o, n) in zip(ref, [(o, n) for o, n, hg in eng.table if hg]):
            q.grad = g[o:o + n].clone()
        opt.step()
        eng.adam_step(1e-3, weight_decay=5e-4, foreach=foreach is not False)
    want = torch.cat([q.detach() for q in ref])
    assert _same(eng.state.params[has], want)
    assert _same(st.exp_avg[has], torch.cat([opt.state[q]['exp_avg'] for q in ref]))
    assert _same(st.exp_avg_sq[has], torch.cat([opt.state[q]['exp_avg_sq'] for q in ref]))
    assert st.step == 3
    assert torch.equal(eng.state.params[~has], before['params'][~has])
    assert torch.equal(st.exp_avg[~has], sentinel[~has]) and torch.equal(st.exp_avg_sq[~has], sentinel[~has])
    assert bool((eng.state.grads[~has] == 123.0).all())
    if head == 'mlp':
        assert (~has).any()
    # the packed weights follow: eval features equal a fresh engine's loaded with the stepped weights
    fresh = _engine(head, seed=99)
    fresh.state.params.copy_(eng.state.params)
    fresh.state.bn_stats.copy_(eng.state.bn_stats)
    fresh.pack()
    x = torch.rand(8, 3, 32, 32, generator=gen, device='cuda')
    assert torch.equal(eng.features_eval(x), fresh.features_eval(x))


@pytest.mark.parametrize('name', ['plain', 'both', 'kd_chain', 'mlp'])
def test_ewc_adam_step_matches_torch(name):
    """The EWC++ step under Adam: the reference's sequence (EMA, loss with the penalty, backward, accum_fisher, then
    opt.step() of torch.optim.Adam) run in torch on the device against b200ocl_net_adam_step_ewc."""
    import test_gpu_ewc as tewc
    from b200ocl import learners
    head, lam, t, kdt, kds, penalty, ema, zero = tewc.CASES[name]
    alpha, fua, lr, wd = 0.9, 50, 1e-3, 1e-4
    eng = tewc._engine(head, zero_grad=zero)
    st, ad = eng.ewc_state(), eng.adam_state()
    has = tewc._has_grad(eng)
    g_t, tmp_t, run_t = tewc._torch_step(eng, lam, t, kdt, kds, penalty, ema, alpha, fua)
    if kdt or kds:
        eng.state.grads.copy_(tewc._ce_part(eng, t, kdt, kds))
    stepped = [(o, n) for o, n, hg in eng.table if hg]
    ref = [torch.nn.Parameter(eng.state.params[o:o + n].clone()) for o, n in stepped]
    for q, (o, n) in zip(ref, stepped):
        q.grad = g_t[o:o + n].clone()
    opt = torch.optim.Adam(ref, lr=lr, weight_decay=wd)
    opt.step()
    up = learners.ewc_penalty_up(lam, t, kdt, kds)
    keep, add = learners.ewc_ema_coefficients(alpha, fua)
    p_before = eng.state.params.clone()
    eng.adam_step_ewc(lr, (0.9, 0.999), 1e-8, wd, True, up, penalty, ema, keep, add)
    assert torch.equal(eng.state.grads[has], g_t[has]), name
    assert torch.equal(st.tmp[has], tmp_t[has]) and torch.equal(st.running[has], run_t[has]), name
    assert _same(eng.state.params[has], torch.cat([q.detach() for q in ref])), name
    assert _same(ad.exp_avg[has], torch.cat([opt.state[q]['exp_avg'] for q in ref])), name
    assert _same(ad.exp_avg_sq[has], torch.cat([opt.state[q]['exp_avg_sq'] for q in ref])), name
    assert torch.equal(eng.state.params[~has], p_before[~has])
    assert not ad.exp_avg[~has].any() and not ad.exp_avg_sq[~has].any()


def test_launches_per_step_equal_sgd():
    import test_gpu_ewc as tewc
    from b200ocl import _native
    eng = tewc._engine()
    counts = {}
    for name, fn in (('sgd', lambda: eng.sgd_step(0.05)), ('adam', lambda: eng.adam_step(1e-3)),
                     ('adam_review', lambda: eng.adam_step(1e-3, grad_div=10.0)),
                     ('sgd_ewc', lambda: eng.sgd_step_ewc(0.05, 0.0, 100.0, True, True, 0.1, 0.018)),
                     ('adam_ewc', lambda: eng.adam_step_ewc(1e-3, (0.9, 0.999), 1e-8, 0.0, True, 100.0, True, True,
                                                            0.1, 0.018))):
        n0 = _native.launch_count()
        fn()
        counts[name] = _native.launch_count() - n0
    assert counts['adam'] == counts['adam_review'] == counts['sgd'], counts          # the update, then the repack
    assert counts['adam_ewc'] == counts['sgd_ewc'], counts                              # one fused launch, as under SGD


def _er_params(**over):
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick',
                                'kd_trick_star')}
    base = dict(data='cifar10', cuda=True, epoch=1, batch=10, verbose=False, mem_size=40, eps_mem_batch=10,
                mem_iters=1, update='random', retrieve='random', agent='ER', k=3, aser_type='asvm', n_smp_cls=1.5,
                num_tasks=5, buffer_tracker=False, optimizer='Adam', learning_rate=1e-3, weight_decay=0, temp=0.07,
                head='mlp', subsample=20, error_analysis=False, trick=trick)
    base.update(over)
    return SimpleNamespace(**base)


def _task(rs, n, labels):
    return rs.randint(0, 256, (n, 32, 32, 3)).astype(np.uint8), np.asarray(labels, dtype=np.int64)[rs.permutation(n) % len(labels)]


def _er(params, opt_kw=None, seed=1):
    from b200ocl import nets, registry
    np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
    model = nets.setup_architecture(params)
    opt = torch.optim.Adam(model.parameters(), **opt_kw) if opt_kw is not None else None
    return registry.agents[params.agent](model, opt, params), opt


def _call(agent, rs_seed, c):
    np.random.seed(50 + c); random.seed(50 + c); torch.manual_seed(50 + c)
    rs = np.random.RandomState(rs_seed + c)
    agent.train_learner(*_task(rs, 33, range(5 * c, 5 * c + 5)))
    torch.cuda.synchronize()


def test_state_dict_after_a_run_and_round_trip():
    params = _er_params()
    kw = dict(lr=1e-3, weight_decay=5e-4)
    a, opt_a = _er(params, kw)
    _call(a, 7, 0)
    sd = opt_a.state_dict()
    stepped = [q for q, (_, _, hg) in zip(a.model.parameters(), a.engine.table) if hg]
    assert len(sd['state']) == len(stepped) == len(list(a.model.parameters()))
    n_steps = 3                                                     # 33 samples, batches of 10, drop_last
    for q in stepped:
        s = opt_a.state[q]
        assert set(s) == {'step', 'exp_avg', 'exp_avg_sq'}
        assert s['step'].dtype == torch.float32 and s['step'].device.type == 'cpu' and float(s['step']) == n_steps
        assert s['exp_avg'].shape == q.shape and s['exp_avg'].dtype == torch.float32 and s['exp_avg'].is_cuda
        assert s['exp_avg_sq'].shape == q.shape
    assert a.engine.adam_state().step == n_steps
    # straight through: a second call on the same learner
    _call(a, 7, 1)
    # round trip: a fresh engine and optimizer loaded with the first call's weights, statistics and state
    b, opt_b = _er(params, kw, seed=2)
    b1, opt_b1 = _er(params, kw)
    _call(b1, 7, 0)
    b.engine.load(list(b1.engine.param_views()), [(m.clone(), v.clone()) for m, v in b1.engine.bn_views()])
    opt_b.load_state_dict(opt_b1.state_dict())
    b.buffer, b.old_labels, b.task_seen = b1.buffer, list(b1.old_labels), b1.task_seen
    b.lbl_inv_map, b.class_task_map = dict(b1.lbl_inv_map), dict(b1.class_task_map)
    _call(b, 7, 1)
    assert torch.equal(a.engine.state.params, b.engine.state.params)
    assert torch.equal(a.engine.adam_state().exp_avg, b.engine.adam_state().exp_avg)
    assert torch.equal(a.engine.adam_state().exp_avg_sq, b.engine.adam_state().exp_avg_sq)
    assert float(opt_b.state[next(iter(b.model.parameters()))]['step']) == 2 * n_steps


def test_whole_runs_are_deterministic_and_follow_lr_changes():
    def run(lr_change):
        a, opt = _er(_er_params(agent='SCR', mem_size=60, eps_mem_batch=20), dict(lr=1e-3))
        for c in range(3):
            if lr_change and c == 2:
                opt.param_groups[0]['lr'] = 5e-4
            _call(a, 3, c)
        return a.engine.state.params.clone(), a.engine.adam_state().exp_avg.clone()
    u, v = run(False), run(False)
    assert all(torch.equal(x, y) for x, y in zip(u, v))
    w = run(True)
    assert not torch.equal(u[0], w[0])                                # the changed lr is followed


def test_opt_none_follows_params_optimizer_and_grad_sync_is_refused():
    a, _ = _er(_er_params())
    _call(a, 5, 0)
    assert a.engine.adam_state().step == 3
    assert a.engine.adam_state().exp_avg_sq.any()
    s, _ = _er(_er_params(optimizer='SGD'))
    _call(s, 5, 0)
    assert getattr(s.engine, '_adam', None) is None                   # SGD never allocates Adam state
    a.grad_sync = lambda eng: None
    with pytest.raises(NotImplementedError, match='data-parallel'):
        _call(a, 5, 1)


def _dropin_cases():
    return range(int(np.load(GOLDEN)['n_dropin']))


@pytest.mark.parametrize('case', _dropin_cases())
def test_adam_dropin_matches_reference_run(case):
    from b200ocl import memory, nets, registry
    from b200ocl.augment import Identity
    from oracle import resnet as oresnet
    g = np.load(GOLDEN)
    tag = 'c%d_' % case
    kind, n_calls, n_label, wseed, seed, dseed = json.loads(str(g[tag + 'case']))
    params = SimpleNamespace(**json.loads(str(g[tag + 'params'])))
    params.cuda = True
    hw = 84 if params.data == 'mini_imagenet' else 32
    spec = oresnet.Spec(hw, 20, 10 if params.data == 'cifar10' else 100, head='mlp' if params.agent == 'SCR' else None)
    memory.set_mode(True, 'cpu')
    memory.ClassBalancedRandomSampling.reset()
    try:
        cls = registry.agents[params.agent] if params.agent != 'EWC' else registry.extra_agents['EWC']
        agent = cls(nets.setup_architecture(params), None, params)
        if hasattr(agent, 'transform'):
            agent.transform = Identity()
        p, bn = oresnet.seeded_state(spec, wseed)
        agent.engine.load(list(p.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
        w0 = torch.cat([t.reshape(-1) for t in p.values()]).numpy()
        pick = dropin.dropin_sample(w0.size)
        w0 = w0[pick].astype(np.float64)
        np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
        rs = np.random.RandomState(dseed)
        x, y, calls, tests = dropin.dropin_inputs(rs, params.mem_size, hw, n_label, params.batch, n_calls)
        has_buffer = hasattr(agent, 'buffer')
        if has_buffer:
            dev = agent.buffer.buffer_img.device
            agent.buffer.update(torch.from_numpy(x).to(dev), torch.from_numpy(y).to(dev))
        for c, (xt, yt) in enumerate(calls):
            where = '%s case %d call %d' % (kind, case, c)
            agent.train_learner(xt, yt)
            torch.cuda.synchronize()
            if has_buffer:
                buf = agent.buffer
                assert buf.current_index == int(g[tag + 'index%d' % c]) and buf.n_seen_so_far == int(g[tag + 'seen%d' % c])
                assert np.array_equal(buf.buffer_label.cpu().numpy(), g[tag + 'label%d' % c]), where
                assert hashlib.sha1(buf.buffer_img.cpu().numpy().tobytes()).hexdigest() == str(g[tag + 'img%d' % c]), where
            w = agent.engine.state.params.cpu().numpy()[pick]
            err = dropin._rel(w - w0, g[tag + 'w%d' % c].astype(np.float64) - w0)
            assert err <= max(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_w'][c]), \
                (where, 'sampled weight update', err, 'one-ulp spread', g[tag + 'spread_w'][c])
            err = dropin._rel(agent.engine.state.bn_stats.cpu().numpy(), g[tag + 'bn%d' % c].astype(np.float64))
            assert err <= max(dropin.BN_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_bn'][c]), (where, 'BN statistics', err)
        loaders = [[(torch.from_numpy(tx).permute(0, 3, 1, 2).float().div(255), torch.from_numpy(ty))] for tx, ty in tests]
        acc = np.asarray(agent.evaluate(loaders))
        assert np.abs(acc - g[tag + 'acc']).max() <= 3.1 / 96, (kind, case, acc, g[tag + 'acc'])
    finally:
        memory.set_mode(False)
        memory.ClassBalancedRandomSampling.reset()
