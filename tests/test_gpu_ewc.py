"""GPU: the EWC++ agent on the engine.
  * b200ocl_net_sgd_step_ewc against torch on the same device: g_ce injected as (p * g_ce).sum(), the regulariser
    through autograd with the reference's mixing, tmp += g ** 2 and the EMA by the reference's expressions.  The
    kernel's gradient, tmp and running are bit-identical to torch's; params and packed are bit-identical to
    b200ocl_net_sgd_step applied to torch's gradient; the penalty value is within 1e-6 of fp64.  Penalty off, EMA only,
    both, lambda = 0, the kd mixing chain, head='mlp' (the skip range untouched in every arena), a zero gradient;
  * b200ocl_ewc_consolidate against torch's expression bit for bit, an all-zero running, prev == params;
  * repeat launches and two seeded train_learner sequences are bit-identical;
  * learner steps from a common state against the oracle (oracle/ewc.py on oracle/resnet.py) within 1e-3;
  * whole train_learner calls step by step against oracle.ewc.step from the learner's own arenas: the EMA schedule,
    the penalty from the second call on and its coefficient with the mixing weights, bit for bit;
  * drop-in runs against the reference's (tests/golden/ewc.npz): parameters, BN statistics and the four EWC arenas
    within the larger of the fp32 bar and 10x the reference's own one-ulp spread, accuracies within 3 of 96;
  * launches: a step issues at most 2 more than the plain step, consolidation at most 3;
  * the data-parallel refusal."""
import json
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import ewc as oewc
from oracle import gdumb as ogd
from oracle import resnet as oresnet

import test_gpu_dropin as dropin
from test_oracle_ewc import _params

pytestmark = pytest.mark.gpu

GOLDEN = dropin.os.path.join(dropin.os.path.dirname(dropin.os.path.abspath(__file__)), 'golden', 'ewc.npz')


def _engine(head=None, seed=5, zero_grad=False):
    from b200ocl import nets
    eng = nets.EngineModel(32, 100, head=head).engine
    rs = np.random.RandomState(seed)
    n = eng.state.params.numel()
    f = lambda a: torch.from_numpy(a.astype(np.float32)).cuda()
    eng.state.params.copy_(f(rs.standard_normal(n) * 0.1))
    eng.state.grads.copy_(f(rs.standard_normal(n) * 0.01 * (not zero_grad)))
    st = eng.ewc_state()
    st.running.copy_(f(np.abs(rs.standard_normal(n)) * 1e-3))
    st.tmp.copy_(f(np.abs(rs.standard_normal(n)) * 1e-4))
    st.normalized.copy_(f(rs.rand(n)))
    st.prev.copy_(eng.state.params + f(rs.standard_normal(n) * 0.01))
    eng.pack()
    return eng


def _has_grad(eng):
    has = torch.zeros(eng.state.params.numel(), dtype=torch.bool, device='cuda')
    for o, n, hg in eng.table:
        has[o:o + n] = hg
    return has


def _torch_step(eng, lam, t, kdt, kds, penalty, ema, alpha, fua):
    """ewc_pp.py:40-62 in torch on copies of the arenas: (g, tmp, running) as flat device tensors."""
    st = eng.ewc_state()
    views = lambda a: [a[o:o + n] for (o, n, _) in eng.table]
    live = [hg for (_, _, hg) in eng.table]
    running = [r.clone() for r in views(st.running)]
    tmp = [r.clone() for r in views(st.tmp)]
    if ema:                                                                 # ewc_pp.py:104-108
        running = [(1. - alpha) * r + 1. / fua * alpha * q if h else r for r, q, h in zip(running, tmp, live)]
        tmp = [torch.zeros_like(q) if h else q for q, h in zip(tmp, live)]
    ps = [torch.nn.Parameter(p.clone()) for p in views(eng.state.params)]
    gce = views(eng.state.grads)
    loss = sum((p * g).sum() for p, g, h in zip(ps, gce, live) if h)       # the network's gradient, injected
    if penalty:                                                             # ewc_pp.py:85-92
        reg = 0
        for p, f, q, h in zip(ps, views(st.normalized), views(st.prev), live):
            if h:
                reg += (f * (p - q) ** 2).sum()
        loss += lam * reg
    if kdt:
        loss = 1 / (t + 1) * loss + (1 - 1 / (t + 1)) * 0
    if kds:
        loss = 1 / ((t + 1) ** 0.5) * loss + (1 - 1 / ((t + 1) ** 0.5)) * 0
    loss.backward()
    g = [p.grad if h else gc for p, gc, h in zip(ps, gce, live)]
    for q, gg, h in zip(tmp, g, live):
        if h:
            q += gg ** 2                                                    # ewc_pp.py:110-112
    return torch.cat(g), torch.cat(tmp), torch.cat(running)


def _ce_part(eng, t, kdt, kds):
    """The gradient of the (mixed) criterion alone, as autograd forms it: what the backward pass leaves in the arena."""
    ps = [torch.nn.Parameter(p.clone()) for p in eng.param_views()]
    loss = sum((p * g).sum() for p, g in zip(ps, eng.grad_views()))
    if kdt:
        loss = 1 / (t + 1) * loss + (1 - 1 / (t + 1)) * 0
    if kds:
        loss = 1 / ((t + 1) ** 0.5) * loss + (1 - 1 / ((t + 1) ** 0.5)) * 0
    loss.backward()
    return torch.cat([p.grad for p in ps])


CASES = {   # name: (head, lam, task_seen, kd_trick, kd_trick_star, penalty, ema, zero gradient)
    'plain': (None, 100.0, 1, False, False, False, False, False),
    'ema_only': (None, 100.0, 1, False, False, False, True, False),
    'penalty_only': (None, 100.0, 1, False, False, True, False, False),
    'both': (None, 100.0, 1, False, False, True, True, False),
    'lambda0': (None, 0.0, 1, False, False, True, True, False),
    'kd_chain': (None, 37.5, 2, True, True, True, True, False),
    'mlp': ('mlp', 100.0, 1, False, False, True, True, False),
    'zero_grad': (None, 100.0, 1, False, False, True, True, True),
    'zero_grad_ema': (None, 100.0, 1, False, False, False, True, True),
}


@pytest.mark.parametrize('name', sorted(CASES))
def test_fused_step_matches_torch(name):
    from b200ocl import learners
    head, lam, t, kdt, kds, penalty, ema, zero = CASES[name]
    alpha, fua, lr, wd = 0.9, 50, 0.05, 1e-4
    eng = _engine(head, zero_grad=zero)
    st = eng.ewc_state()
    before = {k: getattr(st, k).clone() for k in ('running', 'tmp', 'normalized', 'prev')}
    before.update(params=eng.state.params.clone(), grads=eng.state.grads.clone())
    g_t, tmp_t, run_t = _torch_step(eng, lam, t, kdt, kds, penalty, ema, alpha, fua)
    if kdt or kds:
        eng.state.grads.copy_(_ce_part(eng, t, kdt, kds))                  # the mixed criterion's gradient
    # the plain step applied to torch's gradient, on a second engine
    ref = _engine(head, zero_grad=zero)
    ref.state.grads.copy_(g_t)
    ref.sgd_step(lr, wd)
    up = learners.ewc_penalty_up(lam, t, kdt, kds)
    keep, add = learners.ewc_ema_coefficients(alpha, fua)
    pen = eng.sgd_step_ewc(lr, wd, up, penalty, ema, keep, add, want_penalty=True)
    has = _has_grad(eng)
    assert torch.equal(eng.state.grads[has], g_t[has]), name
    assert torch.equal(st.tmp[has], tmp_t[has]), name
    assert torch.equal(st.running[has], run_t[has]), name
    assert torch.equal(eng.state.params, ref.state.params), name
    assert torch.equal(eng.state.packed, ref.state.packed), name
    d = (before['params'] - before['prev']).double()
    want = float((before['normalized'].double() * d * d)[has].sum()) if penalty else 0.0
    assert abs(float(pen) - want) <= 1e-6 * abs(want), (name, float(pen), want)
    for k in ('running', 'tmp', 'normalized', 'prev'):                      # the skip range is untouched
        assert torch.equal(getattr(st, k)[~has], before[k][~has]), (name, k)
    assert torch.equal(eng.state.grads[~has], before['grads'][~has])
    assert torch.equal(eng.state.params[~has], before['params'][~has])
    if head == 'mlp':
        assert (~has).any()
    if zero and ema and not penalty:                                       # tmp restarts at 0 and adds 0 * 0
        assert not st.tmp[has].any()


@pytest.mark.parametrize('head', [None, 'mlp'])
@pytest.mark.parametrize('zero', [False, True])
def test_consolidate_matches_torch(head, zero):
    eng = _engine(head)
    st = eng.ewc_state()
    if zero:
        st.running.zero_()
    has = _has_grad(eng)
    before = {k: getattr(st, k).clone() for k in ('normalized', 'prev')}
    rv = [st.running[o:o + n] for (o, n, hg) in eng.table if hg]
    mx = max([torch.max(m) for m in rv])                                     # ewc_pp.py:74-77
    mn = min([torch.min(m) for m in rv])
    want = torch.cat([(p - mn) / (mx - mn + 1e-32) for p in rv])
    eng.ewc_consolidate()
    assert torch.equal(st.normalized[has], want)
    assert torch.equal(st.prev[has], eng.state.params[has])
    for k in ('normalized', 'prev'):
        assert torch.equal(getattr(st, k)[~has], before[k][~has])
    if zero:
        assert not st.normalized[has].any()
    else:
        assert float(st.normalized[has].max()) == 1.0 and float(st.normalized[has].min()) == 0.0


def test_repeat_launches_are_bit_identical():
    out = []
    for _ in range(2):
        eng = _engine(seed=8)
        pens = [eng.sgd_step_ewc(0.05, 1e-4, 100.0, True, k == 1, 0.1, 0.018, want_penalty=True).clone()
                for k in range(3)]
        eng.ewc_consolidate()
        st = eng.ewc_state()
        out.append([torch.cat(pens), eng.state.params.clone(), eng.state.grads.clone(), st.running.clone(),
                    st.tmp.clone(), st.normalized.clone(), st.prev.clone()])
    for u, v in zip(*out):
        assert torch.equal(u, v)


def test_launch_counts():
    from b200ocl import _native
    eng = _engine()
    n0 = _native.launch_count()
    eng.sgd_step(0.05)
    plain = _native.launch_count() - n0
    n0 = _native.launch_count()
    eng.sgd_step_ewc(0.05, 0.0, 100.0, True, True, 0.1, 0.018, want_penalty=True)
    step = _native.launch_count() - n0
    n0 = _native.launch_count()
    eng.ewc_consolidate()
    cons = _native.launch_count() - n0
    assert step <= plain + 2, (step, plain)
    assert cons <= 3, cons


def _ewc(params):
    from b200ocl import nets, registry
    return registry.extra_agents['EWC'](nets.setup_architecture(params), None, params)


def _task(rs, n, labels):
    return rs.randint(0, 256, (n, 32, 32, 3)).astype(np.uint8), np.asarray(labels, dtype=np.int64)[rs.permutation(n) % len(labels)]


def test_whole_calls_are_deterministic():
    def run():
        np.random.seed(1); random.seed(1); torch.manual_seed(1)              # the network's initialisation draws too
        agent = _ewc(_params(fisher_update_after=3))
        rs = np.random.RandomState(2)
        for t in range(3):
            agent.train_learner(*_task(rs, 45, range(5 * t, 5 * t + 5)))
        torch.cuda.synchronize()
        eng, st = agent.engine, agent.engine.ewc_state()
        return [eng.state.params.clone(), eng.state.grads.clone(), eng.state.bn_stats.clone(), st.running.clone(),
                st.tmp.clone(), st.normalized.clone(), st.prev.clone(), agent.last_loss.clone()]
    for u, v in zip(run(), run()):
        assert torch.equal(u, v)


ARENAS = ('running', 'tmp', 'normalized', 'prev')
WIRING = {   # name: (overrides, calls, samples per call)
    'plain': (dict(), 3, 33),
    'epoch2': (dict(epoch=2), 2, 23),
    'kd_tricks': (dict(kd_trick=True, kd_trick_star=True), 3, 33),
    'labels_trick': (dict(labels_trick=True), 2, 33),
    'lambda0': (dict(lambda_=0.0), 2, 23),
}


@pytest.mark.parametrize('name', sorted(WIRING))
def test_train_learner_steps_match_the_oracle(name, monkeypatch):
    """The learner's wiring over whole train_learner calls: every EWC++ step is checked against oracle.ewc.step taken
    from the arenas the learner left just before it, with the flags and coefficients the reference would use (the EMA
    by ewc_pp.py:40-41's counter, restarted per call; the penalty from the second call on; up from lambda and the mixing
    weights of that call's task_seen).  The gradient, tmp and running must be bit-identical to the oracle's (numpy
    rounds every op in fp32 as the reference's torch ops do), the weights within 1e-6 (the oracle's SGD is fp64); each
    consolidation must give the oracle's normalisation bit for bit and prev == params.  A penalty that is missing,
    scaled, or live a call early or late changes the gradient at the first step it affects."""
    over, n_calls, n = WIRING[name]
    over = dict(over)
    trick = dict(_params().trick, **{k: over.pop(k) for k in ('kd_trick', 'kd_trick_star', 'labels_trick') if k in over})
    params = _params(fisher_update_after=2, learning_rate=0.005, weight_decay=1e-4, trick=trick, **over)
    np.random.seed(4); random.seed(4); torch.manual_seed(4)
    agent = _ewc(params)
    eng, st = agent.engine, agent.engine.ewc_state()
    real_step, real_consolidate = eng.sgd_step_ewc, eng.ewc_consolidate
    sched = oewc.ema_schedule(n // params.batch, params.epoch, params.fisher_update_after)
    log = {'call': 0, 'k': 0, 'penalty_steps': 0, 'ema_steps': 0, 'consolidations': 0}
    cpu = lambda t: t.cpu().numpy().copy()

    def step(lr, wd, up, penalty, ema, keep, add, want_penalty=False):
        c, k = log['call'], log['k']
        P, G = {'w': cpu(eng.state.params)}, {'w': cpu(eng.state.grads)}
        S = {a: {'w': cpu(getattr(st, a))} for a in ARENAS}
        out = real_step(lr, wd, up, penalty, ema, keep, add, want_penalty=want_penalty)
        want_up = oewc.penalty_up(params.lambda_, c, trick['kd_trick'], trick['kd_trick_star'])
        new_p, new_g, S2, _ = oewc.step(P, G, S, params.learning_rate, params.weight_decay, want_up, c > 0, sched[k],
                                        params.alpha, params.fisher_update_after)
        where = '%s call %d step %d' % (name, c, k)
        assert np.array_equal(cpu(eng.state.grads), new_g['w']), (where, 'gradient')
        assert np.array_equal(cpu(st.tmp), S2['tmp']['w']), (where, 'tmp')
        assert np.array_equal(cpu(st.running), S2['running']['w']), (where, 'running')
        w = cpu(eng.state.params)
        assert float(np.abs(w - new_p['w']).max()) <= 1e-6 * float(np.abs(new_p['w']).max()), (where, 'weights')
        log['k'] += 1
        log['penalty_steps'] += c > 0
        log['ema_steps'] += sched[k]
        return out

    def consolidate():
        w, running = cpu(eng.state.params), cpu(st.running)
        real_consolidate()
        assert np.array_equal(cpu(st.normalized), oewc.normalize({'w': running})['w'])
        assert np.array_equal(cpu(st.prev), w)
        log['consolidations'] += 1

    monkeypatch.setattr(eng, 'sgd_step_ewc', step)
    monkeypatch.setattr(eng, 'ewc_consolidate', consolidate)
    rs = np.random.RandomState(5)
    for c in range(n_calls):
        log['call'], log['k'] = c, 0
        agent.train_learner(*_task(rs, n, range(5 * c, 5 * c + 5)))
        assert log['k'] == len(sched), (c, log)
        assert log['consolidations'] == c + 1
    assert log['penalty_steps'] == (n_calls - 1) * len(sched) > 0
    assert log['ema_steps'] == n_calls * sum(sched) > 0


def test_dicts_are_views_and_refusals():
    agent = _ewc(_params())
    names = [n for n, _ in agent.model.named_parameters()]
    assert list(agent.running_fisher) == names and agent.prev_params == {}
    agent.running_fisher[names[0]].fill_(3.0)
    assert float(agent.engine.ewc_state().running[0]) == 3.0
    assert not hasattr(agent, 'buffer')
    rs = np.random.RandomState(3)
    agent.train_learner(*_task(rs, 20, range(3)))
    assert list(agent.prev_params) == names
    agent.grad_sync = lambda eng: None
    with pytest.raises(NotImplementedError, match='data-parallel'):
        agent.train_learner(*_task(rs, 20, range(3)))


def test_learner_steps_match_the_oracle():
    """Steps of the learner from a common state against oracle.resnet's forward / backward and oracle.ewc's step: the
    penalty live, the EMA firing at the second step."""
    from b200ocl import learners
    spec = oresnet.Spec(32, 20, 100)
    p, bn = oresnet.seeded_state(spec, 23)
    agent = _ewc(_params(fisher_update_after=2, learning_rate=0.005, weight_decay=1e-4))
    eng = agent.engine
    names = list(p)
    rs = np.random.RandomState(24)
    flat = lambda d: np.concatenate([d[n].reshape(-1) for n in names])
    n = eng.state.params.numel()
    state = {'running': np.abs(rs.standard_normal(n)).astype(np.float32) * np.float32(1e-3),
             'tmp': np.abs(rs.standard_normal(n)).astype(np.float32) * np.float32(1e-4),
             'normalized': rs.rand(n).astype(np.float32)}
    state['prev'] = (flat({k: v.numpy() for k, v in p.items()}) + rs.standard_normal(n).astype(np.float32) * np.float32(0.01)).astype(np.float32)
    split = lambda a: {k: v.reshape(p[k].shape)
                       for k, v in zip(names, np.split(a, np.cumsum([p[k].numel() for k in names])[:-1]))}
    agent._penalty_live = True
    agent.task_seen = 1
    for i in range(3):
        eng.load(list(p.values()), [(bn[m + '.running_mean'], bn[m + '.running_var']) for m in oresnet.bn_names(spec)])
        st = eng.ewc_state()
        for k in ('running', 'tmp', 'normalized', 'prev'):
            getattr(st, k).copy_(torch.from_numpy(state[k]))
        x = torch.from_numpy(rs.randint(0, 256, (10, 3, 32, 32)).astype(np.float32) / 255.0)
        y = torch.from_numpy(rs.randint(0, 100, 10))
        ema = i == 1
        agent.replay_step(x.cuda(), y.cuda(), y.numpy(), ema=ema)
        torch.cuda.synchronize()
        _, _, grads = oresnet.ce_loss_and_grads(spec, p, bn, x, y)
        pd = {k: v.numpy() for k, v in p.items()}
        gd = {k: grads[k].numpy() for k in names}
        sd = {k: split(v) for k, v in state.items()}
        up = float(oewc.penalty_up(100.0, 1))
        assert up == learners.ewc_penalty_up(100.0, 1)
        new_p, new_g, sd, pen = oewc.step(pd, gd, sd, 0.005, 1e-4, up, True, ema, 0.9, 2)
        state = {k: flat(v) for k, v in sd.items()}
        for k, v in new_p.items():
            p[k] = torch.from_numpy(v)
        rel = lambda a, b: float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))
        assert rel(eng.state.params.cpu().numpy(), flat(new_p)) < 1e-3, i
        assert rel(eng.state.grads.cpu().numpy(), flat(new_g)) < 1e-3, i
        assert rel(st.tmp.cpu().numpy(), state['tmp']) < 1e-3, i
        assert rel(st.running.cpu().numpy(), state['running']) < 1e-3, i


@pytest.mark.parametrize('case', range(int(np.load(GOLDEN)['n_dropin'])))
def test_ewc_dropin_matches_reference_run(case):
    from b200ocl import memory
    g = np.load(GOLDEN)
    tag = 'c%d_' % case
    n_calls, n_label, n_per_call, wseed, seed, dseed = json.loads(str(g[tag + 'case']))
    params = SimpleNamespace(**json.loads(str(g[tag + 'params'])))
    params.cuda = True
    spec = oresnet.Spec(32, 20, 10 if params.data == 'cifar10' else 100)
    memory.set_mode(True, 'cpu')                    # the reference ran on the CPU: its draws came from CPU generators
    try:
        agent = _ewc(params)
        eng = agent.engine
        p, bn = oresnet.seeded_state(spec, wseed)
        eng.load(list(p.values()), [(bn[m + '.running_mean'], bn[m + '.running_var']) for m in oresnet.bn_names(spec)])
        w0 = torch.cat([t.reshape(-1) for t in p.values()]).numpy()
        pick = dropin.dropin_sample(w0.size)
        w0 = w0[pick].astype(np.float64)
        np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
        calls, tests = ogd.dropin_inputs(np.random.RandomState(dseed), 32, n_label, n_per_call, n_calls)
        st = eng.ewc_state()
        arenas = {'running_fisher': st.running, 'tmp_fisher': st.tmp, 'normalized_fisher': st.normalized,
                  'prev_params': st.prev}
        for c, (xt, yt) in enumerate(calls):
            where = 'case %d call %d' % (case, c)
            agent.train_learner(xt, yt)
            torch.cuda.synchronize()
            w = eng.state.params.cpu().numpy()[pick]
            err = dropin._rel(w - w0, g[tag + 'w%d' % c].astype(np.float64) - w0)
            assert err <= max(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_w'][c]), \
                (where, 'sampled weight update', err, 'one-ulp spread', g[tag + 'spread_w'][c])
            err = dropin._rel(eng.state.bn_stats.cpu().numpy(), g[tag + 'bn%d' % c].astype(np.float64))
            assert err <= max(dropin.BN_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_bn'][c]), (where, 'BN statistics', err)
            for a, t in arenas.items():
                err = dropin._rel(t.cpu().numpy()[pick[::4]], g[tag + '%s%d' % (a, c)].astype(np.float64))
                assert err <= max(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_' + a][c]), (where, a, err)
        loaders = [[(torch.from_numpy(tx).permute(0, 3, 1, 2).float().div(255), torch.from_numpy(ty))] for tx, ty in tests]
        acc = np.asarray(agent.evaluate(loaders))
        assert np.abs(acc - g[tag + 'acc']).max() <= 3.1 / 96, (case, acc, g[tag + 'acc'])   # <= 3 of 96 samples
    finally:
        memory.set_mode(False)
