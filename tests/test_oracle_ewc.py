"""CPU: EWC++'s arithmetic against the reference's own code (tests/golden/ewc.npz, written by
tests/golden/make_golden_ewc.py): the oracle (oracle/ewc.py) reproduces update_running_fisher, the end-of-call
normalisation, the penalty's autograd gradient and accum_fisher bit for bit, and the loss with the penalty within 1e-6;
the learner's host-side EMA schedule, EMA coefficients and penalty coefficient are the oracle's; the construction
refusal; the opt-in registration of agents['EWC'] and the launcher's B200OCL_EXTRA_AGENTS."""
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import ewc as oewc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ewc.npz')
SHAPES = {'0.weight': (8, 12), '0.bias': (8,), '1.weight': (5, 8), '1.bias': (5,)}   # make_golden_ewc.SHAPES


def _flat(d):
    return np.concatenate([d[n].reshape(-1) for n in SHAPES])


def _ce(logits, labels):
    z = logits.astype(np.float64)
    z = z - z.max(1, keepdims=True)
    return float(np.mean(np.log(np.exp(z).sum(1)) - z[np.arange(len(labels)), labels]))


@pytest.mark.parametrize('k', range(int(np.load(GOLDEN)['n_element'])))
def test_oracle_matches_the_reference_bit_for_bit(k):
    g = np.load(GOLDEN)
    tag = 'e%d_' % k
    lam, t, kdt, kds, scale, zero, alpha, fua = json.loads(str(g[tag + 'case']))
    params, prev, running, tmp, logits, labels = oewc.element_case_inputs(7000 + k, SHAPES, scale, zero)
    running, tmp = oewc.update_running_fisher(running, tmp, alpha, fua)
    assert np.array_equal(_flat(running), g[tag + 'ema_running'])
    assert np.array_equal(_flat(tmp), g[tag + 'ema_tmp'])
    fisher = oewc.normalize(running)
    assert np.array_equal(_flat(fisher), g[tag + 'normalized'])
    if zero:
        assert not _flat(fisher).any()
    assert np.array_equal(_flat(params), g[tag + 'prev_end'])
    up = oewc.penalty_up(lam, t, kdt, kds)
    grads = oewc.penalty_grad(params, prev, fisher, up)
    assert np.array_equal(_flat(grads), g[tag + 'grad'])
    assert np.array_equal(_flat(oewc.accum_fisher(oewc.accum_fisher(tmp, grads), grads)), g[tag + 'accum_tmp'])
    mix = 1.0
    if kds:
        mix *= 1 / ((t + 1) ** 0.5)
    if kdt:
        mix *= 1 / (t + 1)
    assert abs(float(g[tag + 'ce']) - _ce(logits, labels)) <= 1e-6 * abs(float(g[tag + 'ce']))
    want = mix * (float(g[tag + 'ce']) + lam * oewc.penalty_value(params, prev, fisher))
    assert abs(float(g[tag + 'loss']) - want) <= 1e-6 * abs(want), (float(g[tag + 'loss']), want)


def test_element_golden_covers_the_cases():
    g = np.load(GOLDEN)
    cases = [json.loads(str(g['e%d_case' % k])) for k in range(int(g['n_element']))]
    assert {c[0] for c in cases} >= {0.0, 1.0, 100.0}
    assert any(c[2] for c in cases) and any(c[3] for c in cases) and any(c[2] and c[3] for c in cases)
    assert any(c[5] for c in cases)
    assert len({c[4] for c in cases if not c[5]}) >= 3


def test_learner_coefficients_are_the_oracles():
    from b200ocl import learners
    for lam in (0.0, 1.0, 37.5, 100.0):
        for t in range(4):
            for kdt in (False, True):
                for kds in (False, True):
                    assert learners.ewc_penalty_up(lam, t, kdt, kds) == float(oewc.penalty_up(lam, t, kdt, kds))
    # the chain is the fp32 product from the outermost weight inward, not the double product rounded once
    assert learners.ewc_penalty_up(1.0, 2, True, True) == float(np.float32(np.float32(3 ** -0.5) * np.float32(1 / 3)))
    for alpha, fua in ((0.9, 50), (0.5, 3), (0.3, 7)):
        assert learners.ewc_ema_coefficients(alpha, fua) == tuple(float(c) for c in oewc.ema_coefficients(alpha, fua))


@pytest.mark.parametrize('n_batches,epochs,fua', [(6, 1, 3), (4, 2, 3), (5, 3, 7), (500, 1, 50), (6, 1, 50), (1, 4, 1)])
def test_ema_schedule_is_the_references(n_batches, epochs, fua):
    """ewc_pp.py:33-41: the loop counter (ep * len(loader) + i + 1), restarted by every call."""
    from b200ocl import learners
    want = []
    for ep in range(epochs):
        for i in range(n_batches):
            want.append((ep * n_batches + i + 1) % fua == 0)
    assert learners.ewc_ema_schedule(n_batches, epochs, fua) == want == oewc.ema_schedule(n_batches, epochs, fua)
    assert sum(want) == (n_batches * epochs) // fua


def _params(**over):
    flags = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick', 'kd_trick_star')}
    p = dict(data='cifar100', cuda=True, epoch=1, batch=10, verbose=False, mem_size=100, eps_mem_batch=10, mem_iters=1,
             update='random', retrieve='random', agent='EWC', optimizer='SGD', learning_rate=0.005, weight_decay=0,
             lambda_=100.0, alpha=0.9, fisher_update_after=50, error_analysis=False, trick=flags)
    p.update(over)
    return SimpleNamespace(**p)


def test_ewc_refuses_ncm_trick_before_building_anything():
    """Checked before the base constructor, so no model or device is touched (model=None would fail there)."""
    from b200ocl import registry
    trick = dict(_params().trick, ncm_trick=True)
    with pytest.raises(NotImplementedError, match='ncm_trick'):
        registry.extra_agents['EWC'](None, None, _params(trick=trick))


def _with_stub_reference(fn):
    import test_install
    nm, mods = test_install._stub_reference()
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    try:
        fn(nm)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_install_registers_ewc_only_on_request():
    from b200ocl import registry

    def check(nm):
        ewc = nm.agents['EWC']
        registry.install(nm)
        assert nm.agents['EWC'] is ewc                                   # not by default
        registry.uninstall(nm)
        import b200ocl
        b200ocl.install(nm, extra=('EWC',))
        assert nm.agents['EWC'] is registry.extra_agents['EWC']
        assert registry.extra_agents['EWC'].__module__.startswith('b200ocl')
        assert nm.agents['ER'] is registry.agents['ER']
        registry.uninstall(nm)
        assert nm.agents['EWC'] is ewc
        with pytest.raises(ValueError, match='CNDPM'):
            registry.install(nm, extra=('CNDPM',))
        assert nm.agents['EWC'] is ewc and nm.agents['ER'] is not registry.agents['ER']   # nothing was replaced
    _with_stub_reference(check)


@pytest.mark.parametrize('env,want', [(None, []), ('EWC', ['EWC']), (' EWC , ', ['EWC'])])
def test_launcher_passes_the_extra_agents_through(monkeypatch, tmp_path, env, want):
    import runpy
    from b200ocl import launch, registry
    seen = []
    monkeypatch.setattr(registry, 'install', lambda reference_name_match=None, extra=(): seen.append(list(extra)))
    monkeypatch.setattr(runpy, 'run_path', lambda *a, **k: None)
    monkeypatch.setattr(sys, 'argv', list(sys.argv))
    monkeypatch.setattr(sys, 'path', list(sys.path))
    if env is None:
        monkeypatch.delenv('B200OCL_EXTRA_AGENTS', raising=False)
    else:
        monkeypatch.setenv('B200OCL_EXTRA_AGENTS', env)
    launch.main([str(tmp_path / 'general_main.py'), '--agent', 'EWC'])
    assert seen == [want]
