"""CPU: DER++'s oracle (oracle/derpp.py) and the learner's host side.  With der_alpha = 0 and der_beta = 1 the oracle's
step is er_step (random retrieval, reservoir update) bit for bit, memory, parameters and BN statistics included; the
written-out logit-term gradient is torch autograd's of alpha * F.mse_loss in float64; the logit memory follows the
reservoir's writes; the construction refusals; the opt-in registration of agents['DERPP'] and the launcher's
B200OCL_EXTRA_AGENTS."""
import copy
import math
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import derpp as oder
from oracle import replay_step as ors
from oracle import resnet as oresnet


def _batches(seed, n_steps, n_lab, n=10):
    rs = np.random.RandomState(seed)
    for _ in range(n_steps):
        x = rs.randint(0, 256, (n, 3, 32, 32)).astype(np.float32) / 255.0
        yield torch.tensor(x), torch.tensor(rs.randint(0, n_lab, n))


def _state(cls, seed, dtype=torch.float32, mem=30, ncls=10):
    spec = oresnet.Spec(32, 20, ncls)
    p0, bn0 = oresnet.seeded_state(spec, seed, dtype=dtype)
    return cls(spec, p0, bn0, mem, (3, 32, 32), ncls, lr=0.05)


def test_oracle_with_alpha_0_and_beta_1_is_er_bit_for_bit():
    der, er = _state(oder.DerState, 3), _state(ors.ReplayState, 3)
    for i, (x, y) in enumerate(_batches(5, 6, 4)):
        np.random.seed(40 + i); torch.manual_seed(40 + i)
        got = oder.derpp_step(der, x, y, 0.0, 1.0)
        np.random.seed(40 + i); torch.manual_seed(40 + i)
        want = ors.er_step(er, x, y, retrieve='random', update='random')
        assert got[0] == want and got[1] is None, i
        assert (got[2] is None) == (i == 0), i                       # the first step meets an empty memory
        assert list(der.log['written']) == list(er.log['written']), i
        for k in er.params:
            assert torch.equal(der.params[k], er.params[k]), (i, k)
        for k in er.bn:
            assert torch.equal(der.bn[k], er.bn[k]), (i, k)
        assert torch.equal(der.buffer_img, er.buffer_img) and torch.equal(der.buffer_label, er.buffer_label), i
        assert (der.current_index, der.n_seen_so_far) == (er.current_index, er.n_seen_so_far), i
    assert der.current_index == 30 and der.n_seen_so_far == 60       # the reservoir's draws were reached


@pytest.mark.parametrize('n,C', [(1, 10), (10, 100), (20, 69), (7, 1)])
def test_logit_term_gradient_is_autograds(n, C):
    rs = np.random.RandomState(n * 1000 + C)
    z = torch.tensor(rs.standard_normal((n, C)) * 3, dtype=torch.float64, requires_grad=True)
    t = torch.tensor(rs.standard_normal((n, C)) * 3, dtype=torch.float64)
    alpha = 0.3
    ref = alpha * F.mse_loss(z, t)
    ref.backward()
    loss, dz = oder.logit_mse(z.detach().numpy(), t.numpy(), alpha)
    assert math.isclose(loss, float(ref.detach()), rel_tol=1e-14)
    np.testing.assert_allclose(dz, z.grad.numpy(), rtol=1e-14, atol=0)


def test_logit_memory_follows_the_reservoir():
    """fp64 steps with both terms on: every slot the reservoir writes (fill phase and draws) holds the stream logits of
    the row stored there, taken before the step's update."""
    st = _state(oder.DerState, 4, dtype=torch.float64, mem=25)
    for i, (x, y) in enumerate(_batches(6, 6, 5)):
        np.random.seed(70 + i); torch.manual_seed(70 + i)
        before = copy.deepcopy(st.params), copy.deepcopy(st.bn)
        probe = SimpleNamespace(spec=st.spec, params=before[0], bn=before[1])
        z = oresnet.forward(probe.spec, probe.params, probe.bn, x.double(), train=True).detach()
        s0 = st.current_index
        out = oder.derpp_step(st, x, y, 0.5, 0.7)
        assert all(v is not None for v in out) or i == 0, (i, out)
        fill = list(range(s0, st.current_index)) if s0 < 25 else []
        rows = {s: j for j, s in enumerate(fill)}
        if 'reservoir_draws' in st.log and s0 + 10 > 25:
            from oracle import aser as oaser
            slots, src = oaser.reservoir_slots(st.log['reservoir_draws'], 25)
            rows.update({s: len(fill) + j for s, j in zip(slots, src)})
        for s, j in rows.items():
            assert torch.equal(st.buffer_logits[s], z[j]), (i, s, j)
            assert torch.equal(st.buffer_img[s], x[j]), (i, s, j)
    assert st.n_seen_so_far == 60


def _params(**kw):
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick',
                                'kd_trick_star')}
    base = dict(data='cifar100', cuda=True, epoch=1, batch=10, verbose=False, mem_size=40, eps_mem_batch=10,
                mem_iters=1, update='random', retrieve='random', agent='DERPP', optimizer='SGD', learning_rate=0.1,
                weight_decay=0, error_analysis=False, der_alpha=0.3, der_beta=0.5, trick=trick)
    trick_on = kw.pop('trick_on', ())
    base.update(kw)
    base['trick'] = dict(trick, **{k: True for k in trick_on})
    return SimpleNamespace(**base)


class _NoModel(object):
    """Anything the learner touched after its refusals would fail on this."""


@pytest.mark.parametrize('kw', [dict(update='ASER'), dict(update='GSS'), dict(retrieve='MIR'), dict(retrieve='ASER'),
                                dict(trick_on=('labels_trick',)), dict(trick_on=('separated_softmax',)),
                                dict(trick_on=('kd_trick',)), dict(trick_on=('kd_trick_star',))])
def test_refusals(kw):
    from b200ocl import learners
    with pytest.raises(NotImplementedError):
        learners.DERPP(_NoModel(), None, _params(**kw))


@pytest.mark.parametrize('name', ['der_alpha', 'der_beta'])
@pytest.mark.parametrize('value', ['missing', None, -0.1, float('nan'), float('inf'), '0.5x', True])
def test_weights_must_be_given_finite_and_non_negative(name, value):
    from b200ocl import learners
    p = _params()
    if value == 'missing':
        delattr(p, name)
    else:
        setattr(p, name, value)
    with pytest.raises(ValueError, match=name):
        learners.DERPP(_NoModel(), None, p)


def test_weights_are_read_as_floats():
    from b200ocl import learners
    assert learners.der_weights(_params(der_alpha=0, der_beta='1.5')) == (0.0, 1.5)
    assert learners.der_weights(_params(der_alpha=np.float32(0.25), der_beta=0)) == (0.25, 0.0)


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


def test_install_registers_derpp_only_on_request():
    from b200ocl import registry

    def check(nm):
        assert 'DERPP' not in nm.agents
        registry.install(nm)
        assert 'DERPP' not in nm.agents                                   # not by default
        registry.uninstall(nm)
        import b200ocl
        b200ocl.install(nm, extra=('DERPP',))
        assert nm.agents['DERPP'] is registry.extra_agents['DERPP']
        assert registry.extra_agents['DERPP'].__name__ == 'DERPP'
        assert registry.extra_agents['DERPP'].__module__.startswith('b200ocl')
        assert registry.installed_extra == ('DERPP',)
        registry.uninstall(nm)
        assert 'DERPP' not in nm.agents and registry.installed_extra == ()
        b200ocl.install(nm, extra=('EWC', 'DERPP'))
        assert nm.agents['DERPP'] is registry.extra_agents['DERPP'] and nm.agents['EWC'] is registry.extra_agents['EWC']
        registry.uninstall(nm)
        assert 'DERPP' not in nm.agents
    _with_stub_reference(check)


@pytest.mark.parametrize('env,want', [('DERPP', ['DERPP']), ('EWC, DERPP', ['EWC', 'DERPP'])])
def test_launcher_passes_derpp_through(monkeypatch, tmp_path, env, want):
    import runpy
    from b200ocl import launch, registry
    seen = []
    monkeypatch.setattr(registry, 'install', lambda reference_name_match=None, extra=(): seen.append(list(extra)))
    monkeypatch.setattr(runpy, 'run_path', lambda *a, **k: None)
    monkeypatch.setattr(sys, 'argv', list(sys.argv))
    monkeypatch.setattr(sys, 'path', list(sys.path))
    monkeypatch.setenv('B200OCL_EXTRA_AGENTS', env)
    launch.main([str(tmp_path / 'main_config.py')])
    assert seen == [want]
