"""CPU: PCR's oracle (oracle/pcr.py) and the learner's host side.  The written-out loss and gradients are torch
autograd's of a literal restatement of SupConLoss's steps (row max, self mask, mean over the positives) over [R, 2, d]
features whose second view is the normalised W[y], in float64; gradcheck holds at tiny shapes; a zero-norm row follows
the eps rule; an anchor without positives makes the loss NaN and keeps only its log Z gradient; the construction
refusals; the opt-in registration of agents['PCR'] and the launcher's B200OCL_EXTRA_AGENTS."""
import math
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import pcr as opcr

EPS = 1e-6


def supcon_literal(F, W, y, tau, drop_singleton_positive=False):
    """SupConLoss (anchor = the normalised features, contrast = the normalised proxies of the same rows), step by step:
    logits, detached row max, self mask, log-probabilities, mean over the positives, mean over the anchors."""
    u = F / (F.norm(dim=1, keepdim=True) + EPS)
    v = W / (W.norm(dim=1, keepdim=True) + EPS)
    feats = torch.stack((u, v[y]), dim=1)                        # [R, 2, d]
    anchor, contrast = feats[:, 0], feats[:, 1]
    R = F.shape[0]
    logits = anchor @ contrast.T / tau
    logits = logits - logits.max(dim=1, keepdim=True).values.detach()
    self_mask = 1.0 - torch.eye(R, dtype=F.dtype)
    mask = (y[:, None] == y[None, :]).to(F.dtype) * self_mask
    exp_logits = torch.exp(logits) * self_mask
    log_prob = logits - torch.log(exp_logits.sum(1, keepdim=True))
    npos = mask.sum(1)
    if drop_singleton_positive:
        # the kernels' finite-gradient convention: an anchor without positives keeps its log-sum-exp and nothing else
        mean_pos = (mask * log_prob).sum(1) / torch.where(npos > 0, npos, torch.ones_like(npos))
        mean_pos = torch.where(npos > 0, mean_pos, -torch.log(exp_logits.sum(1)))
    else:
        mean_pos = (mask * log_prob).sum(1) / npos
    return -mean_pos.mean()


def _case(R, d, C, seed, pattern='pairs'):
    rs = np.random.RandomState(seed)
    F = torch.tensor(rs.standard_normal((R, d)), dtype=torch.float64)
    W = torch.tensor(rs.standard_normal((C, d)) * 0.3, dtype=torch.float64)
    if pattern == 'pairs':
        half = rs.randint(0, C, (R + 1) // 2)
        y = np.concatenate((half, half))[:R]
        if R % 2:
            y[R // 2] = y[0]                                     # every class at least twice
    elif pattern == 'single_class':
        y = np.full(R, rs.randint(0, C))
    else:
        y = rs.randint(0, C, R)
    return F, W, torch.tensor(y, dtype=torch.int64)


@pytest.mark.parametrize('R,d,C,tau', [(2, 8, 3, 0.09), (4, 16, 5, 0.07), (40, 160, 100, 0.09), (22, 32, 7, 1.0),
                                       (11, 12, 4, 0.5)])
@pytest.mark.parametrize('pattern', ['pairs', 'single_class'])
def test_oracle_is_autograd_of_the_supcon_literal(R, d, C, tau, pattern):
    F, W, y = _case(R, d, C, R * 31 + d + C, pattern)
    Fl, Wl = F.clone().requires_grad_(True), W.clone().requires_grad_(True)
    ref = supcon_literal(Fl, Wl, y, tau)
    ref.backward()
    loss, dF, dW = opcr.loss_and_grads(F, y, W, tau)
    assert math.isclose(float(loss), float(ref.detach()), rel_tol=1e-12)
    torch.testing.assert_close(dF, Fl.grad, rtol=1e-10, atol=1e-13)
    torch.testing.assert_close(dW, Wl.grad, rtol=1e-10, atol=1e-13)
    absent = torch.ones(C, dtype=torch.bool)
    absent[y] = False
    assert torch.equal(dW[absent], torch.zeros_like(dW[absent]))


def test_multiplicity_form_counts_each_proxy_once_per_row():
    """Z_i = sum_c (n_c - [c = y_i]) exp(g_ic): three rows of one class and two of another."""
    F, W, _ = _case(5, 6, 2, 5)
    y = torch.tensor([0, 0, 0, 1, 1])
    u = F / (F.norm(dim=1, keepdim=True) + EPS)
    v = W / (W.norm(dim=1, keepdim=True) + EPS)
    g = u @ v.T / 0.09
    want = 0.0
    for i in range(5):
        m = torch.tensor([3.0, 2.0]) - torch.nn.functional.one_hot(y[i], 2).double()
        want += float(torch.log((m * torch.exp(g[i])).sum()) - g[i, y[i]])
    assert math.isclose(float(opcr.loss_and_grads(F, y, W, 0.09)[0]), want / 5, rel_tol=1e-12)


class _OracleLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, F, W, y, tau):
        loss, dF, dW = opcr.loss_and_grads(F.detach(), y, W.detach(), tau)
        ctx.save_for_backward(dF, dW)
        return loss

    @staticmethod
    def backward(ctx, g):
        dF, dW = ctx.saved_tensors
        return g * dF, g * dW, None, None


@pytest.mark.parametrize('R,d,C', [(2, 3, 2), (4, 5, 3), (6, 4, 4)])
def test_gradcheck(R, d, C):
    F, W, y = _case(R, d, C, 100 + R, 'pairs')
    F.requires_grad_(True)
    W.requires_grad_(True)
    assert torch.autograd.gradcheck(lambda a, b: _OracleLoss.apply(a, b, y, 0.3), (F, W), eps=1e-6, atol=1e-7)


def test_zero_norm_row_follows_the_eps_rule():
    F, W, y = _case(6, 10, 3, 9, 'pairs')
    F[2] = 0.0
    Fl, Wl = F.clone().requires_grad_(True), W.clone().requires_grad_(True)
    supcon_literal(Fl, Wl, y, 0.09).backward()
    loss, dF, dW = opcr.loss_and_grads(F, y, W, 0.09)
    assert torch.isfinite(dF).all() and torch.isfinite(dW).all() and math.isfinite(float(loss))
    torch.testing.assert_close(dF, Fl.grad, rtol=1e-10, atol=1e-13)
    torch.testing.assert_close(dW, Wl.grad, rtol=1e-10, atol=1e-13)
    # the zero row: du / (0 + eps), nothing from the second term
    u = torch.zeros(10, dtype=torch.float64)
    assert torch.isfinite(dF[2]).all() and not torch.equal(dF[2], u)


def test_anchor_without_positives_makes_the_loss_nan_and_keeps_log_z():
    F, W, y = _case(5, 8, 4, 11, 'pairs')
    y = torch.tensor([0, 0, 1, 1, 3])                            # row 4 is its class's only row
    loss, dF, dW = opcr.loss_and_grads(F, y, W, 0.09)
    assert math.isnan(float(loss))
    assert torch.isfinite(dF).all() and torch.isfinite(dW).all()
    Fl, Wl = F.clone().requires_grad_(True), W.clone().requires_grad_(True)
    supcon_literal(Fl, Wl, y, 0.09, drop_singleton_positive=True).backward()
    torch.testing.assert_close(dF, Fl.grad, rtol=1e-10, atol=1e-13)
    torch.testing.assert_close(dW, Wl.grad, rtol=1e-10, atol=1e-13)


def test_cosine_argmax_takes_the_first_maximum():
    W = np.array([[0.0, 1.0], [2.0, 0.5], [2.0, 0.5], [1.0, 0.0]])   # rows 1 and 2 are duplicates
    f = np.array([[3.0, 0.8], [0.0, 2.0], [0.0, 0.0], [1.0, -0.1]])
    assert opcr.cosine_argmax(f, W).tolist() == [1, 0, 0, 3]


def test_step_moves_bn_stream_pair_first():
    """The step's BN statistics equal those of two train-mode passes made in the order [x; x'], [m; m']."""
    from collections import OrderedDict
    from oracle import replay_step as ors
    from oracle import resnet as oresnet
    spec = oresnet.Spec(32, 20, 10)
    p0, bn0 = oresnet.seeded_state(spec, 3, dtype=torch.float64)
    st = ors.ReplayState(spec, p0, bn0, 30, (3, 32, 32), 10, lr=0.05)
    rs = np.random.RandomState(1)
    st.buffer_img[:20] = torch.tensor(rs.rand(20, 3, 32, 32).astype(np.float32))
    st.buffer_label[:20] = torch.tensor(rs.randint(0, 5, 20))
    st.current_index = st.n_seen_so_far = 20
    x = torch.tensor(rs.rand(10, 3, 32, 32).astype(np.float32))
    y = torch.tensor(rs.randint(0, 5, 10))
    bn = OrderedDict((k, v.clone()) for k, v in st.bn.items())
    p0 = OrderedDict((k, v.clone()) for k, v in st.params.items())
    np.random.seed(0)
    logs = opcr.step(st, x, y, eps_mem_batch=10)
    idx = logs[0]['ret_idx']
    with torch.no_grad():
        oresnet.features(spec, p0, bn, torch.cat((x, x)).double(), train=True)
        oresnet.features(spec, p0, bn, torch.cat((st.buffer_img[idx], st.buffer_img[idx])).double(), train=True)
    for k in bn:
        assert torch.equal(bn[k], st.bn[k]), k
    assert st.current_index == 30 and logs[0]['loss'] is not None


def _params(**kw):
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick',
                                'kd_trick_star')}
    base = dict(data='cifar100', cuda=True, epoch=1, batch=10, verbose=False, mem_size=40, eps_mem_batch=10,
                mem_iters=1, update='random', retrieve='random', agent='PCR', optimizer='SGD', learning_rate=0.1,
                weight_decay=0, error_analysis=False, trick=trick)
    trick_on = kw.pop('trick_on', ())
    base.update(kw)
    base['trick'] = dict(trick, **{k: True for k in trick_on})
    return SimpleNamespace(**base)


class _NoModel(object):
    """Anything the learner touched after its refusals would fail on this."""


@pytest.mark.parametrize('kw', [dict(update='ASER'), dict(update='GSS'), dict(retrieve='MIR'), dict(retrieve='ASER'),
                                dict(trick_on=('labels_trick',)), dict(trick_on=('separated_softmax',)),
                                dict(trick_on=('kd_trick',)), dict(trick_on=('kd_trick_star',)),
                                dict(trick_on=('review_trick',)), dict(trick_on=('ncm_trick',))])
def test_refusals(kw):
    from b200ocl import learners
    with pytest.raises(NotImplementedError):
        learners.PCR(_NoModel(), None, _params(**kw))


@pytest.mark.parametrize('value', [0, -0.1, float('nan'), float('inf'), '0.5x', True, [0.1]])
def test_temperature_must_be_finite_and_positive(value):
    from b200ocl import learners
    with pytest.raises(ValueError, match='pcr_temp'):
        learners.PCR(_NoModel(), None, _params(pcr_temp=value))


def test_temperature_defaults_and_is_read_as_float():
    from b200ocl import learners
    assert learners.pcr_temperature(_params()) == 0.09
    assert learners.pcr_temperature(_params(pcr_temp='0.5')) == 0.5
    assert learners.pcr_temperature(_params(pcr_temp=np.float32(0.25))) == 0.25


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


def test_install_registers_pcr_only_on_request():
    from b200ocl import registry

    def check(nm):
        assert 'PCR' not in nm.agents
        registry.install(nm)
        assert 'PCR' not in nm.agents                                     # not by default
        registry.uninstall(nm)
        import b200ocl
        b200ocl.install(nm, extra=('PCR',))
        assert nm.agents['PCR'] is registry.extra_agents['PCR']
        assert registry.extra_agents['PCR'].__name__ == 'PCR'
        assert registry.extra_agents['PCR'].__module__.startswith('b200ocl')
        assert registry.installed_extra == ('PCR',)
        registry.uninstall(nm)
        assert 'PCR' not in nm.agents and registry.installed_extra == ()
        b200ocl.install(nm, extra=('DERPP', 'PCR'))
        assert nm.agents['PCR'] is registry.extra_agents['PCR'] and nm.agents['DERPP'] is registry.extra_agents['DERPP']
        registry.uninstall(nm)
        assert 'PCR' not in nm.agents
    _with_stub_reference(check)


@pytest.mark.parametrize('env,want', [('PCR', ['PCR']), ('EWC, PCR', ['EWC', 'PCR'])])
def test_launcher_passes_pcr_through(monkeypatch, tmp_path, env, want):
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
