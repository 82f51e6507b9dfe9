"""CPU: Adam's oracle and the optimizer descriptor.
  * oracle.adam.step against the reference's torch.optim.Adam (tests/golden/adam.npz, the CPU optimizer over seeded
    tensors, up to 300 steps, weight decay, other betas / eps, zero and tiny gradients, the review trick's / 10.):
    every recorded step from the recorded state: exp_avg bit for bit, exp_avg_sq within 2 ulp and the weights within
    1 ulp or 3e-5 of their update (the CPU rounds addcmul without fma), the counts reported;
  * the host scalars against torch/optim/adam.py's Python expressions, for both of its paths;
  * the descriptor (learners.ContinualLearner._optimizer): opt None with params.optimizer 'SGD' / 'Adam', the caller's
    SGD and Adam, a changed lr followed, and every refusal (AdamW, amsgrad, maximize, fused, capturable,
    differentiable, two param groups, another optimizer class, data-parallel gradient sync);
  * install() / uninstall() leave the registry as before."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import adam as oadam

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'adam.npz')


def test_oracle_matches_reference_adam_elements():
    """The golden steps ran on the CPU, whose kernels round two ops differently from the CUDA ones the oracle restates:
    addcmul forms value * g * g in two roundings and adds (CUDA: one fma over the rounded g * g), and the division by
    bc2_sqrt is a true division.  So exp_avg must be bit-identical, exp_avg_sq within 2 ulp, and the weights within
    1 ulp or 3e-5 of their own update (a 1-ulp denominator moves the update by ~6e-8 of itself, 300 steps in)."""
    g = np.load(GOLDEN)
    counts = {'m': [0, 0], 'v': [0, 0], 'p': [0, 0]}
    for k in range(int(g['n_element'])):
        lr, b1, b2, eps, wd, n_steps, kind, rec = json.loads(str(g['e%d_case' % k]))
        for s in rec:
            t = 'e%d_s%d_' % (k, s)
            p, gr, m, v = oadam.step(g[t + 'p'], g[t + 'g'], g[t + 'm'], g[t + 'v'], s, lr, (b1, b2), eps, wd,
                                     foreach=True)
            assert np.array_equal(m, g[t + 'm_out']), (k, s, 'exp_avg')
            dv = oadam.ulp_distance(v, g[t + 'v_out'])
            assert dv.max() <= 2, (k, s, 'exp_avg_sq', int(dv.max()))
            dp = oadam.ulp_distance(p, g[t + 'p_out'])
            upd = np.abs(g[t + 'p_out'].astype(np.float64) - g[t + 'p'])
            err = np.abs(p.astype(np.float64) - g[t + 'p_out'])
            assert ((dp <= 1) | (err <= 3e-5 * upd)).all(), (k, s, 'weights', int(dp.max()))
            for key, d in (('m', oadam.ulp_distance(m, g[t + 'm_out'])), ('v', dv), ('p', dp)):
                counts[key][0] += int((d > 0).sum())
                counts[key][1] += d.size
    print('oracle vs the reference CPU Adam, elements not bit-identical: ' +
          ', '.join('%s %d of %d' % (k, a, b) for k, (a, b) in counts.items()))
    assert counts['v'][0] <= 0.2 * counts['v'][1] and counts['p'][0] <= 0.05 * counts['p'][1]


def test_oracle_review_prescale_is_the_recorded_gradient():
    """The review trick's g / 10. as the oracle forms it on CUDA (g * fp32(1/10)) against the CPU division."""
    g = np.load(GOLDEN)
    for k in range(int(g['n_element'])):
        case = json.loads(str(g['e%d_case' % k]))
        if case[6] != 'review':
            continue
        raw = (np.random.RandomState(1).standard_normal(4096) * 0.05).astype(np.float32)
        want = (torch.from_numpy(raw).clone() / 10.).numpy()
        _, got, _, _ = oadam.step(np.zeros(4096, np.float32), raw, np.zeros(4096, np.float32),
                                  np.zeros(4096, np.float32), 1, 1e-3, grad_div=10.0)
        assert oadam.ulp_distance(got, want).max() <= 1


@pytest.mark.parametrize('lr,betas', [(1e-3, (0.9, 0.999)), (3e-4, (0.8, 0.99)), (0.1, (0.5, 0.0))])
def test_host_scalars_match_torch_expressions(lr, betas):
    from b200ocl import ops
    beta1, beta2 = betas
    for step in (1, 2, 3, 10, 100, 1000, 12345):
        st = torch.tensor(float(step), dtype=torch.float32)         # torch keeps the count as an fp32 CPU tensor
        s = st.item()
        bc1, bc2 = 1 - beta1 ** s, 1 - beta2 ** s
        single = (lr / bc1, bc2 ** 0.5)                              # _single_tensor_adam
        multi = ((lr / bc1) * -1, bc2 ** 0.5)                        # _multi_tensor_adam
        assert -single[0] == multi[0]
        assert oadam.host_scalars(lr, beta1, beta2, step) == multi
        c = ops.adam_scalars(lr, betas, 1e-8, 5e-4, step)
        assert c.step_size == float(np.float32(multi[0])) and c.bc2_sqrt == float(np.float32(multi[1]))
        assert c.beta1_c == float(np.float32(1 - beta1)) and c.beta2_c == float(np.float32(1 - beta2))
        assert c.beta2 == float(np.float32(beta2)) and c.eps == float(np.float32(1e-8))
        assert c.weight_decay == float(np.float32(5e-4)) and c.grad_scale == 1.0
        assert c.bc2_sqrt_inv == float(np.float32(1 / multi[1]))   # CUDA Tensor / Python float: the double reciprocal


class _Stub(object):
    """The descriptor and step dispatch of learners.ContinualLearner without an engine."""

    def __init__(self, opt, **params):
        from b200ocl import learners
        self.opt = opt
        self.params = SimpleNamespace(**dict(dict(learning_rate=0.01, weight_decay=0.0), **params))
        self.grad_sync = None
        self._optimizer = learners.ContinualLearner._optimizer.__get__(self)
        self._optimizer_step = learners.ContinualLearner._optimizer_step.__get__(self)
        self._begin_call = learners.ContinualLearner._begin_call.__get__(self)


def _params():
    return [torch.nn.Parameter(torch.zeros(3))]


def test_descriptor_without_an_optimizer_follows_params():
    s = _Stub(None, optimizer='Adam', learning_rate=0.002, weight_decay=1e-4)._optimizer()
    assert (s.kind, s.lr, s.weight_decay, s.betas, s.eps, s.foreach) == ('adam', 0.002, 1e-4, (0.9, 0.999), 1e-8, True)
    s = _Stub(None, optimizer='SGD', learning_rate=0.1)._optimizer()
    assert (s.kind, s.lr, s.weight_decay) == ('sgd', 0.1, 0.0)
    s = _Stub(None)._optimizer()                                     # no params.optimizer: SGD, as before
    assert s.kind == 'sgd'
    with pytest.raises(NotImplementedError):
        _Stub(None, optimizer='RMSprop')._optimizer()


def test_descriptor_reads_the_callers_optimizer_at_every_step():
    opt = torch.optim.Adam(_params(), lr=3e-4, betas=(0.8, 0.99), eps=1e-6, weight_decay=5e-4)
    stub = _Stub(opt)
    s = stub._optimizer()
    assert (s.kind, s.lr, s.weight_decay, s.betas, s.eps, s.foreach) == ('adam', 3e-4, 5e-4, (0.8, 0.99), 1e-6, True)
    opt.param_groups[0]['lr'] = 1e-4
    assert stub._optimizer().lr == 1e-4
    assert not _Stub(torch.optim.Adam(_params(), foreach=False))._optimizer().foreach
    s = _Stub(torch.optim.SGD(_params(), lr=0.05, weight_decay=1e-4))._optimizer()
    assert (s.kind, s.lr, s.weight_decay) == ('sgd', 0.05, 1e-4)


@pytest.mark.parametrize('make', [
    lambda: torch.optim.AdamW(_params()),
    lambda: torch.optim.Adam(_params(), decoupled_weight_decay=True),
    lambda: torch.optim.Adam(_params(), amsgrad=True),
    lambda: torch.optim.Adam(_params(), maximize=True),
    lambda: torch.optim.Adam(_params(), fused=True),
    lambda: torch.optim.Adam(_params(), capturable=True),
    lambda: torch.optim.Adam(_params(), differentiable=True),
    lambda: torch.optim.Adam([{'params': _params()}, {'params': _params(), 'lr': 1e-4}]),
    lambda: torch.optim.RMSprop(_params()),
    lambda: torch.optim.SGD(_params(), lr=0.1, momentum=0.9),
], ids=['AdamW', 'decoupled', 'amsgrad', 'maximize', 'fused', 'capturable', 'differentiable', 'two_groups', 'RMSprop',
        'momentum'])
def test_descriptor_refusals(make):
    with pytest.raises(NotImplementedError):
        _Stub(make())._optimizer()


def test_data_parallel_adam_is_refused():
    stub = _Stub(None, optimizer='Adam')
    stub.grad_sync = lambda eng: None
    with pytest.raises(NotImplementedError, match='data-parallel'):
        stub._begin_call()
    with pytest.raises(NotImplementedError, match='data-parallel'):
        stub._optimizer_step(stub._optimizer())


def test_install_and_uninstall_are_unaffected():
    """Adam adds no agent: install() replaces the same agents as before and uninstall() restores every original."""
    import sys
    import test_install
    from b200ocl import registry
    nm, mods = test_install._stub_reference()
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    try:
        before = dict(nm.agents)
        registry.install(nm)
        replaced = sorted(k for k in before if nm.agents[k] is not before[k])
        assert replaced == sorted(k for k in registry.agents if k in before)
        assert 'EWC' not in replaced
        registry.uninstall(nm)
        assert all(nm.agents[k] is before[k] for k in before)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
