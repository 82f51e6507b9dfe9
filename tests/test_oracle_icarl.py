"""CPU: the fp64 oracle of iCaRL's criterion (oracle/icarl.py) against the reference's own Icarl.update_representation
(tests/golden/icarl.npz, written by tests/golden/make_golden_icarl.py), and the registration of agents['ICARL'] by the
drop-in switch."""
import os
import sys

import numpy as np
import pytest

from oracle import icarl as oic

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'icarl.npz')


def loss_case(g, k):
    """One loss-level golden case: (logits, teacher or None, labels, old_labels, new_labels)."""
    tag = 'l%d_' % k
    rows, C = (int(v) for v in g[tag + 'shape'])
    logits, teacher = oic.case_logits(oic.LOSS_SEED + k, rows, C, float(g[tag + 'scale']), bool(g[tag + 'teacher']))
    return logits, teacher, g[tag + 'labels'].astype(np.int64), g[tag + 'old'].tolist(), g[tag + 'new'].tolist()


def _n_loss_cases():
    return int(np.load(GOLDEN)['n_loss_cases'])


@pytest.mark.parametrize('k', range(_n_loss_cases()))
def test_oracle_matches_reference_icarl_loss(k):
    g = np.load(GOLDEN)
    logits, teacher, labels, old, new = loss_case(g, k)
    loss, grad = oic.icarl_loss(logits, labels, old, new, teacher)
    want = float(g['l%d_loss' % k])
    assert abs(loss - want) <= 1e-5 * abs(want), (k, loss, want)
    assert np.abs(grad - g['l%d_dlogits' % k]).max() <= 1e-6, k
    K = len(old) + len(new)
    assert not g['l%d_dlogits' % k][:, K:].any()          # the reference's columns beyond K get no gradient either


def test_golden_covers_the_cases():
    g = np.load(GOLDEN)
    cases = [loss_case(g, k) for k in range(_n_loss_cases())]
    assert any(t is None for _, t, _, _, _ in cases) and any(t is not None for _, t, _, _, _ in cases)
    assert {lg.shape[1] for lg, _, _, _, _ in cases} == {10, 100}
    # recurring labels with K = C and K = C - 1, and logits in the hundreds
    recurring = [(lg.shape[1], len(o) + len(n)) for lg, _, _, o, n in cases if len(set(o)) < len(o) or set(o) & set(n)]
    assert any(C == K for C, K in recurring) and any(K == C - 1 for C, K in recurring)
    assert max(float(np.abs(lg).max()) for lg, _, _, _, _ in cases) >= 200
    assert int(g['dropin_n_cases']) >= 3


def test_targets_follow_the_reference_construction():
    """icarl.py:42-61: one-hot at len(old) + new.index(y), zero memory rows, teacher sigmoids in the columns k < n_old."""
    old, new = [3, 1, 3], [7, 1]
    teacher = np.array([[0.0, 2.0, -2.0, 5.0, 5.0]] * 4)
    t = oic.targets(4, [7, 1], old, new, teacher)
    assert t.shape == (4, 5)
    np.testing.assert_allclose(t[:, :3], 1 / (1 + np.exp(-teacher[:, :3])), rtol=1e-15)
    assert t[0, 3:].tolist() == [1, 0] and t[1, 3:].tolist() == [0, 1] and not t[2:, 3:].any()
    with pytest.raises(ValueError):
        oic.icarl_loss(np.zeros((4, 4)), [7, 1], old, new, teacher)     # K = 5 positions over 4 logits


def test_install_registers_and_removes_icarl():
    from b200ocl import registry
    import test_install
    for has_ref_icarl in (False, True):
        nm, mods = test_install._stub_reference()
        if has_ref_icarl:
            nm.agents['ICARL'] = ref = object()
        saved = {k: sys.modules.get(k) for k in mods}
        sys.modules.update(mods)
        try:
            registry.install(nm)
            assert nm.agents['ICARL'] is registry.agents['ICARL']
            assert registry.agents['ICARL'].__module__.startswith('b200ocl')
            registry.uninstall(nm)
            if has_ref_icarl:
                assert nm.agents['ICARL'] is ref
            else:
                assert 'ICARL' not in nm.agents
        finally:
            for k, v in saved.items():
                if v is None:
                    sys.modules.pop(k, None)
                else:
                    sys.modules[k] = v
