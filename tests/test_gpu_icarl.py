"""GPU: the iCaRL agent on the engine.
  * b200ocl_icarl_loss against the fp64 oracle (oracle/icarl.py) on every loss-level golden case of
    tests/golden/icarl.npz and on a seeded sweep of shapes, teachers and logits up to |z| = 200; the columns at or beyond
    K get exactly zero; repeat launches are bit-identical; a label without a position of this task sets the error flag;
  * the refusals on the host: more label positions than logits, a short memory draw, an update plugin other than the
    reservoir;
  * concurrent and sequential teacher forwards give bit-identical weights, BN statistics and losses;
  * drop-in runs against the reference's (icarl.npz), with the comparison and tolerances of test_gpu_dropin.py."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import icarl as oic

import test_gpu_dropin as dropin
from test_oracle_icarl import GOLDEN, loss_case

pytestmark = pytest.mark.gpu


def _pos_table(old, new, inv=None):
    """before_train's lbl_inv_map for this task (positions len(old) + i; inv: earlier tasks' entries kept as well) as
    the device table the learner uploads."""
    from b200ocl.learners import separated_softmax_table
    inv = dict(inv or {})
    inv.update({int(c): len(old) + i for i, c in enumerate(new)})
    return torch.from_numpy(separated_softmax_table(old, new, inv)[2]).cuda()


def _kernel(logits, teacher, labels, old, new, err=None, inv=None):
    from b200ocl.engine import icarl_loss
    t = None if teacher is None else torch.from_numpy(np.ascontiguousarray(teacher)).cuda()
    return icarl_loss(torch.from_numpy(logits).cuda(), torch.from_numpy(np.asarray(labels, np.int64)).cuda(),
                      _pos_table(old, new, inv), len(old) + len(new), len(old) if teacher is not None else 0, teacher=t,
                      err=err)


def _check(logits, teacher, labels, old, new, where):
    err = torch.zeros(1, dtype=torch.int32, device='cuda')
    out = _kernel(logits, teacher, labels, old, new, err)
    loss, grad = oic.icarl_loss(logits, labels, old, new, teacher)
    got = float(out['loss'])
    assert np.isfinite(got) and abs(got - loss) <= 1e-5 * abs(loss), (where, got, loss)
    d = out['dlogits'].cpu().numpy()
    assert np.abs(d - grad).max() <= 1e-6 + 1e-5 * np.abs(grad).max(), (where, np.abs(d - grad).max())
    K = len(old) + len(new)
    assert not d[:, K:].any(), where
    assert int(err) == 0, where


@pytest.mark.parametrize('k', range(int(np.load(GOLDEN)['n_loss_cases'])))
def test_icarl_loss_matches_oracle_on_golden_cases(k):
    g = np.load(GOLDEN)
    logits, teacher, labels, old, new = loss_case(g, k)
    _check(logits, teacher, labels, old, new, k)


def _sweep_case(N, C, with_old, K_eq_C, seed):
    rs = np.random.RandomState(seed)
    K = C if K_eq_C else C - 3
    n_old = K // 3 if with_old else 0
    old = rs.randint(0, C, n_old).tolist()                     # old_labels may repeat
    new = rs.permutation(C)[:K - n_old].tolist()
    logits = (rs.standard_normal((N, C)) * 3).astype(np.float32)
    big = rs.rand(N, C) < 0.1
    logits[big] = rs.uniform(-200, 200, big.sum())
    teacher = None
    n_stream = N
    if with_old:
        teacher = (rs.standard_normal((N, C)) * 3).astype(np.float32)
        big_t = rs.rand(N, C) < 0.1
        teacher[big_t] = rs.uniform(-200, 200, big_t.sum())
        n_stream = (N + 1) // 2                                # the rest are memory rows
    labels = np.asarray(new)[rs.randint(0, len(new), n_stream)]
    return logits, teacher, labels, old, new


@pytest.mark.parametrize('N', [1, 10, 20, 110])
@pytest.mark.parametrize('C', [10, 100, 1024])
@pytest.mark.parametrize('with_old', [False, True])
@pytest.mark.parametrize('K_eq_C', [False, True])
def test_icarl_loss_matches_oracle_on_a_seeded_sweep(N, C, with_old, K_eq_C):
    seed = 400 + 7 * N + C + 2 * with_old + K_eq_C
    _check(*_sweep_case(N, C, with_old, K_eq_C, seed), (N, C, with_old, K_eq_C))


def test_icarl_loss_repeat_launches_are_bit_identical():
    logits, teacher, labels, old, new = _sweep_case(110, 100, True, False, 9)
    a = _kernel(logits, teacher, labels, old, new)
    b = _kernel(logits, teacher, labels, old, new)
    assert torch.equal(a['loss'], b['loss']) and torch.equal(a['dlogits'], b['dlogits'])


def test_icarl_loss_flags_labels_outside_the_task():
    """A stream label needs a position in [n_old, K).  The table keeps the earlier tasks' labels at their old positions
    below n_old, as the learner's lbl_inv_map does, so an old label is mapped and must still be refused."""
    old, new = [0, 1, 2], [3, 4]
    logits = np.ones((6, 10), np.float32)
    teacher = np.zeros((6, 10), np.float32)
    # fine; old labels mapped below n_old (position 0 and 2); a negative label; a label beyond the table
    for labels in ([3, 4, 3], [3, 0, 4], [2, 4, 3], [3, -1, 4], [3, 4, 11]):
        err = torch.zeros(1, dtype=torch.int32, device='cuda')
        out = _kernel(logits, teacher, labels, old, new, err, inv={0: 0, 1: 1, 2: 2})
        bad = [i for i, y in enumerate(labels) if y not in new]
        assert int(err) == (1 if bad else 0), labels
        d = out['dlogits'].cpu().numpy()
        for i in bad:
            assert not d[i].any(), labels
        if not bad:
            loss, _ = oic.icarl_loss(logits, labels, old, new, teacher)
            assert abs(float(out['loss']) - loss) <= 1e-5 * loss


def test_icarl_loss_refuses_bad_arguments():
    from b200ocl import _native
    from b200ocl.engine import icarl_loss
    z = torch.zeros(4, 10, device='cuda')
    y = torch.zeros(2, dtype=torch.int64, device='cuda')
    pos = torch.zeros(1, dtype=torch.int64, device='cuda')
    with pytest.raises(_native.NativeError):
        icarl_loss(z, y, pos, 11, 0)                 # K > C
    with pytest.raises(_native.NativeError):
        icarl_loss(z, y, pos, 5, 2)                  # old columns without a teacher
    with pytest.raises(_native.NativeError):
        icarl_loss(z, y, pos, 5, 6, teacher=z)       # n_old > K


def _params(**over):
    flags = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick', 'kd_trick_star')}
    p = dict(data='cifar100', cuda=True, epoch=1, batch=10, verbose=False, mem_size=100, eps_mem_batch=10, mem_iters=1,
             update='random', retrieve='random', agent='ICARL', k=3, aser_type='asvm', n_smp_cls=1.5, num_tasks=5,
             buffer_tracker=False, optimizer='SGD', learning_rate=0.1, weight_decay=0, temp=0.07, head='mlp',
             subsample=20, error_analysis=False, trick=flags)
    p.update(over)
    return SimpleNamespace(**p)


def _agent(params, seed=5):
    from b200ocl import nets, registry
    from oracle import resnet as oresnet
    spec = oresnet.Spec(32, 20, 10 if params.data == 'cifar10' else 100)
    p, bn = oresnet.seeded_state(spec, seed)
    agent = registry.agents['ICARL'](nets.setup_architecture(params), None, params)
    agent.model.engine.load(list(p.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
    return agent


def _task(rs, n, labels):
    return rs.randint(0, 256, (n, 32, 32, 3)).astype(np.uint8), np.asarray(labels, dtype=np.int64)[np.arange(n) % len(labels)]


def test_icarl_refuses_more_positions_than_logits():
    """Labels that recur across tasks count again: the second task over the same 10 labels needs 20 of 10 columns.
    The step refuses before it launches anything."""
    from b200ocl import _native
    agent = _agent(_params(data='cifar10'))
    rs = np.random.RandomState(0)
    agent.train_learner(*_task(rs, 20, range(10)))
    x, y = _task(rs, 10, range(10))
    agent.before_train(x, y)
    bx = torch.rand(10, 3, 32, 32, device='cuda')
    torch.cuda.synchronize()
    before = _native.launch_count()
    with pytest.raises(ValueError, match='exceed'):
        agent.replay_step(bx, torch.from_numpy(y).cuda(), y)
    assert _native.launch_count() == before


def test_icarl_refuses_a_short_memory_draw():
    """A 12-slot memory, 10 slots filled by the first task: the first step of the second task fills the last two and
    writes 8 reservoir draws over the 12 slots, which leaves fewer than 10 slots for the second step to draw from."""
    agent = _agent(_params(mem_size=12))
    torch.manual_seed(0)
    np.random.seed(0)
    rs = np.random.RandomState(1)
    agent.train_learner(*_task(rs, 10, range(5)))
    assert agent.buffer.current_index == 10
    with pytest.raises(ValueError, match='memory rows'):
        agent.train_learner(*_task(rs, 20, range(5, 10)))


@pytest.mark.parametrize('update', ['GSS', 'ASER'])
def test_icarl_refuses_other_update_plugins(update):
    from b200ocl import nets, registry
    params = _params(update=update)
    with pytest.raises(NotImplementedError):
        registry.agents['ICARL'](nets.setup_architecture(params), None, params)


def _run(concurrent):
    from b200ocl import learners
    learners.set_concurrent(concurrent)
    try:
        agent = _agent(_params(epoch=2))
        torch.manual_seed(3)
        np.random.seed(3)
        rs = np.random.RandomState(4)
        x0 = torch.from_numpy(rs.rand(100, 3, 32, 32).astype(np.float32)).cuda()
        agent.buffer.update(x0, torch.from_numpy(rs.randint(0, 100, 100)).cuda())
        losses = []
        for t in range(3):
            agent.train_learner(*_task(rs, 30, range(10 * t, 10 * t + 10)))
            losses.append(float(agent.last_loss))
        torch.cuda.synchronize()
        eng = agent.engine
        return ([eng.state.params.clone(), eng.state.bn_stats.clone(), eng.state.bn_tracked.clone(),
                 eng.teacher.bn_stats.clone(), agent.buffer.buffer_label.clone()], losses)
    finally:
        learners.set_concurrent(True)


def test_icarl_concurrent_teacher_forward_is_bit_identical_to_sequential():
    a, la = _run(True)
    b, lb = _run(False)
    assert la == lb
    for u, v in zip(a, b):
        assert torch.equal(u, v)


class _DropinGolden(dict):
    """The drop-in part of icarl.npz under the key names of dropin.npz."""

    def __init__(self):
        g = np.load(GOLDEN)
        super().__init__((k[len('dropin_'):], g[k]) for k in g.files if k.startswith('dropin_'))


@pytest.mark.parametrize('case', range(int(np.load(GOLDEN)['dropin_n_cases'])))
def test_icarl_dropin_matches_reference_run(case, monkeypatch, tmp_path):
    """test_gpu_dropin's own comparison, fed with these cases."""
    path = str(tmp_path / 'dropin.npz')
    np.savez(path, **_DropinGolden())
    monkeypatch.setattr(dropin, 'GOLDEN', path)
    dropin.test_dropin_matches_reference_run(case)
