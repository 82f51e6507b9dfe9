"""GPU: the training tricks and LwF on the engine.
  * b200ocl_cls_loss against the fp64 oracle on every loss-level golden case of tests/golden/tricks.npz and on a seeded
    sweep, n_correct against the arg-max count, and bit-identical repeat launches;
  * the teacher arena: untouched by the student's SGD, its forward leaves the student's BN statistics alone, matches a
    fresh engine loaded with the same weights, and its graphed replay equals the eager forward;
  * drop-in runs of the trick configurations and of LwF against the reference's (tricks.npz), with the tolerances of
    test_gpu_dropin.py;
  * SCR refuses labels_trick and separated_softmax."""
import json
import os
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import tricks as otr

import test_gpu_dropin as dropin
from test_oracle_tricks import GOLDEN, loss_case

pytestmark = pytest.mark.gpu


def _kernel(logits, labels, kw, want_correct=True):
    from b200ocl.engine import cls_loss
    from b200ocl.learners import separated_softmax_table
    cols = pos = None
    n_old = 0
    if kw['mode'] == 'separated_softmax':
        c, n_old, p = separated_softmax_table(kw['old_labels'], kw['new_labels'], kw['lbl_inv_map'])
        cols, pos = torch.from_numpy(c).cuda(), torch.from_numpy(p).cuda()
    teacher = None if kw.get('teacher') is None else torch.from_numpy(np.ascontiguousarray(kw['teacher'])).cuda()
    err = torch.zeros(1, dtype=torch.int32, device='cuda')
    out = cls_loss(torch.from_numpy(logits).cuda(), torch.from_numpy(labels).cuda(), kw['mode'], cols=cols, n_old=n_old,
                   pos_table=pos, teacher=teacher, w_ce=kw['w_ce'], w_kd=kw['w_kd'], err=err, want_correct=want_correct)
    return out, err


def _check(logits, labels, kw, where):
    out, err = _kernel(logits, labels, kw)
    loss, grad = otr.criterion(logits, labels, **kw)
    got = float(out['loss'])
    assert abs(got - loss) <= 1e-5 * max(abs(loss), 1e-3), (where, got, loss)
    d = out['dlogits'].cpu().numpy()
    assert np.abs(d - grad).max() <= 1e-6 + 1e-5 * np.abs(grad).max(), (where, np.abs(d - grad).max())
    want_hits = int((np.argmax(logits, axis=1) == labels).sum())         # numpy: first maximum, like the kernel
    assert int(out['n_correct']) == want_hits, where
    assert int(err) == 0, where


@pytest.mark.parametrize('k', range(int(np.load(GOLDEN)['n_loss_cases'])))
def test_cls_loss_matches_oracle_on_golden_cases(k):
    g = np.load(GOLDEN)
    logits, labels, kw = loss_case(g, k)
    _check(logits, labels, kw, (k, kw['mode']))


@pytest.mark.parametrize('seed', range(12))
def test_cls_loss_matches_oracle_on_a_seeded_sweep(seed):
    rs = np.random.RandomState(300 + seed)
    C = [10, 100, 37, 200][seed % 4]
    N = [1, 10, 20, 110, 33, 257][seed % 6]
    logits = (rs.standard_normal((N, C)) * rs.uniform(0.5, 8)).astype(np.float32)
    if seed % 3 == 0:            # ties in the arg-max
        logits[:, C // 2] = logits[:, 1] = logits.max(axis=1)
    mode = ['ce', 'labels_trick', 'separated_softmax'][seed % 3]
    kw = dict(mode=mode, teacher=None, w_ce=1.0, w_kd=0.0)
    if mode == 'separated_softmax':
        old = rs.randint(0, C, rs.randint(0, 2 * C)).tolist()
        new = sorted(set(rs.randint(0, C, C // 2).tolist()))
        inv = {}
        for c in sorted(set(old)):
            inv[c] = old.index(c)
        for i, c in enumerate(new):
            inv[c] = len(old) + i
        kw.update(old_labels=old, new_labels=new, lbl_inv_map=inv)
        labels = np.array(sorted(inv))[rs.randint(0, len(inv), N)]
    else:
        labels = rs.randint(0, C, N)
    if seed % 2 == 1:
        kw.update(teacher=(rs.standard_normal((N, C)) * 3).astype(np.float32), w_ce=0.4, w_kd=0.6)
    _check(logits, labels.astype(np.int64), kw, (seed, mode, N, C))


def test_cls_loss_repeat_launches_are_bit_identical():
    rs = np.random.RandomState(9)
    logits = rs.standard_normal((110, 100)).astype(np.float32)
    teacher = rs.standard_normal((110, 100)).astype(np.float32)
    labels = rs.randint(0, 100, 110)
    old, new = list(range(60)) + list(range(30, 80)), list(range(80, 100))
    inv = {c: i for i, c in enumerate(old)}
    inv.update({c: len(old) + i for i, c in enumerate(new)})
    for mode in ('ce', 'labels_trick', 'separated_softmax'):
        kw = dict(mode=mode, teacher=teacher, w_ce=0.25, w_kd=0.75, old_labels=old, new_labels=new, lbl_inv_map=inv)
        a, _ = _kernel(logits, labels, kw)
        b, _ = _kernel(logits, labels, kw)
        assert torch.equal(a['loss'], b['loss']) and torch.equal(a['dlogits'], b['dlogits']), mode
        assert int(a['n_correct']) == int(b['n_correct'])


def test_cls_loss_flags_unmapped_labels():
    logits = np.zeros((4, 10), np.float32)
    kw = dict(mode='separated_softmax', teacher=None, w_ce=1.0, w_kd=0.0, old_labels=[0, 1], new_labels=[2, 3],
              lbl_inv_map={0: 0, 1: 1, 2: 2, 3: 3})
    _, err = _kernel(logits, np.array([0, 1, 2, 3]), kw)
    assert int(err) == 0
    out, err = _kernel(logits, np.array([0, 1, 5, 3]), kw)
    assert int(err) == 1
    assert float(out['dlogits'][2].abs().sum()) == 0.0
    _, err = _kernel(logits, np.array([0, 11, 2, 3]), dict(kw, mode='labels_trick'))
    assert int(err) == 1


def _engine(seed, n_classes=100):
    from b200ocl.engine import Engine
    from oracle import resnet as oresnet
    spec = oresnet.Spec(32, 20, n_classes)
    p, bn = oresnet.seeded_state(spec, seed)
    eng = Engine(32, n_classes)
    eng.load(list(p.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
    return eng


def test_teacher_arena():
    from b200ocl import engine as E
    eng = _engine(61)
    x = torch.rand(10, 3, 32, 32, device='cuda')
    y = torch.randint(0, 100, (10,), device='cuda')
    eng.update_teacher()
    t = eng.teacher
    snap = [a.clone() for a in (t.params, t.packed, t.bn_stats, t.bn_tracked)]
    # the student's SGD leaves the teacher alone
    logits, ws = eng.forward_train(x, slot=0)
    eng.backward(x, E.ce_loss(logits, y)['dlogits'], ws)
    eng.sgd_step(0.1)
    torch.cuda.synchronize()
    for a, b in zip((t.params, t.packed, t.bn_stats, t.bn_tracked), snap):
        assert torch.equal(a, b)
    assert not torch.equal(eng.state.params, t.params)
    # a teacher forward leaves the student's BN statistics bit-unchanged; it equals a fresh engine with the same weights
    fresh = E.Engine(32, 100)
    fresh.state.params.copy_(t.params)
    fresh.state.bn_stats.copy_(t.bn_stats)
    fresh.state.bn_tracked.copy_(t.bn_tracked)
    fresh.pack()
    bn_before = eng.state.bn_stats.clone()
    tracked_before = eng.state.bn_tracked.clone()
    outs = [eng.teacher_forward(x) for _ in range(4)]               # eager, capture, then graph replays
    torch.cuda.synchronize()
    assert torch.equal(eng.state.bn_stats, bn_before) and torch.equal(eng.state.bn_tracked, tracked_before)
    want, _ = fresh.forward_train(x, slot=0, ws=fresh.new_train_workspace(10))     # eager
    for o in outs:
        assert torch.equal(o, want)
    assert ('teacher', 10, eng.TEACHER_SLOT, False) in eng._graphs and eng._graphs[('teacher', 10, eng.TEACHER_SLOT, False)].graphs
    # the teacher's own running statistics moved, as the reference's train-mode copy's do
    assert not torch.equal(t.bn_stats, snap[2])
    # a later update writes the same buffers (captured graphs stay valid) and follows the student
    ptrs = (t.params.data_ptr(), t.packed.data_ptr(), t.bn_stats.data_ptr())
    eng.update_teacher()
    assert (eng.teacher.params.data_ptr(), eng.teacher.packed.data_ptr(), eng.teacher.bn_stats.data_ptr()) == ptrs
    assert torch.equal(eng.teacher.params, eng.state.params)
    student, _ = eng.forward_train(x, slot=0, ws=eng.new_train_workspace(10))
    assert torch.equal(eng.teacher_forward(x), student)


TRICK_GOLDEN = os.path.join(os.path.dirname(GOLDEN), 'tricks.npz')


class _DropinGolden(dict):
    """The drop-in part of tricks.npz under the key names of dropin.npz."""

    def __init__(self):
        g = np.load(TRICK_GOLDEN)
        super().__init__((k[len('dropin_'):], g[k]) for k in g.files if k.startswith('dropin_'))


def _trick_cases():
    return range(int(np.load(TRICK_GOLDEN)['dropin_n_cases']))


@pytest.mark.parametrize('case', _trick_cases())
def test_trick_dropin_matches_reference_run(case, monkeypatch, tmp_path):
    g = _DropinGolden()
    kind = json.loads(str(g['c%d_case' % case]))[0]
    if kind == 'lwf':
        _lwf_dropin(g, case)
        return
    # the memory-based agents: test_gpu_dropin's own comparison, fed with these cases
    path = str(tmp_path / 'dropin.npz')
    np.savez(path, **g)
    monkeypatch.setattr(dropin, 'GOLDEN', path)
    dropin.test_dropin_matches_reference_run(case)


def _lwf_dropin(g, case):
    """LwF has no memory: the same script without the buffer fill and buffer checks."""
    from b200ocl import memory, nets, registry
    from oracle import resnet as oresnet
    tag = 'c%d_' % case
    kind, n_calls, n_label, wseed, seed, dseed = json.loads(str(g[tag + 'case']))
    params = SimpleNamespace(**json.loads(str(g[tag + 'params'])))
    spec = oresnet.Spec(32, 20, 10 if params.data == 'cifar10' else 100)
    memory.set_mode(True, 'cpu')
    try:
        agent = registry.agents[params.agent](nets.setup_architecture(params), None, params)
        assert not hasattr(agent, 'buffer')
        p, bn = oresnet.seeded_state(spec, wseed)
        agent.model.engine.load(list(p.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])
        w0 = torch.cat([t.reshape(-1) for t in p.values()]).numpy()
        pick = dropin.dropin_sample(w0.size)
        w0 = w0[pick].astype(np.float64)
        np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
        rs = np.random.RandomState(dseed)
        x, y, calls, tests = dropin.dropin_inputs(rs, params.mem_size, 32, n_label, params.batch, n_calls)
        for c, (xt, yt) in enumerate(calls):
            agent.train_learner(xt, yt)
            torch.cuda.synchronize()
            w = agent.engine.state.params.cpu().numpy()[pick]
            err = dropin._rel(w - w0, g[tag + 'w%d' % c].astype(np.float64) - w0)
            assert err <= max(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_w'][c]), (case, c, err)
            err = dropin._rel(agent.engine.state.bn_stats.cpu().numpy(), g[tag + 'bn%d' % c].astype(np.float64))
            assert err <= max(dropin.BN_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_bn'][c]), (case, c, err)
        loaders = [[(torch.from_numpy(tx).permute(0, 3, 1, 2).float().div(255), torch.from_numpy(ty))] for tx, ty in tests]
        acc = np.asarray(agent.evaluate(loaders))
        assert np.abs(acc - g[tag + 'acc']).max() <= 3.1 / 96, (case, acc, g[tag + 'acc'])
    finally:
        memory.set_mode(False)


def _scr_params(trick):
    flags = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick', 'kd_trick_star')}
    flags[trick] = True
    return SimpleNamespace(data='cifar100', cuda=True, epoch=1, batch=10, verbose=False, mem_size=200, eps_mem_batch=100,
                           mem_iters=1, update='random', retrieve='random', agent='SCR', k=3, aser_type='asvm',
                           n_smp_cls=1.5, num_tasks=5, buffer_tracker=False, optimizer='SGD', learning_rate=0.1,
                           weight_decay=0, temp=0.07, head='mlp', subsample=20, error_analysis=False, trick=flags)


@pytest.mark.parametrize('trick', ['labels_trick', 'separated_softmax'])
def test_scr_refuses_ce_tricks(trick):
    from b200ocl import nets, registry
    params = _scr_params(trick)
    with pytest.raises(NotImplementedError):
        registry.agents['SCR'](nets.setup_architecture(params), None, params)


def test_scr_accepts_kd_trick_without_a_teacher():
    from b200ocl import nets, registry
    params = _scr_params('kd_trick')
    agent = registry.agents['SCR'](nets.setup_architecture(params), None, params)
    assert not agent._takes_teacher
