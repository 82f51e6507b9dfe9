"""CPU: oracle/agem.py, the fp64 A-GEM step, against the per-parameter list form of agents/agem.py:71-80 (prod as a
sum of per-tensor sums, the projection per tensor), written here directly in torch float64: the projection alone on
edge rows, and whole steps with both decisions; AdamState against torch.optim.Adam; and the step against the
reference's own A-GEM runs at 84x84 and 128x128 (tests/golden/agem_maps.npz, written by
tests/golden/make_golden_agem_maps.py) on their first calls."""
import copy
import json
import os

import numpy as np
import pytest
import torch

from oracle import agem as oagem
from oracle import replay_step as ors
from oracle import resnet as oresnet

import test_gpu_agem_fp64 as tg


def list_project(grad, grad_ref):
    """agem.py:72-80 on per-parameter float64 tensors."""
    prod = sum([torch.sum(g * g_r) for g, g_r in zip(grad, grad_ref)])
    if prod < 0:
        prod_ref = sum([torch.sum(g_r ** 2) for g_r in grad_ref])
        grad = [g - prod / prod_ref * g_r for g, g_r in zip(grad, grad_ref)]
    return grad, bool(prod < 0)


def _tensors(rs, shapes, scale=1.0):
    return [torch.from_numpy(rs.standard_normal(s) * scale) for s in shapes]


@pytest.mark.parametrize('case', ['negative', 'positive', 'zero_ref', 'disjoint', 'opposite', 'tiny'])
def test_project_matches_list_form(case):
    rs = np.random.RandomState(5)
    shapes = [(20, 3, 3, 3), (20,), (40, 20, 3, 3), (100, 160), (100,)]
    g, r = _tensors(rs, shapes), _tensors(rs, shapes, 0.5)
    if case == 'negative':
        g = [a - 3 * b for a, b in zip(g, r)]
    elif case == 'positive':
        g = [a + 3 * b for a, b in zip(g, r)]
    elif case == 'zero_ref':
        r = [torch.zeros_like(b) for b in r]
    elif case == 'disjoint':
        r = [b * (torch.arange(b.numel()).reshape(b.shape) % 2) for b in r]
        g = [a * (1 - torch.arange(a.numel()).reshape(a.shape) % 2) for a in g]
    elif case == 'opposite':
        g = [-b for b in r]
    elif case == 'tiny':
        g, r = [torch.zeros_like(a) for a in g], [torch.zeros_like(b) for b in r]
        g[2][0, 0, 0, 0], r[2][0, 0, 0, 0] = -1e-15, 1e-15
        r[3][1, 1] = 1.0
    want, proj = list_project(g, r)
    out, prod, prod_ref, got = oagem.project(torch.cat([a.reshape(-1) for a in g]).numpy(),
                                             torch.cat([b.reshape(-1) for b in r]).numpy())
    assert got == proj == (case in ('negative', 'opposite', 'tiny'))
    want = torch.cat([a.reshape(-1) for a in want]).numpy()
    assert np.all(np.isfinite(out))
    np.testing.assert_allclose(out, want, rtol=1e-13, atol=1e-13 * np.abs(want).max() + 1e-300)
    if case == 'opposite':
        assert np.abs(out).max() <= 1e-14 * np.abs(want).max() + 1e-15
    if case in ('zero_ref', 'disjoint'):
        assert prod == 0.0


def _state(spec, seed, mem_size, lr):
    p, bn = oresnet.seeded_state(spec, seed, dtype=torch.float64)
    return ors.ReplayState(spec, p, bn, mem_size, (3, spec.in_hw, spec.in_hw), spec.num_classes, lr=lr)


def _list_step(st, x, y, task_seen, eps_mem_batch):
    """agem.py:39-83 for one memory iteration with plain CE and SGD, per parameter, on st."""
    x = x.double()
    _, _, grads = oresnet.ce_loss_and_grads(st.spec, st.params, st.bn, x, y)
    names = list(grads)
    proj = None
    if task_seen > 0:
        idx = ors._random_indices(st, eps_mem_batch)
        if idx.size:
            grad = [grads[k].clone() for k in names]
            _, _, gr = oresnet.ce_loss_and_grads(st.spec, st.params, st.bn, st.buffer_img[idx].double(), st.buffer_label[idx])
            grad, proj = list_project(grad, [gr[k] for k in names])
            grads = dict(zip(names, grad))
    oresnet.sgd_step(st.params, grads, st.lr)
    ors._reservoir_update(st, x.float(), y, None)
    return proj


def test_step_matches_list_form():
    """Whole steps of oracle.agem.step against the per-parameter form: the same draws, decisions, parameters, running
    statistics and memory.  Both decisions occur."""
    spec = oresnet.Spec(32, 20, 100)
    a, b = _state(spec, 41, 10, 0.1), None
    rs = np.random.RandomState(42)
    seen = set()
    for i, kind in enumerate(('fill', 'fill', 'neg', 'pos', 'neg')):
        task_seen = int(kind != 'fill')
        np.random.seed(700 + i)
        x, y = tg._batch(rs, a, kind, 32, ors._random_indices(a, 10) if task_seen else None)
        b = copy.deepcopy(a)
        np.random.seed(700 + i); torch.manual_seed(700 + i)
        logs = oagem.step(a, x, y, task_seen)
        np.random.seed(700 + i); torch.manual_seed(700 + i)
        proj = _list_step(b, x, y, task_seen, 10)
        assert logs[0]['project'] == proj, i
        seen.add(proj)
        for k in a.params:
            np.testing.assert_allclose(a.params[k].numpy(), b.params[k].numpy(), rtol=1e-12, atol=1e-14, err_msg=k)
        for k in a.bn:
            np.testing.assert_allclose(a.bn[k].numpy(), b.bn[k].numpy(), rtol=1e-12, atol=1e-14, err_msg=k)
        assert torch.equal(a.buffer_label, b.buffer_label) and torch.equal(a.buffer_img, b.buffer_img)
    assert seen == {None, True, False}


def test_step_logs_what_it_projects():
    """The log's vectors are the flat gradients in parameter order, the projection is project()'s, and a memory smaller
    than eps_mem_batch replays every stored row."""
    spec = oresnet.Spec(32, 20, 100)
    st = _state(spec, 33, 4, 0.1)
    rs = np.random.RandomState(34)
    x = torch.from_numpy(rs.rand(10, 3, 32, 32).astype(np.float32))
    np.random.seed(1); torch.manual_seed(1)
    oagem.step(st, x, torch.from_numpy(rs.randint(0, 5, 10)), 0)
    assert st.current_index == 4
    x = torch.from_numpy(rs.rand(10, 3, 32, 32).astype(np.float32))
    np.random.seed(2); torch.manual_seed(2)
    log, = oagem.step(st, x, torch.from_numpy(rs.randint(5, 10, 10)), 1)
    assert sorted(log['ret_idx'].tolist()) == [0, 1, 2, 3]
    n = sum(int(np.prod(s)) for s in oresnet.param_shapes(spec).values())
    assert log['g'].shape == log['g_ref'].shape == (n,)
    out, prod, prod_ref, proj = oagem.project(log['g'], log['g_ref'])
    assert (prod, prod_ref, proj) == (log['prod'], log['prod_ref'], log['project'])
    assert np.array_equal(out, log['out'])


def test_adam_state_matches_torch_adam():
    """AdamState against torch.optim.Adam in float64 over three steps, with and without weight decay."""
    rs = np.random.RandomState(9)
    for wd in (0.0, 0.01):
        params = {k: torch.from_numpy(rs.standard_normal(s)) for k, s in (('a', (4, 3)), ('b', (5,)))}
        leaves = [v.clone().requires_grad_(True) for v in params.values()]
        opt = torch.optim.Adam(leaves, lr=1e-3, weight_decay=wd)
        mine = oagem.AdamState(1e-3, weight_decay=wd)
        for _ in range(3):
            grads = {k: torch.from_numpy(rs.standard_normal(tuple(v.shape))) for k, v in params.items()}
            for leaf, gr in zip(leaves, grads.values()):
                leaf.grad = gr.clone()
            opt.step()
            mine.step(params, grads)
            for leaf, v in zip(leaves, params.values()):
                np.testing.assert_allclose(v.numpy(), leaf.detach().numpy(), rtol=1e-13, atol=1e-15)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'agem_maps.npz')
REF_CALLS = 2         # the first calls: one without a memory draw (task_seen = 0), one with


@pytest.mark.parametrize('data', ['mini_imagenet', 'core50'])
def test_step_matches_reference_run(data):
    """oracle.agem.step in float64 against the reference's own run (tests/golden/agem_maps.npz) on its first calls,
    with the loader order and the memory slots the reference drew: the drop-in bars on the sampled weight update and
    the BN statistics, the reference's stream and memory gradients (sampled) and dot products, and its decision.
    Between calls the memory is rebuilt from the recorded slot sources, whose labels must be the reference's."""
    import test_gpu_dropin as dropin
    g = np.load(GOLDEN)
    tag = data + '_'
    _, n_calls, wseed, seed, dseed = json.loads(str(g[tag + 'case']))
    params = json.loads(str(g[tag + 'params']))
    hw, ncls = tg.NETS[data]
    spec = tg.spec_of(data)
    st = _state(spec, wseed, params['mem_size'], params['learning_rate'])
    x, y, calls, _ = oagem.dropin_inputs(np.random.RandomState(dseed), params['mem_size'], hw, params['batch'], n_calls)
    st.buffer_img[:] = torch.from_numpy(x)
    st.buffer_label[:] = torch.from_numpy(y)
    st.current_index = st.n_seen_so_far = params['mem_size']
    w0 = oagem.flat(st.params)
    pick = dropin.dropin_sample(w0.size)
    w0 = w0[pick]
    images = [torch.from_numpy(xt).permute(0, 3, 1, 2).float().div(255) for xt, _ in calls]
    for c in range(REF_CALLS):
        perm = g[tag + 'perm%d' % c]
        xb, yb = images[c][perm], torch.from_numpy(calls[c][1][perm])
        ret = [g[tag + 'ret%d' % c]] if c else None
        log, = oagem.step(st, xb, yb, c, eps_mem_batch=params['eps_mem_batch'], ret_idx=ret)
        w = oagem.flat(st.params)[pick]
        err = dropin._rel(w - w0, g[tag + 'w%d' % c].astype(np.float64) - w0)
        assert err <= max(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_w'][c]), (data, c, 'update', err)
        err = dropin._rel(tg._bn_flat_oracle(st), g[tag + 'bn%d' % c].astype(np.float64))
        assert err <= max(dropin.BN_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_bn'][c]), (data, c, 'BN', err)
        if c:
            # each sampled gradient within the drop-in bar of its own one-ulp spread; the dots within twice the larger
            # of the two gradients' bars times |g| |g_ref|
            tol = 0.0
            for k, key in (('g', 'g'), ('g_ref', 'gref'), ('out', 'out')):
                bar = max(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * g[tag + 'spread_' + key][c])
                err = dropin._rel(log[k][pick], g[tag + key + '%d' % c].astype(np.float64))
                assert err <= bar, (data, c, k, err, bar)
                tol = max(tol, bar) if k != 'out' else tol
            P, R = g[tag + 'dots%d' % c]
            bar = 2 * tol * np.linalg.norm(log['g']) * np.linalg.norm(log['g_ref'])
            assert abs(log['prod'] - P) <= bar and abs(log['prod_ref'] - R) <= 2 * tol * R, (data, c, P, log['prod'])
            assert abs(P) > bar and log['project'] == bool(g[tag + 'proj%d' % c])
        src = g[tag + 'src%d' % c]
        for sl, s in enumerate(src.tolist()):
            st.buffer_img[sl] = torch.from_numpy(x[s]) if s < 1000 else images[s // 1000 - 1][s % 1000]
            st.buffer_label[sl] = int(y[s] if s < 1000 else calls[s // 1000 - 1][1][s % 1000])
        np.testing.assert_array_equal(st.buffer_label.numpy(), g[tag + 'label%d' % c])
        st.n_seen_so_far = int(g[tag + 'seen%d' % c])
