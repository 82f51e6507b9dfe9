"""CPU: GDumb's host side against the reference's own code (tests/golden/gdumb.npz, written by
tests/golden/make_golden_gdumb.py): the re-initialisation nets.reference_init draws (digest, sample and generator
position, bit for bit), the greedy class-balanced memory planner (mem_c order, per-class lists and Python generator
position, exactly), the fp64 clip of oracle/gdumb.py against torch.nn.utils.clip_grad_norm_, the construction refusals,
and the registration of agents['GDUMB'] by the drop-in switch."""
import hashlib
import os
import random
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import gdumb as ogd

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'gdumb.npz')


@pytest.mark.parametrize('k', range(int(np.load(GOLDEN)['n_init'])))
def test_reference_init_draws_what_setup_architecture_draws(k):
    from b200ocl import memory, nets
    g = np.load(GOLDEN)
    tag = 'init%d_' % k
    data = str(g[tag + 'data'])
    torch.manual_seed(int(g[tag + 'seed']))
    flat = torch.cat([t.reshape(-1) for t in nets.reference_init(data, memory.n_classes[data],
                                                                 memory.input_size_match[data][1])]).numpy()
    assert hashlib.sha1(flat.tobytes()).hexdigest() == str(g[tag + 'sha1']), data
    pick = np.sort(np.random.RandomState(7).choice(flat.size, 2048, replace=False))
    assert np.array_equal(flat[pick], g[tag + 'sample']), data
    assert np.array_equal(torch.rand(4).numpy(), g[tag + 'after']), data


def test_reference_init_matches_the_engine_layout():
    from b200ocl import nets
    for hw, dim_in in ((32, 160), (84, 640)):
        assert nets.reduced_resnet_dim_in(hw) == dim_in
        shapes = [tuple(t.shape) for t in nets.reference_init('mini_imagenet' if hw == 84 else 'cifar100', 100, hw)]
        assert shapes == [sh for _, sh in nets.param_layout(dim_in, 100)]


def _replay_greedy(g, k):
    """The planner over the golden streams: (mem_c items, per-class source lists concatenated, random.random())."""
    from b200ocl import memory
    tag = 'greedy%d_' % k
    mem = memory.GreedyBalancedMemory(int(g[tag + 'mem']), 4, 'cpu')
    src_of_slot = np.full(mem.mem_size, -1, dtype=np.int64)
    random.seed(int(g[tag + 'seed']))
    base = 0
    for s in range(int(g[tag + 'n_streams'])):
        y = g[tag + 'stream%d' % s]
        slots, sources = mem.plan(y)
        src_of_slot[slots] = base + sources
        base += y.size
    lists = [int(src_of_slot[sl]) for c in mem.mem_c for sl in mem.slots[c]]
    return mem, np.array(list(mem.mem_c.items()), dtype=np.int64).reshape(-1, 2), np.array(lists), random.random()


@pytest.mark.parametrize('k', range(int(np.load(GOLDEN)['n_greedy'])))
def test_greedy_planner_matches_reference(k):
    g = np.load(GOLDEN)
    tag = 'greedy%d_' % k
    mem, mem_c, lists, after = _replay_greedy(g, k)
    assert np.array_equal(mem_c, g[tag + 'mem_c']), (mem_c, g[tag + 'mem_c'])
    assert np.array_equal(lists, g[tag + 'lists'])
    assert after == float(g[tag + 'after'])
    assert len(mem) == int(mem_c[:, 1].sum()) <= mem.mem_size
    order = mem.order()
    assert order.size == len(mem) and np.unique(order).size == order.size


def test_greedy_golden_covers_the_cases():
    g = np.load(GOLDEN)
    seen = set()
    for k in range(int(g['n_greedy'])):
        tag = 'greedy%d_' % k
        n = sum(g[tag + 'stream%d' % s].size for s in range(int(g[tag + 'n_streams'])))
        m, counts = int(g[tag + 'mem']), g[tag + 'mem_c'][:, 1]
        seen.add('short' if n < m else 'long' if n >= 10 * m else 'mid')
        if (counts == 0).any():
            seen.add('zero')
        if int(g[tag + 'n_streams']) > 1:
            seen.add('calls')
    assert {'short', 'long', 'zero', 'calls'} <= seen


def test_planner_keeps_the_last_source_of_a_slot_written_twice():
    """Memory 2: the third sample of a new class evicts one of the two slots the pass wrote; that slot is planned once,
    with the later source."""
    from b200ocl import memory
    mem = memory.GreedyBalancedMemory(2, 4, 'cpu')
    random.seed(0)
    slots, sources = mem.plan([0, 0, 1])
    assert sorted(slots.tolist()) == [0, 1] and 2 in sources.tolist() and len(set(sources.tolist())) == 2
    assert list(mem.mem_c.items()) == [(0, 1), (1, 1)]


def test_oracle_clip_matches_clip_grad_norm():
    rs = np.random.RandomState(3)
    shapes = [(20, 3, 3, 3), (20,), (100, 160), (100,)]
    for max_norm in (0.5, 10.0, 1e6):
        ps = [torch.nn.Parameter(torch.zeros(s, dtype=torch.float64)) for s in shapes]
        grads = [rs.standard_normal(s) for s in shapes]
        for p, gr in zip(ps, grads):
            p.grad = torch.from_numpy(gr.copy())
        norm = torch.nn.utils.clip_grad_norm_(ps, max_norm)
        clipped, onorm = ogd.clip_grads(grads + [None], max_norm)
        assert abs(onorm - float(norm)) <= 1e-12 * onorm
        assert clipped[-1] is None
        for p, c in zip(ps, clipped):
            np.testing.assert_allclose(c, p.grad.numpy(), rtol=1e-13, atol=0)
        if max_norm > onorm:
            assert all(np.array_equal(c, gr) for c, gr in zip(clipped, grads))


def _params(**over):
    flags = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick', 'kd_trick_star')}
    p = dict(data='cifar100', cuda=True, epoch=1, batch=10, verbose=False, mem_size=100, eps_mem_batch=10, mem_iters=1,
             update='random', retrieve='random', agent='GDUMB', optimizer='SGD', learning_rate=0.01, weight_decay=0,
             mem_epoch=2, clip=10.0, minlr=0.0005, error_analysis=False, trick=flags)
    p.update(over)
    return SimpleNamespace(**p)


def test_gdumb_refuses_adam_and_ncm_trick_before_building_anything():
    """Checked before the base constructor, so no model or device is touched (model=None would fail there)."""
    from b200ocl import registry
    with pytest.raises(NotImplementedError, match='SGD'):
        registry.agents['GDUMB'](None, None, _params(optimizer='Adam'))
    trick = dict(_params().trick, ncm_trick=True)
    with pytest.raises(NotImplementedError, match='ncm_trick'):
        registry.agents['GDUMB'](None, None, _params(trick=trick))


def test_install_registers_and_removes_gdumb():
    from b200ocl import registry
    import test_install
    for has_ref_gdumb in (False, True):
        nm, mods = test_install._stub_reference()
        ewc = nm.agents['EWC']
        if has_ref_gdumb:
            nm.agents['GDUMB'] = ref = object()
        saved = {k: sys.modules.get(k) for k in mods}
        sys.modules.update(mods)
        try:
            registry.install(nm)
            assert nm.agents['GDUMB'] is registry.agents['GDUMB']
            assert registry.agents['GDUMB'].__module__.startswith('b200ocl')
            assert nm.agents['EWC'] is ewc
            registry.uninstall(nm)
            if has_ref_gdumb:
                assert nm.agents['GDUMB'] is ref
            else:
                assert 'GDUMB' not in nm.agents
            assert nm.agents['EWC'] is ewc
        finally:
            for k, v in saved.items():
                if v is None:
                    sys.modules.pop(k, None)
                else:
                    sys.modules[k] = v
