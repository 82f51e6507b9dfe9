"""CPU: GEM's oracle (oracle/gem.py), the launch plan of b200ocl_gem_project, the refusals of learners.GEM and its
registration.

  * The QP oracle (active-set search, final free set solved directly) against enumeration of every free set with a KKT
    check and against scipy.optimize.nnls on the Cholesky form (A = L^T, b = -L^-1 c of H = L L^T), at t = 1 ... 10,
    margins 0 and 0.5, on random, duplicate-row, zero-row and near-parallel G.
  * The ring bookkeeping (oracle.gem.Rings and memory.TaskRingMemory on CPU tensors) against a plain restatement of
    the authors' rule: batches that do not divide M, a task shorter than M, a batch larger than M.
  * b200ocl_gem_plan at 132, 114, 60 and 16 SMs for t = 1 ... 64 and the four arena lengths: the partials fit the
    workspace, every CTA has columns, the grid covers n exactly, the shared memory fits one SM.
  * Every refusal at construction, before anything is allocated; the 64-task limit; registration."""
import math
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.optimize
import torch

from oracle import gem as ogem

ARENAS = {'cifar100': 1109240, 'mini_imagenet': 1157240, 'openloris': 1104249, 'core50': 1221190}


def _G(kind, t, n, rs):
    G = rs.standard_normal((t, n))
    if kind == 'duplicate' and t > 1:
        G[t // 2] = G[0]
    elif kind == 'zero':
        G[t - 1] = 0.0
    elif kind == 'parallel' and t > 1:
        G[1] = G[0] * 1.5 + 1e-7 * rs.standard_normal(n)
    return G


def _problem(kind, t, seed):
    rs = np.random.RandomState(seed)
    n = 40
    G = _G(kind, t, n, rs)
    g = rs.standard_normal(n) - 0.5 * G.sum(axis=0)          # conflicts with several rows
    return ogem.gram(G, g)


def _nnls(P, q, margin):
    H = np.asarray(P) + ogem.EPS * np.eye(len(q))
    c = np.asarray(q) + margin * H.sum(axis=1)
    L = np.linalg.cholesky(H)
    w, _ = scipy.optimize.nnls(L.T, -np.linalg.solve(L, c), maxiter=1000)
    return w + margin


@pytest.mark.parametrize('kind', ['random', 'duplicate', 'zero', 'parallel'])
@pytest.mark.parametrize('margin', [0.0, 0.5])
@pytest.mark.parametrize('t', list(range(1, 11)))
def test_qp_oracle_against_enumeration_and_nnls(kind, margin, t):
    P, q = _problem(kind, t, 100 * t + len(kind))
    v = ogem.solve_qp(P, q, margin)
    assert np.all(v >= margin) and np.all(v[v == margin] == margin)
    H = P + ogem.EPS * np.eye(t)
    c = q + margin * H.sum(axis=1)
    scale = np.abs(c).max() + np.abs(H).max() * max((v - margin).max(), 1.0)
    pr, du, co = ogem.kkt_residuals(H, c, v - margin)
    assert pr == 0.0 and du <= 1e-9 * scale and co <= 1e-9 * scale * max((v - margin).max(), 1.0), (pr, du, co)
    ve = ogem.solve_qp_enumerate(P, q, margin)
    vn = _nnls(P, q, margin)
    f, fe, fn = ogem.objective(P, q, v), ogem.objective(P, q, ve), ogem.objective(P, q, vn)
    assert abs(f - fe) <= 1e-12 * max(abs(fe), 1.0) and abs(f - fn) <= 1e-10 * max(abs(fn), 1.0), (f, fe, fn)
    cond = np.linalg.cond(H)
    if cond < 1e6:
        assert np.abs(v - ve).max() <= 1e-9 * max(np.abs(ve).max(), 1.0)
        assert np.abs(v - vn).max() <= 1e-7 * max(np.abs(vn).max(), 1.0)


def test_qp_with_no_conflict_keeps_the_margin():
    """q > 0 everywhere: the oracle's project leaves g alone; the QP itself still has its solution at or above margin."""
    G = np.eye(3, 5)
    g = np.ones(5)
    out, v, flag = ogem.project(G, g)
    assert not flag and np.array_equal(out, g) and np.all(v == 0)


def test_orthogonal_pair_is_no_conflict():
    G = np.array([[1.0, 0.0, 0.0]])
    g = np.array([0.0, 2.0, 0.0])
    out, v, flag = ogem.project(G, g)
    assert not flag and np.array_equal(out, g)


def test_projection_satisfies_the_constraint():
    rs = np.random.RandomState(4)
    G = rs.standard_normal((6, 50))
    g = -G.sum(axis=0)
    out, v, flag = ogem.project(G, g, margin=0.0)
    assert flag
    assert (G @ out + ogem.EPS * v).min() >= -1e-9 * np.abs(G @ g).max()


# ----------------------------------------------------------------------------- rings
def _restated(M, batches):
    """Plain restatement: (start, count) per batch, filled count."""
    cnt, pos, seen = 0, [], 0
    for b in batches:
        end = cnt + b
        if end > M:
            end = M
        pos.append((cnt, end - cnt))
        seen += end - cnt
        cnt = end
        if cnt == M:
            cnt = 0
    return pos, min(seen, M)


@pytest.mark.parametrize('M,batches', [(25, [10] * 7), (30, [10] * 3), (250, [10] * 30), (40, [10, 10]),
                                       (7, [10, 10, 3]), (5, [10]), (12, [5, 5, 5, 5, 5])],
                         ids=['not_dividing', 'dividing', 'cifar', 'short_task', 'batch_larger', 'one_large', 'fives'])
def test_ring_bookkeeping_matches_the_restatement(M, batches):
    from b200ocl import memory
    want_pos, want_filled = _restated(M, batches)
    assert ogem.ring_positions(M, batches) == (want_pos, want_filled)
    rings = ogem.Rings(M, (3, 2, 2))
    mem = memory.TaskRingMemory(M, 2, 'cpu')
    rs = np.random.RandomState(M)
    truth = np.full(M, -1)
    for task in range(2):
        rings.begin_task(task)
        mem.begin_task(task)
        for b, (s, k) in zip(batches, want_pos):
            x = torch.tensor(rs.rand(b, 3, 2, 2).astype(np.float32))
            y = torch.arange(b) + 100 * task
            assert rings.write(task, x, y) == (s, k)
            assert mem.write(task, x, y, y.numpy()) == (s, k)
            if task == 1:
                truth[s:s + k] = y[:k].numpy()
        assert rings.filled[task] == mem.filled[task] == want_filled
    assert np.array_equal(rings.labels[1][:want_filled].numpy(), truth[:want_filled])
    assert np.array_equal(mem.labels[1][:want_filled].numpy(), truth[:want_filled])
    assert np.array_equal(mem.labels_host[1][:want_filled], truth[:want_filled])
    assert torch.equal(mem.images[1], rings.images[1])


def test_ring_counter_restarts_with_every_task():
    from b200ocl import memory
    mem = memory.TaskRingMemory(25, 2, 'cpu')
    mem.begin_task(0)
    for _ in range(3):
        mem.write(0, torch.zeros(10, 3, 2, 2), torch.zeros(10, dtype=torch.int64), np.zeros(10))
    assert mem.cnt[0] == 0 and mem.filled[0] == 25           # 10, 20, then 5 rows to the end
    mem.write(0, torch.zeros(10, 3, 2, 2), torch.zeros(10, dtype=torch.int64), np.zeros(10))
    assert mem.cnt[0] == 10
    mem.begin_task(2)
    assert len(mem) == 3 and mem.filled[1] == 0 and mem.cnt[2] == 0
    mem.begin_task(0)
    assert mem.cnt[0] == 0 and mem.filled[0] == 25


def test_memory_snapshot_round_trip():
    from b200ocl import memory
    mem = memory.TaskRingMemory(8, 2, 'cpu')
    rs = np.random.RandomState(0)
    for task in range(3):
        mem.begin_task(task)
        if task != 1:
            y = torch.tensor(rs.randint(0, 9, 5))
            mem.write(task, torch.tensor(rs.rand(5, 3, 2, 2).astype(np.float32)), y, y.numpy())
    snap = mem.snapshot()
    back = memory.TaskRingMemory(8, 2, 'cpu')
    back.restore(snap)
    assert back.filled == mem.filled and back.cnt == mem.cnt
    for k in range(3):
        assert torch.equal(back.images[k], mem.images[k]) and torch.equal(back.labels[k], mem.labels[k])
    assert sorted(snap['images']) == [0, 2]
    with pytest.raises(ValueError):
        memory.TaskRingMemory(9, 2, 'cpu').restore(snap)


# ----------------------------------------------------------------------------- the launch plan
@pytest.mark.parametrize('sms', [132, 114, 60, 16])
@pytest.mark.parametrize('data', list(ARENAS))
def test_plan_fits_and_covers_every_column(sms, data):
    from b200ocl import _build, ops
    _build.build()
    n = ARENAS[data]
    for t in range(1, 65):
        L = ops.gem_plan(t, n, sms)
        assert L.sms == sms and L.rows == t + 1 and L.pairs == (t + 1) * (t + 2) // 2
        assert L.rows_padded % 4 == 0 and L.rows_padded >= L.rows and L.row_blocks * 4 == L.rows_padded
        assert 1 <= L.block_pairs * L.lanes <= 256 and L.lanes >= 1
        assert L.tile_cols % 4 == 0 and L.tile_stride >= L.tile_cols
        assert L.smem_bytes >= 2 * L.rows_padded * L.tile_stride * 4 and L.smem_bytes >= 256 * 16 * 8
        assert L.smem_bytes <= 227 * 1024
        assert L.part_bytes == L.grid * L.pairs * 8 <= L.workspace_bytes
        assert 1 <= L.grid <= 2 * sms
        assert (L.grid - 1) * L.chunk < n <= L.grid * L.chunk          # every CTA has columns, all are covered
        assert L.tiles_per_cta == -(-L.chunk // L.tile_cols)
        assert 1 <= L.proj_grid <= 4 * sms


def test_plan_at_small_lengths_and_refusals():
    from b200ocl import _native, ops
    for n in (1, 31, 32, 33, 1023, 1024, 1025):
        for t in (1, 5, 64):
            L = ops.gem_plan(t, n, 132)
            assert (L.grid - 1) * L.chunk < n <= L.grid * L.chunk
    for t, n in ((0, 10), (65, 10), (1, 0)):
        with pytest.raises(_native.NativeError):
            ops.gem_plan(t, n, 132)
    lib = _native.lib()
    assert lib.b200ocl_gem_project_workspace_bytes(0, 10) == 0
    assert lib.b200ocl_gem_project_workspace_bytes(65, 10) == 0


def test_workspace_query_is_the_plans_at_the_device_count():
    from b200ocl import _native, ops
    lib = _native.lib()
    for t in (1, 19, 64):
        assert lib.b200ocl_gem_project_workspace_bytes(t, 1109240) == ops.gem_plan(t, 1109240).workspace_bytes


# ----------------------------------------------------------------------------- refusals and registration
def _params(**kw):
    trick = {k: False for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick',
                                'kd_trick_star')}
    base = dict(data='cifar100', cuda=True, epoch=1, batch=10, verbose=False, mem_size=100, eps_mem_batch=10,
                mem_iters=1, update='random', retrieve='random', agent='GEM', optimizer='SGD', learning_rate=0.1,
                weight_decay=0, error_analysis=False, num_tasks=5, trick=trick)
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
        learners.GEM(_NoModel(), None, _params(**kw))


@pytest.mark.parametrize('value', [-0.1, float('nan'), float('inf'), '0.5x', True, [0.1]])
def test_margin_must_be_finite_and_non_negative(value):
    from b200ocl import learners
    with pytest.raises(ValueError, match='gem_margin'):
        learners.GEM(_NoModel(), None, _params(gem_margin=value))


def test_margin_defaults_and_is_read_as_float():
    from b200ocl import learners
    assert learners.gem_margin(_params()) == 0.5
    assert learners.gem_margin(_params(gem_margin=0)) == 0.0
    assert learners.gem_margin(_params(gem_margin='1.5')) == 1.5


@pytest.mark.parametrize('mem_size,num_tasks', [(4, 5), (0, 5), (19, 20)])
def test_no_row_per_task_is_refused(mem_size, num_tasks):
    from b200ocl import learners
    with pytest.raises(ValueError, match='num_tasks'):
        learners.GEM(_NoModel(), None, _params(mem_size=mem_size, num_tasks=num_tasks))


def test_more_than_64_earlier_tasks_is_refused_before_anything_runs():
    from b200ocl import learners
    agent = learners.GEM.__new__(learners.GEM)
    torch.nn.Module.__init__(agent)
    agent.task_seen = 65
    with pytest.raises(ValueError, match='64'):
        agent.train_learner(np.zeros((10, 32, 32, 3), np.uint8), np.zeros(10, np.int64))


def test_data_parallel_step_is_refused():
    from b200ocl import learners
    agent = learners.GEM.__new__(learners.GEM)
    torch.nn.Module.__init__(agent)
    agent.grad_sync = lambda eng: None
    with pytest.raises(NotImplementedError, match='data-parallel'):
        agent.replay_step(None, None, None)


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


def test_install_registers_gem_only_on_request():
    from b200ocl import registry

    def check(nm):
        assert 'GEM' not in nm.agents
        registry.install(nm)
        assert 'GEM' not in nm.agents                                     # not by default
        registry.uninstall(nm)
        import b200ocl
        b200ocl.install(nm, extra=('GEM',))
        assert nm.agents['GEM'] is registry.extra_agents['GEM']
        assert registry.extra_agents['GEM'].__name__ == 'GEM'
        assert registry.extra_agents['GEM'].__module__.startswith('b200ocl')
        assert registry.installed_extra == ('GEM',)
        registry.uninstall(nm)
        assert 'GEM' not in nm.agents and registry.installed_extra == ()
        b200ocl.install(nm, extra=('PCR', 'GEM'))
        assert nm.agents['GEM'] is registry.extra_agents['GEM'] and nm.agents['PCR'] is registry.extra_agents['PCR']
        registry.uninstall(nm)
        assert 'GEM' not in nm.agents
    _with_stub_reference(check)


@pytest.mark.parametrize('env,want', [('GEM', ['GEM']), ('DERPP, GEM', ['DERPP', 'GEM'])])
def test_launcher_passes_gem_through(monkeypatch, tmp_path, env, want):
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
