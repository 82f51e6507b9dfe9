"""The error analysis of evaluate() (agents/base.py:144-226, --error_analysis) on the GPU:
  * b200ocl_linear_argmax_ea against the fp64 oracle at C in {10, 50, 69, 100}, d in {160, 640, 2560} (the 32x32,
    84x84 and 128x128 features) and B in {1, 7, 128, 129, 1000}, with planted exact ties (duplicated classifier rows),
    empty class sets, all-wrong and all-right batches and predictions into unmapped classes: predicted tasks and the
    four counts exactly, the two per-row logit sums within SUM_TOL; predictions and hits bit-identical to
    b200ocl_linear_argmax on the same inputs;
  * b200ocl_rows_mean against the fp64 mean rounded to fp32;
  * evaluate() accuracies bit-identical with the analysis on and off at 32x32 and 128x128, its confusion lists equal to
    the arg-max kernel's predictions mapped through class_task_map;
  * drop-in runs of ER, ER + ASER, A-GEM, LwF, EWC++ and GDumb with the analysis at every call against the reference's
    own runs (tests/golden/error_analysis.npz);
  * the refusal on the nearest-class-mean branch (SCR, iCaRL, ncm_trick) before anything launches.
Bars are about 3x the largest error measured on an H100 80GB HBM3 (132 SMs, 700 W power limit); the measured maxima are
printed by each test."""
import contextlib
import io
import json
import os
import pickle
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import test_gpu_dropin as dropin

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'error_analysis.npz')
# per-row logit sums: |got - fp64| / sum over the set of (|f| . |w_c| + |b_c|) [6.0e-8, C = 10, d = 640]
SUM_TOL = 2e-7
MARGIN = 1e-4   # inputs are redrawn until every row's best class beats the next distinct one by this share of its scale


def _inputs(C, d, B, seed):
    """Features, classifier, truth, class sets and task table for one kernel case.  Two pairs of classifier rows are
    duplicated (an exact tie: the first of the pair must win) and some rows are aimed at them; rows whose best and
    next-best distinct logits lie within MARGIN of each other in fp64 are redrawn, so that every prediction is decided."""
    rs = np.random.RandomState(seed)
    W = (rs.standard_normal((C, d)) * 0.05).astype(np.float32)
    b = (rs.standard_normal(C) * 0.1).astype(np.float32)
    pairs = [(0, C - 1), (1, C // 2)]
    for k1, k2 in pairs:
        W[k2], b[k2] = W[k1], b[k1]
    distinct = [c for c in range(C) if c not in [k2 for _, k2 in pairs]]

    def draw(n):
        f = np.abs(rs.standard_normal((n, d))).astype(np.float32)
        aim = rs.rand(n) < 0.3
        f[aim] += (40 * np.maximum(W[rs.choice([k1 for k1, _ in pairs], aim.sum())], 0)).astype(np.float32)
        return f
    f = draw(B)
    W64, b64 = W[distinct].astype(np.float64), b[distinct].astype(np.float64)
    for _ in range(50):
        lg = f.astype(np.float64) @ W64.T + b64
        top = np.sort(lg, axis=1)
        scale = (np.abs(f).astype(np.float64) @ np.abs(W64).T + np.abs(b64)).max(1)
        bad = (top[:, -1] - top[:, -2]) <= MARGIN * scale
        if not bad.any():
            break
        f[bad] = draw(int(bad.sum()))
    else:
        raise AssertionError('could not draw decided rows')
    sets = np.zeros(C, dtype=np.uint8)
    kind = seed % 4                                     # both sets, no new classes, no old classes, neither
    perm = rs.permutation(C)
    if kind in (0, 2):
        sets[perm[:max(1, C // 5)]] |= 1
    if kind in (0, 1):
        sets[perm[max(1, C // 5):C // 2]] |= 2
    task = rs.randint(0, 10, C).astype(np.int64)
    task[perm[-max(1, C // 10):]] = -1                  # unmapped classes
    return f, W, b, sets, task


def _oracle(f, W, b, truth, sets, task):
    from oracle.evaluate import linear_logits
    lg = linear_logits(f, W, b)
    # a duplicated classifier row gives the same fp32 logit in the kernel; BLAS may round the two fp64 columns apart
    for c in range(1, W.shape[0]):
        same = np.flatnonzero((W[:c] == W[c]).all(1) & (b[:c] == b[c]))
        if same.size:
            lg[:, c] = lg[:, same[0]]
    pred = np.argmax(lg, axis=1)                        # the first maximum
    wrong = pred != truth
    m = sets[pred]
    counts = np.array([(wrong & ((m & 1) != 0)).sum(), (wrong & ((m & 1) == 0) & ((m & 2) != 0)).sum(),
                       (wrong & ((m & 3) == 0)).sum(), (task[pred] < 0).sum()], dtype=np.int64)
    sums = np.stack([(lg * ((sets & bit) != 0)).sum(1) for bit in (1, 2)], 1)
    absl = np.abs(f.astype(np.float64)) @ np.abs(W.astype(np.float64)).T + np.abs(b.astype(np.float64))
    scale = np.stack([(absl * ((sets & bit) != 0)).sum(1) for bit in (1, 2)], 1)
    return pred, task[pred], counts, sums, scale


@pytest.mark.parametrize('C', [10, 50, 69, 100])
@pytest.mark.parametrize('d', [160, 640, 2560])
def test_linear_argmax_ea_against_fp64(C, d):
    from b200ocl import ops
    worst = 0.0
    for B in (1, 7, 128, 129, 1000):
        for v, truth_kind in enumerate(('random', 'right', 'wrong')):
            seed = 1000 * C + 10 * d + B + v
            f, W, b, sets, task = _inputs(C, d, B, seed)
            pred, ptask, _, sums, scale = _oracle(f, W, b, np.zeros(B, np.int64), sets, task)
            truth = {'random': np.random.RandomState(seed).randint(0, C, B), 'right': pred,
                     'wrong': (pred + 1 + np.random.RandomState(seed).randint(0, C - 1, B)) % C}[truth_kind]
            truth = truth.astype(np.int64)
            pred, ptask, counts, sums, scale = _oracle(f, W, b, truth, sets, task)
            ft, Wt, bt, yt = (torch.from_numpy(a).cuda() for a in (f, W, b, truth))
            st, tt = torch.from_numpy(sets).cuda(), torch.from_numpy(task).cuda()
            cnt = torch.zeros(4, dtype=torch.int64, device='cuda')
            hits = torch.zeros(1, dtype=torch.int64, device='cuda')
            p_ea = torch.empty(B, dtype=torch.int64, device='cuda')
            got_task, got_sums = ops.linear_argmax_ea(ft, Wt, bt, yt, st, tt, cnt, n_correct=hits, pred=p_ea)
            hits_ref = torch.zeros(1, dtype=torch.int64, device='cuda')
            p_ref = ops.linear_argmax(ft, Wt, bt, truth=yt, n_correct=hits_ref)
            where = (C, d, B, truth_kind)
            assert torch.equal(p_ea, p_ref) and torch.equal(hits, hits_ref), where
            assert np.array_equal(p_ea.cpu().numpy(), pred), where
            assert int(hits) == int((pred == truth).sum()), where
            assert np.array_equal(got_task.cpu().numpy(), ptask), where
            assert np.array_equal(cnt.cpu().numpy(), counts), (where, cnt.cpu().numpy(), counts)
            err = np.abs(got_sums.cpu().numpy() - sums) / np.maximum(scale, 1e-30)
            err[scale == 0] = np.abs(got_sums.cpu().numpy() - sums)[scale == 0]
            worst = max(worst, float(err.max()))
            assert err.max() <= SUM_TOL, (where, float(err.max()))
            if truth_kind == 'right':
                assert counts[:3].sum() == 0
            if truth_kind == 'wrong':
                assert int(hits) == 0 and counts[:3].sum() == B
    print('linear_argmax_ea C=%d d=%d: worst sum error %.3g' % (C, d, worst))


def test_linear_argmax_ea_plants_what_it_claims():
    """The inputs reach the planted ties, unmapped predictions and every set kind."""
    seen_tie = seen_unmapped = 0
    kinds = set()
    for seed in range(8):
        f, W, b, sets, task = _inputs(69, 160, 1000, seed)
        pred, ptask, _, _, _ = _oracle(f, W, b, np.zeros(1000, np.int64), sets, task)
        seen_tie += int(np.isin(pred, [0, 1]).sum())
        assert not np.isin(pred, [68, 34]).any()       # the second of a duplicated pair never wins
        seen_unmapped += int((ptask < 0).sum())
        kinds.add((bool((sets & 1).any()), bool((sets & 2).any())))
    assert seen_tie > 0 and seen_unmapped > 0 and len(kinds) == 4


def test_linear_argmax_ea_refuses_bad_tables():
    from b200ocl import ops
    f = torch.zeros(4, 16, device='cuda')
    W, b = torch.zeros(3, 16, device='cuda'), torch.zeros(3, device='cuda')
    y = torch.zeros(4, dtype=torch.int64, device='cuda')
    s, t = torch.zeros(3, dtype=torch.uint8, device='cuda'), torch.zeros(3, dtype=torch.int64, device='cuda')
    cnt = torch.zeros(4, dtype=torch.int64, device='cuda')
    with pytest.raises(ValueError):
        ops.linear_argmax_ea(f, W, b, y, s[:2], t, cnt)
    with pytest.raises(ValueError):
        ops.linear_argmax_ea(f, W, b, y, s, t.int(), cnt)
    with pytest.raises(ValueError):
        ops.linear_argmax_ea(f, W, b, y, s, t, cnt[:3])
    with pytest.raises(ValueError):
        ops.linear_argmax_ea(f, W, b, y[:3], s, t, cnt)
    pt, sums = ops.linear_argmax_ea(f[:0], W, b, y[:0], s, t, cnt)      # B = 0: nothing launched, nothing counted
    assert pt.numel() == 0 and sums.shape == (0, 2) and int(cnt.abs().sum()) == 0


@pytest.mark.parametrize('C,d', [(10, 160), (69, 160), (100, 640), (50, 2560)])
def test_rows_mean_against_fp64(C, d):
    from b200ocl import ops
    rs = np.random.RandomState(C + d)
    W = (rs.standard_normal((C, d)) * 0.05 + 0.01).astype(np.float32)
    b = (rs.standard_normal(C) * 0.1).astype(np.float32)
    Wt, bt = torch.from_numpy(W).cuda(), torch.from_numpy(b).cuda()
    for rows in (list(range(C)), sorted(rs.choice(C, C // 3, replace=False).tolist()), [C - 1], []):
        got = ops.rows_mean(Wt, bt, rows).cpu().numpy()
        if not rows:
            assert np.isnan(got).all()
            continue
        want = np.array([W[rows].astype(np.float64).mean(), b[rows].astype(np.float64).mean()])
        # one fp32 rounding of a sum accumulated in fp64: within half an fp32 ulp of the exact mean, plus slack
        assert (np.abs(got - want) <= np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)).all(), (rows, got, want)
    with pytest.raises(IndexError):
        ops.rows_mean(Wt, bt, [C])


# ----------------------------------------------------------------------------- evaluate()
def _learner(data, agent='ER', **over):
    from b200ocl import nets, registry
    params = SimpleNamespace(data=data, cuda=True, epoch=1, batch=10, verbose=False, mem_size=50, eps_mem_batch=10,
                             mem_iters=1, update='random', retrieve='random', agent=agent, k=3, aser_type='asvm',
                             n_smp_cls=1.5, num_tasks=10, buffer_tracker=False, optimizer='SGD', learning_rate=0.1,
                             weight_decay=0, temp=0.07, head='mlp', subsample=50, error_analysis=False,
                             trick={'labels_trick': False, 'kd_trick': False, 'separated_softmax': False,
                                    'review_trick': False, 'ncm_trick': False, 'kd_trick_star': False}, test_batch=128)
    for k, v in over.items():
        setattr(params, k, v)
    return registry.agents[agent](nets.setup_architecture(params), None, params)


@pytest.mark.parametrize('data,hw,n_cls,n_test', [('cifar100', 32, 100, 1000), ('core50', 128, 50, 300)])
def test_evaluate_accuracies_do_not_move(data, hw, n_cls, n_test, tmp_path, monkeypatch):
    """The same evaluate() with and without the analysis: bit-identical accuracies; the confusion lists are the arg-max
    kernel's predictions mapped through class_task_map, the counts follow from them."""
    from b200ocl import ops
    from b200ocl.learners import error_analysis_tables
    monkeypatch.chdir(tmp_path)
    torch.manual_seed(0)
    agent = _learner(data)
    tasks = [list(range(t, t + 10)) for t in range(0, n_cls, 10)]
    for labels in tasks:
        agent.before_train(None, np.asarray(labels))
        agent.after_train()
    rs = np.random.RandomState(hw)
    loaders = []
    for labels in tasks:
        x = torch.from_numpy(rs.rand(n_test // len(tasks), 3, hw, hw).astype(np.float32))
        y = torch.from_numpy(rs.choice(labels, n_test // len(tasks)).astype(np.int64))
        loaders.append([(x[i:i + 64], y[i:i + 64]) for i in range(0, x.shape[0], 64)])
    with contextlib.redirect_stdout(io.StringIO()):
        off = agent.evaluate(loaders)
        agent.params.error_analysis = True
        on = agent.evaluate(loaders)
    assert np.array_equal(off, on), (off, on)
    with open('confusion', 'rb') as fp:
        correct_lb, predict_lb = pickle.load(fp)
    _, task_of = error_analysis_tables(agent.old_labels, agent.new_labels_zombie, agent.class_task_map, n_cls)
    W, b = agent.model.linear__weight, agent.model.linear__bias
    want_task, want_lb, no_nn_oo_on = [], [], [0, 0, 0, 0]
    zombie, old = set(agent.new_labels_zombie), set(agent.old_labels) - set(agent.new_labels_zombie)
    for t, ld in enumerate(loaders):
        for x, y in ld:
            pred = ops.linear_argmax(agent.engine.features_eval(x.cuda()), W, b).cpu().numpy()
            want_task += task_of[pred].tolist()
            want_lb += [t] * len(y)
            wrong = pred[pred != y.numpy()]
            if t < agent.task_seen - 1:
                on = int(np.isin(wrong, list(zombie)).sum())
                no_nn_oo_on[2] += wrong.size - on
                no_nn_oo_on[3] += on
            elif t == agent.task_seen - 1:
                no = int(np.isin(wrong, list(old)).sum())
                no_nn_oo_on[0] += no
                no_nn_oo_on[1] += wrong.size - no
    assert correct_lb == want_lb and predict_lb == want_task
    assert agent.error_list == [tuple(no_nn_oo_on)]
    assert len(agent.new_class_score) == len(agent.fc_norm_old) == 1


def test_evaluate_raises_keyerror_before_appending(tmp_path, monkeypatch):
    """A prediction into a class never trained on: KeyError, nothing appended, printed or written."""
    monkeypatch.chdir(tmp_path)
    agent = _learner('cifar10', error_analysis=True)
    agent.before_train(None, np.array([0, 1]))
    agent.after_train()
    with torch.no_grad():
        agent.model.linear__bias[7] = 1000.0
    agent.engine.pack()
    x = torch.rand(20, 3, 32, 32)
    out = io.StringIO()
    with contextlib.redirect_stdout(out), pytest.raises(KeyError):
        agent.evaluate([[(x, torch.zeros(20, dtype=torch.int64))]])
    assert out.getvalue() == '' and not agent.error_list and not os.path.exists('confusion')


@pytest.mark.parametrize('agent,over', [('SCR', {}), ('ICARL', {}), ('ER', {'ncm_trick': True})])
def test_ncm_branch_refuses_before_any_launch(agent, over):
    from b200ocl import _native
    trick = {'labels_trick': False, 'kd_trick': False, 'separated_softmax': False, 'review_trick': False,
             'ncm_trick': False, 'kd_trick_star': False}
    trick.update(over)
    a = _learner('cifar100', agent, error_analysis=True, trick=trick)
    torch.cuda.synchronize()
    before = _native.launch_count()
    x = torch.rand(4, 3, 32, 32)
    with pytest.raises(UnboundLocalError):
        a.evaluate([[(x, torch.zeros(4, dtype=torch.int64))]])
    with pytest.raises(NotImplementedError):
        a.evaluate([[(x, torch.zeros(4, dtype=torch.int64))]])
    assert _native.launch_count() == before


# ----------------------------------------------------------------------------- drop-in runs against the reference
def dropin_inputs(rs, mem, batch):
    """tests/golden/make_golden_error_analysis.py dropin_inputs()."""
    call_labels = [list(range(10)), [0, 1, 2, 3, 4], [5, 6, 7, 8, 9]]
    x = rs.rand(mem, 3, 32, 32).astype(np.float32)
    y = rs.randint(0, 10, mem).astype(np.int64)
    calls = []
    for labels in call_labels:
        n = batch + 3
        calls.append((rs.randint(0, 256, (n, 32, 32, 3)).astype(np.uint8),
                      rs.permutation(np.asarray(labels)[np.arange(n) % len(labels)]).astype(np.int64)))
    tests = [(rs.randint(0, 256, (96, 32, 32, 3)).astype(np.uint8),
              rs.permutation(np.asarray(labels)[np.arange(96) % len(labels)]).astype(np.int64)) for labels in call_labels]
    return x, y, calls, tests


def _scales(agent, loaders):
    """The mean absolute value of the elements each analysis mean averages, from the engine's own logits and classifier:
    [logits over the last task's columns, over the older columns, weight rows of each, bias entries of each] (1 where a
    set is empty).  A mean of mixed signs near zero carries the error of its elements' scale, not of its own."""
    from b200ocl.learners import error_analysis_tables
    W, b = agent.model.linear__weight.detach(), agent.model.linear__bias.detach()
    sets, _ = error_analysis_tables(agent.old_labels, agent.new_labels_zombie, agent.class_task_map, W.shape[0])
    new, old = [torch.from_numpy(np.flatnonzero(sets & bit)).cuda() for bit in (1, 2)]
    lg = torch.cat([agent.engine.features_eval(x.cuda()) @ W.T + b for ld in loaders for x, _ in ld]).abs()
    out = []
    for t in (lg[:, new], lg[:, old], W[new].abs(), W[old].abs(), b[new].abs(), b[old].abs()):
        out.append(float(t.double().mean()) if t.numel() else 1.0)
    return np.array(out)


def _close(got, want, spread, scale):
    """NaN where the reference has NaN; elsewhere |got - want| / scale within the larger of test_gpu_dropin.py's vector
    bar and 10x the reference's own one-ulp spread (recorded relative to want), in the same units."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (got, want)
    ok = ~np.isnan(want)
    err = np.abs(got[ok] - want[ok]) / scale[ok]
    bar = np.maximum(dropin.VECTOR_TOL, dropin.SPREAD_FACTOR * np.asarray(spread)[ok] * np.abs(want[ok]) / scale[ok])
    return err, bar


@pytest.mark.parametrize('case', range(int(np.load(GOLDEN)['n_dropin'])))
def test_dropin_error_analysis_matches_reference(case, tmp_path, monkeypatch):
    from b200ocl import memory, nets, registry
    from oracle import resnet as oresnet
    g = np.load(GOLDEN)
    tag = 'd%d_' % case
    kind, n_calls, seed, dseed = json.loads(str(g[tag + 'case']))
    params = SimpleNamespace(**json.loads(str(g[tag + 'params'])))
    params.cuda = True
    monkeypatch.chdir(tmp_path)
    memory.set_mode(True, 'cpu')                    # the reference ran on the CPU: its draws came from CPU generators
    memory.ClassBalancedRandomSampling.reset()
    try:
        cls = registry.agents.get(params.agent) or registry.extra_agents[params.agent]
        agent = cls(nets.setup_architecture(params), None, params)
        if kind != 'gdumb':
            spec = oresnet.Spec(32, 20, 10)
            p, bn = oresnet.seeded_state(spec, 40 + seed)
            agent.engine.load(list(p.values()), [(bn[n + '.running_mean'], bn[n + '.running_var'])
                                                 for n in oresnet.bn_names(spec)])
        np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
        x, y, calls, tests = dropin_inputs(np.random.RandomState(dseed), params.mem_size, params.batch)
        buf = getattr(agent, 'buffer', None)
        if buf is not None:
            buf.update(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda())
        loaders = [[(torch.from_numpy(tx[i:i + 32]).permute(0, 3, 1, 2).float().div(255), torch.from_numpy(ty[i:i + 32]))
                    for i in range(0, 96, 32)] for tx, ty in tests]
        for c, (xt, yt) in enumerate(calls):
            where = '%s call %d' % (kind, c)
            agent.train_learner(xt, yt)
            state = torch.get_rng_state()
            with contextlib.redirect_stdout(io.StringIO()):
                acc = np.asarray(agent.evaluate(loaders))
            torch.set_rng_state(state)
            with open('confusion', 'rb') as fp:
                correct_lb, predict_lb = pickle.load(fp)
            slack = max(int(g[tag + 'spread_pred%d' % c]), 3)          # rows a prediction may move (3 of 96, as dropin)
            assert np.abs(acc - g[tag + 'acc%d' % c]).max() <= 3.1 / 96, (where, acc, g[tag + 'acc%d' % c])
            assert correct_lb == g[tag + 'correct_lb%d' % c].tolist(), where
            moved = int((np.asarray(predict_lb) != g[tag + 'predict_lb%d' % c]).sum())
            d_err = int(np.abs(np.asarray(agent.error_list[-1]) - g[tag + 'error%d' % c]).sum())
            assert moved <= slack and d_err <= 2 * slack, (where, agent.error_list[-1], g[tag + 'error%d' % c], moved)
            got = [agent.new_class_score[-1], agent.old_class_score[-1], agent.fc_norm_new[-1], agent.fc_norm_old[-1],
                   agent.bias_norm_new[-1], agent.bias_norm_old[-1]]
            err, bar = _close(got, g[tag + 'scores%d' % c], g[tag + 'spread_scores%d' % c], _scales(agent, loaders))
            print('error analysis %s: moved %d, count diff %d, worst mean error %.3g' % (where, moved, d_err,
                                                                                        float(err.max(initial=0))))
            assert (err <= bar).all(), (where, got, g[tag + 'scores%d' % c], err, bar)
    finally:
        memory.set_mode(False)
        memory.ClassBalancedRandomSampling.reset()
