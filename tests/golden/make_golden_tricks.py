"""Generate tests/golden/tricks.npz by EXECUTING THE REFERENCE (build container only): the training tricks
(agents/base.py:93-113, utils/kd_manager.py, exp_replay.py:41-47, agem.py:40-46) and the LwF agent (agents/lwf.py).

    python tests/golden/make_golden_tricks.py REFERENCE_CHECKOUT

Uses the import recipe, stubs, seeded weights and drop-in inputs of make_golden.py (imported, not changed), and
records (a) the reference's own ContinualLearner.criterion and loss_fn_kd with autograd's d loss / d logits on seeded
logits, (b) its label bookkeeping over recurring label sets, (c) drop-in runs of the trick configurations and LwF in
the format of make_golden.py gen_dropin (tests/test_gpu_tricks.py runs tests/test_gpu_dropin.py's comparison on them).
The loss-level logits are not stored: case k draws them from RandomState(LOSS_SEED + k) (case_logits, kept identical
to tests/test_oracle_tricks.py).
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402  (reads the reference checkout from sys.argv[1], installs the stubs)

sys.path.insert(0, os.path.join(mg.ROOT, 'baseline'))
import ref_harness  # noqa: E402

ref_harness.import_reference(mg.REF)
REF = mg.REF
LOSS_SEED = 5000


def case_logits(seed, N, C, teacher):
    """Logits [N,C] (and teacher logits when asked) of one loss-level case."""
    rs = np.random.RandomState(seed)
    logits = (rs.standard_normal((N, C)) * 3).astype(np.float32)
    return logits, ((rs.standard_normal((N, C)) * 3).astype(np.float32) if teacher else None)


def _dropin_run(i, kind, n_calls, n_label, over, perturb):
    """One seeded drop-in run of the reference's agent: buffer fill, train_learner per call, evaluate.  Returns the
    record and the sampled initial weights.  Agents without a memory (LwF) skip the buffer fill and records."""
    import hashlib
    import json
    import random
    from continuum.data_utils import setup_test_loader
    over = dict(over)
    trick = dict(ref_harness.TRICK, **over.pop('trick', {}))
    params = ref_harness.make_params(kind, cuda=False, trick=trick, **over)
    hw = 84 if params.data == 'mini_imagenet' else 32
    spec = mg.oresnet.Spec(hw, 20, 10 if params.data == 'cifar10' else 100, head='mlp' if params.agent == 'SCR' else None)
    mg.buffer_utils.ClassBalancedRandomSampling.class_index_cache = None
    mg.buffer_utils.ClassBalancedRandomSampling.class_num_cache = None
    agent = ref_harness.build_agent(params)
    p, bn = mg.oresnet.seeded_state(spec, 40 + i)
    sd = dict(p)
    sd.update(bn)
    agent.model.load_state_dict(sd, strict=True)
    if perturb:
        gen = torch.Generator().manual_seed(1234)
        with torch.no_grad():
            for prm in agent.model.parameters():
                prm.mul_(1 + (torch.randint(0, 2, prm.shape, generator=gen).float() * 2 - 1) * 2.0 ** -23)
    np.random.seed(i); random.seed(i); torch.manual_seed(i)
    rs = np.random.RandomState(100 + i)
    x, y, calls, tests = mg.dropin_inputs(rs, params.mem_size, hw, n_label, params.batch, n_calls)
    has_buffer = hasattr(agent, 'buffer')
    if has_buffer:
        agent.buffer.update(torch.from_numpy(x), torch.from_numpy(y))
    rec, pick = {}, None
    for c, (xt, yt) in enumerate(calls):
        agent.train_learner(xt, yt)
        flat = torch.cat([q.detach().reshape(-1) for q in agent.model.parameters()]).numpy()
        pick = mg.dropin_sample(flat.size) if pick is None else pick
        if has_buffer:
            rec['label%d' % c] = agent.buffer.buffer_label.numpy().astype(np.int16)
            rec['index%d' % c] = np.int64(agent.buffer.current_index)
            rec['seen%d' % c] = np.int64(agent.buffer.n_seen_so_far)
            rec['img%d' % c] = np.array(hashlib.sha1(agent.buffer.buffer_img.numpy().tobytes()).hexdigest())
        rec['w%d' % c] = flat[pick]
        rec['bn%d' % c] = torch.cat([torch.cat([m.running_mean, m.running_var]) for m in agent.model.modules()
                                     if isinstance(m, torch.nn.BatchNorm2d)]).numpy()
    rec['acc'] = np.asarray(agent.evaluate(setup_test_loader(tests, params)), dtype=np.float64)
    rec['params'] = np.array(json.dumps(vars(params), sort_keys=True))
    w0 = torch.cat([t.reshape(-1) for t in p.values()]).numpy()[pick].astype(np.float64)
    return rec, w0


def _dropin_record(cases, first, out):
    """Per case two runs of the reference: the recorded one, and one from the same weights perturbed by one ulp
    (x * (1 +- 2^-23), fixed random signs) whose distance from the first is the reference's own fp32 spread -- the
    yardstick for how far another fp32 implementation may land (tolerance = max(base, 10 x spread)).  Case k runs
    with seed index first + k and is stored under 'c<k>_'."""
    import json

    def rel(a, b):
        return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))

    for k, (kind, n_calls, n_label, over) in enumerate(cases):
        i = first + k
        tag = 'c%d_' % k
        rec, w0 = _dropin_run(i, kind, n_calls, n_label, over, False)
        alt, _ = _dropin_run(i, kind, n_calls, n_label, over, True)
        for key, v in rec.items():
            out[tag + key] = v
        out[tag + 'spread_w'] = np.array([rel(alt['w%d' % c] - w0, rec['w%d' % c] - w0) for c in range(n_calls)])
        out[tag + 'spread_bn'] = np.array([rel(alt['bn%d' % c].astype(np.float64), rec['bn%d' % c].astype(np.float64))
                                           for c in range(n_calls)])
        if 'label0' in rec:
            out[tag + 'spread_slots'] = np.array([int((alt['label%d' % c] != rec['label%d' % c]).sum())
                                                  for c in range(n_calls)])
        out[tag + 'case'] = np.array(json.dumps([kind, n_calls, n_label, 40 + i, i, 100 + i]))
        print('dropin', i, kind, rec['acc'], 'one-ulp spread', out[tag + 'spread_w'], out[tag + 'spread_bn'],
              out.get(tag + 'spread_slots'))


# Drop-in cases (kind, calls, labels, overrides); seed indices start at 20 so that no case shares its seeds with
# make_golden.DROPIN_CASES.  Distillation cases run three calls: the teacher is taken after the first.
TRICK_DROPIN_CASES = [
    ('er', 2, 10, dict(data='cifar10', mem_size=500, trick={'labels_trick': True})),
    ('er', 2, 10, dict(data='cifar10', mem_size=500, trick={'separated_softmax': True})),   # old_labels recur
    ('er', 3, 100, dict(mem_size=1000, trick={'kd_trick': True})),                             # teacher from call 2
    ('aser', 2, 100, dict(trick={'kd_trick_star': True})),                                     # memory 5000
    ('agem', 2, 100, dict(mem_size=1000, trick={'kd_trick': True, 'labels_trick': True})),
    ('er', 2, 10, dict(data='cifar10', mem_size=40, trick={'review_trick': True, 'labels_trick': True})),
    ('lwf', 3, 100, dict(mem_size=10)),
]


def _ref_learner(trick):
    """The reference's ContinualLearner (agents/base.py) with the given trick flags, for its bookkeeping and criterion."""
    from utils import name_match  # noqa: F401  (resolves the reference's circular import first)
    from agents.base import ContinualLearner

    class Learner(ContinualLearner):
        def train_learner(self, x_train, y_train):
            pass
    params = SimpleNamespace(data='cifar100', cuda=False, epoch=1, batch=10, verbose=False, agent='ER', temp=0.07,
                             trick=dict(ref_harness.TRICK, **trick))
    return Learner(torch.nn.Linear(1, 1), None, params)


def gen_tricks():
    """(a) Loss level: the reference's own ContinualLearner.criterion and loss_fn_kd, mixed as exp_replay.py:41-47
    mixes them, on seeded logits, with autograd's d loss / d logits.  (b) The label bookkeeping of base.py:43-60 over
    recurring label sets.  (c) Drop-in runs of the trick configurations and LwF."""
    from utils.kd_manager import loss_fn_kd
    rs = np.random.RandomState(2024)
    out = {}
    # label histories: (C, task label sets); after each set before_train runs, after all but the last after_train
    hist = {'first10': (10, [range(10)]), 'first100': (100, [range(100)]),
            'recur10': (10, [range(10), range(10), range(10)]),
            'overlap100': (100, [range(0, 50), range(40, 60), range(60, 70)])}
    tables = {}
    for name, (C, sets) in hist.items():
        lrn = _ref_learner({'separated_softmax': True})
        for t, lab in enumerate(sets):
            lrn.before_train(np.array(list(lab)), np.array(list(lab)))
            out['hist_%s_old%d' % (name, t)] = np.array(lrn.old_labels, dtype=np.int64)
            out['hist_%s_new%d' % (name, t)] = np.array(lrn.new_labels, dtype=np.int64)
            inv = sorted(lrn.lbl_inv_map.items())
            out['hist_%s_inv%d' % (name, t)] = np.array(inv, dtype=np.int64).reshape(-1, 2)
            if t < len(sets) - 1:
                lrn.after_train()
        out['hist_%s_n' % name] = np.int64(len(sets))
        tables[name] = lrn
    cases = []     # (C, N, mode, history, one_class, teacher, task_seen, kd_trick, kd_trick_star, kd_alone)
    for C, N in ((10, 10), (10, 20), (10, 110), (100, 10), (100, 20), (100, 110)):
        cases.append((C, N, 'labels_trick', None, False, False, 0, False, False, False))
    cases.append((100, 10, 'labels_trick', None, True, False, 0, False, False, False))
    cases.append((10, 20, 'separated_softmax', 'first10', False, False, 0, False, False, False))     # empty old_labels
    cases.append((100, 20, 'separated_softmax', 'first100', False, False, 0, False, False, False))
    cases.append((10, 20, 'separated_softmax', 'recur10', False, False, 0, False, False, False))     # duplicates
    cases.append((100, 20, 'separated_softmax', 'overlap100', False, False, 0, False, False, False))   # target in old
    cases.append((100, 20, 'ce', None, False, True, 0, False, False, True))                          # KD alone
    cases.append((10, 110, 'ce', None, False, True, 0, False, False, True))
    for C, N, mode, hname in ((10, 20, 'ce', None), (10, 20, 'labels_trick', None),
                              (100, 10, 'separated_softmax', 'overlap100')):
        for t in range(4):
            cases.append((C, N, mode, hname, False, t > 0, t, True, False, False))
    for t in range(4):
        cases.append((10, 20, 'ce', None, False, t > 0, t, True, True, False))                         # both flags
        cases.append((10, 10, 'labels_trick', None, False, t > 0, t, False, True, False))
    for k, (C, N, mode, hname, one, teach, t, kdt, kds, alone) in enumerate(cases):
        tag = 'l%d_' % k
        lrn = tables[hname] if hname else _ref_learner({})
        lrn.params.trick = dict(ref_harness.TRICK, **({mode: True} if mode != 'ce' else {}))
        logits, teacher = case_logits(LOSS_SEED + k, N, C, teach)
        if hname:
            pool = np.array(sorted(lrn.lbl_inv_map), dtype=np.int64)
        else:
            pool = np.arange(C)
        labels = np.full(N, pool[rs.randint(len(pool))]) if one else pool[rs.randint(0, len(pool), N)]
        lg = torch.tensor(logits, requires_grad=True)
        kd = loss_fn_kd(lg, torch.tensor(teacher)) if teach else 0
        if alone:
            loss = kd
        else:
            loss = lrn.criterion(lg, torch.tensor(labels))
            if kdt:
                loss = 1 / (t + 1) * loss + (1 - 1 / (t + 1)) * kd
            if kds:
                loss = 1 / ((t + 1) ** 0.5) * loss + (1 - 1 / ((t + 1) ** 0.5)) * kd
        loss.backward()
        out.update({tag + 'shape': np.array([N, C], dtype=np.int64), tag + 'labels': labels.astype(np.int16),
                    tag + 'mode': np.array(mode), tag + 'hist': np.array(hname or ''), tag + 'task_seen': np.int64(t),
                    tag + 'flags': np.array([kdt, kds, alone]), tag + 'loss': np.float64(loss.item()),
                    tag + 'dlogits': lg.grad.numpy().copy()})
        out[tag + 'teacher'] = np.bool_(teach)
        if hname:
            out[tag + 'old'] = np.array(lrn.old_labels, dtype=np.int64)
            out[tag + 'new'] = np.array(lrn.new_labels, dtype=np.int64)
            out[tag + 'inv'] = np.array(sorted(lrn.lbl_inv_map.items()), dtype=np.int64).reshape(-1, 2)
    out['n_loss_cases'] = np.int64(len(cases))
    dropin = {'n_cases': np.int64(len(TRICK_DROPIN_CASES))}
    _dropin_record(TRICK_DROPIN_CASES, 20, dropin)
    out.update({'dropin_' + k: v for k, v in dropin.items()})
    np.savez_compressed(os.path.join(mg.HERE, 'tricks.npz'), **out)


if __name__ == '__main__':
    gen_tricks()
    print('tricks.npz', os.path.getsize(os.path.join(mg.HERE, 'tricks.npz')))
