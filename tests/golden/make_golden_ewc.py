"""Generate tests/golden/ewc.npz by EXECUTING THE REFERENCE (build container only): the EWC++ agent (agents/ewc_pp.py).

    python tests/golden/make_golden_ewc.py REFERENCE_CHECKOUT

Uses the import recipe of make_golden_tricks.py (imported, not changed) and records
  (a) element level: the reference's own EWC_pp over a small two-layer network with seeded named-parameter dicts
      (oracle.ewc.element_case_inputs): update_running_fisher (running and tmp after it); the end-of-call
      normalisation and prev_params, from a train_learner call too short for one batch; total_loss(...).backward()
      with the kd_trick / kd_trick_star mixing of ewc_pp.py:46-51 on detached stub logits, so that p.grad is the
      penalty's gradient alone (the gradient and the loss); accum_fisher twice (tmp after it).  Several lambda, mixing
      weights, an all-zero running and running at several scales;
  (b) drop-in runs of the agent (construction, seeded weights, seeds, train_learner per call, evaluate): per call a
      2048-parameter sample, the BN running statistics, every fourth of those positions of running, tmp, normalized
      and prev, and the
      reference's own one-ulp spread (the same run from weights perturbed by one ulp).  At the end the accuracies.
"""
import json
import os
import random
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_tricks as mgt  # noqa: E402  (make_golden's import recipe: reads the checkout from sys.argv[1])

from oracle import ewc as oewc  # noqa: E402  (the repository root is on sys.path: make_golden)
from oracle import gdumb as ogd  # noqa: E402

mg = mgt.mg
ref_harness = mgt.ref_harness

SHAPES = {'0.weight': (8, 12), '0.bias': (8,), '1.weight': (5, 8), '1.bias': (5,)}

# (lambda, task_seen, kd_trick, kd_trick_star, running scale, all-zero running, alpha, fisher_update_after)
ELEMENT_CASES = [
    (100.0, 0, False, False, 1.0, False, 0.9, 50),
    (1.0, 0, False, False, 1e-3, False, 0.9, 3),
    (0.0, 0, False, False, 1.0, False, 0.5, 50),
    (100.0, 1, True, False, 1.0, False, 0.9, 50),
    (100.0, 2, True, False, 1e4, False, 0.9, 7),
    (100.0, 3, False, True, 1.0, False, 0.9, 50),
    (37.5, 2, True, True, 1e-8, False, 0.3, 3),
    (100.0, 0, False, False, 1.0, True, 0.9, 50),
    (100.0, 1, False, False, 1e2, False, 0.9, 50),
]
ELEMENT_SEED = 7000


def _ref_agent(lam, alpha, fua, kd_trick, kd_trick_star):
    from utils import name_match  # noqa: F401  (resolves the reference's circular import first)
    from agents.ewc_pp import EWC_pp
    trick = dict(ref_harness.TRICK, kd_trick=kd_trick, kd_trick_star=kd_trick_star)
    params = ref_harness.make_params('ewc', cuda=False, trick=trick, lambda_=lam, alpha=alpha, fisher_update_after=fua)
    model = torch.nn.Sequential(torch.nn.Linear(12, 8), torch.nn.Linear(8, 5))
    return EWC_pp(model, torch.optim.SGD(model.parameters(), lr=0.1), params)


def gen_element(out):
    for k, (lam, t, kdt, kds, scale, zero, alpha, fua) in enumerate(ELEMENT_CASES):
        tag = 'e%d_' % k
        params, prev, running, tmp, logits, labels = oewc.element_case_inputs(ELEMENT_SEED + k, SHAPES, scale, zero)
        agent = _ref_agent(lam, alpha, fua, kdt, kds)
        with torch.no_grad():
            for n, p in agent.model.named_parameters():
                p.copy_(torch.from_numpy(params[n]))
        agent.running_fisher = {n: torch.from_numpy(v.copy()) for n, v in running.items()}
        agent.tmp_fisher = {n: torch.from_numpy(v.copy()) for n, v in tmp.items()}
        agent.update_running_fisher()                                        # ewc_pp.py:103-108
        snap = lambda d: {n: v.detach().clone() for n, v in d.items()}          # later steps update tensors in place
        rec = {'ema_running': snap(agent.running_fisher), 'ema_tmp': snap(agent.tmp_fisher)}
        # the end of a call: a train_learner call shorter than one batch runs no step (drop_last), only :70-79
        agent.train_learner(np.zeros((agent.batch - 1, 32, 32, 3), np.uint8), np.arange(agent.batch - 1) % 5)
        rec['normalized'] = snap(agent.normalized_fisher)
        rec['prev_end'] = snap(agent.prev_params)
        agent.prev_params = {n: torch.from_numpy(v.copy()) for n, v in prev.items()}
        agent.task_seen = t
        agent.kd_manager.teacher_model = None                                 # the stub has no teacher: kd = 0
        agent.opt.zero_grad()
        out_t = torch.tensor(logits, requires_grad=True).detach()             # the stub: no path to the parameters
        y = torch.from_numpy(labels)
        loss = agent.total_loss(out_t, y)                                     # ewc_pp.py:44
        ce = agent.criterion(out_t, y)
        if kdt:                                                               # ewc_pp.py:46-51
            loss = 1 / (t + 1) * loss + (1 - 1 / (t + 1)) * agent.kd_manager.get_kd_loss(out_t, None)
        if kds:
            loss = 1 / ((t + 1) ** 0.5) * loss + (1 - 1 / ((t + 1) ** 0.5)) * agent.kd_manager.get_kd_loss(out_t, None)
        loss.backward()
        rec['grad'] = {n: p.grad.clone() for n, p in agent.weights.items()}
        agent.accum_fisher()                                                  # ewc_pp.py:110-112, twice
        agent.accum_fisher()
        rec['accum_tmp'] = snap(agent.tmp_fisher)
        for key, d in rec.items():
            out[tag + key] = torch.cat([d[n].detach().reshape(-1) for n in SHAPES]).numpy()
        out[tag + 'loss'] = np.float64(loss.item())
        out[tag + 'ce'] = np.float64(ce.item())
        out[tag + 'case'] = np.array(json.dumps([lam, t, kdt, kds, scale, zero, alpha, fua]))
    out['n_element'] = np.int64(len(ELEMENT_CASES))


# Drop-in cases (calls, labels, samples per call, overrides); seed indices start at 80 so that no case shares its seeds
# with the other drop-in goldens.  23 samples per call: 2 batches of 10, so that fua=1 fires twice per call; lr 0.001.
# Longer calls or larger steps from seeded weights are chaotic in the reference itself: with 6 batches per call at
# lr 0.005 its own one-ulp spread reaches 4-30 % of the weight update, and then a 10x bar checks nothing.  The
# penalty's wiring (live from the second call, with the mixing weights) is pinned step by step by
# tests/test_gpu_ewc.py::test_train_learner_steps_match_the_oracle.
_LR = dict(learning_rate=0.001)
EWC_DROPIN_CASES = [
    (3, 30, 23, dict(_LR, lambda_=100.0, alpha=0.9, fisher_update_after=1)),
    (2, 30, 23, dict(_LR, lambda_=100.0, alpha=0.9, fisher_update_after=3, epoch=2)),
    (3, 30, 23, dict(_LR, lambda_=100.0, alpha=0.9, fisher_update_after=1, trick={'labels_trick': True})),
    (3, 30, 23, dict(_LR, lambda_=100.0, alpha=0.9, fisher_update_after=1,
                     trick={'kd_trick': True, 'kd_trick_star': True})),
    (2, 10, 23, dict(_LR, data='cifar10', lambda_=100.0, alpha=0.9, fisher_update_after=1)),
    (3, 30, 23, dict(_LR, lambda_=0.0, alpha=0.9, fisher_update_after=50)),       # the published setting
]
ARENAS = ('running_fisher', 'tmp_fisher', 'normalized_fisher', 'prev_params')


def _dropin_run(i, n_calls, n_label, n_per_call, over, perturb):
    from continuum.data_utils import setup_test_loader
    over = dict(over)
    trick = dict(ref_harness.TRICK, **over.pop('trick', {}))
    params = ref_harness.make_params('ewc', cuda=False, trick=trick, **over)
    spec = mg.oresnet.Spec(32, 20, 10 if params.data == 'cifar10' else 100)
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
    calls, tests = ogd.dropin_inputs(np.random.RandomState(100 + i), 32, n_label, n_per_call, n_calls)
    names = [n for n, _ in agent.model.named_parameters()]
    flat = lambda d: torch.cat([d[n].detach().reshape(-1) for n in names]).numpy()
    pick = mg.dropin_sample(sum(q.numel() for q in agent.model.parameters()))
    rec = {}
    for c, (xt, yt) in enumerate(calls):
        agent.train_learner(xt, yt)
        rec['w%d' % c] = flat(dict(agent.model.named_parameters()))[pick]
        rec['bn%d' % c] = torch.cat([torch.cat([m.running_mean, m.running_var]) for m in agent.model.modules()
                                     if isinstance(m, torch.nn.BatchNorm2d)]).numpy()
        for a in ARENAS:
            rec['%s%d' % (a, c)] = flat(getattr(agent, a))[pick[::4]]
    rec['acc'] = np.asarray(agent.evaluate(setup_test_loader(tests, params)), dtype=np.float64)
    rec['params'] = np.array(json.dumps(vars(params), sort_keys=True))
    w0 = torch.cat([t.reshape(-1) for t in p.values()]).numpy()[pick].astype(np.float64)
    return rec, w0


def gen_dropin(out):
    def rel(a, b):
        return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))

    for k, (n_calls, n_label, n_per_call, over) in enumerate(EWC_DROPIN_CASES):
        i = 80 + k
        tag = 'c%d_' % k
        rec, w0 = _dropin_run(i, n_calls, n_label, n_per_call, over, False)
        alt, _ = _dropin_run(i, n_calls, n_label, n_per_call, over, True)
        for key, v in rec.items():
            out[tag + key] = v
        out[tag + 'spread_w'] = np.array([rel(alt['w%d' % c] - w0, rec['w%d' % c] - w0) for c in range(n_calls)])
        for key in ('bn',) + ARENAS:
            out[tag + 'spread_' + key] = np.array([rel(alt['%s%d' % (key, c)].astype(np.float64),
                                                       rec['%s%d' % (key, c)].astype(np.float64))
                                                   for c in range(n_calls)])
        out[tag + 'case'] = np.array(json.dumps([n_calls, n_label, n_per_call, 40 + i, i, 100 + i]))
        print('dropin', k, rec['acc'], 'one-ulp spread', out[tag + 'spread_w'], out[tag + 'spread_bn'],
              [out[tag + 'spread_' + a] for a in ARENAS])
    out['n_dropin'] = np.int64(len(EWC_DROPIN_CASES))


if __name__ == '__main__':
    out = {}
    gen_element(out)
    gen_dropin(out)
    path = os.path.join(mg.HERE, 'ewc.npz')
    np.savez_compressed(path, **out)
    print('ewc.npz', os.path.getsize(path))
