"""Generate tests/golden/adam.npz by EXECUTING THE REFERENCE (build container only): torch.optim.Adam as the reference
builds it (utils/setup_elements.py:76-78, --optimizer Adam) and its agents running with it.

    python tests/golden/make_golden_adam.py REFERENCE_CHECKOUT

Uses the import recipe of make_golden_tricks.py (imported, not changed) and records
  (a) element level: the CPU torch.optim.Adam over seeded fp32 tensors for several steps with state carried: weight
      decay 0 / 5e-4, default and other betas / eps / lr, steps up to 300, all-zero and tiny gradients, and the review
      trick's p.grad.clone() / 10. before the step.  At the recorded steps: the state before the step (p, g, exp_avg,
      exp_avg_sq) and after it;
  (b) drop-in runs of the reference's agents with optimizer='Adam' at lr 0.001 (construction, seeded weights, seeds,
      buffer fill, train_learner per call, evaluate) in dropin.npz's format: per call the 2048-parameter sample, the BN
      running statistics and the buffer digest, at the end the accuracies, and the reference's own one-ulp spread.
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_tricks as mgt  # noqa: E402  (make_golden's import recipe: reads the checkout from sys.argv[1])

mg = mgt.mg
ref_harness = mgt.ref_harness

N_ELEM = 257
# (lr, beta1, beta2, eps, weight_decay, steps, gradient kind, recorded steps)
ELEMENT_CASES = [
    (1e-3, 0.9, 0.999, 1e-8, 0.0, 300, 'normal', (1, 2, 3, 10, 100, 300)),
    (1e-3, 0.9, 0.999, 1e-8, 5e-4, 300, 'normal', (1, 2, 50, 300)),
    (3e-4, 0.8, 0.99, 1e-6, 0.0, 40, 'normal', (1, 5, 40)),
    (1e-2, 0.5, 0.9, 1e-3, 5e-4, 20, 'normal', (1, 2, 20)),        # lerp weight 0.5: Lerp.h's other branch
    (1e-3, 0.3, 0.0, 1e-8, 0.0, 10, 'normal', (1, 10)),            # addcmul value 1 (beta2 = 0)
    (1e-3, 0.9, 0.999, 1e-8, 0.0, 5, 'zero', (1, 5)),
    (1e-3, 0.9, 0.999, 1e-8, 5e-4, 5, 'zero', (1, 5)),
    (1e-3, 0.9, 0.999, 1e-8, 0.0, 8, 'tiny', (1, 2, 8)),
    (1e-3, 0.9, 0.999, 1e-8, 0.0, 6, 'review', (1, 2, 6)),          # g / 10. then the step
    (1e-3, 0.9, 0.999, 1e-8, 5e-4, 6, 'review', (1, 6)),
]
ELEMENT_SEED = 9000


def element_gradient(rs, kind, n):
    if kind == 'zero':
        return np.zeros(n, np.float32)
    g = (rs.standard_normal(n) * 0.05).astype(np.float32)
    if kind == 'tiny':
        g = (g * np.float32(1e-30)).astype(np.float32)
        g[::7] = np.float32(1e-41)                                    # subnormal
        g[1::11] = 0
    return g


def gen_element(out):
    for k, (lr, b1, b2, eps, wd, n_steps, kind, rec_steps) in enumerate(ELEMENT_CASES):
        tag = 'e%d_' % k
        rs = np.random.RandomState(ELEMENT_SEED + k)
        p = torch.nn.Parameter(torch.from_numpy((rs.standard_normal(N_ELEM) * 0.1).astype(np.float32)))
        opt = torch.optim.Adam([p], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
        for s in range(1, n_steps + 1):
            p.grad = torch.from_numpy(element_gradient(rs, kind, N_ELEM))
            if kind == 'review':                                      # agents/base.py:84-87
                grad = [q.grad.clone() / 10. for q in [p]]
                for g0, q in zip(grad, [p]):
                    q.grad.data.copy_(g0)
            if s in rec_steps:
                st = opt.state.get(p, {})
                zeros = np.zeros(N_ELEM, np.float32)
                pre = [p.detach().numpy().copy(), p.grad.numpy().copy(),
                       st['exp_avg'].numpy().copy() if st else zeros, st['exp_avg_sq'].numpy().copy() if st else zeros]
            opt.step()
            if s in rec_steps:
                st = opt.state[p]
                assert float(st['step']) == s
                post = [p.detach().numpy(), st['exp_avg'].numpy(), st['exp_avg_sq'].numpy()]
                for name, a in zip(('p', 'g', 'm', 'v'), pre):
                    out['%ss%d_%s' % (tag, s, name)] = a
                for name, a in zip(('p_out', 'm_out', 'v_out'), post):
                    out['%ss%d_%s' % (tag, s, name)] = a.copy()
        out[tag + 'case'] = np.array(json.dumps([lr, b1, b2, eps, wd, n_steps, kind, list(rec_steps)]))
    out['n_element'] = np.int64(len(ELEMENT_CASES))


# Drop-in cases (kind, calls, labels, overrides); seed indices start at 120 so that no case shares its seeds with the
# other drop-in goldens.  Adam at lr 0.001 (its default, and the scale at which Adam is run).
_ADAM = dict(optimizer='Adam', learning_rate=0.001)
ADAM_DROPIN_CASES = [
    ('er', 3, 10, dict(_ADAM, data='cifar10', mem_size=500)),
    ('scr', 3, 10, dict(_ADAM)),
    ('agem', 3, 100, dict(_ADAM, mem_size=1000)),
    ('lwf', 3, 10, dict(_ADAM, data='cifar10')),
    ('icarl', 3, 10, dict(_ADAM, mem_size=200)),
    ('er', 2, 10, dict(_ADAM, data='cifar10', mem_size=40, trick={'review_trick': True})),
    ('ewc', 3, 10, dict(_ADAM, data='cifar10', lambda_=100.0, alpha=0.9, fisher_update_after=1)),
]


if __name__ == '__main__':
    out = {}
    gen_element(out)
    mgt._dropin_record(ADAM_DROPIN_CASES, 120, out)
    out['n_dropin'] = np.int64(len(ADAM_DROPIN_CASES))
    path = os.path.join(mg.HERE, 'adam.npz')
    np.savez_compressed(path, **out)
    print('adam.npz', os.path.getsize(path))
