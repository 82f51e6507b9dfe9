"""Generate tests/golden/gdumb.npz by EXECUTING THE REFERENCE (build container only): the GDumb agent (agents/gdumb.py).

    python tests/golden/make_golden_gdumb.py REFERENCE_CHECKOUT

Uses the import recipe of make_golden.py and its drop-in weight sample (imported, not changed), and records
  (a) init: the reference's setup_architecture under torch.manual_seed(s) for cifar100, cifar10 and mini_imagenet: a
      sha1 of all parameter bytes in parameters() order, a 2048-element sample, and torch.rand(4) drawn afterwards
      (how far the generator advanced);
  (b) greedy memory: the reference's own Gdumb.greedy_balancing_update over seeded label streams after random.seed(s),
      with x = torch.tensor(i) so that the lists hold source ids: the final mem_c items in order, each class's source
      list, and random.random() drawn afterwards;
  (c) drop-in runs of the agent (construction, seeds, train_learner per call, evaluate), per call mem_c, a sha1 of the
      memory rows in train_mem's order, a 2048-parameter sample of the re-initialised and of the trained network, the
      BN running statistics, and the reference's own one-ulp spread: the same run with the network perturbed by one ulp
      inside every setup_architecture call of train_mem.  At the end the accuracies.
"""
import hashlib
import json
import os
import random
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_tricks as mgt  # noqa: E402  (make_golden's import recipe: reads the checkout from sys.argv[1])

from oracle import gdumb as ogd  # noqa: E402  (the repository root is on sys.path: make_golden)

mg = mgt.mg
ref_harness = mgt.ref_harness

INIT_CASES = [('cifar100', 3), ('cifar100', 11), ('cifar10', 3), ('cifar10', 11), ('mini_imagenet', 3),
              ('mini_imagenet', 11)]


def _flat(model):
    return torch.cat([p.detach().reshape(-1) for p in model.parameters()])


def gen_init(out):
    from utils.setup_elements import setup_architecture
    for k, (data, seed) in enumerate(INIT_CASES):
        params = ref_harness.make_params('gdumb', data=data, cuda=False)
        torch.manual_seed(seed)
        flat = _flat(setup_architecture(params)).numpy()
        tag = 'init%d_' % k
        out[tag + 'data'] = np.array(data)
        out[tag + 'seed'] = np.int64(seed)
        out[tag + 'sha1'] = np.array(hashlib.sha1(flat.tobytes()).hexdigest())
        out[tag + 'sample'] = flat[mg.dropin_sample(flat.size)]
        out[tag + 'after'] = torch.rand(4).numpy()
    out['n_init'] = np.int64(len(INIT_CASES))


def greedy_cases():
    """(mem_size, seed, label streams): shorter than the memory, many times the memory, ties for the largest class, a
    class whose count falls to 0, several calls with recurring and new labels."""
    rs = np.random.RandomState(2026)
    return [
        (50, 1, [rs.randint(0, 5, 30)]),
        (20, 2, [rs.randint(0, 10, 500)]),
        (10, 3, [np.array([0, 1, 2, 3, 4] * 2 + [5, 6, 0, 7, 1, 8, 9, 2, 5, 6])]),
        (4, 4, [np.array([0, 0, 0, 0, 1, 2, 3, 4, 0, 5, 0, 1, 6])]),
        (30, 5, [rs.randint(0, 10, 60), rs.randint(5, 15, 60), np.r_[rs.randint(0, 20, 40), np.arange(20, 26)]]),
    ]


def gen_greedy(out):
    cases = greedy_cases()
    for k, (mem, seed, streams) in enumerate(cases):
        params = ref_harness.make_params('gdumb', cuda=False, mem_size=mem)
        agent = ref_harness.build_agent(params)
        random.seed(seed)
        i = 0
        for y in streams:
            for lbl in np.asarray(y).tolist():
                agent.greedy_balancing_update(torch.tensor(i), int(lbl))
                i += 1
        tag = 'greedy%d_' % k
        out[tag + 'mem'] = np.int64(mem)
        out[tag + 'seed'] = np.int64(seed)
        out[tag + 'n_streams'] = np.int64(len(streams))
        for s, y in enumerate(streams):
            out[tag + 'stream%d' % s] = np.asarray(y, dtype=np.int64)
        out[tag + 'mem_c'] = np.array(list(agent.mem_c.items()), dtype=np.int64).reshape(-1, 2)
        out[tag + 'lists'] = np.array([int(t) for c in agent.mem_img for t in agent.mem_img[c]], dtype=np.int64)
        out[tag + 'after'] = np.float64(random.random())
        print('greedy', k, list(agent.mem_c.items()))
    out['n_greedy'] = np.int64(len(cases))


# Drop-in cases (calls, labels, samples per call, overrides); seed indices start at 60 so that no case shares its seeds
# with the other drop-in goldens.  lr 0.01: over tens of from-scratch steps lr 0.1 is chaotic.
GDUMB_DROPIN_CASES = [
    (3, 30, 83, dict(mem_size=100, mem_epoch=3, learning_rate=0.01)),
    (3, 30, 83, dict(mem_size=150, mem_epoch=2, learning_rate=0.01, trick={'labels_trick': True})),
    (3, 30, 83, dict(mem_size=120, mem_epoch=2, learning_rate=0.01, trick={'separated_softmax': True})),
    (2, 10, 123, dict(data='cifar10', mem_size=200, mem_epoch=3, learning_rate=0.01)),
]


def _dropin_run(i, n_calls, n_label, n_per_call, over, perturb):
    from agents import gdumb as ref_gdumb
    from continuum.data_utils import setup_test_loader
    over = dict(over)
    trick = dict(ref_harness.TRICK, **over.pop('trick', {}))
    params = ref_harness.make_params('gdumb', cuda=False, trick=trick, **over)
    hw = 84 if params.data == 'mini_imagenet' else 32
    agent = ref_harness.build_agent(params)
    inits = []
    orig = ref_gdumb.setup_architecture

    def setup_architecture(p):
        model = orig(p)
        flat = _flat(model).numpy()
        inits.append(flat[mg.dropin_sample(flat.size)].copy())
        if perturb:
            gen = torch.Generator().manual_seed(1234)
            with torch.no_grad():
                for prm in model.parameters():
                    prm.mul_(1 + (torch.randint(0, 2, prm.shape, generator=gen).float() * 2 - 1) * 2.0 ** -23)
        return model
    ref_gdumb.setup_architecture = setup_architecture
    try:
        np.random.seed(i); random.seed(i); torch.manual_seed(i)
        calls, tests = ogd.dropin_inputs(np.random.RandomState(100 + i), hw, n_label, n_per_call, n_calls)
        rec = {}
        for c, (xt, yt) in enumerate(calls):
            agent.train_learner(xt, yt)
            flat = _flat(agent.model).numpy()
            rec['mem_c%d' % c] = np.array(list(agent.mem_c.items()), dtype=np.int64).reshape(-1, 2)
            rows = torch.stack([t for k in agent.mem_img for t in agent.mem_img[k]]).numpy()
            rec['mem%d' % c] = np.array(hashlib.sha1(rows.tobytes()).hexdigest())
            rec['w_init%d' % c] = inits[-1]
            rec['w%d' % c] = flat[mg.dropin_sample(flat.size)]
            rec['bn%d' % c] = torch.cat([torch.cat([m.running_mean, m.running_var]) for m in agent.model.modules()
                                         if isinstance(m, torch.nn.BatchNorm2d)]).numpy()
        rec['acc'] = np.asarray(agent.evaluate(setup_test_loader(tests, params)), dtype=np.float64)
        rec['params'] = np.array(json.dumps(vars(params), sort_keys=True))
    finally:
        ref_gdumb.setup_architecture = orig
    return rec


def gen_dropin(out):
    def rel(a, b):
        return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))

    for k, (n_calls, n_label, n_per_call, over) in enumerate(GDUMB_DROPIN_CASES):
        i = 60 + k
        tag = 'c%d_' % k
        rec = _dropin_run(i, n_calls, n_label, n_per_call, over, False)
        alt = _dropin_run(i, n_calls, n_label, n_per_call, over, True)
        for key, v in rec.items():
            out[tag + key] = v
        out[tag + 'spread_w'] = np.array([rel(alt['w%d' % c].astype(np.float64) - rec['w_init%d' % c],
                                              rec['w%d' % c].astype(np.float64) - rec['w_init%d' % c])
                                          for c in range(n_calls)])
        out[tag + 'spread_bn'] = np.array([rel(alt['bn%d' % c].astype(np.float64), rec['bn%d' % c].astype(np.float64))
                                           for c in range(n_calls)])
        out[tag + 'case'] = np.array(json.dumps([n_calls, n_label, n_per_call, i, 100 + i]))
        print('dropin', k, rec['acc'], 'one-ulp spread', out[tag + 'spread_w'], out[tag + 'spread_bn'])
    out['n_dropin'] = np.int64(len(GDUMB_DROPIN_CASES))


if __name__ == '__main__':
    out = {}
    gen_init(out)
    gen_greedy(out)
    gen_dropin(out)
    path = os.path.join(mg.HERE, 'gdumb.npz')
    np.savez_compressed(path, **out)
    print('gdumb.npz', os.path.getsize(path))
