"""Generate tests/golden/core50.npz by EXECUTING THE REFERENCE (build container only): CORe50's network (128x128
inputs, Reduced_ResNet18(50) with the 2560-input classifier, utils/setup_elements.py:59-62) and short drop-in runs of
the agents on it.

    python tests/golden/make_golden_core50.py REFERENCE_CHECKOUT

Uses the import recipe of make_golden.py, its dropin_inputs / dropin_sample and the one-ulp spread of its drop-in
recorder (imported, not changed), and records
  (a) setup_architecture for 'core50' under two seeds: the sha1 of the flat parameters, a 2048-element sample and the
      torch.rand(4) drawn afterwards (the draws GDumb's re-initialisation follows);
  (b) the reference network's train-mode forward and backward from the oracle's seeded weights on a seeded batch: the
      logits, the loss, a gradient sample per tensor and the BN running statistics afterwards;
  (c) drop-in runs at 128x128 with 50 classes and a small memory: ER, ER with ASER, ER with MIR, iCaRL, EWC++ (the
      format of make_golden.py gen_dropin) and GDumb (the format of make_golden_gdumb.py).
No image is stored: every input is drawn from a seed.
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
HW, NCLS = 128, 50

INIT_SEEDS = [3, 11]
NET_SEED, NET_BATCH = 7, 6

# (kind, calls, labels, overrides); seed indices start at 120 so that no case shares its seeds with another golden.
# Every case steps at lr 0.01: at 0.1 the reference's own one-ulp runs drift apart by 5-50 % of the update from the
# second call on, so the bar (10x that spread) would check nothing after the first call.
DROPIN_CASES = [
    ('er', 3, 10, dict(mem_size=200, learning_rate=0.01)),
    ('aser', 2, 10, dict(mem_size=200, learning_rate=0.01)),
    ('mir', 2, 10, dict(mem_size=200, learning_rate=0.01)),
    ('icarl', 3, 13, dict(mem_size=200, learning_rate=0.01)),
    ('ewc', 3, 10, dict(mem_size=10, learning_rate=0.01, lambda_=100.0, alpha=0.9, fisher_update_after=1)),
]
FIRST = 120
# GDumb: (calls, labels, images per call, overrides)
GDUMB_CASES = [(2, 10, 43, dict(mem_size=40, mem_epoch=2, learning_rate=0.01))]
GDUMB_FIRST = 140


def _flat(model):
    return torch.cat([p.detach().reshape(-1) for p in model.parameters()])


def _perturb(model):
    gen = torch.Generator().manual_seed(1234)
    with torch.no_grad():
        for prm in model.parameters():
            prm.mul_(1 + (torch.randint(0, 2, prm.shape, generator=gen).float() * 2 - 1) * 2.0 ** -23)


def _bn(model):
    return torch.cat([torch.cat([m.running_mean, m.running_var]) for m in model.modules()
                      if isinstance(m, torch.nn.BatchNorm2d)]).numpy()


def _rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def gen_init(out):
    from utils.setup_elements import setup_architecture
    for k, seed in enumerate(INIT_SEEDS):
        params = ref_harness.make_params('er', data='core50', cuda=False)
        torch.manual_seed(seed)
        flat = _flat(setup_architecture(params)).numpy()
        tag = 'init%d_' % k
        out[tag + 'seed'] = np.int64(seed)
        out[tag + 'sha1'] = np.array(hashlib.sha1(flat.tobytes()).hexdigest())
        out[tag + 'sample'] = flat[mg.dropin_sample(flat.size)]
        out[tag + 'after'] = torch.rand(4).numpy()
    out['n_init'] = np.int64(len(INIT_SEEDS))


def net_inputs():
    """The seeded batch of the network case (tests/test_core50_plan.py draws it the same way)."""
    rs = np.random.RandomState(NET_SEED + 1)
    return rs.rand(NET_BATCH, 3, HW, HW).astype(np.float32), rs.randint(0, NCLS, NET_BATCH).astype(np.int64)


def gen_net(out):
    from utils.setup_elements import setup_architecture
    model = setup_architecture(ref_harness.make_params('er', data='core50', cuda=False))
    spec = mg.oresnet.Spec(HW, 20, NCLS)
    p, bn = mg.oresnet.seeded_state(spec, NET_SEED)
    sd = dict(p)
    sd.update(bn)
    model.load_state_dict(sd, strict=True)
    model.train()
    x, y = net_inputs()
    logits = model(torch.from_numpy(x))
    loss = torch.nn.functional.cross_entropy(logits, torch.from_numpy(y))
    loss.backward()
    out['net_logits'] = logits.detach().numpy()
    out['net_loss'] = np.float64(loss.item())
    for i, q in enumerate(model.parameters()):
        g = q.grad.reshape(-1).numpy()
        out['net_grad%d' % i] = g[np.random.RandomState(i).choice(g.size, min(g.size, 64), replace=False)]
    out['net_bn'] = _bn(model)
    out['net_n_tensors'] = np.int64(len(list(model.parameters())))


def _dropin_run(i, kind, n_calls, n_label, over, perturb):
    """make_golden_tricks._dropin_run at 128x128 inputs and 50 classes."""
    from continuum.data_utils import setup_test_loader
    params = ref_harness.make_params(kind, cuda=False, data='core50', trick=dict(ref_harness.TRICK), **over)
    spec = mg.oresnet.Spec(HW, 20, NCLS)
    mg.buffer_utils.ClassBalancedRandomSampling.class_index_cache = None
    mg.buffer_utils.ClassBalancedRandomSampling.class_num_cache = None
    agent = ref_harness.build_agent(params)
    p, bn = mg.oresnet.seeded_state(spec, 40 + i)
    sd = dict(p)
    sd.update(bn)
    agent.model.load_state_dict(sd, strict=True)
    if perturb:
        _perturb(agent.model)
    np.random.seed(i); random.seed(i); torch.manual_seed(i)
    rs = np.random.RandomState(100 + i)
    x, y, calls, tests = mg.dropin_inputs(rs, params.mem_size, HW, n_label, params.batch, n_calls)
    has_buffer = hasattr(agent, 'buffer')
    if has_buffer:
        agent.buffer.update(torch.from_numpy(x), torch.from_numpy(y))
    rec, pick = {}, None
    for c, (xt, yt) in enumerate(calls):
        agent.train_learner(xt, yt)
        flat = _flat(agent.model).numpy()
        pick = mg.dropin_sample(flat.size) if pick is None else pick
        if has_buffer:
            rec['label%d' % c] = agent.buffer.buffer_label.numpy().astype(np.int16)
            rec['index%d' % c] = np.int64(agent.buffer.current_index)
            rec['seen%d' % c] = np.int64(agent.buffer.n_seen_so_far)
            rec['img%d' % c] = np.array(hashlib.sha1(agent.buffer.buffer_img.numpy().tobytes()).hexdigest())
        rec['w%d' % c] = flat[pick]
        rec['bn%d' % c] = _bn(agent.model)
    rec['acc'] = np.asarray(agent.evaluate(setup_test_loader(tests, params)), dtype=np.float64)
    rec['params'] = np.array(json.dumps(vars(params), sort_keys=True))
    w0 = torch.cat([t.reshape(-1) for t in p.values()]).numpy()[pick].astype(np.float64)
    return rec, w0


def gen_dropin(out):
    for k, (kind, n_calls, n_label, over) in enumerate(DROPIN_CASES):
        i = FIRST + k
        tag = 'c%d_' % k
        rec, w0 = _dropin_run(i, kind, n_calls, n_label, over, False)
        alt, _ = _dropin_run(i, kind, n_calls, n_label, over, True)
        for key, v in rec.items():
            out[tag + key] = v
        out[tag + 'spread_w'] = np.array([_rel(alt['w%d' % c] - w0, rec['w%d' % c] - w0) for c in range(n_calls)])
        out[tag + 'spread_bn'] = np.array([_rel(alt['bn%d' % c].astype(np.float64), rec['bn%d' % c].astype(np.float64))
                                           for c in range(n_calls)])
        if 'label0' in rec:
            out[tag + 'spread_slots'] = np.array([int((alt['label%d' % c] != rec['label%d' % c]).sum())
                                                  for c in range(n_calls)])
        out[tag + 'case'] = np.array(json.dumps([kind, n_calls, n_label, 40 + i, i, 100 + i]))
        print('dropin', k, kind, rec['acc'], 'one-ulp spread', out[tag + 'spread_w'], out[tag + 'spread_bn'], flush=True)
    out['n_dropin'] = np.int64(len(DROPIN_CASES))


def _gdumb_run(i, n_calls, n_label, n_per_call, over, perturb):
    """make_golden_gdumb._dropin_run at 128x128 inputs."""
    from agents import gdumb as ref_gdumb
    from continuum.data_utils import setup_test_loader
    params = ref_harness.make_params('gdumb', cuda=False, data='core50', trick=dict(ref_harness.TRICK), **over)
    agent = ref_harness.build_agent(params)
    inits = []
    orig = ref_gdumb.setup_architecture

    def setup_architecture(p):
        model = orig(p)
        flat = _flat(model).numpy()
        inits.append(flat[mg.dropin_sample(flat.size)].copy())
        if perturb:
            _perturb(model)
        return model
    ref_gdumb.setup_architecture = setup_architecture
    try:
        np.random.seed(i); random.seed(i); torch.manual_seed(i)
        calls, tests = ogd.dropin_inputs(np.random.RandomState(100 + i), HW, n_label, n_per_call, n_calls)
        rec = {}
        for c, (xt, yt) in enumerate(calls):
            agent.train_learner(xt, yt)
            flat = _flat(agent.model).numpy()
            rec['mem_c%d' % c] = np.array(list(agent.mem_c.items()), dtype=np.int64).reshape(-1, 2)
            rows = torch.stack([t for k in agent.mem_img for t in agent.mem_img[k]]).numpy()
            rec['mem%d' % c] = np.array(hashlib.sha1(rows.tobytes()).hexdigest())
            rec['w_init%d' % c] = inits[-1]
            rec['w%d' % c] = flat[mg.dropin_sample(flat.size)]
            rec['bn%d' % c] = _bn(agent.model)
        rec['acc'] = np.asarray(agent.evaluate(setup_test_loader(tests, params)), dtype=np.float64)
        rec['params'] = np.array(json.dumps(vars(params), sort_keys=True))
    finally:
        ref_gdumb.setup_architecture = orig
    return rec


def gen_gdumb(out):
    for k, (n_calls, n_label, n_per_call, over) in enumerate(GDUMB_CASES):
        i = GDUMB_FIRST + k
        tag = 'g%d_' % k
        rec = _gdumb_run(i, n_calls, n_label, n_per_call, over, False)
        alt = _gdumb_run(i, n_calls, n_label, n_per_call, over, True)
        for key, v in rec.items():
            out[tag + key] = v
        out[tag + 'spread_w'] = np.array([_rel(alt['w%d' % c].astype(np.float64) - rec['w_init%d' % c],
                                               rec['w%d' % c].astype(np.float64) - rec['w_init%d' % c])
                                          for c in range(n_calls)])
        out[tag + 'spread_bn'] = np.array([_rel(alt['bn%d' % c].astype(np.float64), rec['bn%d' % c].astype(np.float64))
                                           for c in range(n_calls)])
        out[tag + 'case'] = np.array(json.dumps([n_calls, n_label, n_per_call, i, 100 + i]))
        print('gdumb', k, rec['acc'], 'one-ulp spread', out[tag + 'spread_w'], out[tag + 'spread_bn'], flush=True)
    out['n_gdumb'] = np.int64(len(GDUMB_CASES))


if __name__ == '__main__':
    torch.set_num_threads(16)
    out = {}
    gen_init(out)
    gen_net(out)
    gen_dropin(out)
    gen_gdumb(out)
    path = os.path.join(mg.HERE, 'core50.npz')
    np.savez_compressed(path, **out)
    print('core50.npz', os.path.getsize(path))
