"""Generate tests/golden/openloris.npz by EXECUTING THE REFERENCE (build container only): OpenLORIS's network (50x50
inputs, plain Reduced_ResNet18(69), utils/setup_elements.py:67-68) and short drop-in runs of the agents on it over
new-instance streams, where every call carries all 69 classes and old_labels repeats them from the second call on.

    python tests/golden/make_golden_openloris.py REFERENCE_CHECKOUT

Uses the import recipe of make_golden.py (kornia's augmentations stubbed to Identity, which SCR's transform uses), the
dropin_sample of its drop-in recorder and make_golden_core50.py's one-ulp spread helpers (imported, not changed), and
records
  (a) setup_architecture for 'openloris' under two seeds: the sha1 of the flat parameters, a 2048-element sample and
      the torch.rand(4) drawn afterwards (the draws GDumb's re-initialisation follows);
  (b) the reference network's train-mode forward and backward from the oracle's seeded weights on a seeded 50x50 batch:
      the logits, the loss, a gradient sample per tensor and the BN running statistics afterwards;
  (c) drop-in runs at 50x50 with 69 classes on new-instance streams (ni_inputs: every call holds all the classes): ER,
      ER with ASER (2 x 69 = 138 candidates), ER with MIR, A-GEM, LwF, EWC++, SCR with the mlp head, ER with the
      separated softmax, ER with the NCM trick over a memory too small to hold every class, and iCaRL over its first
      call (the format of make_golden.py gen_dropin); GDumb (the format of make_golden_gdumb.py).
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
import make_golden_core50 as mgc  # noqa: E402  (make_golden's import recipe: reads the checkout from sys.argv[1])

mg = mgc.mg
ref_harness = mgc.ref_harness
HW, NCLS = 50, 69
DATA = 'openloris'

INIT_SEEDS = [5, 13]
NET_SEED, NET_BATCH = 9, 6
BATCH = 72                     # stream batch: one replay step per call carries all 69 classes
PER_CALL = BATCH + 3           # images per train_learner call (the 3 extra rows exercise drop_last)

# (kind, calls, overrides); seed indices start at 160 so that no case shares its seeds with another golden.  Every case
# takes one step per call at lr 0.01, as make_golden_core50.py's do: with seven steps of 10 per call the reference's
# own one-ulp runs drift apart by 40-50 % of the update within the first call, and the bar (10x that spread) would
# check nothing.
DROPIN_CASES = [
    ('er', 2, dict(mem_size=200, learning_rate=0.01)),
    ('aser', 2, dict(mem_size=400, n_smp_cls=2.0, learning_rate=0.01)),           # 138 candidates
    ('mir', 2, dict(mem_size=200, learning_rate=0.01)),
    ('agem', 2, dict(mem_size=200, learning_rate=0.01)),
    ('lwf', 2, dict(mem_size=10, learning_rate=0.01)),                             # the teacher from the second call
    ('ewc', 2, dict(mem_size=10, learning_rate=0.01, lambda_=100.0, alpha=0.9, fisher_update_after=1)),
    ('scr', 2, dict(mem_size=200, learning_rate=0.01, head='mlp')),
    ('er', 2, dict(mem_size=200, learning_rate=0.01, trick={'separated_softmax': True})),
    ('er', 2, dict(mem_size=40, learning_rate=0.01, trick={'ncm_trick': True})),   # most classes without exemplars
    ('icarl', 1, dict(mem_size=200, learning_rate=0.01)),                          # its second call is refused
]
FIRST = 160
# GDumb: (calls, images per call, overrides): 80 slots shared by 69 classes hold one image of each, trained in two
# batches of 34 per epoch (at batch 10 the one-ulp runs drift apart by half the update over the steps of a call)
GDUMB_CASES = [(2, PER_CALL, dict(mem_size=80, mem_epoch=2, batch=34, learning_rate=0.01))]
GDUMB_FIRST = 190


def ni_inputs(rs, mem, hw, n_label, per_call, n_calls):
    """Seeded inputs of a new-instance drop-in run (tests/test_gpu_openloris.py draws them the same way): a memory
    prefill of mem float images, n_calls calls of per_call uint8 NHWC images whose labels cover all n_label classes
    (per_call >= n_label), and two test sets of 96 images over all the classes."""
    x = rs.rand(mem, 3, hw, hw).astype(np.float32)
    y = rs.randint(0, n_label, mem).astype(np.int64)
    calls = [(rs.randint(0, 256, (per_call, hw, hw, 3)).astype(np.uint8),
              rs.permutation(np.arange(per_call) % n_label).astype(np.int64)) for _ in range(n_calls)]
    tests = [(rs.randint(0, 256, (96, hw, hw, 3)).astype(np.uint8), rs.permutation(np.arange(96) % n_label).astype(np.int64))
             for _ in range(2)]
    return x, y, calls, tests


def gen_init(out):
    from utils.setup_elements import setup_architecture
    for k, seed in enumerate(INIT_SEEDS):
        params = ref_harness.make_params('er', data=DATA, cuda=False)
        torch.manual_seed(seed)
        flat = mgc._flat(setup_architecture(params)).numpy()
        tag = 'init%d_' % k
        out[tag + 'seed'] = np.int64(seed)
        out[tag + 'sha1'] = np.array(hashlib.sha1(flat.tobytes()).hexdigest())
        out[tag + 'sample'] = flat[mg.dropin_sample(flat.size)]
        out[tag + 'after'] = torch.rand(4).numpy()
    out['n_init'] = np.int64(len(INIT_SEEDS))


def net_inputs():
    """The seeded batch of the network case (tests/test_openloris_plan.py draws it the same way)."""
    rs = np.random.RandomState(NET_SEED + 1)
    return rs.rand(NET_BATCH, 3, HW, HW).astype(np.float32), rs.randint(0, NCLS, NET_BATCH).astype(np.int64)


def gen_net(out):
    from utils.setup_elements import setup_architecture
    model = setup_architecture(ref_harness.make_params('er', data=DATA, cuda=False))
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
    out['net_bn'] = mgc._bn(model)
    out['net_n_tensors'] = np.int64(len(list(model.parameters())))


def _dropin_run(i, kind, n_calls, over, perturb):
    """make_golden_core50._dropin_run at 50x50 inputs and 69 classes on new-instance calls."""
    from continuum.data_utils import setup_test_loader
    over = dict(over)
    trick = dict(ref_harness.TRICK, **over.pop('trick', {}))
    params = ref_harness.make_params(kind, cuda=False, data=DATA, trick=trick, batch=BATCH, **over)
    spec = mg.oresnet.Spec(HW, 20, 100, head='mlp') if params.agent == 'SCR' else mg.oresnet.Spec(HW, 20, NCLS)
    mg.buffer_utils.ClassBalancedRandomSampling.class_index_cache = None
    mg.buffer_utils.ClassBalancedRandomSampling.class_num_cache = None
    agent = ref_harness.build_agent(params)
    p, bn = mg.oresnet.seeded_state(spec, 40 + i)
    sd = dict(p)
    sd.update(bn)
    agent.model.load_state_dict(sd, strict=True)
    if perturb:
        mgc._perturb(agent.model)
    np.random.seed(i); random.seed(i); torch.manual_seed(i)
    rs = np.random.RandomState(100 + i)
    x, y, calls, tests = ni_inputs(rs, params.mem_size, HW, NCLS, PER_CALL, n_calls)
    assert all(np.unique(yt).size == NCLS for _, yt in calls)
    has_buffer = hasattr(agent, 'buffer')
    if has_buffer:
        agent.buffer.update(torch.from_numpy(x), torch.from_numpy(y))
    rec, pick = {}, None
    for c, (xt, yt) in enumerate(calls):
        agent.train_learner(xt, yt)
        flat = mgc._flat(agent.model).numpy()
        pick = mg.dropin_sample(flat.size) if pick is None else pick
        if has_buffer:
            rec['label%d' % c] = agent.buffer.buffer_label.numpy().astype(np.int16)
            rec['index%d' % c] = np.int64(agent.buffer.current_index)
            rec['seen%d' % c] = np.int64(agent.buffer.n_seen_so_far)
            rec['img%d' % c] = np.array(hashlib.sha1(agent.buffer.buffer_img.numpy().tobytes()).hexdigest())
        rec['w%d' % c] = flat[pick]
        rec['bn%d' % c] = mgc._bn(agent.model)
    rec['old_labels'] = np.array(agent.old_labels, dtype=np.int64)
    rec['acc'] = np.asarray(agent.evaluate(setup_test_loader(tests, params)), dtype=np.float64)
    rec['params'] = np.array(json.dumps(vars(params), sort_keys=True))
    w0 = torch.cat([t.reshape(-1) for t in p.values()]).numpy()[pick].astype(np.float64)
    return rec, w0


def gen_dropin(out):
    for k, (kind, n_calls, over) in enumerate(DROPIN_CASES):
        i = FIRST + k
        tag = 'c%d_' % k
        rec, w0 = _dropin_run(i, kind, n_calls, over, False)
        alt, _ = _dropin_run(i, kind, n_calls, over, True)
        for key, v in rec.items():
            out[tag + key] = v
        out[tag + 'spread_w'] = np.array([mgc._rel(alt['w%d' % c] - w0, rec['w%d' % c] - w0) for c in range(n_calls)])
        out[tag + 'spread_bn'] = np.array([mgc._rel(alt['bn%d' % c].astype(np.float64), rec['bn%d' % c].astype(np.float64))
                                           for c in range(n_calls)])
        if 'label0' in rec:
            out[tag + 'spread_slots'] = np.array([int((alt['label%d' % c] != rec['label%d' % c]).sum())
                                                  for c in range(n_calls)])
        out[tag + 'case'] = np.array(json.dumps([kind, n_calls, PER_CALL, 40 + i, i, 100 + i]))
        print('dropin', k, kind, over.get('trick'), rec['acc'], 'one-ulp spread', out[tag + 'spread_w'],
              out[tag + 'spread_bn'], flush=True)
    out['n_dropin'] = np.int64(len(DROPIN_CASES))


def _gdumb_run(i, n_calls, n_per_call, over, perturb):
    """make_golden_core50._gdumb_run at 50x50 inputs on new-instance calls."""
    from agents import gdumb as ref_gdumb
    from continuum.data_utils import setup_test_loader
    params = ref_harness.make_params('gdumb', cuda=False, data=DATA, trick=dict(ref_harness.TRICK), **over)
    agent = ref_harness.build_agent(params)
    inits = []
    orig = ref_gdumb.setup_architecture

    def setup_architecture(p):
        model = orig(p)
        flat = mgc._flat(model).numpy()
        inits.append(flat[mg.dropin_sample(flat.size)].copy())
        if perturb:
            mgc._perturb(model)
        return model
    ref_gdumb.setup_architecture = setup_architecture
    try:
        np.random.seed(i); random.seed(i); torch.manual_seed(i)
        _, _, calls, tests = ni_inputs(np.random.RandomState(100 + i), 0, HW, NCLS, n_per_call, n_calls)
        rec = {}
        for c, (xt, yt) in enumerate(calls):
            agent.train_learner(xt, yt)
            flat = mgc._flat(agent.model).numpy()
            rec['mem_c%d' % c] = np.array(list(agent.mem_c.items()), dtype=np.int64).reshape(-1, 2)
            rows = torch.stack([t for k in agent.mem_img for t in agent.mem_img[k]]).numpy()
            rec['mem%d' % c] = np.array(hashlib.sha1(rows.tobytes()).hexdigest())
            rec['w_init%d' % c] = inits[-1]
            rec['w%d' % c] = flat[mg.dropin_sample(flat.size)]
            rec['bn%d' % c] = mgc._bn(agent.model)
        rec['acc'] = np.asarray(agent.evaluate(setup_test_loader(tests, params)), dtype=np.float64)
        rec['params'] = np.array(json.dumps(vars(params), sort_keys=True))
    finally:
        ref_gdumb.setup_architecture = orig
    return rec


def gen_gdumb(out):
    for k, (n_calls, n_per_call, over) in enumerate(GDUMB_CASES):
        i = GDUMB_FIRST + k
        tag = 'g%d_' % k
        rec = _gdumb_run(i, n_calls, n_per_call, over, False)
        alt = _gdumb_run(i, n_calls, n_per_call, over, True)
        for key, v in rec.items():
            out[tag + key] = v
        out[tag + 'spread_w'] = np.array([mgc._rel(alt['w%d' % c].astype(np.float64) - rec['w_init%d' % c],
                                                   rec['w%d' % c].astype(np.float64) - rec['w_init%d' % c])
                                          for c in range(n_calls)])
        out[tag + 'spread_bn'] = np.array([mgc._rel(alt['bn%d' % c].astype(np.float64), rec['bn%d' % c].astype(np.float64))
                                           for c in range(n_calls)])
        out[tag + 'case'] = np.array(json.dumps([n_calls, n_per_call, i, 100 + i]))
        print('gdumb', k, rec['acc'], 'one-ulp spread', out[tag + 'spread_w'], out[tag + 'spread_bn'], flush=True)
    out['n_gdumb'] = np.int64(len(GDUMB_CASES))


if __name__ == '__main__':
    torch.set_num_threads(16)
    out = {}
    gen_init(out)
    gen_net(out)
    gen_dropin(out)
    gen_gdumb(out)
    path = os.path.join(mg.HERE, 'openloris.npz')
    np.savez_compressed(path, **out)
    print('openloris.npz', os.path.getsize(path))
