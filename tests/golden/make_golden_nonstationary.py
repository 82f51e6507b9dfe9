"""Generate tests/golden/nonstationary.npz by EXECUTING THE REFERENCE (build container only): the non-stationary
new-instance tasks (--cl_type ni --ns_type noise|occlusion, continuum/non_stationary.py), whose images reach the agents
as float64 NHWC arrays in [0, 1], and short drop-in runs of the agents on them.

    python tests/golden/make_golden_nonstationary.py REFERENCE_CHECKOUT

Uses the import recipe of make_golden.py (skimage and matplotlib stubbed: neither is on the noise or occlusion path;
kornia's augmentations stubbed to Identity, which SCR's transform uses), the dropin_sample of its drop-in recorder and
make_golden_core50.py's one-ulp spread helpers (imported, not changed), and records
  (a) the sha1 of every array the reference's construct_ns_multiple builds from seeded uint8 splits, for noise and
      occlusion with several factors including 0, at 32x32 and 84x84, and one numpy and one `random` draw taken
      afterwards (they pin the number of draws);
  (b) drop-in runs on such streams, one factor per call (the format of make_golden_openloris.py): at 32x32 (cifar100)
      ER, ER with MIR, ER with ASER, A-GEM, LwF, EWC++, SCR with the mlp head and iCaRL over its first call; at 84x84
      (mini_imagenet, float64 labels as its loader makes them) ER, ER with ASER and SCR; GDumb at both sizes.
      Every call holds all 100 classes in one 100-image step at lr 0.01, as the OpenLORIS runs do, so that the
      reference's own one-ulp spread stays small enough for the 10x bar to check something.
No image is stored: every input is drawn from a seed and built by oracle/nonstationary.py on the test side.
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
from continuum import non_stationary as ref_ns  # noqa: E402  (skimage / matplotlib are stubs: make_golden)

NCLS = 100
BATCH = 100                    # stream batch: one replay step per call carries all 100 classes
PER_CALL = BATCH + 3           # images per train_learner call (the 3 extra rows exercise drop_last)
N_TEST = 100                   # test images per task, every class once
DATA = {32: 'cifar100', 84: 'mini_imagenet'}

# (a) (hw, ns_type, factors, seed): each task of the split has 5 train, 2 val and 3 test images
SHA_CASES = [(32, 'noise', [0, 0.6, 1.4, 2.2, 3], 300), (32, 'occlusion', [0, 0.2, 0.4, 0.8], 301),
             (84, 'noise', [0.0, 0.4, 2.0, 3.6], 302), (84, 'occlusion', [0.0, 0.1, 0.6, 1.0], 303)]

# (b) (kind, hw, ns_type, factors, overrides); seed indices start at 310 so that no case shares its seeds with another
# golden.  One factor per call; iCaRL runs one call (its second is refused).
DROPIN_CASES = [
    ('er', 32, 'noise', [0, 1.4], dict(mem_size=200, learning_rate=0.01)),
    ('mir', 32, 'occlusion', [0.4, 0.8], dict(mem_size=200, learning_rate=0.01)),
    ('aser', 32, 'noise', [0.6, 3], dict(mem_size=400, n_smp_cls=2.0, learning_rate=0.01)),   # 200 candidates
    ('agem', 32, 'occlusion', [0, 0.4], dict(mem_size=200, learning_rate=0.01)),
    ('lwf', 32, 'noise', [1.4, 2.2], dict(mem_size=10, learning_rate=0.01)),
    ('ewc', 32, 'occlusion', [0.2, 0.6], dict(mem_size=10, learning_rate=0.01, lambda_=100.0, alpha=0.9,
                                              fisher_update_after=1)),
    ('scr', 32, 'noise', [0.6, 1.4], dict(mem_size=200, learning_rate=0.01, head='mlp')),
    ('icarl', 32, 'noise', [2.2], dict(mem_size=200, learning_rate=0.01)),
    ('er', 84, 'noise', [0.0, 1.2], dict(mem_size=200, learning_rate=0.01)),
    ('aser', 84, 'occlusion', [0.2, 0.6], dict(mem_size=400, n_smp_cls=2.0, learning_rate=0.01)),
    ('scr', 84, 'noise', [0.8, 2.0], dict(mem_size=200, learning_rate=0.01, head='mlp')),
]
FIRST = 310
# GDumb: (hw, ns_type, factors, overrides): 110 slots hold one image of each class (the class cap is 110 // 100 = 1),
# trained in two batches of 50 per epoch
GDUMB_CASES = [(32, 'occlusion', [0.4, 0.8], dict(mem_size=110, mem_epoch=2, batch=50, learning_rate=0.01)),
               (84, 'noise', [0.4, 1.6], dict(mem_size=110, mem_epoch=2, batch=50, learning_rate=0.01))]
GDUMB_FIRST = 340


def sha_splits(rs, hw, n_tasks):
    """Seeded uint8 splits of (a) (tests/test_oracle_nonstationary.py draws them the same way)."""
    def split(n):
        return ([rs.randint(0, 256, (n, hw, hw, 3)).astype(np.uint8) for _ in range(n_tasks)],
                [rs.randint(0, NCLS, n).astype(np.int64) for _ in range(n_tasks)])
    tr, va, te = split(5), split(2), split(3)
    return tr[0], tr[1], va[0], va[1], te[0], te[1]


def ns_inputs(rs, mem, hw, per_call, ns_type, factors, label_dtype, build):
    """Seeded inputs of a drop-in run (tests/test_gpu_nonstationary.py draws them the same way): a memory prefill of
    mem float images, then uint8 splits whose labels cover all the classes in every task, turned into float64 tasks by
    build (the reference's construct_ns_multiple here, oracle/nonstationary.py on the test side) under the global
    seeds dseed.  Returns the prefill, the calls and the test sets, one per task."""
    x = rs.rand(mem, 3, hw, hw).astype(np.float32)
    y = rs.randint(0, NCLS, mem).astype(np.int64)
    n = len(factors)
    tr_x = [rs.randint(0, 256, (per_call, hw, hw, 3)).astype(np.uint8) for _ in range(n)]
    tr_y = [rs.permutation(np.arange(per_call) % NCLS).astype(label_dtype) for _ in range(n)]
    va_x = [rs.randint(0, 256, (1, hw, hw, 3)).astype(np.uint8) for _ in range(n)]
    va_y = [np.zeros(1, dtype=label_dtype) for _ in range(n)]
    te_x = [rs.randint(0, 256, (N_TEST, hw, hw, 3)).astype(np.uint8) for _ in range(n)]
    te_y = [rs.permutation(np.arange(N_TEST) % NCLS).astype(label_dtype) for _ in range(n)]
    train, _, test = build(tr_x, tr_y, va_x, va_y, te_x, te_y, ns_type, factors)
    return x, y, train, test


def ref_build(*a):
    return ref_ns.construct_ns_multiple(*a, plot=False)


def _sha(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


def gen_sha(out):
    for k, (hw, ns_type, factors, seed) in enumerate(SHA_CASES):
        tag = 's%d_' % k
        splits = sha_splits(np.random.RandomState(seed), hw, len(factors))
        np.random.seed(seed); random.seed(seed)
        lists = ref_build(*splits, ns_type, factors)
        shas = []
        for part in lists:
            for xt, yt in part:
                assert xt.dtype == np.float64 and xt.shape[1:] == (hw, hw, 3) and 0 <= xt.min() and xt.max() <= 1
                shas += [_sha(xt), _sha(yt)]
        out[tag + 'sha1'] = np.array(shas)
        out[tag + 'after'] = np.array([np.random.rand(), random.random()])
        out[tag + 'case'] = np.array(json.dumps([hw, ns_type, factors, seed]))
    out['n_sha'] = np.int64(len(SHA_CASES))


def _dropin_run(i, kind, hw, ns_type, factors, over, perturb):
    """make_golden_openloris._dropin_run on float64 non-stationary calls at hw x hw with 100 classes."""
    from continuum.data_utils import setup_test_loader
    over = dict(over)
    trick = dict(ref_harness.TRICK, **over.pop('trick', {}))
    data = DATA[hw]
    params = ref_harness.make_params(kind, cuda=False, data=data, trick=trick, batch=BATCH, **over)
    spec = mg.oresnet.Spec(hw, 20, 100, head='mlp') if params.agent == 'SCR' else mg.oresnet.Spec(hw, 20, NCLS)
    mg.buffer_utils.ClassBalancedRandomSampling.class_index_cache = None
    mg.buffer_utils.ClassBalancedRandomSampling.class_num_cache = None
    agent = ref_harness.build_agent(params)
    p, bn = mg.oresnet.seeded_state(spec, 40 + i)
    sd = dict(p)
    sd.update(bn)
    agent.model.load_state_dict(sd, strict=True)
    if perturb:
        mgc._perturb(agent.model)
    dseed = 100 + i
    np.random.seed(dseed); random.seed(dseed)
    x, y, calls, tests = ns_inputs(np.random.RandomState(dseed), params.mem_size, hw, PER_CALL, ns_type, factors,
                                   np.float64 if data == 'mini_imagenet' else np.int64, ref_build)
    assert all(xt.dtype == np.float64 and np.unique(yt).size == NCLS for xt, yt in calls)
    np.random.seed(i); random.seed(i); torch.manual_seed(i)
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
    for k, (kind, hw, ns_type, factors, over) in enumerate(DROPIN_CASES):
        i = FIRST + k
        tag = 'c%d_' % k
        rec, w0 = _dropin_run(i, kind, hw, ns_type, factors, over, False)
        alt, _ = _dropin_run(i, kind, hw, ns_type, factors, over, True)
        n_calls = len(factors)
        for key, v in rec.items():
            out[tag + key] = v
        out[tag + 'spread_w'] = np.array([mgc._rel(alt['w%d' % c] - w0, rec['w%d' % c] - w0) for c in range(n_calls)])
        out[tag + 'spread_bn'] = np.array([mgc._rel(alt['bn%d' % c].astype(np.float64), rec['bn%d' % c].astype(np.float64))
                                           for c in range(n_calls)])
        if 'label0' in rec:
            out[tag + 'spread_slots'] = np.array([int((alt['label%d' % c] != rec['label%d' % c]).sum())
                                                  for c in range(n_calls)])
        out[tag + 'case'] = np.array(json.dumps([kind, hw, ns_type, factors, PER_CALL, 40 + i, i, 100 + i]))
        print('dropin', k, kind, hw, ns_type, factors, rec['acc'], 'one-ulp spread', out[tag + 'spread_w'],
              out[tag + 'spread_bn'], flush=True)
    out['n_dropin'] = np.int64(len(DROPIN_CASES))


def _gdumb_run(i, hw, ns_type, factors, over, perturb):
    """make_golden_openloris._gdumb_run on float64 non-stationary calls at hw x hw with 100 classes."""
    from agents import gdumb as ref_gdumb
    from continuum.data_utils import setup_test_loader
    data = DATA[hw]
    params = ref_harness.make_params('gdumb', cuda=False, data=data, trick=dict(ref_harness.TRICK), **over)
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
        dseed = 100 + i
        np.random.seed(dseed); random.seed(dseed)
        _, _, calls, tests = ns_inputs(np.random.RandomState(dseed), 0, hw, PER_CALL, ns_type, factors,
                                       np.float64 if data == 'mini_imagenet' else np.int64, ref_build)
        np.random.seed(i); random.seed(i); torch.manual_seed(i)
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
    for k, (hw, ns_type, factors, over) in enumerate(GDUMB_CASES):
        i = GDUMB_FIRST + k
        tag = 'g%d_' % k
        rec = _gdumb_run(i, hw, ns_type, factors, over, False)
        alt = _gdumb_run(i, hw, ns_type, factors, over, True)
        n_calls = len(factors)
        for key, v in rec.items():
            out[tag + key] = v
        out[tag + 'spread_w'] = np.array([mgc._rel(alt['w%d' % c].astype(np.float64) - rec['w_init%d' % c],
                                                   rec['w%d' % c].astype(np.float64) - rec['w_init%d' % c])
                                          for c in range(n_calls)])
        out[tag + 'spread_bn'] = np.array([mgc._rel(alt['bn%d' % c].astype(np.float64), rec['bn%d' % c].astype(np.float64))
                                           for c in range(n_calls)])
        out[tag + 'case'] = np.array(json.dumps([hw, ns_type, factors, PER_CALL, i, 100 + i]))
        print('gdumb', k, hw, rec['acc'], 'one-ulp spread', out[tag + 'spread_w'], out[tag + 'spread_bn'], flush=True)
    out['n_gdumb'] = np.int64(len(GDUMB_CASES))


if __name__ == '__main__':
    torch.set_num_threads(16)
    out = {}
    gen_sha(out)
    gen_dropin(out)
    gen_gdumb(out)
    path = os.path.join(mg.HERE, 'nonstationary.npz')
    np.savez_compressed(path, **out)
    print('nonstationary.npz', os.path.getsize(path))
