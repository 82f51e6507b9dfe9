"""Generate tests/golden/error_analysis.npz by EXECUTING THE REFERENCE (build container only): its evaluate() with
--error_analysis (agents/base.py:144-226).

    python tests/golden/make_golden_error_analysis.py REFERENCE_CHECKOUT

Uses make_golden.py's import recipe and drop-in inputs (through make_golden_core50.py's helpers, imported, not changed)
and runs every evaluate() in a temporary working directory, where the reference writes its `confusion` pickle.  Records
  (a) the reference's evaluate(error_analysis=True) on a seeded CIFAR-10 ER network and seeded test loaders at several
      label-bookkeeping states (set by before_train / after_train, no training): class-incremental after 1, 3 and 5
      tasks of two classes (the classes no task has reached get bias -1000, so that nothing predicts them), new-instance
      after two tasks of all ten classes (old_labels repeats every label: the old-class means are NaN), and one state
      where every row predicts a class never trained on (KeyError).  Per state: the logits the network produced for
      every test batch, the labels, the bookkeeping, the classifier and what the analysis appended, printed and wrote;
  (b) short drop-in runs (make_golden.py gen_dropin's recipe at CIFAR-10, lr 0.01) of ER, ER + ASER, A-GEM, LwF, EWC++
      and GDumb with the analysis on at every call: call 0 holds all ten classes, call 1 classes 0-4, call 2 classes
      5-9, so that every prediction has a task and the four error counts all occur.  After every call: the accuracies,
      the appended analysis and the confusion lists, for the recorded run and for the run from weights perturbed by one
      ulp (the reference's own fp32 spread).  The test loaders are unshuffled, batch 32, and the default torch generator
      is restored around each evaluate() so that the analysis does not move the training draws.
No image is stored: every input is drawn from a seed.
"""
import contextlib
import io
import json
import os
import pickle
import random
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_core50 as mgc  # noqa: E402  (make_golden's import recipe: reads the checkout from sys.argv[1])

mg = mgc.mg
ref_harness = mgc.ref_harness
HW, NCLS = 32, 10
TEST_BATCH = 32
CI_TASKS = [[0, 1], [2, 3], [4, 5], [6, 7], [8, 9]]
NI_TASKS = [list(range(NCLS))] * 2
# (name, tasks of the bookkeeping, task_seen, forced class: every row predicts it)
EVAL_CASES = [('ci1', CI_TASKS, 1, None), ('ci3', CI_TASKS, 3, None), ('ci5', CI_TASKS, 5, None),
              ('ni2', NI_TASKS, 2, None), ('unseen', CI_TASKS, 2, 9)]
EVAL_FIRST = 300
# (kind, overrides) of the drop-in runs, seed indices from 320; GDumb as make_golden_gdumb.py runs it
DROPIN_CASES = [('er', dict(mem_size=200)), ('aser', dict(mem_size=200)), ('agem', dict(mem_size=200)),
                ('lwf', dict(mem_size=10)), ('ewc', dict(mem_size=10, fisher_update_after=1)),
                ('gdumb', dict(mem_size=40, mem_epoch=2))]
DROPIN_FIRST = 320
CALL_LABELS = [list(range(NCLS)), [0, 1, 2, 3, 4], [5, 6, 7, 8, 9]]


def eval_inputs(rs, tasks, n=50):
    """Seeded test sets, one per task of the bookkeeping: n uint8 NHWC images with labels drawn from the task's."""
    return [(rs.randint(0, 256, (n, HW, HW, 3)).astype(np.uint8), rs.choice(t, n).astype(np.int64)) for t in tasks]


def dropin_inputs(rs, mem, batch):
    """make_golden.py dropin_inputs with the labels of CALL_LABELS per call and one test set per call's labels."""
    x = rs.rand(mem, 3, HW, HW).astype(np.float32)
    y = rs.randint(0, NCLS, mem).astype(np.int64)
    calls = []
    for labels in CALL_LABELS:
        n = batch + 3
        calls.append((rs.randint(0, 256, (n, HW, HW, 3)).astype(np.uint8),
                      rs.permutation(np.asarray(labels)[np.arange(n) % len(labels)]).astype(np.int64)))
    tests = [(rs.randint(0, 256, (96, HW, HW, 3)).astype(np.uint8),
              rs.permutation(np.asarray(labels)[np.arange(96) % len(labels)]).astype(np.int64)) for labels in CALL_LABELS]
    return x, y, calls, tests


def loaders(tests, params):
    """The reference's test loaders (continuum/data_utils.py:57-64) without the shuffle."""
    from continuum.data_utils import dataset_transform
    from utils.setup_elements import transforms_match
    return [torch.utils.data.DataLoader(dataset_transform(x, y, transform=transforms_match[params.data]),
                                        batch_size=params.test_batch, shuffle=False, num_workers=0) for x, y in tests]


def run_evaluate(agent, test_loaders):
    """agent.evaluate in a temporary directory with the default generator restored afterwards: (acc or None,
    raised exception name or '', stdout, [correct_lb, predict_lb] or None)."""
    state = torch.get_rng_state()
    cwd = os.getcwd()
    out = io.StringIO()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            with contextlib.redirect_stdout(out):
                acc, raised = np.asarray(agent.evaluate(test_loaders), dtype=np.float64), ''
        except Exception as e:          # noqa: BLE001  (recorded: the test expects the same exception)
            acc, raised = None, type(e).__name__
        finally:
            os.chdir(cwd)
        conf = None
        if os.path.exists(os.path.join(tmp, 'confusion')):
            with open(os.path.join(tmp, 'confusion'), 'rb') as fp:
                conf = pickle.load(fp)
    torch.set_rng_state(state)
    return acc, raised, out.getvalue(), conf


def analysis(agent):
    """The last entries the analysis appended: (no, nn, oo, on) and [new score, old score, fc new, fc old, bias new,
    bias old]."""
    return (np.array(agent.error_list[-1], dtype=np.int64),
            np.array([agent.new_class_score[-1], agent.old_class_score[-1], agent.fc_norm_new[-1], agent.fc_norm_old[-1],
                      agent.bias_norm_new[-1], agent.bias_norm_old[-1]], dtype=np.float64))


def gen_eval(out):
    for k, (name, tasks, task_seen, forced) in enumerate(EVAL_CASES):
        i = EVAL_FIRST + k
        tag = 'e%d_' % k
        params = ref_harness.make_params('er', cuda=False, data='cifar10', error_analysis=True, test_batch=TEST_BATCH,
                                         mem_size=10)
        agent = ref_harness.build_agent(params)
        p, bn = mg.oresnet.seeded_state(mg.oresnet.Spec(HW, 20, NCLS), i)
        sd = dict(p)
        sd.update(bn)
        agent.model.load_state_dict(sd, strict=True)
        for t in range(task_seen):
            agent.before_train(None, np.asarray(tasks[t], dtype=np.int64))
            agent.after_train()
        with torch.no_grad():
            seen = set(agent.old_labels)
            for c in range(NCLS):
                if c not in seen:
                    agent.model.linear.bias[c] = -1000.0
            if forced is not None:
                agent.model.linear.bias[forced] = 1000.0
        rec_logits = []
        fwd = agent.model.forward

        def forward(x):
            y = fwd(x)
            rec_logits.append(y.detach().numpy().copy())
            return y
        agent.model.forward = forward
        test_loaders = loaders(eval_inputs(np.random.RandomState(100 + i), tasks), params)
        labels = [y.numpy() for ld in test_loaders for _, y in ld]
        batch_task = [t for t, ld in enumerate(test_loaders) for _ in ld]
        acc, raised, printed, conf = run_evaluate(agent, test_loaders)
        out[tag + 'name'] = np.array(name)
        out[tag + 'task_seen'] = np.int64(task_seen)
        out[tag + 'old_labels'] = np.array(agent.old_labels, dtype=np.int64)
        out[tag + 'zombie'] = np.array(agent.new_labels_zombie, dtype=np.int64)
        out[tag + 'class_task_map'] = np.array(sorted(agent.class_task_map.items()), dtype=np.int64).reshape(-1, 2)
        out[tag + 'W'] = agent.model.linear.weight.detach().numpy().copy()
        out[tag + 'b'] = agent.model.linear.bias.detach().numpy().copy()
        out[tag + 'logits'] = np.concatenate(rec_logits[:len(labels)]) if rec_logits else np.zeros((0, NCLS), np.float32)
        out[tag + 'n_rows'] = np.array([len(y) for y in labels[:len(rec_logits)]], dtype=np.int64)
        out[tag + 'batch_task'] = np.array(batch_task, dtype=np.int64)
        out[tag + 'labels'] = np.concatenate(labels)
        out[tag + 'raised'] = np.array(raised)
        out[tag + 'printed'] = np.array(printed)
        if not raised:
            err, scores = analysis(agent)
            out[tag + 'error'], out[tag + 'scores'] = err, scores
            out[tag + 'acc'] = acc
            out[tag + 'correct_lb'] = np.array(conf[0], dtype=np.int64)
            out[tag + 'predict_lb'] = np.array(conf[1], dtype=np.int64)
        else:
            assert not agent.error_list and conf is None
        print('eval', name, raised or (out[tag + 'error'], out[tag + 'scores']), flush=True)
    out['n_eval'] = np.int64(len(EVAL_CASES))


def _dropin_run(i, kind, over, perturb):
    over = dict(over)
    params = ref_harness.make_params(kind, cuda=False, data='cifar10', error_analysis=True, test_batch=TEST_BATCH,
                                     learning_rate=0.01, trick=dict(ref_harness.TRICK), **over)
    agent = ref_harness.build_agent(params)
    if kind == 'gdumb':
        from agents import gdumb as ref_gdumb
        orig = ref_gdumb.setup_architecture

        def setup_architecture(p):
            model = orig(p)
            if perturb:
                mgc._perturb(model)
            return model
        ref_gdumb.setup_architecture = setup_architecture
    else:
        mg.buffer_utils.ClassBalancedRandomSampling.class_index_cache = None
        mg.buffer_utils.ClassBalancedRandomSampling.class_num_cache = None
        p, bn = mg.oresnet.seeded_state(mg.oresnet.Spec(HW, 20, NCLS), 40 + i)
        sd = dict(p)
        sd.update(bn)
        agent.model.load_state_dict(sd, strict=True)
        if perturb:
            mgc._perturb(agent.model)
    try:
        np.random.seed(i); random.seed(i); torch.manual_seed(i)
        x, y, calls, tests = dropin_inputs(np.random.RandomState(100 + i), params.mem_size, params.batch)
        if hasattr(agent, 'buffer'):
            agent.buffer.update(torch.from_numpy(x), torch.from_numpy(y))
        test_loaders = loaders(tests, params)
        rec = {}
        for c, (xt, yt) in enumerate(calls):
            agent.train_learner(xt, yt)
            acc, raised, _, conf = run_evaluate(agent, test_loaders)
            assert not raised, (kind, c, raised)
            err, scores = analysis(agent)
            rec.update({'acc%d' % c: acc, 'error%d' % c: err, 'scores%d' % c: scores,
                        'correct_lb%d' % c: np.array(conf[0], dtype=np.int64),
                        'predict_lb%d' % c: np.array(conf[1], dtype=np.int64)})
        rec['params'] = np.array(json.dumps(vars(params), sort_keys=True))
    finally:
        if kind == 'gdumb':
            ref_gdumb.setup_architecture = orig
    return rec


def gen_dropin(out):
    for k, (kind, over) in enumerate(DROPIN_CASES):
        i = DROPIN_FIRST + k
        tag = 'd%d_' % k
        rec = _dropin_run(i, kind, over, False)
        alt = _dropin_run(i, kind, over, True)
        for key, v in rec.items():
            out[tag + key] = v
        for c in range(len(CALL_LABELS)):
            # the reference's own one-ulp spread: rows whose predicted task moved, and the relative move of each mean
            out[tag + 'spread_pred%d' % c] = np.int64((alt['predict_lb%d' % c] != rec['predict_lb%d' % c]).sum()
                                                      + np.abs(alt['error%d' % c] - rec['error%d' % c]).sum())
            a, r = alt['scores%d' % c], rec['scores%d' % c]
            with np.errstate(invalid='ignore', divide='ignore'):
                out[tag + 'spread_scores%d' % c] = np.where(np.isnan(r), 0.0, np.abs(a - r) / np.maximum(np.abs(r), 1e-30))
        out[tag + 'case'] = np.array(json.dumps([kind, len(CALL_LABELS), i, 100 + i]))
        print('dropin', k, kind, [rec['error%d' % c].tolist() for c in range(len(CALL_LABELS))],
              [out[tag + 'spread_pred%d' % c] for c in range(len(CALL_LABELS))], flush=True)
    out['n_dropin'] = np.int64(len(DROPIN_CASES))


if __name__ == '__main__':
    torch.set_num_threads(16)
    out = {}
    gen_eval(out)
    gen_dropin(out)
    path = os.path.join(mg.HERE, 'error_analysis.npz')
    np.savez_compressed(path, **out)
    print('error_analysis.npz', os.path.getsize(path))
