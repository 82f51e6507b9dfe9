"""Generate tests/golden/agem_maps.npz by EXECUTING THE REFERENCE (build container only): the reference's A-GEM
(agents/agem.py through its train_learner) on the CPU at Mini-ImageNet's 84x84 and CORe50's 128x128 (the 2560-input
classifier setup_elements.py puts in place), in the drop-in format of make_golden_core50.py.

    python tests/golden/make_golden_agem_maps.py REFERENCE_CHECKOUT

Per network: a memory of MEM rows filled from a seed, then N_CALLS train_learner calls of one step each (the first with
task_seen = 0, the later ones projecting against a memory draw), recorded twice as make_golden.py gen_dropin does: from
the seeded weights and from weights perturbed by one ulp (the reference's own spread, of the weights, the BN statistics
and the recorded gradients).  Besides the drop-in record
(labels, index, seen, image digest, sampled weights, BN statistics, accuracies; the inputs are
oracle.agem.dropin_inputs: memory classes 0-4, call classes 5-9) each call stores what
tests/test_oracle_agem.py replays the step from: the loader's order of the call's images, the memory slots the retrieve
returned, the source of every memory slot afterwards, the sampled stream and memory gradients, their fp64 dot products
and whether the gradient was projected.  No image is stored: every input is drawn from a seed.
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

from oracle import agem as oagem  # noqa: E402  (the repository root is on sys.path: make_golden)

mg, ref_harness = mgc.mg, mgc.ref_harness

# (data, in_hw, classes, case index: weights seed 40 + i, torch/numpy seed i, data seed 100 + i)
NETS = [('mini_imagenet', 84, 100, 160), ('core50', 128, 50, 161)]
MEM, N_CALLS, LR = 20, 3, 0.01


def _run(data, hw, ncls, i, perturb):
    from continuum.data_utils import setup_test_loader
    params = ref_harness.make_params('agem', cuda=False, data=data, trick=dict(ref_harness.TRICK), mem_size=MEM,
                                     learning_rate=LR)
    spec = mg.oresnet.Spec(hw, 20, ncls)
    agent = ref_harness.build_agent(params)
    p, bn = mg.oresnet.seeded_state(spec, 40 + i)
    sd = dict(p)
    sd.update(bn)
    agent.model.load_state_dict(sd, strict=True)
    if perturb:
        mgc._perturb(agent.model)
    prms = [q for q in agent.model.parameters() if q.requires_grad]
    grads = []                                          # one flat gradient per backward pass
    pending = {}

    def hook(k):
        def fn(gr):
            pending[k] = gr.detach().reshape(-1).clone()
            if len(pending) == len(prms):
                grads.append(torch.cat([pending[j] for j in range(len(prms))]))
                pending.clear()
        return fn
    for k, q in enumerate(prms):
        q.register_hook(hook(k))
    inputs, retrieved, stepped = [], [], []
    fwd, ret, step = agent.forward, agent.buffer.retrieve, agent.opt.step
    agent.forward = lambda x: (inputs.append(x.detach().clone()), fwd(x))[1]

    def retrieve(*a, **k):
        before = agent.buffer.buffer_img.clone()
        mx, my = ret(*a, **k)
        retrieved.append([int((before == r).flatten(1).all(1).nonzero()[0]) for r in mx])
        return mx, my
    agent.buffer.retrieve = retrieve
    agent.opt.step = lambda *a, **k: (stepped.append(torch.cat([q.grad.reshape(-1).clone() for q in prms])), step(*a, **k))[1]

    np.random.seed(i); random.seed(i); torch.manual_seed(i)
    rs = np.random.RandomState(100 + i)
    x, y, calls, tests = oagem.dropin_inputs(rs, MEM, hw, params.batch, N_CALLS)
    agent.buffer.update(torch.from_numpy(x), torch.from_numpy(y))
    src = np.arange(MEM, dtype=np.int64)                # slot sources: prefill row r, or 1000 (c + 1) + image of call c
    rec, pick = {}, None
    for c, (xt, yt) in enumerate(calls):
        n_in, n_ret, n_g = len(inputs), len(retrieved), len(grads)
        before = agent.buffer.buffer_img.clone()
        agent.train_learner(xt, yt)
        flat = mgc._flat(agent.model).numpy()
        pick = mg.dropin_sample(flat.size) if pick is None else pick
        imgs = torch.from_numpy(xt).permute(0, 3, 1, 2).float().div(255)
        rec['perm%d' % c] = np.array([int((imgs == r).flatten(1).all(1).nonzero()[0]) for r in inputs[n_in]], np.int64)
        buf = agent.buffer
        for sl in (buf.buffer_img != before).flatten(1).any(1).nonzero().flatten().tolist():
            src[sl] = 1000 * (c + 1) + int((imgs == buf.buffer_img[sl]).flatten(1).all(1).nonzero()[0])
        rec['src%d' % c] = src.copy()
        if len(retrieved) > n_ret:
            g, gr = grads[n_g].double(), grads[n_g + 1].double()
            rec['ret%d' % c] = np.array(retrieved[n_ret], np.int64)
            rec['dots%d' % c] = np.array([float(g @ gr), float(gr @ gr)])
            rec['proj%d' % c] = np.bool_(not torch.equal(stepped[-1], grads[n_g]))
            rec['g%d' % c], rec['gref%d' % c] = g.float().numpy()[pick], gr.float().numpy()[pick]
            rec['out%d' % c] = stepped[-1].numpy()[pick]
        rec['label%d' % c] = buf.buffer_label.numpy().astype(np.int16)
        rec['index%d' % c] = np.int64(buf.current_index)
        rec['seen%d' % c] = np.int64(buf.n_seen_so_far)
        rec['img%d' % c] = np.array(hashlib.sha1(buf.buffer_img.numpy().tobytes()).hexdigest())
        rec['w%d' % c] = flat[pick]
        rec['bn%d' % c] = mgc._bn(agent.model)
    rec['acc'] = np.asarray(agent.evaluate(setup_test_loader(tests, params)), dtype=np.float64)
    rec['params'] = np.array(json.dumps(vars(params), sort_keys=True))
    w0 = torch.cat([t.reshape(-1) for t in p.values()]).numpy()[pick].astype(np.float64)
    return rec, w0


def _rel_vec(alt, rec, key):
    if key not in rec:
        return np.nan
    return mgc._rel(alt[key].astype(np.float64), rec[key].astype(np.float64))


def gen_net(out, data, hw, ncls, i):
    rec, w0 = _run(data, hw, ncls, i, False)
    alt, _ = _run(data, hw, ncls, i, True)
    tag = data + '_'
    for k, v in rec.items():
        out[tag + k] = v
    out[tag + 'spread_w'] = np.array([mgc._rel(alt['w%d' % c] - w0, rec['w%d' % c] - w0) for c in range(N_CALLS)])
    out[tag + 'spread_bn'] = np.array([mgc._rel(alt['bn%d' % c].astype(np.float64), rec['bn%d' % c].astype(np.float64))
                                       for c in range(N_CALLS)])
    out[tag + 'spread_slots'] = np.array([int((alt['label%d' % c] != rec['label%d' % c]).sum()) for c in range(N_CALLS)])
    for key in ('g', 'gref', 'out'):                    # the one-ulp spread of the recorded gradients, per call with a draw
        out[tag + 'spread_' + key] = np.array([_rel_vec(alt, rec, key + '%d' % c) for c in range(N_CALLS)])
    out[tag + 'case'] = np.array(json.dumps(['agem', N_CALLS, 40 + i, i, 100 + i]))
    print(data, 'projected', [bool(rec.get('proj%d' % c)) for c in range(N_CALLS)], 'acc', rec['acc'],
          'one-ulp spread', out[tag + 'spread_w'], out[tag + 'spread_bn'], flush=True)


if __name__ == '__main__':
    torch.set_num_threads(16)
    out = {}
    for args in NETS:
        gen_net(out, *args)
    path = os.path.join(mg.HERE, 'agem_maps.npz')
    np.savez(path, **out)
    print('agem_maps.npz', os.path.getsize(path))
