"""Generate tests/golden/gss_maps.npz by EXECUTING THE REFERENCE (build container only): the reference's
GSSGreedyUpdate (utils/buffer/gss_greedy_update.py) driven through its Buffer on a seeded Reduced_ResNet18 on the CPU,
for OpenLORIS (50x50, 69 classes) and CORe50 (128x128, 50 classes, the 2560-input classifier setup_elements.py puts in
place), the way make_golden.py gen_gss records the CIFAR-10 run.

    python tests/golden/make_golden_gss_maps.py REFERENCE_CHECKOUT

Per network: two fill batches, then full-memory updates with classes the memory does not hold (batch_sim < 0: the
replacement lottery) and with seen classes.  The images come from a numpy stream tests/test_gpu_gss_maps_fp64.py
regenerates, so only the seeds, the labels fed, the labels and the source (update, batch position) of every slot,
the scores and batch_sim after every update are stored.
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402  (reads the reference checkout from sys.argv[1], installs the stubs)

# (data, in_hw, classes, model seed, data seed, first torch seed)
NETS = [('openloris', 50, 69, 81, 810, 2000), ('core50', 128, 50, 83, 830, 3000)]
MEM, BATCH, N_UPD = 20, 10, 6


def gen_net(out, data, hw, ncls, model_seed, data_seed, torch_seed0):
    from utils import name_match  # noqa: F401  (resolves the reference's circular import first)
    from utils.buffer.buffer import Buffer
    from utils.buffer import gss_greedy_update
    spec = mg.oresnet.Spec(hw, 20, ncls)
    model, _, _ = mg._ref_model(data, 'ER', None, spec, model_seed)
    with torch.no_grad():            # a small classifier, as gen_gss: the sign of batch_sim follows the label overlap
        model.linear.weight.mul_(0.02)
        model.linear.bias.zero_()
    params = SimpleNamespace(data=data, cuda=False, mem_size=MEM, update='GSS', retrieve='random',
                             gss_mem_strength=10, gss_batch_size=10, buffer_tracker=False, eps_mem_batch=10)
    buf = Buffer(model, params)
    upd = buf.update_method
    assert isinstance(upd, gss_greedy_update.GSSGreedyUpdate)
    sims = []
    orig = upd.get_batch_sim

    def hook(*a, **k):
        s, m = orig(*a, **k)
        sims.append(float(s))
        return s, m
    upd.get_batch_sim = hook
    rs = np.random.RandomState(data_seed)
    src = np.full((MEM, 2), -1, dtype=np.int64)
    labels, scores, srcs, batch_sim, ys = [], [], [], [], []
    for u in range(N_UPD):
        x = torch.from_numpy(rs.rand(BATCH, 3, hw, hw).astype(np.float32))
        lab = rs.randint(0, 3, BATCH)
        if u >= 2 and u % 2 == 0:
            lab = lab + 3 + 3 * ((u // 2) % 2)        # classes the memory does not hold
        y = torch.from_numpy(lab.astype(np.int64))
        torch.manual_seed(torch_seed0 + u)
        before = buf.buffer_img.clone()
        n_sims = len(sims)
        buf.update(x, y)
        for sl in (buf.buffer_img != before).flatten(1).any(1).nonzero().flatten().tolist():
            pos = [i for i in range(BATCH) if torch.equal(buf.buffer_img[sl], x[i])]
            assert len(pos) == 1
            src[sl] = (u, pos[0])
        ys.append(lab.astype(np.int64))
        labels.append(buf.buffer_label.numpy().copy())
        scores.append(upd.buffer_score.numpy().copy())
        srcs.append(src.copy())
        batch_sim.append(sims[-1] if len(sims) > n_sims else np.nan)
        print(data, 'update', u, 'batch_sim', batch_sim[-1], flush=True)
    assert model.training
    assert any(b < 0 for b in batch_sim if b == b) and any(b >= 0 for b in batch_sim if b == b)
    tag = data + '_'
    out.update({tag + 'y': np.stack(ys), tag + 'labels': np.stack(labels), tag + 'scores': np.stack(scores),
                tag + 'src': np.stack(srcs), tag + 'batch_sim': np.array(batch_sim), tag + 'mem': np.int64(MEM),
                tag + 'batch': np.int64(BATCH), tag + 'model_seed': np.int64(model_seed),
                tag + 'data_seed': np.int64(data_seed), tag + 'torch_seed0': np.int64(torch_seed0)})


if __name__ == '__main__':
    torch.set_num_threads(16)
    out = {}
    for args in NETS:
        gen_net(out, *args)
    path = os.path.join(mg.HERE, 'gss_maps.npz')
    np.savez(path, **out)
    print('gss_maps.npz', os.path.getsize(path))
