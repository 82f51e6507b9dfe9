"""CPU: the non-stationary new-instance tasks (--cl_type ni --ns_type noise|occlusion):
  * oracle/nonstationary.py rebuilds every array the reference's construct_ns_multiple built from seeded uint8 splits
    (tests/golden/nonstationary.npz, recorded by tests/golden/make_golden_nonstationary.py), bit for bit, and leaves
    numpy's and `random`'s global generators where the reference left them;
  * learners.StreamFeeder on the CPU in parity mode turns a float64 NHWC task into the batches of the reference's
    DataLoader(shuffle=True, drop_last=True) over dataset_transform with torchvision's ToTensor and .float()
    (continuum/data_utils.py:38-54), bit for bit, and leaves the default torch generator in the same state;
  * float layouts no reference caller produces raise ValueError before any draw."""
import hashlib
import json
import os
import random

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, 'golden', 'nonstationary.npz')
NCLS = 100


def sha_splits(rs, hw, n_tasks):
    """tests/golden/make_golden_nonstationary.py sha_splits()."""
    def split(n):
        return ([rs.randint(0, 256, (n, hw, hw, 3)).astype(np.uint8) for _ in range(n_tasks)],
                [rs.randint(0, NCLS, n).astype(np.int64) for _ in range(n_tasks)])
    tr, va, te = split(5), split(2), split(3)
    return tr[0], tr[1], va[0], va[1], te[0], te[1]


def _sha(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize('case', range(int(np.load(GOLDEN)['n_sha'])))
def test_oracle_reproduces_reference_tasks(case):
    from oracle import nonstationary as ons
    g = np.load(GOLDEN)
    tag = 's%d_' % case
    hw, ns_type, factors, seed = json.loads(str(g[tag + 'case']))
    splits = sha_splits(np.random.RandomState(seed), hw, len(factors))
    np.random.seed(seed); random.seed(seed)
    lists = ons.construct_ns_multiple(*splits, ns_type, factors)
    shas = [s for part in lists for xt, yt in part for s in (_sha(xt), _sha(yt))]
    after = np.array([np.random.rand(), random.random()])
    assert shas == [str(s) for s in g[tag + 'sha1']]
    assert np.array_equal(after, g[tag + 'after'])
    # the factors cover the original task, a change that leaves pixels untouched and one that saturates some
    assert 0 in factors and all(xt.dtype == np.float64 for part in lists for xt, _ in part)


def _transform_batches(x, y, batch, seed):
    """The reference's stream: DataLoader(dataset_transform(x, y, ToTensor()), shuffle=True, drop_last=True), with
    dataset_transform restated (continuum/data_utils.py:38-54: transform, then .float())."""
    from torch.utils.data import DataLoader, Dataset
    from torchvision import transforms

    class DatasetTransform(Dataset):
        def __init__(self, x, y, transform):
            self.x, self.y, self.transform = x, torch.from_numpy(y).type(torch.LongTensor), transform

        def __len__(self):
            return len(self.y)

        def __getitem__(self, idx):
            return self.transform(self.x[idx]).float(), self.y[idx]
    torch.manual_seed(seed)
    out = list(DataLoader(DatasetTransform(x, y, transforms.Compose([transforms.ToTensor()])), batch_size=batch,
                          shuffle=True, num_workers=0, drop_last=True))
    return out, torch.rand(1)


@pytest.mark.parametrize('hw,ns_type,factor,label_dtype', [(32, 'noise', 1.4, np.int64), (84, 'occlusion', 0.4, np.float64),
                                                           (84, 'noise', 0, np.float64)])
def test_stream_feeder_matches_dataloader_on_float64_tasks(hw, ns_type, factor, label_dtype):
    from b200ocl import memory
    from b200ocl.learners import StreamFeeder
    from oracle import nonstationary as ons
    rs = np.random.RandomState(hw)
    np.random.seed(hw); random.seed(hw)
    x = ons.next_task(rs.randint(0, 256, (57, hw, hw, 3)).astype(np.uint8), ns_type, factor)
    x[0, 0, 0, 0] = 2.0 ** -140          # rounds to an fp32 subnormal
    x[0, 0, 0, 1] = 1.0 / 3.0            # rounds, not truncates
    y = rs.randint(0, 10, 57).astype(label_dtype)
    assert x.dtype == np.float64
    ref, ref_after = _transform_batches(x, y, 10, 11)
    memory.set_mode(True)
    try:
        torch.manual_seed(11)
        mine = list(StreamFeeder(x, y, 10, 'cpu'))
        after = torch.rand(1)
    finally:
        memory.set_mode(False)
    assert len(mine) == len(ref) == 5
    for (rx, ry), (mx, my, myh) in zip(ref, mine):
        assert mx.dtype == torch.float32 and mx.shape == (10, 3, hw, hw) and mx.is_contiguous()
        assert torch.equal(rx.view(torch.int32), mx.view(torch.int32))
        assert torch.equal(ry, my) and np.array_equal(ry.numpy(), myh)
    assert torch.equal(after, ref_after)


@pytest.mark.parametrize('shape,dtype', [((6, 32, 32, 3), np.float32), ((6, 32, 32, 1), np.float64),
                                         ((6, 32, 32, 1), np.float32), ((6, 32, 30, 3), np.float64),
                                         ((6, 3 * 32 * 32), np.float64)])
def test_stream_feeder_refuses_other_float_layouts(shape, dtype):
    """Float32 NHWC, one-channel, non-square and flat images are refused before the stream order is drawn."""
    from b200ocl.learners import StreamFeeder
    x = np.zeros(shape, dtype=dtype)
    y = np.arange(6, dtype=np.int64)
    torch.manual_seed(5)
    with pytest.raises(ValueError, match=r'float64 \[n,H,H,3\]'):
        StreamFeeder(x, y, 2, 'cpu')
    after = torch.rand(1)
    torch.manual_seed(5)
    assert torch.equal(after, torch.rand(1))


def test_stream_feeder_keeps_float_nchw():
    """Float NCHW tasks (the float path the feeder had before) are taken as they are."""
    from b200ocl.learners import StreamFeeder
    rs = np.random.RandomState(2)
    x = rs.rand(8, 3, 32, 32).astype(np.float32)
    torch.manual_seed(3)
    feed = StreamFeeder(x, np.arange(8), 4, 'cpu')
    torch.manual_seed(3)
    perm = torch.randperm(8).numpy()
    assert torch.equal(feed.x, torch.from_numpy(x[perm]))
