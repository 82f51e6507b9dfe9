"""GPU: the halo-strip convolution (csrc/conv_tcp.cu) at the launches of the benchmark's step -- eval forward at
N = 210 with folded BN, residual and ReLU, and the data gradient at N = 110 and N = 20, raw and accumulating -- on
seeded inputs, bit for bit against tests/golden/conv_tcp_parent.npz.

That record holds what the kernel computed when its in-kernel timeline was added (make_golden_conv_tcp.py).  A change
of its schedule may change how taps, slices and tiles overlap, but every output element's MMAs and the order in which
its taps are added into the fp32 sum must stay as they were, so the outputs must not move by a single bit."""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import make_golden_conv_tcp as mg  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'conv_tcp_parent.npz')


@pytest.mark.gpu
@pytest.mark.parametrize('case', mg.CASES, ids=mg.key)
def test_conv_tcp_bit_identical_to_recorded(case):
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    rec = np.load(GOLDEN)
    y = mg.run(case)
    k = mg.key(case)
    if k + '_out' in rec:
        want = rec[k + '_out']
        assert np.array_equal(y.view(np.uint32), want.view(np.uint32)), \
            (k, np.flatnonzero(y.view(np.uint32) != want.view(np.uint32))[:8])
    assert mg.sha(y) == str(rec[k + '_sha256']), k


def test_golden_records_every_case():
    rec = np.load(GOLDEN)
    assert len(mg.CASES) == 20
    for c in mg.CASES:
        sha = str(rec[mg.key(c) + '_sha256'])
        assert len(sha) == 64
        if c in mg.KEEP:
            y = rec[mg.key(c) + '_out']
            _, N, C, H = c
            assert y.shape == (N, H, H, C) and y.dtype == np.float32
            assert hashlib.sha256(y.astype('<f4').tobytes()).hexdigest() == sha
