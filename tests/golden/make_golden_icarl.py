"""Generate tests/golden/icarl.npz by EXECUTING THE REFERENCE (build container only): the iCaRL agent (agents/icarl.py).

    python tests/golden/make_golden_icarl.py REFERENCE_CHECKOUT

Uses the import recipe of make_golden.py and the drop-in recorder of make_golden_tricks.py (both imported, not
changed), and records
  (a) loss-level cases: the reference's own Icarl.update_representation over one batch, with a stub model whose forward
      returns seeded logits as a leaf tensor, a stub previous model returning seeded teacher logits and lr = 0; the
      loss handed to backward() and autograd's d loss / d logits.  The logits are not stored: case k draws them from
      RandomState(LOSS_SEED + k) (oracle/icarl.py case_logits, which the tests use too);
  (b) drop-in runs of the agent in the format of make_golden.py gen_dropin, with the one-ulp spread
      (tests/test_gpu_icarl.py runs tests/test_gpu_dropin.py's comparison on them).
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_tricks as mgt  # noqa: E402  (make_golden's import recipe: reads the checkout from sys.argv[1])

from oracle.icarl import LOSS_SEED, case_logits  # noqa: E402  (the repository root is on sys.path: make_golden)

mg = mgt.mg
ref_harness = mgt.ref_harness


def loss_cases():
    """(C, B, old_labels, new_labels, teacher, scale): the first task (no teacher), later tasks with a teacher,
    recurring labels with K at or just below C, 10 and 100 classes, and logits in the hundreds."""
    rs = np.random.RandomState(2025)
    p10, p100 = rs.permutation(10).tolist(), rs.permutation(100).tolist()
    return [
        (10, 10, [], p10, False, 3.0),                                            # first task
        (100, 10, [], p100[:10], False, 3.0),
        (100, 20, [], p100[:20], False, 3.0),
        (10, 10, p10[:5], p10[5:], True, 3.0),                                    # teacher from the second task on
        (100, 10, p100[:30], p100[30:40], True, 3.0),
        (100, 20, p100[:50], p100[50:60], True, 3.0),
        (10, 10, [0, 1, 2, 3, 4, 0, 1, 2], [1, 0], True, 3.0),                    # recurring labels, K = C
        (100, 10, list(range(60)) + list(range(30, 50)), list(range(40, 60)), True, 3.0),   # K = C
        (100, 10, list(range(40)) + list(range(40)), p100[:19], True, 3.0),       # K = C - 1
        (10, 10, [], p10, False, 150.0),                                          # extreme logits
        (10, 10, p10[:5], p10[5:], True, 150.0),
        (100, 10, p100[:30], p100[30:40], True, 100.0),
    ]


class _Fixed(torch.nn.Module):
    """A model whose forward returns fixed logits (a parameter, so that autograd and the optimizer see a leaf)."""

    def __init__(self, z, grad=True):
        super().__init__()
        self.z = torch.nn.Parameter(torch.tensor(z), requires_grad=grad)

    def forward(self, x):
        assert x.shape[0] == self.z.shape[0], (x.shape, self.z.shape)
        return self.z


def _reference_loss(C, B, old, new, logits, teacher, labels):
    """One batch through the reference's Icarl.update_representation: (loss, d loss / d logits)."""
    params = ref_harness.make_params('icarl', cuda=False, batch=B, mem_size=50, data='cifar100')
    agent = ref_harness.build_agent(params)
    agent.buffer.update(torch.zeros(50, 3, 32, 32), torch.zeros(50, dtype=torch.int64))    # memory rows to draw
    agent.old_labels, agent.new_labels = list(old), list(new)
    student = _Fixed(logits)
    agent.model = student
    agent.opt = torch.optim.SGD(student.parameters(), lr=0.0)
    agent.prev_model = _Fixed(teacher, grad=False) if teacher is not None else None
    seen = []
    orig = torch.Tensor.backward

    def backward(self, *a, **k):
        seen.append(float(self.detach()))
        return orig(self, *a, **k)
    torch.Tensor.backward = backward
    try:
        agent.update_representation([(torch.zeros(B, 3, 32, 32), torch.tensor(labels))])
    finally:
        torch.Tensor.backward = orig
    assert len(seen) == 1
    return seen[0], student.z.grad.numpy().copy()


def gen_icarl():
    out = {}
    rs = np.random.RandomState(77)
    cases = loss_cases()
    for k, (C, B, old, new, teach, scale) in enumerate(cases):
        tag = 'l%d_' % k
        rows = 2 * B if teach else B
        logits, teacher = case_logits(LOSS_SEED + k, rows, C, scale, teach)
        labels = np.asarray(new, dtype=np.int64)[rs.randint(0, len(new), B)]
        loss, grad = _reference_loss(C, B, old, new, logits, teacher, labels)
        out.update({tag + 'shape': np.array([rows, C], dtype=np.int64), tag + 'labels': labels.astype(np.int16),
                    tag + 'old': np.array(old, dtype=np.int64), tag + 'new': np.array(new, dtype=np.int64),
                    tag + 'teacher': np.bool_(teach), tag + 'scale': np.float64(scale), tag + 'loss': np.float64(loss),
                    tag + 'dlogits': grad})
        print('loss case', k, C, B, len(old), len(new), teach, scale, loss)
    out['n_loss_cases'] = np.int64(len(cases))
    dropin = {'n_cases': np.int64(len(ICARL_DROPIN_CASES))}
    mgt._dropin_record(ICARL_DROPIN_CASES, 40, dropin)
    out.update({'dropin_' + k: v for k, v in dropin.items()})
    np.savez_compressed(os.path.join(mg.HERE, 'icarl.npz'), **out)


# Drop-in cases (kind, calls, labels, overrides); seed indices start at 40 so that no case shares its seeds with the
# other drop-in goldens.  Each call holds one batch of labels 0..12, which recur in every call; the previous model
# exists from the second call on.  13 labels: every buffered label is seen in training, which the nearest-class-mean
# evaluation of the reference requires (agents/base.py:126).
# The runs with more than one step per call take lr 0.01: at 0.1 the reference's own one-ulp runs end several test
# samples apart, beyond the fixed accuracy bar of the comparison.
ICARL_DROPIN_CASES = [
    ('icarl', 3, 13, dict(mem_size=1000)),
    ('icarl', 3, 13, dict(mem_size=1000, epoch=3, learning_rate=0.01)),     # written slots leave the later draws
    ('icarl', 3, 13, dict(mem_size=200, learning_rate=0.01, trick={'review_trick': True, 'kd_trick': True})),   # teacher
]                                                                           # from before the review


if __name__ == '__main__':
    gen_icarl()
    print('icarl.npz', os.path.getsize(os.path.join(mg.HERE, 'icarl.npz')))
