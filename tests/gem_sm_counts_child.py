"""Child process of test_gpu_gem.py::test_kernels_at_other_sm_counts: the Gram, QP and projection checks of
test_gpu_gem.py with the library planning for B200OCL_SM_COUNT SMs (read once per process).  Every t = 1 ... 64 runs at
a length of two CTA slices + 1 of that count's plan and at the edge lengths around its tile and slice, so the checks
reach every geometry the plan takes there (rows_padded, tile_cols, lanes for each t; a full grid and one CTA with a
partial slice).  Prints one JSON line: the count, whether that coverage holds, and the worst ratios."""
import json
import os
import sys
from types import SimpleNamespace

import torch

import test_gpu_gem as tg


def main():
    sms = int(os.environ['B200OCL_SM_COUNT'])
    from b200ocl import _native, ops
    b = SimpleNamespace(native=_native, ops=ops)
    assert _native.lib().b200ocl_sm_count() == sms
    want, got = set(), set()
    for t in range(1, 65):
        L = ops.gem_plan(t, 1 << 22, sms)
        want.add((t, L.rows_padded, L.tile_cols, L.lanes, 'full'))
        n = 2 * int(L.chunk) + 1
        Ln = ops.gem_plan(t, n)
        got.add((t, Ln.rows_padded, Ln.tile_cols, Ln.lanes, 'full' if Ln.grid >= 3 else 'small'))
        tg._worst('gram', tg.gram_case(b, t, n, 500 + t, pitch_pad=t % 3))
    for t in (1, 5, 19, 64):
        for n in tg.edge_lengths(b, t, sms):
            tg._worst('gram', tg.gram_case(b, t, n, n + t))
    for t in (1, 3, 10, 40, 64):
        for kind in ('random', 'duplicate', 'parallel'):
            for margin in (0.0, 0.5):
                tg.qp_case(b, kind, t, margin, 2000 * t + len(kind) + int(10 * margin))
    torch.cuda.synchronize()
    print(json.dumps({'sms': sms, 'covered': want <= got, 'worst': tg.WORST}))


if __name__ == '__main__':
    sys.exit(main())
