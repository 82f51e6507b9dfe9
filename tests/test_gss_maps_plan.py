"""CPU: the case table of tests/test_gpu_gss_maps_fp64.py and the rounding bound its cosine test asserts.

  * The networks are the four GSS runs on, with memory.py's input sizes and class counts, and their gradient arenas
    have the lengths the cosine test uses.
  * BATCHES reaches every convolution template of the eval-statistics forward and of the data gradient that some
    N in 1...10 takes, at 114, 132 and 148 SMs (b200ocl_net_conv_geom takes the SM count; nothing is launched), and
    every BN-backward form and weight-gradient kernel at the SM count the library plans for here.
  * cos_bound holds for an fp32 emulation of grad_cosine_final_kernel's arithmetic over dots and norms that span the
    decades real gradients do, including denominators on both sides of the 1e-8 clamp, and is not loose by more than
    a small factor.
  * The update plan covers the first insertion, a memory smaller than gss_batch_size, a batch that only partly fits
    and full-memory updates."""
import numpy as np
import pytest

import test_gpu_gss_maps_fp64 as gm

SMS = (114, 132, 148)


def test_networks_and_arenas():
    from b200ocl import engine, memory
    assert set(gm.DATASETS) == set(gm.ARENA)
    for data in gm.DATASETS:
        hw, ncls = memory.input_size_match[data][1], memory.n_classes[data]
        assert gm.net(data) == (hw, ncls)
        _, info, _ = engine.describe(hw, ncls)
        assert info.n_params == gm.ARENA[data], data
        assert all(1 <= n <= gm.GSS_NMAX for n in gm.BATCHES[data]) and 1 in gm.BATCHES[data]
    assert len(gm.CASES) == len(set(gm.CASES))


@pytest.mark.parametrize('data', gm.DATASETS)
def test_batches_reach_every_launch(data):
    from b200ocl import engine
    hw, ncls = gm.net(data)
    desc, info, _ = engine.describe(hw, ncls)

    def conv(N, sms):
        out = set()
        for i in range(info.n_bn):
            out.add(('train', engine.conv_geom(desc, N, i, 'train', sms).template))
            if i:
                out.add(('dgrad', engine.conv_geom(desc, N, i, 'dgrad', sms).template))
        return out

    def bwd(N):
        out = set()
        for i in range(info.n_bn):
            L = engine.train_ws_layout(desc, N, i)
            out |= {('bn', L.cout, bool(L.bn_fused)), ('wgrad', L.wgrad_kernel)}
        return out

    for sms in SMS:
        every = set().union(*[conv(N, sms) for N in range(1, gm.GSS_NMAX + 1)])
        reached = set().union(*[conv(N, sms) for N in gm.BATCHES[data]])
        assert reached == every, (sms, sorted(every - reached))
    every = set().union(*[bwd(N) for N in range(1, gm.GSS_NMAX + 1)])
    assert set().union(*[bwd(N) for N in gm.BATCHES[data]]) == every


def test_cos_bound_covers_the_final_kernel():
    """fl(fl(dot) / fmaxf(sqrtf(fl(|m|^2)) * sqrtf(fl(|g|^2)), fl(1e-8))) in numpy float32 (correctly rounded, like
    the kernel's sqrtf and division) against the fp64 cosine."""
    import torch
    rs = np.random.RandomState(0)
    n = 1221190
    worst = 0.0
    for _ in range(20):
        nm = 10.0 ** rs.uniform(-24, 6, 20000)
        ng = 10.0 ** rs.uniform(-12, 6, 20000)
        # denominators within 1e-3 of the clamp on both sides
        ng[:2000] = (1e-8 * (1 + rs.uniform(-1e-3, 1e-3, 2000))) ** 2 / nm[:2000]
        cos = np.concatenate([rs.uniform(-1, 1, 10000), rs.uniform(-1e-6, 1e-6, 10000)])
        dot = cos * np.sqrt(nm * ng)
        den32 = np.maximum(np.sqrt(nm.astype(np.float32)) * np.sqrt(ng.astype(np.float32)), np.float32(1e-8))
        got = (dot.astype(np.float32) / den32).astype(np.float64)
        ref = dot / np.maximum(np.sqrt(nm) * np.sqrt(ng), 1e-8)
        bound = gm.cos_bound(torch.from_numpy(ref), n).numpy()
        assert (np.abs(got - ref) <= bound).all()
        worst = max(worst, float((np.abs(got - ref) / bound).max()))
    assert worst > 0.3           # a bound many times the worst case would check little


def test_update_plan():
    for data, strength, gbs, mem, _ in gm.UPDATE_CASES:
        plan = gm.update_plan(mem, gbs)
        sizes = [n for n, _ in plan]
        assert sizes[0] < gbs                               # the next fill draws sub-batches of current_index < gbs
        filled = np.cumsum(sizes)
        assert mem in filled or any(a < mem < b for a, b in zip(filled, filled[1:]))
        assert sum(1 for f in filled[:-1] if f >= mem) >= 4  # full-memory updates
        assert mem // gbs >= strength                      # the full memory gives K = gss_mem_strength rows
