"""CPU: the C-ABI library builds, loads, and exports every symbol declared in include/b200ocl.h
(no compute calls -- there is no GPU here)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions():
    text = open(os.path.join(ROOT, 'include', 'b200ocl.h')).read()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    return sorted(set(re.findall(r'\b(b200ocl_[a-z0-9_]+)\s*\(', text)))


def test_library_exports_every_declared_symbol():
    from b200ocl import _build, _native
    _build.build()
    lib = _native.lib()
    names = _declared_functions()
    assert len(names) >= 10
    for n in names:
        assert hasattr(lib, n), 'missing export ' + n
        assert n in _native.SIGNATURES, 'ctypes signature missing for ' + n
    assert set(_native.SIGNATURES) == set(names)
    assert lib.b200ocl_version() >= 100


def test_ctypes_signatures_take_the_declared_number_of_arguments():
    """A parameter added to a declaration but not to its ctypes signature shifts every argument after it."""
    from b200ocl import _native
    text = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'b200ocl.h')).read(), flags=re.S)
    decls = dict(re.findall(r'\b(b200ocl_[a-z0-9_]+)\s*\(([^()]*)\)\s*;', text))
    assert set(decls) == set(_native.SIGNATURES)
    for name, params in decls.items():
        params = params.strip()
        n = 0 if params in ('', 'void') else params.count(',') + 1
        assert len(_native.SIGNATURES[name][1]) == n, name


def test_workspace_queries_are_pure_host_calls():
    from b200ocl import _native
    lib = _native.lib()
    assert lib.b200ocl_knn_sv_workspace_bytes(110, 160, 160) >= 256
    assert lib.b200ocl_supcon_workspace_bytes(110, 2, 128) >= 256 + 2 * 220 * 4


def test_weight_gradient_workspace_query_follows_the_kernel_geometry():
    """Host-only: the wgmma weight gradient covers 3x3 stride-1 layers on maps up to 37 wide with channel counts that are
    multiples of 4 (csrc/wgrad_tc.cuh); its partial buffer holds one [9*cin, cout] block per chain of two 128-position tiles."""
    from b200ocl import _native
    lib = _native.lib()
    q = lib.b200ocl_wgrad_tc_selftest_workspace_bytes
    for (N, H, W, cin, cout) in [(110, 32, 32, 20, 20), (10, 4, 4, 160, 160), (3, 37, 5, 8, 12)]:
        positions = (N - 1) * (H + 2) * (W + 2) + (H - 1) * (W + 2) + W          # last useful strip position + 1
        tiles = (positions + 127) // 128
        chains = (tiles + 1) // 2
        want = chains * 9 * cin * cout * 4
        got = q(N, H, W, cin, cout)
        assert want <= got < want + 256, (N, H, W, cin, cout, got, want)
    assert q(4, 38, 38, 20, 20) == 0          # wider than the staged strip
    assert q(4, 8, 8, 6, 20) == 0             # channels not a multiple of 4
    assert q(0, 8, 8, 20, 20) == 0


def test_train_workspace_grows_with_the_batch():
    """Host-only: b200ocl_net_train_workspace_bytes is monotonic in N and covers the partial buffers of both weight-gradient
    kernels (the split count of the kernel each layer runs)."""
    from b200ocl import engine
    import ctypes
    from b200ocl import _native
    desc, info, _ = engine.describe(32, 100, None)
    lib = _native.lib()
    sizes = [lib.b200ocl_net_train_workspace_bytes(ctypes.byref(desc), n) for n in (1, 10, 20, 110, 220)]
    assert all(b > a > 0 for a, b in zip(sizes, sizes[1:])), sizes
    assert sizes[2] < 2.2 * sizes[1] and sizes[4] < 2.2 * sizes[3]


def test_ops_refuse_cpu_tensors():
    import torch
    from b200ocl import _native, ops
    with pytest.raises(_native.NativeError):
        ops.knn_sv(torch.zeros(2, 4), torch.zeros(2, dtype=torch.long), torch.zeros(3, 4),
                   torch.zeros(3, dtype=torch.long), 3)
    with pytest.raises(_native.NativeError):
        ops.supcon(torch.zeros(4, 2, 8), torch.zeros(4, dtype=torch.long), 0.07)
