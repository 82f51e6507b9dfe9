"""Where the halo-strip convolution's time goes (GPU box): an in-kernel timeline of conv_tcp_kernel per role.

    python tools/tcp_trace.py [--build-dir DIR] [--out OUT.json]

Builds the library as usual, then a traced copy of it in its own directory (default: a fresh temporary directory):
csrc/conv_tcp.cu compiled with -DB200OCL_TCP_TRACE and linked with the other objects of the normal build.  The
shipped library never carries the stamps.  One launch per shape, at the 12 conv_tcp launches of the benchmark's step
(4 maps x {eval N = 210 with residual and ReLU, data gradient N = 110, accumulating data gradient N = 20}) on seeded
inputs through b200ocl_conv_selftest.  For every role it prints the share of its time spent in each wait, and the
time per tap next to the tensor-core floor: the 3xTF32 MMAs of both warpgroups for one tap at 1024 dense TF32 FMA
per SM and clock, at the SM clock the trace itself measures.  The card name and power limit are printed with it."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

EV = 9                                                    # TCP_EV in conv_tcp.cu
C0, C1, WLOAD, PLOAD, EPI, HDR, ROLES = range(7)
LAYERS = [(20, 32), (40, 16), (80, 8), (160, 4)]          # (channels, map) of the 3x3 stride-1 convolutions
# (label, N, dgrad, selftest mode): eval with residual + ReLU, raw data gradient, accumulating data gradient
LAUNCHES = [('eval', 210, 0, 4), ('dgrad', 110, 1, 0), ('dgrad', 20, 1, 1)]
TC_PATCH = 3


def build_traced(build_dir):
    from b200ocl import _build
    _build.build()
    os.makedirs(build_dir, exist_ok=True)
    obj = os.path.join(build_dir, 'conv_tcp_trace.o')
    src = os.path.join(_build.CSRC, 'conv_tcp.cu')
    subprocess.run([_build.NVCC] + _build.FLAGS + ['-DB200OCL_TCP_TRACE', '-c', src, '-o', obj], check=True)
    objs = [os.path.join(_build.OBJ, os.path.basename(s)[:-3] + '.o') for s in _build.sources()
            if os.path.basename(s) != 'conv_tcp.cu']
    lib = os.path.join(build_dir, 'libb200ocl_tcp_trace.so')
    subprocess.run([_build.NVCC, '-shared', '-o', lib] + objs + [obj] + _build.ARCH, check=True)
    return lib


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = 'unknown'
    return name, q


def run_shape(lib, C, H, N, dgrad, mode):
    from b200ocl import _native
    from b200ocl.ops import _stream
    from b200ocl.engine import ConvGeom
    geom = ConvGeom()
    _native.check(lib.b200ocl_conv_selftest_geom(N, H, H, C, C, 3, 1, dgrad, TC_PATCH, mode, 0, ctypes.byref(geom)),
                  'b200ocl_conv_selftest_geom')
    assert geom.kernel == 1, 'not a conv_tcp launch'
    slices = (C + 31) // 32
    T = 9 * slices
    pitch = (H + 1) * (H + 1)
    tiles = ((N - 1) * pitch + (H - 1) * (H + 1) + (H - 1)) // 128 + 1
    rounds = (tiles + geom.grid_x - 1) // geom.grid_x
    units = rounds * T
    ctas = geom.grid_x * geom.grid_y
    buf = torch.zeros(ctas * ROLES * units * EV, dtype=torch.int64, device='cuda')
    _native.check(lib.b200ocl_tcp_trace_set(buf.data_ptr(), units), 'b200ocl_tcp_trace_set')

    g = torch.Generator(device='cuda').manual_seed(1000 * C + N + dgrad)
    w = torch.randn(C, C, 3, 3, device='cuda', generator=g) / np.sqrt(9 * C)
    x = torch.randn(N, H, H, C, device='cuda', generator=g)
    if not dgrad:
        x = torch.relu(x)
    out = torch.randn(N, H, H, C, device='cuda', generator=g)
    stats = torch.cat([0.1 * torch.randn(C, device='cuda', generator=g), 0.5 + torch.rand(C, device='cuda', generator=g),
                       1 + 0.1 * torch.randn(C, device='cuda', generator=g), 0.1 * torch.randn(C, device='cuda', generator=g)])
    nbytes = lib.b200ocl_conv_selftest_workspace_bytes(N, C, C, H, H, 3, 1)
    ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
    torch.cuda.synchronize()
    rc = lib.b200ocl_conv_selftest(x.data_ptr(), w.data_ptr(), out.data_ptr(), N, H, H, C, C, 3, 1, dgrad, TC_PATCH,
                                   mode, stats.data_ptr() if mode >= 3 else None, ws.data_ptr(), nbytes, _stream())
    _native.check(rc, 'b200ocl_conv_selftest')
    torch.cuda.synchronize()
    tr = buf.view(ctas, ROLES, units, EV).cpu().numpy().astype(np.float64)
    ks = [((min(32, C - 32 * s) + 7) // 8) for s in range(slices)]
    return analyse(tr, geom, tiles, T, ks)


def analyse(tr, geom, tiles, T, ks):
    ctas = tr.shape[0]
    hdr = tr[:, HDR, 0, :]
    span_ns = hdr[:, 2].max() - hdr[:, 0].min()
    ghz = float(np.median((hdr[:, 3] - hdr[:, 1]) / (hdr[:, 2] - hdr[:, 0])))   # SM clock, cycles per ns
    cta_tiles = [len(range(c % geom.grid_x, tiles, geom.grid_x)) for c in range(ctas)]
    taps_max = max(cta_tiles) * T
    per_tap_us = span_ns / taps_max / 1e3
    floor_cyc = 2 * 128 * geom.nt * 8 * 3 * (sum(ks) / len(ks)) / 2048.0
    r = {'ctas': ctas, 'taps_per_cta': taps_max, 'span_us': span_ns / 1e3, 'sm_ghz': ghz, 'per_tap_us': per_tap_us,
         'floor_per_tap_us': floor_cyc / ghz / 1e3, 'ps': geom.tp_ps, 'bs': geom.tp_bs, 'nt': geom.nt}

    def shares(role, n_of, parts, start_ev, end_ev):
        tot = {k: 0.0 for k in parts}
        active = 0.0
        for c in range(ctas):
            n = n_of(cta_tiles[c])
            if n == 0:
                continue
            t = tr[c, role, :n]
            active += t[-1, end_ev] - t[0, start_ev]
            for k, (a, b, last_only) in parts.items():
                rows = t[T - 1::T] if last_only else t
                tot[k] += float((rows[:, b] - rows[:, a]).sum())
        out = {k: v / active for k, v in tot.items()}
        out['other'] = 1.0 - sum(out.values())
        return out

    cons = {'pfull': (0, 1, False), 'bfull': (1, 2, False), 'issue': (2, 3, False), 'wait_group': (4, 5, False),
            'promote': (5, 6, False), 'aempty': (6, 7, True), 'to_s_acc': (7, 8, True)}
    r['consumer0'] = shares(C0, lambda n: n * T, cons, 0, 8)
    r['consumer1'] = shares(C1, lambda n: n * T, cons, 0, 8)
    if not (len(ks) == 1 and geom.nt == 32):
        r['weight_loader'] = shares(WLOAD, lambda n: n * T, {'bempty': (0, 1, False), 'copy': (1, 2, False)}, 0, 2)
    slices = len(ks)
    r['patch_loaders'] = shares(PLOAD, lambda n: n * slices, {'loads': (0, 1, False), 'pempty': (1, 2, False),
                                                                'split_store': (2, 3, False)}, 0, 3)
    r['epilogue'] = shares(EPI, lambda n: n, {'loads': (0, 1, False), 'afull': (1, 2, False),
                                               'store': (2, 3, False)}, 0, 3)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--build-dir', default=None)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'the timeline needs a GPU'
    from b200ocl import _native
    build_dir = args.build_dir or tempfile.mkdtemp(prefix='b200ocl_tcp_trace_')
    _native.LIB_PATH = build_traced(build_dir)
    _native.SIGNATURES['b200ocl_tcp_trace_set'] = (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int])
    lib = _native.lib()
    name, smi = card()
    print('card: %s, power limit / max SM clock: %s' % (name, smi))
    rows = []
    for label, N, dgrad, mode in LAUNCHES:
        for C, H in LAYERS:
            r = run_shape(lib, C, H, N, dgrad, mode)
            r.update(launch='%s%s N=%d %dx%d C=%d' % (label, ' acc' if mode == 1 else '', N, H, H, C))
            rows.append(r)
            print('\n%-28s %3d CTAs x %3d taps  %6.1f us  %.2f GHz  per tap %.3f us (floor %.3f)  stages %d + %d' % (
                r['launch'], r['ctas'], r['taps_per_cta'], r['span_us'], r['sm_ghz'], r['per_tap_us'],
                r['floor_per_tap_us'], r['ps'], r['bs']))
            for role in ('consumer0', 'consumer1', 'weight_loader', 'patch_loaders', 'epilogue'):
                if role in r:
                    print('  %-14s %s' % (role, '  '.join('%s %4.1f%%' % (k, 100 * v) for k, v in r[role].items())))
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump({'card': name, 'nvidia_smi': smi, 'launches': rows}, fh, indent=1)


if __name__ == '__main__':
    main()
