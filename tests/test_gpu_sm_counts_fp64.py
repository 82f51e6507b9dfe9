"""The fp64 pins at SM counts other than the card's: 114 (an H100 PCIe), 60 and 16 (H100 MIG 3g and 1g slices).

Nearly every launch geometry of the engine is a function of the SM count: the convolution plans and their statistics
partials, the halo-strip grid, the weight-gradient splits and chains per CTA, the BN backward's form and rows per CTA,
the SupCon and kNN-SV families, the 2 x SMs grids of agem_project and grad_cosine, the optimizer's norm partials, and
the train workspace sized from all of them.  The other GPU files pin those kernels against fp64 at the geometries of
the card they run on; B200OCL_SM_COUNT makes the library plan for fewer SMs than the device has, so one card can run
the geometries of the others.  It reads the variable once per process, so each count runs in a child process
(sm_counts_child.py) with the other files' references and tolerances, at batch sizes and lengths chosen from the plan
hooks at that count; its coverage tests prove they reach every geometry the four datasets' networks take there.

The override only goes down: the fused BN backward and the fused SupCon kernel wait on each other across a grid of at
most one CTA per SM, which need not be resident if it were planned for more SMs than the device has.  Values above the
device's count, zero, negative or not integers are refused before anything launches (the CPU test below).

Largest error per kind measured on an H100 80GB HBM3 (SXM, 132 SMs, 700 W power limit, 1980 MHz), emulating
114 / 60 / 16 SMs, with the bar of the file each check comes from in brackets (the child prints these as WORST lines):
  forward   z 1.1e-6 / 9.1e-7 / 9.4e-7 [2.6e-6], mean 2.1e-8 / 2.1e-8 / 2.3e-8 [6.6e-8], invstd 5.5e-8 / 5.8e-8 /
            5.5e-8 [1.8e-7], a 1.3e-7 / 1.4e-7 / 1.4e-7 [4.1e-7], feat 1.9e-7 / 1.8e-7 / 1.7e-7 [5.6e-7], head 2.6e-7 /
            2.6e-7 / 2.2e-7 [5.7e-7], run 2.3e-9 / 0 / 0 [2.4e-7], e2e 1.4e-6 / 1.7e-6 / 1.1e-6 [3.8e-6],
            eval 2.4e-6 / 2.3e-6 / 2.2e-6 [6.1e-6]
  backward  conv 1.2e-5 / 9.4e-6 / 8.8e-6 [3e-5], bn 1.4e-5 / 8.1e-6 / 8.6e-6 [4e-5], head 8.3e-7 / 7.2e-7 / 4.9e-7 [2e-6]
  strip     conv_tcp forward, data gradient, eval forms <= 6.6e-7 [5e-6]; wgrad_tc max 2.4e-6 [5e-6], rms 1.8e-6 [2e-6]:
            the same bits at every count (a strip tile's arithmetic does not depend on the grid)
  SupCon    loss 1.2e-8 at every count [4e-8]; gradient 1.4e-5 / 1.9e-5 / 1.6e-5 [5e-5] (ring64 / ring16 / ring16, NC = 4)
  kNN-SV    row 1.0e-7 / 7.6e-8 / 7.2e-8 [3e-7], column sums 4.6e-7 / 3.8e-7 / 4.0e-7 [1.5e-6]
  cosine    grad_cosine error 0.54 / 0.55 / 0.54 of its derived bound (K = 64)
A-GEM's projection, the optimizer steps and the whole ER, SCR and GDumb steps pass their files' checks at every count.
The whole file ran in 3 min 45 s there (pytest's count: 221 s, about 70 s per count)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = os.path.join(ROOT, 'tests', 'sm_counts_child.py')
COUNTS = (114, 60, 16)
TIMEOUT = 1200          # seconds per count; the child is killed, never retried, past it


def _refused(value, device_sms=132):
    from b200ocl import _native
    with pytest.raises(ValueError):
        _native.parse_sm_count(value, device_sms)


def test_sm_count_override_parsing_and_refusals():
    from b200ocl import _native
    assert _native.parse_sm_count(None, 132) is None
    assert _native.parse_sm_count('16', 132) == 16
    assert _native.parse_sm_count(' 114\n', 114) == 114
    assert _native.parse_sm_count('1', 16) == 1
    for bad in ('133', '999', '0', '-1', '-16', '', ' ', '16.0', '1e2', 'sixteen', '0x10', '16 SMs'):
        _refused(bad)
    _refused('115', 114)
    _refused('17', 16)


@pytest.mark.parametrize('value', ['999', '0', 'garbage'])
def test_library_refuses_a_bad_count_before_loading(value):
    """_native.lib() raises ValueError for the count, in a fresh process, before the library is loaded or anything
    launches (the check needs no GPU)."""
    code = ('from b200ocl import _native\n'
            'try:\n    _native.lib()\nexcept ValueError as e:\n    print("refused", e)\n'
            '    assert _native._lib is None\n    raise SystemExit(0)\n'
            'raise SystemExit(1)\n')
    env = dict(os.environ, B200OCL_SM_COUNT=value, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, '-c', code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and 'refused' in r.stdout, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])


@pytest.mark.gpu
@pytest.mark.parametrize('sms', COUNTS)
def test_fp64_pins_at_sm_count(sms):
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    have = torch.cuda.get_device_properties(0).multi_processor_count
    if sms > have:
        pytest.skip('the device has %d SMs; the override only goes down' % have)
    env = dict(os.environ, B200OCL_SM_COUNT=str(sms))
    cmd = [sys.executable, '-m', 'pytest', CHILD, '-q', '-s', '-p', 'no:cacheprovider']
    # subprocess.run kills the child when the timeout expires, so no child outlives this test
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=TIMEOUT)
    lines = r.stdout.splitlines()
    for line in lines:
        if line.startswith(('WORST', 'sms %d batches' % sms)):
            print(line)
    summary = [line for line in lines if ' passed' in line or ' failed' in line or ' error' in line]
    failed = [line for line in lines if line.startswith(('FAILED', 'ERROR'))]
    assert r.returncode == 0, (sms, summary[-1:], failed[:20], '\n'.join(lines[-60:]), r.stderr[-3000:])
    assert 'skipped' not in (summary[-1] if summary else ''), summary
