"""GPU: snapshots written behind the run (B200OCL_CHECKPOINT_ASYNC=1).

  * The encoder of b200ocl_snapshot_pack over all 2^32 fp32 bit patterns: exactly the 256 values u / 255 are stored at
    8 bits, and every pattern, 8-bit or fp32, comes back bit for bit through b200ocl_snapshot_unpack.
  * For each agent configuration of test_gpu_checkpoint.py (RESUME_CASES: ER with random, ASER, MIR and GSS, SCR,
    A-GEM, LwF with kd_trick, ER with the review trick and separated softmax, iCaRL, GDumb, EWC++, ER with Adam, DER++,
    PCR and GEM), the staged snapshot of every task boundary, read back from its file, equals agent.snapshot() at
    that boundary array for array, bit for bit, although the write is held until the next task has taken a step.
  * Interrupted experiments resumed with the switch on end with the uninterrupted results bit for bit (test_gpu_checkpoint
    .py's tests run with the switch on), at R = 1 and 3, on workers 0,0 and in main_tune.py's tuning stage.
  * Rows that are not 8-bit values (float64-sourced, as in the non-stationary streams) keep fp32; CORe50-shaped 8-bit
    rows are stored at one byte per value; both restore bit for bit through the device decode."""
import os
import threading

import numpy as np
import pytest
import torch

from b200ocl import checkpoint, memory, multirun, ops

import test_gpu_checkpoint as gc
from test_gpu_checkpoint import stub_tree  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    return torch.device('cuda', torch.cuda.current_device())


def _table(rows):
    t = np.zeros(len(rows), ops.SNAP_SEGMENT)
    for k, r in enumerate(rows):
        t[k] = tuple(r) + (0,)
    return torch.from_numpy(t.view(np.uint8)).to('cuda')


def _units():
    """The 256 fp32 values u / 255 (numpy's float32 division is the IEEE one), as int32 bit patterns."""
    return (np.arange(256, dtype=np.float32) / np.float32(255)).view(np.int32)


def test_the_256_units_are_stored_at_8_bits_and_a_foreign_value_falls_back():
    dev = _cuda()
    vals = torch.from_numpy(_units().view(np.float32).copy()).to(dev)
    rows = torch.cat([vals, vals.flip(0)]).reshape(2, 256)
    staging = torch.empty(1 << 12, dtype=torch.uint8, device=dev)
    ws = ops.snapshot_workspace(1, dev)
    for foreign in (None, 0.3, -0.0, float('nan')):
        src = rows.clone()
        if foreign is not None:
            src[1, 17] = foreign
        ops.snapshot_pack(_table([(src.data_ptr(), src.numel() * 4, 0, ops.SNAP_U8)]), 1, staging, ws)
        counters = ws[:8].view(torch.int32).cpu().tolist()
        assert counters == [0 if foreign is None else 1, 0], (foreign, counters)
        out = torch.full_like(src, 7.0)
        kind = ops.SNAP_U8 if foreign is None else ops.SNAP_COPY
        ops.snapshot_unpack(_table([(out.data_ptr(), src.numel() * 4, 0, kind)]), 1, staging, ws)
        assert torch.equal(out.view(torch.int32), src.view(torch.int32)), foreign
        if foreign is None:
            assert torch.equal(staging[:512].cpu(), torch.cat([torch.arange(256), torch.arange(255, -1, -1)]).byte())


def test_the_encoder_accepts_exactly_the_256_units_over_all_fp32_patterns():
    """2^32 patterns in 16 chunks of 2^28, 2^16 segments of 2^12 values each: a segment's counter is its number of
    rejected values, so the accepted ones per segment must be the units in it; together with the test above (every unit
    is accepted) the accepted set is the 256 units.  Every chunk is also unpacked (8-bit or fp32 by its counters) and
    compared with its input bit for bit."""
    dev = _cuda()
    CHUNK, SEG = 1 << 28, 1 << 12
    nseg = CHUNK // SEG
    units = _units().astype(np.int64) & 0xffffffff
    staging = torch.empty(CHUNK * 4, dtype=torch.uint8, device=dev)
    ws = ops.snapshot_workspace(nseg, dev)
    out = torch.empty(CHUNK, dtype=torch.int32, device=dev)
    offs = np.arange(nseg, dtype=np.uint64) * np.uint64(SEG * 4)
    accepted = 0
    for c in range((1 << 32) // CHUNK):
        base = c * CHUNK
        bits = torch.arange(base, base + CHUNK, dtype=torch.int64, device=dev)
        bits = torch.where(bits >= 1 << 31, bits - (1 << 32), bits).to(torch.int32)
        src = bits.view(torch.float32)
        t = np.zeros(nseg, ops.SNAP_SEGMENT)
        t['ptr'] = np.uint64(src.data_ptr()) + offs
        t['bytes'], t['offset'], t['kind'] = SEG * 4, offs, ops.SNAP_U8
        ops.snapshot_pack(torch.from_numpy(t.view(np.uint8)).to(dev), nseg, staging, ws)
        counters = ws[:4 * (nseg + 1)].view(torch.int32).cpu().numpy()
        assert counters[nseg] == 0
        mine = units[(units >= base) & (units < base + CHUNK)]
        want = np.bincount(((mine - base) // SEG).astype(np.int64), minlength=nseg)
        assert np.array_equal(SEG - counters[:nseg], want), c
        accepted += int((SEG - counters[:nseg]).sum())
        t['ptr'] = np.uint64(out.data_ptr()) + offs
        t['kind'] = np.where(counters[:nseg] == 0, ops.SNAP_U8, ops.SNAP_COPY)
        ops.snapshot_unpack(torch.from_numpy(t.view(np.uint8)).to(dev), nseg, staging, ws)
        assert torch.equal(out, bits), c
    assert accepted == 256


def _switch_on(tree, monkeypatch):
    """The switch with the directory the experiments are given (install() refuses it without one)."""
    monkeypatch.setenv(checkpoint.ENV, str(tree / 'ck'))
    monkeypatch.setenv(checkpoint.ASYNC_ENV, '1')


def _same_tree(got, want, where):
    if isinstance(want, dict):
        assert isinstance(got, dict) and list(got) == list(want), where
        for k in want:
            _same_tree(got[k], want[k], where + (k,))
    elif isinstance(want, (list, tuple)):                  # GEM's rings: one label array per task
        assert type(got) is type(want) and len(got) == len(want), where
        for k, (g, w) in enumerate(zip(got, want)):
            _same_tree(g, w, where + (k,))
    elif isinstance(want, torch.Tensor):
        assert got.dtype == want.dtype and got.shape == want.shape, where
        assert torch.equal(got.cpu().view(torch.uint8), want.cpu().view(torch.uint8)), where
    elif isinstance(want, np.ndarray):
        assert np.array_equal(got, want) and got.dtype == want.dtype, where
    else:
        assert got == want, where


@pytest.mark.parametrize('case', sorted(gc.RESUME_CASES))
def test_a_staged_snapshot_equals_the_agent_snapshot_at_its_boundary(case, stub_tree, monkeypatch, capsys):  # noqa: F811
    _switch_on(stub_tree, monkeypatch)
    stepped = threading.Event()
    want, got = {}, {}
    stage, next_step, write = multirun._Run.stage, multirun._next_step, checkpoint._Job.write

    def staging(run, task):
        out = stage(run, task)
        want[run.index, task] = run.snapshot(task)
        stepped.clear()
        return out

    def step(steps):
        stepped.set()
        return next_step(steps)

    def held(job):
        assert stepped.wait(60), 'no step after the boundary'          # the next task is training
        write(job)
        i = int(os.path.basename(job.path)[3:-len('.snapshot')])
        snap = checkpoint.Checkpoint(os.path.dirname(os.path.dirname(job.path)), 'runs').snapshot(i)
        got[i, snap['task']] = snap
    monkeypatch.setattr(multirun._Run, 'stage', staging)
    monkeypatch.setattr(multirun, '_next_step', step)
    monkeypatch.setattr(checkpoint._Job, 'write', held)
    uninstall = gc._install(case)
    try:
        gc._experiment(case, 1, 'staged', str(stub_tree / 'ck'), monkeypatch, capsys)
    finally:
        uninstall()
    assert sorted(got) == sorted(want) == [(r, t) for r in range(gc.N_RUNS) for t in range(2)]
    for key in want:
        assert got[key]['task'] == want[key]['task']
        assert all(np.array_equal(a, b) for a, b in zip(got[key]['acc'], want[key]['acc']))
        _same_tree(got[key]['agent'], want[key]['agent'], (case,) + key)


@pytest.mark.parametrize('R', [1, 3])
@pytest.mark.parametrize('case', sorted(gc.RESUME_CASES))
def test_a_resumed_experiment_with_staged_snapshots_matches_an_uninterrupted_one(case, R, stub_tree, monkeypatch,  # noqa: F811
                                                                                capsys):
    _switch_on(stub_tree, monkeypatch)
    before = checkpoint.stats['snapshots']
    gc.test_a_resumed_experiment_matches_an_uninterrupted_one(case, R, 'step', stub_tree, monkeypatch, capsys)
    assert checkpoint.stats['snapshots'] > before


def test_runs_on_two_workers_resume_with_staged_snapshots(stub_tree, monkeypatch, capsys):  # noqa: F811
    _switch_on(stub_tree, monkeypatch)
    gc.test_runs_on_two_workers_resume_like_runs_in_process(stub_tree, monkeypatch, capsys)


def test_tuning_resumed_with_staged_snapshots_chooses_the_same_points(stub_tree, monkeypatch, capsys):  # noqa: F811
    _switch_on(stub_tree, monkeypatch)
    before = checkpoint.stats['snapshots']
    gc.test_tuning_resumed_in_its_tuning_stage_chooses_the_same_points(stub_tree, monkeypatch, capsys)
    assert checkpoint.stats['snapshots'] > before


@pytest.mark.parametrize('shape', ['nonstationary_f64', 'core50_u8'])
def test_memory_rows_keep_their_bits_through_a_staged_file(shape, tmp_path):
    dev = _cuda()
    rs = np.random.RandomState(3)
    if shape == 'nonstationary_f64':                 # float64 images in [0, 1] converted as the stream converts them
        src = torch.from_numpy(rs.rand(200, 32, 32, 3)).to(dev)
    else:                                            # 8-bit CORe50 frames
        src = torch.from_numpy(rs.randint(0, 256, (300, 128, 128, 3)).astype(np.uint8)).to(dev)
    rows = ops.stream_prepare(src)
    labels = torch.from_numpy(rs.randint(0, 50, rows.shape[0])).to(dev)
    parts = {'engine': {'params': torch.randn(1000, device=dev)}, 'buffer': {'images': memory.Rows8(rows),
                                                                             'labels': labels, 'current_index': 7}}
    want = memory.host_tree(parts)
    nbytes = rows.numel() * 4 + labels.numel() * 8 + 4000
    staging = checkpoint.Staging(nbytes, dev)
    ck = checkpoint.Checkpoint(str(tmp_path), 'runs', async_write=True)
    tree, job = staging.stage(parts)
    ck.save_staged(0, {'task': 0, 'acc': [], 'rng': None, 'sampler': None, 'agent': tree}, job)
    checkpoint.writer().drain()
    size = os.path.getsize(ck._path(0, 'snapshot'))
    u8 = shape == 'core50_u8'
    assert size < rows.numel() * (1 if u8 else 4) + labels.numel() * 8 + 4000 + 4096
    assert size >= rows.numel() * (1 if u8 else 4)
    for where in (None, staging):                   # host decode, and the device decode a restore uses
        got = ck.snapshot(0, where)['agent']
        _same_tree(got, want, (shape, where is None))
