"""The fp64 pins of the other GPU files, run in one process whose launches are planned for B200OCL_SM_COUNT SMs.

test_gpu_sm_counts_fp64.py runs this module in a child process per SM count (its file name keeps it out of the normal
collection; without the variable it skips).  Every tolerance and reference is the one of the file a check comes from;
what changes is the geometry: batch sizes and lengths are chosen here from the plan hooks at this count, and the
coverage tests prove they reach every geometry the planner gives the four datasets' networks at this count."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

if not os.environ.get('B200OCL_SM_COUNT'):
    pytest.skip('runs only as the child of test_gpu_sm_counts_fp64.py', allow_module_level=True)

import test_gpu_agem_fp64 as agem  # noqa: E402
import test_gpu_backward_fp64 as bwd  # noqa: E402
import test_gpu_conv_maps_fp64 as cm  # noqa: E402
import test_gpu_ewc as ewc  # noqa: E402
import test_gpu_forward_fp64 as fwd  # noqa: E402
import test_gpu_gdumb as gdumb  # noqa: E402
import test_gpu_gss_maps_fp64 as gss  # noqa: E402
import test_gpu_knn_sv_fp64 as knn  # noqa: E402
import test_gpu_replay as replay  # noqa: E402
import test_gpu_supcon_fp64 as sup  # noqa: E402

pytestmark = pytest.mark.gpu

SMS = int(os.environ['B200OCL_SM_COUNT'])
MAPS = (32, 50, 84, 128)                 # CIFAR-100, OpenLORIS, Mini-ImageNet, CORe50 inputs
# the batch sizes searched per map: the agents' batches there (SCR's 220 and ASER's eval passes on the small maps,
# GDumb's and CORe50's up to 110) with room above
N_MAX = {32: 512, 50: 256, 84: 256, 128: 128}


# ------------------------------------------------------------------------------------------------- plan features
def _rounds(tiles, grid_x):
    return min(3, -(-tiles // grid_x))


def _strip_tiles(N, H):
    return cm.strip_tiles(N, H)[0]


def _net(hw):
    from b200ocl import engine
    desc, info, _ = engine.describe(hw, 100)
    return desc, [engine.train_ws_layout(desc, 1, i) for i in range(info.n_bn)]


def fwd_features(hw, N):
    """What the train and eval forwards at N launch: (pass, template) per layer, and how many strip tiles the
    halo-strip CTAs walk."""
    from b200ocl import engine
    desc, L = _net(hw)
    out = set()
    for i, l in enumerate(L):
        for pass_ in ('train', 'eval'):
            g = engine.conv_geom(desc, N, i, pass_)
            assert g.sms == SMS
            out.add((pass_, g.template))
            if g.name == 'tcp':
                out.add(('walk', pass_, _rounds(_strip_tiles(N, l.hout), g.grid_x)))
    return out


def bwd_features(hw, N):
    """What the backward at N launches: data-gradient templates and strip walks, per width the BN backward's form
    (fused or two-phase) and whether a fused grid covers more than half the SMs, the weight-gradient kernels and how
    many chains each wgmma weight-gradient CTA walks (1, 2, 3+)."""
    from b200ocl import engine
    desc, L = _net(hw)
    out = set()
    for i, l in enumerate(L):
        if i:
            g = engine.conv_geom(desc, N, i, 'dgrad')
            out.add(('dgrad', g.template))
            if g.name == 'tcp':
                out.add(('walk', 'dgrad', _rounds(_strip_tiles(N, l.hout), g.grid_x)))
        w = engine.train_ws_layout(desc, N, i)
        assert w.sms == SMS
        out.add(('bn', w.cout, bool(w.bn_fused)))
        if w.bn_fused and 2 * w.bn_grid > SMS:
            out.add(('bn_wide',))
        out.add(('wgrad', w.wgrad_kernel))
        if w.wgrad_kernel == 1:
            t = engine.wgrad_tc_selftest_geom(N, l.hout, l.wout, l.cin, l.cout)
            assert t.eligible and t.sms == SMS
            out.add(('chains', min(3, t.chains_per_cta)))
    return out


def cover(features, candidates):
    """Greedy set cover: the fewest batches (smallest first on ties) whose features together are every candidate's.
    Returns (batches, the union over every candidate)."""
    feats = {N: features(N) for N in candidates}
    every = set().union(*feats.values())
    left, chosen = set(every), []
    while left:
        N = max(candidates, key=lambda n: (len(feats[n] & left), -n))
        chosen.append(N)
        left -= feats[N]
    return sorted(chosen), every


_PLANS = {}


def plans():
    """{map: (forward batches, backward batches)} at this SM count, cached per process."""
    if not _PLANS:
        for hw in MAPS:
            cand = range(1, N_MAX[hw] + 1)
            _PLANS[hw] = (cover(lambda N: fwd_features(hw, N), cand)[0], cover(lambda N: bwd_features(hw, N), cand)[0])
    return _PLANS


def fwd_cases():
    out = []
    for hw in MAPS:
        f, _ = plans()[hw]
        out += [(hw, None, N) for N in f] + [(hw, 'mlp', max(f))]
    return out


def bwd_cases():
    out = []
    for hw in MAPS:
        _, b = plans()[hw]
        out += [(hw, None, N) for N in b] + [(hw, 'mlp', max(b))]
    return out


# halo-strip pairs: cm.batches plus, where those miss one at this count, the smallest batch that reaches each of the
# pair's launches (template, patch stages, weight ring depth), strip walks of 1, 2 and 3+ tiles, a last tile inside and
# past the last image, and weight-gradient grids with one chain per CTA, an even rounding and CTAs cut by the SM count
def strip_features(C, H, N):
    from b200ocl import engine
    out = set()
    for pass_, dgrad, mode in (('eval', 0, 3), ('dgrad', 1, 0)):
        g = engine.conv_selftest_geom(N, H, H, C, C, 3, 1, dgrad, cm.PATHS['tcp'], mode)
        assert g.sms == SMS
        tiles, past = cm.strip_tiles(N, H)
        out |= {(pass_, g.template, g.tp_ps, g.tp_bs), (pass_, 'walk', _rounds(tiles, g.grid_x)), (pass_, 'past', past > 0)}
    t = engine.wgrad_tc_selftest_geom(N, H, H, C, C)
    out |= {('wgrad', k) for k in cm.wgrad_classes(t)}
    return out


def strip_batches(C, H):
    base = cm.batches(C, H)
    have = set().union(*[strip_features(C, H, N) for N in base])
    extra = []
    for N in range(1, cm.MAX_N + 1):
        new = strip_features(C, H, N) - have
        if new:
            extra.append(N)
            have |= new
    return sorted(set(base) | set(extra))


def strip_cases():
    return [(C, H, N) for C, H in cm.TABLE for N in strip_batches(C, H)]


# SupCon: the SupCon file's cases at this count, plus both sides of A = 16 * SMS (ring16 / ring64 at 64 and 128 wide)
_SUP_CASES = sup.case_list


def supcon_cases(sms):
    return _SUP_CASES(sms) + [('edge16-at', 16 * sms, 1, 128, 0.05, 'few', 3.0, False),
                                 ('edge16-past', 16 * sms + 1, 1, 128, 0.05, 'few', 3.0, False),
                                 ('edge16-at-v2', 8 * sms, 2, 64, 0.07, 'pairs', 1.0, False),
                                 ('edge16-past-v2', 8 * sms + 1, 2, 64, 0.07, 'pairs', 1.0, False)]


def grid():
    """The grid of agem_project and grad_cosine at this count."""
    return min(2 * SMS, 296)


def cosine_lengths():
    G = grid() * 256
    return [1, 255, 257, G - 1, G, G + 1, 2 * G + 1] + sorted(gss.ARENA.values())


# ------------------------------------------------------------------------------------------------------ fixtures
@pytest.fixture(scope='module')
def engine():
    from b200ocl import engine as _engine
    return _engine


@pytest.fixture(scope='module')
def ops():
    from b200ocl import ops as _ops
    return _ops


@pytest.fixture(scope='module')
def b():
    from types import SimpleNamespace
    from b200ocl import _native, engine, learners, memory, nets, ops, registry, retrieve, update
    return SimpleNamespace(native=_native, engine=engine, learners=learners, memory=memory, nets=nets, ops=ops,
                           registry=registry, retrieve=retrieve, update=update)


# ----------------------------------------------------------------------------------------------- the count itself
def test_emulated_count_is_in_force(engine, ops):
    from b200ocl import _native
    assert torch.cuda.is_available()
    assert _native.lib().b200ocl_sm_count() == SMS
    assert SMS <= torch.cuda.get_device_properties(0).multi_processor_count
    desc, _ = _net(32)
    assert engine.conv_geom(desc, 10, 1, 'train').sms == SMS
    assert engine.train_ws_layout(desc, 10, 1).sms == SMS
    assert engine.wgrad_tc_selftest_geom(10, 32, 32, 20, 20).sms == SMS
    assert ops.supcon_plan(110, 2, 128, True, 0).sms == SMS
    assert ops.knn_sv_plan(110, 160, 160, True, True, 0).sms == SMS


# --------------------------------------------------------------------------------------- 1. forward and backward
def test_cases_reach_every_network_geometry():
    """The chosen batches reach every forward and backward geometry the four maps' networks take at this count for
    N <= N_MAX, including both BN-backward forms, a fused grid over half the SMs, all three weight-gradient kernels,
    wgmma weight-gradient CTAs walking 3+ chains and halo-strip CTAs walking 1, 2 and 3+ tiles."""
    everything = set()
    for hw in MAPS:
        cand = range(1, N_MAX[hw] + 1)
        f, b = plans()[hw]
        for features, chosen in ((fwd_features, f), (bwd_features, b)):
            every = cover(lambda N: features(hw, N), cand)[1]
            reached = set().union(*[features(hw, N) for N in chosen])
            assert reached == every, (hw, sorted(every - reached, key=str))
            everything |= {(hw,) + k for k in every}
    print('\nsms %d batches %s' % (SMS, plans()))
    kinds = {k[1:] for k in everything}
    assert {('wgrad', 0), ('wgrad', 1), ('wgrad', 2)} <= kinds
    assert ('chains', 3) in kinds and ('bn_wide',) in kinds
    assert {True, False} <= {k[2] for k in kinds if k[0] == 'bn'}
    for pass_ in ('eval', 'dgrad'):
        assert {('walk', pass_, r) for r in (1, 2, 3)} <= kinds, pass_


def net_id(c):
    return '%d-%s-N%d' % tuple(c)


@pytest.mark.parametrize('case', fwd_cases(), ids=net_id)
def test_forward_matches_fp64(engine, case):
    hw, head, N = case
    rows = fwd.run_case(engine, hw, head, N)
    _record('fwd', rows, lambda r: (r[0], r[2]))
    fwd.check(rows, N)


@pytest.mark.parametrize('case', bwd_cases(), ids=net_id)
def test_backward_matches_fp64(engine, case):
    hw, head, N = case
    _, _, rows = bwd.run_case(engine, hw, head, N)
    _record('bwd', rows, lambda r: (r[1], r[2]))
    bwd.check(rows, N)


@pytest.mark.parametrize('hw', MAPS)
def test_network_repeat_is_bit_identical(engine, hw):
    """Forward and backward at the map's largest backward batch, twice: the same bits (and the backward file's
    accumulate, second-arena and graph-replay properties)."""
    N = max(plans()[hw][1])
    bwd.test_backward_bit_properties(engine, hw, None, N)


# ------------------------------------------------------------------------------- 2. halo strip and wgmma wgrad
def test_strip_cases_reach_every_strip_launch(engine):
    """The strip cases reach every launch the networks give conv_tcp and wgrad_tc at this count (cm's coverage tests
    with this count's batches), and each case's launch is the network's."""
    every = set()
    for hw in cm.DATASETS.values():
        desc, info, _ = engine.describe(hw, 100)
        for i in range(1, info.n_bn):
            L = engine.train_ws_layout(desc, 1, i)
            for pass_ in ('eval', 'dgrad'):
                for N in range(1, cm.MAX_N + 1):
                    g = engine.conv_geom(desc, N, i, pass_)
                    if g.name == 'tcp':
                        every.add(((L.cout, L.hout), pass_, g.template, g.tp_ps, g.tp_bs))
    reached, per_pair = set(), {}
    for C, H, N in strip_cases():
        desc, i = cm.network_layer(engine, C, H)
        for pass_, dgrad, mode in (('eval', 0, 3), ('dgrad', 1, 0)):
            g = engine.conv_selftest_geom(N, H, H, C, C, 3, 1, dgrad, cm.PATHS['tcp'], mode)
            net = engine.conv_geom(desc, N, i, pass_)
            assert (g.template, g.grid_x, g.grid_y, g.tp_ps, g.tp_bs) == \
                (net.template, net.grid_x, net.grid_y, net.tp_ps, net.tp_bs), (C, H, N, pass_)
            reached.add(((C, H), pass_, g.template, g.tp_ps, g.tp_bs))
        assert engine.train_ws_layout(desc, N, i).wgrad_kernel == 1
        per_pair.setdefault((C, H), set()).update(strip_features(C, H, N))
    assert reached == every, sorted(every ^ reached)
    # per pair, every class some batch up to MAX_N takes at this count (a few are out of reach: at 16 SMs no batch
    # leaves (80, 32)'s CTAs one tile each); over all pairs, every class
    for (C, H), feats in per_pair.items():
        possible = set().union(*[strip_features(C, H, N) for N in range(1, cm.MAX_N + 1)])
        assert feats == possible, ((C, H), sorted(possible - feats, key=str))
    kinds = set().union(*per_pair.values())
    for pass_ in ('eval', 'dgrad'):
        assert {(pass_, 'walk', r) for r in (1, 2, 3)} <= kinds, pass_
        assert {(pass_, 'past', False), (pass_, 'past', True)} <= kinds, pass_
    assert {('wgrad', 'one'), ('wgrad', 'even'), ('wgrad', 'cut')} <= kinds


@pytest.mark.parametrize('case', strip_cases(), ids=cm.case_id)
def test_conv_tcp_and_wgrad_tc_match_fp64(engine, case, capsys):
    cm.test_conv_tcp_matches_fp64(engine, case)
    cm.test_wgrad_tc_matches_fp64(engine, case)
    for line in capsys.readouterr().out.splitlines():
        w = line.split()
        if w[:1] == ['MAXERR']:
            _WORST_PUT('strip_' + w[1], float(w[3]), w[2])
            if w[1] == 'wgrad':
                _WORST_PUT('strip_wgrad_rms', float(w[5]), w[2])


# ---------------------------------------------------------------------------------------------- 3. SupCon
def test_supcon_cases_reach_every_launch(ops):
    want = sup.reachable(ops, SMS)
    got = {ops.supcon_plan(c[1], c[2], c[3], not c[7], SMS).kernel for c in supcon_cases(SMS)}
    assert want <= got, sorted(want - got)
    fam = [ops.supcon_plan(c[1], c[2], c[3], True, SMS).name for c in supcon_cases(SMS) if c[0].startswith('edge16')]
    assert fam[0] != fam[1] and fam[2] != fam[3], fam            # A = 16 SMS and 16 SMS + 1 take different families


@pytest.mark.parametrize('idx', range(len(supcon_cases(SMS))))
def test_supcon_matches_fp64(ops, idx, monkeypatch, capsys):
    monkeypatch.setattr(sup, 'device_sms', lambda: SMS)
    monkeypatch.setattr(sup, 'case_list', supcon_cases)
    try:
        sup.test_supcon_against_fp64(ops, idx)
    finally:
        _parse(capsys, r'supcon (\S+) .* loss (\S+) grad (\S+) \|', ('supcon_loss', 'supcon_grad'))


# ----------------------------------------------------------------------------------------------- 4. kNN-SV
def test_knn_sv_cases_reach_every_launch(ops, monkeypatch):
    monkeypatch.setattr(knn, 'device_sms', lambda: SMS)
    knn.test_cases_reach_every_launch(ops)


@pytest.mark.parametrize('idx', range(len(knn.case_list(SMS))))
def test_knn_sv_matches_fp64(ops, idx, monkeypatch, capsys):
    monkeypatch.setattr(knn, 'device_sms', lambda: SMS)
    try:
        knn.test_knn_sv_against_fp64(ops, idx)
    finally:
        _parse(capsys, r'knn (\S+) .* row err (\S+) .* sum err (\S+)', ('knn_row', 'knn_sum'))


# ------------------------------------------------------------------------------- 5. A-GEM projection, GSS cosine
def test_agem_edge_lengths_reach_the_launch_edges(b, monkeypatch):
    monkeypatch.setattr(agem, 'grid_of', grid)
    agem.test_edge_lengths_reach_the_launch_edges(b)


def test_agem_projection_at_edge_lengths(b, monkeypatch):
    monkeypatch.setattr(agem, 'grid_of', grid)
    agem.test_projection_at_edge_lengths(b)


@pytest.mark.parametrize('data', list(agem.NETS))
def test_agem_projection_at_arena_lengths(b, data, monkeypatch):
    monkeypatch.setattr(agem, 'grid_of', grid)
    agem.test_projection_at_arena_lengths(b, data)


@pytest.mark.parametrize('K', (1, 7, 64))
def test_grad_cosine_matches_fp64(ops, K):
    """b200ocl_grad_cosine at lengths around the grid stride (2 SMS CTAs of 256) and the four arena lengths, with rows
    of mixed signs and scales, within gss.cos_bound of fp64, no row excused; repeat launches give the same bits."""
    worst = 0.0
    for n in cosine_lengths():
        gen = torch.Generator(device='cuda').manual_seed(17 * n + K)
        g = torch.randn(n, device='cuda', generator=gen)
        mem = torch.randn(K, n, device='cuda', generator=gen) * 10 ** torch.linspace(-3, 2, K, device='cuda')[:, None]
        mem[::2] += 0.3 * g                                   # positive and negative cosines both
        mem[1::3] -= 0.5 * g
        m64, g64 = mem.double(), g.double()
        ref = (m64 @ g64) / (m64.norm(dim=1) * g64.norm()).clamp(min=1e-8)
        cos, mx = ops.grad_cosine(mem, g)
        cos2, mx2 = ops.grad_cosine(mem, g)
        assert torch.equal(cos.view(torch.int32), cos2.view(torch.int32)) and torch.equal(mx, mx2), n
        assert torch.equal(mx, cos.max().reshape(1)), n
        err, bound = (cos.double() - ref).abs(), gss.cos_bound(ref, n)
        bad = (~(err <= bound)).nonzero().flatten().tolist()
        assert not bad, (n, [(i, float(cos[i]), float(ref[i]), float(bound[i])) for i in bad[:4]])
        worst = max(worst, float((err / bound).max()))
    _WORST_PUT('cosine_of_bound', worst, 'K=%d' % K)


# ------------------------------------------------------------------------------------- 6. optimizer reductions
@pytest.mark.parametrize('head', [None, 'mlp'])
@pytest.mark.parametrize('max_norm', [0.05, 1.0])
def test_gdumb_clipped_step(head, max_norm):
    gdumb.test_clipped_step_matches_clip_grad_norm_and_sgd(head, max_norm)


def test_gdumb_clipped_step_repeats():
    gdumb.test_clipped_step_repeat_launches_are_bit_identical()


@pytest.mark.parametrize('name', sorted(ewc.CASES))
def test_ewc_step(name):
    ewc.test_fused_step_matches_torch(name)


@pytest.mark.parametrize('head', [None, 'mlp'])
@pytest.mark.parametrize('zero', [False, True])
def test_ewc_consolidate(head, zero):
    ewc.test_consolidate_matches_torch(head, zero)


def test_ewc_repeats():
    ewc.test_repeat_launches_are_bit_identical()


# -------------------------------------------------------------------------------------- 8. whole steps, oracle
def test_er_steps(b):
    replay.test_er_random_steps(b)


def test_scr_steps(b):
    replay.test_scr_steps(b)


def test_gdumb_train_mem_steps():
    gdumb.test_train_mem_steps_match_the_oracle()


# --------------------------------------------------------------------------------------------- the worst errors
_WORST = {}


def _WORST_PUT(kind, err, where):
    if err == err and err > _WORST.get(kind, (-1.0, ''))[0]:
        _WORST[kind] = (err, where)


def _parse(capsys, pattern, kinds):
    import re
    out = capsys.readouterr().out
    sys.stdout.write(out)
    for m in re.finditer(pattern, out):
        for k, v in zip(kinds, m.groups()[1:]):
            _WORST_PUT(k, float(v), m.group(1))


def _record(pass_, rows, key):
    for r in rows:
        k, err = key(r)
        _WORST_PUT('%s_%s' % (pass_, k), err, r[1] if pass_ == 'fwd' else r[0])


def test_zz_report_worst_errors():
    """Runs last (pytest keeps file order): one line per kind, for the parent to print."""
    print()
    for k, (e, where) in sorted(_WORST.items()):
        print('WORST sms=%d %s %.2e (%s)' % (SMS, k, e, where))
