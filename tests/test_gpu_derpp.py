"""GPU: DER++ (learners.DERPP, opt-in as agents['DERPP']).

  * b200ocl_logit_mse against fp64 at the shapes the agent feeds it (n in {1, 2, 10, 20, 110}, C in {10, 50, 69, 100},
    slot indices with repeats): every gradient element within a relative 1e-6, the loss within 1e-5, two calls
    bit-identical; its argument refusals and the flag for a slot outside the memory.
  * With der_alpha = 0 and der_beta = 1 a DER++ learner and an ER learner (random retrieval, reservoir update) built
    from the same seed and fed the same three tasks end bit for bit equal: parameters, BN statistics, memory and
    evaluate().
  * Whole DER++ and DER steps against oracle/derpp.py (fp64) at CIFAR-100, CORe50 and OpenLORIS shapes, with
    test_gpu_replay.py::test_er_random_steps's tolerances; after every update each written slot's logit row is the
    matching row of the last stream forward's logits, bit for bit.  Two-task CORe50 and OpenLORIS runs evaluate.
  * Adam's state in opt.state.
Checkpoint resume, staged snapshots, concurrent runs and graphs against eager launches are checked with the other
agents, as agent_cases.CASES['derpp'] (test_gpu_checkpoint.py, test_gpu_checkpoint_async.py, test_gpu_multirun.py,
test_gpu_graphs.py)."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from agent_cases import HW, NCLS, _learner, _load
from oracle import derpp as oder
from oracle import resnet as oresnet

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def b():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    import b200ocl
    from b200ocl import _native, engine, learners, memory, nets, registry, update
    return SimpleNamespace(native=_native, engine=engine, learners=learners, memory=memory, nets=nets,
                           registry=registry, update=update)


# ----------------------------------------------------------------------------- the kernel
@pytest.mark.parametrize('C', [10, 50, 69, 100])
@pytest.mark.parametrize('n', [1, 2, 10, 20, 110])
def test_logit_mse_against_fp64(b, n, C):
    rs = np.random.RandomState(n * 131 + C)
    mem_rows = 200
    z = (rs.standard_normal((n, C)) * 4).astype(np.float32)
    mem = (rs.standard_normal((mem_rows, C)) * 4).astype(np.float32)
    idx = rs.randint(0, mem_rows, n)
    if n > 1:
        idx[1::2] = idx[0]                                       # repeated slots
    mem[idx[0]] = z[0] + np.float32(1e-3) * rs.standard_normal(C).astype(np.float32)   # a row close to its target
    alpha = 0.37
    want_loss, want_dz = oder.logit_mse(z, mem[idx], alpha)
    zt, mt, it = torch.tensor(z).cuda(), torch.tensor(mem).cuda(), torch.tensor(idx).cuda()
    out = b.engine.logit_mse(zt, mt, it, alpha)
    again = b.engine.logit_mse(zt, mt, it, alpha)
    dz = out['dlogits'].cpu().numpy().astype(np.float64)
    assert np.all(np.abs(dz - want_dz) <= 1e-6 * np.abs(want_dz)), np.max(np.abs(dz - want_dz) / np.abs(want_dz))
    assert abs(float(out['loss']) - want_loss) <= 1e-5 * want_loss, (float(out['loss']), want_loss)
    assert torch.equal(out['loss'], again['loss']) and torch.equal(out['dlogits'], again['dlogits'])


def test_logit_mse_refusals_and_flag(b):
    lib = b.native.lib()
    z = torch.ones((4, 10), device='cuda')
    mem = torch.zeros((6, 10), device='cuda')
    idx = torch.tensor([0, 5, 6, -1], device='cuda')
    loss, dz = torch.empty(1, device='cuda'), torch.empty_like(z)
    s = torch.cuda.current_stream().cuda_stream
    args = [z.data_ptr(), mem.data_ptr(), 6, idx.data_ptr(), 4, 10, 1.0, loss.data_ptr(), dz.data_ptr(), None, s]
    for k in (0, 1, 3, 7, 8):
        bad = list(args)
        bad[k] = None
        assert lib.b200ocl_logit_mse(*bad) == 1, k                     # B200OCL_EINVAL
    for k in (2, 4, 5):
        for v in (0, -3):
            bad = list(args)
            bad[k] = v
            assert lib.b200ocl_logit_mse(*bad) == 1, (k, v)
    err = torch.zeros(1, dtype=torch.int32, device='cuda')
    out = b.engine.logit_mse(z, mem, idx, 2.0, err=err)
    assert int(err) == 1
    dz = out['dlogits'].cpu()
    assert torch.equal(dz[2:], torch.zeros(2, 10)) and torch.all(dz[:2] == 2.0 * 2 / 40)
    assert float(out['loss']) == 2.0 * 20 / 40                         # two rows of ten unit differences, over 40


# ----------------------------------------------------------------------------- the learner
def make_params(**kw):
    base = dict(data='cifar100', cuda=True, epoch=1, batch=10, verbose=False, mem_size=40, eps_mem_batch=10,
                mem_iters=1, update='random', retrieve='random', agent='DERPP', k=3, aser_type='asvm', n_smp_cls=1.5,
                num_tasks=5, buffer_tracker=False, optimizer='SGD', learning_rate=0.05, weight_decay=0, temp=0.07,
                head='mlp', subsample=20, error_analysis=False, der_alpha=0.3, der_beta=0.5,
                trick={'labels_trick': False, 'kd_trick': False, 'separated_softmax': False, 'review_trick': False,
                       'ncm_trick': False, 'kd_trick_star': False})
    base.update(kw)
    return SimpleNamespace(**base)


def _task(rs, n, labels, hw):
    x = rs.randint(0, 256, (n, hw, hw, 3)).astype(np.uint8)
    return x, rs.choice(np.asarray(list(labels)), n)


def _loaders(rs, hw, labels):
    out = []
    for labs in labels:
        x, y = _task(rs, 30, labs, hw)
        out.append([(torch.from_numpy(x).permute(0, 3, 1, 2).float().div(255), torch.from_numpy(y))])
    return out


def test_alpha_0_beta_1_is_er_bit_for_bit(b):
    results = []
    for agent_name in ('ER', 'DERPP'):
        params = make_params(agent=agent_name, der_alpha=0.0, der_beta=1.0, mem_size=50)
        agent, _ = _learner(params, 31)
        rs = np.random.RandomState(5)
        tasks = [_task(rs, 73, range(4 * t, 4 * t + 4), 32) for t in range(3)]
        loaders = _loaders(rs, 32, [range(4 * t, 4 * t + 4) for t in range(3)])
        accs = []
        for t, (x, y) in enumerate(tasks):
            np.random.seed(60 + t); torch.manual_seed(60 + t)
            agent.train_learner(x, y)
            accs.append(agent.evaluate(loaders))
        eng, buf = agent.engine, agent.buffer
        results.append([eng.state.params.cpu(), eng.state.bn_stats.cpu(), eng.state.bn_tracked.cpu(),
                        buf.buffer_img.cpu(), buf.buffer_label.cpu(), torch.tensor(buf.labels_host),
                        torch.tensor(np.array(accs)), torch.tensor([buf.current_index, buf.n_seen_so_far])])
    assert isinstance(agent.buffer, b.memory.LogitBuffer)
    for i, (er, der) in enumerate(zip(*results)):
        assert torch.equal(er, der), i
    assert results[0][-1].tolist() == [50, 210]


def _record_stream_logits(agent):
    """Wrap the engine's forward_train so that the learner's last stream forward (slot 0) is kept."""
    eng = agent.engine
    fwd = eng.forward_train
    seen = {}

    def wrapped(x, *a, **k):
        out = fwd(x, *a, **k)
        if k.get('slot', 0) == 0:
            seen['z'] = out[0].clone()
        return out
    eng.forward_train = wrapped
    return seen


def _written_rows(b, buf, s0, n, mem):
    """{slot: stream row} of the update that just ran (fill phase, then the reservoir's draws)."""
    fill = min(max(0, mem - s0), n)
    rows = {s0 + j: j for j in range(fill)}
    if fill < n:
        slots, src = b.update.reservoir_plan(buf.last_draws, mem)
        rows.update({s: fill + j for s, j in zip(slots, src)})
    return rows


def _steps_against_oracle(b, data, alpha, beta, n_steps, seed):
    params = make_params(data=data, der_alpha=alpha, der_beta=beta, mem_size=30)
    agent, spec = _learner(params, seed)
    hw, ncls = HW[data], NCLS[data]
    p64, bn64 = oresnet.seeded_state(spec, seed, dtype=torch.float64)
    st = oder.DerState(spec, p64, bn64, params.mem_size, (3, hw, hw), ncls, lr=params.learning_rate)
    seen = _record_stream_logits(agent)
    agent.model.train()
    rs = np.random.RandomState(seed + 1)
    n_logit = 0
    for i in range(n_steps):
        x = torch.tensor(rs.randint(0, 256, (10, 3, hw, hw)).astype(np.float32) / 255.0)
        y = torch.tensor(rs.randint(0, 5, 10))
        s0 = agent.buffer.current_index
        np.random.seed(100 + i); torch.manual_seed(100 + i)
        agent.replay_step(x.cuda(), y.cuda(), y.numpy())
        np.random.seed(100 + i); torch.manual_seed(100 + i)
        cpu = oder.derpp_step(st, x, y, alpha, beta)
        where = (data, alpha, beta, i)
        assert abs(float(agent.last_loss) - cpu[0]) < 2e-4 * abs(cpu[0]), (where, float(agent.last_loss), cpu)
        for got, want, w in ((agent.last_loss_logit, cpu[1], alpha), (agent.last_loss_mem, cpu[2], beta)):
            assert (got is None) == (want is None), where
            if want is not None:
                floor = 2e-4 * w * float(st.buffer_logits[:st.current_index].pow(2).mean())
                assert abs(float(got) - want) < 2e-4 * abs(want) + floor, (where, float(got), want)
        n_logit += agent.last_loss_logit is not None
        flat = torch.cat([v.reshape(-1) for v in st.params.values()])
        err = float((agent.engine.state.params.cpu().double() - flat).abs().max() / flat.abs().max())
        assert err < 2e-4, (where, err)
        np.testing.assert_array_equal(agent.buffer.buffer_label.cpu().numpy(), st.buffer_label.numpy())
        torch.testing.assert_close(agent.buffer.buffer_img.cpu(), st.buffer_img, rtol=0, atol=0)
        # each written slot holds the last stream forward's logits row, bit for bit
        rows = _written_rows(b, agent.buffer, s0, 10, params.mem_size)
        assert rows, where
        got = agent.buffer.buffer_logits.cpu()
        for s, j in rows.items():
            assert torch.equal(got[s], seen['z'][j].cpu()), (where, s, j)
        # the next step starts from the oracle's weights and statistics and from the engine's logit memory
        _load(agent, st.params, st.bn, spec)
        st.buffer_logits.copy_(got.double())
    assert agent.buffer.n_seen_so_far == st.n_seen_so_far == 10 * n_steps
    assert n_logit == (n_steps - 1 if alpha else 0)


@pytest.mark.parametrize('alpha,beta', [(0.3, 0.5), (0.5, 0.0)], ids=['derpp', 'der'])
def test_steps_against_oracle_cifar100(b, alpha, beta):
    _steps_against_oracle(b, 'cifar100', alpha, beta, 6, 201)


@pytest.mark.parametrize('data', ['core50', 'openloris'])
def test_steps_against_oracle_core50_openloris(b, data):
    _steps_against_oracle(b, data, 0.3, 0.5, 4, 202)


@pytest.mark.parametrize('data', ['core50', 'openloris'])
def test_two_task_run_evaluates(b, data):
    params = make_params(data=data, mem_size=40)
    agent, _ = _learner(params, 9)
    hw = HW[data]
    rs = np.random.RandomState(3)
    # CORe50: new classes per task; OpenLORIS: new instances of the same classes
    labels = [range(0, 5), range(5, 10)] if data == 'core50' else [range(0, 6), range(0, 6)]
    loaders = _loaders(rs, hw, labels)
    for t, labs in enumerate(labels):
        agent.train_learner(*_task(rs, 42, labs, hw))
        acc = agent.evaluate(loaders)
    torch.cuda.synchronize()
    assert acc.shape == (2,) and np.all((acc >= 0) & (acc <= 1))
    assert agent.buffer.current_index == 40 and agent.buffer.n_seen_so_far == 80
    assert torch.isfinite(agent.engine.state.params).all() and torch.isfinite(agent.buffer.buffer_logits).all()


def test_adam_state_is_the_engines(b):
    params = make_params(optimizer='Adam', learning_rate=1e-3)
    agent, _ = _learner(params, 11, opt=lambda m: torch.optim.Adam(m.parameters(), lr=1e-3))
    rs = np.random.RandomState(4)
    agent.train_learner(*_task(rs, 33, range(5), 32))
    opt, st = agent.opt, agent.engine.adam_state()
    stepped = [(q, o, k) for q, (o, k, hg) in zip(agent.model.parameters(), agent.engine.table) if hg]
    assert len(stepped) == len(opt.state) > 0
    for q, o, k in stepped:
        s = opt.state[q]
        assert set(s) == {'step', 'exp_avg', 'exp_avg_sq'} and float(s['step']) == 3 == st.step
        assert s['exp_avg'].data_ptr() == st.exp_avg[o:o + k].data_ptr()
        assert s['exp_avg_sq'].data_ptr() == st.exp_avg_sq[o:o + k].data_ptr()
    assert float(st.exp_avg_sq.abs().max()) > 0
