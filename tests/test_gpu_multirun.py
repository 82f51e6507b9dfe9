"""GPU: runs trained side by side (multirun.run_group, R = 3, three groups) give every run, bit for bit, what it gives
alone (R = 1, the same (seed, r)): accuracy arrays, final parameter arena, BN statistics and buffer contents, for ER
(random, ASER, MIR, Adam), SCR with the review trick, A-GEM, LwF, iCaRL, GDumb and EWC++.  A solo run through the driver
also matches a direct train_learner / evaluate loop from the same random state, so the step generators kept the
learners' behaviour.  Built with nets.setup_architecture on seeded synthetic uint8 tasks."""
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N_RUNS, R, SEED = 9, 3, 11
N_TASKS, PER_TASK, N_TEST = 3, 30, 40

CASES = {
    'er_random': dict(),
    'er_aser': dict(update='ASER', retrieve='ASER'),
    'er_mir': dict(retrieve='MIR'),
    'scr': dict(agent='SCR', trick_on=('review_trick',)),
    'agem': dict(agent='AGEM'),
    'lwf': dict(agent='LWF'),
    'icarl': dict(agent='ICARL', mem_size=100),
    'gdumb': dict(agent='GDUMB'),
    'ewc': dict(agent='EWC'),
    'er_adam': dict(optimizer='Adam', learning_rate=1e-3),
}


def _params(case):
    over = dict(CASES[case])
    trick = {k: k in over.pop('trick_on', ()) for k in ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick',
                                                         'ncm_trick', 'kd_trick_star')}
    base = dict(data='cifar10', cuda=True, epoch=1, batch=10, verbose=False, mem_size=20, eps_mem_batch=10,
                mem_iters=1, update='random', retrieve='random', agent='ER', k=3, aser_type='asvm', n_smp_cls=1.5,
                num_tasks=N_TASKS, buffer_tracker=False, optimizer='SGD', learning_rate=0.1, weight_decay=0,
                temp=0.07, head='mlp', subsample=20, error_analysis=False, mem_epoch=2, clip=10.0, lambda_=100.0,
                alpha=0.9, fisher_update_after=2, test_batch=128, trick=trick)
    base.update(over)
    return SimpleNamespace(**base)


def _data(r):
    """Run r's tasks (two classes each) and test loaders, from a generator of its own."""
    rs = np.random.RandomState(1000 + r)
    tasks, loaders = [], []
    for t in range(N_TASKS):
        labels = np.array([2 * t, 2 * t + 1])
        tasks.append((rs.randint(0, 256, (PER_TASK, 32, 32, 3)).astype(np.uint8), labels[rs.permutation(PER_TASK) % 2]))
        x = torch.from_numpy(rs.rand(N_TEST, 3, 32, 32).astype(np.float32))
        loaders.append([(x[:25], torch.from_numpy(labels[np.arange(25) % 2])),
                        (x[25:], torch.from_numpy(labels[np.arange(15) % 2]))])
    return tasks, loaders


def _maker(params, agents):
    from b200ocl import nets, registry

    def make(r):
        cls = registry.extra_agents.get(params.agent) or registry.agents[params.agent]
        model = nets.setup_architecture(params)
        opt = None if params.optimizer == 'Adam' else torch.optim.SGD(model.parameters(), lr=params.learning_rate)
        agents[r] = cls(model, opt, params)
        return agents[r]
    return make


def _final(agent):
    """What must match: the parameter arena, the BN statistics (and counters), the memory."""
    eng = agent.engine
    out = [eng.state.params, eng.state.bn_stats, eng.state.bn_tracked]
    if hasattr(agent, 'buffer'):
        out += [agent.buffer.buffer_img, agent.buffer.buffer_label]
    if hasattr(agent, 'memory'):
        out += [agent.memory.images, agent.memory.labels]
    return [t.detach().clone() for t in out]


def _group(case, n_concurrent, runs):
    from b200ocl import multirun
    params, agents = _params(case), {}
    data = [_data(r) for r in runs]
    acc = multirun.run_group([d[0] for d in data], [d[1] for d in data], _maker(params, agents), n_concurrent,
                             seed=SEED, first_run=runs[0])
    torch.cuda.synchronize()
    return {r: (a, _final(agents[r])) for r, a in zip(runs, acc)}


def _same(a, b, what):
    assert np.array_equal(a[0], b[0]), (what, a[0], b[0])
    for i, (x, y) in enumerate(zip(a[1], b[1])):
        assert torch.equal(x, y), (what, i)


@pytest.mark.parametrize('case', sorted(CASES))
def test_concurrent_runs_match_solo_runs_bit_for_bit(case):
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    runs = list(range(N_RUNS))
    grouped = _group(case, R, runs)
    for r in runs:
        solo = _group(case, 1, [r])[r]
        _same(grouped[r], solo, (case, r))
        assert grouped[r][0].shape == (N_TASKS, N_TASKS)
    assert not np.array_equal(grouped[0][1][0].cpu().numpy(), grouped[1][1][0].cpu().numpy())   # runs differ


@pytest.mark.parametrize('case', sorted(CASES))
def test_a_solo_run_matches_a_direct_train_learner_loop(case):
    """The driver at R = 1 against train_learner / evaluate from the same random state on the default stream."""
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import memory, multirun
    r = 4
    via = _group(case, 1, [r])[r]
    memory.flush_pending()
    multirun.RunRng(multirun.run_seed(SEED, r)).swap_in()
    params, agents = _params(case), {}
    agent = _maker(params, agents)(r)
    tasks, loaders = _data(r)
    acc = []
    for x, y in tasks:
        agent.train_learner(x, y)
        acc.append(agent.evaluate(loaders))
    torch.cuda.synchronize()
    _same(via, (np.array(acc), _final(agent)), case)


def test_the_cuda_generator_travels_with_its_run():
    """Steps that draw from all four generators, the CUDA one included: the same numbers alone and in a group."""
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import multirun

    class Stub(object):
        def __init__(self):
            self.draws = []

        def _steps(self, x, y):
            for _ in range(len(x)):
                self.draws.append((random.random(), float(np.random.rand()), float(torch.rand(1)),
                                   torch.rand(4, device='cuda').cpu().tolist()))
                yield

        def evaluate(self, loaders):
            return np.array([float(torch.rand(1, device='cuda'))])

    def go(runs, n):
        agents = {}

        def make(r):
            agents[r] = Stub()
            return agents[r]
        acc = multirun.run_group([[(np.zeros(3), None), (np.zeros(2), None)]] * len(runs), [[None]] * len(runs), make,
                                 n, seed=3, first_run=runs[0])
        return agents, acc
    grouped, acc = go([0, 1, 2], 3)
    for r in range(3):
        solo, acc_solo = go([r], 1)
        assert solo[r].draws == grouped[r].draws and np.array_equal(acc_solo[0], acc[r])
    assert grouped[0].draws != grouped[1].draws
