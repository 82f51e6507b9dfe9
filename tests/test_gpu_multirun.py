"""GPU: runs trained side by side (multirun.run_group, R = 3, three groups) give every run, bit for bit, what it gives
alone (R = 1, the same (seed, r)): accuracy arrays and final state (agent_cases.final_state: parameters, BN statistics,
Adam and EWC++ arenas, the memory with DER++'s logits and GEM's rings), for RUN_CASES of agent_cases.CASES: ER (random,
ASER, MIR, Adam), SCR with the review trick, A-GEM, LwF, iCaRL, GDumb, EWC++, DER++, PCR and GEM.  A solo run through
the driver also matches a direct train_learner / evaluate loop from the same random state, so the step generators kept
the learners' behaviour.  Built with nets.setup_architecture on seeded synthetic uint8 tasks."""
import random

import numpy as np
import pytest
import torch

import agent_cases

pytestmark = pytest.mark.gpu

N_RUNS, R, SEED = 9, 3, 11
N_TASKS, PER_TASK, N_TEST = 3, 30, 40

RUN_CASES = ('er_random', 'er_aser', 'er_mir', 'scr_review', 'agem', 'lwf', 'icarl', 'gdumb', 'ewc', 'er_adam', 'derpp',
             'pcr', 'gem')


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


def _group(case, n_concurrent, runs):
    from b200ocl import multirun
    params, agents = agent_cases.params(case), {}
    data = [_data(r) for r in runs]
    acc = multirun.run_group([d[0] for d in data], [d[1] for d in data], _maker(params, agents), n_concurrent,
                             seed=SEED, first_run=runs[0])
    torch.cuda.synchronize()
    return {r: (a, agent_cases.final_state(agents[r])) for r, a in zip(runs, acc)}


def _same(a, b, what):
    assert np.array_equal(a[0], b[0]), (what, a[0], b[0])
    for i, (x, y) in enumerate(zip(a[1], b[1])):
        assert torch.equal(x, y), (what, i)


@pytest.mark.parametrize('case', sorted(RUN_CASES))
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


@pytest.mark.parametrize('case', sorted(RUN_CASES))
def test_a_solo_run_matches_a_direct_train_learner_loop(case):
    """The driver at R = 1 against train_learner / evaluate from the same random state on the default stream."""
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from b200ocl import memory, multirun
    r = 4
    via = _group(case, 1, [r])[r]
    memory.flush_pending()
    multirun.RunRng(multirun.run_seed(SEED, r)).swap_in()
    params, agents = agent_cases.params(case), {}
    agent = _maker(params, agents)(r)
    tasks, loaders = _data(r)
    acc = []
    for x, y in tasks:
        agent.train_learner(x, y)
        acc.append(agent.evaluate(loaders))
    torch.cuda.synchronize()
    _same(via, (np.array(acc), agent_cases.final_state(agent)), case)


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
