"""The agent configurations the experiment-level GPU tests run, and what those tests compare.

  * CASES: every configuration by name.  test_gpu_checkpoint.py, test_gpu_checkpoint_async.py, test_gpu_multirun.py
    (and through it test_gpu_graphs.py) and test_gpu_multidevice.py each name the ones they run.
  * params(case): the params namespace of a case on the CIFAR-10-shaped synthetic tasks of those files; the experiment
    drivers add their own fields (num_runs, seed, stub_data, ...) on top.
  * extra(case): the install(extra=...) of a case, for the agents registered only on request.
  * final_state(agent): everything a run must reproduce bit for bit.  The stub reference trees of
    test_gpu_checkpoint.py and test_gpu_multidevice.py import it (their worker processes find this directory on the
    sys.path they inherit).
  * HW, NCLS, _load, _learner: a learner with seeded weights at a dataset's shapes, for the per-agent files."""
from types import SimpleNamespace

import torch

from oracle import resnet as oresnet

CASES = {
    'er_random': dict(),
    'er_aser': dict(update='ASER', retrieve='ASER'),
    'er_mir': dict(retrieve='MIR'),
    'er_gss': dict(update='GSS'),
    'er_review_sep': dict(trick_on=('review_trick', 'separated_softmax')),
    'er_adam': dict(optimizer='Adam', learning_rate=1e-3),
    'scr': dict(agent='SCR'),
    'scr_review': dict(agent='SCR', trick_on=('review_trick',)),
    'agem': dict(agent='AGEM'),
    'lwf': dict(agent='LWF'),
    'lwf_kd': dict(agent='LWF', trick_on=('kd_trick',)),
    'icarl': dict(agent='ICARL', mem_size=100),
    'gdumb': dict(agent='GDUMB'),
    'ewc': dict(agent='EWC'),
    'derpp': dict(agent='DERPP', der_alpha=0.3, der_beta=0.5),
    'pcr': dict(agent='PCR'),
    'gem': dict(agent='GEM'),
}

TRICKS = ('labels_trick', 'kd_trick', 'separated_softmax', 'review_trick', 'ncm_trick', 'kd_trick_star')


def params(case):
    over = dict(CASES[case])
    trick = {k: k in over.pop('trick_on', ()) for k in TRICKS}
    base = dict(data='cifar10', cuda=True, epoch=1, batch=10, verbose=False, mem_size=20, eps_mem_batch=10,
                mem_iters=1, update='random', retrieve='random', agent='ER', k=3, aser_type='asvm', n_smp_cls=1.5,
                num_tasks=3, buffer_tracker=False, optimizer='SGD', learning_rate=0.1, weight_decay=0, temp=0.07,
                head='mlp', subsample=20, error_analysis=False, mem_epoch=2, clip=10.0, gss_mem_strength=10,
                gss_batch_size=10, lambda_=100.0, alpha=0.9, fisher_update_after=2, test_batch=128, trick=trick)
    base.update(over)
    return SimpleNamespace(**base)


def extra(case):
    from b200ocl import registry
    agent = CASES[case].get('agent', 'ER')
    return (agent,) if agent in registry.extra_agents else ()


def final_state(agent):
    """What must match, on the host: the arenas (parameters, BN statistics and counters, Adam, EWC++) and the memory
    (buffer with its logits, GDumb's memory, GEM's rings).  The first three entries are always params, bn_stats and
    bn_tracked."""
    eng = agent.engine
    out = [eng.state.params, eng.state.bn_stats, eng.state.bn_tracked]
    adam, ewc = getattr(eng, '_adam', None), getattr(eng, '_ewc', None)
    if adam is not None:
        out += [adam.exp_avg, adam.exp_avg_sq, torch.tensor(adam.step)]
    if ewc is not None:
        out += [ewc.running, ewc.tmp, ewc.normalized, ewc.prev]
    if hasattr(agent, 'buffer'):
        out += [agent.buffer.buffer_img, agent.buffer.buffer_label]
        if hasattr(agent.buffer, 'buffer_logits'):
            out.append(agent.buffer.buffer_logits)
    if hasattr(agent, 'memory'):
        out += [agent.memory.images, agent.memory.labels]
    if hasattr(agent, 'rings'):
        for images, labels in zip(agent.rings.images, agent.rings.labels):
            out += [images, labels]
    return [t.detach().cpu().clone() for t in out]


HW = {'cifar100': 32, 'mini_imagenet': 84, 'core50': 128, 'openloris': 50}
NCLS = {'cifar100': 100, 'mini_imagenet': 100, 'core50': 50, 'openloris': 69}


def _load(agent, p, bn, spec):
    agent.engine.load(list(p.values()), [(bn[n + '.running_mean'], bn[n + '.running_var']) for n in oresnet.bn_names(spec)])


def _learner(params, seed, opt=None):
    """params.agent's learner (registered or opt-in) at params.data's shapes, loaded with oresnet.seeded_state(seed);
    returns (agent, spec)."""
    from b200ocl import nets, registry
    spec = oresnet.Spec(HW[params.data], 20, NCLS[params.data])
    p0, bn0 = oresnet.seeded_state(spec, seed)
    model = nets.setup_architecture(params)
    cls = registry.agents.get(params.agent) or registry.extra_agents[params.agent]
    agent = cls(model, opt(model) if opt else None, params)
    _load(agent, p0, bn0, spec)
    return agent, spec
