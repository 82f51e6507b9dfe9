"""CPU: the task loop of every agent's train_learner, with the engine, the memory and replay_step replaced by recorders.

For each agent class, one call over two epochs of a 211-sample stream in batches of 2 (105 batches per epoch, the last
sample dropped; the verbose progress lines fall at i = 1 and i = 101) pins:
  * the event log: begin and end of the call, before_train, pack, model.train(), the agent's own actions at the start
    and end of the task (rings.begin_task, update_teacher, ewc_consolidate), every replay_step with the stream rows it
    got, its meter keys and EWC++'s ema flag, each yield, the review trick's steps and the teacher update after them;
  * the stream order: one StreamFeeder per epoch drawn from the default generator, in both the randperm and the parity
    (DataLoader) orders, and nothing else drawn;
  * the verbose progress lines, byte for byte;
  * which exception a call raises when several error flags are set, and what ran before it."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

N, BATCH, EPOCHS = 211, 2, 2
NB = N // BATCH
REVIEW = 3                  # steps of the stand-in review trick
SEED = 1234
FISHER_UPDATE_AFTER = 4     # does not divide NB: the EMA counter runs on across the epoch boundary

X = np.zeros((N, 2, 2, 3), np.uint8)
X[:, 0, 0, 0] = np.arange(N)             # each image carries its row number
Y = np.arange(N) % 3

# the value each meter takes at step s (1-based) of the call: its average after m steps is VALUES[k] * (m + 1) / 2
VALUES = {'losses_batch': 0.25, 'acc_batch': 0.5, 'losses_mem': 0.125, 'acc_mem': 0.75, 'losses_logit': 0.0625,
          'losses': 1.5}

BATCH_LINE = ('==>>> it: {}, avg. loss: {:.6f}, running train acc: {:.3f}', ('losses_batch', 'acc_batch'))
LOSS_LINE = ('==>>> it: {}, avg. loss: {:.6f}, ', ('losses',))
MEM_LINE = ('==>>> it: {}, mem avg. loss: {:.6f}, running mem acc: {:.3f}', ('losses_mem', 'acc_mem'))
DER_MEM_LINE = ('==>>> it: {}, mem logit loss: {:.6f}, mem avg. loss: {:.6f}, running mem acc: {:.3f}',
                ('losses_logit', 'losses_mem', 'acc_mem'))

# lines: the verbose progress lines; head / tail: the agent's events after before_train / after the last step;
# buffer: the agent keeps a replay buffer (the review trick runs over it); review: params.trick['review_trick'];
# teacher: the teacher is taken after the review (kd_trick, LwF)
SPECS = {
    'ExperienceReplay': dict(lines=[BATCH_LINE, MEM_LINE], buffer=True, review=True, teacher=True),
    'SupContrastReplay': dict(lines=[LOSS_LINE], buffer=True, review=True),
    'AGEM': dict(lines=[BATCH_LINE], buffer=True, review=True),
    'Lwf': dict(lines=[BATCH_LINE], review=True, teacher=True),
    'Icarl': dict(lines=[], buffer=True, review=True, tail=['update_teacher']),
    'DERPP': dict(lines=[BATCH_LINE, DER_MEM_LINE], buffer=True, review=True),
    'PCR': dict(lines=[LOSS_LINE], buffer=True),
    'GEM': dict(lines=[BATCH_LINE], head=[('rings.begin_task', 0)]),
    'EWC_pp': dict(lines=[BATCH_LINE], review=True, tail=['ewc_consolidate']),
}
AGENTS = sorted(SPECS)


class _Engine(object):
    out_dim = 10

    def __init__(self, log):
        self.log = log

    def pack(self):
        self.log.append('pack')

    def update_teacher(self):
        self.log.append('update_teacher')

    def ewc_consolidate(self):
        self.log.append('ewc_consolidate')


class _Model(object):
    def __init__(self, log):
        self.log = log

    def train(self):
        self.log.append('train')
        return self


class _Rings(object):
    def __init__(self, log):
        self.log = log

    def begin_task(self, t):
        self.log.append(('rings.begin_task', t))


class _Memory(object):
    def __init__(self, log):
        self.log = log

    def plan(self, labels):
        self.log.append(('memory.plan', tuple(labels.tolist())))
        return 'slots', 'sources'

    def write(self, x, y_host, slots, sources):
        self.log.append(('memory.write', _rows(x), tuple(y_host.tolist()), slots, sources))


def _rows(x):
    return tuple(int(v) for v in (x[:, 0, 0, 0] * 255).round().tolist())


def _review(log):
    for k in range(REVIEW):
        log.append(('review', k))
        yield


def _train_mem(log):
    for k in range(REVIEW):
        log.append(('train_mem', k))
        yield


def _replay_step(log, ewc):
    steps = [0]

    def record(batch_x, batch_y, batch_y_host, meters, extra):
        steps[0] += 1
        assert batch_y.tolist() == batch_y_host.tolist()
        if meters is not None:
            for k in meters:
                meters[k].update(VALUES[k] * steps[0], 1)
        log.append(('step', _rows(batch_x), None if meters is None else tuple(sorted(meters))) + extra)

    if ewc:
        def replay_step(batch_x, batch_y, batch_y_host, ema=False, meters=None):
            record(batch_x, batch_y, batch_y_host, meters, (ema,))
    else:
        def replay_step(batch_x, batch_y, batch_y_host, meters=None):
            record(batch_x, batch_y, batch_y_host, meters, ())
    return replay_step


def _agent(name, log, verbose=False):
    from b200ocl import learners
    cls = getattr(learners, name)
    spec = SPECS.get(name, {})
    a = cls.__new__(cls)
    torch.nn.Module.__init__(a)
    a.params = SimpleNamespace(trick={'review_trick': spec.get('review', False)})
    a.epoch, a.batch, a.verbose, a.device = EPOCHS, BATCH, verbose, 'cpu'
    a.old_labels, a.new_labels, a.task_seen, a.lbl_inv_map, a.class_task_map = [], [], 0, {}, {}
    a._mode, a._err, a._takes_teacher, a._teacher_live = 'ce', None, spec.get('teacher', False), False
    a.engine, a.model = _Engine(log), _Model(log)
    a._begin_call = lambda: log.append('begin_call')
    a._end_call = lambda: log.append('end_call')
    before_train = a.before_train
    a.before_train = lambda x, y: (log.append('before_train'), before_train(x, y))[1]
    a._review_steps = lambda: _review(log)
    a.replay_step = _replay_step(log, ewc=name == 'EWC_pp')
    if spec.get('buffer'):
        a.buffer = object()
    if name == 'Icarl':
        a._updated, a._pos, a._pos_err, a._prev_live = np.ones(8, bool), None, None, False
    elif name == 'GEM':
        a.rings, a._task, a._qp_err = _Rings(log), None, torch.zeros(1, dtype=torch.int32)
    elif name == 'EWC_pp':
        a.fisher_update_after, a._penalty_live = FISHER_UPDATE_AFTER, False
    elif name == 'Gdumb':
        a.memory = _Memory(log)
        a._train_mem_steps = lambda: _train_mem(log)
    return a


def _feeders(n):
    """The first n StreamFeeders drawn from the seeded default generator, and the draw that follows them."""
    from b200ocl import learners
    torch.manual_seed(SEED)
    feeders = [learners.StreamFeeder(X, Y, BATCH, 'cpu') for _ in range(n)]
    return feeders, torch.rand(1)


def _drive(steps, log):
    torch.manual_seed(SEED)
    for _ in steps:
        log.append('yield')
    return torch.rand(1)


def _expected(name, verbose):
    spec = SPECS[name]
    keys = sorted(k for _, ks in spec['lines'] for k in ks)
    keys = tuple(keys) if verbose and keys else None
    feeders, after = _feeders(EPOCHS)
    log = ['begin_call', 'before_train'] + spec.get('head', []) + ['pack', 'train']
    s = 0
    for f in feeders:
        for bx, _, _ in f:
            extra = ((s + 1) % FISHER_UPDATE_AFTER == 0,) if name == 'EWC_pp' else ()
            log += [('step', _rows(bx), keys) + extra, 'yield']
            s += 1
    tail = len(log) + len(spec.get('tail', []))
    log += spec.get('tail', [])
    if spec.get('buffer') and spec.get('review'):
        for k in range(REVIEW):
            log += [('review', k), 'yield']
    if spec.get('teacher'):
        log.append('update_teacher')
    log.append('end_call')
    text = ''
    if verbose:
        for ep in range(EPOCHS):
            for i in (1, 101):
                m = ep * NB + i + 1
                for fmt, ks in spec['lines']:
                    text += fmt.format(i, *[VALUES[k] * (m + 1) / 2 for k in ks]) + '\n'
    return log, after, tail, text


@pytest.fixture(params=['randperm', 'parity'])
def order(request, monkeypatch):
    from b200ocl import memory
    monkeypatch.setitem(memory._mode, 'parity', request.param == 'parity')
    return request.param


@pytest.mark.parametrize('verbose', [False, True])
@pytest.mark.parametrize('name', AGENTS)
def test_task_loop(name, verbose, order, capsys):
    log = []
    a = _agent(name, log, verbose)
    after = _drive(a._steps(X, Y), log)
    want, want_after, _, text = _expected(name, verbose)
    assert log == want
    assert log.count('yield') == EPOCHS * NB + (REVIEW if SPECS[name].get('buffer') and SPECS[name].get('review')
                                                else 0)
    assert torch.equal(after, want_after)                                # one StreamFeeder per epoch, nothing else
    assert capsys.readouterr().out == text
    assert a.task_seen == 1 and a.old_labels == [0, 1, 2] and a.new_labels == []
    if name == 'Icarl':
        assert a._prev_live and not a._updated.any()
    elif name == 'GEM':
        assert a._task == 0
    elif name == 'EWC_pp':
        assert a._penalty_live


@pytest.mark.parametrize('name', AGENTS + ['Gdumb'])
def test_train_learner_drains_the_same_loop(name):
    log, drained = [], []
    _drive(_agent(name, log)._steps(X, Y), log)
    torch.manual_seed(SEED)
    _agent(name, drained).train_learner(X, Y)
    assert drained == [e for e in log if e != 'yield']


def test_gdumb_task(order):
    log = []
    a = _agent('Gdumb', log)
    after = _drive(a._steps(X, Y), log)
    (f,), want_after = _feeders(1)
    assert log == ['before_train', ('memory.plan', tuple(f.y_host[:NB * BATCH].tolist())),
                   ('memory.write', _rows(f.x), tuple(f.y_host.tolist()), 'slots', 'sources')] + \
        [e for k in range(REVIEW) for e in (('train_mem', k), 'yield')]
    assert torch.equal(after, want_after)
    assert a.task_seen == 1


@pytest.mark.parametrize('name', [n for n in AGENTS if n != 'SupContrastReplay'] + ['Gdumb'])
def test_label_error_is_raised_after_the_last_step(name):
    """The criterion's flag raises KeyError once the task's steps (and the agent's end-of-task actions) have run,
    before the review trick.  (SCR's SupCon loss never raises the flag.)"""
    log = []
    a = _agent(name, log)
    a._err = torch.ones(1, dtype=torch.int32)
    with pytest.raises(KeyError):
        _drive(a._steps(X, Y), log)
    assert int(a._err) == 0
    if name == 'Gdumb':
        assert log[-2:] == [('train_mem', REVIEW - 1), 'yield']
    else:
        want, _, tail, _ = _expected(name, False)
        assert log == want[:tail]


def test_icarl_position_error_wins_over_label_error():
    log = []
    a = _agent('Icarl', log)
    a._pos_err = torch.ones(1, dtype=torch.int32)
    a._err = torch.ones(1, dtype=torch.int32)
    with pytest.raises(ValueError, match="task's labels"):
        _drive(a._steps(X, Y), log)
    want, _, tail, _ = _expected('Icarl', False)
    assert log == want[:tail - 1]                                         # no teacher taken
    assert int(a._pos_err) == 0 and int(a._err) == 1 and not a._prev_live


def test_icarl_too_many_label_positions_is_refused_before_pack():
    log = []
    a = _agent('Icarl', log)
    a.engine.out_dim = 2
    with pytest.raises(ValueError, match='label positions'):
        _drive(a._steps(X, Y), log)
    assert log == ['begin_call', 'before_train']


def test_gem_label_error_wins_over_qp_error():
    log = []
    a = _agent('GEM', log)
    a._err = torch.ones(1, dtype=torch.int32)
    a._qp_err = torch.ones(1, dtype=torch.int32)
    with pytest.raises(KeyError):
        _drive(a._steps(X, Y), log)
    assert int(a._err) == 0 and int(a._qp_err) == 1


def test_gem_qp_error_is_raised_after_the_last_step():
    log = []
    a = _agent('GEM', log)
    a._qp_err = torch.ones(1, dtype=torch.int32)
    with pytest.raises(RuntimeError, match='QP'):
        _drive(a._steps(X, Y), log)
    want, _, tail, _ = _expected('GEM', False)
    assert log == want[:tail] and int(a._qp_err) == 0
