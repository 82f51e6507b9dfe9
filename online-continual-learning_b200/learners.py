"""Agents of the replay path with the reference surface `cls(model, opt, params)`,
`.train_learner(x_train, y_train)`, `.evaluate(test_loaders)`:
ExperienceReplay (agents/exp_replay.py:10-104: ER / MIR / ASER), SupContrastReplay (agents/scr.py:11-69), AGEM
(agents/agem.py), Lwf (agents/lwf.py), Icarl (agents/icarl.py), Gdumb (agents/gdumb.py), and EWC_pp (agents/ewc_pp.py),
DERPP (DER++), PCR and GEM, the last three lacking in the reference, all registered only on request
(registry.extra_agents), over
ContinualLearner (agents/base.py:14-113) with its training tricks (labels trick, separated softmax, kd_trick /
kd_trick_star, review trick).

The loop structure, the order of train-mode forwards (they move BN running statistics) and the
order of buffer operations follow the reference step exactly; what changes is who does the
arithmetic (the CUDA engine, not autograd) and that dead work is not executed: in the ASER
branch the reference computes and then discards two backward passes (exp_replay.py:55,77,81) --
their forwards are kept for the BN side effect, their backwards are skipped.
"""
import collections
import math
import pickle

import numpy as np
import torch

from . import memory, nets, ops
from .augment import SCRTransform
from .engine import ce_loss, cls_loss, icarl_loss, logit_mse, pcr_loss
from .memory import Buffer, input_size_match
from .nets import adopt, engine_of, EngineModel


# The train-mode passes of one replay step only interact through the BatchNorm running statistics and the gradient arena.
# With this switch on (default; B200OCL_CONCURRENT=0 turns it off) independent passes are issued on two streams -- SCR's two
# views (forward and backward), the memory / combined forwards of the ASER branch, iCaRL's teacher and student forwards --
# with deferred statistics applied in the reference's order and the second backward pass into a second gradient arena:
# most launches of this network fill a fraction of the GPU (tools/overlap_probe.py times the overlap).
import os as _os
_CONCURRENT = _os.environ.get('B200OCL_CONCURRENT', '1') != '0'


def set_concurrent(on):
    global _CONCURRENT
    _CONCURRENT = bool(on)


class AverageMeter(object):
    """utils/utils.py:25-42, but values may stay on the device until avg() is read."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.sum = 0
        self.count = 0

    def update(self, val, n):
        self.sum = self.sum + val * n
        self.count += n

    def avg(self):
        if self.count == 0:
            return 0
        return float(self.sum) / self.count


class StreamFeeder(object):
    """One task's stream: uint8 NHWC images -> fp32 NCHW in [0,1] on the device (ToTensor,
    continuum/data_utils.py:38-54), shuffled, batches of `batch`, last partial batch dropped
    (exp_replay.py:21-23).  The whole task is converted once; batches are views.

    The non-stationary tasks (--cl_type ni --ns_type noise|occlusion|blur, continuum/non_stationary.py:9-124) arrive as
    float64 NHWC [n,H,W,3] in [0,1] (H = W), on which ToTensor only transposes and .float() rounds to fp32.  Float NCHW
    [n,3,H,W] is taken as it is; any other float layout raises ValueError before anything is drawn or uploaded."""

    def __init__(self, x_train, y_train, batch, device):
        self.batch = batch
        x = np.asarray(x_train)
        if x.dtype == np.uint8:
            kind = 'u8'
        elif x.dtype.kind == 'f' and x.ndim == 4 and x.shape[1] == 3:
            kind = 'nchw'
        elif x.dtype == np.float64 and x.ndim == 4 and x.shape[3] == 3 and x.shape[1] == x.shape[2]:
            kind = 'f64'
        else:
            raise ValueError('stream images must be uint8 [n,H,W,3], float64 [n,H,H,3] in [0,1] (non-stationary tasks) '
                             'or float [n,3,H,W]; got %s %s' % (x.dtype, tuple(x.shape)))
        y = np.asarray(y_train).astype(np.int64)
        if memory.parity():
            # the reference's DataLoader(shuffle=True, drop_last=True) itself, over slot numbers: consumes the
            # default CPU generator exactly as exp_replay.py:21-23 / scr.py:29-31 do (base seed + sampler seed)
            from torch.utils.data import DataLoader, TensorDataset
            order = [b[0] for b in DataLoader(TensorDataset(torch.arange(len(y))), batch_size=batch, shuffle=True,
                                              num_workers=0, drop_last=True)]
            perm = torch.cat(order).numpy() if order else np.zeros(0, dtype=np.int64)
        else:
            perm = torch.randperm(len(y)).numpy()        # DataLoader(shuffle=True) draws from the torch CPU generator
        x = torch.from_numpy(np.ascontiguousarray(x))
        if kind in ('u8', 'f64') and torch.device(device).type == 'cuda':
            # one upload of the raw values, then shuffle + HWC->CHW (+ /255 for uint8) in one kernel (csrc/misc.cu)
            x = ops.stream_prepare(x.to(device), torch.from_numpy(perm).to(device))
        elif kind == 'u8':
            x = x[torch.from_numpy(perm)].permute(0, 3, 1, 2).to(torch.float32).div_(255.0).contiguous()
        elif kind == 'f64':
            x = x[torch.from_numpy(perm)].permute(0, 3, 1, 2).to(torch.float32).contiguous()
        else:                                             # already float NCHW
            x = x[torch.from_numpy(perm)].to(device=device, dtype=torch.float32).contiguous()
        self.x = x
        self.y_host = y[perm]
        self.y = torch.from_numpy(self.y_host).to(device)

    def __len__(self):
        return len(self.y_host) // self.batch

    def __iter__(self):
        b = self.batch
        for i in range(len(self)):
            yield self.x[i * b:(i + 1) * b], self.y[i * b:(i + 1) * b], self.y_host[i * b:(i + 1) * b]


def separated_softmax_table(old_labels, new_labels, lbl_inv_map):
    """Host side of the separated-softmax criterion (agents/base.py:100-106): the column list old_labels ++ new_labels
    (a label recurs in it when it recurs across tasks), the segment boundary, and the label -> position table of
    lbl_inv_map as an int64 array (-1 where a label has no entry: the reference raises KeyError there)."""
    cols = np.asarray(list(old_labels) + list(new_labels), dtype=np.int64)
    keys = [int(k) for k in lbl_inv_map if int(k) >= 0]
    pos = np.full(max(keys) + 1 if keys else 1, -1, dtype=np.int64)
    for k, v in lbl_inv_map.items():
        if int(k) >= 0:
            pos[int(k)] = int(v)
    return cols, len(old_labels), pos


def error_analysis_tables(old_labels, zombie, class_task_map, n_classes):
    """The per-class tables of the error analysis (agents/base.py:186-205): sets, uint8 [n_classes], bit 0 for the
    labels of new_labels_zombie (the last task's) and bit 1 for set(old_labels) - set(zombie); task, int64
    [n_classes], class_task_map with -1 where a class has no entry (the reference raises KeyError on predicting it).
    A label of either set outside the classifier's rows raises IndexError, as the reference's column indexing does."""
    zombie = set(int(c) for c in zombie)
    old = set(int(c) for c in old_labels) - zombie
    bad = sorted(c for c in zombie | old if c < 0 or c >= n_classes)
    if bad:
        raise IndexError('labels %s lie outside the %d classifier rows' % (bad, n_classes))
    sets = np.zeros(n_classes, dtype=np.uint8)
    sets[sorted(zombie)] |= 1
    sets[sorted(old)] |= 2
    task = np.full(n_classes, -1, dtype=np.int64)
    for c, t in class_task_map.items():
        if 0 <= int(c) < n_classes:
            task[int(c)] = int(t)
    return sets, task


class ErrorAnalysisUnsupported(NotImplementedError, UnboundLocalError):
    """error_analysis on the nearest-class-mean branch (SCR, iCaRL, ncm_trick).  The reference reads logits there that
    this branch never computes and dies with UnboundLocalError (agents/base.py:194,203); this is raised instead, before
    anything launches, and is caught wherever either exception is."""


def ncm_class_ids(old_labels):
    """The classes nearest-class-mean evaluation keeps one mean for: the distinct labels of old_labels in
    first-occurrence order, the keys of the reference's cls_exemplar dict (agents/base.py:124).  Under new-instance
    streams old_labels repeats every label once per task; the reference's repeated means are identical and its arg-min
    takes the first, so classifying against the distinct labels predicts what it predicts.  Without repeats this is
    old_labels itself."""
    return list(dict.fromkeys(int(c) for c in old_labels))


def ncm_fill_empty(means, counts):
    """agents/base.py:135-138: each class without exemplars (counts 0) gets one unit-norm direction drawn by
    torch.normal from the default CPU generator, in class order."""
    for k in (counts == 0).nonzero().flatten().tolist():
        mu = torch.normal(0, 1, size=(1, means.size(1))).to(means.device).squeeze()
        means[k] = mu / mu.norm()
    return means


def _drain(steps):
    for _ in steps:
        pass


def _after_train_steps(self):
    """ContinualLearner.after_train (agents/base.py:56-91) as a generator: yields after every step of the review trick's
    pass.  A function rather than a method, so that after_train also serves objects that only borrow it."""
    self.old_labels += self.new_labels
    self.new_labels_zombie = list(self.new_labels)
    self.new_labels.clear()
    self.task_seen += 1
    self._task_tables()
    if (getattr(self.params, 'trick', None) or {}).get('review_trick') and hasattr(self, 'buffer'):
        yield from self._review_steps()
    if self._takes_teacher:                                                     # base.py:90-91, after the review
        self.engine.update_teacher()
        self._teacher_live = True


def kd_mix(task_seen, kd_trick=False, kd_trick_star=False, lwf=False):
    """(w_ce, w_kd): the loss is w_ce * criterion + w_kd * distillation.  kd_trick: a = 1/(task_seen+1),
    a * loss + (1-a) * kd; kd_trick_star: the same with 1/sqrt(task_seen+1), applied after kd_trick when both are set
    (exp_replay.py:41-47, agem.py:40-46); LwF: the kd_trick mixing whatever the flags (lwf.py:38-40)."""
    w_ce, w_kd = 1.0, 0.0
    if kd_trick or lwf:
        a = 1.0 / (task_seen + 1)
        w_ce, w_kd = a, 1.0 - a
    if kd_trick_star and not lwf:
        b = 1.0 / ((task_seen + 1) ** 0.5)
        w_ce, w_kd = b * w_ce, b * w_kd + (1.0 - b)
    return w_ce, w_kd


class OptimizerSpec(collections.namedtuple('OptimizerSpec', 'kind lr weight_decay betas eps foreach')):
    """What one opt.step() runs: kind 'sgd' (lr, weight_decay) or 'adam' (also betas, eps and foreach: torch's
    multi-tensor path, else its single-tensor one; the two round sqrt(v) / bc2_sqrt differently)."""
    __slots__ = ()

    def __new__(cls, kind, lr, weight_decay, betas=None, eps=None, foreach=None):
        return super().__new__(cls, kind, lr, weight_decay, betas, eps, foreach)


class ContinualLearner(torch.nn.Module):
    """Label bookkeeping and loss dispatch of agents/base.py:14-113 for the replay path."""

    def __init__(self, model, opt, params):
        super().__init__()
        self.params = params
        self.model = model
        self.opt = opt
        self.data = params.data
        self.cuda = params.cuda
        self.epoch = params.epoch
        self.batch = params.batch
        self.verbose = params.verbose
        self.old_labels = []
        self.new_labels = []
        self.task_seen = 0
        self.lbl_inv_map = {}
        self.class_task_map = {}
        self.error_list = []       # the error analysis' history, one entry per evaluate (agents/base.py:33-39)
        self.new_class_score = []
        self.old_class_score = []
        self.fc_norm_new = []
        self.fc_norm_old = []
        self.bias_norm_new = []
        self.bias_norm_old = []
        trick = getattr(params, 'trick', None) or {}
        self._trick = {k: bool(trick.get(k)) for k in ('labels_trick', 'separated_softmax', 'kd_trick', 'kd_trick_star')}
        contrastive = params.agent in ('SCR', 'SCP')
        if contrastive and (self._trick['labels_trick'] or self._trick['separated_softmax']):
            # base.py:95-107 would feed [B,2,128] projections to a CE branch
            raise NotImplementedError('labels_trick / separated_softmax do not apply to the SupCon loss of %s' % params.agent)
        # base.py:96-107: exactly one criterion, labels trick first
        self._mode = ('labels_trick' if self._trick['labels_trick'] else
                      'separated_softmax' if self._trick['separated_softmax'] else 'ce')
        self._lwf = params.agent == 'LWF'
        # base.py:90-91 takes the teacher for kd_trick or LwF; SCR never reads it, so it is not taken there
        self._takes_teacher = (self._trick['kd_trick'] or self._lwf) and not contrastive
        self._teacher_live = False
        self._sep = None           # separated softmax: (cols, n_old, position table) on the device, one upload per task
        self._err = None           # device flag: a label the criterion cannot map (KeyError in the reference)
        if isinstance(model, EngineModel):
            self.engine = model.engine
        else:
            self.engine = adopt(model, input_size_match[params.data][1])
        self.device = self.engine.device
        self.grad_sync = None      # data-parallel stream shards: callable(engine) summing gradients over ranks
        self.grad_world = 1
        self._adam_started = False  # this learner has stepped Adam (its state is the engine's from then on)
        self._adam_synced = False   # the engine's Adam state was matched with opt.state in this train_learner call

    def _fork(self):
        """(main, side) streams with side ordered after everything issued on main so far."""
        main = torch.cuda.current_stream()
        side = self.__dict__.get('_side_stream')
        if side is None:
            side = self.__dict__['_side_stream'] = torch.cuda.Stream(device=self.device)
        side.wait_stream(main)
        return main, side

    def _throttle(self, depth=2):
        """Keep the host at most `depth` replay steps ahead of the GPU: the stream never runs dry, the launch
        queue stays short, and a CUDA-graph executable is never relaunched while it is still running."""
        if not torch.cuda.is_available():
            return
        ring = self.__dict__.setdefault('_step_events', [])
        ev = torch.cuda.Event()
        ev.record()
        ring.append(ev)
        if len(ring) > depth:
            ring.pop(0).synchronize()

    def _optimizer(self):
        """The optimizer this step runs, read afresh at every step so that a caller who changes its param group is
        followed (run.py:40 builds it with setup_opt, setup_elements.py:71-82):
          * torch.optim.SGD without momentum: OptimizerSpec('sgd', lr, weight_decay);
          * torch.optim.Adam with one param group and amsgrad, maximize, fused, capturable, differentiable and
            decoupled_weight_decay off: OptimizerSpec('adam', lr, weight_decay, betas, eps, foreach), foreach being
            the path torch takes for CUDA parameters (the multi-tensor one unless foreach=False);
          * opt None: params.optimizer selects, with params.learning_rate / weight_decay and, for 'Adam', the defaults
            setup_opt's torch.optim.Adam(lr, weight_decay) takes.
        Anything else raises NotImplementedError (AdamW is an Adam with decoupled_weight_decay=True)."""
        opt = self.opt
        if opt is None:
            name = getattr(self.params, 'optimizer', 'SGD')
            lr, wd = float(self.params.learning_rate), float(getattr(self.params, 'weight_decay', 0.0))
            if name == 'SGD':
                return OptimizerSpec('sgd', lr, wd)
            if name == 'Adam':
                return OptimizerSpec('adam', lr, wd, (0.9, 0.999), 1e-8, True)
            raise NotImplementedError('the b200ocl engine implements SGD and Adam, not %r' % name)
        if isinstance(opt, torch.optim.SGD):
            g = opt.param_groups[0]
            if g.get('momentum', 0) or g.get('nesterov', False) or g.get('dampening', 0):
                raise NotImplementedError('SGD momentum/nesterov are not used by the reference and not implemented')
            return OptimizerSpec('sgd', float(g['lr']), float(g['weight_decay']))
        if not isinstance(opt, torch.optim.Adam):
            raise NotImplementedError('the b200ocl engine implements torch.optim.SGD and torch.optim.Adam, not %s'
                                      % type(opt).__name__)
        if len(opt.param_groups) != 1:
            raise NotImplementedError('Adam with %d param groups: the engine steps one' % len(opt.param_groups))
        g = opt.param_groups[0]
        for k in ('amsgrad', 'maximize', 'fused', 'capturable', 'differentiable', 'decoupled_weight_decay'):
            if g.get(k):
                raise NotImplementedError('Adam with %s=True is not implemented (AdamW: decoupled_weight_decay)' % k)
        return OptimizerSpec('adam', float(g['lr']), float(g['weight_decay']),
                             (float(g['betas'][0]), float(g['betas'][1])), float(g['eps']), g.get('foreach') is not False)

    def _optimizer_step(self, spec, review=False):
        """opt.step() with the optimizer `spec` describes.  review: the review trick's step on p.grad.clone() / 10.
        (agents/base.py:84-88); for SGD that is SGD(lr / 10, 10 * wd) on the gradient, for Adam the division is made
        on the device and written back to the gradient arena.  With data-parallel stream shards the summed gradient is
        averaged first (one all-reduce of the flat gradient arena, folded into SGD's step size)."""
        if spec.kind == 'adam':
            if self.grad_sync is not None:
                raise NotImplementedError('data-parallel Adam: the gradient average cannot be folded into its step')
            self._adam_begin()
            self.engine.adam_step(spec.lr, spec.betas, spec.eps, spec.weight_decay, spec.foreach,
                                  grad_div=10.0 if review else None)
            return
        lr, wd = (spec.lr / 10.0, spec.weight_decay * 10.0) if review else (spec.lr, spec.weight_decay)
        if self.grad_sync is not None:
            self.grad_sync(self.engine)
            if wd != 0.0:
                raise NotImplementedError('weight decay with gradient averaging')
            lr = lr / self.grad_world
        self.engine.sgd_step(lr, wd)

    def _begin_call(self):
        """Start of a train_learner call that steps self.opt: an optimizer the engine cannot step is refused before
        anything launches, and the Adam state is matched with opt.state again at the call's first step."""
        if self._optimizer().kind == 'adam' and self.grad_sync is not None:
            raise NotImplementedError('data-parallel Adam: the gradient average cannot be folded into its step')
        self._adam_synced = False

    def _end_call(self):
        """End of a train_learner call, after after_train (and its review trick): opt.state shows the Adam state."""
        self._adam_export()

    # ------------------------------------------------------------------ Adam state (torch.optim.Adam.state)
    def _stepped(self):
        """[(parameter, arena offset, numel)] of the tensors the optimizer steps (the ones with a gradient)."""
        return [(p, o, n) for p, (o, n, hg) in zip(self.model.parameters(), self.engine.table) if hg]

    def _adam_begin(self):
        """Before the first Adam step of a train_learner call: make the engine's Adam state the optimizer's.  When the
        caller's opt.state already holds the arenas (a previous call of this learner exported them) nothing moves.
        Otherwise its state for the stepped tensors (a resumed or load_state_dict-ed optimizer) is copied into the
        arenas; every stepped tensor must then carry state with one common step.  A fresh optimizer (no state, or opt
        None on this learner's first step) starts from zero moments and step 0."""
        if self._adam_synced:
            return
        self._adam_synced = True
        st = self.engine.adam_state()
        if self.opt is None:
            if not self._adam_started:
                st.exp_avg.zero_(), st.exp_avg_sq.zero_()
                st.step = 0
            self._adam_started = True
            return
        self._adam_started = True
        stepped = self._stepped()
        states = [self.opt.state.get(p) or {} for p, _, _ in stepped]
        if all(s.get('exp_avg') is not None and s['exp_avg'].data_ptr() == st.exp_avg[o:o + n].data_ptr()
               and s.get('exp_avg_sq') is not None and s['exp_avg_sq'].data_ptr() == st.exp_avg_sq[o:o + n].data_ptr()
               and float(s['step']) == st.step for s, (_, o, n) in zip(states, stepped)):
            return
        if not any(states):
            st.exp_avg.zero_(), st.exp_avg_sq.zero_()
            st.step = 0
            return
        steps = set()
        for s, (p, o, n) in zip(states, stepped):
            if not all(k in s for k in ('step', 'exp_avg', 'exp_avg_sq')):
                raise ValueError('Adam state covers some of the stepped tensors only: the engine steps all of them '
                                 'with one step count')
            steps.add(float(s['step']))
            st.exp_avg[o:o + n].copy_(s['exp_avg'].detach().reshape(-1))
            st.exp_avg_sq[o:o + n].copy_(s['exp_avg_sq'].detach().reshape(-1))
        if len(steps) != 1:
            raise ValueError('Adam state with different step counts %s: the engine steps every tensor together'
                             % sorted(steps))
        st.step = int(steps.pop())

    def _adam_export(self):
        """After train_learner: opt.state[p] = {'step', 'exp_avg', 'exp_avg_sq'} with torch's keys and dtypes for every
        stepped tensor, the moments as views of the arenas (so opt.state_dict() reflects the engine)."""
        if self.opt is None or not self._adam_started:
            return
        st = self.engine.adam_state()
        for p, o, n in self._stepped():
            self.opt.state[p] = {'step': torch.tensor(float(st.step), dtype=torch.float32),
                                 'exp_avg': st.exp_avg[o:o + n].view(p.shape),
                                 'exp_avg_sq': st.exp_avg_sq[o:o + n].view(p.shape)}

    # ------------------------------------------------------------------ snapshot / restore (checkpoint.py)
    _TABLES = ('old_labels', 'new_labels', 'task_seen', 'lbl_inv_map', 'class_task_map', 'error_list', 'new_class_score',
               'old_class_score', 'fc_norm_new', 'fc_norm_old', 'bias_norm_new', 'bias_norm_old')

    def snapshot_parts(self):
        """What train_learner and evaluate read next, at a task boundary, with the device arrays left on the device:
        the engine's arenas (Engine.snapshot_parts), the buffer's (Buffer.snapshot_parts) when the learner has one, and
        copies of the label bookkeeping, the error-analysis history, whether the teacher is live and whether Adam has
        started."""
        out = {k: pickle.loads(pickle.dumps(getattr(self, k))) for k in self._TABLES}
        out['new_labels_zombie'] = list(getattr(self, 'new_labels_zombie', []))
        out['teacher_live'], out['adam_started'] = self._teacher_live, self._adam_started
        out['engine'] = self.engine.snapshot_parts()
        if isinstance(getattr(self, 'buffer', None), Buffer):
            out['buffer'] = self.buffer.snapshot_parts()
        return out

    def snapshot(self):
        """snapshot_parts() on the host.  restore() on a learner built with the same params takes it back."""
        return memory.host_tree(self.snapshot_parts())

    def snapshot_capacity(self):
        """Bytes of the largest snapshot_parts() device tree this learner can give."""
        n = self.engine.snapshot_capacity()
        if isinstance(getattr(self, 'buffer', None), Buffer):
            n += self.buffer.snapshot_capacity()
        return n

    def restore(self, state):
        """The inverse of snapshot(), on a learner built with the same params and not trained yet.  The derived device
        tables (separated softmax) are uploaded again and, with a torch.optim.Adam, opt.state shows the restored
        moments, as after a train_learner call."""
        self.engine.restore(state['engine'])
        for k in self._TABLES:
            setattr(self, k, state[k])
        self.new_labels_zombie = list(state['new_labels_zombie'])
        self._teacher_live, self._adam_started = state['teacher_live'], state['adam_started']
        if 'buffer' in state:
            self.buffer.restore(state['buffer'])
        self._task_tables()
        self._adam_export()

    def before_train(self, x_train, y_train):
        new_labels = list(set(np.asarray(y_train).tolist()))
        self.new_labels += new_labels
        for i, lbl in enumerate(new_labels):
            self.lbl_inv_map[lbl] = len(self.old_labels) + i
        for i in new_labels:
            self.class_task_map[i] = self.task_seen
        self._task_tables()

    def after_train(self):
        _drain(_after_train_steps(self))

    # ------------------------------------------------------------------ criterion (agents/base.py:93-113)
    def _task_tables(self):
        """Upload the separated-softmax column list and position table (they change only between tasks)."""
        if self._mode != 'separated_softmax':
            return
        cols, n_old, pos = separated_softmax_table(self.old_labels, self.new_labels, self.lbl_inv_map)
        if cols.size == 0:
            cols = np.zeros(1, dtype=np.int64)       # no label is mapped yet: every position lookup fails first
        self._sep = (torch.from_numpy(cols).to(self.device), n_old, torch.from_numpy(pos).to(self.device))

    def _err_flag(self):
        if self._err is None:
            self._err = torch.zeros(1, dtype=torch.int32, device=self.device)
        return self._err

    def _raise_label_errors(self):
        """One read per task.  The reference raises KeyError at the step that meets an unmapped label
        (base.py:105); here the steps of the task run to the end and the error surfaces when train_learner returns."""
        if self._err is not None and int(self._err.item()):
            self._err.zero_()
            raise KeyError('a label outside the logits or without a separated-softmax position was trained on '
                           '(the reference raises at agents/base.py:105)')

    def criterion(self, logits, labels, teacher_logits=None, w_ce=1.0, w_kd=0.0, want_grad=True, want_correct=False):
        """self.criterion(logits, labels) on the device, times w_ce, plus w_kd times the distillation loss against
        teacher_logits when given: dict(loss[1], dlogits, n_correct[1]).  Plain CE goes through b200ocl_ce_loss; the
        tricks and the distillation mixing through b200ocl_cls_loss.  Both raise the same device flag on a label they
        cannot map, read once per task by _raise_label_errors."""
        if self._mode == 'ce' and teacher_logits is None and w_ce == 1.0:
            return ce_loss(logits, labels, want_grad=want_grad, want_correct=want_correct, err=self._err_flag())
        cols, n_old, pos = self._sep if self._mode == 'separated_softmax' else (None, 0, None)
        return cls_loss(logits, labels, self._mode, cols=cols, n_old=n_old, pos_table=pos, teacher=teacher_logits,
                        w_ce=w_ce, w_kd=w_kd, err=self._err_flag(), want_grad=want_grad, want_correct=want_correct)

    def _kd_loss(self, logits, labels, x, want_grad=True, want_correct=False):
        """criterion mixed with the distillation term for the flags in force (exp_replay.py:41-47; lwf.py:37-39):
        the teacher forward runs only once a teacher exists and its term has a non-zero weight."""
        w_ce, w_kd = kd_mix(self.task_seen, self._trick['kd_trick'], self._trick['kd_trick_star'], self._lwf)
        t = self.engine.teacher_forward(x) if (self._teacher_live and w_kd != 0.0) else None
        return self.criterion(logits, labels, t, w_ce, w_kd if t is not None else 0.0, want_grad=want_grad,
                              want_correct=want_correct)

    def _review(self):
        _drain(self._review_steps())

    def _review_steps(self):
        """Review trick (agents/base.py:62-88, the published SCR setting config_CVPR/agent/scr/scr_5k.yml:10): one
        pass over the filled memory in shuffled batches of eps_mem_batch (drop_last), gradients divided by 10.
        g/10 followed by SGD(lr, wd) is p -= lr*(g/10 + wd*p) = SGD(lr/10, 10*wd) on g: folded into the step."""
        eng = self.engine
        spec = self._optimizer()
        n = self.buffer.current_index
        bs = self.params.eps_mem_batch
        if n == 0 or n < bs:
            return
        self.model.train()
        if memory.parity():
            from torch.utils.data import DataLoader, TensorDataset
            batches = [b[0] for b in DataLoader(TensorDataset(torch.arange(n)), batch_size=bs, shuffle=True, num_workers=0,
                                                drop_last=True)]
        else:
            perm = torch.randperm(n)
            batches = [perm[i * bs:(i + 1) * bs] for i in range(n // bs)]
        scr = self.params.agent == 'SCR'
        for idx in batches:
            idx_t = memory.to_device_i64(idx.numpy(), self.device)
            bx = ops.gather_rows(self.buffer.buffer_img, idx_t)
            by = ops.gather_rows(self.buffer.buffer_label, idx_t)
            out, ws = eng.forward_train(bx, slot=0)                                  # base.py:76 (for SCR: BN side effect only)
            if scr:
                f1, ws1 = eng.forward_train(bx, slot=0)                              # base.py:78-79
                aug = self.transform(bx)
                f2, ws2 = eng.forward_train(aug, slot=1)
                loss, dfeat = ops.supcon(torch.stack((f1, f2), dim=1), by, self.params.temp)
                eng.backward(bx, dfeat[:, 0].contiguous(), ws1)
                eng.backward(aug, dfeat[:, 1].contiguous(), ws2, accumulate=True)
            else:
                ce = self.criterion(out, by)                                         # base.py:80 (tricks apply, no KD)
                eng.backward(bx, ce['dlogits'], ws)
            self._optimizer_step(spec, review=True)                                  # base.py:83-88
            self._throttle()
            yield

    def train_learner(self, x_train, y_train):
        _drain(self._steps(x_train, y_train))

    def _steps(self, x_train, y_train):
        """train_learner as a generator that yields after every replay step (and every step of the review trick), so
        that a driver can interleave the steps of several learners (multirun.run_group).  Draining it is
        train_learner: the same launches in the same order."""
        raise NotImplementedError

    def forward(self, x):
        return self.model.forward(x)

    # ------------------------------------------------------------------ evaluate (SURVEY section 8f: next)
    _eval_cosine = False        # PCR: arg-max of the cosine between feature and classifier row (ops.cosine_argmax)

    def _ncm(self):
        return (getattr(self.params, 'trick', None) or {}).get('ncm_trick') or self.params.agent in ['ICARL', 'SCR', 'SCP']

    @torch.no_grad()
    def evaluate(self, test_loaders):
        """Accuracy per task (agents/base.py:118-227): nearest-class-mean over buffer features for SCR /
        ncm_trick, arg-max of the classifier otherwise.  Encoder features come from the engine's batched
        eval pass (the reference runs model.features once per buffered image, base.py:125-134); class
        means, nearest-mean / arg-max and the hit count are the kernels of csrc/ncm.cu; one device -> host
        read per test loader.  With params.error_analysis the arg-max runs as b200ocl_linear_argmax_ea and the
        analysis of base.py:144-226 follows (_error_analysis); on the nearest-class-mean branch it is refused."""
        ea = getattr(self.params, 'error_analysis', False)
        ncm = self._ncm()
        if ea and ncm:
            raise ErrorAnalysisUnsupported('error_analysis reads classifier logits, which the nearest-class-mean '
                                           'evaluation of %s does not compute (the reference fails with '
                                           'UnboundLocalError there)' % self.params.agent)
        if ea and self._eval_cosine:
            raise ErrorAnalysisUnsupported('error_analysis reads classifier logits, which the cosine evaluation of %s '
                                           'does not compute' % self.params.agent)
        eng = self.engine
        eng.pack()                  # the caller may have written the Parameters since the last step
        self.model.eval()           # base.py:119 (the next train_learner switches back)
        acc_array = np.zeros(len(test_loaders))
        if ncm:
            n = self.buffer.current_index
            class_ids = torch.tensor(ncm_class_ids(self.old_labels), dtype=torch.int64, device=self.device)
            feats = torch.cat([eng.features_eval(self.buffer.buffer_img[s:s + 500]) for s in range(0, n, 500)]) \
                if n else torch.zeros((0, eng.dim_in), device=self.device)
            if n and not bool(torch.isin(self.buffer.buffer_label[:n], class_ids).all()):
                raise KeyError('a buffered label was never seen in training (the reference raises here, base.py:126)')
            means, counts = ops.ncm_class_means(feats, self.buffer.buffer_label[:n], class_ids)
            ncm_fill_empty(means, counts)
        else:
            if isinstance(self.model, EngineModel):
                W, b = self.model.linear__weight, self.model.linear__bias
            else:
                W, b = self.model.linear.weight, self.model.linear.bias
        if ea:
            zombie = list(getattr(self, 'new_labels_zombie', []))
            sets, task_of = error_analysis_tables(self.old_labels, zombie, self.class_task_map, W.shape[0])
            sets_t, task_t = torch.from_numpy(sets).to(self.device), torch.from_numpy(task_of).to(self.device)
            counts = torch.zeros((len(test_loaders), 4), dtype=torch.int64, device=self.device)
            recs, batches = [], []
        for task, loader in enumerate(test_loaders):
            hits = torch.zeros(1, dtype=torch.int64, device=self.device)
            total = 0
            for batch_x, batch_y in loader:
                batch_x, batch_y = batch_x.to(self.device), batch_y.to(self.device)
                f = eng.features_eval(batch_x)
                if ncm:
                    ops.ncm_classify(f, means, class_ids, truth=batch_y, n_correct=hits)
                elif self._eval_cosine:
                    ops.cosine_argmax(f, W, truth=batch_y, n_correct=hits)
                elif ea:
                    pred_task, sums = ops.linear_argmax_ea(f, W, b, batch_y, sets_t, task_t, counts[task], n_correct=hits)
                    recs += [pred_task, sums.view(torch.int64).reshape(-1)]
                    batches.append((task, batch_y.numel()))
                else:
                    ops.linear_argmax(f, W, b, truth=batch_y, n_correct=hits)
                total += batch_y.numel()
            acc_array[task] = int(hits) / max(total, 1)
        if ea:
            # the weight / bias means of base.py:217-220 (NaN for an empty row set), then one read of everything
            old = sorted(set(int(c) for c in self.old_labels) - set(int(c) for c in zombie))
            wb = torch.cat((ops.rows_mean(W, b, zombie), ops.rows_mean(W, b, old))).view(torch.int64)
            host = torch.cat([counts.reshape(-1), wb] + recs).cpu().numpy()
            self._error_analysis(host, len(test_loaders), batches, int((sets & 1).astype(bool).sum()), int((sets & 2).astype(bool).sum()),
                                 acc_array)
        else:
            print(acc_array)
        return acc_array

    def _error_analysis(self, host, n_loaders, batches, n_new, n_old, acc_array):
        """The host side of the error analysis (agents/base.py:182-226) from the one read of evaluate: per loader the
        counts of b200ocl_linear_argmax_ea, the weight / bias means, then per batch the predicted tasks and the two
        logit sums of every row.  A prediction without a task raises KeyError before anything is appended, printed
        or written, as the reference's class_task_map lookup leaves it."""
        counts = host[:4 * n_loaders].reshape(n_loaders, 4)
        if counts[:, 3].any():
            raise KeyError('a test sample was predicted as a class never trained on (class_task_map has no entry; the '
                           'reference raises at agents/base.py:185)')
        wb = host[4 * n_loaders:4 * n_loaders + 2].view(np.float32)
        off = 4 * n_loaders + 2
        no = nn = oo = on = 0
        new_class_score, old_class_score = AverageMeter(), AverageMeter()
        correct_lb, predict_lb = [], []
        for task, n in batches:
            pred_task = host[off:off + n]
            sums = host[off + n:off + 3 * n].view(np.float64).reshape(n, 2)
            off += 3 * n
            correct_lb += [task] * n
            predict_lb += pred_task.tolist()
            if task < self.task_seen - 1:                                            # old test (:186-194)
                old_class_score.update(_set_mean(sums[:, 1], n * n_old), n)
            elif task == self.task_seen - 1:                                         # new test (:195-203)
                new_class_score.update(_set_mean(sums[:, 0], n * n_new), n)
        for task in range(n_loaders):
            if task < self.task_seen - 1:                # wrong into the last task's classes: on; anywhere else: oo
                on += int(counts[task, 0])
                oo += int(counts[task, 1] + counts[task, 2])
            elif task == self.task_seen - 1:             # wrong into the older classes: no; anywhere else: nn
                no += int(counts[task, 1])
                nn += int(counts[task, 0] + counts[task, 2])
        print(acc_array)
        self.error_list.append((no, nn, oo, on))                                     # :209-226
        self.new_class_score.append(new_class_score.avg())
        self.old_class_score.append(old_class_score.avg())
        print("no ratio: {}\non ratio: {}".format(no / (no + nn + 0.1), on / (oo + on + 0.1)))
        print(self.error_list)
        print(self.new_class_score)
        print(self.old_class_score)
        self.fc_norm_new.append(float(wb[0]))
        self.fc_norm_old.append(float(wb[2]))
        self.bias_norm_new.append(float(wb[1]))
        self.bias_norm_old.append(float(wb[3]))
        print(self.fc_norm_old)
        print(self.fc_norm_new)
        print(self.bias_norm_old)
        print(self.bias_norm_new)
        with open('confusion', 'wb') as fp:
            pickle.dump([correct_lb, predict_lb], fp)


def _set_mean(row_sums, n):
    """logits[:, S].mean().item() of one batch from the rows' fp64 sums over S: their correctly rounded total over the
    number of elements, rounded to fp32 once (NaN when S is empty)."""
    with np.errstate(invalid='ignore', divide='ignore'):
        return float(np.float32(np.float64(math.fsum(row_sums.tolist())) / np.float64(n)))


class ExperienceReplay(ContinualLearner):
    def __init__(self, model, opt, params):
        super().__init__(model, opt, params)
        self.buffer = Buffer(model, params)
        self.mem_size = params.mem_size
        self.eps_mem_batch = params.eps_mem_batch
        self.mem_iters = params.mem_iters
        self._aser_branch = params.update == 'ASER' or params.retrieve == 'ASER'
        self._needs_batch_grad = params.retrieve == 'MIR' or not self._aser_branch

    def replay_step(self, batch_x, batch_y, batch_y_host, meters=None):
        """One iteration of exp_replay.py:34-92."""
        eng = self.engine
        spec = self._optimizer()
        aser = self._aser_branch
        # in the ASER branch the stream and memory losses reach only the meters (and MIR's virtual step): their
        # distillation terms, and so the teacher forwards, are skipped when nothing reads them
        kd = not aser or meters is not None
        for _ in range(self.mem_iters):
            logits, ws = eng.forward_train(batch_x, slot=0)                         # :40  (BN stats move)
            ce = self._kd_loss(logits, batch_y, batch_x, want_grad=self._needs_batch_grad, want_correct=meters is not None) \
                if (kd or self._needs_batch_grad) else \
                self.criterion(logits, batch_y, want_grad=self._needs_batch_grad, want_correct=meters is not None)   # :41-47
            if meters is not None:
                meters['acc_batch'].update(ce['n_correct'] / batch_y.size(0), batch_y.size(0))
                meters['losses_batch'].update(ce['loss'], batch_y.size(0))
            if self._needs_batch_grad:
                eng.backward(batch_x, ce['dlogits'], ws)                            # :54-55
            mem_x, mem_y = self.buffer.retrieve(x=batch_x, y=batch_y)               # :58
            both = _CONCURRENT and aser and mem_x.size(0) > 0
            if both:
                # ASER branch: the memory forward (:62, kept for its BN side effect and the meters) and the forward of the
                # concatenated batch (:84) are independent -- two streams, statistics applied in call order
                main, side = self._fork()
                with torch.cuda.stream(side):
                    mem_logits, ws_m = eng.forward_train(mem_x, slot=1, defer_stats=True)
                    if meters is not None:
                        ce_m = self._kd_loss(mem_logits, mem_y, mem_x, want_grad=False, want_correct=True)
            elif mem_x.size(0) > 0:
                mem_logits, ws_m = eng.forward_train(mem_x, slot=1)                 # :62  (BN stats move)
                ce_m = (self._kd_loss(mem_logits, mem_y, mem_x, want_grad=not aser, want_correct=meters is not None) if kd
                        else self.criterion(mem_logits, mem_y, want_grad=False))    # :63-70
            if mem_x.size(0) > 0 and not both:
                if meters is not None:
                    meters['losses_mem'].update(ce_m['loss'], mem_y.size(0))
                    meters['acc_mem'].update(ce_m['n_correct'] / mem_y.size(0), mem_y.size(0))
                if not aser:
                    eng.backward(mem_x, ce_m['dlogits'], ws_m, accumulate=True)     # :77 (gradients accumulate)
            if aser:
                combined = torch.cat((mem_x, batch_x))                              # :82-83
                labels = torch.cat((mem_y, batch_y))
                logits_c, ws_c = eng.forward_train(combined, slot=3, defer_stats=both)   # :84
                if both:
                    main.wait_stream(side)
                    eng.apply_running_stats(ws_m, mem_x.size(0))
                    eng.apply_running_stats(ws_c, combined.size(0))
                    if meters is not None:
                        meters['losses_mem'].update(ce_m['loss'], mem_y.size(0))
                        meters['acc_mem'].update(ce_m['n_correct'] / mem_y.size(0), mem_y.size(0))
                ce_c = self.criterion(logits_c, labels)                             # :85 (no distillation term)
                eng.backward(combined, ce_c['dlogits'], ws_c)                       # :86
                self.last_loss = ce_c['loss']
            else:
                self.last_loss = ce['loss']
            self._optimizer_step(spec)                                            # :87 / :89
        # (Not overlapped with the FOLLOWING iteration's first forward on a second stream: the update's eval-feature pass
        # runs persistent one-CTA-per-SM kernels the forward cannot share the SMs with, and the host then waits for the
        # update's decision at the next retrieval.)
        self.buffer.update(batch_x, batch_y, y_host=batch_y_host)                   # :92
        self._throttle()

    def _steps(self, x_train, y_train):
        self._begin_call()
        self.before_train(x_train, y_train)
        self.engine.pack()          # the caller may have written the Parameters (load_state_dict, weight surgery)
        self.model = self.model.train()
        meters = {k: AverageMeter() for k in ('losses_batch', 'losses_mem', 'acc_batch', 'acc_mem')}
        for ep in range(self.epoch):
            stream = StreamFeeder(x_train, y_train, self.batch, self.device)   # DataLoader(shuffle=True): new order per epoch
            for i, (batch_x, batch_y, y_host) in enumerate(stream):
                self.replay_step(batch_x, batch_y, y_host, meters if self.verbose else None)
                yield
                if i % 100 == 1 and self.verbose:
                    print('==>>> it: {}, avg. loss: {:.6f}, running train acc: {:.3f}'
                          .format(i, meters['losses_batch'].avg(), meters['acc_batch'].avg()))
                    print('==>>> it: {}, mem avg. loss: {:.6f}, running mem acc: {:.3f}'
                          .format(i, meters['losses_mem'].avg(), meters['acc_mem'].avg()))
        self._raise_label_errors()
        yield from _after_train_steps(self)
        self._end_call()


class SupContrastReplay(ContinualLearner):
    def __init__(self, model, opt, params):
        nets.check_supcon(input_size_match[params.data][1], getattr(params, 'head', 'mlp'))   # before adopt() allocates
        super().__init__(model, opt, params)
        self.buffer = Buffer(model, params)
        self.mem_size = params.mem_size
        self.eps_mem_batch = params.eps_mem_batch
        self.mem_iters = params.mem_iters
        hw = input_size_match[params.data]
        self.transform = SCRTransform(size=(hw[1], hw[2]))        # scr.py:18-24

    def replay_step(self, batch_x, batch_y, batch_y_host, meters=None):
        """One iteration of scr.py:40-63."""
        eng = self.engine
        spec = self._optimizer()
        for _ in range(self.mem_iters):
            mem_x, mem_y = self.buffer.retrieve(x=batch_x, y=batch_y)               # :47
            if mem_x.size(0) > 0:                                                   # :49 (no training on an empty buffer)
                combined = torch.cat((mem_x, batch_x))                              # :52-53
                labels = torch.cat((mem_y, batch_y))
                combined_aug = self.transform(combined)                             # :54
                if _CONCURRENT:
                    n = combined.size(0)
                    main, side = self._fork()
                    with torch.cuda.stream(side):                                   # :55 two train-mode forwards, side by side
                        f2, ws2 = eng.forward_train(combined_aug, slot=1, defer_stats=True)
                    f1, ws1 = eng.forward_train(combined, slot=0, defer_stats=True)
                    main.wait_stream(side)
                    eng.apply_running_stats(ws1, n)                                 # the running statistics move in call order
                    eng.apply_running_stats(ws2, n)
                    feats = torch.stack((f1, f2), dim=1)
                    loss, dfeat = ops.supcon(feats, labels, self.params.temp)       # :56  (base.py:109-111)
                    d1, d2 = dfeat[:, 0].contiguous(), dfeat[:, 1].contiguous()
                    main, side = self._fork()
                    with torch.cuda.stream(side):                                   # :58-59 one backward per view
                        eng.backward(combined_aug, d2, ws2, alt=True)
                    eng.backward(combined, d1, ws1)
                    main.wait_stream(side)
                    eng.add_alt_grads()
                else:
                    f1, ws1 = eng.forward_train(combined, slot=0)                   # :55 two train-mode forwards
                    f2, ws2 = eng.forward_train(combined_aug, slot=1)
                    feats = torch.stack((f1, f2), dim=1)
                    loss, dfeat = ops.supcon(feats, labels, self.params.temp)       # :56  (base.py:109-111)
                    eng.backward(combined, dfeat[:, 0].contiguous(), ws1)           # :58-59
                    eng.backward(combined_aug, dfeat[:, 1].contiguous(), ws2, accumulate=True)
                self._optimizer_step(spec)                                        # :60
                self.last_loss = loss
                if meters is not None:
                    meters['losses'].update(loss, batch_y.size(0))
        self.buffer.update(batch_x, batch_y, y_host=batch_y_host)                   # :63
        self._throttle()

    def _steps(self, x_train, y_train):
        self._begin_call()
        self.before_train(x_train, y_train)
        self.engine.pack()          # the caller may have written the Parameters (load_state_dict, weight surgery)
        self.model = self.model.train()
        meters = {'losses': AverageMeter()}
        for ep in range(self.epoch):
            stream = StreamFeeder(x_train, y_train, self.batch, self.device)   # DataLoader(shuffle=True): new order per epoch
            for i, (batch_x, batch_y, y_host) in enumerate(stream):
                self.replay_step(batch_x, batch_y, y_host, meters if self.verbose else None)
                yield
                if i % 100 == 1 and self.verbose:
                    print('==>>> it: {}, avg. loss: {:.6f}, '.format(i, meters['losses'].avg()))
        yield from _after_train_steps(self)
        self._end_call()


class AGEM(ContinualLearner):
    """Averaged GEM (agents/agem.py:11-90) on the engine: the gradient of the stream batch is projected against the
    gradient of a memory batch of earlier tasks when their inner product is negative -- two train-mode
    forward / backward passes over the flat gradient arena and one projection kernel (no per-parameter Python loops)."""

    def __init__(self, model, opt, params):
        super().__init__(model, opt, params)
        self.buffer = Buffer(model, params)
        self.mem_size = params.mem_size
        self.eps_mem_batch = params.eps_mem_batch
        self.mem_iters = params.mem_iters
        self._g_cur = torch.empty_like(self.engine.state.grads)

    def replay_step(self, batch_x, batch_y, batch_y_host, meters=None):
        """One iteration of agem.py:36-84."""
        eng = self.engine
        spec = self._optimizer()
        for _ in range(self.mem_iters):
            logits, ws = eng.forward_train(batch_x, slot=0)                          # :39
            ce = self._kd_loss(logits, batch_y, batch_x, want_grad=True, want_correct=meters is not None)   # :40-46
            if meters is not None:
                meters['acc_batch'].update(ce['n_correct'] / batch_y.size(0), batch_y.size(0))
                meters['losses_batch'].update(ce['loss'], batch_y.size(0))
            eng.backward(batch_x, ce['dlogits'], ws)                                 # :53-54
            self.last_loss = ce['loss']
            if self.task_seen > 0:
                mem_x, mem_y = self.buffer.retrieve()                                # :58 (no kwargs)
                if mem_x.size(0) > 0:
                    self._g_cur.copy_(eng.state.grads)                               # :62 grad of the current batch
                    mem_logits, ws_m = eng.forward_train(mem_x, slot=1)              # :65
                    ce_m = self.criterion(mem_logits, mem_y)                         # :66 (no distillation term)
                    eng.backward(mem_x, ce_m['dlogits'], ws_m)                       # :67-68 -> grad_ref in the arena
                    ops.agem_project(self._g_cur, eng.state.grads, out=eng.state.grads)   # :73-80
            self._optimizer_step(spec)                                             # :81
        self.buffer.update(batch_x, batch_y, y_host=batch_y_host)                    # :83
        self._throttle()

    def _steps(self, x_train, y_train):
        self._begin_call()
        self.before_train(x_train, y_train)
        self.engine.pack()
        self.model = self.model.train()
        meters = {k: AverageMeter() for k in ('losses_batch', 'acc_batch')}
        for ep in range(self.epoch):
            stream = StreamFeeder(x_train, y_train, self.batch, self.device)
            for i, (batch_x, batch_y, y_host) in enumerate(stream):
                self.replay_step(batch_x, batch_y, y_host, meters if self.verbose else None)
                yield
                if i % 100 == 1 and self.verbose:
                    print('==>>> it: {}, avg. loss: {:.6f}, running train acc: {:.3f}'
                          .format(i, meters['losses_batch'].avg(), meters['acc_batch'].avg()))
        self._raise_label_errors()
        yield from _after_train_steps(self)
        self._end_call()


class Lwf(ContinualLearner):
    """Learning without Forgetting (agents/lwf.py:10-56) on the engine: no memory; per batch one train-mode forward,
    loss = a * criterion + (1 - a) * distillation against the teacher taken after the previous task, a = 1/(task_seen+1),
    one backward pass and one SGD step.  Evaluation is the classifier's arg-max."""

    def replay_step(self, batch_x, batch_y, batch_y_host, meters=None):
        """One iteration of lwf.py:30-46."""
        eng = self.engine
        spec = self._optimizer()
        logits, ws = eng.forward_train(batch_x, slot=0)                              # :35
        out = self._kd_loss(logits, batch_y, batch_x, want_grad=True, want_correct=meters is not None)   # :36-38
        if meters is not None:
            meters['acc_batch'].update(out['n_correct'] / batch_y.size(0), batch_y.size(0))
            meters['losses_batch'].update(out['loss'], batch_y.size(0))
        eng.backward(batch_x, out['dlogits'], ws)                                    # :45-46
        self._optimizer_step(spec)                                                 # :47
        self.last_loss = out['loss']
        self._throttle()

    def _steps(self, x_train, y_train):
        self._begin_call()
        self.before_train(x_train, y_train)
        self.engine.pack()
        self.model = self.model.train()
        meters = {k: AverageMeter() for k in ('losses_batch', 'acc_batch')}
        for ep in range(self.epoch):
            stream = StreamFeeder(x_train, y_train, self.batch, self.device)
            for i, (batch_x, batch_y, y_host) in enumerate(stream):
                self.replay_step(batch_x, batch_y, y_host, meters if self.verbose else None)
                yield
                if i % 100 == 1 and self.verbose:
                    print('==>>> it: {}, avg. loss: {:.6f}, running train acc: {:.3f}'
                          .format(i, meters['losses_batch'].avg(), meters['acc_batch'].avg()))
        self._raise_label_errors()
        yield from _after_train_steps(self)
        self._end_call()


class Icarl(ContinualLearner):
    """iCaRL (agents/icarl.py:15-65) on the engine.  Per batch of B stream rows: from the second task on, B memory rows
    drawn uniformly from the slots this train_learner call has not written yet are appended; one train-mode forward of
    the student and, with a previous model, one of the teacher arena (the reference's deep copy, taken at the end of
    each call before after_train and its review trick, so it holds the pre-review weights); BCE with logits against
    one-hot targets whose first n_old columns are the teacher's sigmoids (one fused kernel, b200ocl_icarl_loss); one
    backward pass and one SGD step; then the reservoir update, whose written slots are excluded from the later draws of
    the call.  Evaluation is the inherited nearest-class-mean path."""

    def __init__(self, model, opt, params):
        if params.update != 'random':
            # icarl.py:65 extends a list with what buffer.update returns; only the reservoir returns its slots
            raise NotImplementedError('iCaRL runs with the reservoir update (update=random), not %r' % params.update)
        super().__init__(model, opt, params)
        self.mem_size = params.mem_size
        self.buffer = Buffer(model, params)
        self._takes_teacher = False      # the previous model is taken in train_learner; kd_trick's teacher is never read
        self._prev_live = False
        self._updated = np.zeros(params.mem_size, dtype=bool)   # icarl.py:35 updated_idx, as a mask over the slots
        self._pos = None                 # (label -> position table on the device, n_old, K), one upload per task
        # device flag: a stream label that is not one of this task's labels.  Kept apart from the criterion's _err:
        # the reference fails here in list.index (ValueError, icarl.py:44), not in a dict lookup (KeyError, base.py:105)
        self._pos_err = None

    def snapshot_parts(self):
        out = super().snapshot_parts()
        out['prev_live'], out['updated'] = self._prev_live, self._updated.copy()
        return out

    def restore(self, state):
        super().restore(state)
        self._prev_live, self._updated = state['prev_live'], np.array(state['updated'], dtype=bool)

    def _task_tables(self):
        super()._task_tables()
        if not self.new_labels:
            return
        _, n_old, pos = separated_softmax_table(self.old_labels, self.new_labels, self.lbl_inv_map)
        self._pos = (torch.from_numpy(pos).to(self.device), n_old, n_old + len(self.new_labels))

    def replay_step(self, batch_x, batch_y, batch_y_host, meters=None):
        """One iteration of icarl.py:37-65."""
        eng = self.engine
        spec = self._optimizer()
        pos, n_old, K = self._pos
        B = batch_x.size(0)
        if K > eng.out_dim:
            # recurring labels count again in K = len(old_labels) + len(new_labels) (icarl.py:45,62 fail here)
            raise ValueError('iCaRL: %d label positions exceed the %d logits' % (K, eng.out_dim))
        if self._pos_err is None:
            self._pos_err = torch.zeros(1, dtype=torch.int32, device=self.device)
        teacher = None
        if self._prev_live:
            n = self.buffer.current_index
            excl = np.flatnonzero(self._updated[:n])
            if min(self.batch, n - excl.size) != B:
                # icarl.py:52 pads the target with B zero rows whatever the retrieval returned
                raise ValueError('iCaRL: %d memory rows can be drawn for a batch of %d (%d of %d filled slots were '
                                 'written in this call)' % (n - excl.size, B, excl.size, n))
            idx = memory.uniform_indices(n, self.batch, excl)                        # icarl.py:48-49
            mem_x = ops.gather_rows(self.buffer.buffer_img, memory.to_device_i64(idx, self.device))
            x = torch.cat((batch_x, mem_x))                                          # :51
            if _CONCURRENT:
                # the teacher's forward runs over its own arenas and workspace, side by side with the student's
                main, side = self._fork()
                with torch.cuda.stream(side):
                    teacher = eng.teacher_forward(x)                                 # :58-59
                logits, ws = eng.forward_train(x, slot=0)                            # :55
                main.wait_stream(side)
            else:
                logits, ws = eng.forward_train(x, slot=0)
                teacher = eng.teacher_forward(x)
        else:
            x = batch_x
            logits, ws = eng.forward_train(x, slot=0)
        out = icarl_loss(logits, batch_y, pos, K, n_old if teacher is not None else 0, teacher=teacher,
                         err=self._pos_err)                                          # :43-62
        eng.backward(x, out['dlogits'], ws)                                          # :63
        self._optimizer_step(spec)                                                 # :64
        self.last_loss = out['loss']
        slots = self.buffer.update(batch_x, batch_y, y_host=batch_y_host)            # :65
        self._updated[np.asarray(slots, dtype=np.int64)] = True
        self._throttle()

    def _steps(self, x_train, y_train):
        self._begin_call()
        self.before_train(x_train, y_train)
        K = self._pos[2] if self._pos is not None else 0
        if K > self.engine.out_dim:
            # replay_step's refusal, raised before this call launches anything (new-instance streams reach it at
            # their second task: every label recurs)
            raise ValueError('iCaRL: %d label positions exceed the %d logits' % (K, self.engine.out_dim))
        self.engine.pack()
        self.model = self.model.train()
        self._updated[:] = False                                                     # icarl.py:35, once per call
        for ep in range(self.epoch):
            stream = StreamFeeder(x_train, y_train, self.batch, self.device)
            for batch_x, batch_y, y_host in stream:
                self.replay_step(batch_x, batch_y, y_host)
                yield
        if self._pos_err is not None and int(self._pos_err.item()):
            self._pos_err.zero_()
            raise ValueError("iCaRL trained on a label outside the task's labels (icarl.py:44 raises there)")
        self.engine.update_teacher()                                                 # icarl.py:31, before after_train
        self._prev_live = True
        self._raise_label_errors()
        yield from _after_train_steps(self)
        self._end_call()


class Gdumb(ContinualLearner):
    """GDumb (agents/gdumb.py:12-83) on the engine.  Per train_learner call: one pass over the stream in the reference's
    batch order puts each sample through the greedy class-balanced memory (the decisions on the host, the rows moved by
    one gather and one scatter); then train_mem() trains the network from a fresh initialisation, drawn as the
    reference's setup_architecture draws it, over the whole memory for mem_epoch epochs: per batch one train-mode
    forward, the criterion (the labels trick and separated softmax apply), one backward pass and one SGD step on the
    gradient clipped to norm params.clip (b200ocl_net_sgd_step_clipped).  Evaluation is the inherited arg-max path."""

    def __init__(self, model, opt, params):
        if params.optimizer != 'SGD':
            # train_mem builds its own optimizer with setup_opt(params.optimizer, ...) (gdumb.py:63); the engine steps SGD
            raise NotImplementedError('GDumb on the b200ocl engine trains with SGD, not %r' % params.optimizer)
        if (getattr(params, 'trick', None) or {}).get('ncm_trick'):
            # the reference's nearest-class-mean evaluation reads self.buffer, which GDumb does not have
            raise NotImplementedError('ncm_trick reads a buffer GDumb does not keep')
        super().__init__(model, opt, params)
        self._takes_teacher = False      # GDumb never reads a teacher
        # not named `buffer`: after_train runs the review trick when the learner has one, and for GDumb the reference does not
        self.memory = memory.GreedyBalancedMemory(params.mem_size, input_size_match[params.data][1], self.device)

    @property
    def mem_c(self):
        """The reference's mem_c: label -> count in insertion order."""
        return self.memory.mem_c

    def snapshot_parts(self):
        out = super().snapshot_parts()
        out['memory'] = self.memory.snapshot_parts()
        return out

    def snapshot_capacity(self):
        return super().snapshot_capacity() + self.memory.snapshot_capacity()

    def restore(self, state):
        super().restore(state)
        self.memory.restore(state['memory'])

    def train_mem(self):
        """gdumb.py:52-83."""
        _drain(self._train_mem_steps())

    def _train_mem_steps(self):
        """train_mem as a generator: yields after every memory batch."""
        if self.grad_sync is not None:
            raise NotImplementedError('data-parallel GDumb: the clipping would have to follow the gradient all-reduce')
        order = self.memory.order()
        n = order.size
        if n == 0:
            raise RuntimeError('GDumb: the memory is empty (the reference fails in torch.stack, gdumb.py:57)')
        eng = self.engine
        params = nets.reference_init(self.data, eng.out_dim, eng.in_hw)                       # :61
        eng.load(params, [(torch.zeros_like(rm), torch.ones_like(rv), 0) for rm, rv in eng.bn_views()])
        self.model.train()
        lr, wd = float(self.params.learning_rate), float(self.params.weight_decay)            # :63 setup_opt
        clip = float(self.params.clip)
        bs = self.batch
        images, labels = self.memory.images, self.memory.labels
        for _ in range(self.params.mem_epoch):
            order = order[np.random.permutation(n)]                                            # :67-69, cumulative
            order_t = memory.to_device_i64(order, self.device)
            for j in range(n // bs):
                idx = order_t[j * bs:(j + 1) * bs]
                bx, by = ops.gather_rows(images, idx), ops.gather_rows(labels, idx)
                logits, ws = eng.forward_train(bx, slot=0)                                     # :78
                out = self.criterion(logits, by)                                               # :79
                eng.backward(bx, out['dlogits'], ws)                                           # :80-81
                eng.sgd_step_clipped(lr, wd, clip)                                             # :82-83
                self.last_loss = out['loss']
                self._throttle()
                yield

    def _steps(self, x_train, y_train):
        self.before_train(x_train, y_train)
        stream = StreamFeeder(x_train, y_train, self.batch, self.device)                       # :35-38 (drop_last)
        n = len(stream) * self.batch
        slots, sources = self.memory.plan(stream.y_host[:n])                                   # :40-47
        self.memory.write(stream.x, stream.y_host, slots, sources)
        yield from self._train_mem_steps()                                                     # :49
        self._raise_label_errors()
        yield from _after_train_steps(self)                                                   # :50


def der_weights(params):
    """(der_alpha, der_beta) of params as floats: each must be present, finite and >= 0 (ValueError otherwise; there is
    no default)."""
    out = []
    for name in ('der_alpha', 'der_beta'):
        v = getattr(params, name, None)
        if v is None or isinstance(v, bool):
            raise ValueError('DER++ needs params.%s (a finite number >= 0), got %r' % (name, v))
        try:
            f = float(v)
        except (TypeError, ValueError):
            raise ValueError('DER++ needs params.%s (a finite number >= 0), got %r' % (name, v)) from None
        if not math.isfinite(f) or f < 0:
            raise ValueError('DER++ needs params.%s (a finite number >= 0), got %r' % (name, v))
        out.append(f)
    return tuple(out)


class DERPP(ContinualLearner):
    """DER++ (Buzzega et al., NeurIPS 2020, online and without augmentation) on the engine; DER when der_beta = 0.  Each
    slot of the reservoir memory (memory.LogitBuffer) also keeps the logits the network gave the sample when it was
    stored.  Per stream batch (x, y), mem_iters times:
      1. the stream forward z_s, mean CE at y, backward into the gradient arena (ER's stream half);
      2. when der_alpha != 0: a uniform draw idx1 of eps_mem_batch filled slots (memory.random_retrieve, ER's numpy
         draw), their forward z1, der_alpha * mean((z1 - L[idx1])^2) (b200ocl_logit_mse, targets read in place), an
         accumulating backward;
      3. when der_beta != 0: a second, independent draw idx2, its forward, der_beta * CE at the stored labels, an
         accumulating backward;
      4. one optimizer step (SGD or Adam).
    An empty draw skips its term's passes.  The BN running statistics move in the order stream, mem1, mem2.  Then one
    reservoir update of (x, y) writes, for every slot it fills, the fp32 row of the last iteration's z_s.  With
    der_alpha = 0 and der_beta = 1 every draw and every result bit is ER's (random retrieval, reservoir update).
    Evaluation is the inherited arg-max path."""

    def __init__(self, model, opt, params):
        if params.update != 'random' or params.retrieve != 'random':
            raise NotImplementedError('DER++ keeps each slot\'s logits beside it through the reservoir update and the '
                                      'random retrieval (update=random, retrieve=random), not update=%r, retrieve=%r'
                                      % (params.update, params.retrieve))
        trick = getattr(params, 'trick', None) or {}
        on = [k for k in ('labels_trick', 'separated_softmax', 'kd_trick', 'kd_trick_star') if trick.get(k)]
        if on:
            raise NotImplementedError('DER++ runs with plain cross-entropy; %s not implemented' % ', '.join(on))
        alpha, beta = der_weights(params)
        super().__init__(model, opt, params)
        self.der_alpha, self.der_beta = alpha, beta
        self.buffer = memory.LogitBuffer(model, params, self.engine.out_dim)
        self.mem_size = params.mem_size
        self.eps_mem_batch = params.eps_mem_batch
        self.mem_iters = params.mem_iters

    def replay_step(self, batch_x, batch_y, batch_y_host, meters=None):
        if self.grad_sync is not None:
            raise NotImplementedError('data-parallel DER++: the logit memory is not kept consistent across ranks')
        eng = self.engine
        spec = self._optimizer()
        for _ in range(self.mem_iters):
            logits, ws = eng.forward_train(batch_x, slot=0)                          # 1. stream (BN stats move)
            ce = self.criterion(logits, batch_y, want_correct=meters is not None)
            if meters is not None:
                meters['acc_batch'].update(ce['n_correct'] / batch_y.size(0), batch_y.size(0))
                meters['losses_batch'].update(ce['loss'], batch_y.size(0))
            eng.backward(batch_x, ce['dlogits'], ws)
            self.last_loss_logit = self.last_loss_mem = None
            if self.der_alpha != 0.0:                                                # 2. logit term
                mem_x, _, idx = memory.random_retrieve(self.buffer, self.eps_mem_batch, return_indices=True)
                if mem_x.size(0) > 0:
                    z1, ws1 = eng.forward_train(mem_x, slot=1)
                    lm = logit_mse(z1, self.buffer.buffer_logits, idx, self.der_alpha)
                    eng.backward(mem_x, lm['dlogits'], ws1, accumulate=True)
                    self.last_loss_logit = lm['loss']
                    if meters is not None:
                        meters['losses_logit'].update(lm['loss'], mem_x.size(0))
            if self.der_beta != 0.0:                                                 # 3. memory CE term
                mem_x, mem_y, _ = memory.random_retrieve(self.buffer, self.eps_mem_batch, return_indices=True)
                if mem_x.size(0) > 0:
                    z2, ws2 = eng.forward_train(mem_x, slot=1)
                    ce_m = self.criterion(z2, mem_y, w_ce=self.der_beta, want_correct=meters is not None)
                    eng.backward(mem_x, ce_m['dlogits'], ws2, accumulate=True)
                    self.last_loss_mem = ce_m['loss']
                    if meters is not None:
                        meters['losses_mem'].update(ce_m['loss'], mem_y.size(0))
                        meters['acc_mem'].update(ce_m['n_correct'] / mem_y.size(0), mem_y.size(0))
            self.last_loss = ce['loss']
            self._optimizer_step(spec)                                               # 4.
        self.buffer.update(batch_x, batch_y, logits=logits, y_host=batch_y_host)     # z_s of the last iteration
        self._throttle()

    def _steps(self, x_train, y_train):
        self._begin_call()
        self.before_train(x_train, y_train)
        self.engine.pack()          # the caller may have written the Parameters (load_state_dict, weight surgery)
        self.model = self.model.train()
        meters = {k: AverageMeter() for k in ('losses_batch', 'losses_logit', 'losses_mem', 'acc_batch', 'acc_mem')}
        for ep in range(self.epoch):
            stream = StreamFeeder(x_train, y_train, self.batch, self.device)   # DataLoader(shuffle=True): new order per epoch
            for i, (batch_x, batch_y, y_host) in enumerate(stream):
                self.replay_step(batch_x, batch_y, y_host, meters if self.verbose else None)
                yield
                if i % 100 == 1 and self.verbose:
                    print('==>>> it: {}, avg. loss: {:.6f}, running train acc: {:.3f}'
                          .format(i, meters['losses_batch'].avg(), meters['acc_batch'].avg()))
                    print('==>>> it: {}, mem logit loss: {:.6f}, mem avg. loss: {:.6f}, running mem acc: {:.3f}'
                          .format(i, meters['losses_logit'].avg(), meters['losses_mem'].avg(), meters['acc_mem'].avg()))
        self._raise_label_errors()
        yield from _after_train_steps(self)
        self._end_call()


def pcr_temperature(params):
    """params.pcr_temp as a float, 0.09 when absent; ValueError unless it is finite and positive."""
    v = getattr(params, 'pcr_temp', None)
    if v is None:
        return 0.09
    try:
        t = float(v) if not isinstance(v, bool) else float('nan')
    except (TypeError, ValueError):
        t = float('nan')
    if not (math.isfinite(t) and t > 0):
        raise ValueError('PCR needs params.pcr_temp to be a finite number > 0, got %r' % (v,))
    return t


class PCR(ContinualLearner):
    """PCR (Lin et al., "PCR: Proxy-based Contrastive Replay for Online Class-Incremental Continual Learning", CVPR 2023)
    on the engine.  The proxies are the rows of the classifier weight linear.weight [C, d]; linear.bias never enters the
    loss and gets a zero gradient.  Per stream batch (x, y), mem_iters times:
      1. a random retrieval of eps_mem_batch memory rows (m, y_m); an empty draw skips the iteration (no pass, no step);
      2. x' = T(x), then m' = T(m), T being SCR's augmentation for the dataset's size;
      3. the train-mode forward of [x; x'], then of [m; m'] (the BN running statistics move in that order), keeping the
         encoder features;
      4. the proxy-contrastive loss of F = [F_m; F_m'; F_x; F_x'] at [y_m; y_m; y; y] (engine.pcr_loss: dF, and the
         proxies' gradient written into the gradient arena), the two backward passes from dF, one optimizer step.
    Then the reservoir update of the unaugmented (x, y).  Evaluation: the arg-max of the cosine between the eval-mode
    feature and each proxy (ops.cosine_argmax)."""

    _eval_cosine = True

    def __init__(self, model, opt, params):
        if params.update != 'random' or params.retrieve != 'random':
            raise NotImplementedError('PCR runs with the random retrieval and the reservoir update (update=random, '
                                      'retrieve=random), not update=%r, retrieve=%r' % (params.update, params.retrieve))
        trick = getattr(params, 'trick', None) or {}
        on = [k for k in ('labels_trick', 'separated_softmax', 'kd_trick', 'kd_trick_star', 'review_trick', 'ncm_trick')
              if trick.get(k)]
        if on:
            raise NotImplementedError('PCR runs its proxy-contrastive loss alone; %s not implemented' % ', '.join(on))
        temp = pcr_temperature(params)
        super().__init__(model, opt, params)
        self.temp = temp
        self.buffer = Buffer(model, params)
        self.mem_size = params.mem_size
        self.eps_mem_batch = params.eps_mem_batch
        self.mem_iters = params.mem_iters
        hw = input_size_match[params.data]
        self.transform = SCRTransform(size=(hw[1], hw[2]))
        eng = self.engine
        (wo, wn, _), (bo, bn, _) = eng.table[-2], eng.table[-1]
        c = bn
        self._proxies = eng.state.params[wo:wo + wn].view(c, wn // c)
        self._dproxies = eng.state.grads[wo:wo + wn].view(c, wn // c)
        self._dbias = eng.state.grads[bo:bo + bn]

    def replay_step(self, batch_x, batch_y, batch_y_host, meters=None):
        if self.grad_sync is not None:
            raise NotImplementedError('data-parallel PCR: the proxies\' gradient is not summed across ranks')
        eng = self.engine
        spec = self._optimizer()
        for _ in range(self.mem_iters):
            mem_x, mem_y = self.buffer.retrieve(x=batch_x, y=batch_y)                # 1.
            m = mem_x.size(0)
            if m == 0:
                continue
            x_aug = self.transform(batch_x)                                          # 2. stream first
            m_aug = self.transform(mem_x)
            xx = torch.cat((batch_x.to(torch.float32), x_aug))
            mm = torch.cat((mem_x, m_aug))
            fx, ws_x = eng.forward_train(xx, slot=0, features=True)                  # 3. BN stats: stream pair first
            fm, ws_m = eng.forward_train(mm, slot=1, features=True)
            feats = torch.cat((fm, fx))                                              # 4.
            labels = torch.cat((mem_y, mem_y, batch_y, batch_y))
            out = pcr_loss(feats, labels, self._proxies, self.temp, dproxies=self._dproxies, dbias=self._dbias,
                           err=self._err_flag())
            eng.backward(mm, out['dfeats'][:2 * m], ws_m, features=True)
            eng.backward(xx, out['dfeats'][2 * m:], ws_x, accumulate=True, features=True)
            self._optimizer_step(spec)
            self.last_loss = out['loss']
            if meters is not None:
                meters['losses'].update(out['loss'], labels.size(0))
        self.buffer.update(batch_x, batch_y, y_host=batch_y_host)
        self._throttle()

    def _steps(self, x_train, y_train):
        self._begin_call()
        self.before_train(x_train, y_train)
        self.engine.pack()          # the caller may have written the Parameters (load_state_dict, weight surgery)
        self.model = self.model.train()
        meters = {'losses': AverageMeter()}
        for ep in range(self.epoch):
            stream = StreamFeeder(x_train, y_train, self.batch, self.device)   # DataLoader(shuffle=True): new order per epoch
            for i, (batch_x, batch_y, y_host) in enumerate(stream):
                self.replay_step(batch_x, batch_y, y_host, meters if self.verbose else None)
                yield
                if i % 100 == 1 and self.verbose:
                    print('==>>> it: {}, avg. loss: {:.6f}, '.format(i, meters['losses'].avg()))
        self._raise_label_errors()
        yield from _after_train_steps(self)
        self._end_call()


def gem_margin(params):
    """params.gem_margin as a float, 0.5 when absent; ValueError unless it is finite and >= 0."""
    v = getattr(params, 'gem_margin', None)
    if v is None:
        return 0.5
    try:
        m = float(v) if not isinstance(v, bool) else float('nan')
    except (TypeError, ValueError):
        m = float('nan')
    if not (math.isfinite(m) and m >= 0):
        raise ValueError('GEM needs params.gem_margin to be a finite number >= 0, got %r' % (v,))
    return m


class GEM(ContinualLearner):
    """GEM (Lopez-Paz & Ranzato, "Gradient Episodic Memory for Continual Learning", NeurIPS 2017) on the engine, in the
    single-head form.  Each task keeps its own ring of M = mem_size // num_tasks rows (memory.TaskRingMemory).  Per
    stream batch (x, y), mem_iters times:
      1. for every earlier task whose ring is not empty, in task order: a train-mode forward over its filled rows, mean
         CE and backward; the gradient arena is copied into row k of G [t, n] (these BN statistics move first);
      2. the stream batch's train-mode forward, mean CE and backward: g in the arena;
      3. when t >= 1, ops.gem_project: P = G G^T, q = G g in fp64 and, when min q < 0, g <- g + G^T v with v the
         solution of min 1/2 v^T (P + 1e-3 I) v + q^T v subject to v >= gem_margin (the authors' project2cone2, their
         memory_strength); otherwise g is left bit for bit;
      4. one optimizer step (SGD or Adam).
    Then the batch is written into the current task's ring.  Evaluation is the inherited arg-max path."""

    MEM_SLOT = 2          # the memory passes' workspace (and graph) slot: one capture per row count
    EPS = 1e-3

    def __init__(self, model, opt, params):
        if params.update != 'random' or params.retrieve != 'random':
            raise NotImplementedError('GEM keeps its own per-task memory (update=random, retrieve=random), not '
                                      'update=%r, retrieve=%r' % (params.update, params.retrieve))
        trick = getattr(params, 'trick', None) or {}
        on = [k for k in ('labels_trick', 'separated_softmax', 'kd_trick', 'kd_trick_star', 'review_trick', 'ncm_trick')
              if trick.get(k)]
        if on:
            raise NotImplementedError('GEM runs with plain cross-entropy and arg-max evaluation; %s not implemented'
                                      % ', '.join(on))
        margin = gem_margin(params)
        M = int(params.mem_size) // int(params.num_tasks)
        if M < 1:
            raise ValueError('GEM splits mem_size=%d over num_tasks=%d: no row per task' % (params.mem_size,
                                                                                         params.num_tasks))
        super().__init__(model, opt, params)
        self.margin = margin
        self.mem_iters = params.mem_iters
        # not named `memory` or `buffer`: those names carry GDumb's and the replay buffer's layouts elsewhere
        self.rings = memory.TaskRingMemory(M, input_size_match[params.data][1], self.device)
        self._task = 0
        self._G = None                                   # [t, n] task gradients, grown when t grows
        self._v = torch.zeros(ops.GEM_MAX_T, dtype=torch.float64, device=self.device)
        self._flag = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._qp_err = torch.zeros(1, dtype=torch.int32, device=self.device)

    def snapshot_parts(self):
        out = super().snapshot_parts()
        out['rings'] = self.rings.snapshot_parts()
        return out

    def snapshot_capacity(self):
        # num_tasks rings, or 12, the most tasks of the OpenLORIS and CORe50 (ni, nc) streams, which set their own count
        return super().snapshot_capacity() + self.rings.snapshot_capacity(max(int(self.params.num_tasks), 12))

    def restore(self, state):
        super().restore(state)
        self.rings.restore(state['rings'])

    def _task_grads(self, t):
        n = self.engine.info.n_params
        if self._G is None or self._G.shape[0] < t:
            self._G = torch.empty((t, n), dtype=torch.float32, device=self.device)
        return self._G

    def replay_step(self, batch_x, batch_y, batch_y_host, meters=None):
        if self.grad_sync is not None:
            raise NotImplementedError('data-parallel GEM: the task gradients and the QP are not reduced across ranks')
        eng = self.engine
        spec = self._optimizer()
        past = [k for k in range(self._task) if self.rings.filled[k]]
        t = len(past)
        G = self._task_grads(t) if t else None
        for _ in range(self.mem_iters):
            for j, k in enumerate(past):                                              # 1.
                mx, my = self.rings.rows(k)
                logits_k, ws_k = eng.forward_train(mx, slot=self.MEM_SLOT)
                ce_k = self.criterion(logits_k, my)
                eng.backward(mx, ce_k['dlogits'], ws_k)
                G[j].copy_(eng.state.grads)
            logits, ws = eng.forward_train(batch_x, slot=0)                           # 2.
            ce = self.criterion(logits, batch_y, want_correct=meters is not None)
            eng.backward(batch_x, ce['dlogits'], ws)
            if meters is not None:
                meters['acc_batch'].update(ce['n_correct'] / batch_y.size(0), batch_y.size(0))
                meters['losses_batch'].update(ce['loss'], batch_y.size(0))
            if t:                                                                     # 3.
                ops.gem_project(G, t, eng.state.grads, out=eng.state.grads, margin=self.margin, eps=self.EPS,
                                v=self._v, flag=self._flag, err=self._qp_err)
            self.last_loss = ce['loss']
            self._optimizer_step(spec)                                                # 4.
        self.rings.write(self._task, batch_x, batch_y, batch_y_host)
        self._throttle()

    def _raise_qp_errors(self):
        if int(self._qp_err.item()):
            self._qp_err.zero_()
            raise RuntimeError('GEM: the projection QP ran out of iterations (b200ocl_gem_project set its error flag)')

    def _steps(self, x_train, y_train):
        if self.task_seen > ops.GEM_MAX_T:
            raise ValueError('GEM projects against at most %d earlier tasks; this task has %d'
                             % (ops.GEM_MAX_T, self.task_seen))
        self._begin_call()
        self.before_train(x_train, y_train)
        self._task = self.task_seen
        self.rings.begin_task(self._task)
        self.engine.pack()          # the caller may have written the Parameters (load_state_dict, weight surgery)
        self.model = self.model.train()
        meters = {k: AverageMeter() for k in ('losses_batch', 'acc_batch')}
        for ep in range(self.epoch):
            stream = StreamFeeder(x_train, y_train, self.batch, self.device)   # DataLoader(shuffle=True): new order per epoch
            for i, (batch_x, batch_y, y_host) in enumerate(stream):
                self.replay_step(batch_x, batch_y, y_host, meters if self.verbose else None)
                yield
                if i % 100 == 1 and self.verbose:
                    print('==>>> it: {}, avg. loss: {:.6f}, running train acc: {:.3f}'
                          .format(i, meters['losses_batch'].avg(), meters['acc_batch'].avg()))
        self._raise_label_errors()
        self._raise_qp_errors()
        yield from _after_train_steps(self)
        self._end_call()


def ewc_ema_schedule(n_batches, epochs, fisher_update_after):
    """Per step of one train_learner call, in order: whether update_running_fisher fires before it (ewc_pp.py:40-41;
    the counter restarts with every call)."""
    return [(ep * n_batches + i + 1) % fisher_update_after == 0 for ep in range(epochs) for i in range(n_batches)]


def ewc_ema_coefficients(alpha, fisher_update_after):
    """(keep, add) of running = (1 - alpha) * running + (1/fua * alpha) * tmp: each formed in double, as Python forms
    it, then rounded to fp32 where torch multiplies with it (ewc_pp.py:104-106)."""
    return float(np.float32(1. - alpha)), float(np.float32(1. / fisher_update_after * alpha))


def ewc_penalty_up(lambda_, task_seen, kd_trick=False, kd_trick_star=False):
    """The gradient autograd delivers to the regulariser sum F * (p - prev)^2: fp32(lambda) times the kd_trick /
    kd_trick_star mixing weights (ewc_pp.py:46-51 scale the whole loss, penalty included), multiplied in fp32 from the
    outermost weight inward, as the backward pass multiplies them (not kd_mix's double w_ce)."""
    up = np.float32(1.0)
    if kd_trick_star:
        up = np.float32(up * np.float32(1 / ((task_seen + 1) ** 0.5)))
    if kd_trick:
        up = np.float32(up * np.float32(1 / (task_seen + 1)))
    return float(np.float32(up * np.float32(lambda_)))


class EWC_pp(ContinualLearner):
    """EWC++ (agents/ewc_pp.py) on the engine.  Per batch: one train-mode forward, the criterion (the labels trick and
    separated softmax apply, mixed with the distillation term under kd_trick / kd_trick_star), one backward pass, then
    one fused launch (b200ocl_net_sgd_step_ewc) that runs, per element, the running-Fisher EMA when the host-side
    schedule says it fires before this batch, the penalty's gradient from the second call on, tmp += g*g and the SGD
    step.  At the end of each call b200ocl_ewc_consolidate sets prev = params and min-max normalises the running
    Fisher.  running_fisher, tmp_fisher, normalized_fisher and prev_params are name -> view dicts over the EWC arenas,
    as the reference's dicts are.  There is no memory; evaluation is the inherited arg-max path."""

    def __init__(self, model, opt, params):
        if (getattr(params, 'trick', None) or {}).get('ncm_trick'):
            # the reference's nearest-class-mean evaluation reads self.buffer, which EWC++ does not have
            raise NotImplementedError('ncm_trick reads a buffer EWC++ does not keep')
        super().__init__(model, opt, params)
        self.lambda_ = params.lambda_
        self.alpha = params.alpha
        self.fisher_update_after = params.fisher_update_after
        self._penalty_live = False              # ewc_pp.py:88: prev_params is filled at the end of the first call
        st = self.engine.ewc_state()
        names = [n for n, _ in self.model.named_parameters()]
        views = lambda arena: {n: arena[o:o + k].view(p.shape) for n, (o, k, _), p in
                               zip(names, self.engine.table, self.model.parameters())}
        self.running_fisher, self.tmp_fisher = views(st.running), views(st.tmp)
        self.normalized_fisher, self._prev = views(st.normalized), views(st.prev)

    def snapshot_parts(self):
        out = super().snapshot_parts()
        out['penalty_live'] = self._penalty_live
        return out

    def restore(self, state):
        super().restore(state)
        self._penalty_live = state['penalty_live']

    @property
    def prev_params(self):
        """The reference's prev_params: empty until the end of the first call."""
        return self._prev if self._penalty_live else {}

    def replay_step(self, batch_x, batch_y, batch_y_host, ema=False, meters=None):
        """One iteration of ewc_pp.py:40-62, with update_running_fisher (ema) folded into the step launch."""
        if self.grad_sync is not None:
            raise NotImplementedError('data-parallel EWC++: the Fisher accumulation would have to follow the all-reduce')
        eng = self.engine
        spec = self._optimizer()
        logits, ws = eng.forward_train(batch_x, slot=0)                              # :43
        out = self._kd_loss(logits, batch_y, batch_x, want_grad=True, want_correct=meters is not None)   # :44-51
        eng.backward(batch_x, out['dlogits'], ws)                                    # :58-59
        up = ewc_penalty_up(self.lambda_, self.task_seen, self._trick['kd_trick'], self._trick['kd_trick_star'])
        keep, add = ewc_ema_coefficients(self.alpha, self.fisher_update_after)
        want = meters is not None and self._penalty_live
        if spec.kind == 'adam':                                                      # :41, :62-63
            self._adam_begin()
            pen = eng.adam_step_ewc(spec.lr, spec.betas, spec.eps, spec.weight_decay, spec.foreach, up,
                                    self._penalty_live, ema, keep, add, want_penalty=want)
        else:
            pen = eng.sgd_step_ewc(spec.lr, spec.weight_decay, up, self._penalty_live, ema, keep, add,
                                   want_penalty=want)
        self.last_loss = out['loss']
        if meters is not None:
            loss = out['loss'] if pen is None else out['loss'] + up * pen
            meters['acc_batch'].update(out['n_correct'] / batch_y.size(0), batch_y.size(0))
            meters['losses_batch'].update(loss, batch_y.size(0))
        self._throttle()

    def _steps(self, x_train, y_train):
        self._begin_call()
        self.before_train(x_train, y_train)
        self.engine.pack()
        self.model = self.model.train()
        meters = {k: AverageMeter() for k in ('losses_batch', 'acc_batch')}
        schedule = None
        for ep in range(self.epoch):
            stream = StreamFeeder(x_train, y_train, self.batch, self.device)
            if schedule is None:
                schedule = ewc_ema_schedule(len(stream), self.epoch, self.fisher_update_after)
            for i, (batch_x, batch_y, y_host) in enumerate(stream):
                self.replay_step(batch_x, batch_y, y_host, schedule[ep * len(stream) + i],
                                 meters if self.verbose else None)
                yield
                if i % 100 == 1 and self.verbose:
                    print('==>>> it: {}, avg. loss: {:.6f}, running train acc: {:.3f}'
                          .format(i, meters['losses_batch'].avg(), meters['acc_batch'].avg()))
        self.engine.ewc_consolidate()                                                # :71-78
        self._penalty_live = True
        self._raise_label_errors()
        yield from _after_train_steps(self)                                         # :79
        self._end_call()
