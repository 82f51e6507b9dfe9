"""Agents of the replay path with the reference surface `cls(model, opt, params)`,
`.train_learner(x_train, y_train)`, `.evaluate(test_loaders)`:
ExperienceReplay (agents/exp_replay.py:10-104: ER / MIR / ASER), SupContrastReplay (agents/scr.py:11-69), AGEM
(agents/agem.py), Lwf (agents/lwf.py), Icarl (agents/icarl.py), Gdumb (agents/gdumb.py) and EWC_pp (agents/ewc_pp.py, registered
only on request: registry.extra_agents), over ContinualLearner (agents/base.py:14-113) with its training tricks (labels
trick, separated softmax, kd_trick / kd_trick_star, review trick).

The loop structure, the order of train-mode forwards (they move BN running statistics) and the
order of buffer operations follow the reference step exactly; what changes is who does the
arithmetic (the CUDA engine, not autograd) and that dead work is not executed: in the ASER
branch the reference computes and then discards two backward passes (exp_replay.py:55,77,81) --
their forwards are kept for the BN side effect, their backwards are skipped.
"""
import numpy as np
import torch

from . import memory, nets, ops
from .augment import SCRTransform
from .engine import ce_loss, cls_loss, icarl_loss
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
    (exp_replay.py:21-23).  The whole task is converted once; batches are views."""

    def __init__(self, x_train, y_train, batch, device):
        self.batch = batch
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
        x = torch.from_numpy(np.ascontiguousarray(np.asarray(x_train)))
        if x.dtype == torch.uint8 and torch.device(device).type == 'cuda':
            # one upload of the raw bytes, then shuffle + HWC->CHW + /255 in one kernel (csrc/misc.cu)
            x = ops.stream_prepare(x.to(device), torch.from_numpy(perm).to(device))
        elif x.dtype == torch.uint8:
            x = x[torch.from_numpy(perm)].permute(0, 3, 1, 2).to(torch.float32).div_(255.0).contiguous()
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

    def _lr_wd(self):
        """Step size / weight decay from the optimizer the caller built (run.py:40).  Only plain
        SGD is implemented (setup_elements.py:73-75, the reference default)."""
        opt = self.opt
        if opt is None:
            return float(self.params.learning_rate), float(getattr(self.params, 'weight_decay', 0.0))
        if not isinstance(opt, torch.optim.SGD):
            raise NotImplementedError('the b200ocl engine implements torch.optim.SGD only')
        g = opt.param_groups[0]
        if g.get('momentum', 0) or g.get('nesterov', False) or g.get('dampening', 0):
            raise NotImplementedError('SGD momentum/nesterov are not used by the reference and not implemented')
        return float(g['lr']), float(g['weight_decay'])

    def _optimizer_step(self, lr, wd):
        """opt.step(); with data-parallel stream shards the summed gradient is averaged first
        (one all-reduce of the flat gradient arena, folded into the step size)."""
        if self.grad_sync is not None:
            self.grad_sync(self.engine)
            if wd != 0.0:
                raise NotImplementedError('weight decay with gradient averaging')
            lr = lr / self.grad_world
        self.engine.sgd_step(lr, wd)

    def before_train(self, x_train, y_train):
        new_labels = list(set(np.asarray(y_train).tolist()))
        self.new_labels += new_labels
        for i, lbl in enumerate(new_labels):
            self.lbl_inv_map[lbl] = len(self.old_labels) + i
        for i in new_labels:
            self.class_task_map[i] = self.task_seen
        self._task_tables()

    def after_train(self):
        self.old_labels += self.new_labels
        self.new_labels_zombie = list(self.new_labels)
        self.new_labels.clear()
        self.task_seen += 1
        self._task_tables()
        if (getattr(self.params, 'trick', None) or {}).get('review_trick') and hasattr(self, 'buffer'):
            self._review()
        if self._takes_teacher:                                                     # base.py:90-91, after the review
            self.engine.update_teacher()
            self._teacher_live = True

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
        teacher_logits when given: dict(loss[1], dlogits, n_correct[1]).  Plain CE goes through b200ocl_ce_loss as
        before; the tricks and the distillation mixing through b200ocl_cls_loss."""
        if self._mode == 'ce' and teacher_logits is None and w_ce == 1.0:
            return ce_loss(logits, labels, want_grad=want_grad, want_correct=want_correct)
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
        """Review trick (agents/base.py:62-88, the published SCR setting config_CVPR/agent/scr/scr_5k.yml:10): one
        pass over the filled memory in shuffled batches of eps_mem_batch (drop_last), gradients divided by 10.
        g/10 followed by SGD(lr, wd) is p -= lr*(g/10 + wd*p) = SGD(lr/10, 10*wd) on g: folded into the step."""
        eng = self.engine
        lr, wd = self._lr_wd()
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
            self._optimizer_step(lr / 10.0, wd * 10.0)                               # base.py:83-87
            self._throttle()

    def train_learner(self, x_train, y_train):
        raise NotImplementedError

    def forward(self, x):
        return self.model.forward(x)

    # ------------------------------------------------------------------ evaluate (SURVEY section 8f: next)
    def _ncm(self):
        return (getattr(self.params, 'trick', None) or {}).get('ncm_trick') or self.params.agent in ['ICARL', 'SCR', 'SCP']

    @torch.no_grad()
    def evaluate(self, test_loaders):
        """Accuracy per task (agents/base.py:118-227): nearest-class-mean over buffer features for SCR /
        ncm_trick, arg-max of the classifier otherwise.  Encoder features come from the engine's batched
        eval pass (the reference runs model.features once per buffered image, base.py:125-134); class
        means, nearest-mean / arg-max and the hit count are the kernels of csrc/ncm.cu; one device -> host
        read per test loader.  error_analysis is not implemented."""
        if getattr(self.params, 'error_analysis', False):
            raise NotImplementedError('error_analysis is outside the replay-path scope')
        eng = self.engine
        eng.pack()                  # the caller may have written the Parameters since the last step
        self.model.eval()           # base.py:119 (the next train_learner switches back)
        acc_array = np.zeros(len(test_loaders))
        ncm = self._ncm()
        if ncm:
            n = self.buffer.current_index
            class_ids = torch.tensor(self.old_labels, dtype=torch.int64, device=self.device)
            feats = torch.cat([eng.features_eval(self.buffer.buffer_img[s:s + 500]) for s in range(0, n, 500)]) \
                if n else torch.zeros((0, eng.dim_in), device=self.device)
            if n and not bool(torch.isin(self.buffer.buffer_label[:n], class_ids).all()):
                raise KeyError('a buffered label was never seen in training (the reference raises here, base.py:126)')
            means, counts = ops.ncm_class_means(feats, self.buffer.buffer_label[:n], class_ids)
            empty = (counts == 0).nonzero().flatten().tolist()
            for k in empty:         # base.py:135-137: a random direction for a class without exemplars
                mu = torch.normal(0, 1, size=(1, eng.dim_in)).to(self.device).squeeze()
                means[k] = mu / mu.norm()
        else:
            if isinstance(self.model, EngineModel):
                W, b = self.model.linear__weight, self.model.linear__bias
            else:
                W, b = self.model.linear.weight, self.model.linear.bias
        for task, loader in enumerate(test_loaders):
            hits = torch.zeros(1, dtype=torch.int64, device=self.device)
            total = 0
            for batch_x, batch_y in loader:
                batch_x, batch_y = batch_x.to(self.device), batch_y.to(self.device)
                f = eng.features_eval(batch_x)
                if ncm:
                    ops.ncm_classify(f, means, class_ids, truth=batch_y, n_correct=hits)
                else:
                    ops.linear_argmax(f, W, b, truth=batch_y, n_correct=hits)
                total += batch_y.numel()
            acc_array[task] = int(hits) / max(total, 1)
        print(acc_array)
        return acc_array


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
        lr, wd = self._lr_wd()
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
            self._optimizer_step(lr, wd)                                            # :87 / :89
        # (Not overlapped with the FOLLOWING iteration's first forward on a second stream: the update's eval-feature pass
        # runs persistent one-CTA-per-SM kernels the forward cannot share the SMs with, and the host then waits for the
        # update's decision at the next retrieval.)
        self.buffer.update(batch_x, batch_y, y_host=batch_y_host)                   # :92
        self._throttle()

    def train_learner(self, x_train, y_train):
        self.before_train(x_train, y_train)
        self.engine.pack()          # the caller may have written the Parameters (load_state_dict, weight surgery)
        self.model = self.model.train()
        meters = {k: AverageMeter() for k in ('losses_batch', 'losses_mem', 'acc_batch', 'acc_mem')}
        for ep in range(self.epoch):
            stream = StreamFeeder(x_train, y_train, self.batch, self.device)   # DataLoader(shuffle=True): new order per epoch
            for i, (batch_x, batch_y, y_host) in enumerate(stream):
                self.replay_step(batch_x, batch_y, y_host, meters if self.verbose else None)
                if i % 100 == 1 and self.verbose:
                    print('==>>> it: {}, avg. loss: {:.6f}, running train acc: {:.3f}'
                          .format(i, meters['losses_batch'].avg(), meters['acc_batch'].avg()))
                    print('==>>> it: {}, mem avg. loss: {:.6f}, running mem acc: {:.3f}'
                          .format(i, meters['losses_mem'].avg(), meters['acc_mem'].avg()))
        self._raise_label_errors()
        self.after_train()


class SupContrastReplay(ContinualLearner):
    def __init__(self, model, opt, params):
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
        lr, wd = self._lr_wd()
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
                self._optimizer_step(lr, wd)                                        # :60
                self.last_loss = loss
                if meters is not None:
                    meters['losses'].update(loss, batch_y.size(0))
        self.buffer.update(batch_x, batch_y, y_host=batch_y_host)                   # :63
        self._throttle()

    def train_learner(self, x_train, y_train):
        self.before_train(x_train, y_train)
        self.engine.pack()          # the caller may have written the Parameters (load_state_dict, weight surgery)
        self.model = self.model.train()
        meters = {'losses': AverageMeter()}
        for ep in range(self.epoch):
            stream = StreamFeeder(x_train, y_train, self.batch, self.device)   # DataLoader(shuffle=True): new order per epoch
            for i, (batch_x, batch_y, y_host) in enumerate(stream):
                self.replay_step(batch_x, batch_y, y_host, meters if self.verbose else None)
                if i % 100 == 1 and self.verbose:
                    print('==>>> it: {}, avg. loss: {:.6f}, '.format(i, meters['losses'].avg()))
        self.after_train()


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
        lr, wd = self._lr_wd()
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
            self._optimizer_step(lr, wd)                                             # :81
        self.buffer.update(batch_x, batch_y, y_host=batch_y_host)                    # :83
        self._throttle()

    def train_learner(self, x_train, y_train):
        self.before_train(x_train, y_train)
        self.engine.pack()
        self.model = self.model.train()
        meters = {k: AverageMeter() for k in ('losses_batch', 'acc_batch')}
        for ep in range(self.epoch):
            stream = StreamFeeder(x_train, y_train, self.batch, self.device)
            for i, (batch_x, batch_y, y_host) in enumerate(stream):
                self.replay_step(batch_x, batch_y, y_host, meters if self.verbose else None)
                if i % 100 == 1 and self.verbose:
                    print('==>>> it: {}, avg. loss: {:.6f}, running train acc: {:.3f}'
                          .format(i, meters['losses_batch'].avg(), meters['acc_batch'].avg()))
        self._raise_label_errors()
        self.after_train()


class Lwf(ContinualLearner):
    """Learning without Forgetting (agents/lwf.py:10-56) on the engine: no memory; per batch one train-mode forward,
    loss = a * criterion + (1 - a) * distillation against the teacher taken after the previous task, a = 1/(task_seen+1),
    one backward pass and one SGD step.  Evaluation is the classifier's arg-max."""

    def replay_step(self, batch_x, batch_y, batch_y_host, meters=None):
        """One iteration of lwf.py:30-46."""
        eng = self.engine
        lr, wd = self._lr_wd()
        logits, ws = eng.forward_train(batch_x, slot=0)                              # :35
        out = self._kd_loss(logits, batch_y, batch_x, want_grad=True, want_correct=meters is not None)   # :36-38
        if meters is not None:
            meters['acc_batch'].update(out['n_correct'] / batch_y.size(0), batch_y.size(0))
            meters['losses_batch'].update(out['loss'], batch_y.size(0))
        eng.backward(batch_x, out['dlogits'], ws)                                    # :45-46
        self._optimizer_step(lr, wd)                                                 # :47
        self.last_loss = out['loss']
        self._throttle()

    def train_learner(self, x_train, y_train):
        self.before_train(x_train, y_train)
        self.engine.pack()
        self.model = self.model.train()
        meters = {k: AverageMeter() for k in ('losses_batch', 'acc_batch')}
        for ep in range(self.epoch):
            stream = StreamFeeder(x_train, y_train, self.batch, self.device)
            for i, (batch_x, batch_y, y_host) in enumerate(stream):
                self.replay_step(batch_x, batch_y, y_host, meters if self.verbose else None)
                if i % 100 == 1 and self.verbose:
                    print('==>>> it: {}, avg. loss: {:.6f}, running train acc: {:.3f}'
                          .format(i, meters['losses_batch'].avg(), meters['acc_batch'].avg()))
        self._raise_label_errors()
        self.after_train()


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

    def _task_tables(self):
        super()._task_tables()
        if not self.new_labels:
            return
        _, n_old, pos = separated_softmax_table(self.old_labels, self.new_labels, self.lbl_inv_map)
        self._pos = (torch.from_numpy(pos).to(self.device), n_old, n_old + len(self.new_labels))

    def replay_step(self, batch_x, batch_y, batch_y_host, meters=None):
        """One iteration of icarl.py:37-65."""
        eng = self.engine
        lr, wd = self._lr_wd()
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
        self._optimizer_step(lr, wd)                                                 # :64
        self.last_loss = out['loss']
        slots = self.buffer.update(batch_x, batch_y, y_host=batch_y_host)            # :65
        self._updated[np.asarray(slots, dtype=np.int64)] = True
        self._throttle()

    def train_learner(self, x_train, y_train):
        self.before_train(x_train, y_train)
        self.engine.pack()
        self.model = self.model.train()
        self._updated[:] = False                                                     # icarl.py:35, once per call
        for ep in range(self.epoch):
            stream = StreamFeeder(x_train, y_train, self.batch, self.device)
            for batch_x, batch_y, y_host in stream:
                self.replay_step(batch_x, batch_y, y_host)
        if self._pos_err is not None and int(self._pos_err.item()):
            self._pos_err.zero_()
            raise ValueError("iCaRL trained on a label outside the task's labels (icarl.py:44 raises there)")
        self.engine.update_teacher()                                                 # icarl.py:31, before after_train
        self._prev_live = True
        self._raise_label_errors()
        self.after_train()


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

    def train_mem(self):
        """gdumb.py:52-83."""
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

    def train_learner(self, x_train, y_train):
        self.before_train(x_train, y_train)
        stream = StreamFeeder(x_train, y_train, self.batch, self.device)                       # :35-38 (drop_last)
        n = len(stream) * self.batch
        slots, sources = self.memory.plan(stream.y_host[:n])                                   # :40-47
        self.memory.write(stream.x, stream.y_host, slots, sources)
        self.train_mem()                                                                       # :49
        self._raise_label_errors()
        self.after_train()                                                                     # :50


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

    @property
    def prev_params(self):
        """The reference's prev_params: empty until the end of the first call."""
        return self._prev if self._penalty_live else {}

    def replay_step(self, batch_x, batch_y, batch_y_host, ema=False, meters=None):
        """One iteration of ewc_pp.py:40-62, with update_running_fisher (ema) folded into the step launch."""
        if self.grad_sync is not None:
            raise NotImplementedError('data-parallel EWC++: the Fisher accumulation would have to follow the all-reduce')
        eng = self.engine
        lr, wd = self._lr_wd()
        logits, ws = eng.forward_train(batch_x, slot=0)                              # :43
        out = self._kd_loss(logits, batch_y, batch_x, want_grad=True, want_correct=meters is not None)   # :44-51
        eng.backward(batch_x, out['dlogits'], ws)                                    # :58-59
        up = ewc_penalty_up(self.lambda_, self.task_seen, self._trick['kd_trick'], self._trick['kd_trick_star'])
        keep, add = ewc_ema_coefficients(self.alpha, self.fisher_update_after)
        pen = eng.sgd_step_ewc(lr, wd, up, self._penalty_live, ema, keep, add,
                               want_penalty=meters is not None and self._penalty_live)   # :41, :62-63
        self.last_loss = out['loss']
        if meters is not None:
            loss = out['loss'] if pen is None else out['loss'] + up * pen
            meters['acc_batch'].update(out['n_correct'] / batch_y.size(0), batch_y.size(0))
            meters['losses_batch'].update(loss, batch_y.size(0))
        self._throttle()

    def train_learner(self, x_train, y_train):
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
                if i % 100 == 1 and self.verbose:
                    print('==>>> it: {}, avg. loss: {:.6f}, running train acc: {:.3f}'
                          .format(i, meters['losses_batch'].avg(), meters['acc_batch'].avg()))
        self.engine.ewc_consolidate()                                                # :71-78
        self._penalty_live = True
        self._raise_label_errors()
        self.after_train()                                                           # :79
