"""Buffer update plugins with the reference surface: Reservoir_update
(utils/buffer/reservoir_update.py:3-60) and ASER_update (utils/buffer/aser_update.py:9-112)."""
import numpy as np
import torch

from . import memory, ops
from .memory import ClassBalancedRandomSampling, n_classes, to_device_i64, uniform_indices
from .nets import engine_of


def _host_labels(y, kwargs):
    """Labels of the incoming batch on the host: the learners pass y_host=; anything else pays one
    device->host copy."""
    yh = kwargs.get('y_host')
    if yh is None:
        yh = y.detach().cpu().numpy()
    return np.asarray(yh, dtype=np.int64)


def reservoir_draws(n, n_seen, device=None):
    """The reference draws float32 uniforms in [0, n_seen) and truncates (reservoir_update.py:35), on x's
    device.  Default mode: the same call on the CPU generator (no device -> host sync in the step); parity
    mode: the reference's call on the reference's device, then one copy to the host."""
    if memory.parity() and device is not None:
        dev = memory.parity_rng_device(device)
        return torch.FloatTensor(n).to(dev).uniform_(0, n_seen).long().cpu().numpy()
    return torch.FloatTensor(n).uniform_(0, n_seen).long().numpy()


def reservoir_plan(draws, mem_size):
    """Overwrite map of reservoir sampling: slot -> position in the incoming batch; a slot drawn
    twice keeps the last writer; slots in first-seen order (dict semantics, reservoir_update.py:53)."""
    idx_map = {}
    for i, s in enumerate(np.asarray(draws).tolist()):
        if s < mem_size:
            idx_map[int(s)] = i
    return list(idx_map.keys()), list(idx_map.values())


class Reservoir_update(object):
    def __init__(self, params):
        super().__init__()

    def update(self, buffer, x, y, **kwargs):
        y_host = _host_labels(y, kwargs)
        batch_size = x.size(0)
        mem = buffer.buffer_img.size(0)
        place_left = max(0, mem - buffer.current_index)
        if place_left:
            offset = min(place_left, batch_size)
            s, e = buffer.current_index, buffer.current_index + offset
            buffer.buffer_img[s:e].copy_(x[:offset])
            buffer.buffer_label[s:e].copy_(y[:offset])
            buffer.labels_host[s:e] = y_host[:offset]
            buffer.current_index += offset
            buffer.n_seen_so_far += offset
            if offset == batch_size:
                return list(range(s, e))
        x, y, y_host = x[place_left:], y[place_left:], y_host[place_left:]
        draws = reservoir_draws(x.size(0), buffer.n_seen_so_far, x.device)
        self.last_draws = draws
        buffer.n_seen_so_far += x.size(0)
        slots, src = reservoir_plan(draws, mem)
        if not slots:
            return []
        src_t = to_device_i64(src, x.device)
        buffer.write(slots, ops.gather_rows(x, src_t) if x.is_cuda else x[src_t],
                     ops.gather_rows(y, src_t) if y.is_cuda else y[src_t], y_host[src])
        return slots


def aser_update_partition(order, n_cand_buf, cand_ind):
    """Replacement sets from the descending SV ranking (aser_update.py:88-102): the first
    n_cand_buf ranks are kept; current-batch samples among them replace the buffered samples
    among the rest."""
    order = np.asarray(order)
    large, small = order[:n_cand_buf], order[n_cand_buf:]
    ind_cur = large[large >= n_cand_buf] - n_cand_buf
    ind_buffer = np.asarray(cand_ind)[small[small < n_cand_buf]]
    return ind_cur, ind_buffer


class ASER_update(object):
    def __init__(self, params, **kwargs):
        super().__init__()
        self.device = 'cuda' if torch.cuda.is_available() else 'cpu'
        self.k = params.k
        self.mem_size = params.mem_size
        self.num_tasks = params.num_tasks
        self.out_dim = n_classes[params.data]
        self.n_smp_cls = int(params.n_smp_cls)
        self.n_total_smp = int(params.n_smp_cls * self.out_dim)
        self.reservoir_update = Reservoir_update(params)
        self._last_decision = None
        if self.n_total_smp + int(getattr(params, 'batch', 0)) > min(ops.KNN_MAX_CAND, ops.RANK_MAX):
            raise ValueError('ASER update: n_smp_cls*num_classes + batch = %d candidates exceed the kNN-SV / ranking kernel limit %d'
                             % (self.n_total_smp + int(params.batch), min(ops.KNN_MAX_CAND, ops.RANK_MAX)))
        ClassBalancedRandomSampling.reset()

    def update(self, buffer, x, y, **kwargs):
        memory.flush_pending()
        y_host = _host_labels(y, kwargs)
        place_left = self.mem_size - buffer.current_index
        if place_left:
            # fill phase: sequential insert + class-cache update (aser_update.py:28-35)
            n_fit = min(place_left, x.size(0))
            ind = np.arange(buffer.current_index, buffer.current_index + n_fit)
            ClassBalancedRandomSampling.update_cache(buffer.buffer_label, self.out_dim, new_y=y_host[:n_fit], ind=ind)
            self.reservoir_update.update(buffer, x[:n_fit], y[:n_fit], y_host=y_host[:n_fit])
        if buffer.current_index == self.mem_size:
            self._update_by_knn_sv(buffer, x[place_left:], y[place_left:], y_host[place_left:])

    def minority_positions(self, cur_y_host):
        """aser_utils.py:148-157: threshold ~ U(0, 1/num_class) from the CPU torch generator."""
        threshold = torch.tensor(1).float().uniform_(0, 1 / self.out_dim).item()
        self.last_threshold = threshold
        share = ClassBalancedRandomSampling.class_num_cache.astype(np.float32) / np.float32(self.mem_size)
        return np.flatnonzero(share[cur_y_host] < np.float32(threshold))

    def _update_by_knn_sv(self, buffer, cur_x, cur_y, cur_y_host):
        eng = engine_of(buffer.model)
        CB = ClassBalancedRandomSampling
        dev = cur_x.device
        n_cur = cur_x.size(0)
        minority = self.minority_positions(cur_y_host)
        eval_ind = CB.sample_indices(self.n_smp_cls)
        cand_ind = uniform_indices(buffer.current_index, self.n_total_smp, excl_indices=eval_ind)
        n_eval_buf, n_cand_buf = eval_ind.size, cand_ind.size
        self.last_choices = {'upd_eval_ind': eval_ind, 'upd_cand_ind': cand_ind, 'upd_threshold': self.last_threshold}
        # one batch [eval_buf | cand_buf | cur]; candidates = [cand_buf | cur] are contiguous rows
        batch = torch.empty((n_eval_buf + n_cand_buf + n_cur,) + tuple(cur_x.shape[1:]), dtype=torch.float32, device=dev)
        idx_t = to_device_i64(np.concatenate([eval_ind, cand_ind]), dev)
        ops.gather_rows(buffer.buffer_img, idx_t, out=batch)
        batch[n_eval_buf + n_cand_buf:].copy_(cur_x)
        feats = eng.features_eval(batch)
        cand_f = feats[n_eval_buf:]
        cand_y = to_device_i64(np.concatenate([buffer.labels_host[cand_ind], cur_y_host]), dev)
        if minority.size:
            rows = np.concatenate([np.arange(n_eval_buf), n_eval_buf + n_cand_buf + minority])
            eval_f = ops.gather_rows(feats, to_device_i64(rows, dev))
        else:
            eval_f = feats[:n_eval_buf]
        eval_y = to_device_i64(np.concatenate([buffer.labels_host[eval_ind], cur_y_host[minority]]), dev)
        sv_sum = ops.knn_sv(eval_f, eval_y, cand_f, cand_y, self.k, want_sum=True)['sum']
        order = ops.rank_desc(sv_sum)                                  # full descending ranking
        self.last_sv_sum = sv_sum                                      # kept for inspection (tests: tie analysis)
        buffer.n_seen_so_far += n_cur
        # The replacement itself (aser_update.py:88-112) happens on the device; the host mirror (labels,
        # class caches) follows from an asynchronous copy of the decision, applied the next time host-side
        # index logic runs -- the step has no device -> host synchronisation.
        cur_xc = cur_x.detach().to(torch.float32).contiguous()
        pairs = ops.aser_replace(order, n_cand_buf, idx_t[n_eval_buf:], cur_xc, cur_y, buffer.buffer_img, buffer.buffer_label)
        host = memory.pinned_i64(pairs.numel())
        host[:pairs.numel()].copy_(pairs, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        y_host = np.array(cur_y_host, dtype=np.int64, copy=True)
        out_dim = self.out_dim

        def apply():
            done.synchronize()
            arr = host[:1 + 2 * n_cur].numpy().copy()
            memory.release_pinned(host)
            cnt = int(arr[0])
            ind_cur, ind_buffer = arr[1:1 + cnt], arr[1 + n_cur:1 + n_cur + cnt]
            if cnt:
                CB._update_cache_now(buffer.buffer_label, out_dim, new_y=y_host[ind_cur], ind=ind_buffer)
                buffer._labels_host[ind_buffer] = y_host[ind_cur]
            self._last_decision = (ind_cur, ind_buffer)
        memory.defer(apply, owner=buffer)

    @property
    def last_decision(self):
        """(positions in the current batch, buffer slots they replaced) of the latest update."""
        memory.flush_pending()
        return self._last_decision


class GSSGreedyUpdate(object):
    """GSS-greedy (utils/buffer/gss_greedy_update.py:7-124) on the flat gradient arena.

    Every gradient the rule needs is one differentiable EVAL-mode pass of the engine
    (`b200ocl_net_forward_evalgrad` + `b200ocl_net_backward` with the eval-statistics bit: the reference switches the
    model to eval() before it differentiates it, gss_greedy_update.py:16) that leaves the gradient of all parameters,
    in parameters() order, in the engine's gradient arena -- the vector get_grad_vector() assembles tensor by tensor
    (buffer_utils.py:58-73).  The cosine similarities against the stored memory gradients and their maximum are one
    kernel (`b200ocl_grad_cosine`).  The random decisions are the reference's calls on the reference's generators:
    torch.randperm / the first torch.multinomial on the CPU generator, the replacement lottery on the generator of the
    scores' device."""

    SLOT = 5          # workspace slot of the engine that these passes use (the learners use 0, 1, 3)

    def __init__(self, params):
        super().__init__()
        self.mem_strength = params.gss_mem_strength
        self.gss_batch_size = params.gss_batch_size
        dev = 'cuda' if torch.cuda.is_available() else 'cpu'
        self.buffer_score = torch.zeros(params.mem_size, dtype=torch.float32, device=dev)
        self.last_batch_sim = None        # kept for inspection (tests: near-zero decisions)
        self.last_replaced = None

    def snapshot_parts(self):
        """The score of every slot, on the device."""
        return {'buffer_score': self.buffer_score}

    def snapshot(self):
        """The score of every slot, on the host."""
        return memory.host_tree(self.snapshot_parts())

    def restore(self, state):
        self.buffer_score.copy_(state['buffer_score'])

    # ---- one gradient: model.zero_grad(); F.cross_entropy(model.forward(x), y).backward()  (:80-83, :100-103, :117-119)
    def _gradient(self, eng, x, y):
        from .engine import ce_loss
        logits, ws = eng.forward_train(x, slot=self.SLOT, eval_stats=True)
        ce = ce_loss(logits, y, want_grad=True)
        eng.backward(x, ce['dlogits'], ws, eval_stats=True)
        return eng.state.grads

    def update(self, buffer, x, y, **kwargs):
        eng = engine_of(buffer.model)
        y_host = _host_labels(y, kwargs)
        buffer.model.eval()                                                     # :16
        x = x.detach().to(torch.float32).contiguous()
        self.last_replaced = None
        place_left = buffer.buffer_img.size(0) - buffer.current_index
        if place_left <= 0:                                                     # buffer is full (:22)
            batch_sim, mem_grads = self.get_batch_sim(buffer, eng, x, y)
            self.last_batch_sim = float(batch_sim)                              # the reference's `if batch_sim < 0` reads it too
            if self.last_batch_sim < 0:
                buffer_score = self.buffer_score[:buffer.current_index].cpu()
                buffer_sim = (buffer_score - torch.min(buffer_score)) / \
                             ((torch.max(buffer_score) - torch.min(buffer_score)) + 0.01)
                index = torch.multinomial(buffer_sim, x.size(0), replacement=False)          # CPU generator (:30)
                batch_item_sim = self.get_each_batch_sample_sim(buffer, eng, mem_grads, x, y)
                index_dev = index.to(self.buffer_score.device)
                scaled_batch_item_sim = ((batch_item_sim + 1) / 2).unsqueeze(1)
                buffer_repl_batch_sim = ((self.buffer_score[index_dev] + 1) / 2).unsqueeze(1)
                outcome = torch.multinomial(torch.cat((scaled_batch_item_sim, buffer_repl_batch_sim), dim=1), 1,
                                            replacement=False)                               # the scores' device generator (:38)
                sub = outcome.squeeze(1).bool().cpu().numpy()
                slots = index.numpy()[sub]
                src = np.flatnonzero(sub)
                self.last_replaced = (src, slots)
                if slots.size:
                    src_t = to_device_i64(src, x.device)
                    buffer.write(slots, ops.gather_rows(x, src_t) if x.is_cuda else x[src_t],
                                 ops.gather_rows(y, src_t) if y.is_cuda else y[src_t], y_host[src])
                    new_scores = ops.gather_rows(batch_item_sim, src_t) if batch_item_sim.is_cuda else batch_item_sim[src_t]
                    slots_t = to_device_i64(slots, self.buffer_score.device)
                    if self.buffer_score.is_cuda:
                        ops.scatter_rows(self.buffer_score, slots_t, new_scores)
                    else:
                        self.buffer_score[slots_t] = new_scores
        else:
            offset = min(place_left, x.size(0))
            x, y, y_host = x[:offset], y[:offset], y_host[:offset]
            if buffer.current_index == 0:                                       # first insertion (:52-53)
                batch_sample_memory_cos = torch.zeros(x.size(0)) + 0.1
            else:
                mem_grads = self.get_rand_mem_grads(buffer, eng)
                batch_sample_memory_cos = self.get_each_batch_sample_sim(buffer, eng, mem_grads, x, y)
            s, e = buffer.current_index, buffer.current_index + offset
            buffer.buffer_img[s:e].copy_(x)
            buffer.buffer_label[s:e].copy_(y)
            buffer.labels_host[s:e] = y_host
            self.buffer_score[s:e].copy_(batch_sample_memory_cos)
            buffer.current_index += offset
        buffer.model.train()                                                    # :64

    def get_batch_sim(self, buffer, eng, batch_x, batch_y):
        """(score of the incoming batch [1], memory gradients [K, n_params])  (:66-85)."""
        mem_grads = self.get_rand_mem_grads(buffer, eng)
        g = self._gradient(eng, batch_x, batch_y)
        _, batch_sim = ops.grad_cosine(mem_grads, g)
        return batch_sim, mem_grads

    def get_rand_mem_grads(self, buffer, eng):
        """Gradients of num_mem_subs random memory minibatches (:87-107)."""
        gss_batch_size = min(self.gss_batch_size, buffer.current_index)
        num_mem_subs = min(self.mem_strength, buffer.current_index // gss_batch_size)
        if num_mem_subs > ops.GRAD_COSINE_MAX_K:
            raise ValueError('gss_mem_strength %d exceeds the kernel limit %d' % (num_mem_subs, ops.GRAD_COSINE_MAX_K))
        mem_grads = torch.zeros((num_mem_subs, eng.info.n_params), dtype=torch.float32, device=eng.device)
        shuffeled_inds = torch.randperm(buffer.current_index).numpy()            # CPU generator (:98)
        for i in range(num_mem_subs):
            bx, by, _ = buffer.gather(shuffeled_inds[i * gss_batch_size:i * gss_batch_size + gss_batch_size])
            mem_grads[i].copy_(self._gradient(eng, bx, by))
        return mem_grads

    def get_each_batch_sample_sim(self, buffer, eng, mem_grads, batch_x, batch_y):
        """Score of every sample of the batch: the largest cosine similarity of its own gradient with the memory
        gradients (:109-124)."""
        n = batch_x.size(0)
        cosine_sim = torch.zeros(n, dtype=torch.float32, device=eng.device)
        for i in range(n):
            g = self._gradient(eng, batch_x[i:i + 1], batch_y[i:i + 1])
            ops.grad_cosine(mem_grads, g, max_out=cosine_sim[i:i + 1])
        return cosine_sim
