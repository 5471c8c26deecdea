# -*-coding:utf-8 -*-
"""Train ops with the reference's surface (reference tools/train_utils.py:246-390), run as fused
kernels over ONE flat fp32 buffer per state (params / grads / m / v):

  custom_train_op(loss, init_lr, step_per_epoch, decay_rate)   tf.train.AdamOptimizer + staircase
        exponential decay + clip_by_value(+-5)                  (reference :340-350, 365-390)
  bert_train_op(loss, init_lr, num_train_steps, warmup_ratio, diff_lr_times)
        AdamWeightDecayOptimizer per LR group + clip_by_global_norm(1.0)   (reference :246-337)

Data parallel: gradients live in one contiguous buffer, so a step issues exactly ONE NCCL
all-reduce (SURVEY.md §8e); the 1/world scaling is folded into the optimizer kernel.
"""
import ctypes
import re

import torch

from .. import ops, variables


class FlatState:
    """Re-homes every trainable variable (and its gradient) as a view of one flat buffer."""

    def __init__(self, store, group_of=None):
        self.store = store
        names = store.trainable_names()
        group_of = group_of or (lambda n: 0)
        # stable: groups become contiguous ranges; inside a group the BertModel variables follow the order in which the
        # backward pass completes them (encoder layer 11 first ... layer 0, embeddings last), so that the gradients of a
        # few consecutive layers are ONE contiguous slice — a bucket of the overlapped data-parallel exchange
        names.sort(key=lambda n: (group_of(n), _backward_order(n)))
        self.names = names
        self.group_ranges = {}                                # group -> [start, end)
        ALIGN = 64   # floats: every variable starts 256-byte aligned (TMA / 16-byte vector accesses on grads)
        pad = lambda k: (k + ALIGN - 1) // ALIGN * ALIGN
        total = sum(pad(store.vars[n].numel()) for n in names)
        dev = store.device
        self.params = torch.zeros(total, dtype=torch.float32, device=dev)
        self.grads = torch.zeros(total, dtype=torch.float32, device=dev)
        self.m = torch.zeros(total, dtype=torch.float32, device=dev)
        self.v = torch.zeros(total, dtype=torch.float32, device=dev)
        self.slices = {}
        off = 0
        for n in names:
            t = store.vars[n]
            k = t.numel()
            self.params[off:off + k].copy_(t.reshape(-1))
            store.vars[n] = self.params[off:off + k].view(t.shape)
            g_old = store.grads.get(n)
            store.grads[n] = self.grads[off:off + k].view(t.shape)
            if g_old is not None:
                store.grads[n].copy_(g_old)
            self.slices[n] = (off, off + k)
            g = group_of(n)
            s, e = self.group_ranges.get(g, (off, off))
            self.group_ranges[g] = (min(s, off), off + pad(k))
            off += pad(k)
        store.touch()
        # optimizer slots restored from a checkpoint before this buffer existed, or carried over from the buffer this one
        # replaces (the trainable set changed): Adam moments survive by variable name
        slots = getattr(store, "_slot_init", None)
        if slots:
            self.load_slots(slots)
            store._slot_init = None

    def slot_dict(self):
        """name -> (m, v) views, for checkpoints (TF checkpoints carry `<var>/adam_m`, `<var>/adam_v`)."""
        return {n: (self.m[s:e].view(self.store.vars[n].shape), self.v[s:e].view(self.store.vars[n].shape))
                for n, (s, e) in self.slices.items()}

    def load_slots(self, slots):
        for n, (m, v) in slots.items():
            if n in self.slices:
                s, e = self.slices[n]
                self.m[s:e].copy_(torch.as_tensor(m, dtype=torch.float32).reshape(-1))
                self.v[s:e].copy_(torch.as_tensor(v, dtype=torch.float32).reshape(-1))

    def zero_grads(self):
        self.grads.zero_()


_LAYER_RE = re.compile(r'encoder/layer_(\d+)/')


def _backward_order(name):
    m = _LAYER_RE.search(name)
    if m:
        return (0, -int(m.group(1)))
    return (1, 0) if '/embeddings/' in name else (0, -10 ** 6)


class GradExchange(object):
    """The data-parallel gradient exchange of one TRAIN step, overlapped with the backward pass (SURVEY 8e).

    The reference is single device; this engine shards sentences over ranks and sums gradients.  Instead of one
    all-reduce after the whole backward, the flat gradient buffer (laid out in backward-completion order, FlatState) is
    cut into contiguous buckets — the dense kernels of each encoder layer, 11 first ... 0, then the rest (embeddings,
    LayerNorm / bias ranges, the layers above BertModel) — and a layer bucket is all-reduced on a side stream as soon as the event recorded behind its last
    gradient kernel has fired (ner_bert_train_bwd_set_layer_events), while the layers below are still being differentiated.
    dtype 'bf16': a bucket travels as bf16 (half the NVLink bytes: cast, all-reduce, cast back on the side stream); the
    global-norm clip and Adam read the fp32 buffer either way."""

    LAYERS_PER_BUCKET = 1      # one encoder layer (28 MB of fp32 gradients) per all-reduce: the exposed tail is the last layer + embeddings

    def __init__(self, fs, dtype='fp32'):
        self.fs, self.dtype = fs, dtype
        # highest priority: the all-reduce kernels take SM slots as soon as CTAs of the (persistent, all-SM) backward GEMMs retire
        self.comm = torch.cuda.Stream(priority=-1)
        self.tail_event = torch.cuda.Event()
        layers = sorted({int(m.group(1)) for n in fs.names for m in [_LAYER_RE.search(n)] if m})
        self.num_layers = (max(layers) + 1) if layers else 0
        self.layer_events = [torch.cuda.Event() for _ in range(self.num_layers)]
        for ev in [self.tail_event] + self.layer_events:
            ev.record()                                  # materialise the handles
        self._handles = (ctypes.c_void_p * max(self.num_layers, 1))(*[ev.cuda_event for ev in self.layer_events])
        self.armed = False
        # buckets: maximal runs of consecutive variables with the same readiness key, in flat-buffer order.  A key is
        # ('layer', g) for the dense kernels of encoder layers [NL-1-3g .. NL-3-3g] — ready when the lowest of them is
        # differentiated — and ('tail',) for everything else (embeddings, LayerNorm / bias ranges, the variables of the
        # layers above BertModel): reduced once the whole backward pass is enqueued.
        runs = []
        for n in fs.names:
            m = _LAYER_RE.search(n)
            if m and n.startswith('bert/') and _decays(n):
                key = ('layer', (self.num_layers - 1 - int(m.group(1))) // self.LAYERS_PER_BUCKET)
            else:
                key = ('tail',)
            s, e = fs.slices[n]
            if runs and runs[-1][0] == key:
                runs[-1][2] = e
            else:
                runs.append([key, s, e])
        total = fs.grads.numel()
        self.buckets = []
        for i, (key, s, e) in enumerate(runs):
            end = runs[i + 1][1] if i + 1 < len(runs) else total           # cover the alignment padding up to the next run
            if key[0] == 'layer':
                lowest = max(self.num_layers - (key[1] + 1) * self.LAYERS_PER_BUCKET, 0)     # last layer of the group to finish
                ev = self.layer_events[lowest]
            else:
                ev = self.tail_event
            self.buckets.append((key, s, end, ev))
        self.buckets.sort(key=lambda b: (b[0][0] != 'layer', b[0][1] if b[0][0] == 'layer' else 0, b[1]))   # readiness order
        self._stage = torch.empty(max(e - s for _, s, e, _ in self.buckets), dtype=torch.bfloat16,
                                  device=fs.grads.device) if dtype == 'bf16' else None

    # -- called from the BertModel backward closure (bert.py) around the C composite
    def before_bert_backward(self):
        from .. import _lib
        _lib.lib().ner_bert_train_bwd_set_layer_events(self._handles, self.num_layers)
        self.armed = True

    def after_bert_backward(self):
        from .. import _lib
        _lib.lib().ner_bert_train_bwd_set_layer_events(None, 0)

    def finish(self):
        """Enqueue the bucket all-reduces (each behind its readiness event) and make the caller's stream wait for them.
        -> world size."""
        import torch.distributed as dist
        world = dist.get_world_size()
        main = torch.cuda.current_stream()
        self.tail_event.record(main)
        if not self.armed:                       # no BertModel backward ran in this step: nothing was recorded
            for ev in self.layer_events:
                ev.record(main)
        with torch.cuda.stream(self.comm):
            for key, s, e, ev in self.buckets:
                self.comm.wait_event(ev)
                piece = self.fs.grads[s:e]
                if self._stage is not None:
                    half = self._stage[:e - s]
                    half.copy_(piece)
                    dist.all_reduce(half, op=dist.ReduceOp.SUM)
                    piece.copy_(half)
                else:
                    dist.all_reduce(piece, op=dist.ReduceOp.SUM)
        main.wait_stream(self.comm)
        self.armed = False
        return world


def _flat(store, group_of=None):
    fs = getattr(store, "_flat_state", None)
    if fs is None or set(fs.names) != set(store.trainable_names()):
        if fs is not None:
            store._slot_init = {n: (m.clone(), v.clone()) for n, (m, v) in fs.slot_dict().items()}
        fs = FlatState(store, group_of)
        store._flat_state = fs
    return fs


def allreduce_gradients(flat_grads):
    """The single data-parallel exchange of a step: sum of the flat gradient buffer over ranks."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(flat_grads, op=dist.ReduceOp.SUM)
        return dist.get_world_size()
    return 1


def exchange_gradients(store, fs):
    """Bucketed, backward-overlapped exchange when the step armed one (GradExchange), else the single all-reduce.  The
    exchange object is created here on the first multi-rank step — FlatState exists only after the first backward — and
    the BertModel backward closure of the following steps finds it at `store._grad_exchange`."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        return 1
    mode = getattr(store, 'grad_exchange', 'overlap')          # 'overlap' | 'overlap_bf16' | 'single'
    if mode == 'skip':                                          # timing diagnostic only: the step without its exchange
        return dist.get_world_size()
    if mode == 'single' or not fs.grads.is_cuda:
        return allreduce_gradients(fs.grads)
    ex = getattr(store, '_grad_exchange', None)
    if ex is None or ex.fs is not fs:
        ex = store._grad_exchange = GradExchange(fs, 'bf16' if mode == 'overlap_bf16' else 'fp32')
    return ex.finish()


def lr_decay(init_lr, global_step, step_per_epoch, decay_rate):
    """tf.train.exponential_decay(..., staircase=True) (reference :365-376)."""
    return init_lr * decay_rate ** (global_step // max(int(step_per_epoch), 1))


def custom_train_op(loss, init_lr, step_per_epoch, decay_rate, store=None):
    """Adam + exponential LR decay + clip_by_value(-5, 5) (reference :340-350, 378-390)."""
    store = store or variables.default_store()
    fs = _flat(store)
    world = allreduce_gradients(fs.grads)
    t = store.global_step + 1
    lr = lr_decay(init_lr, store.global_step, step_per_epoch, decay_rate)
    b1, b2 = 0.9, 0.999
    lr_t = lr * (1 - b2 ** t) ** 0.5 / (1 - b1 ** t)
    ops.adam_step(fs.params, fs.grads, fs.m, fs.v, lr=lr_t, beta1=b1, beta2=b2, eps=1e-8, mode=1, clip=5.0,
                  grad_scale=1.0 / world)
    store.global_step += 1
    store.touch()
    fs.zero_grads()
    return lr


def bert_lr(init_lr, global_step, num_train_steps, num_warmup_steps):
    """create_optimizer's schedule (reference :252-274): linear warm-up, then linear decay to 0."""
    lr = init_lr * max(0.0, 1.0 - min(global_step, num_train_steps) / float(num_train_steps))
    if num_warmup_steps and global_step < num_warmup_steps:
        lr = init_lr * global_step / float(num_warmup_steps)
    return lr


def bert_train_op(loss, init_lr, num_train_steps, warmup_ratio, diff_lr_times, verbose=False, store=None):
    """AdamWeightDecayOptimizer with per-scope LR multipliers + clip_by_global_norm(1.0) (reference :287-337).

    Groups are matched by substring of the variable name exactly like the reference (:300-303);
    weight decay skips names containing LayerNorm / layer_norm / bias (:276-282)."""
    store = store or variables.default_store()
    keys = list((diff_lr_times or {}).keys())

    def group_of(name):
        for gi, k in enumerate(keys):
            if k in name:
                return (gi, 0 if _decays(name) else 1)
        return (len(keys), 0 if _decays(name) else 1)

    fs = _flat(store, group_of)
    world = exchange_gradients(store, fs)
    gsq = torch.zeros(1, dtype=torch.float32, device=fs.grads.device)
    ops.sumsq_add(fs.grads, gsq)
    num_warmup = int(num_train_steps * warmup_ratio)
    lrs = {}
    for g, (s, e) in fs.group_ranges.items():
        gi, nodecay = g
        mult = diff_lr_times[keys[gi]] if gi < len(keys) else 1
        lr = bert_lr(init_lr * mult, store.global_step, num_train_steps, num_warmup)
        lrs[g] = lr
        ops.adam_step(fs.params[s:e], fs.grads[s:e], fs.m[s:e], fs.v[s:e], lr=lr, beta1=0.9, beta2=0.999, eps=1e-6,
                      weight_decay=0.0 if nodecay else 0.01, mode=0, clip=1.0, gnorm_sq=gsq, grad_scale=1.0 / world)
    store.global_step += 1
    store.touch()
    fs.zero_grads()
    return lrs


def noam_scheme(init_lr, global_step, warmup_steps=4000.):
    """reference tools/transformer/modules.py:209-217: lr rises linearly to init_lr over warmup_steps, then ~ step^-0.5."""
    step = float(global_step + 1)
    if warmup_steps <= 0:      # runs shorter than 1/warmup_ratio steps: the factor warmup_steps ** 0.5 is 0 (the reference's
        return 0.0             # Python-side 0 ** -1.5 raises while building the graph; lr = 0 is the limit it stands for)
    return init_lr * warmup_steps ** 0.5 * min(step * warmup_steps ** -1.5, step ** -0.5)


def transformer_train_op(loss, init_lr, num_train_steps, warmup_ratio, store=None):
    """tf.train.AdamOptimizer(noam_scheme(...)).minimize(loss) (reference :353-362) — plain Adam, no clipping."""
    store = store or variables.default_store()
    fs = _flat(store)
    world = allreduce_gradients(fs.grads)
    lr = noam_scheme(init_lr, store.global_step, int(num_train_steps * warmup_ratio))
    t = store.global_step + 1
    b1, b2 = 0.9, 0.999
    lr_t = lr * (1 - b2 ** t) ** 0.5 / (1 - b1 ** t)
    ops.adam_step(fs.params, fs.grads, fs.m, fs.v, lr=lr_t, beta1=b1, beta2=b2, eps=1e-8, mode=1, clip=0.0,
                  grad_scale=1.0 / world)
    store.global_step += 1
    store.touch()
    fs.zero_grads()
    return lr


def _decays(name):
    return not any(tok in name for tok in ("LayerNorm", "layer_norm", "bias"))


def load_bert_checkpoint(pretrain_dir, store=None):
    """reference tools/train_utils.py:91-102 (kept at the reference's location; the reader lives in bert.py)."""
    from ..bert import load_bert_checkpoint as _load
    return _load(pretrain_dir, store)
