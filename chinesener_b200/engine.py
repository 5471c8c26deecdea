"""model_fn-equivalent glue: picks a plugin by name and runs PREDICT / EVAL steps.

Mirrors reference tools/train_utils.py:145-187 (build_model_fn): the plugin is looked up by
`importlib` under `model.<name>`, called as build_graph(features, labels, params, is_training)
and its PREDICT output dict carries the keys 'pred_ids', 'label_ids', 'tokens'
(tools/train_utils.py:181-185).  Host batches come in as (pinned) CPU tensors and are copied
to the device inside `predict` — that copy is part of the end-to-end number bench.py reports.
"""
import contextlib
import importlib

import numpy as np
import torch

from . import autodiff, variables

_DEVICE_KEYS = ('token_ids', 'mask', 'segment_ids', 'label_ids', 'seq_len', 'softlexicon_ids', 'softlexicon_weights',
                'bichar_ids', 'softword_ids', 'ex_softword_ids', 'task_ids', 'lattice_ids', 'lattice_lens', 'label_mask')


# Plugins that refuse params['crf_nbest'] > 1, with the reason (checked by Estimator.crf_nbest before anything is launched)
NBEST_REFUSED = {
    'bert_ce': "it has no CRF: its tags are a per-token argmax",
    'bert_dice': "it has no CRF: its tags are a per-token argmax",
    'bert_mrc': "it has no CRF: its tags come from per-type span pointers",
    'bert_mrc_span': "it has no CRF: its tags come from span scores",
    'bert_global_pointer': "it has no CRF: its tags come from span scores",
    'bert_bilstm_crf_mtl': "its pred_ids are a per-task selection of several CRF decodes",
    'bert_bilstm_crf_adv': "its pred_ids are a per-task selection of several CRF decodes",
}
NBEST_MAX = 16
# The CRF kernels take up to 128 tags (ner_crf_wide_*), but N-best decoding, the partial-label loss (a 32-bit mask of
# allowed tags), distillation and the token heads of these plugins stop at 32: past that, Estimator refuses them.
NARROW_TAGS = 32
WIDE_TAGS_REFUSED = {
    'bert_ce': "its fused cross-entropy kernel takes at most 32 tags",
    'bert_dice': "its fused Dice-loss kernel takes at most 32 tags",
}


def load_plugin(model_name):
    mod = importlib.import_module(f'{__package__}.model.{model_name}')
    return getattr(mod, 'build_graph'), getattr(mod, 'TRAIN_PARAMS')


class Estimator:
    """Minimal stand-in for tf.estimator.Estimator over one plugin + one variable store."""

    def __init__(self, model_name, params, store=None, device='cuda', teacher=None):
        self.model_name = model_name
        self.build_graph, train_params = load_plugin(model_name)
        self.params = dict(train_params)
        self.params.update(params)
        self.device = torch.device(device)
        self.teacher = teacher
        self.tag_set_limits()
        if teacher is not None:
            self.distill_settings()
        if self.params.get('augment'):
            from . import augment
            augment.check_estimator(self)
        self.store = store or variables.VariableStore(self.device)
        # data-parallel gradient exchange (N > 1): 'overlap' = bucketed all-reduces behind the backward pass, 'overlap_bf16' =
        # the same with bf16 buckets, 'single' = one all-reduce of the flat buffer after the backward pass
        self.store.grad_exchange = self.params.get('grad_exchange', 'overlap')

    def to_device(self, features):
        out = {}
        for k, v in features.items():
            if k in _DEVICE_KEYS and torch.is_tensor(v):
                out[k] = v.to(self.device, non_blocking=True)
            else:
                out[k] = v
        m = features.get('mask')
        if torch.is_tensor(m) and not m.is_cuda and 'mask' in out:
            # host-side token count rides along so sequence packing needs no device sync; the count of non-empty rows
            # sizes the query/context pairs of bert_mrc the same way, and the per-row lengths the windows of document mode
            lens = m.sum(1)
            out['mask'].row_lengths = lens.numpy()
            out['mask'].total_tokens = int(lens.sum())
            out['mask'].nonempty_rows = int((lens > 0).sum())
        return out

    def predict_device(self, dev_features):
        """PREDICT on device-resident features -> pred_ids (device).  One fused C call when the plugin has an
        executor in fastpath.FUSED_PREDICT (same kernels as build_graph, see fastpath.py), else build_graph.  A
        `label_mask` (partial labels) is dropped: decoding does not read labels."""
        if 'label_mask' in dev_features:
            dev_features = {k: v for k, v in dev_features.items() if k != 'label_mask'}
        self.crf_nbest()
        if self.params.get('fused_predict', True):
            from . import fastpath
            fn = fastpath.FUSED_PREDICT.get(self.model_name)
            if fn is not None:
                with variables.use_store(self.store):
                    pred = fn(self, dev_features)
                if pred is not None:
                    return pred
        return self.forward_device(dev_features, False)[1]      # multi-task plugins return (loss, pred_ids, task_ids)

    def document_window(self):
        """-> (W, S) of the BERT plugins' document mode from params['bert_window'] / ['bert_window_stride'] (ValueError when
        out of range), None for a plugin without BERT."""
        if 'bert' not in self.model_name:
            return None
        from . import bert, windows
        max_pos = bert.load_bert_config(self.params.get('pretrain_dir', ''))["max_position_embeddings"]
        return windows.settings(self.params.get('bert_window'), self.params.get('bert_window_stride'), max_pos)

    def label_size(self):
        K = self.params.get('label_size')
        return int(K) if isinstance(K, (int, np.integer)) and not isinstance(K, bool) else 0

    def tag_set_limits(self, features=None):
        """ValueError, before anything is launched, for what does not run past 32 tags: the plugins in
        WIDE_TAGS_REFUSED, and a batch with a `label_mask` (partial labels).  N-best decoding and distillation are
        refused by crf_nbest and distill_settings."""
        K = self.label_size()
        if K <= NARROW_TAGS:
            return
        if self.model_name in WIDE_TAGS_REFUSED:
            raise ValueError(f"{self.model_name} cannot run label_size = {K} tags: {WIDE_TAGS_REFUSED[self.model_name]}")
        if features is not None and features.get('label_mask') is not None:
            raise ValueError(f"partial labels (label_mask) take at most {NARROW_TAGS} tags, a 32-bit mask of allowed "
                             f"tags; this tag set has label_size = {K}")

    def crf_nbest(self):
        """params['crf_nbest'] (default 1): how many best CRF paths PREDICT / EVAL decode.  ValueError outside
        1..NBEST_MAX, or above 1 for a plugin in NBEST_REFUSED."""
        n = self.params.get('crf_nbest', 1)
        if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or not 1 <= n <= NBEST_MAX:
            raise ValueError(f"crf_nbest must be an integer in 1..{NBEST_MAX} (got {n!r})")
        if n > 1 and self.model_name in NBEST_REFUSED:
            raise ValueError(f"{self.model_name} cannot decode crf_nbest = {n} paths: {NBEST_REFUSED[self.model_name]}")
        if n > 1 and self.label_size() > NARROW_TAGS:
            raise ValueError(f"crf_nbest = {n} takes at most {NARROW_TAGS} tags; this tag set has label_size = "
                             f"{self.label_size()}")
        return int(n)

    def distill_settings(self):
        """(alpha, tau) of knowledge distillation from self.teacher: params['distill_alpha'] in (0, 1] (default 0.5) and
        params['distill_temperature'] > 0 (default 1).  ValueError, before anything is launched, for a teacher or
        student without exactly one CRF, different tag sets, different tokenizers, or a student word-enhance method
        other than none or the teacher's own: the two CRFs must score the same tags at the same positions."""
        from .data.base_preprocess import extract_prefix_surfix
        t = self.teacher
        if self.label_size() > NARROW_TAGS:
            raise ValueError(f"distillation takes at most {NARROW_TAGS} tags; this tag set has label_size = "
                             f"{self.label_size()}")
        for who, name in (("teacher", t.model_name), ("student", self.model_name)):
            if name in NBEST_REFUSED:
                raise ValueError(f"cannot distill with {who} {name}: {NBEST_REFUSED[name]}")
        for key in ('label_size', 'idx2tag'):
            if t.params.get(key) != self.params.get(key):
                raise ValueError(f"teacher {t.model_name} and student {self.model_name} have a different {key}")
        t_we, t_tok = extract_prefix_surfix(t.model_name)
        s_we, s_tok = extract_prefix_surfix(self.model_name)
        if t_tok != s_tok:
            raise ValueError(f"teacher {t.model_name} ({t_tok} tokenizer) and student {self.model_name} ({s_tok} "
                             f"tokenizer) do not tag the same positions")
        if s_we is not None and s_we != t_we:
            raise ValueError(f"student {self.model_name} needs {s_we} features, which teacher {t.model_name}'s "
                             f"dataset does not carry")
        a = self.params.get('distill_alpha', 0.5)
        tau = self.params.get('distill_temperature', 1.0)
        if isinstance(a, bool) or not isinstance(a, (int, float, np.number)) or not 0 < a <= 1:
            raise ValueError(f"distill_alpha must be in (0, 1] (got {a!r})")
        if isinstance(tau, bool) or not isinstance(tau, (int, float, np.number)) or not 0 < tau < float('inf'):
            raise ValueError(f"distill_temperature must be > 0 (got {tau!r})")
        return float(a), float(tau)

    def teacher_potentials(self, dev_features):
        """The teacher's PREDICT-mode emissions [B,L,K] and CRF transitions on a device batch (its `label_mask`
        dropped, nothing decoded).  The teacher's store is only read."""
        from .tools import layer
        feats = {k: v for k, v in dev_features.items() if k != 'label_mask'}
        saved = layer.CRF_CAPTURE
        layer.CRF_CAPTURE = captured = []
        try:
            self.teacher.forward_device(feats, False)
        finally:
            layer.CRF_CAPTURE = saved
        if len(captured) != 1:
            raise ValueError(f"teacher {self.teacher.model_name} ran {len(captured)} CRF layers, not one")
        return captured[0]

    @contextlib.contextmanager
    def _layer_settings(self, dev_features):
        """The module settings of tools/layer.py this Estimator's params select, checked before anything is launched."""
        from . import windows
        from .tools import layer
        nbest = self.crf_nbest()
        self.tag_set_limits(dev_features)
        ws = self.document_window()
        if ws is not None and torch.is_tensor(dev_features.get('token_ids')):
            windows.check_batch(self.model_name, dev_features['token_ids'].shape[1], ws[0])
        keys = ('BERT_PRECISION', 'BERT_WINDOW', 'BERT_WINDOW_STRIDE', 'DOCUMENT_REFUSAL', 'CRF_NBEST', 'CRF_TEACHER')
        saved = {k: getattr(layer, k) for k in keys}
        layer.BERT_PRECISION = self.params.get('bert_precision', saved['BERT_PRECISION'])
        layer.CRF_NBEST = nbest
        if ws is not None:
            layer.BERT_WINDOW, layer.BERT_WINDOW_STRIDE = ws
            if self.model_name in windows.REFUSED:
                layer.DOCUMENT_REFUSAL = (f"{self.model_name} cannot run BERT over sequences longer than bert_window = {ws[0]}: "
                                          f"{windows.REFUSED[self.model_name]}")
        try:
            yield
        finally:
            for k, v in saved.items():
                setattr(layer, k, v)

    def forward_device(self, dev_features, is_training=False):
        with self._layer_settings(dev_features), variables.use_store(self.store):
            return self.build_graph(dev_features, None, self.params, is_training)

    def predict(self, features):
        """PREDICT mode on one host batch -> dict(pred_ids int32 [B,L] on host, label_ids, tokens), and 'pred_spans' (per
        sentence a list of (type name, start, end_exclusive, probability)) when the plugin's pred_ids carries spans, and
        'pred_nbest' (per sentence a list of (tags int32 [L], score, probability), best first, empty for seq_len <= 0) when
        params['crf_nbest'] > 1."""
        dev = self.to_device(features)
        pred_ids = self.predict_device(dev)
        out = {'pred_ids': pred_ids.cpu(), 'label_ids': features.get('label_ids'), 'tokens': features.get('tokens')}
        from .tools.infer_utils import nbest_lists, span_lists
        spans = span_lists(pred_ids)
        if spans is not None:
            out['pred_spans'] = spans
        nbest = nbest_lists(pred_ids, features['seq_len']) if 'seq_len' in features else None
        if nbest is not None:
            out['pred_nbest'] = nbest
        return out

    def stack_to_device(self, feature_list):
        """Several host batches -> ONE device batch (rows concatenated in order): every device feature is allocated once
        at the summed batch size and each host part is copied straight into its row slice (pinned -> non-blocking)."""
        if len(feature_list) == 1:
            return self.to_device(feature_list[0])
        out = {}
        first = feature_list[0]
        for k, v in first.items():
            if k in _DEVICE_KEYS and torch.is_tensor(v):
                rows = sum(f[k].shape[0] for f in feature_list)
                dst = torch.empty((rows,) + tuple(v.shape[1:]), dtype=v.dtype, device=self.device)
                r = 0
                for f in feature_list:
                    n = f[k].shape[0]
                    dst[r:r + n].copy_(f[k], non_blocking=True)
                    r += n
                out[k] = dst
        lens = []
        for f in feature_list:
            m = f.get('mask')
            if not (torch.is_tensor(m) and not m.is_cuda):
                lens = None
                break
            lens.append(m.sum(1))
        if lens is not None and 'mask' in out:
            lens = torch.cat(lens)
            out['mask'].row_lengths = lens.numpy()
            out['mask'].total_tokens = int(lens.sum())
            out['mask'].nonempty_rows = int((lens > 0).sum())
        return out

    def predict_iter(self, batches, depth=2, streams=1, group=1):
        """Generator form of PREDICT — the shape of tf.estimator.Estimator.predict(input_fn), which the
        reference drives at main.py:52-55: yields one result dict per host batch, in order.  The device work
        of up to `depth` calls is in flight before the oldest result is awaited, so the host->device copy
        of batch i+1 and the enqueue of its kernels overlap batch i on the GPU; results come back through
        a small ring of pinned host buffers.
        streams > 1: consecutive calls run on different CUDA streams (sentences are independent, SURVEY
        8(e)), so the SMs a kernel of one call leaves idle are taken by the other call's kernels.
        group > 1: `group` consecutive host batches are stacked into one device batch per call (sentences are
        independent, so the tags are those of the separate calls): the packed token count of a 64-sentence MSRA batch
        (~3.2 k rows) fills 0.6 / 1.7 / 2.3 waves of 128x256 GEMM tiles on 132 SMs, two batches (~6.3 k rows) fill
        1.1 / 3.4 / 4.5 — the tensor-core tiles stop idling in partial waves without relying on stream overlap."""
        from . import ops
        ring, inflight = {}, []
        depth = max(depth, streams + 1) if streams > 1 else depth
        side = [torch.cuda.Stream() for _ in range(streams)] if streams > 1 else None
        if side is not None:
            torch.cuda.synchronize()          # weight packs / caches built on the caller's stream are complete

        def finish(item):
            ev, buf, feats_list = item
            ev.synchronize()
            r = 0
            for feats in feats_list:
                n = feats['token_ids'].shape[0] if torch.is_tensor(feats.get('token_ids')) else buf.shape[0]
                yield {'pred_ids': buf[r:r + n].clone(), 'label_ids': feats.get('label_ids'), 'tokens': feats.get('tokens')}
                r += n

        def grouped(it):
            cur = []
            for f in it:
                cur.append(f)
                if len(cur) == group:
                    yield cur
                    cur = []
            if cur:
                yield cur

        # streams > 1: the host->device copies of a call run on their own stream, so the inputs of call k+1 travel while the
        # compute streams are busy with calls k-1 / k (a compute stream that copies its own inputs idles for the ~20 small
        # transfers of a stacked call)
        copy_stream = torch.cuda.Stream() if side is not None else None
        k = 0
        for feats_list in grouped(batches):
            ctx = torch.cuda.stream(side[k % streams]) if side is not None else contextlib.nullcontext()
            if copy_stream is not None:
                with torch.cuda.stream(copy_stream):
                    dev = self.stack_to_device(feats_list)
                    copied = torch.cuda.Event()
                    copied.record()
            with ctx:
                if copy_stream is not None:
                    st = side[k % streams]
                    st.wait_event(copied)
                    for t in dev.values():
                        if torch.is_tensor(t) and t.is_cuda:
                            t.record_stream(st)          # allocated on the copy stream, consumed here
                else:
                    dev = self.stack_to_device(feats_list)
                tile0 = ops.DEFAULT_TILE
                if side is not None or group > 1:   # partial waves are filled (other streams / 2x rows): take the fastest tile
                    ops.DEFAULT_TILE = ops.TILE_AUTO_THROUGHPUT
                try:
                    pred_ids = self.predict_device(dev)
                finally:
                    ops.DEFAULT_TILE = tile0
                key = (tuple(pred_ids.shape), k % (depth + 1))
                buf = ring.get(key)
                if buf is None:
                    buf = ring[key] = torch.empty(pred_ids.shape, dtype=pred_ids.dtype, pin_memory=True)
                buf.copy_(pred_ids, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record()
            inflight.append((ev, buf, feats_list))
            k += 1
            if len(inflight) >= depth:
                yield from finish(inflight.pop(0))
        while inflight:
            yield from finish(inflight.pop(0))
        if side is not None:
            for st in side:
                torch.cuda.current_stream().wait_stream(st)

    def predict_sentences(self, batches, depth=2, streams=1, group=1):
        """tf.estimator.Estimator.predict(input_fn) as the reference consumes it (main.py:52-55, evaluation.py:16-24):
        one dict PER SENTENCE — {'pred_ids': int32 [L], 'label_ids': int32 [L], 'tokens': [L]} as numpy arrays / lists —
        the element type of `<model>_predict.pkl` and the input of evaluation.SingleEval.  (predict / predict_iter yield
        one dict per batch.)"""
        for out in self.predict_iter(batches, depth=depth, streams=streams, group=group):
            pred = out['pred_ids'].numpy()
            lab = out['label_ids'].numpy() if torch.is_tensor(out['label_ids']) else out['label_ids']
            tok = out['tokens']
            for b in range(pred.shape[0]):
                yield {'pred_ids': pred[b], 'label_ids': None if lab is None else lab[b], 'tokens': None if tok is None else tok[b]}

    def train_step(self, features):
        """TRAIN mode of model_fn (reference tools/train_utils.py:151-168): forward with the tape,
        backward, then the train op the reference picks by model name (:156-164).  -> loss (float)."""
        from .tools import train_utils
        self.tag_set_limits(features)
        dev = features if all(not torch.is_tensor(v) or v.is_cuda for v in features.values()) else self.to_device(features)
        teacher = None
        if self.teacher is not None:
            teacher = self.teacher_potentials(dev) + self.distill_settings()
        self.store.dropout_calls = 0
        with self._layer_settings(dev), variables.use_store(self.store), autodiff.recording(self.store) as tape:
            from .tools import layer
            layer.CRF_TEACHER = teacher
            loss = self.build_graph(dev, None, self.params, True)[0]
            tape.backward()
            p = self.params
            if 'bert' in self.model_name:
                train_utils.bert_train_op(loss, p['lr'], p['num_train_steps'], p['warmup_ratio'], p['diff_lr_times'])
            elif 'transformer' in self.model_name:
                train_utils.transformer_train_op(loss, p['lr'], p['num_train_steps'], p['warmup_ratio'])
            else:
                train_utils.custom_train_op(loss, p['lr'], p['step_per_epoch'], p['decay_rate'])
        return loss

    def evaluate(self, features):
        dev = self.to_device(features)
        loss, pred_ids = self.forward_device(dev, False)[:2]
        return {'loss': float(loss), 'pred_ids': pred_ids.cpu()}
