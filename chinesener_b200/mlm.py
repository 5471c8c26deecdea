"""BERT's masked-LM head and loss (google-research/bert run_pretraining.py, get_masked_lm_output) on the variable store,
under its TF variable names, for continued (domain-adaptive) pretraining: dynamic whole-word masking on the device
(ner_mlm_mask), the encoder, then

    h = sequence_output[positions]                      [M, H]
    t = LayerNorm(GELU(h W + b))                        cls/predictions/transform/{dense, LayerNorm}, eps 1e-12
    logits = t E^T + output_bias                        E = bert/embeddings/word_embeddings (tied decoder)
    loss = mean over the counted positions of CE(logits, label)      (ner_vocab_xent)

The loss is the exact mean over the predicted positions.  Google's code divides by sum(weights) + 1e-5 instead; this is a
restatement of its head, not a parity port.  Unused prediction slots (label -1) count nowhere.

This is not an NER plugin: its output is not tags.  `export_pretrained` writes a `bert_model.ckpt` tensor bundle that
every BERT plugin fine-tunes from with `pretrain_dir`.
"""
import json
import os
import shutil
import warnings

import numpy as np
import torch

from . import _lib, bert, ops, variables

SCOPE = "cls/predictions"
GELU = "tanh"                      # the encoder's GELU variant (bert.bert_forward_train's default)
SYNTHETIC_MASK_ID = 103            # [MASK] of the Chinese BERT vocabulary ([CLS] 101, [SEP] 102)


def prediction_budget(lengths, masked_lm_prob, max_predictions_per_seq):
    """Per-row prediction budget k_b, the only place it is computed: 0 for n <= 2 tokens, else
    min(max_pred, max(1, round(n * p))) with Python 3's round (google-research/bert create_pretraining_data.py
    num_to_predict, counted over the [CLS] ... [SEP] tokens).  -> int32 [B]."""
    out = np.zeros(len(lengths), np.int32)
    for i, n in enumerate(lengths):
        n = int(n)
        if n > 2:
            out[i] = min(max_predictions_per_seq, max(1, int(round(n * masked_lm_prob))))
    return out


def pred_offsets(budget):
    """Exclusive prefix sum [B+1] of the budgets (int32, host)."""
    return np.concatenate([[0], np.cumsum(budget, dtype=np.int64)]).astype(np.int32)


def head_names():
    return [f"{SCOPE}/transform/dense/kernel", f"{SCOPE}/transform/dense/bias", f"{SCOPE}/transform/LayerNorm/gamma",
            f"{SCOPE}/transform/LayerNorm/beta", f"{SCOPE}/output_bias"]


def _checkpoint_names(pretrain_dir):
    from . import tf_checkpoint
    prefix = tf_checkpoint.find_checkpoint(pretrain_dir)
    if prefix is not None:
        return set(tf_checkpoint.read_bundle_index(prefix + ".index")[1])
    npz = os.path.join(pretrain_dir or "", "bert_model.npz")
    if pretrain_dir and os.path.exists(npz):
        with np.load(npz) as z:
            return set(z.files)
    return set()


def create_head_variables(cfg, store):
    """The cls/predictions variables with BERT's initialisers (truncated normal 0.02, zeros, ones), then loaded from
    cfg's pretrain_dir when its checkpoint holds them (Google's Chinese checkpoint does); a warning names the ones it
    lacks."""
    H, V = cfg["hidden_size"], cfg["vocab_size"]
    fresh = f"{SCOPE}/output_bias" not in store.vars
    tn = variables.truncated_normal(cfg.get("initializer_range", 0.02))
    gv = store.get_variable
    gv(f"{SCOPE}/transform/dense/kernel", (H, H), tn)
    gv(f"{SCOPE}/transform/dense/bias", (H,), variables.zeros)
    gv(f"{SCOPE}/transform/LayerNorm/gamma", (H,), variables.ones)
    gv(f"{SCOPE}/transform/LayerNorm/beta", (H,), variables.zeros)
    gv(f"{SCOPE}/output_bias", (V,), variables.zeros)
    pretrain_dir = cfg.get("_pretrain_dir")
    if fresh and pretrain_dir:
        missing = [n for n in head_names() if n not in _checkpoint_names(pretrain_dir)]
        if missing:
            warnings.warn(f"the checkpoint under {pretrain_dir!r} lacks {missing}: they keep BERT's initialisation")
        bert.load_bert_checkpoint(pretrain_dir, store, scope="cls")


def _decoder(store, cfg):
    """bf16 operands of the head, refreshed from the store's values whenever its version moved: the dense kernel as
    [out, in] (forward) and [in, out] (data gradient), the tied decoder E zero-padded to V_pad = ceil(V / 32) * 32 rows
    (ner_gemm_bf16 needs N % 32 == 0) and its transpose [H, V_pad], and output_bias padded with zeros.  The buffers are
    allocated once; the pad rows stay zero."""
    v = store.vars
    H, V = cfg["hidden_size"], cfg["vocab_size"]
    Vp = (V + 31) // 32 * 32
    E = v["bert/embeddings/word_embeddings"]
    ent = store.caches.get("mlm_decoder")
    if ent is None:
        dev = E.device
        ent = store.caches["mlm_decoder"] = dict(
            version=-1, Vp=Vp, E=torch.zeros((Vp, H), dtype=torch.bfloat16, device=dev),
            Et=torch.empty((H, Vp), dtype=torch.bfloat16, device=dev), bias=torch.zeros((Vp,), dtype=torch.float32, device=dev))
    if ent["version"] != store.version:
        lib = _lib.lib()
        ops.check(lib.ner_cast_bf16(E.data_ptr(), ent["E"].data_ptr(), V * H, ops.stream()))
        ops.check(lib.ner_transpose_bf16(ent["E"].data_ptr(), ent["Et"].data_ptr(), V, H, Vp, ops.stream()))
        ent["bias"][:V].copy_(v[f"{SCOPE}/output_bias"])
        ent["w_nk"] = ops.pack_weight_bf16(v[f"{SCOPE}/transform/dense/kernel"])
        ent["w_kn"] = ops.cast_bf16(v[f"{SCOPE}/transform/dense/kernel"])
        ent["version"] = store.version
    return ent


def head_logits(h16, positions, M, cfg, store):
    """The head's forward on the encoder output h16 [rows, H] bf16 at the flat row indices positions [M] i32: gather,
    transform (dense, GELU, LayerNorm) and the tied decoder.  -> (logits [M, V_pad] f32, (h, pre, act, t16, decoder
    operands), what the backward reads)."""
    v = store.vars
    dec = _decoder(store, cfg)
    h = ops.gather_rows(h16, positions, M)
    pre = ops.gemm_bf16(h, dec["w_nk"], v[f"{SCOPE}/transform/dense/bias"], epilogue=ops.EPI_BF16)
    act = ops.gelu_bf16(pre, GELU == "erf")
    _, t16 = ops.layernorm(act, v[f"{SCOPE}/transform/LayerNorm/gamma"], v[f"{SCOPE}/transform/LayerNorm/beta"],
                           eps=1e-12, want_f32=False)
    logits = ops.gemm_bf16(t16, dec["E"], dec["bias"], epilogue=ops.EPI_F32)          # [M, V_pad]
    return logits, (h, pre, act, t16, dec)


class MaskedLMOutput:
    """loss [] f32, count / correct [] i32 (device scalars), pred [M] i32, and the masking: masked_ids [B,L],
    positions / labels [M]."""

    def __init__(self, loss, count, correct, pred, masked_ids, positions, labels):
        self.loss, self.count, self.correct, self.pred = loss, count, correct, pred
        self.masked_ids, self.positions, self.labels = masked_ids, positions, labels


def masked_lm(features, cfg, store, seed, masked_lm_prob, max_predictions_per_seq, mask_id, is_training, tape=None):
    """One masked-LM forward on a device batch (token_ids, mask, segment_ids, seq_len [, word_start u8]); the mask carries
    its host row lengths (engine.Estimator.to_device), so budgets, offsets and the sequence pack need no device sync.
    TRAIN (`tape`): the packed training encoder, and the head's backward recorded on the tape.  EVAL: the inference
    encoder on the padded layout."""
    ids, mask, seg = features["token_ids"], features["mask"], features.get("segment_ids")
    B, L = ids.shape
    H, V = cfg["hidden_size"], cfg["vocab_size"]
    bert.create_bert_variables(cfg, store)
    create_head_variables(cfg, store)
    lengths = getattr(mask, "row_lengths", None)
    if lengths is None:
        lengths = mask.sum(1).cpu().numpy()          # device sync; Estimator.to_device attaches the host lengths
    offsets = pred_offsets(prediction_budget(lengths, masked_lm_prob, max_predictions_per_seq))
    M = int(offsets[-1])
    off_dev = torch.from_numpy(offsets).to(ids.device, non_blocking=True)
    ws = features.get("word_start")
    if ws is not None and ws.dtype != torch.uint8:
        ws = ws.to(torch.uint8)
    masked, positions, labels = ops.mlm_mask(ids, features["seq_len"], off_dev, M, seed, V, mask_id, word_start=ws)
    if is_training:
        pack = bert.make_pack(mask, getattr(mask, "total_tokens", None))
        out = bert.bert_forward_train(masked, mask, seg, cfg, store, tape, pack=pack)
        h16 = out.bf16.reshape(B * L, H)
    else:
        _, h16 = bert.bert_forward(masked, mask, seg, cfg, store)
    dev = ids.device
    if M == 0:
        z = torch.zeros((), dtype=torch.float32, device=dev)
        zi = torch.zeros((), dtype=torch.int32, device=dev)
        return MaskedLMOutput(z, zi, zi.clone(), positions, masked, positions, labels)
    v = store.vars
    erf = GELU == "erf"
    logits, (h, pre, act, t16, dec) = head_logits(h16, positions, M, cfg, store)
    gamma = v[f"{SCOPE}/transform/LayerNorm/gamma"]
    loss, count, correct, pred, d_logits = ops.vocab_xent(logits, labels, V, want_grad=is_training)
    res = MaskedLMOutput(loss, count, correct, pred, masked, positions, labels)
    if not is_training:
        return res
    Vp = dec["Vp"]

    def bwd(_):
        gr = store.grad
        db = torch.zeros((Vp,), dtype=torch.float32, device=dev)
        ops.colsum_bf16_add(d_logits, db)
        gr(f"{SCOPE}/output_bias").add_(db[:V])
        dt = ops.gemm_bf16(d_logits, dec["Et"], None, epilogue=ops.EPI_F32)            # d_logits E: K = V_pad
        # The decoder is tied to bert/embeddings/word_embeddings: its gradient buffer receives d_logits^T t here (the pad
        # rows dropped) and the encoder's embedding backward scatters the input-side contribution into the same buffer.
        Mp = (M + 7) // 8 * 8
        dlt = ops.transpose_bf16(d_logits, Mp)[:V]
        gE = gr("bert/embeddings/word_embeddings")
        ops.gemm_bf16(dlt, ops.transpose_bf16(t16, Mp), None, residual=gE, epilogue=ops.EPI_RES_F32, out=gE)
        _, dact = ops.layernorm_bwd(act, gamma, dt, gr(f"{SCOPE}/transform/LayerNorm/gamma"),
                                    gr(f"{SCOPE}/transform/LayerNorm/beta"), eps=1e-12, want_f32=False)
        dpre = ops.gelu_bwd_bias_bf16(pre, dact, gr(f"{SCOPE}/transform/dense/bias"), erf)
        ops.wgrad_gemm_bf16(h, dpre, gr(f"{SCOPE}/transform/dense/kernel"))
        dh = ops.gemm_bf16(dpre, dec["w_kn"], None, epilogue=ops.EPI_F32)
        tape.add_grad(out, ops.scatter_rows(dh, positions, B * L).view(B, L, H))
    tape.record(loss, bwd)
    return res


def export_pretrained(store, out_dir, pretrain_dir):
    """`out_dir/bert_model.ckpt.{index,data-00000-of-00001}` (a TensorFlow tensor bundle) holding every bert/* variable,
    the untouched pooler included, and every cls/predictions/* variable; plus bert_config.json and vocab.txt from
    pretrain_dir (the config of the synthetic BERT-base-Chinese when pretrain_dir is empty).  -> the checkpoint prefix."""
    from . import tf_checkpoint
    os.makedirs(out_dir, exist_ok=True)
    tensors = {n: t.detach().cpu().numpy() for n, t in store.vars.items()
               if n.startswith("bert/") or n.startswith(SCOPE + "/")}
    prefix = os.path.join(out_dir, "bert_model.ckpt")
    tf_checkpoint.save_tf_checkpoint(prefix, tensors)
    same = pretrain_dir and os.path.abspath(pretrain_dir) == os.path.abspath(out_dir)
    for name in ("bert_config.json", "vocab.txt"):
        src = os.path.join(pretrain_dir or "", name)
        if pretrain_dir and os.path.exists(src):
            if not same:
                shutil.copyfile(src, os.path.join(out_dir, name))
        elif name == "bert_config.json":
            cfg = {k: v for k, v in bert.load_bert_config(pretrain_dir or "").items() if not k.startswith("_")}
            with open(os.path.join(out_dir, name), "w") as f:
                json.dump(cfg, f, indent=2)
    return prefix
