"""BertModel forward on the sm_90a kernels (bert_base.bert.modeling.BertModel as driven by
reference tools/layer.py:63-81; variable names per SURVEY.md §8 a9 / Appendix A.3).

Per layer: fused-QKV wgmma GEMM -> attention kernel -> wgmma GEMM (+bias, bf16 out) ->
LayerNorm(+fp32 residual; writes fp32 + bf16 copies) -> wgmma GEMM (+bias, GELU) -> wgmma
GEMM (+bias, bf16 out) -> LayerNorm(+fp32 residual).  The residual stream stays fp32; GEMM
operands and dense sub-layer outputs are bf16.
"""
import json
import os

import torch

from . import ops, variables
from .config import BERT_BASE_CHINESE


_cfg_cache = {}
FUSED_PACKS = os.environ.get("NER_B200_FUSED_PACKS", "1") != "0"   # TRAIN: one launch re-packs every encoder kernel


def load_bert_config(pretrain_dir):
    """bert_config.json of params['pretrain_dir'] over the Google chinese_L-12_H-768_A-12 defaults (read once per
    directory: the layer functions ask for it on every call).  An empty pretrain_dir is the explicit synthetic mode
    (BERT-base-Chinese architecture, random initialisation: bench.py, tests); a non-empty one must hold
    bert_config.json — the reference's modeling.BertConfig.from_json_file fails loudly there, and so does this."""
    cfg = _cfg_cache.get(pretrain_dir)
    if cfg is None:
        cfg = dict(BERT_BASE_CHINESE)
        if pretrain_dir:
            path = os.path.join(pretrain_dir, "bert_config.json")
            if not os.path.exists(path):
                raise FileNotFoundError(f"{path} not found: params['pretrain_dir'] must hold bert_config.json (+ bert_model.ckpt); "
                                        "pass pretrain_dir='' for a randomly initialised BERT-base-Chinese")
            with open(path) as f:
                cfg.update(json.load(f))
        cfg["_pretrain_dir"] = pretrain_dir
        _cfg_cache[pretrain_dir] = cfg
    return cfg


def load_bert_checkpoint(pretrain_dir, store=None, scope="bert"):
    """reference tools/train_utils.py:91-102 — initialise the BertModel variables from `<pretrain_dir>/bert_model.ckpt`
    (a TensorFlow tensor bundle, read by tf_checkpoint.py) or `<pretrain_dir>/bert_model.npz` (name -> array).  As
    get_assignment_map_from_checkpoint does, every store variable whose name the checkpoint holds is assigned; shapes
    must agree.  -> number of variables loaded (0 and a warning when the directory holds no checkpoint)."""
    import warnings

    import numpy as np

    from . import tf_checkpoint
    store = store or variables.default_store()
    prefix = tf_checkpoint.find_checkpoint(pretrain_dir)
    npz = os.path.join(pretrain_dir or "", "bert_model.npz")
    if prefix is not None:
        names = [n for n in store.vars if n.startswith(scope + "/")]
        tensors = tf_checkpoint.load_tf_checkpoint(prefix, names=set(names))
    elif pretrain_dir and os.path.exists(npz):
        with np.load(npz) as z:
            tensors = {k: z[k] for k in z.files if k in store.vars}
    else:
        warnings.warn(f"no bert_model.ckpt / bert_model.npz under {pretrain_dir!r}: the BertModel variables keep their random "
                      "initialisation (the reference would load pretrained weights here)")
        return 0
    store.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in tensors.items()}, strict=True)
    return len(tensors)


def create_bert_variables(cfg, store, scope="bert"):
    """Create (or fetch) every BertModel variable with google-research/bert's initializers."""
    H, I = cfg["hidden_size"], cfg["intermediate_size"]
    tn = variables.truncated_normal(cfg.get("initializer_range", 0.02))
    gv = store.get_variable
    fresh = f"{scope}/embeddings/word_embeddings" not in store.vars
    gv(f"{scope}/embeddings/word_embeddings", (cfg["vocab_size"], H), tn)
    gv(f"{scope}/embeddings/token_type_embeddings", (cfg["type_vocab_size"], H), tn)
    gv(f"{scope}/embeddings/position_embeddings", (cfg["max_position_embeddings"], H), tn)
    gv(f"{scope}/embeddings/LayerNorm/beta", (H,), variables.zeros)
    gv(f"{scope}/embeddings/LayerNorm/gamma", (H,), variables.ones)
    for l in range(cfg["num_hidden_layers"]):
        p = f"{scope}/encoder/layer_{l}"
        for n in ("query", "key", "value"):
            gv(f"{p}/attention/self/{n}/kernel", (H, H), tn)
            gv(f"{p}/attention/self/{n}/bias", (H,), variables.zeros)
        gv(f"{p}/attention/output/dense/kernel", (H, H), tn)
        gv(f"{p}/attention/output/dense/bias", (H,), variables.zeros)
        gv(f"{p}/attention/output/LayerNorm/beta", (H,), variables.zeros)
        gv(f"{p}/attention/output/LayerNorm/gamma", (H,), variables.ones)
        gv(f"{p}/intermediate/dense/kernel", (H, I), tn)
        gv(f"{p}/intermediate/dense/bias", (I,), variables.zeros)
        gv(f"{p}/output/dense/kernel", (I, H), tn)
        gv(f"{p}/output/dense/bias", (H,), variables.zeros)
        gv(f"{p}/output/LayerNorm/beta", (H,), variables.zeros)
        gv(f"{p}/output/LayerNorm/gamma", (H,), variables.ones)
    # pooler exists in the checkpoint but is unused by the reference (only sequence_output): its
    # gradients are None there, so apply_gradients never touches it -> not trainable here
    gv(f"{scope}/pooler/dense/kernel", (H, H), tn, trainable=False)
    gv(f"{scope}/pooler/dense/bias", (H,), variables.zeros, trainable=False)
    if fresh and cfg.get("_pretrain_dir"):
        # every bert plugin of the reference calls load_bert_checkpoint(params['pretrain_dir']) right after building
        # BertModel (model/bert_bilstm_crf.py:21): do it when the variables come into existence
        load_bert_checkpoint(cfg["_pretrain_dir"], store, scope)


def _fused_packs(store, cfg, scope):
    """TRAIN: both bf16 layouts of every encoder dense kernel — the [N, K] packs of the forward GEMMs (Q | K | V stacked into
    one [3H, H] operand) and the TF-layout casts of the data-gradient GEMMs (Q | K | V side by side in one [H, 3H]) — refreshed
    by ONE launch (ops.PackGroup) whenever the store version moved.  The destination buffers and the device table are built
    once: after the first optimizer step the variables are views of the flat parameter buffer and never move."""
    v = store.vars
    NL, H, I = cfg["num_hidden_layers"], cfg["hidden_size"], cfg["intermediate_size"]
    names = []
    for l in range(NL):
        p = f"{scope}/encoder/layer_{l}"
        names += [f"{p}/attention/self/query/kernel", f"{p}/attention/self/key/kernel", f"{p}/attention/self/value/kernel",
                  f"{p}/attention/output/dense/kernel", f"{p}/intermediate/dense/kernel", f"{p}/output/dense/kernel"]
    sig = tuple(v[n].data_ptr() for n in names)
    ent = store.caches.get(("bert_fused_packs", scope))
    if ent is None or ent["sig"] != sig:
        dev = v[names[0]].device
        bf = lambda *shape: torch.empty(shape, dtype=torch.bfloat16, device=dev)
        nk = [dict(wqkv=bf(3 * H, H), wo=bf(H, H), wi=bf(I, H), wd=bf(H, I)) for _ in range(NL)]
        kn = [dict(wqkv=bf(H, 3 * H), wo=bf(H, H), wi=bf(H, I), wd=bf(I, H)) for _ in range(NL)]
        triples = []
        for l in range(NL):
            q, k, vv, o, wi, wd = (v[n] for n in names[6 * l:6 * l + 6])
            for j, src in enumerate((q, k, vv)):
                triples.append((src, nk[l]["wqkv"][j * H:(j + 1) * H], kn[l]["wqkv"][:, j * H:(j + 1) * H]))
            triples += [(o, nk[l]["wo"], kn[l]["wo"]), (wi, nk[l]["wi"], kn[l]["wi"]), (wd, nk[l]["wd"], kn[l]["wd"])]
        ent = store.caches[("bert_fused_packs", scope)] = dict(sig=sig, nk=nk, kn=kn, group=ops.PackGroup(triples), version=-1)
    if ent["version"] != store.version:
        ent["group"].run()
        ent["version"] = store.version
    return ent


def _packed(store, cfg, scope):
    """bf16 [N,K] packs of every dense kernel (+ fused QKV), rebuilt when the store changes."""
    def build():
        if getattr(store, "_flat_state", None) is not None and FUSED_PACKS:
            ent, v, out = _fused_packs(store, cfg, scope), store.vars, []
            ball = torch.cat([v[f"{scope}/encoder/layer_{l}/attention/self/{n}/bias"] for l in range(cfg["num_hidden_layers"])
                              for n in ("query", "key", "value")]).view(cfg["num_hidden_layers"], -1)
            for l in range(cfg["num_hidden_layers"]):
                p, w = f"{scope}/encoder/layer_{l}", ent["nk"][l]
                out.append(dict(wqkv=w["wqkv"], bqkv=ball[l], wo=w["wo"], bo=v[f"{p}/attention/output/dense/bias"],
                                g1=v[f"{p}/attention/output/LayerNorm/gamma"], b1=v[f"{p}/attention/output/LayerNorm/beta"],
                                wi=w["wi"], bi=v[f"{p}/intermediate/dense/bias"], wd=w["wd"], bd=v[f"{p}/output/dense/bias"],
                                g2=v[f"{p}/output/LayerNorm/gamma"], b2=v[f"{p}/output/LayerNorm/beta"]))
            return out
        v = store.vars
        out = []
        for l in range(cfg["num_hidden_layers"]):
            p = f"{scope}/encoder/layer_{l}"
            wqkv = torch.cat([v[f"{p}/attention/self/{n}/kernel"] for n in ("query", "key", "value")], dim=1).contiguous()
            bqkv = torch.cat([v[f"{p}/attention/self/{n}/bias"] for n in ("query", "key", "value")]).contiguous()
            out.append(dict(
                wqkv=ops.pack_weight_bf16(wqkv), bqkv=bqkv,
                wo=ops.pack_weight_bf16(v[f"{p}/attention/output/dense/kernel"]), bo=v[f"{p}/attention/output/dense/bias"],
                g1=v[f"{p}/attention/output/LayerNorm/gamma"], b1=v[f"{p}/attention/output/LayerNorm/beta"],
                wi=ops.pack_weight_bf16(v[f"{p}/intermediate/dense/kernel"]), bi=v[f"{p}/intermediate/dense/bias"],
                wd=ops.pack_weight_bf16(v[f"{p}/output/dense/kernel"]), bd=v[f"{p}/output/dense/bias"],
                g2=v[f"{p}/output/LayerNorm/gamma"], b2=v[f"{p}/output/LayerNorm/beta"]))
        return out
    return store.cached(("bert_pack", scope), build)


class PackInfo:
    """Sequence-packing plan of one batch: token rows of all sequences back to back, no padding."""

    def __init__(self, cu_seqlens, tok_src, total, B, L):
        self.cu_seqlens, self.tok_src, self.total, self.B, self.L = cu_seqlens, tok_src, int(total), B, L


def make_pack(input_mask, total_tokens=None):
    """Plan from a prefix mask [B,L].  `total_tokens` (host int) avoids a device sync."""
    B, L = input_mask.shape
    if total_tokens is None:
        total_tokens = getattr(input_mask, "total_tokens", None)
    if total_tokens is None:
        total_tokens = int(input_mask.sum().item())      # device sync; engine.Estimator passes the host count
    cu, tok_src = ops.seq_pack_plan(input_mask)
    return PackInfo(cu, tok_src, total_tokens, B, L)


def _c_tables(store, cfg, scope, gelu):
    """ctypes config + per-layer pointer table for ner_bert_encoder_fwd (rebuilt with the packs)."""
    layers = _packed(store, cfg, scope)

    def build():
        from . import _lib
        c = _lib.BertConfig(cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                            cfg["num_hidden_layers"], cfg["vocab_size"], cfg["type_vocab_size"],
                            cfg["max_position_embeddings"], 1e-12, 1 if gelu == "erf" else 0, 0)
        arr = (_lib.BertLayerWeights * len(layers))()
        for i, w in enumerate(layers):
            arr[i] = _lib.BertLayerWeights(w["wqkv"].data_ptr(), w["bqkv"].data_ptr(), w["wo"].data_ptr(), w["bo"].data_ptr(),
                                           w["g1"].data_ptr(), w["b1"].data_ptr(), w["wi"].data_ptr(), w["bi"].data_ptr(),
                                           w["wd"].data_ptr(), w["bd"].data_ptr(), w["g2"].data_ptr(), w["b2"].data_ptr())
        return c, arr, layers  # keep `layers` alive with the table
    return store.cached(("bert_ctable", scope, gelu), build)


_ws_cache = {}
PER_KERNEL = False   # True: drive the encoder one ops.* call per kernel (bench.py's per-kernel timing pass)


def bert_forward(input_ids, input_mask, segment_ids, cfg, store=None, scope="bert", gelu="tanh", pack=None,
                 per_kernel=None):
    """-> (sequence_output f32 [rows,H], bf16 copy [rows,H]); rows = B*L, or pack.total in packed mode.

    Default: ONE C-ABI call (ner_bert_encoder_fwd) enqueues the whole encoder.  per_kernel=True drives
    the same kernels one ops.* call at a time (used by bench.py's per-kernel timing and the tests)."""
    store = store or variables.default_store()
    create_bert_variables(cfg, store, scope)
    if per_kernel is None:
        per_kernel = PER_KERNEL
    if not per_kernel:
        import ctypes
        from . import _lib
        B, L = input_ids.shape
        H = cfg["hidden_size"]
        v = store.vars
        c, arr, _ = _c_tables(store, cfg, scope, gelu)
        c.gemm_tile = ops.DEFAULT_TILE            # latency (0) or throughput tile policy, see ops.DEFAULT_TILE
        rows = pack.total if pack else B * L
        dev = input_ids.device
        of = torch.empty((rows, H), dtype=torch.float32, device=dev)
        ob = torch.empty((rows, H), dtype=torch.bfloat16, device=dev)
        need = _lib.lib().ner_bert_encoder_workspace_bytes(ctypes.byref(c), rows)
        key = (dev.index, _lib.stream())
        ws = _ws_cache.get(key)
        if ws is None or ws.numel() < need:
            ws = torch.empty((need,), dtype=torch.uint8, device=dev)
            _ws_cache[key] = ws
        ids = ops._i32(input_ids)
        seg = None if segment_ids is None else ops._i32(segment_ids)
        mask = ops._i32(input_mask)
        _lib.check(_lib.lib().ner_bert_encoder_fwd(
            ctypes.byref(c), v[f"{scope}/embeddings/word_embeddings"].data_ptr(),
            v[f"{scope}/embeddings/token_type_embeddings"].data_ptr(), v[f"{scope}/embeddings/position_embeddings"].data_ptr(),
            v[f"{scope}/embeddings/LayerNorm/gamma"].data_ptr(), v[f"{scope}/embeddings/LayerNorm/beta"].data_ptr(), arr,
            ids.data_ptr(), mask.data_ptr(), _lib.ptr(seg), B, L, _lib.ptr(pack.cu_seqlens if pack else None),
            _lib.ptr(pack.tok_src if pack else None), pack.total if pack else 0, of.data_ptr(), ob.data_ptr(),
            ws.data_ptr(), ws.numel(), _lib.stream()))
        _lib.LAUNCHES += 7 * cfg["num_hidden_layers"]      # the call above enqueued 1 + 7/layer kernels
        return of, ob
    B, L = input_ids.shape
    H, NH = cfg["hidden_size"], cfg["num_attention_heads"]
    v = store.vars
    layers = _packed(store, cfg, scope)
    x32, x16 = ops.bert_embed_ln(v[f"{scope}/embeddings/word_embeddings"], v[f"{scope}/embeddings/token_type_embeddings"],
                                 v[f"{scope}/embeddings/position_embeddings"], v[f"{scope}/embeddings/LayerNorm/gamma"],
                                 v[f"{scope}/embeddings/LayerNorm/beta"], input_ids, segment_ids, eps=1e-12,
                                 tok_src=pack.tok_src if pack else None, n_packed=pack.total if pack else 0)
    epi_gelu = ops.EPI_GELU_ERF_BF16 if gelu == "erf" else ops.EPI_GELU_TANH_BF16
    cu = pack.cu_seqlens if pack else None
    for w in layers:
        qkv = ops.gemm_bf16(x16, w["wqkv"], w["bqkv"], epilogue=ops.EPI_BF16)
        ctx = ops.bert_attention(qkv, input_mask, B, L, NH, H // NH, cu_seqlens=cu)
        y = ops.gemm_bf16(ctx, w["wo"], w["bo"], epilogue=ops.EPI_BF16)
        x32, x16 = ops.layernorm(y, w["g1"], w["b1"], residual=x32, eps=1e-12)
        inter = ops.gemm_bf16(x16, w["wi"], w["bi"], epilogue=epi_gelu)
        y = ops.gemm_bf16(inter, w["wd"], w["bd"], epilogue=ops.EPI_BF16)
        x32, x16 = ops.layernorm(y, w["g2"], w["b2"], residual=x32, eps=1e-12)
    return x32, x16


# =========================================================================== FP8 inference
def _packed_fp8(store, cfg, scope):
    """FP8 operands of every layer, rebuilt when the store changes: e4m3 [N,K] packs + per-channel scales of the QKV (query |
    key | value fused), FFN1 and FFN2 kernels; the out-projection keeps its bf16 pack (shared with the bf16 path)."""
    bf = _packed(store, cfg, scope)

    def build():
        v, out = store.vars, []
        for l, w in enumerate(bf):
            p = f"{scope}/encoder/layer_{l}"
            wqkv = torch.cat([v[f"{p}/attention/self/{n}/kernel"] for n in ("query", "key", "value")], dim=1).contiguous()
            (wq, sq), (wi, si), (wd, sd) = (ops.quantize_weight_e4m3(t) for t in
                                            (wqkv, v[f"{p}/intermediate/dense/kernel"], v[f"{p}/output/dense/kernel"]))
            out.append(dict(w, wqkv=wq, sqkv=sq, wi=wi, si=si, wd=wd, sd=sd))
        return out
    return store.cached(("bert_pack_fp8", scope), build)


def _c_tables_fp8(store, cfg, scope, gelu):
    """ctypes config + per-layer pointer table for ner_bert_encoder_fwd_fp8 (rebuilt with the packs)."""
    layers = _packed_fp8(store, cfg, scope)

    def build():
        from . import _lib
        c = _lib.BertConfig(cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                            cfg["num_hidden_layers"], cfg["vocab_size"], cfg["type_vocab_size"],
                            cfg["max_position_embeddings"], 1e-12, 1 if gelu == "erf" else 0, 0)
        arr = (_lib.BertLayerWeightsFp8 * len(layers))()
        for i, w in enumerate(layers):
            arr[i] = _lib.BertLayerWeightsFp8(*[w[k].data_ptr() for k in ("wqkv", "sqkv", "bqkv", "wo", "bo", "g1", "b1", "wi", "si",
                                                                         "bi", "wd", "sd", "bd", "g2", "b2")])
        return c, arr, layers
    return store.cached(("bert_ctable_fp8", scope, gelu), build)


def _check_fp8_shape(cfg):
    H, I = cfg["hidden_size"], cfg["intermediate_size"]
    if H % 128 or I % 128:
        raise ValueError(f"bert_precision='fp8' needs hidden_size and intermediate_size to be multiples of 128 (its activation "
                         f"scales cover 1 x 128 blocks); this BERT has hidden_size={H}, intermediate_size={I}")


def bert_forward_fp8(input_ids, input_mask, segment_ids, cfg, store=None, scope="bert", gelu="tanh", pack=None,
                     per_kernel=None):
    """Inference BertModel forward with FP8 (e4m3, block-scaled) QKV / FFN1 / FFN2 GEMMs -> (f32 [rows,H], bf16 [rows,H]),
    the outputs of bert_forward.  Default: ONE C-ABI call (ner_bert_encoder_fwd_fp8); per_kernel=True drives the same kernels
    one ops.* call at a time."""
    store = store or variables.default_store()
    create_bert_variables(cfg, store, scope)
    _check_fp8_shape(cfg)
    if per_kernel is None:
        per_kernel = PER_KERNEL
    B, L = input_ids.shape
    H, NH = cfg["hidden_size"], cfg["num_attention_heads"]
    v = store.vars
    rows = pack.total if pack else B * L
    dev = input_ids.device
    if not per_kernel:
        import ctypes
        from . import _lib
        c, arr, _ = _c_tables_fp8(store, cfg, scope, gelu)
        c.gemm_tile = ops.DEFAULT_TILE
        of = torch.empty((rows, H), dtype=torch.float32, device=dev)
        ob = torch.empty((rows, H), dtype=torch.bfloat16, device=dev)
        need = _lib.lib().ner_bert_encoder_fp8_workspace_bytes(ctypes.byref(c), rows)
        key = (dev.index, _lib.stream())
        ws = _ws_cache.get(key)
        if ws is None or ws.numel() < need:
            ws = torch.empty((need,), dtype=torch.uint8, device=dev)
            _ws_cache[key] = ws
        ids, mask = ops._i32(input_ids), ops._i32(input_mask)
        seg = None if segment_ids is None else ops._i32(segment_ids)
        _lib.check(_lib.lib().ner_bert_encoder_fwd_fp8(
            ctypes.byref(c), v[f"{scope}/embeddings/word_embeddings"].data_ptr(),
            v[f"{scope}/embeddings/token_type_embeddings"].data_ptr(), v[f"{scope}/embeddings/position_embeddings"].data_ptr(),
            v[f"{scope}/embeddings/LayerNorm/gamma"].data_ptr(), v[f"{scope}/embeddings/LayerNorm/beta"].data_ptr(), arr,
            ids.data_ptr(), mask.data_ptr(), _lib.ptr(seg), B, L, _lib.ptr(pack.cu_seqlens if pack else None),
            _lib.ptr(pack.tok_src if pack else None), pack.total if pack else 0, of.data_ptr(), ob.data_ptr(),
            ws.data_ptr(), ws.numel(), _lib.stream()))
        _lib.LAUNCHES += 7 * cfg["num_hidden_layers"]      # the call above enqueued 1 + 7/layer kernels
        return of, ob
    layers = _packed_fp8(store, cfg, scope)
    x32, xq, xs = ops.bert_embed_ln_e4m3(v[f"{scope}/embeddings/word_embeddings"], v[f"{scope}/embeddings/token_type_embeddings"],
                                         v[f"{scope}/embeddings/position_embeddings"], v[f"{scope}/embeddings/LayerNorm/gamma"],
                                         v[f"{scope}/embeddings/LayerNorm/beta"], input_ids, segment_ids, eps=1e-12,
                                         tok_src=pack.tok_src if pack else None, n_packed=pack.total if pack else 0)
    epi_gelu = ops.EPI_GELU_ERF_E4M3 if gelu == "erf" else ops.EPI_GELU_TANH_E4M3
    cu = pack.cu_seqlens if pack else None
    for i, w in enumerate(layers):
        qkv = ops.gemm_e4m3(xq, xs, w["wqkv"], w["sqkv"], w["bqkv"], epilogue=ops.EPI_BF16)
        ctx = ops.bert_attention(qkv, input_mask, B, L, NH, H // NH, cu_seqlens=cu)
        y = ops.gemm_bf16(ctx, w["wo"], w["bo"], epilogue=ops.EPI_BF16)
        x1, xq, xs = ops.layernorm_e4m3(y, w["g1"], w["b1"], residual=x32, eps=1e-12)
        iq, isc = ops.gemm_e4m3(xq, xs, w["wi"], w["si"], w["bi"], epilogue=epi_gelu)
        y = ops.gemm_e4m3(iq, isc, w["wd"], w["sd"], w["bd"], epilogue=ops.EPI_BF16)
        if i + 1 < len(layers):
            x32, xq, xs = ops.layernorm_e4m3(y, w["g2"], w["b2"], residual=x1, eps=1e-12)
        else:
            x32, x16 = ops.layernorm(y, w["g2"], w["b2"], residual=x1, eps=1e-12)
    return x32, x16


# =========================================================================== training
def _tf_casts(store, cfg, scope):
    """bf16 casts of the dense kernels in their TF layout [in, out]: the K-major B operand of the
    data-gradient GEMMs (dX = dY · W^T)."""
    def build():
        if getattr(store, "_flat_state", None) is not None and FUSED_PACKS:
            return _fused_packs(store, cfg, scope)["kn"]
        v = store.vars
        out = []
        for l in range(cfg["num_hidden_layers"]):
            p = f"{scope}/encoder/layer_{l}"
            wqkv = torch.cat([v[f"{p}/attention/self/{n}/kernel"] for n in ("query", "key", "value")], dim=1).contiguous()
            out.append(dict(wqkv=ops.cast_bf16(wqkv), wo=ops.cast_bf16(v[f"{p}/attention/output/dense/kernel"]),
                            wi=ops.cast_bf16(v[f"{p}/intermediate/dense/kernel"]), wd=ops.cast_bf16(v[f"{p}/output/dense/kernel"])))
        return out
    return store.cached(("bert_tf_casts", scope), build)


def bert_forward_f32(input_ids, input_mask, segment_ids, cfg, store=None, scope="bert", gelu="tanh"):
    """BertModel forward at fp32 accuracy (BASELINE config 2: "bert_crf ... fp32", logits within 1e-3 of the
    reference): every dense layer is the 3-term split-bf16 product on the wgmma kernel (ops.gemm_split_f32,
    ~2^-16 relative), attention is the fp32 kernel (ner_attention_f32, head_dim 64), LayerNorm / GELU / residual
    stream in f32.  Padded layout; keys are limited to the mask's prefix length, which equals the additive
    (1-mask)*-10000 of attention_layer() because exp(-10000 - max) is exactly 0 in fp32.  ~3x the GEMM work of the
    bf16 path: a parity mode, not the benchmark path."""
    from .tools.transformer.modules import dense_f32
    store = store or variables.default_store()
    create_bert_variables(cfg, store, scope)
    B, L = input_ids.shape
    H, NH, I = cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"]
    v = store.vars
    ids, seg = ops._i32(input_ids), (None if segment_ids is None else ops._i32(segment_ids))
    lens = ops._i32(input_mask).sum(1).to(torch.int32)
    we, te, pe = (v[f"{scope}/embeddings/{n}"] for n in ("word_embeddings", "token_type_embeddings", "position_embeddings"))
    x, _ = ops.bert_embed_ln(we, te, pe, v[f"{scope}/embeddings/LayerNorm/gamma"], v[f"{scope}/embeddings/LayerNorm/beta"], ids, seg,
                             eps=1e-12)
    with variables.use_store(store):
        for li in range(cfg["num_hidden_layers"]):
            p = f"{scope}/encoder/layer_{li}"
            q = dense_f32(x, H, f"{p}/attention/self/query")
            k = dense_f32(x, H, f"{p}/attention/self/key")
            val = dense_f32(x, H, f"{p}/attention/self/value")
            ctx, _, _ = ops.attention_f32(q, k, val, lens, B, L, NH, H // NH, scale=(H // NH) ** -0.5)
            y = dense_f32(ctx, H, f"{p}/attention/output/dense", residual=x)
            x1, _ = ops.layernorm(y, v[f"{p}/attention/output/LayerNorm/gamma"], v[f"{p}/attention/output/LayerNorm/beta"],
                                  eps=1e-12, want_bf16=False)
            h = ops.gelu_f32(dense_f32(x1, I, f"{p}/intermediate/dense"), erf=(gelu == "erf"), inplace=True)
            y2 = dense_f32(h, H, f"{p}/output/dense", residual=x1)
            x, _ = ops.layernorm(y2, v[f"{p}/output/LayerNorm/gamma"], v[f"{p}/output/LayerNorm/beta"], eps=1e-12,
                                 want_bf16=False)
    return x


def _train_composite(input_ids, input_mask, segment_ids, cfg, store, tape, scope, gelu, keep_h, keep_a, pack=None):
    """TRAIN forward + recorded backward through the two C-ABI composites (bert_train.cu): the host
    enqueues the whole encoder with two calls instead of ~480 (the per-kernel path is launch-bound).
    pack (PackInfo): the sequence-packed composites — every per-token kernel runs on the real tokens only; the output
    keeps the padded [B,L,H] shape with zero rows at [PAD]."""
    import ctypes
    from . import _lib
    B, L = input_ids.shape
    H = cfg["hidden_size"]
    rows = B * L
    v = store.vars
    c, arr, layers = _c_tables(store, cfg, scope, gelu)
    dev = input_ids.device
    ids, seg, mask = ops._i32(input_ids), (None if segment_ids is None else ops._i32(segment_ids)), ops._i32(input_mask)
    if pack is not None:
        return _train_composite_packed(ids, seg, cfg, store, tape, scope, keep_h, keep_a, pack, c, arr, layers)
    saved_b = _lib.lib().ner_bert_train_saved_bytes(ctypes.byref(c), rows)
    saved = torch.empty(saved_b, dtype=torch.uint8, device=dev)
    out32 = torch.empty((rows, H), dtype=torch.float32, device=dev)
    out16 = torch.empty((rows, H), dtype=torch.bfloat16, device=dev)
    store.dropout_calls += 1
    seed = (4321 * 1000003 + store.global_step) * 1009 + 64 * store.dropout_calls     # the call uses seed .. seed + 3*layers
    emb = [v[f"{scope}/embeddings/{n}"] for n in ("word_embeddings", "token_type_embeddings", "position_embeddings",
                                                  "LayerNorm/gamma", "LayerNorm/beta")]
    st = ops.stream()
    ops.check(_lib.lib().ner_bert_encoder_train_fwd(
        ctypes.byref(c), *[ops.ptr(t) for t in emb], arr, ops.ptr(ids), ops.ptr(mask), ops.ptr(seg), B, L, float(keep_h),
        float(keep_a), seed & 0xFFFFFFFFFFFFFFFF, ops.ptr(out32), ops.ptr(out16), ops.ptr(saved), saved_b, st))
    _lib.LAUNCHES += 3 + 11 * len(layers)
    out = out32.view(B, L, H)
    out.bf16 = out16.view(B, L, H)

    def bwd(g):
        if g is None:
            return
        casts = _tf_casts(store, cfg, scope)
        gr = store.grad
        garr = (_lib.BertLayerGrads * len(layers))()
        for li in range(len(layers)):
            p = f"{scope}/encoder/layer_{li}"
            cs = casts[li]
            ptrs = [cs["wqkv"], cs["wo"], cs["wi"], cs["wd"]]
            ptrs += [gr(f"{p}/attention/self/{n}/kernel") for n in ("query", "key", "value")]
            ptrs += [gr(f"{p}/attention/self/{n}/bias") for n in ("query", "key", "value")]
            ptrs += [gr(f"{p}/attention/output/dense/kernel"), gr(f"{p}/attention/output/dense/bias"),
                     gr(f"{p}/attention/output/LayerNorm/gamma"), gr(f"{p}/attention/output/LayerNorm/beta"),
                     gr(f"{p}/intermediate/dense/kernel"), gr(f"{p}/intermediate/dense/bias"),
                     gr(f"{p}/output/dense/kernel"), gr(f"{p}/output/dense/bias"),
                     gr(f"{p}/output/LayerNorm/gamma"), gr(f"{p}/output/LayerNorm/beta")]
            garr[li] = _lib.BertLayerGrads(*[t.data_ptr() for t in ptrs])
        scratch_b = _lib.lib().ner_bert_train_scratch_bytes(ctypes.byref(c), rows)
        scratch = torch.empty(scratch_b, dtype=torch.uint8, device=dev)
        d = g.reshape(rows, H).contiguous()
        demb = [gr(f"{scope}/embeddings/{n}") for n in ("word_embeddings", "token_type_embeddings", "position_embeddings",
                                                        "LayerNorm/gamma", "LayerNorm/beta")]
        ex = getattr(store, '_grad_exchange', None)
        if ex is not None:
            ex.before_bert_backward()
        ops.check(_lib.lib().ner_bert_encoder_train_bwd(
            ctypes.byref(c), ops.ptr(emb[3]), arr, garr, *[ops.ptr(t) for t in demb], ops.ptr(ids), ops.ptr(mask), ops.ptr(seg),
            B, L, float(keep_h), float(keep_a), seed & 0xFFFFFFFFFFFFFFFF, ops.ptr(d), ops.ptr(saved), saved_b, ops.ptr(scratch),
            scratch_b, ops.stream()))
        if ex is not None:
            ex.after_bert_backward()
        _lib.LAUNCHES += 3 + 33 * len(layers)
    tape.record(out, bwd)
    return out


def _layer_grad_table(store, cfg, scope, layers):
    from . import _lib
    casts = _tf_casts(store, cfg, scope)
    gr = store.grad
    garr = (_lib.BertLayerGrads * len(layers))()
    for li in range(len(layers)):
        p = f"{scope}/encoder/layer_{li}"
        cs = casts[li]
        ptrs = [cs["wqkv"], cs["wo"], cs["wi"], cs["wd"]]
        ptrs += [gr(f"{p}/attention/self/{n}/kernel") for n in ("query", "key", "value")]
        ptrs += [gr(f"{p}/attention/self/{n}/bias") for n in ("query", "key", "value")]
        ptrs += [gr(f"{p}/attention/output/dense/kernel"), gr(f"{p}/attention/output/dense/bias"),
                 gr(f"{p}/attention/output/LayerNorm/gamma"), gr(f"{p}/attention/output/LayerNorm/beta"),
                 gr(f"{p}/intermediate/dense/kernel"), gr(f"{p}/intermediate/dense/bias"),
                 gr(f"{p}/output/dense/kernel"), gr(f"{p}/output/dense/bias"),
                 gr(f"{p}/output/LayerNorm/gamma"), gr(f"{p}/output/LayerNorm/beta")]
        garr[li] = _lib.BertLayerGrads(*[t.data_ptr() for t in ptrs])
    return garr


def _train_composite_packed(ids, seg, cfg, store, tape, scope, keep_h, keep_a, pack, c, arr, layers):
    import ctypes
    from . import _lib
    B, L = ids.shape
    H = cfg["hidden_size"]
    n = pack.total
    v = store.vars
    dev = ids.device
    saved_b = _lib.lib().ner_bert_train_packed_saved_bytes(ctypes.byref(c), n)
    saved = torch.empty(saved_b, dtype=torch.uint8, device=dev)
    out32 = torch.empty((B * L, H), dtype=torch.float32, device=dev)
    out16 = torch.empty((B * L, H), dtype=torch.bfloat16, device=dev)
    store.dropout_calls += 1
    seed = ((4321 * 1000003 + store.global_step) * 1009 + 64 * store.dropout_calls) & 0xFFFFFFFFFFFFFFFF
    names = ("word_embeddings", "token_type_embeddings", "position_embeddings", "LayerNorm/gamma", "LayerNorm/beta")
    emb = [v[f"{scope}/embeddings/{k}"] for k in names]
    ops.check(_lib.lib().ner_bert_encoder_train_fwd_packed(
        ctypes.byref(c), *[ops.ptr(t) for t in emb], arr, ops.ptr(ids), ops.ptr(seg), B, L, ops.ptr(pack.cu_seqlens),
        ops.ptr(pack.tok_src), n, float(keep_h), float(keep_a), seed, ops.ptr(out32), ops.ptr(out16), ops.ptr(saved), saved_b,
        ops.stream()))
    _lib.LAUNCHES += 9 + 11 * len(layers)
    out = out32.view(B, L, H)
    out.bf16 = out16.view(B, L, H)

    def bwd(g):
        if g is None:
            return
        garr = _layer_grad_table(store, cfg, scope, layers)
        scratch_b = _lib.lib().ner_bert_train_packed_scratch_bytes(ctypes.byref(c), n, B * L)
        scratch = torch.empty(scratch_b, dtype=torch.uint8, device=dev)
        d = g.reshape(B * L, H).contiguous()
        demb = [store.grad(f"{scope}/embeddings/{k}") for k in names]
        ex = getattr(store, '_grad_exchange', None)
        if ex is not None:
            ex.before_bert_backward()
        ops.check(_lib.lib().ner_bert_encoder_train_bwd_packed(
            ctypes.byref(c), ops.ptr(emb[3]), arr, garr, *[ops.ptr(t) for t in demb], ops.ptr(ids), ops.ptr(seg), B, L,
            ops.ptr(pack.cu_seqlens), ops.ptr(pack.tok_src), n, float(keep_h), float(keep_a), seed, ops.ptr(d), ops.ptr(saved),
            saved_b, ops.ptr(scratch), scratch_b, ops.stream()))
        if ex is not None:
            ex.after_bert_backward()
        _lib.LAUNCHES += 6 + 33 * len(layers)
    tape.record(out, bwd)
    return out


def bert_forward_train(input_ids, input_mask, segment_ids, cfg, store, tape, scope="bert", gelu="tanh", pack=None):
    """Training-mode BertModel forward on the padded layout: same kernels, every intermediate the
    backward pass needs is kept, and the backward closure is recorded on `tape`.
    BertModel(is_training=True) dropout (bert modeling.py: hidden_dropout_prob after the embedding
    LayerNorm and after the attention-output / FFN-output dense layers, attention_probs_dropout_prob
    on the softmax output; both 0.1 in bert_config.json) uses the same counter-based masks as every
    other dropout site: the backward pass regenerates them from (seed, element)."""
    create_bert_variables(cfg, store, scope)
    keep_h = 1.0 - float(cfg.get("hidden_dropout_prob", 0.1))
    keep_a = 1.0 - float(cfg.get("attention_probs_dropout_prob", 0.1))
    if not PER_KERNEL:
        return _train_composite(input_ids, input_mask, segment_ids, cfg, store, tape, scope, gelu, keep_h, keep_a, pack=pack)

    def next_seed():
        store.dropout_calls += 1
        return (4321 * 1000003 + store.global_step) * 1009 + store.dropout_calls
    B, L = input_ids.shape
    H, NH, I = cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"]
    v = store.vars
    layers = _packed(store, cfg, scope)
    erf = gelu == "erf"
    ids, seg, mask = ops._i32(input_ids), (None if segment_ids is None else ops._i32(segment_ids)), ops._i32(input_mask)
    we, te, pe = (v[f"{scope}/embeddings/{n}"] for n in ("word_embeddings", "token_type_embeddings", "position_embeddings"))
    ge, be = v[f"{scope}/embeddings/LayerNorm/gamma"], v[f"{scope}/embeddings/LayerNorm/beta"]
    x32, x16 = ops.bert_embed_ln(we, te, pe, ge, be, ids, seg, eps=1e-12)
    seed_e = next_seed()
    if keep_h < 1.0:
        x32 = ops.dropout(x32, keep_h, seed_e)
        x16 = ops.cast_bf16(x32)
    saved = []
    for w in layers:
        sa, s1, s2 = next_seed(), next_seed(), next_seed()
        qkv = ops.gemm_bf16(x16, w["wqkv"], w["bqkv"], epilogue=ops.EPI_BF16)
        ctx = ops.bert_attention(qkv, mask, B, L, NH, H // NH, keep_prob=keep_a, seed=sa)
        y1 = ops.gemm_bf16(ctx, w["wo"], w["bo"], epilogue=ops.EPI_BF16)
        x1_32, x1_16 = ops.layernorm(y1, w["g1"], w["b1"], residual=x32, eps=1e-12, keep_prob=keep_h, seed=s1)
        pre = ops.gemm_bf16(x1_16, w["wi"], w["bi"], epilogue=ops.EPI_BF16)
        inter = ops.gelu_bf16(pre, erf)
        y2 = ops.gemm_bf16(inter, w["wd"], w["bd"], epilogue=ops.EPI_BF16)
        x2_32, x2_16 = ops.layernorm(y2, w["g2"], w["b2"], residual=x1_32, eps=1e-12, keep_prob=keep_h, seed=s2)
        saved.append((x32, x16, qkv, ctx, y1, x1_32, x1_16, pre, inter, y2, sa, s1, s2))
        x32, x16 = x2_32, x2_16
    out = x32.view(B, L, H)
    out.bf16 = x16.view(B, L, H)

    def bwd(g):
        if g is None:
            return
        casts = _tf_casts(store, cfg, scope)
        gr = store.grad
        d = g.reshape(B * L, H).contiguous()
        for li in reversed(range(len(layers))):
            w, c = layers[li], casts[li]
            x32_, x16_, qkv, ctx, y1, x1_32, x1_16, pre, inter, y2, sa, s1, s2 = saved[li]
            p = f"{scope}/encoder/layer_{li}"
            # ---- output LayerNorm + FFN
            dz2_32, dz2_16 = ops.layernorm_bwd(y2, w["g2"], d, gr(f"{p}/output/LayerNorm/gamma"), gr(f"{p}/output/LayerNorm/beta"),
                                               residual=x1_32, eps=1e-12, keep_prob=keep_h, seed=s2)
            # (dz2_32 feeds the residual path, dz2_16 — masked like the forward — the dense output)
            ops.colsum_bf16_add(dz2_16, gr(f"{p}/output/dense/bias"))
            ops.wgrad_gemm_bf16(inter, dz2_16, gr(f"{p}/output/dense/kernel"))
            dinter = ops.gemm_bf16(dz2_16, c["wd"], None, epilogue=ops.EPI_BF16)
            dpre = ops.gelu_bwd_bf16(pre, dinter, erf)
            ops.colsum_bf16_add(dpre, gr(f"{p}/intermediate/dense/bias"))
            ops.wgrad_gemm_bf16(x1_16, dpre, gr(f"{p}/intermediate/dense/kernel"))
            dx1 = ops.gemm_bf16(dpre, c["wi"], None, residual=dz2_32, epilogue=ops.EPI_RES_F32)
            # ---- attention LayerNorm + output projection
            dz1_32, dz1_16 = ops.layernorm_bwd(y1, w["g1"], dx1, gr(f"{p}/attention/output/LayerNorm/gamma"),
                                               gr(f"{p}/attention/output/LayerNorm/beta"), residual=x32_, eps=1e-12,
                                               keep_prob=keep_h, seed=s1)
            ops.colsum_bf16_add(dz1_16, gr(f"{p}/attention/output/dense/bias"))
            ops.wgrad_gemm_bf16(ctx, dz1_16, gr(f"{p}/attention/output/dense/kernel"))
            dctx = ops.gemm_bf16(dz1_16, c["wo"], None, epilogue=ops.EPI_BF16)
            # ---- attention core + fused QKV projection
            dqkv = ops.bert_attention_bwd(qkv, mask, ctx, dctx, B, L, NH, H // NH, keep_prob=keep_a, seed=sa)
            dbqkv = torch.zeros(3 * H, dtype=torch.float32, device=d.device)
            ops.colsum_bf16_add(dqkv, dbqkv)
            dwqkv = ops.wgrad_gemm_bf16(x16_, dqkv)                       # [H, 3H]
            for k, n in enumerate(("query", "key", "value")):
                gr(f"{p}/attention/self/{n}/kernel").add_(dwqkv[:, k * H:(k + 1) * H])
                gr(f"{p}/attention/self/{n}/bias").add_(dbqkv[k * H:(k + 1) * H])
            d = ops.gemm_bf16(dqkv, c["wqkv"], None, residual=dz1_32, epilogue=ops.EPI_RES_F32)
        # ---- embeddings: dropout, then LayerNorm of (word + type + position)
        if keep_h < 1.0:
            d = ops.dropout(d.contiguous(), keep_h, seed_e)
        segl = torch.zeros_like(ids) if seg is None else seg
        emb_sum = (we[ids.long()] + te[segl.long()] + pe[:L][None]).reshape(B * L, H).contiguous()
        dsum, _ = ops.layernorm_bwd(emb_sum, ge, d, gr(f"{scope}/embeddings/LayerNorm/gamma"), gr(f"{scope}/embeddings/LayerNorm/beta"),
                                    eps=1e-12, want_bf16=False)
        ops.bert_embed_bwd(dsum, ids, seg, gr(f"{scope}/embeddings/word_embeddings"), gr(f"{scope}/embeddings/token_type_embeddings"),
                           gr(f"{scope}/embeddings/position_embeddings"))
    tape.record(out, bwd)
    return out
