"""Single-call PREDICT executors for plugins whose whole step exists as one C-ABI composite.

`build_graph()` of the plugin stays the definition of the model (and the only path for EVAL / TRAIN); a fused
executor launches the same kernels in the same order from ONE ctypes call, so the ~20 Python-level calls of a
step leave the host's critical path (eight 4-stream pipelines share one host at N=8, DESIGN.md §7).
`Estimator.predict*` uses it when every variable already exists and the host knows the batch's token count;
tests/test_models_gpu.py pins fused == build_graph.
"""
import ctypes

import torch

from . import _lib, bert as _bert, ops
from .tools import layer as _layer

_ws = {}


def _workspace(nbytes, device):
    key = (device.index, _lib.stream())
    ws = _ws.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = _ws[key] = torch.empty((nbytes,), dtype=torch.uint8, device=device)
    return ws


def bert_bilstm_crf_predict(est, dev):
    """-> pred_ids [B,L] int32 on the device, or None when the fused call does not apply."""
    store, params = est.store, est.params
    mask = dev['mask']
    total = getattr(mask, "total_tokens", None)
    if total is None or not _layer.PACK_SEQUENCES or _bert.PER_KERNEL or params.get('bert_precision', _layer.BERT_PRECISION) != 'bf16':
        return None
    if params.get('cell_type', 'lstm').lower() != 'lstm' or params.get('cell_size', 1) != 1:
        return None
    if params.get('crf_nbest', 1) > 1:
        return None                                    # N-best decoding: build_graph's crf_decode attaches the paths
    if dev['token_ids'].shape[1] > est.document_window()[0]:
        return None                                    # document mode: build_graph stitches the windows
    if params['label_size'] > 32:
        return None                                    # the fused executor's CRF takes 32 tags: build_graph's takes 128
    Hl, K = params['hidden_units_list'][0], params['label_size']
    v = store.vars
    lscope = "bilstm_layer/bidirectional_rnn"
    need = ("logits/kernel", "logits/bias", "crf_layer/transitions", f"{lscope}/fw/multi_rnn_cell/cell_0/lstm_cell/kernel",
            "bert/embeddings/word_embeddings")
    if any(n not in v for n in need):
        return None                                    # first call: build_graph creates the variables
    cfg = _bert.load_bert_config(params['pretrain_dir'])
    H = cfg["hidden_size"]
    c, arr, _ = _bert._c_tables(store, cfg, "bert", "tanh")
    c.gemm_tile = ops.DEFAULT_TILE
    pk = _layer._rnn_pack(store, {d: _layer._rnn_names(lscope, d, "lstm", 0) for d in ("fw", "bw")}, H, False)
    if pk["Dp"] != H:
        return None
    ids, seg, m32, sl = ops._i32(dev['token_ids']), ops._i32(dev['segment_ids']), ops._i32(mask), ops._i32(dev['seq_len'])
    B, L = ids.shape
    lib = _lib.lib()
    nbytes = lib.ner_bert_bilstm_crf_predict_workspace_bytes(ctypes.byref(c), B, L, int(total), Hl, K)
    ws = _workspace(nbytes, ids.device)
    pred = torch.empty((B, L), dtype=torch.int32, device=ids.device)
    emb = [v[f"bert/embeddings/{n}"] for n in ("word_embeddings", "token_type_embeddings", "position_embeddings",
                                               "LayerNorm/gamma", "LayerNorm/beta")]
    _lib.check(lib.ner_bert_bilstm_crf_predict(
        ctypes.byref(c), *[t.data_ptr() for t in emb], arr, pk["wx"].data_ptr(), pk["bias"].data_ptr(), pk["wh_fw"].data_ptr(),
        pk["wh_bw"].data_ptr(), Hl, 1 if params['rnn_activation'] == 'relu' else 0, v["logits/kernel"].data_ptr(),
        v["logits/bias"].data_ptr(), v["crf_layer/transitions"].data_ptr(), K, ids.data_ptr(), m32.data_ptr(), seg.data_ptr(),
        sl.data_ptr(), B, L, int(total), pred.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream()))
    _lib.LAUNCHES += 5 + 7 * cfg["num_hidden_layers"]   # plan, embed, 7/layer, projection, recurrence, logits, Viterbi (+1 by check)
    return pred


FUSED_PREDICT = {"bert_bilstm_crf": bert_bilstm_crf_predict}
