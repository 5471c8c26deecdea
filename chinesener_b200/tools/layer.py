"""Layer library with the reference's function surface (reference tools/layer.py), each a thin
wrapper over the C-ABI kernels.  Same names, argument order and meaning; tensors are torch
CUDA tensors, variables live in `chinesener_b200.variables` under the reference's TF names.
"""
import os

import torch

from .. import autodiff
from .. import bert as _bert
from .. import ops, variables
from .. import windows as _windows

# Remove padding rows from the token-major activations of the BERT plugins (exact for loss and
# pred_ids: the CRF never reads t >= seq_len).  NER_B200_PACK=0 keeps the padded layout.
PACK_SEQUENCES = os.environ.get("NER_B200_PACK", "1") != "0"
# TRAIN mode of BertModel on the packed layout too (ner_bert_encoder_train_fwd_packed / _bwd_packed)
TRAIN_PACK = os.environ.get("NER_B200_TRAIN_PACK", "1") != "0"
# 'bf16': bf16 wgmma operands (BASELINE config 3, the benchmark path); 'fp32': fp32-accurate encoder (config 2's
# "fp32": split-bf16 dense + fp32 attention, emission logits within 1e-3 of the reference); 'fp8': PREDICT / EVAL only,
# the QKV and FFN GEMMs on block-scaled e4m3 wgmma (bert.bert_forward_fp8; TRAIN ignores it, as it does 'fp32').
# Estimator sets it from params['bert_precision'] around build_graph.
BERT_PRECISION = os.environ.get("NER_B200_BERT_PRECISION", "bf16")
# Document mode (chinesener_b200/windows.py): a batch longer than the window W is encoded as overlapping windows and stitched
# back.  None = the defaults (W = max_position_embeddings, S = (W - 2) // 2).  Estimator sets both from
# params['bert_window'] / params['bert_window_stride'], and DOCUMENT_REFUSAL to the reason a plugin cannot take document
# mode (windows.REFUSED), around build_graph.
BERT_WINDOW = None
BERT_WINDOW_STRIDE = None
DOCUMENT_REFUSAL = None
# N-best decoding: with CRF_NBEST > 1, crf_decode outside TRAIN also returns the CRF_NBEST best paths (as attributes of
# pred_ids, whose values stay the Viterbi path).  Estimator sets it from params['crf_nbest'] around build_graph.
CRF_NBEST = 1
# Knowledge distillation (Estimator(teacher=...)): CRF_TEACHER = (teacher logits [B,L,K], teacher transitions, alpha, tau)
# makes crf_layer in TRAIN return the row value (1 - alpha) ll - alpha tau^2 KL(teacher || student), so a plugin's
# (-ll).mean() is the distillation loss.  CRF_CAPTURE = [] makes crf_layer append its (logits, transitions) there and
# crf_decode decode nothing: how Estimator reads the teacher's potentials.  Estimator sets both around build_graph.
CRF_TEACHER = None
CRF_CAPTURE = None


class TrainingPathNotBuilt(NotImplementedError):
    pass


def pretrain_bert_embedding(input_ids, input_mask, segment_ids, pretrain_dir, drop_out, is_training):
    """reference tools/layer.py:63-81 — BertModel(...).get_sequence_output() (+ dropout when training).

    Returns sequence_output [B,L,H] f32; its bf16 copy (what the next GEMM consumes) rides along
    as attribute `.bf16`.  A batch longer than the window takes document mode (_document_embedding), with the same
    output layouts.
    """
    cfg = _bert.load_bert_config(pretrain_dir)
    B, L = input_ids.shape
    W, S = _windows.settings(BERT_WINDOW, BERT_WINDOW_STRIDE, cfg["max_position_embeddings"])
    if L > W:
        if DOCUMENT_REFUSAL:
            raise ValueError(DOCUMENT_REFUSAL)
        _windows.check_batch(None, L, W)
        return _document_embedding(input_ids, input_mask, segment_ids, cfg, W, S, drop_out, is_training)
    if is_training:
        tape = autodiff.current()
        if tape is None:
            raise TrainingPathNotBuilt("pretrain_bert_embedding(is_training=True) needs an autodiff tape (engine.train_step)")
        # TRAIN_PACK: the encoder runs on the real tokens only; its output keeps the [B,L,H] shape, zero at [PAD] (positions
        # no layer after it reads when PACK_SEQUENCES holds — plugins whose next layer does read them switch it off)
        pack = _bert.make_pack(input_mask) if (PACK_SEQUENCES and TRAIN_PACK and not _bert.PER_KERNEL) else None
        emb = _bert.bert_forward_train(input_ids, input_mask, segment_ids, cfg, variables.default_store(), tape, pack=pack)
        return dropout(emb, rate=drop_out, is_training=True, seed=1234)
    if BERT_PRECISION == 'fp32':
        return _bert.bert_forward_f32(input_ids, input_mask, segment_ids, cfg).view(B, L, -1)
    forward = _bert.bert_forward_fp8 if BERT_PRECISION == 'fp8' else _bert.bert_forward
    if PACK_SEQUENCES:
        pack = _bert.make_pack(input_mask)
        x32, x16 = forward(input_ids, input_mask, segment_ids, cfg, pack=pack)
        emb = x32                      # [total_tokens, H]: packed rows, see PackInfo
        emb.bf16, emb.pack = x16, pack
        return emb
    x32, x16 = forward(input_ids, input_mask, segment_ids, cfg)
    emb = x32.view(B, L, -1)
    emb.bf16 = x16.view(B, L, -1)
    return emb


def _document_embedding(input_ids, input_mask, segment_ids, cfg, W, S, drop_out, is_training):
    """Document mode of pretrain_bert_embedding: ner_window_plan cuts the documents into W-token windows, the encoder of
    the current mode runs on the window batch, and row gathers take each document token's row from its owner window.
    The result has the layouts of the plain path: packed [total_tokens, H] with .bf16 and .pack of the document mask, or
    [B, L, H] with zero rows at [PAD] (padded, fp32 and TRAIN).  TRAIN's stitch backward scatters each document row's
    gradient to its owner window row; window rows that own no token get zero."""
    B, L = input_ids.shape
    lengths = getattr(input_mask, "row_lengths", None)
    if lengths is None:
        lengths = input_mask.sum(1).cpu()                 # device sync; engine.Estimator attaches the host lengths
    NW, n_win = _windows.window_counts(lengths, W, S)
    n_doc = int(getattr(input_mask, "total_tokens", None) or sum(int(n) for n in lengths))
    doc_pack = _bert.make_pack(input_mask, n_doc)
    seq_len = input_mask.sum(1, dtype=torch.int32)
    train_pack = is_training and PACK_SEQUENCES and TRAIN_PACK and not _bert.PER_KERNEL
    packed = not is_training and PACK_SEQUENCES and BERT_PRECISION != 'fp32'
    plan = ops.window_plan(input_ids, segment_ids, seq_len, W, S, NW, n_doc, packed=packed, padded=not packed)
    ids, mask, seg = plan['ids'], plan['mask'], plan['segment_ids']
    mask.total_tokens = n_win

    def to_doc(rows, src):
        """window rows -> [B, L, H], zero at [PAD]"""
        H = rows.shape[-1]
        return ops.scatter_rows(ops.gather_rows(rows.reshape(-1, H), src, n_doc), doc_pack.tok_src, B * L).view(B, L, H)

    if is_training:
        tape = autodiff.current()
        if tape is None:
            raise TrainingPathNotBuilt("pretrain_bert_embedding(is_training=True) needs an autodiff tape (engine.train_step)")
        win_pack = _bert.make_pack(mask, n_win) if train_pack else None
        win = _bert.bert_forward_train(ids, mask, seg, cfg, variables.default_store(), tape, pack=win_pack)
        src = plan['doc_src_padded']
        emb = to_doc(win, src)
        n_rows, H = NW * W, win.shape[-1]

        def bwd(g):
            if g is not None:
                g_doc = ops.gather_rows(g.reshape(-1, H).contiguous(), doc_pack.tok_src, n_doc)
                tape.add_grad(win, ops.scatter_rows(g_doc, src, n_rows).view(win.shape))
        tape.record(emb, bwd)
        return dropout(emb, rate=drop_out, is_training=True, seed=1234)
    if BERT_PRECISION == 'fp32':
        return to_doc(_bert.bert_forward_f32(ids, mask, seg, cfg), plan['doc_src_padded'])
    forward = _bert.bert_forward_fp8 if BERT_PRECISION == 'fp8' else _bert.bert_forward
    if packed:
        x32, x16 = forward(ids, mask, seg, cfg, pack=_bert.make_pack(mask, n_win))
        src = plan['doc_src_packed']
        emb = ops.gather_rows(x32, src, n_doc)
        emb.bf16, emb.pack = ops.gather_rows(x16, src, n_doc), doc_pack
        return emb
    x32, x16 = forward(ids, mask, seg, cfg)
    emb = to_doc(x32, plan['doc_src_padded'])
    emb.bf16 = to_doc(x16, plan['doc_src_padded'])
    return emb


def dropout(inputs, rate, is_training, seed=1234):
    """tf.layers.dropout(inputs, rate=rate, seed=seed, training=is_training) — identity in eval mode.

    The mask is a counter-based hash of (seed, global_step, call index, element index): the backward
    pass regenerates it instead of storing it.  (TF's own RNG stream cannot be reproduced; the
    reference's seed=1234 only fixes ITS stream.)
    """
    if not is_training or rate <= 0.0:
        return inputs
    store = variables.default_store()
    store.dropout_calls += 1
    s = (int(seed) * 1000003 + store.global_step) * 1009 + store.dropout_calls
    keep = 1.0 - rate
    x = inputs.contiguous()
    y = ops.dropout(x, keep, s)
    tape = autodiff.current()
    if tape is not None and tape.needs_grad(inputs):
        def bwd(g):
            if g is not None:
                tape.add_grad(inputs, ops.dropout(g.contiguous(), keep, s))
        tape.record(y, bwd)
    return y


RNN_COLUMNS = {'lstm': 4, 'gru': 3}   # recurrent columns per hidden unit: LSTMCell (i, j, f, o), GRUCell (r, u, c)


def _rnn_config(cell_type, hidden_units_list, keep_prob_list, cell_size):
    """-> (cell, n_layers) after checking bilstm()'s RNN arguments.  The reference indexes hidden_units_list[i] and
    keep_prob_list[i] per layer (an IndexError there); here a list shorter than cell_size is a ValueError naming it."""
    cell = str(cell_type).lower()
    if cell not in RNN_COLUMNS:
        raise Exception(f"cell_type={cell_type!r}: only 'lstm' and 'gru' are built on the sm_90a path")
    n = int(cell_size)
    if n < 1:
        raise ValueError(f"cell_size must be >= 1, got {cell_size}")
    for name, lst in (("hidden_units_list", hidden_units_list), ("keep_prob_list", keep_prob_list)):
        if len(lst) < n:
            raise ValueError(f"{name} has {len(lst)} entries but cell_size={n} needs one per layer")
    return cell, n


def _rnn_names(scope, d, cell, i):
    """[(kernel, bias), ...] of layer i of direction d: one pair for LSTMCell, gates then candidate for GRUCell."""
    base = f"{scope}/{d}/multi_rnn_cell/cell_{i}"
    if cell == 'lstm':
        return [(f"{base}/lstm_cell/kernel", f"{base}/lstm_cell/bias")]
    return [(f"{base}/gru_cell/gates/kernel", f"{base}/gru_cell/gates/bias"),
            (f"{base}/gru_cell/candidate/kernel", f"{base}/gru_cell/candidate/bias")]


def _rnn_variables(store, scope, cell, i, Din, H):
    """Create layer i of both directions under the reference's names -> {d: _rnn_names(...)}.  Initialisers as TF:
    glorot_uniform kernels, zero LSTM bias, GRU gates bias 1.0 and candidate bias 0."""
    names = {d: _rnn_names(scope, d, cell, i) for d in ("fw", "bw")}
    for d in ("fw", "bw"):
        if cell == 'lstm':
            store.get_variable(names[d][0][0], (Din + H, 4 * H), variables.glorot_uniform)
            store.get_variable(names[d][0][1], (4 * H,), variables.zeros)
        else:
            store.get_variable(names[d][0][0], (Din + H, 2 * H), variables.glorot_uniform)
            store.get_variable(names[d][0][1], (2 * H,), variables.ones)
            store.get_variable(names[d][1][0], (Din + H, H), variables.glorot_uniform)
            store.get_variable(names[d][1][1], (H,), variables.zeros)
    return names


def _rnn_kernels(store, names):
    """[Din + H, G*H] per direction: the cell's kernels side by side (GRU: [gates | candidate], columns r, u, c)."""
    return [torch.cat([store.vars[k] for k, _ in names[d]], dim=1) if len(names[d]) > 1 else store.vars[names[d][0][0]]
            for d in ("fw", "bw")]


def _rnn_input_kernel(ks, Din, split):
    """Input half of both directions -> f32 [D, 2GH] (fw columns | bw columns).  split: the layer reads [fw | bw] of the
    layer below and each direction only its own half, so the kernel is block-diagonal (D = 2 Din)."""
    if not split:
        return torch.cat([k[:Din] for k in ks], dim=1)
    G = ks[0].shape[1]
    wx = torch.zeros((2 * Din, 2 * G), dtype=torch.float32, device=ks[0].device)
    wx[:Din, :G] = ks[0][:Din]
    wx[Din:, G:] = ks[1][:Din]
    return wx


def _rnn_pack(store, names, Din, split):
    """bf16 [Np, Dp] input-projection pack (fw | bw), fused bias [Np], fp32 recurrent matrices [H, GH].  Np = 2GH, padded
    with zero columns to the GEMM's 32-column granule (GRU with H % 16 != 0; the recurrence reads the row stride)."""
    D = 2 * Din if split else Din
    Dp = (D + 7) // 8 * 8

    def build():
        ks = _rnn_kernels(store, names)
        bs = [store.vars[b] for d in ("fw", "bw") for _, b in names[d]]
        wx = _rnn_input_kernel(ks, Din, split)
        N = wx.shape[1]
        Np = (N + 31) // 32 * 32
        if Dp != D or Np != N:
            wx = torch.nn.functional.pad(wx, (0, Np - N, 0, Dp - D))    # zero rows for the K padding, columns for N
        bias = torch.cat(bs)
        if Np != N:
            bias = torch.nn.functional.pad(bias, (0, Np - N))
        return dict(wx=ops.pack_weight_bf16(wx.contiguous()), bias=bias.contiguous(),
                    wh_fw=ks[0][Din:].contiguous(), wh_bw=ks[1][Din:].contiguous(), Dp=Dp)
    return store.cached(("rnn_pack", names["fw"][0][0], Din, split), build)


def bilstm(embedding, cell_type, activation, hidden_units_list, keep_prob_list, cell_size, seq_len, dtype, is_training):
    """reference tools/layer.py:27-41 — bidirectional_dynamic_rnn over a MultiRNNCell of `cell_size` DropoutWrapper-ed
    LSTMCell / GRUCell layers; -> [B,L,2H] f32 of the top layer.

    The fw and bw stacks are independent: layer i+1 of a direction reads layer i of the same direction (not the
    [fw | bw] concat torch.nn.LSTM(bidirectional=True) feeds forward), through one GEMM with a block-diagonal weight.
    Layer i has hidden_units_list[i] units and keep_prob_list[i] (TRAIN) on its output and carried state, each layer
    with its own dropout seed.  PREDICT keeps a packed BERT layout for layer 0; upper layers read the padded output."""
    cell, n = _rnn_config(cell_type, hidden_units_list, keep_prob_list, cell_size)
    scope = variables.scoped("bilstm_layer/bidirectional_rnn")
    x = embedding
    for i in range(n):
        H = int(hidden_units_list[i])
        if is_training:
            x = _rnn_layer_train(x, cell, i, scope, activation, H, float(keep_prob_list[i]), seq_len)
        else:
            x = _rnn_layer_predict(x, cell, i, scope, activation, H, seq_len)
    return x


def _rnn_layer_predict(embedding, cell, i, scope, activation, H, seq_len):
    pack = getattr(embedding, "pack", None)
    if pack is not None:
        B, L, D = pack.B, pack.L, embedding.shape[-1]
    else:
        B, L, D = embedding.shape
    Din = D if i == 0 else D // 2
    store = variables.default_store()
    names = _rnn_variables(store, scope, cell, i, Din, H)
    pk = _rnn_pack(store, names, Din, i > 0)
    x16 = getattr(embedding, "bf16", None)
    if x16 is not None and pk["Dp"] == D:
        x16 = x16.reshape(-1, D)
    else:
        x16 = ops.cast_pad_bf16(embedding.reshape(-1, D), pk["Dp"])
    xproj = ops.gemm_bf16(x16, pk["wx"], pk["bias"], epilogue=ops.EPI_F32)
    cu = pack.cu_seqlens if pack is not None else None
    if cell == 'lstm':
        return ops.bilstm_recurrence(xproj, pk["wh_fw"], pk["wh_bw"], seq_len, B, L, H, activation=activation,
                                     forget_bias=1.0, cu_seqlens=cu)
    return ops.bigru_recurrence(xproj, pk["wh_fw"], pk["wh_bw"], seq_len, B, L, H, activation=activation, cu_seqlens=cu)


def _rnn_layer_train(embedding, cell, i, scope, activation, H, keep, seq_len):
    """Training-mode layer i: same kernels on the padded layout, saves what BPTT reads and records the backward closure.
    keep < 1 = DropoutWrapper(output_keep_prob, state_keep_prob) (reference tools/layer.py:20-23): counter-based masks
    inside the recurrence kernels."""
    B, L, D = embedding.shape
    split = i > 0
    Din = D // 2 if split else D
    G = RNN_COLUMNS[cell] * H
    store = variables.default_store()
    names = _rnn_variables(store, scope, cell, i, Din, H)
    pk = _rnn_pack(store, names, Din, split)
    x2d = embedding.reshape(B * L, D).contiguous()
    x16 = ops.cast_pad_bf16(x2d, pk["Dp"])
    xproj = ops.gemm_bf16(x16, pk["wx"], pk["bias"], epilogue=ops.EPI_F32)
    store.dropout_calls += 1
    seed = (1234 * 1000003 + store.global_step) * 1009 + store.dropout_calls
    if cell == 'lstm':
        out, gates, cst, hst = ops.bilstm_recurrence(xproj, pk["wh_fw"], pk["wh_bw"], seq_len, B, L, H,
                                                     activation=activation, forget_bias=1.0, save_for_backward=True,
                                                     keep_prob=keep, seed=seed)
    else:
        out, gates, hst, rh = ops.bigru_recurrence(xproj, pk["wh_fw"], pk["wh_bw"], seq_len, B, L, H,
                                                   activation=activation, save_for_backward=True, keep_prob=keep,
                                                   seed=seed)
    tape = autodiff.current()
    if tape is not None:
        need_dx = tape.needs_grad(embedding)

        def bwd(g):
            if g is None:
                return
            if cell == 'lstm':
                dxp = ops.bilstm_recurrence_bwd(g.contiguous(), gates, cst, pk["wh_fw"], pk["wh_bw"], seq_len, B, L, H,
                                                activation=activation, keep_prob=keep, seed=seed)
            else:
                dxp = ops.bigru_recurrence_bwd(g.contiguous(), gates, hst, pk["wh_fw"], pk["wh_bw"], seq_len, B, L, H,
                                               activation=activation, keep_prob=keep, seed=seed)
            dxp16 = ops.cast_bf16(dxp)
            for di, d in enumerate(("fw", "bw")):
                col = di * G
                for k, b in names[d]:
                    n_col = store.vars[b].shape[0]
                    ops.colsum_add(dxp[:, col:col + n_col], store.grad(b), 1.0)
                    col += n_col
            gks = [store.grad(names[d][0][0]) for d in ("fw", "bw")]
            grouped = cell == 'lstm' and not split and pk["Dp"] == D and D % 128 == 0 and H % 128 == 0 \
                and (4 * H) % 256 == 0 and all(k.is_contiguous() for k in gks)
            if grouped:
                # dW_x (both directions) and dW_h (both directions) as ONE grouped launch: token-major operands read in place
                # (ner_wgrad_group_bf16) instead of fp32 transposes + three stream-K GEMMs
                hprev16 = torch.zeros((2, B, L, H), dtype=torch.bfloat16, device=out.device)
                hprev16[0, :, 1:] = hst[:, :-1, :H]          # carried (state-dropped) h of the previous forward step
                hprev16[1, :, :-1] = hst[:, 1:, H:]
                probs = []
                for di in range(2):
                    probs.append((x16, dxp16, di * 4 * H, gks[di][:D]))
                    probs.append((hprev16[di].view(B * L, H), dxp16, di * 4 * H, gks[di][D:]))
                ops.wgrad_group(probs, B * L)
            else:
                dwx = ops.wgrad_gemm(x2d, dxp)                                   # [D, 2GH] = x^T d_xproj
                for di, d in enumerate(("fw", "bw")):
                    dz = dxp[:, di * G:(di + 1) * G]
                    rows = slice(di * Din, (di + 1) * Din) if split else slice(0, Din)
                    hprev = torch.zeros((B, L, H), dtype=torch.float32, device=out.device)
                    if di == 0:                       # carried (state-dropped) h of the previous forward step
                        hprev[:, 1:] = hst[:, :-1, :H]
                    else:
                        hprev[:, :-1] = hst[:, 1:, H:]
                    if cell == 'lstm':
                        gks[di][:Din] += dwx[rows, di * G:(di + 1) * G]
                        gks[di][Din:] += ops.wgrad_gemm(hprev.view(B * L, H), dz)   # dW_h = h_prev^T dz
                    else:
                        gc = store.grad(names[d][1][0])
                        gks[di][:Din] += dwx[rows, di * G:di * G + 2 * H]
                        gc[:Din] += dwx[rows, di * G + 2 * H:(di + 1) * G]
                        gks[di][Din:] += ops.wgrad_gemm(hprev.view(B * L, H), dz[:, :2 * H])   # dW_g^h = h_prev^T da_g
                        rh_d = rh.view(B * L, 2 * H)[:, di * H:(di + 1) * H]
                        gc[Din:] += ops.wgrad_gemm(rh_d, dz[:, 2 * H:])                     # dW_c^h = (r h_prev)^T da_c
            if need_dx:
                wx = _rnn_input_kernel(_rnn_kernels(store, names), Din, split)       # [D, 2GH]: K-major for dx
                Dn = (D + 31) // 32 * 32
                wxp = torch.nn.functional.pad(wx, (0, 0, 0, Dn - D)).to(torch.bfloat16).contiguous()
                dx = ops.gemm_bf16(dxp16, wxp, None, epilogue=ops.EPI_F32)[:, :D]
                tape.add_grad(embedding, dx.reshape(B, L, D).contiguous())
        tape.record(out, bwd)
    return out


LATTICE_PARTS = ("char_cell", "word_cell", "alpha")


def _lattice_variables(store, scope, Ec, Ew, H):
    """{d: {part: (kernel, bias)}} of the lattice layer, created fw then bw: char_cell [Ec+H, 3H] (i, o, g), word_cell
    [Ew+H, 3H] (f, i, g), alpha [Ec+H, H]; glorot-uniform kernels, zero biases."""
    names = {}
    for d in ("fw", "bw"):
        names[d] = {}
        for part, din, n in (("char_cell", Ec, 3 * H), ("word_cell", Ew, 3 * H), ("alpha", Ec, H)):
            k, b = f"{scope}/{d}/{part}/kernel", f"{scope}/{d}/{part}/bias"
            store.get_variable(k, (din + H, n), variables.glorot_uniform)
            store.get_variable(b, (n,), variables.zeros)
            names[d][part] = (k, b)
    return names


def _pack_kn(w, b):
    """[K, N] f32 kernel + [N] bias -> (bf16 [Np, Kp] GEMM operand, f32 [Np] bias, Kp, Np): K padded to 8, N to 32."""
    K, N = w.shape
    Kp, Np = (K + 7) // 8 * 8, (N + 31) // 32 * 32
    w = torch.nn.functional.pad(w, (0, Np - N, 0, Kp - K))
    return ops.pack_weight_bf16(w.contiguous()), torch.nn.functional.pad(b, (0, Np - N)).contiguous(), Kp, Np


def _lattice_pack(store, names, Ec, Ew, H):
    def build():
        v = store.vars
        k = {d: {p: v[names[d][p][0]] for p in LATTICE_PARTS} for d in ("fw", "bw")}
        b = {d: {p: v[names[d][p][1]] for p in LATTICE_PARTS} for d in ("fw", "bw")}
        wx = torch.cat([torch.cat([k[d]["char_cell"][:Ec], k[d]["alpha"][:Ec]], 1) for d in ("fw", "bw")], 1)   # [Ec, 8H]
        bx = torch.cat([torch.cat([b[d]["char_cell"], b[d]["alpha"]]) for d in ("fw", "bw")])
        ww = torch.cat([k[d]["word_cell"][:Ew] for d in ("fw", "bw")], 1)                                      # [Ew, 6H]
        bw = torch.cat([b[d]["word_cell"] for d in ("fw", "bw")])
        xc, xcb, Kc, _ = _pack_kn(wx, bx)
        xw, xwb, Kw_, _ = _pack_kn(ww, bw)
        return dict(wx=wx, ww=ww, xc=xc, xcb=xcb, Kc=Kc, xw=xw, xwb=xwb, Kw=Kw_,
                    wrec={d: torch.cat([k[d]["char_cell"][Ec:], k[d]["word_cell"][Ew:]], 1).contiguous() for d in ("fw", "bw")},
                    wac={d: k[d]["alpha"][Ec:].contiguous() for d in ("fw", "bw")})
    return store.cached(("lattice_pack", names["fw"]["char_cell"][0], Ec, Ew), build)


def _proj(x2d, w16, bias, Kp, N):
    """x [M, K] f32 @ packed weight + bias -> f32 [M, N] (bf16 operands, fp32 accumulate)."""
    y = ops.gemm_bf16(ops.cast_pad_bf16(x2d, Kp), w16, bias, epilogue=ops.EPI_F32)
    return y if y.shape[1] == N else y[:, :N].contiguous()


def _input_grad(dy, w_kn):
    """dx [M, K] = dy [M, N] · w [K, N]^T on the tensor cores."""
    K, N = w_kn.shape
    Np, Kp = (N + 7) // 8 * 8, (K + 31) // 32 * 32
    wt = torch.nn.functional.pad(w_kn, (0, Np - N, 0, Kp - K)).to(torch.bfloat16).contiguous()
    return ops.gemm_bf16(ops.cast_pad_bf16(dy, Np), wt, None, epilogue=ops.EPI_F32)[:, :K]


def lattice_lstm(char_input, word_input, lattice_lens, hidden_units, seq_len, is_training):
    """Bidirectional Lattice LSTM (Zhang & Yang, ACL 2018) as defined in model/lattice_lstm_crf.py -> [B, L, 2H] f32.

    char_input [B, L, Ec] f32; word_input [B*L, Kw*Ew] f32: the embedding of word slot (b, p, k) in row b*L + p, columns
    k*Ew.. (zero rows for empty slots are fine); lattice_lens int32 [B, L*Kw]: slot lengths, a slot is empty when its length
    is outside [2, 10] or the word reaches past seq_len.  The char/alpha and word-cell input projections are bf16 GEMMs
    (fp32 accumulate) for both directions; the recurrence is ner_lattice_recurrence.  TRAIN records the backward:
    ner_lattice_recurrence_bwd, then every weight and bias gradient as a GEMM over its outputs (no float atomics)."""
    B, L, Ec = char_input.shape
    H = int(hidden_units)
    Kw = lattice_lens.shape[1] // L
    Ew = word_input.shape[1] // Kw
    store = variables.default_store()
    names = _lattice_variables(store, variables.scoped("lattice_layer"), Ec, Ew, H)
    pk = _lattice_pack(store, names, Ec, Ew, H)
    x2d = char_input.reshape(B * L, Ec).contiguous()
    w2d = word_input.reshape(B * L * Kw, Ew).contiguous()
    xproj = _proj(x2d, pk["xc"], pk["xcb"], pk["Kc"], 8 * H)
    wproj = _proj(w2d, pk["xw"], pk["xwb"], pk["Kw"], 6 * H)
    lens = lattice_lens.to(torch.int32).contiguous()
    args = (lens, pk["wrec"]["fw"], pk["wrec"]["bw"], pk["wac"]["fw"], pk["wac"]["bw"], seq_len, B, L, H, Kw)
    tape = autodiff.current() if is_training else None
    if tape is None:
        return ops.lattice_recurrence(xproj, wproj, *args)
    out, saved = ops.lattice_recurrence(xproj, wproj, *args, save_for_backward=True)
    need_dc, need_dw = tape.needs_grad(char_input), tape.needs_grad(word_input)

    def bwd(g):
        if g is None:
            return
        dxp, dwp, dal = ops.lattice_recurrence_bwd(g.contiguous(), saved, *args)
        gr = store.grad
        dwx = ops.wgrad_gemm(x2d, dxp)            # [Ec, 8H]
        dww = ops.wgrad_gemm(w2d, dwp)            # [Ew, 6H]
        db_x = ops.wgrad_gemm(torch.ones((B * L, 8), dtype=torch.float32, device=out.device), dxp)
        db_w = ops.wgrad_gemm(torch.ones((B * L * Kw, 8), dtype=torch.float32, device=out.device), dwp)
        for di, d in enumerate(("fw", "bw")):
            nm = names[d]
            c0, w0 = di * 4 * H, di * 3 * H
            hprev = torch.zeros((B, L, H), dtype=torch.float32, device=out.device)
            if di == 0:
                hprev[:, 1:] = out[:, :-1, :H]
            else:
                hprev[:, :-1] = out[:, 1:, H:]
            dz_c, da_x, dz_w = dxp[:, c0:c0 + 3 * H], dxp[:, c0 + 3 * H:c0 + 4 * H], dwp[:, w0:w0 + 3 * H]
            # bias gradients as GEMMs against a ones operand: fixed summation order, so repeats are bit-identical
            gr(nm["char_cell"][1]).add_(db_x[0, c0:c0 + 3 * H])
            gr(nm["alpha"][1]).add_(db_x[0, c0 + 3 * H:c0 + 4 * H])
            gr(nm["word_cell"][1]).add_(db_w[0, w0:w0 + 3 * H])
            gc, gw, ga = gr(nm["char_cell"][0]), gr(nm["word_cell"][0]), gr(nm["alpha"][0])
            gc[:Ec] += dwx[:, c0:c0 + 3 * H]
            ga[:Ec] += dwx[:, c0 + 3 * H:c0 + 4 * H]
            gw[:Ew] += dww[:, w0:w0 + 3 * H]
            gc[Ec:] += ops.wgrad_gemm(hprev.view(B * L, H), dz_c)                                   # h_prev^T dz
            gw[Ew:] += ops.wgrad_gemm(saved["hw"][:, di * H:(di + 1) * H], dz_w)                    # h_start^T dz_w
            ga[Ec:] += ops.wgrad_gemm(saved["cw"][:, di * H:(di + 1) * H], dal[:, di * H:(di + 1) * H])   # C^w^T da
        if need_dc:
            tape.add_grad(char_input, _input_grad(dxp, pk["wx"]).reshape(B, L, Ec).contiguous())
        if need_dw:
            tape.add_grad(word_input, _input_grad(dwp, pk["ww"]).reshape(word_input.shape).contiguous())
    tape.record(out, bwd)
    return out


def cnn_layer(embedding, filter_list, kernel_size_list, activation, drop_out, is_training):
    """reference tools/layer.py:44-60 — tf.layers.conv1d(padding='SAME') per kernel size (+ dropout), concatenated.
    A kernel-k convolution over [B, L, C] is the label-projection kernel (ner_dense_small_n, filters <= 32) applied to the
    k shifted copies of the sequence laid side by side (TF 'SAME': (k-1)//2 zero rows before, k//2 after); the shifts are
    slices of one zero-padded buffer.  TRAIN: the same kernel's backward tap by tap, the shifted gradient slices are added back."""
    if activation not in ('relu', None):
        raise Exception("cnn_layer: only activation='relu' / None is built")
    B, L, C = embedding.shape
    store, tape = variables.default_store(), (autodiff.current() if is_training else None)
    x = embedding.float() if embedding.dtype != torch.float32 else embedding
    outputs = []
    for filters, k in zip(filter_list, kernel_size_list):
        name = f"cnn_kernel{k}"
        w = store.get_variable(f"{name}/kernel", (k, C, filters), variables.glorot_uniform)       # TF conv1d kernel [k, in, out]
        b = store.get_variable(f"{name}/bias", (filters,), variables.zeros)
        pl, pr = (k - 1) // 2, k // 2
        xp = torch.nn.functional.pad(x, (0, 0, pl, pr))
        cols = torch.cat([xp[:, j:j + L] for j in range(k)], dim=-1).reshape(B * L, k * C).contiguous()
        w2d = w.reshape(k * C, filters)
        pre = ops.dense_small_n(cols, w2d, b)
        out = ops.relu(pre) if activation == 'relu' else pre
        if tape is not None:
            need_dx = tape.needs_grad(embedding)

            def bwd(g, xp=xp, w=w, out=out, name=name, k=k, pl=pl):
                if g is None:
                    return
                g = g.reshape(B * L, -1).contiguous()
                if activation == 'relu':
                    g = ops.relu_bwd(out, g)
                dW, db = store.grad(f"{name}/kernel"), store.grad(f"{name}/bias")
                dxp = torch.zeros_like(xp) if need_dx else None
                for j in range(k):            # one tap at a time: [C, filters] weight + its partial fit the kernel's smem
                    xj = xp[:, j:j + L].reshape(B * L, C)
                    dxj = ops.dense_small_n_bwd(xj, w[j], g, dW[j], db if j == 0 else None, want_dx=need_dx)
                    if need_dx:
                        dxp[:, j:j + L] += dxj.view(B, L, C)
                if need_dx:
                    tape.add_grad(embedding, dxp[:, pl:pl + L].contiguous())
            tape.record(out, bwd)
        out = dropout(out, drop_out, is_training, seed=1234)
        out3 = out.view(B, L, filters)
        if tape is not None:                      # the tape keys on tensor identity: record the reshape
            tape.record(out3, lambda g, out=out: tape.add_grad(out, g.reshape(out.shape)) if g is not None else None)
        outputs.append(out3)
    output = outputs[0] if len(outputs) == 1 else torch.cat(outputs, dim=-1)
    if tape is not None and len(outputs) > 1:
        widths = [o.shape[-1] for o in outputs]

        def cat_bwd(g):
            if g is not None:
                off = 0
                for o, wd in zip(outputs, widths):
                    tape.add_grad(o, g[..., off:off + wd].contiguous())
                    off += wd
        tape.record(output, cat_bwd)
    return output


def _dense_wide_pack(store, name, F, N, for_dx=False):
    """Split-bf16 (hi, lo) weight operands of ner_gemm_bf16 from `name/kernel` [F, N], zero-padded; rebuilt when the
    store's variables change.  Forward: packs of W, [Np, Fp] (N padded to the GEMM's 32-column granule, F to 8).
    for_dx: packs of W^T, [Fo, Np] (F padded to 32), the operand of dx = dy·W^T."""
    Fp, Fo, Np = (F + 7) // 8 * 8, (F + 31) // 32 * 32, (N + 31) // 32 * 32

    def build():
        w = variables.default_store().vars[f"{name}/kernel"]
        w = (torch.nn.functional.pad(w, (0, Np - N, 0, Fo - F)).t() if for_dx
             else torch.nn.functional.pad(w, (0, Np - N, 0, Fp - F))).contiguous()
        hi = ops.pack_weight_bf16(w)
        lo = ops.pack_weight_bf16((w - hi.float().t()).contiguous())
        return hi, lo
    return store.cached(("dense_wide_pack", name, F, N, for_dx), build)


def _dense_wide(inputs, units, name, b, is_training):
    """dense() for units > 32: the fp32-accurate split-bf16 wgmma GEMM of the transformer plugins (A_hi·W_hi + A_hi·W_lo +
    A_lo·W_hi), on N padded to 32 columns and sliced.  TRAIN records db = colsum(dy) in fp32, dW = x^T·dy on bf16
    operands (fp32 accumulation) as tools/transformer/modules.py's dense_train does, and dx = dy·W^T on the same split
    GEMM as the forward, so the gradient that reaches the encoder keeps fp32 accuracy."""
    F = inputs.shape[-1]
    lead = inputs.shape[:-1]
    store = variables.default_store()
    x2d = inputs.reshape(-1, F).contiguous()
    w_hi, w_lo = _dense_wide_pack(store, name, F, units)
    a_hi, a_lo = ops.split_bf16(x2d, w_hi.shape[1])
    Np = w_hi.shape[0]
    bias = torch.nn.functional.pad(b, (0, Np - units)) if Np != units else b
    y = ops.gemm_split_f32(a_hi, a_lo, w_hi, w_lo, bias)[:, :units]
    pack = getattr(inputs, "pack", None)
    if pack is not None:                  # packed rows -> padded [B, L, units]; padded positions stay 0
        out = ops.scatter_rows(y.contiguous(), pack.tok_src[:x2d.shape[0]], pack.B * pack.L)
        return out.view(pack.B, pack.L, units)
    out = y.contiguous().view(*lead, units)
    tape = autodiff.current()
    if is_training and tape is not None:
        need_dx = tape.needs_grad(inputs)

        def bwd(g):
            if g is None:
                return
            g2d = g.reshape(-1, units).contiguous()
            ops.colsum_add(g2d, store.grad(f"{name}/bias"))
            ops.wgrad_gemm(x2d, g2d, out=store.grad(f"{name}/kernel"))
            if need_dx:
                wt_hi, wt_lo = _dense_wide_pack(store, name, F, units, for_dx=True)
                g_hi, g_lo = ops.split_bf16(g2d, Np)
                dx = ops.gemm_split_f32(g_hi, g_lo, wt_hi, wt_lo)[:, :F]
                tape.add_grad(inputs, dx.contiguous().view(*lead, F))
        tape.record(out, bwd)
    return out


def dense(inputs, units, name='logits', is_training=False):
    """tf.layers.dense(inputs, units, activation=None, use_bias=True, name=name): ner_dense_small_n for units <= 32,
    the split-bf16 tensor-core GEMM above that."""
    F = inputs.shape[-1]
    lead = inputs.shape[:-1]
    name = variables.scoped(name)
    w = variables.get_variable(f"{name}/kernel", (F, units), variables.glorot_uniform)
    b = variables.get_variable(f"{name}/bias", (units,), variables.zeros)
    if units > 32:
        return _dense_wide(inputs, units, name, b, is_training)
    tape = autodiff.current()
    if is_training and tape is not None:
        store = variables.default_store()
        x2d = inputs.reshape(-1, F).contiguous()
        out = ops.dense_small_n(x2d, w, b).view(*lead, units)
        need_dx = tape.needs_grad(inputs)

        def bwd(g):
            if g is None:
                return
            dx = ops.dense_small_n_bwd(x2d, w, g.reshape(-1, units).contiguous(), store.grad(f"{name}/kernel"),
                                       store.grad(f"{name}/bias"), want_dx=need_dx)
            if need_dx:
                tape.add_grad(inputs, dx.view(*lead, F))
        tape.record(out, bwd)
        return out
    x = getattr(inputs, "bf16", None)
    x = inputs if x is None else x
    pack = getattr(inputs, "pack", None)
    if pack is not None:
        # packed rows -> padded [B, L, units]; padded positions stay 0 (never read by the CRF)
        out = torch.zeros((pack.B * pack.L, units), dtype=torch.float32, device=x.device)
        ops.dense_small_n(x.reshape(-1, F), w, b, row_map=pack.tok_src, out=out)
        return out.view(pack.B, pack.L, units)
    out = ops.dense_small_n(x.reshape(-1, F), w, b)
    return out.view(*lead, units)


def crf_layer(logits, label_ids, seq_len, label_size, is_training, label_mask=None):
    """reference tools/layer.py:112-131 -> (trans, log_likelihood [B]).

    label_mask [B, L] int32 (partially annotated batches): bit j of label_mask[b, t] allows tag j at t, and the
    log-likelihood is that of the partial-annotation CRF (ner_crf_partial_loglik_fwd); label_ids is then not read."""
    tname = variables.scoped("crf_layer/transitions")
    trans = variables.get_variable(tname, (label_size, label_size), variables.xavier)
    if CRF_CAPTURE is not None and not is_training:
        CRF_CAPTURE.append((logits, trans))
    if label_ids is None:
        return trans, None
    if label_mask is None:
        fwd, bwd_op, labels = ops.crf_loglik_fwd, ops.crf_loglik_bwd, label_ids
    else:
        fwd, bwd_op, labels = ops.crf_partial_loglik_fwd, ops.crf_partial_loglik_bwd, label_mask
    tape = autodiff.current()
    if is_training and tape is not None and CRF_TEACHER is not None:
        return trans, _distilled_loglik(logits, labels, seq_len, trans, tname, fwd, bwd_op, tape)
    if is_training and tape is not None:
        store = variables.default_store()
        lg = logits.contiguous()
        ll, logz, alpha = fwd(lg, labels, seq_len, trans, want_alpha=True)

        def bwd(g):
            # g = d loss / d ll  [B]; the plugins use loss = mean(-ll)  ->  g = -1/B
            B = lg.shape[0]
            d_ll = g if g is not None else torch.full((B,), -1.0 / B, dtype=torch.float32, device=lg.device)
            d_logits, d_trans = bwd_op(lg, labels, seq_len, trans, alpha, logz, d_ll.contiguous(), 1.0)
            store.grad(tname).add_(d_trans)
            tape.add_grad(logits, d_logits)
        tape.record(ll, bwd)
        return trans, ll
    # EVAL / PREDICT: built lazily — evaluated when the loss is fetched (EVAL), never in PREDICT
    return trans, variables.Deferred(lambda: fwd(logits, labels, seq_len, trans)[0])


def _distilled_loglik(logits, labels, seq_len, trans, tname, fwd, bwd_op, tape):
    """TRAIN row value ll' = (1 - a) ll - a tau^2 KL_b with CRF_TEACHER = (t_logits, t_trans, a, tau), and its tape entry.
    KL_b is written by the distillation backward kernel, so that kernel runs here, with the coefficient the plugins'
    (-ll').mean() gives it (a tau^2 / B); a tape that seeds another gradient reruns it with that one.  The gold term is
    skipped at a = 1.  The teacher's potentials get no gradient."""
    t_logits, t_trans, a, tau = CRF_TEACHER
    store = variables.default_store()
    lg = logits.contiguous()
    B = lg.shape[0]
    c = float(a) * float(tau) ** 2
    logz_d, alpha_d = ops.crf_distill_fwd(t_logits, t_trans, lg, trans, seq_len, tau)
    kl, dl_kl, dt_kl = ops.crf_distill_bwd(t_logits, t_trans, lg, trans, seq_len, alpha_d, logz_d, tau, scale=c / B)
    gold = None
    row = kl * -c
    if a < 1:
        gold = fwd(lg, labels, seq_len, trans, want_alpha=True)
        row = row + gold[0] * (1.0 - a)

    def bwd(g):
        if g is None:                       # loss = mean(-ll'): d loss / d ll'_b = -1/B
            d_logits, d_trans = dl_kl, dt_kl
        else:
            _, d_logits, d_trans = ops.crf_distill_bwd(t_logits, t_trans, lg, trans, seq_len, alpha_d, logz_d, tau,
                                                       d_kl=(g * -c).contiguous())
        if gold is not None:
            d_ll = g if g is not None else torch.full((B,), -1.0 / B, dtype=torch.float32, device=lg.device)
            dl_g, dt_g = bwd_op(lg, labels, seq_len, trans, gold[2], gold[1], d_ll.contiguous(), 1.0 - a)
            d_logits, d_trans = d_logits + dl_g, d_trans + dt_g
        store.grad(tname).add_(d_trans)
        tape.add_grad(logits, d_logits)
    tape.record(row, bwd)
    return row


def concat(tensors, is_training=False):
    """tf.concat(tensors, axis=-1) with the tape entry that splits the gradient back."""
    out = torch.cat(tensors, dim=-1)
    tape = autodiff.current() if is_training else None
    if tape is not None:
        widths = [t.shape[-1] for t in tensors]

        def bwd(g):
            if g is not None:
                off = 0
                for t, wd in zip(tensors, widths):
                    tape.add_grad(t, g[..., off:off + wd].contiguous())
                    off += wd
        tape.record(out, bwd)
    return out


def reduce_max_flip(x, shrink, is_training):
    """flip_gradient(tf.reduce_max(x, axis=1), shrink) (reference model/bert_bilstm_crf_adv.py:35-37,
    tools/train_utils.py:47-63): max over time forward; backward sends -shrink * g to every position that attains it."""
    x = x.contiguous()
    y = ops.reduce_max_time(x)
    tape = autodiff.current() if is_training else None
    if tape is not None and tape.needs_grad(x):
        def bwd(g):
            if g is not None:
                tape.add_grad(x, ops.reduce_max_time_bwd(x, y, g.contiguous(), torch.zeros_like(x), scale=-float(shrink)))
        tape.record(y, bwd)
    return y


def softmax_cross_entropy_mean(logits, labels, weight, is_training):
    """weight * tf.reduce_mean(tf.nn.sparse_softmax_cross_entropy_with_logits(labels, logits)); a loss root: TRAIN seeds
    d/d logits = weight / B * (softmax - onehot) on the tape."""
    B = logits.shape[0]
    tape = autodiff.current() if is_training else None
    lg = logits.contiguous()
    if tape is None:
        return ops.softmax_xent(lg, labels).mean() * weight
    xent, dz = ops.softmax_xent(lg, labels, scale=float(weight) / B, want_grad=True)
    loss = xent.mean() * weight
    tape.record(loss, lambda g: tape.add_grad(logits, dz))
    return loss


def masked_task_loss(log_likelihoods, masks, weights, batch_size, is_training):
    """sum_t w_t * sum(-ll_t[mask_t]) / batch — the loss of the multi-task plugins (reference
    model/bert_bilstm_crf_mtl.py:42,61,64).  TRAIN: seeds d loss / d ll_t = -w_t mask_t / batch on the tape."""
    coef = [m.to(torch.float32) * (float(w) / batch_size) for m, w in zip(masks, weights)]
    tape = autodiff.current() if is_training else None
    if tape is None:
        return variables.Deferred(lambda: sum((-(ll.value() if isinstance(ll, variables.Deferred) else ll) * c).sum()
                                              for ll, c in zip(log_likelihoods, coef)))
    loss = sum((-ll * c).sum() for ll, c in zip(log_likelihoods, coef))

    def bwd(g):
        for ll, c in zip(log_likelihoods, coef):
            tape.add_grad(ll, -c)
    tape.record(loss, bwd)
    return loss


def crf_decode(logits, trans, seq_len, idx2tag, is_training, mask=None):
    """reference tools/layer.py:134-149 -> pred_ids [B,L] int32, zero beyond seq_len.

    CRF_NBEST > 1 (PREDICT / EVAL): pred_ids is rank 0 of ops.crf_viterbi_nbest, the same tags, and carries the
    CRF_NBEST best paths as .nbest_ids [B,N,L] int32, .nbest_scores [B,N] f32, .nbest_counts [B] int32 and .nbest_logz
    [B] f32 (log Z of ner_crf_loglik_fwd), so that path r has probability exp(nbest_scores[:, r] - nbest_logz)."""
    if CRF_CAPTURE is not None and not is_training:
        return torch.zeros(logits.shape[:2], dtype=torch.int32, device=logits.device)
    if CRF_NBEST <= 1 or is_training:
        return ops.crf_viterbi(logits, seq_len, trans)
    tags, scores, counts = ops.crf_viterbi_nbest(logits, seq_len, trans, CRF_NBEST)
    pred = tags[:, 0].contiguous()
    logz = ops.crf_loglik_fwd(logits, pred, seq_len, trans)[1]
    pred.nbest_ids, pred.nbest_scores, pred.nbest_counts, pred.nbest_logz = tags, scores, counts, logz
    return pred
