"""Float64 CPU restatement of the bidirectional RNN layer with the reference's other RNN knobs (tools/layer.py:10-41):
GRUCell and a MultiRNNCell of `cell_size` DropoutWrapper-ed cells inside bidirectional_dynamic_rnn (SURVEY.md Appendix
A.2), and the bilstm_crf / bert_bilstm_crf / bilstm_crf_softlexicon graphs (oracle/models.py) on top of it.  The checker
of tests/test_rnn_cells_gpu.py, itself pinned by tests/test_rnn_oracle.py.  GRU arithmetic restates TF 1.14's GRUCell,
not reference artefacts."""
import torch

from oracle import nn
from oracle.models import _crf_tail

_rb = nn._rb


def gru_direction(x, kernel, bias, seq_len, activation="tanh", reverse=False, emulate_bf16=False, out_mask=None,
                  state_mask=None):
    """One direction of dynamic_rnn(GRUCell) (TF 1.14): kernel [D+H, 3H] = [gates/kernel | candidate/kernel] (columns
    r, u, c), bias [3H] = [gates/bias | candidate/bias].
        r, u = split(sigmoid([x, h] @ Wg + bg)),  c = act([x, r * h] @ Wc + bc),  h' = u * h + (1 - u) * c
    out_mask / state_mask: optional [B, L, H] multipliers (keep / keep_prob) in original positions, the DropoutWrapper's
    output and state filters."""
    return rnn_direction(x, kernel, bias, seq_len, "gru", activation, 1.0, reverse, emulate_bf16, out_mask, state_mask)


def rnn_direction(x, kernel, bias, seq_len, cell="lstm", activation="tanh", forget_bias=1.0, reverse=False,
                  emulate_bf16=False, out_mask=None, state_mask=None, saved=False):
    """One direction of dynamic_rnn(DropoutWrapper(cell)), cell 'lstm' (kernel [D+H, 4H], gates i, j, f, o; as
    lstm_direction) or 'gru' (see gru_direction).  For t >= seq_len the output is 0 and the state is carried.
    saved=True: -> (out, per-step values [B, L, .] in original positions, 0 past seq_len): 'gates' (LSTM: sigmoid(i),
    act(j), sigmoid(f + forget_bias), sigmoid(o); GRU: r, u, act(c)), 'h' (the carried, state-dropped h) and, LSTM,
    'c' (the cell state) or, GRU, 'rh' (r * h_prev) -- what the recurrence kernels save for back-propagation."""
    B, L, D = x.shape
    H = kernel.shape[1] // (4 if cell == "lstm" else 3)
    act = torch.relu if activation == "relu" else torch.tanh
    wx, wh = kernel[:D], kernel[D:]
    xproj = _rb(x, emulate_bf16) @ _rb(wx, emulate_bf16) + bias
    h = x.new_zeros(B, H)
    c = x.new_zeros(B, H)
    out = x.new_zeros(B, L, H)
    lens = seq_len.long()
    ar = torch.arange(B)
    per_step = {k: x.new_zeros(B, L, n * H) for k, n in
                (("gates", 4 if cell == "lstm" else 3), ("h", 1), ("c" if cell == "lstm" else "rh", 1))}
    for s in range(L):
        active = s < lens
        if not bool(active.any()):
            break
        pos = torch.where(active, (lens - 1 - s) if reverse else torch.full_like(lens, s), torch.zeros_like(lens))
        xp = xproj[ar, pos]
        if cell == "lstm":
            i, j, f, o = (xp + h @ wh).split(H, dim=1)
            gates = (torch.sigmoid(i), act(j), torch.sigmoid(f + forget_bias), torch.sigmoid(o))
            c_new = gates[2] * c + gates[0] * gates[1]
            h_new = gates[3] * act(c_new)
            c = torch.where(active[:, None], c_new, c)
            extra = c_new
        else:
            r, u = torch.sigmoid(xp[:, :2 * H] + h @ wh[:, :2 * H]).split(H, dim=1)
            cand = act(xp[:, 2 * H:] + (r * h) @ wh[:, 2 * H:])
            h_new = u * h + (1 - u) * cand
            gates, extra = (r, u, cand), r * h
        h_state = h_new if state_mask is None else h_new * state_mask[ar, pos]
        h_out = h_new if out_mask is None else h_new * out_mask[ar, pos]
        h = torch.where(active[:, None], h_state, h)
        idx = ar[active]
        out[idx, pos[active]] = h_out[active]
        if saved:
            for k, v in (("gates", torch.cat(gates, 1)), ("h", h_state), ("c" if cell == "lstm" else "rh", extra)):
                per_step[k][idx, pos[active]] = v[active].detach()
    return (out, per_step) if saved else out


def rnn_cell_weights(w, prefix, d, i, cell, dtype=torch.float64):
    """(kernel, bias) of layer i of direction d under the reference's names; GRU: gates and candidate side by side."""
    base = f"{prefix}/{d}/multi_rnn_cell/cell_{i}"
    if cell == "lstm":
        return w[f"{base}/lstm_cell/kernel"].to(dtype), w[f"{base}/lstm_cell/bias"].to(dtype)
    k = torch.cat([w[f"{base}/gru_cell/gates/kernel"], w[f"{base}/gru_cell/candidate/kernel"]], dim=1)
    b = torch.cat([w[f"{base}/gru_cell/gates/bias"], w[f"{base}/gru_cell/candidate/bias"]])
    return k.to(dtype), b.to(dtype)


def birnn(x, w, seq_len, cell_type="lstm", hidden_units_list=(128,), activation="tanh", forget_bias=1.0,
          dtype=torch.float64, emulate_bf16=False, prefix="bilstm_layer/bidirectional_rnn", masks=None):
    """bidirectional_dynamic_rnn over MultiRNNCell([DropoutWrapper(cell_i)] * len(hidden_units_list)) -> [B, L, 2H_top].

    The fw and bw stacks are independent: layer i+1 of a direction reads layer i OF THE SAME DIRECTION (not the [fw | bw]
    concat that torch.nn.LSTM(bidirectional=True, num_layers=n) feeds forward); the bw stack runs on
    reverse_sequence(x, seq_len), so in original positions bw layer i+1 at p reads bw layer i at p.  The output is
    concat(fw_top, bw_top).  masks: optional {(i, d): (out_mask, state_mask)} of rnn_direction (TRAIN dropout)."""
    x = x.to(dtype)
    outs = []
    for d, rev in (("fw", False), ("bw", True)):
        h = x
        for i in range(len(hidden_units_list)):
            k, b = rnn_cell_weights(w, prefix, d, i, cell_type, dtype)
            om, sm = (masks or {}).get((i, d), (None, None))
            h = rnn_direction(h, k, b, seq_len, cell_type, activation, forget_bias, rev, emulate_bf16, om, sm)
        outs.append(h)
    return torch.cat(outs, dim=-1)


def _plugin_rnn(x, w, features, params, dtype, emulate_bf16):
    n = int(params["cell_size"])
    return birnn(x, w, features["seq_len"], params["cell_type"].lower(), params["hidden_units_list"][:n],
                 params["rnn_activation"], 1.0, dtype, emulate_bf16)


def _head(rnn_out, w, features, dtype):
    logits = nn.dense(rnn_out, w["logits/kernel"].to(dtype), w["logits/bias"].to(dtype))
    return _crf_tail(logits, w, features)


def bilstm_crf(w, features, params, dtype=torch.float32, emulate_bf16=False):
    """oracle/models.bilstm_crf with params['cell_type'] / params['cell_size']."""
    emb = torch.as_tensor(params["embedding"]).to(dtype)[features["token_ids"].long()]
    return _head(_plugin_rnn(emb, w, features, params, dtype, emulate_bf16), w, features, dtype)


def bert_bilstm_crf(w, features, params, dtype=torch.float32, emulate_bf16=False, gelu_variant="tanh"):
    """oracle/models.bert_bilstm_crf with params['cell_type'] / params['cell_size']."""
    seq = nn.bert_encoder(w, features["token_ids"], features["mask"], features["segment_ids"],
                          num_layers=params.get("num_hidden_layers", 12), num_heads=params.get("num_attention_heads", 12),
                          dtype=dtype, gelu_variant=gelu_variant, emulate_bf16=emulate_bf16)
    return _head(_plugin_rnn(seq, w, features, params, dtype, emulate_bf16), w, features, dtype)


def bilstm_crf_softlexicon(w, features, params, dtype=torch.float32, emulate_bf16=False):
    """oracle/models.bilstm_crf_softlexicon with params['cell_type'] / params['cell_size']."""
    B = features["token_ids"].shape[0]
    L = params["max_seq_len"]
    G, S = params["word_enhance_dim"], params["max_lexicon_len"]
    emb = torch.as_tensor(params["embedding"]).to(dtype)[features["token_ids"].long()]
    ids = features["softlexicon_ids"].view(B, L, G * S)
    wts = features["softlexicon_weights"].view(B, L, G * S)
    wh = nn.softlexicon_pool(w["word_enhance/softlexicon_embedding"].to(dtype), ids, wts, G, S)
    return _head(_plugin_rnn(torch.cat([wh, emb], dim=-1), w, features, params, dtype, emulate_bf16), w, features, dtype)
