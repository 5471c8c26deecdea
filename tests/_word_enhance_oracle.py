"""Float64 CPU restatements (eval mode) of the word-enhance plugins, the checker of tests/test_word_enhance_gpu.py:
bilstm_crf_bichar, bilstm_crf_softword and bilstm_crf_ex_softword are bilstm_crf (oracle/models.py) with a wider BiLSTM
input.  The reference's plugin files are not available, so these follow this project's restatement of the graphs
(chinesener_b200/model/bilstm_crf_{bichar,softword,ex_softword}.py).  Each returns dict(logits, loss, pred_ids, ll)."""
import torch

from oracle import nn
from oracle.models import _crf_tail


def _bilstm_crf_on(x, w, features, params, dtype, emulate_bf16):
    lstm = nn.bilstm(x, w, features["seq_len"], params["rnn_activation"], 1.0, dtype, emulate_bf16)
    logits = nn.dense(lstm, w["logits/kernel"].to(dtype), w["logits/bias"].to(dtype))
    return _crf_tail(logits, w, features)


def bilstm_crf_bichar(w, features, params, dtype=torch.float32, emulate_bf16=False):
    """concat([char, bichar]) -> bilstm_crf."""
    char = torch.as_tensor(params["embedding"]).to(dtype)[features["token_ids"].long()]
    bichar = torch.as_tensor(params["bichar_embedding"]).to(dtype)[features["bichar_ids"].long()]
    return _bilstm_crf_on(torch.cat([char, bichar], dim=-1), w, features, params, dtype, emulate_bf16)


def bilstm_crf_softword(w, features, params, dtype=torch.float32, emulate_bf16=False):
    """concat([W[softword_ids], char]) -> bilstm_crf."""
    char = torch.as_tensor(params["embedding"]).to(dtype)[features["token_ids"].long()]
    seg = w["word_enhance/softword_embedding"].to(dtype)[features["softword_ids"].long()]
    return _bilstm_crf_on(torch.cat([seg, char], dim=-1), w, features, params, dtype, emulate_bf16)


def bilstm_crf_ex_softword(w, features, params, dtype=torch.float32, emulate_bf16=False):
    """concat([ex_softword_ids @ W, char]) -> bilstm_crf."""
    B, L = features["token_ids"].shape
    char = torch.as_tensor(params["embedding"]).to(dtype)[features["token_ids"].long()]
    table = w["word_enhance/softword_embedding"].to(dtype)
    seg = features["ex_softword_ids"].to(dtype).view(B, L, table.shape[0]) @ table
    return _bilstm_crf_on(torch.cat([seg, char], dim=-1), w, features, params, dtype, emulate_bf16)
