"""The word-enhance small-table kernels and plugins on the GPU.

usage: python scripts/bench_word_enhance.py        (prints one JSON line)

  * kernels, V = E = 5 (the Softword / ExSoftword table), n_tok = 64 * 128 (one batch) and 2^22: ner_multihot_embed_fwd
    and ner_small_table_grad in both modes.  Time = median of CUDA events over many launches; GB/s and share of the
    H100 SXM's 3.35 TB/s (data sheet) from algorithmic bytes per token: forward 4V weights in + 4E out; gradient 4E d_out
    in + 4 ids or 4V weights in (the [V, E] table and the partials are negligible).
  * the deterministic gradient against the float-atomic ner_softlexicon_pool_bwd on the same input (G = 1, S = 5, ids
    the constant 0..4, the multi-hot weights), outputs compared.
  * sentences/s of PREDICT (Estimator.predict_device) and TRAIN (Estimator.train_step, host batch included) of the three
    word-enhance plugins against bilstm_crf on one seeded MSRA-shaped batch (B = 32, L = 150).
The card's name and power limit are read in the same run: a number is only meaningful next to them.
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from chinesener_b200 import engine, ops, synthetic  # noqa: E402
from bench_token_head import card, timeit  # noqa: E402

HBM_BPS = 3.35e12


def _rate(ms, nbytes):
    return dict(ms=ms, bytes=nbytes, GBps=nbytes / ms / 1e6, share_of_3p35TBps=nbytes / (ms * 1e-3) / HBM_BPS)


def bench_kernels(n_tok, V=5, E=5):
    g = torch.Generator(device="cuda").manual_seed(n_tok)
    table = torch.randn(V, E, device="cuda", generator=g)
    w = (torch.rand(n_tok, V, device="cuda", generator=g) < 0.35).float()
    ids = torch.randint(0, V, (n_tok,), device="cuda", dtype=torch.int32, generator=g)
    d_out = torch.randn(n_tok, E, device="cuda", generator=g)
    out = torch.empty(n_tok, E, device="cuda")
    d_table = torch.zeros(V, E, device="cuda")
    fwd = timeit(lambda: ops.multihot_embed(table, w, out=out), warm=5, iters=50)[0]
    g_ids = timeit(lambda: ops.small_table_grad(d_table, d_out, ids=ids), warm=5, iters=50)[0]
    g_w = timeit(lambda: ops.small_table_grad(d_table, d_out, weights=w), warm=5, iters=50)[0]
    const_ids = torch.arange(V, device="cuda", dtype=torch.int32).repeat(n_tok, 1).contiguous()
    atomic = timeit(lambda: ops.softlexicon_pool_bwd(d_table, const_ids, w, d_out, 1, V), warm=5, iters=50)[0]
    # outputs on the same input, from zero
    a, b = torch.zeros(V, E, device="cuda"), torch.zeros(V, E, device="cuda")
    ops.small_table_grad(a, d_out, weights=w)
    ops.softlexicon_pool_bwd(b, const_ids, w, d_out, 1, V)
    ref = (w.double().t() @ d_out.double())
    scale = float(ref.abs().max())
    return dict(n_tok=n_tok, V=V, E=E,
                multihot_fwd=_rate(fwd, n_tok * 4 * (V + E)),
                grad_ids=_rate(g_ids, n_tok * 4 * (1 + E)),
                grad_weights=_rate(g_w, n_tok * 4 * (V + E)),
                atomic_softlexicon_bwd=dict(_rate(atomic, n_tok * 4 * (2 * V + E)), over_grad_weights=atomic / g_w),
                max_rel_err_deterministic=float((a.double() - ref).abs().max()) / scale,
                max_rel_err_atomic=float((b.double() - ref).abs().max()) / scale,
                max_rel_diff_between=float((a - b).abs().max()) / scale)


def bench_models(B=32, L=150, V=11329, NB=40000, iters=30):
    feats = synthetic.msra_batch(B, L, vocab=V, seed=1000)
    rng = np.random.default_rng(1000)
    live = np.arange(L)[None, :] < feats['seq_len'].numpy()[:, None]
    feats['bichar_ids'] = torch.from_numpy(rng.integers(0, NB, (B, L)).astype(np.int32))
    feats['softword_ids'] = torch.from_numpy((rng.integers(1, 5, (B, L)) * live).astype(np.int32))
    ex = (rng.random((B, L, 5)) < 0.35).astype(np.float32)
    ex[..., 4] = ex[..., :4].sum(-1) == 0
    feats['ex_softword_ids'] = torch.from_numpy((ex * live[..., None]).reshape(B, L * 5))
    emb = rng.normal(size=(V, 50)).astype(np.float32)
    bemb = rng.normal(size=(NB, 50)).astype(np.float32)
    out = {}
    for name in ("bilstm_crf", "bilstm_crf_bichar", "bilstm_crf_softword", "bilstm_crf_ex_softword"):
        est = engine.Estimator(name, dict(synthetic.data_params(L), embedding=emb, bichar_embedding=bemb))
        est.evaluate(feats)
        dev = est.to_device(feats)
        pred_ms = timeit(lambda: est.predict_device(dev), warm=5, iters=iters)[0]
        train_ms = timeit(lambda: est.train_step(feats), warm=3, iters=iters)[0]
        out[name] = dict(predict_ms=pred_ms, predict_sentences_per_s=B / pred_ms * 1e3,
                         train_ms=train_ms, train_sentences_per_s=B / train_ms * 1e3)
        del est
        torch.cuda.empty_cache()
    for name in ("bilstm_crf_bichar", "bilstm_crf_softword", "bilstm_crf_ex_softword"):
        out[name]["predict_time_over_bilstm_crf"] = out[name]["predict_ms"] / out["bilstm_crf"]["predict_ms"]
        out[name]["train_time_over_bilstm_crf"] = out[name]["train_ms"] / out["bilstm_crf"]["train_ms"]
    return dict(B=B, L=L, token_fill=float(feats["mask"].float().mean()), **out)


def main():
    assert torch.cuda.is_available(), "bench_word_enhance.py measures on a CUDA device"
    res = dict(card=card(), kernels=[bench_kernels(64 * 128), bench_kernels(1 << 22)], models=bench_models())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
