"""The Lattice LSTM recurrence and the lattice_lstm_crf plugin on the GPU.

usage: python scripts/bench_lattice.py        (prints one JSON line)

  * recurrence at B = 64, L = 128, on MSRA-shaped lengths and on full-length rows, with two synthetic lexicons:
    "sparse" (a Poisson(1) number of words per start, capped at Kw = 4, lengths mostly 2-4) and "full" (all Kw slots filled,
    lengths 2..10).  ner_lattice_recurrence in PREDICT and in TRAIN (saving for BPTT) and ner_lattice_recurrence_bwd, in us
    and us per step, next to ner_bigru_recurrence / ner_bilstm_recurrence (+ their BPTT) at the same B, L and H, for
    H = 100 (the plugin's) and H = 128.  Median of CUDA events over many launches.
  * lattice_lstm_crf PREDICT sentences/s (Estimator.predict_device) and TRAIN step time (Estimator.train_step, host batch
    included) next to bilstm_crf and bilstm_crf_softlexicon on one seeded MSRA-shaped batch with the sparse lexicon.
  * the float64 CPU restatement (tests/_lattice_oracle.py, one sentence and one step at a time, the shape of the public
    one-sentence implementation) in sentences/s on the same kind of batch.
The card's name and power limit are read in the same run: a number is only meaningful next to them.
"""
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
from chinesener_b200 import engine, ops, synthetic  # noqa: E402
from bench_token_head import card, timeit  # noqa: E402
import _lattice_oracle as olat  # noqa: E402

B, L, KW = 64, 128, 4


def lexicon(lens, kind, seed):
    """Slot lengths int32 [B, L * KW] of a synthetic lexicon."""
    rng = np.random.default_rng(seed)
    Bn = lens.shape[0]
    if kind == "full":
        out = rng.integers(2, 11, (Bn, L, KW))
    else:
        count = np.minimum(rng.poisson(1.0, (Bn, L)), KW)
        out = rng.choice([2, 3, 4, 5, 6], p=[0.55, 0.25, 0.12, 0.05, 0.03], size=(Bn, L, KW))
        out[np.arange(KW)[None, None, :] >= count[..., None]] = 0
    return torch.from_numpy(out.reshape(Bn, L * KW).astype(np.int32))


def seq_lengths(full, seed):
    if full:
        return torch.full((B,), L, dtype=torch.int32)
    return torch.from_numpy(synthetic.msra_lengths(B, L, np.random.default_rng(seed)).astype(np.int32))


def bench_recurrence(H, full, kind):
    g = torch.Generator(device="cuda").manual_seed(H)
    lens = seq_lengths(full, 7)
    lat = lexicon(lens, kind, 8).cuda()
    sl = lens.cuda()
    xproj = torch.randn(B * L, 8 * H, device="cuda", generator=g)
    wproj = torch.randn(B * L * KW, 6 * H, device="cuda", generator=g)
    wrec = [(torch.rand(H, 6 * H, device="cuda", generator=g) - 0.5) * 0.2 for _ in range(2)]
    wac = [(torch.rand(H, H, device="cuda", generator=g) - 0.5) * 0.2 for _ in range(2)]
    d_out = torch.randn(B, L, 2 * H, device="cuda", generator=g)
    args = (lat, wrec[0], wrec[1], wac[0], wac[1], sl, B, L, H, KW)
    fwd = timeit(lambda: ops.lattice_recurrence(xproj, wproj, *args), warm=3, iters=30)[0]
    train = timeit(lambda: ops.lattice_recurrence(xproj, wproj, *args, save_for_backward=True), warm=3, iters=30)[0]
    _, sv = ops.lattice_recurrence(xproj, wproj, *args, save_for_backward=True)
    bwd = timeit(lambda: ops.lattice_recurrence_bwd(d_out, sv, *args), warm=3, iters=30)[0]
    steps = int(lens.max())
    res = dict(H=H, lengths="full" if full else "msra", lexicon=kind, steps=steps,
               words_per_start=float((lat.view(B, L, KW) > 0).sum(-1).float().mean()),
               lattice_fwd_us=fwd * 1e3, lattice_fwd_train_us=train * 1e3, lattice_bwd_us=bwd * 1e3,
               lattice_fwd_us_per_step=fwd * 1e3 / steps, lattice_bwd_us_per_step=bwd * 1e3 / steps)
    xg = torch.randn(B * L, 6 * H, device="cuda", generator=g)
    whg = [(torch.rand(H, 3 * H, device="cuda", generator=g) - 0.5) * 0.2 for _ in range(2)]
    res["gru_fwd_us"] = timeit(lambda: ops.bigru_recurrence(xg, whg[0], whg[1], sl, B, L, H), warm=3, iters=30)[0] * 1e3
    _, gates, hst, _ = ops.bigru_recurrence(xg, whg[0], whg[1], sl, B, L, H, save_for_backward=True)
    res["gru_bwd_us"] = timeit(lambda: ops.bigru_recurrence_bwd(d_out, gates, hst, whg[0], whg[1], sl, B, L, H),
                               warm=3, iters=30)[0] * 1e3
    xl = torch.randn(B * L, 8 * H, device="cuda", generator=g)
    whl = [(torch.rand(H, 4 * H, device="cuda", generator=g) - 0.5) * 0.2 for _ in range(2)]
    res["lstm_fwd_us"] = timeit(lambda: ops.bilstm_recurrence(xl, whl[0], whl[1], sl, B, L, H), warm=3, iters=30)[0] * 1e3
    _, gl, cl, _ = ops.bilstm_recurrence(xl, whl[0], whl[1], sl, B, L, H, save_for_backward=True)
    res["lstm_bwd_us"] = timeit(lambda: ops.bilstm_recurrence_bwd(d_out, gl, cl, whl[0], whl[1], sl, B, L, H),
                                warm=3, iters=30)[0] * 1e3
    res["fwd_over_gru"] = res["lattice_fwd_us"] / res["gru_fwd_us"]
    res["bwd_over_gru"] = res["lattice_bwd_us"] / res["gru_bwd_us"]
    return res


def plugin_batch(V=11329, NW=50000, Ew=50, seed=1000):
    feats = synthetic.msra_batch(B, L, vocab=V, seed=seed)
    rng = np.random.default_rng(seed)
    lat = lexicon(feats['seq_len'].numpy(), "sparse", seed)
    feats['lattice_lens'] = lat
    feats['lattice_ids'] = torch.from_numpy(np.where(lat.numpy() > 0, rng.integers(0, NW, lat.shape), NW + 1).astype(np.int32))
    ids, w = synthetic.softlexicon_features(B, L, NW, seed=seed)
    feats['softlexicon_ids'], feats['softlexicon_weights'] = ids, w
    emb = rng.normal(size=(V, 50)).astype(np.float32)
    wemb = rng.normal(size=(NW + 3, Ew)).astype(np.float32)
    return feats, dict(synthetic.data_params(L), embedding=emb, word_embedding=wemb, max_lattice_words=KW, word_enhance_dim=4,
                       max_lexicon_len=10)


def bench_models(iters=20):
    feats, params = plugin_batch()
    out = {}
    for name in ("bilstm_crf", "bilstm_crf_softlexicon", "lattice_lstm_crf"):
        est = engine.Estimator(name, dict(params))
        est.evaluate(feats)
        dev = est.to_device(feats)
        pred_ms = timeit(lambda: est.predict_device(dev), warm=5, iters=iters)[0]
        train_ms = timeit(lambda: est.train_step(feats), warm=3, iters=iters)[0]
        out[name] = dict(predict_ms=pred_ms, predict_sentences_per_s=B / pred_ms * 1e3, train_step_ms=train_ms)
        del est
        torch.cuda.empty_cache()
    return dict(B=B, L=L, token_fill=float(feats["mask"].float().mean()), **out)


def bench_oracle(n=4):
    lens = seq_lengths(False, 3)[:n]
    lat = lexicon(lens, "sparse", 3)
    H, Ec, Ew = 100, 50, 50
    x = torch.randn(n, L, Ec, dtype=torch.float64)
    xw = torch.randn(n, L, KW, Ew, dtype=torch.float64)
    w = {k: v.double() for k, v in olat.random_weights(Ec, Ew, H, seed=1).items()}
    t0 = time.perf_counter()
    with torch.no_grad():
        olat.lattice_lstm(x, xw, lat, lens, w, H)
    return dict(sentences=n, sentences_per_s=n / (time.perf_counter() - t0), threads=torch.get_num_threads())


def main():
    assert torch.cuda.is_available(), "bench_lattice.py measures on a CUDA device"
    rec = [bench_recurrence(H, full, kind) for H in (100, 128) for full in (False, True) for kind in ("sparse", "full")]
    res = dict(card=card(), recurrence=rec, models=bench_models(), cpu_oracle=bench_oracle())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
