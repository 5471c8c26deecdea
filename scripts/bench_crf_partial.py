"""The partial-annotation CRF kernels on the GPU.

usage: python scripts/bench_crf_partial.py [--tiny]        (prints one JSON line)

  * kernel time (median of CUDA events) of the fused pair ner_crf_partial_loglik_fwd + _bwd against the composition of
    the existing kernels (-inf-masked logits, ner_crf_loglik_fwd twice, ner_crf_loglik_bwd twice and a subtraction), at
    B = 64 and B = 262144, L = 128, K = 10, full-length rows, masks mixing one-hot, open and subset positions;
  * achieved bytes/s of the forward and the backward at B = 262144 against the 3.35 TB/s of the H100 SXM data sheet,
    from algorithmic bytes per row: forward reads 4LK + 4L (logits, mask) and writes 8LK + 12 (alpha_A, alpha, ll,
    logZ_A, logZ); backward reads 12LK + 4L + 12 (logits, both alphas, mask, logZ pair, d_ll) and writes 4LK;
  * the TRAIN step (Estimator.train_step, host batch included) of bilstm_crf and bert_bilstm_crf on one MSRA-shaped
    B = 64 batch, with full labels and with 30 % of the real tokens opened to every tag.
The card's name and power limit are read in the same run.  --tiny runs the host parts at a toy size (no timing).
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from chinesener_b200 import engine, ops, synthetic  # noqa: E402

L, K = 128, 10
HBM_BPS = 3.35e12


def fwd_bytes(B):
    return B * (4 * L * K + 4 * L + 8 * L * K + 12)


def bwd_bytes(B):
    return B * (12 * L * K + 4 * L + 12 + 4 * L * K)


def make(B, seed=0, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, K, generator=g) * 2
    tr = torch.randn(K, K, generator=g) * 0.5
    lens = torch.full((B,), L, dtype=torch.int32)
    onehot = torch.ones((B, L), dtype=torch.int64) << torch.randint(1, K, (B, L), generator=g)
    pick = torch.rand((B, L), generator=g)
    mask = torch.where(pick < 0.3, torch.full_like(onehot, ((1 << K) - 1) & ~1),
                       torch.where(pick < 0.4, onehot | (onehot << 1) % (1 << K), onehot)).to(torch.int32)
    d_ll = torch.full((B,), -1.0 / B)
    return [t.to(device) for t in (x, mask, lens, tr, d_ll)]


def fused(x, mask, lens, tr, d_ll):
    ll, logz, alpha = ops.crf_partial_loglik_fwd(x, mask, lens, tr, want_alpha=True)
    return ll, ops.crf_partial_loglik_bwd(x, mask, lens, tr, alpha, logz, d_ll, 1.0)


def composed(x, mask, lens, tr, d_ll):
    allowed = ((mask.long()[..., None] & 0xFFFFFFFF) >> torch.arange(K, device=x.device)) & 1
    xa = torch.where(allowed.bool(), x, torch.full_like(x, -float("inf")))
    tags = torch.zeros(mask.shape, dtype=torch.int32, device=x.device)
    _, lza, aa = ops.crf_loglik_fwd(xa, tags, lens, tr, want_alpha=True)
    _, lzf, af = ops.crf_loglik_fwd(x, tags, lens, tr, want_alpha=True)
    da, ta = ops.crf_loglik_bwd(xa, tags, lens, tr, aa, lza, d_ll, 1.0)
    df, tf = ops.crf_loglik_bwd(x, tags, lens, tr, af, lzf, d_ll, 1.0)
    return lza - lzf, (df - da, tf - ta)


def bench_kernels(B, iters):
    from bench_token_head import timeit
    x, mask, lens, tr, d_ll = make(B)
    t_fused = timeit(lambda: fused(x, mask, lens, tr, d_ll), warm=3, iters=iters)[0]
    t_comp = timeit(lambda: composed(x, mask, lens, tr, d_ll), warm=3, iters=iters)[0]
    ll, logz, alpha = ops.crf_partial_loglik_fwd(x, mask, lens, tr, want_alpha=True)
    t_fwd = timeit(lambda: ops.crf_partial_loglik_fwd(x, mask, lens, tr, want_alpha=True), warm=3, iters=iters)[0]
    t_bwd = timeit(lambda: ops.crf_partial_loglik_bwd(x, mask, lens, tr, alpha, logz, d_ll, 1.0), warm=3,
                   iters=iters)[0]
    (lf, (df, _)), (lc, (dc, _)) = fused(x, mask, lens, tr, d_ll), composed(x, mask, lens, tr, d_ll)
    out = dict(B=B, fused_us=t_fused * 1e3, composed_us=t_comp * 1e3, speedup=t_comp / t_fused,
               fwd_us=t_fwd * 1e3, bwd_us=t_bwd * 1e3,
               max_ll_diff=float((lf - lc).abs().max()), max_dlogits_diff_over_g=float((df - dc).abs().max()) * B)
    out.update(fwd_tb_s=fwd_bytes(B) / (t_fwd * 1e-3) / 1e12, bwd_tb_s=bwd_bytes(B) / (t_bwd * 1e-3) / 1e12)
    out.update(fwd_share_of_hbm=out["fwd_tb_s"] * 1e12 / HBM_BPS, bwd_share_of_hbm=out["bwd_tb_s"] * 1e12 / HBM_BPS)
    return out


def open_tokens(feats, frac=0.3, seed=0):
    """The batch with `frac` of its real tokens opened to every real tag (label_id -1, label_mask bits 1..7)."""
    lab = feats['label_ids'].long()
    g = torch.Generator().manual_seed(seed)
    opened = (torch.rand(lab.shape, generator=g) < frac) & (lab > 0) & (lab < 8)
    out = dict(feats)
    out['label_mask'] = torch.where(opened, torch.full_like(lab, (1 << 8) - 2), torch.ones_like(lab) << lab.clamp(min=0))
    out['label_mask'] = out['label_mask'].to(torch.int32)
    out['label_ids'] = torch.where(opened, torch.full_like(lab, -1), lab).to(torch.int32)
    return out, float(opened.sum()) / float((lab > 0).sum())


def bench_train(tmp, iters):
    from bench_token_head import timeit
    Bt, Lt = 64, 128
    res = {}
    for name in ("bilstm_crf", "bert_bilstm_crf"):
        if name.startswith("bert"):
            cfg = {'vocab_size': 21128, 'hidden_size': 768, 'num_hidden_layers': 12, 'num_attention_heads': 12,
                   'intermediate_size': 3072, 'max_position_embeddings': 512, 'type_vocab_size': 2,
                   'initializer_range': 0.02}
            with open(os.path.join(tmp, "bert_config.json"), "w") as f:
                json.dump(cfg, f)
            params = dict(synthetic.data_params(Lt), pretrain_dir=tmp)
            feats = synthetic.msra_batch(Bt, Lt, seed=3)
        else:
            emb = torch.nn.functional.normalize(torch.randn(21128, 50), dim=1).numpy()
            params = dict(synthetic.data_params(Lt), embedding=emb)
            feats = synthetic.msra_batch(Bt, Lt, seed=3)
        partial, frac = open_tokens(feats)
        est = engine.Estimator(name, params)
        t_full = timeit(lambda: est.train_step(feats), warm=3, iters=iters)[0]
        t_part = timeit(lambda: est.train_step(partial), warm=3, iters=iters)[0]
        t_full2 = timeit(lambda: est.train_step(feats), warm=0, iters=iters)[0]
        res[name] = dict(full_ms=min(t_full, t_full2), partial_ms=t_part, opened_fraction=frac,
                         overhead=t_part / min(t_full, t_full2) - 1)
    return res


def main():
    import tempfile
    if "--tiny" in sys.argv:                                  # host parts only: shapes, bytes, masks
        x, mask, lens, tr, d_ll = make(4, device="cpu")
        feats = synthetic.msra_batch(4, 16, seed=3)
        partial, frac = open_tokens(feats)
        print(json.dumps(dict(tiny=True, mask_shape=list(mask.shape), fwd_bytes_per_row=fwd_bytes(1),
                              bwd_bytes_per_row=bwd_bytes(1), opened_fraction=frac,
                              label_mask_dtype=str(partial['label_mask'].dtype))))
        return
    from bench_token_head import card
    out = dict(card=card(), L=L, K=K)
    out["kernels"] = [bench_kernels(64, 200), bench_kernels(262144, 20)]
    with tempfile.TemporaryDirectory() as tmp:
        out["train_step"] = bench_train(tmp, 30)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
