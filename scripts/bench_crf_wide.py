"""Wide-tag-set CRF kernels (ner_crf_wide_*) against the K-specialised ones, and the plugins on a 108-tag set.  Prints one
JSON line.

Kernel rows: median CUDA-event time of Viterbi, log-likelihood forward (with the alpha workspace) and backward at
B = 64, L = 128 (the model's batch) and at B = 65536 (throughput), for K = 40, 108, 128 on the wide kernels and K = 10 on
today's.  The large-B rows also give FP32 FMA/s (K*K per row and step: one multiply-add per transition) and HBM bytes/s
(logits read, alpha written / read, d_logits written) against the H100 SXM data sheet's 67 TFLOP/s FP32 (33.5 T FMA/s)
and 3.35 TB/s.  Model rows: bilstm_crf TRAIN step and bert_bilstm_crf PREDICT (layer path; plus the fused executor at
K = 10) on one MSRA-shaped B = 64, L = 128 batch.

    python scripts/bench_crf_wide.py [--tiny]      # --tiny: shapes and counts only, no GPU (a rehearsal)
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FMA_PEAK = 67e12 / 2
HBM_PEAK = 3.35e12


def work(kind, B, L, K):
    """(FMAs, HBM bytes) one call needs."""
    fma = B * L * K * K
    io = {"viterbi": B * L * K * 4 + B * L * K + B * L * 4,          # logits, byte backpointers, tags
          "fwd": 2 * B * L * K * 4 + B * L * 4,                       # logits, alpha, tags
          "bwd": 3 * B * L * K * 4 + B * L * 4}[kind]                 # logits, alpha, d_logits, tags
    return fma, io


def time_ms(fn, reps):
    import torch
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def kernel_rows(B, L, Ks, reps):
    import torch
    from chinesener_b200 import ops
    rows = []
    for K in Ks:
        g = torch.Generator(device="cuda").manual_seed(K)
        x = torch.randn(B, L, K, device="cuda", generator=g)
        tr = torch.randn(K, K, device="cuda", generator=g)
        lens = torch.full((B,), L, dtype=torch.int32, device="cuda")
        tags = torch.randint(0, K, (B, L), dtype=torch.int32, device="cuda", generator=g)
        wide = K > ops.MAX_TAGS
        _, logz, alpha = ops.crf_loglik_fwd(x, tags, lens, tr, want_alpha=True)
        t = {"viterbi": time_ms(lambda: ops.crf_viterbi(x, lens, tr), reps),
             "fwd": time_ms(lambda: ops.crf_loglik_fwd(x, tags, lens, tr, want_alpha=True), reps),
             "bwd": time_ms(lambda: ops.crf_loglik_bwd(x, tags, lens, tr, alpha, logz, None, -1.0 / B), reps)}
        row = {"B": B, "L": L, "K": K, "kernel": "wide" if wide else "narrow"}
        for kind, ms in t.items():
            fma, io = work(kind, B, L, K)
            row[kind + "_us"] = round(ms * 1e3, 1)
            if B > 4096:
                row[kind + "_fma_share"] = round(fma / (ms * 1e-3) / FMA_PEAK, 4)
                row[kind + "_hbm_share"] = round(io / (ms * 1e-3) / HBM_PEAK, 4)
        rows.append(row)
        del x, alpha
        torch.cuda.empty_cache()
    return rows


def model_rows(reps):
    import numpy as np
    import torch
    from chinesener_b200 import engine, synthetic
    B, L = 64, 128
    rows = {}
    for K in (10, 108):
        feats = synthetic.msra_batch(B, L, vocab=3000, seed=1)
        if K != 10:
            rng = np.random.default_rng(0)
            lab = rng.integers(1, K - 2, size=(B, L)).astype(np.int32) * feats['mask'].numpy()
            feats['label_ids'] = torch.from_numpy(lab)
        emb = torch.nn.functional.normalize(torch.randn(3000, 50, generator=torch.Generator().manual_seed(0)), dim=1).numpy()
        est = engine.Estimator("bilstm_crf", dict(synthetic.data_params(L, label_size=K), embedding=emb))
        dev = est.to_device(feats)
        rows[f"bilstm_crf_train_ms_K{K}"] = round(time_ms(lambda: est.train_step(dev), reps), 3)
        with tempfile.TemporaryDirectory() as d:
            cfg = {'vocab_size': 3000, 'hidden_size': 768, 'num_hidden_layers': 12, 'num_attention_heads': 12,
                   'intermediate_size': 3072, 'max_position_embeddings': 512, 'type_vocab_size': 2,
                   'initializer_range': 0.02}
            with open(os.path.join(d, "bert_config.json"), "w") as f:
                json.dump(cfg, f)
            for fused in ((False, True) if K == 10 else (False,)):
                est = engine.Estimator("bert_bilstm_crf", dict(synthetic.data_params(L, label_size=K), pretrain_dir=d,
                                                               fused_predict=fused))
                dev = est.to_device(feats)
                est.predict_device(dev)
                ms = time_ms(lambda: est.predict_device(dev), reps)
                rows[f"bert_bilstm_crf_predict_sent_per_s_K{K}" + ("_fused" if fused else "")] = round(B / (ms * 1e-3), 1)
    rows["train_ratio_K108_vs_K10"] = round(rows["bilstm_crf_train_ms_K108"] / rows["bilstm_crf_train_ms_K10"], 3)
    rows["predict_ratio_K108_vs_K10_layer"] = round(rows["bert_bilstm_crf_predict_sent_per_s_K108"]
                                                    / rows["bert_bilstm_crf_predict_sent_per_s_K10"], 3)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiny", action="store_true", help="no GPU: print the shapes and the work they need")
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    Ks = (10, 40, 108, 128)
    if args.tiny:
        out = {"tiny": True, "work": {f"{kind}_B{B}_K{K}": work(kind, B, 128, K)
                                      for B in (64, 65536) for K in Ks for kind in ("viterbi", "fwd", "bwd")}}
        print(json.dumps(out))
        return
    import torch
    assert torch.cuda.is_available(), "bench_crf_wide.py measures on the GPU; --tiny rehearses without one"
    p = torch.cuda.get_device_properties(0)
    out = {"device": p.name, "sms": p.multi_processor_count,
           "kernels_B64": kernel_rows(64, 128, Ks, args.reps),
           "kernels_B65536": kernel_rows(65536, 128, Ks, max(5, args.reps // 6)),
           "models": model_rows(max(5, args.reps // 3))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
