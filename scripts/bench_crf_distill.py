"""CRF-to-CRF distillation on the GPU.

usage: python scripts/bench_crf_distill.py        (prints one JSON line)

  * kernel time (median of CUDA events) of the pair ner_crf_distill_fwd + _bwd at L = 128, K = 10, full-length rows,
    against the ordinary pair ner_crf_loglik_fwd + _bwd and the partial pair ner_crf_partial_loglik_fwd + _bwd on the
    same shape, at B = 64 (the lane-per-tag route training batches take) and B = 262144 (thread per sequence);
  * achieved bytes/s of the distillation pair at B = 262144 against the 3.35 TB/s of the H100 SXM data sheet, where the
    bytes are both emission tensors read plus d_s_logits written (12 LK bytes per row);
  * the TRAIN step (Estimator.train_step, host batch included) on one MSRA-shaped B = 64, L = 128 batch of bilstm_crf
    alone and with a bilstm_crf_softlexicon or a lattice_lstm_crf teacher, and of a 4-layer bert_crf alone and with a
    12-layer bert_bilstm_crf teacher; each distilled step is also split into the teacher's forward
    (Estimator.teacher_potentials) and the rest, and set against the aim of the student's step + the teacher's PREDICT
    on a device-resident batch + 0.2 ms.
The card's name and power limit are read in the same run.
"""
import json
import os
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from chinesener_b200 import engine, ops, synthetic  # noqa: E402

L, K = 128, 10
HBM_BPS = 3.35e12


def make(B, seed=0):
    g = torch.Generator().manual_seed(seed)
    xt, xs = torch.randn(B, L, K, generator=g) * 2, torch.randn(B, L, K, generator=g) * 2
    trt, trs = torch.randn(K, K, generator=g) * 0.5, torch.randn(K, K, generator=g) * 0.5
    lens = torch.full((B,), L, dtype=torch.int32)
    tags = torch.randint(0, K, (B, L), generator=g, dtype=torch.int32)
    d = torch.full((B,), -1.0 / B)
    return [t.cuda() for t in (xt, trt, xs, trs, lens, tags, d)]


def bench_kernels(B, iters):
    from bench_token_head import timeit
    xt, trt, xs, trs, lens, tags, d = make(B)
    mask = (torch.ones_like(tags) << tags).contiguous()

    def distill():
        logz, alpha = ops.crf_distill_fwd(xt, trt, xs, trs, lens, 2.0)
        return ops.crf_distill_bwd(xt, trt, xs, trs, lens, alpha, logz, 2.0, d_kl=d)

    def ordinary():
        _, logz, alpha = ops.crf_loglik_fwd(xs, tags, lens, trs, want_alpha=True)
        return ops.crf_loglik_bwd(xs, tags, lens, trs, alpha, logz, d, 1.0)

    def partial():
        _, logz, alpha = ops.crf_partial_loglik_fwd(xs, mask, lens, trs, want_alpha=True)
        return ops.crf_partial_loglik_bwd(xs, mask, lens, trs, alpha, logz, d, 1.0)

    t_d = timeit(distill, warm=3, iters=iters)[0]
    t_o = timeit(ordinary, warm=3, iters=iters)[0]
    t_p = timeit(partial, warm=3, iters=iters)[0]
    out = dict(B=B, distill_pair_us=t_d * 1e3, ordinary_pair_us=t_o * 1e3, partial_pair_us=t_p * 1e3,
               distill_over_partial=t_d / t_p)
    tb = B * 12 * L * K / (t_d * 1e-3) / 1e12
    out.update(distill_pair_tb_s=tb, distill_pair_share_of_hbm=tb * 1e12 / HBM_BPS)
    return out


def softlexicon_batch(B, Lt, n_word=5000, seed=3):
    feats = synthetic.msra_batch(B, Lt, seed=seed)
    ids, w = synthetic.softlexicon_features(B, Lt, n_word, seed=seed, lens=feats['seq_len'].numpy())
    feats['softlexicon_ids'], feats['softlexicon_weights'] = ids, w
    return feats


def lattice_batch(B, Lt, n_word=5000, Kw=4, seed=3):
    """An MSRA-shaped batch with lattice word features: each of the Kw slots of a position holds a word of 2..10
    characters starting there with probability 0.4 (slots reaching past seq_len count as empty, as in the kernels)."""
    import numpy as np
    feats = synthetic.msra_batch(B, Lt, seed=seed)
    rng = np.random.default_rng(seed)
    lens = rng.integers(2, 11, (B, Lt * Kw)) * (rng.random((B, Lt * Kw)) < 0.4)
    feats['lattice_lens'] = torch.from_numpy(lens.astype(np.int32))
    feats['lattice_ids'] = torch.from_numpy(np.where(lens > 0, rng.integers(0, n_word, lens.shape), n_word + 1)
                                            .astype(np.int32))
    return feats


def timed_steps(student, feats, iters):
    """-> (student step ms, teacher forward ms) of Estimator.train_step with a teacher."""
    from bench_token_head import timeit
    step = timeit(lambda: student.train_step(feats), warm=3, iters=iters)[0]
    dev = student.to_device(feats)
    fwd = timeit(lambda: student.teacher_potentials(dev), warm=3, iters=iters)[0]
    return step, fwd


def bench_train(tmp, iters):
    from bench_token_head import timeit
    Bt, Lt = 64, 128
    res = {}
    emb = torch.nn.functional.normalize(torch.randn(21128, 50), dim=1).numpy()
    wemb = torch.nn.functional.normalize(torch.randn(5000, 50), dim=1).numpy()
    feats = softlexicon_batch(Bt, Lt)
    base = dict(synthetic.data_params(Lt), embedding=emb)
    alone = engine.Estimator("bilstm_crf", base)
    t_alone = timeit(lambda: alone.train_step(feats), warm=3, iters=iters)[0]
    teacher = engine.Estimator("bilstm_crf_softlexicon", dict(base, word_embedding=wemb, word_enhance_dim=4,
                                                               max_lexicon_len=10))
    res["bilstm_crf<-bilstm_crf_softlexicon"] = distilled(teacher, "bilstm_crf", base, feats, t_alone, iters)

    lfeats = lattice_batch(Bt, Lt)
    t_alone = timeit(lambda: alone.train_step(lfeats), warm=3, iters=iters)[0]
    lwemb = (torch.randn(5003, 50) * 0.5).numpy()
    teacher = engine.Estimator("lattice_lstm_crf", dict(base, word_embedding=lwemb, max_lattice_words=4))
    res["bilstm_crf<-lattice_lstm_crf"] = distilled(teacher, "bilstm_crf", base, lfeats, t_alone, iters)

    cfg = {'vocab_size': 21128, 'hidden_size': 768, 'num_hidden_layers': 12, 'num_attention_heads': 12,
           'intermediate_size': 3072, 'max_position_embeddings': 512, 'type_vocab_size': 2, 'initializer_range': 0.02}
    dirs = {}
    for layers in (12, 4):
        dirs[layers] = os.path.join(tmp, "bert%d" % layers)
        os.makedirs(dirs[layers])
        with open(os.path.join(dirs[layers], "bert_config.json"), "w") as f:
            json.dump(dict(cfg, num_hidden_layers=layers), f)
    bfeats = synthetic.msra_batch(Bt, Lt, seed=3)
    alone = engine.Estimator("bert_crf", dict(synthetic.data_params(Lt), pretrain_dir=dirs[4]))
    t_alone = timeit(lambda: alone.train_step(bfeats), warm=3, iters=iters)[0]
    teacher = engine.Estimator("bert_bilstm_crf", dict(synthetic.data_params(Lt), pretrain_dir=dirs[12]))
    res["bert_crf(4)<-bert_bilstm_crf(12)"] = distilled(teacher, "bert_crf",
                                                        dict(synthetic.data_params(Lt), pretrain_dir=dirs[4]), bfeats,
                                                        t_alone, iters)
    return res


def distilled(teacher, student_name, params, feats, t_alone, iters):
    """Times of the distilled TRAIN step against the aim: the student's own step + the teacher's PREDICT + 0.2 ms.  The
    teacher's PREDICT is timed on a batch already on the device: the distilled step copies its host batch once, and
    t_alone already holds that copy."""
    from bench_token_head import timeit
    teacher.evaluate(feats)
    dev = teacher.to_device(feats)
    teacher_predict = timeit(lambda: teacher.predict_device(dev), warm=3, iters=iters)[0]
    student = engine.Estimator(student_name, params, teacher=teacher)
    step, fwd = timed_steps(student, feats, iters)
    return dict(alone_ms=t_alone, distilled_ms=step, teacher_forward_ms=fwd, student_part_ms=step - fwd,
                teacher_predict_device_ms=teacher_predict, excess_over_aim_ms=step - (t_alone + teacher_predict + 0.2))


def main():
    from bench_token_head import card
    out = dict(card=card(), L=L, K=K)
    out["kernels"] = [bench_kernels(64, 200), bench_kernels(262144, 20)]
    with tempfile.TemporaryDirectory() as tmp:
        out["train_step"] = bench_train(tmp, 20)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
