"""GPU: ner_mlm_mask bit-exact against the numpy rule, ner_vocab_xent against float64, the masked-LM head's gradients against
float64 autograd over oracle.nn.bert_encoder, learning on a synthetic corpus, and pretrain -> export -> fine-tune."""
import json
import math

import numpy as np
import pytest
import torch

import _mlm_oracle as mo
from chinesener_b200 import autodiff, bert, engine, mlm, ops, synthetic, variables
from chinesener_b200.tools import train_utils
from oracle import nn as onn

pytestmark = pytest.mark.gpu


def _batch(B, L, seed, V=21128, with_ws=True):
    rng = np.random.default_rng(seed)
    toks = rng.integers(106, V, (B, L)).astype(np.int32)
    n = rng.integers(0, L + 1, B).astype(np.int32)
    n[: min(B, 6)] = [0, 1, 2, 3, L, -4][: min(B, 6)]
    ws = (rng.random((B, L)) < 0.5).astype(np.uint8) if with_ws else None
    return toks, n, ws


def _run_mask(toks, n, ws, p, seed, V=21128, mask_id=103, max_pred=20):
    L = toks.shape[1]
    k = mlm.prediction_budget(np.clip(n, 0, L), p, max_pred)
    off = mlm.pred_offsets(k)
    d = lambda a: None if a is None else torch.from_numpy(a).cuda()
    out = ops.mlm_mask(d(toks), d(n), d(off), int(off[-1]), seed, V, mask_id, word_start=d(ws))
    return [t.cpu().numpy() for t in out], off, k


@pytest.mark.parametrize("with_ws", [False, True])
@pytest.mark.parametrize("L", [8, 128, 512])
@pytest.mark.parametrize("Bk", ["1", "64", "4sm+3"])
def test_mask_is_bit_exact_against_the_oracle(Bk, L, with_ws):
    B = {"1": 1, "64": 64, "4sm+3": 4 * torch.cuda.get_device_properties(0).multi_processor_count + 3}[Bk]
    toks, n, ws = _batch(B, L, 7 + L, with_ws=with_ws)
    seed = 0x1234_5678_9abc
    (masked, pos, lab), off, k = _run_mask(toks, n, ws, 0.15, seed)
    rm, rp, rl = mo.mlm_mask(toks, n, ws, off, seed, 21128, 103)
    assert (masked == rm).all() and (pos == rp).all() and (lab == rl).all()
    nn_ = np.clip(n, 0, L)
    for b in range(B):
        sel = [p - b * L for p, y in zip(pos[off[b]:off[b + 1]], lab[off[b]:off[b + 1]]) if y >= 0]
        assert all(1 <= t <= nn_[b] - 2 for t in sel)
        if not with_ws:
            assert len(sel) == k[b]
        else:                                           # whole words or nothing
            for s, ln in mo.words_of_row(nn_[b], ws[b]):
                inside = sum(s <= t < s + ln for t in sel)
                assert inside in (0, ln)
    # repeats are identical, another seed differs
    again = _run_mask(toks, n, ws, 0.15, seed)[0]
    assert all((a == b_).all() for a, b_ in zip(again, (masked, pos, lab)))
    if k.sum() > 4:
        other = _run_mask(toks, n, ws, 0.15, seed + 1)[0]
        assert not all((a == b_).all() for a, b_ in zip(other, (masked, pos, lab)))


def test_mask_split_is_within_binomial_bounds():
    B, L, V = 16384, 128, 21128
    toks = np.full((B, L), 7000, np.int32)
    n = np.full(B, L, np.int32)
    (masked, pos, lab), off, k = _run_mask(toks, n, None, 0.15, 42, V=V, mask_id=103)
    got = masked.reshape(-1)[pos]
    N = len(pos)
    for frac, cnt in ((0.8, (got == 103).sum()), (0.1, (got == 7000).sum()), (0.1, ((got != 103) & (got != 7000)).sum())):
        sd = math.sqrt(N * frac * (1 - frac))
        assert abs(cnt - N * frac) < 5 * sd + 30, (frac, cnt, N)    # random ids that hit 103 / 7000: < N / V each


@pytest.mark.parametrize("V,ld", [(1, 4), (7, 8), (1000, 1024), (21128, 21152), (50000, 50000)])
def test_vocab_xent_matches_float64(V, ld):
    rng = np.random.default_rng(V)
    M = 300
    z = rng.normal(0, 4, (M, ld)).astype(np.float32)
    z[5, :V] = 1e4
    z[6, :V] = -1e4
    z[7, : min(V, 3)] = 1e4
    y = rng.integers(0, V, M).astype(np.int32)
    y[::7] = -1
    y[3] = V                                              # out of range: not counted
    zd, yd = torch.from_numpy(z).cuda(), torch.from_numpy(y).cuda()
    loss, count, correct, pred, d = ops.vocab_xent(zd, yd, V, want_grad=True, d_loss=3.0)
    rl, rc, rcor, rp, rd = mo.vocab_xent(z, y, V, d_loss=3.0)
    assert int(count) == rc and int(correct) == rcor and (pred.cpu().numpy() == rp).all()
    assert abs(float(loss) - rl) < 1e-5 * max(1.0, abs(rl))
    dn = d.float().cpu().numpy()
    assert np.abs(dn - rd).max() <= 1e-2 * np.abs(rd).max() + 1e-12
    ign = (y < 0) | (y >= V)
    assert (dn[ign] == 0).all() and (dn[:, V:] == 0).all()
    loss2 = ops.vocab_xent(zd, yd, V, want_grad=True, d_loss=3.0)[0]
    assert float(loss2) == float(loss)                    # bit-identical repeat
    # an all-ignored batch
    l0, c0, k0, _, d0 = ops.vocab_xent(zd, torch.full_like(yd, -1), V, want_grad=True)
    assert float(l0) == 0.0 and int(c0) == 0 and int(k0) == 0 and not d0.float().abs().any()


TINY = {'vocab_size': 1000, 'hidden_size': 128, 'num_hidden_layers': 2, 'num_attention_heads': 2, 'intermediate_size': 512,
        'max_position_embeddings': 64, 'type_vocab_size': 2, 'initializer_range': 0.02, 'hidden_dropout_prob': 0.0,
        'attention_probs_dropout_prob': 0.0}


def _tiny_dir(tmp_path):
    (tmp_path / "bert_config.json").write_text(json.dumps(TINY))
    return str(tmp_path)


def _dev_batch(toks, n, ws=None):
    from chinesener_b200 import pretrain
    B, L = toks.shape
    mask = (np.arange(L)[None] < np.clip(n, 0, L)[:, None]).astype(np.int32)
    host = {'token_ids': torch.from_numpy(toks), 'mask': torch.from_numpy(mask), 'segment_ids': torch.zeros_like(torch.from_numpy(toks)),
            'seq_len': torch.from_numpy(n.astype(np.int32))}
    if ws is not None:
        host['word_start'] = torch.from_numpy(ws)
    return pretrain.to_device(host, torch.device('cuda'))


def test_head_gradients_match_float64_autograd(tmp_path):
    cfg = bert.load_bert_config(_tiny_dir(tmp_path))
    store = variables.VariableStore('cuda', seed=3)
    rng = np.random.default_rng(5)
    B, L, V = 6, 32, TINY['vocab_size']
    toks = rng.integers(106, V, (B, L)).astype(np.int32)
    n = np.array([32, 20, 9, 3, 2, 27], np.int32)
    toks[np.arange(B), 0] = 101
    dev = _dev_batch(toks, n)
    bert.create_bert_variables(cfg, store)
    mlm.create_head_variables(cfg, store)
    store.vars["cls/predictions/output_bias"].normal_(0, 0.5)
    store.touch()
    w = store.state_dict()
    with variables.use_store(store), autodiff.recording(store) as tape:
        out = mlm.masked_lm(dev, cfg, store, 11, 0.3, 8, 103, True, tape=tape)
        tape.backward()
    masked, pos, lab = (t.cpu() for t in (out.masked_ids, out.positions, out.labels))
    wd = {k: v.double().clone().requires_grad_(True) for k, v in w.items()}
    seq = onn.bert_encoder(wd, masked, dev['mask'].cpu(), None, num_layers=2, num_heads=2, dtype=torch.float64)
    h = seq.reshape(B * L, -1)[pos.long()]
    ref = mo.masked_lm_loss(mo.head_logits(h, wd, V), lab.long())
    ref.backward()
    assert abs(float(out.loss) - float(ref.detach())) < 2e-2 * max(1.0, float(ref.detach()))
    gscale = max(v.grad.abs().max().item() for n_, v in wd.items() if v.grad is not None)
    worst = {}
    for name, v in wd.items():
        if v.grad is None or "pooler" in name:
            continue
        g = store.grads[name].cpu().double()
        scale = max(v.grad.abs().max().item(), 1e-3 * gscale)
        worst[name] = (g - v.grad).abs().max().item() / scale
    print("max relative gradient error:", max(worst.values()), "over", len(worst), "variables")
    assert "cls/predictions/output_bias" in worst and "bert/embeddings/word_embeddings" in worst
    bad = {k: v for k, v in worst.items() if v > 8e-2}
    assert not bad, bad


def _corpus(N, L, rng, span=50):
    """Rows of successive token ids, token t = start + t mod span, with the start one of 0, 10, 20, 30: a masked token
    follows from its neighbours and from its position.  Predicting the ids' frequencies alone gives log(span) = 3.9 nats,
    above half the initial loss of log(V) = 6.9."""
    toks = (rng.choice([0, 10, 20, 30], N)[:, None] + np.arange(L)[None]) % span + 106
    toks[:, 0], toks[:, L - 1] = 101, 102
    return toks.astype(np.int32)


def _eval(dev, cfg, store):
    out = mlm.masked_lm(dev, cfg, store, 777, 0.15, 20, 103, False)
    return float(out.loss), int(out.correct) / max(1, int(out.count))


def test_masked_lm_learns_a_synthetic_corpus(tmp_path):
    cfg = bert.load_bert_config(_tiny_dir(tmp_path))
    store = variables.VariableStore('cuda', seed=4)
    rng = np.random.default_rng(0)
    B, L, V = 32, 32, TINY['vocab_size']
    train = _corpus(B * 40, L, rng)
    valid = _dev_batch(_corpus(128, L, rng), np.full(128, L, np.int32))
    with variables.use_store(store):
        bert.create_bert_variables(cfg, store)
        mlm.create_head_variables(cfg, store)
        loss0, acc0 = _eval(valid, cfg, store)
        for step in range(300):
            rows = train[(step * B) % len(train):][:B]
            dev = _dev_batch(rows, np.full(B, L, np.int32))
            store.dropout_calls = 0
            with autodiff.recording(store) as tape:
                out = mlm.masked_lm(dev, cfg, store, 1000 + step, 0.15, 20, 103, True, tape=tape)
                tape.backward()
                train_utils.bert_train_op(out.loss, 1e-3, 300, 0.1, None, store=store)
        loss1, acc1 = _eval(valid, cfg, store)
    print("held-out masked-LM loss %.3f -> %.3f, accuracy %.3f -> %.3f" % (loss0, loss1, acc0, acc1))
    assert loss1 < 0.5 * loss0 and acc1 > acc0


def test_pretrain_export_and_fine_tune(tmp_path):
    from chinesener_b200 import pretrain
    from chinesener_b200.data import corpus, records
    pdir = tmp_path / "tiny"
    pdir.mkdir()
    _tiny_dir(pdir)
    vocab = ["[PAD]"] + ["[unused%d]" % i for i in range(1, 100)] + ["[UNK]", "[CLS]", "[SEP]", "[MASK]"]
    vocab += [chr(0x4e00 + i) for i in range(TINY['vocab_size'] - len(vocab))]
    (pdir / "vocab.txt").write_text("\n".join(vocab) + "\n", encoding="utf-8")
    src = tmp_path / "a.txt"
    rng = np.random.default_rng(1)
    src.write_text("\n".join("".join(chr(0x4e00 + int(c)) for c in rng.integers(0, 800, 40)) for _ in range(60)), encoding="utf-8")
    data = tmp_path / "data"
    corpus.main(["--src", str(src), "--out", str(data), "--bert_dir", str(pdir), "--max_seq_len", "32", "--valid_fraction", "0.1"])
    out = tmp_path / "out"
    args = ["--data_dir", str(data), "--pretrain_dir", str(pdir), "--output_dir", str(out), "--num_train_steps", "4",
            "--batch_size", "8", "--save_steps", "2", "--report", str(tmp_path / "report.json")]
    rep = pretrain.main(args)
    assert rep["global_step"] == 4 and np.isfinite(rep["valid"][-1]["perplexity"])
    est = engine.Estimator('bert_crf', dict(synthetic.data_params(32), pretrain_dir=str(out)))
    feats = synthetic.msra_batch(4, 32, vocab=TINY['vocab_size'], seed=2)
    est.train_step(feats)                                 # one TRAIN step from the exported checkpoint
    exported = np.load(str(out / "model.ckpt-4.npz"))
    fresh = engine.Estimator('bert_crf', dict(synthetic.data_params(32), pretrain_dir=str(out)))
    fresh.evaluate(feats)
    for name, v in fresh.store.vars.items():
        if name.startswith("bert/"):
            assert np.array_equal(v.cpu().numpy(), exported[name]), name
    rep2 = pretrain.main([a if a != "4" else "6" for a in args])         # resumes at global_step 4
    assert rep2["resumed_from"] == 4 and rep2["global_step"] == 6
