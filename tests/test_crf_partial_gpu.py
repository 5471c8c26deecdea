"""GPU: the partial-annotation CRF kernels (ner_crf_partial_loglik_fwd / _bwd) against the float64 reference of
tests/_crf_partial_oracle.py, their exactness properties, and the CRF plugins trained and evaluated on partial labels.

`bwd_route` (tests/_crf_grad_oracle.py) restates the kernels' choice: lane per tag up to 4096 sequences, 64-thread CTAs
above 128 sequences per SM (the backward only while its staging ring fits in shared memory), 32-thread CTAs otherwise.
Every case weights its rows with a random d_ll and a scale != 1 and is judged by assert_close_to_ref with the bound of
its route.
"""
import os

import numpy as np
import pytest
import torch

from chinesener_b200 import autodiff, engine, ops, synthetic, variables

from _crf_grad_oracle import TOL as _ROUTE_TOL, _worst_ratio, bwd_route, grad_errors
from _crf_partial_oracle import partial_grad_ref, partial_ll_torch

pytestmark = pytest.mark.gpu

SCALE = 0.75
# d_logits: the bound of the existing route for the same batch sizes (lanes / nt32 / nt64 of _crf_grad_oracle.TOL).
# d_trans: |err| <= tol_s S + C_T U, with tol_s of that route and U the float32 rounding of log-domain marginals
# (_crf_partial_oracle.partial_grad_ref).  U is what makes rows with large |log Z| (long rows, wide transitions, allowed
# tags far below a disallowed one) err beyond tol_s S; ner_crf_loglik_bwd does the same on those rows
# (test_existing_backward_meets_the_same_bound).  At L = 128 a skipped step is > 16 C_T U (test_crf_partial_oracle.py).
TOL = _ROUTE_TOL
C_T = 4.0
NF = 3          # staged float tensors of the backward: logits, alpha_A, alpha (64-thread CTAs fit up to K = 17)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def assert_close_to_ref(d_logits, d_trans, ref, B, K):
    """-> (d_logits error in u_b, d_trans error in U beyond tol_s S, d_trans error in S)."""
    rtol, c_dl, tol_s = TOL[bwd_route(B, K, NF)]
    e_dl, e_s, e_g = grad_errors(d_logits, d_trans, ref.grad, rtol)
    assert e_dl <= c_dl, f"d_logits error {e_dl:.3g} u_b ({e_g:.3e} |g_b|) exceeds {c_dl:.3g} u_b"
    err = (d_trans.to(ref.grad.d_trans.device, torch.float64) - ref.grad.d_trans).abs()
    e_u = _worst_ratio((err - tol_s * ref.grad.trans_scale).clamp(min=0), ref.trans_unit)
    assert e_u <= C_T, f"d_trans error {e_s:.3e} S: {e_u:.3g} U beyond {tol_s:.1e} S exceeds {C_T} U"
    return e_dl, e_u, e_s


def _batch(B):
    return 128 * _sms() + 301 if B == "big" else B


def _case(B, L, K, seed, trans="fast", low=False):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, K, generator=gen) * 2
    if trans == "fast":
        tr = torch.randn(K, K, generator=gen) * 0.5
    elif trans == "wide":
        tr = torch.randn(K, K, generator=gen) * 12
    else:                                                     # forbidden transitions
        tr = torch.randn(K, K, generator=gen)
        if K > 1:
            tr[0, 1] = tr[1, 0] = -float("inf")
    lens = torch.randint(0, L + 1, (B,), generator=gen, dtype=torch.int32)
    for i, n in enumerate((0, 1, 2, L)):
        if i < B:
            lens[i] = n
    full = (1 << K) - 1 if K < 32 else -1
    onehot = torch.ones((B, L), dtype=torch.int64) << torch.randint(0, K, (B, L), generator=gen)
    subset = torch.randint(0, 1 << min(K, 31), (B, L), generator=gen, dtype=torch.int64) | onehot
    pick = torch.randint(0, 3, (B, L), generator=gen)
    mask = torch.where(pick == 0, onehot, torch.where(pick == 1, torch.full_like(onehot, full), subset))
    mask = ((mask + (1 << 31)) % (1 << 32) - (1 << 31)).to(torch.int32)
    if low:                                                   # allowed tags 70 nats below the best disallowed one
        allowed = ((mask.long()[..., None] & 0xFFFFFFFF) >> torch.arange(K)) & 1
        x = torch.where(allowed.bool() & (allowed.sum(-1, keepdim=True) < K), x - 70.0, x)
    d_ll = torch.randn(B, generator=gen)
    return x, mask, lens, tr, d_ll


def _run(x, mask, lens, tr, d_ll, exact=False):
    dev = [t.cuda() for t in (x, mask, lens, tr, d_ll)]
    ll, logz, alpha = ops.crf_partial_loglik_fwd(dev[0], dev[1], dev[2], dev[3], want_alpha=True, exact=exact)
    nan = torch.full_like(dev[0], float("nan"))               # d_logits lands where NaNs were last held
    del nan
    d_logits, d_trans = ops.crf_partial_loglik_bwd(dev[0], dev[1], dev[2], dev[3], alpha, logz, dev[4], SCALE)
    torch.cuda.synchronize()
    return ll.cpu(), logz.cpu(), d_logits, d_trans


def _check(x, mask, lens, tr, d_ll, B, K, exact=False):
    ll, _, d_logits, d_trans = _run(x, mask, lens, tr, d_ll, exact)
    ref = partial_grad_ref(x.cuda().double(), mask.cuda(), lens.cuda(), tr.cuda(), (d_ll * SCALE).cuda())
    rll = ref.ll.cpu()
    fin = torch.isfinite(rll)
    assert torch.equal(torch.isfinite(ll), fin) and (ll[~fin] == -float("inf")).all()
    err = (ll[fin].double() - rll[fin]).abs()
    assert (err <= 1e-4 * rll[fin].abs() + 1e-4).all(), float(err.max())
    L = x.shape[1]
    past = torch.arange(L, device="cuda")[None, :] >= lens.cuda().clamp(0, L)[:, None]
    assert (d_logits[past] == 0).all()
    e = assert_close_to_ref(d_logits, d_trans, ref, B, K)
    print(f"B={B} L={L} K={K} route={bwd_route(B, K, NF)}: d_logits {e[0]:.3g} u_b, d_trans {e[2]:.2e} S, {e[1]:.3g} U")
    return ll, d_logits, d_trans


CASES = [  # B, L, K, trans
    (1, 1, 1, "fast"), (7, 2, 2, "fast"), (64, 128, 10, "fast"), (64, 128, 10, "wide"), (64, 128, 10, "inf"),
    (7, 512, 17, "fast"), (64, 128, 32, "fast"), (4097, 128, 10, "fast"), ("big", 128, 10, "fast"),
    ("big", 128, 17, "inf"), ("big", 64, 32, "wide"), (7, 2048, 10, "fast"), (64, 128, 1, "wide"),
    (4097, 2, 2, "inf"), (4097, 128, 10, "wide"), (4097, 128, 10, "inf"), (4097, 256, 17, "fast"),
    (4097, 64, 32, "fast"), (4097, 128, 10, "fast", True), (4096, 128, 10, "fast"),
]


@pytest.mark.parametrize("case", CASES)
def test_kernels_match_the_float64_reference(case):
    B, L, K, trans = case[:4]
    low = len(case) > 4
    B = _batch(B)
    _check(*_case(B, L, K, seed=B + L + K, trans=trans, low=low), B, K)


@pytest.mark.parametrize("B,L,K,trans", [(7, 2048, 10, "fast"), (64, 128, 10, "wide"), (4097, 256, 17, "fast")])
def test_existing_backward_meets_the_same_bound(B, L, K, trans):
    """ner_crf_loglik_bwd on the same kind of rows, against the same float64 reference (a one-hot mask is the ordinary
    CRF): beyond tol_s S its d_trans error is of the size of U too."""
    x, _, lens, tr, d_ll = _case(B, L, K, seed=B + L + K, trans=trans)
    tags = torch.randint(0, K, (B, L), generator=torch.Generator().manual_seed(7), dtype=torch.int32)
    mask = (torch.ones_like(tags, dtype=torch.int64) << tags.long()).to(torch.int32)
    dev = [t.cuda() for t in (x, tags, lens, tr, d_ll)]
    _, logz, alpha = ops.crf_loglik_fwd(dev[0], dev[1], dev[2], dev[3], want_alpha=True)
    d_logits, d_trans = ops.crf_loglik_bwd(dev[0], dev[1], dev[2], dev[3], alpha, logz, dev[4], SCALE)
    ref = partial_grad_ref(x.cuda().double(), mask.cuda(), lens.cuda(), tr.cuda(), (d_ll * SCALE).cuda())
    e = assert_close_to_ref(d_logits, d_trans, ref, B, K)
    print(f"ner_crf_loglik_bwd B={B} L={L} K={K} {trans}: d_trans {e[2]:.2e} S, {e[1]:.3g} U")


@pytest.mark.parametrize("B,L,K", [(64, 128, 10), (7, 60, 17), ("big", 128, 10)])
def test_exact_path_flag(B, L, K):
    B = _batch(B)
    _check(*_case(B, L, K, seed=5 + K), B, K, exact=True)


@pytest.mark.parametrize("B,K", [(64, 10), ("big", 10), (64, 32)])
def test_allowed_tags_far_below_a_disallowed_one(B, K):
    B = _batch(B)
    ll, d_logits, _ = _check(*_case(B, 128, K, seed=9, low=True), B, K)
    assert torch.isfinite(ll).all() and torch.isfinite(d_logits).all()


@pytest.mark.parametrize("B,K", [(64, 10), ("big", 10), (7, 32)])
def test_one_hot_masks_equal_the_ordinary_crf(B, K):
    B = _batch(B)
    x, _, lens, tr, d_ll = _case(B, 96, K, seed=13)
    tags = torch.randint(0, K, (B, 96), generator=torch.Generator().manual_seed(2), dtype=torch.int32)
    mask = (((torch.ones_like(tags, dtype=torch.int64) << tags.long()) + (1 << 31)) % (1 << 32) - (1 << 31)).to(torch.int32)
    ll, _, d_logits, d_trans = _run(x, mask, lens, tr, d_ll)
    ref = partial_grad_ref(x.cuda().double(), mask.cuda(), lens.cuda(), tr.cuda(), (d_ll * SCALE).cuda())
    ll_full, _, _ = ops.crf_loglik_fwd(x.cuda(), tags.cuda(), lens.cuda(), tr.cuda())
    torch.testing.assert_close(ll, ll_full.cpu(), rtol=1e-4, atol=1e-4)
    assert_close_to_ref(d_logits, d_trans, ref, B, K)


def test_exactness_properties():
    B, L, K = 256, 128, 10
    x, mask, lens, tr, d_ll = _case(B, L, K, seed=21)
    full = (1 << K) - 1
    mask[:64] = full                                          # all-allowed rows
    mask[64, 0] = 0                                           # an empty set at t = 0 ...
    lens[64] = L
    mask[65, L // 2] = 0                                      # ... and mid-row
    lens[65] = L
    ll, logz, d_logits, d_trans = _run(x, mask, lens, tr, d_ll)
    assert (ll[:64] == 0).all() and (d_logits[:64] == 0).all()
    assert ll[64] == -float("inf") and ll[65] == -float("inf")
    assert (d_logits[64:66] == 0).all()
    # the two empty rows add nothing to d_trans
    keep = torch.ones(B, dtype=torch.bool)
    keep[64:66] = False
    _, _, _, d_trans_wo = _run(x, torch.where(keep[:, None], mask, torch.full_like(mask, full)), lens, tr,
                               torch.where(keep, d_ll, torch.zeros_like(d_ll)))
    torch.testing.assert_close(d_trans, d_trans_wo, rtol=1e-6, atol=1e-6)
    # garbage bits >= K change nothing, bit for bit; repeats are bit-identical
    garbage = (mask.long() | (((1 << 32) - 1) ^ full)).to(torch.int64)
    garbage = ((garbage + (1 << 31)) % (1 << 32) - (1 << 31)).to(torch.int32)
    ll_g, _, dl_g, dt_g = _run(x, garbage, lens, tr, d_ll)
    assert torch.equal(ll_g, ll) and torch.equal(dl_g, d_logits)
    torch.testing.assert_close(dt_g, d_trans, rtol=1e-6, atol=1e-6)   # float atomics: the summation order varies
    ll_r, _, dl_r, _ = _run(x, mask, lens, tr, d_ll)
    assert torch.equal(ll_r, ll) and torch.equal(dl_r, d_logits)


def compose(x, mask, lens, tr, d_ll, scale):
    """The same result from the existing kernels: -inf-masked logits, ner_crf_loglik_fwd and _bwd twice, a
    subtraction (tags 0 in both halves, so the gold-path terms cancel)."""
    B, L, K = x.shape
    allowed = ((mask.long()[..., None] & 0xFFFFFFFF) >> torch.arange(K, device=x.device)) & 1
    xa = torch.where(allowed.bool(), x, torch.full_like(x, -float("inf")))
    tags = torch.zeros((B, L), dtype=torch.int32, device=x.device)
    _, lza, aa = ops.crf_loglik_fwd(xa, tags, lens, tr, want_alpha=True)
    _, lzf, af = ops.crf_loglik_fwd(x, tags, lens, tr, want_alpha=True)
    da, ta = ops.crf_loglik_bwd(xa, tags, lens, tr, aa, lza, d_ll, scale)
    df, tf = ops.crf_loglik_bwd(x, tags, lens, tr, af, lzf, d_ll, scale)
    return lza - lzf, df - da, tf - ta


@pytest.mark.parametrize("B", [64, "big"])
def test_fused_kernels_agree_with_the_composition(B):
    B = _batch(B)
    x, mask, lens, tr, d_ll = _case(B, 128, 10, seed=31)
    lens[:] = lens.clamp(min=1)                               # the composition has no empty-set rule
    ll, _, d_logits, d_trans = _run(x, mask, lens, tr, d_ll)
    cl, cd, ct = compose(x.cuda(), mask.cuda(), lens.cuda(), tr.cuda(), d_ll.cuda(), SCALE)
    torch.testing.assert_close(ll, cl.cpu(), rtol=1e-4, atol=1e-4)
    ref = partial_grad_ref(x.cuda().double(), mask.cuda(), lens.cuda(), tr.cuda(), (d_ll * SCALE).cuda())
    e_fused = grad_errors(d_logits, d_trans, ref.grad, 0.0)
    e_comp = grad_errors(cd, ct, ref.grad, 0.0)
    print(f"B={B}: fused {e_fused[2]:.2e} |g|, composition {e_comp[2]:.2e} |g|")
    g = (SCALE * d_ll.abs()).cuda()[:, None, None]
    assert ((d_logits - cd).abs() <= 2e-3 * g).all()


# ------------------------------------------------------------------------------------------------------ plugin level

def _partial_mask(feats, K, frac=0.3, seed=0):
    """label_mask of a batch: the one-hot of label_ids, with `frac` of the real tokens opened to every real tag."""
    lab = feats['label_ids'].long().clamp(0, K - 1)
    mask = torch.ones_like(lab) << lab
    g = torch.Generator().manual_seed(seed)
    L = lab.shape[1]
    real = torch.arange(L)[None, :] < feats['seq_len'][:, None]
    opened = (torch.rand(lab.shape, generator=g) < frac) & real
    return torch.where(opened, torch.full_like(mask, ((1 << K) - 1) & ~1), mask).to(torch.int32)


def _train_grads(est, feats):
    dev = est.to_device(feats)
    for g in est.store.grads.values():
        g.zero_()
    with variables.use_store(est.store), autodiff.recording(est.store) as tape:
        loss, _ = est.build_graph(dev, None, est.params, True)
        tape.backward()
    return float(loss), {k: v.detach().clone().cpu().double() for k, v in est.store.grads.items()}


def _bilstm_setup():
    from test_training_gpu import _setup
    return _setup(B=8, L=48)


def test_bilstm_crf_partial_gradients_match_oracle_autograd():
    from oracle import nn as onn
    est, feats, emb = _bilstm_setup()
    feats['label_mask'] = _partial_mask(feats, 10)
    est.evaluate(feats)
    w = est.store.state_dict()
    wd = {k: v.double().clone().requires_grad_(True) for k, v in w.items()}
    x = torch.from_numpy(emb).double()[feats['token_ids'].long()]
    lstm = onn.bilstm(x, wd, feats['seq_len'], est.params['rnn_activation'], 1.0, torch.float64)
    logits = lstm @ wd['logits/kernel'] + wd['logits/bias']
    ref_loss = (-partial_ll_torch(logits, feats['label_mask'], feats['seq_len'], wd['crf_layer/transitions'])).mean()
    ref_loss.backward()
    loss, grads = _train_grads(est, feats)
    assert abs(loss - ref_loss.item()) < 2e-3 * max(1.0, abs(ref_loss.item()))
    for name, v in wd.items():
        scale = max(v.grad.abs().max().item(), 1e-6)
        assert (grads[name] - v.grad).abs().max().item() < 2e-2 * scale, name


def test_lattice_lstm_crf_partial_gradients_match_oracle_autograd():
    from test_lattice_gpu import _oracle_loss, _setup
    est, feats = _setup(L=32)
    feats['label_mask'] = _partial_mask(feats, 10, seed=1)
    est.evaluate(feats)
    wd = {k: v.double().clone().requires_grad_(True) for k, v in est.store.state_dict().items()}
    _, logits = _oracle_loss(wd, feats, est.params)
    ref_loss = (-partial_ll_torch(logits, feats['label_mask'], feats['seq_len'], wd['crf_layer/transitions'])).mean()
    ref_loss.backward()
    loss, grads = _train_grads(est, feats)
    assert abs(loss - ref_loss.item()) < 2e-3 * max(1.0, abs(ref_loss.item()))
    for name, v in wd.items():
        scale = max(v.grad.abs().max().item(), 1e-6)
        assert (grads[name] - v.grad).abs().max().item() < 2e-2 * scale, name


def test_bert_bilstm_crf_partial_gradients_match_oracle_autograd(tmp_path):
    from oracle import crf_torch  # noqa: F401  (the oracle graph's CRF is replaced by the partial loss below)
    from oracle import nn as onn
    from test_bert_training_gpu import _est
    est, feats = _est(tmp_path, model="bert_bilstm_crf")
    feats['label_mask'] = _partial_mask(feats, 10, seed=4)
    est.evaluate(feats)
    est.store.vars["logits/kernel"].mul_(4.0)
    est.store.touch()
    wd = {k: v.double().clone().requires_grad_(True) for k, v in est.store.state_dict().items()}
    seq = onn.bert_encoder(wd, feats['token_ids'], feats['mask'], feats['segment_ids'], num_layers=2, num_heads=12,
                           dtype=torch.float64)
    seq = onn.bilstm(seq, wd, feats['seq_len'], est.params['rnn_activation'], 1.0, torch.float64)
    logits = seq @ wd['logits/kernel'] + wd['logits/bias']
    ref_loss = (-partial_ll_torch(logits, feats['label_mask'], feats['seq_len'], wd['crf_layer/transitions'])).mean()
    ref_loss.backward()
    loss, grads = _train_grads(est, feats)
    assert abs(loss - ref_loss.item()) < 2e-2 * max(1.0, abs(ref_loss.item()))
    ref = {k: v.grad for k, v in wd.items() if v.grad is not None and "pooler" not in k}
    top = max(g.abs().max().item() for g in ref.values())
    for name, g_ref in ref.items():            # the bert_bilstm_crf TRAIN bar of DESIGN.md §4
        scale = max(g_ref.abs().max().item(), 1e-3 * top)
        assert (grads[name] - g_ref).abs().max().item() < 8e-2 * scale, name


def _bert_estimator(tmp_path, name="bert_bilstm_crf", B=6, L=48):
    import json
    from test_models_gpu import SMALL_BERT
    cfg = dict(SMALL_BERT, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    (tmp_path / "bert_config.json").write_text(json.dumps(cfg))
    feats = synthetic.msra_batch(B, L, vocab=SMALL_BERT['vocab_size'], seed=5)
    params = dict(synthetic.data_params(L), pretrain_dir=str(tmp_path), embedding_dropout=0.0, keep_prob_list=[1.0])
    return engine.Estimator(name, params), feats


@pytest.mark.parametrize("plugin", ["bilstm_crf", "bert_bilstm_crf", "lattice_lstm_crf"])
def test_one_hot_label_mask_trains_like_full_labels(plugin, tmp_path):
    if plugin == "bilstm_crf":
        est, feats, _ = _bilstm_setup()
    elif plugin == "lattice_lstm_crf":
        from test_lattice_gpu import _setup
        est, feats = _setup(L=32)
    else:
        est, feats = _bert_estimator(tmp_path)
    est.evaluate(feats)
    loss0, g0 = _train_grads(est, feats)
    onehot = dict(feats, label_mask=(torch.ones_like(feats['label_ids'], dtype=torch.int64)
                                     << feats['label_ids'].long()).to(torch.int32))
    loss1, g1 = _train_grads(est, onehot)
    assert abs(loss1 - loss0) < 1e-4 * max(1.0, abs(loss0))
    # the plugins' TRAIN gradient bars (DESIGN.md §4): of max(|g|, 1e-3 * global scale)
    bar = 8e-2 if plugin.startswith("bert") else 2e-2
    top = max(g.abs().max().item() for g in g0.values())
    for name in g0:
        scale = max(g0[name].abs().max().item(), 1e-3 * top, 1e-6)
        assert (g1[name] - g0[name]).abs().max().item() < bar * scale, name


def _plugin(name, tmp_path):
    """An Estimator and a batch of each CRF plugin, from the setups of that plugin's own tests."""
    if name == "bilstm_crf":
        return _bilstm_setup()[:2]
    if name in ("bert_bilstm_crf", "bert_crf", "bert_cnn_crf"):
        return _bert_estimator(tmp_path, name)
    if name == "lattice_lstm_crf":
        from test_lattice_gpu import _setup
        return _setup(L=32)
    if name == "transformer_crf_bichar":
        from test_tener_gpu import _abs_setup
        return _abs_setup()[:2]
    if name == "transformer_tener_crf_bichar":
        from test_tener_gpu import _tener_setup
        return _tener_setup()[:2]
    from test_word_enhance_gpu import _setup
    return _setup(name, dropout=0.0, keep=1.0)


EVAL_PLUGINS = ["bilstm_crf", "bert_bilstm_crf", "bert_crf", "bert_cnn_crf", "lattice_lstm_crf", "transformer_crf_bichar",
                "transformer_tener_crf_bichar", "bilstm_crf_bichar", "bilstm_crf_softword", "bilstm_crf_ex_softword"]


@pytest.mark.parametrize("plugin", EVAL_PLUGINS)
def test_eval_loss_with_a_mask(plugin, tmp_path, monkeypatch):
    """Through crf_head / crf_layer (transformer_crf_bichar calls crf_layer itself): the EVAL loss of a masked batch is
    mean(-ll) of the partial CRF on the plugin's own emissions, and an all-open mask gives a loss of exactly 0."""
    from chinesener_b200.tools import layer
    seen = {}
    orig = layer.crf_layer

    def spy(logits, label_ids, seq_len, label_size, is_training, label_mask=None):
        seen['args'] = (logits, seq_len, label_mask)
        return orig(logits, label_ids, seq_len, label_size, is_training, label_mask=label_mask)

    import importlib
    est, feats = _plugin(plugin, tmp_path)
    monkeypatch.setattr(layer, "crf_layer", spy)
    mod = importlib.import_module("chinesener_b200.model." + plugin)
    if hasattr(mod, "crf_layer"):                             # imported by name (transformer_crf_bichar)
        monkeypatch.setattr(mod, "crf_layer", spy)
    feats['label_mask'] = _partial_mask(feats, 10, seed=3)
    out = est.evaluate(feats)
    logits, seq_len, mask = seen['args']
    assert mask is not None
    tr = est.store.vars['crf_layer/transitions']
    ref = partial_grad_ref(logits.double(), mask, seq_len, tr)
    assert abs(out['loss'] - float((-ref.ll).mean())) < 1e-4 * max(1.0, abs(out['loss']))
    feats['label_mask'] = torch.full_like(feats['label_mask'], (1 << 10) - 1)
    assert est.evaluate(feats)['loss'] == 0.0


def test_main_driver_on_a_partially_labelled_split(tmp_path):
    """A synthetic split with 30 % of its real tokens opened to every tag: main.py trains, evaluates and writes its
    predict pickle, and skips the entity report."""
    import pickle
    from chinesener_b200 import main as driver
    from chinesener_b200.data.records import RecordFile, write_records
    from chinesener_b200.data.tokenizer import TokenizerBert
    from test_main_driver_gpu import _setup
    root, pre = _setup(tmp_path)
    data_dir = os.path.join(root, 'msra')
    rng = np.random.default_rng(0)
    for split in ('train', 'valid', 'predict'):
        path = os.path.join(data_dir, '{}_{}.nerrec'.format(TokenizerBert, split))
        rec = RecordFile(path)
        b = rec.batch(slice(0, rec.n))
        lab = b['label_ids'].numpy()
        opened = (rng.random(lab.shape) < 0.3) & (lab > 0) & (lab < 8)
        feats = []
        for i in range(rec.n):
            f = {k: (v[i].tolist() if torch.is_tensor(v) else v[i]) for k, v in b.items()}
            f['label_ids'] = [-1 if o else int(t) for t, o in zip(lab[i], opened[i])]
            f['label_mask'] = [(1 << 8) - 2 if o else 1 << int(t) for t, o in zip(lab[i], opened[i])]
            feats.append(f)
        del rec, b
        write_records(path, feats, lab.shape[1])
    with pytest.warns(UserWarning):                    # no BERT checkpoint in pretrain_dir: random init
        s = driver.main(['--model_name', 'bert_bilstm_crf', '--data', 'msra', '--data_dir', data_dir,
                         '--checkpoint_root', str(tmp_path / 'ckpt'), '--pretrain_dir', pre, '--epoch_size', '2',
                         '--batch_size', '4'])
    assert s['history']['final_step'] > 0 and np.isfinite(s['history']['evals'][-1]['loss'])
    assert 'entity_micro_f1' not in s and 0 <= s['tag_accuracy'] <= 1
    pred = pickle.load(open(os.path.join(data_dir, 'bert_bilstm_crf_predict.pkl'), 'rb'))
    assert len(pred) == s['n_predict'] and (np.concatenate([p['label_ids'] for p in pred]) == -1).any()
