"""GPU: the CRF distillation kernels (ner_crf_distill_fwd / _bwd) against the float64 reference of
tests/_crf_distill_oracle.py, their exactness properties, and a CRF student trained against a teacher through
Estimator(teacher=...).

Every kernel case weights its rows with a random d_kl and a scale != 1 and is judged with the bound of its route
(_crf_grad_oracle.TOL): lane per tag up to 4096 sequences, 64-thread CTAs above 128 sequences per SM where the
backward's four-tensor staging ring fits in shared memory (K <= 13), 32-thread CTAs where it fits (K <= 25), lane per
tag beyond.
"""
import numpy as np
import pytest
import torch

from chinesener_b200 import autodiff, engine, ops, synthetic, variables

from _crf_distill_oracle import distill_ref
from _crf_grad_oracle import EPS32, TOL, SMALL_B, _worst_ratio, grad_errors

pytestmark = pytest.mark.gpu

SCALE = 0.75
C_T = 4.0       # d_trans: |err| <= tol_s S + C_T U, U the float32 rounding of log-domain marginals (as the partial CRF)
C_T_DOC = 32.0  # at document length (L > 2048): 17.4 U on an H100 at L = 4095; ner_crf_loglik_bwd 14.5 U on those rows
C_KL = 8.0      # KL: |err| <= 1e-4 (1 + |logZ_T| + |logZ_S| + |KL|) + C_KL r_b M_b (4.9 r_b M_b measured at L = 2048)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _smem(K, NT):
    return 4 * (6 * ((K * K + 3) & ~3) + 64 + NT + 4 * 2 * NT * (8 * K + 4))


def route(B, K):
    if B <= SMALL_B:
        return "lanes"
    if B > 128 * _sms() and _smem(K, 64) <= 227 * 1024:
        return "nt64"
    return "nt32" if _smem(K, 32) <= 227 * 1024 else "lanes"


def _batch(B):
    return 128 * _sms() + 301 if B == "big" else B


def _trans(kind, K, gen):
    if kind == "fast":
        return torch.randn(K, K, generator=gen) * 0.5
    if kind == "wide":
        return torch.randn(K, K, generator=gen) * 12
    tr = torch.randn(K, K, generator=gen)                   # forbidden transitions
    if K > 1:
        tr[0, 1] = tr[1, 0] = -float("inf")
    return tr


def _case(B, L, K, seed, t_kind="fast", s_kind="fast"):
    gen = torch.Generator().manual_seed(seed)
    xt = torch.randn(B, L, K, generator=gen) * 2
    xs = torch.randn(B, L, K, generator=gen) * 2
    trt, trs = _trans(t_kind, K, gen), _trans(s_kind, K, gen)
    lens = torch.randint(-1, L + 3, (B,), generator=gen, dtype=torch.int32)        # seq_len <= 0 and > L included
    for i, n in enumerate((0, 1, 2, L, -3, L + 5)):
        if i < B:
            lens[i] = n
    return xt, trt, xs, trs, lens, torch.randn(B, generator=gen)


def _run(xt, trt, xs, trs, lens, d_kl, tau=1.0, exact=False):
    dev = [t.cuda() for t in (xt, trt, xs, trs, lens, d_kl)]
    logz, alpha = ops.crf_distill_fwd(*dev[:5], tau, exact=exact)
    kl, d_logits, d_trans = ops.crf_distill_bwd(*dev[:5], alpha, logz, tau, d_kl=dev[5], scale=SCALE, exact=exact)
    torch.cuda.synchronize()
    return kl.cpu(), d_logits, d_trans


def _check(xt, trt, xs, trs, lens, d_kl, tau=1.0, exact=False, kernel_inputs=None):
    """kernel_inputs: run the kernels at tau = 1 on these instead (and judge them against the reference at tau)."""
    B, L, K = xs.shape
    if kernel_inputs is None:
        kl, d_logits, d_trans = _run(xt, trt, xs, trs, lens, d_kl, tau=tau, exact=exact)
    else:
        kl, d_logits, d_trans = _run(*kernel_inputs, tau=1.0, exact=exact)
        d_logits, d_trans = d_logits / tau, d_trans / tau       # d/dx of KL at tau is (1/tau) d/d(x/tau)
    c = [t.cuda() for t in (xt, trt, xs, trs, lens)]
    ref = distill_ref(*c, tau=tau, g=(d_kl * SCALE).cuda())
    g = ref.grad
    valid = (torch.arange(L, device="cuda")[None, :] < g.lens[:, None])[:, :, None] & torch.isfinite(g.alpha)
    amax = torch.where(valid, g.alpha.abs(), torch.zeros_like(g.alpha)).reshape(B, -1).max(dim=1).values
    r = EPS32 * (1 + g.logz.abs() + amax)
    # KL: 1e-4 relative to the log-partitions it cancels, plus C_T times the float32 rounding of the log-domain
    # marginals (r_b) over the size of the terms it sums (M_b)
    rkl = ref.kl.cpu()
    err = (kl.double() - rkl).abs()
    bound = 1e-4 * (1 + ref.logz_t.abs().cpu() + ref.logz_s.abs().cpu() + rkl.abs()) + C_KL * (r * ref.kl_scale).cpu()
    assert (err <= bound).all(), float((err / bound).max())
    past = torch.arange(L, device="cuda")[None, :] >= lens.cuda().clamp(0, L)[:, None]
    assert (d_logits[past] == 0).all()
    rtol, c_dl, tol_s = TOL[route(B, K)]
    e_dl, e_s, e_g = grad_errors(d_logits, d_trans, ref.grad, rtol)
    assert e_dl <= c_dl, f"d_logits error {e_dl:.3g} u_b ({e_g:.3e} |g_b|) exceeds {c_dl:.3g} u_b"
    unit = distill_ref(*c, tau=tau, g=(d_kl * SCALE).cuda().double().abs() * r).grad.trans_scale
    err_t = (d_trans.double() - g.d_trans).abs()
    e_u = _worst_ratio((err_t - tol_s * g.trans_scale).clamp(min=0), unit)
    c_t = C_T if L <= 2048 else C_T_DOC
    assert e_u <= c_t, f"d_trans error {e_s:.3e} S: {e_u:.3g} U beyond {tol_s:.1e} S exceeds {c_t} U"
    print(f"B={B} L={L} K={K} route={route(B, K)}: kl {float((err / bound).max()):.3g}, d_logits {e_dl:.3g} u_b, "
          f"d_trans {e_s:.2e} S, {e_u:.3g} U")


CASES = [  # B, L, K, teacher transitions, student transitions
    (1, 1, 1, "fast", "fast"), (1, 2, 2, "wide", "fast"), (63, 128, 10, "fast", "fast"), (63, 128, 10, "wide", "fast"),
    (63, 128, 10, "fast", "wide"), (63, 128, 10, "inf", "fast"), (63, 2048, 7, "fast", "fast"),
    (4, 4095, 10, "fast", "fast"), (63, 128, 32, "fast", "fast"), (4096, 128, 10, "fast", "fast"),
    (4097, 128, 10, "fast", "fast"), (4097, 128, 10, "inf", "wide"), (4097, 128, 17, "fast", "fast"),
    (4097, 64, 32, "fast", "fast"), (4097, 2, 3, "wide", "wide"), ("big", 128, 10, "fast", "fast"),
    ("big", 128, 10, "inf", "fast"), ("big", 64, 26, "fast", "wide"), ("big", 32, 32, "fast", "fast"),
    ("big", 128, 5, "fast", "fast"), (63, 128, 13, "fast", "fast"), (4097, 1, 4, "fast", "fast"),
]


@pytest.mark.parametrize("case", CASES)
def test_kernels_match_the_float64_reference(case):
    B, L, K, tk, sk = case
    B = _batch(B)
    _check(*_case(B, L, K, seed=B + L + K, t_kind=tk, s_kind=sk))


@pytest.mark.parametrize("B", [63, 4097])
@pytest.mark.parametrize("K", list(range(1, 33)))
def test_every_tag_count(B, K):
    _check(*_case(B, 24, K, seed=K, t_kind="fast", s_kind="fast"))


@pytest.mark.parametrize("B", [63, 4097, "big"])
def test_exact_path_flag(B):
    B = _batch(B)
    _check(*_case(B, 128, 10, seed=5), exact=True)


@pytest.mark.parametrize("tau", [0.5, 2.0])
@pytest.mark.parametrize("B", [63, 4097])
def test_temperature_equals_scaled_inputs(B, tau):
    xt, trt, xs, trs, lens, d_kl = _case(B, 128, 10, seed=11)
    _check(xt, trt, xs, trs, lens, d_kl, tau=tau)
    # the kernel at tau = 1 on (x / tau, T / tau) meets the same bound against the reference at tau
    scaled = (xt / tau, trt / tau, xs / tau, trs / tau, lens, d_kl)
    _check(xt, trt, xs, trs, lens, d_kl, tau=tau, kernel_inputs=scaled)


@pytest.mark.parametrize("B", [63, 4097, "big"])
@pytest.mark.parametrize("kind", ["fast", "wide", "inf"])
def test_teacher_equal_to_student_is_exactly_zero(B, kind):
    B = _batch(B)
    xt, trt, _, _, lens, d_kl = _case(B, 128, 10, seed=3, t_kind=kind)
    kl, d_logits, d_trans = _run(xt, trt, xt, trt, lens, d_kl, tau=0.7)
    assert (kl == 0).all()
    assert (d_logits == 0).all() and (d_trans == 0).all()


# ----------------------------------------------------------------------------------------------------- plugins

def _train_grads(est, feats):
    dev = est.to_device(feats)
    for g in est.store.grads.values():
        g.zero_()
    est.store.dropout_calls = 0
    teacher = est.teacher_potentials(dev) + est.distill_settings()
    from chinesener_b200.tools import layer
    with est._layer_settings(dev), variables.use_store(est.store), autodiff.recording(est.store) as tape:
        layer.CRF_TEACHER = teacher
        loss, _ = est.build_graph(dev, None, est.params, True)
        tape.backward()
    return float(loss), {k: v.detach().clone().cpu().double() for k, v in est.store.grads.items()}, teacher


def _bilstm_pair(alpha=0.5, tau=2.0, teacher="bilstm_crf_softlexicon"):
    """A bilstm_crf student, its teacher (bilstm_crf_softlexicon or lattice_lstm_crf) and a batch carrying the
    teacher's features, from the setups of the teacher's own tests."""
    if teacher == "lattice_lstm_crf":
        from test_lattice_gpu import _setup
        t_est, feats = _setup(L=32, dropout=0.0)
        emb = t_est.params['embedding']
    else:
        from test_training_gpu import _softlex_setup
        t_est, feats, emb = _softlex_setup(L=32)
    t_est.evaluate(feats)
    params = dict(synthetic.data_params(32), embedding=emb, embedding_dropout=0.0, keep_prob_list=[1.0],
                  distill_alpha=alpha, distill_temperature=tau)
    student = engine.Estimator("bilstm_crf", params, teacher=t_est)
    student.evaluate(feats)
    return student, feats, emb


def _ref_loss(logits, trans, feats, pot, alpha, tau):
    from oracle import crf_torch
    from _crf_partial_oracle import partial_ll_torch
    lens = feats['seq_len']
    if 'label_mask' in feats:
        ll = partial_ll_torch(logits, feats['label_mask'], lens, trans)
    else:
        ll = crf_torch.crf_log_likelihood(logits, feats['label_ids'], lens, trans)
    t_logits, t_trans = (p.detach().cpu().double() for p in pot)
    kl = distill_ref(t_logits, t_trans, logits, trans, lens, tau).kl
    return (1 - alpha) * (-ll).mean() + alpha * tau * tau * kl.mean()


def _open_rows(feats, K, rows):
    lab = feats['label_ids'].long().clamp(0, K - 1)
    mask = torch.ones_like(lab) << lab
    mask[rows] = (1 << K) - 1
    return mask.to(torch.int32)


@pytest.mark.parametrize("teacher", ["bilstm_crf_softlexicon", "lattice_lstm_crf"])
@pytest.mark.parametrize("masked", [False, True])
def test_bilstm_crf_student_gradients_match_oracle_autograd(masked, teacher):
    from oracle import nn as onn
    alpha, tau = 0.5, 2.0
    est, feats, emb = _bilstm_pair(alpha, tau, teacher)
    if masked:
        feats['label_mask'] = _open_rows(feats, 10, [0, 3])
    loss, grads, teacher = _train_grads(est, feats)
    wd = {k: v.double().clone().requires_grad_(True) for k, v in est.store.state_dict().items()}
    x = torch.from_numpy(emb).double()[feats['token_ids'].long()]
    lstm = onn.bilstm(x, wd, feats['seq_len'], est.params['rnn_activation'], 1.0, torch.float64)
    logits = lstm @ wd['logits/kernel'] + wd['logits/bias']
    ref = _ref_loss(logits, wd['crf_layer/transitions'], feats, teacher[:2], alpha, tau)
    ref.backward()
    assert abs(loss - ref.item()) < 2e-3 * max(1.0, abs(ref.item())), (loss, ref.item())
    for name, v in wd.items():
        scale = max(v.grad.abs().max().item(), 1e-6)
        assert (grads[name] - v.grad).abs().max().item() < 2e-2 * scale, name
    assert set(grads) == set(est.store.state_dict())          # no teacher variable in the student's store


def test_fully_open_rows_train_on_the_distillation_term_alone():
    est, feats, _ = _bilstm_pair(alpha=0.5, tau=1.0)
    B = feats['label_ids'].shape[0]
    feats['label_mask'] = _open_rows(feats, 10, list(range(B)))
    dev = est.to_device(feats)
    lens = dev['seq_len']
    lg, tr = est.teacher_potentials(dev)
    from chinesener_b200.tools import layer
    cap = []
    layer.CRF_CAPTURE = cap
    try:
        est.forward_device({k: v for k, v in dev.items() if k != 'label_mask'}, False)
    finally:
        layer.CRF_CAPTURE = None
    s_logits, s_trans = cap[0]
    gold = ops.crf_partial_loglik_fwd(s_logits.contiguous(), dev['label_mask'], lens, s_trans)[0]
    assert (gold == 0).all()                                  # a fully open row adds exactly 0 to the gold loss
    logz, alpha = ops.crf_distill_fwd(lg, tr, s_logits.contiguous(), s_trans, lens, 1.0)
    kl = ops.crf_distill_bwd(lg, tr, s_logits.contiguous(), s_trans, lens, alpha, logz, 1.0)[0]
    loss, _, _ = _train_grads(est, feats)
    assert abs(loss - 0.5 * float(kl.mean())) <= 1e-5 * max(1.0, abs(loss))


def test_student_learns_the_teacher():
    """alpha = 1 against a fixed, randomly initialised bilstm_crf teacher (another seed), on synthetic batches."""
    from test_training_gpu import _setup
    teacher, _, emb = _setup(B=32, L=32, V=2000, seed=3)
    torch.manual_seed(123)
    np.random.seed(123)
    teacher.evaluate(synthetic.msra_batch(32, 32, vocab=2000, seed=99))
    teacher.store.vars['logits/kernel'].mul_(3.0)             # a teacher with some confidence to copy
    teacher.store.touch()
    params = dict(synthetic.data_params(32), embedding=emb, embedding_dropout=0.0, keep_prob_list=[1.0],
                  distill_alpha=1.0, distill_temperature=1.0, lr=0.01)
    student = engine.Estimator("bilstm_crf", params, teacher=teacher)
    held = [synthetic.msra_batch(32, 32, vocab=2000, seed=1000 + i) for i in range(2)]
    torch.manual_seed(7)
    student.evaluate(held[0])

    def measure():
        kls, agree = [], 0
        for f in held:
            dev = student.to_device(f)
            t_lg, t_tr = student.teacher_potentials(dev)
            cap = []
            from chinesener_b200.tools import layer
            layer.CRF_CAPTURE = cap
            try:
                student.forward_device(dev, False)
            finally:
                layer.CRF_CAPTURE = None
            s_lg, s_tr = cap[0]
            logz, al = ops.crf_distill_fwd(t_lg, t_tr, s_lg.contiguous(), s_tr, dev['seq_len'], 1.0)
            kls.append(float(ops.crf_distill_bwd(t_lg, t_tr, s_lg.contiguous(), s_tr, dev['seq_len'], al, logz)[0].mean()))
            tt = ops.crf_viterbi(t_lg, dev['seq_len'], t_tr)
            st = ops.crf_viterbi(s_lg.contiguous(), dev['seq_len'], s_tr)
            real = torch.arange(32, device='cuda')[None, :] < dev['seq_len'][:, None]
            agree += int(((tt == st) & real).sum())
        return float(np.mean(kls)), agree

    kl0, agree0 = measure()
    for step in range(300):
        student.train_step(synthetic.msra_batch(32, 32, vocab=2000, seed=step))
    kl1, agree1 = measure()
    print(f"held-out mean KL {kl0:.4g} -> {kl1:.4g}; Viterbi agreement {agree0} -> {agree1} positions")
    assert kl1 < 0.1 * kl0
    assert agree1 > agree0


def test_main_driver_with_a_teacher(tmp_path):
    """main.py trains a bert_bilstm_crf teacher, then a bert_crf student against its checkpoint: the student trains,
    evaluates and writes its pickle, and its checkpoint holds none of the teacher's variables."""
    import os
    from chinesener_b200 import checkpoint
    from chinesener_b200 import main as driver
    from test_main_driver_gpu import _setup
    root, pre = _setup(tmp_path)
    data_dir = os.path.join(root, 'msra')
    ck = str(tmp_path / 'ckpt')
    common = ['--data', 'msra', '--data_dir', data_dir, '--checkpoint_root', ck, '--pretrain_dir', pre,
              '--epoch_size', '1', '--batch_size', '4']
    with pytest.warns(UserWarning):                    # no BERT checkpoint in pretrain_dir: random init
        driver.main(['--model_name', 'bert_bilstm_crf'] + common)
    teacher_dir = os.path.join(ck, 'ner_msra_bert_bilstm_crf')
    with pytest.warns(UserWarning):
        s = driver.main(['--model_name', 'bert_crf', '--teacher_model', 'bert_bilstm_crf', '--teacher_dir', teacher_dir,
                         '--distill_alpha', '0.7', '--distill_temperature', '2'] + common)
    assert s['teacher'] == 'bert_bilstm_crf' and s['distill_alpha'] == 0.7 and s['distill_temperature'] == 2.0
    assert s['history']['final_step'] > 0 and np.isfinite(s['history']['evals'][-1]['loss'])
    assert os.path.exists(os.path.join(data_dir, 'bert_crf_predict.pkl'))
    student = np.load(checkpoint.latest_checkpoint(os.path.join(ck, 'ner_msra_bert_crf')))
    saved = {k for k in student.files if k != 'global_step' and not k.endswith((checkpoint.SLOT_M, checkpoint.SLOT_V))}
    # exactly the variables of a bert_crf student's store, nothing of the teacher's
    from chinesener_b200 import bert
    fresh = engine.Estimator('bert_crf', dict(synthetic.data_params(16), pretrain_dir=pre))
    with pytest.warns(UserWarning):
        fresh.evaluate(synthetic.msra_batch(2, 16, vocab=bert.load_bert_config(pre)['vocab_size'], seed=0))
    assert saved == set(fresh.store.state_dict())
    with pytest.raises(ValueError, match='teacher_dir'):
        driver.main(['--model_name', 'bert_crf', '--teacher_model', 'bert_bilstm_crf', '--teacher_dir',
                     str(tmp_path / 'empty')] + common)


@pytest.mark.parametrize("masked", [False, True])
def test_bert_crf_student_gradients_match_oracle_autograd(tmp_path, masked):
    """A 1-layer bert_crf student against a 2-layer bert_bilstm_crf teacher (temporary bert_config.json files)."""
    import json
    from oracle import nn as onn
    from test_bert_training_gpu import CFG
    alpha, tau = 0.6, 1.5
    dirs = {}
    for layers in (1, 2):
        dirs[layers] = tmp_path / ("bert%d" % layers)
        dirs[layers].mkdir()
        (dirs[layers] / "bert_config.json").write_text(json.dumps(dict(CFG, num_hidden_layers=layers,
                                                                       hidden_dropout_prob=0.0,
                                                                       attention_probs_dropout_prob=0.0)))
    feats = synthetic.msra_batch(4, 32, vocab=CFG['vocab_size'], seed=21)
    base = dict(synthetic.data_params(32), embedding_dropout=0.0, keep_prob_list=[1.0])
    teacher = engine.Estimator("bert_bilstm_crf", dict(base, pretrain_dir=str(dirs[2])))
    teacher.evaluate(feats)
    est = engine.Estimator("bert_crf", dict(base, pretrain_dir=str(dirs[1]), distill_alpha=alpha,
                                            distill_temperature=tau), teacher=teacher)
    if masked:
        feats['label_mask'] = _open_rows(feats, 10, [1])
    est.evaluate({k: v for k, v in feats.items() if k != 'label_mask'})
    est.store.vars["logits/kernel"].mul_(4.0)
    est.store.touch()
    loss, grads, pot = _train_grads(est, feats)
    wd = {k: v.double().clone().requires_grad_(True) for k, v in est.store.state_dict().items()}
    seq = onn.bert_encoder(wd, feats['token_ids'], feats['mask'], feats['segment_ids'], num_layers=1, num_heads=12,
                           dtype=torch.float64)
    logits = seq @ wd['logits/kernel'] + wd['logits/bias']
    ref = _ref_loss(logits, wd['crf_layer/transitions'], feats, pot[:2], alpha, tau)
    ref.backward()
    assert abs(loss - ref.item()) < 2e-2 * max(1.0, abs(ref.item())), (loss, ref.item())
    refg = {k: v.grad for k, v in wd.items() if v.grad is not None and "pooler" not in k}
    top = max(g.abs().max().item() for g in refg.values())
    for name, g_ref in refg.items():            # the BERT TRAIN bar of DESIGN.md §4
        scale = max(g_ref.abs().max().item(), 1e-3 * top)
        assert (grads[name] - g_ref).abs().max().item() < 8e-2 * scale, name
    assert not any("bilstm" in k for k in grads)


def test_document_length_rows_err_as_the_ordinary_loss_does():
    """At L = 4095 the d_s_trans bound is C_T_DOC U rather than C_T U.  The ordinary ner_crf_loglik_bwd, run on the
    teacher's and on the student's potentials of the same rows, errs by the same order: the excess is the float32
    log-domain rounding every CRF loss kernel carries at that length, not something of the distillation kernel."""
    from _crf_grad_oracle import crf_grad_ref
    xt, trt, xs, trs, lens, d_kl = _case(4, 4095, 10, seed=4 + 4095 + 10)
    worst = 0.0
    for x, tr in ((xt, trt), (xs, trs)):
        x, tr, n, g = x.cuda(), tr.cuda(), lens.cuda(), (d_kl * SCALE).cuda()
        tags = torch.randint(0, 10, x.shape[:2], generator=torch.Generator().manual_seed(0), dtype=torch.int32).cuda()
        _, logz, alpha = ops.crf_loglik_fwd(x, tags, n, tr, want_alpha=True)
        d_logits, d_trans = ops.crf_loglik_bwd(x, tags, n, tr, alpha, logz, g, 1.0)
        ref = crf_grad_ref(x.double(), tags, n, tr, g)
        L = x.shape[1]
        valid = (torch.arange(L, device="cuda")[None, :] < ref.lens[:, None])[:, :, None]
        amax = torch.where(valid, ref.alpha.abs(), torch.zeros_like(ref.alpha)).reshape(4, -1).max(dim=1).values
        r = EPS32 * (1 + ref.logz.abs() + amax)
        unit = crf_grad_ref(x.double(), tags, n, tr, g.double().abs() * r).trans_scale
        err = (d_trans.double() - ref.d_trans).abs()
        e_u = _worst_ratio((err - TOL["lanes"][2] * ref.trans_scale).clamp(min=0), unit)
        print(f"ner_crf_loglik_bwd at L = 4095: d_trans {e_u:.3g} U beyond tol_s S")
        worst = max(worst, e_u)
    assert C_T < worst <= C_T_DOC
