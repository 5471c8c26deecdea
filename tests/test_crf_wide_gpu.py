"""GPU: the wide-tag-set CRF kernels (ner_crf_wide_*) against oracle/crf.py and, for K <= 32, against the K-specialised
kernels on the same inputs.

- Viterbi: tags and best_score bit-equal to oracle.crf.crf_decode (fp32) for K in 33..128, and to ner_crf_viterbi for
  K in {1, 10, 32}, with ragged rows (seq_len 0, 1, > L), deliberate ties, an L = 4095 row and B on both sides of the
  four-rows-per-CTA threshold (8 * SMs).
- Forward: ll, logz and the alpha workspace within the tolerances of test_crf_gpu.py of float64, on the fast path and the
  exact one (flags bit0, and transitions spanning >= 30 nats or holding -inf).
- Backward: d_logits / d_trans within test_crf_bwd_gpu.py's tolerances of float64 forward-backward, with d_ll, scale and
  accumulation into d_trans.
"""
import numpy as np
import pytest
import torch

from chinesener_b200 import _lib, ops
from oracle import crf

from _crf_grad_oracle import assert_grads_close, crf_grad_ref

pytestmark = pytest.mark.gpu

WIDE_K = (33, 40, 64, 97, 108, 128)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def make(B, L, K, seed, mode="fast"):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(B, L, K)).astype(np.float32) * 2
    tr = rng.normal(size=(K, K)).astype(np.float32)
    lens = rng.integers(1, L + 1, size=B).astype(np.int32)
    lens[0] = L
    if B > 3:
        lens[1], lens[2], lens[3] = 1, 0, L + 7                      # one position, empty, past L
    tags = rng.integers(0, K, size=(B, L)).astype(np.int32)
    if mode != "fast" and K > 2:
        tr[0, 1] = tr.max() - 35.0 if mode == "wide" else -np.inf
        tags[tags == 0] = 2                                           # keep the gold path off the forbidden edge
    return x, tr, lens, tags


def _dev(*arrs):
    return [torch.from_numpy(a).cuda() for a in arrs]


def _plan(B, L, K):
    return _lib.lib().ner_crf_wide_plan(B, L, K, _sms())


# ------------------------------------------------------------------------------------------------------------ Viterbi
@pytest.mark.parametrize("K", WIDE_K)
@pytest.mark.parametrize("B,L", [(1, 7), (13, 40), ("g4", 12)])
def test_viterbi_matches_oracle(B, L, K):
    B = 8 * _sms() + 5 if B == "g4" else B
    x, tr, lens, _ = make(B, L, K, seed=B * 7 + L + K)
    x[4 % B, :, 5] = x[4 % B, :, 3]                                  # ties between two tags in one row
    tr[:, 5] = tr[:, 3]
    if B > 5:
        x[5] = np.round(x[5])                                         # ties everywhere in another
        tr = np.round(tr)
    tags, score = ops.crf_viterbi(*_dev(x, lens, tr), return_score=True, wide=True)
    ref_tags, ref_score = crf.crf_decode(x, tr, np.minimum(lens, L))
    np.testing.assert_array_equal(tags.cpu().numpy(), ref_tags)
    np.testing.assert_array_equal(score.cpu().numpy(), ref_score.astype(np.float32))
    assert _plan(B, L, K) in ((1, 3) if B >= 8 * _sms() else (0, 2))


@pytest.mark.parametrize("K", (1, 10, 32))
@pytest.mark.parametrize("B,L", [(1, 9), (37, 64), (300, 128), ("g4", 24), (5000, 20)])
def test_viterbi_matches_narrow_kernel(B, L, K):
    B = 8 * _sms() + 3 if B == "g4" else B
    x, tr, lens, _ = make(B, L, K, seed=B + L + K)
    if K > 1:
        x[0, :, K - 1] = x[0, :, 0]
        tr[:, K - 1] = tr[:, 0]
    xd, ld, trd = _dev(x, lens, tr)
    tags, score = ops.crf_viterbi(xd, ld, trd, return_score=True, wide=True)
    ref_tags, ref_score = ops.crf_viterbi(xd, ld, trd, return_score=True)
    assert torch.equal(tags, ref_tags)
    assert torch.equal(score, ref_score)


@pytest.mark.parametrize("K", (40, 128))
def test_viterbi_document_length_row(K):
    L = 4095                                                          # windows.MAX_DOCUMENT_LEN
    x, tr, lens, _ = make(3, L, K, seed=K)
    lens[:] = (L, 1, 2000)
    tags, score = ops.crf_viterbi(*_dev(x, lens, tr), return_score=True, wide=True)
    ref_tags, ref_score = crf.crf_decode(x, tr, lens)
    np.testing.assert_array_equal(tags.cpu().numpy(), ref_tags)
    np.testing.assert_array_equal(score.cpu().numpy(), ref_score.astype(np.float32))


# ------------------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize("K", WIDE_K + (1, 10, 32))
@pytest.mark.parametrize("mode", ["fast", "exact", "wide", "inf"])
@pytest.mark.parametrize("B,L", [(6, 33), ("g4", 9)])
def test_forward_matches_float64(B, L, K, mode):
    if K <= 2 and mode in ("wide", "inf"):
        pytest.skip("needs a third tag to route the gold path around the forbidden edge")
    B = 8 * _sms() + 1 if B == "g4" else B
    x, tr, lens, tags = make(B, L, K, seed=B + L + K + len(mode), mode="fast" if mode == "exact" else mode)
    ll, logz, alpha = ops.crf_loglik_fwd(*_dev(x, tags, lens, tr), want_alpha=True, exact=(mode == "exact"), wide=True)
    x64, tr64 = x.astype(np.float64), tr.astype(np.float64)
    ref = crf.crf_log_likelihood(x, tags, lens, tr, dtype=np.float64)
    ref_logz, ref_alpha = crf.crf_log_norm(x64, lens, tr64, return_alphas=True)
    np.testing.assert_allclose(ll.cpu().numpy(), ref, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(logz.cpu().numpy(), ref_logz, rtol=1e-4, atol=1e-4)
    a = alpha.cpu().numpy()
    for b in range(min(B, 40)):
        n = min(max(int(lens[b]), 1), L)
        np.testing.assert_allclose(a[b, :n], ref_alpha[b, :n], rtol=1e-4, atol=1e-4)


def test_forward_optional_outputs():
    x, tr, lens, tags = make(5, 20, 97, seed=4)
    args = _dev(x, tags, lens, tr)
    ll, logz, _ = ops.crf_loglik_fwd(*args)                            # K > 32: the wide kernel without wide=True
    ll2, logz2, _ = ops.crf_loglik_fwd(*args, want_alpha=True)
    assert torch.equal(ll, ll2) and torch.equal(logz, logz2)
    ll3 = torch.empty_like(ll)
    xd, td, ld, trd = args
    _lib.check(_lib.lib().ner_crf_wide_loglik_fwd(xd.data_ptr(), td.data_ptr(), ld.data_ptr(), trd.data_ptr(),
                                                  ll3.data_ptr(), None, None, 5, 20, 97, 0, _lib.stream()))
    assert torch.equal(ll, ll3)


# ----------------------------------------------------------------------------------------------------------- backward
@pytest.mark.parametrize("K", WIDE_K + (1, 10, 32))
@pytest.mark.parametrize("mode", ["fast", "wide"])
@pytest.mark.parametrize("B,L", [(7, 29), ("g4", 8)])
def test_backward_matches_float64(B, L, K, mode):
    if K <= 2 and mode == "wide":
        pytest.skip("needs a third tag to route the gold path around the forbidden edge")
    B = 8 * _sms() + 2 if B == "g4" else B
    x, tr, lens, tags = make(B, L, K, seed=3 * B + L + K, mode=mode)
    d_ll = np.random.default_rng(K).uniform(-2, 2, size=B).astype(np.float32)
    d_ll[2::5] = 0
    scale = 0.75
    xd, td, ld, trd, gd = _dev(x, tags, lens, tr, d_ll)
    _, logz, alpha = ops.crf_loglik_fwd(xd, td, ld, trd, want_alpha=True, wide=True)
    d_logits, d_trans = ops.crf_loglik_bwd(xd, td, ld, trd, alpha, logz, gd, scale, wide=True)
    ref = crf_grad_ref(xd, td, ld, trd, gd.double() * scale)
    assert (d_logits[torch.from_numpy(d_ll == 0).cuda()] == 0).all()
    assert_grads_close(d_logits, d_trans, ref, 0.0, 1.0, 1e-4)
    d_trans2, scratch = d_trans.clone(), torch.empty_like(d_logits)
    _lib.check(_lib.lib().ner_crf_wide_loglik_bwd(*(t.data_ptr() for t in (xd, td, ld, trd, alpha, logz, gd)), scale,
                                                  scratch.data_ptr(), d_trans2.data_ptr(), B, L, K, _lib.stream()))
    # d_trans is accumulated into; the CTAs' global adds land in any order, so the sums agree to fp32 rounding only
    torch.testing.assert_close(d_trans2, 2 * d_trans, rtol=1e-5, atol=1e-6 * max(1.0, float(d_trans.abs().max())))
    if B <= 16:                                                       # and the numpy forward-backward, row by row
        g = d_ll.astype(np.float64) * scale
        dx_ref = np.zeros(x.shape)
        dtr_ref = np.zeros(tr.shape)
        for b in range(B):
            dxb, dtb = crf.crf_marginal_grads(x[b:b + 1], tags[b:b + 1], lens[b:b + 1], tr)
            dx_ref[b] = g[b] * dxb[0]
            dtr_ref += g[b] * dtb
        np.testing.assert_allclose(d_logits.cpu().numpy(), dx_ref, rtol=2e-3, atol=2e-5)
        np.testing.assert_allclose(d_trans.cpu().numpy(), dtr_ref, rtol=2e-3, atol=2e-4)


@pytest.mark.parametrize("K", (1, 10, 32))
def test_backward_matches_narrow_kernel(K):
    B, L = 50, 40
    x, tr, lens, tags = make(B, L, K, seed=K)
    xd, td, ld, trd = _dev(x, tags, lens, tr)
    _, logz, alpha = ops.crf_loglik_fwd(xd, td, ld, trd, want_alpha=True)
    dl, dt = ops.crf_loglik_bwd(xd, td, ld, trd, alpha, logz, None, -1.0 / B)
    dl_w, dt_w = ops.crf_loglik_bwd(xd, td, ld, trd, alpha, logz, None, -1.0 / B, wide=True)
    torch.testing.assert_close(dl_w, dl, rtol=2e-3, atol=2e-5)
    torch.testing.assert_close(dt_w, dt, rtol=2e-3, atol=2e-4)


@pytest.mark.parametrize("K", (32, 108, 128))
@pytest.mark.parametrize("mode", ["fast", "wide"])
def test_long_rows_keep_fp32_accuracy(K, mode):
    """Rows of 1100 steps (document mode) against float64.  log Z stays within 1e-6 relative.  The gradients, in the
    units of tests/_crf_grad_oracle.py (u_b grows with the row's length and log Z; S is what d_trans sums), stay within
    2x of the K-specialised kernels on the same rows at K = 32.  At K = 108 and 128 they stay within 0.5 u_b and
    1e-2 S, twice the worst the K-specialised kernels measure on such rows at K = 32 (0.12 u_b, 4.7e-3 S)."""
    from _crf_grad_oracle import grad_errors
    B, L = 3, 1100
    x, tr, lens, tags = make(B, L, K, seed=K + len(mode), mode=mode)
    lens[:] = (1100, 300, 37)
    xd, td, ld, trd = _dev(x, tags, lens, tr)
    ref = crf_grad_ref(xd, td, ld, trd, torch.full((B,), -1.0 / B, dtype=torch.float64, device="cuda"))

    def errors(wide):
        _, logz, alpha = ops.crf_loglik_fwd(xd, td, ld, trd, want_alpha=True, wide=wide)
        d_logits, d_trans = ops.crf_loglik_bwd(xd, td, ld, trd, alpha, logz, None, -1.0 / B, wide=wide)
        e_dl, e_dt, _ = grad_errors(d_logits, d_trans, ref, 0.0)
        return ((logz.double() - ref.logz).abs() / ref.logz.abs()).max().item(), e_dl, e_dt

    e_lz, e_dl, e_dt = errors(True)
    print(f"K={K} {mode}: log Z {e_lz:.2e} rel, d_logits {e_dl:.3g} u_b, d_trans {e_dt:.3e} S")
    assert e_lz <= 1e-6
    if K <= 32:
        _, n_dl, n_dt = errors(False)
        print(f"   K-specialised kernels: d_logits {n_dl:.3g} u_b, d_trans {n_dt:.3e} S")
        assert e_dl <= 2 * n_dl + 0.05 and e_dt <= 2 * n_dt + 1e-4
    else:
        assert e_dl <= 0.5 and e_dt <= 1e-2
