"""GPU parity: CUDA CRF kernels (through the C-ABI) vs the numpy oracle.

Viterbi tag indices must be BIT-EXACT (integer output); log-likelihood within 1e-4 relative
(+1e-4 absolute) of the float64 oracle (SURVEY.md §7 step 3).
"""
import numpy as np
import pytest
import torch

from chinesener_b200 import ops
from chinesener_b200._lib import VIT_PLANS, check, lib, ptr, stream
from oracle import crf

from _crf_grad_oracle import crf_grad_ref

pytestmark = pytest.mark.gpu

# |alpha - ref| <= ALPHA_RTOL |ref| + ALPHA_ATOL at every valid step, and the same for log Z
ALPHA_RTOL, ALPHA_ATOL = 5e-6, 5e-6


def _case(B, L, K, seed, ragged=True, scale=2.0):
    rng = np.random.default_rng(seed)
    x = (rng.normal(size=(B, L, K)) * scale).astype(np.float32)
    tr = (rng.normal(size=(K, K))).astype(np.float32)
    lens = rng.integers(1, L + 1, size=B).astype(np.int32) if ragged else np.full(B, L, np.int32)
    tags = rng.integers(0, K, size=(B, L)).astype(np.int32)
    return x, tr, lens, tags


def _plan(B, L, K, aligned=True):
    """Name of the kernel ner_crf_viterbi runs for this shape on this device."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return VIT_PLANS[lib().ner_crf_viterbi_plan(B, L, K, int(aligned), sms)]


@pytest.mark.parametrize("B,L,K", [(64, 128, 10), (8, 64, 10), (37, 150, 7), (5, 1, 4), (3, 17, 1), (130, 33, 13),
                                   (9, 50, 20), (4, 40, 32), (300, 21, 3), (70, 150, 10), (33, 9, 16), (6, 256, 10)])
def test_viterbi_bit_exact(B, L, K):
    x, tr, lens, _ = _case(B, L, K, seed=B * 1000 + L * 10 + K)
    lens[0] = L
    if B > 2:
        lens[1] = 1
        lens[2] = 0                                      # TF quirk: decodes like len 1
    ref_tags, ref_best = crf.crf_decode(x, tr, lens, dtype=np.float32)
    tags, best = ops.crf_viterbi(torch.from_numpy(x).cuda(), torch.from_numpy(lens).cuda(),
                                 torch.from_numpy(tr).cuda(), return_score=True)
    assert tags.dtype == torch.int32
    np.testing.assert_array_equal(tags.cpu().numpy(), ref_tags)
    np.testing.assert_array_equal(best.cpu().numpy(), ref_best.astype(np.float32))


def test_viterbi_ties_resolve_to_lowest_index():
    B, L, K = 40, 30, 10
    rng = np.random.default_rng(7)
    x = rng.integers(-1, 2, size=(B, L, K)).astype(np.float32)     # many exact ties
    tr = rng.integers(-1, 2, size=(K, K)).astype(np.float32)
    lens = rng.integers(1, L + 1, size=B).astype(np.int32)
    ref_tags, _ = crf.crf_decode(x, tr, lens, dtype=np.float32)
    tags = ops.crf_viterbi(torch.from_numpy(x).cuda(), torch.from_numpy(lens).cuda(), torch.from_numpy(tr).cuda())
    np.testing.assert_array_equal(tags.cpu().numpy(), ref_tags)


def test_viterbi_mid_batch_uses_all_on_chip_kernel_with_32_thread_ctas():
    B, L, K = 5000, 40, 10                              # above the lane-per-tag threshold, below the big-batch one
    assert _plan(B, L, K) == "onchip_32"
    x, tr, lens, _ = _case(B, L, K, seed=17)
    ref_tags, _ = crf.crf_decode(x, tr, lens, dtype=np.float32)
    tags = ops.crf_viterbi(torch.from_numpy(x).cuda(), torch.from_numpy(lens).cuda(), torch.from_numpy(tr).cuda())
    np.testing.assert_array_equal(tags.cpu().numpy(), ref_tags)


def test_viterbi_large_batch_uses_tma_kernel():
    B, L, K = 148 * 64 + 77, 128, 10                    # > big-batch threshold, ragged tail CTA
    assert _plan(B, L, K) == "tma"
    x, tr, lens, _ = _case(B, L, K, seed=11)
    ref_tags, _ = crf.crf_decode(x, tr, lens, dtype=np.float32)
    tags = ops.crf_viterbi(torch.from_numpy(x).cuda(), torch.from_numpy(lens).cuda(), torch.from_numpy(tr).cuda())
    np.testing.assert_array_equal(tags.cpu().numpy(), ref_tags)


@pytest.mark.parametrize("B,L,K", [(64, 128, 10), (8, 64, 10), (37, 150, 7), (5, 1, 4), (3, 17, 1), (130, 33, 13),
                                   (9, 50, 20), (4, 40, 32), (19000, 24, 10), (6, 256, 10), (33, 10, 16), (5000, 16, 10)])
@pytest.mark.parametrize("exact", [False, True])
def test_loglik_forward(B, L, K, exact):
    x, tr, lens, tags = _case(B, L, K, seed=B + L + K)
    if B > 2:
        lens[1] = 1
        lens[2] = 0
    ref = crf.crf_log_likelihood(x, tags, lens, tr, dtype=np.float64)
    ref_logz = crf.crf_log_norm(x.astype(np.float64), lens, tr.astype(np.float64))
    ll, logz, _ = ops.crf_loglik_fwd(torch.from_numpy(x).cuda(), torch.from_numpy(tags).cuda(),
                                     torch.from_numpy(lens).cuda(), torch.from_numpy(tr).cuda(), exact=exact)
    np.testing.assert_allclose(ll.cpu().numpy(), ref, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(logz.cpu().numpy(), ref_logz, rtol=1e-4, atol=1e-4)


def test_loglik_wide_transitions_fall_back_to_exact_path():
    B, L, K = 16, 40, 10
    x, tr, lens, tags = _case(B, L, K, seed=3)
    tr[2, 5] = -1e4                                      # hard "forbidden" transition
    tr[7, 1] = -np.inf
    tags[:, :] = 0
    ref = crf.crf_log_likelihood(x, tags, lens, tr, dtype=np.float64)
    ll, _, _ = ops.crf_loglik_fwd(torch.from_numpy(x).cuda(), torch.from_numpy(tags).cuda(),
                                  torch.from_numpy(lens).cuda(), torch.from_numpy(tr).cuda())
    np.testing.assert_allclose(ll.cpu().numpy(), ref, rtol=1e-4, atol=1e-4)


def test_loglik_alpha_workspace():
    B, L, K = 20, 31, 10
    x, tr, lens, tags = _case(B, L, K, seed=9)
    _, alphas = crf.crf_log_norm(x.astype(np.float64), lens, tr.astype(np.float64), return_alphas=True)
    _, _, a = ops.crf_loglik_fwd(torch.from_numpy(x).cuda(), torch.from_numpy(tags).cuda(),
                                 torch.from_numpy(lens).cuda(), torch.from_numpy(tr).cuda(), want_alpha=True)
    a = a.cpu().numpy()
    for b in range(B):
        n = int(lens[b])
        np.testing.assert_allclose(a[b, :n], alphas[b, :n], rtol=1e-4, atol=1e-4)


# (B, L, K, logits 16-byte aligned, kernel the plan must name).  A big batch has more than 64 sequences per SM: 8448 on
# the 132 SMs of an H100 SXM.
_PLANNED = [
    # logits by TMA: K <= 16, L*K % 4 == 0, aligned
    (148 * 64 + 77, 128, 10, True, "tma"), (9500, 50, 16, True, "tma"), (9601, 21, 12, True, "tma"),
    (9500, 12, 5, True, "tma"), (9533, 16, 9, True, "tma"), (9480, 20, 8, True, "tma"), (9479, 8, 11, True, "tma"),
    (9600, 256, 10, True, "tma"), (9500, 6, 2, True, "tma"), (9490, 1200, 10, True, "tma"),
    # parked nibbles: L*K % 4 != 0, logits off a 16-byte boundary, or L past the TMA kernel's shared memory
    (9600, 37, 7, True, "parked"), (9490, 9, 3, True, "parked"), (19000, 150, 7, True, "parked"),
    (9500, 127, 10, True, "parked"), (9500, 33, 13, True, "parked"), (9511, 21, 15, True, "parked"),
    (148 * 64 + 77, 128, 10, False, "parked"), (9500, 50, 16, False, "parked"), (9480, 20, 8, False, "parked"),
    (9601, 21, 12, False, "parked"), (9479, 8, 11, False, "parked"), (9490, 1500, 10, True, "parked"),
    # all on chip, 128-thread CTAs: big batches of more than 16 tags
    (9500, 20, 20, True, "onchip_128"), (9600, 30, 17, True, "onchip_128"), (9490, 24, 18, True, "onchip_128"),
    (9479, 8, 24, True, "onchip_128"), (9500, 20, 20, False, "onchip_128"),
    # all on chip, 32-thread CTAs: mid batches, and big ones past the 128-thread slab (every L at K >= 28)
    (9490, 24, 32, True, "onchip_32"),
    (5000, 40, 10, True, "onchip_32"), (6000, 33, 13, True, "onchip_32"), (4500, 30, 20, True, "onchip_32"),
    (7000, 37, 7, False, "onchip_32"), (9500, 120, 20, True, "onchip_32"), (9490, 100, 32, True, "onchip_32"),
    # lane per tag: up to 4096 sequences, and any B when L is past every thread-per-sequence limit
    (4096, 16, 10, True, "small"), (4200, 1500, 20, True, "small_any_b"), (4200, 800, 10, True, "small_any_b"),
]


@pytest.mark.parametrize("B,L,K,aligned,plan", _PLANNED)
def test_viterbi_large_batch_kernels_bit_exact(B, L, K, aligned, plan):
    """Every kernel the plan can name must reproduce the oracle's tags and scores, ragged lengths and a partial tail CTA
    included, on shapes that reach it by themselves."""
    assert _plan(B, L, K, aligned) == plan
    x, tr, lens, _ = _case(B, L, K, seed=100 * len(plan) + K)
    lens[0], lens[1], lens[2] = L, 1, 0
    x[5] = np.round(x[5])                                # a row with many exact ties
    ref_tags, ref_best = crf.crf_decode(x, tr, lens, dtype=np.float32)
    if aligned:
        xd = torch.from_numpy(x).cuda()
    else:                                                # the same logits 4 bytes past a 16-byte boundary
        flat = torch.empty(x.size + 1, dtype=torch.float32, device="cuda")
        xd = flat[1:].view(B, L, K)
        xd.copy_(torch.from_numpy(x))
    assert (xd.data_ptr() % 16 == 0) == aligned
    tags, best = ops.crf_viterbi(xd, torch.from_numpy(lens).cuda(), torch.from_numpy(tr).cuda(), return_score=True)
    np.testing.assert_array_equal(tags.cpu().numpy(), ref_tags)
    np.testing.assert_array_equal(best.cpu().numpy(), ref_best.astype(np.float32))


def fwd_route(B, forced=False):
    """The kernel ner_crf_loglik_fwd runs for B sequences: the lane-per-tag kernel of crf_small.cu up to
    NER_CRF_SMALL_B unless flags bit 1 forces the throughput kernel; that one runs 4-step chunks in 64-thread CTAs
    above 128 sequences per SM and 8-step chunks in 32-thread CTAs below (launch_fwd, crf_loglik.cu:344)."""
    if B <= 4096 and not forced:
        return "lanes"
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return "t4_nt64" if B > 128 * sms else "t8_nt32"


def _loglik_fwd_flags(xd, td, ld, trd, flags):
    """ner_crf_loglik_fwd with raw flags (bit 0: exact path, bit 1: throughput kernel at any B)."""
    B, L, K = xd.shape
    ll = torch.empty(B, dtype=torch.float32, device="cuda")
    logz = torch.empty(B, dtype=torch.float32, device="cuda")
    alpha = torch.full((B, L, K), float("nan"), dtype=torch.float32, device="cuda")
    check(lib().ner_crf_loglik_fwd(ptr(xd), ptr(td), ptr(ld), ptr(trd), ptr(ll), ptr(logz), ptr(alpha), B, L, K, flags,
                                   stream()))
    return ll, logz, alpha


# (B: "big" above 128 sequences per SM, "mid" between NER_CRF_SMALL_B and that, or a small B forced onto the throughput
# kernel; L, K, mode, logits 16-byte aligned).  mode "wide" spans the transitions over >= 30 nats, "inf" forbids an
# edge, "flag" asks for the exact path through flags bit 0.
_FWD_CASES = [
    ("big", 40, 10, "fast", True), ("big", 37, 7, "inf", True), ("big", 33, 13, "wide", False),
    ("big", 24, 32, "fast", True), ("big", 30, 13, "fast", False), ("big", 9, 4, "flag", True),
    ("mid", 40, 10, "fast", True), ("mid", 9, 11, "wide", True), ("mid", 37, 20, "inf", False),
    ("mid", 17, 4, "fast", True), ("mid", 33, 7, "fast", False), ("mid", 512, 10, "fast", True),
    (37, 31, 10, "fast", True), (5, 1, 4, "flag", True), (70, 45, 13, "wide", False), (3, 9, 1, "fast", True),
    (33, 16, 32, "inf", True), (40, 21, 7, "fast", False), (64, 128, 10, "fast", True),
]


@pytest.mark.parametrize("Bs,L,K,mode,aligned", _FWD_CASES)
def test_loglik_alpha_workspace_throughput_kernels(Bs, L, K, mode, aligned):
    """alpha at every valid step and log Z of the throughput forward (the alpha the backward consumes) against float64,
    on both chunkings, fast and exact, vector and scalar staging."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = {"big": 128 * sms + 301, "mid": 5003}.get(Bs, Bs)
    forced = not isinstance(Bs, str)
    assert fwd_route(B, forced) == ("t4_nt64" if Bs == "big" else "t8_nt32")
    gen = torch.Generator().manual_seed(B + L + K)
    x = torch.randn(B, L, K, generator=gen) * 2
    tr = torch.randn(K, K, generator=gen)
    lens = torch.randint(0, L + 1, (B,), generator=gen, dtype=torch.int32)
    lens[0] = L
    if B > 2:
        lens[1], lens[2] = 1, 0
    tags = torch.randint(0, K, (B, L), generator=gen, dtype=torch.int32)
    if mode == "wide":
        tr[0, 1] = tr.max() - 35.0
    elif mode == "inf":
        tr[0, 1] = -float("inf")
    if aligned:
        xd = x.cuda()
    else:                                                # the same logits 4 bytes past a 16-byte boundary
        flat = torch.empty(x.numel() + 1, dtype=torch.float32, device="cuda")
        xd = flat[1:].view(B, L, K)
        xd.copy_(x)
    assert (xd.data_ptr() % 16 == 0) == aligned
    td, ld, trd = tags.cuda(), lens.cuda(), tr.cuda()
    flags = 2 * forced + (mode == "flag")
    _, logz, alpha = _loglik_fwd_flags(xd, td, ld, trd, flags)
    ref = crf_grad_ref(xd, td, ld, trd)
    valid = (torch.arange(L, device="cuda")[None, :] < ld[:, None].long())[:, :, None].expand(B, L, K)
    got, want = alpha.double()[valid], ref.alpha[valid]
    assert torch.isfinite(got).all()
    assert ((got - want).abs() <= ALPHA_RTOL * want.abs() + ALPHA_ATOL).all(), \
        f"alpha error {((got - want).abs() - ALPHA_RTOL * want.abs()).max().item():.3e}"
    assert ((logz.double() - ref.logz).abs() <= ALPHA_RTOL * ref.logz.abs() + ALPHA_ATOL).all()


@pytest.mark.parametrize("B", [19000, 5000])             # 64-thread CTAs with 4-step chunks / 32-thread CTAs
@pytest.mark.parametrize("K", [10, 7, 13])
def test_loglik_large_batch_configurations(B, K):
    L = 40
    x, tr, lens, tags = _case(B, L, K, seed=B % 7 + K)
    ref = crf.crf_log_likelihood(x, tags, lens, tr, dtype=np.float64)
    ll, _, _ = ops.crf_loglik_fwd(torch.from_numpy(x).cuda(), torch.from_numpy(tags).cuda(),
                                  torch.from_numpy(lens).cuda(), torch.from_numpy(tr).cuda())
    np.testing.assert_allclose(ll.cpu().numpy(), ref, rtol=1e-4, atol=1e-4)
