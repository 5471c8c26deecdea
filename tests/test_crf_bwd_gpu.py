"""GPU: the CRF log-likelihood gradient kernels vs forward-backward in float64 (tests/_crf_grad_oracle.py).

ner_crf_loglik_bwd picks one of three kernels from B and K; `bwd_route` (tests/_crf_grad_oracle.py) restates that rule
and every case asserts which kernel its shape reaches.  Every case weights its rows with a per-sequence upstream gradient d_ll (as crf_layer and
masked_task_loss pass it in TRAIN) and a scale != 1, and is judged with tolerances proportional to each row's
|g_b| = |d_ll_b * scale| (see row_unit), not to 1/B.
"""
import numpy as np
import pytest
import torch

from chinesener_b200 import ops
from oracle import crf

from _crf_grad_oracle import TOL, assert_grads_close, bwd_route, crf_grad_ref

pytestmark = pytest.mark.gpu

SCALE = 0.75
NF = 2                  # staged float tensors of ner_crf_loglik_bwd: logits, alpha (64-thread CTAs fit up to K = 26)


def route_batch(B):
    """An explicit B, or "mid" / "big": a batch on either side of 128 sequences per SM with a partial tail CTA."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {"mid": 5003, "big": 128 * sms + 301}.get(B, B)


def make_case(B, L, K, seed, mode="fast", confident=False):
    """Random logits / transitions / ragged lengths with rows of length L, 1 and 0, tags, and d_ll in [-2, 2] with
    exact zeros on every 7th row, whose tags lie past K (the rows of the other task under masked_task_loss).
    mode "wide" spans the transitions over >= 30 nats, "inf" forbids one edge with -inf: both take the exact path.
    With B >= 192, rows [64, 128) all have length 0 and rows [128, 192) stop at least 16 steps short of L."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, K, generator=gen) * 2
    tr = torch.randn(K, K, generator=gen)
    lens = torch.randint(0, L + 1, (B,), generator=gen, dtype=torch.int32)
    tags = torch.randint(0, K, (B, L), generator=gen, dtype=torch.int32)
    lens[0] = L
    if B > 2:
        lens[1], lens[2] = 1, 0
    if B >= 192:
        lens[64:128] = 0
        lens[128:192] = torch.randint(1, max(L - 15, 2), (64,), generator=gen, dtype=torch.int32).clamp(max=L)
    if mode != "fast":
        assert K > 1
        if mode == "wide":
            tr[0, 1] = tr.max() - 35.0
        else:
            tr[0, 1] = -float("inf")
        tags[tags == 0] = 1                              # keep the gold path off the forbidden edge
    if confident:                                        # marginals near 0 or 1
        x = x * 8
        x.scatter_add_(2, tags.long()[:, :, None], torch.full((B, L, 1), 16.0))
    d_ll = torch.empty(B).uniform_(-2, 2, generator=gen)
    d_ll[3::7] = 0
    tags[3::7] = K + 2 + torch.arange(tags[3::7].numel(), dtype=torch.int32).view(-1, L) % 5
    return x, tr, lens, tags, d_ll


def _device_logits(x, aligned):
    if aligned:
        return x.cuda()
    flat = torch.empty(x.numel() + 1, dtype=torch.float32, device="cuda")   # 4 bytes past a 16-byte boundary
    xd = flat[1:].view(x.shape)
    xd.copy_(x)
    assert xd.data_ptr() % 16 == 4
    return xd


def run_backward(x, tr, lens, tags, d_ll, aligned=True):
    """Forward with the alpha workspace, then the backward into a d_logits block the allocator last held NaNs in, so
    any element the kernel fails to write shows up."""
    xd = _device_logits(x, aligned)
    td, ld, trd, gd = tags.cuda(), lens.cuda(), tr.cuda(), d_ll.cuda()
    _, logz, alpha = ops.crf_loglik_fwd(xd, td, ld, trd, want_alpha=True)
    poison = torch.full_like(xd, float("nan"))
    poison_ptr = poison.data_ptr()
    del poison
    d_logits, d_trans = ops.crf_loglik_bwd(xd, td, ld, trd, alpha, logz, gd, SCALE)
    assert d_logits.data_ptr() == poison_ptr
    return d_logits, d_trans


def check_case(route, x, tr, lens, tags, d_ll, aligned=True):
    B, _, K = x.shape
    assert bwd_route(B, K, NF) == route
    d_logits, d_trans = run_backward(x, tr, lens, tags, d_ll, aligned)
    ref = crf_grad_ref(x.cuda(), tags.cuda(), lens.cuda(), tr.cuda(), d_ll.cuda().double() * SCALE)
    masked = (d_ll == 0).cuda()
    assert (d_logits[masked] == 0).all()
    return assert_grads_close(d_logits, d_trans, ref, *TOL[route])


@pytest.mark.parametrize("B,L,K", [(16, 24, 10), (64, 128, 10), (9, 31, 7), (5, 1, 4), (40, 17, 13), (3, 9, 1),
                                   (19000, 8, 10), (5000, 12, 10), (130, 40, 20), (4, 50, 32)])
@pytest.mark.parametrize("wide", [False, True])
def test_crf_backward(B, L, K, wide):
    rng = np.random.default_rng(B + L + K)
    x = rng.normal(size=(B, L, K)).astype(np.float32) * 2
    tr = rng.normal(size=(K, K)).astype(np.float32)
    if wide and K > 2:
        tr[0, 1] = -1e4                                  # forces the exact path
    lens = rng.integers(1, L + 1, size=B).astype(np.int32)
    if B > 2:
        lens[1] = 1
        lens[2] = 0
    tags = rng.integers(0, K, size=(B, L)).astype(np.int32)
    if wide and K > 2:                                   # keep the gold path off the forbidden edge
        tags[tags == 0] = 2
    xd, td, ld, trd = (torch.from_numpy(a).cuda() for a in (x, tags, lens, tr))
    ll, logz, alpha = ops.crf_loglik_fwd(xd, td, ld, trd, want_alpha=True)
    scale = -1.0 / B
    d_logits, d_trans = ops.crf_loglik_bwd(xd, td, ld, trd, alpha, logz, None, scale)
    if B <= 200:
        dx_ref, dtr_ref = crf.crf_marginal_grads(x, tags, lens, tr)
        np.testing.assert_allclose(d_logits.cpu().numpy(), scale * dx_ref, rtol=2e-3, atol=2e-5)
        np.testing.assert_allclose(d_trans.cpu().numpy(), scale * dtr_ref, rtol=2e-3, atol=2e-4)
    ref = crf_grad_ref(xd, td, ld, trd, torch.full((B,), scale, dtype=torch.float64, device="cuda"))
    assert_grads_close(d_logits, d_trans, ref, *TOL[bwd_route(B, K, NF)])


# (route the shape must reach, B, L, K, mode, logits 16-byte aligned, confident)
_CASES = [
    # lane per tag: one K in each lane-group width (8 / 16 / 32 lanes), B up to the threshold itself
    ("lanes", 37, 24, 5, "fast", True, False), ("lanes", 45, 31, 10, "inf", True, False),
    ("lanes", 19, 512, 10, "fast", True, False), ("lanes", 33, 9, 13, "wide", False, False),
    ("lanes", 4096, 40, 20, "fast", True, False), ("lanes", 11, 17, 32, "inf", True, False),
    ("lanes", 7, 1, 4, "fast", True, False), ("lanes", 9, 33, 1, "fast", True, False),
    ("lanes", 250, 24, 10, "fast", True, True),
    # 32-thread CTAs: K reaches ACC_REGS on (<= 10) and off, UNROLL on (<= 12) and off, step groups G = 4 / 2 / 1
    ("nt32", "mid", 24, 10, "fast", True, False), ("nt32", "mid", 33, 1, "fast", True, False),
    ("nt32", "mid", 9, 3, "wide", True, False), ("nt32", "mid", 16, 4, "fast", True, False),
    ("nt32", "mid", 37, 7, "inf", True, False), ("nt32", "mid", 7, 11, "fast", True, False),
    ("nt32", "mid", 40, 13, "wide", False, False), ("nt32", "mid", 20, 16, "inf", True, False),
    ("nt32", "mid", 12, 20, "fast", True, False), ("nt32", "mid", 17, 32, "fast", True, False),
    ("nt32", "mid", 512, 10, "fast", True, False), ("nt32", "mid", 1, 10, "fast", True, False),
    ("nt32", "mid", 30, 13, "fast", False, False), ("nt32", "mid", 24, 10, "fast", True, True),
    # big batches past K = 26: 64-thread CTAs would need more shared memory than a CTA can have
    ("nt32", "big", 20, 32, "wide", True, False), ("nt32", "big", 13, 27, "fast", True, False),
    # 64-thread CTAs
    ("nt64", "big", 24, 10, "fast", True, False), ("nt64", "big", 9, 7, "inf", True, False),
    ("nt64", "big", 33, 13, "fast", False, False), ("nt64", "big", 20, 26, "wide", True, False),
    ("nt64", "big", 16, 4, "fast", True, False), ("nt64", "big", 1, 3, "fast", True, False),
    ("nt64", "big", 37, 11, "fast", True, False), ("nt64", "big", 12, 20, "inf", False, False),
    ("nt64", "big", 40, 16, "fast", True, False), ("nt64", "big", 16, 7, "fast", True, True),
]


@pytest.mark.parametrize("route,B,L,K,mode,aligned,confident", _CASES)
def test_crf_backward_routes(route, B, L, K, mode, aligned, confident):
    B = route_batch(B)
    x, tr, lens, tags, d_ll = make_case(B, L, K, seed=B + 31 * L + K, mode=mode, confident=confident)
    check_case(route, x, tr, lens, tags, d_ll, aligned)


def test_crf_backward_rejects_mistyped_inputs():
    B, L, K = 6, 5, 4
    x, tr, lens, tags, d_ll = make_case(B, L, K, seed=1)
    xd, td, ld, trd = x.cuda(), tags.cuda(), lens.cuda(), tr.cuda()
    _, logz, alpha = ops.crf_loglik_fwd(xd, td, ld, trd, want_alpha=True)
    ops.crf_loglik_bwd(xd, td, ld, trd, alpha, logz, d_ll.cuda(), SCALE)
    bad = [dict(d_ll=d_ll.double().cuda()), dict(d_ll=d_ll[:-1].cuda()), dict(trans=trd.double()),
           dict(trans=trd[:-1]), dict(alpha=alpha[:, :-1].contiguous()), dict(alpha=alpha.half()), dict(logz=logz[:-1]),
           dict(logz=logz.double())]
    for kw in bad:
        args = dict(logits=xd, tags=td, seq_len=ld, trans=trd, alpha=alpha, logz=logz, d_ll=d_ll.cuda())
        args.update(kw)
        with pytest.raises(AssertionError):
            ops.crf_loglik_bwd(args["logits"], args["tags"], args["seq_len"], args["trans"], args["alpha"],
                               args["logz"], args["d_ll"], SCALE)
