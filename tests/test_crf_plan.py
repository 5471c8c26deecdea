"""CPU: `ner_crf_viterbi_plan`, the one place that decides which Viterbi kernel serves a call.

The plan is a pure function of (B, L, K, alignment of the logits, number of SMs).  It is checked here against the
shared-memory formulas of the kernels written out independently in Python, at every boundary where the choice flips, and
against the process environment, which must not enter into it.
"""
import itertools

import pytest

from chinesener_b200 import _lib
from test_viterbi_kernel_model import _smem_bytes as _tma_smem

SMS = 132                       # H100 SXM
SMALL_B = 4096                  # NER_CRF_SMALL_B
BIG_B = SMS * 64                # big = B > 64 * num_sms
MAX_SMEM = 227 * 1024
SMALL, TMA, PARKED, ONCHIP_128, ONCHIP_32, SMALL_ANY_B, NONE = range(7)


def _plan(B, L, K, aligned=1, sms=SMS):
    return _lib.lib().ner_crf_viterbi_plan(B, L, K, aligned, sms)


def _lanes_smem(L, K):          # crf_viterbi_lanes_kernel: [L][32] bytes + [SPW][L] ints
    spw = 4 if K <= 8 else 2 if K <= 16 else 1
    return ((L * 32 + 15) & ~15) + spw * L * 4


def _onchip_smem(L, K, NT):     # crf_viterbi_kernel<K, NT>: 8-step chunks, W words of backpointers per step
    W = (K + 7) // 8 if K <= 16 else (K + 3) // 4
    P = 4 * ((8 * K // 4) | 1)
    return 4 * (((K * K + 3) & ~3) + NT + 2 * NT * P + L * W * (NT + 1))


def _parked_smem(L, K, NT=64):  # crf_viterbi_gs_kernel<K, 64, 4, 6>: 4-step chunks, HB bytes of high nibbles per step
    HB = 0 if K <= 8 else 1 if K <= 10 else 2 if K <= 12 else 4
    stage = 2 * NT * 4 * (K | 1) * 4
    dec = NT * (((L + 3) & ~3) + 4)
    return (((2 * K * ((K + 1) // 2) + 3) & ~3) + NT) * 4 + max(stage, dec) + ((L * NT * HB + 15) & ~15)


def _expected(B, L, K, aligned, sms=SMS):
    lanes = _lanes_smem(L, K) <= MAX_SMEM
    if B <= SMALL_B and lanes:
        return SMALL
    big = B > 64 * sms
    if big and K <= 16:
        if aligned and L * K % 4 == 0 and _tma_smem(L, K) <= MAX_SMEM:
            return TMA
        if _parked_smem(L, K) <= MAX_SMEM:
            return PARKED
    if big and _onchip_smem(L, K, 128) <= MAX_SMEM:
        return ONCHIP_128
    if _onchip_smem(L, K, 32) <= MAX_SMEM:
        return ONCHIP_32
    return SMALL_ANY_B if B > SMALL_B and lanes else NONE


def _last_fit(smem, K, hi=8000):
    """Largest L whose shared memory fits; 0 when not even L = 1 does."""
    return max((L for L in range(1, hi) if smem(L, K) <= MAX_SMEM), default=0)


GRID_B = (1, 64, SMALL_B, SMALL_B + 1, BIG_B, BIG_B + 1, 262144)
GRID_L = (1, 2, 3, 4, 9, 37, 128, 256, 440, 441, 512, 1400, 1500, 1800, 3600, 4900, 5900, 6500, 8000)


def test_plan_matches_the_kernels_limits_on_a_grid():
    for B, L, K, aligned in itertools.product(GRID_B, GRID_L, range(1, 33), (0, 1)):
        assert _plan(B, L, K, aligned) == _expected(B, L, K, aligned), (B, L, K, aligned)


def test_plan_is_none_only_past_the_lane_per_tag_limit():
    for B, L, K, aligned in itertools.product(GRID_B, GRID_L, range(1, 33), (0, 1)):
        if _plan(B, L, K, aligned) == NONE:
            assert _lanes_smem(L, K) > MAX_SMEM, (B, L, K, aligned)
    assert _plan(64, 8000, 10) == NONE and _plan(9000, 8000, 10) == NONE
    for bad in ((0, 8, 10), (8, 0, 10), (8, 8, 0), (8, 8, 33)):
        assert _plan(*bad) == NONE


def test_batch_size_boundaries():
    assert (_plan(SMALL_B, 128, 10), _plan(SMALL_B + 1, 128, 10)) == (SMALL, ONCHIP_32)
    assert (_plan(BIG_B, 128, 10), _plan(BIG_B + 1, 128, 10)) == (ONCHIP_32, TMA)
    assert (_plan(BIG_B, 20, 20), _plan(BIG_B + 1, 20, 20)) == (ONCHIP_32, ONCHIP_128)
    assert _plan(66 * 64 + 1, 128, 10, 1, 66) == TMA          # "big" scales with the number of SMs


def test_tag_count_alignment_and_divisibility_boundaries():
    B = BIG_B + 1
    assert (_plan(B, 16, 16), _plan(B, 16, 17)) == (TMA, ONCHIP_128)
    assert (_plan(B, 128, 10, 1), _plan(B, 128, 10, 0)) == (TMA, PARKED)
    assert [_plan(B, L, 7) for L in (36, 37, 38, 39, 40)] == [TMA, PARKED, PARKED, PARKED, TMA]
    assert [_plan(B, L, 10) for L in (126, 127, 128)] == [TMA, PARKED, TMA]


@pytest.mark.parametrize("K", range(1, 33))
def test_shared_memory_boundaries(K):
    B = BIG_B + 1
    step = 4 if K % 2 else 2 if K % 4 else 1                  # keeps L*K % 4 == 0
    last = {"lanes": _last_fit(_lanes_smem, K), "onchip_128": _last_fit(lambda L, k: _onchip_smem(L, k, 128), K),
            "onchip_32": _last_fit(lambda L, k: _onchip_smem(L, k, 32), K)}
    if K <= 16:
        last["tma"] = max(L for L in range(step, 8000, step) if _tma_smem(L, K) <= MAX_SMEM)
        last["parked"] = _last_fit(_parked_smem, K)
    for L0, dL, Bx, aligned in itertools.product(filter(None, last.values()), (0, 1, step), (64, 5000, B), (0, 1)):
        assert _plan(Bx, L0 + dL, K, aligned) == _expected(Bx, L0 + dL, K, aligned), (Bx, L0 + dL, K, aligned)
    # the kernel whose limit it is serves the last L that fits, and not the next one
    if K <= 16:
        assert _plan(B, last["tma"], K) == TMA and _plan(B, last["tma"] + step, K) != TMA
        assert _plan(B, last["parked"], K, 0) == PARKED and _plan(B, last["parked"] + 1, K, 0) != PARKED
    elif last["onchip_128"]:
        assert (_plan(B, last["onchip_128"], K), _plan(B, last["onchip_128"] + 1, K)) == (ONCHIP_128, ONCHIP_32)
    else:                                                     # K >= 28: the logits ring of 128 rows alone is past 227 KB
        assert K >= 28 and _plan(B, 1, K) == ONCHIP_32
    assert (_plan(5000, last["onchip_32"], K), _plan(5000, last["onchip_32"] + 1, K)) == (ONCHIP_32, SMALL_ANY_B)
    assert (_plan(B, last["lanes"], K), _plan(B, last["lanes"] + 1, K)) == (SMALL_ANY_B, NONE)
    assert (_plan(64, last["lanes"], K), _plan(64, last["lanes"] + 1, K)) == (SMALL, NONE)


def test_environment_does_not_enter_the_plan(monkeypatch):
    shapes = [(B, L, K, a) for B in (64, 5000, BIG_B + 1) for L in (37, 128, 1500) for K in (7, 10, 20) for a in (0, 1)]
    before = [_plan(*s) for s in shapes]
    for variant in ("1", "2"):
        monkeypatch.setenv("NER_CRF_VIT_VARIANT", variant)
        monkeypatch.setenv("NER_CRF_FWD_VARIANT", variant)
        assert [_plan(*s) for s in shapes] == before
