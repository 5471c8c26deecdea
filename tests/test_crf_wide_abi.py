"""CPU: the wide-tag-set CRF entry points (ner_crf_wide_*) are declared, bound and exported, check their arguments before
any CUDA call, size the Viterbi workspace as documented, and choose their kernel configuration from (B, L, K, SMs)
alone."""
import os
import re
import subprocess
import sys

import pytest

from chinesener_b200 import _lib

INVALID, UNSUPPORTED, WORKSPACE = -1, -2, -3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("ner_crf_wide_viterbi", "ner_crf_wide_viterbi_workspace_bytes", "ner_crf_wide_loglik_fwd",
         "ner_crf_wide_loglik_bwd", "ner_crf_wide_plan")
NONE = 4


def _lib_():
    return _lib.lib()


def _ws(B, L, K):
    return _lib_().ner_crf_wide_viterbi_workspace_bytes(B, L, K)


def _viterbi(B=2, L=8, K=40, ptrs=None, ws=1, nbytes=None):
    p = [1] * 5 if ptrs is None else ptrs                          # logits, seq_len, trans, tags_out, best_score
    n = _ws(max(B, 0), L, K) if nbytes is None else nbytes
    return _lib_().ner_crf_wide_viterbi(p[0], p[1], p[2], p[3], p[4], ws, n, B, L, K, None)


def _fwd(B=2, L=8, K=40, ptrs=None):
    p = [1] * 7 if ptrs is None else ptrs                          # logits, tags, seq_len, trans, ll, logz, alpha
    return _lib_().ner_crf_wide_loglik_fwd(*p, B, L, K, 0, None)


def _bwd(B=2, L=8, K=40, ptrs=None):
    p = [1] * 9 if ptrs is None else ptrs   # logits, tags, seq_len, trans, alpha, logz, d_ll, d_logits, d_trans
    return _lib_().ner_crf_wide_loglik_bwd(*p[:7], 1.0, p[7], p[8], B, L, K, None)


def test_symbols_are_declared_exported_and_bound():
    with open(os.path.join(ROOT, "include", "ner_b200.h")) as f:
        header = f.read()
    assert re.search(r"#define NER_MAX_TAGS_WIDE 128\b", header)
    for name in NAMES:
        assert re.search(r"\b(int|size_t) %s\(" % name, header), name
        assert name in _lib.SIGNATURES
        assert getattr(_lib_(), name) is not None


def test_workspace_bytes():
    for B, L, K in ((1, 1, 1), (64, 128, 108), (3, 4095, 128), (65536, 128, 40)):
        assert _ws(B, L, K) == B * L * K                            # one byte-wide backpointer per (row, step, tag)
    assert _ws(0, 8, 40) == 0
    assert _ws(2, 8, 0) == 0 and _ws(2, 8, 129) == 0 and _ws(2, 0, 40) == 0 and _ws(-1, 8, 40) == 0


@pytest.mark.parametrize("call,nptr,optional", [(_viterbi, 5, {4}), (_fwd, 7, {5, 6}), (_bwd, 9, {6})])
def test_argument_checks(call, nptr, optional):
    for K in (0, 129, -3):
        assert call(K=K) == UNSUPPORTED
    assert call(B=-1) == INVALID
    assert call(L=0) == INVALID
    kw = {"ws": None} if call is _viterbi else {}
    assert call(B=0, ptrs=[None] * nptr, **kw) == 0                 # empty batch: no-op
    for i in range(nptr):
        if i in optional:
            continue
        p = [1] * nptr
        p[i] = None
        assert call(ptrs=p) == INVALID, i


def test_viterbi_workspace_checks():
    assert _viterbi(ws=None) == WORKSPACE
    assert _viterbi(nbytes=_ws(2, 8, 40) - 1) == WORKSPACE
    assert _viterbi(B=3, L=4095, K=128, ws=None) == WORKSPACE        # document-length rows are served


def plan_ref(B, L, K, sms):
    """ner_crf_wide_plan restated: 64 threads up to K = 64, else 128; four rows per CTA from B = 8 * SMs on.  Shared
    memory does not enter the plan: crf_wide.cu static_asserts that every configuration fits at its widest K."""
    if B < 1 or L < 1 or K < 1 or K > 128 or sms < 1:
        return NONE
    g4 = B >= 8 * sms
    return (1 if g4 else 0) if K <= 64 else (3 if g4 else 2)


def test_plan_matches_the_restatement_at_every_boundary():
    for sms in (1, 16, 66, 114, 132):
        for B in sorted({1, 2, 4, 8 * sms - 1, 8 * sms, 8 * sms + 1, 65536, 0, -1}):
            for K in (0, 1, 10, 32, 33, 63, 64, 65, 97, 108, 127, 128, 129):
                for L in (0, 1, 128, 4095):
                    assert _lib_().ner_crf_wide_plan(B, L, K, sms) == plan_ref(B, L, K, sms), (B, L, K, sms)
    assert _lib_().ner_crf_wide_plan(64, 128, 40, 0) == NONE


def test_plan_ignores_the_environment():
    code = ("from chinesener_b200 import _lib; l = _lib.lib(); "
            "print([l.ner_crf_wide_plan(B, 128, K, 132) for B in (64, 1056, 65536) for K in (33, 108)])")
    env = dict(os.environ, NER_CRF_WIDE_PLAN="3", NER_CRF_WIDE_G="1", CUDA_VISIBLE_DEVICES="")
    out = [subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True, cwd=ROOT,
                          env=e).stdout for e in (env, dict(os.environ))]
    assert out[0] == out[1] and out[0].strip() == "[0, 2, 1, 3, 1, 3]"
