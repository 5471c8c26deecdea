"""CPU: ner_crf_distill_fwd / _bwd are exported and declared and reject bad arguments before any CUDA call, and an
Estimator refuses a teacher it cannot distill from before launching anything."""
import os
import re

import pytest

from chinesener_b200 import _lib, engine

INVALID, UNSUPPORTED = -1, -2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("ner_crf_distill_fwd", "ner_crf_distill_bwd")


def _fwd(B=2, L=8, K=4, inv_temp=1.0, ptrs=None):
    p = [1] * 7 if ptrs is None else ptrs         # t_logits, t_trans, s_logits, s_trans, seq_len, logz, alpha_ws
    return _lib.lib().ner_crf_distill_fwd(*p[:5], inv_temp, *p[5:], B, L, K, 0, None)


def _bwd(B=2, L=8, K=4, inv_temp=1.0, ptrs=None):
    p = [1] * 11 if ptrs is None else ptrs        # t_logits .. seq_len, alpha_ws, logz, d_kl, kl, d_s_logits, d_s_trans
    return _lib.lib().ner_crf_distill_bwd(*p[:5], inv_temp, *p[5:8], 1.0, *p[8:], B, L, K, 0, None)


def test_symbols_are_declared_exported_and_bound():
    with open(os.path.join(ROOT, "include", "ner_b200.h")) as f:
        header = f.read()
    for name in NAMES:
        assert re.search(r"\bint %s\(" % name, header), name
        assert name in _lib.SIGNATURES
        assert getattr(_lib.lib(), name) is not None


@pytest.mark.parametrize("call", [_fwd, _bwd])
def test_argument_checks(call):
    assert call(B=-1) == INVALID
    assert call(L=0) == INVALID
    assert call(K=0) == INVALID
    assert call(K=33) == UNSUPPORTED
    assert call(L=4096) == UNSUPPORTED
    for t in (0.0, -1.0, float("nan"), float("inf")):
        assert call(inv_temp=t) == INVALID, t
        assert call(B=0, inv_temp=t) == INVALID, t
    n = 7 if call is _fwd else 11
    assert call(B=0, ptrs=[None] * n) == 0                   # empty batch: no-op
    optional = () if call is _fwd else (7,)                  # d_kl
    for i in range(n):
        if i in optional:
            continue
        p = [1] * n
        p[i] = None
        assert call(ptrs=p) == INVALID, i


PARAMS = dict(label_size=10, idx2tag={i: str(i) for i in range(10)})


def _est(name, teacher=None, **params):
    return engine.Estimator(name, dict(PARAMS, **params), device="cpu", teacher=teacher)


@pytest.mark.parametrize("student,teacher", [
    ("bilstm_crf", "bilstm_crf_softlexicon"), ("bilstm_crf", "lattice_lstm_crf"), ("bilstm_crf", "bilstm_crf_bichar"),
    ("bert_crf", "bert_bilstm_crf"), ("bilstm_crf_softlexicon", "bilstm_crf_softlexicon"), ("bilstm_crf", "bilstm_crf"),
])
def test_supported_pairs(student, teacher):
    assert _est(student, _est(teacher)).distill_settings() == (0.5, 1.0)


@pytest.mark.parametrize("student,teacher,match", [
    ("bilstm_crf", "bert_ce", "no CRF"), ("bert_mrc", "bert_bilstm_crf", "no CRF"),
    ("bert_bilstm_crf_mtl", "bert_bilstm_crf", "per-task"), ("bilstm_crf", "bert_bilstm_crf", "tokenizer"),
    ("bert_crf", "bilstm_crf", "tokenizer"), ("bilstm_crf_softlexicon", "bilstm_crf", "softlexicon"),
    ("bilstm_crf_bichar", "bilstm_crf_softlexicon", "bichar"),
])
def test_refused_pairs(student, teacher, match):
    with pytest.raises(ValueError, match=match):
        _est(student, _est(teacher))


def test_refused_tag_sets_and_settings():
    with pytest.raises(ValueError, match="label_size"):
        _est("bilstm_crf", _est("bilstm_crf", label_size=7))
    with pytest.raises(ValueError, match="idx2tag"):
        _est("bilstm_crf", _est("bilstm_crf", idx2tag={i: "x" + str(i) for i in range(10)}))
    for a in (0, -0.5, 1.5, float("nan"), True):
        with pytest.raises(ValueError, match="distill_alpha"):
            _est("bilstm_crf", _est("bilstm_crf"), distill_alpha=a)
    for t in (0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="distill_temperature"):
            _est("bilstm_crf", _est("bilstm_crf"), distill_temperature=t)
    assert _est("bilstm_crf", _est("bilstm_crf"), distill_alpha=1, distill_temperature=2).distill_settings() == (1.0, 2.0)


def test_driver_refuses_a_teacher_without_a_checkpoint(tmp_path):
    from chinesener_b200 import main
    with pytest.raises(ValueError, match="teacher_dir"):
        main.main(["--model_name", "bilstm_crf", "--teacher_model", "bilstm_crf_softlexicon", "--teacher_dir",
                   str(tmp_path), "--data_dir", str(tmp_path / "absent"), "--checkpoint_root", str(tmp_path)])
    with pytest.raises(ValueError, match="teacher_dir"):
        main.main(["--model_name", "bilstm_crf", "--teacher_model", "bilstm_crf_softlexicon",
                   "--data_dir", str(tmp_path / "absent"), "--checkpoint_root", str(tmp_path)])


def test_driver_refuses_a_teacher_for_multi_task(tmp_path):
    from chinesener_b200 import main
    with pytest.raises(ValueError, match="multi-task"):
        main.main(["--model_name", "bert_bilstm_crf_mtl", "--data", "a,b", "--teacher_model", "bert_bilstm_crf",
                   "--teacher_dir", str(tmp_path), "--checkpoint_root", str(tmp_path)])


def test_driver_refuses_teacher_flags_without_a_teacher(tmp_path):
    from chinesener_b200 import main
    for flag in ("--teacher_dir", "--teacher_pretrain_dir"):
        with pytest.raises(ValueError, match="need --teacher_model"):
            main.main(["--model_name", "bilstm_crf", flag, str(tmp_path), "--data_dir", str(tmp_path / "absent"),
                       "--checkpoint_root", str(tmp_path)])
