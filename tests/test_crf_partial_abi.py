"""CPU: ner_crf_partial_loglik_fwd / _bwd are exported and declared, reject bad arguments before any CUDA call, and the
plugins that read label_ids as complete gold labels refuse a partially labelled batch before launching anything."""
import importlib
import os
import re

import pytest
import torch

from chinesener_b200 import _lib

INVALID, UNSUPPORTED = -1, -2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("ner_crf_partial_loglik_fwd", "ner_crf_partial_loglik_bwd")


def _fwd(B=2, L=8, K=4, ptrs=None):
    p = [1] * 4 + [1, None, None] if ptrs is None else ptrs       # logits, mask, seq_len, trans, ll, logz, alpha_ws
    return _lib.lib().ner_crf_partial_loglik_fwd(*p, B, L, K, 0, None)


def _bwd(B=2, L=8, K=4, ptrs=None):
    p = [1] * 7 if ptrs is None else ptrs                          # logits .. d_ll
    return _lib.lib().ner_crf_partial_loglik_bwd(*p[:7], 1.0, 1, 1, B, L, K, None)


def test_symbols_are_declared_exported_and_bound():
    with open(os.path.join(ROOT, "include", "ner_b200.h")) as f:
        header = f.read()
    for name in NAMES:
        assert re.search(r"\bint %s\(" % name, header), name
        assert name in _lib.SIGNATURES
        assert getattr(_lib.lib(), name) is not None


def test_forward_argument_checks():
    assert _fwd(B=-1) == INVALID
    assert _fwd(L=0) == INVALID
    assert _fwd(K=0) == INVALID
    assert _fwd(K=33) == UNSUPPORTED
    assert _fwd(B=0, ptrs=[None] * 7) == 0                  # empty batch: no-op
    for i in range(5):                                       # logz and alpha_ws are optional
        p = [1] * 5 + [None, None]
        p[i] = None
        assert _fwd(ptrs=p) == INVALID, i


def test_backward_argument_checks():
    assert _bwd(B=-1) == INVALID
    assert _bwd(L=0) == INVALID
    assert _bwd(K=0) == INVALID
    assert _bwd(K=33) == UNSUPPORTED
    assert _bwd(B=0, ptrs=[None] * 7) == 0
    for i in range(6):                                       # d_ll (index 6) is optional
        p = [1] * 7
        p[i] = None
        assert _bwd(ptrs=p) == INVALID, i
    f = _lib.lib().ner_crf_partial_loglik_bwd
    assert f(1, 1, 1, 1, 1, 1, None, 1.0, None, 1, 2, 8, 4, None) == INVALID     # d_logits
    assert f(1, 1, 1, 1, 1, 1, None, 1.0, 1, None, 2, 8, 4, None) == INVALID     # d_trans


REFUSING = ("bert_ce", "bert_dice", "bert_mrc", "bert_mrc_span", "bert_global_pointer", "bert_bilstm_crf_mtl",
            "bert_bilstm_crf_adv")


class _NoTensor(dict):
    """A feature dict whose only readable entries are label_ids and label_mask: reading anything else (the start of a
    launch) fails the test."""

    def __getitem__(self, k):
        if k not in ("label_ids", "label_mask"):
            raise AssertionError("read {!r} before refusing the label_mask".format(k))
        return super().__getitem__(k)

    def get(self, k, default=None):
        return self[k] if k in self else default


@pytest.mark.parametrize("plugin", REFUSING)
@pytest.mark.parametrize("is_training", [True, False])
def test_plugins_without_a_crf_head_refuse_partial_labels(plugin, is_training):
    build_graph = importlib.import_module("chinesener_b200.model." + plugin).build_graph
    feats = _NoTensor(label_ids=torch.zeros((2, 8), dtype=torch.int32),
                      label_mask=torch.ones((2, 8), dtype=torch.int32))
    with pytest.raises(ValueError, match=plugin):
        build_graph(feats, None, {}, is_training)
