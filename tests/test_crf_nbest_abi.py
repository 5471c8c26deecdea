"""CPU: ner_crf_viterbi_nbest is exported and declared, sizes its workspace as documented, rejects bad arguments before any
CUDA call, and params['crf_nbest'] is range-checked and refused by the plugins without one CRF decode before anything is
launched."""
import importlib
import os
import re

import pytest

from chinesener_b200 import _lib, engine, main

INVALID, UNSUPPORTED, WORKSPACE = -1, -2, -3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("ner_crf_viterbi_nbest", "ner_crf_viterbi_nbest_workspace_bytes")


def _ws_bytes(B, L, K, N):
    return _lib.lib().ner_crf_viterbi_nbest_workspace_bytes(B, L, K, N)


def _call(B=2, L=8, K=4, N=3, ptrs=None, ws=1, ws_bytes=None):
    p = [1] * 3 + [1, 1, 1] if ptrs is None else ptrs              # logits, seq_len, trans, tags, scores, count
    nbytes = _ws_bytes(max(B, 0), L, K, N) if ws_bytes is None else ws_bytes
    return _lib.lib().ner_crf_viterbi_nbest(p[0], p[1], p[2], N, p[3], p[4], p[5], ws, nbytes, B, L, K, None)


def test_symbols_are_declared_exported_and_bound():
    with open(os.path.join(ROOT, "include", "ner_b200.h")) as f:
        header = f.read()
    for name in NAMES:
        assert re.search(r"\b(int|size_t) %s\(" % name, header), name
        assert name in _lib.SIGNATURES
        assert getattr(_lib.lib(), name) is not None


def test_workspace_bytes():
    for B, L, K, N in ((1, 1, 1, 1), (64, 128, 10, 8), (3, 4095, 32, 16), (16384, 128, 10, 16)):
        assert _ws_bytes(B, L, K, N) == B * L * K * N * 2          # one 16-bit (i, r) backpointer per list entry
    assert _ws_bytes(0, 8, 4, 2) == 0
    assert _ws_bytes(2, 8, 33, 2) == 0 and _ws_bytes(2, 8, 4, 17) == 0 and _ws_bytes(2, 0, 4, 2) == 0


def test_argument_checks():
    assert _call(K=0) == UNSUPPORTED
    assert _call(K=33) == UNSUPPORTED
    assert _call(N=0) == UNSUPPORTED
    assert _call(N=17) == UNSUPPORTED
    assert _call(B=-1) == INVALID
    assert _call(L=0) == INVALID
    assert _call(B=0, ptrs=[None] * 6, ws=None) == 0                # empty batch: no-op
    for i in range(5):                                               # count_out is optional
        p = [1] * 6
        p[i] = None
        assert _call(ptrs=p) == INVALID, i
    assert _call(ws=None) == WORKSPACE
    assert _call(ws_bytes=_ws_bytes(2, 8, 4, 3) - 1) == WORKSPACE
    assert _call(ptrs=[1] * 5 + [None], ws=None) == WORKSPACE       # a null count_out passes the pointer checks


REFUSING = ("bert_ce", "bert_dice", "bert_mrc", "bert_mrc_span", "bert_global_pointer", "bert_bilstm_crf_mtl",
            "bert_bilstm_crf_adv")


class _NoTensor(dict):
    """A feature dict of which reading any entry (the start of a launch) fails the test."""

    def __getitem__(self, k):
        raise AssertionError("read {!r} before refusing crf_nbest".format(k))

    def get(self, k, default=None):
        raise AssertionError("read {!r} before refusing crf_nbest".format(k))


def test_refusal_list_is_the_plugins_without_one_crf_decode():
    assert set(engine.NBEST_REFUSED) == set(REFUSING)
    for plugin in REFUSING:
        importlib.import_module("chinesener_b200.model." + plugin)


@pytest.mark.parametrize("plugin", REFUSING)
@pytest.mark.parametrize("mode", ["predict", "eval", "train"])
def test_plugins_refuse_nbest_before_launch(plugin, mode):
    est = engine.Estimator(plugin, {'crf_nbest': 4})
    with pytest.raises(ValueError, match=plugin):
        if mode == "predict":
            est.predict_device(_NoTensor())
        elif mode == "eval":
            est.forward_device(_NoTensor(), False)
        else:
            est.train_step(_NoTensor())


@pytest.mark.parametrize("plugin", ["bilstm_crf", "bert_bilstm_crf"])
@pytest.mark.parametrize("n", [0, 17, -1, 2.0, True, "4"])
def test_crf_nbest_range(plugin, n):
    est = engine.Estimator(plugin, {'crf_nbest': n})
    with pytest.raises(ValueError, match="crf_nbest"):
        est.predict_device(_NoTensor())
    with pytest.raises(ValueError, match="crf_nbest"):
        est.forward_device(_NoTensor(), False)


def test_crf_nbest_default_and_accepted():
    assert engine.Estimator("bilstm_crf", {}).crf_nbest() == 1
    for n in (1, 2, 16):
        assert engine.Estimator("bert_bilstm_crf", {'crf_nbest': n}).crf_nbest() == n


def test_multitask_driver_refuses_the_flag(tmp_path):
    with pytest.raises(ValueError, match="crf_nbest"):
        main.main(["--model_name", "bert_bilstm_crf_mtl", "--data", "a,b", "--crf_nbest", "4",
                   "--data_dir", str(tmp_path), "--checkpoint_root", str(tmp_path)])
