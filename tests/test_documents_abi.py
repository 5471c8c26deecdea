"""ner_window_plan (document mode's window plan) rejects bad arguments before any CUDA call, so this runs without a GPU."""
from chinesener_b200 import _lib


def test_window_plan_argument_checks():
    h = _lib.lib()

    def plan(B=4, L=1024, W=512, S=255, NW=9, ptrs=1, seg=1, packed=1, padded=1):
        # (token_ids, segment_ids, seq_len, B, L, W, S, NW, win_ids, win_segment_ids, win_mask, doc_src_packed,
        #  doc_src_padded, stream)
        p = ptrs or None
        return h.ner_window_plan(p, seg or None, p, B, L, W, S, NW, p, p, p, packed or None, padded or None, None)

    assert plan(ptrs=0) == -1                         # null pointers
    assert plan(B=-1) == -1
    assert plan(L=0) == -1
    assert plan(NW=-1) == -1
    assert plan(W=2, S=1) == -1                       # a window holds [CLS], [SEP] and one token at least
    assert plan(S=0) == -1
    assert plan(S=511) == -1                          # S > W - 2
    assert plan(W=3, S=2) == -1
    assert plan(NW=1 << 22) == -2                     # NW * W >= 2^31: int32 window rows
    assert plan(B=1 << 21, L=1024) == -2              # B * L >= 2^31: int32 doc rows
    assert plan(B=0, ptrs=0, seg=0, packed=0, padded=0, NW=0) == 0    # empty batch: no-op
