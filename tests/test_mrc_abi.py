"""ner_mrc_pairs and ner_mrc_merge (the bert_mrc glue) reject bad arguments before any CUDA call, so this runs without a
GPU."""
from chinesener_b200 import _lib


def test_mrc_pairs_argument_checks():
    h = _lib.lib()

    def pairs(B=4, L=8, T=3, Qmax=5, L2=14, ptrs=1, labels_in=1, labels_out=1):
        # (token_ids, seq_len, label_ids, query_ids, query_len, type_tag, B, L, T, Qmax, L2, sep_id,
        #  pair_ids, pair_segment_ids, pair_mask, pair_seq_len, pair_labels, align_rows, stream)
        p = ptrs or None
        return h.ner_mrc_pairs(p, p, labels_in or None, p, p, p, B, L, T, Qmax, L2, 102, p, p, p, p, labels_out or None, p,
                               None)

    assert pairs(ptrs=0, labels_in=0, labels_out=0) == -1       # null pointers
    assert pairs(B=-1) == -1
    assert pairs(L=0) == -1
    assert pairs(Qmax=-1) == -1
    assert pairs(T=0) == -1
    assert pairs(T=33) == -2                                    # more than 32 entity types
    assert pairs(L2=13) == -1                                   # L2 < Qmax + 1 + L
    assert pairs(labels_in=0) == -1                             # BIO labels need label_ids
    assert pairs(B=0, ptrs=0, labels_in=0, labels_out=0) == 0   # empty batch: no-op
    assert pairs(B=1 << 20, L=128, L2=2000) == -2               # B*T*L2 >= 2^31: int32 row indices


def test_mrc_merge_argument_checks():
    h = _lib.lib()
    # (logits, seq_len, type_tag, B, L, T, o_id, cls_id, sep_id, pred_ids, stream)
    assert h.ner_mrc_merge(None, None, None, 4, 8, 3, 1, 8, 9, None, None) == -1      # null pointers
    assert h.ner_mrc_merge(1, 1, 1, 4, 8, 3, 1, 8, 9, None, None) == -1               # null pred_ids
    assert h.ner_mrc_merge(1, 1, 1, -1, 8, 3, 1, 8, 9, 1, None) == -1
    assert h.ner_mrc_merge(1, 1, 1, 4, 0, 3, 1, 8, 9, 1, None) == -1
    assert h.ner_mrc_merge(1, 1, 1, 4, 8, 0, 1, 8, 9, 1, None) == -1
    assert h.ner_mrc_merge(1, 1, 1, 4, 8, 33, 1, 8, 9, 1, None) == -2
    assert h.ner_mrc_merge(None, None, None, 0, 8, 3, 1, 8, 9, None, None) == 0       # empty batch: no-op
