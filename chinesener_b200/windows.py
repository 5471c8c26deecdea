"""Document mode of the BERT plugins (DESIGN.md §7b): the host half of the window plan.

A batch whose padded length L exceeds the window W is encoded as overlapping W-token windows, each keeping the document's
own [CLS] and [SEP] around C = W - 2 content tokens, started every S content tokens (the last one pulled back to end at the
document's end).  Each document token takes its encoder row from the window where it has the most context; everything
after the encoder runs over the whole document.  The device plan is ner_window_plan (csrc/window.cu); this module holds
the settings check and the window counts the layer sizes its buffers with, and the tests share them."""
import numpy as np

MAX_DOCUMENT_LEN = 4095     # ner_extract_spans keeps positions in 12 bits; the lanes Viterbi keeps backpointers on chip

# plugins whose graph reads the sequence output in a way one stitched row per document token cannot serve
REFUSED = {
    'bert_cnn_crf': "its convolution reads encoder rows at [PAD] positions",
    'bert_ce': "its PREDICT argmax covers [PAD] positions",
    'bert_dice': "its PREDICT argmax covers [PAD] positions",
    'bert_mrc': "its query/context pairs would need the query repeated in every window",
    'bert_mrc_span': "its query/context pairs would need the query repeated in every window",
    'bert_global_pointer': "its PREDICT decode keeps a [B, T, L, L] score tensor",
}


def settings(window, stride, max_position):
    """(params['bert_window'], params['bert_window_stride'], max_position_embeddings) -> (W, S).  None takes the default:
    W = max_position_embeddings, S = (W - 2) // 2.  Raises ValueError outside 3 <= W <= max_position, 1 <= S <= W - 2."""
    W = int(max_position) if window is None else int(window)
    if not 3 <= W <= int(max_position):
        raise ValueError(f"bert_window={window!r}: the window must hold [CLS], [SEP] and at least one token and fit the "
                         f"position table (3 <= bert_window <= max_position_embeddings = {max_position})")
    C = W - 2
    S = C // 2 if stride is None else int(stride)
    if not 1 <= S <= C:
        raise ValueError(f"bert_window_stride={stride!r}: the stride must be in [1, bert_window - 2] = [1, {C}]")
    return W, S


def check_batch(model_name, L, W):
    """ValueError when a batch of padded length L would take document mode (L > W) and cannot."""
    if L <= W:
        return
    if model_name in REFUSED:
        raise ValueError(f"{model_name} cannot tag documents longer than bert_window = {W} (this batch has L = {L}): "
                         f"{REFUSED[model_name]}")
    if L > MAX_DOCUMENT_LEN:
        raise ValueError(f"document mode takes L <= {MAX_DOCUMENT_LEN} (this batch has L = {L}): span positions are 12-bit "
                         "and the Viterbi backpointers of a document are kept on chip")


def document_windows(n, W, S):
    """Windows of documents with n tokens each (scalar or array): 0 for n = 0, 1 for n <= W, else 1 + ceil((n - W) / S)."""
    n = np.asarray(n, dtype=np.int64)
    return np.where(n <= 0, 0, np.where(n <= W, 1, 1 + (n - W + S - 1) // S))


def window_counts(lengths, W, S):
    """Per-document token counts -> (NW windows, window tokens of the window-packed layout)."""
    n = np.asarray(lengths, dtype=np.int64)
    nw = document_windows(n, W, S)
    return int(nw.sum()), int(np.where(n <= W, np.maximum(n, 0), nw * W).sum())
