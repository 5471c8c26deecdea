"""Entity extraction for the in-process inference path — behaviour of reference tools/infer_utils.py:76-118
(`extract_entity`, `fix_tokens`), which `inference.InferHelper.infer` applies to the PREDICT output."""
from collections import defaultdict

import numpy as np

_SPECIAL_TOKENS = frozenset(('[PAD]', '[CLS]', '[SEP]'))


def extract_entity(tokens, pred_ids, idx2tag):
    """{entity type: set of surface strings} read off a BIO tag sequence.

    Rules kept from the reference (:76-101): an `I-*` tag extends the open span only when the previous tag starts with
    B or I; any other tag closes the span, whose type is the type of the tag just before; `B-*` opens a new one."""
    if len(tokens) != len(pred_ids):
        raise AssertionError('{}!={} tokens and pred_ids must have same length'.format(len(tokens), len(pred_ids)))
    found = defaultdict(set)
    pieces, last = [], idx2tag[pred_ids[0]]

    def close():
        text = ''.join(pieces)
        if text != '':
            found[last.split('-')[1]].add(text)

    for tok, idx in zip(tokens, pred_ids):
        tag = idx2tag[idx]
        kind = tag.split('-')[0]
        if kind == 'I':
            if last[:1] in ('B', 'I'):
                pieces.append(tok)
        else:
            close()
            pieces = [tok] if kind == 'B' else []
        last = tag
    close()
    return found


def fix_tokens(sentence, tokens):
    """Restore the raw characters WordPiece replaced: `[UNK]` becomes the character under the cursor, `##xx` loses its
    continuation mark (reference :104-118).  Edits `tokens` in place and returns it."""
    cursor = 0
    for k, tok in enumerate(tokens):
        if tok in _SPECIAL_TOKENS:
            continue
        if tok == '[UNK]':
            tokens[k] = sentence[cursor]
            cursor += 1
            continue
        if tok.startswith('##'):
            tok = tokens[k] = tok.replace('##', '')
        cursor += len(tok)
    return tokens


def nbest_lists(pred_ids, seq_len):
    """The N best paths a CRF plugin attaches to its device pred_ids when params['crf_nbest'] > 1 (tools/layer.py
    crf_decode) -> per sentence a list of (tags int32 [L], score, probability), best first, counts[b] long (empty for
    seq_len <= 0); probability = exp(score - log Z).  None when pred_ids carries no N-best paths."""
    ids = getattr(pred_ids, 'nbest_ids', None)
    if ids is None:
        return None
    ids, scores = ids.cpu().numpy(), pred_ids.nbest_scores.cpu().numpy()
    counts, logz = pred_ids.nbest_counts.cpu().numpy(), pred_ids.nbest_logz.cpu().numpy()
    lens = np.asarray(seq_len.cpu() if hasattr(seq_len, 'cpu') else seq_len).reshape(-1)
    out = []
    for b in range(ids.shape[0]):
        c = int(counts[b]) if lens[b] > 0 else 0
        probs = np.exp(scores[b, :c].astype(np.float64) - float(logz[b]))
        out.append([(ids[b, r], float(scores[b, r]), float(probs[r])) for r in range(c)])
    return out


def span_lists(pred_ids):
    """The spans a span-pointer plugin (bert_mrc_span) attaches to its device pred_ids -> per sentence a list of
    (type name, start, end_exclusive, probability), ordered by (start, end, type); None when pred_ids carries no spans."""
    spans = getattr(pred_ids, 'spans', None)
    if spans is None:
        return None
    names = pred_ids.span_types
    counts = pred_ids.span_counts.cpu().numpy()
    words, probs = spans.cpu().numpy(), pred_ids.span_probs.cpu().numpy()
    out = []
    for b in range(len(counts)):
        n = min(int(counts[b]), words.shape[1])
        out.append([(names[int(w) >> 24], int(w) & 0xFFF, (int(w) >> 12) & 0xFFF, float(p))
                    for w, p in zip(words[b, :n], probs[b, :n])])
    return out


def span_entities(tokens_batch, spans_batch):
    """Per sentence {type: set of surface strings} from span_lists' output, by the host join of extract_entity_device:
    overlapping and nested entities are all returned."""
    out = []
    for toks, spans in zip(tokens_batch, spans_batch):
        found = defaultdict(set)
        for name, s, e, _ in spans:
            text = ''.join(toks[s:e])
            if text != '':
                found[name].add(text)
        out.append(found)
    return out


def extract_entity_device(tokens_batch, pred_ids, idx2tag):
    """Batched extract_entity with the tag scan on the GPU (ner_extract_spans): pred_ids [B, L] int32 on the device,
    tokens_batch B lists of L token strings -> list of {type: set of surface strings}, equal to
    [extract_entity(tokens, pred_ids[b], idx2tag) for b ...].  Only the spans (4 bytes each) cross to the host."""
    out = []
    for toks, spans in zip(tokens_batch, tag_spans_device(pred_ids, idx2tag)):
        found = defaultdict(set)
        for t, s, e in spans:
            text = ''.join(toks[s:e])
            if text != '':
                found[t].add(text)
        out.append(found)
    return out


def tag_spans_device(pred_ids, idx2tag, _cache={}):
    """The spans of extract_entity's tag scan, run on the GPU (ner_extract_spans): pred_ids [B, L] int32 on the device ->
    per sentence a list of (entity type, start, end_exclusive) in scan order."""
    from .. import ops
    key = tuple(sorted(idx2tag.items()))
    ent = _cache.get(key)
    if ent is None:
        table, types = ops.tag_classes(idx2tag)
        ent = _cache[key] = (table.to(pred_ids.device), types)
    table, types = ent
    if table.device != pred_ids.device:
        table = table.to(pred_ids.device)
    spans, counts = ops.extract_spans(pred_ids, table)
    counts = counts.cpu().numpy()
    spans = spans[:, :max(int(counts.max()), 1)].cpu().numpy() if len(counts) else spans.cpu().numpy()
    return [[(types[int(w) >> 24], int(w) & 0xFFF, (int(w) >> 12) & 0xFFF) for w in spans[b, :counts[b]]]
            for b in range(len(counts))]
