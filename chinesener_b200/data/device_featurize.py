# -*-coding:utf-8 -*-
"""Raw text -> the features BasicProc.build_seq_feature builds, on the device (ner_featurize_wordpiece /
ner_featurize_chars, csrc/featurize.cu).

The kernels hold no Unicode data of their own: every property the host tokenizer asks `unicodedata` and `str` for is
read into two-stage tables from the running Python once per process, through the host tokenizer's own predicates, so
the device and host tokenizers agree by construction.  The vocabulary becomes an open-addressing hash table over the
UTF-8 bytes of the keys of the tokenizer's dict (not its file), so a duplicated vocabulary line resolves to the id the
host resolves it to.
"""
import unicodedata

import numpy as np
import torch

from .tokenizer import FullTokenizer, TokenizerAdapter, _is_chinese_char, _is_control, _is_punctuation, _is_whitespace

N_CODEPOINTS = 0x110000
F_CONTROL, F_WHITESPACE, F_SPACE, F_PUNCT, F_CJK, F_MN, F_CASED, F_IGNORABLE = (1 << i for i in range(8))
MAX_EXPANSION = 4

_UNICODE = None
_UNICODE_DEV = {}


def _casing(ch):
    """(cased, case-ignorable) as str.lower()'s Final_Sigma rule sees `ch`, read off lower() itself: 'AΣ' + ch + 'A'
    ends its sigma finally iff ch is neither; ch + 'Σ' iff ch is cased and not case-ignorable.  (Whether a
    case-ignorable character is also cased never matters: the rule skips it either way.)"""
    neither = ('AΣ' + ch + 'A').lower()[1] == 'ς'
    cased = (ch + 'Σ').lower()[-1] == 'ς'
    return cased, not neither and not cased


def unicode_tables():
    """-> dict of numpy arrays (built once per process):
    'stage1' uint16 [0x1100], 'stage2' uint32 [n_blocks * 256]: record of code point cp =
    stage2[stage1[cp >> 8] * 256 + (cp & 255)] = flags | combining class << 8 | x << 16, flags F_* above; x > 0 names
    'expand' uint32 [n, 4] row x = NFD(cp.lower()) zero-padded (x = 0: cp maps to itself)."""
    global _UNICODE
    if _UNICODE is not None:
        return _UNICODE
    rec = np.zeros(N_CODEPOINTS, dtype=np.uint32)
    expansions, index = [(0,) * MAX_EXPANSION], {}
    for cp in range(N_CODEPOINTS):
        ch = chr(cp)
        cat = unicodedata.category(ch)
        f = (F_CONTROL * _is_control(ch) | F_WHITESPACE * _is_whitespace(ch) | F_SPACE * ch.isspace()
             | F_PUNCT * _is_punctuation(ch) | F_CJK * _is_chinese_char(cp) | F_MN * (cat == 'Mn'))
        if cat != 'Cn':               # unassigned code points are neither cased nor case-ignorable and map to themselves
            cased, ignorable = _casing(ch)
            f |= F_CASED * cased | F_IGNORABLE * ignorable
        ccc = unicodedata.combining(ch)
        if ccc and f & F_PUNCT:
            raise ValueError(f'U+{cp:04X} is punctuation with combining class {ccc}: the featurise kernel splits '
                             'punctuation before canonical ordering could move a mark across it')
        x = 0
        if cat != 'Cn':
            e = unicodedata.normalize('NFD', ch.lower())
            if e != ch:
                if len(e) > MAX_EXPANSION:
                    raise ValueError(f'NFD(lower(U+{cp:04X})) has {len(e)} code points, more than {MAX_EXPANSION}')
                x = index.get(e)
                if x is None:
                    x = index[e] = len(expansions)
                    expansions.append(tuple(map(ord, e)) + (0,) * (MAX_EXPANSION - len(e)))
        rec[cp] = f | ccc << 8 | x << 16
    if len(expansions) >= 1 << 16:
        raise ValueError('more than 65535 distinct expansions')
    blocks, stage1 = np.unique(rec.reshape(-1, 256), axis=0, return_inverse=True)
    _UNICODE = {'stage1': stage1.reshape(-1).astype(np.uint16), 'stage2': blocks.reshape(-1).astype(np.uint32),
                'expand': np.asarray(expansions, dtype=np.uint32)}
    return _UNICODE


def unicode_record(tables, cps):
    """Records of the code points `cps` (numpy int array) read through the two-stage tables."""
    cps = np.asarray(cps, dtype=np.int64)
    return tables['stage2'][tables['stage1'][cps >> 8].astype(np.int64) * 256 + (cps & 255)]


def _fnv1a(data):
    h = 2166136261
    for byte in data:
        h = ((h ^ byte) * 16777619) & 0xFFFFFFFF
    return h


def vocab_table(vocab):
    """{key: id} -> dict(slots int32 [n_slots] (power of two, -1 empty), entries int32 [n_keys, 3] (blob offset, byte
    length, id), blob uint8, max_piece = the longest key in code points).  FNV-1a over the key's UTF-8 bytes with
    linear probing, as csrc/featurize.cu looks it up."""
    n_slots = 1
    while n_slots < 2 * max(len(vocab), 1):
        n_slots *= 2
    slots = np.full(n_slots, -1, dtype=np.int32)
    entries = np.zeros((max(len(vocab), 1), 3), dtype=np.int32)
    blob = bytearray()
    for e, (key, i) in enumerate(vocab.items()):
        if not 0 <= int(i) < 1 << 24:
            raise ValueError(f'vocabulary id {i} of {key!r} outside [0, 2^24)')
        data = key.encode('utf-8', 'surrogatepass')
        entries[e] = (len(blob), len(data), int(i))
        blob += data
        s = _fnv1a(data) & (n_slots - 1)
        while slots[s] >= 0:
            s = (s + 1) & (n_slots - 1)
        slots[s] = e
    return {'slots': slots, 'entries': entries, 'blob': np.array(bytearray(blob or b'\0'), dtype=np.uint8),
            'max_piece': max((len(k) for k in vocab), default=1)}


class DeviceFeaturizer(object):
    """BasicProc.build_seq_feature + features_to_batch for a whole batch of raw texts in one kernel launch.

    `tokenizer` is a FullTokenizer (WordPiece, either do_lower_case) or a TokenizerAdapter (characters); anything else
    is a TypeError.  featurize(texts) -> the device feature dict of the host path (token_ids, mask, segment_ids,
    seq_len, label_ids zeros, task_ids when asked for) plus 'unk_cursor' [B, L] int32: fix_tokens' cursor at every
    WordPiece [UNK] (the raw character index for the character tokenizer), -1 elsewhere.  entity_text() rebuilds the
    token strings InferHelper.make_feature gives, for the spans that are asked for only."""

    def __init__(self, tokenizer, max_seq_len, device='cuda'):
        if isinstance(tokenizer, FullTokenizer):
            self.wordpiece, vocab = True, tokenizer.vocab
            self.lower = bool(tokenizer.basic_tokenizer.do_lower_case)
            self.special = tuple(vocab[t] for t in ('[CLS]', '[SEP]', '[PAD]', '[UNK]'))
            surface = {i: (k.replace('##', '') if k.startswith('##') else k) for k, i in vocab.items()}
        elif isinstance(tokenizer, TokenizerAdapter):
            self.wordpiece, vocab, self.lower = False, tokenizer.vocab2idx, False
            self.special = (vocab['[PAD]'], vocab['[UNK]'])
            surface = {i: k for k, i in vocab.items() if len(k) == 1}
        else:
            raise TypeError(f'DeviceFeaturizer takes a FullTokenizer or a TokenizerAdapter, not {type(tokenizer).__name__}')
        if max_seq_len < (2 if self.wordpiece else 1):
            raise ValueError(f'max_seq_len {max_seq_len} too small')
        self.max_seq_len, self.device = int(max_seq_len), torch.device(device)
        self.surface = [surface.get(i, '') for i in range(max(surface, default=0) + 1)]
        key = str(self.device)
        if key not in _UNICODE_DEV:
            _UNICODE_DEV[key] = {k: torch.from_numpy(v.view(np.int32 if v.dtype == np.uint32 else np.int16)).to(self.device)
                                 for k, v in unicode_tables().items()}
        self.uni = _UNICODE_DEV[key]
        vt = vocab_table(vocab)
        self.max_piece = vt.pop('max_piece')
        self.vocab = {k: torch.from_numpy(v).to(self.device) for k, v in vt.items()}

    def featurize(self, texts, task_id=None):
        """texts -> device features.  One pinned host-to-device copy carries the offsets and the UTF-8 bytes; after the
        kernel, one 4*B-byte device-to-host copy of seq_len fills mask.row_lengths / total_tokens / nonempty_rows (what
        sequence packing, the MRC pair builder and document windows read without a sync).  That copy is the only
        synchronisation of the call."""
        from .. import ops
        B, L = len(texts), self.max_seq_len
        data = [t.encode('utf-8', 'surrogatepass') for t in texts]
        offsets = np.zeros(B + 1, dtype=np.int64)
        np.cumsum([len(d) for d in data], out=offsets[1:])
        head = 8 * (B + 1)
        host = torch.empty(head + int(offsets[-1]), dtype=torch.uint8, pin_memory=True)
        hv = host.numpy()
        hv[:head] = offsets.view(np.uint8)
        hv[head:] = np.frombuffer(b''.join(data), dtype=np.uint8)
        dev = host.to(self.device, non_blocking=True)
        out = {k: torch.empty((B, L), dtype=torch.int32, device=self.device)
               for k in ('token_ids', 'mask', 'segment_ids', 'unk_cursor')}
        out['seq_len'] = torch.empty((B,), dtype=torch.int32, device=self.device)
        fn = ops.featurize_wordpiece if self.wordpiece else ops.featurize_chars
        fn(dev, host, B, L, self.uni, self.vocab, self.max_piece, self.lower, self.special, out)
        out['label_ids'] = torch.zeros((B, L), dtype=torch.int32, device=self.device)
        if task_id is not None:
            out['task_ids'] = torch.full((B,), int(task_id), dtype=torch.int32, device=self.device)
        lens = out['seq_len'].cpu().numpy().astype(np.int64)
        out['mask'].row_lengths = lens
        out['mask'].total_tokens = int(lens.sum())
        out['mask'].nonempty_rows = int((lens > 0).sum())
        return out

    def entity_text(self, texts, token_ids, unk_cursor, seq_len):
        """Host copies of featurize()'s token_ids / unk_cursor / seq_len -> fn(b, start, end) = ''.join of the token
        strings InferHelper.make_feature gives at positions [start, end) of row b (after fix_tokens for WordPiece).
        Raises IndexError where fix_tokens would: an [UNK] whose cursor is past its sentence's end."""
        if self.wordpiece:
            for b, text in enumerate(texts):
                cur = unk_cursor[b]
                if cur.max(initial=-1) >= len(text):
                    raise IndexError('string index out of range')

        def token(b, p):
            n = int(seq_len[b])
            if p >= n:
                return '[PAD]'
            if self.wordpiece and (p == 0 or p == n - 1):
                return '[CLS]' if p == 0 else '[SEP]'
            c = int(unk_cursor[b, p])
            if c >= 0:
                return texts[b][c] if self.wordpiece else '[UNK]'
            return self.surface[int(token_ids[b, p])]

        return lambda b, s, e: ''.join(token(b, p) for p in range(s, e))
