"""Training-data augmentation drawn fresh at every step on the device (Dai & Adel, COLING 2020, "An Analysis of Simple Data
Augmentation for Named Entity Recognition"; masked-LM replacement after Kobayashi, NAACL 2018 and Wu et al. 2019).

params['augment'] maps an operation to its probability p in [0, 1] (main.py: --augment mr=0.3,lwtr=0.3,sis=0.3,mlm=0.15);
params['augment_rows'] (default 0.5) is the share of rows augmented at all, the others stay byte-identical.  On each
augmented row, in this order (ner_augment_rows in ner_b200.h states every rule and hash stream exactly):

  mr    mention replacement: each mention (a B-X token and its run of I-X tokens) is chosen with p and replaced by a
        mention drawn uniformly from the train split's occurrences of type X (tags B-X I-X ...).  Mentions are processed
        left to right with a running row length; a replacement that would push the row past L is skipped.
  lwtr  label-wise token replacement: each token (not [CLS] / [SEP] / [PAD]) is chosen with p and replaced by a token
        drawn from the train split's occurrences of the same tag, O included.
  sis   shuffle within segments: a segment is a mention or a maximal run of O tokens; each one of length >= 2 is chosen
        with p and its tokens are permuted, its tags stay in place.
  mlm   masked-LM replacement: each O token is chosen with p, up to 20 per row in position order; the chosen positions
        become [MASK], a frozen BERT with its masked-LM head scores the row, and each position takes a sample of
        softmax(logits / params['augment_mlm_temperature']) that excludes the original id, [PAD], [UNK], [CLS], [SEP],
        [MASK], [unused*] and ## pieces (ner_vocab_sample).  BERT-tokenized plugins only, with the tagger's vocab.txt.

[CLS], [SEP] and [PAD] tags are never touched, a stray I-X is a segment of its own, and a BERT row's [SEP] moves to the
new end.  Every draw hashes (step seed, operation stream, row, position), the step seed being (seed * 1000003 + step)
mod 2^64 as in pretrain.py, so a run is reproducible.  The pools come from the train split only, and augmentation
applies to TRAIN only.

    python -m chinesener_b200.augment --data_dir D --model_name NAME --augment mr=0.3,sis=0.3 --show 10

prints train sentences next to their augmented versions, entities bracketed.
"""
import argparse
import math
import os

import numpy as np
import torch

from . import ops

OPS = ('mr', 'lwtr', 'sis', 'mlm')
DEFAULT_ROWS = 0.5
SPECIAL_TAGS = ('[PAD]', '[CLS]', '[SEP]')
EXCLUDED_IDS = ('[PAD]', '[UNK]', '[CLS]', '[SEP]', '[MASK]')
REFUSED_WORD_ENHANCE = "its word-enhance features are derived from the text, and augmentation changes the text"


def step_seed(seed, step):
    """The 64-bit seed of one training step (pretrain.py derives its masking seed the same way)."""
    return (int(seed) * 1000003 + int(step)) & 0xFFFFFFFFFFFFFFFF


def _prob(name, p):
    if isinstance(p, bool) or not isinstance(p, (int, float, np.number)) or not 0 <= p <= 1:
        raise ValueError(f"{name} must be a probability in [0, 1] (got {p!r})")
    return float(p)


def parse_augment(text):
    """'mr=0.3,lwtr=0.3' -> {'mr': 0.3, 'lwtr': 0.3}.  ValueError for an unknown operation, a repeated one or a value
    that is not a probability."""
    out = {}
    for part in filter(None, (s.strip() for s in text.split(','))):
        op, eq, val = part.partition('=')
        op = op.strip()
        if op not in OPS:
            raise ValueError(f"unknown augmentation {op!r}: choose from {', '.join(OPS)}")
        if not eq:
            raise ValueError(f"augmentation {op!r} needs a probability: {op}=p")
        if op in out:
            raise ValueError(f"augmentation {op!r} is given twice")
        try:
            p = float(val)
        except ValueError:
            raise ValueError(f"augment {op}: {val!r} is not a number") from None
        out[op] = _prob(f"augment {op}", p)
    return out


def settings(params):
    """The augmentation a params dict asks for, checked -> dict(probs {op: p}, rows, temperature, mlm_dir, seed), or None
    when params['augment'] is unset or empty."""
    aug = params.get('augment')
    if not aug:
        return None
    if isinstance(aug, str):
        aug = parse_augment(aug)
    if not isinstance(aug, dict):
        raise ValueError(f"params['augment'] must map operations to probabilities (got {aug!r})")
    probs = {}
    for op, p in aug.items():
        if op not in OPS:
            raise ValueError(f"unknown augmentation {op!r}: choose from {', '.join(OPS)}")
        probs[op] = _prob(f"augment {op}", p)
    rows = _prob('augment_rows', params.get('augment_rows', DEFAULT_ROWS))
    t = params.get('augment_mlm_temperature', 1.0)
    if isinstance(t, bool) or not isinstance(t, (int, float, np.number)) or not 0 < t < math.inf:
        raise ValueError(f"augment_mlm_temperature must be > 0 (got {t!r})")
    mlm_dir = params.get('augment_mlm_dir') or params.get('pretrain_dir', '')
    return dict(probs=probs, rows=rows, temperature=float(t), mlm_dir=mlm_dir, seed=int(params.get('augment_seed', 1234)))


def check_estimator(est):
    """ValueError, before anything is launched, for what augmentation cannot run with: word-enhance plugins and teachers,
    multi-task / adversarial plugins, and mlm on a plugin without the BERT tokenizer, without the tagger's vocab.txt or
    with an MLM checkpoint that lacks the cls/predictions head.  -> settings(est.params)."""
    from .data.base_preprocess import extract_prefix_surfix
    s = settings(est.params)
    if s is None:
        return None
    name = est.model_name
    we, tok = extract_prefix_surfix(name)
    if we is not None:
        raise ValueError(f"cannot augment {name}: {REFUSED_WORD_ENHANCE}")
    if name.endswith('_mtl') or name.endswith('_adv'):
        raise ValueError(f"cannot augment {name}: its batches mix tasks whose tags are not one BIO tag set")
    if est.teacher is not None and extract_prefix_surfix(est.teacher.model_name)[0] is not None:
        raise ValueError(f"cannot augment with teacher {est.teacher.model_name}: {REFUSED_WORD_ENHANCE}")
    if s['probs'].get('mlm', 0) > 0:
        mlm_vocab(s['mlm_dir'], est.params.get('pretrain_dir', ''), tok)
    return s


def mlm_vocab(mlm_dir, tagger_dir, tokenizer):
    """Checks of the masked-LM replacement's BERT -> its vocabulary (token -> id).  ValueError for a tagger without the
    BERT tokenizer, a missing bert_config.json / vocab.txt, a vocabulary other than the tagger's, or a checkpoint without
    every cls/predictions variable."""
    from . import mlm
    from .data.tokenizer import load_vocab
    if tokenizer != 'bert':
        raise ValueError("augment mlm replaces WordPiece ids: it needs a BERT-tokenized plugin")
    if not mlm_dir:
        raise ValueError("augment mlm needs a BERT with its masked-LM head: set augment_mlm_dir (or pretrain_dir)")
    for f in ('bert_config.json', 'vocab.txt'):
        if not os.path.exists(os.path.join(mlm_dir, f)):
            raise ValueError(f"augment mlm: {os.path.join(mlm_dir, f)} not found")
    vocab = load_vocab(os.path.join(mlm_dir, 'vocab.txt'))
    tv = os.path.join(tagger_dir or '', 'vocab.txt')
    if not tagger_dir or not os.path.exists(tv) or load_vocab(tv) != vocab:
        raise ValueError(f"augment mlm: the vocab.txt under {mlm_dir!r} is not the tagger's ({tv!r})")
    missing = [n for n in mlm.head_names() if n not in mlm._checkpoint_names(mlm_dir)]
    if missing:
        raise ValueError(f"augment mlm: the checkpoint under {mlm_dir!r} lacks the masked-LM head {missing}")
    if '[MASK]' not in vocab:
        raise ValueError(f"augment mlm: {mlm_dir}/vocab.txt has no [MASK]")
    return vocab


def eligible_ids(vocab):
    """u8 [V]: 1 for the ids masked-LM replacement may draw (not [PAD] / [UNK] / [CLS] / [SEP] / [MASK], [unused*] or a
    ## piece)."""
    V = max(vocab.values()) + 1
    ok = np.zeros(V, np.uint8)
    for tok, i in vocab.items():
        ok[i] = not (tok in EXCLUDED_IDS or tok.startswith('[unused') or tok.startswith('##'))
    return ok


def tag_tables(idx2tag):
    """-> (tag_class int32 [K], type_tag int32 [T, 2], type names): class 0 for [PAD] / [CLS] / [SEP] and any other
    non-BIO name, 1 for O, 2 + 2x for B-<type x>, 3 + 2x for I-<type x>, the types in sorted name order; type_tag[x] =
    (B id, I id), -1 for a missing one."""
    idx2tag = {int(k): v for k, v in idx2tag.items()}
    K = max(idx2tag) + 1
    types = sorted({v[2:] for v in idx2tag.values() if v[:2] in ('B-', 'I-')})
    tx = {t: x for x, t in enumerate(types)}
    cls = np.zeros(K, np.int32)
    tt = np.full((len(types), 2), -1, np.int32)
    for k, v in idx2tag.items():
        if v == 'O':
            cls[k] = 1
        elif v[:2] in ('B-', 'I-'):
            x = tx[v[2:]]
            inside = v[0] == 'I'
            cls[k] = 2 + 2 * x + inside
            tt[x, int(inside)] = k
    return cls, tt, types


class Pool:
    """The train split's mention and token pools (numpy; `tables(device)` uploads them once):
    mention_type_off [T+1] / mention_tok_off [n_mentions+1] / mention_tokens: every mention of every type, types in
    tag_tables order and mentions in (row, start) order, so a uniform draw is frequency-weighted;
    tag_tok_off [K+1] / tag_tokens: the token id of every non-special position, grouped by tag in (row, position) order.
    pad_id / pad_tag: the ids the split pads its rows with."""

    def __init__(self, **arrays):
        self.__dict__.update(arrays)
        self._dev = {}

    @classmethod
    def from_arrays(cls, token_ids, label_ids, seq_len, idx2tag):
        ids = np.asarray(token_ids, np.int64)
        lab = np.asarray(label_ids, np.int64)
        B, L = ids.shape
        n = np.clip(np.asarray(seq_len, np.int64), 0, L)
        tag_class, type_tag, types = tag_tables(idx2tag)
        K, T = len(tag_class), len(types)
        valid = np.arange(L)[None, :] < n[:, None]
        cls_at = np.where((lab >= 0) & (lab < K), tag_class[np.clip(lab, 0, K - 1)], 0)
        keep = valid & (cls_at >= 1)
        y, x = lab[keep], ids[keep]                        # row-major: (row, position) order
        order = np.argsort(y, kind='stable')
        tag_tokens = x[order].astype(np.int32)
        tag_tok_off = np.concatenate([[0], np.cumsum(np.bincount(y, minlength=K))]).astype(np.int32)
        per_type = [[] for _ in range(T)]
        rows, starts = np.nonzero(valid & (cls_at >= 2) & (cls_at % 2 == 0))
        for r, s in zip(rows.tolist(), starts.tolist()):
            xt = (int(cls_at[r, s]) - 2) // 2
            inside, e = type_tag[xt, 1], s
            while e + 1 < n[r] and inside >= 0 and lab[r, e + 1] == inside:
                e += 1
            per_type[xt].append(ids[r, s:e + 1])
        mentions = [m for ms in per_type for m in ms]
        mention_type_off = np.concatenate([[0], np.cumsum([len(ms) for ms in per_type])]).astype(np.int32)
        mention_tok_off = np.concatenate([[0], np.cumsum([len(m) for m in mentions])]).astype(np.int32)
        mention_tokens = (np.concatenate(mentions) if mentions else np.zeros(0)).astype(np.int32)
        padded = ~valid
        pad_id = int(np.bincount(ids[padded]).argmax()) if padded.any() and ids[padded].min() >= 0 else 0
        tag2idx = {v: int(k) for k, v in idx2tag.items()}
        return cls(tag_class=tag_class, type_tag=type_tag, types=types, mention_type_off=mention_type_off,
                   mention_tok_off=mention_tok_off, mention_tokens=mention_tokens, tag_tok_off=tag_tok_off,
                   tag_tokens=tag_tokens, pad_id=pad_id, pad_tag=tag2idx.get('[PAD]', 0))

    @classmethod
    def from_records(cls, path, idx2tag):
        """Pools of one .nerrec file (the train split)."""
        from .data import records
        rec = records.RecordFile(path)
        col = lambda k: rec.cols[k][1]
        return cls.from_arrays(col('token_ids'), col('label_ids'), col('seq_len'), idx2tag)

    def tables(self, device):
        """The tables ner_augment_rows reads, on `device` (uploaded once per device)."""
        key = str(device)
        if key not in self._dev:
            up = lambda a: torch.from_numpy(np.ascontiguousarray(a if a.size else np.zeros(1, np.int32),
                                                                 dtype=np.int32)).to(device)
            self._dev[key] = dict(
                tag_class=up(self.tag_class), type_tag=up(self.type_tag.reshape(-1)), n_types=len(self.types),
                mention_type_off=up(self.mention_type_off), mention_tok_off=up(self.mention_tok_off),
                mention_tokens=up(self.mention_tokens), n_mentions=len(self.mention_tok_off) - 1,
                n_mention_tokens=len(self.mention_tokens), tag_tok_off=up(self.tag_tok_off),
                tag_tokens=up(self.tag_tokens), n_tag_tokens=len(self.tag_tokens))
        return self._dev[key]


class FrozenMLM:
    """A BERT and its masked-LM head on a variable store of their own, loaded once from mlm_dir and never trained or
    checkpointed.  `replace` scores [MASK]ed rows with the inference encoder and mlm.head_logits, and writes a
    ner_vocab_sample draw at each position."""

    def __init__(self, mlm_dir, vocab, temperature, device):
        from . import bert, mlm, variables
        self.cfg = bert.load_bert_config(mlm_dir)
        self.V = self.cfg['vocab_size']
        ok = eligible_ids(vocab)
        if len(ok) > self.V:
            raise ValueError(f"augment mlm: vocab.txt holds ids up to {len(ok) - 1}, bert_config.json says vocab_size = "
                             f"{self.V}")
        self.mask_id = vocab['[MASK]']
        self.temperature = temperature
        self.store = variables.VariableStore(device)
        bert.create_bert_variables(self.cfg, self.store)
        mlm.create_head_variables(self.cfg, self.store)
        self.eligible = torch.from_numpy(np.pad(ok, (0, self.V - len(ok)))).to(device)

    def replace(self, mlm_ids, mask, segment_ids, positions, token_ids, seed):
        from . import bert, mlm
        M = positions.numel()
        _, h16 = bert.bert_forward(mlm_ids, mask, segment_ids, self.cfg, self.store)     # padded layout: no sync
        logits, _ = mlm.head_logits(h16, positions.clamp(min=0), M, self.cfg, self.store)
        ops.vocab_sample(logits, self.V, self.eligible, positions, token_ids, self.temperature, seed)


AUGMENTED = ('token_ids', 'label_ids', 'seq_len', 'mask', 'segment_ids')


class Augmenter:
    """Augments device batches with one ner_augment_rows launch (and, with mlm, the frozen BERT and ner_vocab_sample),
    then one 4*B-byte read-back of seq_len for the host-side row lengths the encoders pack by."""

    def __init__(self, s, pool, device, mlm=None):
        self.s, self.pool, self.device, self.mlm = s, pool, torch.device(device), mlm
        p = s['probs']
        self.probs = (s['rows'], p.get('mr', 0.0), p.get('lwtr', 0.0), p.get('sis', 0.0), p.get('mlm', 0.0))
        self.want_mlm = self.probs[4] > 0
        if self.want_mlm and mlm is None:
            raise ValueError("augment mlm needs the frozen masked-LM BERT")

    def launch(self, dev, step):
        """Enqueue the augmentation of device batch `dev` at training step `step` on the current stream -> the new
        device batch (its mask without host lengths yet)."""
        if dev.get('label_mask') is not None:
            raise ValueError("cannot augment partially labelled batches (label_mask): a replaced token has no tag set")
        seed = step_seed(self.s['seed'], step)
        ids = dev['token_ids']
        seg = dev.get('segment_ids')
        if seg is None:
            seg = torch.zeros_like(ids)
        out = ops.augment_rows(ids, dev['label_ids'], dev['seq_len'], dev['mask'], seg, self.pool.tables(ids.device),
                               self.probs, seed, self.pool.pad_id, self.pool.pad_tag,
                               self.mlm.mask_id if self.want_mlm else -1, self.want_mlm)
        if self.want_mlm:
            self.mlm.replace(out['mlm_ids'], out['mask'], out['segment_ids'], out['mlm_positions'].view(-1),
                             out['token_ids'], seed)
        res = dict(dev)
        res.update({k: out[k] for k in AUGMENTED})
        return res

    @staticmethod
    def attach_lengths(dev, lens):
        m = dev['mask']
        m.row_lengths = lens
        m.total_tokens = int(lens.sum())
        m.nonempty_rows = int((lens > 0).sum())
        return dev

    def augment(self, dev, step):
        """The direct path: augment on the current stream and wait for the seq_len read-back."""
        out = self.launch(dev, step)
        lens = out['seq_len'].cpu().numpy()
        return self.attach_lengths(out, lens)

    def pipeline(self, batches, first_step, to_device):
        """Host batches -> augmented device batches for steps first_step, first_step + 1, ...  The copy and augmentation
        of batch i+1 are enqueued on a side stream before batch i is handed out, so they run while step i does; the
        training stream only waits on the side stream's event."""
        main = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(main)

        def enqueue(feats, step):
            with torch.cuda.stream(side):
                out = self.launch(to_device(feats), step)
                lens = torch.empty(out['seq_len'].shape, dtype=torch.int32, pin_memory=True)
                lens.copy_(out['seq_len'], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(side)
            return out, lens, ev

        def finish(item):
            out, lens, ev = item
            ev.synchronize()
            main.wait_event(ev)
            for t in out.values():
                if torch.is_tensor(t) and t.is_cuda:
                    t.record_stream(main)
            return self.attach_lengths(out, lens.numpy().copy())

        it = iter(batches)
        try:
            pending = enqueue(next(it), first_step)
        except StopIteration:
            return
        step = first_step
        for feats in it:
            step += 1
            nxt = enqueue(feats, step)
            yield finish(pending)
            pending = nxt
        yield finish(pending)


def build(params, idx2tag, train_path, device, model_name):
    """The Augmenter of a training run from its params and train split, or None when augmentation is off.  ValueError
    (before anything is launched) for a partially labelled train split."""
    from .data import records
    from .data.base_preprocess import extract_prefix_surfix
    s = settings(params)
    if s is None:
        return None
    if 'label_mask' in records.RecordFile(train_path).names():
        raise ValueError("cannot augment a partially labelled train split (label_mask): a replaced token has no tag set")
    frozen = None
    if s['probs'].get('mlm', 0) > 0:
        vocab = mlm_vocab(s['mlm_dir'], params.get('pretrain_dir', ''), extract_prefix_surfix(model_name)[1])
        frozen = FrozenMLM(s['mlm_dir'], vocab, s['temperature'], device)
    return Augmenter(s, Pool.from_records(train_path, idx2tag), device, frozen)


def bracketed(tokens, tags):
    """'[张三]PER在[北京]LOC' from tokens and tag names ([CLS] / [SEP] / [PAD] left out)."""
    out, i = [], 0
    while i < len(tokens):
        t = tags[i]
        if t in SPECIAL_TAGS:
            i += 1
            continue
        if t[:2] == 'B-':
            j = i + 1
            while j < len(tokens) and tags[j] == 'I-' + t[2:]:
                j += 1
            out.append('[' + ''.join(tokens[i:j]) + ']' + t[2:])
            i = j
        else:
            out.append(tokens[i])
            i += 1
    return ''.join(out)


def main(argv=None):
    from .data.base_preprocess import extract_prefix_surfix
    from .data.records import NerDataset, RecordFile
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--data_dir', required=True)
    ap.add_argument('--model_name', required=True, help='the plugin whose dataset files are read')
    ap.add_argument('--augment', required=True, help='op=p[,op=p ...] with op in ' + ', '.join(OPS))
    ap.add_argument('--augment_rows', type=float, default=DEFAULT_ROWS)
    ap.add_argument('--augment_mlm_dir', default='')
    ap.add_argument('--augment_mlm_temperature', type=float, default=1.0)
    ap.add_argument('--pretrain_dir', default='', help="the tagger's BERT directory (its vocab.txt)")
    ap.add_argument('--show', type=int, default=10, help='how many train sentences to print')
    ap.add_argument('--seed', type=int, default=1234)
    ap.add_argument('--step', type=int, default=0, help='the training step whose draws are shown')
    args = ap.parse_args(argv)
    params = {'augment': parse_augment(args.augment), 'augment_rows': args.augment_rows,
              'augment_mlm_dir': args.augment_mlm_dir, 'augment_mlm_temperature': args.augment_mlm_temperature,
              'pretrain_dir': args.pretrain_dir, 'augment_seed': args.seed}
    ds = NerDataset(args.data_dir, max(args.show, 1), 1, args.model_name)
    idx2tag = {int(k): v for k, v in ds.params['idx2tag'].items()}
    path = ds.file_path('train')
    aug = build(params, idx2tag, path, 'cuda', args.model_name)
    rec = RecordFile(path)
    rows = np.arange(min(args.show, len(rec)))
    host = rec.batch(rows, with_strings=True)
    id2tok = {}
    for toks, ids in zip(host['tokens'], host['token_ids'].numpy()):
        id2tok.update(zip(ids.tolist(), toks))
    for p in (aug.pool.mention_tokens, aug.pool.tag_tokens):
        for i in np.unique(p).tolist():
            id2tok.setdefault(i, None)
    if any(v is None for v in id2tok.values()) or aug.want_mlm:      # ids only the pools or the MLM hold: the vocabulary
        vdir = args.pretrain_dir or args.augment_mlm_dir
        if extract_prefix_surfix(args.model_name)[1] == 'bert' and vdir:
            from .data.tokenizer import load_vocab
            for tok, i in load_vocab(os.path.join(vdir, 'vocab.txt')).items():
                if id2tok.get(i) is None:
                    id2tok[i] = tok
        full = RecordFile(path).batch(slice(0, len(rec)), with_strings=True)
        for toks, ids in zip(full['tokens'], full['token_ids'].numpy()):
            for i, t in zip(ids.tolist(), toks):
                if id2tok.get(i) is None:
                    id2tok[i] = t
    dev = {k: v.cuda() for k, v in host.items() if torch.is_tensor(v)}
    out = aug.augment(dev, args.step)
    new_ids, new_tags, new_len = (out[k].cpu().numpy() for k in ('token_ids', 'label_ids', 'seq_len'))
    for r in range(len(rows)):
        n0 = int(host['seq_len'][r])
        print('orig: ' + bracketed(host['tokens'][r][:n0], host['labels'][r][:n0]))
        n1 = int(new_len[r])
        toks = [id2tok.get(int(i)) or '[{}]'.format(int(i)) for i in new_ids[r, :n1]]
        print('aug:  ' + bracketed(toks, [idx2tag[int(y)] for y in new_tags[r, :n1]]))
        print()


if __name__ == '__main__':
    main()
