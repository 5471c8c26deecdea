# -*-coding:utf-8 -*-
"""Entity types and queries of the `bert_mrc` plugin (MRC-style NER: one BERT query per entity type).

The reference's mrc/ code, its query texts and its dataset format are not part of this repository, so this is a
restatement, not a pinned parity point.  The entity types are every X with a `B-X` tag in params['idx2tag'], in
ascending tag-id order (ORG, PER, LOC with the MSRA tags).  params['mrc_queries'] (type -> text) defaults to the MSRA
queries released with Li et al., "A Unified MRC Framework for Named Entity Recognition" (ACL 2020); they are tokenized
once with the BERT FullTokenizer of `<pretrain_dir>/vocab.txt`.  params['mrc_query_ids'] (type -> token ids) replaces
the tokenization, which is what synthetic mode (pretrain_dir '', no vocabulary) needs.
"""
import os

import torch

from .. import bert
from .tokenizer import get_bert_tokenizer

DEFAULT_QUERIES = {
    'PER': '人名和虚构的人物形象',
    'LOC': '按照地理位置划分的国家,城市,乡镇,大洲',
    'ORG': '组织包括公司,政府党派,学校,政府,新闻机构',
}
MAX_TYPES = 32              # ner_mrc_pairs / ner_mrc_merge
SEP_TOKEN_ID = 102          # '[SEP]' of the BERT-Base-Chinese vocabulary: the query separator when there is no vocab.txt


def entity_types(idx2tag):
    """-> [(X, id of B-X, id of I-X)] for every X with a B-X tag, in ascending B-X id."""
    tag2idx = {tag: i for i, tag in idx2tag.items()}
    types = []
    for i in sorted(idx2tag):
        tag = idx2tag[i]
        if tag.startswith('B-'):
            name = tag[2:]
            if 'I-' + name not in tag2idx:
                raise ValueError(f"bert_mrc: entity type {name!r} has a B-{name} tag but no I-{name} tag")
            types.append((name, i, tag2idx['I-' + name]))
    if not 1 <= len(types) <= MAX_TYPES:
        raise ValueError(f"bert_mrc needs 1 to {MAX_TYPES} entity types (B-X tags), idx2tag has {len(types)}")
    return types


def query_token_ids(params, names):
    """-> ([token ids of each type's query, in the order of `names`], id of [SEP]).  Tokenizes params['mrc_queries']
    (default DEFAULT_QUERIES) with the vocabulary of pretrain_dir unless params['mrc_query_ids'] gives the ids."""
    vocab_file = os.path.join(params.get('pretrain_dir') or '', 'vocab.txt')
    tokenizer = get_bert_tokenizer(params['pretrain_dir']) if os.path.exists(vocab_file) else None
    given = params.get('mrc_query_ids')
    if given is None:
        if tokenizer is None:
            raise FileNotFoundError(f"{vocab_file} not found: bert_mrc tokenizes its queries with the BERT vocabulary; "
                                    "pass params['mrc_query_ids'] (entity type -> token ids) to run without one")
        texts = params.get('mrc_queries') or DEFAULT_QUERIES
        missing = [n for n in names if n not in texts]
        if missing:
            raise KeyError(f"bert_mrc: no query for entity type {missing[0]!r} in params['mrc_queries']")
        ids = [tokenizer.convert_tokens_to_ids(tokenizer.tokenize(texts[n])) for n in names]
    else:
        missing = [n for n in names if n not in given]
        if missing:
            raise KeyError(f"bert_mrc: no query for entity type {missing[0]!r} in params['mrc_query_ids']")
        ids = [[int(i) for i in given[n]] for n in names]
    return ids, tokenizer.vocab['[SEP]'] if tokenizer is not None else SEP_TOKEN_ID


class TypeTable:
    """The entity types of params['idx2tag'] (entity_types) and the tag ids a per-type decode writes: names, T, type_tag
    [T, 2] (B-X, I-X ids) on `device`, o_tag, and cls_tag / sep_tag (o_tag when idx2tag has no [CLS] / [SEP])."""

    def __init__(self, params, device='cuda'):
        idx2tag = params['idx2tag']
        types = entity_types(idx2tag)
        self.names = [n for n, _, _ in types]
        self.T = len(types)
        self.L = int(params['max_seq_len'])
        self.type_tag = torch.tensor([[b, i] for _, b, i in types], dtype=torch.int32).to(device)
        tag2idx = {tag: i for i, tag in idx2tag.items()}
        if 'O' not in tag2idx:
            raise ValueError("idx2tag has no 'O' tag: the per-type decode writes it outside the entities")
        self.o_tag = tag2idx['O']
        self.cls_tag = tag2idx.get('[CLS]', self.o_tag)
        self.sep_tag = tag2idx.get('[SEP]', self.o_tag)


class MrcTable(TypeTable):
    """Everything the bert_mrc graph needs about its queries: host sizes and the device tables of ner_mrc_pairs /
    ner_mrc_merge, on top of the TypeTable."""

    def __init__(self, params, device='cuda'):
        super().__init__(params, device)
        ids, self.sep_id = query_token_ids(params, self.names)
        self.query_lens = [len(q) for q in ids]
        self.qmax = max(self.query_lens)
        self.L2 = self.qmax + 1 + self.L
        max_pos = bert.load_bert_config(params['pretrain_dir'])['max_position_embeddings']
        if self.L2 > max_pos:
            raise ValueError(f"bert_mrc: a pair holds up to {self.L2} tokens (longest query {self.qmax} + [SEP] + max_seq_len "
                             f"{self.L}), more than BERT's max_position_embeddings = {max_pos}")
        self.query_overhead = sum(q + 1 for q in self.query_lens)          # tokens each non-empty sentence adds
        table = torch.zeros((self.T, self.qmax), dtype=torch.int32)
        for t, q in enumerate(ids):
            table[t, :len(q)] = torch.tensor(q, dtype=torch.int32)
        self.query_ids = table.to(device)
        self.query_len = torch.tensor(self.query_lens, dtype=torch.int32).to(device)

    def pair_tokens(self, mask):
        """Real tokens of the B*T pairs of a batch, from the host counts Estimator.to_device attaches to its mask
        (total_tokens, nonempty_rows); None without them.  Exact when mask[b] is 1 on the first seq_len[b] positions
        only, as in every BERT feature batch."""
        total, rows = getattr(mask, 'total_tokens', None), getattr(mask, 'nonempty_rows', None)
        if total is None or rows is None:
            return None
        return self.T * total + self.query_overhead * rows


def device_table(params):
    """The MrcTable of a params dict, built once (as model/_blocks.device_constant caches its tables)."""
    cache = params.setdefault('_device_consts', {})
    if 'mrc_table' not in cache:
        cache['mrc_table'] = MrcTable(params)
    return cache['mrc_table']


def type_table(params):
    """The TypeTable of a params dict, built once: what a plugin without queries (bert_global_pointer) needs."""
    cache = params.setdefault('_device_consts', {})
    if 'type_table' not in cache:
        cache['type_table'] = TypeTable(params)
    return cache['type_table']
