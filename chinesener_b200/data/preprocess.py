# -*-coding:utf-8 -*-
"""Dataset preparation: raw `<split>/sentences.txt` + `<split>/tags.txt` -> `.nerrec` column files + `data_params.pkl`.

Counterpart of the reference's per-dataset scripts (data/msra/preprocess.py:1-52) and of BasicProc.init_data /
dump_tfrecord (data/base_preprocess.py:152-156, 229-253): same split renaming (train/val/test -> train/valid/predict),
same file naming `<tokenizer>_<split>[_<word_enhance>]`, same `data_params.pkl` contents, a sentence whose token and tag
counts differ is dropped and counted — but the output is the memory-mappable format of data/records.py instead of
TFRecords.

    python -m chinesener_b200.data.preprocess --src <dir with train/ val/ test/> --out datasets/msra \
        --tokenizer giga --giga_vec <gigaword .vec>  [--bert_vocab <vocab.txt>]
        [--word_enhance bichar --bichar_vec <bigram .vec> | --word_enhance ex_softword --word_vec <word .vec>
         | --word_enhance lattice --word_vec <word .vec> | --word_enhance softword]  [--partial_labels]
        [--tag_set msra|data]  [--tag_scheme bio|bioes]

--tag_set data takes the tag set from the train split's tags.txt instead of MSRA's (data_tag2idx); --tag_scheme bioes
rewrites B/I/E/S/M-T tags to BIO as they are read (bioes_to_bio), so evaluation and entity extraction, which follow
BIO, see the same entities.
"""
import argparse
import os
import pickle

from .base_preprocess import BiChar, ExSoftWord, Lattice, SoftWord, get_instance
from .records import write_records
from .tokenizer import TextVectors, TokenizerBert, TokenizerGiga, get_bert_tokenizer, get_giga_tokenizer
from .word_enhance import WordVocab, lattice_word_embedding

# data/msra/preprocess.py:7-27 (people_daily uses the same tag set and length)
MSRA_TAG2IDX = {'[PAD]': 0, 'O': 1, 'B-ORG': 2, 'I-ORG': 3, 'B-PER': 4, 'I-PER': 5, 'B-LOC': 6, 'I-LOC': 7, '[CLS]': 8, '[SEP]': 9}
MSRA_MAX_SEQ_LEN = 150
MAPPING = {'train': 'train', 'val': 'valid', 'test': 'predict'}


# data/msr/preprocess.py:7-22 (Chinese word segmentation as a tagging task: the auxiliary task of the multi-task plugins)
MSR_TAG2IDX = {'[PAD]': 0, 'B': 1, 'I': 2, 'E': 3, 'S': 4, '[CLS]': 5, '[SEP]': 6}
MSR_MAPPING = {'training': 'train', 'test_gold': 'valid', 'test': 'predict'}

MAX_TAGS = 128          # the wide CRF kernels' limit (NER_MAX_TAGS_WIDE)
MAX_PARTIAL_TAGS = 32   # a partial label is a 32-bit mask of allowed tags
_BIOES_TO_BIO = {'B': 'B', 'I': 'I', 'E': 'I', 'M': 'I', 'S': 'B'}


def bioes_to_bio(tag_line):
    """One tags.txt line from BIOES (with M as a synonym of I) to BIO: E-T, M-T -> I-T and S-T -> B-T.  Partial labels
    ('?' and 'T1|T2' alternatives) are rewritten alternative by alternative."""
    def one(tag):
        if tag == '?':
            return tag
        if '|' in tag:
            return '|'.join(one(t) for t in tag.split('|'))
        prefix, sep, typ = tag.partition('-')
        if sep and prefix in _BIOES_TO_BIO:
            return _BIOES_TO_BIO[prefix] + '-' + typ
        return tag
    return ' '.join(one(t) for t in tag_line.split(' '))


def data_tag2idx(tag_lines):
    """The tag set of a corpus in the MSRA layout: [PAD] = 0, O = 1, then B-T, I-T for each entity type T in sorted
    order, then [CLS], [SEP].  tag_lines are BIO lines (partial-label alternatives count; '?' adds nothing)."""
    types = set()
    for line in tag_lines:
        for tag in line.split(' '):
            for t in tag.split('|'):
                prefix, sep, typ = t.partition('-')
                if sep and prefix in ('B', 'I') and typ:
                    types.add(typ)
    tags = ['[PAD]', 'O'] + [p + '-' + t for t in sorted(types) for p in ('B', 'I')] + ['[CLS]', '[SEP]']
    if len(tags) > MAX_TAGS:
        raise ValueError('the train split has {} entity types, {} tags; the CRF kernels take at most {} tags'.format(
            len(types), len(tags), MAX_TAGS))
    return {t: i for i, t in enumerate(tags)}


def scheme_loader(tag_scheme, load=None):
    """load_data for a tag scheme: BIO files as they are, BIOES files rewritten to BIO line by line."""
    load = load or load_data
    if tag_scheme == 'bio':
        return load

    def load_bioes(data_dir, file_name):
        sentences, tags = load(data_dir, file_name)
        return sentences, [bioes_to_bio(t) for t in tags]
    return load_bioes


def msr_gen_tag(length):
    """data/msr/preprocess.py:27-33"""
    if length == 1:
        return 'S'
    if length == 2:
        return 'B E'
    return ' '.join(['B'] + ['I'] * (length - 2) + ['E'])


def load_msr_data(data_dir, file_name):
    """data/msr/preprocess.py:36-52 — `msr_<split>.utf8`: words separated by spaces -> characters + B/I/E/S tags."""
    sentences, tags = [], []
    for line in read_text(data_dir, 'msr_{}.utf8'.format(file_name)):
        if line == '':
            continue
        words = [t for t in line.split(' ') if t not in ['', '"']]
        tags.append(' '.join(msr_gen_tag(len(t)) for t in words))
        sentences.append(' '.join(c for t in words for c in t))
    return sentences, tags


def read_text(data_dir, filename):
    with open(os.path.join(data_dir, filename), 'r', encoding='utf-8') as f:
        return [line.strip() for line in f]


def load_data(data_dir, file_name):
    sentences = read_text(data_dir, os.path.join(file_name, 'sentences.txt'))
    tags = read_text(data_dir, os.path.join(file_name, 'tags.txt'))
    assert len(sentences) == len(tags)
    return sentences, tags


def dump_records(proc, src_dir, out_dir, file_name, mapping=MAPPING, word_enhance=None, embedding=None, verbose=True,
                 load_data=None, bichar_embedding=None):
    """One split through `proc.build_feature` -> `<out_dir>/<tokenizer>_<renamed>[_<enhance>].nerrec`; the train split
    also writes `<tokenizer>[_<enhance>]_data_params.pkl` (data/base_preprocess.py:206-227, 247-253), with the bigram
    table as `bichar_embedding` when one is given."""
    sentences, tags = (load_data or globals()['load_data'])(src_dir, file_name)
    feats, n_invalid = [], 0
    for sentence, tag in zip(sentences, tags):
        try:
            feats.append(proc.build_feature(sentence, tag))
        except Exception as e:          # the reference prints and skips (n_token != n_tag after tokenisation, unknown tag)
            n_invalid += 1
            if verbose:
                print(e)
    if not any(-1 in f['label_ids'] for f in feats if 'label_mask' in f):
        for f in feats:             # a split without open positions is written exactly as without --partial_labels
            f.pop('label_mask', None)
    os.makedirs(out_dir, exist_ok=True)
    stem = '_'.join(filter(None, [proc.tokenizer_type, mapping[file_name], word_enhance]))
    write_records(os.path.join(out_dir, stem + '.nerrec'), feats, proc.max_seq_len)
    if verbose:
        print('Dump {} sample, invalid_sample = {}'.format(len(feats), n_invalid))
    if 'train' in file_name:
        params = proc.build_data_params(len(feats))
        if proc.tokenizer_type == TokenizerGiga and embedding is not None:
            params['embedding'] = embedding
        if bichar_embedding is not None:
            params['bichar_embedding'] = bichar_embedding
        with open(os.path.join(out_dir, '_'.join(filter(None, [proc.tokenizer_type, word_enhance, 'data_params.pkl']))), 'wb') as f:
            pickle.dump(params, f)
    return len(feats), n_invalid


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--src', required=True, help='directory holding train/ val/ test/ with sentences.txt + tags.txt')
    ap.add_argument('--out', required=True)
    ap.add_argument('--tokenizer', default=TokenizerGiga, choices=[TokenizerGiga, TokenizerBert])
    ap.add_argument('--giga_vec', default='./pretrain_model/giga/gigaword_chn.all.a2b.uni.ite50.vec')
    ap.add_argument('--bert_dir', default='./pretrain_model/ch_google/')
    ap.add_argument('--max_seq_len', type=int, default=MSRA_MAX_SEQ_LEN)
    ap.add_argument('--seed', type=int, default=1234, help='seed of the two add-on embedding rows ([PAD], [UNK])')
    ap.add_argument('--format', default='ner', choices=['ner', 'msr'], help="'msr': word-segmented msr_<split>.utf8 files (CWS tags)")
    ap.add_argument('--word_enhance', default=None, choices=[BiChar, SoftWord, ExSoftWord, Lattice],
                    help='extra input of the bilstm_crf_<word_enhance> plugins (giga tokenizer); softword segments with jieba')
    ap.add_argument('--bichar_vec', default='./pretrain_model/giga/gigaword_chn.all.a2b.bi.ite50.vec',
                    help='bigram vectors (giga .vec format) for --word_enhance bichar')
    ap.add_argument('--word_vec', default='./pretrain_model/ctb50/ctb.50d.vec',
                    help='word vectors (giga .vec format) whose vocabulary is the lexicon of --word_enhance ex_softword / '
                         'lattice (lattice also keeps the vectors as the word table)')
    ap.add_argument('--tag_set', default='msra', choices=['msra', 'data'],
                    help="'msra': MSRA's ten tags; 'data': [PAD], O, B-/I- of every entity type in the train split's "
                         "tags.txt (sorted), [CLS], [SEP]; at most 128 tags")
    ap.add_argument('--tag_scheme', default='bio', choices=['bio', 'bioes'],
                    help="'bioes': tags.txt uses B/I/E/S(/M)-T; they are rewritten to BIO before indexing")
    ap.add_argument('--partial_labels', action='store_true',
                    help="tags.txt may leave a token's tag open: '?' (any tag) or a set 'T1|T2|...'; such splits get a "
                         "label_mask column and label_id -1 at the open positions, for the CRF plugins")
    args = ap.parse_args(argv)
    msr = args.format == 'msr'
    if msr and (args.tag_set != 'msra' or args.tag_scheme != 'bio'):
        ap.error("--format msr has its own tag set: --tag_set and --tag_scheme apply to --format ner")
    load = scheme_loader(args.tag_scheme)
    tag2idx = MSR_TAG2IDX if msr else MSRA_TAG2IDX
    if args.tag_set == 'data':
        tag2idx = data_tag2idx(load(args.src, 'train')[1])
        print('tag set from the train split: {} tags'.format(len(tag2idx)))
    if args.partial_labels and len(tag2idx) > MAX_PARTIAL_TAGS:
        ap.error('--partial_labels takes at most {} tags (a 32-bit mask of allowed tags); this tag set has {}'.format(
            MAX_PARTIAL_TAGS, len(tag2idx)))
    if args.tokenizer == TokenizerGiga:
        tok = get_giga_tokenizer(args.giga_vec)
        emb = tok.embedding(args.seed)
    else:
        tok, emb = get_bert_tokenizer(args.bert_dir), None
    kwargs, bichar_emb = {}, None
    if args.word_enhance == BiChar:
        kwargs['bichar_tokenizer'] = get_giga_tokenizer(args.bichar_vec)
        bichar_emb = kwargs['bichar_tokenizer'].embedding(args.seed)
    elif args.word_enhance == ExSoftWord:
        words = TextVectors(args.word_vec).index2word
        kwargs['vocab'] = WordVocab(words, dict.fromkeys(words, 1))
    elif args.word_enhance == Lattice:
        vec = TextVectors(args.word_vec)
        kwargs['vocab'] = WordVocab(vec.index2word, dict.fromkeys(vec.index2word, 1))
        kwargs['word_embedding'] = lattice_word_embedding(vec, args.seed)
    proc = get_instance(args.tokenizer, args.max_seq_len, tag2idx, tok,
                        word_enhance=args.word_enhance, **kwargs)
    proc.partial_labels = args.partial_labels
    for file in (MSR_MAPPING if msr else MAPPING):
        print('Dumping records for {} tokenizer = {}'.format(file, args.tokenizer))
        dump_records(proc, args.src, args.out, file, mapping=MSR_MAPPING if msr else MAPPING, embedding=emb,
                     load_data=load_msr_data if msr else load, word_enhance=args.word_enhance, bichar_embedding=bichar_emb)
        if args.word_enhance == Lattice:
            print('lattice words dropped by the max_lattice_words cap so far: {}'.format(proc.dropped))


if __name__ == '__main__':
    main()
