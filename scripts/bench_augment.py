"""Training-data augmentation on the GPU.

usage: python scripts/bench_augment.py        (prints one JSON line)

  * ner_augment_rows with mr, lwtr and sis at p = 0.3 on every row, at B = 64 and B = 16 384 MSRA-shaped rows (L = 128):
    kernel time, median of CUDA events;
  * ner_vocab_sample at M = 1 280 (64 rows x 20), V = 21 128: kernel time, bytes/s over the M V f32 logits it reads, and
    the share of the 3.35 TB/s of the H100 SXM data sheet;
  * the TRAIN step (Estimator.train_step, host batch included) of bilstm_crf and bert_bilstm_crf on one MSRA-shaped
    B = 64, L = 128 batch, with augmentation off, with mr + lwtr + sis (p = 0.3, augment_rows 0.5), and for
    bert_bilstm_crf the same plus mlm (p = 0.15), alternated over three rounds.  An augmented step runs through
    Augmenter.pipeline, so the next batch's augmentation overlaps the step as it does in training.  mlm needs a BERT
    vocabulary, so bilstm_crf (character vocabulary) has no mlm row.
The card's name, power limit and max SM clock are read in the same run.  A temporary directory holds the BERT-base
checkpoint with its masked-LM head that mlm loads.
"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from chinesener_b200 import augment, bert, engine, mlm, ops, synthetic, variables  # noqa: E402
from chinesener_b200.synthetic import MSRA_IDX2TAG  # noqa: E402

HBM_BPS = 3.35e12
ROUNDS = 3


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def events(fn, warm=3, iters=50):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def pool_of(vocab):
    b = synthetic.msra_batch(4096, 128, vocab=vocab, seed=99)
    return augment.Pool.from_arrays(b['token_ids'].numpy(), b['label_ids'].numpy(), b['seq_len'].numpy(), MSRA_IDX2TAG)


def bench_rows():
    pool = pool_of(21128)
    tb = pool.tables('cuda')
    out = []
    for B in (64, 16384):
        f = {k: v.cuda() for k, v in synthetic.msra_batch(B, 128, seed=1).items()}
        fn = lambda: ops.augment_rows(f['token_ids'], f['label_ids'], f['seq_len'], f['mask'], f['segment_ids'], tb,
                                      (1.0, .3, .3, .3, 0.0), 7, pool.pad_id, pool.pad_tag)
        out.append(dict(B=B, L=128, us=events(fn) * 1e3))
    return out


def bench_sample():
    M, V, ld = 1280, 21128, 21152
    g = torch.Generator().manual_seed(0)
    z = (torch.randn(M, ld, generator=g) * 3).cuda()
    elig = torch.ones(V, dtype=torch.uint8).cuda()
    pos = torch.arange(M, dtype=torch.int32).cuda() * 3
    toks = torch.zeros(64 * 128, dtype=torch.int32).cuda()
    t = events(lambda: ops.vocab_sample(z, V, elig, pos, toks, 1.0, 7), iters=100)
    nbytes = M * V * 4
    return dict(M=M, V=V, us=t * 1e3, tb_s=nbytes / (t * 1e-3) / 1e12, share_of_hbm=nbytes / (t * 1e-3) / HBM_BPS)


def bert_dir(tmp):
    """BERT-base-Chinese (random) with its masked-LM head and a 21 128-line vocab.txt."""
    cfg = bert.load_bert_config('')
    V = cfg['vocab_size']
    vocab = ['[PAD]'] + ['[unused%d]' % i for i in range(1, 100)] + ['[UNK]', '[CLS]', '[SEP]', '[MASK]']
    vocab += ['##%d' % i for i in range(10)] + [chr(0x4E00 + i) for i in range(V - len(vocab) - 10)]
    with open(os.path.join(tmp, 'vocab.txt'), 'w') as f:
        f.write('\n'.join(vocab) + '\n')
    store = variables.VariableStore('cuda', seed=1)
    bert.create_bert_variables(cfg, store)
    mlm.create_head_variables(cfg, store)
    mlm.export_pretrained(store, tmp, '')
    return tmp


def bench_steps(tmp):
    d = bert_dir(tmp)
    base = synthetic.data_params(128, batch_size=64)
    emb = np.random.default_rng(0).standard_normal((21128, 100)).astype(np.float32) * 0.1
    configs = {'bilstm_crf': dict(base, embedding=emb), 'bert_bilstm_crf': dict(base, pretrain_dir=d)}
    variants = {'off': None, 'mr+lwtr+sis': {'mr': .3, 'lwtr': .3, 'sis': .3},
                'mr+lwtr+sis+mlm': {'mr': .3, 'lwtr': .3, 'sis': .3, 'mlm': .15}}
    batch = synthetic.msra_batch(64, 128, seed=3)
    pool = pool_of(21128)
    res = {}
    for model, params in configs.items():
        runs = {}
        for name, probs in variants.items():
            if name.endswith('mlm') and model == 'bilstm_crf':
                continue
            p = dict(params, **({'augment': probs, 'augment_seed': 5} if probs else {}))
            est = engine.Estimator(model, p)
            aug = None
            if probs:
                frozen = (augment.FrozenMLM(d, augment.mlm_vocab(d, d, 'bert'), 1.0, 'cuda') if 'mlm' in probs else None)
                aug = augment.Augmenter(augment.settings(p), pool, 'cuda', frozen)
            runs[name] = (est, aug)
        times = {k: [] for k in runs}

        def steps(est, aug, n):
            it = (batch for _ in range(n))
            feed = aug.pipeline(it, est.store.global_step, est.to_device) if aug else it
            torch.cuda.synchronize()
            s = time.perf_counter()
            for f in feed:
                loss = est.train_step(f)
            float(loss)
            torch.cuda.synchronize()
            return (time.perf_counter() - s) / n * 1e3
        for name, (est, aug) in runs.items():
            steps(est, aug, 5)
        for _ in range(ROUNDS):
            for name, (est, aug) in runs.items():
                times[name].append(steps(est, aug, 20))
        off = np.median(times['off'])
        res[model] = {k: dict(ms=float(np.median(v)), runs=[round(x, 3) for x in v], vs_off=float(np.median(v) / off))
                      for k, v in times.items()}
    return res


def main():
    out = dict(card=card(), augment_rows=bench_rows(), vocab_sample=bench_sample())
    with tempfile.TemporaryDirectory() as tmp:
        out['train_step'] = bench_steps(tmp)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
