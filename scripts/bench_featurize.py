"""Raw text -> features on the device (ner_featurize_wordpiece / ner_featurize_chars) against the host featuriser.

One run: first checks that both featurisers give equal features on the timed sentences, and that
InferHelper.infer_batch gives the same entities on both paths; then times
  - the featurise kernels alone (CUDA events) at B = 64 and B = 16384 MSRA-shaped sentences, in characters/s;
  - InferHelper.infer_batch end to end, host featuriser against device featuriser, alternated, for bert_bilstm_crf
    (BERT-base shaped encoder, random weights) and bilstm_crf at B = 64;
  - Estimator.predict_device on a pre-built device batch of the same sentences: the ceiling infer_batch approaches.
Prints the card's name and power limit beside the numbers, and one JSON line at the end.

    python scripts/bench_featurize.py [--reps 20]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from chinesener_b200 import engine, synthetic                                       # noqa: E402
from chinesener_b200.data.base_preprocess import BasicProc, features_to_batch       # noqa: E402
from chinesener_b200.data.device_featurize import DeviceFeaturizer                  # noqa: E402
from chinesener_b200.data.tokenizer import FullTokenizer, TokenizerAdapter, TokenizerBert, TokenizerGiga  # noqa: E402
from chinesener_b200.inference import TAG2IDX, InferHelper                          # noqa: E402

L = 128
CJK = [chr(0x4E00 + i) for i in range(20000)]


def sentences(n, seed):
    """MSRA-shaped: about 46 characters, mostly CJK, some digits, punctuation and Latin letters."""
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        s = []
        for _ in range(max(3, int(rng.gauss(46, 20)))):
            r = rng.random()
            s.append(CJK[rng.randrange(3000)] if r < 0.9 else str(rng.randrange(10)) if r < 0.95
                     else rng.choice('，。、abcXYZ '))
        out.append(''.join(s))
    return out


def tokenizers():
    vocab = (['[PAD]', '[UNK]', '[CLS]', '[SEP]', '[MASK]'] + CJK + [str(d) for d in range(10)]
             + list('abcdefghijklmnopqrstuvwxyz，。、；：“”（）') + ['##' + str(d) for d in range(10)]
             + ['##' + c for c in 'abcdefghijklmnopqrstuvwxyz'])
    return FullTokenizer({t: i for i, t in enumerate(vocab)}), TokenizerAdapter(CJK[:6000] + list('0123456789，。、abc'))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, check=True).stdout.strip().splitlines()[0]
        return q
    except (OSError, subprocess.CalledProcessError, IndexError):
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def check_features(tok, kind, texts):
    want = features_to_batch([BasicProc(kind, L, TAG2IDX, tok).build_seq_feature(t) for t in texts])
    got = DeviceFeaturizer(tok, L).featurize(texts)
    for k in ('token_ids', 'mask', 'segment_ids', 'seq_len'):
        assert torch.equal(got[k].cpu(), want[k]), (kind, k)


def time_kernel(tok, texts, reps):
    f = DeviceFeaturizer(tok, L)
    f.featurize(texts)
    chars = sum(len(t) for t in texts)
    from chinesener_b200 import ops
    B = len(texts)
    data = [t.encode('utf-8', 'surrogatepass') for t in texts]
    offsets = np.zeros(B + 1, dtype=np.int64)
    np.cumsum([len(d) for d in data], out=offsets[1:])
    host = torch.from_numpy(np.concatenate([offsets.view(np.uint8), np.frombuffer(b''.join(data), np.uint8)])).pin_memory()
    dev = host.cuda()
    out = {k: torch.empty((B, L), dtype=torch.int32, device='cuda') for k in ('token_ids', 'mask', 'segment_ids', 'unk_cursor')}
    out['seq_len'] = torch.empty((B,), dtype=torch.int32, device='cuda')
    fn = ops.featurize_wordpiece if f.wordpiece else ops.featurize_chars
    run = lambda: fn(dev, host, B, L, f.uni, f.vocab, f.max_piece, f.lower, f.special, out)   # noqa: E731
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    e1.synchronize()
    sec = e0.elapsed_time(e1) / 1e3 / reps
    return {'B': B, 'us_per_call': sec * 1e6, 'chars_per_s': chars / sec, 'sentences_per_s': B / sec}


def helper_for(model, tok, tmp):
    if 'bert' in model:
        cfg = {'vocab_size': max(tok.vocab.values()) + 1, 'hidden_size': 768, 'num_hidden_layers': 12,
               'num_attention_heads': 12, 'intermediate_size': 3072, 'max_position_embeddings': 512,
               'type_vocab_size': 2, 'initializer_range': 0.02}
        with open(os.path.join(tmp, 'bert_config.json'), 'w') as fh:
            json.dump(cfg, fh)
        params = dict(synthetic.data_params(L), pretrain_dir=tmp)
    else:
        params = dict(synthetic.data_params(L), embedding=np.random.default_rng(0).standard_normal(
            (max(tok.vocab2idx.values()) + 1, 50)).astype(np.float32))
    est = engine.Estimator(model, params)
    return InferHelper(L, TAG2IDX, model, tok, estimator=est)


def host_infer_batch(helper, texts):
    """infer_batch as it featurises on the host (make_feature + features_to_batch)."""
    from chinesener_b200.tools.infer_utils import extract_entity_device
    feats = [dict(helper.make_feature(t)) for t in texts]
    pred = helper.estimator.predict_device(helper.estimator.to_device(features_to_batch(feats, pin_memory=True)))
    return extract_entity_device([f['tokens'] for f in feats], pred, helper.idx2tag)


def time_infer(helper, texts, reps):
    assert [dict(e) for e in helper.infer_batch(texts)] == [dict(e) for e in host_infer_batch(helper, texts)]
    feats = features_to_batch([dict(helper.make_feature(t)) for t in texts], pin_memory=True)
    t = {'host': [], 'device': [], 'predict': []}
    for _ in range(reps):
        for name, fn in (('host', lambda: host_infer_batch(helper, texts)), ('device', lambda: helper.infer_batch(texts)),
                         ('predict', lambda: helper.estimator.predict_device(helper.estimator.to_device(feats)))):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            t[name].append(time.perf_counter() - t0)
    B = len(texts)
    return {k: {'median_ms': 1e3 * float(np.median(v)), 'sentences_per_s': B / float(np.median(v))} for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_featurize measures on the GPU'
    wp, ch = tokenizers()
    gpu = card()
    print('card:', gpu, flush=True)
    res = {'card': gpu, 'L': L}
    small, big = sentences(64, 0), sentences(16384, 1)
    for tok, kind in ((wp, TokenizerBert), (ch, TokenizerGiga)):
        check_features(tok, kind, small + big[:2048])
    for tok, name in ((wp, 'wordpiece'), (ch, 'chars')):
        for texts in (small, big):
            r = time_kernel(tok, texts, args.reps)
            res[f'kernel_{name}_B{len(texts)}'] = r
            print(f'kernel {name:9s} B={len(texts):5d}: {r["us_per_call"]:9.1f} us/call  {r["chars_per_s"] / 1e6:8.1f} M chars/s',
                  flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        for model, tok in (('bert_bilstm_crf', wp), ('bilstm_crf', ch)):
            helper = helper_for(model, tok, tmp)
            r = time_infer(helper, small, args.reps)
            res[f'infer_batch_{model}_B64'] = r
            print(f'{model:16s} B=64: host featuriser {r["host"]["sentences_per_s"]:8.0f}/s, device featuriser '
                  f'{r["device"]["sentences_per_s"]:8.0f}/s, predict_device ceiling {r["predict"]["sentences_per_s"]:8.0f}/s '
                  f'(device / ceiling = {r["device"]["sentences_per_s"] / r["predict"]["sentences_per_s"]:.2f})', flush=True)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
