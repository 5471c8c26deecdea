"""Continued masked-LM pretraining of BERT on unlabelled in-domain text (Gururangan et al., ACL 2020, "Don't Stop
Pretraining"), the step before fine-tuning any BERT plugin from the result:

    python -m chinesener_b200.data.corpus --src domain.txt --out data/domain --bert_dir P --max_seq_len 128 [--whole_word]
    python -m chinesener_b200.pretrain --data_dir data/domain --pretrain_dir P --output_dir out --num_train_steps 10000
    python -m chinesener_b200.main --model_name bert_crf --pretrain_dir out ...

Dynamic (whole-word) masking is drawn on the device at every step (mlm.masked_lm); the optimizer is the BERT plugins'
AdamW recipe (train_utils.bert_train_op).  At every save: an EVAL pass over valid.nerrec with one fixed masking seed (so
every evaluation masks the same positions), the resumable `model.ckpt-<step>.npz` and `export_pretrained` into
output_dir (bert_model.ckpt + bert_config.json + vocab.txt).  A restart resumes from the latest .npz with its Adam slots
and LR schedule position.
"""
import argparse
import json
import math
import os

import numpy as np
import torch

from . import autodiff, bert, checkpoint, mlm, variables
from .data import records
from .data.tokenizer import load_vocab
from .tools import train_utils

EVAL_SEED = 0x5EED


def to_device(batch, device):
    """Host batch -> device tensors; the mask carries its host row lengths and token count (engine.Estimator.to_device),
    so the prediction budgets and the sequence pack need no device synchronisation.  word_start travels as u8."""
    out = {k: v.to(device, non_blocking=True) for k, v in batch.items() if torch.is_tensor(v)}
    lens = batch['mask'].sum(1)
    out['mask'].row_lengths = lens.numpy()
    out['mask'].total_tokens = int(lens.sum())
    if 'word_start' in out:
        out['word_start'] = out['word_start'].to(torch.uint8)
    return out


def settings(args):
    """Check the run before anything is launched -> (cfg, mask_id, max_seq_len).  ValueError for p outside (0, 1],
    max_pred < 1, records longer than the position table, a vocab.txt whose size differs from vocab_size or without
    [MASK], or V above the vocabulary kernels' limit."""
    p, k = args.masked_lm_prob, args.max_predictions_per_seq
    if not (isinstance(p, (int, float)) and 0 < p <= 1):
        raise ValueError(f"masked_lm_prob must be in (0, 1] (got {p!r})")
    if k < 1:
        raise ValueError(f"max_predictions_per_seq must be >= 1 (got {k})")
    cfg = bert.load_bert_config(args.pretrain_dir)
    V = cfg['vocab_size']
    if V > 50000:
        raise ValueError(f"vocab_size {V} is above the masked-LM kernels' limit of 50000")
    path = os.path.join(args.data_dir, 'train.nerrec')
    if not os.path.exists(path):
        raise ValueError(f"{path} not found: build it with python -m chinesener_b200.data.corpus")
    max_seq_len = records.RecordFile(path).max_seq_len
    if max_seq_len > cfg['max_position_embeddings']:
        raise ValueError(f"the records' max_seq_len {max_seq_len} is above max_position_embeddings "
                         f"{cfg['max_position_embeddings']}")
    mask_id = mlm.SYNTHETIC_MASK_ID
    if args.pretrain_dir:
        vpath = os.path.join(args.pretrain_dir, 'vocab.txt')
        if not os.path.exists(vpath):
            raise ValueError(f"{vpath} not found")
        vocab = load_vocab(vpath)
        if len(vocab) != V:
            raise ValueError(f"{vpath} holds {len(vocab)} tokens, bert_config.json says vocab_size = {V}")
        if '[MASK]' not in vocab:
            raise ValueError(f"{vpath} has no [MASK] token")
        mask_id = vocab['[MASK]']
    return cfg, mask_id, max_seq_len


def evaluate(rec, cfg, store, args, mask_id):
    """Masked-LM loss, accuracy and perplexity over every row of `rec`, masked with EVAL_SEED."""
    tot, cnt, cor = 0.0, 0, 0
    for s in range(0, len(rec), args.batch_size):
        dev = to_device(rec.batch(slice(s, s + args.batch_size), with_strings=False), store.device)
        out = mlm.masked_lm(dev, cfg, store, EVAL_SEED + s, args.masked_lm_prob, args.max_predictions_per_seq, mask_id, False)
        c = int(out.count)
        tot += float(out.loss) * c
        cnt += c
        cor += int(out.correct)
    loss = tot / cnt if cnt else float('nan')
    return {'loss': loss, 'accuracy': cor / cnt if cnt else float('nan'), 'perplexity': math.exp(loss) if cnt else float('nan'),
            'predictions': cnt}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--data_dir', required=True, help='train.nerrec / valid.nerrec of chinesener_b200.data.corpus')
    ap.add_argument('--pretrain_dir', default='', help="BERT to continue from ('': random BERT-base-Chinese)")
    ap.add_argument('--output_dir', required=True)
    ap.add_argument('--num_train_steps', type=int, default=10000)
    ap.add_argument('--batch_size', type=int, default=32)
    ap.add_argument('--lr', type=float, default=5e-5)
    ap.add_argument('--warmup_ratio', type=float, default=0.1)
    ap.add_argument('--masked_lm_prob', type=float, default=0.15)
    ap.add_argument('--max_predictions_per_seq', type=int, default=20)
    ap.add_argument('--save_steps', type=int, default=500)
    ap.add_argument('--seed', type=int, default=1234)
    ap.add_argument('--report', default='', help='JSON report path (default output_dir/pretrain_report.json)')
    args = ap.parse_args(argv)
    cfg, mask_id, _ = settings(args)
    train = records.RecordFile(os.path.join(args.data_dir, 'train.nerrec'))
    vpath = os.path.join(args.data_dir, 'valid.nerrec')
    valid = records.RecordFile(vpath) if os.path.exists(vpath) else None
    store = variables.VariableStore('cuda', seed=args.seed)
    with variables.use_store(store):
        bert.create_bert_variables(cfg, store)
        mlm.create_head_variables(cfg, store)
    last = checkpoint.latest_checkpoint(args.output_dir)
    resumed = checkpoint.restore_checkpoint(store, last) if last else 0
    report = {'settings': vars(args), 'mask_id': mask_id, 'resumed_from': resumed, 'train': [], 'valid': []}
    rng_epoch, per_epoch = -1, len(train) // args.batch_size
    if per_epoch < 1:
        raise ValueError(f"train.nerrec holds {len(train)} rows, fewer than one batch of {args.batch_size}")
    pending = []

    def save():
        for step, loss, cnt, cor in pending:
            c = int(cnt)
            report['train'].append({'step': step, 'loss': float(loss), 'accuracy': int(cor) / c if c else None})
        pending.clear()
        if valid is not None and len(valid):
            report['valid'].append(dict(evaluate(valid, cfg, store, args, mask_id), step=store.global_step))
        checkpoint.save_checkpoint(store, args.output_dir)
        mlm.export_pretrained(store, args.output_dir, args.pretrain_dir)

    order = None
    while store.global_step < args.num_train_steps:
        step = store.global_step
        epoch, i = divmod(step, per_epoch)
        if epoch != rng_epoch:
            order, rng_epoch = np.random.default_rng(args.seed + epoch).permutation(len(train)), epoch
        dev = to_device(train.batch(np.sort(order[i * args.batch_size:(i + 1) * args.batch_size]), pin_memory=True,
                                    with_strings=False), store.device)
        store.dropout_calls = 0
        with variables.use_store(store), autodiff.recording(store) as tape:
            out = mlm.masked_lm(dev, cfg, store, (args.seed * 1000003 + step) & 0xFFFFFFFFFFFFFFFF, args.masked_lm_prob,
                                args.max_predictions_per_seq, mask_id, True, tape=tape)
            tape.backward()
            train_utils.bert_train_op(out.loss, args.lr, args.num_train_steps, args.warmup_ratio, None, store=store)
        pending.append((step, out.loss, out.count, out.correct))
        if store.global_step % args.save_steps == 0 or store.global_step == args.num_train_steps:
            save()
    report['global_step'] = store.global_step
    if report['valid']:
        report['final_valid_perplexity'] = report['valid'][-1]['perplexity']
    path = args.report or os.path.join(args.output_dir, 'pretrain_report.json')
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, 'w') as f:
        json.dump(report, f, indent=1)
    return report


if __name__ == '__main__':
    main()
