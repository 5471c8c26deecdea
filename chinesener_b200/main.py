# -*-coding:utf-8 -*-
"""Train / evaluate / predict driver with the reference's command line (reference main.py:14-140).

    python -m chinesener_b200.main --model_name bilstm_crf --data msra [--clear_model 1] [--data_dir datasets/msra]

What `singletask_train` does, in the reference's order (main.py:14-62):
  * TRAIN_PARAMS of the plugin + the dataset's params (NerDataset -> label_size, max_seq_len, step_per_epoch,
    num_train_steps, embedding ...);
  * an Estimator over `./checkpoint/ner_<data>_<model>`, warm-started from its latest checkpoint (tools/utils.py:52-66);
  * tf.estimator.train_and_evaluate: TRAIN over shuffle(64).repeat(epoch_size).batch(batch_size); a checkpoint every
    RUN_CONFIG['save_steps'] steps, each followed by an EVAL pass over the `valid` split; the
    stop_if_no_decrease_hook(metric 'loss', max_steps_without_decrease = step_per_epoch * early_stop_ratio) ends
    training when the best eval loss is that many steps old;
  * PREDICT over the `predict` split with the LAST checkpoint's weights; the list of per-sentence dicts
    {'pred_ids' int32[L], 'label_ids' int32[L], 'tokens' bytes[L]} is pickled to `<data_dir>/<model>_predict.pkl`
    (main.py:52-55) — the file evaluation.py scores.
The Estimator's own evaluation cadence is time based (throttle_secs=60, the hook polls every 60 s); on an H100 a whole
epoch takes seconds, so the cadence here is the step-based one those timers converge to on the reference's hardware:
evaluate at every checkpoint.  Exporting a SavedModel (main.py:57-60) has no counterpart: the in-process InferHelper
serves from the checkpoint.
"""
import argparse
import json
import os
import pickle
import shutil
import time

import numpy as np

RUN_CONFIG = {'summary_steps': 10, 'log_steps': 100, 'save_steps': 500, 'keep_checkpoint_max': 3}     # config.py:19-30


def clear_model(model_dir):
    """tools/utils.py:17-23"""
    try:
        shutil.rmtree(model_dir)
    except Exception as e:
        print('Error! {} occured at model cleaning'.format(e))
    else:
        print('{} model cleaned'.format(model_dir))


def evaluate(estimator, input_fn):
    """EVAL pass: mean of the per-batch losses (tf.estimator averages the `loss` metric over batches) + tag accuracy over
    the real tokens (tools/train_utils.py:107-127 weights by the non-[PAD] mask)."""
    losses, right, total = [], 0, 0
    for feats in input_fn():
        out = estimator.evaluate(feats)
        losses.append(out['loss'])
        lab, pred = feats['label_ids'].numpy(), out['pred_ids'].numpy()
        real = lab > 0
        right += int(((lab == pred) & real).sum())
        total += int(real.sum())
    return {'loss': float(np.mean(losses)), 'accuracy': right / max(total, 1), 'batches': len(losses)}


def train_and_evaluate(estimator, input_pipe, model_dir, run_config=RUN_CONFIG, log=print, max_steps=None):
    """-> history dict.  See the module docstring for the correspondence with tf.estimator.train_and_evaluate."""
    from . import checkpoint
    p = estimator.params
    max_no_decrease = int(p['step_per_epoch'] * p['early_stop_ratio'])
    evals, best = [], (None, None)               # best = (loss, step)
    t0 = time.time()
    loss_sum, loss_n = None, 0
    stopped = 'input exhausted'
    store = estimator.store

    def checkpoint_and_eval():
        nonlocal best
        path = checkpoint.save_checkpoint(store, model_dir, run_config['keep_checkpoint_max'])
        ev = evaluate(estimator, input_pipe.build_input_fn('valid', is_predict=True, with_strings=False))
        ev.update(step=store.global_step, seconds=round(time.time() - t0, 1))
        evals.append(ev)
        if best[0] is None or ev['loss'] < best[0]:
            best = (ev['loss'], store.global_step)
        log('eval @ step {step}: loss = {loss:.4f} accuracy = {accuracy:.4f} ({seconds}s) -> {0}'.format(os.path.basename(path), **ev))
        # stop_if_no_decrease_hook: the best (lowest) eval loss is at least max_steps_without_decrease steps old
        return store.global_step - best[1] >= max_no_decrease

    batches = input_pipe.build_input_fn('train')()
    if p.get('augment'):
        from . import augment
        aug = augment.build(p, p['idx2tag'], input_pipe.file_path('train'), estimator.device, estimator.model_name)
        batches = aug.pipeline(batches, store.global_step, estimator.to_device)
    for feats in batches:
        loss = estimator.train_step(feats)
        loss_sum = loss.detach() if loss_sum is None else loss_sum + loss.detach()
        loss_n += 1
        step = store.global_step
        if step % run_config['log_steps'] == 0:
            log('step {}: loss = {:.4f} ({:.1f}s)'.format(step, float(loss_sum) / loss_n, time.time() - t0))
            loss_sum, loss_n = None, 0
        if step % run_config['save_steps'] == 0 and checkpoint_and_eval():
            stopped = 'no decrease of the eval loss for {} steps (best {:.4f} @ {})'.format(max_no_decrease, *best)
            break
        if max_steps is not None and step >= max_steps:
            stopped = 'max_steps'
            break
    if not evals or evals[-1]['step'] != store.global_step:
        checkpoint_and_eval()                     # the Estimator always saves and evaluates at the end of training
    log('training stopped at step {}: {}'.format(store.global_step, stopped))
    return {'evals': evals, 'best_eval_loss': best[0], 'best_eval_step': best[1], 'final_step': store.global_step,
            'stopped': stopped, 'train_seconds': round(time.time() - t0, 1)}


def predict_to_list(estimator, input_fn):
    """estimator.predict(input_fn) of the reference: one dict per SENTENCE, numpy values as tf.estimator yields them."""
    out = []
    for res in estimator.predict_sentences(input_fn()):
        out.append({'pred_ids': res['pred_ids'].astype(np.int32), 'label_ids': res['label_ids'].astype(np.int32),
                    'tokens': np.array([t.encode('utf-8') if isinstance(t, str) else t for t in res['tokens']], dtype=object)})
    return out


def predict_nbest_to_list(estimator, input_fn):
    """predict_to_list with params['crf_nbest'] > 1, batch by batch through Estimator.predict: each sentence's dict also
    holds its candidate paths, best first, as nbest_ids int32 [count, L], nbest_scores f32 [count] and nbest_probs f32
    [count].  -> (that list, seq_len of every sentence)."""
    out, lens = [], []
    for feats in input_fn():
        res = estimator.predict(feats)
        pred, lab, tok = res['pred_ids'].numpy(), feats['label_ids'].numpy(), feats['tokens']
        L = pred.shape[1]
        lens.extend(int(n) for n in feats['seq_len'])
        for b, paths in enumerate(res['pred_nbest']):
            out.append({'pred_ids': pred[b].astype(np.int32), 'label_ids': lab[b].astype(np.int32),
                        'tokens': np.array([t.encode('utf-8') if isinstance(t, str) else t for t in tok[b]], dtype=object),
                        'nbest_ids': np.array([p[0] for p in paths], dtype=np.int32).reshape(len(paths), L),
                        'nbest_scores': np.array([p[1] for p in paths], dtype=np.float32),
                        'nbest_probs': np.array([p[2] for p in paths], dtype=np.float32)})
    return out, lens


def exact_match_rates(prediction, lens):
    """-> (exact_match_at_1, exact_match_at_n): the share of sentences whose gold label_ids over t < seq_len equal the
    best candidate path / one of the candidate paths."""
    at1 = atn = 0
    for p, n in zip(prediction, lens):
        hits = [np.array_equal(c[:n], p['label_ids'][:n]) for c in p['nbest_ids']] if n > 0 else []
        at1 += bool(hits and hits[0])
        atn += any(hits)
    total = max(len(prediction), 1)
    return at1 / total, atn / total


def singletask_train(args):
    from . import checkpoint, engine
    from .data.records import NerDataset, RecordFile
    model_name = args.rename if args.rename else args.model_name
    model_dir = os.path.join(args.checkpoint_root, 'ner_{}_{}'.format(args.data, model_name))
    data_dir = args.data_dir or './data/{}'.format(args.data)
    if args.clear_model:
        clear_model(model_dir)

    _, TRAIN_PARAMS = engine.load_plugin(args.model_name)
    TRAIN_PARAMS = dict(TRAIN_PARAMS)
    if args.epoch_size:
        TRAIN_PARAMS['epoch_size'] = args.epoch_size
    if args.pretrain_dir:
        TRAIN_PARAMS['pretrain_dir'] = args.pretrain_dir
    if args.batch_size:
        TRAIN_PARAMS['batch_size'] = args.batch_size
    _window_params(TRAIN_PARAMS, args)
    if args.crf_nbest != 1:
        TRAIN_PARAMS['crf_nbest'] = args.crf_nbest
    _augment_params(TRAIN_PARAMS, args)
    teacher_ck = None
    if not args.teacher_model and (args.teacher_dir or args.teacher_pretrain_dir):
        raise ValueError('--teacher_dir / --teacher_pretrain_dir need --teacher_model')
    if args.teacher_model:
        # a missing teacher checkpoint is an error before anything is built, not a randomly initialised teacher
        teacher_ck = checkpoint.latest_checkpoint(args.teacher_dir) if args.teacher_dir else None
        if teacher_ck is None:
            raise ValueError('--teacher_model {} needs --teacher_dir with a checkpoint (found none in {!r})'.format(
                args.teacher_model, args.teacher_dir))
        TRAIN_PARAMS['distill_alpha'] = args.distill_alpha
        TRAIN_PARAMS['distill_temperature'] = args.distill_temperature
    # with a teacher, the dataset is the teacher's: its features are a superset of the student's
    input_pipe = NerDataset(data_dir, TRAIN_PARAMS['batch_size'], TRAIN_PARAMS['epoch_size'],
                            args.teacher_model or model_name, seed=args.seed)
    TRAIN_PARAMS.update(input_pipe.params)       # label_size, max_seq_len, num_train_steps ... (main.py:25)
    print('=' * 10 + 'TRAIN PARAMS' + '=' * 10)
    print(dict((i, j) for i, j in TRAIN_PARAMS.items() if ('emb' not in i) and ('vocab' not in i)))
    print('=' * 10 + 'RUN PARAMS' + '=' * 10)
    print(RUN_CONFIG)

    teacher = None
    if teacher_ck is not None:
        teacher_params = dict(engine.load_plugin(args.teacher_model)[1])
        teacher_params.update(input_pipe.params)
        if args.teacher_pretrain_dir or args.pretrain_dir:
            teacher_params['pretrain_dir'] = args.teacher_pretrain_dir or args.pretrain_dir
        _window_params(teacher_params, args)     # the teacher encodes the same (document-length) batches as the student
        teacher = engine.Estimator(args.teacher_model, teacher_params)
        teacher.document_window()                # ValueError before training: a window the teacher's BERT cannot take
    estimator = engine.Estimator(args.model_name, TRAIN_PARAMS, teacher=teacher)   # ValueError for a pair it cannot distill
    nbest = estimator.crf_nbest()                # ValueError before training: out of range, or a plugin without one CRF
    if teacher is not None:
        first = next(iter(input_pipe.build_input_fn('valid', is_predict=True, with_strings=False)()))
        teacher.evaluate(first)                  # creates the teacher's variables, then the checkpoint overwrites them
        print('teacher {} from {} (step {})'.format(args.teacher_model, teacher_ck,
                                                    checkpoint.restore_checkpoint(teacher.store, teacher_ck)))
    estimator.store.gen.manual_seed(args.seed)
    warm = checkpoint.latest_checkpoint(model_dir)
    if warm:
        # variables exist only after the first build_graph: run one EVAL batch, then overwrite them from the checkpoint
        first = next(iter(input_pipe.build_input_fn('valid', is_predict=True, with_strings=False)()))
        estimator.evaluate(first)
        print('warm start from {} (step {})'.format(warm, checkpoint.restore_checkpoint(estimator.store, warm)))

    history = None
    if not args.predict_only:
        history = train_and_evaluate(estimator, input_pipe, model_dir, max_steps=args.max_steps)

    if nbest > 1:
        prediction, lens = predict_nbest_to_list(estimator, input_pipe.build_input_fn('predict', is_predict=True))
    else:
        prediction = predict_to_list(estimator, input_pipe.build_input_fn('predict', is_predict=True))
    out_pkl = os.path.join(data_dir, '{}_predict.pkl'.format(model_name))
    with open(out_pkl, 'wb') as f:
        pickle.dump(prediction, f)
    print('{} sentences -> {}'.format(len(prediction), out_pkl))

    summary = {'model': model_name, 'data': args.data, 'history': history, 'n_predict': len(prediction), 'seed': args.seed}
    if teacher is not None:
        summary['teacher'] = args.teacher_model
        summary['distill_alpha'], summary['distill_temperature'] = estimator.distill_settings()
    if nbest > 1:
        summary['crf_nbest'] = nbest
        summary['exact_match_at_1'], summary['exact_match_at_n'] = exact_match_rates(prediction, lens)
        print('exact match of the gold tags: {:.4f} at 1, {:.4f} within {} paths'.format(
            summary['exact_match_at_1'], summary['exact_match_at_n'], nbest))
    if 'label_mask' in RecordFile(input_pipe.file_path('predict')).names():
        # partially labelled: the gold entities are unknown, only the labelled positions (label_id > 0) can be scored
        real = [(int(a), int(b)) for i in prediction for a, b in zip(i['label_ids'], i['pred_ids']) if a > 0]
        summary['tag_accuracy'] = sum(a == b for a, b in real) / max(len(real), 1)
        print('entity report skipped: the predict split is partially labelled, so its gold entities are unknown; '
              'tag accuracy over the labelled positions = {:.4f}'.format(summary['tag_accuracy']))
    else:
        from .evaluation import SingleEval
        tag_rep, ent_rep = SingleEval(prediction, TRAIN_PARAMS['idx2tag']).gen_report()
        summary.update({'entity_micro_f1': ent_rep['micro avg']['f1-score'],
                        'entity_weighted_f1': ent_rep['weighted avg']['f1-score'],
                        'entity_report': ent_rep, 'tag_weighted_f1': tag_rep['weighted avg']['f1-score']})
        print('entity micro-F1 = {:.4f}  weighted-F1 = {:.4f}'.format(summary['entity_micro_f1'], summary['entity_weighted_f1']))
    if args.report:
        with open(args.report, 'w') as f:
            json.dump(summary, f, indent=1, default=float)
    return summary


def multitask_train(args):
    """reference main.py:65-118: `--data a,b` with an mtl / adv plugin.  One Estimator over
    `./checkpoint/ner_<a_b>_<model>`, TRAIN / EVAL over the sample-by-sample mix of the datasets (MultiDataset), then one
    PREDICT pass per dataset with that dataset's task id -> `<data_root>/<data>/<model>_<a_b>_predict.pkl`."""
    from . import checkpoint, engine
    from .data.records import MultiDataset
    model_name = args.rename if args.rename else args.model_name
    data_list = args.data.split(',')
    joined = '_'.join(data_list)
    if args.crf_nbest != 1:
        raise ValueError('--crf_nbest is for single-task plugins: the multi-task pred_ids are a per-task selection of '
                         'several CRF decodes')
    if args.augment:
        raise ValueError('--augment is for single-task plugins: a multi-task batch mixes tag sets')
    model_dir = os.path.join(args.checkpoint_root, 'ner_{}_{}'.format(joined, model_name))
    data_root = args.data_dir or './data'
    if args.clear_model:
        clear_model(model_dir)

    _, TRAIN_PARAMS = engine.load_plugin(args.model_name)
    TRAIN_PARAMS = dict(TRAIN_PARAMS)
    if args.epoch_size:
        TRAIN_PARAMS['epoch_size'] = args.epoch_size
    if args.pretrain_dir:
        TRAIN_PARAMS['pretrain_dir'] = args.pretrain_dir
    if args.batch_size:
        TRAIN_PARAMS['batch_size'] = args.batch_size
    _window_params(TRAIN_PARAMS, args)
    input_pipe = MultiDataset(data_root, data_list, TRAIN_PARAMS['batch_size'], TRAIN_PARAMS['epoch_size'], model_name, seed=args.seed)
    TRAIN_PARAMS.update(input_pipe.params)       # per-dataset params, task_list, step_per_epoch, num_train_steps, max_seq_len
    print('=' * 10 + 'TRAIN PARAMS' + '=' * 10)
    print(dict((i, j) for i, j in TRAIN_PARAMS.items() if i not in data_list))
    print('=' * 10 + 'RUN PARAMS' + '=' * 10)
    print(RUN_CONFIG)

    estimator = engine.Estimator(args.model_name, TRAIN_PARAMS)
    estimator.store.gen.manual_seed(args.seed)
    warm = checkpoint.latest_checkpoint(model_dir)
    if warm:
        first = next(iter(input_pipe.build_input_fn('valid', is_predict=True)()))
        estimator.evaluate(first)
        print('warm start from {} (step {})'.format(warm, checkpoint.restore_checkpoint(estimator.store, warm)))

    history = None
    if not args.predict_only:
        history = train_and_evaluate(estimator, input_pipe, model_dir, max_steps=args.max_steps)

    summary = {'model': model_name, 'data': data_list, 'history': history, 'seed': args.seed, 'tasks': {}}
    for data in data_list:
        print('Prediction for {}'.format(data))
        prediction = predict_to_list(estimator, input_pipe.build_predict_fn(data))
        out_pkl = os.path.join(data_root, data, '{}_{}_predict.pkl'.format(model_name, joined))
        with open(out_pkl, 'wb') as f:
            pickle.dump(prediction, f)
        # the entity report of evaluation.py is NER specific (a B/I/E/S segmentation tag has no entity type): tag accuracy here
        real = [(int(a), int(b)) for i in prediction for a, b in zip(i['label_ids'], i['pred_ids']) if a > 0]
        acc = sum(a == b for a, b in real) / max(len(real), 1)
        summary['tasks'][data] = {'n_predict': len(prediction), 'file': out_pkl, 'tag_accuracy': acc}
        print('{} sentences -> {} (tag accuracy {:.4f})'.format(len(prediction), out_pkl, acc))
    if args.report:
        with open(args.report, 'w') as f:
            json.dump(summary, f, indent=1, default=float)
    return summary


def build_parser():
    parser = argparse.ArgumentParser()
    # the reference's flags (main.py:121-136); argparse accepts unambiguous prefixes, so `--model` works as it does there
    parser.add_argument('--model_name', type=str, help='model_name[bert_bilstm_crf, bert_crf, bilstm_crf ...]', required=True)
    parser.add_argument('--clear_model', type=int, help='Whether to clear existing model', required=False, default=0)
    parser.add_argument('--data', type=str, help='which data to use[msra, people_daily]', required=False, default='msra')
    parser.add_argument('--gpu', type=int, help='kept for compatibility: the sm_90a path always runs on the GPU', required=False, default=1)
    parser.add_argument('--device', type=int, help='which gpu to use', required=False, default=-1)
    parser.add_argument('--rename', type=str, help='Allow rename model with special parameter', required=False, default='')
    parser.add_argument('--export_only', type=int, help='kept for compatibility (no SavedModel export: InferHelper serves in-process)',
                        required=False, default=0)
    # additions
    parser.add_argument('--data_dir', type=str, default='', help='directory of the .nerrec files (default ./data/<data>); with --data a,b: the root '
                        'holding one directory per dataset (default ./data)')
    parser.add_argument('--checkpoint_root', type=str, default='./checkpoint')
    parser.add_argument('--predict_only', type=int, default=0)
    parser.add_argument('--epoch_size', type=int, default=0, help='override TRAIN_PARAMS["epoch_size"]')
    parser.add_argument('--pretrain_dir', type=str, default='', help='override TRAIN_PARAMS["pretrain_dir"] (bert_config.json [+ checkpoint])')
    parser.add_argument('--batch_size', type=int, default=0, help='override TRAIN_PARAMS["batch_size"]')
    parser.add_argument('--max_steps', type=int, default=None)
    parser.add_argument('--seed', type=int, default=1234)
    parser.add_argument('--report', type=str, default='', help='write a JSON summary (eval history + test F1) here')
    parser.add_argument('--bert_window', type=int, default=0, help='override params["bert_window"]: BERT plugins encode '
                        'longer batches as overlapping windows of this many tokens (default max_position_embeddings)')
    parser.add_argument('--bert_window_stride', type=int, default=0, help='override params["bert_window_stride"]: content '
                        'tokens between window starts (default (bert_window - 2) // 2)')
    parser.add_argument('--crf_nbest', type=int, default=1, help='CRF plugins: decode the N best tag paths (1..16) at '
                        'PREDICT; the pickle gains nbest_ids / nbest_scores / nbest_probs and the summary exact_match_at_1 / '
                        'exact_match_at_n')
    parser.add_argument('--teacher_model', type=str, default='', help='distil from this CRF plugin (a trained teacher); '
                        'the dataset is opened by its name')
    parser.add_argument('--teacher_dir', type=str, default='', help="the teacher's checkpoint directory (latest checkpoint)")
    parser.add_argument('--teacher_pretrain_dir', type=str, default='', help="the teacher's bert_config.json directory "
                        '(default --pretrain_dir)')
    parser.add_argument('--distill_alpha', type=float, default=0.5, help='weight of the distillation term, in (0, 1]')
    parser.add_argument('--distill_temperature', type=float, default=1.0, help='temperature of the distillation term, > 0')
    parser.add_argument('--augment', type=str, default='', help='augment every TRAIN batch on the GPU: op=p[,op=p ...] '
                        'with op in mr (mention replacement), lwtr (label-wise token replacement), sis (shuffle within '
                        'segments), mlm (masked-LM replacement), e.g. mr=0.3,lwtr=0.3,sis=0.3,mlm=0.15')
    parser.add_argument('--augment_rows', type=float, default=None, help='share of rows augmented at all (default 0.5)')
    parser.add_argument('--augment_mlm_dir', type=str, default='', help='BERT with its masked-LM head for mlm (default '
                        '--pretrain_dir)')
    parser.add_argument('--augment_mlm_temperature', type=float, default=None, help='sampling temperature of mlm '
                        '(default 1)')
    return parser


def _augment_params(params, args):
    """--augment* over the params (read by augment.settings); nothing is set without --augment."""
    if not args.augment:
        return
    from .augment import parse_augment
    params['augment'] = parse_augment(args.augment)
    params['augment_seed'] = args.seed
    if args.augment_rows is not None:
        params['augment_rows'] = args.augment_rows
    if args.augment_mlm_dir:
        params['augment_mlm_dir'] = args.augment_mlm_dir
    if args.augment_mlm_temperature is not None:
        params['augment_mlm_temperature'] = args.augment_mlm_temperature


def _window_params(params, args):
    """--bert_window / --bert_window_stride over the params (read with params.get by the BERT plugins' document mode)."""
    for k in ('bert_window', 'bert_window_stride'):
        if getattr(args, k, 0):
            params[k] = getattr(args, k)


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.device >= 0:
        os.environ['CUDA_VISIBLE_DEVICES'] = '{}'.format(args.device)
    if len(args.data.split(',')) > 1:
        if args.teacher_model or args.teacher_dir:
            raise ValueError('multi-task training (--data a,b) cannot distil from a teacher')
        return multitask_train(args)
    return singletask_train(args)


if __name__ == '__main__':
    main()
