"""Document mode of the BERT plugins without a GPU: the plain restatement of the window plan (oracle/windows.py) against
the definition, the shared window-count formula, and the parameter checks that refuse a batch before any launch."""
import json

import numpy as np
import pytest
import torch

from chinesener_b200 import engine, main, synthetic, windows
from oracle import windows as ow

SETTINGS = [(3, 1), (128, 1), (128, 37), (128, 126), (512, 255), (512, 510)]


@pytest.mark.parametrize("W,S", SETTINGS)
def test_plan_restatement(W, S):
    C = W - 2
    for n in range(0, 1301):
        pos = ow.window_positions(n, W, S)
        assert len(pos) == windows.document_windows(n, W, S)
        if n == 0:
            continue
        assert pos.shape[1] == (W if n > W else n)
        own = np.array(ow.owners(n, W, S))
        assert own.shape == (n, 2)
        k, p = own[:, 0], own[:, 1]
        assert (pos[k, p] == np.arange(n)).all()            # exactly one owner per doc position, and it holds it
        if n <= W:
            continue
        assert (pos[:, 0] == 0).all() and (pos[:, -1] == n - 1).all()
        assert own[0].tolist() == [0, 0] and own[-1].tolist() == [len(pos) - 1, W - 1]
        # every (window, content row): the doc content index it holds and that index's context there
        a = pos[:, 1] - 1
        assert (np.diff(a) > 0).all() and a[0] == 0 and a[-1] == n - 2 - C
        rows = np.arange(1, C + 1)
        c_all = (a[:, None] + rows - 1).ravel()
        score = np.broadcast_to(np.minimum(rows - 1, C - rows), (len(a), C)).ravel()
        k_all = np.repeat(np.arange(len(a)), C)
        best = np.full(n - 2, -1)
        np.maximum.at(best, c_all, score)
        first = np.full(n - 2, len(a))
        hit = score == best[c_all]
        np.minimum.at(first, c_all[hit], k_all[hit])
        kc, pc = k[1:-1], p[1:-1]
        assert (np.minimum(pc - 1, C - pc) == best).all()     # no window holding c gives it more context
        assert (kc == first).all()                            # ties go to the lowest window


@pytest.mark.parametrize("W,S", SETTINGS)
def test_window_counts_match_the_restated_plan(W, S):
    rng = np.random.default_rng(W * 1000 + S)
    lengths = np.concatenate([[0, 1, 2, W, W + 1, 1300], rng.integers(0, 1301, size=20)])
    pl = ow.plan(lengths, W, S)
    NW, n_win = windows.window_counts(lengths, W, S)
    assert NW == len(pl['doc']) == pl['pos'].shape[0]
    assert n_win == int((pl['pos'] >= 0).sum())
    assert len(pl['src_packed']) == len(pl['src_padded']) == int(lengths.sum())
    assert pl['src_packed'].max() < n_win and pl['src_padded'].max() < NW * W


def test_window_settings():
    assert windows.settings(None, None, 512) == (512, 255)
    assert windows.settings(128, None, 512) == (128, 63)
    assert windows.settings(3, 1, 512) == (3, 1)
    for w, s in [(2, None), (513, None), (0, None), (128, 0), (128, 127), (3, 2), (512, -1)]:
        with pytest.raises(ValueError):
            windows.settings(w, s, 512)


def test_batch_checks():
    windows.check_batch('bert_crf', 512, 512)
    windows.check_batch('bert_cnn_crf', 512, 512)               # fits one window: nothing to refuse
    windows.check_batch('bert_bilstm_crf', 4095, 512)
    with pytest.raises(ValueError, match="4095"):
        windows.check_batch('bert_bilstm_crf', 4096, 512)
    for name in ('bert_cnn_crf', 'bert_ce', 'bert_dice', 'bert_mrc'):
        with pytest.raises(ValueError, match=name):
            windows.check_batch(name, 513, 512)


def _estimator(tmp_path, model, L, **extra):
    cfg = {'vocab_size': 300, 'hidden_size': 128, 'num_hidden_layers': 1, 'num_attention_heads': 2,
           'intermediate_size': 512, 'max_position_embeddings': 512, 'type_vocab_size': 2}
    (tmp_path / "bert_config.json").write_text(json.dumps(cfg))
    params = dict(synthetic.data_params(L), pretrain_dir=str(tmp_path), **extra)
    return engine.Estimator(model, params, device='cpu')


@pytest.mark.parametrize("extra", [dict(bert_window=2), dict(bert_window=600), dict(bert_window=128, bert_window_stride=127),
                                   dict(bert_window_stride=0)])
def test_estimator_refuses_bad_window_parameters(tmp_path, extra):
    """The checks run before build_graph, so they raise on the host with CPU features."""
    est = _estimator(tmp_path, 'bert_bilstm_crf', 64, **extra)
    feats = synthetic.msra_batch(2, 64, vocab=300, seed=1)
    with pytest.raises(ValueError, match="bert_window"):
        est.forward_device(feats)
    with pytest.raises(ValueError, match="bert_window"):
        est.train_step(feats)


@pytest.mark.parametrize("model", ['bert_cnn_crf', 'bert_ce', 'bert_dice', 'bert_mrc', 'bert_bilstm_crf'])
def test_estimator_refuses_documents_it_cannot_tag(tmp_path, model):
    L = 4096 if model == 'bert_bilstm_crf' else 700
    est = _estimator(tmp_path, model, L)
    feats = synthetic.msra_batch(2, L, vocab=300, seed=1)
    with pytest.raises(ValueError, match="4095" if model == 'bert_bilstm_crf' else model):
        est.forward_device(feats)
    with pytest.raises(ValueError, match="4095" if model == 'bert_bilstm_crf' else model):
        est.train_step(feats)


def test_estimator_attaches_host_lengths():
    est = engine.Estimator('bilstm_crf', dict(synthetic.data_params(16)), device='cpu')
    feats = synthetic.msra_batch(3, 16, vocab=300, seed=2)
    feats['mask'][1, 5:] = 0
    feats['mask'][2, :] = 0
    m = est.stack_to_device([feats, feats])['mask']
    assert m.row_lengths.tolist() == [16, 5, 0] * 2
    assert m.total_tokens == 42 and m.nonempty_rows == 4


def test_driver_window_flags():
    args = main.build_parser().parse_args(['--model_name', 'bert_bilstm_crf', '--bert_window', '256',
                                           '--bert_window_stride', '100'])
    params = {}
    main._window_params(params, args)
    assert params == {'bert_window': 256, 'bert_window_stride': 100}
    params = {}
    main._window_params(params, main.build_parser().parse_args(['--model_name', 'bert_crf']))
    assert params == {}
