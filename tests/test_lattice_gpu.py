# -*-coding:utf-8 -*-
"""GPU: the Lattice LSTM recurrence (ner_lattice_recurrence / _bwd) against the float64 CPU restatement, the layer's
gradients against its autograd, bit-identical repeats, and the lattice_lstm_crf plugin (PREDICT / EVAL, TRAIN,
InferHelper, checkpoint round trip)."""
import numpy as np
import pytest
import torch

from chinesener_b200 import autodiff, checkpoint, engine, ops, synthetic, variables
from chinesener_b200.tools import layer
from oracle import crf as ocrf, crf_torch

import _lattice_oracle as olat
from test_word_enhance_host import write_vec

pytestmark = pytest.mark.gpu


def _edge_lattice(B, L, Kw, lens, seed, density=0.5):
    """Random slots plus the cases the kernels must get right: a row without words, 2- and 10-character words, every
    slot full, words touching [0] and [seq_len - 1], and malformed slots that must behave as empty."""
    lat = olat.random_lattice(B, L, Kw, lens, seed, density)
    lat = lat.view(B, L, Kw)
    if B > 3:
        lat[3] = 0                                        # no words
    n0 = int(lens[0])
    lat[0, :, :] = 0
    if n0 >= 10:
        lat[0, 0, :] = torch.tensor([2, 10, 3, 5][:Kw] + [4] * max(0, Kw - 4))[:Kw]    # all slots full, at [0]
        lat[0, n0 - 2, 0] = 2                            # ends at seq_len - 1
        lat[0, n0 - 10, 1 % Kw] = 10                     # 10 characters ending at seq_len - 1
        lat[0, n0 - 1, 0] = 2                            # reaches past seq_len: empty
        lat[0, 4, 0], lat[0, 5, 0], lat[0, 6, 0] = 1, 11, -7   # malformed lengths
        lat[0, 7, 0] = 1 << 30
    return lat.view(B, L * Kw).contiguous()


def _host_recurrence_inputs(x, xw, w, H):
    """xproj / wproj in float64 on the host (so only the recurrence kernel is under test) and the recurrent weights."""
    B, L, Ec = x.shape
    Ew = xw.shape[-1]
    nm = olat.names()
    xp, wp, wrec, wac = [], [], [], []
    for d in ("fw", "bw"):
        kc, bc = w[nm[d]["char_cell"][0]].double(), w[nm[d]["char_cell"][1]].double()
        ka, ba = w[nm[d]["alpha"][0]].double(), w[nm[d]["alpha"][1]].double()
        kw, bw = w[nm[d]["word_cell"][0]].double(), w[nm[d]["word_cell"][1]].double()
        xp += [x.double().reshape(-1, Ec) @ kc[:Ec] + bc, x.double().reshape(-1, Ec) @ ka[:Ec] + ba]
        wp.append(xw.double().reshape(-1, Ew) @ kw[:Ew] + bw)
        wrec.append(torch.cat([kc[Ec:], kw[Ew:]], 1).float().contiguous().cuda())
        wac.append(ka[Ec:].float().contiguous().cuda())
    return torch.cat(xp, 1).float().cuda(), torch.cat(wp, 1).float().cuda(), wrec, wac


CASES = [(5, 24, 32, 2, 0.5), (6, 40, 100, 4, 0.6), (3, 33, 64, 8, 0.9), (7, 17, 48, 4, 0.0)]


@pytest.mark.parametrize("B,L,H,Kw,density", CASES + [(64, 128, 100, 4, 0.3)])
def test_recurrence_matches_oracle(B, L, H, Kw, density):
    Ec, Ew = 20, 12
    g = torch.Generator().manual_seed(B * L + H)
    x = torch.randn(B, L, Ec, generator=g)
    xw = torch.randn(B, L, Kw, Ew, generator=g)
    lens = torch.randint(1, L + 1, (B,), generator=g, dtype=torch.int32)
    lens[0] = L
    lens[1] = 0
    lens[2] = 1
    lat = _edge_lattice(B, L, Kw, lens, seed=B + L, density=density)
    w = olat.random_weights(Ec, Ew, H, seed=H, scale=1.5)
    ref = olat.lattice_lstm(x.double(), xw.double(), lat, lens, {k: v.double() for k, v in w.items()}, H)
    xproj, wproj, wrec, wac = _host_recurrence_inputs(x, xw, w, H)
    out = ops.lattice_recurrence(xproj, wproj, lat.cuda(), wrec[0], wrec[1], wac[0], wac[1], lens.cuda(), B, L, H, Kw)
    torch.testing.assert_close(out.cpu().double(), ref, rtol=1e-4, atol=1e-4)
    for b in range(B):
        assert (out[b, int(lens[b]):] == 0).all()
    # PREDICT and TRAIN forwards agree bit for bit, and a repeat is bit-identical
    out2, _ = ops.lattice_recurrence(xproj, wproj, lat.cuda(), wrec[0], wrec[1], wac[0], wac[1], lens.cuda(), B, L, H, Kw,
                                     save_for_backward=True)
    assert torch.equal(out, out2)


def test_empty_lexicon_is_the_coupled_gate_lstm():
    B, L, H, Kw, Ec = 4, 30, 64, 4, 16
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, L, Ec, generator=g, dtype=torch.float64)
    lens = torch.tensor([30, 17, 1, 0], dtype=torch.int32)
    w = olat.random_weights(Ec, 8, H, seed=4)
    xproj, wproj, wrec, wac = _host_recurrence_inputs(x.float(), torch.zeros(B, L, Kw, 8), w, H)
    lat = torch.zeros(B, L * Kw, dtype=torch.int32)
    out = ops.lattice_recurrence(xproj, wproj, lat.cuda(), wrec[0], wrec[1], wac[0], wac[1], lens.cuda(), B, L, H, Kw)
    nm = olat.names()
    ref = torch.zeros(B, L, 2 * H, dtype=torch.float64)
    for di, d in enumerate(("fw", "bw")):
        k, bias = w[nm[d]["char_cell"][0]].double(), w[nm[d]["char_cell"][1]].double()
        for b in range(B):
            h = c = torch.zeros(H, dtype=torch.float64)
            n = int(lens[b])
            for t in (range(n) if di == 0 else range(n - 1, -1, -1)):
                z = x[b, t] @ k[:Ec] + h @ k[Ec:] + bias
                i, o, gg = torch.sigmoid(z[:H]), torch.sigmoid(z[H:2 * H]), torch.tanh(z[2 * H:])
                c = (1 - i) * c + i * gg
                h = o * torch.tanh(c)
                ref[b, t, di * H:(di + 1) * H] = h
    torch.testing.assert_close(out.cpu().double(), ref, rtol=1e-4, atol=1e-4)


def _bf16(t):
    return t.to(torch.bfloat16).double()


@pytest.mark.parametrize("B,L,H,Kw,density", CASES)
def test_bptt_matches_oracle_autograd_and_repeats_bit_identically(B, L, H, Kw, density):
    """layer.lattice_lstm in TRAIN: every variable and both inputs against float64 autograd (projection operands rounded
    to bf16 in the oracle, as the GEMMs round them), and the BPTT outputs and dense weight gradients bit-identical."""
    Ec, Ew = 24, 16
    g = torch.Generator().manual_seed(B + L + H)
    x = torch.randn(B, L, Ec, generator=g)
    xw = torch.randn(B * L, Kw * Ew, generator=g)
    lens = torch.randint(1, L + 1, (B,), generator=g, dtype=torch.int32)
    lens[0], lens[1], lens[2] = L, 0, 1
    lat = _edge_lattice(B, L, Kw, lens, seed=L, density=density)
    w = olat.random_weights(Ec, Ew, H, seed=H + 1, scale=1.5)
    wd = {k: v.double().requires_grad_(True) for k, v in w.items()}
    wd_in = {}
    for k, v in wd.items():          # input halves of the kernels go through bf16 GEMM operands
        part = k.split('/')[-2]
        if k.endswith('kernel'):
            din = Ew if part == 'word_cell' else Ec
            wd_in[k] = torch.cat([v[:din] + (_bf16(v[:din].detach()) - v[:din].detach()), v[din:]], 0)
        else:
            wd_in[k] = v
    xd = _bf16(x).requires_grad_(True)
    xwd = _bf16(xw).requires_grad_(True)
    ref = olat.lattice_lstm(xd, xwd.view(B, L, Kw, Ew), lat, lens, wd_in, H)
    d_out = torch.randn(B, L, 2 * H, generator=g, dtype=torch.float64)
    (ref * d_out).sum().backward()

    runs = []
    for _ in range(2):
        store = variables.VariableStore("cuda")
        store.load_state_dict(w)
        got = {}
        with variables.use_store(store), autodiff.recording(store) as tape:
            xg, xwg = x.cuda(), xw.cuda()
            tape.record(xg, lambda gx: got.__setitem__('x', gx))
            tape.record(xwg, lambda gx: got.__setitem__('xw', gx))
            out = layer.lattice_lstm(xg, xwg, lat.cuda(), H, lens.cuda(), True)
            tape.add_grad(out, d_out.float().cuda())
            tape.backward()
        runs.append((out, got, {k: v.clone() for k, v in store.grads.items()}))
    out, got, grads = runs[0]
    torch.testing.assert_close(out.cpu().double(), ref.detach(), rtol=1e-3, atol=1e-3)
    assert set(grads) == set(w)
    for name, v in wd.items():
        scale = max(v.grad.abs().max().item(), 1e-6)
        assert (grads[name].cpu().double() - v.grad).abs().max().item() < 2e-2 * scale, name
    for key, ref_g in (('x', xd.grad), ('xw', xwd.grad)):
        scale = max(ref_g.abs().max().item(), 1e-6)
        assert (got[key].cpu().double().reshape(ref_g.shape) - ref_g).abs().max().item() < 2e-2 * scale, key
    # bit-identical repeats: forward, BPTT inputs' gradients and every weight gradient
    assert torch.equal(runs[0][0], runs[1][0])
    for key in ('x', 'xw'):
        assert torch.equal(runs[0][1][key], runs[1][1][key])
    for name in grads:
        assert torch.equal(runs[0][2][name], runs[1][2][name]), name


def test_bwd_kernel_outputs_repeat_bit_identically():
    B, L, H, Kw = 64, 128, 100, 4
    g = torch.Generator().manual_seed(9)
    lens = torch.randint(1, L + 1, (B,), generator=g, dtype=torch.int32)
    lat = olat.random_lattice(B, L, Kw, lens, seed=9, density=0.4).cuda()
    xproj = torch.randn(B * L, 8 * H, generator=g).cuda()
    wproj = torch.randn(B * L * Kw, 6 * H, generator=g).cuda()
    wrec = [(torch.rand(H, 6 * H, generator=g) - 0.5).div(10).cuda() for _ in range(2)]
    wac = [(torch.rand(H, H, generator=g) - 0.5).div(10).cuda() for _ in range(2)]
    d_out = torch.randn(B, L, 2 * H, generator=g).cuda()
    res = []
    for _ in range(2):
        out, sv = ops.lattice_recurrence(xproj, wproj, lat, wrec[0], wrec[1], wac[0], wac[1], lens.cuda(), B, L, H, Kw,
                                         save_for_backward=True)
        res.append((out,) + ops.lattice_recurrence_bwd(d_out, sv, lat, wrec[0], wrec[1], wac[0], wac[1], lens.cuda(),
                                                       B, L, H, Kw))
    for a, b in zip(*res):
        assert torch.isfinite(a).all() and torch.equal(a, b)


# ----------------------------------------------------------------------------- plugin
MODEL = 'lattice_lstm_crf'


def _setup(B=8, L=48, V=3000, NW=500, Ew=50, Kw=4, seed=2, dropout=0.0):
    feats = synthetic.msra_batch(B, L, vocab=V, seed=seed)
    lat = olat.random_lattice(B, L, Kw, feats['seq_len'], seed, 0.4)
    rng = np.random.default_rng(seed)
    feats['lattice_lens'] = lat
    feats['lattice_ids'] = torch.from_numpy(np.where(lat.numpy() > 0, rng.integers(0, NW, lat.shape), NW + 1)
                                            .astype(np.int32))
    g = torch.Generator().manual_seed(0)
    emb = torch.nn.functional.normalize(torch.randn(V, 50, generator=g), dim=1).numpy()
    wemb = (torch.randn(NW + 3, Ew, generator=g) * 0.5).numpy()
    params = dict(synthetic.data_params(L), embedding=emb, word_embedding=wemb, max_lattice_words=Kw)
    if dropout is not None:
        params['embedding_dropout'] = dropout
    return engine.Estimator(MODEL, params), feats


def _oracle_loss(wd, feats, params):
    B, L = feats['token_ids'].shape
    Kw = params['max_lattice_words']
    x = _bf16(torch.as_tensor(params['embedding']).double()[feats['token_ids'].long()])
    table = wd['word_enhance/lattice_word_embedding']
    filled = ((feats['lattice_lens'] >= 2) & (feats['lattice_lens'] <= 10)).double().view(B, L, Kw, 1)
    xw = table[feats['lattice_ids'].long()].view(B, L, Kw, -1) * filled
    xw = xw + (_bf16(xw.detach()) - xw.detach())
    wd_in = {}
    for k, v in wd.items():
        if k.startswith('lattice_layer') and k.endswith('kernel'):
            din = xw.shape[-1] if '/word_cell/' in k else x.shape[-1]
            v = torch.cat([v[:din] + (_bf16(v[:din].detach()) - v[:din].detach()), v[din:]], 0)
        wd_in[k] = v
    H = params['hidden_units_list'][0]
    hidden = olat.lattice_lstm(x, xw, feats['lattice_lens'], feats['seq_len'], wd_in, H)
    logits = hidden @ wd['logits/kernel'] + wd['logits/bias']
    ll = crf_torch.crf_log_likelihood(logits, feats['label_ids'], feats['seq_len'], wd['crf_layer/transitions'])
    return (-ll).mean(), logits


def test_plugin_predict_eval_match_oracle_and_crf():
    est, feats = _setup()
    est.evaluate(feats)
    est.store.vars['logits/kernel'].mul_(6.0)
    est.store.touch()
    out = est.evaluate(feats)
    wd = {k: v.double() for k, v in est.store.state_dict().items()}
    loss, logits = _oracle_loss(wd, feats, est.params)
    assert abs(out['loss'] - loss.item()) < 2e-3 * max(1.0, abs(loss.item()))
    tags = ocrf.crf_decode(logits.numpy(), wd['crf_layer/transitions'].numpy(), feats['seq_len'].numpy(), np.float64)[0]
    assert (out['pred_ids'].numpy() == np.asarray(tags)).mean() > 0.99
    assert (out['pred_ids'].numpy()[feats['mask'].numpy() == 0] == 0).all()
    pred = est.predict(feats)['pred_ids'].numpy()
    np.testing.assert_array_equal(pred, out['pred_ids'].numpy())


def test_plugin_gradients_match_oracle_autograd():
    est, feats = _setup(L=32)
    est.evaluate(feats)
    w = est.store.state_dict()
    wd = {k: v.double().clone().requires_grad_(True) for k, v in w.items()}
    ref_loss, _ = _oracle_loss(wd, feats, est.params)
    ref_loss.backward()
    dev = est.to_device(feats)
    with variables.use_store(est.store), autodiff.recording(est.store) as tape:
        loss, _ = est.build_graph(dev, None, est.params, True)
        tape.backward()
    assert abs(float(loss) - ref_loss.item()) < 2e-3 * max(1.0, abs(ref_loss.item()))
    for name, v in wd.items():
        gk = est.store.grads[name].cpu().double()
        scale = max(v.grad.abs().max().item(), 1e-6)
        assert (gk - v.grad).abs().max().item() < 2e-2 * scale, name


def test_train_steps_lower_the_loss():
    torch.manual_seed(0)
    est, feats = _setup(L=48, dropout=None)                 # TRAIN_PARAMS dropout on
    losses = [float(est.train_step(feats)) for _ in range(12)]
    assert np.isfinite(losses).all() and losses[-1] < 0.9 * losses[0], losses


def test_plugin_variables_and_checkpoint_round_trip(tmp_path):
    est, feats = _setup()
    pred = est.evaluate(feats)['pred_ids']
    names = sorted(est.store.state_dict())
    want = sorted([f'lattice_layer/{d}/{p}/{kb}' for d in ('fw', 'bw') for p in ('char_cell', 'word_cell', 'alpha')
                   for kb in ('kernel', 'bias')] + ['word_enhance/lattice_word_embedding', 'logits/kernel', 'logits/bias',
                                                    'crf_layer/transitions'])
    assert names == want
    H = est.params['hidden_units_list'][0]
    assert tuple(est.store.vars['lattice_layer/fw/char_cell/kernel'].shape) == (50 + H, 3 * H)
    assert tuple(est.store.vars['lattice_layer/bw/word_cell/kernel'].shape) == (50 + H, 3 * H)
    assert tuple(est.store.vars['lattice_layer/fw/alpha/kernel'].shape) == (50 + H, H)
    path = checkpoint.save_checkpoint(est.store, str(tmp_path))
    est2, _ = _setup()
    checkpoint.restore_checkpoint(est2.store, path)
    assert sorted(est2.store.state_dict()) == names
    np.testing.assert_array_equal(est2.evaluate(feats)['pred_ids'].numpy(), pred.numpy())


def test_cell_type_and_cell_size_are_refused():
    for bad in (dict(cell_type='gru'), dict(cell_size=2, hidden_units_list=[100, 100], keep_prob_list=[1, 1])):
        est, feats = _setup()
        est.params.update(bad)
        with pytest.raises(ValueError):
            est.evaluate(feats)


def test_infer_helper_serves_text(tmp_path):
    from chinesener_b200.data.base_preprocess import features_to_batch
    from chinesener_b200.data.tokenizer import TextVectors, get_giga_tokenizer
    from chinesener_b200.data.word_enhance import WordVocab, lattice_word_embedding
    from chinesener_b200.inference import InferHelper, TAG2IDX
    from chinesener_b200.tools.infer_utils import extract_entity
    text = '中共中央致中国致公党十一大的贺词，各位代表、各位同志：在中国致公党第十一次全国代表大会隆重召开之际。'
    tok = get_giga_tokenizer(write_vec(tmp_path / 'giga.vec', sorted(set(text)), dim=50))
    vec = TextVectors(write_vec(tmp_path / 'word.vec', ['中共中央', '中国', '致公党', '中国致公党', '代表', '代表大会',
                                                        '全国代表大会', '同志', '召开'], dim=16))
    vocab = WordVocab(vec.index2word, dict.fromkeys(vec.index2word, 1))
    params = dict(synthetic.data_params(150), embedding=tok.embedding(0), word_embedding=lattice_word_embedding(vec),
                  max_lattice_words=4)
    est = engine.Estimator(MODEL, params)
    helper = InferHelper(150, TAG2IDX, MODEL, tok, estimator=est, vocab=vocab, word_embedding=params['word_embedding'])
    helper.infer(text)
    est.store.vars['logits/kernel'].mul_(8.0)
    est.store.touch()
    ent = helper.infer(text)
    lens = np.asarray(helper.feature['lattice_lens']).reshape(150, 4)
    assert lens[text.index('中国致公党')].tolist()[:2] == [2, 5]         # 中国, 中国致公党 in increasing length
    pred = est.predict(features_to_batch([helper.feature]))['pred_ids'].numpy()[0]
    assert pred[len(text):].tolist() == [0] * (150 - len(text))
    idx2tag = {v: k for k, v in TAG2IDX.items()}
    assert dict(ent) == dict(extract_entity(helper.feature['tokens'], [int(i) for i in pred], idx2tag))
