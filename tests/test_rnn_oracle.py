"""Pins the stacked / GRU restatement of bidirectional_dynamic_rnn (tests/_rnn_oracle.py: birnn, gru_direction) independently of
the CUDA path: against torch.nn.LSTM / torch.nn.GRU where their semantics coincide, and against hand-worked steps where
TF's GRUCell differs from torch's (the reset gate applied before the recurrent matmul of the candidate)."""
import math

import pytest
import torch

from oracle import nn as onn

import _rnn_oracle as ornn

P = "bilstm_layer/bidirectional_rnn"


def _lens(B, L, g):
    lens = torch.randint(1, L + 1, (B,), generator=g, dtype=torch.int32)
    lens[0] = L
    lens[1] = 1
    return lens


def _lstm_weights(D, Hs, g):
    w = {}
    for d in ("fw", "bw"):
        din = D
        for i, H in enumerate(Hs):
            w[f"{P}/{d}/multi_rnn_cell/cell_{i}/lstm_cell/kernel"] = torch.randn(din + H, 4 * H, generator=g, dtype=torch.float64) * 0.3
            w[f"{P}/{d}/multi_rnn_cell/cell_{i}/lstm_cell/bias"] = torch.randn(4 * H, generator=g, dtype=torch.float64) * 0.1
            din = H
    return w


def _gru_weights(D, Hs, g):
    w = {}
    for d in ("fw", "bw"):
        din = D
        for i, H in enumerate(Hs):
            base = f"{P}/{d}/multi_rnn_cell/cell_{i}/gru_cell"
            w[f"{base}/gates/kernel"] = torch.randn(din + H, 2 * H, generator=g, dtype=torch.float64) * 0.3
            w[f"{base}/gates/bias"] = 1.0 + torch.randn(2 * H, generator=g, dtype=torch.float64) * 0.1
            w[f"{base}/candidate/kernel"] = torch.randn(din + H, H, generator=g, dtype=torch.float64) * 0.3
            w[f"{base}/candidate/bias"] = torch.randn(H, generator=g, dtype=torch.float64) * 0.1
            din = H
    return w


def _reverse_within(x, lens):
    """reverse_sequence(x, lens, seq_axis=1): positions [0, len) reversed, the rest kept."""
    out = x.clone()
    for b, n in enumerate(lens.tolist()):
        out[b, :n] = x[b, :n].flip(0)
    return out


def _torch_stack(module, x, lens, reverse):
    xs = _reverse_within(x, lens) if reverse else x
    keep = lens > 0
    packed = torch.nn.utils.rnn.pack_padded_sequence(xs[keep], lens[keep].long(), batch_first=True, enforce_sorted=False)
    y, _ = module(packed)
    y, _ = torch.nn.utils.rnn.pad_packed_sequence(y, batch_first=True, total_length=x.shape[1])
    out = x.new_zeros(x.shape[0], x.shape[1], y.shape[-1])
    out[keep] = y
    return _reverse_within(out, lens) if reverse else out


@pytest.mark.parametrize("n_layers", [1, 2, 3])
def test_stacked_lstm_equals_two_unidirectional_torch_stacks(n_layers):
    """Per-direction stacking: fw layer i+1 reads fw layer i (torch's bidirectional stacking would feed [fw | bw])."""
    g = torch.Generator().manual_seed(n_layers)
    B, L, D, H = 5, 9, 6, 8
    x = torch.randn(B, L, D, generator=g, dtype=torch.float64)
    lens = _lens(B, L, g)
    w = _lstm_weights(D, [H] * n_layers, g)
    ref = ornn.birnn(x, w, lens, "lstm", [H] * n_layers, "tanh", forget_bias=1.0)
    outs = []
    for d, rev in (("fw", False), ("bw", True)):
        m = torch.nn.LSTM(D, H, num_layers=n_layers, batch_first=True).double()
        with torch.no_grad():
            for i in range(n_layers):
                k = w[f"{P}/{d}/multi_rnn_cell/cell_{i}/lstm_cell/kernel"]
                b = w[f"{P}/{d}/multi_rnn_cell/cell_{i}/lstm_cell/bias"]
                din = k.shape[0] - H
                ki, kj, kf, ko = k.split(H, dim=1)            # TF (i, j, f, o) -> torch (i, f, g, o)
                bi, bj, bf, bo = b.split(H)
                wt = torch.cat([ki, kf + 0, kj, ko], dim=1)
                getattr(m, f"weight_ih_l{i}").copy_(wt[:din].t())
                getattr(m, f"weight_hh_l{i}").copy_(wt[din:].t())
                getattr(m, f"bias_ih_l{i}").copy_(torch.cat([bi, bf + 1.0, bj, bo]))   # forget_bias folded in
                getattr(m, f"bias_hh_l{i}").zero_()
            outs.append(_torch_stack(m, x, lens, rev))
    torch.testing.assert_close(ref, torch.cat(outs, -1), rtol=0, atol=1e-10)


def test_one_lstm_layer_is_bilstm():
    g = torch.Generator().manual_seed(7)
    x = torch.randn(4, 7, 5, generator=g, dtype=torch.float64)
    lens = _lens(4, 7, g)
    w = _lstm_weights(5, [6], g)
    for act in ("tanh", "relu"):
        torch.testing.assert_close(ornn.birnn(x, w, lens, "lstm", [6], act), onn.bilstm(x, w, lens, act, 1.0),
                                   rtol=0, atol=1e-12)


@pytest.mark.parametrize("n_layers", [1, 2])
def test_gru_with_zero_recurrent_candidate_equals_torch_gru(n_layers):
    """With candidate/kernel[D:] = 0, TF's (r * h) @ W_c^h and torch's r * (h @ W_hn) both vanish: gate order r / u,
    h' = u h + (1 - u) c and the masking are then pinned by torch.nn.GRU."""
    g = torch.Generator().manual_seed(10 + n_layers)
    B, L, D, H = 6, 8, 5, 7
    x = torch.randn(B, L, D, generator=g, dtype=torch.float64)
    lens = _lens(B, L, g)
    lens[2] = 0
    w = _gru_weights(D, [H] * n_layers, g)
    for k in list(w):
        if k.endswith("candidate/kernel"):
            w[k][-H:] = 0.0
    ref = ornn.birnn(x, w, lens, "gru", [H] * n_layers, "tanh")
    outs = []
    for d, rev in (("fw", False), ("bw", True)):
        m = torch.nn.GRU(D, H, num_layers=n_layers, batch_first=True).double()
        with torch.no_grad():
            for i in range(n_layers):
                base = f"{P}/{d}/multi_rnn_cell/cell_{i}/gru_cell"
                gk, gb = w[f"{base}/gates/kernel"], w[f"{base}/gates/bias"]
                ck, cb = w[f"{base}/candidate/kernel"], w[f"{base}/candidate/bias"]
                din = gk.shape[0] - H
                getattr(m, f"weight_ih_l{i}").copy_(torch.cat([gk[:din], ck[:din]], dim=1).t())
                getattr(m, f"weight_hh_l{i}").copy_(torch.cat([gk[din:], torch.zeros(H, H, dtype=torch.float64)], 1).t())
                getattr(m, f"bias_ih_l{i}").copy_(torch.cat([gb, cb]))
                getattr(m, f"bias_hh_l{i}").zero_()
            outs.append(_torch_stack(m, x, lens, rev))
    out = torch.cat(outs, -1)
    torch.testing.assert_close(ref, out, rtol=0, atol=1e-10)
    assert (ref[2] == 0).all()


def _sig(v):
    return 1.0 / (1.0 + math.exp(-v))


def test_gru_hand_worked_steps_apply_the_reset_gate_before_the_matmul():
    """D = 1, H = 2, two steps of the fw direction, worked with scalars: the candidate's recurrent term is
    (r * h) @ W_c^h, which torch's GRU (r * (h @ W_hn)) does not share once W_c^h mixes units."""
    Wg = [[0.5, -0.3, 0.2, 0.1],        # row x
          [0.4, 0.2, -0.6, 0.3],        # row h_0
          [-0.2, 0.7, 0.1, -0.5]]       # row h_1   (columns r0, r1, u0, u1)
    bg = [1.0, 1.0, 1.0, 1.0]
    Wc = [[0.3, -0.8],
          [0.9, -0.4],
          [-0.7, 0.6]]                  # columns c0, c1
    bc = [0.05, -0.1]
    xs = [1.5, -0.7]
    h = [0.0, 0.0]
    hand = []
    for xv in xs:
        a = [xv * Wg[0][j] + h[0] * Wg[1][j] + h[1] * Wg[2][j] + bg[j] for j in range(4)]
        r, u = [_sig(a[0]), _sig(a[1])], [_sig(a[2]), _sig(a[3])]
        rh = [r[0] * h[0], r[1] * h[1]]
        c = [math.tanh(xv * Wc[0][j] + rh[0] * Wc[1][j] + rh[1] * Wc[2][j] + bc[j]) for j in range(2)]
        h = [u[j] * h[j] + (1 - u[j]) * c[j] for j in range(2)]
        hand.append(h)
    k = torch.cat([torch.tensor(Wg, dtype=torch.float64), torch.tensor(Wc, dtype=torch.float64)], dim=1)
    b = torch.tensor(bg + bc, dtype=torch.float64)
    x = torch.tensor(xs, dtype=torch.float64).view(1, 2, 1)
    two = ornn.gru_direction(x, k, b, torch.tensor([2]))
    torch.testing.assert_close(two[0], torch.tensor(hand, dtype=torch.float64), rtol=0, atol=1e-15)
    one = ornn.gru_direction(x, k, b, torch.tensor([1]))   # length 1: the second position is zero
    torch.testing.assert_close(one[0], torch.tensor([hand[0], [0.0, 0.0]], dtype=torch.float64), rtol=0, atol=1e-15)
    # the same weights with the reset gate applied after the matmul (torch's form) give a different second step
    h1 = torch.tensor(hand[0], dtype=torch.float64)
    a = torch.tensor(xs[1]) * k[0, :4] + h1 @ k[1:, :4] + b[:4]
    r, u = torch.sigmoid(a[:2]), torch.sigmoid(a[2:])
    c_after = torch.tanh(xs[1] * k[0, 4:] + r * (h1 @ k[1:, 4:]) + b[4:])
    assert (u * h1 + (1 - u) * c_after - two[0, 1]).abs().max() > 1e-3


def test_gru_masks_are_the_dropout_wrapper_filters():
    """state_mask feeds the next step (the whole GRU state), out_mask only the emitted output."""
    g = torch.Generator().manual_seed(3)
    B, L, D, H = 3, 5, 4, 6
    x = torch.randn(B, L, D, generator=g, dtype=torch.float64)
    lens = torch.tensor([5, 3, 0])
    k = torch.randn(D + H, 3 * H, generator=g, dtype=torch.float64) * 0.4
    b = torch.randn(3 * H, generator=g, dtype=torch.float64) * 0.1
    om = (torch.rand(B, L, H, generator=g) < 0.7).double() / 0.7
    ones = torch.ones(B, L, H, dtype=torch.float64)
    plain = ornn.gru_direction(x, k, b, lens)
    torch.testing.assert_close(ornn.gru_direction(x, k, b, lens, out_mask=om), plain * om, rtol=0, atol=1e-15)
    torch.testing.assert_close(ornn.gru_direction(x, k, b, lens, state_mask=ones), plain, rtol=0, atol=0)
    sm = om.flip(-1)
    dropped = ornn.gru_direction(x, k, b, lens, state_mask=sm)
    assert torch.equal(dropped[:, 0], plain[:, 0]) and not torch.allclose(dropped[0, 1:], plain[0, 1:])
