"""GPU: persistent cluster BiLSTM recurrence (+ wgmma input projection) vs the CPU oracle."""
import pytest
import torch

from chinesener_b200 import ops, variables
from chinesener_b200.tools import layer
from oracle import nn as onn

pytestmark = pytest.mark.gpu


def _weights(D, H, seed):
    g = torch.Generator().manual_seed(seed)
    w = {}
    for d in ("fw", "bw"):
        lim = (6.0 / (D + H + 4 * H)) ** 0.5
        w[f"bilstm_layer/bidirectional_rnn/{d}/multi_rnn_cell/cell_0/lstm_cell/kernel"] = \
            (torch.rand(D + H, 4 * H, generator=g) * 2 - 1) * lim
        w[f"bilstm_layer/bidirectional_rnn/{d}/multi_rnn_cell/cell_0/lstm_cell/bias"] = torch.randn(4 * H, generator=g) * 0.1
    return w


@pytest.mark.parametrize("B,L,H,act", [(64, 128, 128, "relu"), (8, 64, 128, "tanh"), (5, 33, 200, "tanh"),
                                       (150, 20, 128, "tanh"), (3, 150, 64, "relu"), (300, 12, 128, "relu"), (256, 40, 128, "relu")])
def test_recurrence_matches_oracle_fp32_inputs(B, L, H, act):
    """Recurrence alone: xproj computed in fp64 on the host, so only the cluster kernel is under test."""
    D = 40
    g = torch.Generator().manual_seed(B + L + H)
    x = torch.randn(B, L, D, generator=g)
    w = _weights(D, H, seed=H)
    lens = torch.randint(1, L + 1, (B,), generator=g, dtype=torch.int32)
    lens[0] = L
    if B > 2:
        lens[1] = 1
        lens[2] = 0
    ref = onn.bilstm(x, w, lens, act, 1.0, torch.float64)
    ks = [w[f"bilstm_layer/bidirectional_rnn/{d}/multi_rnn_cell/cell_0/lstm_cell/kernel"] for d in ("fw", "bw")]
    bs = [w[f"bilstm_layer/bidirectional_rnn/{d}/multi_rnn_cell/cell_0/lstm_cell/bias"] for d in ("fw", "bw")]
    xproj = torch.cat([x.double().view(B * L, D) @ k[:D].double() + b.double() for k, b in zip(ks, bs)], dim=1).float()
    out = ops.bilstm_recurrence(xproj.cuda(), ks[0][D:].contiguous().cuda(), ks[1][D:].contiguous().cuda(), lens.cuda(),
                                B, L, H, activation=act)
    torch.testing.assert_close(out.cpu().double(), ref, rtol=1e-4, atol=1e-4)
    # dynamic_rnn contract: zero output for t >= len
    for b in range(B):
        assert (out[b, int(lens[b]):] == 0).all()


@pytest.mark.parametrize("D,H,act", [(768, 128, "relu"), (250, 200, "tanh"), (50, 128, "tanh")])
def test_bilstm_layer_with_tensor_core_projection(D, H, act):
    B, L = 16, 48
    g = torch.Generator().manual_seed(D + H)
    x = torch.randn(B, L, D, generator=g) * 0.5
    w = _weights(D, H, seed=D)
    lens = torch.randint(1, L + 1, (B,), generator=g, dtype=torch.int32)
    store = variables.VariableStore("cuda")
    store.load_state_dict(w)
    with variables.use_store(store):
        out = layer.bilstm(x.cuda(), "lstm", act, [H], [1.0], 1, lens.cuda(), "float32", False)
    ref_emul = onn.bilstm(x, w, lens, act, 1.0, torch.float64, emulate_bf16=True)
    ref_true = onn.bilstm(x, w, lens, act, 1.0, torch.float64)
    torch.testing.assert_close(out.cpu().double(), ref_emul, rtol=1e-3, atol=1e-3)
    # bf16 operand rounding of the input projection stays small against the fp64 truth
    assert (out.cpu().double() - ref_true).abs().max() < 5e-2
