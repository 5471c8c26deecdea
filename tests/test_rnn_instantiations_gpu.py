"""GPU: every instantiation of the BiLSTM, BiGRU and Lattice LSTM recurrence kernels against float64.

The host picks one of 38 kernel instantiations from (B, H, Kw, number of SMs) through `ner_rnn_plan`, so which of them a
fixed B reaches depends on the device.  Each case here asks the plan, on this device's SM count, for the smallest B that
reaches its instantiation and for one more B with B % R != 0, and calls the C entry points directly with every output
pre-filled with NaN (a position the kernel skips shows up).  The projections are computed in float64 on the host, so
only the recurrence is under test.  Lengths include 0, 1, 2, L, -3 and L + 5 (the reference gets clamp(len, 0, L)), a
row group of zero-length rows and a row group whose longest row is shorter than L.
"""
import ctypes
import os
import re

import pytest
import torch

import _lattice_oracle as olat
import _rnn_oracle as ornn
from chinesener_b200._lib import check, lib, ptr, stream
from test_bilstm_gpu import _weights as _lstm_weights
from test_lattice_gpu import _edge_lattice, _host_recurrence_inputs
from test_rnn_cells_gpu import P, _gru_w, _rnn_masks

pytestmark = pytest.mark.gpu

LSTM_FWD, LSTM_BWD, GRU_FWD, GRU_BWD, LAT_FWD, LAT_BWD = range(6)
NAMES = ("bilstm_rec", "bilstm_bwd", "bigru_rec", "bigru_bwd", "lattice_fwd", "lattice_bwd")

# (kernel, R, resident, ACT): the template arguments of the GO(...) lines of csrc/bilstm.cu, bilstm_bwd.cu, bigru.cu,
# bigru_bwd.cu and lattice.cu, each LSTM / GRU line for ACT = 0 (tanh) and 1 (relu); the lattice has no activation.
INSTANTIATIONS = {
    (LSTM_FWD, 8, 1, 0), (LSTM_FWD, 8, 1, 1), (LSTM_FWD, 2, 1, 0), (LSTM_FWD, 2, 1, 1),
    (LSTM_FWD, 1, 1, 0), (LSTM_FWD, 1, 1, 1), (LSTM_FWD, 4, 0, 0), (LSTM_FWD, 4, 0, 1),
    (LSTM_FWD, 2, 0, 0), (LSTM_FWD, 2, 0, 1), (LSTM_FWD, 1, 0, 0), (LSTM_FWD, 1, 0, 1),
    (LSTM_BWD, 2, 1, 0), (LSTM_BWD, 2, 1, 1), (LSTM_BWD, 1, 1, 0), (LSTM_BWD, 1, 1, 1),
    (LSTM_BWD, 2, 0, 0), (LSTM_BWD, 2, 0, 1), (LSTM_BWD, 1, 0, 0), (LSTM_BWD, 1, 0, 1),
    (GRU_FWD, 4, 0, 0), (GRU_FWD, 4, 0, 1), (GRU_FWD, 2, 0, 0), (GRU_FWD, 2, 0, 1), (GRU_FWD, 1, 0, 0), (GRU_FWD, 1, 0, 1),
    (GRU_BWD, 4, 0, 0), (GRU_BWD, 4, 0, 1), (GRU_BWD, 2, 0, 0), (GRU_BWD, 2, 0, 1), (GRU_BWD, 1, 0, 0), (GRU_BWD, 1, 0, 1),
    (LAT_FWD, 4, 0, 0), (LAT_FWD, 2, 0, 0), (LAT_FWD, 1, 0, 0),
    (LAT_BWD, 4, 0, 0), (LAT_BWD, 2, 0, 0), (LAT_BWD, 1, 0, 0),
}
SRC = {LSTM_FWD: "bilstm.cu", LSTM_BWD: "bilstm_bwd.cu", GRU_FWD: "bigru.cu", GRU_BWD: "bigru_bwd.cu"}
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "chinesener_b200", "csrc")

L = 24                          # the lattice oracle loops over rows in Python: L stays small at B > 128
LAT_H, LAT_KW = 64, 4


def _shape(kernel, resident):
    """(H, Kw) of a case: the plugins' H = 128 (register-resident LSTM), the softlexicon plugin's H = 200 (LSTM in
    shared memory), H = 128 for the GRU and a small lattice."""
    if kernel in (LAT_FWD, LAT_BWD):
        return LAT_H, LAT_KW
    return (128 if resident or kernel in (GRU_FWD, GRU_BWD) else 200), 1


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _plan(kernel, B, H, Kw, sms):
    R, C, res = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    st = lib().ner_rnn_plan(kernel, B, H, Kw, sms, ctypes.byref(R), ctypes.byref(C), ctypes.byref(res))
    return (R.value, res.value) if st == 0 else None


def _batches(inst, sms, limit=1100):
    """The smallest B whose plan is `inst`, and one more: the next B with B % R != 0 at least one row group further,
    or for R = 1 the largest B that still runs one row per cluster."""
    kernel, R, res, _ = inst
    H, Kw = _shape(kernel, res)
    hits = [B for B in range(1, limit) if _plan(kernel, B, H, Kw, sms) == (R, res)]
    assert hits, inst
    if R == 1:
        return hits[0], hits[-1]
    return hits[0], next(B for B in hits if B >= hits[0] + R and B % R)


def _go_lines():
    """The instantiations the launchers' GO(...) lines name, read from the sources."""
    found = set()
    for kernel, f in SRC.items():
        text = open(os.path.join(CSRC, f)).read().split("#define GO")[1]
        for m in re.finditer(r"\bGO\((\d+)(?:, (\d+))?\);", text):
            for act in (0, 1):
                found.add((kernel, int(m.group(1)), int(m.group(2) is not None and m.group(2) != "0"), act))
    text = open(os.path.join(CSRC, "lattice.cu")).read()
    for kernel, part in ((LAT_FWD, text.split("ner_lattice_recurrence(")[1].split("ner_lattice_recurrence_bwd(")[0]),
                         (LAT_BWD, text.split("ner_lattice_recurrence_bwd(")[1])):
        found |= {(kernel, int(r), 0, 0) for r in re.findall(r"\bGO\((\d+)\);", part)}
    return found


def test_cases_cover_every_instantiation():
    """Before any kernel runs: the table below names each instantiation once, the plan reaches each of them on this
    device and no other, and the launchers' GO(...) lines name the same set."""
    assert len(INSTANTIATIONS) == 38
    assert _go_lines() == INSTANTIATIONS
    sms = _sms()
    reached = set()
    for kernel in range(6):
        for H in (range(4, 348, 4) if kernel < LAT_FWD else (32, 64, 100, 128, 200)):
            for B in range(1, 1100, 1 if H in (128, 200, 64) else 7):
                p = _plan(kernel, B, H, LAT_KW, sms)
                if p is not None:
                    reached |= {(kernel, p[0], p[1], a) for a in ((0, 1) if kernel < LAT_FWD else (0,))}
    assert reached == INSTANTIATIONS
    print(f"\n{sms} SMs: {torch.cuda.get_device_name(0)}")
    print(f"{'kernel':12} {'R':>2} {'regs':>4} {'act':>4}  {'H':>4} {'Kw':>2}  B")
    for inst in sorted(INSTANTIATIONS):
        H, Kw = _shape(inst[0], inst[2])
        print(f"{NAMES[inst[0]]:12} {inst[1]:2d} {inst[2]:4d} {('tanh', 'relu')[inst[3]]:>4}  {H:4d} {Kw:2d}  "
              f"{_batches(inst, sms)}")


# ---- inputs

def _lengths(B, R, g):
    """Random lengths in [1, L] with 0, 1, 2, L, -3 and L + 5; row group 1 all zero-length, the last group (from four
    groups on) shorter than L."""
    lens = torch.randint(1, L + 1, (B,), generator=g, dtype=torch.int32)
    ng = -(-B // R)
    zero_g = 1 if ng >= 3 else None
    short_g = ng - 1 if ng >= 4 else None
    for b in range(B):
        if b // R == zero_g:
            lens[b] = 0
        elif b // R == short_g:
            lens[b] = int(torch.randint(1, L - 2, (1,), generator=g))
    free = [b for b in range(B) if b // R not in (zero_g, short_g)]
    for b, v in zip(free, (L, 0, 1, 2, -3, L + 5)):
        lens[b] = v
    return lens


def _valid(lens):
    return torch.arange(L)[None, :] < lens.clamp(0, L)[:, None].long()


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


CELLS = {LSTM_FWD: "lstm", LSTM_BWD: "lstm", GRU_FWD: "gru", GRU_BWD: "gru"}


def _rnn_inputs(cell, B, H, seed):
    """xproj [B*L, 2 G H] float32 computed in float64 from plugin-initialised weights, the recurrent matrices and lengths."""
    g = torch.Generator().manual_seed(seed)
    D = 48
    x = torch.randn(B, L, D, generator=g)
    if cell == "lstm":
        w = _lstm_weights(D, H, seed)
        ks = [(w[f"{P}/{d}/multi_rnn_cell/cell_0/lstm_cell/kernel"].double(),
               w[f"{P}/{d}/multi_rnn_cell/cell_0/lstm_cell/bias"].double()) for d in ("fw", "bw")]
    else:
        ks = [ornn.rnn_cell_weights(_gru_w(D, H, g), P, d, 0, "gru") for d in ("fw", "bw")]
    xproj = torch.cat([x.double().view(B * L, D) @ k[:D] + b for k, b in ks], dim=1).float()
    wh = [k[D:].float().contiguous() for k, _ in ks]
    return xproj, wh, g


def _forward(cell, xproj, wh, lens, B, H, act, keep, seed, save=True, cu=None):
    """One call of the forward entry point; -> (out, gates, extra, h) with extra = c (LSTM) or r * h (GRU)."""
    G = 4 if cell == "lstm" else 3
    out = _nan(B, L, 2 * H)
    gates, extra, h = (_nan(B * L, 2 * G * H), _nan(B, L, 2 * H), _nan(B, L, 2 * H)) if save else (None, None, None)
    args = (ptr(xproj), ptr(wh[0]), ptr(wh[1]), ptr(lens), ptr(out), B, L, H)
    if cell == "lstm":
        check(lib().ner_bilstm_recurrence(*args, act, 1.0, ptr(cu), ptr(gates), ptr(extra), ptr(h), keep, seed, stream()))
    else:
        check(lib().ner_bigru_recurrence(*args, 6 * H, act, ptr(cu), ptr(gates), ptr(h), ptr(extra), keep, seed, stream()))
    torch.cuda.synchronize()
    return out, gates, extra, h


def _reference(cell, xp64, wh64, lens, B, H, act, keep, seed, saved=False):
    """Both directions through ornn.rnn_direction with an identity input half (x = xproj) and the kernels' masks."""
    G = 4 if cell == "lstm" else 3
    om, sm = _rnn_masks(B, L, H, keep, seed)
    outs, steps = [], []
    for di in range(2):
        cols = slice(di * H, (di + 1) * H)
        kernel = torch.cat([torch.eye(G * H, dtype=torch.float64), wh64[di]], dim=0)
        r = ornn.rnn_direction(xp64.view(B, L, 2 * G * H)[..., di * G * H:(di + 1) * G * H], kernel,
                               torch.zeros(G * H, dtype=torch.float64), lens.clamp(0, L), cell, act, 1.0, di == 1, False,
                               None if om is None else om[..., cols], None if sm is None else sm[..., cols], saved)
        outs.append(r[0] if saved else r)
        if saved:
            steps.append(r[1])
    return torch.cat(outs, -1), steps


def _close(got, ref, tol=1e-4):
    torch.testing.assert_close(got.cpu().double(), ref, rtol=tol, atol=tol)


# ---- LSTM and GRU

def _rnn_ids(kernels):
    return [i for i in sorted(INSTANTIATIONS) if i[0] in kernels]


def _ident(i):
    return f"{NAMES[i[0]]}-R{i[1]}-{'reg' if i[2] else 'smem'}-{('tanh', 'relu')[i[3]]}"


@pytest.mark.parametrize("keep", [1.0, 0.8])
@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("inst", _rnn_ids((LSTM_FWD, GRU_FWD)), ids=_ident)
def test_forward_matches_float64(inst, which, keep):
    """out, the saved gates / cell state / carried h (LSTM) or gates / carried h / r * h (GRU) against float64; PREDICT
    == TRAIN, packed == padded and repeated calls bit for bit."""
    kernel, R, res, a = inst
    cell, act = CELLS[kernel], ("tanh", "relu")[a]
    H, _ = _shape(kernel, res)
    B = _batches(inst, _sms())[which]
    assert _plan(kernel, B, H, 1, _sms()) == (R, res)
    seed = 0x5DEECE66D * (B + 1) + kernel
    xproj, wh, g = _rnn_inputs(cell, B, H, 1000 * B + H + a)
    lens = _lengths(B, R, g)
    xpc, whc, lc = xproj.cuda(), [w.cuda() for w in wh], lens.cuda()
    out, gates, extra, h = _forward(cell, xpc, whc, lc, B, H, a, keep, seed)
    ref, steps = _reference(cell, xproj.double(), [w.double() for w in wh], lens, B, H, act, keep, seed, saved=True)
    valid = _valid(lens)
    _close(out, ref)
    assert (out.cpu()[~valid] == 0).all()
    G = 4 if cell == "lstm" else 3
    gv = gates.view(B, L, 2, G * H).cpu()
    for di in range(2):
        cols = slice(di * H, (di + 1) * H)
        _close(gv[:, :, di][valid], steps[di]["gates"][valid])
        _close(h.cpu()[..., cols][valid], steps[di]["h"][valid])
        _close(extra.cpu()[..., cols][valid], steps[di]["c" if cell == "lstm" else "rh"][valid])
    if keep == 1.0:
        assert torch.equal(h.cpu()[valid], out.cpu()[valid])   # carried h == emitted output without dropout
    predict = _forward(cell, xpc, whc, lc, B, H, a, keep, seed, save=False)[0]
    assert torch.equal(predict, out)
    clamped = lens.clamp(0, L)
    cu = torch.zeros(B + 1, dtype=torch.int32)
    cu[1:] = clamped.cumsum(0)
    packed = xproj.view(B, L, -1)[valid].contiguous().cuda()
    outp = _forward(cell, packed, whc, clamped.cuda(), B, H, a, keep, seed, save=False, cu=cu.cuda())[0]
    assert torch.equal(outp, out)
    again = _forward(cell, xpc, whc, lc, B, H, a, keep, seed)
    for x, y in zip(again, (out, gates, extra, h)):
        assert torch.equal(x.nan_to_num(7.0), y.nan_to_num(7.0))


@pytest.mark.parametrize("keep", [1.0, 0.8])
@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("inst", _rnn_ids((LSTM_BWD, GRU_BWD)), ids=_ident)
def test_bptt_matches_float64_autograd(inst, which, keep):
    """d_xproj against float64 autograd through rnn_direction (identity input half) with the kernels' dropout masks,
    exactly 0 where no step runs, dW_h formed from the saved carried h as the caller forms it, and repeats bit for bit."""
    kernel, R, res, a = inst
    cell, act = CELLS[kernel], ("tanh", "relu")[a]
    H, _ = _shape(kernel, res)
    G = 4 if cell == "lstm" else 3
    B = _batches(inst, _sms())[which]
    assert _plan(kernel, B, H, 1, _sms()) == (R, res)
    seed = 0x2545F4914F6CDD1D + B + kernel
    xproj, wh, g = _rnn_inputs(cell, B, H, 2000 * B + H + a)
    lens = _lengths(B, R, g)
    xpc, whc, lc = xproj.cuda(), [w.cuda() for w in wh], lens.cuda()
    out, gates, extra, h = _forward(cell, xpc, whc, lc, B, H, a, keep, seed)
    xp64 = xproj.double().requires_grad_(True)
    whd = [w.double().requires_grad_(True) for w in wh]
    ref, _ = _reference(cell, xp64, whd, lens, B, H, act, keep, seed)
    d_out = torch.randn(B, L, 2 * H, generator=g, dtype=torch.float64)
    (ref * d_out).sum().backward()
    _close(out, ref.detach())

    def bwd():
        dx = _nan(B * L, 2 * G * H)
        args = (ptr(d_out.float().cuda()), ptr(gates), ptr(extra if cell == "lstm" else h), ptr(whc[0]), ptr(whc[1]),
                ptr(lc), ptr(dx), B, L, H, a, keep, seed, stream())
        check(lib().ner_bilstm_recurrence_bwd(*args) if cell == "lstm" else lib().ner_bigru_recurrence_bwd(*args))
        torch.cuda.synchronize()
        return dx

    dxp = bwd()
    _close(dxp, xp64.grad)
    valid = _valid(lens)
    assert (dxp.cpu().view(B, L, -1)[~valid] == 0).all()
    d = dxp.cpu().double()
    hs = torch.where(valid[..., None], h.cpu().double(), 0.0)
    for di in range(2):
        hprev = torch.zeros(B, L, H, dtype=torch.float64)
        if di == 0:
            hprev[:, 1:] = hs[:, :-1, :H]
        else:
            hprev[:, :-1] = hs[:, 1:, H:]
        dz = d[:, di * G * H:(di + 1) * G * H]
        if cell == "lstm":
            dw = hprev.view(B * L, H).t() @ dz
        else:
            rh = torch.where(valid[..., None], extra.cpu().double(), 0.0)[..., di * H:(di + 1) * H]
            dw = torch.cat([hprev.view(B * L, H).t() @ dz[:, :2 * H], rh.reshape(B * L, H).t() @ dz[:, 2 * H:]], 1)
        gref = whd[di].grad
        assert (dw - gref).abs().max().item() < 1e-4 * max(1.0, gref.abs().max().item()), di
    assert torch.equal(bwd(), dxp)


# ---- Lattice LSTM

@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("R", [4, 2, 1])
def test_lattice_matches_float64_autograd(R, which):
    """Forward against _lattice_oracle.lattice_lstm, and d_xproj, d_wproj and d_alpha against its float64 autograd with
    the two projections (and a zero shift of each word's alpha pre-activation) as leaves.  Covers lattice_fwd_kernel<R>
    and lattice_bwd_kernel<R>, which share the plan."""
    H, Kw = LAT_H, LAT_KW
    B = _batches((LAT_FWD, R, 0, 0), _sms())[which]
    assert _plan(LAT_FWD, B, H, Kw, _sms()) == (R, 0) == _plan(LAT_BWD, B, H, Kw, _sms())
    g = torch.Generator().manual_seed(B * 31 + R)
    Ec, Ew = 20, 12
    x = torch.randn(B, L, Ec, generator=g)
    xw = torch.randn(B, L, Kw, Ew, generator=g)
    lens = _lengths(B, R, g)
    lat = _edge_lattice(B, L, Kw, lens.clamp(0, L), seed=B + R, density=0.5)
    w = olat.random_weights(Ec, Ew, H, seed=B + H)
    xproj, wproj, wrec, wac = _host_recurrence_inputs(x, xw, w, H)
    lc, latc = lens.cuda(), lat.cuda()
    wargs = (ptr(wrec[0]), ptr(wrec[1]), ptr(wac[0]), ptr(wac[1]), ptr(lc))

    def fwd(save):
        out = _nan(B, L, 2 * H)
        sv = dict(gates=_nan(B * L, 6 * H), cstate=_nan(B, L, 2 * H), norm=_nan(B, L, 2 * H),
                  wgates=_nan(B * L * Kw, 6 * H), cw=_nan(B * L * Kw, 2 * H), aw=_nan(B * L * Kw, 2 * H),
                  hw=_nan(B * L * Kw, 2 * H)) if save else {}
        check(lib().ner_lattice_recurrence(ptr(xproj), ptr(wproj), ptr(latc), *wargs, ptr(out), B, L, H, Kw,
                                           *(ptr(sv.get(k)) for k in ("gates", "cstate", "norm", "wgates", "cw", "aw",
                                                                      "hw")), stream()))
        torch.cuda.synchronize()
        return out, sv

    def bwd(sv, d_out):
        dx, dw, da = _nan(B * L, 8 * H), _nan(B * L * Kw, 6 * H), _nan(B * L * Kw, 2 * H)
        check(lib().ner_lattice_recurrence_bwd(ptr(d_out), *(ptr(sv[k]) for k in ("gates", "cstate", "norm", "wgates",
                                                                                  "cw", "aw")),
                                               ptr(latc), *wargs, ptr(dx), ptr(dw), ptr(da), B, L, H, Kw, stream()))
        torch.cuda.synchronize()
        return dx, dw, da

    # float64 reference with the projections as leaves: identity input halves select each direction's columns
    xp = xproj.cpu().double().view(B, L, 8 * H).requires_grad_(True)
    wp = wproj.cpu().double().view(B, L, Kw, 6 * H).requires_grad_(True)
    shift = torch.zeros(B, L, Kw, 2 * H, dtype=torch.float64, requires_grad=True)
    e8, e6, z = torch.eye(8 * H, dtype=torch.float64), torch.eye(6 * H, dtype=torch.float64), torch.zeros
    wref = {}
    for di, d in enumerate(("fw", "bw")):
        nm, wr, wa = olat.names()[d], wrec[di].cpu().double(), wac[di].cpu().double()
        c0 = di * 4 * H
        wref[nm["char_cell"][0]] = torch.cat([e8[:, c0:c0 + 3 * H], wr[:, :3 * H]], 0)
        wref[nm["alpha"][0]] = torch.cat([e8[:, c0 + 3 * H:c0 + 4 * H], wa], 0)
        wref[nm["word_cell"][0]] = torch.cat([e6[:, di * 3 * H:(di + 1) * 3 * H], wr[:, 3 * H:]], 0)
        for p, n in (("char_cell", 3 * H), ("alpha", H), ("word_cell", 3 * H)):
            wref[nm[p][1]] = z(n, dtype=torch.float64)
    ref = olat.lattice_lstm(xp, wp, lat, lens, wref, H, alpha_shift=shift)
    d_out = torch.randn(B, L, 2 * H, generator=g, dtype=torch.float64)
    (ref * d_out).sum().backward()

    out = fwd(False)[0]
    _close(out, ref.detach())
    valid = _valid(lens)
    assert (out.cpu()[~valid] == 0).all()
    out_t, sv = fwd(True)
    assert torch.equal(out_t, out)
    dx, dw, da = bwd(sv, d_out.float().cuda())
    words = torch.zeros(B, L, Kw, dtype=torch.bool)
    for b in range(B):
        for (p, _, k) in olat.words_of(lat[b], int(lens.clamp(0, L)[b]), Kw):
            words[b, p, k] = True
    for name, got, leaf in (("d_xproj", dx, xp), ("d_wproj", dw, wp), ("d_alpha", da, shift)):
        got = got.cpu().double().view(leaf.shape)
        scale = max(leaf.grad.abs().max().item(), 1e-6)
        if name == "d_xproj":
            assert torch.isfinite(got).all() and (got[~valid] == 0).all()
        else:           # written at the slots of valid words only; the caller zero-fills the rest
            assert torch.isfinite(got[words]).all(), name
        err = (got.nan_to_num(0.0) - leaf.grad).abs().max().item()
        print(f"B={B} R={R}: {name} max err {err:.2e} of scale {scale:.2e}")
        assert err < 1e-4 * scale, name
    again = bwd(sv, d_out.float().cuda())
    for x, y in zip(again, (dx, dw, da)):
        assert torch.equal(x.nan_to_num(7.0), y.nan_to_num(7.0))
