"""CPU: `ner_rnn_plan`, the one place that decides which instantiation of the BiLSTM, BiGRU and Lattice LSTM recurrence
kernels serves a call.

The plan is a pure function of (kernel, B, H, Kw, number of SMs).  It is checked here against the cluster, shared-memory
and rows-per-cluster rules of the kernels written out independently in Python, on a grid that puts B at every boundary
where the rows per cluster flip, and against the process environment, which must not enter into it.
"""
import ctypes
import itertools

from chinesener_b200 import _lib

LSTM_FWD, LSTM_BWD, GRU_FWD, GRU_BWD, LAT_FWD, LAT_BWD = range(6)
OK, INVALID, UNSUPPORTED = 0, -1, -2
SMS = (132, 114, 66, 16)        # H100 SXM, H100 PCIe, and two partial devices
HS = range(4, 533, 4)           # past the largest H any kernel supports (LSTM: 304, GRU: 336, lattice: 240)
KWS = range(1, 9)


def plan(kernel, B, H, Kw=1, sms=132):
    R, C, res = ctypes.c_int(-7), ctypes.c_int(-7), ctypes.c_int(-7)
    st = _lib.lib().ner_rnn_plan(kernel, B, H, Kw, sms, ctypes.byref(R), ctypes.byref(C), ctypes.byref(res))
    return st, R.value, C.value, res.value


# ---- the rules, restated from the kernels' shared-memory layouts (csrc/bilstm.cu, bilstm_bwd.cu, bigru.cu, lattice.cu)

def _first_cluster(H, fits):
    return next((C for C in (1, 2, 4, 8) if H % C == 0 and fits(C)), 0)


def _rows(B, C, sms):           # 1 row per cluster while 2 B C CTAs fit the SMs, 4 once 2 waves would not
    return 4 if 2 * ((B + 1) // 2) * C > 2 * sms else 2 if 2 * B * C > sms else 1


def _lstm_fwd(B, H, sms):
    if H % 4:
        return UNSUPPORTED, 0, 0, 0
    C = _first_cluster(H, lambda C: H * 4 * (H // C) * 4 <= 190 * 1024 and 4 * (H // C) <= 512)   # W_h slice, fp32
    if not C:
        return UNSUPPORTED, 0, 0, 0
    R = _rows(B, C, sms)
    if H == 128 and 4 * (H // C) <= 256:                       # one W_h column per thread, in registers
        return OK, 8 if 2 * -(-B // 4) * C > sms else 2 if R == 2 else 1, C, 1
    return OK, R, C, 0


def _lstm_bwd(B, H, sms):
    C = _first_cluster(H, lambda C: 4 * H * (H // C + 1) * 4 <= 180 * 1024)                       # [4H][H/C + 1] fp32
    if not C or H // C > 256:
        return UNSUPPORTED, 0, 0, 0
    return OK, min(_rows(B, C, sms), 2), C, int(H == 128 and C == 2)


def _gru(B, H, sms):
    if H % 4:
        return UNSUPPORTED, 0, 0, 0
    H4 = H // 4

    def fits(C):                 # 4 lanes per unit; gate and candidate float4 streams + 3 double-buffered vectors at R = 4
        NT = 4 * (H // C)
        return NT <= 512 and ((H4 + 1) // 2 + (H4 + 3) // 4) * NT * 16 + 6 * 4 * H * 4 + 64 <= 200 * 1024
    C = _first_cluster(H, fits)
    return (OK, _rows(B, C, sms), C, 0) if C else (UNSUPPORTED, 0, 0, 0)


def _lattice(B, H, Kw, sms):
    if Kw > 8:
        return UNSUPPORTED, 0, 0, 0
    lst = 9 * 8                 # word-list entries: 9 starts x 8 slots

    def fits(C, R):
        HU = H // C
        fwd = (7 * H * HU + 2 * R * H + R * 6 * HU + R * 8 * H + 2 * R * 10 * Kw * HU) * 4 + (2 * R * lst + 3 * R) * 4
        bwd = (7 * H * HU + 2 * R * 6 * H + R * HU + R * 8 * H + R * 10 * Kw * HU) * 4 + (2 * R * lst + 3 * R) * 4
        return R * HU <= 512 and fwd <= 226 * 1024 and bwd <= 226 * 1024

    R, C = 1, _first_cluster(H, lambda C: fits(C, 1))
    if not C:
        return UNSUPPORTED, 0, 0, 0
    for r in (2, 4):            # more rows per cluster only while one wave of clusters does not fit
        if 2 * -(-B // R) * C <= sms:
            break
        c = _first_cluster(H, lambda C: fits(C, r))
        if not c:
            break
        R, C = r, c
    return OK, R, C, 0


def expected(kernel, B, H, Kw=1, sms=132):
    if B < 0 or H < 1 or sms < 1 or (kernel >= LAT_FWD and Kw < 1):
        return INVALID, 0, 0, 0
    if kernel == LSTM_FWD:
        return _lstm_fwd(B, H, sms)
    if kernel == LSTM_BWD:
        return _lstm_bwd(B, H, sms)
    if kernel in (GRU_FWD, GRU_BWD):
        return _gru(B, H, sms)
    return _lattice(B, H, Kw, sms)


def _boundaries(sms, Cs=(1, 2, 4, 8)):
    """Every B where a rule of _rows, the LSTM's R = 8 rule or the lattice's wave test can flip, +-1."""
    out = {0, 1, 2, 3}
    for C in Cs:
        for edge in (sms // (2 * C), sms // C, 2 * (sms // C), 4 * (sms // (2 * C)), 2 * (sms // (2 * C))):
            out.update(edge + d for d in (-1, 0, 1, 2))
    out.update((1000, 4096))
    return sorted(b for b in out if b >= 0)


def test_plan_matches_the_rules_on_a_grid():
    n = 0
    for sms in SMS:
        for B, H in itertools.product(_boundaries(sms), HS):
            for kernel in (LSTM_FWD, LSTM_BWD, GRU_FWD, GRU_BWD):
                assert plan(kernel, B, H, 1, sms) == expected(kernel, B, H, 1, sms), (kernel, B, H, sms)
                n += 1
            for Kw in KWS:
                for kernel in (LAT_FWD, LAT_BWD):
                    assert plan(kernel, B, H, Kw, sms) == expected(kernel, B, H, Kw, sms), (kernel, B, H, Kw, sms)
                    n += 1
    assert n > 100000


def test_every_rows_value_is_reached_and_flips_where_the_rules_say():
    # B where R flips, on a 132-SM H100 (C = 2 for H = 128 and 200)
    assert [plan(LSTM_FWD, B, 200)[1] for B in (16, 17, 33, 34, 66, 67)] == [1, 2, 2, 2, 2, 4]
    assert [plan(LSTM_FWD, B, 128)[1] for B in (33, 34, 132, 133)] == [1, 2, 2, 8]
    assert [plan(LSTM_BWD, B, 128)[1] for B in (33, 34, 1000)] == [1, 2, 2]
    assert [plan(GRU_FWD, B, 128)[1] for B in (33, 34, 132, 133)] == [1, 2, 2, 4]
    assert {plan(k, 64, 100, 4)[1:3] for k in (LAT_FWD, LAT_BWD)} == {(2, 2)}
    # the same B reaches different instantiations on a 114-SM H100
    assert plan(LSTM_FWD, 30, 128, 1, 114)[1] == 2 and plan(LSTM_FWD, 30, 128, 1, 132)[1] == 1
    # the register-resident LSTM kernels serve H = 128 alone
    assert all(plan(k, 8, H)[3] == int(H == 128) for k in (LSTM_FWD, LSTM_BWD) for H in (64, 124, 128, 132, 200, 256))


def test_unsupported_shapes_give_the_launchers_status():
    for k in (LSTM_FWD, GRU_FWD, GRU_BWD):
        assert plan(k, 8, 130)[0] == UNSUPPORTED                       # H % 4 != 0
    assert plan(LSTM_BWD, 8, 130)[0] == OK                             # the BPTT kernel takes any H its slice holds
    # the largest H each kernel holds, and the next multiple of 8
    for k, H in ((LSTM_FWD, 304), (LSTM_BWD, 296), (GRU_FWD, 336), (GRU_BWD, 336), (LAT_FWD, 240), (LAT_BWD, 240)):
        assert plan(k, 8, H)[0] == OK and plan(k, 8, H + 8)[0] == UNSUPPORTED, k
    assert plan(LSTM_FWD, 8, 228)[0] == UNSUPPORTED                    # 4 CTAs do not hold it, 8 do not divide it
    assert plan(LAT_FWD, 8, 100, 8)[0] == OK and plan(LAT_FWD, 8, 100, 9)[0] == UNSUPPORTED
    for k in range(6):
        assert plan(k, -1, 128, 4) == (INVALID, 0, 0, 0)
        assert plan(k, 8, 0, 4) == (INVALID, 0, 0, 0)
        assert plan(k, 8, 128, 4, 0) == (INVALID, 0, 0, 0)
    assert plan(LAT_FWD, 8, 64, 0)[0] == INVALID and plan(LSTM_FWD, 8, 64, 0)[0] == OK   # Kw read only by the lattice
    assert plan(6, 8, 128)[0] == INVALID and plan(-1, 8, 128)[0] == INVALID
    assert _lib.lib().ner_rnn_plan(LSTM_FWD, 64, 128, 0, 132, None, None, None) == OK


def test_the_launchers_return_the_plans_status_without_a_gpu():
    """Shapes the plan refuses are refused by the launchers with the same status, before any launch."""
    h, p = _lib.lib(), ctypes.c_void_p(16)
    assert h.ner_bilstm_recurrence(p, p, p, p, p, 8, 4, 130, 0, 1.0, None, None, None, None, 1.0, 0, None) == UNSUPPORTED
    assert h.ner_bigru_recurrence(p, p, p, p, p, 8, 4, 344, 6 * 344, 0, None, None, None, None, 1.0, 0, None) \
        == UNSUPPORTED
    assert h.ner_bigru_recurrence_bwd(p, p, p, p, p, p, p, 8, 4, 130, 0, 1.0, 0, None) == UNSUPPORTED
    assert h.ner_lattice_recurrence(*[p] * 9, 8, 4, 100, 9, *[None] * 8) == UNSUPPORTED
    assert h.ner_lattice_recurrence_bwd(*[p] * 16, 8, 4, 100, 9, None) == UNSUPPORTED


def test_environment_does_not_enter_the_plan(monkeypatch):
    shapes = [(k, B, H, Kw, s) for k in range(6) for B in (1, 17, 64, 256) for H in (100, 128, 200)
              for Kw in (1, 4) for s in (132, 114)]
    before = [plan(*s) for s in shapes]
    for value in ("1", "2", "8"):        # the variables that once chose the BiLSTM rows and the BPTT variant
        monkeypatch.setenv("NER_BILSTM_ROWS", value)
        monkeypatch.setenv("NER_BPTT_VARIANT", value)
        assert [plan(*s) for s in shapes] == before
