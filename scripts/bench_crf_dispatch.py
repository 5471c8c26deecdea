"""ner_crf_viterbi per kernel plan: CUDA-event timings of the shapes that decide which Viterbi kernels are worth keeping.

usage: python scripts/bench_crf_dispatch.py [--lib NAME=OTHER/libner_b200.so ...] [--seconds 0.5] [--rounds 3]

Times the package's library ("tree") and any other builds of it given with --lib on the same inputs, alternating the
libraries round by round so that clock drift hits all alike, and checks that they return the same tags.  Every point is
warmed up and then timed over at least --seconds of back-to-back launches between one pair of events; the median over
--rounds is reported with the spread (max - min) / median.  GB/s is the algorithm's bytes (computed from the shape: logits
and lengths in, tags and scores out) over that time.  The card's name and power limit are printed with the numbers.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from chinesener_b200 import _lib  # noqa: E402

# (B, L, K): big batches the TMA kernel cannot take (L*K % 4 != 0), the roofline shape, and the lane-per-tag regime
SHAPES = [(19000, 150, 7), (9600, 37, 7), (9490, 9, 3), (262144, 127, 10), (262144, 128, 10), (64, 128, 10), (4096, 128, 10)]


def viterbi_bytes(B, L, K):
    return B * L * K * 4 + 4 * B + 4 * K * K + B * L * 4 + 4 * B


def load(path):
    h = _lib.lib() if path is None else ctypes.CDLL(os.path.abspath(path))
    fn = h.ner_crf_viterbi
    fn.restype, fn.argtypes = _lib.SIGNATURES["ner_crf_viterbi"]
    plan = getattr(h, "ner_crf_viterbi_plan", None)      # absent from builds that predate the plan query
    if plan is not None:
        plan.restype, plan.argtypes = _lib.SIGNATURES["ner_crf_viterbi_plan"]
    return fn, plan


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH")
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_crf_dispatch.py needs a CUDA device: timings come from the GPU or not at all")
    libs = {"tree": load(None)}
    for spec in args.lib:
        name, path = spec.split("=", 1)
        libs[name] = load(path)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"# card: {card()}  ({sms} SMs)")
    print(f"# >= {args.seconds} s of launches per timing, median of {args.rounds} alternating rounds, spread = (max - min) / median")
    rows = []
    g = torch.Generator(device="cuda").manual_seed(1234)
    for B, L, K in SHAPES:
        x = torch.randn(B, L, K, device="cuda", generator=g) * 2
        tr = torch.randn(K, K, device="cuda", generator=g)
        lens = torch.randint(1, L + 1, (B,), device="cuda", generator=g, dtype=torch.int32)
        best = torch.empty(B, device="cuda")
        outs, iters, times = {}, {}, {n: [] for n in libs}

        def call(name, tags):
            rc = libs[name][0](x.data_ptr(), lens.data_ptr(), tr.data_ptr(), tags.data_ptr(), best.data_ptr(), B, L, K,
                               _lib.stream())
            if rc != 0:
                raise RuntimeError(f"{name}: ner_crf_viterbi({B}, {L}, {K}) returned {rc}")

        def timed(name, tags, n):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                call(name, tags)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / n

        for name in libs:                                # warm-up, result, and the launch count that fills --seconds
            tags = torch.full((B, L), -1, dtype=torch.int32, device="cuda")
            for _ in range(3):
                call(name, tags)
            outs[name] = tags
            iters[name] = max(5, int(args.seconds * 1e3 / timed(name, tags, 5)) + 1)
        for _ in range(args.rounds):
            for name in libs:
                times[name].append(timed(name, outs[name], iters[name]))
        for name, (_, plan) in libs.items():
            ts = sorted(times[name])
            med = ts[len(ts) // 2]
            rows.append({"B": B, "L": L, "K": K, "lib": name,
                         "plan": _lib.VIT_PLANS[plan(B, L, K, 1, sms)] if plan else "-",
                         "ms": round(med, 5), "spread": round((ts[-1] - ts[0]) / med, 4), "launches": iters[name],
                         "GBps": round(viterbi_bytes(B, L, K) / med / 1e6, 1),
                         "tags_equal_tree": bool(torch.equal(outs[name], outs["tree"]))})
        del x, outs
    print(f"{'B':>7s} {'L':>4s} {'K':>3s} {'lib':12s} {'plan':12s} {'ms':>10s} {'spread':>7s} {'GB/s':>8s} {'launches':>8s} same tags")
    for r in rows:
        print(f"{r['B']:7d} {r['L']:4d} {r['K']:3d} {r['lib']:12s} {r['plan']:12s} {r['ms']:10.5f} {r['spread']:7.2%} "
              f"{r['GBps']:8.1f} {r['launches']:8d} {r['tags_equal_tree']}")
    print(json.dumps({"card": card(), "sms": sms, "rows": rows}))


if __name__ == "__main__":
    main()
