"""GPU time per kernel family of warmed-up bert_bilstm_crf PREDICT calls (torch.profiler, CUDA activities).

Two settings: one 64-sentence batch per call on one stream (tile_n = 0), and bench.py's pipeline (calls alternating over
four streams, TILE_AUTO_THROUGHPUT).  Families are those of scripts/launch_shares.py.

usage: python scripts/prof_predict_kernels.py [--calls N]
"""
import os
import re
import sys
from collections import OrderedDict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from chinesener_b200 import engine, ops, synthetic  # noqa: E402
from launch_shares import FAMILIES  # noqa: E402


def families(events):
    fam = OrderedDict((k, [0.0, 0]) for k in FAMILIES)
    for name, us in events:
        for k, pat in FAMILIES.items():
            if re.search(pat, name):
                fam[k][0] += us
                fam[k][1] += 1
                break
    return fam


def profile(est, batches, calls, streams):
    side = [torch.cuda.Stream() for _ in range(streams)]
    ops.DEFAULT_TILE = ops.TILE_AUTO_THROUGHPUT if streams > 1 else 0
    try:
        def run(n):
            for j in range(n):
                with torch.cuda.stream(side[j % streams]):
                    est.predict_device(batches[j % len(batches)])
            for st in side:
                torch.cuda.current_stream().wait_stream(st)
        run(2 * streams)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            run(calls)
            e.record()
            torch.cuda.synchronize()
    finally:
        ops.DEFAULT_TILE = 0
    kern = [(ev.name, ev.time_range.elapsed_us()) for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA
            and not ev.name.startswith(("Memcpy", "Memset"))]
    return families(kern), s.elapsed_time(e) / calls, len(kern) / calls


def main():
    calls = int(sys.argv[sys.argv.index("--calls") + 1]) if "--calls" in sys.argv else 20
    est = engine.Estimator("bert_bilstm_crf", dict(synthetic.data_params(128, 10), pretrain_dir=""))
    batches = [est.to_device(synthetic.msra_batch(64, 128, seed=1234 + i)) for i in range(4)]
    print(f"# card: {torch.cuda.get_device_name()}")
    for label, streams in (("1 stream, 1 batch per call, tile_n=0", 1), ("4 streams, 1 batch per call, TILE_AUTO_THROUGHPUT", 4)):
        fam, ms, launches = profile(est, batches, calls, streams)
        tot = sum(v for v, _ in fam.values())
        print(f"## {label}: {calls} calls, {ms:.3f} ms per call (events, profiler on), {launches:.0f} kernels per call")
        for k, (us, n) in fam.items():
            print(f"  {k:28s} {us / calls:9.1f} us/call  {n / calls:6.1f} launches/call  {100 * us / tot:5.1f} %")


if __name__ == "__main__":
    main()
