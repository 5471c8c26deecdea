"""Summarise an ncu launch list (`--metrics gpu__time_duration.sum --csv`): time per kernel family and its share.
usage: python scripts/launch_shares.py <launches.csv> [first_row last_row]"""
import csv
import re
import sys
from collections import OrderedDict

FAMILIES = OrderedDict([
    ("gemm (wgmma)", r"gemm_bf16_tc"), ("attention", r"attention"), ("bilstm recurrence", r"bilstm"),
    ("layernorm / embed", r"layernorm|embed"), ("crf", r"crf_"), ("label projection", r"dense_small"),
    ("cast / pack / gelu / misc", r".*"),
])


def main(path, lo=None, hi=None):
    rows = []
    with open(path, newline="") as f:
        lines = [l for l in f if l.startswith('"')]
    for r in csv.DictReader(lines):
        if r.get("Metric Name") == "gpu__time_duration.sum":
            v = float(r["Metric Value"].replace(",", ""))
            unit = r["Metric Unit"]
            v *= {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}.get(unit, 1e-3)
            rows.append((r["Kernel Name"], v))
    rows = rows[lo:hi]
    tot = sum(v for _, v in rows)
    fam = OrderedDict((k, [0.0, 0]) for k in FAMILIES)
    for name, v in rows:
        for k, pat in FAMILIES.items():
            if re.search(pat, name):
                fam[k][0] += v
                fam[k][1] += 1
                break
    print(f"{path}: {len(rows)} launches, {tot:.1f} us")
    for k, (v, n) in fam.items():
        print(f"  {k:28s} {v:10.1f} us  {n:5d} launches  {100 * v / tot:5.1f} %")


if __name__ == "__main__":
    a = sys.argv[1:]
    main(a[0], int(a[1]) if len(a) > 1 else None, int(a[2]) if len(a) > 2 else None)
