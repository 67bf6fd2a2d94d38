#!/usr/bin/env python
"""timeline.py — reads the CSV written by B200_TRACE=<file> (engine.cu: events at the stage boundaries of every picture as
it really ran on its compute lane) and answers what per-kernel tools cannot: how well the pictures overlap.

    B200_TRACE=/tmp/trace.csv python bench.py --steps 16 --warmup 3 --no-cpu-baseline
    python tools/timeline.py /tmp/trace.csv [--from 64]

Prints per-picture stage times under load, the number of pictures in flight over time, the busy fraction of every lane
and the critical-path / throughput bounds of the run.
"""
import argparse
import csv
import statistics


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("--from", dest="first", type=int, default=0, help="ignore the pictures before this index (warm-up)")
    ap.add_argument("--to", dest="last", type=int, default=1 << 30)
    a = ap.parse_args()
    rows = [r for r in csv.DictReader(open(a.csv))]
    pics = []
    for r in rows:
        i = int(r["picture"])
        if i < a.first or i >= a.last:
            continue
        st = float(r["start_us"])
        ends = [float(r[k]) for k in ("mc_us", "residual_us", "intra_us", "deblock_us", "sao_us")]
        pics.append(dict(i=i, lane=int(r["lane"]), n_ref=int(r["n_ref"]), start=st, ends=ends, end=st + ends[-1]))
    if not pics:
        raise SystemExit("no pictures in range")
    t0, t1 = min(p["start"] for p in pics), max(p["end"] for p in pics)
    span = t1 - t0
    print(f"{len(pics)} pictures in {span / 1e3:.2f} ms -> {len(pics) / span * 1e6:.0f} pictures/s")
    names = ("mc", "residual", "intra", "deblock", "sao")
    for kind, sel in (("inter", [p for p in pics if p["n_ref"]]), ("intra-only", [p for p in pics if not p["n_ref"]])):
        if not sel:
            continue
        d = [[p["ends"][0]] + [p["ends"][k] - p["ends"][k - 1] for k in range(1, 5)] for p in sel]
        med = [statistics.median(x[k] for x in d) for k in range(5)]
        tot = statistics.median(p["ends"][-1] for p in sel)
        print(f"  {kind:10s} pictures: {len(sel):4d}, median residence {tot:7.1f} us  (" + ", ".join(f"{n} {m:.0f}" for n, m in zip(names, med)) + ")")
    # pictures in flight (device side) sampled on a fine grid
    step = span / 2000
    hist = {}
    for k in range(2000):
        t = t0 + (k + 0.5) * step
        n = sum(1 for p in pics if p["start"] <= t < p["end"])
        hist[n] = hist.get(n, 0) + 1
    print("  pictures in flight (share of time): " + ", ".join(f"{n}: {100 * c / 2000:.0f}%" for n, c in sorted(hist.items())))
    lanes = sorted(set(p["lane"] for p in pics))
    for l in lanes:
        busy = sum(p["end"] - p["start"] for p in pics if p["lane"] == l)
        print(f"  lane {l}: {sum(1 for p in pics if p['lane'] == l):4d} pictures, busy {100 * busy / span:.0f}%")
    serial = sum(p["end"] - p["start"] for p in pics)
    print(f"  sum of residences {serial / 1e3:.2f} ms = {serial / span:.2f} x the span (average pictures in flight)")


if __name__ == "__main__":
    main()
