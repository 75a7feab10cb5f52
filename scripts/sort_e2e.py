"""sort of a numeric ColumnarRDD on one GPU, end to end and per kernel, against the composition it replaces.

    python scripts/sort_e2e.py [--rows 1e8] [--parts 64] [--runs 7] [--comp-rows 1e6] [--comp-runs 3]

Prints the card and its power limit.  With 1e8 rows in HBM (int64 values uniform over +-2^40) it sorts, as the table of
DESIGN.md section 6 lists: int64 keys uniform over [0, 2^26) by x[0], reversed and by the identity, full-range int64
keys and float64 keys by x[0].  For each: the median materialisation time over --runs runs and the device time of every
kernel (the radix passes summed).  Then the composition over the first --comp-rows rows of the first case."""
import argparse
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.argv, _argv = sys.argv[:1], sys.argv[1:]      # DparkContext parses sys.argv

from dpark_b200 import DparkContext  # noqa: E402
from dpark_b200 import _native as nv  # noqa: E402
from dpark_b200 import sorting  # noqa: E402



def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit or "unknown"


def timed(fn, runs):
    times = []
    for _ in range(runs):
        t0 = time.perf_counter()
        out = fn()
        times.append(time.perf_counter() - t0)
    return statistics.median(times), out


def run_case(name, col, key, reverse, P, runs):
    rdd = col.sort(key=key, reverse=reverse, numSplits=P)

    def materialize():
        parts = sorting.sort_columns(col, rdd.order, reverse, rdd.bounds)
        torch.cuda.synchronize()
        return len(parts)
    timed(materialize, 2)
    med, parts = timed(materialize, runs)
    nv.prof_enable(True)
    materialize()
    nv.prof_enable(False)
    ms = {}
    for lab, t in nv.prof_collect():
        lab = "radix passes" if lab.startswith("radix") else lab
        ms[lab] = ms.get(lab, 0.0) + t
    n = int(col.keys.numel())
    print("%-10s %d rows, %d partitions: median %.2f ms (%d runs) = %.3g rows/s; device ms: %s"
          % (name, n, parts, med * 1e3, runs, n / med, ", ".join("%s %.3f" % kv for kv in sorted(ms.items()))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1e8)
    ap.add_argument("--parts", type=int, default=64)
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--comp-rows", type=float, default=1e6)
    ap.add_argument("--comp-runs", type=int, default=3)
    args = ap.parse_args(_argv)
    if not torch.cuda.is_available():
        raise SystemExit("sort_e2e.py measures on a CUDA device; none found")
    name, limit = card()
    print("device: %s, power limit %s" % (name, limit))
    dc = DparkContext("local")
    g = torch.Generator(device="cuda").manual_seed(1)
    n, P = int(args.rows), args.parts
    vals = torch.randint(-(1 << 40), 1 << 40, (n,), device="cuda", generator=g)
    keys = torch.randint(0, 1 << 26, (n,), device="cuda", generator=g)
    col = dc.parallelizeColumns(keys, vals, P)
    run_case("1 x[0]", col, lambda x: x[0], False, P, args.runs)
    run_case("2 x[0] rev", col, lambda x: x[0], True, P, args.runs)
    run_case("3 identity", col, lambda x: x, False, P, args.runs)
    full = torch.randint(-(1 << 63), (1 << 63) - 1, (n,), device="cuda", generator=g)
    run_case("4 full i64", dc.parallelizeColumns(full, vals, P), lambda x: x[0], False, P, args.runs)
    del full
    floats = torch.randn(n, device="cuda", generator=g, dtype=torch.float64)
    run_case("5 float64", dc.parallelizeColumns(floats, vals, P), lambda x: x[0], False, P, args.runs)
    del floats
    torch.cuda.empty_cache()
    m = int(args.comp_rows)
    small = dc.parallelizeColumns(keys[:m], vals[:m], P)
    med, _ = timed(lambda: small.map(lambda x: x).sort(key=lambda x: x[0], numSplits=P).glom().collect(), args.comp_runs)
    print("composition %d rows by x[0]: median %.2f s (%d runs) = %.3g rows/s" % (m, med, args.comp_runs, m / med))


if __name__ == "__main__":
    main()
