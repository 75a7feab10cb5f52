"""percentilesByKey of a numeric ColumnarRDD on one GPU, end to end and per kernel, against the composition it replaces.

    python scripts/percentilesbykey_e2e.py [--rows 1e8] [--serial-rows 1e7] [--splits 64] [--runs 5]
                                           [--comp-rows 1e6] [--comp-runs 3]

Prints the card and its power limit, then, with int64 keys and float64 values already in HBM and p = [1, 50, 90, 99]:
  - the device percentilesByKey (percentiles.percentiles_columns: the group-by, the segment cut, the digests, the
    absorb chains and the quantiles, the partition cut, then a synchronise) of --rows rows in --splits splits with keys
    uniform over [0, 2^16) and with Zipf(1.1) keys, and of --serial-rows rows under one key in one split (one digest
    built by one warp: the serial worst case): the median time of its materialisation over --runs runs, the segments,
    and the device times of the dpk_tdigest_* kernels (CUDA events) and of everything else (the group-by);
  - the composition (split-tagged groupByKey + quantiles.MergingDigest) of the first --comp-rows uniform rows, every
    partition collected: the median over --comp-runs runs."""
import argparse
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.argv, _argv = sys.argv[:1], sys.argv[1:]      # DparkContext parses sys.argv

from dpark_b200 import DparkContext  # noqa: E402
from dpark_b200 import _native as nv  # noqa: E402
from dpark_b200 import percentiles  # noqa: E402

P_LIST = [1, 50, 90, 99]
KERNELS = ("tdigest_heads", "tdigest_build_short", "tdigest_build_long", "tdigest_merge")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit or "unknown"


def materialize(col, P):
    parts = percentiles.percentiles_columns(col, P, None, [pp / 100. for pp in P_LIST])
    torch.cuda.synchronize()
    if parts is None:
        raise SystemExit("the device path fell back to the composition")
    return sum(int(k.numel()) for k, _ in parts)


def run_case(name, col, P, runs):
    keys = materialize(col, P)
    times = []
    for _ in range(runs):
        t0 = time.perf_counter()
        materialize(col, P)
        times.append(time.perf_counter() - t0)
    nv.prof_enable(True)
    materialize(col, P)
    torch.cuda.synchronize()
    nv.prof_enable(False)
    prof = nv.prof_collect()
    per = {k: sum(ms for lab, ms in prof if lab == k) for k in KERNELS}
    other = sum(ms for lab, ms in prof if lab not in KERNELS)
    n = int(col.keys.numel())
    med = statistics.median(times)
    print("%-8s %d rows, %d splits, P=%d: %d keys; materialisation median %.2f ms (min %.2f, max %.2f, %d runs) = "
          "%.3g rows/s; %s; other kernels (group-by) %.2f ms"
          % (name, n, len(col.splits), P, keys, med * 1e3, min(times) * 1e3, max(times) * 1e3, runs, n / med,
             ", ".join("%s %.3f ms" % (k, per[k]) for k in KERNELS), other), flush=True)


def composition(col, P, runs):
    times = []
    for _ in range(runs):
        t0 = time.perf_counter()
        parts = col._percentiles_rows(P_LIST, P).glom().collect()
        times.append(time.perf_counter() - t0)
    n = int(col.keys.numel())
    med = statistics.median(times)
    print("composition %d rows, %d splits, P=%d: %d keys; median %.2f s (min %.2f, max %.2f, %d runs) = %.3g rows/s"
          % (n, len(col.splits), P, sum(len(p) for p in parts), med, min(times), max(times), runs, n / med),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1e8)
    ap.add_argument("--serial-rows", type=float, default=1e7)
    ap.add_argument("--splits", type=int, default=64)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--comp-rows", type=float, default=1e6)
    ap.add_argument("--comp-runs", type=int, default=3)
    args = ap.parse_args(_argv)
    if not torch.cuda.is_available():
        raise SystemExit("percentilesbykey_e2e.py measures on a CUDA device; none found")
    name, limit = card()
    print("device: %s, power limit %s" % (name, limit), flush=True)
    dc = DparkContext("local")
    g = torch.Generator(device="cuda").manual_seed(1)
    n, M = int(args.rows), args.splits
    vals = torch.randn(n, device="cuda", generator=g, dtype=torch.float64) * 1e3
    uniform = torch.randint(0, 1 << 16, (n,), device="cuda", generator=g)
    run_case("uniform", dc.parallelizeColumns(uniform, vals, M), M, args.runs)
    zipf = torch.from_numpy(np.minimum(np.random.default_rng(2).zipf(1.1, n), 1 << 40)).cuda()
    run_case("zipf1.1", dc.parallelizeColumns(zipf, vals, M), M, args.runs)
    del zipf
    torch.cuda.empty_cache()
    m = int(args.serial_rows)
    run_case("one key", dc.parallelizeColumns(torch.zeros(m, dtype=torch.int64, device="cuda"), vals[:m], 1), 1,
             args.runs)
    c = int(args.comp_rows)
    composition(dc.parallelizeColumns(uniform[:c], vals[:c], M), M, args.comp_runs)


if __name__ == "__main__":
    main()
