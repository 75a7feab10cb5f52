"""top, uniq and hot of a numeric ColumnarRDD on one GPU, end to end and per kernel, against the compositions they replace.

    python scripts/uniq_top_hot_e2e.py [--rows 1e8] [--parts 64] [--runs 5] [--comp-rows 1e6] [--comp-runs 3]

Prints the card and its power limit.  With --rows int64 rows in HBM and --parts splits: top(10) by x[1] of uniform
int64 values, top(10) by the identity with keys in [0, 2^10) (deep ties), top(100000); uniq() of about 4e6 distinct
pairs and of all-distinct pairs (with the peak device memory); hot(10) of Zipf(1.1) pairs.  For each: the median over
--runs runs after one warm-up, the device time of every kernel and the algorithmic bytes/s of the main ones.  Then each
composition over the first --comp-rows rows."""
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
from dpark_b200.rdd import Split  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit or "unknown"


def timed(fn, runs):
    fn()                                          # warm-up
    times = []
    for _ in range(runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return statistics.median(times)


def run_case(name, fn, runs, n, bytes_of):
    """Median time, peak extra device memory, and per kernel the device ms and algorithmic GB/s (bytes_of: label ->
    bytes per call)."""
    med = timed(fn, runs)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    nv.prof_enable(True)
    fn()
    torch.cuda.synchronize()
    nv.prof_enable(False)
    peak = torch.cuda.max_memory_allocated() - base
    ms = {}
    for lab, t in nv.prof_collect():
        lab = "radix passes" if lab.startswith("radix") else lab
        ms[lab] = ms.get(lab, 0.0) + t
    bw = ", ".join("%s %.0f GB/s" % (k, b / (ms[k] * 1e-3) / 1e9) for k, b in bytes_of.items() if ms.get(k))
    print("%-22s %d rows: median %.2f ms (%d runs); peak extra device memory %.2f GB\n    device ms: %s; %s"
          % (name, n, med * 1e3, runs, peak / 1e9, ", ".join("%s %.3f" % kv for kv in sorted(ms.items())), bw),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1e8)
    ap.add_argument("--parts", type=int, default=64)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--comp-rows", type=float, default=1e6)
    ap.add_argument("--comp-runs", type=int, default=3)
    args = ap.parse_args(_argv)
    if not torch.cuda.is_available():
        raise SystemExit("uniq_top_hot_e2e.py measures on a CUDA device; none found")
    print("device: %s, power limit %s" % card(), flush=True)
    dc = DparkContext("local")
    g = torch.Generator(device="cuda").manual_seed(1)
    n, P, runs = int(args.rows), args.parts, args.runs
    second = lambda x: x[1]  # noqa: E731
    ints = lambda hi: torch.randint(0, hi, (n,), device="cuda", generator=g)  # noqa: E731
    vals = torch.randint(-(1 << 62), 1 << 62, (n,), device="cuda", generator=g)
    col = dc.parallelizeColumns(ints(1 << 30), vals, P)
    # sort_keys: V read, 8 (word) + 8 (id) written per row; the first round and the take read 8 per row and word
    one = {"sort_keys": n * 24, "select_tiles": n * 8, "select_write": n * 8}
    run_case("top(10) by x[1]", lambda: col.top(10, key=second), runs, n, one)
    run_case("top(100000) by x[1]", lambda: col.top(100000, key=second), runs, n, one)
    ties = dc.parallelizeColumns(ints(1 << 10), vals, P)
    run_case("top(10) identity ties", lambda: ties.top(10), runs, n,
             {"sort_keys": n * 32, "select_tiles": n * 16, "select_write": n * 16})
    del ties
    # uniq_insert: K + V per row (the owner's pair and the slot are random reads, not credited); emit: 8 per slot
    pairs = {"uniq_insert": n * 16, "uniq_emit": nv.bcast_slots(n) * 8}
    for name, c in (("uniq ~4.2e6 distinct", dc.parallelizeColumns(ints(1 << 21), ints(2), P)),
                    ("uniq all distinct", dc.parallelizeColumns(torch.randperm(n, device="cuda", generator=g), vals, P))):
        run_case(name, lambda: c.uniq(P).columns(Split(0)), runs, n, pairs)
        del c
    rng = np.random.default_rng(3)
    zk = torch.from_numpy(np.minimum(rng.zipf(1.1, n), 1 << 40).astype(np.int64)).cuda()
    cz = dc.parallelizeColumns(zk, torch.from_numpy(rng.integers(0, 4, n)).cuda(), P)
    run_case("hot(10) zipf(1.1)", lambda: cz.hot(10, P), runs, n, pairs)
    torch.cuda.empty_cache()
    m = int(args.comp_rows)
    for label, c, fn in (("top(10) by x[1]", col, lambda r: r.top(10, key=second)),
                         ("uniq()", cz, lambda r: r.uniq(P).glom().collect()),
                         ("hot(10)", cz, lambda r: r.hot(10, P))):
        small = dc.parallelizeColumns(c.keys[:m], c.vals[:m], P)
        comp = timed(lambda: fn(small.map(lambda x: x)), args.comp_runs)
        print("composition %-16s %d rows: median %.3f s (%d runs); device path on the same rows %.2f ms"
              % (label, m, comp, args.comp_runs, timed(lambda: fn(small), runs) * 1e3), flush=True)


if __name__ == "__main__":
    main()
