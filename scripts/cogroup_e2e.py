"""Cogroup and groupByKey of numeric ColumnarRDDs on one GPU, end to end and per kernel, against the row path.

    python scripts/cogroup_e2e.py [--left 1e8] [--right 1e7] [--group 1e8] [--group-host 1e7] [--runs 7]
                                  [--rows-left 1e6] [--rows-right 1e5]

Prints the card and its power limit, then:
  - a 2-way cogroup (keys uniform over [0, 2^26), int64 values, inputs already in HBM): the median time of its
    materialisation (columns() of every partition, then a synchronise), the device times of dpk_cogroup_count and
    dpk_cogroup_emit (CUDA events, the emit summed over its one launch per input) and the emit's algorithmic bytes
    per second;
  - the same for the device part of a groupByKey of one ColumnarRDD, and one run of a groupByKey of its first
    --group-host rows to the host lists its ShuffledRDD hands out;
  - the row path (ctx.parallelize rows, CoGroupedRDD / the row-id group-by) at a smaller size."""
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
from dpark_b200 import join  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit or "unknown"


def emit_bytes(n_out, w):
    """Algorithmic bytes of dpk_cogroup_emit: per output row its row id and its value read, the value written."""
    return n_out * (8 + w + w)


def materialize(rdds, P):
    parts = join.cogroup_columns(rdds, P, None)
    torch.cuda.synchronize()
    return sum(int(p[0].numel()) for p in parts)


def run_case(name, rdds, P, runs):
    for _ in range(2):
        groups = materialize(rdds, P)
    times = []
    for _ in range(runs):
        t0 = time.perf_counter()
        materialize(rdds, P)
        times.append(time.perf_counter() - t0)
    nv.prof_enable(True)
    materialize(rdds, P)
    nv.prof_enable(False)
    prof = nv.prof_collect()
    kt = {lab: sum(ms for l2, ms in prof if l2 == lab) for lab in ("cogroup_count", "cogroup_emit")}
    med = statistics.median(times)
    nin = sum(int(r.keys.numel()) for r in rdds)
    eb = emit_bytes(nin, 8)
    print("%-10s %s rows, P=%d: %d keys; materialisation median %.2f ms (min %.2f, max %.2f, %d runs) = %.3g input "
          "rows/s; dpk_cogroup_count %.3f ms, dpk_cogroup_emit %.3f ms = %.1f GB/s algorithmic"
          % (name, " + ".join(str(int(r.keys.numel())) for r in rdds), P, groups, med * 1e3, min(times) * 1e3,
             max(times) * 1e3, runs, nin / med, kt["cogroup_count"], kt["cogroup_emit"],
             eb / (kt["cogroup_emit"] * 1e-3) / 1e9 if kt["cogroup_emit"] else 0.0))


def group_to_host(dc, col, P):
    t0 = time.perf_counter()
    g = col.groupByKey(P)
    n = sum(len(g.columns(sp)[0]) for sp in g.splits)
    dt = time.perf_counter() - t0
    print("groupByKey %d rows, P=%d, to host lists (one run): %d keys in %.2f s = %.3g input rows/s"
          % (col.keys.numel(), P, n, dt, col.keys.numel() / dt))


def row_path(dc, nl, nr, P):
    rng = np.random.default_rng(2)
    kr = max(1, int((1 << 26) * nl / 1e8))     # keys per row as in the cases above
    ra = list(zip(rng.integers(0, kr, nl).tolist(), range(nl)))
    rb = list(zip(rng.integers(0, kr, nr).tolist(), range(nr)))
    a, b = dc.parallelize(ra, 8), dc.parallelize(rb, 8)
    a.groupWith(b, P).glom().collect()                     # warm-up
    t0 = time.perf_counter()
    n = sum(len(p) for p in a.groupWith(b, P).glom().collect())
    dt = time.perf_counter() - t0
    print("row path cogroup %d + %d rows, P=%d: %d keys in %.2f s = %.3g input rows/s"
          % (nl, nr, P, n, dt, (nl + nr) / dt))
    t0 = time.perf_counter()
    n = sum(len(p) for p in a.groupByKey(P).glom().collect())
    dt = time.perf_counter() - t0
    print("row path groupByKey %d rows, P=%d: %d keys in %.2f s = %.3g input rows/s" % (nl, P, n, dt, nl / dt))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--left", type=float, default=1e8)
    ap.add_argument("--right", type=float, default=1e7)
    ap.add_argument("--group", type=float, default=1e8)
    ap.add_argument("--group-host", type=float, default=1e7)
    ap.add_argument("--parts", type=int, default=64)
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--rows-left", type=float, default=1e6)
    ap.add_argument("--rows-right", type=float, default=1e5)
    args = ap.parse_args(_argv)
    if not torch.cuda.is_available():
        raise SystemExit("cogroup_e2e.py measures on a CUDA device; none found")
    name, limit = card()
    print("device: %s, power limit %s" % (name, limit))
    dc = DparkContext("local")
    g = torch.Generator(device="cuda").manual_seed(1)
    nl, nr = int(args.left), int(args.right)
    lk = torch.randint(0, 1 << 26, (nl,), device="cuda", generator=g)
    rk = torch.randint(0, 1 << 26, (nr,), device="cuda", generator=g)
    a = dc.parallelizeColumns(lk, torch.arange(nl, dtype=torch.int64, device="cuda"), 8)
    b = dc.parallelizeColumns(rk, torch.arange(nr, dtype=torch.int64, device="cuda"), 8)
    run_case("cogroup", [a, b], args.parts, args.runs)
    del a, b, lk, rk
    torch.cuda.empty_cache()
    n = int(args.group)
    k = torch.randint(0, 1 << 26, (n,), device="cuda", generator=g)
    col = dc.parallelizeColumns(k, torch.arange(n, dtype=torch.int64, device="cuda"), 8)
    run_case("groupByKey", [col], args.parts, args.runs)
    group_to_host(dc, dc.parallelizeColumns(k[:int(args.group_host)], col.vals[:int(args.group_host)], 8), args.parts)
    del col, k
    torch.cuda.empty_cache()
    row_path(dc, int(args.rows_left), int(args.rows_right), args.parts)


if __name__ == "__main__":
    main()
