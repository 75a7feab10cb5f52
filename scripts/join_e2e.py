"""Join of two numeric ColumnarRDDs on one GPU, end to end and per kernel, against the row path.

    python scripts/join_e2e.py [--left 1e8] [--right 1e7] [--runs 7] [--rows-left 1e6] [--rows-right 1e5]

Prints the card and its power limit, then per case (uniform keys over [0, 2^26); the same plus one key with 3000 rows
on each side) the median time of the join's materialisation (columns() of every partition, then a synchronise; the
inputs are already in HBM), the device times of dpk_join_count and dpk_join_emit (CUDA events) and the emit's
algorithmic bytes per second, and last the row path (ctx.parallelize rows, cogroup + flatMap) at a smaller size."""
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


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit or "unknown"


def emit_bytes(n_out, lw, rw):
    """Algorithmic bytes of dpk_join_emit for an inner join: per output row the key and both values written, the two
    row ids and both values read."""
    return n_out * (8 + lw + rw) + n_out * (8 + 8 + lw + rw)


def materialize(a, b, P):
    out = a.join(b, P)
    cols = [out.columns(sp) for sp in out.splits]
    torch.cuda.synchronize()
    return sum(int(c[0].numel()) for c in cols)


def run_case(dc, name, lk, rk, P, runs):
    dev = lk.device
    lv = torch.arange(lk.numel(), dtype=torch.int64, device=dev)
    rv = torch.arange(rk.numel(), dtype=torch.int64, device=dev)
    a = dc.parallelizeColumns(lk, lv, 8)
    b = dc.parallelizeColumns(rk, rv, 8)
    for _ in range(2):
        n_out = materialize(a, b, P)
    times = []
    for _ in range(runs):
        t0 = time.perf_counter()
        materialize(a, b, P)
        times.append(time.perf_counter() - t0)
    nv.prof_enable(True)
    materialize(a, b, P)
    nv.prof_enable(False)
    prof = nv.prof_collect()
    kt = {lab: sum(ms for l2, ms in prof if l2 == lab) for lab in ("join_count", "join_emit")}
    med = statistics.median(times)
    nin = lk.numel() + rk.numel()
    eb = emit_bytes(n_out, 8, 8)
    print("%-8s left %d x right %d rows, P=%d: %d output rows; materialisation median %.2f ms (min %.2f, max %.2f, "
          "%d runs) = %.3g input rows/s; dpk_join_count %.3f ms, dpk_join_emit %.3f ms = %.1f GB/s algorithmic"
          % (name, lk.numel(), rk.numel(), P, n_out, med * 1e3, min(times) * 1e3, max(times) * 1e3, runs, nin / med,
             kt["join_count"], kt["join_emit"], eb / (kt["join_emit"] * 1e-3) / 1e9 if kt["join_emit"] else 0.0))
    return med


def row_path(dc, nl, nr, P):
    rng = np.random.default_rng(2)
    kr = max(1, int((1 << 26) * nl / 1e8))     # at a 10:1 size ratio: the output rows per input row of the cases above
    ra = list(zip(rng.integers(0, kr, nl).tolist(), range(nl)))
    rb = list(zip(rng.integers(0, kr, nr).tolist(), range(nr)))
    a, b = dc.parallelize(ra, 8), dc.parallelize(rb, 8)
    a.join(b, P).glom().collect()                       # warm-up
    t0 = time.perf_counter()
    n_out = sum(len(p) for p in a.join(b, P).glom().collect())
    dt = time.perf_counter() - t0
    print("row path left %d x right %d rows, P=%d: %d output rows in %.2f s = %.3g input rows/s"
          % (nl, nr, P, n_out, dt, (nl + nr) / dt))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--left", type=float, default=1e8)
    ap.add_argument("--right", type=float, default=1e7)
    ap.add_argument("--parts", type=int, default=64)
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--rows-left", type=float, default=1e6)
    ap.add_argument("--rows-right", type=float, default=1e5)
    args = ap.parse_args(_argv)
    if not torch.cuda.is_available():
        raise SystemExit("join_e2e.py measures on a CUDA device; none found")
    name, limit = card()
    print("device: %s, power limit %s" % (name, limit))
    dc = DparkContext("local")
    g = torch.Generator(device="cuda").manual_seed(1)
    nl, nr = int(args.left), int(args.right)
    lk = torch.randint(0, 1 << 26, (nl,), device="cuda", generator=g)
    rk = torch.randint(0, 1 << 26, (nr,), device="cuda", generator=g)
    run_case(dc, "uniform", lk, rk, args.parts, args.runs)
    hot = 3000
    lk[torch.randperm(nl, device="cuda", generator=g)[:hot]] = 1 << 27
    rk[torch.randperm(nr, device="cuda", generator=g)[:hot]] = 1 << 27
    run_case(dc, "skewed", lk, rk, args.parts, args.runs)
    del lk, rk
    torch.cuda.empty_cache()
    row_path(dc, int(args.rows_left), int(args.rows_right), args.parts)


if __name__ == "__main__":
    main()
