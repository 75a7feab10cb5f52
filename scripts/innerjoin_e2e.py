"""innerJoin of two numeric ColumnarRDDs on one GPU, end to end and per kernel, against the device join and the row
path.

    python scripts/innerjoin_e2e.py [--big 1e8] [--smalls 1e3,1e5,1e7] [--runs 7] [--parts 64] [--rows-big 1e6]

Prints the card and its power limit, then per workload (big int64 keys uniform over [0, 2^22) against a small side over
the same range; the 1e5 side once more with one key of 1e4 small rows that 1e3 big rows hit) the median time of the
materialisation (columns() of every split, then a synchronise; the inputs are already in HBM), the device times of
dpk_bcast_build / dpk_bcast_probe / dpk_bcast_emit (CUDA events) and the probe's and emit's algorithmic bytes per
second, and the median time of the device join (RDD.join, P partitions) of the same inputs.  Last the row path
(ctx.parallelize rows: a dict on the host and a flatMap) at a smaller big side."""
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

KEY_RANGE = 1 << 22


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit or "unknown"


def probe_bytes(n, kw):
    """Algorithmic bytes of dpk_bcast_probe: per big row the key read, its group (4) and match count (8) written; table
    reads are not credited."""
    return n * (kw + 4 + 8)


def emit_bytes(n_out, kw, lw, rw):
    """Algorithmic bytes of dpk_bcast_emit: per output row the key and both values written, the key, the left value,
    the small row id and the right value read."""
    return n_out * (kw + lw + rw) + n_out * (kw + lw + 8 + rw)


def timed(fn, runs):
    fn()
    fn()
    times = []
    for _ in range(runs):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return times


def materialize(rdd):
    cols = [rdd.columns(sp) for sp in rdd.splits]
    torch.cuda.synchronize()
    return sum(int(c[0].numel()) for c in cols)


def run_case(dc, name, bk, bv, sk, sv, P, runs):
    big = dc.parallelizeColumns(bk, bv, 8)
    small = dc.parallelizeColumns(sk, sv, 8)
    n_out = materialize(big.innerJoin(small))
    times = timed(lambda: materialize(big.innerJoin(small)), runs)
    nv.prof_enable(True)
    materialize(big.innerJoin(small))
    nv.prof_enable(False)
    prof = nv.prof_collect()
    kt = {lab: sum(ms for l2, ms in prof if l2 == lab) for lab in ("bcast_build", "bcast_probe", "bcast_emit")}
    med = statistics.median(times)
    n = bk.numel()
    pb = probe_bytes(n, bk.element_size())
    eb = emit_bytes(n_out, bk.element_size(), bv.element_size(), sv.element_size())
    print("%-9s big %d x small %d rows: %d output rows; materialisation median %.2f ms (min %.2f, max %.2f, %d runs) "
          "= %.3g big rows/s; build %.3f ms, probe %.3f ms = %.1f GB/s, emit %.3f ms = %.1f GB/s algorithmic"
          % (name, n, sk.numel(), n_out, med * 1e3, min(times) * 1e3, max(times) * 1e3, runs, n / med,
             kt["bcast_build"], kt["bcast_probe"], pb / (kt["bcast_probe"] * 1e-3) / 1e9 if kt["bcast_probe"] else 0,
             kt["bcast_emit"], eb / (kt["bcast_emit"] * 1e-3) / 1e9 if kt["bcast_emit"] else 0.0))
    jt = timed(lambda: materialize(big.join(small, P)), runs)
    print("%-9s device join of the same inputs, P=%d: median %.2f ms (min %.2f, max %.2f, %d runs)"
          % (name, P, statistics.median(jt) * 1e3, min(jt) * 1e3, max(jt) * 1e3, runs))
    torch.cuda.empty_cache()


def row_path(dc, nb, ns):
    rng = np.random.default_rng(2)
    kr = max(1, int(KEY_RANGE * nb / 1e8))      # the output rows per big row of the cases above at the same size ratio
    rb = list(zip(rng.integers(0, kr, nb).tolist(), range(nb)))
    rs = list(zip(rng.integers(0, kr, ns).tolist(), range(ns)))
    a, b = dc.parallelize(rb, 8), dc.parallelize(rs, 8)
    a.innerJoin(b).glom().collect()                       # warm-up
    t0 = time.perf_counter()
    n_out = sum(len(p) for p in a.innerJoin(b).glom().collect())
    dt = time.perf_counter() - t0
    print("row path  big %d x small %d rows: %d output rows in %.2f s = %.3g big rows/s" % (nb, ns, n_out, dt, nb / dt))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--big", type=float, default=1e8)
    ap.add_argument("--smalls", default="1e3,1e5,1e7")
    ap.add_argument("--parts", type=int, default=64)
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--rows-big", type=float, default=1e6)
    args = ap.parse_args(_argv)
    if not torch.cuda.is_available():
        raise SystemExit("innerjoin_e2e.py measures on a CUDA device; none found")
    name, limit = card()
    print("device: %s, power limit %s" % (name, limit))
    dc = DparkContext("local")
    g = torch.Generator(device="cuda").manual_seed(1)
    nb = int(args.big)
    bk = torch.randint(0, KEY_RANGE, (nb,), device="cuda", generator=g)
    bv = torch.arange(nb, dtype=torch.int64, device="cuda")
    smalls = [int(float(x)) for x in args.smalls.split(",")]
    for ns in smalls:
        sk = torch.randint(0, KEY_RANGE, (ns,), device="cuda", generator=g)
        sv = torch.arange(ns, dtype=torch.int64, device="cuda")
        run_case(dc, "small %.0e" % ns, bk, bv, sk, sv, args.parts, args.runs)
    ns = smalls[len(smalls) // 2]
    sk = torch.randint(0, KEY_RANGE, (ns,), device="cuda", generator=g)
    sv = torch.arange(ns, dtype=torch.int64, device="cuda")
    hot = KEY_RANGE + 1
    sk[torch.randperm(ns, device="cuda", generator=g)[:min(ns, 10_000)]] = hot
    bk[torch.randperm(nb, device="cuda", generator=g)[:1_000]] = hot
    run_case(dc, "hot %.0e" % ns, bk, bv, sk, sv, args.parts, args.runs)
    del bk, bv, sk, sv
    torch.cuda.empty_cache()
    row_path(dc, int(args.rows_big), int(args.rows_big / 10))


if __name__ == "__main__":
    main()
