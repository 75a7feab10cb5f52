"""topByKey of a numeric ColumnarRDD on one GPU, end to end and per kernel, against the composition it replaces.

    python scripts/topbykey_e2e.py [--rows 1e8] [--top 10] [--parts 64] [--runs 7] [--comp-rows 1e7] [--comp-runs 3]

Prints the card and its power limit, then, with int64 keys and values already in HBM:
  - the device topByKey (topk.topk_columns: the group-by, the selection rounds, the partition cut, then a synchronise)
    with keys uniform over [0, 2^26) and with Zipf(1.1) keys: the median time of its materialisation over --runs runs,
    the rounds it took and the device times of dpk_topk_lengths and dpk_topk_round (CUDA events, summed over rounds),
    the first round's algorithmic bytes per second, and the device time of everything else (the group-by);
  - the composition groupByKey(P).mapValue(sorted(...)[:top]) of the first --comp-rows uniform rows, every partition
    collected: the median over --comp-runs runs."""
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
from dpark_b200 import topk  # noqa: E402
from dpark_b200.rdd import top_values  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit or "unknown"


def round1_bytes(n, kept, w):
    """Algorithmic bytes of the first dpk_topk_round: per row its id and its value read; per kept value the id and the
    value read again and the value written."""
    return n * (8 + w) + kept * (8 + 2 * w)


def materialize(col, P, top_n):
    parts = topk.topk_columns(col, P, None, top_n, False)
    torch.cuda.synchronize()
    return sum(int(k.numel()) for k, _, _ in parts), sum(int(v.numel()) for _, _, v in parts)


def run_case(name, col, P, top_n, runs):
    for _ in range(2):
        keys, kept = materialize(col, P, top_n)
    times = []
    for _ in range(runs):
        t0 = time.perf_counter()
        materialize(col, P, top_n)
        times.append(time.perf_counter() - t0)
    nv.prof_enable(True)
    materialize(col, P, top_n)
    torch.cuda.synchronize()
    nv.prof_enable(False)
    prof = nv.prof_collect()
    rounds = [ms for lab, ms in prof if lab == "topk_round"]
    lengths = sum(ms for lab, ms in prof if lab == "topk_lengths")
    other = sum(ms for lab, ms in prof if lab not in ("topk_round", "topk_lengths"))
    n = int(col.keys.numel())
    med = statistics.median(times)
    longest = int(torch.unique(col.keys, return_counts=True)[1].max()) if n else 0
    print("%-8s %d rows, top %d, P=%d: %d keys (longest %d values), %d values kept; materialisation median %.2f ms "
          "(min %.2f, max %.2f, %d runs) = %.3g rows/s; %d rounds: dpk_topk_round %s ms (first round %.1f GB/s "
          "algorithmic), dpk_topk_lengths %.3f ms; other kernels (group-by) %.2f ms"
          % (name, n, top_n, P, keys, longest, kept, med * 1e3, min(times) * 1e3, max(times) * 1e3, runs, n / med,
             len(rounds), " + ".join("%.3f" % ms for ms in rounds), round1_bytes(n, kept, 8) / (rounds[0] * 1e-3) / 1e9,
             lengths, other))


def composition(dc, col, P, top_n, runs):
    times = []
    for _ in range(runs):
        t0 = time.perf_counter()
        parts = col.groupByKey(P).mapValue(top_values(top_n, None, False)).glom().collect()
        times.append(time.perf_counter() - t0)
    n = int(col.keys.numel())
    med = statistics.median(times)
    print("composition %d rows, top %d, P=%d: %d keys; median %.2f s (min %.2f, max %.2f, %d runs) = %.3g rows/s"
          % (n, top_n, P, sum(len(p) for p in parts), med, min(times), max(times), runs, n / med))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1e8)
    ap.add_argument("--top", type=int, default=10)
    ap.add_argument("--parts", type=int, default=64)
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--comp-rows", type=float, default=1e7)
    ap.add_argument("--comp-runs", type=int, default=3)
    args = ap.parse_args(_argv)
    if not torch.cuda.is_available():
        raise SystemExit("topbykey_e2e.py measures on a CUDA device; none found")
    name, limit = card()
    print("device: %s, power limit %s" % (name, limit))
    dc = DparkContext("local")
    g = torch.Generator(device="cuda").manual_seed(1)
    n = int(args.rows)
    vals = torch.randint(-(1 << 40), 1 << 40, (n,), device="cuda", generator=g)
    uniform = torch.randint(0, 1 << 26, (n,), device="cuda", generator=g)
    run_case("uniform", dc.parallelizeColumns(uniform, vals, 8), args.parts, args.top, args.runs)
    zipf = torch.from_numpy(np.minimum(np.random.default_rng(2).zipf(1.1, n), 1 << 40)).cuda()
    run_case("zipf1.1", dc.parallelizeColumns(zipf, vals, 8), args.parts, args.top, args.runs)
    del zipf
    torch.cuda.empty_cache()
    m = int(args.comp_rows)
    composition(dc, dc.parallelizeColumns(uniform[:m], vals[:m], 8), args.parts, args.top, args.comp_runs)


if __name__ == "__main__":
    main()
