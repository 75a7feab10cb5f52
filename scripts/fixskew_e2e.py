"""The fixSkew partitioner of a numeric ColumnarRDD on one GPU, end to end and per kernel, against the composition.

    python scripts/fixskew_e2e.py [--rows 1e8] [--splits 8,64] [--rates 0.01,0.1,1] [--P 64] [--runs 5]
                                  [--comp-rows 1e6] [--comp-runs 3]

Prints the card and its power limit, then, with int64 keys uniform over [0, 2^40) already in HBM:
  - col._combine_partitioner(P, fixSkew=r) (sampling.skew_thresholds: the key hashes, the MT19937 sample, the per-split
    digests, the merge and the host reads) of --rows rows in M splits for every M of --splits and r of --rates: the
    median time over --runs runs after one warm-up, the rows kept, and the device times (CUDA events) of
    dpk_sample_bernoulli, dpk_hash_keys, dpk_tdigest_build (short and long segments) and dpk_tdigest_merge;
  - the composition (SampleRDD, hashes per partition, quantiles.MergingDigest) over the first --comp-rows rows as
    Python rows in the same number of splits, at every rate: the median over --comp-runs runs, and whether the device
    path gives the same partitioner for those rows."""
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
from dpark_b200 import sampling  # noqa: E402

KERNELS = ("sample_bernoulli", "hash_keys", "tdigest_build_short", "tdigest_build_long", "tdigest_merge")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit or "unknown"


def partitioner(col, P, rate):
    if sampling.thresholds_inputs(col, rate) is None:
        raise SystemExit("the device path does not apply")
    part = col._combine_partitioner(P, rate)
    torch.cuda.synchronize()
    return part


def run_case(col, P, rate, runs):
    part = partitioner(col, P, rate)
    times = []
    for _ in range(runs):
        t0 = time.perf_counter()
        partitioner(col, P, rate)
        times.append(time.perf_counter() - t0)
    nv.prof_enable(True)
    partitioner(col, P, rate)
    torch.cuda.synchronize()
    nv.prof_enable(False)
    prof = nv.prof_collect()
    per = {k: sum(ms for lab, ms in prof if lab == k) for k in KERNELS}
    other = sum(ms for lab, ms in prof if lab not in KERNELS)
    kept = int(col.keys.numel())
    if rate < 1:
        sample = col.sample(rate, False, sampling.SKEW_SEED)
        kept = sum(int(sample.columns(sp)[0].numel()) for sp in sample.splits)
    n = int(col.keys.numel())
    med = statistics.median(times)
    print("device  %d rows, M=%d, P=%d, fixSkew=%g: %d rows kept, %d partitions; median %.2f ms (min %.2f, max %.2f, "
          "%d runs) = %.3g rows/s; %s; other kernels %.2f ms"
          % (n, len(col.splits), P, rate, kept, part.numPartitions, med * 1e3, min(times) * 1e3, max(times) * 1e3,
             runs, n / med, ", ".join("%s %.3f ms" % (k, per[k]) for k in KERNELS), other), flush=True)


def composition(dc, col, P, rate, runs):
    rows = dc.parallelize(list(zip(col.keys.cpu().tolist(), col.vals.cpu().tolist())), len(col.splits))
    times = []
    for _ in range(runs):
        t0 = time.perf_counter()
        want = rows._combine_partitioner(P, rate)
        times.append(time.perf_counter() - t0)
    got = partitioner(col, P, rate)
    n = int(col.keys.numel())
    med = statistics.median(times)
    print("composition %d rows, M=%d, P=%d, fixSkew=%g: median %.3f s (min %.3f, max %.3f, %d runs) = %.3g rows/s; "
          "device partitioner %s" % (n, len(col.splits), P, rate, med, min(times), max(times), runs, n / med,
                                     "equal" if got == want else "DIFFERS"), flush=True)
    return got == want


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1e8)
    ap.add_argument("--splits", default="8,64")
    ap.add_argument("--rates", default="0.01,0.1,1")
    ap.add_argument("--P", type=int, default=64)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--comp-rows", type=float, default=1e6)
    ap.add_argument("--comp-runs", type=int, default=3)
    args = ap.parse_args(_argv)
    if not torch.cuda.is_available():
        raise SystemExit("fixskew_e2e.py measures on a CUDA device; none found")
    name, limit = card()
    print("device: %s, power limit %s" % (name, limit), flush=True)
    dc = DparkContext("local")
    g = torch.Generator(device="cuda").manual_seed(1)
    n = int(args.rows)
    keys = torch.randint(0, 1 << 40, (n,), device="cuda", generator=g)
    vals = torch.arange(n, device="cuda")
    splits = [int(x) for x in args.splits.split(",")]
    rates = [float(x) for x in args.rates.split(",")]
    for M in splits:
        col = dc.parallelizeColumns(keys, vals, M)
        for rate in rates:
            run_case(col, args.P, rate, args.runs)
    c = int(args.comp_rows)
    ok = all([composition(dc, dc.parallelizeColumns(keys[:c], vals[:c], M), args.P, rate, args.comp_runs)
              for M in splits[-1:] for rate in rates])
    if not ok:
        raise SystemExit("the device partitioner differs from the composition's")


if __name__ == "__main__":
    main()
