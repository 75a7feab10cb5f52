#!/usr/bin/env python
"""Numeric text files into ColumnarRDDs on the GPU (DparkContext.textFileColumns, dpark_b200/textcolumns.py).

Two seeded TSVs under a temporary directory, each a 10^6-line block repeated to --lines lines:
  tsv2  `int\\tfloat` (repr floats), key 0 (int) and value 1 (float);
  tsv8  8 columns, fields 3 (int) and 6 (float) parsed.
For each it reports:
  - the kernels on the first piece (textingest.MAX_PIECE_BYTES): line_starts (dpk_textcols_count + the scan + _emit)
    and dpk_textcols_parse, CUDA events, the median of 10 launches, and their algorithmic bytes/s (the text read
    twice, 8 bytes per line start written, 8 read back by the parse, 16 bytes of outputs per line);
  - textFileColumns end to end (file read, host-to-device copy, kernels, host lines), and the host-to-device copy of
    the same bytes alone (its share of the end-to-end time);
  - the same followed by reduceByKey(add)._materialize();
  - the composition (textFile(...).map(parse)) over the first 10^6 lines, whose rows must equal the device's.
Prints the card name and power limit read in the same run, and one JSON line last.

    python scripts/textcolumns_e2e.py [--lines 100000000] [--repeats 3]
"""
import argparse
import json
import os
import random
import shutil
import statistics
import struct
import subprocess
import sys
import tempfile
import time
from operator import add

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BLOCK = 10 ** 6


def block(kind, seed=1):
    rng = random.Random(seed)
    out = []
    for _ in range(BLOCK):
        k = rng.randrange(1 << 20)
        x = struct.unpack("<d", struct.pack("<Q", rng.getrandbits(52) | (rng.randrange(1000, 1050) << 52)))[0]
        if kind == "tsv2":
            out.append("%d\t%r\n" % (k, x))
        else:
            f = ["w%d" % rng.randrange(100), "%d" % rng.randrange(10 ** 6), "x", "%d" % k, "%.3f" % rng.random(),
                 "y%d" % rng.randrange(10), repr(x), "z"]
            out.append("\t".join(f) + "\n")
    return "".join(out).encode("ascii")


def gpu_conditions():
    import torch
    q = "name,power.limit,clocks.max.sm"
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the numbers still stand; say what could not be read
        smi = "nvidia-smi unavailable (%s)" % type(e).__name__
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q + ": " + smi}


def events(fn, n=10):
    import torch
    fn()
    ts = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / 1e3)
    return statistics.median(ts)


def wall(fn, repeats):
    import torch
    ts = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return statistics.median(ts)


def run(ctx, kind, path, prefix, key, value, repeats):
    import numpy as np
    import torch
    from dpark_b200 import _native as nv
    from dpark_b200 import textingest
    size = os.path.getsize(path)
    dev = torch.device("cuda", 0)
    piece = min(size, textingest.cut_pieces(path, 0, size, size)[0][1])
    d = torch.from_numpy(np.fromfile(path, dtype=np.uint8, count=piece)).to(dev)
    starts, _ = nv.line_starts(d)
    lines = int(starts.numel())
    t_starts = events(lambda: nv.line_starts(d))
    outs = [torch.empty(lines, dtype=torch.int64, device=dev) for _ in range(2)] + [
        torch.empty(lines, dtype=torch.uint8, device=dev)]
    t_parse = events(lambda: nv.textcols_parse(d, starts, torch.tensor([9], dtype=torch.uint8, device=dev), key,
                                               value, False, True, *outs))
    nbytes = 2 * piece + 8 * lines + 8 * lines + 16 * lines
    del d, starts, outs
    torch.cuda.empty_cache()

    def ingest():
        return ctx.textFileColumns(path, key, value, (int, float), "\t")
    e2e = wall(ingest, repeats)
    buf = np.fromfile(path, dtype=np.uint8)
    h2d = wall(lambda: torch.from_numpy(buf).to(dev), repeats)
    del buf
    with_reduce = wall(lambda: ingest().reduceByKey(add, 64)._materialize(), repeats)
    # the composition over the first 10^6 lines, and the device rows of the same lines
    def parse(line):
        f = line.split("\t")
        return int(f[key]), float(f[value])
    t = time.perf_counter()
    comp = ctx.textFile(prefix).map(parse).collect()
    t_comp = time.perf_counter() - t
    cols = ctx.textFileColumns(prefix, key, value, (int, float), "\t")
    dev_rows = list(zip(cols.keys.cpu().tolist(), cols.vals.cpu().tolist()))
    same = len(dev_rows) == len(comp) and all(
        a[0] == b[0] and struct.pack("<d", a[1]) == struct.pack("<d", b[1]) for a, b in zip(dev_rows, comp))
    return {"kind": kind, "bytes": size, "piece_bytes": piece, "piece_lines": lines, "kernel_line_starts_s": t_starts,
            "kernel_parse_s": t_parse,
            "kernel_algorithmic_GBps": nbytes / (t_starts + t_parse) / 1e9,
            "textFileColumns_s": e2e, "h2d_same_bytes_s": h2d, "h2d_share": h2d / e2e,
            "textFileColumns_reduceByKey_s": with_reduce, "composition_1e6_lines_s": t_comp,
            "composition_rows_per_s": BLOCK / t_comp, "prefix_equal": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=10 ** 8)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import torch
    from dpark_b200 import DparkContext
    assert torch.cuda.is_available(), "needs a GPU"
    ctx = DparkContext("local")
    tmp = tempfile.mkdtemp(prefix="textcols_")
    results = []
    try:
        for kind, key, value in (("tsv2", 0, 1), ("tsv8", 3, 6)):
            blk = block(kind)
            prefix = os.path.join(tmp, kind + "_prefix.tsv")
            with open(prefix, "wb") as f:
                f.write(blk)
            path = os.path.join(tmp, kind + ".tsv")
            with open(path, "wb") as f:
                for _ in range(max(1, a.lines // BLOCK)):
                    f.write(blk)
            r = run(ctx, kind, path, prefix, key, value, a.repeats)
            r["lines_total"] = max(1, a.lines // BLOCK) * BLOCK
            r["device_rows_per_s_e2e"] = r["lines_total"] / r["textFileColumns_s"]
            print(json.dumps(r), flush=True)
            results.append(r)
            os.remove(path)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    out = dict(gpu_conditions(), results=results)
    print(json.dumps(out))
    assert all(r["prefix_equal"] for r in results)


if __name__ == "__main__":
    main()
