"""topByKey of a numeric ColumnarRDD on one GPU (dpark/rdd.py:552-594).

RDD.topByKey is a groupByKey followed by a stable sort of every key's values, cut at top_n: every value of every key
becomes a Python object so that top_n of them survive.  When the input already is columns the same rows come from the
device:

  1. the keys, converted as join._key_column converts them, go through the numeric group-by (grouping.group_row_ids)
     carrying their row ids: every key's ids in (map split, position) order, the order in which the reference's
     HeapAggregator breaks ties;
  2. selection rounds (dpk_topk.cu): a run longer than TOPK_TILE candidates is cut into chunks that keep their first
     top_n; once every run fits one chunk, one more round leaves per key the first min(top_n, L) values of its stable
     sort.  The first round reads the values through the ids, without a gathered copy;
  3. the partitions are cut as the cogroup's are (join.partition_bounds / join.partition_slices).

A float value column holding a NaN keeps the composition: Python's sort of such a list has no order-free answer, so
only the composition itself reproduces it.
"""
import itertools

import torch

from . import _native as nv
from . import grouping, join
from .rdd import DeviceResultRDD, Split, top_values

TOPK_MAX_N = nv.TOPK_MAX_N


def rounds(longest, top_n):
    """Selection rounds for runs of at most `longest` candidates: one per round in which the longest run is longer than
    a tile, and the last one (the length rule is topk_next_len, dpk_common.cuh; it is monotone in the run length)."""
    T = nv.TOPK_TILE
    r = 1
    while longest > T:
        longest = longest // T * top_n + min(top_n, longest % T)
        r += 1
    return r


def topk_columns(rdd, P, thresholds, top_n, reverse):
    """topByKey of a ColumnarRDD: a list of P tuples (keys[G_p], offsets[G_p + 1], values) of CUDA tensors, one per
    partition.  Keys are int64 or float64 in the group-by's order; keys[j]'s top values are
    values[offsets[j] : offsets[j + 1]], in the input value dtype, best first."""
    from .engine import _device
    dev = _device()
    keys = join._key_column([rdd], dev)
    vals = rdd.vals.to(dev).contiguous()
    n = int(keys.numel())
    if n == 0:
        return [(keys, torch.zeros(1, dtype=torch.int64, device=dev), vals)] * P
    ids = torch.arange(n, dtype=torch.int64, device=dev)
    gk, gs, ov, part_off = grouping.group_row_ids([keys], [ids], P, thresholds)
    runs, cand, cand_ids, m = gs, vals, ov, n
    for _ in range(rounds(int((gs[1:] - gs[:-1]).max()), top_n)):
        nxt = torch.zeros_like(gs)
        torch.cumsum(nv.topk_lengths(runs, top_n), 0, out=nxt[1:])
        cand = nv.topk_round(cand_ids, cand, runs, m, nxt, top_n, reverse)
        runs, cand_ids, m = nxt, None, int(cand.numel())
    off = runs.unsqueeze(0)
    pg, rows = join.partition_bounds(gs, part_off, off)
    return [(k, o[0], v) for k, o, (v,) in join.partition_slices(gk.view(keys.dtype), off, [cand], pg, rows)]


class ColumnarTopByKeyRDD(DeviceResultRDD):
    """The result of topByKey(top_n, reverse=...) of a numeric ColumnarRDD in a one-process job: per key its top_n
    values, the rows of groupByKey(...).mapValue(stable sort, cut), computed on the GPU the first time a partition is
    asked for and kept.  It has the group-by's partitioner, so mapValue keeps it and a later groupWith reads it as a
    narrow dependency.  columns(split) hands out CUDA tensors (keys, offsets, values): keys int64 or float64, offsets
    int64 [keys + 1], values in the input dtype (see topk_columns); when the float values hold a NaN the composition's
    rows stand."""

    def __init__(self, parent, part, top_n, reverse):
        DeviceResultRDD.__init__(self, parent.ctx)
        self.parent = parent
        self.partitioner = part
        self.top_n, self.reverse = top_n, reverse
        self._splits = [Split(i) for i in range(part.numPartitions)]

    def parents(self):
        return [self.parent]

    def _run(self):
        from .engine import _device
        vals, p = self.parent.vals, self.partitioner
        if vals.dtype.is_floating_point and bool(torch.isnan(vals.to(_device())).any()):
            return None
        return topk_columns(self.parent, p.numPartitions, p.thresholds, self.top_n, self.reverse)

    def _composition(self):
        return self.parent.groupByKey(self.partitioner).mapValue(top_values(self.top_n, None, self.reverse))

    def _columns_of_rows(self, rows, dev):
        kdt = torch.float64 if self.parent.keys.dtype.is_floating_point else torch.int64
        off = [0] + list(itertools.accumulate(len(vs) for _, vs in rows))
        return (torch.tensor([k for k, _ in rows], dtype=kdt, device=dev),
                torch.tensor(off, dtype=torch.int64, device=dev),
                torch.tensor([v for _, vs in rows for v in vs], dtype=self.parent.vals.dtype, device=dev))

    def _rows(self, columns):
        keys, offsets, values = columns
        off, vals = offsets.cpu().tolist(), values.cpu().tolist()
        return zip(keys.cpu().tolist(), [vals[off[j]:off[j + 1]] for j in range(len(off) - 1)])
