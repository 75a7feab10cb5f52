"""percentilesByKey of a numeric ColumnarRDD on one GPU (dpark/rdd.py:815-850).

RDD.percentilesByKey tags every row with its split, groups the tagged rows by key into host lists and runs the pure-Python
MergingDigest (quantiles.py) over every value.  When the input already is columns the same numbers come from the device,
bit for bit:

  1. the keys, converted as join._key_column converts them, go through the numeric group-by (grouping.group_row_ids)
     carrying their row ids: every key's ids in (split, position) order;
  2. a key's run is cut where the split changes (dpk_tdigest_heads with per = 1 over each row's split, found by a
     search of the splits' first rows): one segment per (key, split);
  3. every segment's digest, MergingDigest().update(values) + compress(), into compacted scratch of min(L, TD_CAP)
     centroids per segment (dpk_tdigest_build);
  4. per key the first segment's digest absorbs the others in split order, then quantile(pp / 100.) for every pp in p
     (dpk_tdigest_merge);
  5. the partitions are cut as the cogroup's are (join.partition_bounds / join.partition_slices).

The composition stands -- same partitioner, same rows -- when the float values hold a NaN (it raises "Cannot add NaN"),
when a centroid mean comes out NaN (+inf and -inf under one key) or below its predecessor (x - m overflowed), when a fold
would stage more than 2 * TD_CAP entries, and when a q lies outside [0, 1] (it raises its own ValueError).  Host reads:
G, the segment count and the flag word, then the partition bounds.
"""
import torch

from . import _native as nv
from . import grouping, join
from .rdd import DeviceResultRDD, Split

TD_CAP = nv.TD_CAP


def segment_digests(rdd, P, thresholds):
    """Steps 1-3 for a non-empty ColumnarRDD: (group-by (keys, gs, ids, part_off), seg_starts[S + 1], seg_off[S + 1],
    tdigest_build's digests, flag) as CUDA tensors; flag[0] != 0 voids the digests."""
    from .engine import _device
    dev = _device()
    keys = join._key_column([rdd], dev)
    vals = rdd.vals.to(dev).contiguous()
    n = int(keys.numel())
    ids = torch.arange(n, dtype=torch.int64, device=dev)
    gk, gs, ov, part_off = grouping.group_row_ids([keys], [ids], P, thresholds)
    # each row's split (splits may be uneven: ColumnarRDD bounds): a key's run is cut where it changes
    begins = torch.tensor([sp.begin for sp in rdd.splits[1:]], dtype=torch.int64, device=dev)
    head = nv.tdigest_heads(torch.searchsorted(begins, ov, right=True), gs, 1)
    seg_starts = torch.cat([head.nonzero().view(-1), gs[-1:]])
    seg_off = torch.zeros_like(seg_starts)
    torch.cumsum((seg_starts[1:] - seg_starts[:-1]).clamp_(max=TD_CAP), 0, out=seg_off[1:])
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    digests = nv.tdigest_build(ov, vals, seg_starts, seg_off, flag)
    return (gk.view(keys.dtype), gs, ov, part_off), seg_starts, seg_off, digests, flag


def percentiles_columns(rdd, P, thresholds, qs):
    """percentilesByKey of a ColumnarRDD for the fractions qs: a list of P tuples (keys[G_p], quantiles[G_p, len(qs)])
    of CUDA tensors, keys int64 or float64 in the group-by's order, quantiles float64; or None when the composition must
    stand."""
    from .engine import _device
    dev = _device()
    if rdd.keys.numel() == 0:
        keys = join._key_column([rdd], dev)
        return [(keys, torch.empty((0, len(qs)), dtype=torch.float64, device=dev))] * P
    (gk, gs, _, part_off), seg_starts, seg_off, digests, flag = segment_digests(rdd, P, thresholds)
    q = torch.tensor(qs, dtype=torch.float64, device=dev)
    out = nv.tdigest_merge(gs, seg_starts, seg_off, digests, q, flag)
    if int(flag.item()):
        return None
    G = int(gk.numel())
    pg, rows = join.partition_bounds(gs, part_off, torch.arange(G + 1, device=dev).unsqueeze(0))
    return [(k, v) for k, _, (v,) in join.partition_slices(gk, gs.unsqueeze(0), [out], pg, rows)]


class ColumnarPercentilesByKeyRDD(DeviceResultRDD):
    """The result of percentilesByKey(p) of a numeric ColumnarRDD in a one-process job: per key the list of its
    percentiles, the rows of the composition (RDD._percentiles_rows), computed on the GPU the first time a partition is
    asked for and kept.  It has the group-by's partitioner, so mapValue keeps it and a later groupWith reads it as a
    narrow dependency.  columns(split) hands out CUDA tensors (keys, quantiles): keys int64 or float64, quantiles
    float64 [keys, len(p)]; where the module docstring says so the composition's rows stand."""

    def __init__(self, parent, part, p):
        DeviceResultRDD.__init__(self, parent.ctx)
        self.parent = parent
        self.partitioner = part
        self.p = list(p)
        self._splits = [Split(i) for i in range(part.numPartitions)]

    def parents(self):
        return [self.parent]

    def _run(self):
        part = self.partitioner
        qs = [pp / 100. for pp in self.p]
        if all(0 <= q <= 1 for q in qs) or self.parent.keys.numel() == 0:
            return percentiles_columns(self.parent, part.numPartitions, part.thresholds, qs)
        return None

    def _composition(self):
        return self.parent._percentiles_rows(self.p, self.partitioner)

    def _columns_of_rows(self, rows, dev):
        kdt = torch.float64 if self.parent.keys.dtype.is_floating_point else torch.int64
        return (torch.tensor([k for k, _ in rows], dtype=kdt, device=dev),
                torch.tensor([qs for _, qs in rows], dtype=torch.float64, device=dev).view(len(rows), len(self.p)))
