"""join / leftOuterJoin / rightOuterJoin / outerJoin of two numeric ColumnarRDDs on one GPU (dpark/rdd.py:649-676), and
groupWith / cogroup / groupByKey of numeric ColumnarRDDs.

RDD._join is a cogroup followed by a flatMap over Python lists: every row of the inputs and of the result becomes a
Python object.  When both inputs already are columns the same result is computed on the device:

  1. the left keys, then the right keys, converted as columnar._key_column converts Python keys (int32 -> int64,
     float32 -> float64, + 0.0), go through the numeric group-by (grouping.group_row_ids) carrying their row ids, so
     row id < nL is a left row; the values stay where they are, in the same concatenated order;
  2. dpk_join_count: per key its left row count and the L * R rows it produces;
  3. the exclusive scan of those counts places every key's rows; the partitions' row offsets are read back once;
  4. dpk_join_emit: the joined rows, load-balanced over output rows, the values gathered by row id.

The groups come out partition by partition in the order of the group-by of the tagged union, and per key
`for x in left for y in right` -- partitions, rows and order are those of the composition.

groupWith / cogroup of N numeric ColumnarRDDs (CoGroupedRDD, a group-by of the tagged union) and groupByKey of one
(N = 1) take the same CSR without a cross product: dpk_cogroup_count splits every key's id run at the inputs' id
boundaries, and dpk_cogroup_emit gathers each input's value runs, load-balanced like the join's emit.

innerJoin (dpark/rdd.py:626-648) keeps the big side where it lies: no group-by, no shuffle, its splits and row order.
Only the small side is grouped (P = 1, with row ids, so each key's ids ascend: small.collect() order); its distinct
keys go into a device hash table (dpk_bcast_build), every big row is probed in place (dpk_bcast_probe: its group and
match count), and after one scan of the counts dpk_bcast_emit writes the rows, load-balanced like the join's emit.
"""
import torch

from . import _native as nv
from . import grouping
from .rdd import DeviceResultRDD, Split, device_path_applies


def has_nan_key(key_columns):
    return any(k.dtype.is_floating_point and bool(torch.isnan(k).any()) for k in key_columns)


def reject_nan_keys(key_columns, flag=None):
    """TypeError if a float key column holds a NaN, as the row path's ingest raises (columnar._key_column): CPython
    hashes NaN by identity, so every NaN row is a key of its own there, while the device would merge equal bits.
    flag: has_nan_key already evaluated (under torch.distributed: over every rank's columns, so all ranks agree)."""
    if has_nan_key(key_columns) if flag is None else flag:
        raise TypeError("NaN keys are not supported (CPython hashes NaN by identity)")


def _key_column(rdds, dev):
    """The keys of rdds one after the other on the device, as the row path ingests them; raises TypeError where it
    does (NaN keys, int keys on one input and float keys on another)."""
    sides = [r.keys for r in rdds if r.keys.numel()]
    reject_nan_keys(sides)
    kinds = sorted(set("float" if k.dtype.is_floating_point else "int" for k in sides))
    if len(kinds) > 1:
        raise TypeError("mixed key types %s in one shuffle are not supported on the GPU path" % kinds)
    kdt = torch.float64 if kinds == ["float"] else torch.int64
    keys = torch.cat([r.keys.to(dev, kdt) for r in rdds])
    return keys + 0.0 if kdt == torch.float64 else keys     # -0.0 and 0.0 are one key, spelled 0.0


def join_columns(left, right, P, thresholds, keep_left, keep_right):
    """The joined rows of two ColumnarRDDs: a list of P tuples (keys, left, right, left_valid, right_valid) of CUDA
    tensors, one per partition."""
    from .engine import _device
    dev = _device()
    nL = int(left.keys.numel())
    keys = _key_column([left, right], dev)
    lvals, rvals = left.vals.to(dev).contiguous(), right.vals.to(dev).contiguous()
    n = int(keys.numel())
    if n == 0:
        out = (keys, lvals, rvals, torch.empty(0, dtype=torch.uint8, device=dev) if keep_right else None,
               torch.empty(0, dtype=torch.uint8, device=dev) if keep_left else None)
        return [out] * P
    ids = torch.arange(n, dtype=torch.int64, device=dev)
    gk, gs, ov, part_off = grouping.group_row_ids([keys], [ids], P, thresholds)
    G = int(gk.numel())
    nl, cnt = nv.join_count(ov, gs, G, nL, keep_left, keep_right)
    out_off = torch.zeros(G + 1, dtype=torch.int64, device=dev)
    torch.cumsum(cnt, 0, out=out_off[1:])
    # partition p's rows start at the output offset of its first group; the last entry is the total
    bounds = out_off[torch.searchsorted(gs[:-1], part_off)].cpu().tolist()
    cols = nv.join_emit(gk, gs, ov, nl, out_off, nL, lvals, rvals, keep_left, keep_right, bounds[-1])
    if keys.dtype == torch.float64:
        cols = (cols[0].view(torch.float64),) + cols[1:]
    return [tuple(None if c is None else c[bounds[p]:bounds[p + 1]] for c in cols) for p in range(P)]


class ColumnarJoinedRDD(DeviceResultRDD):
    """The result of join / leftOuterJoin / rightOuterJoin / outerJoin of two numeric ColumnarRDDs in a one-process
    job: the rows RDD._join's composition yields, computed on the GPU the first time a partition is asked for and
    kept (like ShuffledRDD).  Like the flatMap it stands for, it has the cogroup's partitions and no partitioner.

    columns(split) hands out CUDA tensors (keys, left, right, left_valid, right_valid).  Keys are int64 or float64,
    values keep their input dtypes; a valid column is uint8 (0 = the side is missing, its value slot holds 0) and None
    for a side the join kind never misses."""

    def __init__(self, left, right, part, keep_left, keep_right):
        DeviceResultRDD.__init__(self, left.ctx)
        self.left, self.right = left, right
        self.join_partitioner = part
        self.keep_left, self.keep_right = keep_left, keep_right
        self._splits = [Split(i) for i in range(part.numPartitions)]

    def parents(self):
        return [self.left, self.right]

    def _run(self):
        p = self.join_partitioner
        return join_columns(self.left, self.right, p.numPartitions, p.thresholds, self.keep_left, self.keep_right)

    def _rows(self, columns):
        keys, left, right, lvalid, rvalid = columns
        ls, rs = left.cpu().tolist(), right.cpu().tolist()
        if lvalid is not None:
            ls = [x if ok else None for x, ok in zip(ls, lvalid.cpu().tolist())]
        if rvalid is not None:
            rs = [y if ok else None for y, ok in zip(rs, rvalid.cpu().tolist())]
        return zip(keys.cpu().tolist(), zip(ls, rs))


def inner_join_applies(big, small):
    """True when big.innerJoin(small) runs on the device: rdd.device_path_applies, and not int keys on one side with
    float keys on the other (both non-empty; Python's 1 == 1.0 is not the device's equality)."""
    if not device_path_applies([big, small]):
        return False
    sides = [r.keys for r in (big, small) if r.keys.numel()]
    return len(set(k.dtype.is_floating_point for k in sides)) <= 1


def inner_join_columns(big, small):
    """big.innerJoin(small) of two ColumnarRDDs: a list of tuples (keys, left, right) of CUDA tensors, one per split of
    big, in big's key and value dtypes and small's value dtype."""
    from .engine import _device
    dev = _device()
    keys, lvals = big.keys.to(dev).contiguous(), big.vals.to(dev).contiguous()
    rvals = small.vals.to(dev).contiguous()
    split_rows = [sp.begin for sp in big.splits] + [big.splits[-1].end]
    # the small keys as the dict holds them: int -> int64, float -> float64 with 0.0 for -0.0; NaN keys find nothing
    sk = small.keys.to(dev)
    ids = torch.arange(sk.numel(), dtype=torch.int64, device=dev)
    if sk.dtype.is_floating_point:
        sk = sk.to(torch.float64) + 0.0
        keep = ~torch.isnan(sk)
        sk, ids = sk[keep], ids[keep]
    else:
        sk = sk.to(torch.int64)
    if keys.numel() == 0 or sk.numel() == 0:
        empty = (keys[:0], lvals[:0], rvals[:0])
        return [empty] * len(big.splits)
    gk, gs, ov, _ = grouping.group_row_ids([sk], [ids], 1, None)
    table = nv.bcast_build(gk)
    grp, cnt = nv.bcast_probe(table, keys, gs)
    off = torch.zeros(keys.numel() + 1, dtype=torch.int64, device=dev)
    torch.cumsum(cnt, 0, out=off[1:])
    rows = off[split_rows].cpu().tolist()
    cols = nv.bcast_emit(keys, lvals, grp, off, gs, ov, rvals, rows[-1])
    return [tuple(c[rows[s]:rows[s + 1]] for c in cols) for s in range(len(big.splits))]


class ColumnarInnerJoinedRDD(DeviceResultRDD):
    """The result of big.innerJoin(small) of two numeric ColumnarRDDs in a one-process job: the rows RDD.innerJoin's
    flatMap yields, computed on the GPU the first time a partition is asked for and kept.  Like the flatMap it has
    big's splits and no partitioner.

    columns(split) hands out the rows of big's split `split` as CUDA tensors (keys, left, right): keys in big's key
    dtype with their own bits, left in big's value dtype, right in small's value dtype."""

    def __init__(self, big, small):
        DeviceResultRDD.__init__(self, big.ctx)
        self.big, self.small = big, small
        self._splits = [Split(i) for i in range(len(big.splits))]

    def parents(self):
        return [self.big, self.small]

    def _run(self):
        return inner_join_columns(self.big, self.small)

    def _rows(self, columns):
        keys, left, right = columns
        return zip(keys.cpu().tolist(), zip(left.cpu().tolist(), right.cpu().tolist()))


def cogroup_columns(rdds, P, thresholds):
    """The cogroup of N ColumnarRDDs: a list of P tuples (keys[G_p], offsets[N, G_p + 1], (values_0, ..., values_N-1))
    of CUDA tensors, one per partition.  Keys are int64 or float64, keys[j]'s values from input t are
    values_t[offsets[t, j] : offsets[t, j + 1]] in input t's dtype and (split, position) order; every offsets row
    starts at 0."""
    from .engine import _device
    dev = _device()
    N = len(rdds)
    keys = _key_column(rdds, dev)
    vals = tuple(r.vals.to(dev).contiguous() for r in rdds)
    sizes = [int(r.keys.numel()) for r in rdds]
    bounds = [0]
    for m in sizes:
        bounds.append(bounds[-1] + m)
    n = bounds[-1]
    if n == 0:
        return [(keys, torch.zeros((N, 1), dtype=torch.int64, device=dev), vals)] * P
    ids = torch.arange(n, dtype=torch.int64, device=dev)
    gk, gs, ov, part_off = grouping.group_row_ids([keys], [ids], P, thresholds)
    G = int(gk.numel())
    first, cnt = nv.cogroup_count(ov, gs, G, torch.tensor(bounds, dtype=torch.int64, device=dev))
    off = torch.zeros((N, G + 1), dtype=torch.int64, device=dev)
    for t in range(N):      # one 1-D scan per input: torch scans a [N, G] tensor along dim 1 one row per CTA
        torch.cumsum(cnt[t], 0, out=off[t, 1:])
    pg, rows = partition_bounds(gs, part_off, off)
    cols = [nv.cogroup_emit(ov, first[t], off[t], bounds[t], vals[t], rows[t][-1]) for t in range(N)]
    return partition_slices(gk.view(keys.dtype), off, cols, pg, rows)


def partition_bounds(gs, part_off, off):
    """Where the partitions of a group-by (group starts gs[G + 1], partition row offsets part_off[P + 1]) lie in its
    per-group outputs: partition p holds the groups [pg[p], pg[p + 1]) and the rows [rows[t][p], rows[t][p + 1]) of
    output t, whose group g starts at row off[t, g] (off: [N, G + 1]).  Host lists."""
    pg = torch.searchsorted(gs[:-1], part_off)
    rows = off[:, pg].cpu().tolist()
    return pg.cpu().tolist(), rows


def partition_slices(gk, off, cols, pg, rows):
    """Per partition (keys[G_p], offsets[N, G_p + 1] starting at 0, (output_0, ...)): views of the group keys, of the
    per-group output offsets off and of the output columns cols, cut at partition_bounds' (pg, rows)."""
    return [(gk[pg[p]:pg[p + 1]], off[:, pg[p]:pg[p + 1] + 1] - off[:, pg[p]:pg[p] + 1],
             tuple(c[r[p]:r[p + 1]] for c, r in zip(cols, rows))) for p in range(len(pg) - 1)]


class ColumnarCoGroupedRDD(DeviceResultRDD):
    """The result of groupWith / cogroup of numeric ColumnarRDDs in a one-process job: per key one value list per
    input, the rows CoGroupedRDD yields, computed on the GPU the first time a partition is asked for and kept.  It has
    the cogroup's partitioner, so mapValue keeps it and a later groupWith reads it as a narrow dependency.

    columns(split) hands out CUDA tensors (keys, offsets, values): keys int64 or float64, offsets int64 [N, keys + 1],
    values a tuple of N columns in the inputs' dtypes (see cogroup_columns)."""

    def __init__(self, rdds, part):
        DeviceResultRDD.__init__(self, rdds[0].ctx)
        self.rdds = list(rdds)
        self.partitioner = part
        self._splits = [Split(i) for i in range(part.numPartitions)]

    def parents(self):
        return list(self.rdds)

    def _run(self):
        p = self.partitioner
        return cogroup_columns(self.rdds, p.numPartitions, p.thresholds)

    def _rows(self, columns):
        keys, offsets, values = columns
        off = offsets.cpu().tolist()
        vals = [v.cpu().tolist() for v in values]
        groups = zip(*[[vs[o[j]:o[j + 1]] for j in range(len(o) - 1)] for o, vs in zip(off, vals)])
        return zip(keys.cpu().tolist(), groups)
