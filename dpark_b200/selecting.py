"""top, uniq and hot of a numeric ColumnarRDD on one GPU (dpark/rdd.py:383-398).

The compositions turn every row into a Python tuple (top) or tuple key (uniq, hot).  On the device:
  top(n, key, reverse): the composition's list is sorted(rows in (split, position) order, key=key, reverse=not
    reverse)[:n] (nlargest / nsmallest are stable, the per-split picks are prefixes): the n smallest rows by
    (dpk_sort_keys' order words, row id), found by select_smallest, ordered by the radix passes and gathered.
  uniq(): every row's (k, v) pair into dpk_uniq_insert's table; the distinct pairs in partition portable_hash((k, v))
    % P, each partition in order of first occurrence with the first row's bits -- the reference's outcome when it
    fetches the map outputs in split order.
  hot(n): uniq's pairs and counts, then select_smallest over ~count with the position in uniq's order as the tie id.
A NaN in an order column keeps top's composition; a NaN in either column raises the row path's TypeError for uniq / hot.
"""
import torch

from . import _native as nv
from . import shuffle, sorting
from .rdd import RDD, DeviceResultRDD, Split, device_path_applies

NAN_KEYS = "NaN keys are not supported (CPython hashes NaN by identity)"
MAX_UNIQ_ROWS = (1 << 31) - 2       # row ids stay below the table's empty mark 0x7FFFFFFF
ID_BITS = 31                        # the (partition, first row id) sort word: partition << 31 | id


def top_order(key):
    """The columns top(n, key) orders by (sorting.ORDER_*), None meaning the identity, or None if key is not
    recognised."""
    return sorting.ORDER_KV if key is None else sorting.order_of(key)


def top_applies(rdd, n, key):
    """True when rdd.top(n, key, reverse) runs on the device: an int n, a numeric ColumnarRDD in a one-process job
    (rdd.device_path_applies) with at most sorting.MAX_ROWS rows, and a recognised key."""
    return type(n) is int and device_path_applies([rdd], sorting.MAX_ROWS) and top_order(key) is not None


def uniq_applies(rdd):
    """True when rdd.uniq(...) runs on the device (given a HashPartitioner): a numeric ColumnarRDD in a one-process job
    (rdd.device_path_applies) with at most MAX_UNIQ_ROWS rows."""
    return device_path_applies([rdd], MAX_UNIQ_ROWS)


def hot_applies(rdd, n):
    """True when rdd.hot(n, ...) runs on the device (given a HashPartitioner): uniq_applies and an int n."""
    return type(n) is int and uniq_applies(rdd)


device_partitioner = RDD._device_partitioner     # (rdd, numSplits): the HashPartitioner uniq / hot take, or None


def select_smallest(w0, w1, n):
    """Row ids of the n smallest rows by (w0[, w1], row id), in that order: int64 device [min(n, rows)].  w0 / w1 are
    int64 tensors of unsigned order words (w1 None for one word).

    Host reads: one per radix round (the chosen bucket's size and whether the threshold is exact).  A round fixes at
    least 8 more bits of the threshold or finishes a word, so there are at most 8 per word; every round after the first
    reads only the previous round's bucket."""
    m = int(w0.numel())
    n = min(n, m)
    if n <= 0:
        return torch.empty(0, dtype=torch.int64, device=w0.device)
    if n == m:
        ids = torch.arange(m, dtype=torch.int64, device=w0.device)
    else:
        st, hist = (t.to(w0.device) for t in nv.select_state(n, m))
        cands, rounds, limit = None, 0, 8 * (1 if w1 is None else 2)
        while True:
            nv.select_round(w0, w1, cands, m, st, hist)
            rounds += 1
            count, _, _, done = st[4:8].tolist()
            if done:
                break
            if rounds >= limit:
                raise AssertionError("radix select did not settle in %d rounds" % limit)
            if count < m:
                cands, m = nv.select_compact(w0, w1, cands, m, st, count), count
        del cands
        ids = nv.select_take(w0, w1, n, st)
    if w1 is not None:              # LSD over the selected rows: by w1, then stably by w0; ids ascend within ties
        _, ids = shuffle.sort_by_key_bits(nv.gather_i64(w1, ids), ids)
    _, ids = shuffle.sort_by_key_bits(nv.gather_i64(w0, ids), ids)
    return ids


def _columns(rdd):
    from .engine import _device
    dev = _device()
    return rdd.keys.to(dev).contiguous(), rdd.vals.to(dev).contiguous()


def top(rdd, n, key, reverse):
    """rdd.top(n, key, reverse) as the composition returns it, or None when an order column holds a NaN."""
    keys, vals = _columns(rdd)
    if n <= 0 or not keys.numel():
        return []
    order = top_order(key)
    col0, col1 = {sorting.ORDER_KV: (keys, vals), sorting.ORDER_K: (keys, None), sorting.ORDER_V: (vals, None)}[order]
    w0, w1, ids, nan = nv.sort_keys(col0, col1, not reverse)     # the largest first: complemented words
    del ids
    if int(nan.item()):
        return None
    ids = select_smallest(w0, w1, n)
    del w0, w1
    k, v = nv.gather_columns(keys, vals, ids)
    return list(zip(k.cpu().tolist(), v.cpu().tolist()))


def distinct(rdd, part):
    """The distinct (k, v) pairs of rdd under HashPartitioner part: (keys, vals, counts, offsets) -- CUDA columns in the
    input dtypes, each pair with the bits of its first row, ordered by (partition, first row id); int64 row counts; and
    the P + 1 partition offsets as a list.  Raises TypeError for a NaN in either column."""
    keys, vals = _columns(rdd)
    n, P = int(keys.numel()), part.numPartitions
    if n == 0:
        return keys, vals, torch.empty(0, dtype=torch.int64, device=keys.device), [0] * (P + 1)
    table, st = nv.uniq_insert(keys, vals)
    first, count = nv.uniq_emit(table, st, n)
    del table
    nan, D = st.tolist()
    if nan:
        raise TypeError(NAN_KEYS)
    first, count = first[:D], count[:D]
    fk, fv = nv.gather_columns(keys, vals, first)
    h = nv.hash_tuple(torch.stack([nv.hash_keys(fk), nv.hash_keys(fv)]))
    pid = nv.partition_ids(h, P, part.thresholds).to(torch.int64)
    word, count = shuffle.sort_by_key_bits((pid << ID_BITS) | first, count)
    bounds = torch.arange(P + 1, dtype=torch.int64, device=keys.device) << ID_BITS
    offsets = torch.searchsorted(word, bounds).tolist()
    k, v = nv.gather_columns(keys, vals, word & ((1 << ID_BITS) - 1))
    return k, v, count, offsets


def hot(rdd, n, part):
    """rdd.hot(n, numSplits) under HashPartitioner part: [((k, v), count)], the n largest counts, ties in uniq's order."""
    k, v, count, _ = distinct(rdd, part)
    if n <= 0 or not count.numel():
        return []
    ids = select_smallest(~count, None, n)      # unsigned order of ~count: the largest count first
    hk, hv = nv.gather_columns(k, v, ids)
    return [((a, b), c) for a, b, c in zip(hk.cpu().tolist(), hv.cpu().tolist(), count[ids].cpu().tolist())]


class ColumnarUniqRDD(DeviceResultRDD):
    """rdd.uniq(numSplits) of a numeric ColumnarRDD in a one-process job: the composition's partition count and no
    partitioner; partition p holds the distinct (k, v) pairs with portable_hash((k, v)) % P == p, in order of first
    occurrence, each with its first row's bits.  Computed on the GPU the first time a partition is asked for and kept;
    columns(split) hands out CUDA tensors (keys, values) in the input dtypes."""

    def __init__(self, parent, part):
        DeviceResultRDD.__init__(self, parent.ctx)
        self.parent, self.part = parent, part
        self._splits = [Split(i) for i in range(part.numPartitions)]

    def parents(self):
        return [self.parent]

    def _run(self):
        return distinct(self.parent, self.part)

    def _part(self, result, i):
        keys, vals, _, off = result
        return keys[off[i]:off[i + 1]], vals[off[i]:off[i + 1]]
