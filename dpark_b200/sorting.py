"""sort of a numeric ColumnarRDD on one GPU (dpark/rdd.py:273-287).

RDD.sort samples range bounds, routes every row with a Python bisect, groups the rows into host lists by range index
and runs Python's sorted per partition.  For columns sorted by the identity ((k, v)), x[0] or x[1] the same partitions
come from one global stable sort: the bounds by the same rule (rdd.range_bounds) over samples read from column slices;
dpk_sort_keys (order words, row ids, a NaN flag); the group-by's radix passes (for (k, v): by the v word, then by the
k word gathered through the sorted ids); dpk_sort_cuts (getPartition is monotone in the key, so partitions are slices
of the sorted rows, found by binary search); dpk_sort_gather.  Equal keys keep (split, position) order in both
directions, as Python's stable sort does.  A NaN in an order column keeps the composition: Python's sort of such a
list has no order-free answer.
"""
import operator
import struct

import torch

from . import _native as nv
from . import shuffle
from .rdd import DeviceResultRDD, Split, device_path_applies, range_bounds
from .textingest import _same

_t_identity = lambda x: x           # noqa: E731
_t_first = lambda x: x[0]           # noqa: E731
_t_second = lambda x: x[1]          # noqa: E731

ORDER_KV, ORDER_K, ORDER_V = "kv", "k", "v"
MAX_ROWS = (1 << 31) - 1            # the radix passes' multisplit takes n < 2^31 rows


def _itemgetter_of(key, index):
    return (type(key) is operator.itemgetter and key.__reduce__() == operator.itemgetter(index).__reduce__()
            and type(key.__reduce__()[1][0]) is int)


def order_of(key):
    """Which columns a recognised sort key orders by -- ORDER_KV (the identity: the (k, v) tuple), ORDER_K (x[0]) or
    ORDER_V (x[1]) -- or None.  Recognition is structural (textingest._same: the same code, no closure, no defaults);
    an operator.itemgetter is compared by its __reduce__()."""
    if _same(key, _t_identity):
        return ORDER_KV
    if _same(key, _t_first) or _itemgetter_of(key, 0):
        return ORDER_K
    if _same(key, _t_second) or _itemgetter_of(key, 1):
        return ORDER_V
    return None


def device_sort_applies(rdd, key):
    """True when rdd.sort(key, ...) runs on the device: rdd.device_path_applies (a plain ColumnarRDD in a one-process
    job with 1-D int32 / int64 / float32 / float64 columns) with fewer than 2^31 rows, and a recognised key."""
    return device_path_applies([rdd], MAX_ROWS) and order_of(key) is not None


def sample_bounds(rdd, key, reverse, numSplits):
    """RDD.sort's range bounds over rdd, from the same samples the composition takes (the first n rows of every split,
    mapped by key), read from column slices instead of through compute.  [] for a single split or none."""
    if len(rdd) <= 1:
        return []
    if numSplits is None:
        numSplits = min(rdd.ctx.defaultMinSplits, len(rdd))
    n = max(numSplits * 10 // len(rdd), 1)
    samples = []
    for sp in rdd.splits:
        end = min(sp.end, sp.begin + n)
        samples.extend(map(key, zip(rdd.keys[sp.begin:end].tolist(), rdd.vals[sp.begin:end].tolist())))
    return range_bounds(samples, numSplits, reverse)


def _bound_bits(values, dtype, dev):
    """Python bound values as the widened bits dpk_sort_cuts reads: int64 for int columns, float64 bits for floats."""
    if dtype.is_floating_point:
        bits = [struct.unpack("<q", struct.pack("<d", float(v)))[0] for v in values]
    else:
        bits = [int(v) for v in values]
    return torch.tensor(bits, dtype=torch.int64).to(dev)


def sort_columns(rdd, order, reverse, bounds):
    """The sorted rows of a ColumnarRDD cut at RangePartitioner(bounds, reverse): a list of len(bounds) + 1 tuples
    (keys, values) of CUDA tensors in the input dtypes, or None when an order column holds a NaN."""
    from .engine import _device
    dev = _device()
    keys, vals = rdd.keys.to(dev).contiguous(), rdd.vals.to(dev).contiguous()
    P = len(bounds) + 1
    n = int(keys.numel())
    if n == 0:
        return [(keys, vals)] * P
    col0, col1 = {ORDER_KV: (keys, vals), ORDER_K: (keys, None), ORDER_V: (vals, None)}[order]
    w0, w1, ids, nan = nv.sort_keys(col0, col1, reverse)
    if int(nan.item()):
        return None
    if order == ORDER_KV:           # LSD over two words: by v, then stably by k
        _, ids = shuffle.sort_by_key_bits(w1, ids)
        del w1
        w0, ids = shuffle.sort_by_key_bits(nv.gather_i64(w0, ids), ids)
    else:
        w0, ids = shuffle.sort_by_key_bits(w0, ids)
    ordered = sorted(bounds)        # RangePartitioner.keys
    if order == ORDER_KV:
        b0 = _bound_bits([b[0] for b in ordered], keys.dtype, dev)
        b1 = _bound_bits([b[1] for b in ordered], vals.dtype, dev)
    else:
        b0, b1 = _bound_bits(ordered, col0.dtype, dev), None
    starts = nv.sort_cuts(w0, ids, vals, b0, col0.dtype, b1, reverse).cpu().tolist()
    del w0
    sk, sv = nv.sort_gather(keys, vals, ids)
    return [(sk[starts[p]:starts[p + 1]], sv[starts[p]:starts[p + 1]]) for p in range(P)]


class ColumnarSortedRDD(DeviceResultRDD):
    """The result of sort(key, reverse, numSplits) of a numeric ColumnarRDD in a one-process job with a recognised key:
    the partitions of RDD.sort's composition, computed on the GPU the first time a partition is asked for and kept.  The
    range bounds are sampled at construction, as the composition samples them.  Like the composition's mapPartitions
    it has no partitioner.  columns(split) hands out CUDA tensors (keys, values) in the input dtypes; when an order
    column holds a NaN the composition's rows stand."""

    def __init__(self, parent, key, reverse, numSplits, taskMemory=None, rddconf=None):
        DeviceResultRDD.__init__(self, parent.ctx)
        self.parent = parent
        self.key, self.reverse, self.numSplits = key, reverse, numSplits
        self.taskMemory, self.sort_rddconf = taskMemory, rddconf
        self.order = order_of(key)
        self.bounds = sample_bounds(parent, key, reverse, numSplits)
        # no partitions for an input without splits, as the composition returns that input itself
        self._splits = [Split(i) for i in range(len(self.bounds) + 1)] if len(parent) else []

    def parents(self):
        return [self.parent]

    def _run(self):
        return sort_columns(self.parent, self.order, self.reverse, self.bounds)

    def _composition(self):
        return self.parent._sort_rows(self.key, self.reverse, self.numSplits, self.taskMemory, self.sort_rddconf)

    def _columns_of_rows(self, rows, dev):
        return (torch.tensor([k for k, _ in rows], dtype=self.parent.keys.dtype, device=dev),
                torch.tensor([v for _, v in rows], dtype=self.parent.vals.dtype, device=dev))
