"""RDD operator surface for the shuffle hot path -- the reference's names,
signatures and result semantics (dpark/rdd.py) over the GPU shuffle engine.

Only what a user of reduceByKey / groupByKey / combineByKey touches is here
(SURVEY.md §8b seam 1): sources (ParallelCollection, TextFileRDD, ColumnarRDD),
narrow Python-side operators that feed or consume a shuffle (map, flatMap,
filter, mapValue, glom, union ...), the shuffle itself (ShuffledRDD) and the
actions (collect, collectAsMap, count, saveAsTextFile ...).  The narrow
operators are plain Python generators, as in the reference; every shuffle runs
on the GPU through dpark_b200.shuffle -- there is no CPU shuffle.
"""
import itertools
import math
import operator
import os
import random
import shutil

import numpy as np

from . import columnar, conf, quantiles, trace
from .dependency import (Aggregator, GroupByAggregator, HashPartitioner, Partitioner, RangePartitioner,
                         ShuffleDependency)
from .errors import DparkUserFatalError  # noqa: F401

_enumerate = enumerate      # RDD.enumerate shadows the builtin inside the class body


def top_values(top_n, order_func, reverse):
    """topByKey's per-key function: the first top_n values of a stable sort by order_func."""
    def best(values):
        return sorted(values, key=order_func, reverse=reverse)[:top_n]
    return best


def range_bounds(samples, numSplits, reverse):
    """RDD.sort's range bounds (dpark/rdd.py:273-287) from its samples (the first rows of every split, mapped by the
    key): every 10th of the sorted samples, from the 6th on, at most numSplits - 1 of them."""
    return sorted(samples, reverse=reverse)[5::10][:numSplits - 1]


class Split(object):
    def __init__(self, index):
        self.index = index


class RDD(object):
    def __init__(self, ctx):
        self.ctx = ctx
        self.id = ctx.newRddId()
        self._splits = []
        self._dependencies = []
        self.partitioner = None
        self.mem = None
        self.rddconf = None
        self._cache = None
        self.should_cache = False

    # ------------------------------------------------------------------ plumbing
    @property
    def splits(self):
        return self._splits

    def __len__(self):
        return len(self.splits)

    def __repr__(self):
        return "<%s>" % self.__class__.__name__

    def compute(self, split):
        raise NotImplementedError

    def parents(self):
        """RDDs this one reads (the lineage walk of dpark_b200.spmd: under torch.distributed every rank must enter a
        shuffle's collectives, also a rank that owns none of the partitions being computed)."""
        return []

    def iterator(self, split):
        if self.should_cache:
            if self._cache is None:
                self._cache = {}
            if split.index not in self._cache:
                self._cache[split.index] = list(self.compute(split))
            return iter(self._cache[split.index])
        return self.compute(split)

    def cache(self):
        self.should_cache = True
        return self

    def uncache(self):
        """Drop the cached partitions (they are recomputed from the lineage if read again)."""
        self._cache = None
        return self

    def set_rddconf(self, rddconf):
        self.rddconf = conf.default_rddconf.dup() if rddconf is None else rddconf

    # -------------------------------------------------------------- narrow ops
    def map(self, f):
        return MappedRDD(self, f)

    def flatMap(self, f):
        return FlatMappedRDD(self, f)

    def filter(self, f):
        return FilteredRDD(self, f)

    def glom(self):
        return GlommedRDD(self)

    def mapPartitions(self, f):
        return MapPartitionsRDD(self, f)

    mapPartition = mapPartitions

    def mapPartitionWithIndex(self, f):
        return MapPartitionsRDD(self, f, with_index=True)

    def mapValue(self, f):
        return MappedValuesRDD(self, f)

    mapValues = mapValue

    def flatMapValue(self, f):
        return FlatMappedValuesRDD(self, f)

    def keyBy(self, f):
        return self.map(lambda x: (f(x), x))

    def union(self, *others):
        return UnionRDD(self.ctx, [self] + list(others))

    def __add__(self, other):
        return self.union(other)

    # ----------------------------------------------------------------- actions
    def collect(self):
        """Concatenation of the partitions in index order (dpark/schedule.py:669-672)."""
        return list(itertools.chain.from_iterable(self.ctx.runJob(self, list)))

    def __iter__(self):
        return iter(self.collect())

    def collectAsMap(self):
        d = {}
        for part in self.ctx.runJob(self, list):
            d.update(part)
        return d

    def count(self):
        return sum(self.ctx.runJob(self, lambda it: sum(1 for _ in it)))

    def reduce(self, f):
        def part(it):
            it = iter(it)
            try:
                acc = next(it)
            except StopIteration:
                return []
            for x in it:
                acc = f(acc, x)
            return [acc]
        vals = list(itertools.chain.from_iterable(self.ctx.runJob(self, part)))
        if not vals:
            return None
        acc = vals[0]
        for x in vals[1:]:
            acc = f(acc, x)
        return acc

    def foreach(self, f):
        def run(it):
            for x in it:
                f(x)
        list(self.ctx.runJob(self, run))

    def take(self, n):
        out = []
        for part in self.ctx.runJob(self, list):
            out.extend(part[:n - len(out)])
            if len(out) >= n:
                break
        return out

    def first(self):
        r = self.take(1)
        return r[0] if r else None

    def saveAsTextFile(self, path, ext="", overwrite=True, compress=False):
        return OutputTextFileRDD(self, path, ext, overwrite, compress).collect()

    def lookup(self, key):
        """dpark/rdd.py lookup: with a partitioner only the key's partition is
        scanned; a (k, v) RDD answers the value, None when absent."""
        if self.partitioner is not None:
            idx = self.partitioner.getPartition(key)
            for k, v in self.iterator(self.splits[idx]):
                if k == key:
                    return v
            return None
        for k, v in self.collect():
            if k == key:
                return v
        return None

    # ------------------------------------------------------------- the shuffle
    def sample(self, faction, withReplacement=False, seed=12345):
        """dpark/rdd.py:267-268.

        A numeric ColumnarRDD in a one-process job, sampled without replacement by an int or float fraction, is sampled
        on the device (dpark_b200/sampling.py), with the same splits and rows as SampleRDD."""
        from . import sampling
        if sampling.sample_applies(self, faction, withReplacement):
            return sampling.ColumnarSampleRDD(self, faction, withReplacement, seed)
        return SampleRDD(self, faction, withReplacement, seed)

    def percentiles(self, p, sampleRate=1.0, func=None):
        """dpark/rdd.py:791-814: one t-digest per partition, merged in partition order."""
        if sampleRate <= 0:
            raise ValueError("Sample Rate should be positive.")
        rdd = self if sampleRate >= 1.0 else self.sample(sampleRate)
        if func:
            rdd = rdd.map(func)
        return quantiles.percentiles_of_partitions(self.ctx.runJob(rdd, list), p)

    def _skew_thresholds(self, splits, sampleRate):
        """Thresholds of combineByKey(fixSkew=sampleRate) (dpark/rdd.py:516-537): approximate percentiles of
        portable_hash(key) over a sample of the rows.

        A numeric ColumnarRDD, or a union of them, in a one-process job is sampled, hashed and digested on the device
        (dpark_b200/sampling.py), with the same thresholds as this composition."""
        from . import sampling
        inputs = sampling.thresholds_inputs(self, sampleRate)
        if inputs is not None:
            res = sampling.skew_thresholds(inputs, splits, sampleRate)
            if res is not None:
                return res
        return self._skew_thresholds_rows(splits, sampleRate)

    def _skew_thresholds_rows(self, splits, sampleRate):
        """_skew_thresholds' composition over the rows: the sampled keys of every partition are hashed on the
        device in one launch; the digest arithmetic is the reference's (dpark_b200/quantiles.py)."""
        rdd = self if sampleRate >= 1.0 else self.sample(sampleRate)
        hashed = [columnar.hashes_of_keys([row[0] for row in part])
                  for part in self.ctx.runJob(rdd, list)]
        return quantiles.skew_thresholds(hashed, splits)

    def combineByKey(self, aggregator, splits=None, taskMemory=None, fixSkew=-1, rddconf=None):
        """dpark/rdd.py:511-541.  `splits` is a partition count or a Partitioner; fixSkew > 0 is the sample
        rate for balancing the partitions by hash thresholds instead of hash modulo."""
        return ShuffledRDD(self, aggregator, self._combine_partitioner(splits, fixSkew), taskMemory, rddconf=rddconf)

    def _combine_partitioner(self, splits, fixSkew):
        """The partitioner of combineByKey(splits, fixSkew=...) (dpark/rdd.py:511-541): splits defaults to
        min(defaultMinSplits, partitions); an int becomes a HashPartitioner, with thresholds sampled over self when
        fixSkew > 0; a Partitioner is taken as it is."""
        if splits is None:
            splits = min(self.ctx.defaultMinSplits, len(self))
        if type(splits) is int:
            thresh = None
            if fixSkew > 0 and splits > 1:
                thresh, splits = self._skew_thresholds(splits, fixSkew)
            splits = HashPartitioner(splits, thresholds=thresh)
        return splits

    def _device_partitioner(self, numSplits, fixSkew=-1):
        """_combine_partitioner(numSplits, fixSkew) if a device group-by can take it -- a HashPartitioner -- else None
        (the composition's group-by refuses every other partitioner as well)."""
        part = self._combine_partitioner(numSplits, fixSkew)
        return part if isinstance(part, HashPartitioner) else None

    def reduceByKey(self, func, numSplits=None, taskMemory=None, fixSkew=-1, rddconf=None):
        """dpark/rdd.py:543-545."""
        aggregator = Aggregator(lambda x: x, func, func)
        return self.combineByKey(aggregator, numSplits, taskMemory, fixSkew=fixSkew, rddconf=rddconf)

    def groupByKey(self, numSplits=None, taskMemory=None, fixSkew=-1, rddconf=None):
        """dpark/rdd.py:547-550."""
        return self.combineByKey(GroupByAggregator(), numSplits, taskMemory, fixSkew=fixSkew, rddconf=rddconf)

    def groupWith(self, others, numSplits=None, taskMemory=None, fixSkew=-1, rddconf=None):
        """dpark/rdd.py:686-731: (k, (values of self, values of others[0], ...)) for every key of any input.

        Numeric ColumnarRDDs in a one-process job are grouped on the device (dpark_b200/join.py), with the same
        partitions, keys and value lists as CoGroupedRDD."""
        if isinstance(others, RDD):
            others = [others]
        others = list(others)
        part = self._cogroup_partitioner(others, numSplits, fixSkew)
        if device_path_applies([self] + others):
            from . import join
            return join.ColumnarCoGroupedRDD([self] + others, part)
        return CoGroupedRDD([self] + others, part, taskMemory, rddconf=rddconf)

    def _cogroup_partitioner(self, others, numSplits, fixSkew):
        """The partitioner of a cogroup of self and others (dpark/rdd.py:686-731): numSplits defaults to self's
        partition count if self is partitioned, else defaultParallelism; fixSkew > 0 samples hash thresholds over
        the union of the inputs."""
        if numSplits is None:
            numSplits = self.partitioner.numPartitions if self.partitioner is not None else self.ctx.defaultParallelism
        thresh = None
        if fixSkew > 0 and numSplits > 1:
            thresh, numSplits = self.union(*others)._skew_thresholds(numSplits, fixSkew)
        return HashPartitioner(numSplits, thresholds=thresh)

    cogroup = groupWith

    def join(self, other, numSplits=None, taskMemory=None, fixSkew=-1, rddconf=None):
        """dpark/rdd.py:649-650."""
        return self._join(other, (), numSplits, taskMemory, fixSkew=fixSkew, rddconf=rddconf)

    def leftOuterJoin(self, other, numSplits=None, taskMemory=None, fixSkew=-1, rddconf=None):
        return self._join(other, (1,), numSplits, taskMemory, fixSkew=fixSkew, rddconf=rddconf)

    def rightOuterJoin(self, other, numSplits=None, taskMemory=None, fixSkew=-1, rddconf=None):
        return self._join(other, (2,), numSplits, taskMemory, fixSkew=fixSkew, rddconf=rddconf)

    def outerJoin(self, other, numSplits=None, taskMemory=None, fixSkew=-1, rddconf=None):
        return self._join(other, (1, 2), numSplits, taskMemory, fixSkew=fixSkew, rddconf=rddconf)

    def _join(self, other, keeps, numSplits=None, taskMemory=None, fixSkew=-1, rddconf=None):
        """dpark/rdd.py:661-676: the cross product of the two value lists of every key; `keeps` names the sides
        (1 = left, 2 = right) whose unmatched keys survive, paired with None.

        Two numeric ColumnarRDDs in a one-process job are joined on the device (dpark_b200/join.py), with the same
        partitions, rows and order as this composition."""
        keep_left, keep_right = 1 in keeps, 2 in keeps
        if device_path_applies([self, other]):
            from . import join
            return join.ColumnarJoinedRDD(self, other, self._cogroup_partitioner([other], numSplits, fixSkew),
                                          keep_left, keep_right)

        def pairs(row):
            k, (left, right) = row
            if not left and keep_right:
                left = [None]
            if not right and keep_left:
                right = [None]
            return ((k, (a, b)) for a in left for b in right)

        return self.cogroup(other, numSplits, taskMemory, fixSkew=fixSkew, rddconf=rddconf).flatMap(pairs)

    def uniq(self, numSplits=None, taskMemory=None, rddconf=None):
        """dpark/rdd.py:383-385: the distinct elements, partitioned by their hash.  The reference merges `None`
        values with `lambda x, y: None`; the GPU shuffle needs a recognised op, so the placeholder value is 0
        merged with `or` -- the keys and their partitions are the same.

        A numeric ColumnarRDD in a one-process job, partitioned by a HashPartitioner, is deduplicated on the device
        (dpark_b200/selecting.py): the same partitions and elements, each partition's elements in order of first
        occurrence with the bits of that occurrence."""
        from . import selecting
        if selecting.uniq_applies(self):
            part = self._device_partitioner(numSplits)
            if part is not None:
                return selecting.ColumnarUniqRDD(self, part)
        import operator
        return self.map(lambda x: (x, 0)).reduceByKey(operator.or_, numSplits, taskMemory, rddconf=rddconf) \
                   .map(lambda kv: kv[0])

    def top(self, n=10, key=None, reverse=False):
        """dpark/rdd.py:387-394: the n largest (smallest with reverse) elements; per partition, then overall.

        A numeric ColumnarRDD in a one-process job, with an int n and the identity (key None), x[0] or x[1] as the key,
        is selected on the device (dpark_b200/selecting.py): the same list, ties in (split, position) order.  A NaN in
        an order column keeps this composition."""
        from . import selecting
        if selecting.top_applies(self, n, key):
            res = selecting.top(self, n, key, reverse)
            if res is not None:
                return res
        import heapq
        pick = heapq.nsmallest if reverse else heapq.nlargest
        best = []
        for part in self.ctx.runJob(self, lambda it: pick(n, it, key)):
            best.extend(part)
        return pick(n, best, key)

    def hot(self, n=10, numSplits=None, taskMemory=None, rddconf=None):
        """dpark/rdd.py:396-398: the n most frequent elements with their counts.

        A numeric ColumnarRDD in a one-process job, with an int n and a HashPartitioner, is counted on the device
        (dpark_b200/selecting.py): a stable top n by count over uniq's order of the elements."""
        from . import selecting
        if selecting.hot_applies(self, n):
            part = self._device_partitioner(numSplits)
            if part is not None:
                return selecting.hot(self, n, part)
        counts = self.map(lambda x: (x, 1)).reduceByKey(lambda a, b: a + b, numSplits, taskMemory, rddconf=rddconf)
        return counts.top(n, key=lambda kv: kv[1])

    def topByKey(self, top_n, order_func=None, reverse=False, num_splits=None, task_memory=None, fixSkew=-1):
        """dpark/rdd.py:552-594: per key the top_n values by `order_func` (the value itself when None), ascending,
        or the top_n largest in descending order with reverse=True; values that compare equal keep the order in
        which they were met -- (input partition, position) -- and the oldest ones win.

        The reference keeps a bounded heap per key on both sides of the shuffle (HeapAggregator,
        dpark/dependency.py:164-193) over (order, partition, sequence, value) tuples.  The GPU group-by already
        delivers every key's values in (partition, position) order, so the same answer is a stable sort of that
        list (Python's sort is stable for reverse=True as well) cut at top_n.

        A numeric ColumnarRDD in a one-process job, with no order_func and top_n <= topk.TOPK_MAX_N, is selected on
        the device (dpark_b200/topk.py), with the same partitions, keys, values and order as this composition."""
        if top_n <= 0:
            raise AssertionError("top_n must be positive")
        from . import topk
        if order_func is None and type(top_n) is int and top_n <= topk.TOPK_MAX_N and device_path_applies([self]):
            part = self._device_partitioner(num_splits, fixSkew)
            if part is not None:
                return topk.ColumnarTopByKeyRDD(self, part, top_n, reverse)
        return self.groupByKey(num_splits, task_memory, fixSkew=fixSkew).mapValue(top_values(top_n, order_func, reverse))

    def sort(self, key=lambda x: x, reverse=False, numSplits=None, taskMemory=None, rddconf=None):
        """dpark/rdd.py:273-287: a globally sorted RDD.  Range bounds come from the first elements of every
        partition exactly as in the reference (range_bounds); each element is routed to its range on the host
        (RangePartitioner) and the shuffle runs on the GPU keyed by the RANGE INDEX -- portable_hash(i) % P == i for
        0 <= i < P, so HashPartitioner(P) reproduces the reference's layout -- then every partition is sorted.

        A numeric ColumnarRDD in a one-process job, sorted by the identity, x[0] or x[1], is sorted on the device
        (dpark_b200/sorting.py), with the same partitions and rows in the same order as this composition."""
        from . import sorting
        if sorting.device_sort_applies(self, key):
            return sorting.ColumnarSortedRDD(self, key, reverse, numSplits, taskMemory, rddconf)
        return self._sort_rows(key, reverse, numSplits, taskMemory, rddconf)

    def _sort_rows(self, key, reverse, numSplits, taskMemory, rddconf):
        """RDD.sort's composition over the rows."""
        if not len(self):
            return self
        if len(self) == 1:
            return self.mapPartitions(lambda it: sorted(it, key=key, reverse=reverse))
        if numSplits is None:
            numSplits = min(self.ctx.defaultMinSplits, len(self))
        n = max(numSplits * 10 // len(self), 1)
        samples = self.mapPartitions(lambda it: itertools.islice(it, n)).map(key).collect()
        ranges = RangePartitioner(range_bounds(samples, numSplits, reverse), reverse=reverse)
        routed = self.map(lambda x: (ranges.getPartition(key(x)), x)) \
                     .groupByKey(ranges.numPartitions, taskMemory, rddconf=rddconf)
        return routed.flatMap(lambda kv: kv[1]).mapPartitions(lambda it: sorted(it, key=key, reverse=reverse))

    def groupBy(self, f, numSplits=None, rddconf=None):
        """dpark/rdd.py:298-301."""
        if numSplits is None:
            numSplits = min(self.ctx.defaultMinSplits, len(self))
        return self.map(lambda x: (f(x), x)).groupByKey(numSplits, rddconf=rddconf)

    def update(self, other, replace_only=False, numSplits=None, taskMemory=None, fixSkew=-1, rddconf=None):
        """dpark/rdd.py:599-624: this (k, v) RDD with the values `other` holds for the same keys put in their
        place; keys only `other` has are added unless replace_only.

        The reference folds (value, origin bit) pairs with an order-sensitive lambda, which the GPU shuffle cannot
        express as one of its ops; the same table falls out of a cogroup: a key's new value is the first one
        `other` holds for it in (input partition, position) order, else its first old value -- the outcome the
        reference's fold gives when it meets the rows in that order."""
        def pick(groups):
            old, new = groups
            return new[0] if new else old[0]

        both = self.groupWith(other, numSplits, taskMemory, fixSkew=fixSkew, rddconf=rddconf)
        if replace_only:
            both = both.filter(lambda kv: bool(kv[1][0]))
        return both.mapValue(pick)

    def innerJoin(self, smallRdd):
        """dpark/rdd.py:626-647: join against a small RDD held as a dict on the host (no shuffle).

        Two numeric ColumnarRDDs in a one-process job, with int keys on both sides or float keys on both (or an empty
        side), are joined on the device (dpark_b200/join.py): the same splits, rows and order as this composition."""
        from . import join
        if join.inner_join_applies(self, smallRdd):
            return join.ColumnarInnerJoinedRDD(self, smallRdd)
        import collections
        table = collections.defaultdict(list)
        for k, v in smallRdd.collect():
            table[k].append(v)

        def matches(kv):
            k, v = kv
            return [(k, (v, w)) for w in table.get(k, ())]

        return self.flatMap(matches)

    def percentilesByKey(self, p, sampleRate=1.0, func=None, numSplits=None, taskMemory=None, fixSkew=-1):
        """dpark/rdd.py:815-850: per key the requested percentiles of its values (t-digest).  The reference builds
        one digest per key and map task and merges them on the reduce side in fetch order; here the values of a key
        arrive grouped and ordered by (input partition, position), each carries its partition index, and the same
        digests are built and merged in partition order -- one of the orders the reference may take.

        A numeric ColumnarRDD in a one-process job, with sampleRate >= 1 and no func, is digested on the device
        (dpark_b200/percentiles.py), with the same partitions, keys and percentiles, bit for bit, as this composition."""
        if sampleRate <= 0:
            raise ValueError("Sample Rate should be positive.")
        from . import percentiles
        if sampleRate >= 1.0 and func is None and device_path_applies([self]):
            part = self._device_partitioner(numSplits, fixSkew)
            if part is not None:
                return percentiles.ColumnarPercentilesByKeyRDD(self, part, p)
        rdd = self if sampleRate >= 1.0 else self.sample(sampleRate)
        if func:
            rdd = rdd.mapValue(func)
        return rdd._percentiles_rows(p, numSplits, taskMemory, fixSkew)

    def _percentiles_rows(self, p, numSplits=None, taskMemory=None, fixSkew=-1):
        """percentilesByKey's composition over the rows of self (already sampled and mapped)."""
        def quantiles_of(tagged):
            merged, current, digest = None, None, None
            for part, x in tagged:
                if part != current:
                    if digest is not None:
                        merged = digest if merged is None else merged.absorb(digest)
                        merged.compress()
                    current, digest = part, quantiles.MergingDigest()
                digest.add(x)
            if digest is not None:
                merged = digest if merged is None else merged.absorb(digest)
                merged.compress()
            return [merged.quantile(pp / 100.) for pp in p]

        tagged = self.mapPartitionWithIndex(lambda i, it: ((k, (i, v)) for k, v in it))
        return tagged.groupByKey(numSplits, taskMemory, fixSkew=fixSkew).mapValue(quantiles_of)

    def fold(self, zero, f):
        """dpark/rdd.py:400-408."""
        import copy
        import functools
        return functools.reduce(f, self.ctx.runJob(self, lambda it: functools.reduce(f, it, copy.copy(zero))), zero)

    def aggregate(self, zero, seqOp, combOp):
        """dpark/rdd.py:410-422."""
        import copy
        import functools
        return functools.reduce(combOp, self.ctx.runJob(self, lambda it: functools.reduce(seqOp, it, copy.copy(zero))),
                                zero)

    def toList(self):
        return self.collect()

    def foreachPartition(self, f):
        list(self.ctx.runJob(self, f))

    def enumeratePartition(self):
        """dpark/rdd.py:326-327: (partition index, element)."""
        return self.mapPartitionWithIndex(lambda i, it: ((i, x) for x in it))

    def enumerate(self):
        """dpark/rdd.py:329-345: (global position, element), positions counted partition after partition."""
        sizes = list(self.ctx.runJob(self, lambda it: sum(1 for _ in it))) if len(self) > 1 else [0]
        starts = [0]
        for c in sizes[:-1]:
            starts.append(starts[-1] + c)
        return self.mapPartitionWithIndex(lambda i, it: ((starts[i] + j, x) for j, x in _enumerate(it)))

    def partitionByKey(self, numSplits=None, taskMemory=None, rddconf=None):
        return self.groupByKey(numSplits, taskMemory, rddconf=rddconf).flatMapValue(lambda x: x)

    def reduceByKeyToDriver(self, func):
        """dpark/rdd.py:503-509 (driver-side merge of per-row dicts); here simply
        the shuffle followed by collectAsMap."""
        return self.reduceByKey(func).collectAsMap()


class DerivedRDD(RDD):
    def __init__(self, prev):
        RDD.__init__(self, prev.ctx)
        self.prev = prev
        self._splits = prev.splits

    def parents(self):
        return [self.prev]

    @property
    def splits(self):
        return self.prev.splits


class MappedRDD(DerivedRDD):
    def __init__(self, prev, f):
        DerivedRDD.__init__(self, prev)
        self.func = f

    def compute(self, split):
        return map(self.func, self.prev.iterator(split))


class FlatMappedRDD(MappedRDD):
    def compute(self, split):
        return itertools.chain.from_iterable(map(self.func, self.prev.iterator(split)))


class FilteredRDD(MappedRDD):
    def compute(self, split):
        return filter(self.func, self.prev.iterator(split))


class SampleRDD(DerivedRDD):
    """dpark/rdd.py:1379-1397: Bernoulli (or with-replacement) sample, `random.Random(seed + split.index)`
    per partition -- the same generator and the same draw order, so the same rows are kept."""

    def __init__(self, prev, frac, withReplacement, seed):
        DerivedRDD.__init__(self, prev)
        self.frac, self.withReplacement, self.seed = frac, withReplacement, seed

    def compute(self, split):
        rd = random.Random(self.seed + split.index)
        if self.withReplacement:
            rows = list(self.prev.iterator(split))
            for _ in range(int(math.ceil(len(rows) * self.frac))):
                yield rd.choice(rows)
        else:
            for row in self.prev.iterator(split):
                if rd.random() <= self.frac:
                    yield row


class GlommedRDD(DerivedRDD):
    def compute(self, split):
        yield list(self.prev.iterator(split))


class MapPartitionsRDD(DerivedRDD):
    def __init__(self, prev, f, with_index=False):
        DerivedRDD.__init__(self, prev)
        self.func, self.with_index = f, with_index

    def compute(self, split):
        it = self.prev.iterator(split)
        return self.func(split.index, it) if self.with_index else self.func(it)


class MappedValuesRDD(MappedRDD):
    """Keeps the parent's partitioner: keys are untouched (dpark/rdd.py MappedValuesRDD)."""

    def __init__(self, prev, f):
        MappedRDD.__init__(self, prev, f)
        self.partitioner = prev.partitioner

    def compute(self, split):
        f = self.func
        return ((k, f(v)) for k, v in self.prev.iterator(split))


class FlatMappedValuesRDD(MappedValuesRDD):
    def compute(self, split):
        f = self.func
        return ((k, x) for k, v in self.prev.iterator(split) for x in f(v))


class UnionRDD(RDD):
    def __init__(self, ctx, rdds):
        RDD.__init__(self, ctx)
        self.rdds = rdds
        self._splits = []
        for r in rdds:
            for s in r.splits:
                sp = Split(len(self._splits))
                sp.rdd, sp.split = r, s
                self._splits.append(sp)

    def compute(self, split):
        return split.rdd.iterator(split.split)


class ParallelCollection(RDD):
    """dpark/rdd.py:1556-1598: a list cut into numSlices contiguous chunks of
    ceil(len/numSlices) (numSlices capped to len; trailing chunks may be empty)."""

    def __init__(self, ctx, data, numSlices, taskMemory=None):
        RDD.__init__(self, ctx)
        data = data if isinstance(data, (list, range)) else list(data)
        self.size = len(data)
        k = max(1, min(self.size, numSlices))
        if k <= 0:
            raise ValueError("invalid numSlices %d" % numSlices)
        if self.size == 0:
            chunks = [[]]
        else:
            per = -(-self.size // k)
            chunks = [data[i * per:i * per + per] for i in range(k)]
        self._splits = []
        for i, c in enumerate(chunks):
            sp = Split(i)
            sp.values = c
            self._splits.append(sp)

    def compute(self, split):
        return iter(split.values)


class ColumnarRDD(RDD):
    """Extension: a (k, v) RDD whose partitions are already columns -- numpy
    arrays or torch tensors (host or cuda).  This is how 1e8..1e9-row inputs
    enter without ever becoming Python tuples; a ShuffledRDD on top of it takes
    the columns as they are."""

    def __init__(self, ctx, keys, vals, numSlices, bounds=None):
        """bounds: optional split row bounds, a non-decreasing int sequence from 0 to the row count -- split i holds
        rows [bounds[i], bounds[i + 1]) and numSlices is not used.  Without it the rows are cut into numSlices
        blocks of ceil(n / numSlices)."""
        RDD.__init__(self, ctx)
        import torch
        self.keys = keys if torch.is_tensor(keys) else torch.from_numpy(np.ascontiguousarray(keys))
        self.vals = vals if torch.is_tensor(vals) else torch.from_numpy(np.ascontiguousarray(vals))
        if self.keys.numel() != self.vals.numel():
            raise DparkUserFatalError("ragged pair columns: %d keys, %d values"
                                      % (self.keys.numel(), self.vals.numel()))
        n = int(self.keys.numel())
        if bounds is not None:
            cuts = _split_bounds(bounds, n)
        else:
            k = max(1, min(n, numSlices)) if n else 1
            per = -(-n // k) if n else 0
            cuts = [min(n, i * per) for i in range(k)] + [min(n, k * per)]
        self._splits = []
        for i in range(len(cuts) - 1):
            sp = Split(i)
            sp.begin, sp.end = cuts[i], cuts[i + 1]
            self._splits.append(sp)

    def columns(self, split):
        return self.keys[split.begin:split.end], self.vals[split.begin:split.end]

    def compute(self, split):
        k, v = self.columns(split)
        return zip(k.cpu().tolist(), v.cpu().tolist())


def _split_bounds(bounds, n):
    try:
        cuts = list(bounds)
        if any(isinstance(b, bool) for b in cuts):
            raise TypeError("bool")
        cuts = [operator.index(b) for b in cuts]
    except TypeError:
        raise DparkUserFatalError("split bounds must be a sequence of ints, got %r" % (bounds,))
    if not cuts or cuts[0] != 0 or cuts[-1] != n or any(a > b for a, b in zip(cuts, cuts[1:])):
        raise DparkUserFatalError("split bounds must rise from 0 to %d without decreasing, got %r" % (n, cuts))
    return cuts


def device_path_applies(rdds, max_rows=None):
    """True when a columnar operator over rdds may run on the device: every input a ColumnarRDD (not a subclass), one
    process, 1-D key and value columns of int32 / int64 / float32 / float64, and at most max_rows rows in each input
    when a cap is given.  Each operator adds its own argument checks (sorting.device_sort_applies, ...)."""
    import torch
    from . import spmd
    if any(type(r) is not ColumnarRDD for r in rdds) or spmd.rank_world()[1] != 1:
        return False
    if max_rows is not None and any(int(r.keys.numel()) > max_rows for r in rdds):
        return False
    dtypes = (torch.int32, torch.int64, torch.float32, torch.float64)
    return all(t.dtype in dtypes and t.dim() == 1 for r in rdds for t in (r.keys, r.vals))


class DeviceResultRDD(RDD):
    """The result of a columnar operator on the device: every partition is computed in one go the first time any
    partition is asked for, and kept (like ShuffledRDD).  A subclass gives

      _run()                   the device result, or None when the composition's rows must stand instead;
      _rows(columns)           one partition's columns as the composition's rows (by default (keys, values) pairs);
      _part(result, index)     one partition's columns cut from the result (by default result[index]);
      _composition()           and _columns_of_rows(rows, device), where _run may return None.

    columns(split) hands out the partition as CUDA tensors, also when the composition stands."""

    _result = None          # the device result, or the composition RDD whose rows stand

    def _materialize(self):
        if self._result is None:
            res = self._run()
            self._result = res if res is not None else self._composition()
        return self._result

    def _part(self, result, index):
        return result[index]

    def _rows(self, columns):
        keys, vals = columns
        return zip(keys.cpu().tolist(), vals.cpu().tolist())

    def columns(self, split):
        res = self._materialize()
        if isinstance(res, RDD):
            from .engine import _device
            return self._columns_of_rows(list(res.iterator(res.splits[split.index])), _device())
        return self._part(res, split.index)

    def compute(self, split):
        res = self._materialize()
        if isinstance(res, RDD):
            return res.iterator(res.splits[split.index])
        return self._rows(self._part(res, split.index))


class TextFileRDD(RDD):
    """dpark/rdd.py:1633-1711: byte-range splits; a split owns the lines that
    START inside its range (a line straddling the end belongs to the split it
    starts in)."""
    DEFAULT_SPLIT_SIZE = 64 * 1024 * 1024

    def __init__(self, ctx, path, numSplits=None, splitSize=None):
        RDD.__init__(self, ctx)
        self.path = path
        size = os.path.getsize(path)
        if splitSize is None:
            splitSize = self.DEFAULT_SPLIT_SIZE if numSplits is None else (size // numSplits or self.DEFAULT_SPLIT_SIZE)
        n = size // splitSize + (1 if size % splitSize > 0 else 0)
        self.splitSize = splitSize
        self._splits = []
        for i in range(n):
            sp = Split(i)
            sp.begin, sp.end = i * splitSize, min(size, (i + 1) * splitSize)
            self._splits.append(sp)

    def compute(self, split):
        with open(self.path, "rb") as f:
            start, end = split.begin, split.end
            if start > 0:
                f.seek(start - 1)
                byte = f.read(1)
                while byte != b"\n":
                    byte = f.read(1)
                    if not byte:
                        return
                    start += 1
            if start >= end:
                return
            for line in f:
                size = len(line)
                text = line.decode("utf-8")
                yield text[:-1] if text.endswith("\n") else text
                start += size
                if start >= end:
                    break


class OutputTextFileRDD(DerivedRDD):
    """dpark/rdd.py:2097-2161: one file `%04d<ext>` per partition, empty
    partitions write nothing; yields the paths written."""

    def __init__(self, rdd, path, ext="", overwrite=False, compress=False):
        from . import spmd
        rank, world = spmd.rank_world()
        if rank == 0:                      # one driver process per GPU: rank 0 prepares the directory, everyone waits
            if os.path.exists(path):
                if not os.path.isdir(path):
                    raise Exception("output must be dir")
                if overwrite:
                    for n in os.listdir(path):
                        p = os.path.join(path, n)
                        if os.path.isdir(p):
                            shutil.rmtree(p)
                        else:
                            os.remove(p)
            else:
                os.makedirs(path, exist_ok=True)
        if world > 1:
            spmd.barrier()
        DerivedRDD.__init__(self, rdd)
        self.path = os.path.abspath(path)
        if ext and not ext.startswith("."):
            ext = "." + ext
        if compress and not ext.endswith("gz"):
            ext += ".gz"
        self.ext, self.overwrite, self.compress = ext, overwrite, compress

    def compute(self, split):
        path = os.path.join(self.path, "%04d%s" % (split.index, self.ext))
        if os.path.exists(path) and not self.overwrite:
            return
        lines = list(self.prev.iterator(split))
        if not lines:
            return
        tmp = path + ".tmp%d" % os.getpid()
        if self.compress:
            import gzip
            opener = lambda p: gzip.open(p, "wt", encoding="utf-8")  # noqa: E731
        else:
            opener = lambda p: open(p, "w", encoding="utf-8")        # noqa: E731
        with opener(tmp) as f:
            for line in lines:
                f.write(line if line.endswith("\n") else line + "\n")
        os.rename(tmp, path)
        yield path


class _TagValue(object):
    """v -> (input index, v): marks which cogroup input a row came from."""

    def __init__(self, index):
        self.index = index

    def __call__(self, v):
        return (self.index, v)


class CoGroupedRDD(RDD):
    """dpark/rdd.py:1264-1376 with the ordered merger (OrderedCoGroupDiskHashMerger, dpark/shuffle.py:683-719):
    per key one value list per input, each ordered by (map split of that input, position).

    On this path a cogroup IS a group-by: the inputs that need a shuffle are concatenated (in dependency order),
    every value is tagged with its input index, one ordered groupByKey runs on the GPU (values are host objects
    addressed by row id, dpark_b200/grouping.py), and the tag splits each key's list again -- a stable split, so
    the (map split, position) order inside every input survives.

    An input that is already partitioned by the same partitioner is NOT shuffled (the reference's narrow
    dependency, dpark/rdd.py:1280-1293): its partition j is read as is and merged into partition j of the result,
    values in the partition's own iteration order.  Iterative jobs live on this -- in Bagel both inputs of the
    superstep's groupWith (the vertices of the previous superstep, the combined messages) carry the partitioner."""

    def __init__(self, rdds, partitioner, taskMemory=None, rddconf=None):
        RDD.__init__(self, rdds[0].ctx)
        self.size = len(rdds)
        self.rdds = list(rdds)
        self.partitioner = partitioner
        if taskMemory:
            self.mem = taskMemory
        self.narrow = [i for i, r in enumerate(rdds) if r.partitioner == partitioner]
        moved = [i for i in range(self.size) if i not in self.narrow]
        self._grouped = None
        if moved:
            tagged = UnionRDD(self.ctx, [MappedValuesRDD(rdds[i], _TagValue(i)) for i in moved])
            self._grouped = ShuffledRDD(tagged, GroupByAggregator(), partitioner, taskMemory, rddconf=rddconf)
            self._dependencies = self._grouped._dependencies
        self.set_rddconf(rddconf)
        self.rddconf = self.rddconf.dup(op=conf.OP_COGROUP)
        self._splits = [Split(i) for i in range(partitioner.numPartitions)]

    def compute(self, split):
        merged = {}

        def lists_of(k):
            groups = merged.get(k)
            if groups is None:
                groups = merged[k] = tuple([] for _ in range(self.size))
            return groups

        if self._grouped is not None:
            for k, tagged in self._grouped.iterator(self._grouped.splits[split.index]):
                groups = lists_of(k)
                for i, v in tagged:
                    groups[i].append(v)
        for i in self.narrow:
            rdd = self.rdds[i]
            for k, v in rdd.iterator(rdd.splits[split.index]):
                lists_of(k)[i].append(v)
        return iter(merged.items())


def _parents_of_union(self):
    return list(self.rdds)


UnionRDD.parents = _parents_of_union


def _parents_of_cogroup(self):
    return ([self._grouped] if self._grouped is not None else []) + [self.rdds[i] for i in self.narrow]


CoGroupedRDD.parents = _parents_of_cogroup


class ShuffledRDD(RDD):
    """dpark/rdd.py:1101-1134.  The plan node is built eagerly (aggregator is
    recognised at construction, so unsupported combiners fail when the job is
    declared, not in the middle of it); the shuffle itself runs once, on the
    GPU, the first time any partition is asked for, and is reused afterwards
    (the reference caches map outputs per shuffleId the same way)."""

    def __init__(self, parent, aggregator, part, taskMemory=None, rddconf=None):
        RDD.__init__(self, parent.ctx)
        if not isinstance(part, Partitioner):
            raise TypeError("splits must be an int or a Partitioner")
        if not isinstance(part, HashPartitioner):
            raise NotImplementedError("only HashPartitioner is supported on the GPU shuffle path")
        self.parent = parent
        self.aggregator = aggregator
        self.partitioner = part
        if taskMemory:
            self.mem = taskMemory
        self._splits = [Split(i) for i in range(part.numPartitions)]
        self.shuffleId = self.ctx.newShuffleId()
        self.set_rddconf(rddconf)
        self._dependencies = [ShuffleDependency(self.shuffleId, parent, aggregator, part, self.rddconf)]
        self.kind, self.op = trace.recognize_aggregator(aggregator)
        if self.kind == "group":
            self.rddconf.op = conf.OP_GROUPBY
        self._result = None

    def parents(self):
        return [self.parent]

    def _materialize(self):
        if self._result is None:
            from . import engine
            self._result = engine.run_shuffle(self)
        return self._result

    def compute(self, split):
        return iter(self._materialize().rows(split.index))

    def columns(self, split):
        """Extension: the partition as columns (numpy) instead of Python rows."""
        return self._materialize().columns(split.index)
