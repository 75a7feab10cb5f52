"""sample and the fixSkew thresholds of numeric ColumnarRDDs on one GPU (dpark/rdd.py:267-268, 516-537, 1379-1397).

SampleRDD keeps row j of split i when the j-th random.Random(seed + i).random() is <= frac, one draw per row, in Python.
combineByKey(fixSkew=rate) and the cogroups derive their HashPartitioner thresholds from such a sample (seed 12345) of
the input, or of the union of the inputs: every kept key is hashed, each split's hashes go into a pure-Python
MergingDigest, the digests are merged in split order and queried (quantiles.skew_thresholds).  When the inputs already
are columns the same numbers come from the device:

  1. the draws: random.Random's generator is MT19937, exact integer arithmetic.  The host takes each split's state
     right after seeding from random.Random(seed + i).getstate(); dpk_sample_bernoulli replays the stream, one CTA per
     split, and writes the kept row ids in row order (one host read: the per-split counts);
  2. the hashes: each input's key column in its own kind (int widened to int64, float to float64 + 0.0), dpk_hash_keys
     -- the keys of one split are all int or all float, as the composition hashes them per split;
  3. the digests: one segment per split with kept rows, MergingDigest().update(hashes) + compress() each
     (dpk_tdigest_build), then one absorb chain in split order and the quantiles at the composition's fractions
     (dpk_tdigest_merge, one group).

The composition starts its chain from the FIRST split's digest even when that split kept nothing: the first non-empty
digest then enters through E.absorb(d), a refold of d's centroids with lo / hi of its own.  The device digest of that
split is refolded on the host with quantiles.MergingDigest (at most TD_CAP centroids) and written back before the merge.

A NaN key among the kept rows raises the composition's TypeError; a NaN key that was not kept is never hashed there and
changes nothing.  When the merge flags a fold too long to stage, the composition stands.
"""
import itertools
import random

import numpy as np
import torch

from . import _native as nv
from . import quantiles
from .rdd import ColumnarRDD, DeviceResultRDD, SampleRDD, UnionRDD, device_path_applies

SKEW_SEED = 12345         # RDD.sample's default seed, the one _skew_thresholds samples with
NAN_KEYS = "NaN keys are not supported (CPython hashes NaN by identity)"


def _number(x):
    return type(x) in (int, float)


def sample_applies(rdd, frac, withReplacement):
    """True when rdd.sample(frac, withReplacement) runs on the device: a numeric ColumnarRDD in a one-process job
    (rdd.device_path_applies), without replacement, with an int or float fraction."""
    return not withReplacement and _number(frac) and device_path_applies([rdd])


def thresholds_inputs(rdd, rate):
    """The ColumnarRDDs whose splits are rdd's, in order, when rdd._skew_thresholds(splits, rate) runs on the device:
    rdd is a numeric ColumnarRDD or a UnionRDD of them (what the cogroups sample), in a one-process job, and rate an int
    or float.  Otherwise None."""
    if type(rdd) is ColumnarRDD:
        inputs = [rdd]
    elif type(rdd) is UnionRDD and rdd.rdds and all(type(r) is ColumnarRDD for r in rdd.rdds):
        inputs = list(rdd.rdds)
    else:
        return None
    return inputs if _number(rate) and device_path_applies(inputs) else None


def mt_states(seed, n):
    """int32 [n, 624] (the words' bits): the MT19937 state of random.Random(seed + i) right after seeding, i < n --
    the very expression SampleRDD draws from, so a seed it refuses raises the same error here."""
    out = np.empty((n, nv.MT_N), dtype=np.uint32)
    for i in range(n):
        version, internal, _ = random.Random(seed + i).getstate()
        if version != 3 or len(internal) != nv.MT_N + 1 or internal[-1] != nv.MT_N:
            raise AssertionError("unexpected random.Random state (version %r, position %r)" % (version, internal[-1]))
        out[i] = internal[:nv.MT_N]
    return torch.from_numpy(out.view(np.int32))


def _frac_arg(frac):
    """frac as the double the kernel compares with: an int is clamped to [-1, 2], which keeps every compare with a draw
    in [0, 1) as Python makes it and keeps huge ints from overflowing."""
    return float(min(max(frac, -1), 2)) if type(frac) is int else float(frac)


def bernoulli(ranges, nrows, frac, seed):
    """The kept row ids of the row ranges [(begin, end)] (split i drawn from random.Random(seed + i)): (ids, counts) --
    int64 device ids, split after split in row order, and the per-split counts as a list."""
    from .engine import _device
    states = mt_states(seed, len(ranges))
    dev = _device()
    states = states.to(dev)
    rng = torch.tensor(ranges, dtype=torch.int64).view(len(ranges), 2).to(dev)
    ids, counts = nv.sample_bernoulli(states, rng, _frac_arg(frac), nrows)
    counts = counts.cpu().tolist()
    return torch.cat([ids[:0]] + [ids[b:b + c] for (b, _), c in zip(ranges, counts)]), counts


def _refold_first(digests):
    """The first segment's digest d replaced by MergingDigest().absorb(d), as the composition's chain takes it after an
    empty first split."""
    cm, cw, cnt, lohi = digests
    c = int(cnt[0])
    if c == 0:                     # not built (the flag is raised): the merge stops there
        return
    d = quantiles.MergingDigest()
    d.means, d.weights = cm[:c].tolist(), cw[:c].tolist()
    d.merged_weight = sum(d.weights)
    e = quantiles.MergingDigest().absorb(d)
    m = len(e.means)
    cm[:m] = torch.tensor(e.means, dtype=torch.float64)
    cw[:m] = torch.tensor(e.weights, dtype=torch.float64)
    cnt[0] = m
    lohi[:2] = torch.tensor([e.lo, e.hi], dtype=torch.float64)


def skew_thresholds(inputs, splits, rate):
    """RDD._skew_thresholds(splits, rate) of the union of the ColumnarRDDs `inputs`: (thresholds, effective number of
    splits) as quantiles.skew_thresholds gives them over the composition's sample, or None when the composition must
    stand.  Raises the composition's TypeError for a NaN key among the kept rows."""
    from .engine import _device
    dev = _device()
    floats = any(r.keys.dtype.is_floating_point for r in inputs)
    hashes, nans, ranges, start = [], [], [], 0
    for r in inputs:
        k = r.keys.to(dev)
        k = k.to(torch.float64) + 0.0 if k.dtype.is_floating_point else k.to(torch.int64)
        if floats:
            nans.append(torch.isnan(k) if k.dtype.is_floating_point else torch.zeros_like(k, dtype=torch.bool))
        hashes.append(nv.hash_keys(k.contiguous()))
        ranges += [(start + s.begin, start + s.end) for s in r.splits]
        start += int(k.numel())
    h = torch.cat(hashes)
    if rate >= 1.0:
        kept, counts = torch.arange(start, dtype=torch.int64, device=dev), [e - b for b, e in ranges]
    else:
        kept, counts = bernoulli(ranges, start, rate, SKEW_SEED)
    if floats and bool(torch.cat(nans)[kept].any()):
        raise TypeError(NAN_KEYS)
    qs = [m / 100. for m in quantiles.skew_marks(splits)]
    K = sum(counts)
    if K == 0 or not qs:
        return quantiles.thresholds_of([float("nan")] * len(qs), splits)
    lens = [c for c in counts if c]
    seg_starts = torch.tensor([0] + list(itertools.accumulate(lens)), dtype=torch.int64, device=dev)
    seg_off = torch.tensor([0] + list(itertools.accumulate(min(c, nv.TD_CAP) for c in lens)), dtype=torch.int64,
                           device=dev)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    digests = nv.tdigest_build(kept, h, seg_starts, seg_off, flag)
    if counts[0] == 0:
        _refold_first(digests)
    groups = torch.tensor([0, K], dtype=torch.int64, device=dev)
    out = nv.tdigest_merge(groups, seg_starts, seg_off, digests, torch.tensor(qs, dtype=torch.float64, device=dev),
                           flag)
    if int(flag.item()):
        return None
    return quantiles.thresholds_of(out.view(-1).cpu().tolist(), splits)


class ColumnarSampleRDD(DeviceResultRDD, SampleRDD):
    """rdd.sample(frac, False, seed) of a numeric ColumnarRDD in a one-process job: the parent's splits, no partitioner,
    and SampleRDD's rows, drawn on the GPU the first time a partition is asked for and kept.  columns(split) hands out
    the kept rows as CUDA tensors in the parent's dtypes and bits."""

    def _run(self):
        p = self.prev
        ids, counts = bernoulli([(s.begin, s.end) for s in p.splits], int(p.keys.numel()), self.frac, self.seed)
        keys, vals = nv.gather_columns(p.keys.to(ids.device).contiguous(), p.vals.to(ids.device).contiguous(), ids)
        return keys, vals, [0] + list(itertools.accumulate(counts))

    def _part(self, result, i):
        keys, vals, off = result
        return keys[off[i]:off[i + 1]], vals[off[i]:off[i + 1]]
