"""Approximate quantiles of a stream: the merging t-digest behind `RDD.percentiles` and
`combineByKey(fixSkew=...)`.

The reference balances skewed shuffles by cutting the HASH space at approximate percentiles of the
keys' hashes (dpark/rdd.py:514-540): one digest per input partition (dpark/rdd.py:791-814), merged
in partition order, queried at i*100/splits percent; the ceil()-ed answers become
`HashPartitioner(thresholds=...)`.  Which partition a key lands in therefore depends on every
floating-point step of the digest, so this module restates dpark/utils/tdigest.py operation for
operation (same buffer size, same scale test `z*z <= q(1-q)` on both ends, same incremental mean
update, same interpolation in `quantile`) -- tests/test_quantiles.py holds vectors captured from
the reference's class (tests/golden/make_tdigest_golden.py) and demands equality to the last bit.

This is host-side control-path code (a few hundred centroids per partition); the rows themselves
are hashed on the device (dpk_hash_keys / dpk_hash_bytes).
"""
import math


class MergingDigest(object):
    """Centroids (mean, weight) sorted by mean + a buffer of not yet merged points."""

    def __init__(self, compression=100, size=None):
        self.compression = compression
        self.capacity = int(2 * math.ceil(compression)) + 10 if size is None else size   # tdigest.py:41-44
        self.means, self.weights = [], []          # merged centroids, ascending means
        self.merged_weight = 0                     # total weight of the merged centroids
        self.buf_means, self.buf_weights = [], []  # points added since the last compress()
        self.buf_weight = 0
        self.lo = self.hi = None                   # smallest / largest centroid mean ever seen at a merge

    def __len__(self):
        return int(self.merged_weight + self.buf_weight)

    # ------------------------------------------------------------------ building
    def add(self, x, w=1):
        x, w = float(x), float(w)
        if math.isnan(x):
            raise ValueError("Cannot add NaN")
        if len(self.buf_weights) + len(self.weights) >= self.capacity - 1:        # tdigest.py:82-83
            self.compress()
        self.buf_means.append(x)
        self.buf_weights.append(w)
        self.buf_weight += w

    def update(self, values):
        for x in values:
            self.add(x)
        return self

    def compress(self):
        if self.buf_weight > 0:
            self._fold(self.buf_means, self.buf_weights)
            self.buf_means, self.buf_weights, self.buf_weight = [], [], 0

    def absorb(self, other):
        """self += other (dpark/utils/tdigest.py:55-74): other's centroids enter as buffered points."""
        if not isinstance(other, MergingDigest):
            raise TypeError("Can not add MergingDigest with %s" % type(other).__name__)
        if len(other) == 0:
            return self
        other.compress()
        self.buf_means.extend(other.means)
        self.buf_weights.extend(other.weights)
        self.buf_weight = sum(other.weights)       # assigned, not accumulated -- as the reference does
        self.compress()
        return self

    __add__ = absorb

    def _fold(self, in_means, in_weights):
        """One merge pass (tdigest.py:96-137): incoming points first, then the old centroids, stably
        sorted by mean; neighbours are fused while the fused weight stays under the scale bound at
        BOTH ends of the quantile range it would cover."""
        ms = in_means + self.means
        ws = in_weights + self.weights
        order = sorted(range(len(ms)), key=ms.__getitem__)
        self.merged_weight += self.buf_weight
        total = self.merged_weight
        norm = self.compression / (math.pi * total)
        first = order[0]
        out_m, out_w = [ms[first]], [ws[first]]
        done = 0.
        for i in order[1:]:
            fused = out_w[-1] + ws[i]
            z = fused * norm
            q_lo = done / total
            q_hi = (done + fused) / total
            if z * z <= q_lo * (1 - q_lo) and z * z <= q_hi * (1 - q_hi):
                out_w[-1] += ws[i]
                out_m[-1] = out_m[-1] + (ms[i] - out_m[-1]) * ws[i] / out_w[-1]
            else:
                done += out_w[-1]
                out_m.append(ms[i])
                out_w.append(ws[i])
        self.means, self.weights = out_m, out_w
        if total > 0:
            self.lo = out_m[0] if self.lo is None else min(self.lo, out_m[0])
            self.hi = out_m[-1] if self.hi is None else max(self.hi, out_m[-1])

    # ------------------------------------------------------------------ queries
    @staticmethod
    def _between(x1, w1, x2, w2):
        lo, hi = min(x1, x2), max(x1, x2)
        return max(lo, min(hi, float(x1 * w1 + x2 * w2) / (w1 + w2)))

    def quantile(self, q):
        q = float(q)
        if not 0 <= q <= 1:
            raise ValueError("q should be in [0, 1], got %s" % q)
        self.compress()
        ws, ms = self.weights, self.means
        if not ws:
            return float("nan")
        if len(ws) == 1:
            return ms[0]
        target = q * self.merged_weight
        if target < ws[0] / 2:
            return self.lo + 2. * target / ws[0] * (ms[0] - self.lo)
        seen = ws[0] / 2.
        for i in range(len(ws) - 1):
            span = (ws[i] + ws[i + 1]) / 2.
            if seen + span > target:
                left = target - seen
                right = seen + span - target
                return self._between(ms[i], right, ms[i + 1], left)
            seen += span
        # beyond the centre of the last centroid (tdigest.py:168-173, including its sign convention)
        left = target - self.merged_weight - ws[-1] / 2.
        right = ws[-1] / 2. - left
        return self._between(ms[-1], left, self.hi, right)


def percentiles_of_partitions(partitions, percents, compression=100):
    """`RDD.percentiles` (dpark/rdd.py:791-814) over already materialised partitions: one digest per
    partition, merged left to right, then queried.  `partitions`: iterable of iterables of numbers."""
    merged = None
    for part in partitions:
        d = MergingDigest(compression).update(part)
        d.compress()
        merged = d if merged is None else merged.absorb(d)
    if merged is None:
        return [float("nan") for _ in percents]
    merged.compress()
    return [merged.quantile(p / 100.) for p in percents]


def skew_marks(splits):
    """The percentiles `combineByKey(fixSkew=...)` queries (dpark/rdd.py:516-537): i*100/splits for 0 < i < splits."""
    step = 100. / splits
    return [step * i for i in range(1, splits)]


def thresholds_of(pcts, splits):
    """The thresholds from the percentiles at skew_marks(splits): NaNs dropped, ceil()-ed, strictly increasing.
    Returns (thresholds or None, effective number of splits)."""
    if not pcts:
        return None, splits
    thr = []
    for p in pcts:
        if math.isnan(p):
            continue
        p = int(math.ceil(p))
        if not thr or p > thr[-1]:
            thr.append(p)
    return thr, len(thr) + 1


def skew_thresholds(hash_partitions, splits):
    """The thresholds `combineByKey(fixSkew=...)` derives (dpark/rdd.py:516-537): percentiles of the
    key hashes at i*100/splits, NaNs dropped, ceil()-ed, strictly increasing.  Returns
    (thresholds or None, effective number of splits)."""
    return thresholds_of(percentiles_of_partitions(hash_partitions, skew_marks(splits)), splits)
