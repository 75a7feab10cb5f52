"""ColumnarRDDs with uneven, empty and no splits on a CPU: what the columnar operators decide before any launch.

textFileColumns gives every result explicit split bounds (ColumnarRDD(bounds=...)): a split owns the lines that start in
its byte range, so splits are uneven, a split can own no line at all, and an empty file gives no split.  Checked here:
  - sort of a ColumnarRDD with no split, and with one: the device class, with the composition's partition count
    (RDD._sort_rows returns an input without splits as it is: no partition);
  - the range bounds sorting.sample_bounds reads from column slices, against the bounds of the composition's own samples
    (the first numSplits * 10 // len(rdd) rows of every split, read through compute), over layouts with empty splits;
  - sampling.thresholds_inputs over unions that hold inputs without splits.
The device results over the same layouts are checked in tests/test_gpu_split_layouts.py."""
import itertools

import pytest
import torch

from tests import cogroup_common as cc

LAYOUTS = {
    "zero": [0],
    "one_empty": [0, 0],
    "one": [0, 40],
    "leading_empty": [0, 0, 0, 40],
    "trailing_empty": [0, 40, 40, 40],
    "middle_empty": [0, 13, 13, 13, 29, 40],
    "singletons": list(range(0, 9)),
    "ragged": [0, 1, 30, 30, 33, 33, 40],
    "mostly_empty": [0, 0, 0, 0, 0, 17, 17, 17, 17, 40],
}


def _columns(dc, bounds, kdt=torch.int64, vdt=torch.float64, seed=0):
    from dpark_b200.rdd import ColumnarRDD
    n = bounds[-1]
    g = torch.Generator().manual_seed(seed + n)
    k = torch.randint(-20, 20, (n,), generator=g).to(kdt)
    v = torch.randint(-50, 50, (n,), generator=g).to(vdt)
    return ColumnarRDD(dc, k, v, 1, bounds=bounds)


def _sorted_cls():
    from dpark_b200.sorting import ColumnarSortedRDD
    return ColumnarSortedRDD


SORT_KEYS = {"id": lambda x: x, "first": lambda x: x[0], "second": lambda x: x[1]}


@pytest.mark.parametrize("key", sorted(SORT_KEYS))
@pytest.mark.parametrize("numSplits", [None, 4])
@pytest.mark.parametrize("reverse", [False, True])
def test_sort_of_no_split_has_no_partition(key, numSplits, reverse):
    dc = cc.ctx()
    e = _columns(dc, [0])
    assert len(e.splits) == 0
    got = e.sort(SORT_KEYS[key], reverse=reverse, numSplits=numSplits)
    assert type(got) is _sorted_cls()
    want = e._sort_rows(SORT_KEYS[key], reverse, numSplits, None, None)
    assert len(got) == len(want) == 0
    assert got.bounds == []
    assert got.glom().collect() == want.glom().collect() == []


@pytest.mark.parametrize("bounds", [[0, 0], [0, 40]], ids=["one_empty", "one"])
@pytest.mark.parametrize("numSplits", [None, 4])
def test_sort_of_one_split_has_one_partition(bounds, numSplits):
    dc = cc.ctx()
    rdd = _columns(dc, bounds)
    got = rdd.sort(numSplits=numSplits)
    assert type(got) is _sorted_cls()
    assert got.bounds == [] and len(got) == 1
    assert len(rdd._sort_rows(lambda x: x, False, numSplits, None, None)) == 1


def _composition_bounds(rdd, key, reverse, numSplits):
    """RDD._sort_rows' range bounds, from samples read through compute."""
    from dpark_b200.rdd import range_bounds
    if numSplits is None:
        numSplits = min(rdd.ctx.defaultMinSplits, len(rdd))
    n = max(numSplits * 10 // len(rdd), 1)
    samples = rdd.mapPartitions(lambda it: itertools.islice(it, n)).map(key).collect()
    return range_bounds(samples, numSplits, reverse)


@pytest.mark.parametrize("layout", [name for name, b in sorted(LAYOUTS.items()) if len(b) > 2])
@pytest.mark.parametrize("kdt, vdt", [(torch.int64, torch.float64), (torch.float32, torch.int32)], ids=["i64f64", "f32i32"])
def test_sample_bounds_over_empty_splits(layout, kdt, vdt):
    from dpark_b200 import sorting
    dc = cc.ctx()
    for n in (40, 200):                # 200 rows: every split holds more than numSplits * 10 // len(rdd) rows
        bounds = [b * n // 40 for b in LAYOUTS[layout]]
        rdd = _columns(dc, bounds, kdt, vdt, seed=n)
        for (name, key), reverse, numSplits in itertools.product(sorted(SORT_KEYS.items()), (False, True),
                                                                  (None, 2, 4, 7)):
            want = _composition_bounds(rdd, key, reverse, numSplits)
            got = sorting.sample_bounds(rdd, key, reverse, numSplits)
            assert got == want, (layout, n, name, reverse, numSplits)
            dev = rdd.sort(key, reverse=reverse, numSplits=numSplits)
            assert type(dev) is _sorted_cls() and dev.bounds == want
            assert len(dev) == len(rdd._sort_rows(key, reverse, numSplits, None, None)) == len(want) + 1


def test_sample_bounds_differ_when_only_non_empty_splits_are_counted():
    """The layouts above are ones where the sample length counts every split: dividing by the non-empty splits only
    reads more rows per split and moves the bounds."""
    from dpark_b200.rdd import range_bounds
    dc = cc.ctx()
    rdd = _columns(dc, [b * 5 for b in LAYOUTS["mostly_empty"]], seed=200)
    full = [sp for sp in rdd.splits if sp.end > sp.begin]
    n_all, n_full = max(4 * 10 // len(rdd), 1), max(4 * 10 // len(full), 1)
    assert n_all != n_full

    def bounds_of(n):
        rows = list(zip(rdd.keys.tolist(), rdd.vals.tolist()))
        return range_bounds([r for sp in rdd.splits for r in rows[sp.begin:min(sp.end, sp.begin + n)]], 4, False)
    assert bounds_of(n_all) != bounds_of(n_full)
    assert _composition_bounds(rdd, lambda x: x, False, 4) == bounds_of(n_all)


@pytest.mark.parametrize("rate", [0.3, 1, 1.0])
def test_thresholds_inputs_over_unions_with_no_split_inputs(rate):
    from dpark_b200 import sampling
    dc = cc.ctx()
    zero, one_empty = _columns(dc, [0]), _columns(dc, [0, 0])
    ragged = _columns(dc, LAYOUTS["ragged"], seed=1)
    lead = _columns(dc, LAYOUTS["leading_empty"], seed=2)
    assert sampling.thresholds_inputs(zero, rate) == [zero]
    for rdds in ([zero], [zero, zero], [zero, ragged], [ragged, zero], [one_empty, zero, lead], [zero, lead, zero],
                 [zero, one_empty, ragged, zero]):
        u = rdds[0].union(*rdds[1:])
        got = sampling.thresholds_inputs(u, rate)
        assert got is not None and len(got) == len(rdds) and all(a is b for a, b in zip(got, rdds))
        # the inputs' splits, one after the other, are the union's splits
        assert [(r, s) for r in got for s in r.splits] == [(sp.rdd, sp.split) for sp in u.splits]
        assert len(u) == sum(len(r) for r in got)
    mixed = zero.union(dc.parallelize([(1, 2.0)], 1))
    assert sampling.thresholds_inputs(mixed, rate) is None
    assert sampling.thresholds_inputs(zero, "0.3") is None
