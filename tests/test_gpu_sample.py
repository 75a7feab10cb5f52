"""The device sample and fixSkew thresholds of numeric ColumnarRDDs (dpark_b200/sampling.py): sample against SampleRDD
row for row and bit for bit, _skew_thresholds against the composition over the same rows (ctx.parallelize cuts a list
into the splits a ColumnarRDD of the same length has), end to end through every operator that takes fixSkew, and at
1e7 rows against numpy's MT19937 and quantiles.skew_thresholds."""
import random

import numpy as np
import pytest
import torch

from dpark_b200 import quantiles, sampling
from dpark_b200.rdd import ColumnarRDD, SampleRDD
from tests import cogroup_common as cc

pytestmark = pytest.mark.gpu

DTYPES = [torch.int32, torch.int64, torch.float32, torch.float64]
FRACS = [0, 1e-4, 0.3, 0.999, 1, 1.5, float("nan")]
SEEDS = [12345, 0, -7, 2 ** 40]
RATES = [1e-3, 0.05, 0.5, 1, 2]
PS = [2, 7, 64, 1000]


def _bits(t):
    t = t.cpu()
    return t.view(torch.int64 if t.element_size() == 8 else torch.int32).numpy()


def _column(rng, dtype, n, lo=-50, hi=50):
    x = rng.integers(lo, hi, n)
    if dtype.is_floating_point:
        x = x * 0.5
        if n:
            x[rng.random(n) < 0.1] = -0.0
            x[rng.random(n) < 0.05] = np.nan
    return torch.from_numpy(x).to(dtype)


def _want_masks(col, frac, seed):
    """SampleRDD's keep decisions per split, drawn with the stdlib generator."""
    out = []
    for s in col.splits:
        rd = random.Random(seed + s.index)
        out.append(np.array([rd.random() <= frac for _ in range(s.end - s.begin)], dtype=bool))
    return out


@pytest.mark.parametrize("vdt", DTYPES, ids=str)
@pytest.mark.parametrize("kdt", DTYPES, ids=str)
def test_sample_rows_and_bits_equal_sample_rdd(kdt, vdt):
    rng = np.random.default_rng(1)
    dc = cc.ctx()
    keys, vals = _column(rng, kdt, 2000), _column(rng, vdt, 2000)
    col = dc.parallelizeColumns(keys, vals, 5)
    for frac in FRACS:
        for seed in SEEDS:
            out = col.sample(frac, False, seed)
            assert isinstance(out, sampling.ColumnarSampleRDD) and out.partitioner is None
            assert out.splits is col.splits
            want = SampleRDD(col, frac, False, seed).glom().collect()
            got = out.glom().collect()
            assert repr(got) == repr(want), (frac, seed)
            for s, mask in zip(col.splits, _want_masks(col, frac, seed)):
                k, v = out.columns(s)
                assert k.is_cuda and k.dtype == kdt and v.dtype == vdt
                assert np.array_equal(_bits(k), _bits(keys[s.begin:s.end][torch.from_numpy(mask)]))
                assert np.array_equal(_bits(v), _bits(vals[s.begin:s.end][torch.from_numpy(mask)]))


@pytest.mark.parametrize("n, M", [(10, 8), (0, 4), (1, 3), (313, 1), (624, 2)])
def test_sample_of_trailing_empty_splits_and_no_rows(n, M):
    rng = np.random.default_rng(2)
    dc = cc.ctx()
    col = dc.parallelizeColumns(_column(rng, torch.int64, n), _column(rng, torch.float64, n), M)
    for frac in (0.5, 1):
        out = col.sample(frac)
        assert isinstance(out, sampling.ColumnarSampleRDD)
        assert repr(out.glom().collect()) == repr(SampleRDD(col, frac, False, 12345).glom().collect())


# ------------------------------------------------------------------------------------------------ thresholds
def _shape_keys(shape, rng, n):
    if shape == "uniform":
        return torch.from_numpy(rng.integers(-10 ** 6, 10 ** 6, n))
    if shape == "zipf":
        return torch.from_numpy(rng.zipf(1.2, n).astype(np.int64))
    if shape == "single":
        return torch.full((n,), 42, dtype=torch.int64)
    if shape == "equal_zeros":              # every key 0.0 or -0.0: one Python key
        return torch.from_numpy(np.where(rng.random(n) < 0.5, -0.0, 0.0))
    if shape == "wide":                     # |k| > 2^53, and -0.0 among float keys elsewhere
        return torch.from_numpy(rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64))
    if shape == "float32":
        k = (rng.standard_normal(n) * 1e4).astype(np.float32)
        k[::7] = -0.0
        return torch.from_numpy(k)
    raise AssertionError(shape)


def _rows_of(dc, col):
    rows = dc.parallelize(col.collect(), len(col.splits))
    assert [len(s.values) for s in rows.splits] == [s.end - s.begin for s in col.splits]
    return rows


@pytest.mark.parametrize("shape", ["uniform", "zipf", "single", "equal_zeros", "wide", "float32"])
def test_skew_thresholds_equal_the_composition(shape, monkeypatch):
    rng = np.random.default_rng(3)
    dc = cc.ctx()
    n = 6000
    keys = _shape_keys(shape, rng, n)
    col = dc.parallelizeColumns(keys, torch.arange(n), 8)
    rows = _rows_of(dc, col)
    for rate in RATES:
        for P in PS:
            want = rows._skew_thresholds(P, rate)
            assert col._skew_thresholds(P, rate) == want, (rate, P)


def _union_inputs(dc, rng, layout):
    out = []
    for n, M, dt in layout:
        out.append(dc.parallelizeColumns(_column(rng, dt, n, -10 ** 5, 10 ** 5) if n else torch.empty(0, dtype=dt),
                                         torch.arange(n, dtype=torch.int32), M))
    return out


UNIONS = {
    "two": [(3000, 4, torch.int64), (2000, 3, torch.int32)],
    "three_mixed_kinds": [(1500, 2, torch.int64), (1000, 3, torch.float64), (500, 2, torch.float32)],
    "empty_first_input": [(0, 3, torch.int64), (3000, 4, torch.int64)],
    "empty_first_of_three": [(0, 2, torch.float64), (2500, 3, torch.float64), (1000, 2, torch.int64)],
    "tiny_first_split": [(2, 2, torch.int64), (4000, 4, torch.int64), (700, 1, torch.int32)],
}


@pytest.mark.parametrize("name", sorted(UNIONS))
def test_union_thresholds_equal_the_composition(name):
    rng = np.random.default_rng(4)
    dc = cc.ctx()
    ins = _union_inputs(dc, rng, UNIONS[name])
    for a in ins:                         # NaN keys are tested below
        if a.keys.dtype.is_floating_point:
            a.keys[torch.isnan(a.keys)] = 1.5
    union = ins[0].union(*ins[1:])
    rows = _rows_of(dc, ins[0]).union(*[_rows_of(dc, a) for a in ins[1:]])
    assert sampling.thresholds_inputs(union, 0.05) is not None
    refolds = 0
    for rate in RATES:
        if rate < 1:
            first = union.splits[0]
            rd = random.Random(12345)
            refolds += not any(rd.random() <= rate for _ in range(first.split.end - first.split.begin))
        for P in PS:
            assert union._skew_thresholds(P, rate) == rows._skew_thresholds(P, rate), (rate, P)
    if name in ("empty_first_input", "empty_first_of_three", "tiny_first_split"):
        assert refolds >= 2                # the first split's sample is empty at the small rates


def test_everything_sampled_away_gives_one_split():
    dc = cc.ctx()
    col = dc.parallelizeColumns(torch.arange(5), torch.arange(5), 2)
    assert col._skew_thresholds(4, 1e-9) == ([], 1) == _rows_of(dc, col)._skew_thresholds(4, 1e-9)
    assert col.reduceByKey(lambda a, b: a + b, 4, fixSkew=1e-9).partitioner.numPartitions == 1


def test_nan_key_raises_only_when_kept():
    dc = cc.ctx()
    n, rate = 4000, 0.01
    keys = torch.arange(n, dtype=torch.float64)
    rd = random.Random(12345)
    draws = [rd.random() for _ in range(n // 2)]              # split 0 of 2
    kept = next(j for j, u in enumerate(draws) if u <= rate)
    dropped = next(j for j, u in enumerate(draws) if u > rate)
    k1 = keys.clone()
    k1[dropped] = float("nan")
    col = dc.parallelizeColumns(k1, torch.arange(n), 2)
    assert col._skew_thresholds(8, rate) == _rows_of(dc, col)._skew_thresholds(8, rate)
    k2 = keys.clone()
    k2[kept] = float("nan")
    col = dc.parallelizeColumns(k2, torch.arange(n), 2)
    with pytest.raises(TypeError) as e_dev:
        col._skew_thresholds(8, rate)
    with pytest.raises(TypeError) as e_rows:
        _rows_of(dc, col)._skew_thresholds(8, rate)
    assert str(e_dev.value) == str(e_rows.value)
    with pytest.raises(TypeError):
        col._skew_thresholds(8, 1)


# ------------------------------------------------------------------------------------------------ end to end
def _sorted_parts(parts):
    return [sorted(repr(x) for x in part) for part in parts]


def test_operators_with_fix_skew_partition_like_the_row_path():
    rng = np.random.default_rng(5)
    dc = cc.ctx()
    n = 5000
    a = dc.parallelizeColumns(torch.from_numpy(rng.zipf(1.3, n).astype(np.int64)),
                              torch.from_numpy(rng.integers(0, 100, n)), 4)
    b = dc.parallelizeColumns(torch.from_numpy(rng.zipf(1.3, n // 2).astype(np.int64)),
                              torch.from_numpy(rng.standard_normal(n // 2)), 3)
    ra, rb = _rows_of(dc, a), _rows_of(dc, b)
    ops = {
        "reduceByKey": lambda x, y: x.reduceByKey(lambda u, v: u + v, 6, fixSkew=0.05),
        "groupByKey": lambda x, y: x.groupByKey(6, fixSkew=0.05).mapValue(sorted),
        "join": lambda x, y: x.join(y, 6, fixSkew=0.05),
        "cogroup": lambda x, y: x.cogroup(y, 6, fixSkew=0.05),
        "topByKey": lambda x, y: x.topByKey(3, num_splits=6, fixSkew=0.05),
        "percentilesByKey": lambda x, y: x.percentilesByKey([10, 90], numSplits=6, fixSkew=0.05),
    }
    for name, op in ops.items():
        got, want = op(a, b), op(ra, rb)
        assert got.partitioner == want.partitioner, name
        assert _sorted_parts(got.glom().collect()) == _sorted_parts(want.glom().collect()), name
    part = a._combine_partitioner(6, 0.05)
    assert part == ra._combine_partitioner(6, 0.05) and part.thresholds
    part = a._cogroup_partitioner([b], 6, 0.05)          # join's, which its flatMap result does not carry
    assert part == ra._cogroup_partitioner([rb], 6, 0.05) and part.thresholds


def test_device_path_reads_no_rows_and_draws_nothing_in_python(monkeypatch):
    rng = np.random.default_rng(6)
    dc = cc.ctx()
    col = dc.parallelizeColumns(torch.from_numpy(rng.integers(0, 10 ** 6, 50000)), torch.arange(50000), 8)
    empty = dc.parallelizeColumns(torch.empty(0, dtype=torch.int64), torch.empty(0, dtype=torch.int64), 2)
    rows = _rows_of(dc, col)
    wants = {rate: rows._skew_thresholds(16, rate) for rate in (0.01, 1)}
    want_u = dc.parallelize([], 2).union(rows)._skew_thresholds(16, 0.01)
    adds = []
    orig_add = quantiles.MergingDigest.add

    def counting_add(self, x, w=1):
        adds.append(x)
        return orig_add(self, x, w)

    def refuse(*a, **k):
        raise AssertionError("row path taken")

    monkeypatch.setattr(ColumnarRDD, "compute", refuse)
    monkeypatch.setattr(random.Random, "random", refuse)
    monkeypatch.setattr(quantiles.MergingDigest, "add", counting_add)
    for rate, want in wants.items():
        assert col._skew_thresholds(16, rate) == want
    assert adds == []
    assert empty.union(col)._skew_thresholds(16, 0.01) == want_u      # the refold of the first non-empty digest
    assert len(adds) <= quantiles.MergingDigest().capacity - 1
    s = col.sample(0.2)
    assert sum(int(s.columns(sp)[0].numel()) for sp in s.splits) > 0


# ------------------------------------------------------------------------------------------------ scale
def test_ten_million_rows_against_numpy_mt19937():
    n, M, P, rate = 10 ** 7, 16, 64, 0.01
    rng = np.random.default_rng(7)
    keys = rng.integers(0, 2 ** 40, n)                # portable_hash(k) == k below 2^61 - 1
    dc = cc.ctx()
    col = dc.parallelizeColumns(torch.from_numpy(keys).cuda(), torch.arange(n, device="cuda"), M)
    parts, masks = [], []
    for s in col.splits:
        L = s.end - s.begin
        bg = np.random.MT19937()
        st = bg.state
        st["state"]["key"] = np.array(random.Random(12345 + s.index).getstate()[1][:624], dtype=np.uint32)
        st["state"]["pos"] = 624
        bg.state = st
        w = bg.random_raw(2 * L).astype(np.uint64)
        u = ((w[0::2] >> 5).astype(np.float64) * 67108864.0 + (w[1::2] >> 6).astype(np.float64)) * 2.0 ** -53
        mask = u <= rate
        masks.append(mask)
        parts.append(keys[s.begin:s.end][mask].tolist())
    sample = col.sample(rate)
    for s, mask in zip(col.splits, masks):
        assert np.array_equal(sample.columns(s)[0].cpu().numpy(), keys[s.begin:s.end][mask])
    assert col._skew_thresholds(P, rate) == quantiles.skew_thresholds(parts, P)
