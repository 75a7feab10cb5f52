"""The device percentilesByKey on a CPU: the digest arithmetic of dpk_common.cuh run through tests/tdigestcheck.cu, step
for step as dpk_tdigest.cu takes it (segment digests, the absorb chain, the quantiles), against quantiles.MergingDigest
and the reference's vectors, compared through float.hex; which calls take the device path, and the partitioner it shares
with the composition.  The device results themselves are checked in tests/test_gpu_percentiles.py."""
import ctypes as C
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from dpark_b200.quantiles import MergingDigest
from tests import cogroup_common as cc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = {np.dtype(np.int64): 0, np.dtype(np.int32): 1, np.dtype(np.float64): 2, np.dtype(np.float32): 4}
PERCENTS = [0, 0.1, 1, 5, 10, 25, 33.3, 50, 66.6, 75, 90, 95, 99, 99.9, 100]


def tdigestcheck():
    path = os.path.join(ROOT, "tests", "_tdigestcheck.so")
    if not os.path.exists(path):
        subprocess.call([sys.executable, "-c", "import __graft_entry__ as g; g.build()"], cwd=ROOT)
    if not os.path.exists(path):
        pytest.skip("tdigestcheck not built")
    L = C.CDLL(path)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    L.tdc_cap.restype = L.tdc_short.restype = i32
    L.tdc_build.restype = i32
    L.tdc_build.argtypes = [vp, vp, i32, vp, vp, i64, vp, vp, vp, vp]
    L.tdc_merge.restype = i32
    L.tdc_merge.argtypes = [vp, i64, vp, vp, i64, vp, vp, vp, vp, vp, i32, vp]
    L.tdc_fold_serial.restype = i32
    L.tdc_fold_serial.argtypes = [vp, vp, i32, C.c_double, vp, vp, vp]
    L.tdc_quantile.restype = C.c_double
    L.tdc_quantile.argtypes = [vp, vp, i32, C.c_double, C.c_double, C.c_double, C.c_double]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def harness_run(L, ids, vals, seg_starts, group_starts, qs):
    """tdc_build + tdc_merge over numpy arrays: (flag, per-segment [(means, weights, lo, hi)], quantiles [G, nq])."""
    ids, vals = np.ascontiguousarray(ids, np.int64), np.ascontiguousarray(vals)
    ss, gs = np.asarray(seg_starts, np.int64), np.asarray(group_starts, np.int64)
    S, G = len(ss) - 1, len(gs) - 1
    so = np.concatenate([[0], np.cumsum(np.minimum(np.diff(ss), L.tdc_cap()))]).astype(np.int64)
    cm, cw = np.zeros(max(1, len(ids))), np.zeros(max(1, len(ids)))
    cnt, lohi = np.zeros(max(1, S), np.int32), np.zeros(max(2, 2 * S))
    flag = L.tdc_build(_p(ids), _p(vals), KINDS[vals.dtype], _p(ss), _p(so), S, _p(cm), _p(cw), _p(cnt), _p(lohi))
    q = np.asarray(qs, np.float64)
    out = np.zeros(max(1, G * len(q)))
    if not flag:
        flag = L.tdc_merge(_p(gs), G, _p(ss), _p(so), S, _p(cnt), _p(lohi), _p(cm), _p(cw), _p(q), len(q), _p(out))
    segs = [(cm[so[s]:so[s] + cnt[s]], cw[so[s]:so[s] + cnt[s]], lohi[2 * s], lohi[2 * s + 1]) for s in range(S)]
    return flag, segs, out[:G * len(q)].reshape(G, len(q))


def run_keys(L, keys, dtype=np.float64, percents=PERCENTS):
    """keys: per key its list of non-empty segments (lists of numbers); one row per value in that order."""
    flat, ss, gs = [], [0], [0]
    for segs in keys:
        for seg in segs:
            flat.extend(seg)
            ss.append(len(flat))
        gs.append(len(flat))
    vals = np.array(flat, dtype=dtype)
    return harness_run(L, np.arange(len(flat)), vals, ss, gs, [pp / 100. for pp in percents])


def py_segment(values):
    d = MergingDigest().update(values)
    d.compress()
    return d


def py_key(segs, percents=PERCENTS):
    """RDD._percentiles_rows' quantiles_of over one key's segments."""
    merged = None
    for seg in segs:
        d = py_segment(seg)
        merged = d if merged is None else merged.absorb(d)
        merged.compress()
    return [merged.quantile(pp / 100.) for pp in percents]


def _hex(xs):
    return [float(x).hex() for x in xs]


def check_keys(L, keys, dtype=np.float64, percents=PERCENTS):
    flag, segs, quant = run_keys(L, keys, dtype, percents)
    assert flag == 0
    conv = (lambda x: float(np.float32(x))) if dtype == np.float32 else (lambda x: x)
    s = 0
    for j, key in enumerate(keys):
        key = [[conv(x) for x in seg] for seg in key]
        for seg in key:
            d = py_segment(seg)
            m, w, lo, hi = segs[s]
            assert _hex(m) == _hex(d.means) and _hex(w) == _hex(d.weights), (j, s, len(seg))
            assert (float(lo).hex(), float(hi).hex()) == (float(d.lo).hex(), float(d.hi).hex()), (j, s)
            s += 1
        assert _hex(quant[j]) == _hex(py_key(key, percents)), j


# ------------------------------------------------------------------------------------------------ harness parity
def test_constants():
    L = tdigestcheck()
    assert L.tdc_cap() == MergingDigest().capacity - 1 == 209
    assert L.tdc_short() <= L.tdc_cap()
    from dpark_b200 import _native as nv
    assert nv.TD_CAP == 209


with open(os.path.join(ROOT, "tests", "golden", "tdigest_vectors.json")) as f:
    GOLD = json.load(f)["cases"]


@pytest.mark.parametrize("case", GOLD, ids=[c["name"] for c in GOLD])
def test_golden_vectors(case):
    """Every case as one key whose splits are the case's parts (an empty split has no segment).  Where the first part
    is not empty the composition's merge is the reference's, and the quantiles are the captured ones."""
    L = tdigestcheck()
    segs = [p for p in case["parts"] if p]
    check_keys(L, [segs], percents=case["percents"])
    if case["parts"][0]:
        _, _, quant = run_keys(L, [segs], percents=case["percents"])
        assert _hex(quant[0]) == case["quantiles"]


def _values(kind, n, rng):
    if kind == "uniform":
        return [rng.random() for _ in range(n)]
    if kind == "normal":
        return [rng.gauss(0, 100) for _ in range(n)]
    if kind == "sorted":
        return sorted(rng.random() for _ in range(n))
    if kind == "reverse":
        return sorted((rng.random() for _ in range(n)), reverse=True)
    if kind == "ties":
        return [float(rng.randrange(3)) for _ in range(n)]
    if kind == "zeros":
        return [rng.choice([-0.0, 0.0, 1.0, -1.0]) for _ in range(n)]
    if kind == "subnormal":
        return [rng.choice([5e-324, -5e-324, 1e-310, -1e-310, 0.0, -0.0]) * rng.randrange(1, 4) for _ in range(n)]
    if kind == "exp":
        return [rng.expovariate(1) for _ in range(n)]
    raise ValueError(kind)


LENGTHS = [1, 2, 31, 32, 33, 208, 209, 210, 211, 418, 1000, 100000]
SHAPES = ["uniform", "normal", "sorted", "reverse", "ties", "zeros", "subnormal", "exp"]


@pytest.mark.parametrize("shape", SHAPES)
def test_segment_lengths_one_split(shape):
    """One key, one segment, of every edge length: the short (one thread) and long (buffered) builds."""
    L = tdigestcheck()
    rng = random.Random(SHAPES.index(shape))
    check_keys(L, [[_values(shape, n, rng)] for n in LENGTHS])


@pytest.mark.parametrize("shape", SHAPES)
def test_absorb_chains(shape):
    """Keys of many segments of mixed lengths: the absorb chain in split order."""
    L = tdigestcheck()
    rng = random.Random(7 + len(shape))
    keys = [[_values(shape, rng.choice(LENGTHS[:-1]), rng) for _ in range(rng.randrange(1, 12))] for _ in range(6)]
    keys.append([_values(shape, 3000, rng) for _ in range(8)])
    check_keys(L, keys)


@pytest.mark.parametrize("dtype", [np.float32, np.int32, np.int64], ids=str)
def test_value_dtypes(dtype):
    L = tdigestcheck()
    rng = random.Random(3)
    if dtype == np.float32:
        keys = [[[rng.gauss(0, 1e3) for _ in range(n)] for n in (5, 300, 40)]]
    elif dtype == np.int32:
        keys = [[[rng.randrange(-2 ** 31, 2 ** 31) for _ in range(n)] for n in (5, 300, 40)]]
    else:       # above 2^53: float() rounds to nearest, ties to even
        big = [2 ** 53 + 1, 2 ** 53 + 3, 2 ** 62 + 1, -(2 ** 63), 2 ** 63 - 1, 2 ** 60 + 2 ** 7 + 1]
        clamp = lambda x: min(max(x, -2 ** 63), 2 ** 63 - 1)
        keys = [[[clamp(rng.choice(big) + rng.randrange(-3, 4)) for _ in range(n)] for n in (5, 300, 40)], [big]]
    flag, segs, quant = run_keys(L, keys, dtype)
    assert flag == 0
    conv = [[[float(x) for x in seg] for seg in key] for key in keys]
    if dtype == np.float32:
        conv = [[[float(np.float32(x)) for x in seg] for seg in key] for key in keys]
    for j, key in enumerate(conv):
        assert _hex(quant[j]) == _hex(py_key(key)), j


def test_infinities_on_one_side_and_flags():
    L = tdigestcheck()
    inf = float("inf")
    check_keys(L, [[[1.0, 2.0, inf]], [[-inf, 0.0, 5.0]], [[inf], [3.0, 4.0]], [[-inf] + [0.5] * 40]])
    # +inf and -inf under one key: a NaN mean, the composition stands
    flag, _, _ = run_keys(L, [[[-inf] * 50 + [inf] * 50 + [1.0] * 300]])
    assert flag == 1
    flag, _, _ = run_keys(L, [[[float("nan"), 1.0]]])          # a NaN value
    assert flag == 1
    flag, _, _ = run_keys(L, [[[1.0] * 40 + [float("nan")]]])
    assert flag == 1


def test_fold_and_quantile_entry_points():
    """tdc_fold_serial is one _fold; tdc_quantile is quantile() of the digest it leaves."""
    L = tdigestcheck()
    rng = random.Random(11)
    for n in (1, 2, 50, 209):
        xs = sorted(rng.gauss(0, 1) for _ in range(n))
        ws = [float(rng.randrange(1, 5)) for _ in range(n)]
        d = MergingDigest()
        d.buf_weight = sum(ws)
        d._fold(xs, ws)
        xm, xw = np.array(xs), np.array(ws)
        om, ow, bad = np.zeros(n), np.zeros(n), np.zeros(1, np.int32)
        c = L.tdc_fold_serial(_p(xm), _p(xw), n, sum(ws), _p(om), _p(ow), _p(bad))
        assert bad[0] == 0 and _hex(om[:c]) == _hex(d.means) and _hex(ow[:c]) == _hex(d.weights)
        for q in (0.0, 0.01, 0.5, 0.99, 1.0):
            got = L.tdc_quantile(_p(om), _p(ow), c, d.merged_weight, d.lo, d.hi, q)
            assert float(got).hex() == float(d.quantile(q)).hex()


# ------------------------------------------------------------------------------------------------ path choice
ELIGIBLE = [torch.int32, torch.int64, torch.float32, torch.float64]
INELIGIBLE = [torch.int16, torch.uint8, torch.bool, torch.float16]


def _col(dc, kdt, vdt, n=6, M=2):
    return dc.parallelizeColumns(torch.arange(n).to(kdt), torch.arange(n).to(vdt), M)


def _cls():
    from dpark_b200.percentiles import ColumnarPercentilesByKeyRDD
    return ColumnarPercentilesByKeyRDD


@pytest.mark.parametrize("kdt", ELIGIBLE + INELIGIBLE, ids=str)
@pytest.mark.parametrize("vdt", ELIGIBLE + INELIGIBLE, ids=str)
def test_device_path_is_chosen_by_dtypes(kdt, vdt):
    from dpark_b200 import HashPartitioner
    from dpark_b200.rdd import MappedValuesRDD
    dc = cc.ctx()
    eligible = kdt in ELIGIBLE and vdt in ELIGIBLE
    out = _col(dc, kdt, vdt).percentilesByKey([50], numSplits=4)
    assert isinstance(out, _cls()) == eligible
    assert isinstance(out, MappedValuesRDD) != eligible
    assert out.partitioner == HashPartitioner(4) and len(out.splits) == 4


def test_func_sample_rate_and_input_type_choose_the_path(monkeypatch):
    from dpark_b200 import spmd
    from dpark_b200.rdd import ColumnarRDD, MappedValuesRDD
    dc = cc.ctx()
    col = _col(dc, torch.int64, torch.float64)

    class MyColumns(ColumnarRDD):
        pass

    assert isinstance(col.percentilesByKey([50]), _cls())
    assert isinstance(col.percentilesByKey([50], sampleRate=1.5), _cls())
    assert isinstance(col.percentilesByKey([50], func=lambda v: v), MappedValuesRDD)
    assert isinstance(col.percentilesByKey([50], sampleRate=0.5), MappedValuesRDD)
    for other in (dc.parallelize([(1, 2.0)], 1), col.map(lambda kv: kv), col.mapValue(lambda v: v),
                  MyColumns(dc, np.arange(4), np.arange(4), 2), col.union(col)):
        assert isinstance(other.percentilesByKey([50]), MappedValuesRDD)
    for bad in (0, -1):
        with pytest.raises(ValueError):
            col.percentilesByKey([50], sampleRate=bad)
    monkeypatch.setattr(spmd, "rank_world", lambda: (0, 2))
    assert isinstance(col.percentilesByKey([50]), MappedValuesRDD)


def test_nothing_is_computed_at_construction(monkeypatch):
    from dpark_b200 import engine, percentiles

    def no_device(*a):
        raise AssertionError("the percentilesByKey ran at construction")

    monkeypatch.setattr(engine, "_device", no_device)
    monkeypatch.setattr(percentiles, "percentiles_columns", no_device)
    dc = cc.ctx()
    out = _col(dc, torch.int64, torch.float64).percentilesByKey([10, 90], numSplits=4)
    out.mapValue(len)
    assert out._result is None


def test_partitioner_is_the_composition_s(monkeypatch):
    """The composition groups the split-tagged rows, which have self's keys, row counts and splits: the same partitioner,
    fixSkew's sample is taken over an RDD of the same length (the thresholds themselves: tests/test_gpu_percentiles.py)."""
    from dpark_b200 import HashPartitioner
    from dpark_b200.rdd import RDD, CoGroupedRDD
    dc = cc.ctx()
    a = dc.parallelizeColumns(torch.arange(40) % 7, torch.arange(40).double(), 3)
    rows = dc.parallelize(a.collect(), 3)
    for splits in (None, 1, 5):
        assert a.percentilesByKey([50], numSplits=splits).partitioner == \
            rows.percentilesByKey([50], numSplits=splits).partitioner
    part = HashPartitioner(6, thresholds=[1, 2, 3, 4, 5])
    assert a.percentilesByKey([50], numSplits=part).partitioner is part
    calls = []

    def fake_thresholds(self, splits, rate):
        calls.append((len(self), splits, rate))
        return [10 * i for i in range(1, splits - 1)], splits - 1

    monkeypatch.setattr(RDD, "_skew_thresholds", fake_thresholds)
    want = HashPartitioner(3, thresholds=[10, 20])
    assert a.percentilesByKey([50], numSplits=4, fixSkew=0.5).partitioner == want
    assert rows.percentilesByKey([50], numSplits=4, fixSkew=0.5).partitioner == want
    assert calls == [(3, 4, 0.5)] * 2
    out = a.percentilesByKey([50], numSplits=6)
    assert out.mapValue(len).partitioner == HashPartitioner(6)
    again = out.groupWith(a)
    assert type(again) is CoGroupedRDD and again.narrow == [0]


def test_other_partitioners_are_refused_as_by_the_composition():
    from dpark_b200.dependency import RangePartitioner
    dc = cc.ctx()
    col = _col(dc, torch.int64, torch.int64)
    for bad in (RangePartitioner([3]), "4"):
        with pytest.raises((TypeError, NotImplementedError)) as e_dev:
            col.percentilesByKey([50], numSplits=bad).collect()
        with pytest.raises((TypeError, NotImplementedError)) as e_rows:
            col.percentilesByKey([50], func=lambda v: v, numSplits=bad).collect()
        assert type(e_dev.value) is type(e_rows.value)

