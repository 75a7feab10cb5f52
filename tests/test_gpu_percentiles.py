"""The device percentilesByKey of numeric ColumnarRDDs (dpark_b200/percentiles.py): against the reference's golden cases,
against the row path (the same rows through ctx.parallelize, which runs the split-tagged groupByKey and
quantiles.MergingDigest), bit for bit, and at scale against the CPU harness tests/tdigestcheck.cu segment by segment."""
import numpy as np
import pytest
import torch

from tests import cogroup_common as cc
from tests.golden_util import load
from tests.test_percentiles_host import harness_run, tdigestcheck

pytestmark = pytest.mark.gpu

DTYPES = [torch.int32, torch.int64, torch.float32, torch.float64]
PS = [[], [0, 100], [10, 50, 90, 99]]


def _cls():
    from dpark_b200.percentiles import ColumnarPercentilesByKeyRDD
    return ColumnarPercentilesByKeyRDD


def _spy(m):
    """Counts the device group-bys; the groupByKey's host lists, MergingDigest and the composition must not be used."""
    from dpark_b200 import engine, grouping, quantiles
    from dpark_b200.rdd import RDD
    calls = {"group": 0}
    real = grouping.group_row_ids

    def group(*a, **kw):
        calls["group"] += 1
        return real(*a, **kw)

    def refuse(*a, **kw):
        raise AssertionError("the device percentilesByKey left the device")

    m.setattr(grouping, "group_row_ids", group)
    m.setattr(engine, "_run_group_columns", refuse)
    m.setattr(quantiles.MergingDigest, "__init__", refuse)
    m.setattr(RDD, "_percentiles_rows", refuse)
    return calls


@pytest.fixture
def device_only(monkeypatch):
    return _spy(monkeypatch)


def _hexparts(parts):
    return [sorted([k, [q.hex() for q in qs]] for k, qs in part) for part in parts]


# ------------------------------------------------------------------------------------------------ golden
MISC = load("misc_cases.json")


@pytest.mark.parametrize("kdt", [torch.int32, torch.int64], ids=str)
def test_golden_one_map(kdt, device_only):
    c = MISC["percentilesByKey_one_map"]
    dc = cc.ctx()
    col = dc.parallelizeColumns(torch.tensor([k for k, _ in c["rows"]], dtype=kdt),
                                torch.tensor([float.fromhex(v) for _, v in c["rows"]], dtype=torch.float64), c["M"])
    out = col.percentilesByKey(c["p"], numSplits=c["P"])
    assert isinstance(out, _cls())
    assert _hexparts(out.glom().collect()) == c["parts"]
    assert device_only["group"] == 1


@pytest.mark.parametrize("kdt", [torch.int32, torch.int64], ids=str)
def test_golden_four_maps_layout_and_composition(kdt):
    c = MISC["percentilesByKey_four_maps"]
    dc = cc.ctx()
    rows = [(k, float.fromhex(v)) for k, v in c["rows"]]
    col = dc.parallelizeColumns(torch.tensor([k for k, _ in rows], dtype=kdt),
                                torch.tensor([v for _, v in rows], dtype=torch.float64), c["M"])
    got = col.percentilesByKey(c["p"], numSplits=c["P"]).glom().collect()
    assert [sorted(k for k, _ in part) for part in got] == [[k for k, _ in part] for part in c["parts"]]
    want = dc.parallelize(col.collect(), c["M"]).percentilesByKey(c["p"], numSplits=c["P"]).glom().collect()
    assert repr(got) == repr(want) and _hexparts(got) == _hexparts(want)


# ------------------------------------------------------------------------------------------------ identity
def _cast(a, dtype):
    return torch.from_numpy(np.asarray(a)).to(dtype)


def _column(dc, rng, shape, kdt, vdt):
    """(ColumnarRDD, P, fixSkew) of one shape; values with ties, -0.0 and (float) subnormals."""
    P, skew, M = 5, -1, 4
    if shape == "uniform":
        k = rng.integers(0, 300, 4000)
    elif shape == "zipf":        # a hot key of 3e4 values over every split: many compresses and absorbs
        k = np.concatenate([np.minimum(rng.zipf(1.3, 6000), 500), np.full(30000, 3)])
        k = k[rng.permutation(len(k))]
        P, M = 4, 7
    elif shape == "partial_overlap":       # split i holds keys [30 i, 30 i + 60)
        k = np.concatenate([rng.integers(30 * i, 30 * i + 60, 400) for i in range(M)])
    elif shape == "fix_skew":
        k, skew = rng.integers(0, 80, 3000), 1
    else:
        k = np.zeros(0, np.int64)
    if kdt.is_floating_point:
        k = k * 0.5
        k[rng.random(len(k)) < 0.05] = -0.0
    if vdt.is_floating_point:
        v = rng.normal(0, 100, len(k))
        v[rng.random(len(v)) < 0.1] = -0.0
        v[rng.random(len(v)) < 0.1] = 0.0
        v[rng.random(len(v)) < 0.02] = 1e-310 if vdt == torch.float64 else 1e-40
    else:
        v = rng.integers(-20, 20, len(k))
    return dc.parallelizeColumns(_cast(k, kdt), _cast(v, vdt), M), P, skew


@pytest.mark.parametrize("kdt", DTYPES, ids=str)
@pytest.mark.parametrize("shape", ["uniform", "zipf", "partial_overlap", "fix_skew", "empty"])
def test_device_percentiles_equal_the_row_path(shape, kdt):
    i = DTYPES.index(kdt)
    rng = np.random.default_rng(10 * i + len(shape))
    dc = cc.ctx()
    for vdt in (DTYPES[i], DTYPES[(i + 1) % 4]):
        col, P, skew = _column(dc, rng, shape, kdt, vdt)
        rows = dc.parallelize(col.collect(), len(col.splits))
        for p in PS:
            out = col.percentilesByKey(p, numSplits=P, fixSkew=skew)
            assert isinstance(out, _cls())
            want = rows.percentilesByKey(p, numSplits=P, fixSkew=skew)
            assert out.partitioner == want.partitioner
            got, want = out.glom().collect(), want.glom().collect()
            assert len(got) == len(want) == out.partitioner.numPartitions
            assert repr(got) == repr(want)
            assert _hexparts(got) == _hexparts(want)
            assert any(len(part) for part in got) == (shape != "empty")


# ------------------------------------------------------------------------------------------------ edges
def _both(dc, k, v, M, p, P=3):
    col = dc.parallelizeColumns(k, v, M)
    out = col.percentilesByKey(p, numSplits=P)
    assert isinstance(out, _cls())
    want = dc.parallelize(col.collect(), M).percentilesByKey(p, numSplits=P)
    return out, want


def test_nan_value_raises_the_composition_s_error():
    dc = cc.ctx()
    k = np.array([1, 2, 1, 1, 2], np.int64)
    v = np.array([3.0, float("nan"), 1.0, 2.0, 0.0])
    out, want = _both(dc, k, v, 2, [50])
    with pytest.raises(ValueError, match="Cannot add NaN"):
        want.collect()
    with pytest.raises(ValueError, match="Cannot add NaN"):
        out.collect()


def test_both_infinities_under_one_key_give_the_composition_s_rows():
    dc = cc.ctx()
    k = np.array([1] * 400 + [2] * 10, np.int64)
    v = np.concatenate([np.full(100, -np.inf), np.full(100, np.inf), np.linspace(0, 1, 200), np.arange(10.)])
    out, want = _both(dc, k, v, 1, [0, 10, 50, 90, 100])
    assert repr(out.glom().collect()) == repr(want.glom().collect())
    assert out._result is not None and not isinstance(out._result, list)       # the composition stood


EDGES = ["plus_inf", "minus_inf", "signed_zeros", "int64_beyond_2_53"]


def _edge(case):
    rng = np.random.default_rng(4)
    n = 5000
    k = rng.integers(0, 6, n).astype(np.int64)
    if case == "signed_zeros":
        return k, rng.choice(np.array([-0.0, 0.0, 1.0, -1.0]), n)
    if case == "int64_beyond_2_53":
        return k, (np.int64(2 ** 62) + rng.integers(-2 ** 20, 2 ** 20, n)).astype(np.int64)
    v = rng.normal(0, 1, n)
    v[rng.random(n) < 0.0005] = np.inf if case == "plus_inf" else -np.inf
    return k, v


@pytest.mark.parametrize("case", EDGES)
def test_edges_stay_on_the_device_and_are_bit_identical(case, monkeypatch):
    """+inf or -inf on one side only, -0.0 / 0.0 ties, int64 values past 2^53 (rounded as float() rounds them)."""
    dc = cc.ctx()
    k, v = _edge(case)
    col = dc.parallelizeColumns(k, v, 3)
    p = [0, 1, 25, 50, 75, 99, 100]
    want = dc.parallelize(col.collect(), 3).percentilesByKey(p, numSplits=2).glom().collect()
    with monkeypatch.context() as m:
        calls = _spy(m)
        got = col.percentilesByKey(p, numSplits=2).glom().collect()
    assert calls["group"] == 1
    assert repr(got) == repr(want) and _hexparts(got) == _hexparts(want)


def test_percent_out_of_range_raises():
    dc = cc.ctx()
    col = dc.parallelizeColumns(np.array([1, 2, 1], np.int64), np.array([1.0, 2.0, 3.0]), 2)
    for p in ([101], [50, -1]):
        with pytest.raises(ValueError, match="q should be in"):
            col.percentilesByKey(p).collect()
    assert col.filter(lambda kv: False).percentilesByKey([101]).collect() == []


# ------------------------------------------------------------------------------------------------ scale
def test_ten_million_zipf_rows_match_the_harness():
    """1e7 float64 values under Zipf(1.1) keys over 16 splits: every segment digest and every key's quantiles equal the
    CPU harness's, bit for bit."""
    from dpark_b200 import _native as nv
    from dpark_b200 import percentiles
    L = tdigestcheck()
    rng = np.random.default_rng(31)
    n = 10_000_000
    k = np.minimum(rng.zipf(1.1, n), 1 << 40).astype(np.int64)
    v = rng.normal(0, 1e3, n)
    dc = cc.ctx()
    col = dc.parallelizeColumns(torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(), 16)
    qs = [pp / 100. for pp in (0, 0.1, 1, 10, 50, 90, 99, 99.9, 100)]
    (gk, gs, ov, _), ss, so, digests, flag = percentiles.segment_digests(col, 8, None)
    out = nv.tdigest_merge(gs, ss, so, digests, torch.tensor(qs, dtype=torch.float64, device="cuda"), flag)
    assert int(flag.item()) == 0
    cm, cw, cnt, lohi = (t.cpu().numpy() for t in digests)
    ss_h, so_h, ov_h, gs_h = ss.cpu().numpy(), so.cpu().numpy(), ov.cpu().numpy(), gs.cpu().numpy()
    split = ov_h // -(-n // 16)
    heads = np.flatnonzero(np.concatenate([[True], split[1:] != split[:-1]]) | np.isin(np.arange(n), gs_h[:-1]))
    assert np.array_equal(ss_h[:-1], heads)
    hflag, segs, hquant = harness_run(L, ov_h, v, ss_h, gs_h, qs)
    assert hflag == 0
    assert np.array_equal(cnt, np.array([len(m) for m, _, _, _ in segs], np.int32))
    assert (np.diff(ss_h) > 32).sum() > 100 and len(segs) > 10 ** 5
    for s, (m, w, lo, hi) in enumerate(segs):
        a, b = so_h[s], so_h[s] + cnt[s]
        assert cm[a:b].tobytes() == m.tobytes() and cw[a:b].tobytes() == w.tobytes(), s
        assert lohi[2 * s:2 * s + 2].tobytes() == np.array([lo, hi]).tobytes(), s
    assert out.cpu().numpy().tobytes() == hquant.tobytes()


# ------------------------------------------------------------------------------------------------ spies, columns
def test_the_device_path_runs_one_group_by(device_only):
    dc = cc.ctx()
    col = dc.parallelizeColumns(np.array([5, 1, 5, 5, -0.0, 0.0]), np.array([4, 9, 2, 7, 1, 3], np.int32), 2)
    out = col.percentilesByKey([0, 50, 100], numSplits=1)
    assert sorted(out.collect()) == [(0.0, [1.0, 2.0, 3.0]), (1.0, [9.0, 9.0, 9.0]), (5.0, [2.0, 4.0, 7.0])]
    out.collect()
    assert device_only["group"] == 1


def test_columns_and_what_lies_on_top():
    from dpark_b200 import HashPartitioner
    dc = cc.ctx()
    a = dc.parallelizeColumns(np.array([1, 2, 2, 3, 2], np.int32), np.array([10, 20, 21, 30, 19], np.float32), 2)
    out = a.percentilesByKey([25, 75], numSplits=3)
    total = 0
    for sp in out.splits:
        keys, quant = out.columns(sp)
        assert keys.is_cuda and quant.is_cuda and keys.dtype == torch.int64 and quant.dtype == torch.float64
        assert quant.shape == (keys.numel(), 2)
        total += keys.numel()
    assert total == 3
    assert out.mapValue(len).partitioner == HashPartitioner(3)
    rows = dc.parallelize(a.collect(), 2)
    got = out.mapValue(sum).groupWith(a).glom().collect()
    want = rows.percentilesByKey([25, 75], numSplits=3).mapValue(sum).groupWith(rows).glom().collect()
    assert repr(got) == repr(want)
