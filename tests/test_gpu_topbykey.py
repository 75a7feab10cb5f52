"""The device topByKey of numeric ColumnarRDDs (dpark_b200/topk.py): against the reference's golden cases, against the
row path (the same rows through ctx.parallelize, which runs groupByKey and Python's sorted), and at scale against a
numpy oracle (np.lexsort by key, order key and position, cut per key)."""
import json

import numpy as np
import pytest
import torch

from tests import cogroup_common as cc
from tests.golden_util import dec, load

pytestmark = pytest.mark.gpu

DTYPES = [torch.int32, torch.int64, torch.float32, torch.float64]
T = 4096


def _topk_cls():
    from dpark_b200.topk import ColumnarTopByKeyRDD
    return ColumnarTopByKeyRDD


@pytest.fixture
def topk_spy(monkeypatch):
    """Counts the device group-bys and selection rounds; the host lists of the device groupByKey must not be built."""
    from dpark_b200 import _native as nv
    from dpark_b200 import engine, grouping
    calls = {"group": 0, "lengths": 0, "round": 0}

    def counted(name, real):
        def run(*args, **kw):
            calls[name] += 1
            return real(*args, **kw)
        return run

    def host_lists(*args):
        raise AssertionError("the device topByKey built the groupByKey's host lists")

    monkeypatch.setattr(grouping, "group_row_ids", counted("group", grouping.group_row_ids))
    monkeypatch.setattr(nv, "topk_lengths", counted("lengths", nv.topk_lengths))
    monkeypatch.setattr(nv, "topk_round", counted("round", nv.topk_round))
    monkeypatch.setattr(engine, "_run_group_columns", host_lists)
    return calls


# ------------------------------------------------------------------------------------------------ golden
TOPK = [c for c in load("topbykey_cases.json")["cases"] if c["order"] == "none"]


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=str)
@pytest.mark.parametrize("case", TOPK, ids=[c["name"] for c in TOPK])
def test_golden_top_by_key_cases_on_the_device(case, dtype, topk_spy):
    from tests.golden.make_golden import enc
    dc = cc.ctx()
    rows = [(dec(k), dec(v)) for k, v in case["rows"]]
    col = dc.parallelizeColumns(torch.tensor([k for k, _ in rows], dtype=dtype),
                                torch.tensor([v for _, v in rows], dtype=dtype), case["M"])
    out = col.topByKey(case["top_n"], reverse=case["reverse"], num_splits=case["P"])
    assert isinstance(out, _topk_cls())
    got = [sorted(([enc(k), enc(list(v))] for k, v in part), key=json.dumps) for part in out.glom().collect()]
    assert got == case["parts"]
    assert topk_spy["group"] == 1 and topk_spy["round"] == 1


# ------------------------------------------------------------------------------------------------ identity
def _cast(a, dtype):
    return torch.from_numpy(np.asarray(a)).to(dtype)


def _column(dc, rng, shape, kdt, vdt):
    """(ColumnarRDD, P, fixSkew) of one shape; values with many ties (and -0.0 among float values)."""
    P, skew, M = 5, -1, 4
    if shape == "uniform":
        k = rng.integers(0, 300, 2000)
    elif shape == "zipf":        # a few hot keys, one of them spanning several chunks of a round
        k = np.concatenate([np.minimum(rng.zipf(1.3, 3000), 500), np.full(2 * T + 700, 3)])
        k = k[rng.permutation(len(k))]
        P, M = 4, 3
    elif shape == "partial_overlap":       # split i holds keys [30 i, 30 i + 60)
        k = np.concatenate([rng.integers(30 * i, 30 * i + 60, 150) for i in range(M)])
    elif shape == "fix_skew":
        k, skew = rng.integers(0, 80, 1500), 1
    else:
        k = np.zeros(0, np.int64)
    if kdt.is_floating_point:
        k = k * 0.5
        k[rng.random(len(k)) < 0.05] = -0.0
    v = rng.integers(-20, 20, len(k)).astype(np.float64)
    if vdt.is_floating_point:
        v = v * 0.5
        v[rng.random(len(v)) < 0.1] = -0.0
        v[rng.random(len(v)) < 0.02] = float("inf")
    return dc.parallelizeColumns(_cast(k, kdt), _cast(v, vdt), M), P, skew


@pytest.mark.parametrize("kdt", DTYPES, ids=str)
@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("top_n", [1, 2, 7, 512])
@pytest.mark.parametrize("shape", ["uniform", "zipf", "partial_overlap", "fix_skew", "empty"])
def test_device_top_by_key_equals_the_row_path(shape, top_n, reverse, kdt):
    i = DTYPES.index(kdt)
    rng = np.random.default_rng(100 * i + top_n + reverse)
    dc = cc.ctx()
    for vdt in (DTYPES[i], DTYPES[(i + 1 + top_n) % 4]):
        col, P, skew = _column(dc, rng, shape, kdt, vdt)
        out = col.topByKey(top_n, reverse=reverse, num_splits=P, fixSkew=skew)
        assert isinstance(out, _topk_cls())
        rows = dc.parallelize(col.collect(), len(col.splits))
        want = rows.topByKey(top_n, reverse=reverse, num_splits=P, fixSkew=skew)
        assert out.partitioner == want.partitioner
        got, want = out.glom().collect(), want.glom().collect()
        assert len(got) == len(want) == out.partitioner.numPartitions      # P, or fewer when fixSkew merges splits
        assert got == want and repr(got) == repr(want)      # -0.0 values keep their sign, keys are spelled 0.0
        assert any(len(p) for p in got) == (shape != "empty")


# ------------------------------------------------------------------------------------------------ scale
def _order_key(v, reverse):
    """numpy sort key of a value column: the value (-0.0 sorts as 0.0), negated (ints: complemented) for reverse."""
    if not reverse:
        return v
    return -v if v.dtype.kind == "f" else ~v


def _oracle_top(k, v, top_n, reverse):
    """{key: its top values} from np.lexsort by (key, order key, position)."""
    order = np.lexsort((np.arange(len(k)), _order_key(v, reverse), k))
    ks, vs = k[order], v[order]
    heads = np.flatnonzero(np.concatenate([[True], ks[1:] != ks[:-1]]))
    ends = np.concatenate([heads[1:], [len(ks)]])
    return {int(ks[h]): vs[h:min(e, h + top_n)] for h, e in zip(heads, ends)}


def _check_against_the_oracle(k, v, M, P, top_n, reverse):
    from oracle import oracle as orc
    dc = cc.ctx()
    col = dc.parallelizeColumns(torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(), M)
    out = col.topByKey(top_n, reverse=reverse, num_splits=P)
    assert isinstance(out, _topk_cls())
    want = _oracle_top(k, v, top_n, reverse)
    bounds = [(sp.begin, sp.end) for sp in col.splits]
    layout = orc.group_by_key([k[b:e] for b, e in bounds], [np.arange(b, e, dtype=np.int64) for b, e in bounds], P)
    seen = 0
    for p, sp in enumerate(out.splits):
        keys, offsets, values = out.columns(sp)
        keys, off, vals = keys.cpu().numpy(), offsets.cpu().numpy(), values.cpu().numpy()
        assert np.array_equal(np.sort(keys), np.sort(layout[p][0])), p    # the partition's keys (their order: the
                                                                          # row-path tests)
        for j, key in enumerate(keys.tolist()):
            got, exp = vals[off[j]:off[j + 1]], want[key]
            assert got.dtype == exp.dtype and np.array_equal(got.view(np.uint8), exp.view(np.uint8)), (p, key)
        seen += len(keys)
    assert seen == len(want)


@pytest.mark.parametrize("reverse", [False, True])
def test_ten_million_zipf_rows_with_a_hot_key_match_the_oracle(reverse, topk_spy):
    """1e7 int64 rows with Zipf(1.1) keys plus one key of 3e6 values: the hot key takes three rounds."""
    rng = np.random.default_rng(21 + reverse)
    k = np.concatenate([np.minimum(rng.zipf(1.1, 7_000_000), 1 << 40), np.full(3_000_000, -5)]).astype(np.int64)
    perm = rng.permutation(len(k))
    k = k[perm]
    v = rng.integers(-10 ** 6, 10 ** 6, len(k)).astype(np.int64)
    _check_against_the_oracle(k, v, 8, 16, 10, reverse)
    assert topk_spy["round"] == 3


@pytest.mark.parametrize("vdt", [np.float32, np.float64])
@pytest.mark.parametrize("reverse", [False, True])
def test_signed_zero_ties_keep_their_bits(vdt, reverse):
    """Float values from {-0.0, 0.0, -1, 1, 2}: -0.0 and 0.0 tie and keep their input order and their sign bit."""
    rng = np.random.default_rng(5 + reverse)
    n = 400_000
    k = rng.integers(0, 40, n).astype(np.int64)
    k[rng.random(n) < 0.3] = 7                        # one key of ~1.2e5 values: two rounds
    v = rng.choice(np.array([-0.0, 0.0, -1.0, 1.0, 2.0], vdt), n, p=[0.3, 0.3, 0.1, 0.1, 0.2])
    for top_n in (1, 10, 512):
        _check_against_the_oracle(k, v, 5, 7, top_n, reverse)


@pytest.mark.parametrize("top_n", [1, 10, 512])
def test_runs_at_chunk_boundaries_with_dense_ties(top_n):
    """Keys of T, T + 1, 2T - 1 and 2T + 1 values (and their neighbours) in one column, values from {0, 1, 2}: ties
    straddle every chunk cut, and chunks of different keys share CTAs."""
    rng = np.random.default_rng(top_n)
    lens = [T, T + 1, 2 * T - 1, 2 * T + 1, T - 1, 1, 3 * T, 513, 2]
    k = np.repeat(np.arange(len(lens), dtype=np.int64) * 7 + 1, lens)
    for order in ("sorted", "shuffled"):
        kk = k if order == "sorted" else k[rng.permutation(len(k))]
        v = rng.integers(0, 3, len(kk)).astype(np.int32)
        for reverse in (False, True):
            _check_against_the_oracle(kk, v, 3, 3, top_n, reverse)


# ------------------------------------------------------------------------------------------------ NaN, spies, columns
def test_nan_values_give_the_composition_s_rows(monkeypatch):
    from dpark_b200 import _native as nv

    def no_round(*a):
        raise AssertionError("a selection round ran over NaN values")

    monkeypatch.setattr(nv, "topk_round", no_round)
    monkeypatch.setattr(nv, "topk_lengths", no_round)
    dc = cc.ctx()
    nan = float("nan")
    k = np.array([1, 2, 1, 1, 2, 3, 1], np.int64)
    v = np.array([3.0, nan, 1.0, nan, -0.0, 2.0, 0.0], np.float32)
    for reverse in (False, True):
        col = dc.parallelizeColumns(k, v, 3)
        out = col.topByKey(2, reverse=reverse, num_splits=2)
        assert isinstance(out, _topk_cls())
        want = dc.parallelize(col.collect(), 3).topByKey(2, reverse=reverse, num_splits=2).glom().collect()
        got = out.glom().collect()
        assert repr(got) == repr(want)
        for sp, part in zip(out.splits, got):
            keys, offsets, values = out.columns(sp)
            assert keys.is_cuda and values.dtype == torch.float32 and offsets.shape == (len(part) + 1,)
            assert keys.tolist() == [key for key, _ in part]
            assert repr(values.tolist()) == repr([x for _, xs in part for x in xs])


def test_the_device_path_runs_the_group_by_and_the_selection(topk_spy):
    dc = cc.ctx()
    col = dc.parallelizeColumns(np.array([5, 1, 5, 5, -0.0, 0.0]), np.array([4, 9, 2, 7, 1, 3], np.int32), 2)
    out = col.topByKey(2, reverse=True, num_splits=1)
    assert repr(sorted(out.collect())) == repr([(0.0, [3, 1]), (1.0, [9]), (5.0, [7, 4])])
    out.collect()                                      # materialised once
    assert topk_spy == {"group": 1, "lengths": 1, "round": 1}


def test_columns_and_what_lies_on_top():
    from dpark_b200 import HashPartitioner
    dc = cc.ctx()
    a = dc.parallelizeColumns(np.array([1, 2, 2, 3, 2], np.int32), np.array([10, 20, 21, 30, 19], np.float64), 2)
    out = a.topByKey(2, num_splits=3)
    total = 0
    for sp in out.splits:
        keys, offsets, values = out.columns(sp)
        assert all(t.is_cuda for t in (keys, offsets, values))
        assert (keys.dtype, offsets.dtype, values.dtype) == (torch.int64, torch.int64, torch.float64)
        assert offsets.shape == (keys.numel() + 1,) and int(offsets[0]) == 0 and int(offsets[-1]) == values.numel()
        total += keys.numel()
    assert total == 3
    assert sorted(out.collect()) == [(1, [10.0]), (2, [19.0, 20.0]), (3, [30.0])]
    rows = dc.parallelize(a.collect(), 2)
    mapped = out.mapValue(len)
    assert mapped.partitioner == HashPartitioner(3)
    b = dc.parallelizeColumns(np.array([2, 4], np.int64), np.array([5, 6], np.int64), 1)
    rb = dc.parallelize(b.collect(), 1)
    got = mapped.groupWith(b).glom().collect()
    want = rows.topByKey(2, num_splits=3).mapValue(len).groupWith(rb).glom().collect()
    assert got == want and repr(got) == repr(want)
