"""The device sort of numeric ColumnarRDDs (dpark_b200/sorting.py): against the composition over the same splits (forced
with col.map(lambda x: x), which is not a ColumnarRDD), against the reference's golden layouts, and at scale against a
numpy oracle (a stable argsort on the order keys, cut at the same bounds by np.searchsorted, or for the (k, v) order by
counting the rows that sort before each bound)."""
import numpy as np
import pytest
import torch

from tests import cogroup_common as cc
from tests.test_sort_host import COLSORT, golden_case

pytestmark = pytest.mark.gpu

DTYPES = [torch.int32, torch.int64, torch.float32, torch.float64]
BITS = {torch.int32: torch.int32, torch.int64: torch.int64, torch.float32: torch.int32, torch.float64: torch.int64}
KEYS = {"id": lambda x: x, "first": lambda x: x[0], "second": lambda x: x[1]}


def _sorted_cls():
    from dpark_b200.sorting import ColumnarSortedRDD
    return ColumnarSortedRDD


@pytest.fixture
def sort_spy(monkeypatch):
    """Counts the sort kernels; the input must not be read through ColumnarRDD.compute and no group-by host lists may
    be built."""
    from dpark_b200 import _native as nv
    from dpark_b200 import engine
    from dpark_b200.rdd import ColumnarRDD
    calls = {"keys": 0, "cuts": 0, "gather": 0}

    def counted(name, real):
        def run(*args, **kw):
            calls[name] += 1
            return real(*args, **kw)
        return run

    def forbidden(*args, **kw):
        raise AssertionError("the device sort read its input row by row or built group-by host lists")

    monkeypatch.setattr(nv, "sort_keys", counted("keys", nv.sort_keys))
    monkeypatch.setattr(nv, "sort_cuts", counted("cuts", nv.sort_cuts))
    monkeypatch.setattr(nv, "sort_gather", counted("gather", nv.sort_gather))
    monkeypatch.setattr(ColumnarRDD, "compute", forbidden)
    monkeypatch.setattr(engine, "_run_group_columns", forbidden)
    return calls


def _check_equal(out, want, kdt, vdt):
    """Same partitions, same rows in the same order, floats compared bit for bit (so -0.0 is checked)."""
    got_parts, want_parts = out.glom().collect(), want.glom().collect()
    assert [len(p) for p in got_parts] == [len(p) for p in want_parts]
    assert got_parts == want_parts and repr(got_parts) == repr(want_parts)
    for sp, part in zip(out.splits, want_parts):
        keys, vals = out.columns(sp)
        assert keys.is_cuda and vals.is_cuda and (keys.dtype, vals.dtype) == (kdt, vdt)
        wk = torch.tensor([k for k, _ in part], dtype=kdt)
        wv = torch.tensor([v for _, v in part], dtype=vdt)
        assert torch.equal(keys.cpu().view(BITS[kdt]), wk.view(BITS[kdt]))
        assert torch.equal(vals.cpu().view(BITS[vdt]), wv.view(BITS[vdt]))


def _columns(rng, kdt, vdt, n):
    """Columns with many ties and both signed zeros among the floats."""
    k = rng.integers(-30, 30, n).astype(np.float64)
    v = rng.integers(-4, 4, n).astype(np.float64)
    for a, dt in ((k, kdt), (v, vdt)):
        if dt.is_floating_point:
            a *= 0.5
            a[rng.random(n) < 0.1] = -0.0
            a[rng.random(n) < 0.02] = float("inf")
            a[rng.random(n) < 0.02] = -float("inf")
    return torch.from_numpy(k).to(kdt), torch.from_numpy(v).to(vdt)


# ------------------------------------------------------------------------------------------------ the composition
@pytest.mark.parametrize("key", ["id", "first", "second"])
@pytest.mark.parametrize("vdt", DTYPES, ids=str)
@pytest.mark.parametrize("kdt", DTYPES, ids=str)
def test_device_sort_equals_the_composition(kdt, vdt, key):
    rng = np.random.default_rng(DTYPES.index(kdt) * 4 + DTYPES.index(vdt))
    dc = cc.ctx()
    k, v = _columns(rng, kdt, vdt, 700)
    col = dc.parallelizeColumns(k.cuda(), v.cuda(), 5)
    for reverse in (False, True):
        out = col.sort(key=KEYS[key], reverse=reverse, numSplits=4)
        assert isinstance(out, _sorted_cls())
        want = col.map(lambda x: x).sort(key=KEYS[key], reverse=reverse, numSplits=4)
        assert not isinstance(want, _sorted_cls())
        _check_equal(out, want, kdt, vdt)


@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("key", ["first", "id"])
def test_heavy_ties_keep_split_and_position_order(key, reverse, sort_spy):
    """4 distinct keys over 16 splits; the value is the row's position, so equal keys must keep ascending values."""
    rng = np.random.default_rng(11 + reverse)
    dc = cc.ctx()
    n = 4000
    k = torch.from_numpy(rng.integers(0, 4, n)).cuda()
    v = torch.arange(n, device="cuda")
    col = dc.parallelizeColumns(k, v, 16)
    out = col.sort(key=KEYS[key], reverse=reverse, numSplits=16)
    rows = out.collect()
    assert [x[0] for x in rows] == sorted(k.tolist(), reverse=reverse)
    for a, b in zip(rows, rows[1:]):
        if a[0] == b[0]:
            assert (a[1] < b[1]) != (key == "id" and reverse)
    out.collect()                                      # materialised once
    assert sort_spy == {"keys": 1, "cuts": 1, "gather": 1}


# ------------------------------------------------------------------------------------------------ golden
@pytest.mark.parametrize("case", COLSORT["cases"], ids=[c["name"] for c in COLSORT["cases"]])
def test_golden_layouts_of_the_reference(case, sort_spy):
    """The reference's partitions: keys in the same positions, the same rows per partition (their order among equal
    keys follows the reference's fetch order)."""
    dc = cc.ctx()
    pairs, want, kdt, vdt = golden_case(case)
    col = dc.parallelizeColumns(torch.tensor([k for k, _ in pairs], dtype=kdt).cuda(),
                                torch.tensor([v for _, v in pairs], dtype=vdt).cuda(), case["M"])
    key = KEYS[case["key"]]
    got = col.sort(key=key, reverse=case["reverse"], numSplits=case["P"]).glom().collect()
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert [key(x) for x in g] == [key(x) for x in w]
        assert sorted(map(repr, g)) == sorted(map(repr, w))
    assert sort_spy["keys"] == 1


# ------------------------------------------------------------------------------------------------ NaN
@pytest.mark.parametrize("key", ["id", "first", "second"])
def test_nan_in_an_order_column_gives_the_composition_s_rows(key):
    from dpark_b200.rdd import RDD
    dc = cc.ctx()
    nan = float("nan")
    k = torch.tensor([3.0, nan, 1.0, -0.0, 0.0, 2.0, nan, 1.0], dtype=torch.float32)
    v = torch.tensor([1.5, 2.0, nan, 0.5, -0.0, 0.0, 1.0, 3.0], dtype=torch.float64)
    col = dc.parallelizeColumns(k.cuda(), v.cuda(), 3)
    for reverse in (False, True):
        out = col.sort(key=KEYS[key], reverse=reverse, numSplits=2)
        assert isinstance(out, _sorted_cls())
        want = col.map(lambda x: x).sort(key=KEYS[key], reverse=reverse, numSplits=2).glom().collect()
        got = out.glom().collect()
        assert repr(got) == repr(want)
        assert isinstance(out._materialize(), RDD)          # the composition's rows stand
        for sp, part in zip(out.splits, got):
            keys, vals = out.columns(sp)
            assert keys.is_cuda and (keys.dtype, vals.dtype) == (torch.float32, torch.float64)
            assert repr(keys.tolist()) == repr([a for a, _ in part]) and repr(vals.tolist()) == repr([b for _, b in part])


def test_nan_in_the_other_column_stays_on_the_device(sort_spy):
    dc = cc.ctx()
    nan = float("nan")
    k = torch.tensor([3, 1, 2, 1, 0, 5], dtype=torch.int64)
    v = torch.tensor([nan, 1.0, -0.0, nan, 2.0, 0.0], dtype=torch.float32)
    col = dc.parallelizeColumns(k.cuda(), v.cuda(), 2)
    out = col.sort(key=lambda x: x[0], numSplits=2)
    rows = out.collect()
    assert [a for a, _ in rows] == [0, 1, 1, 2, 3, 5]
    assert repr([b for _, b in rows]) == repr([2.0, 1.0, nan, -0.0, nan, 0.0])
    assert sort_spy == {"keys": 1, "cuts": 1, "gather": 1}


# ------------------------------------------------------------------------------------------------ scale
def _order_key(a, reverse):
    if not reverse:
        return a
    return -a if a.dtype.kind == "f" else ~a


def _check_oracle(out, order, starts, k, v):
    assert len(out.splits) == len(starts) - 1
    for p, sp in enumerate(out.splits):
        keys, vals = out.columns(sp)
        sel = order[starts[p]:starts[p + 1]]
        assert np.array_equal(keys.cpu().numpy().view(np.uint8), k[sel].view(np.uint8)), p
        assert np.array_equal(vals.cpu().numpy().view(np.uint8), v[sel].view(np.uint8)), p


@pytest.mark.parametrize("reverse", [False, True])
def test_twenty_million_rows_by_key_match_the_oracle(reverse, sort_spy):
    rng = np.random.default_rng(17 + reverse)
    n, M = 20_000_000, 16
    k = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    k[rng.random(n) < 0.2] = 12345                                    # a fifth of the rows tie
    v = rng.integers(-(1 << 20), 1 << 20, n).astype(np.int32)
    dc = cc.ctx()
    col = dc.parallelizeColumns(torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(), M)
    out = col.sort(key=lambda x: x[0], reverse=reverse, numSplits=64)
    order = np.argsort(_order_key(k, reverse), kind="stable")
    ok = _order_key(k, reverse)[order]
    bounds = sorted(out.bounds)
    L = len(bounds)
    if reverse:
        starts = [int(np.searchsorted(ok, ~np.int64(bounds[L - j]), side="right")) for j in range(1, L + 1)]
    else:
        starts = [int(np.searchsorted(ok, np.int64(bounds[j - 1]), side="left")) for j in range(1, L + 1)]
    assert L == 63
    _check_oracle(out, order, [0] + starts + [n], k, v)
    assert sort_spy["keys"] == 1


@pytest.mark.parametrize("reverse", [False, True])
def test_twenty_million_rows_by_tuple_match_the_oracle(reverse, sort_spy):
    rng = np.random.default_rng(23 + reverse)
    n, M = 20_000_000, 12
    k = rng.integers(-1000, 1000, n).astype(np.int32)
    v = rng.integers(-50, 50, n).astype(np.float64) * 0.25
    v[rng.random(n) < 0.05] = -0.0
    dc = cc.ctx()
    col = dc.parallelizeColumns(torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(), M)
    out = col.sort(reverse=reverse, numSplits=32)
    order = np.lexsort((_order_key(v, reverse), _order_key(k, reverse)))     # stable: (k, v, position)
    bounds = sorted(out.bounds)
    L = len(bounds)
    starts = [0]
    for j in range(1, L + 1):
        bk, bv = bounds[L - j] if reverse else bounds[j - 1]
        if reverse:       # rows before the cut: key >= bound (getPartition = the number of bounds > key)
            starts.append(int(np.count_nonzero((k > bk) | ((k == bk) & (v >= bv)))))
        else:             # rows before the cut: key < bound
            starts.append(int(np.count_nonzero((k < bk) | ((k == bk) & (v < bv)))))
    _check_oracle(out, order, starts + [n], k, v)
    assert sort_spy["keys"] == 1
