"""The device sort on a CPU: which calls of RDD.sort take the device path (dpark_b200/sorting.py), the range-bounds rule
both paths share against the layouts captured from the reference, and the sort arithmetic of dpk_common.cuh run through
tests/sortcheck.cu (widening, order words, the two-word order and the partition cut) against Python's sorted and
bisect.  The device results themselves are checked in tests/test_gpu_sort.py."""
import ctypes as C
import operator
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import cogroup_common as cc
from tests.golden_util import dec, load

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KIND = {torch.int64: 0, torch.int32: 1, torch.float64: 2, torch.float32: 4}
DTYPES = [torch.int32, torch.int64, torch.float32, torch.float64]


def _sortcheck():
    path = os.path.join(ROOT, "tests", "_sortcheck.so")
    if not os.path.exists(path):
        subprocess.call([sys.executable, "-c", "import __graft_entry__ as g; g.build()"], cwd=ROOT)
    if not os.path.exists(path):
        pytest.skip("sortcheck not built")
    L = C.CDLL(path)
    u64, i64, i32, vp = C.c_uint64, C.c_int64, C.c_int32, C.c_void_p
    for name, res, args in (("sc_wide_bits", u64, [vp, i32, i64]), ("sc_is_nan", i32, [u64]),
                            ("sc_word", u64, [u64, i32, i32]),
                            ("sc_cuts", None, [vp, vp, vp, i32, i64, vp, i32, vp, i32, i32, vp])):
        getattr(L, name).restype, getattr(L, name).argtypes = res, args
    return L


def _sorted_cls():
    from dpark_b200.sorting import ColumnarSortedRDD
    return ColumnarSortedRDD


def _col(dc, kdt=torch.int64, vdt=torch.int64, n=40, M=4):
    g = torch.Generator().manual_seed(n)
    return dc.parallelizeColumns(torch.randint(-9, 9, (n,), generator=g).to(kdt),
                                 torch.randint(-9, 9, (n,), generator=g).to(vdt), M)


# ------------------------------------------------------------------------------------------------ recognition
DEVICE_KEYS = [
    ("default", None, "kv"),
    ("identity", lambda x: x, "kv"),
    ("identity_renamed", lambda row: row, "kv"),
    ("first", lambda x: x[0], "k"),
    ("itemgetter0", operator.itemgetter(0), "k"),
    ("second", lambda x: x[1], "v"),
    ("itemgetter1", operator.itemgetter(1), "v"),
]


@pytest.mark.parametrize("name,key,order", DEVICE_KEYS, ids=[k[0] for k in DEVICE_KEYS])
@pytest.mark.parametrize("kdt", DTYPES, ids=str)
def test_recognised_keys_take_the_device_path(name, key, order, kdt):
    from dpark_b200 import sorting
    dc = cc.ctx()
    col = _col(dc, kdt, DTYPES[(DTYPES.index(kdt) + 1) % 4])
    out = col.sort() if key is None else col.sort(key=key, reverse=True, numSplits=3)
    assert isinstance(out, _sorted_cls())
    assert out.order == order and out.partitioner is None
    if key is not None:
        assert sorting.order_of(key) == order


def _closure_key():
    i = 0
    return lambda x: x[i]


OTHER_KEYS = [
    ("closure", _closure_key()),
    ("default_arg", lambda x=None: x),
    ("default_arg_first", lambda x, i=0: x[i]),
    ("last", lambda x: x[-1]),
    ("negated_first", lambda x: -x[0]),
    ("index_float", lambda x: x[0.0]),
    ("itemgetter_pair", operator.itemgetter(0, 1)),
    ("itemgetter2", operator.itemgetter(2)),
    ("itemgetter_float", operator.itemgetter(0.0)),
    ("str", str),
]


@pytest.mark.parametrize("name,key", OTHER_KEYS, ids=[k[0] for k in OTHER_KEYS])
def test_other_keys_keep_the_composition(name, key):
    from dpark_b200 import sorting
    assert sorting.order_of(key) is None
    assert not sorting.device_sort_applies(_col(cc.ctx()), key)


def test_other_inputs_keep_the_composition(monkeypatch):
    from dpark_b200 import sorting, spmd
    from dpark_b200.rdd import ColumnarRDD
    dc = cc.ctx()
    col = _col(dc)
    ident = lambda x: x     # noqa: E731
    assert sorting.device_sort_applies(col, ident)

    class MyColumns(ColumnarRDD):
        pass

    sub = MyColumns(dc, col.keys, col.vals, 3)
    wide = ColumnarRDD(dc, torch.arange(6).reshape(6, 1), torch.arange(6), 2)
    narrow = ColumnarRDD(dc, torch.arange(6, dtype=torch.int16), torch.arange(6), 2)
    flags = ColumnarRDD(dc, torch.arange(6), torch.ones(6, dtype=torch.bool), 2)
    for other in (sub, wide, narrow, flags, col.map(ident), col.mapValue(ident), dc.parallelize(col.collect(), 4)):
        assert not sorting.device_sort_applies(other, ident)
    assert not isinstance(sub.sort(ident), _sorted_cls())
    assert not isinstance(narrow.sort(ident), _sorted_cls())
    monkeypatch.setattr(sorting, "MAX_ROWS", col.keys.numel() - 1)
    assert not sorting.device_sort_applies(col, ident)
    monkeypatch.setattr(sorting, "MAX_ROWS", col.keys.numel())
    assert sorting.device_sort_applies(col, ident)
    monkeypatch.setattr(spmd, "rank_world", lambda: (0, 2))
    assert not sorting.device_sort_applies(col, ident)


# ------------------------------------------------------------------------------------------------ bounds
def _slices(xs, M):
    """ParallelCollection's (and ColumnarRDD's) splits: chunks of ceil(len / M)."""
    k = max(1, min(len(xs), M))
    per = -(-len(xs) // k)
    return [xs[i * per:i * per + per] for i in range(k)]


def _reference_bounds(xs, M, key, reverse, P):
    from dpark_b200.rdd import range_bounds
    chunks = _slices(xs, M)
    if len(chunks) == 1:
        return []
    P = min(cc.ctx().defaultMinSplits, len(chunks)) if P is None else P
    n = max(P * 10 // len(chunks), 1)
    return range_bounds([key(x) for c in chunks for x in c[:n]], P, reverse)


def _check_layout(parts, bounds, key, reverse):
    from dpark_b200.dependency import RangePartitioner
    assert len(parts) == len(bounds) + 1
    ranges = RangePartitioner(bounds, reverse=reverse)
    for p, part in enumerate(parts):
        assert all(ranges.getPartition(key(x)) == p for x in part), p


SORT = load("sort_cases.json")["cases"]
SORT_KEYS = {"id": lambda x: x, "neg": lambda x: -x, "second": lambda x: x[1], "mod": lambda x: (x % 10, x)}


@pytest.mark.parametrize("case", SORT, ids=[c["name"] for c in SORT])
def test_bounds_rule_gives_the_reference_layouts(case):
    """The shared bounds rule over the composition's samples puts every row of the reference's partition p into p."""
    xs = [dec(x) for x in case["xs"]]
    xs = [tuple(x) if isinstance(x, list) else x for x in xs]
    key = SORT_KEYS[case["key"]]
    parts = [[dec(x) for x in part] for part in case["parts"]]
    parts = [[tuple(x) if isinstance(x, list) else x for x in part] for part in parts]
    _check_layout(parts, _reference_bounds(xs, case["M"], key, case["reverse"], case["P"]), key, case["reverse"])


COLSORT = load("columnar_sort_cases.json")
COL_KEYS = {"id": lambda x: x, "first": lambda x: x[0], "second": lambda x: x[1]}


def golden_case(case):
    """(pairs, parts, key dtype, value dtype) of a columnar sort case, its partitions as lists of pairs."""
    inp = COLSORT["inputs"][case["input"]]
    pairs = [(dec(k), dec(v)) for k, v in inp["pairs"]]
    kdt, vdt = (torch.float64 if kind == "float" else torch.int64 for kind in inp["kinds"])
    return pairs, [[pairs[i] for i in part] for part in case["parts"]], kdt, vdt


@pytest.mark.parametrize("case", COLSORT["cases"], ids=[c["name"] for c in COLSORT["cases"]])
def test_sampled_bounds_of_columns_give_the_reference_layouts(case):
    """ColumnarSortedRDD's bounds, read from column slices, are the composition's and lay the reference's rows out as
    the reference did; the rows stay sorted across partitions."""
    dc = cc.ctx()
    key, reverse = COL_KEYS[case["key"]], case["reverse"]
    pairs, parts, kdt, vdt = golden_case(case)
    col = dc.parallelizeColumns(torch.tensor([k for k, _ in pairs], dtype=kdt),
                                torch.tensor([v for _, v in pairs], dtype=vdt), case["M"])
    out = col.sort(key=key, reverse=reverse, numSplits=case["P"])
    assert isinstance(out, _sorted_cls())
    assert out.bounds == _reference_bounds(pairs, case["M"], key, reverse, case["P"])
    _check_layout(parts, out.bounds, key, reverse)
    assert len(out.splits) == len(parts)
    flat = [key(x) for part in parts for x in part]
    assert flat == sorted(flat, reverse=reverse)


# ------------------------------------------------------------------------------------------------ sortcheck
def _edges(dt, rng):
    if not dt.is_floating_point:
        info = torch.iinfo(dt)
        xs = [info.min, info.min + 1, -2, -1, 0, 1, 2, info.max - 1, info.max]
        return xs + [rng.randrange(info.min, info.max) for _ in range(6)]
    info = np.finfo(np.float32 if dt == torch.float32 else np.float64)
    sub, tiny, big = float(info.smallest_subnormal), float(info.smallest_normal), float(info.max)
    xs = [float("-inf"), -big, -1.5, -1.0, -tiny, -2 * sub, -sub, -0.0, 0.0, sub, 2 * sub, tiny, 1.0, 1.5, big,
          float("inf")]
    return xs + [rng.uniform(-10, 10) for _ in range(4)]


def _column(dt, values):
    return torch.tensor(values, dtype=dt).numpy()


def _words(L, arr, dt, reverse):
    p = arr.ctypes.data_as(C.c_void_p)
    return [L.sc_word(L.sc_wide_bits(p, KIND[dt], i), int(dt.is_floating_point), int(reverse)) for i in range(len(arr))]


def _rows(rng, kdt, vdt, n):
    ke, ve = _edges(kdt, rng), _edges(vdt, rng)
    k = _column(kdt, [rng.choice(ke) for _ in range(n)])
    v = _column(vdt, [rng.choice(ve[:5]) if rng.random() < 0.5 else rng.choice(ve) for _ in range(n)])
    return k, v, list(zip(k.tolist(), v.tolist()))


def test_widening_is_what_python_sees():
    L = _sortcheck()
    rng = random.Random(1)
    for dt in DTYPES:
        arr = _column(dt, _edges(dt, rng))
        p = arr.ctypes.data_as(C.c_void_p)
        wide = np.array([L.sc_wide_bits(p, KIND[dt], i) for i in range(len(arr))], np.uint64)
        want = np.array(arr.tolist(), np.float64 if dt.is_floating_point else np.int64)
        assert np.array_equal(wide, want.view(np.uint64)), dt
        if dt.is_floating_point:        # only float columns are checked for NaN
            assert not any(L.sc_is_nan(int(w)) for w in wide)
    nans = np.array([float("nan"), -float("nan")], np.float32)
    assert all(L.sc_is_nan(L.sc_wide_bits(nans.ctypes.data_as(C.c_void_p), KIND[torch.float32], i)) for i in range(2))
    assert not L.sc_is_nan(np.array([float("inf")]).view(np.uint64)[0].item())


@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("vdt", DTYPES, ids=str)
@pytest.mark.parametrize("kdt", DTYPES, ids=str)
def test_sorting_by_the_order_words_is_python_sorted(kdt, vdt, reverse):
    """Rows of edge values (int extremes, +-0.0, +-inf, subnormals) with many ties: the stable sort by (k word, v word),
    by the k word alone and by the v word alone is Python's sorted of the tuples, of x[0] and of x[1]."""
    L = _sortcheck()
    rng = random.Random(DTYPES.index(kdt) * 8 + DTYPES.index(vdt) * 2 + reverse)
    k, v, rows = _rows(rng, kdt, vdt, 120)
    wk, wv = _words(L, k, kdt, reverse), _words(L, v, vdt, reverse)
    n = len(rows)
    assert sorted(range(n), key=lambda i: (wk[i], wv[i], i)) == sorted(range(n), key=lambda i: rows[i], reverse=reverse)
    assert sorted(range(n), key=lambda i: (wk[i], i)) == sorted(range(n), key=lambda i: rows[i][0], reverse=reverse)
    assert sorted(range(n), key=lambda i: (wv[i], i)) == sorted(range(n), key=lambda i: rows[i][1], reverse=reverse)


def _expected_starts(sorted_rows, bounds, key, reverse):
    """Partition starts from bisect: getPartition of every sorted row, which must be monotone."""
    from dpark_b200.dependency import RangePartitioner
    ranges = RangePartitioner(bounds, reverse=reverse)
    pids = [ranges.getPartition(key(x)) for x in sorted_rows]
    assert pids == sorted(pids)
    return [sum(1 for q in pids if q < j) for j in range(len(bounds) + 2)]


@pytest.mark.parametrize("order", ["kv", "k", "v"])
@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("vdt", DTYPES, ids=str)
@pytest.mark.parametrize("kdt", DTYPES, ids=str)
def test_cuts_are_the_bisect_partition_starts(kdt, vdt, reverse, order):
    """Bounds drawn from the rows, from values outside them and repeated: the cut of the sorted rows is where
    RangePartitioner(bounds, reverse) changes partition."""
    L = _sortcheck()
    rng = random.Random(DTYPES.index(kdt) * 8 + DTYPES.index(vdt) * 2 + reverse + 100 * len(order))
    ke, ve = _edges(kdt, rng), _edges(vdt, rng)
    k = _column(kdt, [rng.choice(ke[2:-2]) for _ in range(90)])      # the extremes stay outside the data
    v = _column(vdt, [rng.choice(ve[2:-2]) for _ in range(90)])
    rows = list(zip(k.tolist(), v.tolist()))
    key = {"kv": lambda x: x, "k": lambda x: x[0], "v": lambda x: x[1]}[order]
    wk, wv = _words(L, k, kdt, reverse), _words(L, v, vdt, reverse)
    w0, w1 = {"kv": (wk, wv), "k": (wk, None), "v": (wv, None)}[order]
    n = len(rows)
    ids = np.array(sorted(range(n), key=lambda i: (w0[i], w1[i] if w1 else 0, i)), np.int64)
    sorted_rows = [rows[i] for i in ids]
    extra = list(zip(_column(kdt, ke).tolist(), _column(vdt, ve).tolist()))
    for trial in range(6):
        pool = [key(r) for r in rng.sample(rows, 6)] + [key(r) for r in rng.sample(extra, 4)]
        bounds = [rng.choice(pool) for _ in range(rng.randrange(0, 9))]
        bounds += bounds[:2]                                          # duplicates give empty partitions
        ordered = sorted(bounds)
        first = [b[0] for b in ordered] if order == "kv" else ordered
        d0 = {"kv": kdt, "k": kdt, "v": vdt}[order]
        b0 = np.array(first, np.float64 if d0.is_floating_point else np.int64).view(np.uint64)
        b1 = (np.array([b[1] for b in ordered], np.float64 if vdt.is_floating_point else np.int64).view(np.uint64)
              if order == "kv" else None)
        sw0 = np.array([w0[i] for i in ids], np.uint64)
        out = np.zeros(len(bounds) + 2, np.int64)
        ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)   # noqa: E731
        L.sc_cuts(ptr(sw0), ptr(ids), ptr(v), KIND[vdt], n, ptr(b0), KIND[d0], ptr(b1), len(bounds), int(reverse),
                  ptr(out))
        assert out.tolist() == _expected_starts(sorted_rows, bounds, key, reverse), (trial, bounds)
