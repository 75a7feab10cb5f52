"""top, uniq and hot on a CPU: which calls take the device path (dpark_b200/selecting.py), the reference's golden cases
through the composition (stand-in engine), and the select and distinct-table arithmetic of dpk_common.cuh run through
tests/selectcheck.cu -- radix rounds, the stable take and the first-occurrence table -- against Python's sorted and
dict.  The device results themselves are checked in tests/test_gpu_uniq_top_hot.py."""
import ctypes as C
import json
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
from tests.standin import standin_engine  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KIND = {torch.int64: 0, torch.int32: 1, torch.float64: 2, torch.float32: 4}
DTYPES = [torch.int32, torch.int64, torch.float32, torch.float64]
GOLDEN = load("uniq_top_hot_cases.json")["cases"]
GOLDEN_KEYS = {"none": None, "first": lambda x: x[0], "second": lambda x: x[1], "neg": lambda x: -x}


def _selectcheck():
    path = os.path.join(ROOT, "tests", "_selectcheck.so")
    if not os.path.exists(path):
        subprocess.call([sys.executable, "-c", "import __graft_entry__ as g; g.build()"], cwd=ROOT)
    if not os.path.exists(path):
        pytest.skip("selectcheck not built")
    L = C.CDLL(path)
    u64, i64, i32, u32, vp = C.c_uint64, C.c_int64, C.c_int32, C.c_uint32, C.c_void_p
    for name, res, args in (("slc_digit", u32, [u64, i32]), ("slc_bucket", i32, [vp, i64, vp]),
                            ("slc_next_shift", i32, [u64]),
                            ("slc_select", i32, [vp, vp, i64, i64, vp]),
                            ("slc_uniq", i64, [vp, i32, vp, i32, i64, vp, vp])):
        getattr(L, name).restype, getattr(L, name).argtypes = res, args
    return L


def _col(dc, kdt=torch.int64, vdt=torch.int64, n=40, M=4):
    g = torch.Generator().manual_seed(n)
    return dc.parallelizeColumns(torch.randint(-9, 9, (n,), generator=g).to(kdt),
                                 torch.randint(-9, 9, (n,), generator=g).to(vdt), M)


# ------------------------------------------------------------------------------------------------ recognition
TOP_KEYS = [(None, True), (lambda x: x, True), (lambda x: x[0], True), (operator.itemgetter(0), True),
            (lambda x: x[1], True), (operator.itemgetter(1), True), (lambda x: -x[0], False),
            (operator.itemgetter(0, 1), False), (operator.itemgetter(2), False), (len, False)]


@pytest.mark.parametrize("key,device", TOP_KEYS)
def test_top_key_recognition(key, device):
    from dpark_b200 import selecting
    assert selecting.top_applies(_col(cc.ctx()), 10, key) is device


@pytest.mark.parametrize("vdt", DTYPES, ids=str)
@pytest.mark.parametrize("kdt", DTYPES, ids=str)
def test_which_calls_apply(kdt, vdt):
    """Every numeric dtype pair; only an int n (booleans, numpy ints, floats and strings keep the composition)."""
    from dpark_b200 import selecting
    col = _col(cc.ctx(), kdt, vdt)
    assert selecting.top_applies(col, -3, None) and selecting.uniq_applies(col) and selecting.hot_applies(col, 0)
    for n in (10.0, True, np.int64(10), "10", None):
        assert not selecting.top_applies(col, n, None) and not selecting.hot_applies(col, n)


def test_other_inputs_keep_the_composition(monkeypatch):
    from dpark_b200 import selecting, spmd
    from dpark_b200.rdd import ColumnarRDD
    dc = cc.ctx()

    class Sub(ColumnarRDD):
        pass

    sub = Sub(dc, torch.arange(8), torch.arange(8), 2)
    flat = dc.parallelizeColumns(torch.arange(8).view(4, 2), torch.arange(8).view(4, 2), 2)
    u8 = dc.parallelizeColumns(torch.arange(8, dtype=torch.uint8), torch.arange(8), 2)
    rows = dc.parallelize([(1, 2), (3, 4)], 2)
    for rdd in (sub, flat, u8, rows, _col(dc).map(lambda x: x)):
        assert not selecting.top_applies(rdd, 3, None)
        assert not selecting.uniq_applies(rdd) and not selecting.hot_applies(rdd, 3)
    col = _col(dc)
    monkeypatch.setattr(spmd, "rank_world", lambda: (0, 2))
    assert not selecting.top_applies(col, 3, None) and not selecting.uniq_applies(col)


def test_dispatch(monkeypatch):
    """RDD.top / uniq / hot hand device inputs to selecting with the composition's partitioner, and everything else
    to the composition."""
    from dpark_b200 import selecting
    from dpark_b200.dependency import HashPartitioner, RangePartitioner
    dc = cc.ctx()
    seen = []
    monkeypatch.setattr(selecting, "top", lambda rdd, n, key, reverse: seen.append(("top", n, reverse)) or ["dev"])
    monkeypatch.setattr(selecting, "hot", lambda rdd, n, part: seen.append(("hot", n, part)) or ["dev"])
    col = _col(dc, M=5)
    assert col.top(4, reverse=True) == ["dev"] and col.hot(3, 5) == ["dev"] and col.hot(3) == ["dev"]
    default = HashPartitioner(min(dc.defaultMinSplits, 5))
    assert seen == [("top", 4, True), ("hot", 3, HashPartitioner(5)), ("hot", 3, default)]
    u = col.uniq(HashPartitioner(3, [0, 5]))
    assert isinstance(u, selecting.ColumnarUniqRDD) and len(u) == 3 and u.partitioner is None
    assert u.part == HashPartitioner(3, [0, 5]) and selecting.device_partitioner(col, RangePartitioner([1])) is None
    rows = dc.parallelize([(1, 2), (3, 4), (1, 2)], 2)
    assert rows.top(1) == [(3, 4)] and not isinstance(rows.uniq(2), selecting.ColumnarUniqRDD)
    monkeypatch.setattr(selecting, "top", lambda rdd, n, key, reverse: None)      # a NaN in an order column
    assert col.top(2, key=lambda x: x[0]) == col.map(lambda x: x).top(2, key=lambda x: x[0])


# ------------------------------------------------------------------------------------------------ golden cases
def _enc(o):
    from tests.golden.make_golden import enc
    return enc(o)


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_golden_composition(case, standin_engine):  # noqa: F811
    dc = cc.ctx()
    rows = [dec(x) for x in case["rows"]]
    rdd = dc.parallelize(rows, case["M"])
    for t in case["top"]:
        got = rdd.top(t["n"], key=GOLDEN_KEYS[t["key"]], reverse=t["reverse"])
        assert [_enc(x) for x in got] == t["want"]
    check_uniq_hot(rdd, case)


def canon(x):
    """An element as == sees it: a float -0.0 spelled 0.0 (which occurrence's bits a partition keeps is the fetch
    order's choice in the reference)."""
    if isinstance(x, tuple):
        return tuple(canon(e) for e in x)
    return x + 0.0 if isinstance(x, float) else x


def _set(xs):
    return sorted((_enc(canon(x)) for x in xs), key=json.dumps)


def check_uniq_hot(rdd, case):
    """rdd.uniq(P): the golden per-partition sets under ==; rdd.hot(n, P): the golden counts, each element among those
    with its count, and every count above the n-th one with all its elements."""
    parts = [_set(part) for part in rdd.uniq(case["P"]).glom().collect()]
    assert parts == [_set(dec(x) for x in part) for part in case["uniq"]]
    sets = {c: _set(dec(x) for x in xs) for c, xs in case["counts"]}
    for h in case["hot"]:
        got = rdd.hot(h["n"], case["P"])
        assert [c for _, c in got] == h["counts"]
        assert all(_enc(canon(x)) in sets[c] for x, c in got)
        for c in set(h["counts"]) - {min(h["counts"], default=None)}:
            assert _set(x for x, cc_ in got if cc_ == c) == sets[c]


# ------------------------------------------------------------------------------------------------ selectcheck
def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _select(L, w0, w1, n):
    m = len(w0)
    out = np.zeros(max(1, min(n, m)), dtype=np.int64)
    rounds = L.slc_select(_ptr(w0), _ptr(w1), m, n, _ptr(out))
    return out[:min(n, m)].tolist(), rounds


def _want(w0, w1, n):
    key = (lambda i: (int(w0[i]), int(w1[i]))) if w1 is not None else (lambda i: int(w0[i]))
    return sorted(range(len(w0)), key=key)[:n]


WORDS = {
    "uniform": lambda r, m: r.integers(0, 1 << 63, m, dtype=np.uint64) * 2 + r.integers(0, 2, m, dtype=np.uint64),
    "small": lambda r, m: r.integers(0, 1 << 10, m).astype(np.uint64),
    "all_equal": lambda r, m: np.full(m, 0x8000000000000123, dtype=np.uint64),
    "two_values": lambda r, m: np.where(r.random(m) < 0.5, 5, 1 << 62).astype(np.uint64),
    "spread_bits": lambda r, m: (np.uint64(1) << r.integers(0, 64, m).astype(np.uint64)),
    "extremes": lambda r, m: r.choice(np.array([0, 1, (1 << 64) - 1, 1 << 63, (1 << 63) - 1], dtype=np.uint64), m),
}


@pytest.mark.parametrize("two", [False, True], ids=["one_word", "two_words"])
@pytest.mark.parametrize("dist", sorted(WORDS))
def test_selectcheck_matches_sorted(dist, two):
    L = _selectcheck()
    r = np.random.default_rng(len(dist) * 7 + two)
    m = 3000
    w0 = WORDS[dist](r, m)
    w1 = WORDS["small"](r, m) if two else None
    for n in (1, 2, 7, 10, 100, 1499, m - 1, m, m + 5):
        got, rounds = _select(L, w0, w1, n)
        assert rounds >= 0, "select failed (%d) at n=%d" % (rounds, n)
        assert rounds <= 8 * (2 if two else 1)
        assert got == _want(w0, w1, n)


def test_selectcheck_all_equal_is_two_rounds():
    """One round per word when every row agrees: the ORs and ANDs show no differing bit."""
    L = _selectcheck()
    w = np.full(500, 77, dtype=np.uint64)
    assert _select(L, w, None, 10) == (list(range(10)), 1)
    assert _select(L, w, w.copy(), 10) == (list(range(10)), 2)


def test_selectcheck_bucket_and_shift():
    L = _selectcheck()
    hist = np.zeros(256, dtype=np.int64)
    hist[[3, 9, 200]] = [5, 1, 10]
    below = C.c_int64()
    for need, b, bl in ((1, 3, 0), (5, 3, 0), (6, 9, 5), (7, 200, 6), (16, 200, 6)):
        assert L.slc_bucket(_ptr(hist), need, C.byref(below)) == b and below.value == bl
    assert L.slc_digit(0xAB << 48, 48) == 0xAB and L.slc_digit(0x1FF, 1) == 0xFF
    for diff, shift in ((1, 0), (0x80, 0), (0x100, 1), (1 << 55, 48), (0x8000_0000_0000, 40)):
        assert L.slc_next_shift(diff) == shift


@pytest.mark.parametrize("vdt", DTYPES, ids=str)
@pytest.mark.parametrize("kdt", DTYPES, ids=str)
def test_selectcheck_uniq_first_occurrence(kdt, vdt):
    """The table's pairs, counts and first rows are a dict's over the rows in order: each element widened, -0.0 finds
    0.0, int32 extremes stay apart; a NaN in either column is refused."""
    L = _selectcheck()
    rnd = random.Random(KIND[kdt] * 8 + KIND[vdt])
    n = 2000

    def one(dt, lo, hi):
        x = rnd.randrange(lo, hi)
        if dt.is_floating_point:
            return -0.0 if x == 0 and rnd.random() < 0.5 else x * 0.5
        return x if x else rnd.choice([0, -2 ** 31, 2 ** 31 - 1])

    rows = [(one(kdt, -20, 20), one(vdt, -5, 5)) for _ in range(n)]
    k = torch.tensor([a for a, _ in rows], dtype=kdt)
    v = torch.tensor([b for _, b in rows], dtype=vdt)
    first, count = np.zeros(n, dtype=np.int64), np.zeros(n, dtype=np.int64)

    def run(k, v):
        return L.slc_uniq(C.c_void_p(k.data_ptr()), KIND[kdt], C.c_void_p(v.data_ptr()), KIND[vdt], int(k.numel()),
                          _ptr(first), _ptr(count))

    d = run(k, v)
    want = {}
    for i, x in enumerate(zip(k.tolist(), v.tolist())):
        f, c = want.get(x, (i, 0))
        want[x] = (f, c + 1)
    assert d == len(want)
    assert sorted(zip(first[:d].tolist(), count[:d].tolist())) == sorted(want.values())
    for col in (k, v):
        if col.dtype.is_floating_point:
            col[n // 2] = float("nan")
            assert run(k, v) == -1
