"""top, uniq and hot of numeric ColumnarRDDs on the device (dpark_b200/selecting.py): against the composition over the
same splits (forced with col.map(lambda x: x), which is not a ColumnarRDD), against the reference's golden cases, and
against a numpy oracle (a stable argsort of the order words for top; np.unique over the canonical pair bits with
return_index, partitions from the oracle's portable_hash, for uniq and hot)."""
import operator

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tests import cogroup_common as cc
from tests.golden_util import dec
from tests.test_uniq_top_hot_host import GOLDEN, GOLDEN_KEYS, _enc, canon, check_uniq_hot

pytestmark = pytest.mark.gpu

DTYPES = [torch.int32, torch.int64, torch.float32, torch.float64]
BITS = {torch.int32: torch.int32, torch.int64: torch.int64, torch.float32: torch.int32, torch.float64: torch.int64}
KEYS = {"none": None, "first": lambda x: x[0], "second": lambda x: x[1], "itemgetter1": operator.itemgetter(1)}
NAN_MSG = "NaN keys are not supported"


@pytest.fixture
def device_spy(monkeypatch):
    """The device path must not read its input row by row, encode tuple keys or run the bytes reduce."""
    from dpark_b200 import columnar, strings
    from dpark_b200.rdd import ColumnarRDD

    def forbidden(*args, **kw):
        raise AssertionError("the device path read its input as rows or went through the tuple-key shuffle")

    monkeypatch.setattr(ColumnarRDD, "compute", forbidden)
    monkeypatch.setattr(strings, "reduce_by_key_bytes", forbidden)
    monkeypatch.setattr(columnar, "_tuple_identity_bytes", forbidden)


def _columns(rng, kdt, vdt, n, lo=-30, hi=30):
    """Columns with many ties and both signed zeros among the floats."""
    k = rng.integers(lo, hi, n).astype(np.float64)
    v = rng.integers(-4, 4, n).astype(np.float64)
    for a, dt in ((k, kdt), (v, vdt)):
        if dt.is_floating_point:
            a *= 0.5
            a[rng.random(n) < 0.1] = -0.0
            a[rng.random(n) < 0.02] = float("inf")
            a[rng.random(n) < 0.02] = -float("inf")
    return torch.from_numpy(k).to(kdt), torch.from_numpy(v).to(vdt)


def _same(got, want):
    """Equal lists, floats bit for bit (so -0.0 is checked)."""
    assert got == want and repr(got) == repr(want)


# ------------------------------------------------------------------------------------------------ top
@pytest.mark.parametrize("reverse", [False, True], ids=["largest", "smallest"])
@pytest.mark.parametrize("key", sorted(KEYS))
@pytest.mark.parametrize("vdt", DTYPES, ids=str)
@pytest.mark.parametrize("kdt", DTYPES, ids=str)
def test_top_is_the_composition(kdt, vdt, key, reverse):
    dc = cc.ctx()
    rng = np.random.default_rng(DTYPES.index(kdt) * 4 + DTYPES.index(vdt))
    rows = 5000
    k, v = _columns(rng, kdt, vdt, rows)
    col = dc.parallelizeColumns(k.cuda(), v.cuda(), 7)
    rowwise = col.map(lambda x: x)
    for n in (0, 1, 7, 10, 4096, rows - 1, rows, rows + 5):
        _same(col.top(n, key=KEYS[key], reverse=reverse), rowwise.top(n, key=KEYS[key], reverse=reverse))


@pytest.mark.parametrize("case", ["all_equal", "zeros", "int64_extremes"])
def test_top_edges(case, device_spy):
    dc = cc.ctx()
    n = 3000
    if case == "all_equal":
        k, v = torch.full((n,), 7, dtype=torch.int64), torch.full((n,), 2.5, dtype=torch.float64)
    elif case == "zeros":
        k = torch.where(torch.arange(n) % 3 == 0, -0.0, 0.0).to(torch.float64)
        v = torch.where(torch.arange(n) % 5 == 0, -0.0, 0.0).to(torch.float32)
    else:
        ext = torch.tensor([-2 ** 63, 2 ** 63 - 1, 0, -1, 1], dtype=torch.int64)
        k, v = ext[torch.arange(n) % 5], ext[(torch.arange(n) * 7) % 5]
    col = dc.parallelizeColumns(k.cuda(), v.cuda(), 4)
    rows = list(zip(k.tolist(), v.tolist()))
    for key in KEYS.values():
        f = key or (lambda x: x)
        for reverse in (False, True):
            for m in (1, 10, 2999):
                _same(col.top(m, key=key, reverse=reverse), sorted(rows, key=f, reverse=not reverse)[:m])


def test_top_nan_and_empty():
    """A NaN in an order column keeps the composition; one outside it stays on the device."""
    dc = cc.ctx()
    k = torch.tensor([1.0, float("nan"), 3.0, 2.0, 3.0] * 40, dtype=torch.float64)
    col = dc.parallelizeColumns(k.cuda(), torch.arange(200).cuda(), 3)
    assert repr(col.top(9, key=lambda x: x[0])) == repr(col.map(lambda x: x).top(9, key=lambda x: x[0]))
    rows = list(zip(torch.arange(200).tolist(), k.tolist()))
    col = dc.parallelizeColumns(torch.arange(200).cuda(), k.cuda(), 3)
    assert repr(col.top(15, key=lambda x: x[0])) == repr(sorted(rows, key=lambda x: x[0], reverse=True)[:15])
    col = dc.parallelizeColumns(torch.empty(0, dtype=torch.int64).cuda(), torch.empty(0).cuda(), 2)
    assert col.top(5) == [] and col.hot(5) == [] and col.uniq(3).glom().collect() == [[], [], []]


# ------------------------------------------------------------------------------------------------ uniq / hot oracle
def _wide(t):
    """A column as Python sees it: ints as int64, floats as float64."""
    return t.cpu().to(torch.float64 if t.dtype.is_floating_point else torch.int64).numpy()


def _tuple_hash2(h0, h1):
    """portable_hash.pyx tuple_hash of 2 items, vectorised (int64 wraparound)."""
    with np.errstate(over="ignore"):
        value = np.uint64(0x345678)
        value = (value ^ h0.view(np.uint64)) * np.uint64(1000003)
        value = (value ^ h1.view(np.uint64)) * np.uint64(1000003 + 82520 + 2)
        value = value + np.uint64(97531)
    out = value.view(np.int64)
    return np.where(out == -1, -2, out)


def oracle_uniq(k, v, P):
    """Per partition (keys, vals, counts) in order of first occurrence, the first occurrence's bits."""
    pair = np.stack([(_wide(k) + 0).view(np.int64), (_wide(v) + 0).view(np.int64)], axis=1)    # + 0: -0.0 is 0.0
    pair = pair.view([("k", np.int64), ("v", np.int64)]).ravel()
    _, first, counts = np.unique(pair, return_index=True, return_counts=True)
    pid = orc.partition_vec(_tuple_hash2(orc.hash_vec(_wide(k))[first], orc.hash_vec(_wide(v))[first]), P)
    order = np.lexsort((first, pid))
    kn, vn = k.cpu().numpy(), v.cpu().numpy()
    out = []
    for p in range(P):
        sel = order[pid[order] == p]
        out.append((kn[first[sel]], vn[first[sel]], counts[sel]))
    return out


def test_tuple_hash_matches_the_oracle():
    rng = np.random.default_rng(5)
    a = rng.integers(-2 ** 62, 2 ** 62, 200)
    b = rng.integers(-2 ** 62, 2 ** 62, 200)
    got = _tuple_hash2(orc.hash_vec(a), orc.hash_vec(b))
    assert got.tolist() == [orc.portable_hash((int(x), int(y))) for x, y in zip(a, b)]


def _check_uniq_oracle(col, k, v, P):
    u = col.uniq(P)
    want = oracle_uniq(k, v, P)
    assert len(u) == P and u.partitioner is None
    for sp, (wk, wv, _) in zip(u.splits, want):
        gk, gv = u.columns(sp)
        assert gk.is_cuda and gk.dtype == k.dtype and gv.dtype == v.dtype
        assert np.array_equal(gk.cpu().view(BITS[k.dtype]).numpy(), torch.from_numpy(wk).view(BITS[k.dtype]).numpy())
        assert np.array_equal(gv.cpu().view(BITS[v.dtype]).numpy(), torch.from_numpy(wv).view(BITS[v.dtype]).numpy())
    return want


def _hot_oracle(want, n):
    """Stable top n by count over uniq's order."""
    flat = [((a, b), int(c)) for wk, wv, wc in want for a, b, c in zip(wk.tolist(), wv.tolist(), wc.tolist())]
    return sorted(flat, key=lambda x: x[1], reverse=True)[:max(n, 0)]


@pytest.mark.parametrize("vdt", DTYPES, ids=str)
@pytest.mark.parametrize("kdt", DTYPES, ids=str)
def test_uniq_and_hot_against_the_oracle(kdt, vdt, device_spy):
    dc = cc.ctx()
    rng = np.random.default_rng(100 + DTYPES.index(kdt) * 4 + DTYPES.index(vdt))
    k, v = _columns(rng, kdt, vdt, 20000)
    col = dc.parallelizeColumns(k.cuda(), v.cuda(), 6)
    for P in (1, 5, 16):
        want = _check_uniq_oracle(col, k, v, P)
        for n in (0, 1, 10, 100000):
            got = col.hot(n, P)
            _same(got, _hot_oracle(want, n))
            _same(col.hot(n, P), got)


def test_uniq_keeps_the_first_signed_zero(device_spy):
    dc = cc.ctx()
    k = torch.tensor([-0.0, 0.0, 0.0, 1.0, -0.0], dtype=torch.float64)
    v = torch.tensor([0.0, -0.0, 0.0, -0.0, 5.0], dtype=torch.float32)
    col = dc.parallelizeColumns(k.cuda(), v.cuda(), 2)
    got = col.uniq(1).collect()
    assert repr(got) == repr([(-0.0, 0.0), (1.0, -0.0), (-0.0, 5.0)])
    _check_uniq_oracle(col, k, v, 3)


@pytest.mark.parametrize("vdt", DTYPES, ids=str)
@pytest.mark.parametrize("kdt", DTYPES, ids=str)
def test_uniq_and_hot_are_the_composition(kdt, vdt):
    dc = cc.ctx()
    rng = np.random.default_rng(200 + DTYPES.index(kdt) * 4 + DTYPES.index(vdt))
    k, v = _columns(rng, kdt, vdt, 3000, -8, 8)
    col = dc.parallelizeColumns(k.cuda(), v.cuda(), 5)
    rowwise = col.map(lambda x: x)
    for P in (1, 4):
        got = [sorted(map(canon, part)) for part in col.uniq(P).glom().collect()]
        assert got == [sorted(map(canon, part)) for part in rowwise.uniq(P).glom().collect()]
        for n in (1, 10, 50):
            g, w = col.hot(n, P), rowwise.hot(n, P)
            assert [c for _, c in g] == [c for _, c in w]
            cut = w[-1][1]
            assert sorted(canon(x) for x, c in g if c > cut) == sorted(canon(x) for x, c in w if c > cut)


@pytest.mark.parametrize("which", ["key", "value"])
def test_uniq_and_hot_raise_on_nan(which):
    dc = cc.ctx()
    k = torch.tensor([1.0, 2.0, float("nan") if which == "key" else 3.0], dtype=torch.float64)
    v = torch.tensor([1.0, float("nan") if which == "value" else 2.0, 3.0], dtype=torch.float32)
    col = dc.parallelizeColumns(k.cuda(), v.cuda(), 2)
    u = col.uniq(2)                  # nothing is computed before a partition is asked for
    with pytest.raises(TypeError, match=NAN_MSG):
        u.collect()
    with pytest.raises(TypeError, match=NAN_MSG):
        col.hot(3)
    with pytest.raises(TypeError, match=NAN_MSG):
        col.map(lambda x: x).uniq(2).collect()


# ------------------------------------------------------------------------------------------------ golden
PAIR_GOLDEN = [c for c in GOLDEN if c["name"].startswith("pairs_")]
DT = {"i": torch.int64, "f": torch.float64}


@pytest.mark.parametrize("case", PAIR_GOLDEN, ids=[c["name"] for c in PAIR_GOLDEN])
def test_golden(case, device_spy):
    dc = cc.ctx()
    kinds = case["name"].split("_")[1]
    rows = [dec(x) for x in case["rows"]]
    k = torch.tensor([a for a, _ in rows], dtype=DT[kinds[0]])
    v = torch.tensor([b for _, b in rows], dtype=DT[kinds[1]])
    col = dc.parallelizeColumns(k.cuda(), v.cuda(), case["M"])
    for t in case["top"]:
        got = col.top(t["n"], key=GOLDEN_KEYS[t["key"]], reverse=t["reverse"])
        assert [_enc(x) for x in got] == t["want"]
    check_uniq_hot(col, case)


# ------------------------------------------------------------------------------------------------ scale
@pytest.mark.parametrize("dist", ["uniform", "all_distinct", "zipf"])
def test_1e7_rows_against_the_oracle(dist, device_spy):
    dc = cc.ctx()
    rng = np.random.default_rng(7)
    n = 10 ** 7
    if dist == "uniform":
        k, v = rng.integers(0, 1 << 12, n), rng.integers(0, 8, n)
    elif dist == "all_distinct":
        k, v = rng.permutation(n), rng.integers(-2 ** 62, 2 ** 62, n)
    else:
        k, v = np.minimum(rng.zipf(1.1, n), 1 << 40), rng.integers(0, 2, n)
    k, v = torch.from_numpy(k.astype(np.int64)), torch.from_numpy(v.astype(np.int64))
    col = dc.parallelizeColumns(k.cuda(), v.cuda(), 64)
    want = _check_uniq_oracle(col, k, v, 64)
    _same(col.hot(10, 64), _hot_oracle(want, 10))
    order = np.lexsort((np.arange(n), -v.numpy()))           # top(10, x[1]): descending v, ties by row
    _same(col.top(100, key=lambda x: x[1]), [(int(k[i]), int(v[i])) for i in order[:100]])
    order = np.lexsort((np.arange(n), -v.numpy(), -k.numpy()))  # top(1000): descending (k, v), ties by row
    _same(col.top(1000), [(int(k[i]), int(v[i])) for i in order[:1000]])
