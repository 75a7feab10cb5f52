"""The device innerJoin of numeric ColumnarRDDs (dpark_b200/join.py, ColumnarInnerJoinedRDD): against the reference's
golden cases, against the row path (the same rows through ctx.parallelize, whose innerJoin is a dict on the host and a
flatMap), and at scale against a numpy restatement (a stable sort of the small side, a searchsorted per big row,
np.repeat)."""
import numpy as np
import pytest
import torch

from tests import cogroup_common as cc
from tests.golden_util import dec, load

pytestmark = pytest.mark.gpu

INTS = [torch.int32, torch.int64]
FLOATS = [torch.float32, torch.float64]
DTYPES = INTS + FLOATS


def _cls():
    from dpark_b200.join import ColumnarInnerJoinedRDD
    return ColumnarInnerJoinedRDD


@pytest.fixture
def spy(monkeypatch):
    """Counts the small side's group-bys and the three kernels' launches."""
    from dpark_b200 import _native as nv
    from dpark_b200 import grouping
    calls = {"group": 0, "build": 0, "probe": 0, "emit": 0}

    def counted(name, real):
        def run(*args, **kw):
            calls[name] += 1
            return real(*args, **kw)
        return run

    monkeypatch.setattr(grouping, "group_row_ids", counted("group", grouping.group_row_ids))
    for name in ("build", "probe", "emit"):
        monkeypatch.setattr(nv, "bcast_" + name, counted(name, getattr(nv, "bcast_" + name)))
    return calls


# ------------------------------------------------------------------------------------------------ golden
CASES = load("innerjoin_cases.json")["cases"]


@pytest.mark.parametrize("dtype", INTS, ids=str)
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden_inner_join_cases_on_the_device(case, dtype, spy):
    dc = cc.ctx()

    def col(rows, M):
        return dc.parallelizeColumns(torch.tensor([dec(k) for k, _ in rows], dtype=dtype),
                                     torch.tensor([dec(v) for _, v in rows], dtype=dtype), M)

    out = col(case["big"], case["M_big"]).innerJoin(col(case["small"], case["M_small"]))
    assert isinstance(out, _cls())
    assert out.collect() == [(dec(k), dec(v)) for k, v in case["rows"]]
    assert out.glom().collect() == [[(dec(k), dec(v)) for k, v in part] for part in case["parts"]]
    assert spy == {"group": 1, "build": 1, "probe": 1, "emit": 1}


# ------------------------------------------------------------------------------------------------ identity
SHAPES = ["overlap", "empty_big", "empty_small", "disjoint", "all_match", "fewer_rows_than_splits", "one_split",
          "many_splits", "hot", "colliding", "specials", "extremes"]


def _keys(rng, shape, kdt_big, kdt_small):
    """(big keys, small keys, big splits, small splits) as float64 / int64 numpy columns."""
    is_float = kdt_big.is_floating_point
    nb, ns, Mb, Ms, span = 3000, 400, 6, 3, 600
    if shape == "empty_big":
        nb = 0
    elif shape == "empty_small":
        ns = 0
    elif shape == "fewer_rows_than_splits":
        nb, Mb = 5, 9
    elif shape == "one_split":
        Mb = 1
    elif shape == "many_splits":
        Mb, Ms = 97, 13
    bk = rng.integers(-span, span, nb)
    sk = rng.integers(-span, span, ns)
    if shape == "disjoint":
        sk = sk + 10 * span
    elif shape == "all_match":
        bk = rng.choice(sk, nb)
    elif shape == "hot":           # one small key with 3000 values, hit by every 7th big row
        sk = np.concatenate([sk, np.full(3000, 17)])[rng.permutation(ns + 3000)]
        bk[::7] = 17
    elif shape == "colliding":     # keys equal in their low 32 bits (ints) / in their mantissa (floats)
        if is_float:
            bk, sk = np.ldexp(1.0, bk % 300 - 150), np.ldexp(1.0, sk % 300 - 150)
        elif kdt_big == kdt_small == torch.int64:
            bk, sk = (bk % 64) << 32, (sk % 64) << 32
        else:
            bk, sk = (bk % 64) << 24, (sk % 64) << 24
    if is_float:
        bk, sk = bk * 0.25, sk * 0.25
        if shape == "specials":
            bk[rng.random(nb) < 0.1], sk[rng.random(ns) < 0.1] = -0.0, 0.0
            sk[rng.random(ns) < 0.05] = -0.0
            bk[rng.random(nb) < 0.05], sk[rng.random(ns) < 0.05] = np.nan, np.nan
            bk[:2], sk[:2] = np.inf, -np.inf
            bk[2:4], sk[2:4] = -np.inf, np.inf
        if shape == "extremes":
            sub = float(np.finfo(np.float32).smallest_subnormal)
            vals = np.array([sub, -sub, float(np.finfo(np.float32).max), 0.1, -0.0])
            bk[::3], sk[::2] = rng.choice(vals, len(bk[::3])), rng.choice(vals, len(sk[::2]))
    elif shape == "extremes":
        info = torch.iinfo(torch.int32 if torch.int32 in (kdt_big, kdt_small) else torch.int64)
        vals = np.array([info.min, info.min + 1, -1, 0, info.max - 1, info.max], np.int64)
        bk[::3], sk[::2] = rng.choice(vals, len(bk[::3])), rng.choice(vals, len(sk[::2]))
    return bk, sk, Mb, Ms


def _cast(a, dtype):
    return torch.from_numpy(np.asarray(a)).to(dtype)


PAIRS = [(a, b) for a in INTS for b in INTS] + [(a, b) for a in FLOATS for b in FLOATS]


@pytest.mark.parametrize("kdt_big,kdt_small", PAIRS, ids=str)
@pytest.mark.parametrize("shape", SHAPES)
def test_device_inner_join_equals_the_row_path(shape, kdt_big, kdt_small, spy):
    i = PAIRS.index((kdt_big, kdt_small))
    rng = np.random.default_rng(100 * SHAPES.index(shape) + i)
    dc = cc.ctx()
    bk, sk, Mb, Ms = _keys(rng, shape, kdt_big, kdt_small)
    lvdt, rvdt = DTYPES[i % 4], DTYPES[(i + 1 + SHAPES.index(shape)) % 4]
    lv = rng.integers(-50, 50, len(bk)) * (0.5 if lvdt.is_floating_point else 1)
    rv = rng.integers(-10 ** 6, 10 ** 6, len(sk)) * (0.5 if rvdt.is_floating_point else 1)
    big = dc.parallelizeColumns(_cast(bk, kdt_big).cuda(), _cast(lv, lvdt).cuda(), Mb)
    small = dc.parallelizeColumns(_cast(sk, kdt_small), _cast(rv, rvdt), Ms)      # host columns are taken as well
    out = big.innerJoin(small)
    assert isinstance(out, _cls()) and out.partitioner is None and len(out) == len(big.splits)
    got = out.glom().collect()
    want = dc.parallelize(big.collect(), len(big.splits)).innerJoin(dc.parallelize(small.collect(), Ms)).glom().collect()
    assert [len(p) for p in got] == [len(p) for p in want]
    assert got == want and repr(got) == repr(want)          # order, -0.0 keys and value types included
    for sp in out.splits:
        keys, left, right = out.columns(sp)
        assert all(t.is_cuda for t in (keys, left, right))
        assert (keys.dtype, left.dtype, right.dtype) == (kdt_big, lvdt, rvdt)
    if shape in ("overlap", "all_match", "hot", "colliding", "specials", "extremes", "many_splits"):
        assert sum(map(len, got)) > 0
    if shape not in ("empty_big", "empty_small"):
        assert spy == {"group": 1, "build": 1, "probe": 1, "emit": 1}


# ------------------------------------------------------------------------------------------------ scale
def _numpy_inner_join(bk, bv, sk, sv):
    """Every big row's matches in small row order: a stable sort of small, searchsorted per big row, np.repeat."""
    order = np.argsort(sk, kind="stable")
    ks = sk[order]
    lo, hi = np.searchsorted(ks, bk, "left"), np.searchsorted(ks, bk, "right")
    cnt = hi - lo
    off = np.concatenate([[0], np.cumsum(cnt)])
    j = np.arange(off[-1]) - np.repeat(off[:-1], cnt)
    return np.repeat(bk, cnt), np.repeat(bv, cnt), sv[order[np.repeat(lo, cnt) + j]], off


def test_ten_million_big_rows_with_a_hot_small_key_match_numpy(spy):
    """1e7 big x 1e5 small int64 rows, keys uniform over [0, 2^22), plus one small key with 1e4 values that 1e3 big
    rows hit (1e7 of the output rows)."""
    rng = np.random.default_rng(7)
    nb, ns, hot = 10_000_000, 100_000, (1 << 40) + 3
    bk = rng.integers(0, 1 << 22, nb)
    sk = rng.integers(0, 1 << 22, ns)
    sk[rng.choice(ns, 10_000, replace=False)] = hot
    bk[rng.choice(nb, 1_000, replace=False)] = hot
    bv = rng.integers(-10 ** 9, 10 ** 9, nb)
    sv = rng.random(ns).astype(np.float32)
    dc = cc.ctx()
    big = dc.parallelizeColumns(torch.from_numpy(bk).cuda(), torch.from_numpy(bv).cuda(), 16)
    small = dc.parallelizeColumns(torch.from_numpy(sk).cuda(), torch.from_numpy(sv).cuda(), 8)
    out = big.innerJoin(small)
    wk, wl, wr, off = _numpy_inner_join(bk, bv, sk, sv)
    assert len(wk) > 10_000_000
    for sp, bsp in zip(out.splits, big.splits):
        keys, left, right = (c.cpu().numpy() for c in out.columns(sp))
        a, b = off[bsp.begin], off[bsp.end]
        assert np.array_equal(keys, wk[a:b]) and np.array_equal(left, wl[a:b]), sp.index
        assert right.dtype == np.float32 and np.array_equal(right.view(np.uint32), wr[a:b].view(np.uint32)), sp.index
    assert spy == {"group": 1, "build": 1, "probe": 1, "emit": 1}


# ------------------------------------------------------------------------------------------------ spies, fallback
def test_the_device_path_launches_the_three_kernels_once(spy):
    from dpark_b200 import _native as nv
    dc = cc.ctx()
    big = dc.parallelizeColumns(np.array([5, 1, 5, -0.0, 0.0, np.nan]), np.array([4, 9, 2, 7, 1, 3], np.int32), 2)
    small = dc.parallelizeColumns(np.array([0.0, 5.0, np.nan, 5.0], np.float32), np.array([10, 20, 30, 40]), 3)
    before = nv.launch_count()
    out = big.innerJoin(small)
    assert nv.launch_count() == before                  # nothing at construction
    assert repr(out.collect()) == repr([(5.0, (4, 20)), (5.0, (4, 40)), (5.0, (2, 20)), (5.0, (2, 40)),
                                        (-0.0, (7, 10)), (0.0, (1, 10))])
    assert nv.launch_count() > before
    launched = nv.launch_count()
    out.collect()                                        # materialised once
    assert nv.launch_count() == launched
    assert spy == {"group": 1, "build": 1, "probe": 1, "emit": 1}


def test_mixed_int_and_float_keys_fall_back(spy):
    from dpark_b200.rdd import FlatMappedRDD
    dc = cc.ctx()
    ints = dc.parallelizeColumns(torch.arange(6, device="cuda"), torch.arange(6, device="cuda"), 2)
    floats = dc.parallelizeColumns(torch.arange(6.0, device="cuda") * 0.5, torch.arange(6, device="cuda"), 2)
    out = ints.innerJoin(floats)
    assert isinstance(out, FlatMappedRDD)
    assert out.collect() == [(0, (0, 0)), (1, (1, 2)), (2, (2, 4))]
    assert spy == {"group": 0, "build": 0, "probe": 0, "emit": 0}
