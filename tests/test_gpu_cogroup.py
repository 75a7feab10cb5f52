"""The device cogroup of numeric ColumnarRDDs (dpark_b200/join.py) and groupByKey of one: against the reference's
golden cases, against the row path (the same rows through ctx.parallelize, which runs CoGroupedRDD / the row-id
group-by), and at scale against the oracle's group-by of the tagged union split by id range in numpy."""
import json

import numpy as np
import pytest
import torch

from tests import cogroup_common as cc
from tests.golden_util import dec, load

pytestmark = pytest.mark.gpu

KEY_DTYPES = [torch.int32, torch.int64, torch.float32, torch.float64]
VAL_DTYPES = [torch.int64, torch.float32, torch.int32, torch.float64]


def _cogrouped_cls():
    from dpark_b200.join import ColumnarCoGroupedRDD
    return ColumnarCoGroupedRDD


@pytest.fixture
def group_spy(monkeypatch):
    """Counts the groupByKeys that ran on the device cogroup; the row-id group-by must not run."""
    from dpark_b200 import engine
    calls = []
    real = engine._run_group_columns

    def columns(*args):
        calls.append(args[1])
        return real(*args)

    def rows(*args):
        raise AssertionError("groupByKey of a numeric ColumnarRDD took the row path")

    monkeypatch.setattr(engine, "_run_group_columns", columns)
    monkeypatch.setattr(engine, "_run_group", rows)
    return calls


# ------------------------------------------------------------------------------------------------ golden
INT_COGROUP_CASES = [c for c in cc.COGROUP_CASES if c["op"] == "cogroup" and c["name"] != "str_keys"]


@pytest.mark.parametrize("case", INT_COGROUP_CASES, ids=[c["name"] for c in INT_COGROUP_CASES])
def test_golden_cogroup_cases_on_the_device(case):
    dc = cc.ctx()
    rdds = [dc.parallelizeColumns(np.array([dec(k) for k, _ in inp["rows"]], dtype=np.int64),
                                  np.array([dec(v) for _, v in inp["rows"]], dtype=np.int64), inp["M"])
            for inp in case["inputs"]]
    out = rdds[0].groupWith(rdds[1:], case["P"], fixSkew=case.get("fixSkew", -1))
    assert isinstance(out, _cogrouped_cls())
    if case.get("thresholds") is not None:
        assert out.partitioner.thresholds == case["thresholds"]
    parts = out.glom().collect()
    got = [sorted(([cc._enc(k), [cc._enc(list(g)) for g in groups]] for k, groups in part), key=json.dumps)
           for part in parts]
    assert got == case["parts"]
    assert all(isinstance(groups, tuple) and len(groups) == len(rdds) for part in parts for _, groups in part)


SC = load("shuffle_cases.json")
INT_GROUP_CASES = [c for c in SC["cases"] if c["op"] == "groupByKey" and c["name"] != "group_str"]


@pytest.mark.parametrize("case", INT_GROUP_CASES, ids=[c["name"] for c in INT_GROUP_CASES])
def test_golden_group_by_key_cases_on_the_device(case, group_spy):
    from tests.golden.make_golden import enc
    dc = cc.ctx()
    rows = [(dec(k), dec(v)) for k, v in case["rows"]]
    col = dc.parallelizeColumns(np.array([k for k, _ in rows], dtype=np.int64),
                                np.array([v for _, v in rows], dtype=np.int64), case["M"])
    got = col.groupByKey(case["P"]).glom().collect()
    assert group_spy == [case["P"]]
    assert [sorted(([enc(k), enc(list(v))] for k, v in part), key=json.dumps) for part in got] == case["parts"]


# ------------------------------------------------------------------------------------------------ identity
def _keys(rng, dtype, lo, hi, n):
    if dtype.is_floating_point:
        k = rng.integers(lo, hi, n).astype(np.float64) * 0.5
        if n:
            k[rng.random(n) < 0.2] = -0.0
            k[rng.random(n) < 0.1] = 0.0
    else:
        k = rng.integers(lo, hi, n)
    return torch.from_numpy(k).to(dtype)


def _vals(rng, dtype, n):
    v = rng.integers(-1000, 1000, n)
    if dtype.is_floating_point:
        v = v * 0.25
        v[rng.random(n) < 0.05] = -0.0            # a value keeps its sign on both paths
    return torch.from_numpy(v).to(dtype)


# name: per input t of N -> (rows, key range, M); then P, fixSkew
SHAPES = {
    "partial_overlap": (lambda t, N: (200, (30 * t, 30 * t + 60), 2 + t % 3), 5, -1),
    "no_overlap": (lambda t, N: (80, (100 * t, 100 * t + 40), 3), 4, -1),
    "one_empty": (lambda t, N: (0 if t == N // 2 else 90, (0, 30), 2 + t), 4, -1),
    "all_empty": (lambda t, N: (0, (0, 1), 2), 3, -1),
    "fewer_rows_than_splits": (lambda t, N: (3 - t % 2, (0, 4), 5), 3, -1),
    "one_partition": (lambda t, N: (150, (0, 50), 4 - t % 2), 1, -1),
    "p4095": (lambda t, N: (300, (-100, 100), 3 + t), 4095, -1),
    "signed_zeros": (lambda t, N: (120, (-2, 3), 3), 3, -1),
    "fix_skew": (lambda t, N: (300, (0, 40), 3 - t % 2), 4, 1),
    "hot_key": (lambda t, N: (300, (0, 50), 4), 4, -1),
}


def _inputs(dc, rng, N, kdt, vdts, shape):
    spec, P, skew = SHAPES[shape]
    rdds = []
    for t in range(N):
        n, (lo, hi), M = spec(t, N)
        k, v = _keys(rng, kdt, lo, hi, n), _vals(rng, vdts[t % len(vdts)], n)
        if shape == "hot_key":                     # one key of 5000 rows on input 0 and 700 on the others
            h = 5000 if t == 0 else 700
            k = torch.cat([k, torch.full((h,), 7, dtype=kdt)])[torch.from_numpy(rng.permutation(n + h))]
            v = torch.cat([v, _vals(rng, v.dtype, h)])
        rdds.append(dc.parallelizeColumns(k, v, M))
    return rdds, P, skew


def _as_rows(dc, rdds):
    return [dc.parallelize(r.collect(), len(r.splits)) for r in rdds]


def _check_identity(N, kdt, vdts, shape, seed=0):
    rng = np.random.default_rng(seed)
    dc = cc.ctx()
    rdds, P, skew = _inputs(dc, rng, N, kdt, vdts, shape)
    out = rdds[0].groupWith(rdds[1:], P, fixSkew=skew)
    assert isinstance(out, _cogrouped_cls())
    rows = _as_rows(dc, rdds)
    want = rows[0].groupWith(rows[1:], P, fixSkew=skew).glom().collect()
    got = out.glom().collect()
    assert len(got) == len(want) == P
    assert got == want
    assert repr(got) == repr(want)          # also the spelling of every float: 0.0, never -0.0 as a key
    return got


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("kdt", KEY_DTYPES, ids=str)
@pytest.mark.parametrize("N", [1, 2, 3, 4])
def test_device_cogroup_equals_the_row_path(N, kdt, shape):
    i = sorted(SHAPES).index(shape)
    got = _check_identity(N, kdt, VAL_DTYPES[i % 4:] + VAL_DTYPES[:i % 4], shape)
    if shape in ("partial_overlap", "hot_key"):
        assert any(len(p) for p in got)
    if shape == "all_empty":
        assert not any(len(p) for p in got)


@pytest.mark.parametrize("rot", range(4))
@pytest.mark.parametrize("kdt", KEY_DTYPES, ids=str)
def test_device_cogroup_equals_the_row_path_for_value_dtypes(kdt, rot):
    _check_identity(4, kdt, VAL_DTYPES[rot:] + VAL_DTYPES[:rot], "partial_overlap", seed=7)


OPS = {
    "groupByKey": lambda a, b, P: a.groupByKey(P),
    "groupByKey_fixSkew": lambda a, b, P: a.groupByKey(P, fixSkew=1),
    "topByKey": lambda a, b, P: a.topByKey(2, num_splits=P),
    "topByKey_reverse": lambda a, b, P: a.topByKey(3, order_func=lambda v: -v, reverse=True, num_splits=P),
    "partitionByKey": lambda a, b, P: a.partitionByKey(P),
    "update": lambda a, b, P: a.update(b, numSplits=P),
    "update_replace_only": lambda a, b, P: a.update(b, replace_only=True, numSplits=P),
}


@pytest.mark.parametrize("op", sorted(OPS))
@pytest.mark.parametrize("kdt", KEY_DTYPES, ids=str)
def test_grouping_operators_of_columnar_rdds_equal_the_row_path(op, kdt):
    rng = np.random.default_rng(3)
    dc = cc.ctx()
    (a, b), P, _ = _inputs(dc, rng, 2, kdt, [torch.float32, torch.int32], "partial_overlap")
    ra, rb = _as_rows(dc, [a, b])
    got = OPS[op](a, b, P).glom().collect()
    want = OPS[op](ra, rb, P).glom().collect()
    assert got == want and repr(got) == repr(want)
    assert any(len(p) for p in got)


def test_group_by_key_of_a_columnar_rdd_runs_on_the_device(group_spy):
    from dpark_b200.rdd import ShuffledRDD
    dc = cc.ctx()
    col = dc.parallelizeColumns(np.array([3, 1, 3, -0.0, 0.0]), np.array([1, 2, 3, 4, 5], np.float32), 2)
    g = col.groupByKey(2)
    assert type(g) is ShuffledRDD
    got = sorted(g.collect())
    assert repr(got) == repr([(0.0, [4.0, 5.0]), (1.0, [2.0]), (3.0, [1.0, 3.0])])
    keys, vals = g.columns(g.splits[0])                  # host lists, as the row path hands them out
    assert isinstance(keys, list) and all(isinstance(v, list) for v in vals)
    assert group_spy == [2]


def test_columns_of_the_device_cogroup():
    dc = cc.ctx()
    a = dc.parallelizeColumns(np.array([1, 2, 2, 3], np.int32), np.array([10, 20, 21, 30], np.float32), 2)
    b = dc.parallelizeColumns(np.array([2, 4], np.int64), np.array([5, 6], np.int32), 1)
    c = dc.parallelizeColumns(np.array([], np.int64), np.array([], np.float64), 1)
    out = a.groupWith([b, c], 1)
    keys, offsets, values = out.columns(out.splits[0])
    assert all(t.is_cuda for t in (keys, offsets) + values)
    assert (keys.dtype, offsets.dtype) == (torch.int64, torch.int64)
    assert [v.dtype for v in values] == [torch.float32, torch.int32, torch.float64]
    assert offsets.shape == (3, 5) and offsets[:, 0].tolist() == [0, 0, 0]
    ks = keys.tolist()
    assert sorted(ks) == [1, 2, 3, 4]
    want = {1: ([10.0], [], []), 2: ([20.0, 21.0], [5], []), 3: ([30.0], [], []), 4: ([], [6], [])}
    for j, k in enumerate(ks):
        assert tuple(values[t][offsets[t, j]:offsets[t, j + 1]].tolist() for t in range(3)) == want[k]
    rows = list(out.compute(out.splits[0]))
    ra, rb, rc = _as_rows(dc, [a, b, c])
    assert rows == ra.groupWith([rb, rc], 1).collect()
    assert [k for k, _ in rows] == ks


# ------------------------------------------------------------------------------------------------ errors
def _raises_on_both_paths(rdds, P=3):
    dc = rdds[0].ctx
    assert isinstance(rdds[0].groupWith(rdds[1:], P), _cogrouped_cls())
    with pytest.raises(TypeError):
        rdds[0].groupWith(rdds[1:], P).collect()
    rows = _as_rows(dc, rdds)
    with pytest.raises(TypeError):
        rows[0].groupWith(rows[1:], P).collect()


@pytest.mark.parametrize("pos", [0, 1, 2])
def test_nan_keys_raise_type_error(pos):
    dc = cc.ctx()
    rdds = [dc.parallelizeColumns(np.array([1.0, 2.0]), np.array([1, 2]), 2) for _ in range(3)]
    rdds[pos] = dc.parallelizeColumns(np.array([1.0, float("nan"), 2.0], np.float32), np.arange(3), 2)
    _raises_on_both_paths(rdds)


def test_nan_keys_raise_type_error_in_group_by_key():
    dc = cc.ctx()
    k, v = np.array([1.0, float("nan")]), np.arange(2)
    with pytest.raises(TypeError):
        dc.parallelizeColumns(k, v, 1).groupByKey(2).collect()
    with pytest.raises(TypeError):
        dc.parallelize(list(zip(k.tolist(), v.tolist())), 1).groupByKey(2).collect()


@pytest.mark.parametrize("pos", [0, 1, 2])
def test_int_keys_grouped_with_float_keys_raise_type_error(pos):
    dc = cc.ctx()
    rdds = [dc.parallelizeColumns(np.array([1, 2, 3], np.int32), np.arange(3), 2) for _ in range(3)]
    rdds[pos] = dc.parallelizeColumns(np.array([1.0, 2.5], np.float64), np.arange(2), 1)
    _raises_on_both_paths(rdds)


# ------------------------------------------------------------------------------------------------ scale
def _by_key(keys, counts, vals):
    """Rows (key, value) in key order, each key's values in their given order: a layout-independent view of a CSR."""
    rk = np.repeat(keys, counts)
    order = np.argsort(rk, kind="stable")
    return rk[order], vals[order]


def test_cogroup_at_scale_with_a_hot_key_matches_the_oracle():
    """1e7 + 1e6 + 1e6 int64 rows plus one key with 2e6 + 5e5 + 5e5 rows, read through columns(), against the
    oracle's group-by of the tagged union split by id range: per partition the same keys and, per key and input, the
    same values in the same order."""
    from oracle import oracle as orc
    rng = np.random.default_rng(11)
    base, hot, M, P = (10_000_000, 1_000_000, 1_000_000), (2_000_000, 500_000, 500_000), 8, 16
    hot_key = (1 << 24) + 7
    ks, vs = [], []
    for t in range(3):
        k = np.concatenate([rng.integers(0, 1 << 24, base[t]), np.full(hot[t], hot_key)])
        ks.append(k[rng.permutation(len(k))])
        vs.append(rng.integers(-2 ** 62, 2 ** 62, len(k)) if t != 1 else rng.standard_normal(len(k)).astype(np.float32))
    dc = cc.ctx()
    rdds = [dc.parallelizeColumns(torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(), M) for k, v in zip(ks, vs)]
    out = rdds[0].groupWith(rdds[1:], P)
    assert isinstance(out, _cogrouped_cls())
    got = []
    for sp in out.splits:
        keys, offsets, values = out.columns(sp)
        got.append((keys.cpu().numpy(), offsets.cpu().numpy(), [v.cpu().numpy() for v in values]))
    torch.cuda.synchronize()

    bounds = np.concatenate([[0], np.cumsum([len(k) for k in ks])])
    ids = np.arange(bounds[-1], dtype=np.int64)
    ksp = [k[sp.begin:sp.end] for k, r in zip(ks, rdds) for sp in r.splits]
    isp = [ids[bounds[t] + sp.begin:bounds[t] + sp.end] for t, r in enumerate(rdds) for sp in r.splits]
    total = 0
    for p, (gk, off, ov) in enumerate(orc.group_by_key(ksp, isp, P)):
        keys, offsets, values = got[p]
        assert len(keys) == len(gk)
        tag = np.searchsorted(bounds, ov, side="right") - 1
        grp = np.repeat(np.arange(len(gk)), np.diff(off))
        for t in range(3):
            mine = tag == t
            wcount = np.bincount(grp[mine], minlength=len(gk))
            wk, wv = _by_key(gk, wcount, vs[t][ov[mine] - bounds[t]])
            gk_t, gv = _by_key(keys, np.diff(offsets[t]), values[t])
            assert np.array_equal(gk_t, wk) and np.array_equal(gv, wv), (p, t)
            total += len(gv)
        assert np.array_equal(np.sort(keys), np.sort(gk))
    assert total == bounds[-1]


def test_group_by_key_at_scale_matches_the_oracle(group_spy):
    """1e7 int64 rows over 2^16 keys: the host lists of every partition against the oracle's ordered group-by."""
    from oracle import oracle as orc
    rng = np.random.default_rng(5)
    n, M, P = 10_000_000, 8, 16
    k = rng.integers(-(1 << 15), 1 << 15, n)
    v = rng.integers(-2 ** 40, 2 ** 40, n)
    dc = cc.ctx()
    col = dc.parallelizeColumns(torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(), M)
    g = col.groupByKey(P)
    sizes = [(sp.begin, sp.end) for sp in col.splits]
    want = orc.group_by_key([k[b:e] for b, e in sizes], [v[b:e] for b, e in sizes], P)
    for p, sp in enumerate(g.splits):
        keys, lists = g.columns(sp)
        wk, woff, wv = want[p]
        gk, gv = _by_key(np.array(keys, np.int64), [len(x) for x in lists],
                         np.array([x for xs in lists for x in xs], np.int64))
        ek, ev = _by_key(wk, np.diff(woff), wv)
        assert np.array_equal(gk, ek) and np.array_equal(gv, ev), p
    assert group_spy == [P]
