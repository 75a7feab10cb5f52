"""The device join of two numeric ColumnarRDDs (dpark_b200/join.py) against the reference's golden cases, against the
row path (the same rows through ctx.parallelize, which RDD._join runs as cogroup + flatMap), and at scale against the
oracle's group-by of the tagged union expanded in numpy."""
import json
import math

import numpy as np
import pytest
import torch

from tests import cogroup_common as cc
from tests.golden_util import dec

pytestmark = pytest.mark.gpu

KINDS = ["join", "leftOuterJoin", "rightOuterJoin", "outerJoin"]
KEY_DTYPES = [torch.int32, torch.int64, torch.float32, torch.float64]
VAL_PAIRS = [(torch.int64, torch.int64), (torch.int32, torch.float64), (torch.float32, torch.int32),
             (torch.float64, torch.float32)]


def _joined_cls():
    from dpark_b200.join import ColumnarJoinedRDD
    return ColumnarJoinedRDD


@pytest.mark.parametrize("case", cc.JOIN_CASES, ids=[c["name"] for c in cc.JOIN_CASES])
def test_golden_join_cases_on_the_device(case):
    dc = cc.ctx()
    a, b = [dc.parallelizeColumns(np.array([dec(k) for k, _ in inp["rows"]], dtype=np.int64),
                                  np.array([dec(v) for _, v in inp["rows"]], dtype=np.int64), inp["M"])
            for inp in case["inputs"]]
    out = getattr(a, case["op"])(b, case["P"])
    assert isinstance(out, _joined_cls())
    parts = out.glom().collect()
    got = [sorted(([cc._enc(k), cc._enc(tuple(v))] for k, v in part), key=json.dumps) for part in parts]
    assert got == case["parts"]


# ------------------------------------------------------------------------------------------------ identity
def _keys(rng, dtype, lo, hi, n, signed_zero):
    if dtype.is_floating_point:
        k = rng.integers(lo, hi, n).astype(np.float64) * 0.5
        if signed_zero and n:
            k[rng.random(n) < 0.2] = -0.0
            k[rng.random(n) < 0.1] = 0.0
    else:
        k = rng.integers(lo, hi, n)
    return torch.from_numpy(k).to(dtype)


def _vals(rng, dtype, n):
    v = rng.integers(-1000, 1000, n)
    return torch.from_numpy(v * 0.25 if dtype.is_floating_point else v).to(dtype)


# name: (left rows, left key range, right rows, right key range, left M, right M, P, fixSkew)
SHAPES = {
    "partial_overlap": (300, (0, 60), 200, (30, 90), 3, 4, 5, -1),
    "no_overlap": (120, (0, 40), 80, (100, 140), 2, 3, 4, -1),
    "left_empty": (0, (0, 1), 90, (0, 30), 3, 2, 4, -1),
    "right_empty": (90, (0, 30), 0, (0, 1), 2, 3, 4, -1),
    "fewer_rows_than_splits": (3, (0, 4), 2, (2, 6), 5, 4, 3, -1),
    "one_partition": (200, (0, 50), 150, (25, 75), 4, 3, 1, -1),
    "p4095": (400, (-100, 100), 300, (-50, 150), 3, 5, 4095, -1),
    "fix_skew": (300, (0, 40), 200, (20, 60), 3, 2, 4, 1),
}


def _check_identity(kind, kdt, ldt, rdt, shape, seed=0):
    nl, lr, nr, rr, ml, mr, P, skew = SHAPES[shape]
    rng = np.random.default_rng(seed)
    dc = cc.ctx()
    a = dc.parallelizeColumns(_keys(rng, kdt, lr[0], lr[1], nl, True), _vals(rng, ldt, nl), ml)
    b = dc.parallelizeColumns(_keys(rng, kdt, rr[0], rr[1], nr, True), _vals(rng, rdt, nr), mr)
    out = getattr(a, kind)(b, P, fixSkew=skew)
    assert isinstance(out, _joined_cls())
    rows_a, rows_b = dc.parallelize(a.collect(), ml), dc.parallelize(b.collect(), mr)
    want = getattr(rows_a, kind)(rows_b, P, fixSkew=skew).glom().collect()
    got = out.glom().collect()
    assert len(got) == len(want)
    assert got == want
    assert repr(got) == repr(want)          # also the spelling of every float: 0.0, never -0.0
    return got


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("kdt", KEY_DTYPES, ids=str)
@pytest.mark.parametrize("kind", KINDS)
def test_device_join_equals_the_row_path(kind, kdt, shape):
    ldt, rdt = VAL_PAIRS[sorted(SHAPES).index(shape) % len(VAL_PAIRS)]
    got = _check_identity(kind, kdt, ldt, rdt, shape)
    if shape == "partial_overlap":
        assert any(len(p) for p in got)


@pytest.mark.parametrize("vals", VAL_PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("kdt", KEY_DTYPES, ids=str)
@pytest.mark.parametrize("kind", KINDS)
def test_device_join_equals_the_row_path_for_value_dtypes(kind, kdt, vals):
    _check_identity(kind, kdt, vals[0], vals[1], "partial_overlap", seed=7)


@pytest.mark.parametrize("kind", KINDS)
def test_columns_of_the_device_join(kind):
    dc = cc.ctx()
    a = dc.parallelizeColumns(np.array([1, 2, 2, 3], np.int32), np.array([10, 20, 21, 30], np.float32), 2)
    b = dc.parallelizeColumns(np.array([2, 4], np.int64), np.array([5, 6], np.int32), 1)
    out = getattr(a, kind)(b, 1)
    keys, left, right, lvalid, rvalid = out.columns(out.splits[0])
    assert all(t.is_cuda for t in (keys, left, right))
    assert (keys.dtype, left.dtype, right.dtype) == (torch.int64, torch.float32, torch.int32)
    assert (lvalid is None) == (kind in ("join", "leftOuterJoin"))
    assert (rvalid is None) == (kind in ("join", "rightOuterJoin"))
    for valid, vals in ((lvalid, left), (rvalid, right)):
        if valid is not None:
            assert valid.dtype == torch.uint8
            assert bool((vals[valid == 0] == 0).all())        # a missing side's slot holds 0
    rows = list(out.compute(out.splits[0]))
    want = getattr(dc.parallelize(a.collect(), 2), kind)(dc.parallelize(b.collect(), 1), 1).collect()
    assert rows == want


# ------------------------------------------------------------------------------------------------ errors
def _raises_on_both_paths(a, b, kind, P=3):
    dc = a.ctx
    assert isinstance(getattr(a, kind)(b, P), _joined_cls())
    with pytest.raises(TypeError):
        getattr(a, kind)(b, P).collect()
    rows_a = dc.parallelize(a.collect(), len(a.splits))
    rows_b = dc.parallelize(b.collect(), len(b.splits))
    with pytest.raises(TypeError):
        getattr(rows_a, kind)(rows_b, P).collect()


@pytest.mark.parametrize("side", ["left", "right"])
@pytest.mark.parametrize("kind", KINDS)
def test_nan_keys_raise_type_error(kind, side):
    dc = cc.ctx()
    k = np.array([1.0, float("nan"), 2.0])
    good = dc.parallelizeColumns(np.array([1.0, 2.0]), np.array([1, 2]), 2)
    bad = dc.parallelizeColumns(k, np.arange(3), 2)
    a, b = (bad, good) if side == "left" else (good, bad)
    _raises_on_both_paths(a, b, kind)


@pytest.mark.parametrize("kind", KINDS)
def test_int_keys_joined_with_float_keys_raise_type_error(kind):
    dc = cc.ctx()
    a = dc.parallelizeColumns(np.array([1, 2, 3], np.int64), np.arange(3), 2)
    b = dc.parallelizeColumns(np.array([1.0, 2.5], np.float32), np.arange(2), 1)
    _raises_on_both_paths(a, b, kind)
    _raises_on_both_paths(b, a, kind)


# ------------------------------------------------------------------------------------------------ scale
def test_join_at_scale_with_a_hot_key_matches_the_oracle():
    """1e7 x 1e6 int64 rows plus one key with 3000 rows on each side (9e6 output rows from one key), read through
    columns(), against the oracle's group-by of the tagged union expanded in numpy: per partition the same
    (key, left, right) rows, in row-path order inside every key."""
    from oracle import oracle as orc
    rng = np.random.default_rng(11)
    nL0, nR0, hot, M, P = 10_000_000, 1_000_000, 3000, 8, 16
    hot_key = (1 << 24) + 7
    lk = np.concatenate([rng.integers(0, 1 << 24, nL0), np.full(hot, hot_key)])
    rk = np.concatenate([rng.integers(0, 1 << 24, nR0), np.full(hot, hot_key)])
    lk, rk = lk[rng.permutation(len(lk))], rk[rng.permutation(len(rk))]
    lv = rng.integers(-2 ** 62, 2 ** 62, len(lk))
    rv = rng.standard_normal(len(rk)).astype(np.float32)
    nL = len(lk)
    dc = cc.ctx()
    a = dc.parallelizeColumns(torch.from_numpy(lk).cuda(), torch.from_numpy(lv).cuda(), M)
    b = dc.parallelizeColumns(torch.from_numpy(rk).cuda(), torch.from_numpy(rv).cuda(), M)
    out = a.join(b, P)
    assert isinstance(out, _joined_cls())
    got = [[c.cpu().numpy() for c in out.columns(sp)[:3]] for sp in out.splits]
    torch.cuda.synchronize()

    # the oracle: map tasks over the left splits, then the right splits, carrying row ids
    ids = np.arange(nL + len(rk), dtype=np.int64)
    ksp = [lk[sp.begin:sp.end] for sp in a.splits] + [rk[sp.begin:sp.end] for sp in b.splits]
    isp = [ids[sp.begin:sp.end] for sp in a.splits] + [ids[nL + sp.begin:nL + sp.end] for sp in b.splits]
    total = 0
    for p, (gk, off, ov) in enumerate(orc.group_by_key(ksp, isp, P)):
        isl = (ov < nL).astype(np.int64)
        cl = np.concatenate([[0], np.cumsum(isl)])
        nl = cl[off[1:]] - cl[off[:-1]]
        nr = np.diff(off) - nl
        cnt = nl * nr
        G, N = len(gk), int(cnt.sum())
        total += N
        g = np.repeat(np.arange(G), cnt)
        local = np.arange(N) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        R = nr[g]
        ai, bi = local // np.maximum(R, 1), local % np.maximum(R, 1)
        want = (gk[g], lv[ov[off[g] + ai]], rv[ov[off[g] + nl[g] + bi] - nL])
        order = np.argsort(got[p][0], kind="stable")
        worder = np.argsort(want[0], kind="stable")
        for x, y in zip(got[p], want):
            assert len(x) == len(y)
            assert np.array_equal(x[order], y[worder]), p
    assert sum(len(g[0]) for g in got) == total
    assert total >= hot * hot


def test_hot_key_alone_spreads_over_many_tiles():
    """One key with 3000 x 3000 rows and nothing else: every output row, left-major."""
    dc = cc.ctx()
    n = 3000
    a = dc.parallelizeColumns(torch.full((n,), 5, dtype=torch.int64), torch.arange(n, dtype=torch.int32), 4)
    b = dc.parallelizeColumns(torch.full((n,), 5, dtype=torch.int64), torch.arange(n, dtype=torch.float64), 3)
    out = a.outerJoin(b, 2)
    cols = [out.columns(sp) for sp in out.splits]
    keys, left, right, lvalid, rvalid = [c for c in cols if c[0].numel()][0]
    assert keys.numel() == n * n and sum(c[0].numel() for c in cols) == n * n
    assert bool((keys == 5).all()) and bool(lvalid.all()) and bool(rvalid.all())
    idx = torch.arange(n * n, device=keys.device)
    assert torch.equal(left.long(), idx // n)
    assert torch.equal(right, (idx % n).double())
    assert math.isclose(float(right.sum()), n * n * (n - 1) / 2)
