"""Oracle parity of the host-buffer entry points: `shuffle.HostShuffle.run` and `shuffle.HostShuffleStream.submit /
collect` (kind "reduce" and "group", depth 1, 2 and 3), over every key and value kind, every op, with and without
fixSkew thresholds, map-side combine, empty and tiny inputs, and batches of 2^24 rows whose slots overlap.  -m gpu.

References, neither sharing device code with the library:
  * up to a few 10^4 rows, the pure-Python restatement of the reference's loops (oracle.py_reduce_by_key /
    py_group_by_key over Python ints and floats, placed by portable_hash);
  * at 2^24 rows, the oracle's C loops (oracle.reduce_by_key / group_by_key).
Reduce partitions compare as sets of (key, value) rows: integer values and float min/max bit for bit, float prod to
rtol 1e-12, float sums to 1e-9 * sum|v| of the key (DESIGN.md §7).  Integer results are Python's wrapped to int64.
Group partitions compare their keys as sets, each key's values exactly, in (map split, position) order.  Float keys
compare by the bits of their canonical float64: -0.0 and 0.0 are one Python dict key, spelled 0.0 on the device.

Mutations of dpark_b200/shuffle.py this file catches and tests/test_gpu_host_api.py does not, each tried once:
  * `_collect_group` cutting partitions one group late (searchsorted(..., right=True) for `first`);
  * dropping the `+ 0.0` of float group keys (-0.0 and 0.0 become two groups);
  * every slot sharing one set of pinned output buffers (a result changes before its slot is collected again);
  * `d2h_bytes` of the group kind counting 8 bytes per value whatever the value dtype;
  * HostShuffle cutting its splits `n // splits` rows long (the last rows of an n not a multiple of splits lost);
  * HostShuffle.run partitioning without its thresholds.
Both files catch `collect()` not advancing `next_collect`.
"""
import itertools
import operator

import numpy as np
import pytest
import torch

from oracle import oracle as orc

pytestmark = pytest.mark.gpu

KINDS = ["i64", "i32", "f64", "f32"]
_NP = {"i64": np.int64, "i32": np.int32, "f64": np.float64, "f32": np.float32}
_TORCH = {"i64": torch.int64, "i32": torch.int32, "f64": torch.float64, "f32": torch.float32}
INT_OPS = ["sum", "min", "max", "prod", "and", "or", "xor"]
FLOAT_OPS = ["sum", "min", "max", "prod"]


def _wrap(x):
    return (x + 2 ** 63) % 2 ** 64 - 2 ** 63


_PYOP = {"sum": operator.add, "min": min, "max": max, "prod": operator.mul, "and": operator.and_,
         "or": operator.or_, "xor": operator.xor}


def _pyop(op, vk):
    f = _PYOP[op]
    if vk[0] == "i":                          # the device accumulates in int64: Python's result modulo 2^64
        return lambda a, b: _wrap(f(a, b))
    return f


def _combos():
    """(key kind, value kind, op): all seven ops for integer values, sum/min/max/prod for float values."""
    return [(kk, vk, op) for kk in KINDS for vk in KINDS for op in (INT_OPS if vk[0] == "i" else FLOAT_OPS)]


def _pairs(row):
    return {(i, row[i], j, row[j]) for i in range(len(row)) for j in range(i + 1, len(row))}


def _cover(combos, extra):
    """Every combo, each with the setting of the `extra` factors that covers the most pairs of factor values not yet
    covered (greedy, deterministic): every pair that can occur does."""
    seen, out = set(), []
    for c in combos:
        row = max((tuple(c) + e for e in itertools.product(*extra)), key=lambda r: len(_pairs(r) - seen))
        seen |= _pairs(row)
        out.append(row)
    return out


def _pairwise(rows):
    """A greedy covering array: rows of `rows` until every pair of factor values that occurs in `rows` is covered."""
    todo = set().union(*(_pairs(r) for r in rows))
    out = []
    while todo:
        best = max(rows, key=lambda r: len(_pairs(r) & todo))
        out.append(best)
        todo -= _pairs(best)
    return out


# ----------------------------------------------------------------------------------------------------- inputs
I64_EDGES = [-2 ** 63, 2 ** 63 - 1, -2 ** 31, 2 ** 31 - 1, -1, 0]
I32_EDGES = [-2 ** 31, 2 ** 31 - 1, -1, 0]
FLOAT_EDGES = [0.0, -0.0, np.inf, -np.inf, 5e-324, -5e-324, 1e-310, 2.0 ** -149, -(2.0 ** -149), 1e-40, 1.0]


def _keys(kind, n, rng, distinct, hot=True):
    """A key column of `kind` with about `distinct` distinct keys, the kind's edge values among them, and (hot) one
    key on a fifth of the rows, so that a fixSkew sample of it is skewed."""
    if kind[0] == "i":
        edges = I64_EDGES if kind == "i64" else I32_EDGES
        info = np.iinfo(_NP[kind])
        pool = np.concatenate([rng.integers(info.min, info.max, max(1, distinct // 2), dtype=np.int64, endpoint=True),
                               rng.integers(-distinct, distinct, max(1, distinct // 2)), edges]).astype(_NP[kind])
    else:
        rnd = rng.standard_normal(max(1, distinct)) * 10.0 ** rng.integers(-30, 30, max(1, distinct))
        pool = np.concatenate([rnd, FLOAT_EDGES]).astype(_NP[kind])
    k = pool[rng.integers(0, len(pool), n)]
    if n:
        k[: min(n, len(pool))] = pool[: min(n, len(pool))][::-1]          # every edge value occurs
        if hot:
            k[rng.random(n) < 0.2] = pool[0]
        rng.shuffle(k)
    return k


def _vals(kind, op, n, rng):
    if kind[0] == "i":
        if op == "prod":
            v = rng.integers(-3, 4, n)
        elif op in ("and", "or", "xor"):
            v = rng.integers(-2 ** 62, 2 ** 62, n) if kind == "i64" else rng.integers(-2 ** 31, 2 ** 31, n)
        else:
            v = rng.integers(-2 ** 31, 2 ** 31, n)
        return v.astype(_NP[kind])
    if op == "prod":
        return (rng.random(n) + 0.5).astype(_NP[kind])
    return (rng.standard_normal(n) * 1000.0).astype(_NP[kind])


def _zipf_keys(kind, n, rng, support=1.0e6, s=1.1):
    """Zipf(1.1) ranks by inverse CDF (bench.py's C3 column over a smaller support), permuted by an odd multiplier."""
    u = rng.random(n)
    r = np.clip(np.power(1.0 - u * (1.0 - support ** (1.0 - s)), 1.0 / (1.0 - s)), 1.0, support).astype(np.int64)
    r = (r * 0x9E3779B1) & 0x7FFFFFFF
    if kind == "i32":
        return (r - 2 ** 30).astype(np.int32)
    if kind[0] == "f":
        return ((r - 2 ** 30).astype(np.float64) * 0.25).astype(_NP[kind])
    return r


def _bounds(n, splits):
    per = (n + splits - 1) // splits
    return [(min(n, i * per), min(n, (i + 1) * per)) for i in range(splits)]


def _thresholds(keys, P, rng):
    """fixSkew's thresholds (quantiles.skew_thresholds: percentiles of the key hashes) from a sample of the keys, and
    the number of partitions they make."""
    sample = keys[rng.integers(0, len(keys), min(len(keys), 2000))]
    from dpark_b200 import quantiles
    thr, P2 = quantiles.skew_thresholds([orc.hash_vec(sample).tolist()], P)
    assert thr
    return thr, P2


def _pinned(a):
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory()


# ------------------------------------------------------------------------------------------------- references
def _kbits(a, canonical=True):
    """Keys as comparable int64: integers widened, floats by the bits of their float64 (canonical: + 0.0)."""
    a = np.asarray(a)
    if a.dtype.kind == "f":
        a = a.astype(np.float64)
        return (a + 0.0 if canonical else a).view(np.int64)
    return a.astype(np.int64)


def _rows(k, v, n, splits):
    ks, vs = k.tolist(), v.tolist()
    return [list(zip(ks[a:b], vs[a:b])) for a, b in _bounds(n, splits)]


def _sorted_reduce(kb, v, tol):
    o = np.argsort(kb, kind="stable")
    return kb[o], v[o], (None if tol is None else tol[o])


def py_reduce(k, v, splits, P, op, thr=None):
    """Per partition (key bits, values, sum|v| or None) sorted by key, from the pure-Python reduceByKey."""
    n, vk = len(k), ("f" if v.dtype.kind == "f" else "i")
    want = orc.py_reduce_by_key(_rows(k, v, n, splits), P, _pyop(op, vk), thr)
    tol = None
    if vk == "f" and op == "sum":
        tol = orc.py_reduce_by_key(_rows(k, np.abs(v.astype(np.float64)), n, splits), P, operator.add, thr)
    out = []
    for p in range(P):
        keys = list(want[p].keys())
        kb = _kbits(np.array(keys, dtype=np.float64 if k.dtype.kind == "f" else np.int64))
        vals = np.array([want[p][x] for x in keys], dtype=np.float64 if vk == "f" else np.int64)
        t = None if tol is None else np.array([tol[p][x] for x in keys], dtype=np.float64)
        out.append(_sorted_reduce(kb, vals, t))
    return out


def orc_reduce(k, v, P, op, tol_by_key=None):
    """The same from the oracle's C loops; tol_by_key: sum|v| indexed by key (non-negative int keys)."""
    out = []
    for wk, wv in orc.reduce_by_key([k], [v], P, op):
        out.append(_sorted_reduce(_kbits(wk), wv, None if tol_by_key is None else tol_by_key[wk]))
    return out


def check_reduce(parts, want, op, kdt, vdt):
    assert [p for p, _, _ in parts] == list(range(len(want)))
    for p, gk, gv in parts:
        assert gk.dtype == kdt and gv.dtype == (torch.float64 if vdt.is_floating_point else torch.int64)
        gb, gv = _sorted_reduce(_kbits(gk.numpy(), canonical=False), gv.numpy(), None)[:2]
        wb, wv, tol = want[p]
        assert np.array_equal(gb, wb), "partition %d: keys differ" % p
        if gv.dtype.kind != "f" or op in ("min", "max"):
            assert np.array_equal(gv.view(np.int64), wv.view(np.int64)), "partition %d: values differ" % p
        elif op == "prod":
            assert np.allclose(gv, wv, rtol=1e-12, atol=0), "partition %d: products differ" % p
        else:
            assert np.all(np.abs(gv - wv) <= 1e-9 * tol), "partition %d: sums differ beyond 1e-9 * sum|v|" % p


def _csr_sorted(kb, starts, vals):
    """(keys, run lengths, values run after run) with the groups sorted by key bits."""
    o = np.argsort(kb, kind="stable")
    lens = (starts[1:] - starts[:-1])[o]
    first = starts[:-1][o]
    at = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    idx = np.repeat(first - at, lens) + np.arange(int(lens.sum()), dtype=np.int64)
    return kb[o], lens, vals[idx]


def py_group(k, v, splits, P, thr=None):
    want = orc.py_group_by_key(_rows(k, v, len(k), splits), P, thr)
    out = []
    for p in range(P):
        keys = list(want[p].keys())
        kb = _kbits(np.array(keys, dtype=np.float64 if k.dtype.kind == "f" else np.int64))
        lens = np.array([len(want[p][x]) for x in keys], dtype=np.int64)
        starts = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        vals = np.array([y for x in keys for y in want[p][x]], dtype=v.dtype)
        out.append(_csr_sorted(kb, starts, vals))
    return out


def orc_group(k, v, P):
    """The oracle's C group-by over row ids, the values gathered by them (exact for every value kind)."""
    out = []
    for wk, wo, wid in orc.group_by_key([k], [np.arange(len(k), dtype=np.int64)], P):
        out.append(_csr_sorted(_kbits(wk), wo, v[wid[: wo[-1]]]))
    return out


def check_group(parts, want, kdt, vdt):
    assert [p for p, _, _, _ in parts] == list(range(len(want)))
    wide = torch.float64 if kdt.is_floating_point else torch.int64
    for p, gk, gs, gv in parts:
        assert gk.dtype == wide and gv.dtype == vdt and gs.numel() == gk.numel() + 1
        gb, glen, gval = _csr_sorted(_kbits(gk.numpy(), canonical=False), gs.numpy(), gv.numpy())
        wb, wlen, wval = want[p]
        assert np.array_equal(gb, wb), "partition %d: group keys differ" % p
        assert np.array_equal(glen, wlen), "partition %d: group sizes differ" % p
        assert gval.tobytes() == wval.tobytes(), "partition %d: value runs differ" % p


# ------------------------------------------------------------------------------------ 1. HostShuffle.run
RUN_CASES = _cover(_combos(), [(False, True), (False, True), (1, 3, 8)])     # + thresholds, map_combine, splits


@pytest.mark.parametrize("case", range(len(RUN_CASES)),
                         ids=["%s-%s-%s-thr%d-mc%d-s%d" % c for c in RUN_CASES])
def test_host_shuffle_run_matches_python_reference(case):
    """Two runs on one object: many distinct keys, then a batch of 6 distinct keys, so that rows left over in the
    reused pinned output buffers would show."""
    from dpark_b200 import shuffle
    kk, vk, op, use_thr, mc, splits = RUN_CASES[case]
    rng = np.random.default_rng(1000 + case)
    n = 4000 + 7 * case
    n += 1 if splits > 1 and n % splits == 0 else 0
    P = 5
    k1, v1 = _keys(kk, n, rng, n // 3), _vals(vk, op, n, rng)
    k2, v2 = rng.choice(_keys(kk, 64, rng, 6, hot=False)[:6], n), _vals(vk, op, n, rng)
    thr = None
    if use_thr:
        thr, P = _thresholds(k1, P, rng)
    hs = shuffle.HostShuffle(n, _TORCH[kk], _TORCH[vk], P, op, splits=splits, thresholds=thr, map_combine=mc)
    for k, v in ((k1, v1), (k2, v2)):
        hs.h_keys.copy_(torch.from_numpy(k))
        hs.h_vals.copy_(torch.from_numpy(v))
        parts = hs.run()
        want = py_reduce(k, v, splits, P, op, thr)
        check_reduce(parts, want, op, _TORCH[kk], _TORCH[vk])
        nout = sum(len(w[0]) for w in want)
        assert hs.h2d_bytes == n * (hs.h_keys.element_size() + hs.h_vals.element_size())
        assert hs.d2h_bytes == nout * (hs.h_keys.element_size() + 8)
    assert sum(len(w[0]) for w in want) <= 6


SMALL = [(s, n) for s in (1, 3, 8) for n in sorted({0, 1, s - 1, s + 1}) if n >= 0]


@pytest.mark.parametrize("splits,n", SMALL)
def test_host_shuffle_run_empty_and_tiny_inputs(splits, n):
    """n = 0, n = 1 and n below splits: the trailing splits of _bounds are empty."""
    from dpark_b200 import shuffle
    rng = np.random.default_rng(splits * 100 + n)
    for i, (kk, vk, op) in enumerate([("i64", "i64", "sum"), ("f32", "f32", "max"), ("i32", "f64", "min"),
                                      ("f64", "i32", "xor")]):
        k, v = _keys(kk, n, rng, 3, hot=False), _vals(vk, op, n, rng)
        hs = shuffle.HostShuffle(n, _TORCH[kk], _TORCH[vk], 3, op, splits=splits, map_combine=bool(i % 2))
        hs.h_keys.copy_(torch.from_numpy(k))
        hs.h_vals.copy_(torch.from_numpy(v))
        check_reduce(hs.run(), py_reduce(k, v, splits, 3, op), op, _TORCH[kk], _TORCH[vk])


# -------------------------------------------------------------------- 2./3. HostShuffleStream, both kinds
def _drive(st, batches, depth, pattern, check):
    """Submit every batch and collect every result, `fill` (submit depth, collect depth) or `alt` (keep the pipeline
    full: collect one, submit one).  After every collect(), check(parts, batch, fresh) runs on the result of the last
    `depth` collects, fresh for the one just returned: the older views must hold until their slot is collected again."""
    live, inflight = [], []

    def collect():
        b = inflight.pop(0)
        live.append((b, st.collect()))
        del live[:-depth]
        for bb, parts in live:
            check(parts, bb, bb == b)

    for b in range(len(batches)):
        if len(inflight) == depth:
            collect()
            while pattern == "fill" and inflight:
                collect()
        st.submit(*batches[b])
        inflight.append(b)
    while inflight:
        collect()


STREAM_REDUCE = _pairwise([(d, p, t) + c for d in (1, 2, 3) for p in ("fill", "alt") for t in (False, True)
                           for c in _combos()])


@pytest.mark.parametrize("case", range(len(STREAM_REDUCE)), ids=["d%d-%s-thr%d-%s-%s-%s" % c for c in STREAM_REDUCE])
def test_host_shuffle_stream_reduce_matches_python_reference(case):
    from dpark_b200 import shuffle
    depth, pattern, use_thr, kk, vk, op = STREAM_REDUCE[case]
    rng = np.random.default_rng(2000 + case)
    n, P, splits = 3001 + case, 4, 3
    data = []
    for b in range(2 * depth + 1):            # every batch differs, in the size of its key set too
        data.append((_keys(kk, n, rng, 50 + 400 * (b % 3)), _vals(vk, op, n, rng)))
    thr = None
    if use_thr:
        thr, P = _thresholds(data[0][0], P, rng)
    want = [py_reduce(k, v, splits, P, op, thr) for k, v in data]
    st = shuffle.HostShuffleStream(n, _TORCH[kk], _TORCH[vk], P, op, splits=splits, thresholds=thr, depth=depth)
    ksz, vsz = np.dtype(_NP[kk]).itemsize, np.dtype(_NP[vk]).itemsize

    def check(parts, b, fresh):
        check_reduce(parts, want[b], op, _TORCH[kk], _TORCH[vk])
        if fresh:
            assert st.d2h_bytes == sum(len(w[0]) for w in want[b]) * (ksz + 8)
    _drive(st, [(_pinned(k), _pinned(v)) for k, v in data], depth, pattern, check)
    assert st.h2d_bytes == n * (ksz + vsz)


STREAM_GROUP = _pairwise([(kk, vk, d, p, t, z) for kk in KINDS for vk in KINDS for d in (1, 2, 3)
                          for p in ("fill", "alt") for t in (False, True) for z in ("uniform", "zipf")])


@pytest.mark.parametrize("case", range(len(STREAM_GROUP)), ids=["%s-%s-d%d-%s-thr%d-%s" % c for c in STREAM_GROUP])
def test_host_shuffle_stream_group_matches_python_reference(case):
    """groupByKey through the stream: 4-byte keys are widened, float keys come back as canonical float64 (one group
    for -0.0 and 0.0), each key's values in (map split, position) order."""
    from dpark_b200 import shuffle
    kk, vk, depth, pattern, use_thr, dist = STREAM_GROUP[case]
    rng = np.random.default_rng(3000 + case)
    n, P, splits = 2501 + 2 * case, 4, 3
    data = []
    for b in range(2 * depth + 1):
        k = _zipf_keys(kk, n, rng) if dist == "zipf" else _keys(kk, n, rng, 30 + 300 * (b % 3))
        if kk[0] == "f":
            k[rng.integers(0, n, 40)] = rng.choice([0.0, -0.0], 40)
        data.append((k, _vals(vk, "sum", n, rng)))
    thr = None
    if use_thr:
        thr, P = _thresholds(data[0][0], P, rng)
    want = [py_group(k, v, splits, P, thr) for k, v in data]
    st = shuffle.HostShuffleStream(n, _TORCH[kk], _TORCH[vk], P, splits=splits, thresholds=thr, depth=depth,
                                   kind="group")
    vsz = np.dtype(_NP[vk]).itemsize

    def check(parts, b, fresh):
        check_group(parts, want[b], _TORCH[kk], _TORCH[vk])
        if fresh:
            G = sum(len(w[0]) for w in want[b])
            assert st.d2h_bytes == G * 8 + (G + 1) * 8 + n * vsz
    _drive(st, [(_pinned(k), _pinned(v)) for k, v in data], depth, pattern, check)


@pytest.mark.parametrize("kind", ["reduce", "group"])
@pytest.mark.parametrize("kk", KINDS)
def test_host_shuffle_stream_empty_and_tiny_batches(kind, kk):
    """n = 0, 1 and 5 rows over 8 splits: empty trailing splits, empty batches."""
    from dpark_b200 import shuffle
    rng = np.random.default_rng(KINDS.index(kk))
    for n in (0, 1, 5):
        data = [(_keys(kk, n, rng, 2, hot=False), _vals("i32", "sum", n, rng)) for _ in range(3)]
        st = shuffle.HostShuffleStream(n, _TORCH[kk], torch.int32, 3, splits=8, depth=2, kind=kind)
        if kind == "reduce":
            want = [py_reduce(k, v, 8, 3, "sum") for k, v in data]

            def check(parts, b, fresh):
                check_reduce(parts, want[b], "sum", _TORCH[kk], torch.int32)
        else:
            want = [py_group(k, v, 8, 3) for k, v in data]

            def check(parts, b, fresh):
                check_group(parts, want[b], _TORCH[kk], torch.int32)
        _drive(st, [(_pinned(k), _pinned(v)) for k, v in data], 2, "alt", check)


def _group_by_hand(k, v, splits):
    from dpark_b200 import shuffle
    st = shuffle.HostShuffleStream(len(k), torch.from_numpy(k).dtype, torch.int64, 1, splits=splits, depth=1,
                                   kind="group")
    st.submit(_pinned(k), _pinned(v))
    [(p, gk, gs, gv)] = st.collect()
    return gk, {x: gv[int(gs[i]):int(gs[i + 1])].tolist() for i, x in enumerate(gk.tolist())}


V7 = np.array([10, 11, 12, 13, 14, 15, 16], dtype=np.int64)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_host_shuffle_stream_group_float_keys_by_hand(dtype):
    """-0.0 and 0.0 are one key, spelled 0.0 and returned as float64; each key's values in (map split, position)
    order.  (7 rows: float32 keys read two at a time as int64 would raise before any launch.)"""
    gk, got = _group_by_hand(np.array([1.5, -0.0, 2.0, 0.0, 1.5, -0.0, 7.0], dtype=dtype), V7, 2)
    assert gk.numel() == 4, "-0.0 and 0.0 are one key"
    assert gk.dtype == torch.float64
    assert got == {1.5: [10, 14], 0.0: [11, 13, 15], 2.0: [12], 7.0: [16]}
    assert not np.signbit(gk.numpy()).any()


def test_host_shuffle_stream_group_int32_keys_by_hand():
    """int32 keys are grouped by value and come back as int64.  (5 rows: read two at a time as int64 they would
    raise before any launch.)"""
    gk, got = _group_by_hand(np.array([3, -2 ** 31, 3, 2 ** 31 - 1, -2 ** 31], dtype=np.int32), V7[:5], 3)
    assert gk.dtype == torch.int64
    assert got == {3: [10, 12], -2 ** 31: [11, 14], 2 ** 31 - 1: [13]}


# ----------------------------------------------------------------------------------------- 4. overlap at size
def _big_batch(shape, b, n):
    rng = np.random.default_rng(4000 + 10 * b + len(shape))
    if shape == "c2":
        return rng.integers(0, 2 ** 31, n, dtype=np.int64), rng.integers(0, 2 ** 16, n, dtype=np.int64)
    if shape == "c4":
        return rng.integers(0, 2 ** 24, n, dtype=np.int32), rng.random(n, dtype=np.float32)
    return _zipf_keys("i64", n, rng, support=1.0e9), np.arange(b * n, (b + 1) * n, dtype=np.int64)


def _own(parts):
    """Copies of the pinned views one collect() returned (the values column once, however many partitions share it)."""
    memo = {}

    def own(t):
        if (t.data_ptr(), t.numel()) not in memo:
            memo[(t.data_ptr(), t.numel())] = t.clone()
        return memo[(t.data_ptr(), t.numel())]
    return [(p,) + tuple(own(t) for t in ts) for p, *ts in parts]


@pytest.mark.parametrize("shape", ["c2", "c4", "c3"])
def test_host_shuffle_stream_depth3_overlapping_batches_of_2_24_rows(shape):
    """Four batches of 2^24 rows through three slots, the pinned inputs of the first batch rewritten with the fourth
    once the first is collected: submit 0, 1, 2; collect 0; submit 3; collect 1, 2, 3.  Every partition against the
    oracle's C loops.  C2: (int64, int64) sum, C4: (int32, float32) sum, C3: group of Zipf(1.1) int64 keys.  The
    references and the checks run on worker threads (the C loops and numpy's sorts release the GIL)."""
    from concurrent.futures import ThreadPoolExecutor

    from dpark_b200 import shuffle
    n, P, depth, nb = 1 << 24, 8, 3, 4
    kdt, vdt = {"c2": ("i64", "i64"), "c4": ("i32", "f32"), "c3": ("i64", "i64")}[shape]
    kind = "group" if shape == "c3" else "reduce"
    data = [_big_batch(shape, b, n) for b in range(nb)]

    def reference(k, v):
        if kind == "group":
            return orc_group(k, v, P)
        tol = np.bincount(k, np.abs(v.astype(np.float64)), 1 << 24) if shape == "c4" else None
        return orc_reduce(k, v, P, "sum", tol)

    def check(parts, want):
        if kind == "group":
            check_group(parts, want.result(), _TORCH[kdt], _TORCH[vdt])
        else:
            check_reduce(parts, want.result(), "sum", _TORCH[kdt], _TORCH[vdt])

    st = shuffle.HostShuffleStream(n, _TORCH[kdt], _TORCH[vdt], P, splits=8, depth=depth, kind=kind)
    host = [(torch.empty(n, dtype=_TORCH[kdt]).pin_memory(), torch.empty(n, dtype=_TORCH[vdt]).pin_memory())
            for _ in range(depth)]
    with ThreadPoolExecutor(6) as pool:
        want = [pool.submit(reference, k, v) for k, v in data]
        checks = []

        def submit(b):
            hk, hv = host[b % depth]
            hk.copy_(torch.from_numpy(data[b][0]))
            hv.copy_(torch.from_numpy(data[b][1]))
            st.submit(hk, hv)

        def collect(b):
            checks.append(pool.submit(check, _own(st.collect()), want[b]))

        for b in range(depth):
            submit(b)
        collect(0)
        submit(3)
        for b in (1, 2, 3):
            collect(b)
        for c in checks:
            c.result()


# ------------------------------------------------------------------------------------------------ 5. NaN keys
@pytest.mark.parametrize("kk", ["f64", "f32"])
def test_nan_keys_raise_type_error_in_both_entry_points(kk):
    """CPython hashes NaN by identity, so the engine refuses NaN keys (join.reject_nan_keys); so do the host entry
    points.  The object stays usable: the next batch gives the reference's result."""
    from dpark_b200 import shuffle
    rng = np.random.default_rng(5)
    n = 3000
    good_k, v = _keys(kk, n, rng, 100), _vals("i64", "sum", n, rng)
    bad_k = good_k.copy()
    bad_k[1234] = np.nan
    tk = _TORCH[kk]

    hs = shuffle.HostShuffle(n, tk, torch.int64, 3, "sum", splits=3)
    for k in (bad_k, good_k):
        hs.h_keys.copy_(torch.from_numpy(k))
        hs.h_vals.copy_(torch.from_numpy(v))
        if k is bad_k:
            with pytest.raises(TypeError):
                hs.run()
        else:
            check_reduce(hs.run(), py_reduce(k, v, 3, 3, "sum"), "sum", tk, torch.int64)

    for kind in ("reduce", "group"):
        st = shuffle.HostShuffleStream(n, tk, torch.int64, 3, splits=3, depth=2, kind=kind)
        st.submit(_pinned(bad_k), _pinned(v))
        st.submit(_pinned(good_k), _pinned(v))
        with pytest.raises(TypeError):
            st.collect()
        st.submit(_pinned(good_k), _pinned(v))          # the slot of the refused batch is free again
        for _ in range(2):
            if kind == "reduce":
                check_reduce(st.collect(), py_reduce(good_k, v, 3, 3, "sum"), "sum", tk, torch.int64)
            else:
                check_group(st.collect(), py_group(good_k, v, 3, 3), tk, torch.int64)
