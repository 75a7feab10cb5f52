"""Every columnar GPU operator over uneven, empty and zero-split ColumnarRDDs, against references that share no device
code with it.  -m gpu.

ColumnarRDD(bounds=...) -- what textFileColumns builds -- gives split layouts parallelizeColumns never makes: uneven
splits, empty splits anywhere, and no split at all (an empty file).  The layouts, over n rows:

  zero            [0] (n = 0)                  leading_empty   [0, 0, 0, n]
  one_empty       [0, 0] (n = 0)               trailing_empty  [0, n, n, n]
  one             [0, n]                       middle_empty    [0, a, a, a, b, n]
  singletons      one row per split (n <= 300) ragged          sizes 1, n // 2, 0, 3, 0, the rest

at n = 1, 300 and 4 * PT_TILE + 37 (several map-side multisplit tiles), and the ColumnarRDDs textFileColumns builds from
an empty file, an empty directory, a directory whose files the extension filter drops, a directory holding one empty
file, and long lines cut by a small splitSize (most splits own no line).  The columns come in the forms that pick the
two map-side paths of shuffle.map_side: one CUDA tensor or a CUDA view at a storage offset (one launch over
consecutive splits, shuffle._as_one), a CPU tensor or a non-contiguous CUDA column (one launch per split).

The references:
  - reduceByKey (add, min, max): a Python dict fold over the rows in (split, position) order, each key placed by the
    oracle's HashPartitioner.getPartition (oracle/dpk_oracle.c on the host); min, max and int sums exact, float sums
    within 1e-9 * sum |v| (DESIGN.md §7), a float key -0.0 spelled 0.0;
  - groupByKey, groupWith / cogroup (2- and 3-way) and the four joins: per key the value lists in (input, split,
    position) order, placed the same way, the joins' rows per key in `for a in left for b in right` order;
  - innerJoin, sort, top, topByKey, percentilesByKey and sample: the composition -- the same call on
    rdd.map(lambda x: x) -- partition by partition, in order; uniq and hot: the composition's partitions as sets
    (its reduceByKey's order varies), uniq in order against a Python first-occurrence list, hot's counts exactly;
  - the fixSkew thresholds: rdd._skew_thresholds(4, r) against the composition's, also over unions whose first input
    holds only empty splits.
Every case shows it ran on the device: the result is the operator's Columnar*RDD class (reduceByKey / groupByKey: a spy
saw the columns reach the device shuffle), and reading a ColumnarRDD as rows is refused while the result materialises.
Every layout also runs once at the smallest size under tests/test_gpu_buffer_bounds.py's guarded allocator, with the
poison bytes 0x00 and 0xFF: a zero-row launch on the per-split path that stored anywhere would show there.
The file takes 32 s on an H100 80GB HBM3 at a 700 W power limit.

Defects these tests found, fixed with them: sort of a ColumnarRDD without splits raised ZeroDivisionError
(sorting.sample_bounds); the fixSkew thresholds of inputs without splits at a rate below 1 raised ValueError from
torch.cat (sampling.bernoulli); reduceByKey of any RDD without splits raised IndexError (engine._run_reduce), which
also broke the compositions of uniq and hot of such an input.

Mutations run against these tests (tests/test_gpu_sample.py, test_gpu_sort.py, test_gpu_textcolumns.py,
test_sample_host.py and test_sort_host.py all pass under each of the first two):
  - sampling.ColumnarSampleRDD._run drawing over the non-empty splits only, which shifts the seed + i of later splits:
    caught by test_single_input_operators (sample over leading_empty, middle_empty and ragged), by
    test_text_file_columns_inputs[long_lines] and by test_guarded_at_the_smallest_size[middle_empty-1];
  - sorting.sample_bounds dividing by the number of non-empty splits instead of len(rdd): caught by
    test_single_input_operators (sort over leading_empty, trailing_empty, middle_empty and ragged at 300 rows and
    more) and by tests/test_split_layouts_host.py::test_sample_bounds_over_empty_splits;
  - sampling.skew_thresholds without _refold_first: NOT caught, and no output comparison can catch it on the inputs
    tried: refolding a digest's own centroids at the same total weight gives back the same centroids and lo / hi (no
    difference in quantiles.skew_thresholds([[], h, rest], s) against ([h, rest], s) over 29,406 random cases of up to
    2,000 hashes and 2 to 64 splits).  test_skew_thresholds still runs that path over leading_empty and over unions whose
    first input holds only empty splits.
"""
import collections
import operator
import os
import struct

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tests import cogroup_common as cc
from tests.test_gpu_buffer_bounds import POISONS, PT_TILE, _on_the_device, guarded  # noqa: F401

pytestmark = pytest.mark.gpu

SIZES = (1, 300, 4 * PT_TILE + 37)
KINDS = [(np.int32, np.int64), (np.int64, np.float64), (np.float32, np.float64), (np.float64, np.int64)]
FORMS = ["cuda", "cpu", "offset", "strided"]
ZERO = {"zero": [0], "one_empty": [0, 0]}


def layouts(n):
    a, b, big = n // 3, 2 * n // 3, n // 2
    out = {"one": [0, n], "leading_empty": [0, 0, 0, n], "trailing_empty": [0, n, n, n],
           "middle_empty": [0, a, a, a, b, n],
           "ragged": [min(n, c) for c in (0, 1, 1 + big, 1 + big, 4 + big, 4 + big)] + [n]}
    if n <= 300:
        out["singletons"] = list(range(n + 1))
    return out


CASES = [(name, 0, b) for name, b in ZERO.items()] + [(name, n, b) for n in SIZES for name, b in layouts(n).items()]
CASE_IDS = ["%s-%d" % (name, n) for name, n, _ in CASES]
SMALLEST = [c for c in CASES if c[1] <= 1]


def _has_empty(bounds):
    return any(a == b for a, b in zip(bounds, bounds[1:]))


def _data(n, kind, seed):
    """Keys that repeat (a few rows per key at the largest size, so the joins stay near n rows; float keys include -0.0
    beside 0.0), values without signed zeros."""
    kt, vt = kind
    rng = np.random.default_rng(seed)
    hi = max(30, n // 8)
    k = rng.integers(-hi, hi, n)
    v = rng.integers(-1000, 1000, n)
    if np.dtype(kt).kind == "f":
        k = k * 0.5
        k[rng.random(n) < min(0.1, 20 / max(n, 1))] = -0.0      # about 20 at the largest size: key 0.0's join stays small
    if np.dtype(vt).kind == "f":
        v = v * 0.25
    return k.astype(kt), v.astype(vt)


def _form(a, form):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if form == "cpu":
        return t
    if form == "offset":              # a view at storage offset 5 of a larger CUDA buffer
        buf = torch.zeros(len(a) + 9, dtype=t.dtype, device="cuda")
        buf[5:5 + len(a)] = t.cuda()
        return buf[5:5 + len(a)]
    if form == "strided":             # column 0 of an [n, 2] CUDA tensor
        m = torch.zeros((len(a), 2), dtype=t.dtype, device="cuda")
        m[:, 0] = t.cuda()
        return m[:, 0]
    return t.cuda()


def _rdd(dc, bounds, kind, form, seed):
    from dpark_b200.rdd import ColumnarRDD
    k, v = _data(bounds[-1], kind, seed)
    rdd = ColumnarRDD(dc, _form(k, form), _form(v, form), 1, bounds=bounds)
    assert [(s.begin, s.end) for s in rdd.splits] == list(zip(bounds, bounds[1:]))
    return rdd


def _rows(rdd):
    """The ColumnarRDD's rows in (split, position) order, read from the columns on the host."""
    k, v = rdd.keys.cpu().tolist(), rdd.vals.cpu().tolist()
    return [(k[i], v[i]) for sp in rdd.splits for i in range(sp.begin, sp.end)]


def _ident(x):
    return x


_PART = {}


def _part(key, P, thr):
    """HashPartitioner(P, thresholds=thr).getPartition(key) by the host oracle."""
    at = (repr(key), P, None if thr is None else tuple(thr))
    if at not in _PART:
        _PART[at] = orc.get_partition(key, P, thr)
    return _PART[at]


def _canon_key(k):
    return k + 0.0 if isinstance(k, float) else k


def _same(got, want, what=""):
    assert got == want and repr(got) == repr(want), what


def _bits(x):
    return struct.pack("<d", x) if isinstance(x, float) else x


# ------------------------------------------------------------------------------------------------------------ spies
class Spy(object):
    def __init__(self):
        self.reduce_inputs, self.group_columns = [], 0
        self.one_launch, self.per_split = 0, 0


@pytest.fixture
def spy(monkeypatch):
    from dpark_b200 import _native as nv
    from dpark_b200 import engine
    s = Spy()
    real_reduce, real_group, real_part, real_count = (engine._run_reduce, engine._run_group_columns, nv.partition,
                                                      nv.partition_count)

    def run_reduce(splits, *a, **kw):
        s.reduce_inputs.append(list(splits))
        return real_reduce(splits, *a, **kw)

    def run_group_columns(*a, **kw):
        s.group_columns += 1
        return real_group(*a, **kw)

    def partition(*a, **kw):
        s.one_launch += 1
        return real_part(*a, **kw)

    def partition_count(*a, **kw):
        s.per_split += 1
        return real_count(*a, **kw)

    monkeypatch.setattr(engine, "_run_reduce", run_reduce)
    monkeypatch.setattr(engine, "_run_group_columns", run_group_columns)
    monkeypatch.setattr(nv, "partition", partition)
    monkeypatch.setattr(nv, "partition_count", partition_count)
    return s


MAP_SIDE_PATHS = collections.Counter()      # map-side path -> reduceByKey runs over layouts with empty splits


# ------------------------------------------------------------------------------------------------------------ reduceByKey
OPS = {"add": operator.add, "min": min, "max": max}


def _reduce_reference(rows, P, thr, op):
    f = OPS[op]
    parts = [dict() for _ in range(P)]
    mags = {}
    for k, v in rows:
        k = _canon_key(k)
        d = parts[_part(k, P, thr)]
        d[k] = f(d[k], v) if k in d else v
        mags[k] = mags.get(k, 0.0) + abs(v)
    return parts, mags


def _check_reduce(got, rows, P, thr, op):
    want, mags = _reduce_reference(rows, P, thr, op)
    assert len(got) == P
    for p, (part, w) in enumerate(zip(got, want)):
        g = dict(part)
        assert len(g) == len(part), "a key twice in partition %d" % p
        assert sorted(map(repr, g)) == sorted(map(repr, w)), "partition %d keys" % p
        for k, wv in w.items():
            gv = g[k]
            assert type(gv) is type(wv)
            if op == "add" and isinstance(wv, float):
                assert abs(gv - wv) <= 1e-9 * mags[k], (k, gv, wv)
            else:
                assert _bits(gv) == _bits(wv), (k, gv, wv)


def _reduce_case(spy, dc, rdd, op, numSplits, fixSkew=-1):
    rows = _rows(rdd)
    if numSplits is None:
        P, thr = max(1, min(dc.defaultMinSplits, len(rdd))), None
    elif fixSkew > 0 and numSplits > 1:
        thr, P = rdd.map(_ident)._skew_thresholds(numSplits, fixSkew)
    else:
        P, thr = numSplits, None
    before_one, before_per = spy.one_launch, spy.per_split
    res = rdd.reduceByKey(OPS[op], numSplits, fixSkew=fixSkew)
    got = _on_the_device(lambda: res.glom().collect())
    inputs = spy.reduce_inputs[-1]
    assert len(inputs) == len(rdd.splits) and all(torch.is_tensor(k) for k, _ in inputs)
    _check_reduce(got, rows, P, thr, op)
    one, per = spy.one_launch - before_one, spy.per_split - before_per
    return one, per


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("op", sorted(OPS))
def test_reduce_by_key(form, op, spy):
    dc = cc.ctx()
    for i, (name, n, bounds) in enumerate(CASES):
        kind = KINDS[(i + FORMS.index(form)) % len(KINDS)]
        rdd = _rdd(dc, bounds, kind, form, seed=i)
        numSplits = [None, 1, 3, 7][i % 4]
        one, per = _reduce_case(spy, dc, rdd, op, numSplits)
        if len(rdd.splits) > 1:       # the map side's path: one launch over consecutive slices, or one per split
            if form in ("cuda", "offset"):
                assert (one, per) == (1, 0), (name, n)
            elif form == "cpu" or n > 1:      # slices of at most one row of a strided column are contiguous
                assert one == 0 and per == len(rdd.splits), (name, n)
            if _has_empty(bounds):
                MAP_SIDE_PATHS["one_launch" if one else "per_split"] += 1


@pytest.mark.parametrize("rate", [0.3, 1, 1.0])
def test_reduce_by_key_with_fix_skew(rate, spy):
    dc = cc.ctx()
    for i, (name, n, bounds) in enumerate(CASES):
        rdd = _rdd(dc, bounds, KINDS[i % len(KINDS)], FORMS[i % len(FORMS)], seed=100 + i)
        _reduce_case(spy, dc, rdd, "max", 4, fixSkew=rate)


def test_both_map_side_paths_ran_over_empty_splits():
    assert MAP_SIDE_PATHS["one_launch"] > 0 and MAP_SIDE_PATHS["per_split"] > 0, MAP_SIDE_PATHS


# ---------------------------------------------------------------------------------------- groupByKey, cogroup, joins
def _groups_reference(inputs, P, thr):
    """Per partition {key: (values of input 0, values of input 1, ...)} in (input, split, position) order."""
    parts = [dict() for _ in range(P)]
    for t, rdd in enumerate(inputs):
        for k, v in _rows(rdd):
            k = _canon_key(k)
            d = parts[_part(k, P, thr)]
            d.setdefault(k, tuple([] for _ in inputs))[t].append(v)
    return parts


def _check_groups(got, want):
    assert len(got) == len(want)
    for p, (part, w) in enumerate(zip(got, want)):
        g = {k: tuple(vs) for k, vs in part}
        assert len(g) == len(part), "a key twice in partition %d" % p
        _same(sorted(g.items(), key=repr), sorted(w.items(), key=repr), "partition %d" % p)


def _join_rows(groups, keep_left, keep_right):
    out = {}
    for k, (left, right) in groups.items():
        if not left and keep_right:
            left = [None]
        if not right and keep_left:
            right = [None]
        rows = [(a, b) for a in left for b in right]
        if rows:
            out[k] = rows
    return out


JOINS = {"join": (False, False), "leftOuterJoin": (True, False), "rightOuterJoin": (False, True),
         "outerJoin": (True, True)}
SMALL = {name: b for name, b in layouts(300).items()}
PAIRS = [("ragged", "middle_empty"), ("zero", "ragged"), ("ragged", "zero"), ("zero", "zero"),
         ("one_empty", "leading_empty"), ("singletons", "trailing_empty"), ("leading_empty", "one_empty"),
         ("one_empty", "zero"), ("middle_empty", "singletons")]


def _layout(name, n=300):
    return ZERO[name] if name in ZERO else (SMALL[name] if n == 300 else layouts(n)[name])


def _side(dc, name, kind, form, seed, n=300):
    return _rdd(dc, _layout(name, n), kind, form, seed)


def _side_kinds(i):
    """Both sides int keys or both float keys (int32 against int64, float32 against float64), values int64 / float64."""
    if i % 2:
        return (np.float32, np.int64), (np.float64, np.float64)
    return (np.int32, np.float64), (np.int64, np.int64)


PAIR_CASES = [(a, b, 300) for a, b in PAIRS] + [("ragged", "middle_empty", SIZES[-1])]
PAIR_IDS = ["%s-%s-%d" % c for c in PAIR_CASES]


@pytest.mark.parametrize("left, right, n", PAIR_CASES, ids=PAIR_IDS)
def test_group_by_key_cogroup_and_joins(left, right, n, spy):
    from dpark_b200.join import ColumnarCoGroupedRDD, ColumnarJoinedRDD
    dc = cc.ctx()
    i = PAIR_CASES.index((left, right, n))
    lk, rk = _side_kinds(i)
    a = _side(dc, left, lk, FORMS[i % 4], 10 * i, n)
    b = _side(dc, right, rk, FORMS[(i + 1) % 4], 10 * i + 1, n)
    for P in (None, 1, 4):
        Pn = P if P is not None else dc.defaultParallelism
        before = spy.group_columns
        res = a.groupByKey(P)
        got = _on_the_device(lambda: res.glom().collect())
        assert spy.group_columns == before + 1
        Pg = P if P is not None else max(1, min(dc.defaultMinSplits, len(a)))
        _check_groups([[(k, (vs,)) for k, vs in part] for part in got], _groups_reference([a], Pg, None))
        res = a.cogroup(b, P)
        assert type(res) is ColumnarCoGroupedRDD
        want = _groups_reference([a, b], Pn, None)
        _check_groups(_on_the_device(lambda: res.glom().collect()), want)
        for name, (keep_left, keep_right) in JOINS.items():
            res = getattr(a, name)(b, P)
            assert type(res) is ColumnarJoinedRDD
            got = _on_the_device(lambda: res.glom().collect())
            assert len(got) == Pn
            for p, (part, w) in enumerate(zip(got, want)):
                g = collections.OrderedDict()
                for k, pair in part:
                    g.setdefault(k, []).append(pair)
                _same(sorted(g.items(), key=repr), sorted(_join_rows(w, keep_left, keep_right).items(), key=repr),
                      "%s partition %d" % (name, p))


TRIPLES = [("zero", "ragged", "one_empty"), ("middle_empty", "singletons", "leading_empty"),
           ("one_empty", "zero", "zero"), ("trailing_empty", "one", "ragged")]


@pytest.mark.parametrize("names", TRIPLES, ids=["-".join(t) for t in TRIPLES])
def test_three_way_cogroup(names):
    from dpark_b200.join import ColumnarCoGroupedRDD
    dc = cc.ctx()
    i = TRIPLES.index(names)
    kinds = [(np.int64, np.int64), (np.int32, np.float64), (np.int64, np.float64)]
    rdds = [_side(dc, name, kinds[t], FORMS[(i + t) % 4], 30 * i + t) for t, name in enumerate(names)]
    for P in (None, 3):
        res = rdds[0].groupWith(rdds[1:], P)
        assert type(res) is ColumnarCoGroupedRDD
        got = _on_the_device(lambda: res.glom().collect())
        _check_groups(got, _groups_reference(rdds, P if P is not None else dc.defaultParallelism, None))


INNER = [("ragged", "middle_empty"), ("zero", "ragged"), ("ragged", "zero"), ("one_empty", "singletons"),
         ("singletons", "leading_empty"), ("middle_empty", "one_empty"), ("trailing_empty", "ragged")]


@pytest.mark.parametrize("big, small", INNER, ids=["-".join(t) for t in INNER])
def test_inner_join(big, small):
    from dpark_b200.join import ColumnarInnerJoinedRDD
    dc = cc.ctx()
    i = INNER.index((big, small))
    bk, sk = _side_kinds(i)
    for n in (300, SIZES[-1]) if big == "ragged" else (300,):
        a = _side(dc, big, bk, FORMS[i % 4], 50 * i, n)
        b = _side(dc, small, sk, FORMS[(i + 2) % 4], 50 * i + 1)
        want = a.map(_ident).innerJoin(b).glom().collect()
        res = a.innerJoin(b)
        assert type(res) is ColumnarInnerJoinedRDD and len(res) == len(a.splits)
        _same(_on_the_device(lambda: res.glom().collect()), want)


# ------------------------------------------------------------------------------------------- the single-input operators
GLOMMED = []                    # the classes of the RDDs _glom read


def _glom(r):
    GLOMMED.append(type(r).__name__)
    return r.glom().collect()


def _canon_pair(pair):
    """A pair as a set member: the composition keeps either spelling of a float zero (its merge order varies)."""
    return tuple(_canon_key(x) for x in pair)


def _uniq_norm(parts):
    return [sorted(repr(_canon_pair(x)) for x in p) for p in parts]


def _hot_norm(pairs):
    """hot's counts in order, and its pairs as a set within every run of equal counts but the last, which the cut at n
    may split (the composition's order among equal counts varies)."""
    counts = [c for _, c in pairs]
    last = counts[-1] if counts else None
    return counts, sorted(repr(_canon_pair(p)) for p, c in pairs if c != last)


def single_ops(P):
    """(name, operator over an RDD, normal form of its result, the device result's class or None)."""
    ops = [("sort-%s-%s-%s" % (kn, rev, ns), (lambda r, k=k, rev=rev, ns=ns: _glom(r.sort(k, rev, ns))), None,
            "ColumnarSortedRDD")
           for kn, k in (("id", lambda x: x), ("k", lambda x: x[0]), ("v", lambda x: x[1]))
           for rev in (False, True) for ns in (None, 4)]
    ops += [("top-%s-%s" % (kn, rev), (lambda r, k=k, rev=rev: r.top(7, k, rev)), None, None)
            for kn, k in (("id", None), ("k", lambda x: x[0]), ("v", lambda x: x[1])) for rev in (False, True)]
    ops += [("topByKey-%s" % rev, (lambda r, rev=rev: _glom(r.topByKey(3, reverse=rev, num_splits=P))), None,
             "ColumnarTopByKeyRDD") for rev in (False, True)]
    ops += [("percentilesByKey", lambda r: _glom(r.percentilesByKey([0, 10, 50, 99.5, 100], numSplits=P)), None,
             "ColumnarPercentilesByKeyRDD")]
    ops += [("sample-%r-%d" % (f, s), (lambda r, f=f, s=s: _glom(r.sample(f, False, s))), None, "ColumnarSampleRDD")
            for f in (0.3, 0.75, 0, 1) for s in (7, 12345)]
    ops += [("uniq", lambda r: _glom(r.uniq(P)), _uniq_norm, "ColumnarUniqRDD"),
            ("hot", lambda r: r.hot(5, P), _hot_norm, None)]
    return ops


def _run_device(rdd, make, cls):
    """make(rdd) with reading a ColumnarRDD as rows refused; the RDD it read is of class cls (None: make returns a
    list, and the refusal is the proof)."""
    del GLOMMED[:]
    out = _on_the_device(lambda: make(rdd))
    assert GLOMMED == ([cls] if cls is not None else []), (GLOMMED, cls)
    return out


def _check_single(rdd, P):
    for name, make, norm, cls in single_ops(P):
        want = make(rdd.map(_ident))
        got = _run_device(rdd, make, cls)
        norm = norm or _ident
        _same(norm(got), norm(want), name)
        if name.startswith("sort") and len(rdd.splits) == 0:
            assert got == []                    # no partition, as the composition returns the input itself
        if name == "uniq":
            _check_uniq_order(rdd, got, P)
        if name == "hot":
            _check_hot_counts(rdd, got)


def _check_uniq_order(rdd, got, P):
    """uniq in order: per partition the distinct pairs in order of first occurrence, with the first row's bits."""
    Pn = P if P is not None else max(1, min(rdd.ctx.defaultMinSplits, len(rdd)))
    want, seen = [[] for _ in range(Pn)], set()
    for row in _rows(rdd):
        if row not in seen:
            seen.add(row)
            want[_part(row, Pn, None)].append(row)
    _same(got, want, "uniq order")


def _check_hot_counts(rdd, got):
    counts = collections.Counter(_rows(rdd))
    assert [c for _, c in got] == sorted(counts.values(), reverse=True)[:5]
    assert all(counts[p] == c for p, c in got)


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_single_input_operators(case):
    name, n, bounds = case
    dc = cc.ctx()
    i = CASES.index(case)
    rdd = _rdd(dc, bounds, KINDS[i % len(KINDS)], FORMS[i % len(FORMS)], seed=200 + i)
    _check_single(rdd, [None, 4, 1][i % 3])


# ------------------------------------------------------------------------------------------------ the fixSkew thresholds
RATES = [0.3, 1, 1.0]
UNIONS = [("one_empty", "ragged"), ("zero", "ragged"), ("zero", "zero"), ("one_empty", "zero"),
          ("leading_empty", "middle_empty", "one_empty"), ("zero", "one_empty", "singletons"),
          ("one_empty", "one_empty")]


def _check_thresholds(rdd, rate, inputs):
    from dpark_b200 import sampling
    want = rdd_map(rdd)._skew_thresholds(4, rate)
    assert sampling.thresholds_inputs(rdd, rate) == inputs
    got = _on_the_device(lambda: sampling.skew_thresholds(inputs, 4, rate))
    assert got is not None
    _same(got, want)
    _same(_on_the_device(lambda: rdd._skew_thresholds(4, rate)), want)


def rdd_map(rdd):
    """The composition's input: every ColumnarRDD read through map (a union of such maps for a union)."""
    from dpark_b200.rdd import UnionRDD
    if type(rdd) is UnionRDD:
        return UnionRDD(rdd.ctx, [r.map(_ident) for r in rdd.rdds])
    return rdd.map(_ident)


@pytest.mark.parametrize("rate", RATES, ids=["0.3", "int1", "1.0"])
def test_skew_thresholds(rate):
    dc = cc.ctx()
    for i, (name, n, bounds) in enumerate(CASES):
        rdd = _rdd(dc, bounds, KINDS[i % len(KINDS)], FORMS[i % len(FORMS)], seed=300 + i)
        _check_thresholds(rdd, rate, [rdd])
    for i, names in enumerate(UNIONS):
        rdds = [_side(dc, nm, (np.int64, np.int64) if i % 2 else (np.float64, np.int64), FORMS[(i + t) % 4],
                      400 + 10 * i + t) for t, nm in enumerate(names)]
        u = rdds[0].union(*rdds[1:])
        _check_thresholds(u, rate, rdds)


@pytest.mark.parametrize("rate", [0.3, 1])
@pytest.mark.parametrize("layout", sorted(ZERO) + ["leading_empty"])
def test_fix_skew_operators_over_empty_inputs(layout, rate, spy):
    """reduceByKey, groupByKey, topByKey, percentilesByKey and the joins and cogroups with fixSkew over inputs that hold
    no row, or only empty splits before their rows: the composition's partitions."""
    from dpark_b200.join import ColumnarCoGroupedRDD, ColumnarJoinedRDD
    dc = cc.ctx()
    bounds = ZERO[layout] if layout in ZERO else layouts(1)[layout]
    a = _rdd(dc, bounds, (np.int64, np.float64), "cuda", 1)
    b = _rdd(dc, ZERO["zero"] if layout != "zero" else ZERO["one_empty"], (np.int64, np.int64), "cpu", 2)
    comp = rdd_map(a)
    _reduce_case(spy, dc, a, "add", 4, fixSkew=rate)
    before = spy.group_columns
    got = _on_the_device(lambda: _glom(a.groupByKey(4, fixSkew=rate)))
    assert spy.group_columns == before + 1
    _check_groups([[(k, (vs,)) for k, vs in part] for part in got],
                  [{k: (vs,) for k, vs in part} for part in _glom(comp.groupByKey(4, fixSkew=rate))])
    for make, cls in ((lambda r: _glom(r.topByKey(2, num_splits=4, fixSkew=rate)), "ColumnarTopByKeyRDD"),
                      (lambda r: _glom(r.percentilesByKey([50], numSplits=4, fixSkew=rate)),
                       "ColumnarPercentilesByKeyRDD")):
        _same(_run_device(a, make, cls), make(comp))
    for x, y in ((a, b), (b, a), (b, b)):
        res = x.cogroup(y, 4, fixSkew=rate)
        assert type(res) is ColumnarCoGroupedRDD
        _check_groups(_on_the_device(lambda: _glom(res)),
                      [dict(p) for p in _glom(rdd_map(x).cogroup(rdd_map(y), 4, fixSkew=rate))])
        res = x.outerJoin(y, 4, fixSkew=rate)
        assert type(res) is ColumnarJoinedRDD
        want = _glom(rdd_map(x).outerJoin(rdd_map(y), 4, fixSkew=rate))
        _same([sorted(p, key=repr) for p in _on_the_device(lambda: _glom(res))], [sorted(p, key=repr) for p in want])


# ------------------------------------------------------------------------------------------------ textFileColumns inputs
def _write(path, text):
    with open(path, "w") as f:
        f.write(text)
    return path


def _text_inputs(dc, tmp):
    """{name: ColumnarRDD} of the textFileColumns layouts."""
    os.makedirs(os.path.join(tmp, "empty_dir"))
    os.makedirs(os.path.join(tmp, "filtered"))
    os.makedirs(os.path.join(tmp, "one_empty_file"))
    os.makedirs(os.path.join(tmp, "mixed"))
    rng = np.random.default_rng(5)
    _write(os.path.join(tmp, "filtered", "a.txt"), "1 2\n3 4\n")
    _write(os.path.join(tmp, "one_empty_file", "a.txt"), "")
    _write(os.path.join(tmp, "mixed", "a.txt"), "")
    _write(os.path.join(tmp, "mixed", "b.txt"), "".join("%d %d\n" % (rng.integers(-9, 9), rng.integers(-99, 99))
                                                        for _ in range(50)))
    _write(os.path.join(tmp, "mixed", "c.txt"), "")
    long_lines = "".join("%d\t%r\t%s\n" % (rng.integers(-20, 20), float(rng.integers(-400, 400)) / 8, "x" * int(w))
                         for w in rng.integers(0, 400, 120))
    return {
        "empty_file": dc.textFileColumns(_write(os.path.join(tmp, "empty.txt"), "")),
        "empty_dir": dc.textFileColumns(os.path.join(tmp, "empty_dir")),
        "ext_matches_nothing": dc.textFileColumns(os.path.join(tmp, "filtered"), ext=".csv"),
        "dir_one_empty_file": dc.textFileColumns(os.path.join(tmp, "one_empty_file")),
        "dir_mixed": dc.textFileColumns(os.path.join(tmp, "mixed"), splitSize=64),
        "long_lines": dc.textFileColumns(_write(os.path.join(tmp, "long.tsv"), long_lines), 0, 1, (int, float), "\t",
                                         splitSize=64),
    }


TEXT = ["empty_file", "empty_dir", "ext_matches_nothing", "dir_one_empty_file", "dir_mixed", "long_lines"]


@pytest.mark.parametrize("name", TEXT)
def test_text_file_columns_inputs(name, tmp_path, spy):
    dc = cc.ctx()
    rdd = _text_inputs(dc, str(tmp_path))[name]
    if name in ("empty_file", "empty_dir", "ext_matches_nothing"):
        assert len(rdd.splits) == 0
    if name == "long_lines":
        assert sum(sp.begin == sp.end for sp in rdd.splits) > len(rdd.splits) // 2 and rdd.keys.numel() == 120
    for op in ("add", "max"):
        _reduce_case(spy, dc, rdd, op, [None, 4][op == "max"])
    _check_single(rdd, 4)
    for rate in RATES:
        _check_thresholds(rdd, rate, [rdd])
    other = _rdd(dc, SMALL["ragged"], (np.int64, np.float64), "cuda", 9)
    _check_groups(_on_the_device(lambda: _glom(rdd.cogroup(other, 3))), _groups_reference([rdd, other], 3, None))


# ------------------------------------------------------------------------------------------------ guarded, smallest size
@pytest.mark.parametrize("case", SMALLEST, ids=["%s-%d" % (c[0], c[1]) for c in SMALLEST])
def test_guarded_at_the_smallest_size(case, guarded):
    """Every operator over the layout at its smallest size, on guarded, poison-filled buffers: no store outside an
    allocation, and bit-identical results under both poison bytes, equal to the composition's."""
    name, n, bounds = case
    dc = cc.ctx()
    i = SMALLEST.index(case)
    outs = []
    for form in ("cuda", "cpu"):                 # both map-side paths
        rdd = _rdd(dc, bounds, KINDS[i % len(KINDS)], form, seed=500 + i)
        other = _rdd(dc, layouts(1)["ragged"], (KINDS[i % len(KINDS)][0], np.int64), "cuda", 501 + i)
        ops = [(nm, make, norm or _ident) for nm, make, norm, _ in single_ops(4)]
        ops += [("reduceByKey", lambda r: _glom(r.reduceByKey(max, 3)), lambda ps: [sorted(p) for p in ps]),
                ("groupByKey", lambda r: _glom(r.groupByKey(3)), lambda ps: [sorted(p) for p in ps]),
                ("cogroup", lambda r: _glom(r.cogroup(other if type(r) is type(other) else rdd_map(other), 3)),
                 lambda ps: [sorted(p, key=repr) for p in ps]),
                ("outerJoin", lambda r: _glom(r.outerJoin(other if type(r) is type(other) else rdd_map(other), 3)),
                 lambda ps: [sorted(p, key=repr) for p in ps]),
                ("innerJoin", lambda r: _glom(r.innerJoin(other)), _ident),
                ("thresholds", lambda r: r._skew_thresholds(4, 0.3), _ident)]
        want = [norm(make(rdd_map(rdd))) for _, make, norm in ops]
        guarded.check()
        runs = []
        for p in POISONS:
            guarded.poison = p
            got = [norm(_on_the_device(lambda: make(rdd))) for _, make, norm in ops]
            guarded.check()
            for (nm, _, _), g, w in zip(ops, got, want):
                _same(g, w, nm)
            runs.append(repr(got))
        assert runs[0] == runs[1], "the result depends on the poison byte"
        outs.append(runs[0])
    assert outs[0] == outs[1]
