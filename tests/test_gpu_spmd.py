"""The multi-rank engine on the real kernels: two and three driver processes sharing cuda:0, each running the same
script, against references that share no device code with the engine.  -m gpu.

Under torchrun every shuffle goes through engine._run_shuffle_spmd.  Here G = 2 and G = 3 processes are spawned, join a
gloo group over 127.0.0.1 themselves (so DparkContext creates no NCCL group, which refuses two ranks on one device)
and run the cases below in one fixed order.  The engine's device collectives (the counts all-gather and the
all_to_all_single of shuffle.exchange) get CUDA tensors, which gloo takes as they are.  Every case's outcome, a result
or an exception's type and message, must be the same on every rank: rank 0 hands back its outcomes, the other ranks a
digest of theirs.  The cases:

  - numeric reduceByKey from Python rows (engine._device_reduce, exchange with G > 1, reduce_side over G sources):
    int64 keys with INT64_MIN / MAX, float keys with +-0.0, +-inf and subnormals; all seven ops over int values,
    sum / min / max / prod over float values; P in {1, 2, 5, 8} with and without fixSkew; one split (ranks without a
    split), four splits (owners 0, 0, 1, 1 at G = 3), and a 20,000-row split beside a 7-row one, whose own rows
    would choose fewer sub-bucket bits than the agreed maximum; and 2^21 rows with four hot keys.  Reference:
    oracle.py_reduce_by_key over the same splits (oracle.reduce_by_key's C loops for the large case), placed by
    getPartition with the thresholds the ranks agreed on, which must equal one process's; int values and float
    min / max exact, float sums within 1e-9 * sum |v| of the key, float products within a relative 1e-12;
  - reduceByKey of ColumnarRDDs (the tensor branch): every pair of int32 / int64 / float32 / float64 for keys and
    values, CUDA and CPU columns, split bounds with empty splits so that one rank owns only empty splits;
  - the routed shuffle: reduceByKey over str (non-ASCII too), bytes and (int, str) tuple keys with int and float
    values, groupByKey of object values and of a ColumnarRDD, each key's list equal to oracle.py_group_by_key's, in
    order;
  - word count of ASCII and UTF-8 files with numSplits = 5, a one-split file and an empty file, against
    collections.Counter(text.split()); each saveAsTextFile part holds exactly its partition's words;
  - the columnar operators, which take their compositions with G > 1: each glom() equals the one-process device
    result computed in the parent, partition by partition (in order where the operator defines one, per key where
    it groups, as a set for uniq and hot, percentiles bit for bit);
  - Bagel (tests/golden/bagel_cases.json) and an accumulator, whose value every rank must see;
  - errors every rank must raise alike: int keys on one rank and float keys on another, int values on one rank and
    float values on another, an int64 sum and an int64 product that overflow only across ranks, a NaN key in one
    rank's split of a ColumnarRDD, and a str-keyed product whose overflow only the owner of its partition sees:
    the type and message one process raises.

Before engine._run_shuffle_spmd took the one-process checks over from the ranks' descriptors, the multi-rank path
returned -2^62 for the sum, 0 for the product and one merged key for the NaNs; and, as the code shows, the str-keyed
product raised on its owner alone, leaving the other ranks waiting in the all-gather of the results until the group
timed out (not run against that code: it would stall on purpose).

A host-side mutation these tests catch and tests/test_spmd_gloo.py and test_exchange_gloo.py miss (it changes no
buffer size and no kernel argument): shuffle.reduce_by_key dropping `rx.part_first +` from its partition labels, so
that every rank labels its partitions from 0 and rank 1's results overwrite rank 0's.  The CPU files route every
shuffle through oracle stand-ins, so no labels of the device reduce reach them.  Reading `got` in reverse source
order in _routed_shuffle is caught here by the groupByKey value lists and also by test_spmd_gloo.py.

NCCL, the peer-memory forms across devices and multi-GPU timing stay with scripts/spmd_check.py and
scripts/multi_gpu_check.py, which need one GPU per rank.
"""
import collections
import ctypes
import datetime
import hashlib
import math
import operator
import os
import socket
import sys
import time

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tests import bagel_jobs
from tests.golden_util import load

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1
FUNCS = {"sum": operator.add, "min": min, "max": max, "prod": operator.mul,
         "and": operator.and_, "or": operator.or_, "xor": operator.xor}
INT_OPS, FLOAT_OPS = ["sum", "min", "max", "prod", "and", "or", "xor"], ["sum", "min", "max", "prod"]
WORLD_TIMEOUT = 60          # seconds: the gloo group's timeout
RUN_TIMEOUT = 900           # seconds: all cases of one world

CASES = collections.OrderedDict()       # name -> run(dc, env): what every rank computes, in this order
CHECKS = {}                             # name -> check(outcome, env): the parent's comparison with the reference


def case(name, check):
    def deco(run):
        CASES[name] = run
        CHECKS[name] = check
        return run
    return deco


def ctx():
    sys.argv = [sys.argv[0]]
    from dpark_b200 import DparkContext
    return DparkContext("local")


def columnar_rdd(dc, keys, vals, bounds=None, n=4):
    from dpark_b200.rdd import ColumnarRDD
    return ColumnarRDD(dc, keys, vals, n, bounds=bounds)


# ---- numeric reduceByKey from Python rows ----------------------------------------------------------------------------
FLOAT_KEY_EDGES = [0.0, -0.0, math.inf, -math.inf, 5e-324, -5e-324, 2.2250738585072014e-308, 1e-310, 1.5, -2.25]
INT_KEY_EDGES = [I64_MIN, I64_MAX, I64_MIN + 1, I64_MAX - 1, 0, -1, 1]


def numeric_rows(seed, fkeys, op, fvals, n=3000):
    rng = np.random.default_rng(seed)
    if fkeys:
        pool = FLOAT_KEY_EDGES + [float(x) for x in np.round(rng.normal(0, 100, 90), 2)]
    else:
        pool = INT_KEY_EDGES + [int(x) for x in rng.integers(-10 ** 12, 10 ** 12, 90)]
    keys = [pool[i] for i in rng.integers(0, len(pool), n)]
    if fvals:
        if op == "prod":
            vals = (rng.uniform(0.5, 2.0, n) * rng.choice([-1.0, 1.0], n)).tolist()
        else:
            vals = (rng.normal(0, 1e3, n)).tolist()
    elif op == "sum":
        vals = rng.integers(-2 ** 40, 2 ** 40, n).tolist()
    elif op == "prod":
        vals = rng.choice([-1, 1] * 20 + [2, 3], n).tolist()       # products stay well inside int64
    else:
        vals = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True).tolist()
    return list(zip(keys, vals))


def layout_splits(rows, layout):
    if layout == "one":
        return [rows]
    if layout == "four":
        return orc.split_like_parallelize(rows, 4)
    return [rows[:20000], rows[20000:]]          # "lopsided": 20,000 rows beside 7


def layout_rdd(dc, rows, layout):
    if layout == "lopsided":
        a, b = layout_splits(rows, layout)
        return dc.parallelize(a, 1).union(dc.parallelize(b, 1))
    return dc.parallelize(rows, {"one": 1, "four": 4}[layout])


def numeric_specs():
    specs = []
    combos = [(fk, fv, op) for fk in (False, True) for fv in (False, True) for op in (FLOAT_OPS if fv else INT_OPS)]
    for i, (fk, fv, op) in enumerate(combos):
        P = [1, 2, 5, 8][i % 4]
        skew = (i // 4) % 2 == 1
        layout = ["four", "one", "lopsided"][i % 3]
        specs.append((i, fk, fv, op, P, skew, layout))
    return specs


def _rows_of(spec):
    i, fk, fv, op, P, skew, layout = spec
    return numeric_rows(100 + i, fk, op, fv, n=20007 if layout == "lopsided" else 3000)


def reduce_job(dc, rdd, op, P, skew):
    r = rdd.reduceByKey(FUNCS[op], P, fixSkew=0.5 if skew else -1)
    return {"thresholds": r.partitioner.thresholds, "parts": r.glom().collect()}


def check_reduce_parts(parts, want, op, tol=None):
    """parts: the glom of a reduceByKey; want / tol: per partition {key: value} / {key: sum |v|}."""
    assert len(parts) == len(want)
    for p, (rows, w) in enumerate(zip(parts, want)):
        got = dict(rows)
        assert len(got) == len(rows), "partition %d holds a key twice" % p
        assert set(got) == set(w), "partition %d: keys differ" % p
        for k, v in got.items():
            if isinstance(v, float) and op == "sum":
                assert abs(v - w[k]) <= 1e-9 * tol[p][k], (p, k, v, w[k])
            elif isinstance(v, float) and op == "prod":
                assert abs(v - w[k]) <= 1e-12 * abs(w[k]), (p, k, v, w[k])
            else:
                assert v == w[k] and type(v) is type(w[k]), (p, k, v, w[k])


def reference_reduce(splits, P, op, thresholds):
    want = orc.py_reduce_by_key(splits, P, FUNCS[op], thresholds)
    tol = orc.py_reduce_by_key([[(k, abs(v)) for k, v in s] for s in splits], P, operator.add, thresholds)
    return want, tol


def _one_process_thresholds(rows, layout, P, skew):
    if not skew:
        return None
    return layout_rdd(ctx(), rows, layout).reduceByKey(operator.add, P, fixSkew=0.5).partitioner.thresholds


def _numeric_case(spec):
    i, fk, fv, op, P, skew, layout = spec

    def run(dc, env):
        return reduce_job(dc, layout_rdd(dc, _rows_of(spec), layout), op, P, skew)

    def check(out, env):
        rows = _rows_of(spec)
        assert out["thresholds"] == _one_process_thresholds(rows, layout, P, skew)
        want, tol = reference_reduce(layout_splits(rows, layout), P, op, out["thresholds"])
        check_reduce_parts(out["parts"], want, op, tol)
    name = "rows-%s_keys-%s_vals-%s-P%d%s-%s" % ("f64" if fk else "i64", "f64" if fv else "i64", op, P,
                                                 "-skew" if skew else "", layout)
    case(name, check)(run)


for _spec in numeric_specs():
    _numeric_case(_spec)


def _large_columns():
    rng = np.random.default_rng(7)
    n = 1 << 21
    keys = np.where(rng.random(n) < 0.5, rng.integers(0, 4, n), rng.integers(0, 1 << 20, n)).astype(np.int64)
    vals = rng.integers(-1000, 1000, n).astype(np.int64)
    return keys, vals


def _run_large(dc, env):
    keys, vals = _large_columns()
    r = dc.parallelize(list(zip(keys.tolist(), vals.tolist())), 5).reduceByKey(operator.add, 8)
    return [sorted(p) for p in r.glom().collect()]


def _check_large(out, env):
    keys, vals = _large_columns()
    cuts = [len(s) for s in orc.split_like_parallelize(range(len(keys)), 5)]
    at = np.cumsum([0] + cuts)
    want = orc.reduce_by_key([keys[a:b] for a, b in zip(at[:-1], at[1:])], [vals[a:b] for a, b in zip(at[:-1], at[1:])],
                             8, "sum")
    assert len(out) == 8
    for p, (wk, wv) in enumerate(want):
        o = np.argsort(wk, kind="stable")
        assert out[p] == list(zip(wk[o].tolist(), wv[o].tolist())), "partition %d" % p


case("rows-2^21-hot_keys-sum-P8", _check_large)(_run_large)


# ---- reduceByKey of ColumnarRDDs: the tensor branch ------------------------------------------------------------------
DTYPES = [torch.int32, torch.int64, torch.float32, torch.float64]
F32_KEY_EDGES = [0.0, -0.0, math.inf, -math.inf, 1e-45, -1e-45, 1.5, -2.25]


def columns_input(kdt, vdt, seed, n=2000):
    rng = np.random.default_rng(seed)
    if kdt.is_floating_point:
        pool = torch.tensor(F32_KEY_EDGES + np.round(rng.normal(0, 50, 40), 1).tolist(), dtype=kdt)
    else:
        info = torch.iinfo(kdt)
        pool = torch.tensor([info.min, info.max, 0, -1] + rng.integers(-10 ** 6, 10 ** 6, 40).tolist(), dtype=kdt)
    keys = pool[torch.from_numpy(rng.integers(0, len(pool), n))]
    vals = torch.from_numpy(rng.integers(-1000, 1000, n)).to(vdt)
    a, b = n // 3, n // 3 + 5
    return keys, vals, [0, a, b, n, n, n]      # owners 0,0,1,1,2 at G = 3 and 0,0,0,1,1 at G = 2: empty splits only


def _columns_case(ci, kdt, vdt):
    op = ["sum", "min", "max"][ci % 3] if vdt != torch.float32 else ["min", "max"][ci % 2]
    on_cuda = ci % 2 == 0

    def run(dc, env):
        keys, vals, bounds = columns_input(kdt, vdt, 300 + ci)
        if on_cuda:
            keys, vals = keys.cuda(), vals.cuda()
        return reduce_job(dc, columnar_rdd(dc, keys, vals, bounds), op, 5, False)

    def check(out, env):
        keys, vals, bounds = columns_input(kdt, vdt, 300 + ci)
        ks, vs = keys.tolist(), vals.tolist()
        splits = [list(zip(ks[a:b], vs[a:b])) for a, b in zip(bounds[:-1], bounds[1:])]
        want, tol = reference_reduce(splits, 5, op, None)
        check_reduce_parts(out["parts"], want, op, tol)
    name = "columns-%s_keys-%s_vals-%s-%s" % (str(kdt)[6:], str(vdt)[6:], op, "cuda" if on_cuda else "cpu")
    case(name, check)(run)


for _ci, (_kdt, _vdt) in enumerate([(k, v) for k in DTYPES for v in DTYPES]):
    _columns_case(_ci, _kdt, _vdt)


# ---- the routed shuffle ----------------------------------------------------------------------------------------------
def routed_rows(kind, fvals, seed, n=1500):
    rng = np.random.default_rng(seed)
    if kind == "str":
        pool = ["w%d" % i for i in range(40)] + ["é", "naïve", "日本語", "ß", "", "Ω≈ç", "😀"]
    elif kind == "bytes":
        pool = [b"b%d" % i for i in range(40)] + [b"", b"\x00", b"\xff\xfe", b"\x80" * 9]
    else:
        pool = [(i % 7, "t%d" % (i % 3)) for i in range(30)] + [(-1, "é"), (2 ** 40, ""), (I64_MIN, "日本")]
    keys = [pool[i] for i in rng.integers(0, len(pool), n)]
    vals = rng.normal(0, 100, n).tolist() if fvals else rng.integers(-10 ** 9, 10 ** 9, n).tolist()
    return list(zip(keys, vals))


def _routed_case(kind, fvals, P, nsplits, seed):
    def run(dc, env):
        return reduce_job(dc, dc.parallelize(routed_rows(kind, fvals, seed), nsplits), "sum", P, False)

    def check(out, env):
        splits = orc.split_like_parallelize(routed_rows(kind, fvals, seed), nsplits)
        want, tol = reference_reduce(splits, P, "sum", None)
        check_reduce_parts(out["parts"], want, "sum", tol)
    case("routed-reduce-%s_keys-%s_vals-P%d-%dsplits" % (kind, "f64" if fvals else "i64", P, nsplits), check)(run)


for _i, (_kind, _fv) in enumerate([(k, f) for k in ("str", "bytes", "tuple") for f in (False, True)]):
    _routed_case(_kind, _fv, [1, 2, 5][_i % 3], [1, 4, 5][_i % 3], 500 + _i)


def check_group_parts(parts, want):
    assert len(parts) == len(want)
    for p, (rows, w) in enumerate(zip(parts, want)):
        got = dict((k, list(v)) for k, v in rows)
        assert len(got) == len(rows), "partition %d holds a key twice" % p
        assert got == w, "partition %d" % p


def _group_rows():
    rng = np.random.default_rng(11)
    return [(int(k), ("v", i, float(i) / 3)) for i, k in enumerate(rng.integers(0, 50, 1200))]


def _run_group_objects(dc, env):
    return dc.parallelize(_group_rows(), 5).groupByKey(4).glom().collect()


def _check_group_objects(out, env):
    check_group_parts(out, orc.py_group_by_key(orc.split_like_parallelize(_group_rows(), 5), 4))


case("routed-groupByKey-objects-P4-5splits", _check_group_objects)(_run_group_objects)


def _group_columns():
    keys, vals, bounds = columns_input(torch.float64, torch.int64, 17, n=900)
    return keys, vals, bounds


def _run_group_columns(dc, env):
    keys, vals, bounds = _group_columns()
    return columnar_rdd(dc, keys.cuda(), vals.cuda(), bounds).groupByKey(3).glom().collect()


def _check_group_columns(out, env):
    keys, vals, bounds = _group_columns()
    ks, vs = keys.tolist(), vals.tolist()
    splits = [list(zip(ks[a:b], vs[a:b])) for a, b in zip(bounds[:-1], bounds[1:])]
    check_group_parts(out, orc.py_group_by_key(splits, 3))


case("routed-groupByKey-columns-P3", _check_group_columns)(_run_group_columns)


# ---- word count ------------------------------------------------------------------------------------------------------
def fm(x):
    for w in x.strip().split():
        yield (w, 1)


WC_FILES = {
    "ascii-5splits": (5, lambda rng: "\n".join(" ".join("w%d" % int(x) for x in rng.zipf(1.3, 12) % 500)
                                               for _ in range(600)) + "\n"),
    "utf8-5splits": (5, lambda rng: "\n".join(" ".join(["é", "naïve", "日本語", "ß", "Ω", "w%d" % int(x)][int(x) % 6]
                                                       + str(int(x) % 17) for x in rng.integers(0, 10 ** 6, 9))
                                              + "　x y" for _ in range(500))),
    "ascii-1split": (1, lambda rng: "one two  two\tthree three three\n"),
    "empty": (3, lambda rng: ""),
}


def write_wc_files(root):
    for i, (name, (_, make)) in enumerate(WC_FILES.items()):
        with open(os.path.join(root, name + ".txt"), "w", encoding="utf-8") as f:
            f.write(make(np.random.default_rng(i)))


def _wc_case(name, nsplits):
    def run(dc, env):
        path = os.path.join(env["data"], name + ".txt")
        out = os.path.join(env["out"], name)
        counts = dc.textFile(path, numSplits=nsplits).flatMap(fm).reduceByKey(lambda x, y: x + y, numSplits=6)
        got = counts.collectAsMap()
        counts.map(lambda x: " ".join(map(str, x))).saveAsTextFile(out, overwrite=False)
        return got

    def check(out, env):
        with open(os.path.join(env["data"], name + ".txt"), encoding="utf-8") as f:
            text = f.read()
        want = collections.Counter(text.split())
        assert out == dict(want)
        root = os.path.join(env["out"], name)
        names = os.listdir(root) if os.path.isdir(root) else []
        files = {int("".join(c for c in fn if c.isdigit())): fn for fn in names}
        assert set(files) <= set(range(6))
        for p in range(6):
            lines = []
            if p in files:
                with open(os.path.join(root, files[p]), encoding="utf-8") as f:
                    lines = [ln for ln in f.read().split("\n") if ln]
            assert sorted(lines) == sorted("%s %d" % (w, c) for w, c in want.items() if orc.get_partition(w, 6) == p)
    case("wordcount-" + name, check)(run)


for _name, (_ns, _) in WC_FILES.items():
    _wc_case(_name, _ns)


# ---- the columnar operators, compositions with G > 1 against the one-process device result ---------------------------
def op_inputs(dc):
    rng = np.random.default_rng(23)

    def cols(n, kmax, seed_vals, nsl, vdt=torch.float64):
        k = torch.from_numpy(rng.integers(0, kmax, n)).cuda()
        v = torch.from_numpy(rng.normal(0, 10, n) if vdt.is_floating_point else rng.integers(-99, 99, n)).to(vdt).cuda()
        return dc.parallelizeColumns(k, v, nsl)
    return cols(700, 60, 0, 4), cols(300, 80, 1, 3, torch.int64), cols(200, 40, 2, 5)


OPERATORS = collections.OrderedDict([
    ("join", ("by_key", lambda a, b, c: a.join(b, 4))),
    ("leftOuterJoin", ("by_key", lambda a, b, c: a.leftOuterJoin(b, 3, fixSkew=0.5))),
    ("rightOuterJoin", ("by_key", lambda a, b, c: a.rightOuterJoin(b, 5))),
    ("outerJoin", ("by_key", lambda a, b, c: a.outerJoin(b, 2, fixSkew=0.5))),
    ("cogroup3", ("by_key", lambda a, b, c: a.groupWith([b, c], 4))),
    ("groupByKey", ("by_key", lambda a, b, c: a.groupByKey(3, fixSkew=0.5))),
    ("sort", ("ordered", lambda a, b, c: a.sort(numSplits=3))),
    ("sort_x0", ("ordered", lambda a, b, c: a.sort(key=lambda x: x[0], numSplits=4))),
    ("sort_x1_reverse", ("ordered", lambda a, b, c: a.sort(key=lambda x: x[1], reverse=True, numSplits=2))),
    ("top", ("ordered", lambda a, b, c: a.top(25))),
    ("topByKey", ("ordered", lambda a, b, c: a.topByKey(3, num_splits=4, fixSkew=0.5))),
    ("percentilesByKey", ("ordered", lambda a, b, c: a.percentilesByKey([10, 50, 90], numSplits=3))),
    ("uniq", ("as_set", lambda a, b, c: b.uniq(3))),
    ("hot", ("as_set", lambda a, b, c: b.hot(100, 3))),        # n above the distinct count: ties cannot pick
    ("sample", ("ordered", lambda a, b, c: a.sample(0.3, False, 99))),
    ("innerJoin", ("ordered", lambda a, b, c: a.innerJoin(c))),
])


def _glom(r):
    if isinstance(r, list):             # top: already a list
        return r
    return r.glom().collect()


def normalise(kind, res):
    """ordered: as it is; by_key: each partition's rows as {key: [values in order]}; as_set: sorted rows (hot: a list
    of rows, uniq: partitions)."""
    if kind == "ordered":
        return res
    if kind == "by_key":
        out = []
        for p in res:
            d = {}
            for k, v in p:
                d.setdefault(k, []).append(v)
            out.append(d)
        return out
    if res and isinstance(res[0], tuple):
        return sorted(res, key=repr)
    return [sorted(p, key=repr) for p in res]


def _operator_case(name, kind, make):
    def run(dc, env):
        return normalise(kind, _glom(make(*op_inputs(dc))))

    def check(out, env):
        from dpark_b200.rdd import device_path_applies
        dc = ctx()
        ins = op_inputs(dc)
        assert device_path_applies(list(ins))
        assert out == normalise(kind, _glom(make(*ins))), name
    case("operator-" + name, check)(run)


for _name, (_kind, _make) in OPERATORS.items():
    _operator_case(_name, _kind, _make)


# ---- Bagel and accumulators ----------------------------------------------------------------------------------------- 
BAGEL_CASES = load("bagel_cases.json")["cases"]


def _run_bagel(dc, env):
    from dpark_b200 import bagel
    out = []
    for c in BAGEL_CASES:
        run = bagel_jobs.run_pagerank if c["job"] == "pagerank" else bagel_jobs.run_maxprop
        out.append(run(dc, bagel, [[v, ts] for v, ts in c["graph"]], c["parts"]))
    return out


def _check_bagel(out, env):
    for c, got in zip(BAGEL_CASES, out):
        if c["job"] == "pagerank":
            want = {k: float.fromhex(v) for k, v in c["values"].items()}
            assert sorted(got) == sorted(want), c["name"]
            for k in want:
                assert abs(got[k] - want[k]) <= 1e-12 * abs(want[k]), (c["name"], k)
        else:
            assert {str(k): v for k, v in got.items()} == c["values"], c["name"]


case("bagel-golden", _check_bagel)(_run_bagel)


def _run_accumulators(dc, env):
    acc, rows_seen = dc.accumulator(0), dc.accumulator(0)

    def one(x):
        acc.add(x)
        rows_seen.add(1)
        return (x % 13, x)
    total = dc.parallelize(list(range(1000)), 7).map(one).reduceByKey(operator.add, 4).count()
    after_one = (acc.value, rows_seen.value)
    dc.parallelize(list(range(50)), 2).foreach(lambda x: acc.add(x))
    return {"count": total, "after_job": after_one, "after_foreach": acc.value}


def _check_accumulators(out, env):
    assert out == {"count": 13, "after_job": (sum(range(1000)), 1000), "after_foreach": sum(range(1000)) + sum(range(50))}


case("accumulators", _check_accumulators)(_run_accumulators)


# ---- errors every rank raises alike --------------------------------------------------------------------------------- 
def _two_splits(dc, a, b):
    return dc.parallelize(a, 1).union(dc.parallelize(b, 1))


ERROR_JOBS = collections.OrderedDict([
    ("mixed_key_kinds", lambda dc: _two_splits(dc, [(1, 1), (2, 2)], [(1.5, 3)]).reduceByKey(operator.add, 2)),
    ("mixed_value_kinds", lambda dc: _two_splits(dc, [(1, 1), (2, 2)], [(1, 1.5)]).reduceByKey(operator.add, 2)),
    ("int64_sum_overflow", lambda dc: _two_splits(dc, [(7, 2 ** 62)], [(7, 2 ** 62), (7, 2 ** 62)])
     .reduceByKey(operator.add, 2)),
    ("int64_prod_overflow", lambda dc: _two_splits(dc, [(5, 2 ** 32), (6, 3)], [(5, 2 ** 32)])
     .reduceByKey(operator.mul, 2)),
    ("nan_key_columns", lambda dc: columnar_rdd(dc, torch.tensor([1.0, 2.0, 3.0, math.nan], device="cuda"),
                                                torch.arange(4, device="cuda"), [0, 2, 4]).reduceByKey(operator.add, 2)),
    ("str_key_prod_overflow", lambda dc: _two_splits(dc, [("a", 2 ** 32), ("b", 3)], [("a", 2 ** 32)])
     .reduceByKey(operator.mul, 3)),
])


def outcome(f, *a):
    try:
        return ("ok", f(*a))
    except Exception as e:
        return (type(e).__name__, str(e))


def _error_case(name, make):
    def run(dc, env):
        return make(dc).collect()

    def check(out, env):
        want = outcome(lambda: make(ctx()).collect())
        assert want[0] != "ok", want
        assert out == want
    case("error-" + name, check)(run)


for _name, _make in ERROR_JOBS.items():
    _error_case(_name, _make)


# ---- the harness -----------------------------------------------------------------------------------------------------
CUDA_DEV_ATTR_COMPUTE_MODE = 20      # cudaDevAttrComputeMode; 0 = default (shared), 1 / 3 = exclusive, 2 = prohibited


def compute_mode():
    torch.cuda.init()
    v = ctypes.c_int(-1)
    err = ctypes.CDLL("libcudart.so.12").cudaDeviceGetAttribute(ctypes.byref(v), CUDA_DEV_ATTR_COMPUTE_MODE, 0)
    return v.value if err == 0 else None


def digest(x):
    return hashlib.sha256(repr(x).encode()).hexdigest()


def worker(rank, world, port, env, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sys.argv = [sys.argv[0]]
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=WORLD_TIMEOUT))
    try:
        try:
            torch.cuda.set_device(0)
            torch.zeros(1, device="cuda")
        except Exception as e:
            q.put((rank, "skip", "cannot create a CUDA context on cuda:0 (compute mode %s): %s" % (compute_mode(), e)))
            return
        dc = ctx()
        out = collections.OrderedDict()
        for name, run in CASES.items():
            t0 = time.time()
            res = outcome(run, dc, env)
            out[name] = (res if rank == 0 else digest(res), time.time() - t0)
        q.put((rank, "done", out))
    except BaseException as e:
        import traceback
        q.put((rank, "error", "%r\n%s" % (e, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


@pytest.fixture(scope="module")
def env(tmp_path_factory):
    mode = compute_mode()
    if mode not in (0, None):
        pytest.skip("cuda:0 is in compute mode %d (not shared): several processes cannot use it at once" % mode)
    root = tmp_path_factory.mktemp("spmd")
    data = root / "data"
    data.mkdir()
    write_wc_files(str(data))
    return {"data": str(data), "root": str(root)}


_WORLDS = {}


def world_outcomes(G, env):
    """Every rank's outcomes, run once per G: a world that failed or skipped is reported to every test, not rerun."""
    if G not in _WORLDS:
        try:
            _WORLDS[G] = ("ok", _run_world(G, env))
        except pytest.skip.Exception as e:
            _WORLDS[G] = ("skip", str(e))
        except BaseException as e:
            _WORLDS[G] = ("fail", "%s: %s" % (type(e).__name__, e))
    status, res = _WORLDS[G]
    if status == "skip":
        pytest.skip(res)
    if status == "fail":
        pytest.fail("the world of %d ranks failed: %s" % (G, res))
    return res


def _run_world(G, env):
    import multiprocessing
    import queue
    import torch.multiprocessing as mp
    wenv = dict(env, out=os.path.join(env["root"], "out%d" % G))
    spawn = mp.get_context("spawn")
    q = spawn.Queue()
    port = _free_port()
    procs = [spawn.Process(target=worker, args=(r, G, port, wenv, q)) for r in range(G)]
    t0 = time.time()
    got = {}
    try:
        for p in procs:
            p.start()
        while len(got) < G:
            try:
                rank, status, payload = q.get(timeout=5)
                got[rank] = (status, payload)
            except queue.Empty:
                dead = [r for r, p in enumerate(procs) if not p.is_alive() and r not in got]
                if dead or time.time() - t0 > RUN_TIMEOUT:
                    raise AssertionError("ranks %s ended without a result, or the run passed %d s" % (dead, RUN_TIMEOUT))
    finally:
        for p in procs:
            p.join(timeout=30)
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=10)
            if p.is_alive():
                p.kill()
                p.join(timeout=10)
    assert not any(p.is_alive() for p in procs) and not multiprocessing.active_children(), \
        "a worker process outlived the run"
    for rank, (status, payload) in sorted(got.items()):
        if status == "skip":
            pytest.skip(payload)
        assert status == "done", "rank %d: %s" % (rank, payload)
    return got, wenv, time.time() - t0


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("G", [2, 3])
def test_every_rank_computes_what_one_process_computes(G, name, env):
    got, wenv, _ = world_outcomes(G, env)
    res, _ = got[0][1][name]
    for rank in range(1, G):
        assert got[rank][1][name][0] == digest(res), "rank %d disagrees with rank 0" % rank
    assert res[0] == "ok" or name.startswith("error-"), res
    CHECKS[name](res[1] if res[0] == "ok" else res, wenv)
