"""Reduce-side parity at IEEE special values and at the edges of int64, on every dpk_set_option variant of the merge.

The oracle is not the reference here: it restates Python's `min(x, y)`, whose answer on a NaN or a signed-zero tie
depends on the fetch order.  Every expected value below is computed in this file, per key, from the key's values:

  min / max   IEEE 754-2019 minimum / maximum: NaN if any value is NaN, otherwise the usual one with -0.0 < +0.0;
              compared bit for bit.
  sum         exact rational sum (math.fsum is its rounding).  NaN if a value is NaN or both infinities occur, else an
              infinity if one occurs, and the sign rule of IEEE zeros for all-zero keys: bit for bit.  Otherwise
              |gpu - exact| <= gamma(n-1) * sum|v| with gamma(k) = k u / (1 - k u), u = 2^-53 and n the key's rows: the
              bound of every summation order, also of a merge done in two rounds (map_combine).  A key whose partial
              sums can overflow in one order and not in another may give any of those results (one case:
              [DBL_MAX, DBL_MAX, -DBL_MAX] gives DBL_MAX or +inf).
  prod        exact rational product, |gpu - exact| <= gamma(n-1) * |exact| where nothing underflows or overflows;
              a zero's sign is the XOR of the values' signs, inf with a zero is NaN, inf with finite nonzero values is
              +-inf (bit for bit); a product of values |v| >= 1 past DBL_MAX is +-inf in every order.
  ints        exact Python ints.

-m gpu."""
import math
import operator
import struct
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tests.shuffle_cases import AG2_CAP, REDUCE_VARIANTS, dpk_options, variant_id  # noqa: F401

pytestmark = pytest.mark.gpu

NAN = float("nan")
INF = float("inf")
DBL_MAX = float(np.finfo(np.float64).max)
DBL_MIN = float(np.finfo(np.float64).tiny)          # 2.2250738585072014e-308
FLT_MAX = float(np.finfo(np.float32).max)
FLT_MIN = float(np.finfo(np.float32).tiny)
I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1
I32_MIN, I32_MAX = -2 ** 31, 2 ** 31 - 1
NAN_PAYLOAD = struct.unpack("<d", struct.pack("<Q", 0x7FF800000000ABCD))[0]
NEG_NAN = struct.unpack("<d", struct.pack("<Q", 0xFFF8000000000000))[0]

SPECIALS = {
    "f64": [NAN, 0.0, -0.0, INF, -INF, 5e-324, -5e-324, DBL_MIN, -DBL_MIN, DBL_MAX, -DBL_MAX],
    "f32": [NAN, 0.0, -0.0, INF, -INF, 2.0 ** -149, -2.0 ** -149, FLT_MIN, -FLT_MIN, FLT_MAX, -FLT_MAX],
}
NP = {"i64": np.int64, "i32": np.int32, "f64": np.float64, "f32": np.float32}
HOT = AG2_CAP + 452                                  # rows of each hot key: more than one staging window

# every merge variant, and the default one behind a map-side combine (two merge rounds)
VARIANTS = [(opts, False) for opts in REDUCE_VARIANTS] + [({}, True)]
VARIANT_IDS = [variant_id(o) + (",map_combine" if mc else "") for o, mc in VARIANTS]


def _bits(x):
    return struct.pack("<d", x)


# ------------------------------------------------------------------------------------------------ references
def _is_neg(x):
    return math.copysign(1.0, x) < 0


def ieee_min(vs):
    if any(math.isnan(x) for x in vs):
        return NAN
    m = min(vs)
    if m == 0:
        return -0.0 if any(x == 0 and _is_neg(x) for x in vs) else 0.0
    return m


def ieee_max(vs):
    if any(math.isnan(x) for x in vs):
        return NAN
    m = max(vs)
    if m == 0:
        return 0.0 if any(x == 0 and not _is_neg(x) for x in vs) else -0.0
    return m


def _fixed(x):
    """A finite double as the exact integer x * 2^1074 (every double is a multiple of 2^-1074)."""
    n, d = x.as_integer_ratio()
    return n << (1074 - (d.bit_length() - 1))


DBL_MAX_FIXED = _fixed(DBL_MAX)


def expect_sum(vs):
    if any(math.isnan(x) for x in vs) or (INF in vs and -INF in vs):
        return ("bits", NAN)
    if INF in vs or -INF in vs:
        return ("bits", INF if INF in vs else -INF)
    if all(x == 0 for x in vs):
        return ("bits", -0.0 if all(_is_neg(x) for x in vs) else 0.0)
    fx = [_fixed(x) for x in vs]
    exact = sum(fx)
    pos, neg = sum(f for f in fx if f > 0), sum(f for f in fx if f < 0)
    if pos > DBL_MAX_FIXED or -neg > DBL_MAX_FIXED:     # a partial sum overflows in some orders
        allowed = [float(Fraction(exact, 2 ** 1074))] if abs(exact) <= DBL_MAX_FIXED else []
        allowed += [INF] if pos > DBL_MAX_FIXED else []
        allowed += [-INF] if -neg > DBL_MAX_FIXED else []
        allowed += [NAN] if pos > DBL_MAX_FIXED and -neg > DBL_MAX_FIXED else []
        return ("oneof", allowed)
    return ("sum", exact, pos - neg, len(vs) - 1)


def expect_prod(vs):
    if any(math.isnan(x) for x in vs):
        return ("bits", NAN)
    negative = sum(_is_neg(x) for x in vs) % 2 == 1
    has_inf, has_zero = any(math.isinf(x) for x in vs), any(x == 0 for x in vs)
    if has_inf and has_zero:
        return ("bits", NAN)
    if has_inf:
        return ("bits", -INF if negative else INF)
    if has_zero:
        return ("bits", -0.0 if negative else 0.0)
    exact = Fraction(1)
    for x in vs:
        exact *= Fraction(x)
    if abs(exact) > DBL_MAX and all(abs(x) >= 1 for x in vs):   # partial products only grow: inf in every order
        return ("bits", -INF if negative else INF)
    if len(vs) > 1:   # the relative bound needs every partial product in the normal range; the cases keep it there
        assert all(2.0 ** -500 < abs(x) < 2.0 ** 500 for x in vs), vs
    return ("prod", exact, len(vs) - 1)


def expect_int(op, vs):
    f = {"sum": operator.add, "min": min, "max": max, "prod": operator.mul, "and": operator.and_,
         "or": operator.or_, "xor": operator.xor}[op]
    r = vs[0]
    for x in vs[1:]:
        r = f(r, x)
    assert I64_MIN <= r <= I64_MAX, (op, vs)
    return ("int", r)


def expect(op, vs):
    if isinstance(vs[0], int):
        return expect_int(op, vs)
    if op == "min":
        return ("bits", ieee_min(vs))
    if op == "max":
        return ("bits", ieee_max(vs))
    return expect_sum(vs) if op == "sum" else expect_prod(vs)


def agrees(got, want):
    kind = want[0]
    if kind == "int":
        return int(got) == want[1]
    got = float(got)
    if kind == "bits":
        return math.isnan(got) if math.isnan(want[1]) else _bits(got) == _bits(want[1])
    if kind == "oneof":
        return any(agrees(got, ("bits", w)) for w in want[1])
    if not math.isfinite(got):
        return False
    if kind == "sum":      # |got - exact| <= k u / (1 - k u) * sum|v|, in integers: |d| * (2^53 - k) <= k * sum|v|
        _, exact, mag, k = want
        return abs(_fixed(got) - exact) * (2 ** 53 - k) <= k * mag
    _, exact, k = want     # prod
    return abs(Fraction(got) - exact) * (2 ** 53 - k) <= k * abs(exact)


# ------------------------------------------------------------------------------------------------ running a case
def _to_kind(vs, vk):
    """Python values as the value column of kind vk holds them, and back as the Python numbers the kernel sees."""
    arr = np.array(vs, dtype=np.float64 if vk[0] == "f" else np.int64).astype(NP[vk])
    return arr, [float(x) for x in arr.astype(np.float64)] if vk[0] == "f" else [int(x) for x in arr]


def _background(kk, vk, op, n, rng):
    """n rows of random keys >= 0 (the edge keys are negative), about three rows per key, ordinary values."""
    hi = I32_MAX if kk == "i32" else I64_MAX
    pool = rng.integers(0, hi, max(n // 3, 1), dtype=np.int64)
    keys = pool[rng.integers(0, len(pool), n)]
    if vk[0] == "f":
        vals = rng.random(n) + 0.5 if op == "prod" else rng.standard_normal(n) * 1000.0
    elif op == "prod":
        vals = rng.choice(np.array([-1, 1, 2, 3]), n)
    elif op in ("and", "or", "xor", "min", "max"):
        info = np.iinfo(NP[vk])
        vals = rng.integers(info.min, info.max, n, dtype=np.int64, endpoint=True)
    else:
        vals = rng.integers(-2 ** 31, 2 ** 31, n)
    return keys, vals


def run_case(kk, vk, op, groups, variant, rng, background=12_000, P=5):
    """groups: {key: [values]} of edge keys (negative, or INT64_MIN).  Reduces them with `background` ordinary rows,
    the rows shuffled over three map splits, and checks every key's partition and value against its reference."""
    from dpark_b200 import shuffle
    map_combine = variant[1]
    bk, bv = _background(kk, vk, op, background, rng)
    keys, vals = [bk], [bv]
    for k, vs in groups.items():
        keys.append(np.full(len(vs), k, dtype=np.int64))
        vals.append(np.array(vs, dtype=object))
    k = np.concatenate(keys).astype(NP[kk])
    v, seen = _to_kind(np.concatenate(vals).tolist(), vk)
    perm = rng.permutation(len(k))
    k, v = k[perm], v[perm]
    seen = [seen[i] for i in perm.tolist()]
    per_key = {}
    for key, x in zip(k.tolist(), seen):
        per_key.setdefault(key, []).append(x)
    ks, vs = np.array_split(k, 3), np.array_split(v, 3)
    res = shuffle.reduce_by_key([torch.from_numpy(x).cuda() for x in ks], [torch.from_numpy(x).cuda() for x in vs],
                                P, op, map_combine=map_combine)
    all_keys = np.array(sorted(per_key), dtype=np.int64)
    want_part = dict(zip(all_keys.tolist(), orc.partition_vec(orc.hash_vec(all_keys.astype(NP[kk])), P).tolist()))
    assert [p for p, _, _ in res] == list(range(P))
    bad = []
    for p, gk, gv in res:
        gk, gv = gk.cpu().numpy().astype(np.int64), gv.cpu().numpy()
        o = np.argsort(gk, kind="stable")
        gk, gv = gk[o], gv[o]
        assert gk.tolist() == [x for x in all_keys.tolist() if want_part[x] == p], (variant, p)
        for key, got in zip(gk.tolist(), gv.tolist()):
            want = expect(op, per_key[key])
            if not agrees(got, want):
                shown = float(Fraction(want[1], 2 ** 1074)) if want[0] == "sum" else want[1]
                bad.append((key, len(per_key[key]), got, want[0], shown))
    assert not bad, "%s %s %s/%s: %d keys differ, first: %s" % (VARIANT_IDS[VARIANTS.index(variant)], op, kk, vk,
                                                               len(bad), bad[:6])


# ------------------------------------------------------------------------------------------------ float cases
def _mixtures(vk, op):
    """Small keys whose result does not depend on the merge order under the rules above."""
    big, tiny = (DBL_MAX, 5e-324) if vk == "f64" else (FLT_MAX, 2.0 ** -149)
    m = [
        [NAN, 1.0], [1.0, NAN, -3.0], [NAN_PAYLOAD, 2.0, NEG_NAN], [-0.0, NAN, 0.0],
        [0.0, -0.0], [-0.0, 0.0, -0.0], [0.0, 0.0], [-0.0, -0.0, -0.0], [-0.0, 5.0, 0.0, -2.5],
        [INF, -INF], [INF, 1.0], [-INF, -5.0, 2.0], [INF, INF, 3.0], [NAN, INF, -INF], [-INF, -0.0, 0.0],
        [1.5] * 40, [-0.75, 3.0, -1.25, 2.0] * 8, [1e16, 1.0, -1e16], [big / 4, -big / 8, big / 8],
    ]
    if op in ("sum", "min", "max"):     # products of these leave the range the relative bound is stated for
        m += [[tiny] * 7, [tiny, -tiny, tiny], [3 * tiny, tiny, 2 * tiny, -tiny] * 5, [big, big, -big]]
    if op == "prod":
        m += [[big, 2.0, 4.0], [-big, -big, big]] if vk == "f64" else [[big, big, -big]]
    return m


def _hot_groups(op, rng):
    """Keys of HOT rows each: every fine bucket holding one takes the multi-window path (or agg_pipe's second
    launch).  All NaN, all -0.0, three NaNs among finite values, random zeros, one -0.0 among +0.0, and (not for
    prod, whose partial products would leave the range) the finite values alone."""
    finite = (rng.standard_normal(HOT) * 100.0).tolist()
    mixed_nan = list(finite)
    for i in rng.choice(HOT, 3, replace=False).tolist():
        mixed_nan[i] = NAN
    zeros = [-0.0 if b else 0.0 for b in (rng.random(HOT) < 0.5).tolist()]
    hot = [[NAN] * HOT, [-0.0] * HOT, mixed_nan, zeros, [0.0] * (HOT - 1) + [-0.0]]
    return hot if op == "prod" else hot + [finite]


def float_groups(vk, op, rng):
    groups, key = {}, -1000
    for vs in [[x] for x in SPECIALS[vk]] + _hot_groups(op, rng) + _mixtures(vk, op):
        groups[key] = vs
        key -= 1
    return groups


OPS_F = ["sum", "min", "max", "prod"]
KINDS = [("i64", "f64"), ("i32", "f32"), ("i64", "f32"), ("i32", "f64")]   # i64+f64 and i32+f32 travel packed
# variant x op, and the (key, value) kinds as a Latin square over them: every variant meets min and max (and every
# op) with the single-value, hot and mixed keys, and every pair of the four factors occurs
FLOAT_CASES = [(v, op) + KINDS[(v + j) % 4] for v in range(len(VARIANTS)) for j, op in enumerate(OPS_F)]


@pytest.mark.parametrize("case", FLOAT_CASES, ids=["%s-%s-%s-%s" % ((VARIANT_IDS[c[0]],) + c[1:]) for c in FLOAT_CASES])
def test_float_special_values_on_every_variant(case, dpk_options):
    """Single-value keys for every special value (NaN, +-0, +-inf, the smallest subnormal, the smallest normal and
    the largest finite value of the value kind), hot keys of all NaN, all -0.0, NaN among finite values and mixed
    zeros, small order-free mixtures, and background keys that fill the fine buckets."""
    v, op, kk, vk = case
    rng = np.random.default_rng(1000 + FLOAT_CASES.index(case))
    dpk_options(VARIANTS[v][0])
    run_case(kk, vk, op, float_groups(vk, op, rng), VARIANTS[v], rng)


SIDE_MIXTURES = [[NAN, 1.0], [1.0, NAN], [0.0, -0.0], [-0.0, 0.0], [INF, -INF], [-0.0] * 5]


@pytest.mark.parametrize("vk", ["f64", "f32"])
@pytest.mark.parametrize("variant", range(len(VARIANTS)), ids=VARIANT_IDS)
def test_float_special_values_on_the_int64_min_key(variant, vk, dpk_options):
    """The key whose bits equal the slot tables' free marker (INT64_MIN) is merged in a side slot by the kernels that
    have one.  It holds, one run each, every single special value and a few order-free mixtures, under every op."""
    rng = np.random.default_rng(variant * 2 + (vk == "f32"))
    dpk_options(VARIANTS[variant][0])
    for op in OPS_F:
        for vs in [[x] for x in SPECIALS[vk]] + SIDE_MIXTURES:
            run_case("i64", vk, op, {I64_MIN: vs, -7: vs}, VARIANTS[variant], rng, background=2000, P=3)


IDENTITY = {"min": I64_MAX, "max": I64_MIN, "and": -1, "prod": 1, "sum": 0, "or": 0, "xor": 0}


@pytest.mark.parametrize("variant", range(len(VARIANTS)), ids=VARIANT_IDS)
def test_int_single_values_equal_to_the_identity(variant, dpk_options):
    """A key whose only value equals the op's identity (INT64_MAX for min, INT64_MIN for max, -1 for and, 1 for prod,
    0 for sum / or / xor) must come back with that value, also on the INT64_MIN key: a merge that took "accumulator
    == identity" for "not yet seeded" would still pass every other test.  The int64 extremes, 0 and -1 ride along;
    int32 values use the int32 extremes."""
    rng = np.random.default_rng(500 + variant)
    dpk_options(VARIANTS[variant][0])
    for vk in ("i64", "i32"):
        lo, hi = (I64_MIN, I64_MAX) if vk == "i64" else (I32_MIN, I32_MAX)
        for op, ident in IDENTITY.items():
            ident = min(max(ident, lo), hi)
            singles = [ident, lo, hi, 0, -1]
            groups = {-100 - i: [x] for i, x in enumerate(singles)}
            run_case("i64" if vk == "i64" else "i32", vk, op, groups, VARIANTS[variant], rng, background=3000, P=4)
            for x in singles:
                run_case("i64", vk, op, {I64_MIN: [x]}, VARIANTS[variant], rng, background=500, P=2)


# ------------------------------------------------------------------------------------------------ operator surface
def ctx():
    sys.argv = [sys.argv[0]]
    from dpark_b200 import DparkContext
    return DparkContext("local")


SURFACE_GROUPS = {0: [1.0, NAN], 1: [NAN, 1.0], 2: [0.0, -0.0], 3: [-0.0, 0.0], 4: [NAN], 5: [2.0, -0.0, 0.0, NAN, 3.0],
                  6: [-0.0, -0.0], 7: [0.0, 5.0, -0.0], 8: [-INF, NAN], 9: [4.0, -1.5]}


@pytest.mark.parametrize("op,funcs", [
    ("min", [min, lambda x, y: min(x, y), lambda x, y: x if x < y else y, lambda x, y: y if y <= x else x]),
    ("max", [max, lambda x, y: max(x, y), lambda x, y: x if x > y else y, lambda x, y: y if y >= x else x]),
])
def test_min_max_over_nan_and_signed_zeros_do_not_depend_on_the_spelling(op, funcs):
    """Python's min(x, y) keeps its first operand on a NaN or a tie and `x if x < y else y` its second; both are
    recognised as min, and both give the IEEE minimum (maximum) on the GPU path, whatever order the rows come in: the
    keys hold their values in both orders ([1.0, nan] and [nan, 1.0], [0.0, -0.0] and [-0.0, 0.0]), in one map split
    and spread over three."""
    rows = [(k, x) for k, vs in SURFACE_GROUPS.items() for x in vs]
    dc = ctx()
    for f in funcs:
        for splits in (1, 3):
            got = dict(dc.parallelize(rows, splits).reduceByKey(f, 4).collect())
            assert sorted(got) == sorted(SURFACE_GROUPS)
            for k, vs in SURFACE_GROUPS.items():
                want = ieee_min(vs) if op == "min" else ieee_max(vs)
                assert agrees(got[k], ("bits", want)), (f, splits, k, vs, got[k])


MUL_OK = {"a": [2] * 62, "b": [2 ** 40] * 5 + [0] + [2 ** 40] * 5, "c": [46340] * 4, "d": [-2 ** 31] * 2,
          "e": [3, -5, 7], "f": [-2] * 62 + [-1], "g": [I32_MAX, I32_MAX]}
MUL_OVERFLOW = [[2 ** 32, 2 ** 32], [2] * 63, [I32_MAX] * 3, [7, 7, 73, 127, 337, 92737, 649657], [-2] * 63]


@pytest.mark.parametrize("keytype", [int, str])
def test_int_products_are_exact_or_refused(keytype):
    """Integer reduceByKey(mul) multiplies in int64 on the device: the exact product whenever it fits (also past
    wrapped intermediates: a zero among factors totalling 2^400 gives 0), OverflowError when a key's product could
    leave int64 -- where the reference's big ints would not wrap -- for int and str keys alike."""
    dc = ctx()
    key = (lambda k: 10 + ord(k)) if keytype is int else (lambda k: "key-" + k)
    rows = [(key(k), x) for k, vs in MUL_OK.items() for x in vs]
    rows = [rows[i] for i in np.random.default_rng(2).permutation(len(rows)).tolist()]
    got = dict(dc.parallelize(rows, 3).reduceByKey(lambda a, b: a * b, 4).collect())
    assert got == {key(k): math.prod(vs) for k, vs in MUL_OK.items()}
    for vs in MUL_OVERFLOW:
        bad = rows + [(key("z"), x) for x in vs]
        with pytest.raises(OverflowError):
            dc.parallelize(bad, 3).reduceByKey(operator.mul, 4).collect()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("where", ["first_split", "last_split"])
def test_nan_keys_of_columns_raise_type_error_in_reduce_by_key(dtype, where):
    """NaN keys of a ColumnarRDD: TypeError, as on the row path and in groupByKey / join, instead of one merged key
    (the device keys a float by its bits; CPython keeps every NaN row apart)."""
    k = np.array([1.0, 2.0, -0.0, 3.0, 4.0, 0.0], dtype=dtype)
    k[0 if where == "first_split" else -1] = NAN
    v = np.arange(len(k), dtype=np.float64)
    dc = ctx()
    with pytest.raises(TypeError):
        dc.parallelizeColumns(k, v, 3).reduceByKey(operator.add, 2).collect()
    with pytest.raises(TypeError):
        dc.parallelizeColumns(torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda(), 3).reduceByKey(min, 2).collect()
    with pytest.raises(TypeError):
        dc.parallelize(list(zip(k.tolist(), v.tolist())), 3).reduceByKey(operator.add, 2).collect()
    k[np.isnan(k)] = 7.0      # the same columns without the NaN reduce normally
    want = {}
    for x, y in zip(k.tolist(), v.tolist()):
        want[x] = want.get(x, 0.0) + y
    assert dict(dc.parallelizeColumns(k, v, 3).reduceByKey(operator.add, 2).collect()) == want
