"""oracle/oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT.

CPU restatement of the reference's shuffle hot path (SURVEY.md §8a):

* `libdpk_oracle.so` (oracle/dpk_oracle.c) through ctypes: vector hash /
  partition / map-task / merge / group over numpy columns -- fast enough to
  check the CUDA path at 1e6..1e8 rows in seconds;
* pure-Python loops that mirror the reference line by line (dict per bucket,
  dict merge), used for tiny cases, for object keys (str/bytes/tuple) and as the
  *faithful* CPU baseline ("port": the reference is CPython dict loops).

Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl
reference) may import this module.  Parity is pinned against
tests/golden/*.json (captured from the real reference by
tests/golden/make_golden.py) in tests/test_oracle_golden.py.

Reference citations are relative to the reference root.
"""
import bisect
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

K_I64, K_I32, K_F64, K_U64, K_F32 = 0, 1, 2, 3, 4
V_I64, V_F64 = 0, 1
OPS = {"sum": 0, "min": 1, "max": 2, "prod": 3, "and": 4, "or": 5, "xor": 6, "first": 7, "last": 8}

_KIND_OF = {np.dtype(np.int64): K_I64, np.dtype(np.int32): K_I32, np.dtype(np.float64): K_F64,
            np.dtype(np.uint64): K_U64, np.dtype(np.float32): K_F32}


def build():
    """Compile the C restatement (and, if the reference is present, _ref)."""
    subprocess.check_call(["make", "-s", "-C", _HERE, "all"])
    from oracle import build_reference
    if os.path.exists(os.path.join(build_reference.REF, "dpark", "portable_hash.pyx")):
        subprocess.call(["make", "-s", "-C", _HERE, "ref", "REF=" + build_reference.REF])


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "libdpk_oracle.so")
        if not os.path.exists(path):
            build()
        L = C.CDLL(path)
        i64, i32, vp, dbl = C.c_int64, C.c_int32, C.c_void_p, C.c_double
        L.orc_hash_i64.restype = i64; L.orc_hash_i64.argtypes = [i64]
        L.orc_hash_u64.restype = i64; L.orc_hash_u64.argtypes = [C.c_uint64]
        L.orc_hash_f64.restype = i64; L.orc_hash_f64.argtypes = [dbl]
        L.orc_hash_bytes.restype = i64; L.orc_hash_bytes.argtypes = [C.c_char_p, i64]
        L.orc_hash_utf8.restype = i64; L.orc_hash_utf8.argtypes = [C.c_char_p, i64]
        L.orc_hash_codepoints.restype = i64; L.orc_hash_codepoints.argtypes = [vp, i64]
        L.orc_hash_tuple.restype = i64; L.orc_hash_tuple.argtypes = [vp, i64]
        L.orc_partition.restype = i32; L.orc_partition.argtypes = [i64, i32, vp, i32]
        L.orc_hash_vec.restype = None; L.orc_hash_vec.argtypes = [vp, C.c_int, i64, vp]
        L.orc_hash_bytes_vec.restype = None
        L.orc_hash_bytes_vec.argtypes = [vp, vp, i64, C.c_int, vp]
        L.orc_partition_vec.restype = None
        L.orc_partition_vec.argtypes = [vp, i64, i32, vp, i32, vp]
        L.orc_merge.restype = i64
        L.orc_merge.argtypes = [vp, vp, C.c_int, i64, C.c_int, vp, vp]
        L.orc_map_task.restype = i64
        L.orc_map_task.argtypes = [vp, vp, vp, C.c_int, i64, i32, vp, i32, C.c_int, C.c_int,
                                   vp, vp, vp]
        L.orc_group.restype = i64
        L.orc_group.argtypes = [vp, vp, i64, vp, vp, vp]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


# ----------------------------------------------------------------------------
# a1: portable_hash of one Python object (dpark/portable_hash.pyx:51-70)
# ----------------------------------------------------------------------------
def portable_hash(obj):
    L = lib()
    t = type(obj)
    if obj is None:
        return 1315925605                       # portable_hash.pyx:53-54
    if t is bytes:
        return L.orc_hash_bytes(obj, len(obj))  # :55-56 -> string_hash :17-32
    if t is str:
        cps = np.array([ord(c) for c in obj], dtype=np.uint32)
        return L.orc_hash_codepoints(_p(cps), len(cps))   # :57-58 -> unicode_hash :34-48
    if t is tuple:
        hs = np.array([portable_hash(x) for x in obj], dtype=np.int64)
        return L.orc_hash_tuple(_p(hs), len(hs))          # :59-60 -> tuple_hash :3-15
    if t is int:
        if -2 ** 63 <= obj < 2 ** 63:
            return L.orc_hash_i64(obj)
        # big ints: CPython long_hash, same formula, arbitrary precision
        m = (1 << 61) - 1
        h = abs(obj) % m
        h = -h if obj < 0 else h
        return -2 if h == -1 else h
    if t is float:
        return L.orc_hash_f64(obj)
    if isinstance(obj, np.number):              # :64-67
        if isinstance(obj, np.floating):
            return L.orc_hash_f64(float(obj))
        v = int(obj)
        return L.orc_hash_u64(v) if v >= 2 ** 63 else L.orc_hash_i64(v)
    raise TypeError('%s is unhashable by portable_hash' % t)   # :70


def get_partition(key, P, thresholds=None):
    """HashPartitioner.getPartition, dpark/dependency.py:229-233."""
    h = portable_hash(key)
    if thresholds is None:
        return h % P
    return bisect.bisect(thresholds, h)


# ----------------------------------------------------------------------------
# vector entry points over numpy columns
# ----------------------------------------------------------------------------
def hash_vec(keys):
    keys = np.ascontiguousarray(keys)
    out = np.empty(len(keys), dtype=np.int64)
    lib().orc_hash_vec(_p(keys), _KIND_OF[keys.dtype], len(keys), _p(out))
    return out


def hash_bytes_vec(data, offsets, mode):
    """mode 0 = bytes keys (signed chars), 1 = str keys stored as UTF-8."""
    data = np.ascontiguousarray(data, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    n = len(offsets) - 1
    out = np.empty(n, dtype=np.int64)
    if data.size == 0:
        data = np.zeros(1, dtype=np.uint8)
    lib().orc_hash_bytes_vec(_p(data), _p(offsets), n, mode, _p(out))
    return out


def partition_vec(hashes, P, thresholds=None):
    hashes = np.ascontiguousarray(hashes, dtype=np.int64)
    out = np.empty(len(hashes), dtype=np.int32)
    if thresholds is None:
        lib().orc_partition_vec(_p(hashes), len(hashes), P, None, 0, _p(out))
    else:
        thr = np.ascontiguousarray(thresholds, dtype=np.int64)
        lib().orc_partition_vec(_p(hashes), len(hashes), P, _p(thr), len(thr), _p(out))
    return out


def _key_bits(keys):
    """int64 identity of a key column for the C loops: integers widened; floats keyed by the bits of their
    canonical float64 (`arr + 0.0`: -0.0 and 0.0 are one Python dict key, spelled 0.0, as dpark_b200/columnar.py
    does), so distinct floats stay distinct keys."""
    keys = np.asarray(keys)
    if keys.dtype.kind == "f":
        return np.ascontiguousarray(keys.astype(np.float64) + 0.0).view(np.int64)
    return np.ascontiguousarray(keys, dtype=np.int64)


def _keys_from_bits(bits, dtype):
    """Inverse of _key_bits for the keys a C loop returns: floats come back in their input dtype."""
    return bits.view(np.float64).astype(dtype) if dtype.kind == "f" else bits


def _vals8(vals):
    vals = np.asarray(vals)
    if vals.dtype.kind == "f":
        return np.ascontiguousarray(vals, dtype=np.float64), V_F64
    return np.ascontiguousarray(vals, dtype=np.int64), V_I64


def map_task(keys, vals, P, op="sum", thresholds=None, combine=True):
    """ShuffleMapTask._run (dpark/task.py:209-226) over one input split.
    Returns (bucket_keys, bucket_vals, bucket_offsets[P+1]) bucket-major,
    each bucket in first-seen order.  combine=False keeps every row (the layout
    the CUDA partition kernel produces before any combine).  Integer keys come back
    as int64, float keys in their own dtype."""
    keys = np.ascontiguousarray(keys)
    h = hash_vec(keys)
    k64 = _key_bits(keys)
    v8, vk = _vals8(vals)
    n = len(k64)
    ok = np.empty(n, dtype=np.int64)
    ov = np.empty(n, dtype=v8.dtype)
    offs = np.empty(P + 1, dtype=np.int64)
    if thresholds is None:
        thr_p, nthr = None, 0
    else:
        thr = np.ascontiguousarray(thresholds, dtype=np.int64)
        thr_p, nthr = _p(thr), len(thr)
    tot = lib().orc_map_task(_p(k64), _p(h), _p(v8), vk, n, P, thr_p, nthr, OPS[op],
                             1 if combine else 0, _p(ok), _p(ov), _p(offs))
    return _keys_from_bits(ok[:tot], keys.dtype), ov[:tot], offs


def merge(keys, vals, op="sum"):
    """DiskHashMerger._merge (dpark/shuffle.py:600-608): distinct keys in
    first-seen order with combined values."""
    keys = np.asarray(keys)
    k64 = _key_bits(keys)
    v8, vk = _vals8(vals)
    n = len(k64)
    ok = np.empty(n, dtype=np.int64)
    ov = np.empty(n, dtype=v8.dtype)
    nd = lib().orc_merge(_p(k64), _p(v8), vk, n, OPS[op], _p(ok), _p(ov))
    return _keys_from_bits(ok[:nd], keys.dtype), ov[:nd]


def group(keys, vals):
    """OrderedGroupByDiskHashMerger (dpark/shuffle.py:626-646): CSR
    (keys, offsets, values); rows must arrive concatenated in map_id order."""
    keys = np.asarray(keys)
    k64 = _key_bits(keys)
    v = np.ascontiguousarray(vals)
    assert v.dtype.itemsize == 8
    n = len(k64)
    ok = np.empty(n, dtype=np.int64)
    oo = np.empty(n + 1, dtype=np.int64)
    ov = np.empty(n, dtype=v.dtype)
    nd = lib().orc_group(_p(k64), _p(v.view(np.int64)), n, _p(ok), _p(oo), _p(ov.view(np.int64)))
    return _keys_from_bits(ok[:nd], keys.dtype), oo[:nd + 1], ov


def reduce_by_key(key_splits, val_splits, P, op="sum", thresholds=None):
    """Whole path for reduceByKey over M input splits: M map tasks
    (task.py:209-226) -> per reducer, fetch every map's bucket in map order and
    merge (shuffle.py:378-398, 600-608).  Returns a list of P (keys, vals)."""
    maps = [map_task(k, v, P, op, thresholds) for k, v in zip(key_splits, val_splits)]
    out = []
    for r in range(P):
        ks = [mk[mo[r]:mo[r + 1]] for mk, mv, mo in maps]
        vs = [mv[mo[r]:mo[r + 1]] for mk, mv, mo in maps]
        if ks:
            out.append(merge(np.concatenate(ks), np.concatenate(vs), op))
        else:
            out.append((np.empty(0, np.int64), np.empty(0, np.int64)))
    return out


def group_by_key(key_splits, val_splits, P, thresholds=None):
    """groupByKey with ordered_group=True semantics: list of P CSR triples."""
    maps = [map_task(k, v, P, "sum", thresholds, combine=False)
            for k, v in zip(key_splits, val_splits)]
    out = []
    for r in range(P):
        ks = np.concatenate([mk[mo[r]:mo[r + 1]] for mk, mv, mo in maps]) if maps else np.empty(0, np.int64)
        vs = np.concatenate([mv[mo[r]:mo[r + 1]] for mk, mv, mo in maps]) if maps else np.empty(0, np.int64)
        out.append(group(ks, vs))
    return out


# ----------------------------------------------------------------------------
# pure-Python restatement (mirrors the reference loops; any hashable key kind)
# ----------------------------------------------------------------------------
def py_shuffle_map_task(rows, P, create_combiner, merge_value, thresholds=None,
                        hash_fn=portable_hash):
    """dpark/task.py:209-226 -- P dicts {k: combiner}."""
    buckets = [{} for _ in range(P)]
    for item in rows:
        k, v = item
        h = hash_fn(k)
        p = h % P if thresholds is None else bisect.bisect(thresholds, h)
        bucket = buckets[p]
        r = bucket.get(k, None)
        if r is not None:
            bucket[k] = merge_value(r, v)
        else:
            bucket[k] = create_combiner(v)
    return buckets


def py_merge(batches, merge_combiners):
    """dpark/shuffle.py:600-608 -- batches: iterable of lists of (k, combiner)."""
    combined = {}
    for items in batches:
        for k, v in items:
            o = combined.get(k)
            combined[k] = merge_combiners(o, v) if o is not None else v
    return combined


def py_ordered_group_merge(batches_with_map_id, merge_combiners):
    """dpark/shuffle.py:626-646 -- values ordered by map_id then arrival."""
    from functools import reduce
    combined = {}
    for map_id, items in batches_with_map_id:
        for k, v in items:
            combined.setdefault(k, []).append((map_id, v))
    out = {}
    for k, ivs in combined.items():
        ivs.sort(key=lambda t: t[0])
        out[k] = reduce(merge_combiners, (v for _, v in ivs))
    return out


def py_reduce_by_key(splits, P, func, thresholds=None, hash_fn=portable_hash):
    """reduceByKey = Aggregator(identity, func, func) (dpark/rdd.py:543-545).
    splits: list of lists of (k, v).  Returns list of P dicts."""
    maps = [py_shuffle_map_task(s, P, lambda x: x, func, thresholds, hash_fn) for s in splits]
    return [py_merge((list(m[r].items()) for m in maps), func) for r in range(P)]


def py_group_by_key(splits, P, thresholds=None, hash_fn=portable_hash):
    """groupByKey with GroupByAggregator (dpark/dependency.py:107-118) under
    ordered_group=True.  Returns list of P dicts {k: [values]}."""
    def create(x):
        return [x]

    def merge_value(c, x):
        c.append(x)
        return c

    def merge_comb(x, y):
        x.extend(y)
        return x
    maps = [py_shuffle_map_task(s, P, create, merge_value, thresholds, hash_fn) for s in splits]
    return [py_ordered_group_merge(((mid, list(m[r].items())) for mid, m in enumerate(maps)),
                                   merge_comb) for r in range(P)]


def split_like_parallelize(seq, num_slices):
    """ParallelCollection.slice, dpark/rdd.py:1562, 1576-1598: numSlices is
    capped to len(seq); chunks of ceil(len/numSlices); trailing chunks may be
    empty; an empty input is one empty split."""
    seq = list(seq)
    m = len(seq)
    if not m:
        return [[]]
    k = max(1, min(m, num_slices))
    n = m // k + (1 if m % k else 0)
    return [seq[i * n:i * n + n] for i in range(k)]
