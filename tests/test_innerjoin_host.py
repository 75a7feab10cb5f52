"""The device innerJoin on a CPU: the hash table of dpk_common.cuh run through tests/bcastcheck.cu (key normalisation,
slot count, build and probe at colliding keys, special values and the load bound), which calls take the device path,
and join.inner_join_columns on an emulated device.  The device results themselves are checked in
tests/test_gpu_innerjoin.py."""
import ctypes as C
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import cogroup_common as cc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def _bcastcheck():
    path = os.path.join(ROOT, "tests", "_bcastcheck.so")
    if not os.path.exists(path):
        subprocess.call([sys.executable, "-c", "import __graft_entry__ as g; g.build()"], cwd=ROOT)
    if not os.path.exists(path):
        pytest.skip("bcastcheck not built")
    L = C.CDLL(path)
    u64p = C.POINTER(C.c_uint64)
    L.bc_slots.restype = C.c_uint64
    L.bc_slots.argtypes = [C.c_int64]
    L.bc_slot.restype = C.c_uint64
    L.bc_slot.argtypes = [C.c_uint64, C.c_uint64]
    for name, t in (("i32", C.c_int32), ("i64", C.c_int64), ("f32", C.c_float), ("f64", C.c_double)):
        f = getattr(L, "bc_bits_" + name)
        f.restype = C.c_int32
        f.argtypes = [t, u64p]
    L.bc_slot_bytes.restype = C.c_int64
    L.bc_build.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
    L.bc_find.restype = C.c_int32
    L.bc_find.argtypes = [C.c_void_p, C.c_int64, C.c_uint64]
    return L


def _bits(L, x, kind):
    """(ok, normalised bits) of key x read as a column of `kind` would hold it."""
    kb = C.c_uint64()
    ok = getattr(L, "bc_bits_" + kind)(x, C.byref(kb))
    return bool(ok), kb.value


def _u64(x):
    return x & ((1 << 64) - 1)


def _f64_bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


class Table:
    """A table built by the harness from distinct normalised keys (group g = keys[g])."""

    def __init__(self, L, keys):
        self.L = L
        self.S = L.bc_slots(len(keys))
        self.keys = np.array([_u64(k) for k in keys], dtype=np.uint64)
        self.buf = np.zeros(self.S * L.bc_slot_bytes(), np.uint8)
        L.bc_build(self.keys.ctypes.data, len(keys), self.buf.ctypes.data, self.S)

    def find(self, kb):
        return self.L.bc_find(self.buf.ctypes.data, self.S, _u64(kb))


# ------------------------------------------------------------------------------------------------ the table
def test_slot_layout_and_count():
    L = _bcastcheck()
    from dpark_b200 import _native as nv
    assert L.bc_slot_bytes() == 16
    for G, S in ((0, 2), (1, 2), (2, 4), (3, 8), (4, 8), (5, 16), (1 << 20, 1 << 21), ((1 << 20) + 1, 1 << 22)):
        assert L.bc_slots(G) == nv.bcast_slots(G) == S, G


def test_key_normalisation_is_python_equality():
    """Ints widen to int64 whatever their width; floats widen to float64 with -0.0 spelled 0.0 (a dict finds 0.0 under
    -0.0); a float32 key and a float64 key of the same value get the same bits; NaN is refused."""
    L = _bcastcheck()
    for x in (0, 1, -1, -(1 << 31), (1 << 31) - 1):
        assert _bits(L, x, "i32") == _bits(L, x, "i64") == (True, _u64(x))
    for x in (I64_MIN, I64_MAX, 1 << 40):
        assert _bits(L, x, "i64") == (True, _u64(x))
    f32 = np.finfo(np.float32)
    f64 = np.finfo(np.float64)
    for x in (0.0, 1.5, -2.25, float("inf"), float("-inf"), float(f32.smallest_subnormal), float(f32.max),
              -float(f32.smallest_normal)):
        assert _bits(L, x, "f32") == _bits(L, x, "f64") == (True, _f64_bits(x)), x
    for x in (float(f64.smallest_subnormal), -float(f64.smallest_subnormal), float(f64.max), 0.1):
        assert _bits(L, x, "f64") == (True, _f64_bits(x))
    assert _bits(L, -0.0, "f64") == _bits(L, -0.0, "f32") == (True, 0)
    assert _bits(L, 0.1, "f32")[1] != _bits(L, 0.1, "f64")[1]       # float32(0.1) != 0.1, in Python as well
    assert not _bits(L, float("nan"), "f64")[0] and not _bits(L, float("nan"), "f32")[0]
    assert not _bits(L, -float("nan"), "f64")[0]


def _check_table(L, keys, absent):
    t = Table(L, keys)
    for g, k in enumerate(keys):
        assert t.find(k) == g, (g, k)
    for k in absent:
        assert t.find(k) == -1, k
    return t


def test_keys_colliding_in_the_low_bits():
    """Multiples of 2^32 and of 2^40 agree in every bit a small table's mask keeps: the slot function mixes all 64."""
    L = _bcastcheck()
    for step in (1 << 32, 1 << 40):
        keys = [i * step for i in range(-300, 300)]
        t = _check_table(L, keys, [i * step + 1 for i in range(-300, 300)] + [301 * step, -301 * step])
        first = {L.bc_slot(_u64(k), t.S - 1) for k in keys}
        assert len(first) > len(keys) // 2, step


def test_int_extremes_and_small_ints():
    L = _bcastcheck()
    keys = [I64_MIN, -1, 0, I64_MAX, 1, -2, I64_MIN + 1, 1 << 31, -(1 << 31)]
    _check_table(L, keys, [2, -3, I64_MAX - 1, I64_MIN + 2, (1 << 31) + 1])


def test_float_special_values():
    """±0.0 normalise to one key, ±inf and subnormals are keys like any other; probed through the normalisation."""
    L = _bcastcheck()
    sub = float(np.finfo(np.float64).smallest_subnormal)
    vals = [0.0, float("inf"), float("-inf"), sub, -sub, 2 * sub, 1.0, -1.0, float(np.finfo(np.float32).smallest_subnormal)]
    t = _check_table(L, [_bits(L, x, "f64")[1] for x in vals], [_bits(L, x, "f64")[1] for x in (3 * sub, 2.0, -2.0)])
    assert t.find(_bits(L, -0.0, "f64")[1]) == 0
    assert t.find(_bits(L, -0.0, "f32")[1]) == 0
    assert t.find(_bits(L, float(np.finfo(np.float32).smallest_subnormal), "f32")[1]) == len(vals) - 1


@pytest.mark.parametrize("G", [1, 2, 64, 1024, 1 << 14])
def test_tables_at_the_load_bound(G):
    """G a power of two: exactly 2 G slots, half of them full; random keys, and runs of consecutive ints."""
    L = _bcastcheck()
    assert L.bc_slots(G) == 2 * G
    rng = np.random.default_rng(G)
    keys = np.unique(rng.integers(I64_MIN, I64_MAX, 2 * G, dtype=np.int64))[:G]
    rng.shuffle(keys)
    absent = rng.integers(I64_MIN, I64_MAX, 200, dtype=np.int64)
    absent = [int(x) for x in absent if x not in set(keys.tolist())]
    _check_table(L, [int(k) for k in keys], absent)
    _check_table(L, list(range(G)), list(range(G, G + 100)) + [-1])


# ------------------------------------------------------------------------------------------------ path choice
ELIGIBLE = [torch.int32, torch.int64, torch.float32, torch.float64]
INELIGIBLE = [torch.int16, torch.uint8, torch.bool, torch.float16]


def _col(dc, kdt, vdt, n=6, M=2):
    return dc.parallelizeColumns(torch.arange(n).to(kdt), torch.arange(n).to(vdt), M)


def _cls():
    from dpark_b200.join import ColumnarInnerJoinedRDD
    return ColumnarInnerJoinedRDD


@pytest.mark.parametrize("kdt", ELIGIBLE + INELIGIBLE, ids=str)
@pytest.mark.parametrize("vdt", ELIGIBLE + INELIGIBLE, ids=str)
def test_device_inner_join_is_chosen_by_dtypes(kdt, vdt):
    from dpark_b200.rdd import FlatMappedRDD
    dc = cc.ctx()
    same_kind = torch.float64 if kdt.is_floating_point else torch.int64
    ok = _col(dc, same_kind, torch.int64, 3, 1)
    eligible = kdt in ELIGIBLE and vdt in ELIGIBLE
    for big, small in ((_col(dc, kdt, vdt, 6, 3), ok), (ok, _col(dc, kdt, vdt))):
        out = big.innerJoin(small)
        assert isinstance(out, _cls()) == eligible
        assert isinstance(out, FlatMappedRDD) != eligible
        assert out.partitioner is None and len(out) == len(big.splits)


def test_two_dimensional_columns_keep_the_composition():
    from dpark_b200.rdd import ColumnarRDD, FlatMappedRDD
    dc = cc.ctx()
    flat = _col(dc, torch.int64, torch.int64)
    wide = ColumnarRDD(dc, torch.arange(6).reshape(6, 1), torch.arange(6), 2)
    assert isinstance(flat.innerJoin(flat), _cls())
    assert isinstance(wide.innerJoin(flat), FlatMappedRDD)


def test_input_types_choose_the_path():
    from dpark_b200.rdd import ColumnarRDD, FlatMappedRDD
    dc = cc.ctx()
    col = _col(dc, torch.int64, torch.float64)

    class MyColumns(ColumnarRDD):
        pass

    for other in (dc.parallelize([(1, 2)], 1), col.map(lambda kv: kv), col.mapValue(lambda v: v),
                  MyColumns(dc, np.arange(4), np.arange(4), 2), col.union(col), col.filter(bool)):
        assert isinstance(col.innerJoin(other), FlatMappedRDD)
        assert isinstance(other.innerJoin(col), FlatMappedRDD)
    assert isinstance(col.innerJoin(col), _cls())


def test_more_than_one_process_keeps_the_composition(monkeypatch):
    """(The composition itself collects the small side at once, a job of all ranks: only the choice is checked.)"""
    from dpark_b200 import join, spmd
    dc = cc.ctx()
    a, b = _col(dc, torch.int32, torch.float32), _col(dc, torch.int64, torch.int64)
    assert join.inner_join_applies(a, b) and isinstance(a.innerJoin(b), _cls())
    monkeypatch.setattr(spmd, "rank_world", lambda: (0, 2))
    assert not join.inner_join_applies(a, b)


def test_mixed_int_and_float_keys_keep_the_composition_unless_a_side_is_empty():
    from dpark_b200.rdd import FlatMappedRDD
    dc = cc.ctx()
    ints, floats = _col(dc, torch.int32, torch.int64), _col(dc, torch.float32, torch.int64)
    no_ints, no_floats = _col(dc, torch.int64, torch.int64, 0), _col(dc, torch.float64, torch.int64, 0)
    for big, small in ((ints, floats), (floats, ints)):
        out = big.innerJoin(small)
        assert isinstance(out, FlatMappedRDD)
        assert out.collect() == [(k, (v, k)) for k, v in big.collect()]      # 1 == 1.0 in Python's dict
    for big, small in ((ints, no_floats), (floats, no_ints), (no_ints, floats), (no_floats, ints)):
        out = big.innerJoin(small)
        assert isinstance(out, _cls()) and len(out) == len(big.splits)


def test_nothing_is_computed_at_construction(monkeypatch):
    """Building the device innerJoin (and what lies on top of it) touches no device: the CPU has none."""
    from dpark_b200 import engine, join

    def no_device(*a):
        raise AssertionError("the innerJoin ran at construction")

    monkeypatch.setattr(engine, "_device", no_device)
    monkeypatch.setattr(join, "inner_join_columns", no_device)
    dc = cc.ctx()
    a, b = _col(dc, torch.int64, torch.float64), _col(dc, torch.int64, torch.int64)
    out = a.innerJoin(b)
    out.mapValue(lambda v: v[0]).filter(bool)
    assert out._result is None


# ------------------------------------------------------------------------------------------------ emulated device
def _emulated_device(monkeypatch, L):
    """join.inner_join_columns on the CPU: the P = 1 group-by as a dict (groups in first-seen order, ids ascending),
    dpk_bcast_build / probe / emit replaced by loops over the table functions the kernels run (tests/bcastcheck.cu).
    An emit that would read outside the small values raises IndexError here instead of reading past a device
    allocation."""
    from dpark_b200 import engine, grouping, join
    from dpark_b200 import _native as nv

    def group_row_ids(key_chunks, id_chunks, P, thresholds):
        assert P == 1 and thresholds is None
        runs = {}
        for k, i in zip(torch.cat(key_chunks).view(torch.int64).tolist(), torch.cat(id_chunks).tolist()):
            runs.setdefault(k, []).append(i)
        gs = [0]
        for ids in runs.values():
            gs.append(gs[-1] + len(ids))
        return (torch.tensor(list(runs), dtype=torch.int64), torch.tensor(gs, dtype=torch.int64),
                torch.tensor([i for ids in runs.values() for i in ids], dtype=torch.int64),
                torch.tensor([0, gs[-1]], dtype=torch.int64))

    def bcast_build(gk):
        return Table(L, gk.tolist())

    def bcast_probe(table, keys, gs):
        kind = {torch.int32: "i32", torch.int64: "i64", torch.float32: "f32", torch.float64: "f64"}[keys.dtype]
        starts = gs.tolist()
        grp, cnt = [], []
        for x in keys.tolist():
            ok, kb = _bits(L, x, kind)
            g = table.find(kb) if ok else -1
            grp.append(g)
            cnt.append(starts[g + 1] - starts[g] if g >= 0 else 0)
        return torch.tensor(grp, dtype=torch.int32), torch.tensor(cnt, dtype=torch.int64)

    def bcast_emit(keys, lvals, grp, off, gs, ids, rvals, n_out):
        out = (torch.empty(n_out, dtype=keys.dtype), torch.empty(n_out, dtype=lvals.dtype),
               torch.empty(n_out, dtype=rvals.dtype))
        o, g, s, ids = off.tolist(), grp.tolist(), gs.tolist(), ids.tolist()
        assert o[-1] == n_out
        for r in range(keys.numel()):
            for i in range(o[r], o[r + 1]):
                src = ids[s[g[r]] + i - o[r]]
                if not 0 <= src < rvals.numel():
                    raise IndexError("output row %d reads value %d of %d" % (i, src, rvals.numel()))
                out[0][i], out[1][i], out[2][i] = keys[r], lvals[r], rvals[src]
        return out

    monkeypatch.setattr(engine, "_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(grouping, "group_row_ids", group_row_ids)
    monkeypatch.setattr(nv, "bcast_build", bcast_build)
    monkeypatch.setattr(nv, "bcast_probe", bcast_probe)
    monkeypatch.setattr(nv, "bcast_emit", bcast_emit)
    return join


def _as(a, dtype):
    return torch.from_numpy(np.asarray(a)).to(dtype)


SHAPES = ["overlap", "empty_big", "empty_small", "disjoint", "all_match", "one_split", "fewer_rows_than_splits", "hot",
          "specials"]


@pytest.mark.parametrize("kdt_big,kdt_small", [(torch.int64, torch.int32), (torch.int32, torch.int64),
                                               (torch.float32, torch.float64), (torch.float64, torch.float32)],
                         ids=str)
@pytest.mark.parametrize("shape", SHAPES)
def test_inner_join_columns_on_an_emulated_device(monkeypatch, kdt_big, kdt_small, shape):
    """Per split of big, the composition's rows in its order: same keys (their own bits, -0.0 stays -0.0), values and
    dtypes as the row path through ctx.parallelize gives."""
    join = _emulated_device(monkeypatch, _bcastcheck())
    rng = np.random.default_rng(10 * SHAPES.index(shape) + kdt_big.itemsize)
    dc = cc.ctx()
    nb, ns, Mb, Ms, span = 60, 25, 4, 3, 12
    if shape == "empty_big":
        nb = 0
    elif shape == "empty_small":
        ns = 0
    elif shape == "one_split":
        Mb = 1
    elif shape == "fewer_rows_than_splits":
        nb, Mb = 3, 7
    bk = rng.integers(-span, span, nb).astype(np.float64)
    sk = rng.integers(-span, span, ns).astype(np.float64)
    if shape == "disjoint":
        sk = sk + 100
    elif shape == "all_match":
        bk = rng.choice(sk, nb)
    elif shape == "hot":
        sk = np.concatenate([sk, np.full(40, 3.0)])
        bk[::4] = 3.0
    elif shape == "specials":
        if kdt_big.is_floating_point:
            bk[::5], bk[1::7], sk[::4], sk[1::6] = -0.0, float("nan"), 0.0, float("nan")
            sk[2::9] = -0.0
        else:
            info = torch.iinfo(kdt_big if kdt_big.itemsize < kdt_small.itemsize else kdt_small)
            bk[::5], sk[::4] = info.min, info.min
            bk[1::5], sk[1::4] = info.max, info.max
    big = dc.parallelizeColumns(_as(bk, kdt_big), _as(rng.integers(-9, 9, len(bk)), torch.float32), Mb)
    small = dc.parallelizeColumns(_as(sk, kdt_small), _as(rng.integers(0, 1000, len(sk)), torch.int64), Ms)
    out = big.innerJoin(small)
    assert isinstance(out, join.ColumnarInnerJoinedRDD)
    got = out.glom().collect()
    want = dc.parallelize(big.collect(), len(big.splits)).innerJoin(dc.parallelize(small.collect(), Ms)).glom().collect()
    assert [len(p) for p in got] == [len(p) for p in want] and len(got) == len(big.splits)
    assert got == want and repr(got) == repr(want)
    for sp in out.splits:
        keys, left, right = out.columns(sp)
        assert (keys.dtype, left.dtype, right.dtype) == (kdt_big, torch.float32, torch.int64)
    if shape in ("overlap", "hot", "all_match"):
        assert sum(len(p) for p in got) > 0
