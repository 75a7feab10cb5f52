"""The device topByKey on a CPU: the selection arithmetic of dpk_common.cuh run through tests/topkcheck.cu (the order
key, the length rule of a round, the unit a CTA takes of a run and where it writes), which calls take the device path,
the partitioner it shares with the composition, and topk_columns on an emulated device.  The device results themselves
are checked in tests/test_gpu_topbykey.py."""
import ctypes as C
import os
import random
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import cogroup_common as cc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _topkcheck():
    path = os.path.join(ROOT, "tests", "_topkcheck.so")
    if not os.path.exists(path):
        subprocess.call([sys.executable, "-c", "import __graft_entry__ as g; g.build()"], cwd=ROOT)
    if not os.path.exists(path):
        pytest.skip("topkcheck not built")
    L = C.CDLL(path)
    L.tc_order_key.restype = C.c_uint64
    L.tc_order_key.argtypes = [C.c_uint64, C.c_int32, C.c_int32, C.c_int32]
    L.tc_next_len.restype = C.c_int64
    L.tc_next_len.argtypes = [C.c_int64, C.c_int64, C.c_int64]
    L.tc_unit.restype = C.c_int32
    L.tc_unit.argtypes = [C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.tc_unit_out.restype = C.c_int64
    L.tc_unit_out.argtypes = [C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64]
    L.tc_tile.restype = C.c_int64
    L.tc_max_n.restype = C.c_int64
    return L


def test_constants_agree_with_the_library():
    from dpark_b200 import _native as nv
    from dpark_b200 import topk
    L = _topkcheck()
    assert (L.tc_tile(), L.tc_max_n()) == (nv.TOPK_TILE, nv.TOPK_MAX_N) == (4096, topk.TOPK_MAX_N)
    assert nv.TOPK_MAX_N <= nv.TOPK_TILE // 8


# ------------------------------------------------------------------------------------------------ order key
def _bits(x, fmt):
    return struct.unpack({"i": "<I", "q": "<Q", "f": "<I", "d": "<Q"}[fmt], struct.pack("<" + fmt, x))[0]


def _samples(fmt, rng):
    if fmt in "iq":
        w = 32 if fmt == "i" else 64
        lo, hi = -(1 << (w - 1)), (1 << (w - 1)) - 1
        xs = [lo, lo + 1, -2, -1, 0, 1, 2, hi - 1, hi] + [rng.randrange(lo, hi + 1) for _ in range(40)]
        return xs + [rng.randrange(-5, 5) for _ in range(10)]
    info = np.finfo(np.float32 if fmt == "f" else np.float64)
    sub, tiny, big = float(info.smallest_subnormal), float(info.smallest_normal), float(info.max)
    xs = [float("-inf"), -big, -1.5, -1.0, -tiny, -sub, -0.0, 0.0, sub, 2 * sub, tiny, 1.0, 1.5, big, float("inf")]
    xs += [rng.uniform(-1e6, 1e6) for _ in range(30)] + [rng.choice([-0.0, 0.0, 1.0, -1.0]) for _ in range(10)]
    if fmt == "f":      # values a float32 column can hold
        xs = [struct.unpack("<f", struct.pack("<f", x))[0] for x in xs]
    return xs


@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("fmt", ["i", "q", "f", "d"], ids=["int32", "int64", "float32", "float64"])
def test_order_key_orders_as_python_does(fmt, reverse):
    """For every pair of sampled values: key(a) < key(b) exactly when Python orders a before b (a < b, or a > b with
    reverse), and the keys are equal exactly when the values compare equal (-0.0 == 0.0)."""
    L = _topkcheck()
    xs = _samples(fmt, random.Random(ord(fmt) + reverse))
    width = 4 if fmt in "if" else 8
    keys = [L.tc_order_key(_bits(x, fmt), width, fmt in "fd", reverse) for x in xs]
    assert all(k < (1 << (8 * width)) for k in keys)
    for a, ka in zip(xs, keys):
        for b, kb in zip(xs, keys):
            assert (ka < kb) == ((a > b) if reverse else (a < b)), (a, b)
            assert (ka == kb) == (a == b), (a, b)
    # the stable sort by (key, position) is Python's sorted()
    order = sorted(range(len(xs)), key=lambda i: (keys[i], i))
    want = sorted(range(len(xs)), key=lambda i: xs[i], reverse=reverse)
    assert order == want


def test_order_key_ignores_bits_above_the_width():
    L = _topkcheck()
    for x in (-7, 0, 5):
        b = _bits(x, "i")
        assert L.tc_order_key(b | (0xDEAD << 32), 4, 0, 0) == L.tc_order_key(b, 4, 0, 0)


# ------------------------------------------------------------------------------------------------ rounds
def _chunks(s, e, T):
    """A run's units: one for a run of at most T rows, else chunks of T from its start."""
    return [(a, min(e, a + T)) for a in range(s, e, T)]


def _lengths(T, n):
    return [0, 1, n, T - 1, T, T + 1, 2 * T - 1, 2 * T, 2 * T + 1, 3 * T - 1, 3 * T + 1, 7 * T + 5, 12 * T + T // 2]


@pytest.mark.parametrize("T,top_n", [(4096, 1), (4096, 10), (4096, 512), (8, 1), (8, 3), (8, 8), (5, 2)])
def test_length_rule_is_the_chunks_kept(T, top_n):
    L = _topkcheck()
    for length in _lengths(T, top_n) + list(range(3 * T + 2)):
        want = sum(min(top_n, e - a) for a, e in _chunks(0, length, T))
        assert L.tc_next_len(length, T, top_n) == want, length


@pytest.mark.parametrize("T,top_n", [(4096, 10), (4096, 512), (8, 3), (8, 8), (5, 2)])
def test_every_row_lies_in_one_unit_of_one_cta(T, top_n):
    """Runs of the edge lengths in random order: the units CTAs take are exactly the runs' chunks, every row lies in
    exactly one, a unit starts in its CTA's window, a CTA's units are one contiguous range of at most 2T rows, and the
    units' outputs tile every run's next-round range in order."""
    L = _topkcheck()
    rng = random.Random(T * 1000 + top_n)
    lens = [x for x in _lengths(T, top_n) if x] * 2 + [rng.randrange(1, 3 * T) for _ in range(20)]
    rng.shuffle(lens)
    starts = np.concatenate([[0], np.cumsum(lens)]).tolist()
    n = starts[-1]
    out_starts = np.concatenate([[0], np.cumsum([L.tc_next_len(x, T, top_n) for x in lens])]).tolist()
    owner = np.full(n, -1, np.int64)
    u0, u1 = C.c_int64(), C.c_int64()
    written = {g: [] for g in range(len(lens))}
    for w in range(-(-n // T)):
        units = []
        for g in range(len(lens)):
            if L.tc_unit(starts[g], starts[g + 1], w, T, C.byref(u0), C.byref(u1)):
                units.append((g, u0.value, u1.value))
        for g, a, e in units:
            assert (a, e) in _chunks(starts[g], starts[g + 1], T)
            assert w * T <= a < (w + 1) * T
            assert (owner[a:e] == -1).all()
            owner[a:e] = w
            o = L.tc_unit_out(starts[g], a, out_starts[g], T, top_n)
            written[g].append((o, o + min(top_n, e - a)))
        if units:
            assert all(units[i][2] == units[i + 1][1] for i in range(len(units) - 1))   # adjacent
            assert units[-1][2] - units[0][1] <= 2 * T
    assert (owner >= 0).all()
    for g, spans in written.items():
        assert spans[0][0] == out_starts[g] and spans[-1][1] == out_starts[g + 1]
        assert all(spans[i][1] == spans[i + 1][0] for i in range(len(spans) - 1))


@pytest.mark.parametrize("top_n", [1, 10, 512])
def test_rounds_follow_the_length_rule(top_n):
    """topk.rounds(longest): the round in which the longest run is at most one tile is the last, and after it every
    run holds min(top_n, L) candidates."""
    from dpark_b200 import topk
    L = _topkcheck()
    T = L.tc_tile()
    for longest in [1, top_n, T, T + 1, 10 * T, 3_000_000, 10 ** 8, 10 ** 9]:
        x, r = longest, 1
        while x > T:
            x = L.tc_next_len(x, T, top_n)
            r += 1
        assert topk.rounds(longest, top_n) == r
        assert L.tc_next_len(x, T, top_n) == min(top_n, longest)
    assert topk.rounds(10 ** 8, 10) <= 4


# ------------------------------------------------------------------------------------------------ path choice
ELIGIBLE = [torch.int32, torch.int64, torch.float32, torch.float64]
INELIGIBLE = [torch.int16, torch.uint8, torch.bool, torch.float16]


def _col(dc, kdt, vdt, n=6, M=2):
    return dc.parallelizeColumns(torch.arange(n).to(kdt), torch.arange(n).to(vdt), M)


def _topk_cls():
    from dpark_b200.topk import ColumnarTopByKeyRDD
    return ColumnarTopByKeyRDD


@pytest.mark.parametrize("kdt", ELIGIBLE + INELIGIBLE, ids=str)
@pytest.mark.parametrize("vdt", ELIGIBLE + INELIGIBLE, ids=str)
def test_device_top_by_key_is_chosen_by_dtypes(kdt, vdt):
    from dpark_b200 import HashPartitioner
    from dpark_b200.rdd import MappedValuesRDD
    dc = cc.ctx()
    eligible = kdt in ELIGIBLE and vdt in ELIGIBLE
    out = _col(dc, kdt, vdt).topByKey(3, num_splits=4)
    assert isinstance(out, _topk_cls()) == eligible
    assert isinstance(out, MappedValuesRDD) != eligible
    assert out.partitioner == HashPartitioner(4) and len(out.splits) == 4


def test_order_func_top_n_and_input_type_choose_the_path():
    from dpark_b200.rdd import ColumnarRDD
    from dpark_b200.rdd import MappedValuesRDD
    dc = cc.ctx()
    col = _col(dc, torch.int64, torch.float64)

    class MyColumns(ColumnarRDD):
        pass

    for n, rev in ((1, False), (2, True), (512, False)):
        assert isinstance(col.topByKey(n, reverse=rev), _topk_cls())
    assert isinstance(col.topByKey(513), MappedValuesRDD)
    assert isinstance(col.topByKey(3, order_func=lambda v: -v), MappedValuesRDD)
    assert isinstance(col.topByKey(3, order_func=lambda v: -v, reverse=True), MappedValuesRDD)
    for other in (dc.parallelize([(1, 2)], 1), col.map(lambda kv: kv), col.mapValue(lambda v: v),
                  MyColumns(dc, np.arange(4), np.arange(4), 2), col.union(col)):
        assert isinstance(other.topByKey(3), MappedValuesRDD)
    with pytest.raises(AssertionError):
        col.topByKey(0)


def test_more_than_one_process_keeps_the_composition(monkeypatch):
    from dpark_b200 import spmd
    from dpark_b200.rdd import MappedValuesRDD
    dc = cc.ctx()
    col = _col(dc, torch.int32, torch.float32)
    assert isinstance(col.topByKey(2, num_splits=2), _topk_cls())
    monkeypatch.setattr(spmd, "rank_world", lambda: (0, 2))
    assert isinstance(col.topByKey(2, num_splits=2), MappedValuesRDD)


def test_nothing_is_computed_at_construction(monkeypatch):
    """Building the device topByKey (and what lies on top of it) touches no device: the CPU has none."""
    from dpark_b200 import engine, topk

    def no_device(*a):
        raise AssertionError("the topByKey ran at construction")

    monkeypatch.setattr(engine, "_device", no_device)
    monkeypatch.setattr(topk, "topk_columns", no_device)
    dc = cc.ctx()
    a, b = _col(dc, torch.int64, torch.float64), _col(dc, torch.int64, torch.int64)
    out = a.topByKey(3, num_splits=4, reverse=True)
    out.mapValue(len).filter(bool)
    out.groupWith(b)
    assert out._result is None


# ------------------------------------------------------------------------------------------------ partitioner
def test_partitioner_is_the_composition_s(monkeypatch):
    from dpark_b200 import HashPartitioner
    from dpark_b200.rdd import RDD, CoGroupedRDD
    dc = cc.ctx()
    a, c = _col(dc, torch.int64, torch.int64, n=9, M=3), _col(dc, torch.int64, torch.int64)
    for splits in (None, 1, 5):
        assert a.topByKey(2, num_splits=splits).partitioner == a.groupByKey(splits).partitioner
    assert a.topByKey(2).partitioner == HashPartitioner(min(dc.defaultMinSplits, 3))
    part = HashPartitioner(6, thresholds=[1, 2, 3, 4, 5])
    assert a.topByKey(2, num_splits=part).partitioner is part
    calls = []

    def fake_thresholds(self, splits, rate):
        calls.append((type(self).__name__, splits, rate))
        return [10 * i for i in range(1, splits - 1)], splits - 1

    monkeypatch.setattr(RDD, "_skew_thresholds", fake_thresholds)
    want = HashPartitioner(3, thresholds=[10, 20])
    out = a.topByKey(2, num_splits=4, fixSkew=0.5)
    assert out.partitioner == want == a.groupByKey(4, fixSkew=0.5).partitioner
    assert calls == [("ColumnarRDD", 4, 0.5)] * 2          # once for the topByKey, once for the groupByKey
    assert a.topByKey(2, num_splits=1, fixSkew=0.5).partitioner == HashPartitioner(1)
    assert len(calls) == 2
    # the partitioner survives mapValue, and a later groupWith takes the result as a narrow dependency
    top = a.topByKey(2, num_splits=6)
    assert top.mapValue(len).partitioner == HashPartitioner(6)
    again = top.groupWith(c)
    assert type(again) is CoGroupedRDD and again.partitioner == HashPartitioner(6) and again.narrow == [0]


def test_other_partitioners_are_refused_as_by_the_composition():
    from dpark_b200.dependency import RangePartitioner
    dc = cc.ctx()
    col = _col(dc, torch.int64, torch.int64)
    for bad in (RangePartitioner([3]), "4"):
        with pytest.raises((TypeError, NotImplementedError)) as e_dev:
            col.topByKey(2, num_splits=bad)
        with pytest.raises((TypeError, NotImplementedError)) as e_rows:
            col.topByKey(2, order_func=lambda v: v, num_splits=bad)
        assert type(e_dev.value) is type(e_rows.value)


# ------------------------------------------------------------------------------------------------ host orchestration
def _emulated_device(monkeypatch, L, T):
    """topk.topk_columns on the CPU with a tile of T: the numeric group-by from the oracle (as in the cogroup's host
    test), dpk_topk_lengths / dpk_topk_round replaced by loops over the very arithmetic the kernels run."""
    from dpark_b200 import _native as nv
    from tests.test_cogroup_columnar_host import _emulated_device as cogroup_device
    cogroup_device(monkeypatch, None)
    monkeypatch.setattr(nv, "TOPK_TILE", T)

    def topk_lengths(runs, top_n):
        r = runs.tolist()
        return torch.tensor([L.tc_next_len(r[g + 1] - r[g], T, top_n) for g in range(len(r) - 1)], dtype=torch.int64)

    def topk_round(ids, vals, runs, n, out_starts, top_n, reverse):
        r, o = runs.tolist(), out_starts.tolist()
        assert r[-1] == n
        src = [vals[i] for i in ids.tolist()] if ids is not None else list(vals)
        width, is_float = vals.element_size(), vals.dtype.is_floating_point
        raw = torch.stack(src).view(torch.int32 if width == 4 else torch.int64).tolist() if src else []
        out = torch.empty(o[-1], dtype=vals.dtype)
        u0, u1 = C.c_int64(), C.c_int64()
        for g in range(len(r) - 1):
            for w in range(r[g] // T, (r[g + 1] - 1) // T + 1):
                if not L.tc_unit(r[g], r[g + 1], w, T, C.byref(u0), C.byref(u1)):
                    continue
                a, e = u0.value, u1.value
                key = lambda i: (L.tc_order_key(raw[i] & ((1 << 8 * width) - 1), width, is_float, reverse), i)
                best = sorted(range(a, e), key=key)[:top_n]
                base = L.tc_unit_out(r[g], a, o[g], T, top_n)
                for j, i in enumerate(best):
                    out[base + j] = src[i]
        return out

    monkeypatch.setattr(nv, "topk_lengths", topk_lengths)
    monkeypatch.setattr(nv, "topk_round", topk_round)


@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("vdt", ELIGIBLE, ids=str)
@pytest.mark.parametrize("P", [1, 3])
def test_topk_columns_on_an_emulated_device(monkeypatch, P, vdt, reverse):
    """With a tile of 16 a key of 70 rows needs two or three rounds: per partition the keys of the group-by and, per
    key, the first top_n values of Python's stable sort of its values in row order, bit for bit (-0.0 stays -0.0).
    (A round shrinks a long run only while top_n < T; the library's top_n is at most T / 8.)"""
    from dpark_b200 import topk
    from oracle import oracle as orc
    L = _topkcheck()
    _emulated_device(monkeypatch, L, 16)
    rng = np.random.default_rng(P)
    dc = cc.ctx()
    k = np.concatenate([rng.integers(0, 9, 60), np.full(70, 4), [11]])
    k = k[rng.permutation(len(k))]
    v = rng.integers(-4, 4, len(k)).astype(np.float64)
    if vdt.is_floating_point:
        v[rng.random(len(v)) < 0.3] = -0.0
    rdd = dc.parallelizeColumns(torch.from_numpy(k), torch.from_numpy(v).to(vdt), 3)
    for top_n in (1, 3, 7):
        assert topk.rounds(70, top_n) >= 2
        parts = topk.topk_columns(rdd, P, None, top_n, reverse)
        want = orc.group_by_key([k], [np.arange(len(k), dtype=np.int64)], P)
        for p, (gk, off, vals) in enumerate(parts):
            wk, woff, wids = want[p]
            assert gk.dtype == torch.int64 and gk.tolist() == wk.tolist()
            assert vals.dtype == vdt and off.shape == (len(wk) + 1,) and off[0] == 0
            got = [vals[off[j]:off[j + 1]].tolist() for j in range(len(wk))]
            col = rdd.vals.tolist()
            exp = [sorted([col[i] for i in wids[woff[j]:woff[j + 1]]], reverse=reverse)[:top_n] for j in range(len(wk))]
            assert repr(got) == repr(exp), (p, top_n)
