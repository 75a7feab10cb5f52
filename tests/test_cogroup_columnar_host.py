"""The device cogroup on a CPU: the cogroup arithmetic of dpk_common.cuh run through tests/cogroupcheck.cu (the N-way
split of a key's id run, output row -> group -> input row), which inputs take the device path for groupWith / cogroup
and for groupByKey, and the partitioner the device cogroup shares with the join.  The device results themselves are
checked in tests/test_gpu_cogroup.py."""
import ctypes as C
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import cogroup_common as cc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cogroupcheck():
    path = os.path.join(ROOT, "tests", "_cogroupcheck.so")
    if not os.path.exists(path):
        subprocess.call([sys.executable, "-c", "import __graft_entry__ as g; g.build()"], cwd=ROOT)
    if not os.path.exists(path):
        pytest.skip("cogroupcheck not built")
    L = C.CDLL(path)
    L.cc_cogroup_split.restype = None
    L.cc_cogroup_split.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                   C.c_int64]
    L.cc_group_of.restype = C.c_int64
    L.cc_group_of.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int64]
    L.cc_cogroup_source.restype = C.c_int64
    L.cc_cogroup_source.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64]
    return L


def _i64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.int64))


def _split(L, ids, s, length, bounds, stride=1):
    N = len(bounds) - 1
    first = np.full(N * stride, -7, np.int64)
    count = np.full(N * stride, -7, np.int64)
    L.cc_cogroup_split(ids.ctypes.data, s, length, bounds.ctypes.data, N, first.ctypes.data, count.ctypes.data, stride)
    return first, count


@pytest.mark.parametrize("N", [1, 2, 3, 4, 5])
def test_cogroup_split_of_every_small_run(N):
    """Every input holds 0 or 2 rows; a key's run takes any subset of every input's rows (an empty sub-run, the input's
    first id, its last id, both).  The run sits at an offset inside a longer id column.  Every sub-run must start at
    the ids below the input's first id and hold exactly that input's ids."""
    L = _cogroupcheck()
    for sizes in itertools.product((0, 2), repeat=N):
        bounds = _i64(np.concatenate([[0], np.cumsum(sizes)]))
        per_input = [[ids for r in range(m + 1) for ids in itertools.combinations(range(bounds[t], bounds[t] + m), r)]
                     for t, m in enumerate(sizes)]
        for picks in itertools.product(*per_input):
            run = [i for p in picks for i in p]
            s = 3
            ids = _i64([-1] * s + run + [10 ** 9] * 2)
            first, count = _split(L, ids, s, len(run), bounds)
            want_first = s + np.searchsorted(run, bounds[:-1], side="left")
            assert np.array_equal(count, [len(p) for p in picks]), (sizes, picks)
            assert np.array_equal(first, want_first), (sizes, picks)
            for t in range(N):
                sub = ids[first[t]:first[t] + count[t]].tolist()
                assert sub == list(picks[t]), (sizes, picks, t)


def test_cogroup_split_writes_input_major_with_a_stride():
    L = _cogroupcheck()
    bounds = _i64([0, 4, 4, 9])
    ids = _i64([1, 3, 4, 8, 0, 2, 5])
    G = 2                                                  # group 0 = ids[0:4], group 1 = ids[4:7]
    first = np.zeros(3 * G, np.int64)
    count = np.zeros(3 * G, np.int64)
    for g, (s, e) in enumerate(((0, 4), (4, 7))):
        L.cc_cogroup_split(ids.ctypes.data, s, e - s, bounds.ctypes.data, 3,
                           first[g:].ctypes.data, count[g:].ctypes.data, G)
    assert first.reshape(3, G).tolist() == [[0, 4], [2, 6], [2, 6]]
    assert count.reshape(3, G).tolist() == [[2, 2], [0, 0], [2, 1]]


def _random_csr(rng, N, G):
    """A cogroup CSR: N inputs of random sizes (some empty), every row id in one of G groups, every group's run
    ascending.  Returns (ids, starts, bounds)."""
    sizes = rng.integers(0, 12, N)
    sizes[rng.random(N) < 0.3] = 0
    bounds = _i64(np.concatenate([[0], np.cumsum(sizes)]))
    n = int(bounds[-1])
    grp = rng.integers(0, G, n)
    ids = _i64(np.argsort(grp, kind="stable"))           # group-major, ascending inside each group
    starts = _i64(np.concatenate([[0], np.cumsum(np.bincount(grp, minlength=G))]))
    return ids, starts, bounds


@pytest.mark.parametrize("N", [1, 2, 3, 4, 5])
def test_every_output_row_reads_its_input_row(N):
    """Per input: the counts of every group, their exclusive scan, then for every output row its group (group_of on
    the scan, past the groups where the input has no rows) and the input row it copies -- the input's rows of each
    key in ascending id order, counted from the input's own first row."""
    L = _cogroupcheck()
    rng = np.random.default_rng(N)
    for trial in range(60):
        G = int(rng.integers(1, 9))
        ids, starts, bounds = _random_csr(rng, N, G)
        first = np.zeros((N, G), np.int64)
        count = np.zeros((N, G), np.int64)
        for g in range(G):
            f, c = _split(L, ids, int(starts[g]), int(starts[g + 1] - starts[g]), bounds)
            first[:, g], count[:, g] = f, c
        for t in range(N):
            off = _i64(np.concatenate([[0], np.cumsum(count[t])]))
            ft = _i64(first[t])
            want = [int(i) - int(bounds[t]) for g in range(G) for i in ids[starts[g]:starts[g + 1]]
                    if bounds[t] <= i < bounds[t + 1]]
            got, groups = [], []
            for r in range(int(off[-1])):
                g = L.cc_group_of(off.ctypes.data, 0, G, r)
                groups.append(g)
                got.append(L.cc_cogroup_source(ids.ctypes.data, int(ft[g]), int(off[g]), r, int(bounds[t])))
            assert got == want, (trial, t)
            assert groups == np.repeat(np.arange(G), count[t]).tolist(), (trial, t)


# ------------------------------------------------------------------------------------------------ path choice
ELIGIBLE = [torch.int32, torch.int64, torch.float32, torch.float64]
INELIGIBLE = [torch.int16, torch.uint8, torch.bool, torch.float16]


def _col(dc, kdt, vdt, n=6, M=2):
    return dc.parallelizeColumns(torch.arange(n).to(kdt), torch.arange(n).to(vdt), M)


def _cogrouped_cls():
    from dpark_b200.join import ColumnarCoGroupedRDD
    return ColumnarCoGroupedRDD


@pytest.mark.parametrize("N", [1, 2, 3, 4])
@pytest.mark.parametrize("kdt", ELIGIBLE + INELIGIBLE, ids=str)
@pytest.mark.parametrize("vdt", ELIGIBLE + INELIGIBLE, ids=str)
def test_device_cogroup_is_chosen_by_input_type_and_dtypes(N, kdt, vdt):
    from dpark_b200 import HashPartitioner
    from dpark_b200.join import device_path_applies
    from dpark_b200.rdd import CoGroupedRDD
    dc = cc.ctx()
    eligible = kdt in ELIGIBLE and vdt in ELIGIBLE
    a = _col(dc, kdt, vdt)
    others = [_col(dc, torch.int64, torch.float64) for _ in range(N - 1)]
    for rdds in ([a] + others, others + [a]):
        for op in ("groupWith", "cogroup"):
            out = getattr(rdds[0], op)(rdds[1:], 3)
            assert isinstance(out, _cogrouped_cls()) == eligible
            assert isinstance(out, CoGroupedRDD) != eligible
            assert out.partitioner == HashPartitioner(3) and len(out.splits) == 3
            if eligible:
                assert out.parents() == rdds
                assert out._result is None        # nothing ran: the cogroup materialises when a partition is read
        assert device_path_applies(rdds) == eligible
    # groupByKey asks the same question of its one input
    assert device_path_applies([a]) == eligible


@pytest.mark.parametrize("N", [2, 3])
def test_row_subclass_union_and_mapped_inputs_keep_the_cogroup(N):
    from dpark_b200.join import device_path_applies
    from dpark_b200.rdd import CoGroupedRDD, ColumnarRDD
    dc = cc.ctx()

    class MyColumns(ColumnarRDD):
        pass

    col = _col(dc, torch.int64, torch.int64)
    odd = [dc.parallelize([(1, 2), (3, 4)], 2), col.map(lambda kv: kv), MyColumns(dc, np.arange(4), np.arange(4), 2),
           col.union(col), col.mapValue(lambda v: v)]
    for other in odd:
        for pos in range(N):
            rdds = [_col(dc, torch.int64, torch.int64) for _ in range(N - 1)]
            rdds.insert(pos, other)
            out = rdds[0].groupWith(rdds[1:], 2)
            assert type(out) is CoGroupedRDD
            assert not device_path_applies(rdds)
        assert not device_path_applies([other])


def test_more_than_one_process_keeps_the_cogroup(monkeypatch):
    from dpark_b200 import spmd
    from dpark_b200.join import device_path_applies
    from dpark_b200.rdd import CoGroupedRDD
    dc = cc.ctx()
    a, b = _col(dc, torch.int64, torch.int64), _col(dc, torch.int32, torch.float32)
    assert isinstance(a.groupWith(b, 2), _cogrouped_cls())
    assert isinstance(a.groupWith([], 2), _cogrouped_cls())
    monkeypatch.setattr(spmd, "rank_world", lambda: (0, 2))
    assert type(a.groupWith(b, 2)) is CoGroupedRDD
    assert type(a.groupWith([], 2)) is CoGroupedRDD
    assert not device_path_applies([a])


def test_nothing_is_computed_at_construction(monkeypatch):
    """Building the device cogroup (and what lies on top of it) touches no device: the CPU has none."""
    from dpark_b200 import engine, join

    def no_device():
        raise AssertionError("the cogroup ran at construction")

    monkeypatch.setattr(engine, "_device", no_device)
    monkeypatch.setattr(join, "cogroup_columns", lambda *a: no_device())
    dc = cc.ctx()
    a, b, c = (_col(dc, torch.int64, torch.int64) for _ in range(3))
    out = a.groupWith([b, c], 4)
    out.mapValue(len).filter(bool)
    a.update(b, numSplits=3)
    a.groupByKey(3)
    assert out._result is None


# ------------------------------------------------------------------------------------------------ partitioner
def test_partitioner_and_fix_skew_are_shared_with_the_join(monkeypatch):
    from dpark_b200 import HashPartitioner
    from dpark_b200.rdd import RDD, CoGroupedRDD
    dc = cc.ctx()
    a, b, c = (_col(dc, torch.int64, torch.int64) for _ in range(3))
    assert a.groupWith(b, 5).partitioner == HashPartitioner(5) == a.join(b, 5).join_partitioner
    assert a.groupWith([b, c]).partitioner == HashPartitioner(dc.defaultParallelism) == a.join(b).join_partitioner
    assert a.groupWith([]).partitioner == HashPartitioner(dc.defaultParallelism)
    calls = []

    def fake_thresholds(self, splits, rate):
        calls.append(([type(r).__name__ for r in self.rdds], splits, rate))
        return [10 * i for i in range(1, splits - 1)], splits - 1

    monkeypatch.setattr(RDD, "_skew_thresholds", fake_thresholds)
    want = HashPartitioner(3, thresholds=[10, 20])
    assert a.groupWith(b, 4, fixSkew=0.5).partitioner == want == a.leftOuterJoin(b, 4, fixSkew=0.5).join_partitioner
    assert a.cogroup([b, c], 4, fixSkew=0.5).partitioner == want
    assert a.groupWith([], 4, fixSkew=0.5).partitioner == want
    assert calls == [(["ColumnarRDD"] * 2, 4, 0.5)] * 2 + [(["ColumnarRDD"] * 3, 4, 0.5), (["ColumnarRDD"], 4, 0.5)]
    assert a.groupWith(b, 1, fixSkew=0.5).partitioner == HashPartitioner(1)
    assert len(calls) == 4
    # the partitioner survives mapValue, and a later groupWith takes the result as a narrow dependency
    cg = a.groupWith(b, 6)
    assert cg.mapValue(len).partitioner == HashPartitioner(6)
    again = cg.groupWith(c)
    assert type(again) is CoGroupedRDD and again.partitioner == HashPartitioner(6) and again.narrow == [0]


@pytest.mark.parametrize("kdt", ELIGIBLE + INELIGIBLE[:2], ids=str)
def test_group_by_key_takes_the_device_path_when_the_parent_qualifies(monkeypatch, kdt):
    """engine.run_shuffle's group branch: a numeric ColumnarRDD parent goes to the device cogroup, anything else (a
    row parent, an ineligible dtype, a mapped parent) keeps the row-id group-by; the reduce branch is untouched."""
    from dpark_b200 import engine
    from dpark_b200.rdd import ShuffledRDD
    seen = []

    def spy(name):
        def run(*args):
            seen.append(name)
            res = engine.ShuffleResult(args[1])
            res.parts = [([], [])] * args[1]
            return res
        return run

    monkeypatch.setattr(engine, "_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(engine, "_run_group_columns", spy("columns"))
    monkeypatch.setattr(engine, "_run_group", lambda splits, P, thr, dev: spy("rows")(splits, P))
    monkeypatch.setattr(engine, "_run_reduce", lambda splits, P, *a: spy("reduce")(splits, P))
    dc = cc.ctx()
    col = _col(dc, kdt, torch.int64)
    for rdd, want in ((col, "columns" if kdt in ELIGIBLE else "rows"), (col.map(lambda kv: kv), "rows"),
                      (dc.parallelize([(1, 2)], 1), "rows")):
        seen.clear()
        g = rdd.groupByKey(3)
        assert type(g) is ShuffledRDD
        assert g.collect() == []
        assert seen == [want]
    seen.clear()
    col.reduceByKey(lambda x, y: x + y, 3).collect()
    assert seen == ["reduce"]


# ------------------------------------------------------------------------------------------------ host orchestration
def _emulated_device(monkeypatch, L):
    """join.cogroup_columns on the CPU: the numeric group-by from the oracle, dpk_cogroup_count / dpk_cogroup_emit
    replaced by loops over the very arithmetic the kernels run (tests/cogroupcheck.cu).  An emit that would read
    outside an input's values raises IndexError here instead of reading past a device allocation."""
    from dpark_b200 import engine, grouping, join
    from dpark_b200 import _native as nv
    from oracle import oracle as orc

    def group_row_ids(key_chunks, id_chunks, P, thresholds):
        gk, gs, ov, part_off = [], [0], [], [0]
        for k, off, ids in orc.group_by_key([c.numpy() for c in key_chunks], [c.numpy() for c in id_chunks], P,
                                            thresholds):
            gk.extend(k.tolist())
            gs.extend((gs[-1] - off[0] + off[1:]).tolist())
            ov.extend(ids.tolist())
            part_off.append(len(ov))
        return (torch.tensor(gk, dtype=torch.int64), torch.tensor(gs, dtype=torch.int64),
                torch.tensor(ov, dtype=torch.int64), torch.tensor(part_off, dtype=torch.int64))

    def cogroup_count(ids, gs, G, bounds):
        ids, gs, b = _i64(ids.numpy()), gs.numpy(), _i64(bounds.numpy())
        N = len(b) - 1
        first, count = np.zeros(N * G, np.int64), np.zeros(N * G, np.int64)
        for g in range(G):
            L.cc_cogroup_split(ids.ctypes.data, int(gs[g]), int(gs[g + 1] - gs[g]), b.ctypes.data, N,
                               first[g:].ctypes.data, count[g:].ctypes.data, G)
        return torch.from_numpy(first.reshape(N, G)), torch.from_numpy(count.reshape(N, G))

    def cogroup_emit(ids, first, out_off, id_base, vals, n_out):
        ids, first, off = _i64(ids.numpy()), first.numpy(), _i64(out_off.numpy())
        out = torch.empty(n_out, dtype=vals.dtype)
        for r in range(n_out):
            g = L.cc_group_of(off.ctypes.data, 0, len(first), r)
            src = L.cc_cogroup_source(ids.ctypes.data, int(first[g]), int(off[g]), r, id_base)
            if not 0 <= src < vals.numel():
                raise IndexError("output row %d reads value %d of %d" % (r, src, vals.numel()))
            out[r] = vals[src]
        return out

    monkeypatch.setattr(engine, "_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(grouping, "group_row_ids", group_row_ids)
    monkeypatch.setattr(nv, "cogroup_count", cogroup_count)
    monkeypatch.setattr(nv, "cogroup_emit", cogroup_emit)
    return join


@pytest.mark.parametrize("N", [1, 2, 3, 4])
@pytest.mark.parametrize("P", [1, 3, 7])
def test_cogroup_columns_on_an_emulated_device(monkeypatch, N, P):
    """Partition by partition, the keys of the group-by in its order and, per key and input, that input's values in
    row order; every offsets row starts at 0 and the value columns keep their dtypes."""
    join = _emulated_device(monkeypatch, _cogroupcheck())
    rng = np.random.default_rng(10 * N + P)
    dc = cc.ctx()
    vdts = [torch.int64, torch.float32, torch.int32, torch.float64]
    rdds = []
    for t in range(N):
        n = 0 if (t == 1 and P == 3) else int(rng.integers(1, 40))
        rdds.append(dc.parallelizeColumns(torch.from_numpy(rng.integers(0, 12, n)).to(torch.int32 if t % 2 else
                                                                                      torch.int64),
                                          torch.from_numpy(rng.integers(-50, 50, n)).to(vdts[t]), 1 + t))
    parts = join.cogroup_columns(rdds, P, None)
    assert len(parts) == P
    from oracle import oracle as orc
    keys = np.concatenate([r.keys.numpy().astype(np.int64) for r in rdds])
    bounds = np.concatenate([[0], np.cumsum([r.keys.numel() for r in rdds])])
    want = orc.group_by_key([keys], [np.arange(len(keys), dtype=np.int64)], P)
    for p, (gk, offsets, values) in enumerate(parts):
        wk, woff, wids = want[p]
        assert gk.dtype == torch.int64 and gk.tolist() == wk.tolist()
        assert offsets.shape == (N, len(wk) + 1) and offsets[:, 0].tolist() == [0] * N
        assert [v.dtype for v in values] == [r.vals.dtype for r in rdds]
        for t in range(N):
            lists = [values[t][offsets[t, j]:offsets[t, j + 1]].tolist() for j in range(len(wk))]
            wl = [[rdds[t].vals[i - bounds[t]].item() for i in wids[woff[j]:woff[j + 1]]
                   if bounds[t] <= i < bounds[t + 1]] for j in range(len(wk))]
            assert lists == wl, (p, t)
