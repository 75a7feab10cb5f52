"""The device join on a CPU: the join arithmetic of dpk_common.cuh run through tests/joincheck.cu (rows per key, output
row -> (left row, right row), the left rows of an id run), which inputs take the device path, and the partitioner the
device join shares with groupWith.  The device results themselves are checked in tests/test_gpu_join.py."""
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
KINDS = {"join": (False, False), "leftOuterJoin": (True, False), "rightOuterJoin": (False, True),
         "outerJoin": (True, True)}


def _joincheck():
    path = os.path.join(ROOT, "tests", "_joincheck.so")
    if not os.path.exists(path):
        subprocess.call([sys.executable, "-c", "import __graft_entry__ as g; g.build()"], cwd=ROOT)
    if not os.path.exists(path):
        pytest.skip("joincheck not built")
    L = C.CDLL(path)
    L.jc_join_count.restype = C.c_int64
    L.jc_join_count.argtypes = [C.c_int64, C.c_int64, C.c_int, C.c_int]
    L.jc_join_pair.argtypes = [C.c_int64, C.c_int64, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.jc_join_left_rows.restype = C.c_int64
    L.jc_join_left_rows.argtypes = [C.c_void_p, C.c_int64, C.c_int64]
    return L


def _row_path_pairs(nl, nr, keep_left, keep_right):
    """What RDD._join's flatMap yields for one key with nl left and nr right values (as (a, b) row numbers)."""
    left, right = list(range(nl)), list(range(nr))
    if not left and keep_right:
        left = [None]
    if not right and keep_left:
        right = [None]
    return [(a, b) for a in left for b in right]


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_join_count_matches_the_row_path(kind):
    L = _joincheck()
    keep_left, keep_right = KINDS[kind]
    for nl, nr in itertools.product((0, 1, 2, 7), repeat=2):
        want = len(_row_path_pairs(nl, nr, keep_left, keep_right))
        assert L.jc_join_count(nl, nr, keep_left, keep_right) == want, (nl, nr)


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_join_pair_enumerates_left_major(kind):
    """Every output row of a key maps to the (left row, right row) the row path puts there, for every L, R <= 9;
    a missing side is row 0 of that side."""
    L = _joincheck()
    keep_left, keep_right = KINDS[kind]
    a, b = C.c_int64(), C.c_int64()
    for nl, nr in itertools.product(range(10), repeat=2):
        want = [(x or 0, y or 0) for x, y in _row_path_pairs(nl, nr, keep_left, keep_right)]
        got = []
        for i in range(L.jc_join_count(nl, nr, keep_left, keep_right)):
            L.jc_join_pair(i, nr, keep_left, C.byref(a), C.byref(b))
            got.append((a.value, b.value))
        assert got == want, (nl, nr)


def test_join_left_rows_counts_ids_below_nL():
    L = _joincheck()
    rng = np.random.default_rng(3)
    nL = 1000
    for nl, nr in itertools.product((0, 1, 2, 7, 100), repeat=2):
        left = np.sort(rng.choice(nL, nl, replace=False))
        right = np.sort(rng.choice(np.arange(nL, 2 * nL), nr, replace=False))
        if nr:
            right[0] = nL                   # the first right row of the union is a right row
        if nl:
            left[-1] = nL - 1               # the last left row is a left row
        run = np.ascontiguousarray(np.concatenate([left, right]).astype(np.int64))
        assert L.jc_join_left_rows(run.ctypes.data, len(run), nL) == nl, (nl, nr)


# ------------------------------------------------------------------------------------------------ path choice
ELIGIBLE = [torch.int32, torch.int64, torch.float32, torch.float64]
INELIGIBLE = [torch.int16, torch.uint8, torch.bool, torch.float16]


def _col(dc, kdt, vdt, n=6, M=2):
    return dc.parallelizeColumns(torch.arange(n).to(kdt), torch.arange(n).to(vdt), M)


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("kdt", ELIGIBLE + INELIGIBLE, ids=str)
@pytest.mark.parametrize("vdt", ELIGIBLE + INELIGIBLE, ids=str)
def test_device_path_is_chosen_by_input_type_and_dtypes(kind, kdt, vdt):
    from dpark_b200.join import ColumnarJoinedRDD
    dc = cc.ctx()
    eligible = kdt in ELIGIBLE and vdt in ELIGIBLE
    a = _col(dc, kdt, vdt)
    b = _col(dc, torch.int64, torch.float64)
    for x, y in ((a, b), (b, a)):
        out = getattr(x, kind)(y, 3)
        assert isinstance(out, ColumnarJoinedRDD) == eligible
        assert out.partitioner is None and len(out.splits) == 3
        if eligible:
            assert out.parents() == [x, y]
            assert (out.keep_left, out.keep_right) == KINDS[kind]
            assert out._result is None            # nothing ran: the join materialises when a partition is read


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_row_inputs_keep_the_composition(kind):
    from dpark_b200.join import ColumnarJoinedRDD
    from dpark_b200.rdd import ColumnarRDD, FlatMappedRDD
    dc = cc.ctx()

    class MyColumns(ColumnarRDD):
        pass

    col = _col(dc, torch.int64, torch.int64)
    others = [dc.parallelize([(1, 2), (3, 4)], 2), col.map(lambda kv: kv), MyColumns(dc, np.arange(4), np.arange(4), 2),
              col.union(col)]
    for other in others:
        for x, y in ((col, other), (other, col)):
            out = getattr(x, kind)(y, 2)
            assert not isinstance(out, ColumnarJoinedRDD)
            assert isinstance(out, FlatMappedRDD)


def test_more_than_one_process_keeps_the_composition(monkeypatch):
    from dpark_b200 import spmd
    from dpark_b200.join import ColumnarJoinedRDD
    dc = cc.ctx()
    a, b = _col(dc, torch.int64, torch.int64), _col(dc, torch.int64, torch.int64)
    assert isinstance(a.join(b, 2), ColumnarJoinedRDD)
    monkeypatch.setattr(spmd, "rank_world", lambda: (0, 2))
    assert not isinstance(a.join(b, 2), ColumnarJoinedRDD)


# ------------------------------------------------------------------------------------------------ partitioner
def test_group_with_partitioner_is_unchanged_and_shared_with_the_device_join(monkeypatch):
    from dpark_b200 import HashPartitioner
    from dpark_b200.rdd import RDD
    dc = cc.ctx()
    a, b = _col(dc, torch.int64, torch.int64), _col(dc, torch.int64, torch.int64)
    # numSplits: explicit, else defaultParallelism, else the left input's partition count
    assert a.groupWith(b, 5).partitioner == HashPartitioner(5)
    assert a.groupWith(b).partitioner == HashPartitioner(dc.defaultParallelism)
    grouped = a.groupByKey(7)
    assert grouped.groupWith(b).partitioner == HashPartitioner(7)
    assert a.join(b).join_partitioner == HashPartitioner(dc.defaultParallelism)
    assert a.outerJoin(b, 5).join_partitioner == HashPartitioner(5)
    # fixSkew: thresholds sampled over the union of the inputs, only when there is more than one partition
    calls = []

    def fake_thresholds(self, splits, rate):
        calls.append((type(self).__name__, [type(r).__name__ for r in self.rdds], splits, rate))
        return [10 * i for i in range(1, splits - 1)], splits - 1

    monkeypatch.setattr(RDD, "_skew_thresholds", fake_thresholds)
    assert a.groupWith(b, 4, fixSkew=0.5).partitioner == HashPartitioner(3, thresholds=[10, 20])
    assert a.leftOuterJoin(b, 4, fixSkew=0.5).join_partitioner == HashPartitioner(3, thresholds=[10, 20])
    assert calls == [("UnionRDD", ["ColumnarRDD", "ColumnarRDD"], 4, 0.5)] * 2
    assert a.groupWith(b, 1, fixSkew=0.5).partitioner == HashPartitioner(1)
    assert a.join(b, 1, fixSkew=0.5).join_partitioner == HashPartitioner(1)
    assert len(calls) == 2
