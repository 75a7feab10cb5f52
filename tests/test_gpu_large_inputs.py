"""The one-GPU operators near the top of their supported size range, checked against plain references computed on the
same device, and the size caps themselves checked at cap and cap + 1 without allocating either.

The native entry points with a row count take up to 2^31 - 1 rows (innerJoin's probe and emit have no cap), and the
Python layer's caps (sorting.MAX_ROWS, selecting.MAX_UNIQ_ROWS) exist because of 32-bit limits inside the kernels.  The
rest of the suite stays below 2^31 bytes per column, so a kernel that computes a row id, a tile index or an element
offset in 32 bits would pass it.  The cases below run row ids past 2^30 (bit 30 set) through every tile loop, with
every column past 2^32 bytes.  Inputs are built on the device; the references are stock torch ops (sort, bincount,
index_add_, scatter_reduce, searchsorted), the oracle's hash for partition ids, the composition's MergingDigest for
percentiles, and numpy's MT19937 set to random.Random's state for sample.  No reference reads libdpark_b200.

All columns are int32 or float32, so a column of n rows is 4n bytes: past 2^30 rows it is past 2^32 bytes, and every
int64 word, id or offset column the kernels make is past 2^33 bytes.

| case              | n (rows)        | k, v     | limit crossed                                   | peak GiB | s    |
|-------------------|-----------------|----------|-------------------------------------------------|----------|------|
| sort x[0]         | 1,350,000,001   | i32, i32 | ids > 2^30 via keys, radix, cuts, gather (1)    | 70.41    | 0.9  |
| top x[0]          | 2^31 - 1 (cap)  | i32, i32 | the cap; picked, tied rows with bit 30 set      | 48.00    | 0.5  |
| uniq / hot        | 1,850,000,003   | i32, i32 | owners > 2^30, a count > 2^30, 2^32 slots (2)   | 73.58    | 6.4  |
| topByKey          | 2^30 + 2^20 + 5 | i32, f32 | a key's run > 2^30 through the rounds (3)       | 72.26    | 0.6  |
| percentilesByKey  | 2^30 + 2^20 + 5 | i32, f32 | a key's run > 2^30 through group-by, heads (3)  | 72.26    | 71.7 |
| cogroup           | 2^30 + 2^20 + 8 | i32, mix | ids > 2^30 over 2 inputs, 8 + 3 odd splits (3)  | 72.26    | 0.7  |
| leftOuterJoin     | 1,075,314,696   | i32, mix | ids > 2^30 on both sides, None rows (3)         | 72.29    | 1.2  |
| join              | 200,786,436     | i32, mix | 2.4e9 output rows: k_join_emit ids > 2^31       | 44.74    | 1.2  |
| innerJoin         | 1,200,000,007   | i32, i32 | 2.26e9 output rows: output ids > 2^31           | 59.57    | 0.4  |
| sample            | 2^30 + 2^24 + 7 | i32, i32 | kept ids > 2^30, every split's draws            | 18.69    | 17.2 |
| reduceByKey int   | 1,450,000,002   | i32, i32 | 2.18e9 slots (> 2^31), packed rows > 2^33 B (4) | 71.27    | 0.3  |
| reduceByKey float | 1,450,000,002   | i32, f32 | the same, float64 sums within their bound       | 71.27    | 0.7  |
| reduceByKey 8 map | 1,450,000,002   | i32, i32 | the same over 8 odd-sized map splits            | 71.27    | 0.3  |

Peak: torch.cuda.max_memory_allocated over the operator and its reference; s: the case's wall time, input generation
and reference included.  Both measured once on an H100 80GB HBM3 at a 700 W power limit.

Where a case stops short of the operator's cap, the cap does not fit in 80 GB:
(1) sort: the radix passes hold the order words and row ids three times (the caller's, ping and pong), 48 bytes per
    row, on top of the 8-byte input rows: 56 x (2^31 - 1) bytes is 112 GiB.  1.35e9 rows (70.4 GiB) is the largest
    round size that leaves the margin free on an 80 GB part.
(2) uniq: past 2^30 rows the table has 2^32 eight-byte slots (32 GiB) and the emit writes two int64 columns of n rows,
    24 bytes per row with the input: 80 GiB at 2^31 - 2 rows.  1.85e9 rows (73.6 GiB) is the largest round size that
    leaves the margin free; its owner ids reach 86% of the table's empty mark 0x7FFFFFFF.
(3) the group-by under topByKey, percentilesByKey, cogroup, the joins and groupByKey: the int64 keys and row ids, the
    map output and two radix buffers of (key, id), then the heads' [n] columns, 72 bytes per row with the input:
    72 x (2^31 - 2^20) bytes is 144 GiB.  2^30 + 2^20 rows is the least round size with one key past 2^30 values, at
    72.3 GiB.  48 bytes per row of it stay alive through the join's emit, so a join whose group-by ids pass 2^30 has
    room for only about 1.5e9 output rows of 17 bytes: output past 2^31 rows is its own case, on fewer input rows.
(4) reduceByKey: the combine's workspace is 1.5 n 16-byte slots, 24 bytes per row, on top of the input, the packed map
    output and the 12-byte output rows, 52 bytes per row or 104 GiB at 2^31 - 2^20 rows.

Mutations that these cases catch, each made once in the kernel source and reverted (the existing tests of the mutated
kernel, tests/test_gpu_sort.py + tests/test_gpu_uniq_top_hot.py and tests/test_gpu_packed_rows.py +
tests/test_gpu_kernels.py, pass under them):
* dpk_sort.cu, k_sort_gather: the key read `keys[r]` through a 32-bit byte offset, `(uint32_t)(r * sizeof(K))`,
  which wraps for r >= 2^30: the sort, top and uniq / hot cases fail.
* dpk_partition.cu, k_part_scatter_bulk's packed-record copy-out: `flush_run<Rec>(out_rec, g, ...)` with g taken
  through a 32-bit byte offset, `(uint32_t)(g * sizeof(Rec)) / sizeof(Rec)`, which wraps for g >= 2^29: all three
  reduceByKey cases fail.
The plain int32 forms, `int r = ids[i]` in k_sort_gather and `int g = s_gpos[p]` in the copy-out, cannot fail at any
supported size: r and g are row / record indices below n < 2^31, and indexing a typed pointer widens them to 64 bits
before scaling.  An int slot index in k_uniq_emit (2^32 slots in the uniq case) would wrap to a negative address, a
fault rather than a wrong answer, and is not made.

Each case skips when the device has less free memory than its budget (its peak, rounded up) plus a margin, frees
everything it made and empties the caching allocator before the next case, and prints its wall time and peak (run
pytest with -s to see them).
"""
import gc
import itertools
import math
import random
import struct
import time
import traceback

import numpy as np
import pytest
import torch

GiB = 1 << 30
MARGIN = 2 * GiB
CHUNK = 1 << 28                 # rows per step of the chunked torch references


# ------------------------------------------------------------------------------------------------ size caps
def _ctx():
    from tests import cogroup_common as cc
    return cc.ctx()


def _phantom(dc, n, dtype=torch.int32):
    """A ColumnarRDD of n rows that holds no memory: zero-stride expanded columns."""
    col = torch.zeros(1, dtype=dtype).expand(n)
    return dc.parallelizeColumns(col, col, 4)


def test_python_caps_at_cap_and_cap_plus_one():
    """On zero-stride columns: sort and top take the device path at MAX_ROWS rows and leave one more row to the
    composition; uniq and hot do so at MAX_UNIQ_ROWS."""
    from dpark_b200 import selecting, sorting
    dc = _ctx()
    assert sorting.MAX_ROWS == (1 << 31) - 1 and selecting.MAX_UNIQ_ROWS == (1 << 31) - 2
    at, past = _phantom(dc, sorting.MAX_ROWS), _phantom(dc, sorting.MAX_ROWS + 1)
    first = lambda x: x[0]      # noqa: E731
    assert sorting.device_sort_applies(at, first) and not sorting.device_sort_applies(past, first)
    assert selecting.top_applies(at, 5, None) and not selecting.top_applies(past, 5, None)
    at, past = _phantom(dc, selecting.MAX_UNIQ_ROWS), _phantom(dc, selecting.MAX_UNIQ_ROWS + 1)
    assert selecting.uniq_applies(at) and not selecting.uniq_applies(past)
    assert selecting.hot_applies(at, 5) and not selecting.hot_applies(past, 5)


def _native_cases():
    """(name, call(n) -> return code, cap): each entry point called with null buffers, so past the range check it stops
    at its pointer check; no call reaches a launch."""
    from dpark_b200 import _native as nv
    L = nv.lib()
    K_I32 = nv._KEY_KIND[torch.int32]
    return [
        ("dpk_partition", lambda n: L.dpk_partition(None, K_I32, None, None, 4, n, 1, None, 0, 0, None, None, None,
                                                    None, 0, None), (1 << 31) - 1),
        ("dpk_combine", lambda n: L.dpk_combine(None, K_I32, None, None, nv.V_I32, n, 0, 1, None, 0, 0, 0, 1, 1, None,
                                                None, None, None, None, None, 0, None), (1 << 31) - 1),
        ("dpk_radix_pass_seg", lambda n: L.dpk_radix_pass_seg(None, None, 8, n, 0, 8, 1, 1, None, None, None, None,
                                                              None, 0, None), (1 << 31) - 1),
        ("dpk_group_heads", lambda n: L.dpk_group_heads(None, n, None, None, None, None, 0, None), (1 << 31) - 1),
        ("dpk_dict_encode", lambda n: L.dpk_dict_encode(None, None, None, n, None, None, 0, None), (1 << 31) - 1),
        ("dpk_sort_keys", lambda n: L.dpk_sort_keys(None, K_I32, None, -1, n, 0, None, None, None, None, None),
         (1 << 31) - 1),
        ("dpk_select_round", lambda n: L.dpk_select_round(None, None, None, n, None, None, None), (1 << 31) - 1),
        ("dpk_select_take", lambda n: L.dpk_select_take(None, None, n, 1, None, None, None, None, None), (1 << 31) - 1),
        ("dpk_uniq_insert", lambda n: L.dpk_uniq_insert(None, K_I32, None, K_I32, n, None, nv.bcast_slots(n), None,
                                                        None), (1 << 31) - 2),
    ]


@pytest.mark.parametrize("name", ["dpk_partition", "dpk_combine", "dpk_radix_pass_seg", "dpk_group_heads",
                                  "dpk_dict_encode", "dpk_sort_keys", "dpk_select_round", "dpk_select_take",
                                  "dpk_uniq_insert"])
def test_native_row_cap(name):
    """At the cap the range check passes and the null-pointer check refuses; one row more, the range check refuses."""
    from dpark_b200 import _native as nv
    call, cap = {c[0]: c[1:] for c in _native_cases()}[name]
    before = nv.launch_count()
    with pytest.raises(ValueError) as at:
        nv._check(call(cap))
    with pytest.raises(ValueError) as past:
        nv._check(call(cap + 1))
    assert str(cap + 1) in str(past.value) and "2^31" in str(past.value)
    assert str(cap) not in str(at.value) and "2^31" not in str(at.value)
    assert nv.launch_count() == before


def test_tokenizer_byte_cap():
    """The tokenizer launches one block per TK_CHUNK bytes, at most 2^31 - 1 of them: the first longer text is refused
    before any launch (dummy non-null buffers, which the range check rejects first).  This block limit is the only
    tokenizer limit checked here; textingest's refusal of 2^31 tokens needs 2^31 tokens on the device and is not."""
    from dpark_b200 import _native as nv
    L = nv.lib()
    lo, hi = 1, 1 << 20                     # TK_CHUNK: the largest n of one block
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if L.dpk_tokenize_blocks(mid) == 1 else (lo, mid - 1)
    chunk = lo
    cap = chunk * ((1 << 31) - 1)
    assert L.dpk_tokenize_blocks(cap) == (1 << 31) - 1 and L.dpk_tokenize_blocks(cap + 1) == 1 << 31
    before = nv.launch_count()
    dummy = 16
    for call in (lambda: L.dpk_tokenize_count(dummy, cap + 1, dummy, dummy, None),
                 lambda: L.dpk_tokenize_emit(dummy, cap + 1, dummy, dummy, dummy, None)):
        with pytest.raises(ValueError, match="too long for one launch"):
            nv._check(call())
    assert nv.launch_count() == before


# ------------------------------------------------------------------------------------------------ large cases
@pytest.fixture
def large_case():
    """run(name, budget_gib, body): one large case.  Skipped unless the device has budget + MARGIN free once the caching
    allocator is emptied; prints the wall time and peak of body(); a failure's traceback frames are cleared, so a failed
    case does not hold its tensors, and the cache is emptied again after the test."""
    def run(name, budget_gib, body):
        gc.collect()
        torch.cuda.empty_cache()
        free, _ = torch.cuda.mem_get_info()
        if free < budget_gib * GiB + MARGIN:
            pytest.skip("%s needs %.0f GiB + %.0f GiB free on the device, %.1f GiB are"
                        % (name, budget_gib, MARGIN / GiB, free / GiB))
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        try:
            body()
            torch.cuda.synchronize()
        except BaseException as e:
            traceback.clear_frames(e.__traceback__)
            raise
        print("\n[large input] %s: %.1f s, peak %.2f GiB (budget %.0f GiB)"
              % (name, time.perf_counter() - t0, torch.cuda.max_memory_allocated() / GiB, budget_gib))

    yield run
    gc.collect()
    torch.cuda.empty_cache()


def _gen(seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return g


def _randint32(n, lo, hi, seed):
    return torch.randint(lo, hi, (n,), dtype=torch.int32, device="cuda", generator=_gen(seed))


def _spread(n, count, lo, seed):
    """`count` distinct row ids in [lo, n), always including lo and n - 1 (the rows whose ids have bit 30 set when
    lo >= 2^30)."""
    rng = np.random.default_rng(seed)
    ids = np.unique(rng.integers(lo + 1, n - 1, 2 * count))
    ids = set(rng.permutation(ids)[:count - 2].tolist()) | {lo, n - 1}
    assert len(ids) == count
    return torch.tensor(sorted(ids), dtype=torch.int64, device="cuda")


@pytest.mark.gpu
def test_sort_past_2pow32_bytes(large_case):
    """col.sort(x[0]) over 1.35e9 rows in 8 map splits into 6 ranges: the partitions' concatenation is
    torch.sort(stable=True) of the keys, every value (the row id) says which row landed there, the range bounds are
    RDD.sort's (every 10th of the sorted samples from the 6th on, the samples the first 60 // 8 keys of every split),
    and every partition's first and last keys belong to it under RangePartitioner(bounds)."""
    from dpark_b200.dependency import RangePartitioner
    from dpark_b200.sorting import ColumnarSortedRDD
    n = 1_350_000_001

    def body():
        keys = _randint32(n, -(1 << 20), 1 << 20, 11)          # ~520 rows per key: stability decides the order
        keys[_spread(n, 1000, 1 << 30, 12)] = torch.tensor([-(1 << 31), (1 << 31) - 1] * 500, dtype=torch.int32,
                                                             device="cuda")
        vals = torch.arange(n, dtype=torch.int32, device="cuda")
        col = _ctx().parallelizeColumns(keys, vals, 8)
        out = col.sort(lambda x: x[0], numSplits=6)
        assert isinstance(out, ColumnarSortedRDD) and len(out.splits) == 6
        parts = [out.columns(sp) for sp in out.splits]
        assert sum(int(k.numel()) for k, _ in parts) == n
        ref = torch.sort(keys, stable=True)
        take = max(6 * 10 // len(col.splits), 1)
        samples = sorted(x for sp in col.splits for x in keys[sp.begin:sp.begin + take].tolist())
        assert out.bounds == samples[5::10][:5]
        rp, at = RangePartitioner(samples[5::10][:5]), 0
        for p, (k, v) in enumerate(parts):
            m = int(k.numel())
            assert k.dtype == torch.int32 and v.dtype == torch.int32
            assert torch.equal(k, ref.values[at:at + m]), "partition %d: keys differ from torch.sort" % p
            assert torch.equal(v.long(), ref.indices[at:at + m]), "partition %d: rows differ from torch.sort" % p
            if m:
                assert rp.getPartition(int(k[0])) == p and rp.getPartition(int(k[-1])) == p
            at += m
        assert int(ref.indices[-1]) >= 1 << 30
    large_case("sort x[0], n=%d" % n, 71, body)


@pytest.mark.gpu
def test_top_at_max_rows(large_case):
    """col.top(1000, x[0]) over sorting.MAX_ROWS rows: 1000 rows of the largest keys, ties in row order.  600 of them
    are planted at row ids past 2^30 (including the last row), the rest tie at the threshold key across the whole
    column.  The reference finds the threshold with a torch.bincount of the keys."""
    from dpark_b200 import sorting
    n, take, top_key = sorting.MAX_ROWS, 1000, 1 << 24

    def body():
        keys = _randint32(n, 0, top_key, 21)
        planted = _spread(n, 600, 1 << 30, 22)
        keys[planted] = top_key + torch.arange(600, dtype=torch.int32, device="cuda") % 7
        vals = torch.arange(n, dtype=torch.int32, device="cuda")
        col = _ctx().parallelizeColumns(keys, vals, 8)
        got = col.top(take, key=lambda x: x[0])

        counts = torch.zeros(top_key + 7, dtype=torch.int64, device="cuda")
        for a in range(0, n, CHUNK):
            counts += torch.bincount(keys[a:a + CHUNK], minlength=top_key + 7)
        above = torch.flip(torch.cumsum(torch.flip(counts, [0]), 0), [0])      # rows with key >= t
        thr = int((above >= take).nonzero().max())
        over = [], []
        for a in range(0, n, CHUNK):
            ks = keys[a:a + CHUNK]
            over[0].append((ks > thr).nonzero().flatten() + a)
            over[1].append((ks == thr).nonzero().flatten() + a)
        ids = torch.cat([torch.cat(over[0]), torch.cat(over[1])[:take - int(above[thr + 1])]]).cpu().tolist()
        kh = keys[torch.tensor(ids, device="cuda")].cpu().tolist()
        want = sorted(zip(kh, ids), key=lambda r: (-r[0], r[1]))
        assert len(got) == take and got == want
        assert sum(1 for _, i in got if i >= 1 << 30) >= 600 and got[0][1] >= 1 << 30
    large_case("top x[0], n=%d" % n, 49, body)


@pytest.mark.gpu
def test_uniq_and_hot_past_2pow30_rows(large_case):
    """col.uniq(7) and col.hot(5, 7) over 1.85e9 rows (owner ids up to 86% of the table's empty mark 0x7FFFFFFF) of at
    most 131,074 distinct (k, v) pairs, one of which holds more than 2^30 rows and two of which first occur past row
    2^30, one of them only in the last row.  The reference: a dense pair code, its torch.bincount and first row by
    scatter_reduce(amin), partitions from the oracle's portable_hash of (k, v)."""
    from oracle import oracle as orc
    from dpark_b200.selecting import ColumnarUniqRDD
    from tests.test_gpu_uniq_top_hot import _tuple_hash2
    n, P, K, V = 1_850_000_003, 7, 8192, 16                        # k in [0, K + 2), v in [-8, 8)

    def body():
        keys = _randint32(n, 0, K, 31)
        vals = _randint32(n, -8, 8, 32)
        g = _gen(33)
        for a in range(0, n, CHUNK):                               # the hot pair (17, -3): ~ 0.995 of the rows
            hot = torch.rand(min(CHUNK, n - a), device="cuda", generator=g) < 0.995
            keys[a:a + CHUNK][hot] = 17
            vals[a:a + CHUNK][hot] = -3
        late = _spread(n, 50, 1 << 30, 34)                          # (K, 0) first at row 2^30, (K + 1, 7) only last
        keys[late], vals[late] = K, 0
        keys[-1], vals[-1] = K + 1, 7
        col = _ctx().parallelizeColumns(keys, vals, 8)
        u = col.uniq(P)
        assert isinstance(u, ColumnarUniqRDD)
        got = [u.columns(sp) for sp in u.splits]
        ucount = u._materialize()[2]
        hot_got = col.hot(5, P)

        C = (K + 2) * V
        counts = torch.zeros(C, dtype=torch.int64, device="cuda")
        first = torch.full((C,), n, dtype=torch.int64, device="cuda")
        for a in range(0, n, CHUNK):
            code = keys[a:a + CHUNK].long() * V + (vals[a:a + CHUNK].long() + 8)
            counts += torch.bincount(code, minlength=C)
            first.scatter_reduce_(0, code, torch.arange(a, a + code.numel(), device="cuda"), "amin")
        codes = counts.nonzero().flatten()
        ck, cv = (codes // V).cpu().numpy(), (codes % V - 8).cpu().numpy()
        pid = orc.partition_vec(_tuple_hash2(orc.hash_vec(ck), orc.hash_vec(cv)), P)
        fh, ch = first[codes].cpu().numpy(), counts[codes].cpu().numpy()
        assert int(ch.max()) > 1 << 30 and int(fh.max()) == n - 1
        order = np.lexsort((fh, pid))                             # uniq's order: by partition, then first row
        for p in range(P):
            sel = order[pid[order] == p]
            gk, gv = got[p]
            assert gk.dtype == torch.int32 and gv.dtype == torch.int32
            assert gk.cpu().numpy().tolist() == ck[sel].tolist(), "partition %d: keys" % p
            assert gv.cpu().numpy().tolist() == cv[sel].tolist(), "partition %d: values" % p
        want_count = ch[order].tolist()
        assert ucount.cpu().tolist() == want_count
        rank = sorted(range(len(order)), key=lambda i: -want_count[i])[:5]        # stable: ties in uniq's order
        assert hot_got == [((int(ck[order[i]]), int(cv[order[i]])), want_count[i]) for i in rank]
        assert hot_got[0] == ((17, -3), int(ch.max()))
    large_case("uniq / hot, n=%d" % n, 74, body)


@pytest.mark.gpu
def test_topbykey_one_key_past_2pow30_values(large_case):
    """col.topByKey(100) over 2^30 + 2^20 + 5 rows with float32 values, one key holding more than 2^30 of them: every
    key's 100 smallest values, ties in row order, bit for bit.  The hot key's candidates for the cut are signed zeros
    that occur only at rows past 2^30, so which zeros win (and their signs) depends on the group-by keeping row order
    across a run longer than 2^30.  The reference: a stable torch.sort by value (-0.0 as 0.0), then a stable one by
    key, each key's run cut at 100."""
    from dpark_b200.topk import ColumnarTopByKeyRDD
    n, P, top_n, hot_key = (1 << 30) + (1 << 20) + 5, 5, 100, 7

    def body():
        ids = torch.arange(0, n, 4096, device="cuda")             # the other keys' rows
        keys = torch.full((n,), hot_key, dtype=torch.int32, device="cuda")
        keys[ids] = (1000 + (ids // 4096) % 255).int()
        vals = _randint32(n, 1, 1000, 61).float()
        zero = torch.rand(n, device="cuda", generator=_gen(62)) < 1 / 64
        zero[:1 << 30] = False
        vals[zero] = torch.where(torch.rand(n, device="cuda", generator=_gen(63))[zero] < 0.5, -0.0, 0.0)
        del zero
        col = _ctx().parallelizeColumns(keys, vals, 8)
        out = col.topByKey(top_n, num_splits=P)
        assert isinstance(out, ColumnarTopByKeyRDD)
        got = {}
        for sp in out.splits:
            k, off, v = out.columns(sp)
            off, bits = off.tolist(), v.view(torch.int32).tolist()
            for j, key in enumerate(k.tolist()):
                assert key % P == sp.index
                got[key] = bits[off[j]:off[j + 1]]
        del out, k, off, v

        o1 = torch.sort(vals + 0.0, stable=True).indices
        order = o1[torch.sort(keys[o1], stable=True).indices]
        del o1
        gkeys, counts = torch.unique_consecutive(keys[order], return_counts=True)
        take = counts.clamp(max=top_n)
        starts = torch.cumsum(counts, 0) - counts
        first = torch.cumsum(take, 0) - take
        pos = torch.repeat_interleave(starts - first, take) + torch.arange(int(take.sum()), device="cuda")
        want_bits, want_ids = vals[order[pos]].view(torch.int32).tolist(), order[pos].tolist()
        at = (torch.cumsum(take, 0) - take).tolist()
        want = {key: want_bits[at[j]:at[j] + min(top_n, c)] for j, (key, c) in enumerate(zip(gkeys.tolist(),
                                                                                            counts.tolist()))}
        hot = gkeys.tolist().index(hot_key)
        assert counts[hot] > 1 << 30 and min(want_ids[at[hot]:at[hot] + top_n]) >= 1 << 30
        assert set(want[hot_key]) == {0, -(1 << 31)}                 # both zeros among the winners
        assert got == want
    large_case("topByKey, n=%d" % n, 73, body)


@pytest.mark.gpu
def test_percentiles_by_key_one_key_past_2pow30_values(large_case):
    """col.percentilesByKey([5, 50, 95, 99.97]) over 2^30 + 2^20 + 5 rows in 8 splits, one key holding more than 2^30
    of them: that run goes through the group-by and the segment heads whole, and is digested per split (about 1.3e8
    values each), as the composition digests it.  Every other key (255 of them, ~1000 rows each over all splits) bit
    for bit against the composition's digests run on just that key's rows in split order (one MergingDigest per
    split, absorbed in split order).  The hot key, whose digests no host can build in reasonable time: its values
    past row 2^30 (0.1% of them) lie in [1e4, 1e4 + 100], far above the others, so its 99.97th percentile must land
    among them (a lost or misplaced row past 2^30 moves it out); each answer's rank among its values within 1% of
    the percentile, within 0.05% for the 99.97th."""
    from dpark_b200 import quantiles
    from dpark_b200.percentiles import ColumnarPercentilesByKeyRDD
    n, P, hot_key, pcts = (1 << 30) + (1 << 20) + 5, 3, 7, [5, 50, 95, 99.97]

    def body():
        ids = torch.arange(0, n, 4096, device="cuda")             # the other keys' rows
        keys = torch.full((n,), hot_key, dtype=torch.int32, device="cuda")
        keys[ids] = (1000 + (ids // 4096) % 255).int()
        vals = torch.randn(n, dtype=torch.float32, device="cuda", generator=_gen(91)) * 100
        tail = vals[1 << 30:]
        tail[keys[1 << 30:] == hot_key] = 1e4 + torch.rand(n - (1 << 30), device="cuda", generator=_gen(92))[
            keys[1 << 30:] == hot_key] * 100
        col = _ctx().parallelizeColumns(keys, vals, 8)
        out = col.percentilesByKey(pcts, numSplits=P)
        assert isinstance(out, ColumnarPercentilesByKeyRDD)
        got = {}
        for sp in out.splits:
            k, q = out.columns(sp)
            for key, qs in zip(k.tolist(), q.tolist()):
                assert key % P == sp.index
                got[key] = qs
        del out, k, q
        assert len(got) == 256

        per = col.splits[0].end - col.splits[0].begin
        ck, cv, split = keys[ids].tolist(), vals[ids].tolist(), (ids // per).tolist()
        tagged = {}
        for key, v, s in zip(ck, cv, split):
            tagged.setdefault(key, []).append((s, v))
        for key, tv in tagged.items():
            merged = None
            for _, group in itertools.groupby(tv, key=lambda t: t[0]):
                d = quantiles.MergingDigest()
                for _, v in group:
                    d.add(v)
                merged = d if merged is None else merged.absorb(d)
                merged.compress()
            want = [merged.quantile(pp / 100.) for pp in pcts]
            assert [struct.pack("<d", x) for x in got[key]] == [struct.pack("<d", x) for x in want], key

        hv = vals[keys == hot_key]
        assert hv.numel() > 1 << 30
        for pp, x in zip(pcts, got[hot_key]):
            assert abs(int((hv < x).sum()) / hv.numel() - pp / 100.) < (0.0005 if pp > 99 else 0.01), (pp, x)
        assert 1e4 <= got[hot_key][-1] <= 1e4 + 100
    large_case("percentilesByKey, n=%d" % n, 73, body)


def _python_draws(seed, m):
    """The first m random.Random(seed).random() draws, from numpy's MT19937 set to that generator's state (the same
    generator and the same 53-bit double from two words; checked against random.Random on a prefix)."""
    words = random.Random(seed).getstate()[1]
    rs = np.random.RandomState()
    rs.set_state(("MT19937", np.array(words[:624], dtype=np.uint32), words[624]))
    out = rs.random_sample(m)
    rd = random.Random(seed)
    assert [rd.random() for _ in range(1000)] == out[:1000].tolist()
    return out


@pytest.mark.gpu
def test_sample_past_2pow30_rows(large_case):
    """col.sample(0.3, False, 17) over 2^30 + 2^24 + 7 rows in 8 splits: every split's kept rows, in row order, are the
    rows j whose j-th random.Random(17 + i).random() draw of split i is <= 0.3 (values are the row ids)."""
    from dpark_b200.sampling import ColumnarSampleRDD
    n, frac, seed = (1 << 30) + (1 << 24) + 7, 0.3, 17

    def body():
        keys = _randint32(n, -(1 << 31), (1 << 31) - 1, 95)
        vals = torch.arange(n, dtype=torch.int32, device="cuda")
        col = _ctx().parallelizeColumns(keys, vals, 8)
        out = col.sample(frac, False, seed)
        assert isinstance(out, ColumnarSampleRDD)
        for sp, src in zip(out.splits, col.splits):
            k, v = out.columns(sp)
            want = np.flatnonzero(_python_draws(seed + sp.index, src.end - src.begin) <= frac) + src.begin
            assert v.numel() == want.size, "split %d: kept rows" % sp.index
            assert np.array_equal(v.cpu().numpy(), want), "split %d: kept row ids" % sp.index
            assert torch.equal(k, keys[v.long()]), "split %d: kept keys" % sp.index
        assert int(v[-1]) >= 1 << 30
    large_case("sample, n=%d" % n, 19, body)


def _runs_in_key_order(keys, lens, cols):
    """Device groups (keys[G], run lengths lens[G], value columns cols whose runs follow one another in group order)
    reordered by key: (sorted keys, lens in that order, the columns' runs gathered in that order)."""
    perm = torch.argsort(keys)
    starts = torch.cumsum(lens, 0) - lens
    ls = lens[perm]
    idx = torch.repeat_interleave(starts[perm] - (torch.cumsum(ls, 0) - ls), ls) + torch.arange(int(ls.sum()),
                                                                                                 device="cuda")
    return keys[perm], ls, [c[idx] for c in cols]


@pytest.mark.gpu
def test_cogroup_past_2pow30_row_ids(large_case):
    """a.groupWith(b) (the device cogroup) over 2^30 + 2^20 + 8 rows: a in 8 map splits, b in 3, every split of an odd
    size, a's keys a quarter one hot key, b's keys partly disjoint from a's.  Rows are numbered across both inputs, so
    b's ids pass 2^30.  Every key of either input, every key's value count per input and every value, bit for bit and
    in order, against each input's stable torch.sort by key; every key in partition portable_hash(k) % P.

    What this covers of groupByKey is its device group-by (grouping.group_row_ids), here at 1.07e9 rows over 11 map
    splits; ColumnarRDD.groupByKey then builds host value lists, which no host holds at this size, and the group-by at
    2^31 - 2^20 rows needs 144 GiB (note (3))."""
    from dpark_b200.join import ColumnarCoGroupedRDD
    na, nb, P, hot_key = 7 * (1 << 27) + 5, (1 << 27) + (1 << 20) + 3, 6, 12345
    assert na + nb > 1 << 30 and (-(-na // 8)) % 2 and (-(-nb // 3)) % 2

    def body():
        ka = _randint32(na, 0, 1 << 20, 71)
        ka[torch.rand(na, device="cuda", generator=_gen(72)) < 0.25] = hot_key
        va = torch.arange(na, dtype=torch.int32, device="cuda")
        kb = _randint32(nb, 1 << 19, (1 << 20) + (1 << 18), 73)
        vb = _randint32(nb, -8, 8, 74).float() * 0.5
        vb[vb == 0] = torch.where(torch.rand(nb, device="cuda", generator=_gen(75))[vb == 0] < 0.5, -0.0, 0.0)
        dc = _ctx()
        a, b = dc.parallelizeColumns(ka, va, 8), dc.parallelizeColumns(kb, vb, 3)
        out = a.groupWith(b, P)
        assert isinstance(out, ColumnarCoGroupedRDD)
        parts = [out.columns(sp) for sp in out.splits]
        for p, (k, _, _) in enumerate(parts):
            h = k.clone()
            h[h == -1] = -2
            assert bool((torch.remainder(h, P) == p).all()), "partition %d holds another partition's key" % p
        del k, h
        dk = torch.cat([k for k, _, _ in parts])
        lens = [torch.cat([o[t, 1:] - o[t, :-1] for _, o, _ in parts]) for t in range(2)]
        cols = [torch.cat([v[t] for _, _, v in parts]) for t in range(2)]
        del out, parts
        allk = torch.unique(torch.cat([ka, kb]).long())
        for t, (keys, vals) in enumerate(((ka, va), (kb, vb))):
            sk, ls, (got,) = _runs_in_key_order(dk, lens[t], [cols[t]])
            assert torch.equal(sk, allk), "the keys differ"
            assert torch.equal(ls, torch.bincount(keys.long() - int(allk[0]), minlength=int(allk[-1] - allk[0]) + 1)
                               [allk - allk[0]]), "input %d: a key's value count differs" % t
            want = vals[torch.sort(keys, stable=True).indices]
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), "input %d: values differ" % t
            del sk, ls, got, want
    large_case("cogroup, n=%d" % (na + nb), 73, body)


def _join_case(how, nl, nr, lspan, rlo, rspan, P, seed, min_out):
    """left.<how>(right, P) of int32 keys (left in [0, lspan), right in [rlo, rspan)) with int32 left values (the row
    ids) and float32 right values.  Against bincount / index_add_ of each input's keys: every key's output row count
    (L x R, a missing side counting 1 where the join kind keeps the other) and int64 sums of the left values and of the
    right values' bits; every key in partition portable_hash(k) % P; and, bit for bit with their valid flags and in
    `for a in left for b in right` order, the whole output of 40 sampled keys, of the keys of both inputs' last rows
    and of the key at output row 2^31 if there is one.  At least min_out output rows."""
    keep_left, keep_right = how in ("leftOuterJoin", "outerJoin"), how in ("rightOuterJoin", "outerJoin")
    lk = _randint32(nl, 0, lspan, seed)
    lv = torch.arange(nl, dtype=torch.int32, device="cuda")
    rk = _randint32(nr, rlo, rspan, seed + 1)
    rv = torch.randn(nr, dtype=torch.float32, device="cuda", generator=_gen(seed + 2))
    dc = _ctx()
    out = getattr(dc.parallelizeColumns(lk, lv, 8), how)(dc.parallelizeColumns(rk, rv, 3), P)
    assert type(out).__name__ == "ColumnarJoinedRDD"
    parts = [out.columns(sp) for sp in out.splits]
    del out

    span = max(lspan, rspan)
    L, R = torch.bincount(lk.long(), minlength=span), torch.bincount(rk.long(), minlength=span)
    Ls = torch.zeros(span, dtype=torch.int64, device="cuda").index_add_(0, lk.long(), lv.long())
    Rs = torch.zeros(span, dtype=torch.int64, device="cuda").index_add_(0, rk.long(), rv.view(torch.int32).long())
    SL = torch.where(L > 0, L, int(keep_right))
    SR = torch.where(R > 0, R, int(keep_left))
    cnt, lsum, rsum = (torch.zeros(span, dtype=torch.int64, device="cuda") for _ in range(3))
    total = 0
    for p, (ok, ol, orr, olv, orv) in enumerate(parts):
        assert ok.dtype == torch.int64 and ol.dtype == torch.int32 and orr.dtype == torch.float32
        assert (olv is None) != keep_right and (orv is None) != keep_left
        for a in range(0, int(ok.numel()), CHUNK):
            kc = ok[a:a + CHUNK]
            assert bool((kc % P == p).all()), "partition %d holds another partition's key" % p
            cnt += torch.bincount(kc, minlength=span)
            lsum.index_add_(0, kc, ol[a:a + CHUNK].long())
            rsum.index_add_(0, kc, orr[a:a + CHUNK].view(torch.int32).long())
        total += int(ok.numel())
    assert torch.equal(cnt, SL * SR), "a key's output row count differs"
    assert torch.equal(lsum, Ls * SR), "a key's left values differ"
    assert torch.equal(rsum, Rs * SL), "a key's right values differ"

    present = (SL * SR).nonzero().flatten()
    pick = present[torch.randperm(int(present.numel()), device="cuda", generator=_gen(seed + 3))[:40]].tolist()
    pick += [int(lk[-1]), int(rk[-1])]
    assert total >= min_out
    if total > 1 << 31:
        at = 1 << 31
        for ok, _, _, _, _ in parts:
            if at < ok.numel():
                pick.append(int(ok[at]))
                break
            at -= int(ok.numel())
    for k in pick:
        ok, ol, orr, olv, orv = parts[k % P]
        idx = (ok == k).nonzero().flatten()
        a, b = lv[lk == k], rv[rk == k]
        sl, sr = int(SL[k]), int(SR[k])
        if sl * sr == 0:
            assert idx.numel() == 0, "key %d: rows for a key without output" % k
            continue
        assert idx.numel() == sl * sr and int(idx[-1] - idx[0]) + 1 == sl * sr, "key %d: rows not one run" % k
        wl = (a if a.numel() else torch.zeros(1, dtype=a.dtype, device="cuda")).repeat_interleave(sr)
        wr = (b if b.numel() else torch.zeros(1, dtype=b.dtype, device="cuda")).repeat(sl)
        assert torch.equal(ol[idx], wl) and torch.equal(orr[idx].view(torch.int32), wr.view(torch.int32)), k
        if olv is not None:
            assert bool((olv[idx] == int(a.numel() > 0)).all()), k
        if orv is not None:
            assert bool((orv[idx] == int(b.numel() > 0)).all()), k


@pytest.mark.gpu
def test_left_outer_join_past_2pow30_row_ids(large_case):
    """leftOuterJoin over 2^30 + 2^20 + 5 left rows in 8 map splits and 2^19 + 3 right rows in 3, numbered across both
    inputs, so the left input's tail and every right row have ids past 2^30 in the group-by; half the left keys find
    no right row and keep a None.  The group-by needs 72 bytes per row, so output rows stay near 1.07e9 here; the
    join's output past 2^31 rows is the next case."""
    nl, nr = (1 << 30) + (1 << 20) + 5, (1 << 19) + 3
    large_case("leftOuterJoin, n=%d" % (nl + nr), 73,
               lambda: _join_case("leftOuterJoin", nl, nr, 1 << 20, 1 << 19, (1 << 20) + (1 << 19), 5, 101, nl))


@pytest.mark.gpu
def test_join_past_2pow31_output_rows(large_case):
    """join of 2e8 left rows over 2^16 keys with 786,435 right rows over the same keys: about 2.4e9 output rows, so
    k_join_emit's output row ids, tiles and group offsets pass 2^31."""
    nl, nr = 200_000_001, 12 * (1 << 16) + 3
    large_case("join, n=%d" % (nl + nr), 45,
               lambda: _join_case("join", nl, nr, 1 << 16, 0, 1 << 16, 7, 111, (1 << 31) + (1 << 27)))


@pytest.mark.gpu
def test_inner_join_past_2pow31_output_rows(large_case):
    """big.innerJoin(small) with 1.2e9 big rows in 8 splits, 1 in 17 of their keys absent from the small side, which
    holds every other key 1 to 3 times: 2.26e9 output rows, so output row ids pass 2^31 (innerJoin has no row cap).
    Per big split: the output row count and four int64 checksums (of keys, of left values, of right values, of
    left x right, wrapping as the device sums do) against each big row's multiplicity and right-value sum from a
    torch.sort of the small side; and every output row, bit for bit, in windows at each split's start and end and
    around output row 2^31."""
    from dpark_b200.join import ColumnarInnerJoinedRDD
    n, ns, span = 1_200_000_007, 1 << 20, (1 << 20) + (1 << 16)      # big keys >= 2^20 find nothing

    def body():
        keys = _randint32(n, 0, span, 81)
        vals = _randint32(n, -(1 << 31), (1 << 31) - 1, 82)
        skeys = torch.arange(ns, dtype=torch.int32, device="cuda").repeat_interleave(
            torch.arange(ns, device="cuda") % 3 + 1)
        skeys = skeys[torch.randperm(skeys.numel(), device="cuda", generator=_gen(83))]
        svals = _randint32(skeys.numel(), -(1 << 31), (1 << 31) - 1, 84)
        dc = _ctx()
        big, small = dc.parallelizeColumns(keys, vals, 8), dc.parallelizeColumns(skeys, svals, 2)
        out = big.innerJoin(small)
        assert isinstance(out, ColumnarInnerJoinedRDD)
        parts = [out.columns(sp) for sp in out.splits]

        order = torch.sort(skeys, stable=True).indices          # a key's right values in small row order
        rsorted = svals[order].long()
        mult = torch.bincount(skeys.long(), minlength=span)
        first = torch.cumsum(mult, 0) - mult
        rsum = torch.zeros(span, dtype=torch.int64, device="cuda").index_add_(0, skeys.long(), svals.long())
        m = mult[keys.long()]
        off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
        torch.cumsum(m, 0, out=off[1:])
        total = int(off[-1])
        assert total > (1 << 31) + (1 << 20)

        def expect(i):
            r = torch.searchsorted(off, i, right=True) - 1
            k = keys[r]
            return k, vals[r], rsorted[first[k.long()] + i - off[r]].int()

        seen = 0
        for sp, (k, l, r) in zip(big.splits, parts):
            b, e = sp.begin, sp.end
            rows = int(off[e] - off[b])
            assert k.numel() == l.numel() == r.numel() == rows, "split %d: output rows" % sp.index
            ms, kb = m[b:e], keys[b:e].long()
            want = [int((kb * ms).sum()), int((vals[b:e].long() * ms).sum()), int(rsum[kb].sum()),
                    int((vals[b:e].long() * rsum[kb]).sum())]
            got = [int(k.long().sum()), int(l.long().sum()), int(r.long().sum()), int((l.long() * r.long()).sum())]
            assert got == want, "split %d: checksums" % sp.index
            windows = [torch.arange(0, min(rows, 256)), torch.arange(max(0, rows - 256), rows)]
            if seen <= 1 << 31 < seen + rows:
                windows.append(torch.arange(max(0, (1 << 31) - seen - 512), min(rows, (1 << 31) - seen + 512)))
            for w in windows:
                w = w.cuda()
                for got_col, want_col in zip((k[w], l[w], r[w]), expect(w + seen)):
                    assert torch.equal(got_col, want_col), "split %d: output rows %d.." % (sp.index, int(w[0]) + seen)
            seen += rows
        assert seen == total
    large_case("innerJoin, n=%d" % n, 60, body)


def _gamma(m):
    """gamma(m) = m u / (1 - m u), u = 2^-53: |float64 sum of m + 1 terms in any order - exact| <= gamma(m) sum|v|."""
    u = 2.0 ** -53
    return m * u / (1 - m * u)


def _reduce_case(splits, vdt, seed):
    """reduceByKey(sum) over int32 key splits with int32 or float32 values.  Every key in partition portable_hash(k) %
    P (portable_hash of an int is the int, -1 -> -2), the distinct keys those of a torch.bincount, and each key's sum
    against a chunked torch index_add_: int64 sums exactly; float64 sums within 2 gamma(m - 1) sum|v| for a key of m
    rows (both sums are off the exact one by at most half that), and for 1000 sampled keys within gamma(m - 1) sum|v|
    of math.fsum of their rows."""
    from dpark_b200 import shuffle
    P, half = 8, 1 << 22                                           # keys in [-2^22, 2^22): ~170 rows each
    n = sum(splits)
    ks = [_randint32(m, -half, half, seed + i) for i, m in enumerate(splits)]
    if vdt == torch.int32:
        vs = [_randint32(m, -(1 << 31), (1 << 31) - 1, seed + 100 + i) for i, m in enumerate(splits)]
    else:
        vs = [torch.randn(m, dtype=torch.float32, device="cuda", generator=_gen(seed + 100 + i)) * 1e3
              for i, m in enumerate(splits)]
    res = shuffle.reduce_by_key(ks, vs, P, "sum")
    assert [p for p, _, _ in res] == list(range(P))
    gk = torch.cat([k for _, k, _ in res])
    gs = torch.cat([s for _, _, s in res])
    gp = torch.cat([torch.full((int(k.numel()),), p, dtype=torch.int64, device="cuda") for p, k, _ in res])
    del res
    acc = torch.int64 if vdt == torch.int32 else torch.float64
    assert gk.dtype == torch.int32 and gs.dtype == acc

    sums = torch.zeros(2 * half, dtype=acc, device="cuda")
    mags = torch.zeros(2 * half, dtype=torch.float64, device="cuda")
    counts = torch.zeros(2 * half, dtype=torch.int64, device="cuda")
    for k, v in zip(ks, vs):
        for a in range(0, int(k.numel()), CHUNK):
            idx = k[a:a + CHUNK].long() + half
            sums.index_add_(0, idx, v[a:a + CHUNK].to(acc))
            if acc == torch.float64:
                mags.index_add_(0, idx, v[a:a + CHUNK].double().abs())
            counts += torch.bincount(idx, minlength=2 * half)
    assert int(counts.sum()) == n
    present = counts.nonzero().flatten()
    order = torch.argsort(gk)
    gk, gs, gp = gk[order], gs[order], gp[order]
    assert torch.equal(gk.long(), present - half), "the distinct keys differ"
    h = gk.long()
    h[h == -1] = -2
    assert torch.equal(torch.remainder(h, P), gp), "a key is in the wrong partition"
    if acc == torch.int64:
        assert torch.equal(gs, sums[present]), "a key's sum differs"
        return
    m = counts[present].double()
    gam = (m - 1) * 2.0 ** -53 / (1 - (m - 1) * 2.0 ** -53)
    err = (gs - sums[present]).abs()
    assert bool((err <= 2 * gam * mags[present]).all()), "a key's sum is off by more than 2 gamma(m - 1) sum|v|"

    pick = present[torch.randperm(int(present.numel()), device="cuda", generator=_gen(seed + 200))[:1000]] - half
    rows = {}
    for k, v in zip(ks, vs):
        for a in range(0, int(k.numel()), CHUNK):
            kc = k[a:a + CHUNK]
            hit = torch.isin(kc, pick.int())
            for key, val in zip(kc[hit].tolist(), v[a:a + CHUNK][hit].tolist()):
                rows.setdefault(key, []).append(val)
    at = torch.searchsorted(gk.long(), pick)
    for key, dev_sum in zip(pick.tolist(), gs[at].tolist()):
        vals = rows[key]
        exact = math.fsum(vals)
        assert abs(dev_sum - exact) <= _gamma(len(vals) - 1) * math.fsum(abs(x) for x in vals), key


REDUCE_N = 1_450_000_002       # 1.5 n + 40 F + 64 combine slots: past 2^31


@pytest.mark.gpu
@pytest.mark.parametrize("vdt", [torch.int32, torch.float32], ids=str)
def test_reduce_by_key_one_split_past_2pow31_slots(large_case, vdt):
    large_case("reduceByKey %s, 1 split, n=%d" % (vdt, REDUCE_N), 72, lambda: _reduce_case([REDUCE_N], vdt, 41))


@pytest.mark.gpu
def test_reduce_by_key_eight_splits_past_2pow31_slots(large_case):
    """8 separately allocated map splits (one partition launch pair each): sizes are odd, none a multiple of a tile."""
    per = REDUCE_N // 8 + 1
    splits = [per + (14 if i % 2 else -14) for i in range(7)]
    splits.append(REDUCE_N - sum(splits))
    assert all(m % 2 for m in splits)
    large_case("reduceByKey 8 splits, n=%d" % REDUCE_N, 72, lambda: _reduce_case(splits, torch.int32, 51))
