"""Host-buffer entry points (what bench.py's e2e leg times): HostShuffle.run and the
pipelined HostShuffleStream.submit/collect must return exactly the reference's
reduceByKey result (dpark/rdd.py:303-327 over task.py:209-226 + shuffle.py:600-608).  -m gpu."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc

pytestmark = pytest.mark.gpu


def _check(parts, want, P):
    seen = set()
    for p, k, v in parts:
        seen.add(p)
        k, v = k.numpy(), v.numpy()
        o1, o2 = np.argsort(k), np.argsort(want[p][0])
        assert np.array_equal(k[o1], want[p][0][o2])
        assert np.array_equal(v[o1], want[p][1][o2])
    assert seen == set(range(P))


def _batch(seed, n, hi):
    rng = np.random.default_rng(seed)
    return rng.integers(-hi, hi, n, dtype=np.int64), rng.integers(-1000, 1000, n, dtype=np.int64)


@pytest.mark.parametrize("P,splits,hi", [(8, 4, 2 ** 31), (3, 1, 5000), (1, 5, 100)])
def test_host_shuffle_run_matches_oracle(P, splits, hi):
    from dpark_b200 import shuffle
    n = 300_000
    k, v = _batch(P, n, hi)
    hs = shuffle.HostShuffle(n, torch.int64, torch.int64, P, "sum", splits=splits)
    hs.h_keys.copy_(torch.from_numpy(k))
    hs.h_vals.copy_(torch.from_numpy(v))
    want = orc.reduce_by_key(np.array_split(k, splits), np.array_split(v, splits), P, "sum")
    for _ in range(2):                      # buffers are reused between runs
        _check(hs.run(), want, P)


@pytest.mark.parametrize("depth", [1, 2, 3])
def test_host_shuffle_stream_pipelined_batches_keep_their_own_results(depth):
    from dpark_b200 import shuffle
    n, P, nb = 250_000, 8, 7
    st = shuffle.HostShuffleStream(n, torch.int64, torch.int64, P, "sum", splits=4, depth=depth)
    batches = []
    for b in range(nb):                     # every batch differs, so a slot mix-up cannot pass
        k, v = _batch(100 + b, n, 3000 * (b + 1))
        batches.append((torch.from_numpy(k).pin_memory(), torch.from_numpy(v).pin_memory(),
                        orc.reduce_by_key(np.array_split(k, 4), np.array_split(v, 4), P, "sum")))
    inflight, done = [], 0
    for b in range(nb):
        if len(inflight) == depth:
            _check(st.collect(), batches[inflight.pop(0)][2], P)
            done += 1
        st.submit(batches[b][0], batches[b][1])
        inflight.append(b)
    while inflight:
        _check(st.collect(), batches[inflight.pop(0)][2], P)
        done += 1
    assert done == nb
    assert st.h2d_bytes == n * 16


def test_host_shuffle_stream_refuses_overrun_and_underrun():
    from dpark_b200 import shuffle
    n = 1000
    st = shuffle.HostShuffleStream(n, torch.int64, torch.int64, 2, depth=1)
    with pytest.raises(RuntimeError):
        st.collect()
    k = torch.arange(n, dtype=torch.int64).pin_memory()
    st.submit(k, k)
    with pytest.raises(RuntimeError):
        st.submit(k, k)
    parts = st.collect()
    assert sum(int(kk.numel()) for _, kk, _ in parts) == n


def test_copy_segments_moves_every_byte_at_any_alignment():
    """dpk_copy_segments (the exchange as block pushes): segments of very different sizes and
    16/8/4/1-byte alignments land exactly, and bytes outside the segments stay untouched."""
    from dpark_b200 import _native as nv
    rng = np.random.default_rng(5)
    total = 6_000_000
    src = torch.from_numpy(rng.integers(0, 256, total, dtype=np.uint8)).cuda()
    dst = torch.full((total,), 7, dtype=torch.uint8, device="cuda")
    #        src_off   dst_off   bytes
    segs = [(0,        16,       1_000_000),      # 16-byte aligned
            (1_000_008, 1_100_008, 800_000),      # 8-byte
            (2_000_004, 2_100_012, 70_004),       # 4-byte
            (2_500_001, 2_600_003, 33_333),       # bytes
            (3_000_000, 3_000_000, 0),            # empty
            (3_100_000, 3_200_000, 2_500_000),    # much larger than the others
            (5_900_000, 5_900_016, 16)]
    so = torch.tensor([src.data_ptr() + a for a, _, _ in segs], dtype=torch.int64, device="cuda")
    do = torch.tensor([dst.data_ptr() + b for _, b, _ in segs], dtype=torch.int64, device="cuda")
    nb = torch.tensor([c for _, _, c in segs], dtype=torch.int64, device="cuda")
    nv.copy_segments(so, do, nb)
    want = np.full(total, 7, dtype=np.uint8)
    h = src.cpu().numpy()
    for a, b, c in segs:
        want[b:b + c] = h[a:a + c]
    assert np.array_equal(dst.cpu().numpy(), want)
    nv.copy_segments(so[:0], do[:0], nb[:0])      # empty table is a no-op


@pytest.mark.parametrize("op", ["sum", "max"])
def test_map_side_combine_gives_the_same_partitions(op):
    """reduce_by_key(map_combine=True) -- the reference's map-side dict upsert (dpark/task.py:222-226) as a
    local merge before the exchange -- must not change any partition's result, on a Zipf-like key column
    (one key holds ~10 % of the rows) with int32 values (the combined column is int64)."""
    from dpark_b200 import shuffle
    rng = np.random.default_rng(17)
    n, P, M = 800_000, 6, 4
    k = (rng.zipf(1.3, n) % 50_000).astype(np.int64)
    k[rng.random(n) < 0.1] = 7
    v = rng.integers(-500, 500, n).astype(np.int32)
    ks, vs = np.array_split(k, M), np.array_split(v, M)
    want = orc.reduce_by_key(ks, [x.astype(np.int64) for x in vs], P, op)
    for mc in (False, True):
        res = shuffle.reduce_by_key([torch.from_numpy(x).cuda() for x in ks], [torch.from_numpy(x).cuda() for x in vs],
                                    P, op, map_combine=mc)
        _check([(p, a.cpu(), b.cpu()) for p, a, b in res], want, P)
    # the combined map output holds one row per (distinct key): far fewer rows than went in
    mo = shuffle.map_side([torch.from_numpy(k).cuda()], [torch.from_numpy(v).cuda()], P, sub_bits=2, unordered=True)
    mc = shuffle.combine_map_output(mo, op)
    assert int(mc.keys.numel()) == len(np.unique(k)) and int(mc.offsets[-1]) == len(np.unique(k))


@pytest.mark.parametrize("G,P,sb,H", [(2, 8, 0, 1), (3, 5, 1, 1), (8, 64, 3, 1), (4, 1, 3, 1), (8, 5, 2, 2)])
def test_push_plan_kernel_equals_the_tensor_plan_with_landed_segments(G, P, sb, H):
    """dpk_push_plan (one launch) against peer.push_plan (the tensor arithmetic the CPU tests pin to the alltoallv
    layout): segment table of every source row, clamping at the receive-buffer capacity, the capacity flag and the
    segment matrix of the rows that land in the rank's own buckets."""
    from dpark_b200 import _native as nv
    from dpark_b200 import peer, shuffle
    rng = np.random.default_rng(G * 100 + P)
    F = P << sb
    S = G * H
    counts = torch.from_numpy(rng.integers(0, 50, (S, F), dtype=np.int64)).cuda()
    blocks = [b << sb for b in shuffle.owner_blocks(P, G)]
    per_block = ((P + G - 1) // G) << sb
    keys = torch.zeros(int(counts.sum()) + 8, dtype=torch.int64, device="cuda")
    vals = torch.zeros(int(counts.sum()) + 8, dtype=torch.int32, device="cuda")
    dst_base = torch.arange(1, 2 * G + 1, dtype=torch.int64, device="cuda") * (1 << 40)
    for cap in (10 ** 9, int(counts.sum(0).max()) // 2 + 1):
        for rank in range(G):
            for h in range(H):
                me = rank * H + h
                need = torch.zeros(1, dtype=torch.int64, device="cuda")
                src, dst, nby, seg = nv.push_plan(counts, G, per_block, me, rank, keys, vals, dst_base, cap, need)
                sf, df, rows, tot = peer.push_plan(counts, blocks, me)
                rows = torch.minimum(rows, (cap - df).clamp(min=0))
                assert torch.equal(src[:G], keys.data_ptr() + sf * 8) and torch.equal(src[G:], vals.data_ptr() + sf * 4)
                assert torch.equal(dst[:G], dst_base[:G] + df * 8) and torch.equal(dst[G:], dst_base[G:] + df * 4)
                assert torch.equal(nby[:G], rows * 8) and torch.equal(nby[G:], rows * 4)
                assert int(need) == max(0, int(tot.max()) - cap)
                # the segment matrix describes the rows that land: every source's push is clamped at the capacity
                mine = counts[:, blocks[rank]:blocks[rank + 1]]
                assert torch.equal(seg, peer._landed(mine, cap))
                assert int(seg.sum()) == min(int(mine.sum()), cap)
