"""Packed shuffle rows (DPK_K_PACKED): reduceByKey map outputs and reduce-side inputs whose key and value columns have
the same width travel as one [n, 2] buffer of (key, value) records.  The packed path must give what the column
(struct-of-arrays) path gives: bit-identical integer results and min/max, float sums within DESIGN.md §7's tolerance
(1e-9 * sum|v| per key: the merge adds in a run-to-run varying order either way).  -m gpu.

In-bounds mutations these tests are built to catch:
  * a record stride of 8 bytes instead of 16 in the second-level split's load (k_part_scatter_bulk, PK_IN): keys and
    values of neighbouring rows mix -> test_reduce_matches_column_path;
  * key and value halves swapped where the merge reads a record (k_smem_aggregate2, PACKED) -> the same test;
  * the histogram reading packed keys with a stride of 1 (k_part_count, PIN) -> wrong fine-bucket counts, rows merged
    in the wrong bucket -> test_reduce_matches_column_path and test_row_id_keys_packed."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc

pytestmark = pytest.mark.gpu

def nv():
    from dpark_b200 import _native
    return _native


def _columns(kdt, vdt, n, rng, hot=False, nkeys=None):
    k = rng.integers(-(nkeys or 2 ** 30), nkeys or 2 ** 30, n).astype(kdt)
    if hot:                                  # a few keys hold most rows: multi-window fine buckets
        k[rng.random(n) < 0.8] = 7
    if np.dtype(vdt).kind == "f":
        v = rng.normal(0, 1000, n).astype(vdt)
    else:
        v = rng.integers(-1000, 1000, n).astype(vdt)
    return k, v


def _column_path(kc, vc, P, sb, op):
    """The struct-of-arrays path through the native entry points: one map split at a time with column outputs,
    concatenated per bucket, then dpk_combine over the two columns."""
    F = P << sb
    parts = [nv().partition(k, v, P, None, False, sb, None, True, packed=False) for k, v in zip(kc, vc)]
    seg = sum((off[1:] - off[:-1]) for _, _, off in parts).unsqueeze(0).contiguous()
    if len(parts) == 1:
        keys, vals = parts[0][0], parts[0][1]
    else:
        offs = [off.cpu().tolist() for _, _, off in parts]
        keys = torch.cat([ok[o[b]:o[b + 1]] for b in range(F) for (ok, _, _), o in zip(parts, offs)])
        vals = torch.cat([ov[o[b]:o[b + 1]] for b in range(F) for (_, ov, _), o in zip(parts, offs)])
    return nv().combine(keys.contiguous(), vals.contiguous(), op, P, seg, 0, P, None, sb)


def _packed_path(kc, vc, P, sb, op):
    from dpark_b200 import shuffle
    mo = shuffle.map_side(kc, vc, P, None, False, sb, unordered=True)
    assert (mo.rows is not None) == nv().packable(kc[0], vc[0])     # same-width rows travel packed, others as columns
    if mo.rows is not None:
        assert mo.rows.shape == (sum(int(k.numel()) for k in kc), 2)
    return shuffle.reduce_side(shuffle.exchange(mo), op, P)


def _by_partition(res, P):
    ok, ov, po, cnt = (t.cpu().numpy() for t in res)
    assert (cnt >= 0).all()
    out = []
    for p in range(P):
        k, v = ok[po[p]:po[p] + cnt[p]], ov[po[p]:po[p] + cnt[p]]
        o = np.argsort(k, kind="stable")
        out.append((k[o], v[o]))
    return out


def _assert_same(a, b, P, float_sum, tol=None):
    for p, ((ka, va), (kb, vb)) in enumerate(zip(_by_partition(a, P), _by_partition(b, P))):
        assert np.array_equal(ka.view(np.uint8), kb.view(np.uint8)), "partition %d keys" % p
        if float_sum:
            assert np.all(np.abs(va - vb) <= 1e-9 * tol.get(p, 0) + 1e-300), "partition %d sums" % p
        else:
            assert np.array_equal(va.view(np.uint8), vb.view(np.uint8)), "partition %d values" % p


def _abs_sum_tol(k, v, P):
    """Per partition, the largest sum of |v| over one key (an upper bound of every key's tolerance)."""
    pid = orc.partition_vec(orc.hash_vec(k), P)
    tol = {}
    for p in range(P):
        sel = pid == p
        if sel.any():
            _, inv = np.unique(k[sel], return_inverse=True)
            tol[p] = float(np.bincount(inv, np.abs(v[sel].astype(np.float64))).max())
    return tol


def _run_both(k, v, P, sb, op, cuts):
    kd, vd = torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda()
    bounds = [0] + list(cuts) + [len(k)]
    kc = [kd[a:b].clone() for a, b in zip(bounds[:-1], bounds[1:])]      # separate buffers: one launch pair per split
    vc = [vd[a:b].clone() for a, b in zip(bounds[:-1], bounds[1:])]
    if len(kc) == 1:
        kc, vc = [kd], [vd]
    return _packed_path(kc, vc, P, sb, op), _column_path(kc, vc, P, sb, op)


KV = [("i64", "i64"), ("i64", "f64"), ("i32", "i32"), ("i32", "f32"),      # same width: packed
      ("i64", "i32"), ("i32", "i64"), ("i64", "f32")]                      # mixed width: columns all the way


@pytest.mark.parametrize("op", ["sum", "min", "max"])
@pytest.mark.parametrize("kv", KV, ids=lambda kv: "%s-%s" % kv)
def test_reduce_matches_column_path(kv, op):
    kdt, vdt = np.dtype(kv[0].replace("i", "int").replace("f", "float")), np.dtype(kv[1].replace("i", "int").replace("f", "float"))
    rng = np.random.default_rng(10 * KV.index(kv) + ["sum", "min", "max"].index(op))
    n = 3 * 8192 + 17                                       # a tail that is not a multiple of a tile
    k, v = _columns(kdt, vdt, n, rng, nkeys=20000)
    a, b = _run_both(k, v, 8, 3, op, [])
    float_sum = vdt.kind == "f" and op == "sum"
    _assert_same(a, b, 8, float_sum, _abs_sum_tol(k, v, 8) if float_sum else None)


@pytest.mark.parametrize("P,sb", [(1, 0), (8, 0), (8, 3), (8, 6), (4095, 0), (1, 6)])
@pytest.mark.parametrize("kv", [("i64", "i64"), ("i32", "f32")], ids=lambda kv: "%s-%s" % kv)
def test_partition_counts_and_sub_bits(kv, P, sb):
    kdt = np.int64 if kv[0] == "i64" else np.int32
    vdt = np.int64 if kv[1] == "i64" else np.float32
    rng = np.random.default_rng(P * 16 + sb)
    k, v = _columns(kdt, vdt, 200_003, rng, nkeys=50_000)
    a, b = _run_both(k, v, P, sb, "sum", [])
    fs = vdt == np.float32
    _assert_same(a, b, P, fs, _abs_sum_tol(k, v, P) if fs else None)


@pytest.mark.parametrize("shape", ["empty_split", "hot_key", "big_buckets"])
def test_reduce_shapes(shape):
    """An empty map split among others (the multi-split scatter into one packed buffer), one hot key, and fine buckets
    far above one staging window (the multi-window path of smem_aggregate_big)."""
    rng = np.random.default_rng(5)
    if shape == "empty_split":
        k, v = _columns(np.int64, np.int64, 100_000, rng, nkeys=10_000)
        a, b = _run_both(k, v, 8, 2, "sum", [30_000, 30_000, 77_777])
        P = 8
    elif shape == "hot_key":
        k, v = _columns(np.int64, np.float64, 300_000, rng, hot=True)
        a, b = _run_both(k, v, 4, 0, "max", [])
        P = 4
    else:
        k = rng.integers(0, 3000, 1_500_000).astype(np.int64)
        v = rng.integers(-5, 5, len(k)).astype(np.int64)
        a, b = _run_both(k, v, 2, 0, "sum", [])
        P = 2
    _assert_same(a, b, P, False)


def test_map_output_column_views_match_oracle():
    """The packed map output's key / value views hold, per bucket, the multiset of rows the oracle puts there."""
    from dpark_b200 import shuffle
    rng = np.random.default_rng(11)
    k, v = _columns(np.int32, np.float32, 123_457, rng, nkeys=1 << 20)
    P, sb = 8, 3
    mo = shuffle.map_side([torch.from_numpy(k).cuda()], [torch.from_numpy(v).cuda()], P, None, False, sb, unordered=True)
    assert mo.rows is not None and mo.keys.data_ptr() == mo.rows.data_ptr() and mo.keys.stride() == (2,)
    off = mo.offsets.cpu().numpy()
    ok, ov = mo.keys.cpu().numpy(), mo.vals.cpu().numpy()
    wk, wv, woff = orc.map_task(k, v, P, combine=False)
    pid = orc.partition_vec(orc.hash_vec(k), P)
    assert np.array_equal(np.bincount(pid, minlength=P), np.diff(woff))
    for p in range(P):                   # sub-bucket boundaries refine the partition boundaries
        a, b = off[p << sb], off[(p + 1) << sb]
        assert (a, b) == (woff[p], woff[p + 1])
        got = sorted(zip(ok[a:b].tolist(), ov[a:b].view(np.int32).tolist()))
        want = sorted(zip(k[pid == p].tolist(), v[pid == p].view(np.int32).tolist()))
        assert got == want


def test_row_id_keys_packed():
    """Row-id keys (DPK_K_ROWID, the strings / textingest reduce side) through the packed path vs the columns."""
    from dpark_b200 import shuffle
    rng = np.random.default_rng(3)
    words = [("w%d" % i).encode() for i in rng.integers(0, 5000, 60_000)]
    off = np.zeros(len(words) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(w) for w in words])
    data = torch.from_numpy(np.frombuffer(b"".join(words), dtype=np.uint8).copy()).cuda()
    d_off = torch.from_numpy(off).cuda()
    h = nv().hash_bytes(data, d_off, nv().BYTES_SIGNED)
    rep = nv().dict_encode(data, d_off, h)
    vals = torch.from_numpy(rng.integers(0, 100, len(words)).astype(np.int64)).cuda()
    P, sb = 4, 2
    mo = shuffle.map_side([rep], [vals], P, None, False, sb, row_hash=h, unordered=True)
    assert mo.rows is not None
    rx = shuffle.exchange(mo)
    a = nv().combine(rx.keys, rx.vals, "sum", P, rx.seg.contiguous(), rx.part_first, rx.nparts, None, sb, row_hash=h,
                     rows=rx.rows)
    k2, v2, o2 = nv().partition(rep, vals, P, None, False, sb, h, True, packed=False)
    b = nv().combine(k2, v2, "sum", P, (o2[1:] - o2[:-1]).unsqueeze(0).contiguous(), 0, P, None, sb, row_hash=h)
    _assert_same(a, b, P, False)


def test_combine_map_output_packed():
    from dpark_b200 import shuffle
    rng = np.random.default_rng(8)
    k, v = _columns(np.int64, np.int64, 150_000, rng, nkeys=3000)
    mo = shuffle.map_side([torch.from_numpy(k).cuda()], [torch.from_numpy(v).cuda()], 8, None, False, 2, unordered=True)
    mc = shuffle.combine_map_output(mo, "sum")
    assert mc.rows is not None
    res = shuffle.reduce_side(shuffle.exchange(mc), "sum", 8)
    want = orc.reduce_by_key([k], [v], 8, "sum")
    for p, (gk, gv) in enumerate(_by_partition(res, 8)):
        o = np.argsort(want[p][0])
        assert np.array_equal(gk, want[p][0][o]) and np.array_equal(gv, want[p][1][o])


MARK = 0x5A


def test_packed_buffers_stay_in_bounds():
    """Marker bytes behind the packed map output, the combine workspace and the combine outputs survive the step."""
    rng = np.random.default_rng(21)
    n, P, sb = 100_001, 8, 4
    k, v = _columns(np.int64, np.int64, n, rng, nkeys=40_000)
    kd, vd = torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda()
    L = nv().lib()
    F = P << sb
    counts, ws = nv().partition_count(kd, P, None, False, sb, None, None, True)
    off = torch.zeros(F + 1, dtype=torch.int64, device="cuda")
    off[1:] = torch.cumsum(counts, 0)
    pad = 64
    big = torch.full(((n + pad) * 16,), MARK, dtype=torch.uint8, device="cuda")
    rows = big.view(torch.int64).view(n + pad, 2)[:n]
    nv().partition_scatter(kd, vd, P, off[:-1].contiguous(), rows, None, ws, None, False, sb, None, True)
    assert (big[n * 16:] == MARK).all()
    seg = (off[1:] - off[:-1]).unsqueeze(0).contiguous()
    ws_bytes = L.dpk_combine_workspace_bytes(n, F, 1)
    wsb = torch.full((ws_bytes + 4096,), MARK, dtype=torch.uint8, device="cuda")
    ok = torch.full((n + pad,), -1, dtype=torch.int64, device="cuda")
    ov = torch.full((n + pad,), -1, dtype=torch.int64, device="cuda")
    po = torch.empty(P + 1, dtype=torch.int64, device="cuda")
    cnt = torch.empty(P, dtype=torch.int64, device="cuda")
    nv()._check(L.dpk_combine(nv()._ptr(rows), nv().K_I64 | nv().K_PACKED, None, None, nv().V_I64, n, nv().OPS["sum"], P,
                              None, 0, sb, 0, P, 1, nv()._ptr(seg), nv()._ptr(ok), nv()._ptr(ov), nv()._ptr(po),
                              nv()._ptr(cnt), nv()._ptr(wsb), ws_bytes, nv()._stream()))
    torch.cuda.synchronize()
    assert (wsb[ws_bytes:] == MARK).all()
    assert (ok[n:] == -1).all() and (ov[n:] == -1).all()
    b = _column_path([kd], [vd], P, sb, "sum")
    _assert_same((ok[:n], ov[:n], po, cnt), b, P, False)
