"""Parity of the CUDA kernels (through the C ABI) against the oracle.  -m gpu."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tests.shuffle_cases import dpk_options  # noqa: F401

pytestmark = pytest.mark.gpu


def nv():
    from dpark_b200 import _native
    return _native


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


EDGE_I64 = np.array([0, 1, -1, -2, 7, 2 ** 31, 2 ** 61 - 1, 2 ** 61, -(2 ** 61 - 1), -(2 ** 61),
                     2 ** 63 - 1, -2 ** 63, 2 * (2 ** 61 - 1), 4 * (2 ** 61 - 1) - 1], dtype=np.int64)


def rand_keys(dtype, n, seed):
    rng = np.random.default_rng(seed)
    if dtype == np.int64:
        a = rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64, endpoint=True)
        a[: min(n, len(EDGE_I64))] = EDGE_I64[: min(n, len(EDGE_I64))]
        return a
    if dtype == np.int32:
        a = rng.integers(-2 ** 31, 2 ** 31 - 1, n, dtype=np.int32, endpoint=True)
        a[: min(n, 4)] = np.array([-1, -2, 0, 2 ** 31 - 1], dtype=np.int32)[: min(n, 4)]
        return a
    if dtype == np.float64:
        a = rng.standard_normal(n) * 10.0 ** rng.integers(-30, 30, n)
        a[: min(n, 6)] = np.array([0.0, 1.5, -1.0, 2.0 ** 61, np.inf, -np.inf])[: min(n, 6)]
        return a
    if dtype == np.float32:
        return (rng.standard_normal(n) * 100).astype(np.float32)
    raise ValueError(dtype)


@pytest.mark.parametrize("dtype", [np.int64, np.int32, np.float64, np.float32])
def test_hash_keys_bit_exact(dtype):
    k = rand_keys(dtype, 200003, 1)
    got = nv().hash_keys(dev(k)).cpu().numpy()
    assert np.array_equal(got, orc.hash_vec(k))


@pytest.mark.parametrize("mode", [0, 1])
def test_hash_bytes_bit_exact(mode):
    rng = np.random.default_rng(3)
    if mode == 0:
        blobs = [bytes(rng.integers(0, 256, rng.integers(0, 40), dtype=np.uint8)) for _ in range(5000)]
    else:
        alph = [chr(c) for c in list(range(32, 127)) + [0xe9, 0x4f60, 0xffff, 0x10000, 0x1f600]]
        blobs = ["".join(rng.choice(alph, rng.integers(0, 20))).encode("utf-8") for _ in range(5000)]
    offs = np.zeros(len(blobs) + 1, dtype=np.int64)
    offs[1:] = np.cumsum([len(b) for b in blobs])
    data = np.frombuffer(b"".join(blobs), dtype=np.uint8)
    got = nv().hash_bytes(dev(data), dev(offs), mode).cpu().numpy()
    assert np.array_equal(got, orc.hash_bytes_vec(data, offs, mode))


@pytest.mark.parametrize("P", [1, 2, 3, 4, 6, 7, 8, 64, 100, 1000, 4096, 2 ** 20 + 7])
def test_partition_ids_floor_mod(P):
    h = rand_keys(np.int64, 100000, 5)
    got = nv().partition_ids(dev(h), P).cpu().numpy()
    assert np.array_equal(got, orc.partition_vec(h, P))


def test_partition_ids_thresholds_bisect():
    h = rand_keys(np.int64, 50000, 6)
    thr = np.sort(rand_keys(np.int64, 15, 7))
    got = nv().partition_ids(dev(h), 16, dev(thr)).cpu().numpy()
    assert np.array_equal(got, orc.partition_vec(h, 16, thr))


def _check_partition(k, v, P, thresholds=None):
    """The CUDA multisplit must equal a stable sort by oracle partition id:
    bucket-major, input order kept inside each bucket (bit-exact)."""
    ok, ov, off = nv().partition(dev(k), None if v is None else dev(v), P,
                                 None if thresholds is None else dev(thresholds))
    pid = orc.partition_vec(orc.hash_vec(k), P, thresholds)
    order = np.argsort(pid, kind="stable")
    woff = np.zeros(P + 1, dtype=np.int64)
    woff[1:] = np.cumsum(np.bincount(pid, minlength=P))
    assert np.array_equal(off.cpu().numpy(), woff)
    assert np.array_equal(ok.cpu().numpy().view(np.uint8), k[order].view(np.uint8))
    if v is not None:
        assert np.array_equal(ov.cpu().numpy().view(np.uint8), v[order].view(np.uint8))


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 4095, 4096, 4097, 100003, 1000000])
@pytest.mark.parametrize("P", [1, 3, 8, 64])
def test_partition_stable_i64_i64(n, P):
    k = rand_keys(np.int64, n, n + P)
    k[: n // 2] = np.abs(k[: n // 2]) % 1000          # duplicates + small keys
    v = np.arange(n, dtype=np.int64)                   # row index: proves stability
    _check_partition(k, v, P)


@pytest.mark.parametrize("P", [1000, 4096])
def test_partition_many_buckets(P):
    k = rand_keys(np.int64, 300000, P)
    _check_partition(k, np.arange(len(k), dtype=np.int64), P)


def test_partition_i32_f32_and_keys_only():
    k = rand_keys(np.int32, 250000, 11)
    v = rand_keys(np.float32, 250000, 12)
    _check_partition(k, v, 8)
    _check_partition(rand_keys(np.int64, 70000, 13), None, 6)


def test_partition_thresholds():
    k = rand_keys(np.int64, 120000, 14)
    thr = np.sort(rand_keys(np.int64, 7, 15))
    _check_partition(k, np.arange(len(k), dtype=np.int64), 8, thr)


def test_partition_prehashed_uses_hash_as_is():
    h = rand_keys(np.int64, 90000, 16)
    v = np.arange(len(h), dtype=np.int64)
    ok, ov, off = nv().partition(dev(h), dev(v), 7, prehashed=True)
    pid = orc.partition_vec(h, 7)
    order = np.argsort(pid, kind="stable")
    assert np.array_equal(ok.cpu().numpy(), h[order])
    assert np.array_equal(ov.cpu().numpy(), v[order])
    assert np.array_equal(off.cpu().numpy()[1:], np.cumsum(np.bincount(pid, minlength=7)))


def test_map_side_multi_chunk_equals_single_stable_partition():
    from dpark_b200 import shuffle
    k = rand_keys(np.int64, 300000, 17) % 5000
    v = np.arange(len(k), dtype=np.int64)
    cuts = [0, 1000, 1000, 150000, 299999, 300000]
    kc = [dev(k[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
    vc = [dev(v[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
    mo = shuffle.map_side(kc, vc, 8)
    wk, wv, woff = orc.map_task(k, v, 8, combine=False)
    assert np.array_equal(mo.offsets.cpu().numpy(), woff)
    assert np.array_equal(mo.keys.cpu().numpy(), wk)
    assert np.array_equal(mo.vals.cpu().numpy(), wv)


def _parts_from(res):
    return {p: (k.cpu().numpy(), v.cpu().numpy()) for p, k, v in res}


@pytest.mark.parametrize("op", ["sum", "min", "max", "and", "or", "xor"])
def test_reduce_by_key_i64_ops(op):
    from dpark_b200 import shuffle
    rng = np.random.default_rng(21)
    n, P, M = 400000, 8, 4
    k = rng.integers(-3000, 3000, n, dtype=np.int64)
    k[:5] = [-1, -2, -2 ** 63, 2 ** 63 - 1, 2 ** 61 - 1]
    v = rng.integers(-2 ** 31, 2 ** 31, n, dtype=np.int64)
    ks, vs = np.array_split(k, M), np.array_split(v, M)
    got = _parts_from(shuffle.reduce_by_key([dev(x) for x in ks], [dev(x) for x in vs], P, op))
    want = orc.reduce_by_key(ks, vs, P, op)
    for p in range(P):
        gk, gv = got[p]
        wk, wv = want[p]
        o1, o2 = np.argsort(gk), np.argsort(wk)
        assert np.array_equal(gk[o1], wk[o2])
        assert np.array_equal(gv[o1], wv[o2])


def test_reduce_by_key_mostly_distinct_keys():
    from dpark_b200 import shuffle
    rng = np.random.default_rng(22)
    n, P = 2000000, 8
    k = rng.integers(0, 2 ** 31, n, dtype=np.int64)
    v = rng.integers(0, 2 ** 16, n, dtype=np.int64)
    got = _parts_from(shuffle.reduce_by_key([dev(k)], [dev(v)], P, "sum"))
    want = orc.reduce_by_key([k], [v], P, "sum")
    for p in range(P):
        o1, o2 = np.argsort(got[p][0]), np.argsort(want[p][0])
        assert np.array_equal(got[p][0][o1], want[p][0][o2])
        assert np.array_equal(got[p][1][o1], want[p][1][o2])


def test_reduce_by_key_i32_f32_sum_tolerance():
    """C4 shape.  The reference adds Python floats (float64) in a
    nondeterministic order; the kernel accumulates in float64 with atomics.
    Tolerance: |gpu - ref| <= 1e-9 * sum|v| per key (fp64 reassociation)."""
    from dpark_b200 import shuffle
    rng = np.random.default_rng(23)
    n, P = 500000, 8
    k = rng.integers(0, 2 ** 12, n, dtype=np.int32)
    k[:3] = [-1, -2, -2 ** 31]
    v = rng.random(n, dtype=np.float32)
    got = _parts_from(shuffle.reduce_by_key([dev(k)], [dev(v)], P, "sum"))
    want = orc.reduce_by_key([k], [v], P, "sum")
    for p in range(P):
        o1, o2 = np.argsort(got[p][0]), np.argsort(want[p][0])
        assert np.array_equal(got[p][0][o1].astype(np.int64), want[p][0][o2])
        assert got[p][1].dtype == np.float64
        assert np.allclose(got[p][1][o1], want[p][1][o2], rtol=0, atol=1e-9 * n / 2 ** 12)


@pytest.mark.parametrize("op", ["min", "max", "prod"])
def test_reduce_by_key_f64_ops(op):
    from dpark_b200 import shuffle
    rng = np.random.default_rng(24)
    n, P = 100000, 4
    k = rng.integers(0, 500, n, dtype=np.int64)
    v = rng.random(n) + 0.5 if op == "prod" else rng.standard_normal(n)
    if op == "prod":
        k = rng.integers(0, 20000, n, dtype=np.int64)
    got = _parts_from(shuffle.reduce_by_key([dev(k)], [dev(v)], P, op))
    want = orc.reduce_by_key([k], [v], P, op)
    for p in range(P):
        o1, o2 = np.argsort(got[p][0]), np.argsort(want[p][0])
        assert np.array_equal(got[p][0][o1], want[p][0][o2])
        if op == "prod":
            assert np.allclose(got[p][1][o1], want[p][1][o2], rtol=1e-12)
        else:
            assert np.array_equal(got[p][1][o1], want[p][1][o2])


def test_empty_and_unsupported():
    from dpark_b200 import shuffle
    e = torch.empty(0, dtype=torch.int64, device="cuda")
    res = shuffle.reduce_by_key([e], [e], 4, "sum")
    assert [int(k.numel()) for _, k, _ in res] == [0, 0, 0, 0]
    with pytest.raises(TypeError):
        nv().hash_keys(torch.zeros(4, dtype=torch.bool, device="cuda"))      # bool is unhashable in the reference too
    with pytest.raises(TypeError):
        nv().partition(torch.zeros(4, dtype=torch.int64, device="cuda"), None, 5000)
    with pytest.raises(nv().NativeError):
        nv().hash_keys(torch.zeros(4, dtype=torch.int64))                    # CPU tensor: no fallback
    with pytest.raises(TypeError):
        shuffle.reduce_by_key([torch.zeros(4, dtype=torch.int64, device="cuda")],
                              [torch.zeros(4, dtype=torch.float64, device="cuda")], 2, "xor")


def test_full_size_properties_1e8():
    """BASELINE config 2 size; checked through size-independent properties:
    conservation of rows and of the value checksum, every bucket holds only its
    own keys (GPU pid of the output == bucket id), stability (row-index payload
    ascending inside each bucket), and the reduce output: distinct count and
    checksum of sums equal to a sort-based recount in torch."""
    from dpark_b200 import shuffle
    n, P = 100_000_000, 8
    g = torch.Generator(device="cuda"); g.manual_seed(1234)
    k = torch.randint(0, 2 ** 31, (n,), dtype=torch.int64, device="cuda", generator=g)
    idx = torch.arange(n, dtype=torch.int64, device="cuda")
    ok, ov, off = nv().partition(k, idx, P)
    offh = off.cpu().tolist()
    assert offh[0] == 0 and offh[-1] == n
    assert int(ov.sum()) == n * (n - 1) // 2
    pid = nv().partition_ids(nv().hash_keys(ok), P)
    for p in range(P):
        seg = slice(offh[p], offh[p + 1])
        assert bool((pid[seg] == p).all())
        assert bool((ov[seg][1:] > ov[seg][:-1]).all())
        assert bool((k[ov[seg][:1000]] == ok[seg][:1000]).all())
    del ok, ov, pid, idx
    g.manual_seed(1235)
    v = torch.randint(0, 2 ** 16, (n,), dtype=torch.int64, device="cuda", generator=g)
    res = shuffle.reduce_by_key([k], [v], P, "sum")
    total = sum(int(x.numel()) for _, x, _ in res)
    uk = torch.unique(k)
    assert total == int(uk.numel())
    assert sum(int(x.sum()) for _, _, x in res) == int(v.sum())
    allk = torch.cat([x for _, x, _ in res])
    assert bool((torch.sort(allk).values == uk).all())


def _zipf_keys(n, support, s, seed):
    """Zipf(s) ranks by inverse CDF over a finite support, pushed through an odd-multiplier
    permutation so hot keys are not adjacent (SURVEY.md §8d, config C3 generator)."""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, support + 1, dtype=np.float64) ** s
    cdf = np.cumsum(w / w.sum())
    ranks = np.searchsorted(cdf, rng.random(n), side="left").astype(np.int64)
    return (ranks * 2654435761 + 12345) % (1 << 40)


def test_group_by_key_zipf_c3_shape_matches_oracle():
    """BASELINE config 3 shape scaled down: groupByKey over Zipf(1.1) int64 keys, 64 partitions,
    values = row index.  Per partition the same keys and, for every key, the SAME value list in
    (map split, position) order as the oracle's ordered-group merge."""
    from dpark_b200 import shuffle
    n, P, M = 1_000_000, 64, 8
    k = _zipf_keys(n, 200_000, 1.1, 2025)
    v = np.arange(n, dtype=np.int64)
    ks, vs = np.array_split(k, M), np.array_split(v, M)
    mo = shuffle.map_side([dev(x) for x in ks], [dev(x) for x in vs], P)
    rx = shuffle.exchange(mo)
    gk, gs, ng, ov, off = shuffle.group_side(rx, P)
    G = int(ng.item())
    gk, gs, ov, off = gk[:G].cpu().numpy(), gs[:G + 1].cpu().numpy(), ov.cpu().numpy(), off.cpu().numpy()
    want = orc.group_by_key(ks, vs, P)
    first = np.searchsorted(gs[:-1], off, side="left")
    hot = 0
    for p in range(P):
        wk, wo, wv = want[p]
        g0, g1 = first[p], first[p + 1]
        assert g1 - g0 == len(wk)
        pos = {int(key): g for g, key in zip(range(g0, g1), gk[g0:g1])}
        for i, key in enumerate(wk.tolist()):
            g = pos[key]
            assert np.array_equal(ov[gs[g]:gs[g + 1]], wv[wo[i]:wo[i + 1]])
            hot = max(hot, int(wo[i + 1] - wo[i]))
    assert hot > n // 20          # the skew is really there: the hottest key holds > 5 % of the rows


def test_reduce_by_key_zipf_hot_keys_all_impls_sum_exact(dpk_options):
    """Skewed reduceByKey (hot key = ~10 % of the rows): shared-memory and global atomics pile up
    on one accumulator; sums stay exact."""
    from dpark_b200 import shuffle
    n, P = 2_000_000, 8
    k = _zipf_keys(n, 100_000, 1.1, 7)
    v = np.random.default_rng(8).integers(-5, 6, n, dtype=np.int64)
    want = orc.reduce_by_key([k], [v], P, "sum")
    for impl in (2, 1):
        dpk_options({"reduce_impl": impl})
        got = _parts_from(shuffle.reduce_by_key([dev(k)], [dev(v)], P, "sum"))
        for p in range(P):
            o1, o2 = np.argsort(got[p][0]), np.argsort(want[p][0])
            assert np.array_equal(got[p][0][o1], want[p][0][o2])
            assert np.array_equal(got[p][1][o1], want[p][1][o2])
