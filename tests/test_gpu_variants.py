"""Oracle parity of every kernel variant dpk_set_option selects (include/dpark_b200.h: "results are the same for every
setting"), and of the reduce side fed what a multi-GPU exchange delivers, built on one GPU.  -m gpu."""
import itertools
import operator

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tests.shuffle_cases import MULTISPLIT_VARIANTS, REDUCE_VARIANTS, dpk_options, reduce_shape, variant_id  # noqa: F401

pytestmark = pytest.mark.gpu


def nv():
    from dpark_b200 import _native
    return _native


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits(a):
    """Keys as comparable integers: floats by their bits (the kernels and the oracle both spell -0.0 as 0.0)."""
    a = np.asarray(a)
    if a.dtype.kind == "f":
        return a.astype(np.float64).view(np.int64)
    return a.astype(np.int64)


def _check_part(gk, gv, wk, wv, op, tol=None):
    """One reduce partition against the oracle, after sorting both by key: keys exact; integer values and float
    min/max exact; float prod to rtol 1e-12; float sums to 1e-9 * sum|v| of the key (tol, aligned with wk)."""
    gb, wb = _bits(gk), _bits(wk)
    o1, o2 = np.argsort(gb, kind="stable"), np.argsort(wb, kind="stable")
    assert np.array_equal(gb[o1], wb[o2])
    gv, wv = gv[o1], wv[o2]
    if gv.dtype.kind != "f" or op in ("min", "max"):
        assert np.array_equal(gv.view(np.int64), wv.view(np.int64))
    elif op == "prod":
        assert np.allclose(gv, wv, rtol=1e-12, atol=0)
    else:
        assert np.all(np.abs(gv - wv) <= 1e-9 * tol[o2])


def _reduce_and_check(ks, vs, P, op, sub_bits=None):
    from dpark_b200 import shuffle
    res = shuffle.reduce_by_key([dev(x) for x in ks], [dev(x) for x in vs], P, op, sub_bits=sub_bits)
    want = _oracle_reduce(ks, vs, P, op)
    assert [p for p, _, _ in res] == list(range(P))
    for p, gk, gv in res:
        wk, wv, tol = want[p]
        _check_part(gk.cpu().numpy(), gv.cpu().numpy(), wk, wv, op, tol)


def _oracle_reduce(ks, vs, P, op):
    want = orc.reduce_by_key(ks, vs, P, op)
    if np.asarray(vs[0]).dtype.kind == "f" and op == "sum":
        tol = orc.reduce_by_key(ks, [np.abs(v.astype(np.float64)) for v in vs], P, "sum")
        return [(wk, wv, tv) for (wk, wv), (_, tv) in zip(want, tol)]
    return [(wk, wv, None) for wk, wv in want]


# ----------------------------------------------------------------------------- reduce side: variants x shapes
# (tests/test_gpu_subbuckets.py::test_every_reduce_implementation_gives_the_oracle_result runs every variant over every
# shape; tests/test_host_logic.py checks that each shape reaches the path it is named for)


def _pairwise_cases():
    """Variant x key kind x value kind x op (all seven ops for integer values, sum/min/max/prod for floats), every
    pair of the four factors covered at least once (greedy covering array, deterministic)."""
    kinds = ["i64", "i32", "f64", "f32"]
    combos = [(kk, vk, op) for kk in kinds for vk in kinds
              for op in (["sum", "min", "max", "prod", "and", "or", "xor"] if vk[0] == "i" else ["sum", "min", "max", "prod"])]
    nvar = len(REDUCE_VARIANTS)

    def pairs(c):
        var, kk, vk, op = c
        return {("v", var, "k", kk), ("v", var, "v", vk), ("v", var, "o", op), ("k", kk, "v", vk), ("k", kk, "o", op),
                ("vk", vk, "o", op)}
    todo = set().union(*(pairs((var,) + c) for var in range(nvar) for c in combos))
    cases = []
    while todo:
        best = max(((var,) + c for var in range(nvar) for c in combos), key=lambda c: len(pairs(c) & todo))
        cases.append(best)
        todo -= pairs(best)
    return cases


_NP = {"i64": np.int64, "i32": np.int32, "f64": np.float64, "f32": np.float32}


def _keys_of_kind(kind, n, rng):
    if kind in ("i64", "i32"):
        info = np.iinfo(_NP[kind])
        k = rng.integers(info.min, info.max, n, dtype=_NP[kind], endpoint=True)
        k[: n // 2] = rng.integers(-300, 300, n // 2)
        k[:4] = [info.min, info.max, -1, -2]
        return k
    pool = np.concatenate([rng.standard_normal(3000) * 10.0 ** rng.integers(-20, 20, 3000),
                           [0.0, -0.0, np.inf, -np.inf, 5e-324, 1.25, 1.75, 2.0 ** 61, 1.0, 1e-310]]).astype(_NP[kind])
    return pool[rng.integers(0, len(pool), n)]


def _vals_of_kind(kind, op, n, rng):
    if kind[0] == "i":
        if op == "prod":
            v = rng.integers(-3, 4, n)
        elif op in ("and", "or", "xor"):
            v = rng.integers(-2 ** 62, 2 ** 62, n) if kind == "i64" else rng.integers(-2 ** 31, 2 ** 31, n)
        else:
            v = rng.integers(-2 ** 31, 2 ** 31, n)
        return v.astype(_NP[kind])
    if op == "prod":
        return (rng.random(n) + 0.5).astype(_NP[kind])
    return (rng.standard_normal(n) * 1000.0).astype(_NP[kind])


PAIRWISE = _pairwise_cases()


@pytest.mark.parametrize("case", range(len(PAIRWISE)),
                         ids=["%s-%s-%s-%s" % ((variant_id(REDUCE_VARIANTS[c[0]]),) + c[1:]) for c in PAIRWISE])
def test_reduce_variants_over_key_value_kinds_and_ops(case, dpk_options):
    var, kk, vk, op = PAIRWISE[case]
    rng = np.random.default_rng(case)
    n, P = 60_000, 5
    k = _keys_of_kind(kk, n, rng)
    v = _vals_of_kind(vk, op, n, rng)
    dpk_options(REDUCE_VARIANTS[var])
    _reduce_and_check(np.array_split(k, 3), np.array_split(v, 3), P, op)


@pytest.mark.parametrize("P", [1000, 4095, 4096])
@pytest.mark.parametrize("kinds", [("i64", "i64"), ("i32", "f32")])
def test_reduce_by_key_with_many_partitions(P, kinds):
    """P >= 1000 buckets: with 8-byte columns the bulk multisplit's staging no longer fits and the map side falls back
    to the round-1 kernel (unordered for an even bucket count, stable for an odd one)."""
    rng = np.random.default_rng(P)
    n = 400_000
    k = _keys_of_kind(kinds[0], n, rng)
    v = _vals_of_kind(kinds[1], "sum", n, rng)
    _reduce_and_check(np.array_split(k, 2), np.array_split(v, 2), P, "sum")


@pytest.mark.parametrize("variant", REDUCE_VARIANTS, ids=variant_id)
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_float_sum_of_only_negative_zeros_is_negative_zero(variant, dtype, dpk_options):
    """A key whose only values are -0.0 sums to -0.0 (Python: -0.0 + -0.0 == -0.0) on every path, also the ones that
    start an accumulator at the operation's identity, and the INT64_MIN key (the slot tables' free marker).  The other
    keys' values are small integers, so every sum is exact and is compared bit for bit too."""
    rng = np.random.default_rng(5)
    n, P = 6000, 4
    k = rng.integers(0, 300, n, dtype=np.int64)
    k[::11] = -2 ** 63
    v = rng.integers(-8, 9, n).astype(dtype)
    only_neg_zero = (k < 60) | (k == -2 ** 63)
    v[only_neg_zero] = -0.0
    v[(k == 70) | (k == 71)] = 0.0                     # +0.0 only and ...
    v[(k == 71) & (np.arange(n) % 2 == 0)] = -0.0      # ... mixed zeros: +0.0
    ks, vs = np.array_split(k, 2), np.array_split(v, 2)
    want = orc.py_reduce_by_key([list(zip(a.tolist(), (float(x) for x in b))) for a, b in zip(ks, vs)], P, operator.add)
    dpk_options(variant)
    from dpark_b200 import shuffle
    res = shuffle.reduce_by_key([dev(x) for x in ks], [dev(x) for x in vs], P, "sum")
    for p, gk, gv in res:
        gk, gv = gk.cpu().numpy(), gv.cpu().numpy()
        wk = np.array(sorted(want[p]), dtype=np.int64)
        wv = np.array([want[p][x] for x in wk.tolist()], dtype=np.float64)
        o = np.argsort(gk)
        assert np.array_equal(gk[o], wk)
        assert np.array_equal(gv[o].view(np.int64), wv.view(np.int64)), variant_id(variant)


def test_look_back_runs_agree_on_offsets_counts_and_rows(dpk_options):
    """agg_cursor 0 (chained scan with decoupled look-back) fixes where every fine bucket's rows start, but the rows
    reach a fine bucket through unordered multisplits, so which row claims a key -- and with it the order inside the
    bucket -- changes from run to run (DESIGN.md section 7).  What two runs share: the partition offsets, the counts
    and the set of (key, value) rows of every partition."""
    from dpark_b200 import shuffle
    [(k, v)], P, sb = reduce_shape("hot_keys")
    dpk_options({"agg_cursor": 0})
    rx = shuffle.exchange(shuffle.map_side([dev(k)], [dev(v)], P, None, False, sb, unordered=True))
    runs = [[t.cpu().numpy() for t in shuffle.reduce_side(rx, "sum", P)] for _ in range(2)]
    (k1, v1, po1, c1), (k2, v2, po2, c2) = runs
    assert np.array_equal(po1, po2) and np.array_equal(c1, c2)
    for j in range(P):
        a, c = po1[j], c1[j]
        o1, o2 = np.argsort(k1[a:a + c]), np.argsort(k2[a:a + c])
        assert np.array_equal(k1[a:a + c][o1], k2[a:a + c][o2]) and np.array_equal(v1[a:a + c][o1], v2[a:a + c][o2])


# ----------------------------------------------------------------------------- map side: multisplit variants
EDGE_N = [0, 1, 4095, 4096, 4097, 8191, 8192, 8193]
WIDTHS = [(np.int64, None), (np.int64, np.int32), (np.int64, np.float64), (np.int32, None), (np.int32, np.float32),
          (np.int32, np.int64)]


def _expect_partition(k, v, P):
    pid = orc.partition_vec(orc.hash_vec(k), P)
    order = np.argsort(pid, kind="stable")
    off = np.zeros(P + 1, dtype=np.int64)
    off[1:] = np.cumsum(np.bincount(pid, minlength=P))
    return k[order], None if v is None else v[order], off


def _check_multisplit(ok, ov, off, k, v, P, unordered):
    """Stable: bit-identical to the stable argsort by oracle bucket id.  Unordered: the same offsets and, per bucket,
    the same multiset of (key, value) rows."""
    wk, wv, woff = _expect_partition(k, v, P)
    ok = ok.cpu().numpy()
    ov = None if ov is None else ov.cpu().numpy()
    assert np.array_equal(off.cpu().numpy(), woff)
    if unordered:
        bucket = np.repeat(np.arange(P), np.diff(woff))
        cols = [_bits(ok)] if ov is None else [ov.view(np.int64 if ov.itemsize == 8 else np.int32), _bits(ok)]
        wcols = [_bits(wk)] if wv is None else [wv.view(np.int64 if wv.itemsize == 8 else np.int32), _bits(wk)]
        o1, o2 = np.lexsort(cols + [bucket]), np.lexsort(wcols + [bucket])
        ok, wk = ok[o1], wk[o2]
        if ov is not None:
            ov, wv = ov[o1], wv[o2]
    assert np.array_equal(ok.view(np.uint8), wk.view(np.uint8))
    if v is not None:
        assert np.array_equal(ov.view(np.uint8), wv.view(np.uint8))


def _columns(kdt, vdt, n, rng):
    info = np.iinfo(kdt)
    k = rng.integers(info.min, info.max, n, dtype=kdt, endpoint=True)
    k[: n // 3] = rng.integers(-1000, 1000, n // 3)
    v = None if vdt is None else (np.arange(n) * 3 + 1).astype(vdt)
    return k, v


@pytest.mark.parametrize("variant", MULTISPLIT_VARIANTS, ids=variant_id)
@pytest.mark.parametrize("unordered", [False, True], ids=["stable", "unordered"])
@pytest.mark.parametrize("P", [1, 3, 64, 511, 512, 1000, 4095, 4096])
def test_multisplit_variants(variant, unordered, P, dpk_options):
    """nv.partition over 4- and 8-byte keys, values of 0, 4 and 8 bytes, n at the tile edges (4096- and 8192-row
    tiles) and one large n, for every multisplit variant and bucket count (odd counts, the scatter_wide_from step at
    512, bulk staging that no longer fits from ~1000 buckets); the large n also through the multi-chunk
    partition_count / partition_scatter pair."""
    from dpark_b200 import shuffle
    dpk_options(variant)
    rng = np.random.default_rng(P * 2 + unordered)
    for n, (kdt, vdt) in itertools.product(EDGE_N, WIDTHS):
        k, v = _columns(kdt, vdt, n, rng)
        ok, ov, off = nv().partition(dev(k), None if v is None else dev(v), P, unordered=unordered)
        _check_multisplit(ok, ov, off, k, v, P, unordered)
    kdt, vdt = WIDTHS[P % len(WIDTHS)]
    n = 300_001
    k, v = _columns(kdt, vdt, n, rng)
    ok, ov, off = nv().partition(dev(k), None if v is None else dev(v), P, unordered=unordered)
    _check_multisplit(ok, ov, off, k, v, P, unordered)
    cut = 100_000                      # two separate allocations: one count + scatter launch pair per chunk
    mo = shuffle.map_side([dev(k[:cut]), dev(k[cut:])], [None, None] if v is None else [dev(v[:cut]), dev(v[cut:])],
                          P, unordered=unordered)
    _check_multisplit(mo.keys, mo.vals, mo.offsets, k, v, P, unordered)


# ----------------------------------------------------------------------------- exchange-shaped reduce input
def _sources(G, n_per, P, rng, one_key=False):
    """Map splits of G sources: source 0 holds a handful of rows (most of its (source, bucket) segments are empty),
    source 1 none at all.  Values: global row numbers in (source, split, position) order."""
    splits, at = [], 0
    for s in range(G):
        m = 7 if s == 0 else (0 if s == 1 else n_per)
        k = rng.integers(-4000, 4000, m, dtype=np.int64) if not one_key else np.full(m, 4242, dtype=np.int64)
        if not one_key:
            k[: m // 4] = rng.integers(-2 ** 63, 2 ** 63 - 1, m // 4, dtype=np.int64, endpoint=True)
        cut = m // 3
        splits.append([(k[:cut], np.arange(at, at + cut, dtype=np.int64)),
                       (k[cut:], np.arange(at + cut, at + m, dtype=np.int64))])
        at += m
    return splits


def _received(splits, P, G, r, sb, unordered, extra=None):
    """What the exchange delivers to rank r of G: its block of partitions (shuffle.owner_blocks) cut out of every
    source's bucket-major map output, concatenated source-major; seg[s][b] = rows of local fine bucket b from source
    s.  extra: rows appended behind the described ones (a receive buffer larger than what it holds)."""
    from dpark_b200 import shuffle
    blocks = shuffle.owner_blocks(P, G)
    b0, b1 = blocks[r] << sb, blocks[r + 1] << sb
    ks, vs, seg = [], [], []
    for src in splits:
        mo = shuffle.map_side([dev(k) for k, _ in src], [dev(v) for _, v in src], P, None, False, sb,
                              unordered=unordered)
        off = mo.offsets.cpu().numpy()
        ks.append(mo.keys[off[b0]:off[b1]])
        vs.append(mo.vals[off[b0]:off[b1]])
        seg.append(np.diff(off)[b0:b1])
    bound = extra is not None
    if bound:
        ks.append(dev(extra[0]))
        vs.append(dev(extra[1]))
    return shuffle.Received(torch.cat(ks), torch.cat(vs), dev(np.array(seg, dtype=np.int64).reshape(G, b1 - b0)),
                            blocks[r], blocks[r + 1] - blocks[r], sb, bound=bound)


def _unreceived_rows(splits, P, G, r, count=16):
    """Up to `count` rows with distinct keys of rank r's own partitions that appear nowhere in the data."""
    from dpark_b200 import shuffle
    blocks = shuffle.owner_blocks(P, G)
    cand = np.arange(10 ** 15, 10 ** 15 + 4000, dtype=np.int64)
    pid = orc.partition_vec(orc.hash_vec(cand), P)
    k = cand[(pid >= blocks[r]) & (pid < blocks[r + 1])][:count]
    return k, np.full(len(k), 10 ** 9, dtype=np.int64)


EXCHANGE_REDUCE_VARIANTS = [{"reduce_impl": 0}, {"reduce_impl": 1}, {}, {"agg_pipe": 1}]


def _owning_ranks(P, G):
    from dpark_b200 import shuffle
    blocks = shuffle.owner_blocks(P, G)
    return [r for r in range(G) if blocks[r + 1] > blocks[r]]


def _check_reduce_ranks(splits, P, G, sb, bound):
    from dpark_b200 import shuffle
    want = orc.reduce_by_key([k for src in splits for k, _ in src], [v for src in splits for _, v in src], P)
    for r in _owning_ranks(P, G):
        extra = _unreceived_rows(splits, P, G, r) if bound else None
        rx = _received(splits, P, G, r, sb, True, extra)
        ok, ov, po, cnt = (t.cpu().numpy() for t in shuffle.reduce_side(rx, "sum", P))
        assert (cnt >= 0).all()
        for j in range(rx.nparts):
            wk, wv = want[rx.part_first + j]
            _check_part(ok[po[j]:po[j] + cnt[j]], ov[po[j]:po[j] + cnt[j]], wk, wv, "sum")


@pytest.mark.parametrize("variant", EXCHANGE_REDUCE_VARIANTS, ids=variant_id)
@pytest.mark.parametrize("G", [2, 3, 8])
def test_reduce_side_on_exchange_shaped_input(G, variant, dpk_options):
    """nv.combine over rows from G sources (nsrc = G, source-major, bucket-major inside each), for every rank's block
    of partitions (part_first > 0; with P = 10 and G = 8 the last ranks own none), against the oracle over all map
    splits in source order."""
    dpk_options(variant)
    splits = _sources(G, 40_000, 10, np.random.default_rng(G))
    _check_reduce_ranks(splits, 10, G, 2, bound=False)


@pytest.mark.parametrize("variant", EXCHANGE_REDUCE_VARIANTS, ids=variant_id)
@pytest.mark.parametrize("G", [2, 3, 8])
def test_reduce_side_reads_only_the_received_rows_of_a_bound_buffer(G, variant, dpk_options):
    """A receive buffer longer than the rows it holds (Received.bound, the peer exchange): up to 16 rows behind the
    described ones carry keys of this rank's partitions that were never sent, and must not be merged."""
    dpk_options(variant)
    splits = _sources(G, 20_000, 10, np.random.default_rng(100 + G))
    _check_reduce_ranks(splits, 10, G, 2, bound=True)


def _check_group_ranks(splits, P, G, sb, bound):
    from dpark_b200 import shuffle
    want = orc.group_by_key([k for src in splits for k, _ in src], [v for src in splits for _, v in src], P)
    for r in _owning_ranks(P, G):
        extra = _unreceived_rows(splits, P, G, r) if bound else None
        rx = _received(splits, P, G, r, sb, False, extra)
        gk, gs, ng, ov, off = shuffle.group_side(rx, P)
        _check_groups(gk, gs, ng, ov, off, [want[rx.part_first + j] for j in range(rx.nparts)])


def _check_groups(gk, gs, ng, ov, off, want):
    """CSR result of group_side against the oracle's per partition: the same keys and, per key, the same values in
    (source, position) order."""
    G = int(ng.item())
    gk, gs, ov, off = gk[:G].cpu().numpy(), gs[:G + 1].cpu().numpy(), ov.cpu().numpy(), off.cpu().numpy()
    first = np.searchsorted(gs[:-1], off, side="left")
    assert len(off) == len(want) + 1
    for j, (wk, wo, wv) in enumerate(want):
        g0, g1 = first[j], first[j + 1]
        assert g1 - g0 == len(wk)
        pos = {int(key): g for g, key in zip(range(g0, g1), gk[g0:g1])}
        for i, key in enumerate(_bits(wk).tolist()):
            g = pos[key]
            assert np.array_equal(ov[gs[g]:gs[g + 1]], wv[wo[i]:wo[i + 1]])


@pytest.mark.parametrize("G", [2, 3, 8])
@pytest.mark.parametrize("bound", [False, True], ids=["exact", "bound"])
def test_group_side_on_exchange_shaped_input(G, bound):
    """shuffle.group_side over rows from G sources against orc.group_by_key: the same values per key, in (source,
    position) order, also when the receive buffer is longer than the rows it holds."""
    splits = _sources(G, 30_000, 10, np.random.default_rng(200 + G))
    _check_group_ranks(splits, 10, G, 2, bound)


def test_group_side_one_key_from_several_sources():
    """Every row has the same key (no radix digit differs): group_side still has to make the rows of several sources
    bucket-major, in source order (the 1-bit pass)."""
    splits = _sources(3, 5000, 4, np.random.default_rng(9), one_key=True)
    _check_group_ranks(splits, 4, 3, 1, False)


# ----------------------------------------------------------------------------- groupByKey keys
@pytest.mark.parametrize("kind", ["full_range", "above_bit_56", "float64"])
def test_group_side_key_bit_ranges(kind):
    """groupByKey over keys whose differing bits reach every radix digit: full-range int64 (INT64_MIN, INT64_MAX, -1,
    -2), keys that differ only above bit 56, and float keys (sorted by their canonical bits)."""
    from dpark_b200 import shuffle
    rng = np.random.default_rng(3)
    n, P, M = 300_000, 16, 3
    if kind == "full_range":
        pool = rng.integers(-2 ** 63, 2 ** 63 - 1, 20_000, dtype=np.int64, endpoint=True)
        pool[:4] = [-2 ** 63, 2 ** 63 - 1, -1, -2]
        k = pool[rng.integers(0, len(pool), n)]
    elif kind == "above_bit_56":
        k = (rng.integers(-128, 128, n, dtype=np.int64) << 56) | 12345
    else:
        pool = np.concatenate([rng.standard_normal(20_000) * 10.0 ** rng.integers(-300, 300, 20_000),
                               [0.0, np.inf, -np.inf, 5e-324, -5e-324, 1.25, 1.75, 2.0 ** 61, 1.0]]) + 0.0
        k = pool[rng.integers(0, len(pool), n)]
    v = np.arange(n, dtype=np.int64)
    ks, vs = np.array_split(k, M), np.array_split(v, M)
    rx = shuffle.exchange(shuffle.map_side([dev(x) for x in ks], [dev(x) for x in vs], P))
    gk, gs, ng, ov, off = shuffle.group_side(rx, P)
    _check_groups(gk, gs, ng, ov, off, orc.group_by_key(ks, vs, P))


@pytest.mark.parametrize("shift,bits", [(0, 8), (8, 8), (56, 8), (60, 4), (13, 1), (0, 10)])
def test_radix_pass_seg_is_a_stable_split_inside_every_bucket(shift, bits):
    """dpk_radix_pass_seg over source-major input (nsrc = 3, empty segments included): the output is bucket-major and
    every bucket is its rows in (source, position) order, stably split by the digit."""
    rng = np.random.default_rng(shift * 16 + bits)
    nsrc, F = 3, 7
    seg = rng.integers(0, 3000, (nsrc, F)).astype(np.int64)
    seg[1, 2] = seg[0, 5] = seg[2, 0] = 0
    seg[:, 4] = 0
    n = int(seg.sum())
    k = rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64, endpoint=True)
    v = np.arange(n, dtype=np.int64)
    gk, gv = nv().radix_pass_seg(dev(k), dev(v), shift, bits, dev(seg))
    start = np.concatenate([[0], np.cumsum(seg.ravel())[:-1]]).reshape(nsrc, F)
    want = []
    for b in range(F):
        rows = np.concatenate([np.arange(start[s, b], start[s, b] + seg[s, b]) for s in range(nsrc)]).astype(np.int64)
        digit = (k[rows].view(np.uint64) >> np.uint64(shift)) & np.uint64((1 << bits) - 1)
        want.append(rows[np.argsort(digit, kind="stable")])
    want = np.concatenate(want)
    assert np.array_equal(gv.cpu().numpy(), want) and np.array_equal(gk.cpu().numpy(), k[want])
