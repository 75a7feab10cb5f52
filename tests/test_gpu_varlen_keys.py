"""Oracle parity of the variable-length key path (str, bytes, tuple and None keys): dict_encode under forced hash
collisions, representative row ids (DPK_K_ROWID) in every multisplit and merge variant, the operator surface at scale
against Python dicts, tuple and byte hashes on the device, and the overflow check of the string reduce side.  -m gpu.

Byte-key columns are built from int64 keys by a bijective spelling (the 8 little-endian bytes, or the decimal form), so
the expected results are computed on the ints."""
import bisect
import functools
import math
import operator
import sys

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tests.shuffle_cases import MULTISPLIT_VARIANTS, REDUCE_VARIANTS, dpk_options, reduce_shape, variant_id  # noqa: F401
from tests.test_gpu_variants import _check_part, _vals_of_kind

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1


def nv():
    from dpark_b200 import _native
    return _native


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _le_bytes(k):
    """int64 keys as 8-byte little-endian byte keys: (data, offsets)."""
    k = np.ascontiguousarray(k, dtype=np.int64)
    return k.view(np.uint8), np.arange(len(k) + 1, dtype=np.int64) * 8


def _decimal(k):
    """int64 keys spelled in decimal: variable-length byte keys (data, offsets)."""
    s = np.ascontiguousarray(k, dtype=np.int64).astype("S20")
    mat = s.view(np.uint8).reshape(len(k), 20)
    lens = (mat != 0).sum(1)
    data = mat[np.arange(20)[None, :] < lens[:, None]]
    offs = np.zeros(len(k) + 1, dtype=np.int64)
    np.cumsum(lens, out=offs[1:])
    return data, offs


def _columns(blobs):
    offs = np.zeros(len(blobs) + 1, dtype=np.int64)
    np.cumsum([len(b) for b in blobs], out=offs[1:])
    return np.frombuffer(b"".join(blobs) or b"\0", dtype=np.uint8), offs


def _first_ids(k):
    """Representative row id of every row (the first occurrence of its key), the key index of every row and the row
    id of every key."""
    _, first, inv = np.unique(k, return_index=True, return_inverse=True)
    return first[inv].astype(np.int64), inv.astype(np.int64), first.astype(np.int64)


# ----------------------------------------------------------------------------- 1. dict_encode
def _check_rep(rep, group):
    """rep from dict_encode against `group` (group[i] == group[j] <=> rows i and j hold the same bytes)."""
    n = len(group)
    assert rep.shape == (n,)
    assert ((rep >= 0) & (rep < n)).all()
    assert np.array_equal(group[rep], group)                  # a representative holds the bytes of its rows
    assert np.array_equal(rep[rep], rep)                      # and represents itself
    assert len(np.unique(rep)) == len(np.unique(group))       # one representative per distinct key


def _group_of(blobs):
    ids = {}
    return np.array([ids.setdefault(b, len(ids)) for b in blobs], dtype=np.int64)


def _encode(data, offs, h):
    return nv().dict_encode(dev(data), dev(offs), dev(np.asarray(h, dtype=np.int64))).cpu().numpy()


def _random_blobs(n, rng):
    pool = [bytes(rng.integers(0, 256, rng.integers(0, 25), dtype=np.uint8)) for _ in range(max(1, n // 3))]
    return [pool[i] for i in rng.integers(0, len(pool), n)]


@pytest.mark.parametrize("n", [1, 2, 511, 512, 513, 1023, 1024, 1025, 100_003])
def test_dict_encode_with_real_hashes_at_table_size_edges(n):
    """The table has 1024 slots and doubles at 2n: sizes on both sides of every edge, random bytes (high bytes and the
    empty key included), about three rows per key."""
    blobs = _random_blobs(n, np.random.default_rng(n))
    data, offs = _columns(blobs)
    _check_rep(_encode(data, offs, orc.hash_bytes_vec(data, offs, 0)), _group_of(blobs))


def test_dict_encode_zipf_words():
    """2e6 Zipf-distributed decimal words, hashed on the device as str keys (the word-count shape)."""
    rng = np.random.default_rng(1)
    w = np.minimum(rng.zipf(1.2, 2_000_000), 10 ** 12).astype(np.int64)
    data, offs = _decimal(w)
    h = nv().hash_bytes(dev(data), dev(offs), nv().STR_UTF8)
    rep = nv().dict_encode(dev(data), dev(offs), h).cpu().numpy()
    _check_rep(rep, np.unique(w, return_inverse=True)[1])


@pytest.mark.parametrize("const", [0, -1, I64_MIN, I64_MAX])
def test_dict_encode_one_hash_for_every_row(const):
    """The hash is the caller's column: with one value for every row the probe chain holds every distinct key, so only
    the byte compare tells the 20 000 keys apart."""
    rng = np.random.default_rng(2)
    k = rng.integers(0, 20_000, 60_000)
    k[:20_000] = np.arange(20_000)
    data, offs = _decimal(k * 7919 - 10 ** 6)
    _check_rep(_encode(data, offs, np.full(len(k), const)), k)


def test_dict_encode_hash_with_four_bits():
    rng = np.random.default_rng(3)
    k = rng.integers(I64_MIN, I64_MAX, 100_000, dtype=np.int64, endpoint=True)
    k[50_000:] = k[rng.integers(0, 50_000, 50_000)]
    data, offs = _le_bytes(k)
    _check_rep(_encode(data, offs, orc.hash_bytes_vec(data, offs, 0) & 0xF), np.unique(k, return_inverse=True)[1])


def _near_pairs(L, rng):
    base = bytes(rng.integers(0, 256, L, dtype=np.uint8))
    last = base[:-1] + bytes([base[-1] ^ 1])
    first = bytes([base[0] ^ 0x80]) + base[1:]
    return [base, last, first, base[:-1]]


@pytest.mark.parametrize("hash_kind", ["one_hash", "real"])
@pytest.mark.parametrize("L", [1, 4095, 4096, 4097, 65536])
def test_dict_encode_keys_that_differ_in_one_byte(L, hash_kind):
    """Keys built to differ as little as possible: the same length differing only in the last or only in the first
    byte, a key and its prefix, b"" and b"\\0" -- each several times, interleaved."""
    rng = np.random.default_rng(L)
    blobs = (_near_pairs(L, rng) + [b"", b"\0"]) * 5
    blobs = [blobs[i] for i in rng.permutation(len(blobs))]
    data, offs = _columns(blobs)
    h = np.full(len(blobs), 12345) if hash_kind == "one_hash" else orc.hash_bytes_vec(data, offs, 0)
    _check_rep(_encode(data, offs, h), _group_of(blobs))


def test_dict_encode_degenerate_inputs():
    n = 1_000_000
    data, offs = _columns([b"the same key"] * n)
    rep = _encode(data, offs, orc.hash_bytes_vec(data, offs, 0))
    assert (rep == rep[0]).all() and 0 <= rep[0] < n
    data, offs = _columns([b""] * 5000)                      # the data buffer is the 1-byte dummy
    assert data.size == 1
    rep = _encode(data, offs, orc.hash_bytes_vec(data, offs, 0))
    assert (rep == rep[0]).all()
    rng = np.random.default_rng(4)
    blobs = [b"" if x else b for x, b in zip(rng.random(30_000) < 0.3, _random_blobs(30_000, rng))]
    data, offs = _columns(blobs)
    for h in (orc.hash_bytes_vec(data, offs, 0), np.zeros(len(blobs), dtype=np.int64)):
        _check_rep(_encode(data, offs, h), _group_of(blobs))


# ----------------------------------------------------------------------------- 2. row-id keys in the multisplit
SPLIT_N = [1, 4097, 8193, 100_003]
SPLIT_SHAPES = [(1, 0), (1, 3), (3, 0), (3, 3), (64, 0), (64, 3), (512, 0), (512, 3), (4095, 0)]


@functools.lru_cache(maxsize=None)
def _split_input(n):
    """(representative ids, real hash column of the decimal byte keys) of n rows, about three rows per key."""
    rng = np.random.default_rng(n)
    k = rng.integers(0, max(1, n // 3), n, dtype=np.int64)
    k[::5] = rng.integers(I64_MIN, I64_MAX, len(k[::5]), dtype=np.int64, endpoint=True)
    data, offs = _decimal(k)
    return _first_ids(k)[0], orc.hash_bytes_vec(data, offs, 0)


def _check_row_id_split(ok, ov, off, rep, aux, vals, P, thr, sb, unordered):
    """Stable: bit for bit what the prehashed path (pinned to the oracle) gives for the hash of each row's key.
    Unordered: the same offsets and per bucket the same rows.  Both: partition sizes from the oracle."""
    wk, wv, woff = nv().partition(dev(aux[rep]), dev(vals), P, thr, prehashed=True, sub_bits=sb)
    ok, ov, off = ok.cpu().numpy(), ov.cpu().numpy(), off.cpu().numpy()
    wv, woff = wv.cpu().numpy(), woff.cpu().numpy()
    assert np.array_equal(off, woff)
    pid = orc.partition_vec(aux[rep], P, thr)
    assert np.array_equal(np.diff(off[::1 << sb]), np.bincount(pid, minlength=P))
    if unordered:
        bucket = np.repeat(np.arange(len(off) - 1), np.diff(off))
        o1, o2 = np.lexsort((ov, bucket)), np.lexsort((wv, bucket))
        ok, ov, wv = ok[o1], ov[o1], wv[o2]
    assert np.array_equal(ov, wv)
    assert np.array_equal(ok, rep[ov])


def _row_id_split_cases(P, thr, sb, unordered, sizes):
    from dpark_b200 import shuffle
    for n in sizes:
        rep, real = _split_input(n)
        vals = np.arange(n, dtype=np.int64)
        for aux in (real, (real & 0xF) - 8):                 # real hashes, then 16 hash values for all keys
            d_aux = dev(aux)
            ok, ov, off = nv().partition(dev(rep), dev(vals), P, thr, sub_bits=sb, row_hash=d_aux, unordered=unordered)
            _check_row_id_split(ok, ov, off, rep, aux, vals, P, thr, sb, unordered)
            if n > 10_000:                                   # two allocations: one count + scatter pair per chunk
                cut = n // 3
                mo = shuffle.map_side([dev(rep[:cut]), dev(rep[cut:])], [dev(vals[:cut]), dev(vals[cut:])], P, thr,
                                      False, sb, row_hash=d_aux, unordered=unordered)
                _check_row_id_split(mo.keys, mo.vals, mo.offsets, rep, aux, vals, P, thr, sb, unordered)


@pytest.mark.parametrize("P,sb", SPLIT_SHAPES, ids=["P%d-sb%d" % s for s in SPLIT_SHAPES])
@pytest.mark.parametrize("unordered", [False, True], ids=["stable", "unordered"])
@pytest.mark.parametrize("variant", MULTISPLIT_VARIANTS, ids=variant_id)
def test_row_id_multisplit_variants(variant, unordered, P, sb, dpk_options):
    """nv.partition / map_side with representative row ids whose hash is looked up in row_hash (the strings.py map
    side), for every multisplit variant, at tile-edge and large sizes."""
    dpk_options(variant)
    _row_id_split_cases(P, None, sb, unordered, SPLIT_N)


@pytest.mark.parametrize("sb", [0, 3])
@pytest.mark.parametrize("unordered", [False, True], ids=["stable", "unordered"])
@pytest.mark.parametrize("variant", MULTISPLIT_VARIANTS, ids=variant_id)
def test_row_id_multisplit_with_thresholds(variant, unordered, sb, dpk_options):
    """HashPartitioner thresholds (bisect over the hash) with row-id keys; some thresholds sit among the 16 colliding
    hash values."""
    dpk_options(variant)
    rep, real = _split_input(100_003)
    thr = np.sort(np.concatenate([real[::10_000], [-5, 0, 3]])).astype(np.int64)
    _row_id_split_cases(len(thr) + 1, thr, sb, unordered, [100_003])


# ----------------------------------------------------------------------------- 3. row-id keys in the merge
MERGE_SHAPES = ["distinct", "hot_keys", "distinct_overflow", "tiny", "collide", "one_hash"]
VALUE_OPS = [("i64", op) for op in ("sum", "min", "max", "prod", "and", "or", "xor")] + \
            [("f64", op) for op in ("sum", "min", "max", "prod")]
_UFUNC = {"sum": np.add, "min": np.minimum, "max": np.maximum, "prod": np.multiply, "and": np.bitwise_and,
          "or": np.bitwise_or, "xor": np.bitwise_xor}


@functools.lru_cache(maxsize=None)
def _merge_shape(name):
    """[(rep, key index per row, row id per key, hash column)], P, sub_bits of the shape (None: choose_sub_bits).
    The reduce-side shapes of tests/shuffle_cases.py become byte keys (hot_keys and distinct_overflow their 8 bytes,
    the others their decimal form) hashed as bytes; `collide` and `one_hash` inject the hash column."""
    if name in ("collide", "one_hash"):
        rng = np.random.default_rng(11)
        nd, n, P = (100_000, 300_000, 8) if name == "collide" else (50_000, 400_000, 4)
        k = np.concatenate([np.arange(nd), rng.integers(0, nd, n - nd)])
        rng.shuffle(k)
        rep, inv, first = _first_ids(k)
        if name == "collide":                                # 16 hash values over 100 000 keys
            hv = rng.integers(I64_MIN, I64_MAX, 16, dtype=np.int64, endpoint=True)
            hv[:3] = [I64_MIN, -1, 0]
            h = hv[k % 16]
        else:                                                # one hash value: every row in one fine bucket
            h = np.full(n, 0x5DEECE66D, dtype=np.int64)
        return [(rep, inv, first, h)], P, None
    inputs, P, sb = reduce_shape(name)
    runs = []
    for k, _ in inputs:
        if len(k) == 0:                                      # strings.py returns before the shuffle when n == 0
            continue
        data, offs = _le_bytes(k) if name in ("hot_keys", "distinct_overflow") else _decimal(k)
        runs.append(_first_ids(k) + (orc.hash_bytes_vec(data, offs, 0),))
    return runs, P, sb


def _expected_merge(inv, first, h, v, P, op, thr=None):
    """Per partition: (row ids, combined values, sum |v| per key): numpy ufuncs per key, float sums by math.fsum (a
    key of one or two rows: the float64 sum, which is correctly rounded too)."""
    order = np.argsort(inv, kind="stable")
    cnt = np.bincount(inv, minlength=len(first))
    starts = np.zeros(len(first), dtype=np.int64)
    np.cumsum(cnt[:-1], out=starts[1:])
    sv = v[order]
    out = _UFUNC[op].reduceat(sv, starts)
    tol = None
    if v.dtype.kind == "f" and op == "sum":
        for j in np.nonzero(cnt > 2)[0].tolist():
            out[j] = math.fsum(sv[starts[j]:starts[j] + cnt[j]].tolist())
        tol = np.add.reduceat(np.abs(sv), starts)
    pid = orc.partition_vec(h[first], P, thr)
    return [(first[pid == p], out[pid == p], None if tol is None else tol[pid == p]) for p in range(P)]


def _merge_row_ids(rep, vals, h, P, sb, op, thr=None):
    """The strings.py reduce side: map_side over the ids, exchange, combine with row_hash."""
    from dpark_b200 import shuffle
    d_h = dev(h)
    mo = shuffle.map_side([dev(rep)], [dev(vals)], P, thr, False, sb, row_hash=d_h, unordered=True)
    rx = shuffle.exchange(mo)
    return nv().combine(rx.keys, rx.vals, op, P, rx.seg.contiguous(), rx.part_first, rx.nparts, thr, sb, row_hash=d_h)


@pytest.mark.parametrize("shape", MERGE_SHAPES)
@pytest.mark.parametrize("variant", REDUCE_VARIANTS, ids=variant_id)
def test_row_id_merge_variants(variant, shape, dpk_options):
    """Every reduce variant over every shape, with sub_bits as choose_sub_bits picks it and 0 (distinct_overflow: 0
    only, which is what sends it to the hash-disjoint passes).  The value kind and op rotate so that every shape and
    every variant meets all eleven (i64: seven ops, f64: sum/min/max/prod)."""
    from dpark_b200 import shuffle
    vi, si = REDUCE_VARIANTS.index(variant), MERGE_SHAPES.index(shape)
    dpk_options(variant)
    runs, P, _ = _merge_shape(shape)
    j = 0
    for rep, inv, first, h in runs:
        n = len(rep)
        for sb in sorted({shuffle.choose_sub_bits(n, P), 0}) if shape != "distinct_overflow" else [0]:
            vk, op = VALUE_OPS[(2 * vi + j + 3 * si) % len(VALUE_OPS)]
            v = _vals_of_kind(vk, op, n, np.random.default_rng(100 * vi + 10 * si + j))
            j += 1
            ok, ov, off, cnt = (t.cpu().numpy() for t in _merge_row_ids(rep, v, h, P, sb, op))
            assert (cnt >= 0).all(), (sb, vk, op)
            for p, (wk, wv, tol) in enumerate(_expected_merge(inv, first, h, v, P, op)):
                _check_part(ok[off[p]:off[p] + cnt[p]], ov[off[p]:off[p] + cnt[p]], wk, wv, op, tol)


@pytest.mark.parametrize("variant", REDUCE_VARIANTS, ids=variant_id)
def test_row_id_merge_on_exchange_shaped_input(variant, dpk_options):
    """nv.combine with row_hash over what a 3-rank exchange delivers to ranks 1 and 2 (part_first > 0, source-major,
    one source with 7 rows and one with none), in a receive buffer longer than the rows it holds: the 16 rows behind
    the described ones carry VALID ids of this rank's own keys with a marker value, so a merge that reads past the
    described rows gives a wrong sum instead of an out-of-bounds read."""
    from dpark_b200 import shuffle
    dpk_options(variant)
    rng = np.random.default_rng(31)
    G, P, sb, sizes = 3, 10, 2, [7, 0, 30_000]
    k = rng.integers(-3000, 3000, sum(sizes), dtype=np.int64)
    k[::4] = rng.integers(I64_MIN, I64_MAX, len(k[::4]), dtype=np.int64, endpoint=True)
    v = rng.integers(-1000, 1000, len(k), dtype=np.int64)
    rep, inv, first = _first_ids(k)
    h = orc.hash_bytes_vec(*_decimal(k), 0)
    d_h = dev(h)
    want = _expected_merge(inv, first, h, v, P, "sum")
    at = np.concatenate([[0], np.cumsum(sizes)])
    blocks = shuffle.owner_blocks(P, G)
    for r in (1, 2):
        b0, b1 = blocks[r] << sb, blocks[r + 1] << sb
        ks, vs, seg = [], [], []
        for s in range(G):
            mo = shuffle.map_side([dev(rep[at[s]:at[s + 1]])], [dev(v[at[s]:at[s + 1]])], P, None, False, sb,
                                  row_hash=d_h, unordered=True)
            o = mo.offsets.cpu().numpy()
            ks.append(mo.keys[o[b0]:o[b1]])
            vs.append(mo.vals[o[b0]:o[b1]])
            seg.append(np.diff(o)[b0:b1])
        own = np.concatenate([want[p][0] for p in range(blocks[r], blocks[r + 1])])[:16]
        assert len(own) == 16
        ks.append(dev(own))
        vs.append(dev(np.full(16, 10 ** 9, dtype=np.int64)))
        rx = shuffle.Received(torch.cat(ks), torch.cat(vs), dev(np.array(seg, dtype=np.int64)), blocks[r],
                              blocks[r + 1] - blocks[r], sb, bound=True)
        ok, ov, off, cnt = (t.cpu().numpy() for t in nv().combine(rx.keys, rx.vals, "sum", P, rx.seg, rx.part_first,
                                                                    rx.nparts, None, sb, row_hash=d_h))
        assert (cnt >= 0).all()
        for j in range(rx.nparts):
            wk, wv, _ = want[rx.part_first + j]
            _check_part(ok[off[j]:off[j] + cnt[j]], ov[off[j]:off[j] + cnt[j]], wk, wv, "sum")


# ----------------------------------------------------------------------------- 4. the operator surface at scale
N4, D4, M4 = 1_000_000, 200_000, 8
SURFACE_P = [1, 6, 64, 4096]
_NON_ASCII = ["é", "ß", "你", "好", "\U0001f600", "\ud83d", "\ude00", "ÿ", "\u0800",
              "\U0010ffff"]


def _key_table(kind, d):
    """d distinct keys, key 0 the empty one.  non_ascii: the decimal digits of the id spelled with 2-, 3- and 4-byte
    characters and lone surrogates (id 56 is "\\ud83d\\ude00", id 4 "\\U0001f600": two different keys).  bytes: high
    bytes only, or ASCII digits with b"\\x80\\0" behind.  tuple: (float, (str, None))."""
    if kind == "ascii":
        return [""] + ["w%d" % i for i in range(1, d)]
    if kind == "non_ascii":
        return [""] + ["".join(_NON_ASCII[int(c)] for c in str(i)) for i in range(1, d)]
    if kind == "bytes":
        return [b""] + [bytes(0xF0 + int(c) for c in str(i)) if i % 2 else str(i).encode() + b"\x80\0"
                        for i in range(1, d)]
    return [(float(i % 1000 - 500), ("s%d" % (i // 1000), None)) for i in range(d)]


@functools.lru_cache(maxsize=None)
def _surface(kind):
    """(keys of N4 rows, {key: portable_hash}, int values, float values).  Tuple keys whose float is 0.0 are spelled
    (-0.0, ...) in every other row: one Python key.  Tuple keys are ingested leaf by leaf in Python, so that kind runs
    at a fifth of the size (2e5 rows, 4e4 keys)."""
    rng = np.random.default_rng(len(kind))
    n, d = (N4, D4) if kind != "tuple" else (N4 // 5, D4 // 5)
    table = _key_table(kind, d)
    ids = rng.integers(0, d, n).tolist()
    keys = [table[i] for i in ids]
    if kind == "tuple":
        keys = [(-0.0, k[1]) if k[0] == 0.0 and r % 2 else k for r, k in enumerate(keys)]
        assert any(math.copysign(1.0, k[0]) < 0 for k in keys)
        hashes = {k: orc.portable_hash(k) for k in table}
    else:
        data, offs = _columns([k.encode("utf-8", "surrogatepass") for k in table] if kind != "bytes" else table)
        hashes = dict(zip(table, orc.hash_bytes_vec(data, offs, 0 if kind == "bytes" else 1).tolist()))
    return keys, hashes, rng.integers(-1000, 1000, n).tolist(), (rng.standard_normal(n) * 100).tolist()


def ctx():
    sys.argv = [sys.argv[0]]
    from dpark_b200 import DparkContext
    return DparkContext("local")


def _part_of(h, P, thr):
    return h % P if thr is None else bisect.bisect(thr, h)


def _check_reduced(parts, keys, vals, hashes, P, thr, func):
    """Every key once, in its reference partition; ints and max exact, float sums within 1e-9 * sum |v| of the key
    around math.fsum."""
    per = {}
    for k, x in zip(keys, vals):
        per.setdefault(k, []).append(x)
    assert len(parts) == P
    seen = set()
    for p, part in enumerate(parts):
        for k, got in part:
            assert k not in seen
            seen.add(k)
            xs = per[k]
            assert _part_of(hashes[k], P, thr) == p, (k, p)
            if func == "fsum":
                assert abs(got - math.fsum(xs)) <= 1e-9 * math.fsum(abs(x) for x in xs), k
            else:
                assert got == (sum(xs) if func == "add" else max(xs)), k
    assert len(seen) == len(per)


def _check_grouped(parts, keys, hashes, P):
    """Values are the row numbers: a key's list must be its rows in (map split, position) order, i.e. increasing."""
    want = {}
    for i, k in enumerate(keys):
        want.setdefault(k, []).append(i)
    assert len(parts) == P
    n = 0
    for p, part in enumerate(parts):
        for k, vs in part:
            assert _part_of(hashes[k], P, None) == p, (k, p)
            assert list(vs) == want[k], k
            n += 1
    assert n == len(want)


SURFACE_KINDS = ["ascii", "non_ascii", "bytes", "tuple"]


@pytest.mark.parametrize("P", SURFACE_P)
@pytest.mark.parametrize("kind", SURFACE_KINDS)
def test_reduce_and_group_by_key_at_scale(kind, P):
    """1e6 rows, 2e5 keys, 8 map splits: groupByKey at every P and one reduceByKey, against Python dicts -- + on ints
    at P = 1 and 4096, + on floats at P = 6, max at P = 64; the partition of every key is the reference's
    getPartition."""
    keys, hashes, ivals, fvals = _surface(kind)
    dc = ctx()
    func, vals, check = {1: (operator.add, ivals, "add"), 6: (operator.add, fvals, "fsum"), 64: (max, fvals, "max"),
                         4096: (operator.add, ivals, "add")}[P]
    _check_reduced(dc.parallelize(list(zip(keys, vals)), M4).reduceByKey(func, P).glom().collect(),
                   keys, vals, hashes, P, None, check)
    _check_grouped(dc.parallelize([(k, i) for i, k in enumerate(keys)], M4).groupByKey(P).glom().collect(),
                   keys, hashes, P)


@pytest.mark.parametrize("kind", SURFACE_KINDS)
def test_combine_by_key_with_thresholds_at_scale(kind):
    from dpark_b200 import Aggregator, HashPartitioner
    keys, hashes, ivals, _ = _surface(kind)
    thr = sorted(np.quantile(np.array(list(hashes.values()), dtype=np.float64), [0.1, 0.3, 0.5, 0.9]).astype(np.int64)
                 .tolist() + [0])
    add = operator.add
    got = ctx().parallelize(list(zip(keys, ivals)), M4).combineByKey(
        Aggregator(lambda x: x, add, add), HashPartitioner(len(thr) + 1, thresholds=thr)).glom().collect()
    _check_reduced(got, keys, ivals, hashes, len(thr) + 1, thr, "add")


def test_degraded_string_hash_changes_layout_but_never_merges_keys(monkeypatch):
    """hash_bytes keeping only 3 bits: every key lands where its degraded hash says, and distinct strings that now
    share a hash stay distinct (15 000 keys, so the probe chains of dict_encode stay short enough)."""
    from dpark_b200 import _native
    real = _native.hash_bytes
    monkeypatch.setattr(_native, "hash_bytes", lambda d, o, m: real(d, o, m) & 7)
    rng = np.random.default_rng(8)
    table = ["w%d" % i for i in range(15_000)]
    keys = [table[i] for i in rng.integers(0, len(table), 200_000).tolist()]
    data, offs = _columns([k.encode() for k in table])
    hashes = dict(zip(table, (orc.hash_bytes_vec(data, offs, 1) & 7).tolist()))
    vals = rng.integers(-1000, 1000, len(keys)).tolist()
    dc, P = ctx(), 6
    _check_reduced(dc.parallelize(list(zip(keys, vals)), M4).reduceByKey(operator.add, P).glom().collect(),
                   keys, vals, hashes, P, None, "add")
    _check_grouped(dc.parallelize([(k, i) for i, k in enumerate(keys)], M4).groupByKey(P).glom().collect(),
                   keys, hashes, P)


# ----------------------------------------------------------------------------- 5. tuple and byte hashes on the device
def _orc_tuple_hash(items):
    """items: int64 [arity, n] -> tuple_hash of every column, by the oracle."""
    L = orc.lib()
    cols = np.ascontiguousarray(items.T)
    return np.array([L.orc_hash_tuple(orc._p(np.ascontiguousarray(c)), items.shape[0]) for c in cols],
                    dtype=np.int64)


@pytest.mark.parametrize("n", [1, 255, 256, 257, 100_000])
def test_hash_tuple_matches_the_oracle(n):
    rng = np.random.default_rng(n)
    special = np.array([-1, -2, 0, I64_MIN, I64_MAX], dtype=np.int64)
    for arity in (0, 1, 2, 3, 8):
        items = rng.integers(I64_MIN, I64_MAX, (arity, n), dtype=np.int64, endpoint=True)
        if arity:
            mask = rng.random((arity, n)) < 0.3
            items[mask] = special[rng.integers(0, len(special), int(mask.sum()))]
        got = nv().hash_tuple(dev(items)).cpu().numpy()
        assert np.array_equal(got, _orc_tuple_hash(items)), arity
    inner = rng.integers(I64_MIN, I64_MAX, (3, n), dtype=np.int64, endpoint=True)    # ((a, b, c), d, (e,))
    inner[0, ::3] = -1
    last = rng.integers(-3, 3, (1, n), dtype=np.int64)
    outer = np.stack([_orc_tuple_hash(inner), rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True),
                      _orc_tuple_hash(last)])
    d_outer = torch.stack([nv().hash_tuple(dev(inner)), dev(outer[1]), nv().hash_tuple(dev(last))]).contiguous()
    assert np.array_equal(nv().hash_tuple(d_outer).cpu().numpy(), _orc_tuple_hash(outer))


@pytest.mark.parametrize("mode", [0, 1])
def test_hash_bytes_lone_surrogates_and_long_keys(mode):
    """Lone surrogates (UTF-8 with surrogatepass: 3-byte sequences unicode_hash sees as code points D800-DFFF) and
    keys longer than 4096 bytes."""
    rng = np.random.default_rng(12 + mode)
    alph = ["\ud800", "\udbff", "\udc00", "\udfff", "\ud83d", "\ude00", "\U0001f600", "a", "é", "你"]
    strs = ["\ud83d\ude00", "\U0001f600", ""] + ["".join(rng.choice(alph, rng.integers(0, 12))) for _ in range(3000)]
    strs += ["".join(rng.choice(alph, m)) for m in (1366, 1400, 4097, 5000, 20_000)]
    strs += ["x" * m for m in (4095, 4096, 4097, 65_536)]
    blobs = [s.encode("utf-8", "surrogatepass") for s in strs]
    data, offs = _columns(blobs)
    got = nv().hash_bytes(dev(data), dev(offs), mode).cpu().numpy()
    assert np.array_equal(got, orc.hash_bytes_vec(data, offs, mode))
    # and against portable_hash of the Python objects (code points for str, signed chars for bytes)
    objs = strs if mode == 1 else blobs
    assert got[:200].tolist() + got[-9:].tolist() == [orc.portable_hash(x) for x in objs[:200] + objs[-9:]]


# ----------------------------------------------------------------------------- 6. overflow of the string reduce side
def test_string_reduce_raises_when_a_partition_merge_failed(monkeypatch):
    """A merge that fails marks its partition with out_counts = -1; the str/bytes/tuple reduceByKey must raise instead
    of returning that partition empty."""
    from dpark_b200 import _native, columnar, strings
    from dpark_b200.engine import ShuffleResult
    splits = [columnar.ingest_pairs([("w%d" % (i % 50), 1) for i in range(a, a + 500)]) for a in (0, 500)]
    dev0 = torch.device("cuda", torch.cuda.current_device())
    res = strings.reduce_by_key_bytes(splits, columnar.KEY_STR, 4, None, "sum", dev0, ShuffleResult(4))
    assert sorted(k for p in range(4) for k in res.parts[p][0]) == sorted("w%d" % i for i in range(50))
    real = _native.combine

    def failing(*a, **kw):
        ok, ov, off, cnt = real(*a, **kw)
        cnt[1] = -1
        return ok, ov, off, cnt
    monkeypatch.setattr(strings.nv, "combine", failing)
    with pytest.raises(_native.NativeError):
        strings.reduce_by_key_bytes(splits, columnar.KEY_STR, 4, None, "sum", dev0, ShuffleResult(4))
