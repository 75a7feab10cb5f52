"""Guarded, poison-filled device buffers for every one-GPU operator, swept across its kernels' tile boundaries.  -m gpu.

Every buffer a kernel of the library writes comes from torch.empty / zeros / full / ones (or their _like forms) in one
of its modules.  The `guarded` fixture replaces the module attribute `torch` of each of those modules with a proxy
that hands out every CUDA allocation as the body of one flat uint8 buffer [guard | body | guard]:
  - the guards (GUARD bytes, a multiple of 512 so the body keeps the allocator's alignment) hold the poison byte;
  - the body of an empty / empty_like holds the poison byte too; zeros / full / ones are filled as asked.
After every operator call the guards are compared with the poison byte: a kernel store past either end of an output,
scratch buffer or workspace names the allocation, its caller and the first changed offset.  Every case runs under two
poison bytes, 0x00 and 0xFF (NaN in floats, -1 in ints): an output element a kernel should have written but did not
keeps the poison, so the result cannot equal the oracle under both, and the two runs must be bit-identical.  While an
operator runs, reading a ColumnarRDD as rows (the composition's fallback) fails the case, and the operator must have
made at least one guarded allocation: every case proves it ran on the device.

The sizes sit on the kernels' tail paths, with the constants read from dpark_b200/csrc (or _native where it has
them): the multisplit tiles (PT_TILE and its multiples), both map-side paths (one launch over consecutive splits, one
per split otherwise), k_smem_aggregate2's windows (AG2_CAP, with the hot key alone in its fine bucket and with other
keys beside it), the group-by's radix tiles (GR_TILE), the join emit tiles (JN_TILE, in output rows), topByKey's chunks
(TOPK_TILE), the select's tiles (SEL_TILE), its one-CTA tile scan (SEL_SCAN_THREADS tiles) and grid-stride cap, the
t-digest's short / long build split (TD_SHORT) and capacity (TD_CAP), the MT19937 twist (MT_N words, MT_N / 2 draws),
and the tokeniser's TK_BYTES slices and TK_THREADS * TK_BYTES-byte blocks.  Split counts are chosen so that split
starts of 4-byte columns fall on every residue modulo 16.  The oracles are the suite's own.

Not seen by the guards: buffers torch itself makes and kernels only read (torch.arange / tensor / cat / stack, .to(dev)
copies of inputs, cumsum and searchsorted results).  The t-digest fold stage limit TD_STAGE (2 * TD_CAP) is not swept:
k_td_merge folds a digest of at most TD_CAP centroids with another of at most TD_CAP, so no input was found that
stages more than TD_STAGE entries."""
import collections
import os
import re
import sys

import numpy as np
import pytest
import torch

from dpark_b200 import _native as nv
from tests import cogroup_common as cc
from tests.shuffle_cases import REDUCE_VARIANTS, dpk_options, variant_id  # noqa: F401
from tests.test_gpu_sample import _rows_of, _want_masks
from tests.test_gpu_topbykey import _oracle_top
from tests.test_gpu_uniq_top_hot import _hot_oracle, oracle_uniq
from tests.test_gpu_variants import _check_part, _oracle_reduce

pytestmark = pytest.mark.gpu

GUARD = 4096
POISONS = (0x00, 0xFF)
GUARDED_MODULES = ["_native", "shuffle", "grouping", "join", "topk", "sorting", "percentiles", "sampling", "selecting",
                   "columnar", "engine", "strings", "textingest"]

# The native wrappers (and library functions) that allocate a buffer a kernel writes; each must be reached by the sweep.
KERNEL_OUTPUT_SITES = [
    "hash_keys", "hash_bytes", "hash_tuple", "partition_ids", "partition_workspace", "partition_count", "packed_rows",
    "partition", "map_side", "dict_encode", "combine", "sort_by_key_bits", "radix_pass_seg", "group_heads",
    "group_side", "key_or", "gather_i64", "join_count", "join_emit", "cogroup_count", "cogroup_emit", "topk_lengths",
    "topk_round", "bcast_build", "bcast_probe", "bcast_emit", "sort_keys", "sort_cuts", "sort_gather", "gather_columns",
    "tdigest_heads", "tdigest_build", "tdigest_merge", "sample_bernoulli", "select_state", "select_compact",
    "select_take", "uniq_insert", "uniq_emit", "tokenize", "gather_bytes",
]
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dpark_b200", "csrc")


def _csrc_constants(files):
    """The integer constexpr constants of the kernel sources, evaluated in order (those defined in terms of template
    parameters or sizeof are skipped)."""
    env = {}
    for name in files:
        with open(os.path.join(CSRC, name)) as f:
            text = f.read()
        for stmt in re.findall(r"constexpr\s+(?:int|int64_t)\s+([^;]+);", text):
            for const, expr in re.findall(r"(\w+)\s*=\s*([^,]+)", stmt):
                try:
                    env[const] = int(eval(expr, {"__builtins__": {}}, dict(env)))
                except Exception:
                    pass
    return env


K = _csrc_constants(["dpk_common.cuh", "dpk_partition.cu", "dpk_aggregate2.cuh", "dpk_group.cu", "dpk_join.cu",
                     "dpk_select.cu", "dpk_sort.cu", "dpk_tdigest.cu", "dpk_strings.cu"])
with open(os.path.join(CSRC, "dpk_select.cu")) as _f:
    SEL_CTAS_PER_SM = int(re.search(r"sm_count\(\) \* (\d+)", _f.read()).group(1))    # sel_blocks' grid-stride cap
with open(os.path.join(CSRC, "dpk_join.cu")) as _f:
    BCAST_BLOCK = int(re.search(r"k_bcast_probe<int64_t><<<blocks, (\d+)", _f.read()).group(1))   # rows per probe CTA
PT_TILE, AG2_CAP, GR_TILE, JN_TILE, SO_THREADS = K["PT_TILE"], K["AG2_CAP"], K["GR_TILE"], K["JN_TILE"], K["SO_THREADS"]
SEL_TILE, SEL_SCAN_THREADS, SEL_THREADS = K["SEL_TILE"], K["SEL_SCAN_THREADS"], K["SEL_THREADS"]
TD_SHORT, TD_WARPS, TK_BYTES, TK_BLOCK = K["TD_SHORT"], K["TD_WARPS"], K["TK_BYTES"], K["TK_THREADS"] * K["TK_BYTES"]
TD_CAP, TOPK_TILE, MT_N = nv.TD_CAP, nv.TOPK_TILE, nv.MT_N
assert (K["TD_CAP"], K["MT_N"]) == (TD_CAP, MT_N)

REACHED = collections.Counter()     # allocating function -> guarded allocations, over the whole module
SWEEPS_RUN = set()


# ------------------------------------------------------------------------------------------------ the guarded allocator
class _Alloc(object):
    __slots__ = ("buf", "nbytes", "poison", "module", "caller", "shape", "dtype")

    def __init__(self, buf, nbytes, poison, module, caller, shape, dtype):
        self.buf, self.nbytes, self.poison = buf, nbytes, poison
        self.module, self.caller, self.shape, self.dtype = module, caller, shape, dtype

    def __repr__(self):
        return "%s.%s: %s %s (%d bytes)" % (self.module, self.caller, self.dtype, tuple(self.shape), self.nbytes)


class Guard(object):
    """The allocation record of one test and the poison byte the next allocations get."""

    def __init__(self):
        self.poison = POISONS[0]
        self.records = []

    def alloc(self, fn, fill, args, kw, module, caller):
        like = args[0] if fn.__name__.endswith("_like") else None
        dev = kw.get("device")
        dev = torch.device(dev) if dev is not None else (like.device if like is not None else torch.device("cpu"))
        if dev.type != "cuda":
            return fn(*args, **kw)
        meta = fn(*args, **dict(kw, device="meta"))
        if not meta.is_contiguous():
            raise AssertionError("%s.%s: a non-contiguous %s the guard cannot lay out" % (module, caller, fn.__name__))
        nbytes = meta.numel() * meta.element_size()
        buf = torch.full((2 * GUARD + nbytes,), self.poison, dtype=torch.uint8, device=dev)
        body = buf[GUARD:GUARD + nbytes].view(meta.dtype).view(meta.shape)
        if fill is not None:
            body.fill_(fill(args, kw))
        self.records.append(_Alloc(buf, nbytes, self.poison, module, caller, meta.shape, meta.dtype))
        REACHED[caller] += 1
        return body

    def copy_in(self, t, caller):
        """A guarded CUDA copy of the host tensor t."""
        dev = torch.device("cuda", torch.cuda.current_device())
        body = self.alloc(torch.empty, None, (tuple(t.shape),), {"dtype": t.dtype, "device": dev}, "_native", caller)
        body.copy_(t)
        return body

    def check(self):
        """Synchronise, then compare every recorded guard with its poison byte; forget the records."""
        torch.cuda.synchronize()
        recs, self.records = self.records, []
        if not recs:
            return
        heads = torch.stack([r.buf[:GUARD] for r in recs])
        tails = torch.stack([r.buf[GUARD + r.nbytes:] for r in recs])
        pv = torch.tensor([r.poison for r in recs], dtype=torch.uint8, device=heads.device).unsqueeze(1)
        bad_h, bad_t = (heads != pv).any(1).cpu().tolist(), (tails != pv).any(1).cpu().tolist()
        msgs = []
        for i, r in enumerate(recs):
            if bad_h[i]:
                at = int((r.buf[:GUARD] != r.poison).nonzero()[0]) - GUARD
                msgs.append("%r: store before the body at offset %d" % (r, at))
            if bad_t[i]:
                at = r.nbytes + int((r.buf[GUARD + r.nbytes:] != r.poison).nonzero()[0])
                msgs.append("%r: store past the body at offset %d" % (r, at))
        if msgs:
            raise AssertionError("guard bytes changed:\n  " + "\n  ".join(msgs))


def _fill_zero(args, kw):
    return 0


def _fill_one(args, kw):
    return 1


def _fill_value(args, kw):
    return args[1] if len(args) > 1 else kw["fill_value"]


class GuardedTorch(object):
    """torch, except that empty / empty_like / zeros / zeros_like / full / ones of a CUDA tensor go through a Guard."""

    def __init__(self, guard, module):
        self._guard, self._module = guard, module

    def __getattr__(self, name):
        return getattr(torch, name)

    def _alloc(self, fn, fill, args, kw):
        return self._guard.alloc(fn, fill, args, kw, self._module, sys._getframe(2).f_code.co_name)

    def empty(self, *args, **kw):
        return self._alloc(torch.empty, None, args, kw)

    def empty_like(self, *args, **kw):
        return self._alloc(torch.empty_like, None, args, kw)

    def zeros(self, *args, **kw):
        return self._alloc(torch.zeros, _fill_zero, args, kw)

    def zeros_like(self, *args, **kw):
        return self._alloc(torch.zeros_like, _fill_zero, args, kw)

    def full(self, *args, **kw):
        return self._alloc(torch.full, _fill_value, args, kw)

    def ones(self, *args, **kw):
        return self._alloc(torch.ones, _fill_one, args, kw)


@pytest.fixture
def guarded(monkeypatch, request):
    """A Guard installed in every module that allocates kernel buffers.  select_state's state and histogram are made
    on the host and copied to the device by selecting.select_smallest: they are handed out guarded instead."""
    import importlib
    from dpark_b200 import _native as nv
    g = Guard()
    for name in GUARDED_MODULES:
        mod = importlib.import_module("dpark_b200." + name)
        monkeypatch.setattr(mod, "torch", GuardedTorch(g, name))
    real_state = nv.select_state
    monkeypatch.setattr(nv, "select_state", lambda n, m: tuple(g.copy_in(t, "select_state") for t in real_state(n, m)))
    SWEEPS_RUN.add(request.function.__name__)
    yield g
    g.records = []


def _canon(x):
    """A comparable form of a result: tensors and arrays by dtype and bytes, floats by repr."""
    if torch.is_tensor(x):
        x = x.detach().cpu().numpy()
    if isinstance(x, np.ndarray):
        return ("nd", x.dtype.str, x.shape, x.tobytes())
    if isinstance(x, (list, tuple)):
        return tuple(_canon(y) for y in x)
    if isinstance(x, dict):
        return tuple(sorted((repr(k), _canon(v)) for k, v in x.items()))
    return repr(x)


def _read_as_rows(*args, **kw):
    raise AssertionError("the operator read its input as rows: it did not run on the device")


def _on_the_device(op):
    """op() with the row-path fallbacks of the device operators refused (the reads device_spy refuses in
    tests/test_gpu_uniq_top_hot.py)."""
    from dpark_b200 import columnar, strings
    from dpark_b200.rdd import ColumnarRDD
    saved = [(ColumnarRDD, "compute"), (strings, "reduce_by_key_bytes"), (columnar, "_tuple_identity_bytes")]
    saved = [(owner, name, owner.__dict__[name]) for owner, name in saved]
    for owner, name, _ in saved:
        setattr(owner, name, _read_as_rows)
    try:
        return op()
    finally:
        for owner, name, real in saved:
            setattr(owner, name, real)


def sweep(g, op, check):
    """op() on the device under each poison byte, the guards checked after it; check(result) against the oracle; both
    results bit-identical."""
    outs = []
    g.check()                         # what the oracle allocated
    for p in POISONS:
        g.poison = p
        out = _on_the_device(op)
        assert g.records, "the operator made no guarded allocation: it never reached the native code"
        g.check()
        check(out)
        outs.append(_canon(out))
    assert outs[0] == outs[1], "the result depends on the poison byte"


def _m(n, choices=(5, 7, 9, 11, 6, 4, 3)):
    """A split count whose split length ceil(n / M) is odd: the starts of 4-byte columns cycle through every residue
    modulo 16."""
    for M in choices:
        if M <= n and (-(-n // M)) % 2 == 1:
            return M
    return choices[0]


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _rows_equal(got, want):
    assert got == want and repr(got) == repr(want), "differs from the oracle"


# ------------------------------------------------------------------------------------------------ the fixture can fail
def test_a_store_into_a_guard_is_reported(guarded):
    from dpark_b200 import _native as nv
    for p in POISONS:
        guarded.poison = p
        nv.hash_keys(torch.arange(100, device="cuda"))
        rec = [r for r in guarded.records if r.caller == "hash_keys"][-1]
        rec.buf[GUARD + rec.nbytes + 3] = p ^ 0x5A          # 3 bytes past the body's end
        with pytest.raises(AssertionError, match=r"_native\.hash_keys.*past the body at offset 803"):
            guarded.check()
        nv.hash_keys(torch.arange(100, device="cuda"))
        rec = guarded.records[-1]
        rec.buf[GUARD - 1] = p ^ 1
        with pytest.raises(AssertionError, match=r"_native\.hash_keys.*before the body at offset -1"):
            guarded.check()
        guarded.check()                                     # the records went with the report


TOP_KEYS = {"none": None, "first": lambda x: x[0], "second": lambda x: x[1]}


def _top_order(k, v, key, reverse):
    """Row ids in the order of rdd.top(n, key, reverse) = sorted(rows, key=key, reverse=not reverse)[:n], which keeps
    equal rows in row order: a stable np.lexsort (its last key is the primary one)."""
    cols = {"none": (v, k), "first": (k,), "second": (v,)}[key]
    if not reverse:
        cols = tuple(-c for c in cols)                      # the largest first (-0.0 and 0.0 stay equal)
    return np.lexsort((np.arange(len(k)),) + cols)


def _top_case(g, n, key, reverse, m, seed=0):
    rng = np.random.default_rng(seed)
    k = rng.integers(-40, 40, n).astype(np.int32)
    v = rng.integers(-8, 8, n).astype(np.float64) * 0.5
    v[rng.random(n) < 0.1] = -0.0
    sel = _top_order(k, v, key, reverse)[:m]
    want = list(zip(k[sel].tolist(), v[sel].tolist()))
    dk, dv = _cuda(k), _cuda(v)
    dc = cc.ctx()
    sweep(g, lambda: dc.parallelizeColumns(dk, dv, _m(n)).top(m, key=TOP_KEYS[key], reverse=reverse),
          lambda got: _rows_equal(got, want))


def test_a_skipped_output_element_fails_the_oracle(guarded, monkeypatch):
    from dpark_b200 import _native as nv
    real = nv.gather_columns

    def loses_the_last_value(keys, vals, ids):
        ok, ov = real(keys, vals, ids)
        if ov.numel():
            ov.view(torch.uint8)[-ov.element_size():] = guarded.poison
        return ok, ov

    monkeypatch.setattr(nv, "gather_columns", loses_the_last_value)
    with pytest.raises(AssertionError, match="differs from the oracle"):
        _top_case(guarded, 3000, "none", False, 10)


# ------------------------------------------------------------------------------------------------ reduceByKey
KINDS = [(np.int64, np.int64), (np.int32, np.float32), (np.int64, np.int32), (np.float64, np.float64)]
TILE_ROWS = [b + d for b in (PT_TILE, 2 * PT_TILE, 4 * PT_TILE) for d in (-1, 0, 1)]
HOT_ROWS = [b + d for b in (AG2_CAP, 2 * AG2_CAP) for d in (-1, 0, 1)]
PS = [1, 7, 9, 31, 33]


def _reduce_input(rng, kind, n, hot):
    """n rows of keys in [-n, n); with hot: one key of `hot` rows and n other rows of 1000 keys (n = 0: the hot key
    alone in its fine bucket, so the bucket holds exactly `hot` rows)."""
    kt, vt = kind
    k = rng.integers(-n, n, n)
    if hot:
        k = np.concatenate([np.full(hot, 12345), rng.integers(-500, 500, n)])
        k = k[rng.permutation(len(k))]
    v = rng.integers(-1000, 1000, len(k))
    if np.dtype(vt).kind == "f":
        v = v * 0.25
    return k.astype(kt), v.astype(vt)


def _reduce_case(g, k, v, P, map_combine, per_split):
    """per_split: the map splits go in reverse order, so they are no run of consecutive slices (shuffle._as_one) and
    the map side counts and scatters every split by itself, at the split starts parallelizeColumns gives."""
    from dpark_b200 import shuffle
    op = "max" if v.dtype.kind == "f" else "sum"     # exact in every order, so both runs are bit-identical
    M = _m(len(k))
    col = cc.ctx().parallelizeColumns(_cuda(k), _cuda(v), M)
    order = col.splits[::-1] if per_split else col.splits
    splits = [col.columns(sp) for sp in order]
    want = _oracle_reduce([k[sp.begin:sp.end] for sp in order], [v[sp.begin:sp.end] for sp in order], P, op)

    def run():
        before = REACHED["partition_count"]
        res = shuffle.reduce_by_key([a for a, _ in splits], [b for _, b in splits], P, op, map_combine=map_combine)
        assert REACHED["partition_count"] - before == (len(splits) if per_split and len(splits) > 1 else 0)
        out = []
        for p, gk, gv in res:
            gk, gv = gk.cpu().numpy(), gv.cpu().numpy()
            o = np.argsort(gk, kind="stable")
            out.append((p, gk[o], gv[o]))
        return out

    def check(out):
        assert [p for p, _, _ in out] == list(range(P))
        for p, gk, gv in out:
            wk, wv, tol = want[p]
            _check_part(gk, gv, wk, wv, op, tol)

    sweep(g, run, check)


REDUCE_RUNS = [(v, False) for v in REDUCE_VARIANTS] + [({}, True)]


@pytest.mark.parametrize("variant, map_combine", REDUCE_RUNS,
                         ids=[variant_id(v) + ("-map_combine" if mc else "") for v, mc in REDUCE_RUNS])
def test_reduce_by_key_at_tile_and_window_boundaries(variant, map_combine, guarded, dpk_options):
    dpk_options(variant)
    rng = np.random.default_rng(len(variant_id(variant)))
    cases = [(n, None) for n in TILE_ROWS] + [(300, h) for h in HOT_ROWS] + [(0, h) for h in HOT_ROWS]
    for i, (n, hot) in enumerate(cases):
        k, v = _reduce_input(rng, KINDS[i % len(KINDS)], n, hot)
        _reduce_case(guarded, k, v, PS[i % len(PS)], map_combine, per_split=i % 2 == 1)


# ---------------------------------------------------------------------------------------- groupByKey, cogroup, joins
JOINS = ["join", "leftOuterJoin", "rightOuterJoin", "outerJoin"]


def _pair_columns(rng, kdt, vdt, keys):
    v = rng.integers(-1000, 1000, len(keys))
    return (torch.from_numpy(np.asarray(keys)).to(kdt),
            torch.from_numpy(v * 0.25 if vdt.is_floating_point else v).to(vdt))


def _group_case(g, k, v, P):
    dc = cc.ctx()
    dk, dv = k.cuda(), v.cuda()
    M = _m(len(k))
    want = dc.parallelize(list(zip(k.tolist(), v.tolist())), M).groupByKey(P).glom().collect()
    sweep(g, lambda: dc.parallelizeColumns(dk, dv, M).groupByKey(P).glom().collect(),
          lambda got: _rows_equal(got, want))


def test_group_by_key_at_radix_tiles(guarded):
    rng = np.random.default_rng(1)
    for i, n in enumerate((GR_TILE - 1, GR_TILE, GR_TILE + 1, 2 * GR_TILE + 1)):
        kdt, vdt = [(torch.int64, torch.float32), (torch.float64, torch.int32), (torch.int32, torch.int64),
                    (torch.float32, torch.float64)][i]
        keys = rng.integers(-n // 3, n // 3, n).astype(np.float64 if kdt.is_floating_point else np.int64)
        k, v = _pair_columns(rng, kdt, vdt, keys)
        _group_case(guarded, k, v, PS[i % len(PS)])


def _product_sides(products):
    """Left and right key lists whose joined output has the given per-key row counts (L * R each)."""
    left, right = [], []
    for key, (nl, nr) in enumerate(products):
        left += [key] * nl
        right += [key] * nr
    return np.array(left, np.int64), np.array(right, np.int64)


def _products(n_out, L, R):
    """(L, R) per key: keys of L x R rows, and one key of the remainder x 1, n_out joined rows in all."""
    q, r = divmod(n_out, L * R)
    return [(L, R)] * q + ([(r, 1)] if r else [])


# joined rows at the emit tiles (JN_TILE - 1 .. 2 JN_TILE + 1): from one big product, and from many small ones
PRODUCTS = {"%d" % n: _products(n, n // 32, 32) for n in (b + d for b in (JN_TILE, 2 * JN_TILE) for d in (-1, 0, 1))}
PRODUCTS["tiles_of_many_keys"] = _products(2 * JN_TILE + 1, 3, 5)


@pytest.mark.parametrize("products", sorted(PRODUCTS))
def test_joins_and_cogroup_at_emit_tiles(products, guarded):
    rng = np.random.default_rng(len(products))
    lk, rk = _product_sides(PRODUCTS[products])
    lk = np.concatenate([lk, rng.integers(1000, 1100, 50)])       # keys of one side only
    rk = np.concatenate([rk, rng.integers(2000, 2100, 40)])
    lk, rk = lk[rng.permutation(len(lk))], rk[rng.permutation(len(rk))]
    dc = cc.ctx()
    sides = [(lk, torch.int64, torch.float32), (rk, torch.int64, torch.float64)]
    for which in ("both", "right_empty"):
        (a_k, a_v), (b_k, b_v) = [_pair_columns(rng, kdt, vdt, keys if which == "both" or i == 0 else keys[:0])
                                  for i, (keys, kdt, vdt) in enumerate(sides)]
        Ma, Mb = _m(len(a_k)), _m(max(1, len(b_k)))
        ra = dc.parallelize(list(zip(a_k.tolist(), a_v.tolist())), Ma)
        rb = dc.parallelize(list(zip(b_k.tolist(), b_v.tolist())), Mb)
        ca, cb = (a_k.cuda(), a_v.cuda()), (b_k.cuda(), b_v.cuda())
        for kind, P in zip(JOINS + ["groupWith"], (1, 7, 9, 33, 5)):
            if kind == "groupWith":
                want = ra.groupWith([rb], P).glom().collect()
            else:
                want = getattr(ra, kind)(rb, P).glom().collect()
            if kind == "join" and which == "both":
                assert sum(map(len, want)) == sum(nl * nr for nl, nr in PRODUCTS[products])

            def run():
                a, b = dc.parallelizeColumns(*ca, Ma), dc.parallelizeColumns(*cb, Mb)
                if kind == "groupWith":
                    return a.groupWith([b], P).glom().collect()
                return getattr(a, kind)(b, P).glom().collect()
            sweep(guarded, run, lambda got: _rows_equal(got, want))
        # the left side empty: the mirror image
        want = rb.leftOuterJoin(ra.filter(lambda x: False), 3).glom().collect()
        sweep(guarded, lambda: dc.parallelizeColumns(*cb, Mb).leftOuterJoin(
            dc.parallelizeColumns(ca[0][:0], ca[1][:0], 2), 3).glom().collect(), lambda got: _rows_equal(got, want))


# ------------------------------------------------------------------------------------------------ innerJoin
HOT_REPEAT = 32                   # rows of the small side's hot key: each big row of that key emits 32 output rows


def _inner_join_keys(rng, sk, nbig, n_out):
    """Big keys that give exactly n_out output rows against the small keys sk + (HOT_REPEAT - 1) more rows of sk[0]:
    n_out // HOT_REPEAT rows of the hot key, n_out % HOT_REPEAT of single keys, the rest without a match."""
    a, b = divmod(n_out, HOT_REPEAT)
    assert a + b <= nbig
    bk = np.concatenate([np.full(a, sk[0]), sk[1:][rng.integers(0, len(sk) - 1, b)], np.full(nbig - a - b, -7)])
    return bk[rng.permutation(nbig)]


@pytest.mark.parametrize("G", [BCAST_BLOCK - 1, BCAST_BLOCK, BCAST_BLOCK + 1, 2 * BCAST_BLOCK, 4 * BCAST_BLOCK])
def test_inner_join_at_table_doublings_probe_blocks_and_emit_tiles(G, guarded):
    """G distinct small keys at powers of two (the table doubles at 2 G); big rows at the probe blocks; output rows at
    JN_TILE - 1 .. JN_TILE + 1 and 2 JN_TILE - 1 .. 2 JN_TILE + 1, where k_bcast_emit's second CTA and its last
    tile's tail begin."""
    rng = np.random.default_rng(G)
    dc = cc.ctx()
    sk = rng.permutation(G).astype(np.int64) * 3
    small = np.concatenate([sk, np.full(HOT_REPEAT - 1, sk[0])])
    small = small[rng.permutation(len(small))]
    small_k, small_v = _pair_columns(rng, torch.int32, torch.int64, small)
    cs, Ms = (small_k.cuda(), small_v.cuda()), _m(len(small))
    rows_small = dc.parallelize(list(zip(small_k.tolist(), small_v.tolist())), Ms)
    outs = [b + d for b in (JN_TILE, 2 * JN_TILE) for d in (-1, 0, 1)]
    bigs = [BCAST_BLOCK - 1, BCAST_BLOCK, BCAST_BLOCK + 1, JN_TILE - 1, JN_TILE, JN_TILE + 1]
    for i, nbig in enumerate(bigs):
        for n_out in (outs[i], outs[(i + 3) % len(outs)]):
            big_k, big_v = _pair_columns(rng, torch.int64, torch.float32, _inner_join_keys(rng, sk, nbig, n_out))
            Mb = _m(nbig)
            want = dc.parallelize(list(zip(big_k.tolist(), big_v.tolist())), Mb).innerJoin(rows_small).glom().collect()
            assert sum(map(len, want)) == n_out
            cb = (big_k.cuda(), big_v.cuda())
            sweep(guarded,
                  lambda: dc.parallelizeColumns(*cb, Mb).innerJoin(dc.parallelizeColumns(*cs, Ms)).glom().collect(),
                  lambda got: _rows_equal(got, want))


# ------------------------------------------------------------------------------------------------ topByKey
T = TOPK_TILE


@pytest.mark.parametrize("top_n", [1, 511, 512])
def test_top_by_key_at_chunk_boundaries_and_rounds(top_n, guarded):
    from dpark_b200 import topk
    """Runs of T - 1 .. 2T + 1 values and one of 40000 (three rounds at top_n 511 and 512: topk.rounds), ties across
    every chunk cut."""
    rng = np.random.default_rng(top_n)
    lens = [T - 1, T, T + 1, 2 * T - 1, 2 * T, 2 * T + 1, 40000, 511, 512, 513, 1]
    k = np.repeat(np.arange(len(lens), dtype=np.int64) * 5 - 9, lens)
    k = k[rng.permutation(len(k))]
    v = rng.integers(0, 5, len(k)).astype(np.int32)
    dk, dv = _cuda(k), _cuda(v)
    dc = cc.ctx()
    for reverse in (False, True):
        want = _oracle_top(k, v, top_n, reverse)

        def run():
            before = REACHED["topk_round"]
            out = dc.parallelizeColumns(dk, dv, _m(len(k))).topByKey(top_n, reverse=reverse, num_splits=3)
            res = []
            for sp in out.splits:
                keys, off, vals = (t.cpu().numpy() for t in out.columns(sp))
                res.append([(int(key), vals[off[j]:off[j + 1]]) for j, key in enumerate(keys.tolist())])
            return REACHED["topk_round"] - before, res

        def check(out):
            nrounds, res = out
            assert nrounds == topk.rounds(40000, top_n) == (2 if top_n == 1 else 3)
            got = {key: vals for part in res for key, vals in part}
            assert sum(len(part) for part in res) == len(got) == len(want)
            for key, vals in got.items():
                assert np.array_equal(vals.view(np.uint8), want[key].view(np.uint8)), key
        sweep(guarded, run, check)


# ------------------------------------------------------------------------------------------------ sort
SORT_KEYS = {"id": lambda x: x, "first": lambda x: x[0], "second": lambda x: x[1]}


@pytest.mark.parametrize("n", [b + d for b in (SO_THREADS, PT_TILE) for d in (-1, 0, 1)])
def test_sort_at_radix_tiles_with_empty_first_and_last_ranges(n, guarded):
    """Keys from a narrow range over many partitions: the range bounds repeat, so first and last ranges come out
    empty."""
    rng = np.random.default_rng(n)
    dc = cc.ctx()
    k = torch.from_numpy(rng.integers(0, 3, n)).to(torch.float32)
    k[torch.from_numpy(rng.random(n) < 0.2)] = -0.0
    v = torch.from_numpy(rng.integers(-2, 2, n)).to(torch.int64)
    dk, dv = k.cuda(), v.cuda()
    M = _m(n)
    rows = dc.parallelize(list(zip(k.tolist(), v.tolist())), M)
    for key in sorted(SORT_KEYS):
        for reverse in (False, True):
            want = rows.sort(key=SORT_KEYS[key], reverse=reverse, numSplits=9).glom().collect()
            sweep(guarded, lambda: dc.parallelizeColumns(dk, dv, M).sort(key=SORT_KEYS[key], reverse=reverse,
                                                                          numSplits=9).glom().collect(),
                  lambda got: _rows_equal(got, want))


# ------------------------------------------------------------------------------------------------ top, hot, uniq
def _grid_cap():
    """Rows of the select kernels' full grid-stride grid (sel_blocks, dpk_select.cu)."""
    return nv.device_info()["sm_count"] * SEL_CTAS_PER_SM * SEL_THREADS


@pytest.mark.parametrize("n", [b + d for b in (SEL_TILE, 2 * SEL_TILE) for d in (-1, 0, 1)])
def test_top_at_select_tiles(n, guarded):
    for i, (key, reverse) in enumerate([("none", False), ("second", True), ("first", False)]):
        for m in (1, SEL_TILE // 2 + 1, n - 1, n):
            _top_case(guarded, n, key, reverse, m, seed=i)


def test_top_at_the_grid_stride_cap_and_the_tile_scan(guarded):
    """The grid-stride cap, and k_sel_scan's one CTA at SEL_SCAN_THREADS tiles and just above (each thread then scans
    a chunk of two tiles)."""
    cap = _grid_cap()
    scan = SEL_SCAN_THREADS * SEL_TILE
    for n in (cap - 1, cap, cap + 1, scan, scan + 1):
        _top_case(guarded, n, "none", False, n - 1, seed=n)
    _top_case(guarded, cap, "second", True, cap, seed=1)


def _uniq_case(g, k, v, P, hot_ns):
    want = oracle_uniq(k, v, P)
    dk, dv = k.cuda(), v.cuda()
    dc = cc.ctx()
    M = _m(len(k))

    def run():
        u = dc.parallelizeColumns(dk, dv, M).uniq(P)
        return [tuple(t.cpu().numpy() for t in u.columns(sp)) for sp in u.splits]

    def check(parts):
        assert len(parts) == P
        for (gk, gv), (wk, wv, _) in zip(parts, want):
            assert np.array_equal(gk.view(np.uint8), wk.view(np.uint8))
            assert np.array_equal(gv.view(np.uint8), wv.view(np.uint8))
    sweep(g, run, check)
    for n in hot_ns:
        w = _hot_oracle(want, n)
        sweep(g, lambda: dc.parallelizeColumns(dk, dv, M).hot(n, P), lambda got: _rows_equal(got, w))


@pytest.mark.parametrize("n", [1023, 1024, 1025, 2048, 2049, 4097])
def test_uniq_and_hot_at_table_steps(n, guarded):
    """uniq's table doubles at n = 2^k + 1; pairs mostly distinct, then few pairs with tied counts at hot's cut."""
    rng = np.random.default_rng(n)
    k = torch.from_numpy(rng.integers(-n, n, n)).to(torch.float64)
    k[torch.from_numpy(rng.random(n) < 0.1)] = -0.0
    v = torch.from_numpy(rng.integers(0, 3, n)).to(torch.int32)
    _uniq_case(guarded, k, v, PS[n % len(PS)], (1, n - 1, n))
    # 64 pairs of 16 rows each and one of 17: every cut of hot falls inside a tie
    pairs = np.concatenate([np.repeat(np.arange(64), 16), [5]])
    pairs = pairs[rng.permutation(len(pairs))]
    _uniq_case(guarded, torch.from_numpy(pairs % 8).to(torch.int64), torch.from_numpy(pairs // 8).to(torch.float32),
               3, (1, 2, 10, 64, 65))


def test_uniq_and_hot_at_the_grid_stride_cap(guarded):
    cap = _grid_cap()
    rng = np.random.default_rng(3)
    k = torch.from_numpy(rng.integers(0, 1 << 20, cap + 1)).to(torch.int64)
    v = torch.from_numpy(rng.integers(0, 4, cap + 1)).to(torch.int32)
    _uniq_case(guarded, k, v, 9, (10,))


# ------------------------------------------------------------------------------------------------ percentilesByKey
@pytest.mark.parametrize("L", [b + d for b in (TD_SHORT, TD_CAP) for d in (-1, 0, 1)])
def test_percentiles_by_key_at_segment_lengths(L, guarded):
    """Every (key, split) segment holds L values: the one-thread build up to TD_SHORT, the warp build above, the
    capacity TD_CAP; G keys per split at multiples of the merge's TD_WARPS warps per CTA and next to them."""
    rng = np.random.default_rng(L)
    dc = cc.ctx()
    p = [0, 1, 25, 50, 99.5, 100]
    for G in (TD_WARPS - 1, TD_WARPS, TD_WARPS + 1, 2 * TD_WARPS):
        M = 3
        k = np.concatenate([rng.permutation(np.repeat(np.arange(G), L)) for _ in range(M)]).astype(np.int64) * 7 - 3
        v = rng.standard_normal(len(k)) * 100
        v[rng.random(len(k)) < 0.05] = -0.0
        dk, dv = _cuda(k), _cuda(v.astype(np.float32 if G % 2 else np.float64))
        rows = list(zip(k.tolist(), dv.cpu().tolist()))
        for P in (1, 5):
            want = dc.parallelize(rows, M).percentilesByKey(p, numSplits=P).glom().collect()
            sweep(guarded, lambda: dc.parallelizeColumns(dk, dv, M).percentilesByKey(p, numSplits=P).glom().collect(),
                  lambda got: _rows_equal(got, want))


# ------------------------------------------------------------------------------------------------ sample, fixSkew
MT_DRAWS = MT_N // 2      # random() takes two words: one twist of the state gives MT_N / 2 draws


@pytest.mark.parametrize("n, M", [(0, 3), (10, 8)] + [((b + d) * M, M) for b, M in ((MT_DRAWS, 3), (MT_N, 2))
                                                      for d in (-1, 0, 1)] + [(MT_N * 4 + 1, 5)])
def test_sample_at_twist_boundaries(n, M, guarded):
    """Split lengths 0, MT_DRAWS - 1 .. MT_DRAWS + 1 (one twist) and MT_N - 1 .. MT_N + 1 (two)."""
    rng = np.random.default_rng(n)
    dc = cc.ctx()
    k = torch.from_numpy(rng.integers(-50, 50, n)).to(torch.int32)
    v = torch.from_numpy(rng.standard_normal(n))
    dk, dv = k.cuda(), v.cuda()
    for frac in (0, 0.5, 1, float("nan")):
        col = dc.parallelizeColumns(dk, dv, M)
        masks = _want_masks(col, frac, 12345)

        def run():
            out = dc.parallelizeColumns(dk, dv, M).sample(frac, False, 12345)
            return [tuple(t.cpu().numpy() for t in out.columns(sp)) for sp in out.splits]

        def check(parts):
            assert len(parts) == len(masks)
            for (gk, gv), sp, mask in zip(parts, col.splits, masks):
                assert np.array_equal(gk, k[sp.begin:sp.end].numpy()[mask])
                assert np.array_equal(gv.view(np.int64), v[sp.begin:sp.end].numpy()[mask].view(np.int64))
        sweep(guarded, run, check)
    if n:
        rows = _rows_of(dc, dc.parallelizeColumns(dk, dv, M))
        for rate in (0.5, 1):
            want = rows._skew_thresholds(7, rate)
            sweep(guarded, lambda: dc.parallelizeColumns(dk, dv, M)._skew_thresholds(7, rate),
                  lambda got: _rows_equal(got, want))


# ------------------------------------------------------------------------------------------------ textFile ingest
def _text(rng, nbytes, cut=None):
    """Random ASCII words and whitespace, exactly nbytes long; cut: a 20-byte token straddles that byte."""
    alphabet = np.frombuffer(b"abcdefgh" * 4 + b" \t\n\x0b", dtype=np.uint8)
    data = bytearray(alphabet[rng.integers(0, len(alphabet), nbytes)].tobytes())
    if cut is not None:
        data[cut - 11:cut + 11] = b" " + b"z" * 20 + b" "
    return bytes(data)


@pytest.mark.parametrize("nbytes", [b + d for b in (TK_BYTES, TK_BLOCK) for d in (-1, 0, 1)] + [3 * TK_BLOCK + 5])
def test_tokenize_at_slices_and_chunks(nbytes, guarded):
    rng = np.random.default_rng(nbytes)
    data = _text(rng, nbytes, cut=TK_BLOCK if nbytes > TK_BLOCK + 4 else None)
    want = data.decode("ascii").split()
    d = _cuda(np.frombuffer(data, dtype=np.uint8).copy())

    def run():
        starts, lens, ok = nv.tokenize(d)
        assert ok
        out, off = nv.gather_bytes(d, starts, lens)
        return starts.cpu().numpy(), lens.cpu().numpy(), out.cpu().numpy(), off.cpu().numpy()

    def check(res):
        starts, lens, out, off = res
        assert [data[a:a + b].decode() for a, b in zip(starts.tolist(), lens.tolist())] == want
        raw, o = out.tobytes(), off.tolist()
        assert [raw[o[i]:o[i + 1]].decode() for i in range(len(want))] == want
    sweep(guarded, run, check)


def _fm(x):
    for w in x.strip().split():
        yield (w, 1)


@pytest.mark.parametrize("nbytes", [TK_BLOCK - 1, TK_BLOCK, TK_BLOCK + 1, 2 * TK_BLOCK + 1])
def test_word_count_through_text_file_at_chunk_cuts(nbytes, guarded, tmp_path, monkeypatch):
    from dpark_b200 import textingest
    rng = np.random.default_rng(nbytes)
    data = _text(rng, nbytes, cut=TK_BLOCK if nbytes > TK_BLOCK + 4 else None).replace(b"\x0b", b" ")
    path = str(tmp_path / "in.txt")
    with open(path, "wb") as f:
        f.write(data)
    want = dict(collections.Counter(data.decode("ascii").split()))
    calls = []
    real = textingest.reduce_tokens
    monkeypatch.setattr(textingest, "reduce_tokens", lambda *a, **kw: calls.append(real(*a, **kw)) or calls[-1])
    dc = cc.ctx()
    sweep(guarded, lambda: dc.textFile(path, splitSize=1500).flatMap(_fm).reduceByKey(lambda x, y: x + y, 5)
          .collectAsMap(), lambda got: _rows_equal(dict(sorted(got.items())), dict(sorted(want.items()))))
    assert calls and all(r is not None for r in calls)


# ------------------------------------------------------------------------------------------------ coverage
SWEEPS = [name for name in dir(sys.modules[__name__]) if name.startswith("test_") and name not in (
    "test_every_kernel_output_site_was_reached", "test_a_store_into_a_guard_is_reported",
    "test_a_skipped_output_element_fails_the_oracle")]


def test_every_kernel_output_site_was_reached():
    """Runs last: the sweep above went through every allocation site that holds a kernel's output."""
    if set(SWEEPS) - SWEEPS_RUN:
        pytest.skip("only part of the sweep ran: %s" % sorted(set(SWEEPS) - SWEEPS_RUN))
    missing = [s for s in KERNEL_OUTPUT_SITES if not REACHED[s]]
    assert not missing, "never reached: %s (reached: %s)" % (missing, sorted(REACHED))
