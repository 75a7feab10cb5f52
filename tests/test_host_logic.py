"""CPU-only tests of the host side: combiner recognition, columnar ingest, the
operator surface's split semantics, the C-ABI library's exports, and the
__host__ __device__ hash/partition arithmetic run on the CPU (hostcheck)."""
import ctypes as C
import operator
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as orc
from tests.golden_util import dec, load

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ----------------------------------------------------------------- trace
def test_recognize_binary_ops():
    from dpark_b200 import trace
    cases = [
        (lambda x, y: x + y, "sum"), (lambda a, b: b + a, "sum"), (operator.add, "sum"),
        (lambda x, y: x * y, "prod"), (min, "min"), (max, "max"),
        (lambda x, y: min(x, y), "min"), (lambda x, y: max(y, x), "max"),
        (lambda x, y: x if x < y else y, "min"), (lambda x, y: y if y >= x else x, "max"),
        (lambda x, y: x | y, "or"), (lambda x, y: x & y, "and"), (lambda x, y: x ^ y, "xor"),
    ]
    for f, want in cases:
        assert trace.recognize_binary(f) == want


@pytest.mark.parametrize("bad", [
    lambda x, y: x - y, lambda x, y: x + y + 1, lambda x, y: x, lambda x, y: y,
    lambda x, y: (x[0] + y[0], x[1] + y[1]), lambda x, y: x + 2 * y, lambda x, y: str(x) + str(y),
    lambda x, y: x if x < y else x,
])
def test_unrecognised_combiners_raise_no_cpu_fallback(bad):
    from dpark_b200 import trace
    with pytest.raises(NotImplementedError):
        trace.recognize_binary(bad)


def test_recognize_aggregator_kinds():
    from dpark_b200 import trace
    from dpark_b200.dependency import AddAggregator, Aggregator, GroupByAggregator, MergeAggregator
    assert trace.recognize_aggregator(GroupByAggregator()) == ("group", None)
    assert trace.recognize_aggregator(MergeAggregator()) == ("group", None)
    assert trace.recognize_aggregator(AddAggregator()) == ("reduce", "sum")
    f = lambda a, b: a + b  # noqa: E731
    assert trace.recognize_aggregator(Aggregator(lambda x: x, f, f)) == ("reduce", "sum")
    with pytest.raises(NotImplementedError):
        trace.recognize_aggregator(Aggregator(lambda x: [x], f, f))
    with pytest.raises(NotImplementedError):
        trace.recognize_aggregator(Aggregator(lambda x: x, f, lambda a, b: a * b))


# -------------------------------------------------------------- columnar
def test_ingest_pairs_kinds_and_errors():
    from dpark_b200 import columnar
    from dpark_b200.errors import DparkUserFatalError
    c = columnar.ingest_pairs([(1, 2), (-5, 7)])
    assert c.key_kind == "i64" and c.val_kind == "i64" and c.keys.tolist() == [1, -5]
    c = columnar.ingest_pairs([("ab", 1.5), ("你好", 2.0), ("", 0.0)])
    assert c.key_kind == "str" and c.val_kind == "f64"
    assert columnar.decode_keys("str", c.keys, c.key_offsets) == ["ab", "你好", ""]
    c = columnar.ingest_pairs([(b"\xff\x00", 1)])
    assert c.key_kind == "bytes" and columnar.decode_keys("bytes", c.keys, c.key_offsets) == [b"\xff\x00"]
    c = columnar.ingest_pairs([(1, object()), (2, "x")], numeric_values=False)
    assert c.val_kind == "obj" and c.vals.tolist() == [0, 1] and len(c.objs) == 2
    with pytest.raises(DparkUserFatalError):
        columnar.ingest_pairs([(1, 2), 3])                    # dpark/task.py:216-219
    with pytest.raises(DparkUserFatalError):
        columnar.ingest_pairs([(1, 2, 3)])
    with pytest.raises(TypeError, match="unhashable by portable_hash"):
        columnar.ingest_pairs([(True, 1)])                    # bool is not int for the reference
    with pytest.raises(TypeError, match="unhashable by portable_hash"):
        columnar.ingest_pairs([([1], 1)])
    with pytest.raises(TypeError):
        columnar.ingest_pairs([(1, 1), ("a", 1)])
    with pytest.raises(TypeError):
        columnar.ingest_pairs([(2 ** 70, 1)])
    with pytest.raises(TypeError):
        columnar.ingest_pairs([(1, 1), (2, 2.5)])


# ------------------------------------------------------------ rdd surface
def _ctx():
    sys.argv = [sys.argv[0]]
    from dpark_b200 import DparkContext
    return DparkContext("local")


def test_parallelize_split_sizes_match_reference():
    dc = _ctx()
    for case in load("shuffle_cases.json")["cases"]:
        rows = case["rows"]
        got = [len(x) for x in dc.parallelize(rows, case["M"]).glom().collect()]
        assert got == case["split_sizes"], case["name"]


def test_narrow_ops_and_actions():
    dc = _ctx()
    r = dc.parallelize(range(10), 3)
    assert r.map(lambda x: x * 2).filter(lambda x: x % 3 == 0).collect() == [0, 6, 12, 18]
    assert r.flatMap(lambda x: [x] * (x % 3)).count() == sum(x % 3 for x in range(10))
    assert r.reduce(lambda a, b: a + b) == 45
    assert r.take(4) == [0, 1, 2, 3] and r.first() == 0
    kv = dc.makeRDD([(1, 2), (3, 4)], 2)
    assert kv.mapValue(lambda v: v + 1).collectAsMap() == {1: 3, 3: 5}
    assert kv.flatMapValue(lambda v: range(v)).count() == 6
    assert dc.union([r, r]).count() == 20 and len(dc.union([r, r])) == 6
    assert dc.defaultParallelism == 2 and dc.defaultMinSplits == 2


def test_text_file_rdd_splits_own_the_lines_that_start_in_them(tmp_path):
    dc = _ctx()
    from dpark_b200.rdd import TextFileRDD
    lines = ["line %d %s" % (i, "x" * (i % 17)) for i in range(500)] + ["", "你好 world", "last-without-newline"]
    p = tmp_path / "in.txt"
    p.write_bytes("\n".join(lines).encode("utf-8"))
    for split_size in (7, 64, 1000, 10 ** 6):
        rdd = TextFileRDD(dc, str(p), splitSize=split_size)
        assert rdd.collect() == lines, split_size
    assert dc.textFile(str(p), numSplits=4).collect() == lines


def test_save_as_text_file_layout(tmp_path):
    dc = _ctx()
    out = tmp_path / "out"
    paths = dc.parallelize(["a", "b", "c"], 3).filter(lambda x: x != "b").saveAsTextFile(str(out))
    assert sorted(os.path.basename(p) for p in paths) == ["0000", "0002"]   # empty partition: no file
    assert (out / "0000").read_text() == "a\n"


def test_shuffled_rdd_plan_is_checked_at_declaration():
    dc = _ctx()
    kv = dc.parallelize([(1, 1)], 1)
    with pytest.raises(NotImplementedError):
        kv.reduceByKey(lambda x, y: x - y)
    sh = kv.reduceByKey(lambda x, y: x + y, 6)
    assert len(sh) == 6 and sh.partitioner.numPartitions == 6 and sh.op == "sum"
    assert kv.groupByKey(3).rddconf.is_groupby
    assert len(kv.reduceByKey(lambda x, y: x + y)) == 1      # min(defaultMinSplits, len(self))


def test_hash_partitioner_record():
    from dpark_b200 import HashPartitioner
    assert HashPartitioner(4) == HashPartitioner(4) and HashPartitioner(4) != HashPartitioner(5)
    assert HashPartitioner(3, [10, 100]) != HashPartitioner(3)
    with pytest.raises(AssertionError):
        HashPartitioner(3, [1])
    assert HashPartitioner(0).numPartitions == 1


def test_shuffle_without_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    dc = _ctx()
    from dpark_b200 import _native
    with pytest.raises(_native.NativeError):
        dc.parallelize([(1, 1), (2, 2)], 2).reduceByKey(lambda x, y: x + y).collect()


# ------------------------------------------------------------- C ABI library
def test_library_exports_every_symbol_the_header_declares():
    from dpark_b200 import _native
    hdr = open(os.path.join(ROOT, "include", "dpark_b200.h")).read()
    declared = set(re.findall(r"\b(dpk_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations found"
    L = _native.lib()
    missing = [n for n in sorted(declared) if not hasattr(L, n)]
    assert not missing, missing
    assert declared == set(_native.EXPORTS)
    assert L.dpk_abi_version() == 1
    assert L.dpk_partition_workspace_bytes(0, 8) > 0


def test_product_never_imports_the_oracle():
    bad = []
    for dirpath, _, names in os.walk(os.path.join(ROOT, "dpark_b200")):
        for n in names:
            if n.endswith((".py", ".cu", ".cuh", ".h")):
                if re.search(r"^\s*(from|import)\s+oracle|dpk_oracle|orc_", open(os.path.join(dirpath, n)).read(), re.M):
                    bad.append(n)
    assert not bad, bad


# --------------------------------------------------- hostcheck (HD functions)
def _hostcheck():
    path = os.path.join(ROOT, "tests", "_hostcheck.so")
    if not os.path.exists(path):
        subprocess.call([sys.executable, "-c", "import __graft_entry__ as g; g.build()"], cwd=ROOT)
    if not os.path.exists(path):
        pytest.skip("hostcheck not built")
    return C.CDLL(path)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def test_device_hash_functions_on_cpu_match_oracle():
    L = _hostcheck()
    rng = np.random.default_rng(1)
    xs = rng.integers(-2 ** 63, 2 ** 63 - 1, 200000, dtype=np.int64, endpoint=True)
    xs[:8] = [0, -1, 2 ** 61 - 1, 2 ** 61, -(2 ** 61 - 1), 2 ** 63 - 1, -2 ** 63, 4 * (2 ** 61 - 1)]
    o = np.empty_like(xs)
    L.hc_hash_i64(_p(xs), C.c_int64(len(xs)), _p(o))
    assert np.array_equal(o, orc.hash_vec(xs))
    fs = np.concatenate([rng.standard_normal(50000) * 10.0 ** rng.integers(-300, 300, 50000),
                         np.array([0.0, -0.0, np.inf, -np.inf, 5e-324, 1.5, 2.0 ** 61, 2.0 ** 61 - 1])])
    o = np.empty(len(fs), dtype=np.int64)
    L.hc_hash_f64(_p(fs), C.c_int64(len(fs)), _p(o))
    assert np.array_equal(o, orc.hash_vec(fs))
    hv = load("hash_vectors.json")
    for tag, mode, encf in (("b", 0, lambda b: b), ("s", 1, lambda s: s.encode("utf-8", "surrogatepass"))):
        ks = [(dec(r["key"]), r["hash"]) for r in hv["rows"] if isinstance(r["key"], dict) and tag in r["key"]]
        blobs = [encf(k) for k, _ in ks]
        offs = np.zeros(len(blobs) + 1, dtype=np.int64)
        offs[1:] = np.cumsum([len(b) for b in blobs])
        data = np.frombuffer(b"".join(blobs), dtype=np.uint8).copy()
        o = np.empty(len(blobs), dtype=np.int64)
        L.hc_hash_bytes(_p(data), _p(offs), C.c_int64(len(blobs)), mode, _p(o))
        assert o.tolist() == [h for _, h in ks]


@pytest.mark.parametrize("P", [1, 2, 3, 5, 6, 7, 8, 12, 63, 64, 65, 100, 1000, 1023, 1025, 4095, 4096,
                               2 ** 31 - 1, 2 ** 30 + 3])
def test_device_floor_mod_on_cpu_matches_oracle(P):
    L = _hostcheck()
    rng = np.random.default_rng(P)
    h = rng.integers(-2 ** 63, 2 ** 63 - 1, 100000, dtype=np.int64, endpoint=True)
    h[:6] = [0, -1, -2, 2 ** 61 - 2, -(2 ** 61 - 2), 2 ** 63 - 1]
    pid = np.empty(len(h), dtype=np.int32)
    assert L.hc_partition(_p(h), C.c_int64(len(h)), C.c_int32(P), None, 0, _p(pid)) == 0
    assert np.array_equal(pid, orc.partition_vec(h, P))


def test_device_bisect_and_sub_buckets_on_cpu():
    L = _hostcheck()
    rng = np.random.default_rng(5)
    h = rng.integers(-2 ** 63, 2 ** 63 - 1, 50000, dtype=np.int64, endpoint=True)
    thr = np.sort(rng.integers(-2 ** 62, 2 ** 62, 15, dtype=np.int64))
    pid = np.empty(len(h), dtype=np.int32)
    assert L.hc_partition(_p(h), C.c_int64(len(h)), C.c_int32(16), _p(thr), 15, _p(pid)) == 0
    assert np.array_equal(pid, orc.partition_vec(h, 16, thr))
    for P, sb in ((8, 5), (3, 2), (1, 7)):
        b = np.empty(len(h), dtype=np.int32)
        assert L.hc_bucket(_p(h), C.c_int64(len(h)), C.c_int32(P), C.c_int32(sb), _p(b)) == 0
        assert np.array_equal(b >> sb, orc.partition_vec(h, P))     # refinement of the reference partition
        assert b.min() >= 0 and b.max() < (P << sb)
        cnt = np.bincount(b & ((1 << sb) - 1), minlength=1 << sb)
        assert cnt.min() > 0.5 * len(h) / (1 << sb)                 # sub-bucket bits are well mixed


@pytest.mark.parametrize("G,P,sb", [(2, 8, 0), (3, 5, 1), (8, 5, 2), (4, 1, 3), (8, 64, 0)])
def test_push_plan_reproduces_the_alltoallv_layout(G, P, sb):
    """peer.push_plan (segment table of the block-push exchange) against a direct construction of
    what shuffle.exchange delivers: source-rank-major, bucket-major inside, empty owners included."""
    import torch
    from dpark_b200 import peer, shuffle
    rng = np.random.default_rng(G * 100 + P)
    F = P << sb
    counts = rng.integers(0, 7, (G, F))
    counts[rng.random((G, F)) < 0.2] = 0
    blocks = [b << sb for b in shuffle.owner_blocks(P, G)]
    # rows tagged (source, bucket, position) so that any misplacement shows
    bufs = [np.concatenate([np.array([s * 10 ** 6 + b * 1000 + i for i in range(counts[s, b])], dtype=np.int64)
                            for b in range(F)] + [np.zeros(0, np.int64)]) for s in range(G)]
    want = [np.concatenate([bufs[s][counts[s, :blocks[d]].sum():counts[s, :blocks[d + 1]].sum()] for s in range(G)])
            for d in range(G)]
    got = [np.full(len(want[d]), -1, dtype=np.int64) for d in range(G)]
    ac = torch.from_numpy(counts.astype(np.int64))
    for s in range(G):
        send_first, dst_first, rows, recv_total = peer.push_plan(ac, blocks, s)
        assert recv_total.tolist() == [len(w) for w in want]
        for d in range(G):
            a, b, c = int(send_first[d]), int(dst_first[d]), int(rows[d])
            got[d][b:b + c] = bufs[s][a:a + c]
    for d in range(G):
        assert np.array_equal(got[d], want[d])


def test_sample_rdd_draws_like_the_reference():
    """SampleRDD (dpark/rdd.py:1379-1397): random.Random(seed + split.index), one draw per row, keep if <= frac;
    with replacement: ceil(len * frac) choices.  Restated here with the stdlib generator the reference uses."""
    import random
    import sys
    sys.argv = [sys.argv[0]]
    from dpark_b200 import DparkContext
    dc = DparkContext("local")
    rows = list(range(1000))
    rdd = dc.parallelize(rows, 4)
    parts = rdd.glom().collect()
    got = rdd.sample(0.3).glom().collect()
    for i, part in enumerate(parts):
        rd = random.Random(12345 + i)
        assert got[i] == [x for x in part if rd.random() <= 0.3]
    got = rdd.sample(0.1, True, 7).glom().collect()
    for i, part in enumerate(parts):
        rd = random.Random(7 + i)
        assert got[i] == [rd.choice(part) for _ in range(int(np.ceil(len(part) * 0.1)))]
    # percentiles(): host-side digest over the partitions (no shuffle involved)
    p = rdd.percentiles([0, 50, 100])
    assert p[0] == 0.0 and p[2] == 999.0 and abs(p[1] - 499.5) < 5
    with pytest.raises(ValueError):
        rdd.percentiles([50], sampleRate=0)


def test_bench_reference_arm_prints_one_contract_line():
    """`bench.py --impl reference` (the CPU arm timed next to ours): exactly one JSON line on stdout
    with the expected keys, measured on the UNMODIFIED reference when oracle/_ref/baseline was built (oracle/build_reference.py)
    and on the oracle's CPython port otherwise (bounded sample so this stays quick)."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1",
                          "--warmup", "0", "--cpu-sample-rows", "8000"], capture_output=True, text=True, timeout=300,
                         cwd=root)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    b = json.loads(lines[0])
    assert b["impl"] == "reference" and b["unit"] == "rows/s" and b["higher_is_better"] is True
    assert b["metric"] == "shuffled rows/sec (reduceByKey end-to-end)"
    assert b["value"] > 0 and b["n_gpus"] == 1 and b["scaling"] == "weak" and b["dtype"] == "int64"
    assert b["cpu_baseline"]["kind"] in ("reference", "port") and b["cpu_baseline"]["cores"] >= 1
    if b["cpu_baseline"]["kind"] == "reference":     # the reference's own compiled extension was loaded, nothing of ours
        assert any("_ref/baseline/dpark/portable_hash" in x for x in b["cpu_baseline"]["native_so_loaded"])
    assert b["cpu_baseline"]["value"] == b["value"]
    assert b["e2e"] == {"value": b["value"], "unit": "rows/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in b["config"]


def test_only_straight_line_list_collectors_are_recognised_as_group_by():
    """ADVICE r1: an aggregator that merely LOOKS like append/concat on small probes (bounded lists, de-duplication)
    must not be run as an unbounded groupByKey; only straight-line collectors and the known classes are."""
    from dpark_b200 import bagel, trace
    from dpark_b200.dependency import Aggregator

    def mv(c, v):
        c.append(v)
        return c

    def mc(a, b):
        a.extend(b)
        return a
    assert trace.recognize_aggregator(Aggregator(lambda v: [v], lambda c, v: c + [v], lambda a, b: a + b)) == ("group", None)
    assert trace.recognize_aggregator(Aggregator(lambda v: [v], mv, mc)) == ("group", None)
    assert trace.recognize_aggregator(bagel.DefaultListCombiner()) == ("group", None)
    bounded = Aggregator(lambda v: [v], lambda c, v: c + [v] if len(c) < 5 else c, lambda a, b: (a + b)[:5])
    dedup = Aggregator(lambda v: [v], lambda c, v: c if v in c else c + [v], lambda a, b: a + [x for x in b if x not in a])
    srt = Aggregator(lambda v: [v], lambda c, v: sorted(c + [v]), lambda a, b: sorted(a + b))
    for agg in (bounded, dedup, srt):
        with pytest.raises(NotImplementedError):
            trace.recognize_aggregator(agg)


def test_tuple_hash_device_function_matches_the_reference_vectors():
    """a1 for tuple keys (dpark/portable_hash.pyx:3-15): the __host__ __device__ tuple_hash, fed with the item hashes
    of the reference's own golden vectors, must reproduce the golden tuple hashes (incl. the empty tuple, nested
    tuples and None items)."""
    L = _hostcheck()
    hv = load("hash_vectors.json")
    rows = [(dec(r["key"]), r["hash"]) for r in hv["rows"] if isinstance(r["key"], dict) and "tu" in r["key"]]
    assert len(rows) >= 5

    def item_hash(x):
        return orc.portable_hash(x)                 # leaves are pinned separately; here only the combination is tested
    for key, want in rows:
        items = np.array([item_hash(x) for x in key], dtype=np.int64).reshape(len(key), 1)
        o = np.empty(1, dtype=np.int64)
        L.hc_hash_tuple(_p(np.ascontiguousarray(items)), C.c_int64(1), C.c_int32(len(key)), _p(o))
        assert int(o[0]) == want, key


def test_tuple_and_none_keys_become_identity_bytes_with_one_shape():
    from dpark_b200 import columnar
    c = columnar.ingest_pairs([((1, "a"), 1), ((1, "b"), 2), ((1, "a"), 3)])
    assert c.key_kind == "tuple" and c.key_objs == [(1, "a"), (1, "b"), (1, "a")]
    blobs = [bytes(c.keys[c.key_offsets[i]:c.key_offsets[i + 1]]) for i in range(3)]
    assert blobs[0] == blobs[2] != blobs[1]
    c = columnar.ingest_pairs([(None, 1), (None, 2)])
    assert c.key_kind == "tuple" and c.key_offsets.tolist() == [0, 0, 0]
    with pytest.raises(TypeError):
        columnar.ingest_pairs([((1, 2), 1), ((1, 2.0), 2)])          # same value in Python, different shape here
    with pytest.raises(TypeError):
        columnar.ingest_pairs([((1, 2), 1), ((1, 2, 3), 2)])
    with pytest.raises(TypeError):
        columnar.ingest_pairs([(None, 1), (3, 2)])


def test_int_sums_that_could_wrap_are_refused_and_float_zero_keys_are_canonical():
    """ADVICE r1 (low): int64 accumulation must not wrap silently where the reference's big ints would not; -0.0 and
    0.0 are one key on every path (the group-by path used the raw bits)."""
    from dpark_b200 import columnar, engine
    big = columnar.ingest_pairs([(1, 2 ** 62), (2, 2 ** 62), (1, 5)])
    with pytest.raises(OverflowError):
        engine._check_int_sum_range([big], {columnar.VAL_I64}, "sum")
    engine._check_int_sum_range([big], {columnar.VAL_I64}, "max")          # only sums can wrap
    ok = columnar.ingest_pairs([(1, 2 ** 40), (2, -2 ** 40)])
    engine._check_int_sum_range([ok], {columnar.VAL_I64}, "sum")
    c = columnar.ingest_pairs([(-0.0, 1), (0.0, 2)])
    assert np.signbit(c.keys).tolist() == [False, False]


def test_merge_part_results_concatenates_partitions_in_order():
    """peer.merge_part_results: the per-part results of a pipelined step as one reduce_side-shaped result."""
    import torch
    from dpark_b200 import peer
    # part A: partitions 4,5 with 3 + 1 distinct rows (received-row offsets 0, 5, 7); part B: partitions 6,7
    a = (torch.tensor([10, 11, 12, 0, 0, 20, 0]), torch.tensor([1, 2, 3, 0, 0, 4, 0]),
         torch.tensor([0, 5, 7]), torch.tensor([3, 1]), 4, 2)
    b = (torch.tensor([30, 0, 40, 41]), torch.tensor([5, 0, 6, 7]), torch.tensor([0, 2, 4]), torch.tensor([1, 2]), 6, 2)
    k, v, po, cnt = peer.merge_part_results([a, b])
    assert po.tolist() == [0, 5, 7, 9, 11] and cnt.tolist() == [3, 1, 1, 2]
    got = [(k[po[j]:po[j] + cnt[j]].tolist(), v[po[j]:po[j] + cnt[j]].tolist()) for j in range(4)]
    assert got == [([10, 11, 12], [1, 2, 3]), ([20], [4]), ([30], [5]), ([40, 41], [6, 7])]


# ------------------------------------------- oracle float keys, path coverage of the parity shapes
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_oracle_keys_float_columns_by_value(dtype):
    """orc.reduce_by_key / group_by_key key float columns by their canonical bits: 1.25 and 1.75 stay two keys,
    -0.0 and 0.0 are one (spelled 0.0), infinities, subnormals and 2.0**61 (whose hash equals that of 1.0) are keys
    of their own -- as in the reference's dicts (orc.py_reduce_by_key)."""
    rng = np.random.default_rng(11)
    pool = np.array([1.25, 1.75, -1.25, 0.0, -0.0, np.inf, -np.inf, 5e-324, -5e-324, 1e-310, 2.0 ** 61, 1.0, 3.0,
                     2.0 ** -149, 1e-40, -7.5], dtype=np.float64).astype(dtype)
    k = pool[rng.integers(0, len(pool), 600)]
    v = rng.integers(-1000, 1000, len(k), dtype=np.int64)
    ks, vs = np.array_split(k, 3), np.array_split(v, 3)
    P = 3
    want = orc.py_reduce_by_key([list(zip((float(x) for x in a), (int(y) for y in b))) for a, b in zip(ks, vs)],
                                P, operator.add)
    got = orc.reduce_by_key(ks, vs, P, "sum")
    groups = orc.group_by_key(ks, [np.arange(len(a), dtype=np.int64) + 1000 * s for s, a in enumerate(ks)], P)
    for p in range(P):
        gk, gv = got[p]
        assert gk.dtype == dtype
        assert not np.signbit(gk[gk == 0]).any()
        assert dict(zip((float(x) for x in gk), gv.tolist())) == want[p]
        assert len(gk) == len(want[p])
        wk, wo, _ = groups[p]
        assert wk.dtype == dtype and sorted(float(x) for x in wk) == sorted(want[p])
        assert [int(n) for n in np.diff(wo)] == [sum(float(x) == float(key) for x in k
                                                     if orc.get_partition(float(x), P) == p) for key in wk]


def test_every_set_option_switch_is_in_a_variant_table():
    """Every switch dpk_set_option accepts has its default in tests/shuffle_cases.DEFAULT_OPTIONS, and every one
    that selects a kernel variant is run against the oracle by a variant table (agg_timing only prints, copy_sms is
    a parameter of copy_segments)."""
    from tests import shuffle_cases as sc
    src = open(os.path.join(ROOT, "dpark_b200", "csrc", "dpk_combine.cu")).read()
    accepted = set(re.findall(r'strcmp\(name, "(\w+)"\)', src))
    assert accepted == set(sc.DEFAULT_OPTIONS)
    header = open(os.path.join(ROOT, "include", "dpark_b200.h")).read()
    assert all('"%s"' % name in header for name in accepted)
    tables = sc.REDUCE_VARIANTS + sc.MULTISPLIT_VARIANTS + sc.POINTER_VARIANTS + sc.COPY_VARIANTS
    run = {name for opts in tables for name in opts}
    assert accepted - {"agg_timing", "copy_sms"} <= run


def _fine_buckets(L, keys, P, sb, n_total):
    """Fine bucket of every key as dpk_combine's second-level split numbers it, for a combine over n_total rows."""
    sb = 0 if sb is None else sb
    sb2 = L.hc_choose_sb2(C.c_int64(n_total), C.c_int32(P << sb), C.c_int32(2048))
    h = orc.hash_vec(keys)
    fb = np.empty(len(h), dtype=np.int32)
    assert L.hc_fine_bucket(_p(h), C.c_int64(len(h)), C.c_int32(P), C.c_int32(sb), C.c_int32(sb2), _p(fb)) == 0
    return fb, sb2


def test_reduce_parity_shapes_reach_their_kernel_paths():
    """The reduce-side parity shapes (tests/shuffle_cases.reduce_shape) really hold what they are named for under the
    current split tuning: `distinct_overflow` has a fine bucket with more than 2 x 2048 distinct keys (>= 4
    hash-disjoint passes of k_smem_aggregate2, >= 2 of the round-1 kernel with its 3584-key limit), `hot_keys` a fine
    bucket of more than one 2048-row window with few distinct keys, and `distinct` fits one window everywhere."""
    from tests import shuffle_cases as sc
    from dpark_b200 import shuffle
    L = _hostcheck()
    L.hc_choose_sb2.restype = C.c_int
    for target in (64, 2048, 3584):
        assert L.hc_choose_sb2(C.c_int64(6_000_000), C.c_int32(1), C.c_int32(target)) == 10    # capped at 1024-way
    assert L.hc_choose_sb2(C.c_int64(2048), C.c_int32(1), C.c_int32(2048)) == 0
    assert L.hc_choose_sb2(C.c_int64(4096), C.c_int32(1), C.c_int32(2048)) == 1
    assert L.hc_choose_sb2(C.c_int64(4096 * 2), C.c_int32(2), C.c_int32(2048)) == 1

    [(k, _)], P, sb = sc.reduce_shape("distinct_overflow")
    fb, sb2 = _fine_buckets(L, k, P, sb, len(k))
    distinct = np.bincount(fb, minlength=(P << sb) << sb2)          # every key is distinct
    assert len(np.unique(k)) == len(k)
    assert distinct.max() > 2 * sc.AG2_CAP and distinct.max() > sc.AG_LIMIT

    [(k, _)], P, sb = sc.reduce_shape("hot_keys")
    fb, sb2 = _fine_buckets(L, k, P, sb, len(k))
    rows = np.bincount(fb)
    pairs = np.unique(np.stack([fb.astype(np.int64), k]), axis=1)
    nd = np.bincount(pairs[0], minlength=len(rows))
    big = rows > sc.AG2_CAP
    assert big.any() and nd[big].max() < sc.AG2_CAP // 4

    [(k, _)], P, sb = sc.reduce_shape("distinct")
    sb = shuffle.choose_sub_bits(len(k), P)
    fb, sb2 = _fine_buckets(L, k, P, sb, len(k))
    assert np.bincount(fb).max() <= sc.AG2_CAP
