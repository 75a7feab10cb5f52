"""The reference's operator surface on the GPU shuffle, checked against the golden
vectors captured from the real reference (tests/golden/make_golden.py) and the
reference's own shuffle tests (tests/test_rdd.py:246-272).  -m gpu."""
import json
import os
import sys

import pytest

from tests.golden_util import dec, load

pytestmark = pytest.mark.gpu

SC = load("shuffle_cases.json")
FUNCS = {"add": lambda x, y: x + y, "min": lambda x, y: min(x, y), "max": lambda x, y: max(x, y),
         "mul": lambda x, y: x * y, "or": lambda x, y: x | y, "and": lambda x, y: x & y,
         "xor": lambda x, y: x ^ y}


def ctx():
    sys.argv = [sys.argv[0]]
    from dpark_b200 import DparkContext
    return DparkContext("local")


def _canon(parts):
    from tests.golden.make_golden import enc
    return [sorted(([enc(k), enc(v)] for k, v in part), key=json.dumps) for part in parts]


REDUCE_CASES = [c for c in SC["cases"] if c["op"] == "reduceByKey"]


@pytest.mark.parametrize("case", REDUCE_CASES, ids=[c["name"] for c in REDUCE_CASES])
def test_reduce_by_key_matches_reference_per_partition(case):
    """Per-partition multisets equal the reference's glom() output: same keys in
    the same partitions, same combined values (ints bit-exact; float sums within
    1e-9 relative -- the reference's own merge order is nondeterministic)."""
    from dpark_b200 import Aggregator, HashPartitioner
    dc = ctx()
    rows = [(dec(k), dec(v)) for k, v in case["rows"]]
    rdd = dc.parallelize(rows, case["M"])
    f = FUNCS[case["func"]]
    if case["thresholds"] is None:
        got = rdd.reduceByKey(f, case["P"]).glom().collect()
    else:
        got = rdd.combineByKey(Aggregator(lambda x: x, f, f),
                               HashPartitioner(case["P"], thresholds=case["thresholds"])).glom().collect()
    isfloat_sum = rows and isinstance(rows[0][1], float) and case["func"] == "add"
    if not isfloat_sum:
        assert _canon(got) == case["parts"]
    else:
        assert len(got) == len(case["parts"])
        for gp, wp in zip(got, case["parts"]):
            want = {json.dumps(k): dec(v) for k, v in wp}
            from tests.golden.make_golden import enc
            assert len(gp) == len(want)
            for k, v in gp:
                w = want[json.dumps(enc(k))]
                assert abs(v - w) <= 1e-9 * max(1.0, abs(w))


GROUP_CASES = [c for c in SC["cases"] if c["op"] == "groupByKey"]


@pytest.mark.parametrize("case", GROUP_CASES, ids=[c["name"] for c in GROUP_CASES])
def test_group_by_key_matches_reference_ordered_group(case):
    """Per partition: same keys, and for every key the SAME LIST (order included)
    as the reference run with ordered_group=True."""
    dc = ctx()
    rows = [(dec(k), dec(v)) for k, v in case["rows"]]
    got = dc.parallelize(rows, case["M"]).groupByKey(case["P"]).glom().collect()
    assert _canon([[(k, list(v)) for k, v in part] for part in got]) == case["parts"]


def test_reference_test_basic_group_and_lookup():
    """tests/test_rdd.py:246-272 of the reference (groupByKey / lookup / partitionByKey)."""
    dc = ctx()
    d = list(zip([1, 2, 3, 3], list(range(4, 8))))
    nums = dc.makeRDD(d, 2)
    assert nums.groupByKey().mapValue(list).collectAsMap() == {1: [4], 2: [5], 3: [6, 7]}
    assert nums.groupByKey().mapValue(list).lookup(3) == [6, 7]
    assert nums.partitionByKey().lookup(2) == 5
    assert nums.partitionByKey().lookup(4) is None
    assert nums.flatMapValue(lambda x: list(range(x))).count() == 22


def test_radix_sort_is_a_stable_sort_of_key_bits():
    import numpy as np
    import torch
    from dpark_b200 import shuffle
    rng = np.random.default_rng(9)
    for n, lo, hi in ((1, 0, 10), (1000, -50, 50), (300000, 0, 2 ** 31), (300000, -2 ** 63, 2 ** 63 - 1),
                      (200000, 7, 8)):
        k = rng.integers(lo, hi, n, dtype=np.int64)
        v = np.arange(n, dtype=np.int64)
        sk, sv = shuffle.sort_by_key_bits(torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda())
        order = np.argsort(k.view(np.uint64), kind="stable")          # bit order == unsigned order
        assert np.array_equal(sk.cpu().numpy(), k[order])
        assert np.array_equal(sv.cpu().numpy(), v[order])


def test_group_heads_csr():
    import numpy as np
    import torch
    from dpark_b200 import _native as nv
    rng = np.random.default_rng(10)
    k = np.sort(rng.integers(0, 5000, 100003, dtype=np.int64))
    gk, gs, ng = nv.group_heads(torch.from_numpy(k).cuda())
    G = int(ng.item())
    uk, first = np.unique(k, return_index=True)
    assert G == len(uk)
    assert np.array_equal(gk[:G].cpu().numpy(), uk)
    assert np.array_equal(gs[:G + 1].cpu().numpy(), np.concatenate([first, [len(k)]]))


def test_reference_test_basic_reduce():
    """tests/test_rdd.py:246-257 of the reference."""
    dc = ctx()
    d = list(zip([1, 2, 3, 3], list(range(4, 8))))
    nums = dc.makeRDD(d, 2)
    assert nums.reduceByKey(lambda x, y: x + y).collectAsMap() == {1: 4, 2: 5, 3: 13}
    assert nums.reduceByKeyToDriver(lambda x, y: x + y) == {1: 4, 2: 5, 3: 13}
    assert nums.reduceByKey(lambda x, y: x + y).lookup(3) == 13


def test_wc_pipeline_writes_the_files_the_reference_writes(tmp_path):
    """examples/wc.py shape: textFile -> flatMap -> reduceByKey(+, 6) -> map ->
    saveAsTextFile.  The golden fixture holds the reference's output files for
    the same input; file names (= partition ids of str keys) and line sets must match."""
    dc = ctx()
    wc = SC["wc"]
    inp = tmp_path / "in.txt"
    inp.write_text("\n".join(wc["lines"]) + "\n", encoding="utf-8")
    out = tmp_path / "out"

    def fm(x):
        for w in x.strip().split():
            yield (w, 1)

    (dc.textFile(str(inp)).flatMap(fm).reduceByKey(lambda x, y: x + y, numSplits=6)
       .map(lambda x: " ".join(list(map(str, x)))).saveAsTextFile(str(out), overwrite=False))
    got = {fn: sorted(open(os.path.join(str(out), fn), encoding="utf-8").read().splitlines())
           for fn in sorted(os.listdir(str(out)))}
    assert got == wc["files"]


def test_columnar_rdd_reduce_large():
    import numpy as np
    from oracle import oracle as orc
    dc = ctx()
    rng = np.random.default_rng(5)
    n, P = 3_000_000, 8
    k = rng.integers(0, 2 ** 20, n, dtype=np.int64)
    v = rng.integers(0, 2 ** 16, n, dtype=np.int64)
    sh = dc.parallelizeColumns(k, v, 8).reduceByKey(lambda a, b: a + b, P)
    want = orc.reduce_by_key(np.array_split(k, 8), np.array_split(v, 8), P, "sum")
    for p in range(P):
        gk, gv = sh.columns(sh.splits[p])
        gk, gv = np.array(gk), np.array(gv)
        o1, o2 = np.argsort(gk), np.argsort(want[p][0])
        assert np.array_equal(gk[o1], want[p][0][o2]) and np.array_equal(gv[o1], want[p][1][o2])


def test_unsupported_things_fail_loudly():
    dc = ctx()
    with pytest.raises(NotImplementedError):
        dc.parallelize([(1, 1)], 1).reduceByKey(lambda x, y: x - y)
    from dpark_b200 import DparkUserFatalError
    with pytest.raises(DparkUserFatalError):
        dc.parallelize([(1, 1), 5], 1).reduceByKey(lambda x, y: x + y).collect()
    with pytest.raises(TypeError):
        dc.parallelize([(True, 1)], 1).reduceByKey(lambda x, y: x + y).collect()


def test_fix_skew_layout_of_the_reference_test():
    """tests/test_rdd.py:259-266 of the reference: keys 0..9 once and key 10 five times in 10 input
    partitions, groupByKey(3, fixSkew=1) -> the t-digest thresholds [5, 10] put {0..4}, {5..9}, {10}
    into the three partitions (golden glom() output captured from the reference)."""
    dc = ctx()
    dsk = list(zip(range(10), range(10))) + [(10, 10)] * 5
    rdd = dc.makeRDD(dsk, 10).groupByKey(3, fixSkew=1)
    assert rdd.partitioner.thresholds == [5, 10]
    out = rdd.map(lambda kv: (kv[0], list(kv[1]))).glom().collect()
    assert [sorted([[k, sorted(v)] for k, v in part]) for part in out] == SC["fix_skew_test_basic"]


def test_fix_skew_balances_a_hot_hash_range_and_keeps_results():
    """reduceByKey(fixSkew=rate): thresholds come from a seeded sample (random.Random(12345 + split), as the
    reference's SampleRDD), partitions are balanced by hash range, per-key results are unchanged."""
    import random
    dc = ctx()
    rnd = random.Random(3)
    rows = [(rnd.randrange(0, 1000) if rnd.random() < 0.7 else rnd.randrange(-10 ** 12, 10 ** 12), 1)
            for _ in range(20000)]
    plain = dict(dc.parallelize(rows, 5).reduceByKey(lambda a, b: a + b, 4).collect())
    skew = dc.parallelize(rows, 5).reduceByKey(lambda a, b: a + b, 4, fixSkew=0.3)
    thr = skew.partitioner.thresholds
    assert thr is not None and thr == sorted(thr) and len(thr) == len(skew.splits) - 1
    parts = skew.glom().collect()
    assert dict(kv for part in parts for kv in part) == plain
    import bisect
    for i, part in enumerate(parts):                  # every key sits where bisect over the thresholds says
        assert all(bisect.bisect(thr, k if k != -1 else -2) == i for k, _ in part)
    sizes = [sum(v for _, v in part) for part in parts]
    assert max(sizes) < 0.5 * len(rows)               # hash % 4 would not help here either; ranges are balanced
    # percentiles() itself, against exact order statistics of the same numbers
    p50, p90 = dc.parallelize(list(range(1000)), 4).percentiles([50, 90])
    assert abs(p50 - 499.5) < 5 and abs(p90 - 899.5) < 5


# ---- cogroup / join (SURVEY.md §8 f1): the same golden cases as tests/test_cogroup_host.py, real engine
from tests import cogroup_common as _cc  # noqa: E402


@pytest.mark.parametrize("case", _cc.COGROUP_CASES, ids=[c["name"] for c in _cc.COGROUP_CASES])
def test_cogroup_matches_reference_on_the_gpu(case):
    _cc.check_cogroup(case)


@pytest.mark.parametrize("case", _cc.JOIN_CASES, ids=[c["name"] for c in _cc.JOIN_CASES])
def test_joins_match_reference_on_the_gpu(case):
    _cc.check_join(case)


def test_tuple_and_none_keys_reduce_and_group_like_python_and_partition_like_the_reference():
    """a1 for tuple / None keys (dpark/portable_hash.pyx:3-15, 53-54): the device hashes decide the partition, the
    canonical-bytes identity decides equality.  Layout is checked against the oracle's getPartition (pinned to the
    reference's golden tuple vectors in test_oracle_golden.py), contents against plain Python dicts."""
    import random
    from oracle import oracle as orc
    dc = ctx()
    rnd = random.Random(11)
    P = 5
    for make in (lambda: (rnd.randint(-3, 3), "k%d" % rnd.randint(0, 4)),
                 lambda: ("a", (rnd.randint(0, 2), float(rnd.randint(0, 2)))),
                 lambda: (rnd.randint(0, 6), None, b"x" * rnd.randint(0, 2)),
                 lambda: ()):
        rows = [(make(), rnd.randint(-50, 50)) for _ in range(3000)]
        want = {}
        for k, v in rows:
            want[k] = want.get(k, 0) + v
        got = dc.parallelize(rows, 4).reduceByKey(lambda x, y: x + y, P).glom().collect()
        assert len(got) == P
        seen = {}
        for p, part in enumerate(got):
            for k, v in part:
                assert orc.get_partition(k, P) == p, (k, p)
                assert k not in seen
                seen[k] = v
        assert seen == want
        groups = dict(dc.parallelize([(k, i) for i, (k, _) in enumerate(rows)], 4).groupByKey(P).collect())
        wantg = {}
        for i, (k, _) in enumerate(rows):
            wantg.setdefault(k, []).append(i)
        assert {k: list(v) for k, v in groups.items()} == wantg        # values in (map split, position) order
    nones = dc.parallelize([(None, i) for i in range(100)], 3).reduceByKey(lambda x, y: x + y, 4).glom().collect()
    assert [len(p) for p in nones] == [0, 1, 0, 0] and nones[1] == [(None, 4950)]     # portable_hash(None) % 4 == 1
