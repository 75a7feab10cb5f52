#!/usr/bin/env python
"""Golden vectors for top, uniq and hot FROM THE REAL REFERENCE (dpark/rdd.py:383-398); same out-of-tree build as
make_golden.py.

    python tests/golden/make_uniq_top_hot_golden.py     # writes tests/golden/uniq_top_hot_cases.json

The inputs of the reference's own tests (tests/test_rdd.py:441-448, scalar rows) plus seeded (k, v) pair rows with many
ties, both signed zeros and int / float column mixes, over several split counts M and partition counts P.  top lists are
recorded exactly; uniq as per-partition sorted sets and hot as its counts plus, per count, the set of all elements with
that count (hot(n) over every element), because the reference's fetch order is not fixed.  uniq runs the body of the
reference's uniq (see generate())."""
import json
import logging
import os
import random
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import bootstrap, build_reference, enc  # noqa: E402

KEYS = {"none": None, "first": lambda x: x[0], "second": lambda x: x[1], "neg": lambda x: -x}


def _pairs(rnd, n, kinds):
    def one(kind, lo, hi):
        x = rnd.randrange(lo, hi)
        if kind == "i":
            return x
        r = rnd.random()
        return -0.0 if r < 0.1 else (0.0 if r < 0.2 else x * 0.5)
    return [(one(kinds[0], -6, 6), one(kinds[1], -3, 3)) for _ in range(n)]


def generate():
    from dpark import DparkContext
    logging.getLogger("dpark").setLevel(logging.ERROR)
    dc = DparkContext("local")
    dc.init()
    rnd = random.Random(23)
    cases = []

    def case(name, rows, M, P, tops, hots):
        rdd = dc.makeRDD(rows, M)
        c = {"name": name, "rows": [enc(x) for x in rows], "M": M, "P": P, "top": [], "hot": []}
        for key, reverse, n in tops:
            got = rdd.top(n, key=KEYS[key], reverse=reverse) if key != "none" else rdd.top(n, reverse=reverse)
            c["top"].append({"key": key, "reverse": reverse, "n": n, "want": [enc(x) for x in got]})
        # the reference's uniq (dpark/rdd.py:383-385) hands rddconf to reduceByKey's fixSkew position, which fails
        # (None > 0) under Python 3; its body with that argument dropped:
        u = rdd.map(lambda x: (x, None)).reduceByKey(lambda x, y: None, P).map(lambda x_y1: x_y1[0])
        c["uniq"] = [sorted((enc(x) for x in part), key=json.dumps) for part in u.glom().collect()]
        every = rdd.hot(len(rows) + 1, P)
        sets = {}
        for x, cnt in every:
            sets.setdefault(cnt, []).append(enc(x))
        c["counts"] = [[cnt, sorted(xs, key=json.dumps)] for cnt, xs in sorted(sets.items())]
        for n in hots:
            c["hot"].append({"n": n, "counts": [cnt for _, cnt in rdd.hot(n, P)]})
        cases.append(c)

    d = list(range(100))
    random.Random(0).shuffle(d)
    case("test_rdd_top", d, 10, 10, [("none", False, 10), ("neg", False, 15)], [])
    for i in range(10):
        for j in range(i + 1):
            d.append(i)
    case("test_rdd_hot", d, 10, 10, [], [10])
    for kinds, n_rows, M, P in (("ii", 120, 5, 4), ("if", 60, 3, 2), ("fi", 60, 4, 3), ("ff", 80, 7, 5)):
        rows = _pairs(rnd, n_rows, kinds)
        tops = [(key, reverse, n) for key in ("none", "first", "second") for reverse in (False, True) for n in (1, 7)]
        tops += [("none", False, n_rows + 5), ("first", True, 30)]       # the whole sorted list, and a long prefix
        case("pairs_%s_%d_M%d_P%d" % (kinds, n_rows, M, P), rows, M, P, tops, [1, 5, 10])
    json.dump({"cases": cases}, open(os.path.join(HERE, "uniq_top_hot_cases.json"), "w"), separators=(",", ":"))
    dc.stop()
    print("wrote", len(cases), "top / uniq / hot cases")


def main():
    scratch = tempfile.mkdtemp(prefix="dpark_ref_")
    try:
        build_reference(scratch)
        bootstrap(scratch)
        generate()
    finally:
        shutil.rmtree(scratch, ignore_errors=True)


if __name__ == "__main__":
    main()
