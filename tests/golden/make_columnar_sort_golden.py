#!/usr/bin/env python
"""Golden vectors for RDD.sort of (k, v) pairs FROM THE REAL REFERENCE (dpark/rdd.py:273-287); same out-of-tree build as
make_golden.py.

    python tests/golden/make_columnar_sort_golden.py     # writes tests/golden/columnar_sort_cases.json

The pairs a numeric ColumnarRDD holds -- int and float columns with many ties and both signed zeros -- sorted by the
three keys the device sort recognises (the identity, x[0], x[1]) in both directions.  parallelize slices the list in
chunks of ceil(len / M), as ColumnarRDD does.  Stored: every input once, and every output partition in order as indices
into its input (the first pair with the row's repr; -0.0 and 0.0 are told apart).  The reference's order among equal
keys follows its fetch order, so a partition's rows are compared as a multiset and only their keys by position."""
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

KEYS = {"id": lambda x: x, "first": lambda x: x[0], "second": lambda x: x[1]}


def generate():
    from dpark import DparkContext
    logging.getLogger("dpark").setLevel(logging.ERROR)
    dc = DparkContext("local")
    dc.init()
    rnd = random.Random(47)
    inputs, cases = {}, []

    def case(name, data, M, key, reverse, P):
        pairs = inputs[data]["pairs"]
        index = {}
        for i, x in enumerate(pairs):
            index.setdefault(repr(x), i)
        out = dc.parallelize(pairs, M).sort(key=KEYS[key], reverse=reverse, numSplits=P).glom().collect()
        cases.append({"name": name, "input": data, "M": M, "key": key, "reverse": reverse, "P": P,
                      "parts": [[index[repr(x)] for x in part] for part in out]})

    zeros = [-0.0, 0.0, 0.5, -0.5, 1.5, -2.0]
    inputs["ints"] = {"kinds": ["int", "int"], "pairs": [(rnd.randrange(-15, 15), rnd.randrange(-3, 3))
                                                         for _ in range(40)]}
    inputs["floats"] = {"kinds": ["float", "float"],
                        "pairs": [(rnd.choice(zeros) if rnd.random() < 0.4 else rnd.randrange(-3, 3) * 0.5,
                                   rnd.choice(zeros)) for _ in range(40)]}
    inputs["int_float"] = {"kinds": ["int", "float"], "pairs": [(rnd.randrange(-6, 6), rnd.choice(zeros))
                                                               for _ in range(30)]}
    for key in ("id", "first", "second"):
        for reverse in (False, True):
            tag = "%s_%s" % (key, "rev" if reverse else "fwd")
            case("ints_" + tag, "ints", 5, key, reverse, 4)
            case("floats_" + tag, "floats", 3, key, reverse, None)
            case("int_float_" + tag, "int_float", 6, key, reverse, 5)
    case("one_split", "ints", 1, "first", True, 4)
    case("one_partition", "floats", 4, "id", False, 1)
    case("more_splits_than_samples", "int_float", 3, "second", False, 8)
    for inp in inputs.values():
        inp["pairs"] = [[enc(k), enc(v)] for k, v in inp["pairs"]]
    with open(os.path.join(HERE, "columnar_sort_cases.json"), "w") as f:
        json.dump({"inputs": inputs, "cases": cases}, f, separators=(",", ":"))
    dc.stop()
    print("wrote", len(cases), "columnar sort cases")


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
