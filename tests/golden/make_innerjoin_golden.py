#!/usr/bin/env python
"""Golden vectors for innerJoin FROM THE REAL REFERENCE (dpark/rdd.py:626-648); same out-of-tree build as make_golden.py.

    python tests/golden/make_innerjoin_golden.py    # writes tests/golden/innerjoin_cases.json

The inputs of the reference's own innerJoin assertions (tests/test_rdd.py:326-348): per case both inputs with their
split counts, the collect() rows in order and the glom() partitions in order (innerJoin keeps the big side's splits
and row order, so nothing is sorted)."""
import json
import logging
import os
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import bootstrap, build_reference, enc  # noqa: E402


def generate():
    from dpark import DparkContext
    logging.getLogger("dpark").setLevel(logging.ERROR)
    dc = DparkContext("local")
    dc.init()
    cases = []

    def case(name, big, small, M_big, M_small):
        out = dc.makeRDD(big, M_big).innerJoin(dc.makeRDD(small, M_small))
        cases.append({"name": name, "big": [[enc(k), enc(v)] for k, v in big], "M_big": M_big,
                      "small": [[enc(k), enc(v)] for k, v in small], "M_small": M_small,
                      "rows": [[enc(k), enc(tuple(v))] for k, v in out.collect()],
                      "parts": [[[enc(k), enc(tuple(v))] for k, v in part] for part in out.glom().collect()]})

    nums = list(zip([1, 2, 3, 3], range(4, 8)))
    case("test_rdd_inner_join", nums, list(zip([2, 3, 4], [1, 2, 3])), 2, 2)
    case("test_rdd_inner_join_duplicate_key", nums, list(zip([2, 2, 4], [1, 2, 3])), 2, 2)
    json.dump({"cases": cases}, open(os.path.join(HERE, "innerjoin_cases.json"), "w"), separators=(",", ":"))
    dc.stop()
    print("wrote", len(cases), "innerJoin cases")


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
