#!/usr/bin/env python
"""Golden fixture for DparkContext.textFileColumns (dpark_b200/textcolumns.py), captured FROM THE REAL REFERENCE.

Runs only in the build container (needs the reference checkout).  Builds the scratch copy of the reference exactly as
make_golden.py does, writes seeded numeric files -- ints, floats with exponents, -0.0, inf / nan in mixed case, 25-digit
floats, underscores and non-ASCII digits, CRLF lines, extra columns, no final newline -- one per separator (None,
"\\t", ",", "::"), and records for several split sizes (cutting inside lines) what the REFERENCE's
`textFile(path, splitSize=...).map(parse)` yields per split, parse(line) = (types[0](f[key]), types[1](f[value])) for
f = line.split(sep); floats are stored as the hex of their bits.  Three more files hold a bad literal, a short line and
a byte that is not UTF-8; for them the fixture records, per split, the rows or the exception the reference raises.
tests/test_textcolumns_host.py checks the product's lines and its parse arithmetic (run on the CPU) against this file,
tests/test_gpu_textcolumns.py the device result.

    python tests/golden/make_textcolumns_golden.py        # rewrites tests/golden/textcolumns_cases.json
"""
import json
import os
import random
import shutil
import struct
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

SPLIT_SIZES = (7, 97, 1 << 20)
SEPS = (None, "\t", ",", "::")
# (types, key, value): every combination of column types, value < key and key == value
COLUMNS = {"int,float:0,1": ((int, float), 0, 1), "float,int:1,0": ((float, int), 1, 0),
           "float,float:0,1": ((float, float), 0, 1), "int,int:0,0": ((int, int), 0, 0)}


def numeric_lines(seed=20261018):
    rng = random.Random(seed)
    floats = ["-0.0", "0.0", "inf", "-Infinity", "NaN", "-nan", "1e400", "-1e-400", "1.", ".5", "2.2250738585072011e-308",
              "4.9406564584124654e-324", "1.7976931348623157e308", "9007199254740993", "1e23", "1_0.5", "１.５",
              "0.1234567890123456789012345", "+3.25E+02", "7"]
    ints = ["0", "-0", "+42", "9223372036854775807", "-9223372036854775808", "0000000000000000000012", "1_000",
            "٣٠", "-17"]
    out = []
    for i in range(40):
        if i < len(floats):
            f = floats[i]
        elif rng.random() < 0.5:
            f = repr(struct.unpack("<d", struct.pack("<Q", rng.getrandbits(64) & ~(0x7FF << 52) | (rng.randrange(900, 1150) << 52)))[0])
        else:
            f = "%de%d" % (rng.randrange(-10 ** 6, 10 ** 6), rng.randrange(-30, 30))
        k = ints[i] if i < len(ints) else str(rng.randrange(-10 ** 12, 10 ** 12))
        extra = ["x%d" % rng.randrange(100) for _ in range(rng.randrange(0, 3))]
        out.append(([k, f] + extra, rng.random() < 0.15))        # (fields, CRLF)
    return out


def render(lines, sep):
    j = " \t " if sep is None else sep
    return "\n".join(j.join(fs) + ("\r" if crlf else "") for fs, crlf in lines)     # no final newline


ERRORS = {
    "bad_literal": "1 2\n3 4\n5 x6\n7 8\n",
    "short_line": "1 2\n3 4\n5\n7 8\n",
    "not_utf8": b"1 2\n3 4\n5 6\xff\n7 8\n",
}


def enc(x):
    return {"f": struct.pack("<d", x).hex()} if isinstance(x, float) else x


def rows_or_error(rdd, sp):
    try:
        return {"rows": [[enc(k), enc(v)] for k, v in rdd.iterator(sp)]}
    except Exception as e:       # noqa: BLE001 -- the reference's exception is the datum
        return {"error": type(e).__name__, "message": str(e)}


def main():
    scratch = tempfile.mkdtemp(prefix="dpark_ref_")
    try:
        mg.build_reference(scratch)
        mg.bootstrap(scratch)
        import dpark  # the REFERENCE (scratch copy)
        dc = dpark.DparkContext("local")
        lines = numeric_lines()
        files = []
        for si, sep in enumerate(SEPS):
            text = render(lines, sep)
            path = os.path.join(scratch, "num%d.txt" % si)
            with open(path, "wb") as f:
                f.write(text.encode("utf-8"))
            cases = []
            for split_size in SPLIT_SIZES:
                base = dc.textFile(path, splitSize=split_size)
                entry = {"split_size": split_size, "ranges": [[sp.begin, sp.end] for sp in base.splits],
                         "lines": [list(base.iterator(sp)) for sp in base.splits], "rows": {}}
                for name, (types, key, value) in COLUMNS.items():
                    def parse(line, sep=sep, types=types, key=key, value=value):
                        f = line.split(sep)
                        return types[0](f[key]), types[1](f[value])
                    rdd = base.map(parse)
                    entry["rows"][name] = [rows_or_error(rdd, sp) for sp in rdd.splits]
                cases.append(entry)
            files.append({"sep": sep, "text": text, "cases": cases})
        errors = []
        for name, body in ERRORS.items():
            raw = body if isinstance(body, bytes) else body.encode("utf-8")
            path = os.path.join(scratch, name + ".txt")
            with open(path, "wb") as f:
                f.write(raw)
            for split_size in (6, 1 << 20):
                rdd = dc.textFile(path, splitSize=split_size).map(lambda line: (int(line.split()[0]), int(line.split()[1])))
                errors.append({"name": name, "hex": raw.hex(), "split_size": split_size,
                               "splits": [rows_or_error(rdd, sp) for sp in rdd.splits]})
        dc.stop()
        out = {"files": files, "errors": errors,
               "how": "reference textFile(path, splitSize).map(parse), parse(line) = (t0(f[key]), t1(f[value])) for "
                      "f = line.split(sep): per split the rows (floats as {'f': hex of the float64 bits}) or the "
                      "exception; error files with int, int over line.split()"}
        with open(os.path.join(HERE, "textcolumns_cases.json"), "w", encoding="utf-8") as f:
            json.dump(out, f, ensure_ascii=False)
        print("wrote textcolumns_cases.json: %d files, %d error cases" % (len(files), len(errors)))
    finally:
        shutil.rmtree(scratch, ignore_errors=True)


if __name__ == "__main__":
    main()
