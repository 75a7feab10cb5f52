"""The numeric text columns' arithmetic (dpk_common.cuh tc_parse_i64 / tc_parse_f64 / tc_eisel_lemire / tc_fields /
tc_starts16, the per-line step of dpk_strings.cu k_tc_*) run on the CPU through tests/numparsecheck.cu, against Python
itself: every string the device accepts gets the bits of Python's int() / float(), every string Python rejects goes to
the host, and the fields are line.split(sep)'s.  Then the product's lines and rows against what the REAL reference
yields for textFile(...).map(parse) (tests/golden/textcolumns_cases.json), and ColumnarRDD's split bounds.  No GPU
needed."""
import ctypes as C
import decimal
import importlib.util
import itertools
import json
import math
import os
import random
import struct

import numpy as np
import pytest

from dpark_b200 import textcolumns as tc
from dpark_b200 import textingest as ti
from dpark_b200.errors import DparkUserFatalError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_I64, K_F64 = 0, 2
WHITESPACE = [chr(c) for c in range(0x110000) if chr(c).isspace()]


@pytest.fixture(scope="module")
def L():
    path = os.path.join(ROOT, "tests", "_numparsecheck.so")
    if not os.path.exists(path):
        pytest.skip("numparsecheck not built")
    L = C.CDLL(path)
    vp, i64, i32 = C.c_void_p, C.c_int64, C.c_int32
    for name in ("np_parse_i64_many", "np_parse_f64_many"):
        getattr(L, name).restype = None
        getattr(L, name).argtypes = [vp, vp, i64, vp, vp]
    L.np_fields_many.restype = None
    L.np_fields_many.argtypes = [vp, vp, i64, vp, i32, i32, i32, vp, vp]
    L.np_lines_many.restype = None
    L.np_lines_many.argtypes = [vp, vp, i64, vp, i32, i32, i32, i32, i32, vp, vp, vp]
    L.np_line_starts.restype = i64
    L.np_line_starts.argtypes = [vp, i64, vp]
    L.np_pow5.restype = None
    L.np_pow5.argtypes = [vp]
    return L


def _pack(strings):
    bs = [s.encode("utf-8") if isinstance(s, str) else s for s in strings]
    off = np.zeros(len(bs) + 1, np.int64)
    off[1:] = np.cumsum([len(b) for b in bs])
    buf = np.frombuffer(b"".join(bs) + b"\0" * 16, np.uint8).copy()
    return buf, off


def device_f64(L, strings):
    """(bits, accepted) of every string through tc_parse_f64."""
    buf, off = _pack(strings)
    out, ok = np.zeros(len(strings), np.uint64), np.zeros(len(strings), np.uint8)
    L.np_parse_f64_many(buf.ctypes.data, off.ctypes.data, len(strings), out.ctypes.data, ok.ctypes.data)
    return out.tolist(), ok.astype(bool).tolist()


def device_i64(L, strings):
    buf, off = _pack(strings)
    out, ok = np.zeros(len(strings), np.int64), np.zeros(len(strings), np.uint8)
    L.np_parse_i64_many(buf.ctypes.data, off.ctypes.data, len(strings), out.ctypes.data, ok.ctypes.data)
    return out.tolist(), ok.astype(bool).tolist()


def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def check_f64(L, strings):
    """Every accepted string has float()'s bits, every rejected one is rejected by the device; returns the share of
    the strings Python accepts that the device sends to the host."""
    got, ok = device_f64(L, strings)
    python_ok = host = 0
    for s, g, a in zip(strings, got, ok):
        try:
            want = bits(float(s))
        except ValueError:
            assert not a, "device accepts %r, float() rejects it" % (s,)
            continue
        python_ok += 1
        if a:
            assert g == want, "%r: device %016x, float() %016x" % (s, g, want)
        else:
            host += 1
    return host / max(python_ok, 1)


def check_i64(L, strings):
    got, ok = device_i64(L, strings)
    python_ok = host = 0
    for s, g, a in zip(strings, got, ok):
        try:
            want = int(s)
        except ValueError:
            assert not a, "device accepts %r, int() rejects it" % (s,)
            continue
        python_ok += 1
        if a:
            assert g == want, "%r: device %d, int() %d" % (s, g, want)
        else:
            host += 1
    return host / max(python_ok, 1)


# ---- float ----------------------------------------------------------------------------------------------------------
def test_float_every_short_string(L):
    alphabet = list("0123456789.eE+-_ infatyNIx") + ["\x1f"]
    strings = ["".join(t) for n in range(5) for t in itertools.product(alphabet, repeat=n)]
    check_f64(L, strings)


def test_float_random_decimals(L):
    rng = random.Random(5)
    strings = []
    for _ in range(10 ** 6):
        nd = rng.randint(1, 40)
        d = "".join(rng.choice("0123456789") for _ in range(nd))
        k = rng.randint(0, nd)
        s = d[:k] + "." + d[k:] if rng.random() < 0.7 else d
        strings.append(rng.choice(("", "-", "+")) + s + rng.choice(("e", "E")) + str(rng.randint(-360, 330)))
    share = check_f64(L, strings)
    print("random 1-40 digit decimals: %.4f%% host" % (100 * share))
    assert share < 0.01


def test_float_repr_and_17g_of_random_bits(L):
    rng = random.Random(6)
    xs = [struct.unpack("<d", struct.pack("<Q", rng.getrandbits(64)))[0] for _ in range(2 * 10 ** 5)]
    xs = [x for x in xs if math.isfinite(x)]
    assert check_f64(L, [repr(x) for x in xs]) == 0       # repr text never needs the host
    share = check_f64(L, ["%.17g" % x for x in xs])
    print("%%.17g: %.4f%% host" % (100 * share))


def _midpoints(rng, count):
    out = []
    decimal.getcontext().prec = 1200
    for _ in range(count):
        x = abs(struct.unpack("<d", struct.pack("<Q", rng.getrandbits(63)))[0])
        if not math.isfinite(x) or x == 0:
            continue
        mid = (decimal.Decimal(x) + decimal.Decimal(math.nextafter(x, math.inf))) / 2
        s = format(mid, "f") if -30 < mid.adjusted() < 30 else format(mid, "e")
        out.append(s)
        mant, _, exp = s.partition("e")
        last = mant.rstrip("0")
        if last[-1].isdigit() and last[-1] not in "09":
            for dlt in (-1, 1):
                out.append(last[:-1] + str(int(last[-1]) + dlt) + ("e" + exp if exp else ""))
    return out


def test_float_midpoints_between_doubles(L):
    rng = random.Random(7)
    strings = _midpoints(rng, 3000)
    strings += ["9007199254740993", "9007199254740993.0000000000000000001", "9007199254740992.9999999999999999999"]
    check_f64(L, strings)


def test_float_boundaries_and_specials(L):
    strings = ["2.2250738585072011e-308", "2.2250738585072014e-308", "4.9406564584124654e-324",
               "2.4703282292062327e-324", "2.4703282292062328e-324", "1.7976931348623157e308",
               "1.7976931348623158e308", "1.7976931348623159e308", "9007199254740993", "1e23", "8.98846567431158e307",
               "0", "-0", "0.0", "-0.0", "+0e99999999999999999999", "-0e-5", "1e400", "-1e400", "1e-400", "-1e-400",
               "1e99999999999999999999999", "1e-99999999999999999999999", ".5", "1.", "-.5e-3", " 1.5\t", "\r\n2\v\f",
               "1.5\x1f", "1_0.5", "1e1_0", "1__0", "_1", "1_", "1_.5", "1._5", ".", "e5", "1e", "1e+", "0x10",
               "nan(1)", "١.٥"]
    for w in ("inf", "infinity", "nan"):
        for sign in ("", "+", "-"):
            for case in (w, w.upper(), w.title(), "".join(c.upper() if i % 2 else c for i, c in enumerate(w))):
                strings.append(sign + case)
    strings += ["infinit", "infinityy", "nana", "in", "-", "+-1", "--1"]
    check_f64(L, strings)
    got, ok = device_f64(L, ["-nan", "nan", "-0.0", "1e400", "-1e-400"])
    assert ok == [True] * 5
    assert got == [0xFFF8000000000000, 0x7FF8000000000000, 1 << 63, 0x7FF0000000000000, 1 << 63]


# ---- int ------------------------------------------------------------------------------------------------------------
def test_int_every_short_string(L):
    alphabet = list("0123456789+-_ \t")
    strings = ["".join(t) for n in range(6) for t in itertools.product(alphabet, repeat=n)]
    check_i64(L, strings)


def test_int_limits(L):
    strings = [str(x) for x in (2 ** 63 - 1, -2 ** 63 + 1, -2 ** 63, 2 ** 63, -2 ** 63 - 1, 10 ** 18, -10 ** 18)]
    strings += ["9" * 19, "-" + "9" * 19, "1" + "0" * 19, "0" * 19, "0" * 18 + "7", "0" * 20, "0" * 19 + "1",
                "+0000000000000000001", "0" * 5000 + "1", "1_" * 2500 + "1", "٣", "１２", " 12\x1f", "\t-5\r"]
    check_i64(L, strings)
    got, ok = device_i64(L, [str(2 ** 63 - 1), str(-2 ** 63), str(2 ** 63), "0" * 19, "0" * 20])
    assert ok == [True, True, False, True, False] and got[:2] == [2 ** 63 - 1, -2 ** 63]


def test_plain_int_text_never_needs_the_host(L):
    rng = random.Random(8)
    strings = ["%d" % rng.randrange(-2 ** 63, 2 ** 63) for _ in range(10 ** 5)]
    assert check_i64(L, strings) == 0


# ---- fields ---------------------------------------------------------------------------------------------------------
def device_fields(L, lines, sep, k0, k1):
    buf, off = _pack(lines)
    sb = np.frombuffer((sep or "").encode("utf-8") + b"\0", np.uint8).copy()
    f, ok = np.zeros(4 * len(lines), np.int64), np.zeros(len(lines), np.uint8)
    L.np_fields_many(buf.ctypes.data, off.ctypes.data, len(lines), sb.ctypes.data, len(sb) - 1, k0, k1,
                     f.ctypes.data, ok.ctypes.data)
    out = []
    for i, line in enumerate(lines):
        raw = line.encode("utf-8")
        g = f[4 * i:4 * i + 4].tolist()
        out.append((raw[g[0]:g[1]].decode("utf-8"), raw[g[2]:g[3]].decode("utf-8")) if ok[i] else None)
    return out


def python_fields(line, sep, k0, k1):
    f = line.split(sep)
    return (f[k0], f[k1]) if max(k0, k1) < len(f) else None


@pytest.mark.parametrize("sep", [None, ",", "\t", "::", "aa", "→", " "])
def test_fields_are_line_split(L, sep):
    rng = random.Random(hash(sep) & 0xFFFF)
    pieces = ["1", "-2.5", "x", "a", ":", "é", "→", "中", "", "__"]
    glue = WHITESPACE if sep is None else [sep, sep, sep + sep, sep[:-1] or "a", ":"]
    lines = []
    for _ in range(20000):
        n = rng.randint(0, 6)
        line = "".join(rng.choice(pieces) + rng.choice(glue) for _ in range(n)) + rng.choice(pieces)
        lines.append(line.replace("\n", " ") if sep is not None else line.replace("\n", "\x0b"))
    for k0, k1 in ((0, 1), (1, 0), (2, 2), (0, 4)):
        got = device_fields(L, lines, sep, k0, k1)
        for line, g in zip(lines, got):
            assert g == python_fields(line, sep, k0, k1), (line, sep, k0, k1)


def test_line_starts(L):
    rng = random.Random(9)
    for n in list(range(0, 40)) + [4095, 4096, 4097, 10000]:
        for _ in range(3):
            data = bytes(rng.choice(b"ab\n\xc3") for _ in range(n))
            raw = np.zeros(n + 64, np.uint8)
            o = (-raw.ctypes.data) % 16
            raw[o:o + n] = np.frombuffer(data, np.uint8)
            starts = np.zeros(n + 1, np.int64)
            m = L.np_line_starts(raw[o:].ctypes.data, n, starts.ctypes.data)
            want = [0] + [i + 1 for i, c in enumerate(data) if c == 10 and i + 1 < n] if n else []
            assert starts[:m].tolist() == want


# ---- the power-of-five table -----------------------------------------------------------------------------------------
def test_power_of_five_table_is_regenerated_identically(L):
    spec = importlib.util.spec_from_file_location("gen_pow5", os.path.join(ROOT, "dpark_b200", "csrc", "gen_pow5.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    with open(os.path.join(ROOT, "dpark_b200", "csrc", "dpk_pow5.inc")) as f:
        assert f.read() == gen.render()
    compiled = np.zeros(2 * (gen.Q_MAX - gen.Q_MIN + 1), np.uint64)
    L.np_pow5(compiled.ctypes.data)
    assert [x for hl in gen.table() for x in hl] == compiled.tolist()
    for q, (hi, lo) in zip(range(gen.Q_MIN, gen.Q_MAX + 1), gen.table()):
        v = (hi << 64) | lo
        assert v >> 127 == 1
        if q >= 0:      # 5^q * 2^s truncated: within one unit below the exact value
            e = 5 ** q
            s = 127 - (e.bit_length() - 1)
            exact = e << s if s >= 0 else e >> -s
            assert v == exact


# ---- the reference's rows ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "textcolumns_cases.json"), encoding="utf-8") as f:
        return json.load(f)


def _dec(x):
    return struct.unpack("<d", bytes.fromhex(x["f"]))[0] if isinstance(x, dict) else x


def rows_of_lines(L, lines, sep, key, value, types):
    """The rows textFileColumns makes of one split's lines with the device arithmetic run on the CPU: device rows, the
    host lines through the composition's parse (raising what it raises)."""
    buf, off = _pack(lines)
    sb = np.frombuffer((sep or "").encode("utf-8") + b"\0", np.uint8).copy()
    m = len(lines)
    k, v, ok = np.zeros(m, np.int64), np.zeros(m, np.int64), np.zeros(m, np.uint8)
    kinds = [K_F64 if t is float else K_I64 for t in types]
    L.np_lines_many(buf.ctypes.data, off.ctypes.data, m, sb.ctypes.data, len(sb) - 1, key, value, kinds[0], kinds[1],
                    k.ctypes.data, v.ctypes.data, ok.ctypes.data)
    parse = tc.make_parse(key, value, types, sep)
    out = []
    for i, line in enumerate(lines):
        if ok[i]:
            kv = [np.int64(x).view(np.float64).item() if t is float else int(x) for x, t in zip((k[i], v[i]), types)]
        else:
            kv = list(parse(line))
        out.append(kv)
    return out, int(m - ok.sum())


def _same(a, b):
    return all(bits(x) == bits(y) if isinstance(x, float) else (type(x) is type(y) and x == y) for x, y in zip(a, b))


def test_golden_lines_and_rows(L, golden, tmp_path):
    host_lines = 0
    for fi, entry in enumerate(golden["files"]):
        path = tmp_path / ("num%d.txt" % fi)
        path.write_bytes(entry["text"].encode("utf-8"))
        size = path.stat().st_size
        raw = path.read_bytes()
        for case in entry["cases"]:
            for (b, e), lines in zip(case["ranges"], case["lines"]):
                a0, a1 = ti.owned_range(str(path), b, e, size)
                mine = [tc._line(np.frombuffer(raw, np.uint8), s, t) for s, t in _lines_in(raw, a0, a1)]
                assert mine == lines
            for name, per_split in case["rows"].items():
                t, kv = name.split(":")
                types = tuple({"int": int, "float": float}[x] for x in t.split(","))
                key, value = (int(x) for x in kv.split(","))
                for lines, want in zip(case["lines"], per_split):
                    assert "rows" in want
                    got, h = rows_of_lines(L, lines, entry["sep"], key, value, types)
                    host_lines += h
                    assert len(got) == len(want["rows"])
                    for g, w in zip(got, want["rows"]):
                        assert _same(g, [_dec(x) for x in w]), (g, w)
    assert host_lines > 0       # the fixture has underscores, non-ASCII digits, 25-digit floats


def _lines_in(raw, a, b):
    at = a
    while at < b:
        nl = raw.find(b"\n", at, b)
        nxt = b if nl < 0 else nl + 1
        yield at, nxt
        at = nxt


def test_golden_errors(L, golden, tmp_path):
    for case in golden["errors"]:
        raw = bytes.fromhex(case["hex"])
        size = len(raw)
        path = tmp_path / (case["name"] + ".txt")
        path.write_bytes(raw)
        split_size = case["split_size"]
        nsplits = size // split_size + (1 if size % split_size else 0)
        assert len(case["splits"]) == nsplits
        for i, want in enumerate(case["splits"]):
            a, b = ti.owned_range(str(path), i * split_size, min(size, (i + 1) * split_size), size)
            try:
                lines = [tc._line(np.frombuffer(raw, np.uint8), s, t) for s, t in _lines_in(raw, a, b)]
                rows, _ = rows_of_lines(L, lines, None, 0, 1, (int, int))
            except Exception as e:       # noqa: BLE001
                assert want.get("error") == type(e).__name__ and want["message"] == str(e)
            else:
                assert want.get("rows") == rows


# ---- arguments and split bounds -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw, exc", [
    (dict(key=-1), ValueError), (dict(value=1.0), TypeError), (dict(key=True), TypeError),
    (dict(types=(int,)), TypeError), (dict(types=(int, str)), TypeError), (dict(types="if"), TypeError),
    (dict(sep=""), ValueError), (dict(sep="a\nb"), ValueError), (dict(sep=b","), TypeError),
    (dict(numSplits=0), ValueError), (dict(splitSize=1.5), TypeError),
])
def test_arguments_are_checked_before_any_file_is_read(kw, exc):
    args = dict(key=0, value=1, types=(int, int), sep=None, numSplits=None, splitSize=None)
    args.update(kw)
    with pytest.raises(exc) as e:
        tc.check_args(**args)
    if kw.get("sep") == "":
        assert str(e.value) == "empty separator"


def test_columnar_rdd_bounds():
    from dpark_b200 import DparkContext
    from dpark_b200.rdd import ColumnarRDD
    ctx = DparkContext("local")
    k = np.arange(10, dtype=np.int64)
    r = ColumnarRDD(ctx, k, k * 2, 3, bounds=[0, 0, 4, 4, 10])
    assert [(s.begin, s.end) for s in r.splits] == [(0, 0), (0, 4), (4, 4), (4, 10)]
    assert [list(r.iterator(s)) for s in r.splits][1] == [(i, 2 * i) for i in range(4)]
    assert len(ColumnarRDD(ctx, k[:0], k[:0], 3, bounds=[0]).splits) == 0
    assert len(ColumnarRDD(ctx, k, k, 2, bounds=np.array([0, 10])).splits) == 1
    plain, same = ColumnarRDD(ctx, k, k, 3), ColumnarRDD(ctx, k, k, 3, bounds=None)
    assert [(s.begin, s.end) for s in plain.splits] == [(s.begin, s.end) for s in same.splits] == [(0, 4), (4, 8), (8, 10)]
    for bad in ([], [1, 10], [0, 9], [0, 5, 4, 10], [0, 2.5, 10], [0, True, 10], None.__class__, "0a", [0, "5", 10]):
        with pytest.raises(DparkUserFatalError):
            ColumnarRDD(ctx, k, k, 2, bounds=bad)
