"""The UTF-8 tokeniser's arithmetic (dpk_common.cuh tok8_ws / tok8_seq_ok / tok8_starts16, the per-thread step of
dpk_strings.cu k_tok8_count / k_tok8_emit) run on the CPU through tests/utf8check.cu, against Python itself:
whitespace is every code point str.isspace() accepts, a range is well-formed exactly when bytes.decode("utf-8")
succeeds, and the tokens are str.split()'s.  Then the product's splits, lines and tokens against what the REAL
reference hands out for a mixed-language text (tests/golden/textfile_utf8_cases.json).  No GPU needed."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

from dpark_b200 import textingest as ti
from tests import utf8_common as u

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    path = os.path.join(ROOT, "tests", "_utf8check.so")
    if not os.path.exists(path):
        pytest.skip("utf8check not built")
    L = C.CDLL(path)
    L.u8_tokenize.restype = C.c_int64
    L.u8_tokenize.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    L.u8_count_many.restype = None
    L.u8_count_many.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    L.u8_ws_many.restype = None
    L.u8_ws_many.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
    return L


def _aligned(data):
    """data in a 16-byte aligned host buffer, as a device buffer is (the slices' vector loads need it)."""
    raw = np.zeros(len(data) + 64, np.uint8)
    off = (-raw.ctypes.data) % 16
    view = raw[off:off + len(data)]
    view[:] = np.frombuffer(data, dtype=np.uint8)
    return raw, view


def tokens(L, data):
    """The tokens of one byte range, or None when the arithmetic flags it as not strict UTF-8."""
    raw, view = _aligned(data)
    starts = np.zeros(len(data) + 1, np.int64)
    lens = np.zeros(len(data) + 1, np.int64)
    m = L.u8_tokenize(view.ctypes.data, len(data), starts.ctypes.data, lens.ctypes.data)
    if m < 0:
        return None
    return [data[a:a + b] for a, b in zip(starts[:m].tolist(), lens[:m].tolist())]


def counts(L, strings):
    """Token count (-1: flagged ill-formed) of every string, each tokenised as a range of its own that starts on a
    16-byte boundary."""
    begin = np.zeros(len(strings), np.int64)
    end = np.zeros(len(strings), np.int64)
    at = 0
    for i, s in enumerate(strings):
        begin[i], end[i] = at, at + len(s)
        at = (at + len(s) + 15) // 16 * 16
    buf = bytearray(at)
    for s, b in zip(strings, begin.tolist()):
        buf[b:b + len(s)] = s
    raw, view = _aligned(bytes(buf))
    out = np.zeros(len(strings), np.int64)
    L.u8_count_many(view.ctypes.data, begin.ctypes.data, end.ctypes.data, len(strings), out.ctypes.data)
    return out.tolist()


def split_count(b):
    s = u.decodes(b)
    return -1 if s is None else len(s.split())


def test_whitespace_is_what_str_isspace_says(L):
    """tok8_ws of every code point's UTF-8 form: the length of that form when chr(c).isspace(), else 0."""
    cps = u.NON_SURROGATES
    enc = [chr(c).encode("utf-8") for c in cps]
    win = np.frombuffer(b"".join((e + b"\0\0")[:3] for e in enc), dtype=np.uint8).copy()
    got = np.zeros(len(cps), np.int32)
    L.u8_ws_many(win.ctypes.data, len(cps), got.ctypes.data)
    ws = set(u.WHITESPACE)
    want = [len(e) if c in ws else 0 for c, e in zip(cps, enc)]
    bad = [hex(c) for c, g, w in zip(cps, got.tolist(), want) if g != w]
    assert not bad, bad[:20]
    assert {len(chr(c).encode("utf-8")) for c in ws} == {1, 2, 3}
    assert not {0xFEFF, 0x200B, 0x180E} & ws


def test_every_code_point_between_two_letters_splits_as_str_split(L):
    """a<c>b for every code point c that is not a surrogate: each as its own range, and all of them as one text."""
    strings = [("a" + chr(c) + "b").encode("utf-8") for c in u.NON_SURROGATES]
    got = counts(L, strings)
    bad = [hex(c) for c, g, s in zip(u.NON_SURROGATES, got, strings) if g != split_count(s)]
    assert not bad, bad[:20]
    text = "\n".join("a" + chr(c) + "b" for c in u.NON_SURROGATES)
    assert tokens(L, text.encode("utf-8")) == [w.encode("utf-8") for w in text.split()]


@pytest.mark.parametrize("prefix", [0, 1, 13, 14, 15, 16, 17, 30, 31])
def test_well_formed_exactly_when_bytes_decode_succeeds(L, prefix):
    """Every 1- and 2-byte string, every 3- and 4-byte lead with every second byte and valid, invalid and missing later
    bytes: the arithmetic flags a range exactly when bytes.decode("utf-8") raises, and otherwise counts str.split()'s
    tokens.  `prefix` ASCII letters shift each probe across the 16-byte slice boundaries; a probe ends at the end of its
    range (a sequence cut short there is truncated) and, behind 24 more letters, in the middle of a range whose slices
    take the vector loads."""
    strings = []
    for s in u.probe_sequences():
        strings.append(b"x" * prefix + s)
        strings.append(b"x" * prefix + s + b"y" * 24)
    got = counts(L, strings)
    bad = [s.hex() for s, g in zip(strings, got) if g != split_count(s)]
    assert not bad, bad[:20]
    assert -1 in got and any(g > 0 for g in got)


@pytest.mark.parametrize("seq", [b"\x80", b"\xbf", b"\xc0\x80", b"\xc1\xbf", b"\xe0\x80\x80", b"\xe0\x9f\xbf",
                                 b"\xed\xa0\x80", b"\xed\xbf\xbf", b"\xf0\x80\x80\x80", b"\xf0\x8f\xbf\xbf",
                                 b"\xf4\x90\x80\x80", b"\xf4\xbf\xbf\xbf", b"\xf5\x80\x80\x80", b"\xff", b"\xe4\xb8",
                                 b"\xf0\x9f\x98", b"\xc3", b"\xe4\xb8\xad\x80"])
def test_each_ill_formed_class_is_flagged_anywhere_in_a_long_range(L, seq):
    """Stray continuation, C0 / C1, overlong 3- and 4-byte forms, surrogates, above U+10FFFF, F5..FF, cut short (in the
    middle and at the end of the range): flagged at every offset across two 16-byte slices of a range of Chinese text."""
    body = "\u4e2d\u6587 text ok ".encode("utf-8") * 8
    with pytest.raises(UnicodeDecodeError):
        seq.decode("utf-8")
    for at in range(0, 40):
        data = body[:at] + seq + body[at:]
        if u.decodes(body[:at]) is None:       # `at` inside a character of the body: a different byte string
            continue
        assert u.decodes(data) is None and tokens(L, data) is None, at
    assert tokens(L, body + seq) is None
    assert tokens(L, body) == [w.encode("utf-8") for w in body.decode("utf-8").split()]


@pytest.mark.parametrize("seed,nchars", [(1, 17), (2, 1000), (3, 4095), (4, 4096), (5, 70001)])
def test_random_mixed_text_splits_as_str_split(L, seed, nchars):
    text = u.random_text(seed, nchars)
    data = text.encode("utf-8")
    assert tokens(L, data) == [w.encode("utf-8") for w in text.split()]
    for cut in range(1, 8):                       # every suffix that starts inside a character is ill-formed
        if (data[cut] & 0xC0) == 0x80:
            assert tokens(L, data[cut:]) is None


def test_edge_ranges(L):
    for text in ["", " ", "\u3000", "\u3000\u2028\x85\xa0 \n", "a", "\u4e2d", "\U0001f600", "\ufeff",
                 "a\u3000b\u2029c\x85d\xa0e\u1680f\u205fg", "\u00e9" * 20 + "\u2000" + "\u6587" * 20]:
        data = text.encode("utf-8")
        assert tokens(L, data) == [w.encode("utf-8") for w in text.split()], text


def _golden():
    with open(os.path.join(ROOT, "tests", "golden", "textfile_utf8_cases.json"), encoding="utf-8") as f:
        return json.load(f)


def ctx():
    sys.argv = [sys.argv[0]]
    from dpark_b200 import DparkContext
    return DparkContext("local")


def test_owned_ranges_and_tokens_equal_what_the_reference_hands_out(L, tmp_path):
    """For every split size -- 5, 64 and 700 bytes cut inside multi-byte characters -- the product cuts the reference's
    splits, owns exactly the bytes of the lines the reference yields, and the tokeniser arithmetic makes the reference's
    wc.py tokens of that range, in order; cut in pieces at line starts, the pieces make the same tokens."""
    from dpark_b200.rdd import TextFileRDD
    gold = _golden()
    body = gold["text"].encode("utf-8")
    p = tmp_path / "in.txt"
    p.write_bytes(body)
    dc = ctx()
    assert any(c["cuts_inside_a_character"] for c in gold["cases"])
    for case in gold["cases"]:
        tf = TextFileRDD(dc, str(p), splitSize=case["split_size"])
        assert [[sp.begin, sp.end] for sp in tf.splits] == case["ranges"]
        prev = 0
        for sp, want_lines, want_tokens in zip(tf.splits, case["lines"], case["tokens"]):
            a, b = ti.owned_range(str(p), sp.begin, sp.end, len(body))
            chunk = body[a:b]
            got_lines = chunk.decode("utf-8").split("\n")
            if chunk.endswith(b"\n"):
                got_lines = got_lines[:-1]
            assert (got_lines if chunk else []) == want_lines
            assert list(tf.compute(sp)) == want_lines
            assert tokens(L, chunk) == [w.encode("utf-8") for w in want_tokens]
            assert a >= prev
            prev = b
        assert prev == len(body)
    want = [w.encode("utf-8") for w in gold["cases"][-1]["tokens"][0]]
    for limit in (1, 100, 1000):
        pieces = ti.cut_pieces(str(p), 0, len(body), len(body), limit)
        assert [w for a, b in pieces for w in tokens(L, body[a:b])] == want


def test_an_ill_formed_split_raises_the_references_error(L, tmp_path):
    """The text with one byte that is not UTF-8: the split holding it raises the reference's UnicodeDecodeError on the
    row path and its owned range is flagged; the other splits yield the reference's lines and are not flagged."""
    from dpark_b200.rdd import TextFileRDD
    gold = _golden()
    body = bytes.fromhex(gold["invalid_hex"])
    p = tmp_path / "bad.txt"
    p.write_bytes(body)
    dc = ctx()
    for case in gold["invalid"]:
        tf = TextFileRDD(dc, str(p), splitSize=case["split_size"])
        assert [[sp.begin, sp.end] for sp in tf.splits] == case["ranges"]
        for sp, want in zip(tf.splits, case["splits"]):
            a, b = ti.owned_range(str(p), sp.begin, sp.end, len(body))
            if "error" in want:
                with pytest.raises(UnicodeDecodeError) as e:
                    list(tf.compute(sp))
                assert str(e.value) == want["message"]
                assert tokens(L, body[a:b]) is None
            else:
                assert list(tf.compute(sp)) == want["lines"]
                assert tokens(L, body[a:b]) is not None
        assert tokens(L, body) is None
