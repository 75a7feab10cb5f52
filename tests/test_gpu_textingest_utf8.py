"""Device text ingest of UTF-8 text: dpk_tokenize_utf8_* against Python's str.split() and bytes.decode("utf-8"), and the
word-count pipeline through DparkContext with the UTF-8 tokeniser against the same pipeline run row-wise
(engine.TEXT_INGEST = False).  -m gpu."""
import os
import sys

import numpy as np
import pytest
import torch

from tests import utf8_common as u

pytestmark = pytest.mark.gpu

WS2 = [chr(c) for c in u.WHITESPACE if len(chr(c).encode("utf-8")) == 2]
WS3 = [chr(c) for c in u.WHITESPACE if len(chr(c).encode("utf-8")) == 3]
PROBES = WS2 + WS3 + ["\U0001f600", "\U0010ffff"]      # every 2- and 3-byte separator, 4-byte non-separators
ILL_FORMED = [b"\x80", b"\xc0\x80", b"\xc1\xbf", b"\xe0\x9f\xbf", b"\xed\xa0\x80", b"\xf0\x8f\xbf\xbf",
              b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xff", b"\xe4\xb8", b"\xf0\x9f\x98", b"\xe4\xb8\xad\x80"]


def nv():
    from dpark_b200 import _native
    return _native


def _dev(data):
    return torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda() if data else \
        torch.zeros(0, dtype=torch.uint8, device="cuda")


def _tokens(data: bytes):
    starts, lens, ok = nv().tokenize_utf8(_dev(data))
    if not ok:
        return None
    s, l = starts.cpu().tolist(), lens.cpu().tolist()
    return [data[a:a + b] for a, b in zip(s, l)]


def _split(data: bytes):
    return [w.encode("utf-8") for w in data.decode("utf-8").split()]


def _sized(seed, nbytes):
    """Seeded mixed text of exactly nbytes UTF-8 bytes (a character cut by the end is replaced by ASCII letters)."""
    data = u.random_text(seed, nbytes).encode("utf-8")[:nbytes]
    while u.decodes(data) is None:
        data = data[:-1]
    return data + b"z" * (nbytes - len(data))


@pytest.mark.parametrize("probe", PROBES, ids=lambda c: "U+%04X" % ord(c))
def test_probe_at_every_offset_across_a_slice_and_a_block_boundary(probe):
    """A 2- or 3-byte separator (or a 4-byte letter) at every byte offset around the 16-byte thread-slice boundary and
    the 4096-byte block boundary, between ASCII letters and between 3-byte CJK letters."""
    p = probe.encode("utf-8")
    for filler, step in ((b"x", 1), ("\u6587".encode("utf-8"), 3)):
        body = filler * (5000 // len(filler))
        for at in list(range(8, 26)) + list(range(4084, 4102)):
            at -= at % step
            data = body[:at] + p + body[at:]
            assert _tokens(data) == _split(data), (at, filler)
            data = body[:at] + p + p + b"y" + body[at:]
            assert _tokens(data) == _split(data), (at, filler)


@pytest.mark.parametrize("text", ["", " ", "\u3000\u2028\x85\xa0 \n\u1680", "\n\n", "no final newline \u6587\u5b57",
                                  "\u4e2d\u6587\n\u5b57 \u00e9\u00e8\n", "\ufeffbom\u200bzw\u180emv"])
def test_edge_texts(text):
    data = text.encode("utf-8")
    assert _tokens(data) == _split(data)


@pytest.mark.parametrize("seed,n", [(1, 4095), (2, 4096), (3, 4097), (4, 70001), (5, 1 << 20)])
def test_random_mixed_text_matches_str_split(seed, n):
    data = _sized(seed, n)
    assert len(data) == n
    assert _tokens(data) == _split(data)


@pytest.mark.parametrize("seq", ILL_FORMED, ids=lambda s: s.hex())
def test_each_ill_formed_class_sets_the_flag(seq):
    """Stray continuation, C0 / C1, overlong, surrogate, above U+10FFFF, F5..FF, cut short: at the start, at a slice
    and a block boundary, and at the end of the range."""
    body = b"ascii and \xe4\xb8\xad\xe6\x96\x87 " * 400
    for at in (0, 15, 16, 17, 4094, 4096, len(body)):
        while u.decodes(body[:at]) is None:
            at -= 1
        data = body[:at] + seq + body[at:]
        assert u.decodes(data) is None
        assert _tokens(data) is None, at
    assert _tokens(body) == _split(body)


def test_device_token_hashes_equal_the_key_hashes():
    """The tokens' bytes, hashed on the device by code point (dpk_hash_bytes STR_UTF8), equal portable_hash of the
    decoded words -- astral code points included."""
    from dpark_b200 import columnar
    data = _sized(9, 50000)
    d = _dev(data)
    starts, lens, ok = nv().tokenize_utf8(d)
    assert ok
    tok, off = nv().gather_bytes(d, starts, lens)
    h = nv().hash_bytes(tok, off, nv().STR_UTF8).cpu().tolist()
    words = data.decode("utf-8").split()
    assert any(ord(ch) > 0xFFFF for w in words for ch in w)
    assert h == columnar.hashes_of_keys(words)


# ---- the word-count pipeline ------------------------------------------------------------------------------------------
def ctx():
    sys.argv = [sys.argv[0]]
    from dpark_b200 import DparkContext
    return DparkContext("local")


def fm(x):
    for w in x.strip().split():
        yield (w, 1)


def _corpus(tmp_path, seed=11, lines_n=6000, final_newline=True):
    rng = np.random.default_rng(seed)
    vocab = ["w%d" % i for i in range(500)] + u.random_text(seed, 20000).split() + ["caf\u00e9", "\U0001f600"]
    seps = [chr(c) for c in u.WHITESPACE if c != 0x0A] + [" "] * 20
    lines = []
    for _ in range(lines_n):
        words = [vocab[int(i)] for i in (rng.zipf(1.3, int(rng.integers(0, 12))) - 1) % len(vocab)]
        lines.append("".join(w + seps[int(rng.integers(0, len(seps)))] for w in words))
    p = tmp_path / ("in%d.txt" % seed)
    p.write_bytes(("\n".join(lines) + ("\n" if final_newline else "")).encode("utf-8"))
    return str(p)


def _spy(monkeypatch):
    from dpark_b200 import textingest
    calls = []
    for name in ("reduce_tokens", "reduce_tokens_utf8"):
        real = getattr(textingest, name)

        def spy(*a, _real=real, _name=name, **kw):
            r = _real(*a, **kw)
            calls.append((_name, r is not None))
            return r
        monkeypatch.setattr(textingest, name, spy)
    return calls


def _wc(path, out, num_splits):
    dc = ctx()
    counts = dc.textFile(path, numSplits=num_splits).flatMap(fm).reduceByKey(lambda x, y: x + y, numSplits=6)
    got = counts.collectAsMap()
    dc.textFile(path, numSplits=num_splits).flatMap(fm).reduceByKey(lambda x, y: x + y, numSplits=6) \
        .map(lambda x: " ".join(list(map(str, x)))).saveAsTextFile(out, overwrite=False)
    # the lines of each partition's file (their order inside a partition is not part of the result)
    files = {fn: sorted(open(os.path.join(out, fn), encoding="utf-8").read().split("\n")) for fn in sorted(os.listdir(out))}
    return got, files


@pytest.mark.parametrize("num_splits,piece_bytes,final_newline", [(1, None, True), (3, None, False), (3, 4096, True),
                                                                  (1, 10000, False)])
def test_wc_utf8_on_the_device_equals_the_row_wise_pipeline(tmp_path, monkeypatch, num_splits, piece_bytes,
                                                            final_newline):
    """collectAsMap() and the saveAsTextFile files, line for line, are the same whether the tokens come from the
    user's Python generator or from dpk_tokenize_utf8 -- which produced them: the ASCII pass declined, the UTF-8 pass
    ran, once per job."""
    from dpark_b200 import engine, textingest
    path = _corpus(tmp_path, final_newline=final_newline)
    if piece_bytes:
        monkeypatch.setattr(textingest, "MAX_PIECE_BYTES", piece_bytes)
    calls = _spy(monkeypatch)
    got, got_files = _wc(path, str(tmp_path / "dev"), num_splits)
    runs = len(calls) // 2
    assert runs >= 1 and calls == [("reduce_tokens", False), ("reduce_tokens_utf8", True)] * runs
    monkeypatch.setattr(engine, "TEXT_INGEST", False)
    want, want_files = _wc(path, str(tmp_path / "rows"), num_splits)
    assert len(calls) == 2 * runs
    assert got == want and got_files == want_files
    text = open(path, encoding="utf-8").read()
    assert sum(got.values()) == len(text.split()) and any(ord(ch) > 0x7F for w in got for ch in w)


def test_wc_of_ill_formed_text_raises_the_row_paths_error(tmp_path, monkeypatch):
    from dpark_b200 import engine
    p = tmp_path / "bad.txt"
    p.write_bytes("\u597d ok\nfine line\n".encode("utf-8") * 500 + b"bad \xed\xa0\x80 surrogate\n" + b"tail\n")
    calls = _spy(monkeypatch)
    with pytest.raises(UnicodeDecodeError) as dev_err:
        ctx().textFile(str(p), numSplits=3).flatMap(fm).reduceByKey(lambda x, y: x + y).collectAsMap()
    assert calls == [("reduce_tokens", False), ("reduce_tokens_utf8", False)]
    monkeypatch.setattr(engine, "TEXT_INGEST", False)
    with pytest.raises(UnicodeDecodeError) as row_err:
        ctx().textFile(str(p), numSplits=3).flatMap(fm).reduceByKey(lambda x, y: x + y).collectAsMap()
    assert str(dev_err.value) == str(row_err.value)


def test_ascii_text_still_takes_the_ascii_pass_alone(tmp_path, monkeypatch):
    p = tmp_path / "a.txt"
    p.write_text("one two\nthree one\n" * 100, encoding="ascii")
    calls = _spy(monkeypatch)
    got = ctx().textFile(str(p)).flatMap(fm).reduceByKey(lambda x, y: x + y).collectAsMap()
    assert calls == [("reduce_tokens", True)]
    assert got == {"one": 200, "two": 100, "three": 100}
