#!/usr/bin/env python
"""Golden fixture for the device UTF-8 tokeniser (textingest.reduce_tokens_utf8), captured FROM THE REAL REFERENCE.

Runs only in the build container (needs the reference checkout).  Builds the scratch copy of the reference exactly as
make_golden.py does, writes a seeded mixed-language text -- Chinese, Latin-1, Cyrillic, emoji, every code point
str.isspace() accepts (1-, 2- and 3-byte UTF-8 forms), the non-whitespace U+FEFF, U+200B and U+180E, CRLF lines, empty
lines, no final newline -- and records, for several split sizes (some cutting inside multi-byte characters), what the
REFERENCE's `textFile(path, splitSize=...)` hands out: the lines of every split and the rows the tokenising flatMap of
examples/wc.py (`for w in x.strip().split(): yield (w, 1)`) makes of them.  A second text holds one byte that is not
UTF-8; for it the fixture records, per split, the lines or the UnicodeDecodeError the reference raises.
tests/test_textingest_utf8_host.py checks the product's owned byte ranges, its lines and its tokeniser arithmetic (run
on the CPU) against this file.

    python tests/golden/make_textfile_utf8_golden.py        # rewrites tests/golden/textfile_utf8_cases.json
"""
import json
import os
import random
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

SPLIT_SIZES = (5, 64, 700, 1 << 20)


def make_text(seed=20261018):
    rng = random.Random(seed)
    ws = [chr(c) for c in range(0x110000) if chr(c).isspace() and chr(c) != "\n"]
    cjk = [chr(rng.randrange(0x4E00, 0xA000)) for _ in range(300)]
    special = ["caf\u00e9", "na\u00efve", "Stra\u00dfe", "\u00e9lan", "\u043c\u0438\u0440", "\U0001f600", "a\U0001f600b",
               "\U0001f004", "\ufeffbom", "zero\u200bwidth", "mongol\u180eian", "\U0010ffff", "x" * 37, "\x00nul",
               "\x7fdel", "\ufb01"]
    vocab = ["w%d" % i for i in range(20)] + ["".join(rng.sample(cjk, rng.randint(1, 4))) for _ in range(60)] + special
    lines = [" ".join(special), "".join("s" + c for c in ws) + "s"]     # every word kind and every separator, once
    for _ in range(40):
        k = rng.choice([0, 0, 1, 2, 3, 5, 8, 13])
        line = "".join(rng.choice(vocab) + rng.choice(ws + [" "] * 10) for _ in range(k))
        if rng.random() < 0.15:
            line = rng.choice(ws) + line
        if rng.random() < 0.1:
            line += "\r"
        lines.append(line)
    return "\n".join(lines) + "\n\u6700\u540e\u4e00\u884c without newline"


INVALID = "\u597d ok\nfine line\n".encode("utf-8") + b"bad \xff byte\n" + "\u672b\u5c3e tail\n".encode("utf-8")


def fm(x):
    for w in x.strip().split():
        yield (w, 1)


def main():
    scratch = tempfile.mkdtemp(prefix="dpark_ref_")
    try:
        mg.build_reference(scratch)
        mg.bootstrap(scratch)
        import dpark  # the REFERENCE (scratch copy)
        dc = dpark.DparkContext("local")
        text = make_text()
        body = text.encode("utf-8")
        path = os.path.join(scratch, "in.txt")
        with open(path, "wb") as f:
            f.write(body)
        cases = []
        for split_size in SPLIT_SIZES:
            rdd = dc.textFile(path, splitSize=split_size)
            lines = [list(rdd.iterator(sp)) for sp in rdd.splits]
            rows = [list(rdd.flatMap(fm).iterator(sp)) for sp in rdd.splits]
            assert all(one == 1 for r in rows for w, one in r)
            inside = sum(1 for sp in rdd.splits if 0 < sp.begin < len(body) and (body[sp.begin] & 0xC0) == 0x80)
            cases.append({"split_size": split_size, "ranges": [[sp.begin, sp.end] for sp in rdd.splits],
                          "cuts_inside_a_character": inside, "lines": lines, "tokens": [[w for w, _ in r] for r in rows]})
        assert cases[0]["cuts_inside_a_character"] and cases[1]["cuts_inside_a_character"]
        bad_path = os.path.join(scratch, "bad.txt")
        with open(bad_path, "wb") as f:
            f.write(INVALID)
        invalid = []
        for split_size in (8, 1 << 20):
            rdd = dc.textFile(bad_path, splitSize=split_size)
            per_split = []
            for sp in rdd.splits:
                try:
                    per_split.append({"lines": list(rdd.iterator(sp))})
                except UnicodeDecodeError as e:
                    per_split.append({"error": type(e).__name__, "message": str(e)})
            invalid.append({"split_size": split_size, "ranges": [[sp.begin, sp.end] for sp in rdd.splits],
                            "splits": per_split})
        dc.stop()
        out = {"text": text, "cases": cases, "invalid_hex": INVALID.hex(), "invalid": invalid,
               "how": "reference textFile(path, splitSize) -> lines per split; flatMap(wc.py's fm) -> tokens per split; "
                      "a text with one byte that is not UTF-8 -> lines or the UnicodeDecodeError per split"}
        with open(os.path.join(HERE, "textfile_utf8_cases.json"), "w", encoding="utf-8") as f:
            json.dump(out, f, ensure_ascii=False)
        print("wrote textfile_utf8_cases.json: %d bytes of text, %d cases, %d tokens"
              % (len(body), len(cases), sum(len(t) for t in cases[0]["tokens"])))
    finally:
        shutil.rmtree(scratch, ignore_errors=True)


if __name__ == "__main__":
    main()
