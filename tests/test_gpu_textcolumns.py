"""DparkContext.textFileColumns on the GPU (dpk_textcols_count / _emit / _parse, dpark_b200/textcolumns.py): split by
split and bit for bit what textFile(...).map(parse) yields, with the composition's exceptions; the kernels at their
slice and block boundaries, under poison-filled guarded buffers, and the columns fed to the columnar operators."""
import random
import struct
import sys

import numpy as np
import pytest
import torch

from dpark_b200 import _native as nv
from dpark_b200 import textcolumns, textingest
from tests.test_gpu_buffer_bounds import Guard, GuardedTorch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    sys.argv = [sys.argv[0]]          # DparkContext.init parses the command line (pytest's flags are not its own)
    from dpark_b200 import DparkContext
    return DparkContext("local")


def composition(ctx, path, key=0, value=1, types=(int, int), sep=None, **kw):
    """Per split the composition's rows, or the exception it raises first (in split order)."""
    def parse(line):
        f = line.split(sep)
        return types[0](f[key]), types[1](f[value])
    rdd = ctx.textFile(path, kw.get("ext", ""), numSplits=kw.get("numSplits"), splitSize=kw.get("splitSize")).map(parse)
    return [list(rdd.iterator(sp)) for sp in rdd.splits]


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0] if isinstance(x, float) else ("i", x)


def check(ctx, path, **kw):
    """textFileColumns equals the composition split by split, bit for bit -- or both raise the same exception."""
    try:
        want = composition(ctx, path, **kw)
    except Exception as e:       # noqa: BLE001
        with pytest.raises(type(e)) as got:
            ctx.textFileColumns(path, **kw)
        assert str(got.value) == str(e)
        return None
    rdd = ctx.textFileColumns(path, **kw)
    assert type(rdd).__name__ == "ColumnarRDD"
    assert len(rdd.splits) == len(want)
    for sp, w in zip(rdd.splits, want):
        k, v = rdd.columns(sp)
        got = list(zip(k.cpu().tolist(), v.cpu().tolist()))
        assert [tuple(map(_bits, r)) for r in got] == [tuple(map(_bits, r)) for r in w]
    return rdd


def write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data if isinstance(data, bytes) else data.encode("utf-8"))
    return str(p)


def test_line_breaks_at_slice_and_block_boundaries(ctx, tmp_path):
    for at in (15, 16, 17, 4095, 4096, 4097):
        first = "1" + " " * (at - 3) + "2"            # the first '\n' lands at byte `at - 1`, the next line at `at`
        body = first + "\n3 4\n" + "5 6\n" * 1100 + "7 8"
        check(ctx, write(tmp_path, "b%d.txt" % at, body))
        check(ctx, write(tmp_path, "c%d.txt" % at, body + "\n"), splitSize=at)


def test_empty_blank_and_long_lines(ctx, tmp_path):
    rdd = check(ctx, write(tmp_path, "empty.txt", b""))
    assert len(rdd.splits) == 0
    check(ctx, write(tmp_path, "nl.txt", "\n\n\n"))                      # IndexError
    check(ctx, write(tmp_path, "long.txt", "1 " + "0" * 9000 + "7\n2 3\n"))   # a line past a block, a host line
    check(ctx, write(tmp_path, "long2.txt", "1" + " " * 9000 + "2\n2 3"))


def _field(rng, t):
    r = rng.random()
    if t is int:
        if r < 0.8:
            return str(rng.randrange(-10 ** rng.randint(1, 18), 10 ** rng.randint(1, 18)))
        return rng.choice(["+7", "-0", "0007", " 5", "9223372036854775807", "-9223372036854775808", "1_000", "٣"])
    if r < 0.5:
        return repr(struct.unpack("<d", struct.pack("<Q", rng.getrandbits(64) & ~(0x7FF << 52)
                                                    | (rng.randrange(800, 1250) << 52)))[0])
    if r < 0.9:
        return "%de%d" % (rng.randrange(-10 ** 9, 10 ** 9), rng.randrange(-40, 40))
    return rng.choice(["-0.0", "inf", "-Infinity", "nan", "-NaN", "1e400", "1_0.5", "１.５",
                       "0.1234567890123456789012345", ".5", "1."])


def corpus(seed, types, sep, nbytes=1 << 20, ncols=4):
    rng = random.Random(seed)
    joins = [" ", "\t", "  ", " \x0b", "　"] if sep is None else [sep]
    out, size = [], 0
    while size < nbytes:
        fs = [_field(rng, types[i % 2]) for i in range(ncols)]
        line = fs[0]
        for f in fs[1:]:
            line += rng.choice(joins) + f
        if rng.random() < 0.05:
            line += "\r"
        out.append(line)
        size += len(line.encode("utf-8")) + 1
    return "\n".join(out)


@pytest.mark.parametrize("types", [(int, int), (int, float), (float, int), (float, float)])
@pytest.mark.parametrize("sep", [None, "\t", ",", "::", "→"])
def test_random_corpora_match_the_composition(ctx, tmp_path, types, sep):
    path = write(tmp_path, "r.txt", corpus(repr((types, sep)), types, sep))
    check(ctx, path, key=0, value=1, types=types, sep=sep)
    check(ctx, path, key=3, value=2, types=(types[1], types[0]), sep=sep, numSplits=7)
    check(ctx, path, key=2, value=2, types=(types[0], types[0]), sep=sep, splitSize=100003)


def test_directory_of_files(ctx, tmp_path):
    d = tmp_path / "dir"
    d.mkdir()
    for i in range(3):
        (d / ("part%d.tsv" % i)).write_text(corpus(i, (int, float), "\t", nbytes=1 << 16), encoding="utf-8")
    (d / "skip.txt").write_text("x\n")
    check(ctx, str(d), types=(int, float), sep="\t", ext=".tsv", splitSize=30000)
    check(ctx, [str(d / "part0.tsv"), str(d)], types=(int, float), sep="\t", ext=".tsv")


def test_several_pieces(ctx, tmp_path, monkeypatch):
    path = write(tmp_path, "p.txt", corpus(11, (int, float), None))
    monkeypatch.setattr(textingest, "MAX_PIECE_BYTES", 40000)
    check(ctx, path, types=(int, float))
    check(ctx, path, types=(int, float), numSplits=3)


def test_host_lines_and_errors(ctx, tmp_path):
    body = "1_0 2.5\n٣ １.５\n9223372036854775807 0.1234567890123456789012345\n-9223372036854775808 1e400\n"
    check(ctx, write(tmp_path, "h.txt", body), types=(int, float))
    with pytest.raises(OverflowError, match="9223372036854775808"):
        ctx.textFileColumns(write(tmp_path, "o.txt", "1 2\n9223372036854775808 3\n"))
    for name, data in (("bad", "1 2\n3 x\n5\n"), ("short", "1 2\n3\n5 x\n"), ("utf", b"1 2\n3 \xff\n5\n"),
                       ("utf_after", b"1 2\n3 x\n4 \xe4\n"), ("utf_cut", b"1 2\n3 4\xe4")):
        path = write(tmp_path, name + ".txt", data)
        check(ctx, path)
        check(ctx, path, splitSize=4)


def test_feeds_the_columnar_operators(ctx, tmp_path):
    from operator import add
    rng = random.Random(3)
    lines = ["%d\t%d\t%r" % (rng.randrange(50), rng.randrange(1000), rng.random()) for _ in range(20000)]
    path = write(tmp_path, "ops.tsv", "\n".join(lines))
    cols = ctx.textFileColumns(path, 0, 2, (int, float), "\t", splitSize=50000)
    ints = ctx.textFileColumns(path, 0, 1, (int, int), "\t", splitSize=50000)
    bounds = [sp.begin for sp in cols.splits] + [cols.splits[-1].end]
    assert len(set(np.diff(bounds).tolist())) > 1         # uneven splits
    rows = [r for sp in composition(ctx, path, 0, 2, (int, float), "\t", splitSize=50000) for r in sp]
    k = torch.tensor([r[0] for r in rows], dtype=torch.int64)
    v = torch.tensor([r[1] for r in rows], dtype=torch.float64)
    ref = ctx.parallelizeColumns(k, v)
    ref = type(ref)(ctx, k, v, 1, bounds=bounds)
    got, want = sorted(cols.reduceByKey(add, 4).collect()), sorted(ref.reduceByKey(add, 4).collect())
    assert [k for k, _ in got] == [k for k, _ in want]         # float sums: the merge order may differ in the last bits
    assert all(abs(a - b) <= 1e-12 * abs(b) for (_, a), (_, b) in zip(got, want))
    assert cols.sort().collect() == ref.sort().collect()
    assert sorted(cols.topByKey(3).collect()) == sorted(ref.topByKey(3).collect())
    assert sorted(cols.join(ints).collect()) == sorted(ref.join(ints).collect())
    assert cols.sample(False, 0.1, 7).collect() == ref.sample(False, 0.1, 7).collect()
    got = sorted(cols.percentilesByKey([10, 50, 99]).collect())
    assert got == sorted(ref.percentilesByKey([10, 50, 99]).collect())
    comp = ctx.textFile(path, splitSize=50000).map(lambda line: (int(line.split("\t")[0]), float(line.split("\t")[2])))
    assert got == sorted(comp._percentiles_rows([10, 50, 99]).collect())


@pytest.mark.parametrize("poison", [0x00, 0xFF])
def test_guarded_buffers(ctx, tmp_path, monkeypatch, poison):
    path = write(tmp_path, "g.txt", corpus(21, (int, float), None, nbytes=1 << 17))
    want = ctx.textFileColumns(path, types=(int, float), splitSize=20000)
    g = Guard()
    g.poison = poison
    for mod, name in ((textcolumns, "textcolumns"), (nv, "_native")):
        monkeypatch.setattr(mod, "torch", GuardedTorch(g, name))
    got = ctx.textFileColumns(path, types=(int, float), splitSize=20000)
    g.check()
    assert torch.equal(got.keys.cpu(), want.keys.cpu())
    assert torch.equal(got.vals.view(torch.int64).cpu(), want.vals.view(torch.int64).cpu())
    assert [(s.begin, s.end) for s in got.splits] == [(s.begin, s.end) for s in want.splits]
