"""Numeric text files into ColumnarRDDs on the GPU: DparkContext.textFileColumns.

    ctx.textFileColumns(path, key, value, types, sep, ...)

is a plain ColumnarRDD whose split i holds exactly the rows that split i of

    def parse(line):
        f = line.split(sep)
        return types[0](f[key]), types[1](f[value])
    ctx.textFile(path, ext, followLink, maxdepth, numSplits=numSplits, splitSize=splitSize).map(parse)

yields, in the same order: int columns are int64, float columns float64 with the bits of Python's float().  The splits
are the TextFileRDD's (or the UnionRDD's, for a directory or a list of paths); a split owns the lines that start in
its byte range (textingest.owned_range), cut into pieces at line starts (textingest.cut_pieces).  Per piece the bytes
go to the device, where dpk_textcols_count / _emit find the line starts and dpk_textcols_parse parses each line's two
fields -- or marks the line for the host when the device grammar (include/dpark_b200.h) does not cover it.  The host
lines are compacted in line order and run through `parse` itself, so a host line gets Python's values or raises
Python's exception, the first one in file order.  A piece holding a byte >= 0x80 is checked for strict UTF-8
(dpk_tokenize_utf8_count); if it is not, `parse` runs over all its lines as TextFileRDD decodes them, which raises
the row path's UnicodeDecodeError (or an earlier line's error).  An int outside int64 raises OverflowError, since a
column cannot hold it.

The columns are built when the method is called, as parallelizeColumns builds them, so errors are raised there and
not when a job runs.
"""
import os

import numpy as np
import torch

from . import _native as nv
from . import textingest
from .rdd import ColumnarRDD, TextFileRDD, UnionRDD

_I64_MIN, _I64_MAX = -(1 << 63), (1 << 63) - 1


def check_args(key, value, types, sep, numSplits, splitSize):
    for name, x in (("key", key), ("value", value)):
        if type(x) is not int:
            raise TypeError("%s must be an int, got %r" % (name, x))
        if x < 0:
            raise ValueError("%s must be >= 0, got %d" % (name, x))
    if not isinstance(types, (tuple, list)) or len(types) != 2:
        raise TypeError("types must be a pair of int / float, got %r" % (types,))
    if any(t is not int and t is not float for t in types):
        raise TypeError("types must be a pair of int / float, got %r" % (types,))
    if sep is not None:
        if not isinstance(sep, str):
            raise TypeError("sep must be None or a str, got %r" % (sep,))
        if sep == "":
            raise ValueError("empty separator")
        if "\n" in sep:
            raise ValueError("sep must not contain a newline")
    for name, x in (("numSplits", numSplits), ("splitSize", splitSize)):
        if x is None:
            continue
        if type(x) is not int:
            raise TypeError("%s must be None or an int, got %r" % (name, x))
        if x < 1:
            raise ValueError("%s must be >= 1, got %d" % (name, x))


def leaf_splits(rdd):
    """The (TextFileRDD, split) behind every split of what ctx.textFile returned, in split order."""
    if type(rdd) is TextFileRDD:
        return [(rdd, sp) for sp in rdd.splits]
    assert type(rdd) is UnionRDD
    return [leaf for sp in rdd.splits for leaf in leaf_splits_of(sp.rdd, sp.split)]


def leaf_splits_of(rdd, split):
    if type(rdd) is TextFileRDD:
        return [(rdd, split)]
    return leaf_splits_of(split.rdd, split.split)


def make_parse(key, value, types, sep):
    """The composition's parse, with the int64 check a column needs."""
    def parse(line):
        f = line.split(sep)
        k, v = types[0](f[key]), types[1](f[value])
        for i, x in ((key, k), (value, v)):
            if type(x) is int and not _I64_MIN <= x <= _I64_MAX:
                raise OverflowError("int field %d of line %r does not fit int64" % (i, line))
        return k, v
    return parse


def _line(buf, s, e):
    """A line as TextFileRDD.compute makes it: its bytes with the '\\n' decoded, then the '\\n' cut off."""
    text = buf[s:e].tobytes().decode("utf-8")
    return text[:-1] if text.endswith("\n") else text


def _bits(xs, t):
    return np.array(xs, dtype=np.float64).view(np.int64) if t is float else np.array(xs, dtype=np.int64)


def _piece(path, a, b, dev, sep_t, key, value, types, parse):
    """(keys, vals) int64 device columns (float columns as their bits) for the lines of path[a, b)."""
    buf = np.fromfile(path, dtype=np.uint8, count=b - a, offset=a)
    data = torch.from_numpy(buf).to(dev)
    starts, high = nv.line_starts(data)
    m = int(starts.numel())
    if high and not nv.utf8_valid(data):
        st = starts.cpu().tolist() + [b - a]
        rows = [parse(_line(buf, st[i], st[i + 1])) for i in range(m)]
        return (torch.from_numpy(_bits([r[0] for r in rows], types[0])).to(dev),
                torch.from_numpy(_bits([r[1] for r in rows], types[1])).to(dev))
    keys, vals, host = nv.textcols_parse(data, starts, sep_t, key, value, types[0] is float, types[1] is float)
    idx = host.nonzero().view(-1)
    if idx.numel():
        ends = torch.cat([starts[1:], torch.tensor([b - a], dtype=torch.int64, device=dev)])
        st, en = starts[idx].cpu().tolist(), ends[idx].cpu().tolist()
        rows = [parse(_line(buf, s, e)) for s, e in zip(st, en)]
        keys[idx] = torch.from_numpy(_bits([r[0] for r in rows], types[0])).to(dev)
        vals[idx] = torch.from_numpy(_bits([r[1] for r in rows], types[1])).to(dev)
    return keys, vals


def text_file_columns(ctx, path, key=0, value=1, types=(int, int), sep=None, ext="", followLink=True, maxdepth=0,
                      numSplits=None, splitSize=None):
    check_args(key, value, types, sep, numSplits, splitSize)
    types = tuple(types)
    rdd = ctx.textFile(path, ext, followLink, maxdepth, numSplits=numSplits, splitSize=splitSize)
    from .engine import _device
    dev = _device()
    sep_t = None if sep is None else torch.tensor(list(sep.encode("utf-8")), dtype=torch.uint8, device=dev)
    parse = make_parse(key, value, types, sep)
    kcols, vcols, bounds = [], [], [0]
    for text, sp in leaf_splits(rdd):
        size = os.path.getsize(text.path)
        a, b = textingest.owned_range(text.path, sp.begin, sp.end, size)
        rows = 0
        for pa, pb in textingest.cut_pieces(text.path, a, b, size) if b > a else []:
            k, v = _piece(text.path, pa, pb, dev, sep_t, key, value, types, parse)
            kcols.append(k)
            vcols.append(v)
            rows += int(k.numel())
        bounds.append(bounds[-1] + rows)
    dtypes = [torch.float64 if t is float else torch.int64 for t in types]
    keys, vals = [torch.cat(c) if c else torch.zeros(0, dtype=torch.int64, device=dev) for c in (kcols, vcols)]
    return ColumnarRDD(ctx, keys.view(dtypes[0]), vals.view(dtypes[1]), 1, bounds=bounds)
