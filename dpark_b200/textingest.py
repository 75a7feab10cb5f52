"""Device text ingest for the word-count shape (SURVEY.md section 8 row f4; examples/wc.py:10-17).

    dc.textFile(path).flatMap(fm).reduceByKey(add)          fm(x): for w in x.strip().split(): yield (w, 1)

In the reference -- and on this package's row-wise path -- every line is decoded and split by the user's Python
function and every token becomes a (str, int) tuple before the shuffle sees it: the end-to-end time of BASELINE config 1
is that interpreter loop (scripts/wc_e2e.py <lines> rowwise times it).  When the functions between
`textFile` and the shuffle are, byte code for byte code, one of the tokenising shapes below, the same rows are produced
on the GPU instead: the file's bytes go to HBM, `dpk_tokenize_*` finds the tokens (str.split() semantics), and the
token bytes feed the existing variable-length-key shuffle (dpk_hash_bytes -> dpk_dict_encode -> dpk_partition ->
dpk_combine).  Only the distinct words and their counts come back.

Two tokenisers, tried in this order: `reduce_tokens` (dpk_tokenize_count / _emit) takes text that is ASCII throughout
and declines at the first piece holding a byte >= 0x80; `reduce_tokens_utf8` (dpk_tokenize_utf8_count / _emit) then
runs the whole job again over UTF-8 text, with Python's Unicode whitespace (every code point c with chr(c).isspace(),
separators of 1 to 3 bytes) and strict decoding.  TextFileRDD decodes every line with strict utf-8, so when a range is
not well-formed UTF-8 the device declines the whole job and the row-wise path raises the reference's
UnicodeDecodeError.  Keys come back as the decoded tokens, not normalised, exactly as str.split() leaves them.

Recognition is structural and exact -- the user's code object must equal a template's (instructions, constants,
attribute names, signature; no closure, no defaults) -- never a behavioural probe: anything else, any split that is
not well-formed UTF-8, and any subclass of the RDD types involved takes the row-wise path unchanged.
"""
import os
import types

import numpy as np
import torch

from . import _native as nv
from . import shuffle


# ---- the shapes ------------------------------------------------------------------------------------------------------
def _t_gen_strip_split(x):
    for w in x.strip().split():
        yield (w, 1)


def _t_gen_split(x):
    for w in x.split():
        yield (w, 1)


_t_list_strip_split = lambda x: [(w, 1) for w in x.strip().split()]     # noqa: E731
_t_list_split = lambda x: [(w, 1) for w in x.split()]                   # noqa: E731
_t_split = lambda x: x.split()                                          # noqa: E731
_t_strip_split = lambda x: x.strip().split()                            # noqa: E731
_t_pair_one = lambda x: (x, 1)                                          # noqa: E731


def _sig(code):
    """What makes two code objects the same program: instructions, constants (nested code objects recursively),
    attribute/global names, signature and kind flags.  Variable names, file names and line numbers do not matter."""
    consts = tuple(_sig(c) if isinstance(c, types.CodeType) else (type(c).__name__, c) for c in code.co_consts)
    return (code.co_code, consts, code.co_names, code.co_argcount, code.co_posonlyargcount, code.co_kwonlyargcount,
            code.co_flags & 0x2F, len(code.co_freevars), len(code.co_cellvars))   # OPTIMIZED|NEWLOCALS|VARARGS|VARKEYWORDS|GENERATOR


def _same(f, template):
    return (type(f) is types.FunctionType and f.__closure__ is None and not f.__defaults__ and not f.__kwdefaults__
            and _sig(f.__code__) == _sig(template.__code__))


_PAIR_TOKENISERS = (_t_gen_strip_split, _t_gen_split, _t_list_strip_split, _t_list_split)
_TOKENISERS = (_t_split, _t_strip_split)


def recognize(parent):
    """The TextFileRDD whose tokens, each paired with the int 1, are exactly `parent`'s rows -- or None."""
    from .rdd import FlatMappedRDD, MappedRDD, TextFileRDD
    if type(parent) is FlatMappedRDD and type(parent.prev) is TextFileRDD:
        if any(_same(parent.func, t) for t in _PAIR_TOKENISERS):
            return parent.prev
        return None
    if (type(parent) is MappedRDD and _same(parent.func, _t_pair_one) and type(parent.prev) is FlatMappedRDD
            and type(parent.prev.prev) is TextFileRDD and any(_same(parent.prev.func, t) for t in _TOKENISERS)):
        return parent.prev.prev
    return None


# ---- the byte ranges of the splits -------------------------------------------------------------------------------------
def owned_range(path, begin, end, size):
    """Bytes of the lines that START inside [begin, end) (TextFileRDD.compute, dpark/rdd.py:1672-1711): from the first
    line start at or after `begin` to the first line start at or after `end`."""
    def line_start_at_or_after(pos):
        if pos <= 0:
            return 0
        if pos >= size:
            return size
        with open(path, "rb") as f:
            f.seek(pos - 1)
            at = pos - 1
            while True:
                chunk = f.read(1 << 16)
                if not chunk:
                    return size
                i = chunk.find(b"\n")
                if i >= 0:
                    return at + i + 1
                at += len(chunk)
    return line_start_at_or_after(begin), line_start_at_or_after(end)


MAX_PIECE_BYTES = 1 << 30      # a byte range longer than this is tokenised in pieces cut at line starts


def cut_pieces(path, a, b, size, max_bytes=None):
    """[a, b) (both line starts) as consecutive pieces of at most ~max_bytes bytes, every cut on a line start (a token
    never straddles a piece: newlines are whitespace)."""
    max_bytes = max_bytes or MAX_PIECE_BYTES
    out = []
    while b - a > max_bytes:
        cut = owned_range(path, a + max_bytes, a + max_bytes, size)[0]     # first line start at or after a + max_bytes
        if cut >= b:
            break
        out.append([a, cut])
        a = cut
    if b > a:
        out.append([a, b])
    return out


def reduce_tokens(text_rdd, split_indices, P, thresholds, op, dev, res, local_only=True):
    """reduceByKey(op) over (token, 1) for the tokens of the given splits of `text_rdd`, on the device.  Fills
    res.parts[p] = (keys, values) for every partition and returns res; returns None (nothing done) when a split
    holds a non-ASCII byte.  The splits' owned ranges are contiguous when the indices are, and every line belongs to
    exactly one split, so consecutive splits are read as one byte range."""
    return _reduce(text_rdd, split_indices, P, thresholds, op, dev, res, local_only, nv.tokenize, "ascii")


def reduce_tokens_utf8(text_rdd, split_indices, P, thresholds, op, dev, res, local_only=True):
    """reduce_tokens for UTF-8 text: the tokens are those str.split() finds in the decoded lines (Unicode whitespace),
    the keys their `bytes.decode("utf-8")`.  Returns None (nothing done) only when a split is not strict UTF-8 -- the
    row-wise path then raises the UnicodeDecodeError TextFileRDD.compute raises."""
    return _reduce(text_rdd, split_indices, P, thresholds, op, dev, res, local_only, nv.tokenize_utf8, "utf-8")


def _reduce(text_rdd, split_indices, P, thresholds, op, dev, res, local_only, tokenize, encoding):
    path = text_rdd.path
    size = os.path.getsize(path)
    splits = text_rdd.splits
    ranges = []
    for i in sorted(split_indices):
        a, b = owned_range(path, splits[i].begin, splits[i].end, size)
        if b > a:
            if ranges and ranges[-1][1] == a:
                ranges[-1][1] = b
            else:
                ranges.append([a, b])
    pieces = []
    for a, b in [piece for r in ranges for piece in cut_pieces(path, r[0], r[1], size)]:
        host = np.fromfile(path, dtype=np.uint8, count=b - a, offset=a)
        d_text = torch.from_numpy(host).to(dev)
        starts, lens, ok = tokenize(d_text)
        if not ok:
            return None
        if starts.numel():
            pieces.append(nv.gather_bytes(d_text, starts, lens))
        del d_text
    if not pieces:
        for p in range(P):
            res.parts[p] = ([], [])
        return res
    if len(pieces) == 1:
        tok, off = pieces[0]
    else:
        tok = torch.cat([t for t, _ in pieces])
        offs, base = [pieces[0][1]], int(pieces[0][0].numel())
        for t, o in pieces[1:]:
            offs.append(o[1:] + base)
            base += int(t.numel())
        off = torch.cat(offs)
    n = int(off.numel()) - 1
    if n >= (1 << 31):
        raise nv.NativeError("more than 2^31 tokens in one shuffle")
    ones = torch.ones(n, dtype=torch.int64, device=dev)
    h = nv.hash_bytes(tok, off, nv.STR_UTF8)          # str keys hash by code point (unicode_hash, portable_hash.pyx:33-48)
    rep = nv.dict_encode(tok, off, h)                 # strict UTF-8: equal strings are equal bytes
    sb = shuffle.choose_sub_bits(n, P)
    ctx = shuffle.local_only() if local_only else _Null()
    with ctx:
        mo = shuffle.map_side([rep], [ones], P, thresholds, False, sb, row_hash=h, unordered=True)
        rx = shuffle.exchange(mo)
        ok, ov, poff, cnt = nv.combine(rx.keys, rx.vals, op, P, rx.seg.contiguous(), rx.part_first, rx.nparts,
                                       thresholds, sb, row_hash=h, rows=rx.rows)
    off_h, cnt_h = poff.cpu().tolist(), cnt.cpu().tolist()
    shuffle.check_counts(cnt_h)
    # the distinct words: their bytes are gathered on the device, one small copy back
    sel = torch.cat([ok[off_h[p]:off_h[p] + cnt_h[p]] for p in range(P)]) if P else ok[:0]
    lens_all = off[1:] - off[:-1]
    kb, ko = nv.gather_bytes(tok, off[:-1].contiguous(), lens_all.contiguous(), sel.contiguous())
    raw, ko_h = kb.cpu().numpy().tobytes(), ko.cpu().tolist()
    vals = torch.cat([ov[off_h[p]:off_h[p] + cnt_h[p]] for p in range(P)]).cpu().tolist() if P else []
    at = 0
    for p in range(P):
        c = cnt_h[p]
        keys = [raw[ko_h[i]:ko_h[i + 1]].decode(encoding) for i in range(at, at + c)]
        res.parts[p] = (keys, vals[at:at + c])
        at += c
    return res


class _Null(object):
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False
