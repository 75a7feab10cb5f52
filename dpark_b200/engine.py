"""Runs one ShuffledRDD on the GPU: the static two-stage plan that replaces the
reference's DAG scheduler for this path (SURVEY.md §2 row 8: out of scope as a
system; the map stage and the reduce stage are simply run in order).

    stage 1 (map)    every parent split -> columns -> HBM -> dpark_b200.shuffle.map_side
    stage 2 (reduce) exchange + reduce_side / group_side -> per-partition columns

Python rows exist only before stage 1 (ingest of what user lambdas produced) and
after stage 2 (egress to user lambdas); see dpark_b200.columnar.
"""
import numpy as np
import torch

from . import _native as nv
from . import columnar, shuffle


class ShuffleResult(object):
    """Per-partition result columns on the host + lazy conversion to rows."""

    def __init__(self, nparts):
        self.parts = [None] * nparts      # (keys: list, vals: list | (offsets, values)) per partition

    def rows(self, p):
        keys, vals = self.parts[p]
        return list(zip(keys, vals))

    def columns(self, p):
        return self.parts[p]


def _device():
    if not torch.cuda.is_available():
        raise nv.NativeError("the dpark_b200 shuffle needs a CUDA device (there is no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def _gather_parent(srdd, numeric_values, only=None):
    """Stage-1 input: one Columns (host) or a (keys, vals) tensor pair per parent split (`only`: the split indices
    this rank owns under torch.distributed)."""
    from .rdd import ColumnarRDD
    parent = srdd.parent
    out = []
    for i, sp in enumerate(parent.splits):
        if only is not None and i not in only:
            continue
        if isinstance(parent, ColumnarRDD) and numeric_values:
            out.append(parent.columns(sp))
        else:
            out.append(columnar.ingest_pairs(parent.iterator(sp), repr(parent), numeric_values))
    return out


TEXT_INGEST = True            # dpark_b200.textingest: tokenise textFile -> split -> (w, 1) pipelines on the device


def run_shuffle(srdd):
    from . import spmd
    rank, world = spmd.rank_world()
    if world > 1:
        return _run_shuffle_spmd(srdd, rank, world)
    dev = _device()
    P = srdd.partitioner.numPartitions
    thr = srdd.partitioner.thresholds
    if srdd.kind == "reduce":
        from . import textingest
        text = textingest.recognize(srdd.parent) if TEXT_INGEST else None
        if text is not None:     # the word-count shape: tokenise on the device (ASCII first, then UTF-8; None back from
            # both: the text is not strict UTF-8 and the row-wise path raises the reference's UnicodeDecodeError)
            res = textingest.reduce_tokens(text, range(len(text.splits)), P, thr, srdd.op, dev, ShuffleResult(P))
            if res is None:
                res = textingest.reduce_tokens_utf8(text, range(len(text.splits)), P, thr, srdd.op, dev, ShuffleResult(P))
            if res is not None:
                return res
        splits = _gather_parent(srdd, True)
        return _run_reduce(splits, P, thr, srdd.op, dev)
    from .rdd import device_path_applies
    if device_path_applies([srdd.parent]):
        return _run_group_columns(srdd.parent, P, thr)
    splits = _gather_parent(srdd, False)
    return _run_group(splits, P, thr, dev)


def _run_group_columns(parent, P, thr):
    """groupByKey of a numeric ColumnarRDD: the one-input cogroup on the device (dpark_b200/join.py), handed out as
    the host lists the row path gives."""
    from . import join
    res = ShuffleResult(P)
    for p, (keys, offsets, (vals,)) in enumerate(join.cogroup_columns([parent], P, thr)):
        off, vs = offsets[0].cpu().tolist(), vals.cpu().tolist()
        res.parts[p] = (keys.cpu().tolist(), [vs[off[j]:off[j + 1]] for j in range(len(off) - 1)])
    return res


# ---------------------------------------------------------------------------------------------------------------------
# one driver process per GPU (dpark_b200/spmd.py)
# ---------------------------------------------------------------------------------------------------------------------
ROUTE_EVERYTHING = False      # test hook: numeric reduceByKey also takes the routed path (CPU tests have no NCCL)


def _run_shuffle_spmd(srdd, rank, world):
    """The shuffle with the map stage spread over the ranks: every rank ingests the parent splits it owns.

      numeric keys + numeric values + reduce   device columns through shuffle.reduce_by_key: map_side -> NCCL
                                               alltoallv -> reduce_side, partitions owned in contiguous blocks;
      everything else (group-by: values are    the rows are routed on the HOST to the rank owning their partition
      Python objects; str / bytes keys)        (partition ids come from the CUDA hash / getPartition kernels), as
                                               pickled columns in one all_to_all; the owner then runs the one-GPU path
                                               over what it received, sources in rank order = map split order.

    Every rank ends up with the (small, host) result of every partition, so downstream narrow stages can run anywhere."""
    from . import spmd
    dev = _device()
    P = srdd.partitioner.numPartitions
    thr = srdd.partitioner.thresholds
    nsplits = len(srdd.parent.splits)
    mine = set(spmd.my_indices(nsplits, rank, world))
    numeric = srdd.kind == "reduce"
    splits = None
    if numeric and TEXT_INGEST:
        # the word-count shape: this rank's splits are tokenised AND combined on its GPU (the reference's map-side
        # combine, dpark/task.py:221-226); what is routed to the owners are the distinct (word, partial count) pairs
        from . import textingest
        text = textingest.recognize(srdd.parent)
        if text is not None:
            part = textingest.reduce_tokens(text, sorted(mine), P, thr, srdd.op, dev, ShuffleResult(P))
            if part is None:
                part = textingest.reduce_tokens_utf8(text, sorted(mine), P, thr, srdd.op, dev, ShuffleResult(P))
            if part is not None:
                ks = [k for p in range(P) for k in part.parts[p][0]]
                vs = [v for p in range(P) for v in part.parts[p][1]]
                splits = [columnar.ingest_pairs(zip(ks, vs), "textFile", True)]
    if splits is None:
        splits = _gather_parent(srdd, numeric, only=mine)
    blocks = shuffle.owner_blocks(P, world)
    tensor_in = bool(splits) and not isinstance(splits[0], columnar.Columns)
    # what every rank must agree on before any collective: key kind, value kinds, and what the one-process checks
    # read from the whole input (NaN keys of columns; the terms of the int64 sum bound, in split order)
    if tensor_in:
        kc = [k.to(dev).contiguous() for k, v in splits]
        from . import join
        desc = ("tensor", str(splits[0][0].dtype), str(splits[0][1].dtype), join.has_nan_key(kc))
    else:
        desc = ("cols", sorted(set(c.key_kind for c in splits if c.n)), sorted(set(c.val_kind for c in splits if c.n)),
                _int_sum_terms(splits) if numeric and srdd.op == "sum" else [])
    descs = spmd.all_gather_objects(desc)
    if any(d[0] == "tensor" for d in descs):
        if not all(d[0] == "tensor" or d[1] == [] for d in descs):
            raise TypeError("mixed columnar and row inputs in one shuffle are not supported on the GPU path")
        from . import join
        join.reject_nan_keys((), flag=any(d[0] == "tensor" and d[3] for d in descs))
        kd = next(d for d in descs if d[0] == "tensor")
        kdt, vdt = getattr(torch, kd[1].split(".")[1]), getattr(torch, kd[2].split(".")[1])
        kc = kc if tensor_in else [torch.empty(0, dtype=kdt, device=dev)]
        vc = [v.to(dev).contiguous() for k, v in splits] if tensor_in else [torch.empty(0, dtype=vdt, device=dev)]
        return _gathered(_device_reduce(kc, vc, P, thr, srdd.op, world), P)
    kinds = sorted(set(k for d in descs for k in d[1]))
    vkinds = set(k for d in descs for k in d[2])
    if len(kinds) > 1:
        raise TypeError("mixed key types %s in one shuffle are not supported on the GPU path" % kinds)
    kk = kinds[0] if kinds else columnar.KEY_I64
    if numeric:
        if len(vkinds) > 1:
            raise TypeError("reduceByKey values must be all int or all float on the GPU path")
        _check_int_sum_range((), vkinds, srdd.op, terms=[t for d in descs for t in d[3]])
    if numeric and kk in (columnar.KEY_I64, columnar.KEY_F64) and not ROUTE_EVERYTHING:
        def reduce_all(cols, vdt, op):
            kdt = np.int64 if kk == columnar.KEY_I64 else np.float64
            kc = [torch.from_numpy(c.keys.astype(kdt, copy=False)).to(dev) for c in cols] or \
                [torch.empty(0, dtype=torch.int64 if kk == columnar.KEY_I64 else torch.float64, device=dev)]
            vc = [torch.from_numpy(c.vals).to(dev).to(vdt) for c in cols] or [torch.empty(0, dtype=vdt, device=dev)]
            return _gathered(_device_reduce(kc, vc, P, thr, op, world), P)
        _check_int_prod_range(splits, vkinds, srdd.op, lambda logs: reduce_all(logs, torch.float64, "sum"))
        return reduce_all(splits, torch.float64 if vkinds == {columnar.VAL_F64} else torch.int64, srdd.op)
    return _gathered(_routed_shuffle(splits, kk, numeric, P, thr, srdd.op, dev, rank, world, blocks), P)


def _gathered(owned, P):
    """Every rank's {partition: columns} -> the ShuffleResult of all P partitions, on every rank.  A rank may hand in
    the exception its owner stage raised instead: every rank raises the first one, in rank order."""
    from . import spmd
    res = ShuffleResult(P)
    parts = spmd.all_gather_objects(owned)
    for part in parts:
        if isinstance(part, Exception):
            raise part
    for part in parts:
        for p, cols in part.items():
            res.parts[p] = cols
    for p in range(P):
        if res.parts[p] is None:
            res.parts[p] = ([], [])
    return res


def _device_reduce(kc, vc, P, thr, op, world):
    """Numeric reduceByKey across the ranks, columns stay on the devices: {partition: (keys, values)} for the
    partitions this rank owns."""
    from . import spmd
    rows = spmd.agree_max(sum(int(k.numel()) for k in kc))
    sb = shuffle.choose_sub_bits(max(rows, 1), P, world)      # every rank must use the same bucket layout
    parts = shuffle.reduce_by_key(kc, vc, P, op, thr, sub_bits=sb)
    return {p: (k.cpu().numpy().tolist(), v.cpu().numpy().tolist()) for p, k, v in parts}


def _routed_shuffle(splits, kk, numeric, P, thr, op, dev, rank, world, blocks):
    """Rows with Python-object values (group-by) or str / bytes keys: every row goes to the rank that owns its
    partition -- the partition id is computed by the CUDA kernels (portable_hash + getPartition), the rows travel as
    pickled host columns in one all_to_all -- and the owner runs the single-GPU shuffle over the received rows, which
    arrive in source-rank order, i.e. in map split order (splits are owned in contiguous blocks)."""
    from . import spmd
    per_dest = [([], []) for _ in range(world)]
    dest_of_part = np.zeros(P, dtype=np.int64)
    for d in range(world):
        dest_of_part[blocks[d]:blocks[d + 1]] = d
    for c in splits:
        if not c.n:
            continue
        keys = columnar.decode_keys(c.key_kind, c.keys, c.key_offsets, c.key_objs)
        vals = c.objs if c.objs is not None else c.vals.tolist()
        h = columnar._hash_column(keys)
        t = None if thr is None else torch.tensor(thr, dtype=torch.int64, device=h.device)
        pid = nv.partition_ids(h, P, t).cpu().numpy()
        dest = dest_of_part[pid]
        for d in np.unique(dest).tolist():
            idx = np.nonzero(dest == d)[0].tolist()
            per_dest[d][0].extend(keys[i] for i in idx)
            per_dest[d][1].extend(vals[i] for i in idx)
    got = spmd.all_to_all_objects(per_dest)
    local = [columnar.ingest_pairs(zip(ks, vs), "shuffle", numeric) for ks, vs in got]
    try:
        with shuffle.local_only():
            if numeric:
                r = _run_reduce(local, P, thr, op, dev)
            else:
                r = _run_group(local, P, thr, dev)
    except Exception as e:      # raised on this owner alone (the int64 product check of its keys): _gathered raises
        return e                # it on every rank instead of leaving the others waiting in the next collective
    return {p: r.parts[p] for p in range(blocks[rank], blocks[rank + 1])}


def _key_kind_of(splits):
    kinds = set(c.key_kind for c in splits if isinstance(c, columnar.Columns) and c.n)
    if len(kinds) > 1:
        raise TypeError("mixed key types %s in one shuffle are not supported on the GPU path" % sorted(kinds))
    return kinds.pop() if kinds else columnar.KEY_I64


def _run_reduce(splits, P, thr, op, dev):
    res = ShuffleResult(P)
    if not splits:                  # a parent without splits (an empty file): P empty partitions, as group_by_key gives
        res.parts = [([], []) for _ in range(P)]
        return res
    tensor_in = not isinstance(splits[0], columnar.Columns)
    if tensor_in:
        from . import join
        kc = [k.to(dev).contiguous() for k, v in splits]
        join.reject_nan_keys(kc)
        vc = [v.to(dev).contiguous() for k, v in splits]
        parts = shuffle.reduce_by_key(kc, vc, P, op, thr)
        for p, k, v in parts:
            res.parts[p] = (k.cpu().numpy().tolist(), v.cpu().numpy().tolist())
        return res
    kk = _key_kind_of(splits)
    vkinds = set(c.val_kind for c in splits if c.n)
    if len(vkinds) > 1:
        raise TypeError("reduceByKey values must be all int or all float on the GPU path")
    _check_int_sum_range(splits, vkinds, op)
    _check_int_prod_range(splits, vkinds, op, lambda logs: _run_reduce(logs, P, thr, "sum", dev))
    if kk in (columnar.KEY_I64, columnar.KEY_F64):
        kdt = np.int64 if kk == columnar.KEY_I64 else np.float64
        kc = [torch.from_numpy(c.keys.astype(kdt, copy=False)).to(dev) for c in splits]
        vc = [torch.from_numpy(c.vals).to(dev) for c in splits]
        if vkinds:
            vdt = torch.int64 if vkinds == {columnar.VAL_I64} else torch.float64
            vc = [v.to(vdt) for v in vc]
        parts = shuffle.reduce_by_key(kc, vc, P, op, thr)
        for p, k, v in parts:
            res.parts[p] = (k.cpu().numpy().tolist(), v.cpu().numpy().tolist())
        return res
    from . import strings
    return strings.reduce_by_key_bytes(splits, kk, P, thr, op, dev, res)


def _int_sum_terms(splits):
    """The terms of _check_int_sum_range: sum |v| of each split, in split order."""
    return [float(np.abs(c.vals.astype(np.float64)).sum()) for c in splits if c.n]


def _check_int_sum_range(splits, vkinds, op, terms=None):
    """The reference adds Python big ints; the device accumulates in int64.  A cheap sufficient check on the ingested
    columns: if the sum of |v| over the whole shuffle stays below 2^63 no key's sum can wrap.  terms: the
    _int_sum_terms of every split of a distributed shuffle, gathered from the ranks in split order (splits is then
    not read), so that every rank adds the same terms in the same order as one process does."""
    if vkinds == {columnar.VAL_I64} and op == "sum":
        bound = sum(_int_sum_terms(splits) if terms is None else terms)
        if bound >= 2.0 ** 63:
            raise OverflowError("reduceByKey(add): the values' magnitudes sum to %.3g >= 2^63; int64 accumulation on "
                                "the GPU path could wrap where the reference's big ints do not" % bound)


PROD_LOG2_LIMIT = 63 - 1e-9


def _check_int_prod_range(splits, vkinds, op, reduce_sum):
    """The reference multiplies Python big ints; the device multiplies int64 modulo 2^64.  That is exact whenever a
    key's final product fits (wrapped intermediates cancel out, and a zero factor makes the exact 0), so only the
    final magnitude matters: the same reduce, run by `reduce_sum` over log2|v| as float64 sums (a zero gives -inf),
    must keep every key below 2^63.  Like the sum check this is sufficient and conservative at the boundary: the
    margin of 1e-9 covers the rounding of the log sums (at most 63 terms of |v| >= 2 can stay below the limit), so a
    product within a factor 1 - 7e-10 of 2^63, -2^63 included, is refused although it fits."""
    if vkinds != {columnar.VAL_I64} or op != "prod":
        return
    logs = []
    for c in splits:
        with np.errstate(divide="ignore"):
            lv = np.log2(np.abs(c.vals.astype(np.float64)))
        logs.append(columnar.Columns(c.n, c.key_kind, c.keys, c.key_offsets, columnar.VAL_F64, lv,
                                     key_objs=c.key_objs))
    res = reduce_sum(logs)
    worst = max((max(vals) for _, vals in res.parts if len(vals)), default=float("-inf"))
    if worst >= PROD_LOG2_LIMIT:
        raise OverflowError("reduceByKey(mul): a key's integer product has |p| = 2^%.9f, not clearly below 2^63; int64 "
                            "multiplication on the GPU path would wrap where the reference's big ints do not (the check "
                            "is conservative at the boundary: [-2] * 63 is refused although -2**63 fits)" % worst)


def _run_group(splits, P, thr, dev):
    from . import grouping
    return grouping.group_by_key(splits, P, thr, dev, ShuffleResult(P))
