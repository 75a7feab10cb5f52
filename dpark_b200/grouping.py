"""groupByKey on the GPU shuffle (GroupByAggregator, dpark/dependency.py:107-118,
with the deterministic order of OrderedGroupByDiskHashMerger,
dpark/shuffle.py:626-646: values of a key ordered by map split, then arrival).

Values may be arbitrary Python objects, so the device shuffles ROW IDS (int64):
row i of the concatenated map splits carries value-id i; after the shuffle each
group is a run of row ids in (map split, position) order and the host picks the
objects out of the list it kept.  Keys:

  int / float   int64 key bits go through map_side -> exchange -> group_side
  str / bytes   hash_bytes + dict_encode give every row a representative row id
                (key identity by value); rows are sorted by representative id,
                partitioned by the hash of the string they stand for, and the
                group heads are found on the representative ids
"""
import numpy as np
import torch

from . import _native as nv
from . import columnar, shuffle


def _concat_objs(splits):
    objs, sizes = [], []
    for c in splits:
        objs.extend(c.objs if c.objs is not None else c.vals.tolist())
        sizes.append(c.n)
    return objs, sizes


def _emit(res, P, part_off, gkeys, gstarts, ids, objs, key_decoder):
    """Host egress: CSR -> per-partition (keys, [values...])."""
    first_group = np.searchsorted(gstarts[:-1], part_off, side="left")
    for p in range(P):
        g0, g1 = int(first_group[p]), int(first_group[p + 1])
        keys = key_decoder(gkeys[g0:g1])
        st = gstarts[g0:g1 + 1].tolist()
        idl = ids[st[0]:st[-1]].tolist() if g1 > g0 else []
        base = st[0] if g1 > g0 else 0
        vals = [[objs[i] for i in idl[st[j] - base:st[j + 1] - base]] for j in range(g1 - g0)]
        res.parts[p] = (keys, vals)
    return res


def group_row_ids(key_chunks, id_chunks, P, thresholds):
    """The numeric group-by on one GPU: map_side -> exchange -> group_side over int64 / float64 device key columns
    (the map splits in order) carrying int64 row ids.  Returns (group_keys[G] as int64 bits, group_starts[G + 1],
    ids, part_offsets[P + 1]): group g holds ids[group_starts[g] : group_starts[g + 1]] in (map split, position)
    order, groups are partition-major.  One host read (G)."""
    float_keys = key_chunks[0].dtype == torch.float64
    mo = shuffle.map_side(key_chunks, id_chunks, P, thresholds)
    rx = shuffle.exchange(mo)
    rx.keys = rx.keys.view(torch.int64)
    gk, gs, ng, ov, off = shuffle.group_side(rx, P, thresholds, key_view=torch.float64 if float_keys else None)
    G = int(ng.item())
    return gk[:G], gs[:G + 1], ov, off


def group_by_key(splits, P, thresholds, dev, res):
    if shuffle._world() > 1:
        raise NotImplementedError("this is the one-GPU stage; under torch.distributed the rows are first routed to the "
                                  "rank owning their partition (dpark_b200.engine._routed_shuffle)")
    objs, sizes = _concat_objs(splits)
    n = len(objs)
    kinds = set(c.key_kind for c in splits if c.n)
    if len(kinds) > 1:
        raise TypeError("mixed key types %s in one shuffle are not supported on the GPU path" % sorted(kinds))
    kk = kinds.pop() if kinds else columnar.KEY_I64
    if n == 0:
        for p in range(P):
            res.parts[p] = ([], [])
        return res
    bounds = np.concatenate([[0], np.cumsum(sizes)])
    if kk in (columnar.KEY_I64, columnar.KEY_F64):
        kdt = np.int64 if kk == columnar.KEY_I64 else np.float64
        kc = [torch.from_numpy(c.keys.astype(kdt, copy=False)).to(dev) for c in splits]
        vc = [torch.arange(int(bounds[i]), int(bounds[i + 1]), dtype=torch.int64, device=dev)
              for i in range(len(splits))]
        gk, gs, ov, off = group_row_ids(kc, vc, P, thresholds)
        gkeys = gk.cpu().numpy()
        if kk == columnar.KEY_F64:
            gkeys = gkeys.view(np.float64)
        return _emit(res, P, off.cpu().numpy(), gkeys, gs.cpu().numpy(), ov.cpu().numpy(), objs,
                     lambda a: a.tolist())
    # ---- str / bytes keys
    data = np.concatenate([c.keys for c in splits if c.n]) if n else np.zeros(0, np.uint8)
    offs = [np.zeros(1, np.int64)]
    base = 0
    for c in splits:
        if c.n:
            offs.append(c.key_offsets[1:] + base)
            base += int(c.key_offsets[-1])
    offsets = np.concatenate(offs)
    d_data = torch.from_numpy(data if data.size else np.zeros(1, np.uint8)).to(dev)
    d_off = torch.from_numpy(offsets).to(dev)
    key_objs = None
    if kk == columnar.KEY_TUPLE:             # identity = the canonical bytes; hash = tuple_hash of the leaves, on the device
        key_objs = [k for c in splits if c.n for k in c.key_objs]
        h = columnar.tuple_hashes_on_device(key_objs, dev)
    else:
        h = nv.hash_bytes(d_data, d_off, nv.STR_UTF8 if kk == columnar.KEY_STR else nv.BYTES_SIGNED)
    rep = nv.dict_encode(d_data, d_off, h)
    rowid = torch.arange(n, dtype=torch.int64, device=dev)
    # stable sort by representative id (rows of one string become adjacent, arrival order kept)
    rep_s, row_s = shuffle.sort_by_key_bits(rep, rowid)
    # partition-major by the hash of the string (stable: groups stay contiguous and ordered)
    h_s = nv.gather_i64(h, rep_s)
    _, row_p, off = nv.partition(h_s, row_s, P, thresholds, prehashed=True)
    rep_p = nv.gather_i64(rep, row_p)
    gk, gs, ng = nv.group_heads(rep_p)
    G = int(ng.item())
    raw = data.tobytes()
    is_str = kk == columnar.KEY_STR

    def decode(ids):
        out = []
        for r in ids.tolist():
            if key_objs is not None:
                out.append(key_objs[r])
                continue
            b = raw[offsets[r]:offsets[r + 1]]
            out.append(b.decode("utf-8", "surrogatepass") if is_str else b)
        return out
    return _emit(res, P, off.cpu().numpy(), gk[:G].cpu().numpy(), gs[:G + 1].cpu().numpy(), row_p.cpu().numpy(),
                 objs, decode)
