"""The shuffle engine: map-side hash-partition, exchange, reduce-side merge over
columnar partitions held as torch CUDA tensors.

Mirrors, for the hot path only (SURVEY.md §8a):
  ShuffleMapTask._run          dpark/task.py:197-255      -> map_side()
  ShuffleFetcher.fetch         dpark/shuffle.py:309-420   -> exchange()  (one NCCL alltoallv; the NVLink
                                                             peer-memory forms live in dpark_b200/peer.py)
  DiskHashMerger._merge        dpark/shuffle.py:600-608   -> reduce_side()
  MapOutputTracker             dpark/shuffle.py:809-826   -> the counts matrix

Layout.  The map side writes ONE bucket-major buffer per rank.  Buckets are the
reference's P reduce partitions, each refined into 2^sub_bits sub-buckets by
other hash bits (dpk_partition, include/dpark_b200.h): partition p is the
concatenation of its sub-buckets, so everything the reference defines (which
keys a partition owns, row order inside a bucket where it is observable) is
unchanged, while the reduce side gets bounded working sets.

Ownership across G ranks: reduce partition r lives on rank r // ceil(P/G)
(contiguous blocks), so what a rank sends to one peer is one contiguous range of
its buffer.  Map splits are assigned to ranks in contiguous blocks too, so
"source rank order" == "map_id order".
"""
import torch

from . import _native as nv

# rows the reduce side wants in a fine bucket (second-level split, merged in shared memory: dpk_combine.cu,
# implementation 2) and the widest second-level split it can do
FINE_BUCKET_ROWS = 1536
MAX_SECOND_LEVEL = 1024
TARGET_BUCKET_ROWS = FINE_BUCKET_ROWS * MAX_SECOND_LEVEL      # upper end of a first-level bucket (all ranks' rows)
MAX_FIRST_LEVEL = 512        # map-side bucket runs of a 4096-row tile stay >= 8 rows (64 B); 1024 only when forced


def owner_blocks(P, G):
    """[first partition of rank g for g in 0..G] (len G+1), contiguous blocks."""
    per = (P + G - 1) // G
    return [min(P, g * per) for g in range(G + 1)]


def choose_sub_bits(rows, P, world=1):
    """Sub-bucket bits of the map side (first split level) for `rows` rows PER RANK on `world` ranks.

    The job needs rows * world / FINE_BUCKET_ROWS fine buckets in all; they are reached in two levels, the map
    side's P << sub_bits buckets and the reduce side's second-level split (<= 1024-way).  The first level takes about
    twice the square root of the total, leaning on the map side: on an H100 the C2 step (1e8 rows, 8 partitions, one
    GPU) ran in 6.54 ms with 512 x 128 fine buckets against 6.73 ms with 256 x 256, the second-level split losing
    more than the map-side multisplit gains.  The first level stays at <= 512 buckets so that the bucket runs of a
    map-side tile stay long (512 from 1 GPU and 1e8 rows up, 512 x 1024 at 8 GPUs), and grows to 1024 only when the
    second level could not absorb the rest."""
    total = float(rows) * max(1, world)
    nf = total / FINE_BUCKET_ROWS
    if nf <= P:
        return 0
    want = min(float(MAX_FIRST_LEVEL), 2.0 * nf ** 0.5)
    sb = 0
    while sb < 12 and (P << (sb + 1)) <= min(nv.MAX_PARTITIONS, MAX_FIRST_LEVEL) and (P << sb) < want:
        sb += 1
    while sb < 12 and (P << (sb + 1)) <= min(nv.MAX_PARTITIONS, 1024) and total / float(P << sb) > TARGET_BUCKET_ROWS:
        sb += 1
    return sb


def bind_to_gpu_numa_node(local_rank):
    """Pin this process (and with it the pinned host buffers it allocates from now on: first touch) to the CPUs of
    the NUMA node GPU `local_rank` hangs off, so that host-to-device copies of pinned buffers do not cross the socket
    interconnect when several ranks share a host (not measured on H100 machines).  Returns the
    node number, or None when the topology cannot be read (nothing is changed then)."""
    import os
    try:
        props = torch.cuda.get_device_properties(local_rank)
        bus = "%04x:%02x:%02x.0" % (props.pci_domain_id, props.pci_bus_id, props.pci_device_id)
        with open("/sys/bus/pci/devices/%s/numa_node" % bus) as f:
            node = int(f.read().strip())
        if node < 0:
            return None
        with open("/sys/devices/system/node/node%d/cpulist" % node) as f:
            spec = f.read().strip()
        cpus = set()
        for part in spec.split(","):
            if "-" in part:
                lo, hi = part.split("-")
                cpus.update(range(int(lo), int(hi) + 1))
            elif part:
                cpus.add(int(part))
        allowed = cpus & set(os.sched_getaffinity(0))
        if not allowed:
            return None
        os.sched_setaffinity(0, allowed)
        return node
    except Exception:
        return None


class MapOutput(object):
    """Bucket-major output of the map side on one rank: the alltoallv send buffer.  rows: None, or the packed [n, 2]
    buffer of (key, value) records that keys and vals are strided column views of (see map_side)."""
    __slots__ = ("keys", "vals", "offsets", "P", "sub_bits", "rows")

    def __init__(self, keys, vals, offsets, P, sub_bits, rows=None):
        self.keys, self.vals, self.offsets, self.P, self.sub_bits = keys, vals, offsets, P, sub_bits
        self.rows = rows

    def unpacked(self):
        """This map output with contiguous key and value columns (an exchange between ranks moves columns)."""
        if self.rows is None:
            return self
        return MapOutput(self.keys.contiguous(), self.vals.contiguous(), self.offsets, self.P, self.sub_bits)


def _as_one(chunks):
    """One tensor spanning `chunks` if they are consecutive contiguous slices of the same storage, else None.
    Positions are storage offsets: an empty slice's data_ptr() is not its place in the buffer, and a map split may be
    empty."""
    first = chunks[0]
    if first is None or not first.is_contiguous():
        return None
    base = first.untyped_storage().data_ptr()
    at, total = first.storage_offset(), 0
    for c in chunks:
        if (c is None or c.dtype != first.dtype or c.dim() != 1 or not c.is_contiguous() or c.storage_offset() != at
                or c.untyped_storage().data_ptr() != base):
            return None
        at += c.numel()
        total += c.numel()
    return torch.empty(0, dtype=first.dtype, device=first.device).set_(first.untyped_storage(), first.storage_offset(), (total,))


def map_side(key_chunks, val_chunks, P, thresholds=None, prehashed=False, sub_bits=0, row_hash=None,
             unordered=False):
    """Hash-partition all local map splits into ONE bucket-major buffer.

    key_chunks/val_chunks: lists of CUDA tensors (the rank's map splits in map_id
    order).  Rows of a bucket are ordered by (map split, position) -- the order
    OrderedGroupByDiskHashMerger produces (dpark/shuffle.py:626-646).

    Packed rows: an unordered (reduceByKey) split of hashed keys with values of the key's width, whose exchange is the
    identity (one rank, or inside local_only), writes one [n, 2] buffer of (key, value) records instead of two columns
    -- the multisplit stores half as many, twice as long bucket runs and the reduce side reads one record per row.  The
    MapOutput then carries that buffer as `rows`, and keys / vals are strided views of it."""
    F = P << sub_bits
    packed = (unordered and val_chunks[0] is not None and _world() == 1
              and nv.packable(key_chunks[0], val_chunks[0], prehashed))
    if len(key_chunks) > 1:
        # map splits that are consecutive slices of one buffer (the usual case: a batch copied to the device and
        # cut into map tasks) are partitioned in ONE launch pair: rows of a bucket stay in (split, position) order
        # because that IS the buffer's row order; 2 launches instead of 2 per split, no per-split tails
        whole_k, whole_v = _as_one(key_chunks), (_as_one(val_chunks) if val_chunks[0] is not None else None)
        if whole_k is not None and (val_chunks[0] is None or whole_v is not None) and whole_k.numel() < (1 << 31):
            key_chunks, val_chunks = [whole_k], [whole_v]
    if len(key_chunks) == 1:
        k, v, off = nv.partition(key_chunks[0], val_chunks[0], P, thresholds, prehashed, sub_bits, row_hash, unordered,
                                 packed)
        if packed:
            return MapOutput(*nv.packed_views(k, key_chunks[0].dtype, val_chunks[0].dtype), off, P, sub_bits, rows=k)
        return MapOutput(k, v, off, P, sub_bits)
    dev = key_chunks[0].device
    counts, wss = [], []
    for k in key_chunks:
        c, ws = nv.partition_count(k, P, thresholds, prehashed, sub_bits, None, row_hash, unordered)
        counts.append(c)
        wss.append(ws)
    cm = torch.stack(counts)                       # [M, F]
    tot = cm.sum(0)                                # rows per bucket
    offsets = torch.zeros(F + 1, dtype=torch.int64, device=dev)
    torch.cumsum(tot, 0, out=offsets[1:])
    # base[m][b] = offsets[b] + rows of bucket b in earlier splits
    base = offsets[:-1].unsqueeze(0) + (torch.cumsum(cm, 0) - cm)
    n = sum(int(k.numel()) for k in key_chunks)
    has_v = val_chunks[0] is not None
    if packed:
        rows = nv.packed_rows(n, key_chunks[0].dtype, dev)
        out_k, out_v = rows, None
    else:
        out_k = torch.empty(n, dtype=key_chunks[0].dtype, device=dev)
        out_v = torch.empty(n, dtype=val_chunks[0].dtype, device=dev) if has_v else None
    for m, (k, v) in enumerate(zip(key_chunks, val_chunks)):
        nv.partition_scatter(k, v, P, base[m].contiguous(), out_k, out_v, wss[m], thresholds, prehashed, sub_bits,
                             row_hash, unordered)
    if packed:
        return MapOutput(*nv.packed_views(rows, key_chunks[0].dtype, val_chunks[0].dtype), offsets, P, sub_bits,
                         rows=rows)
    return MapOutput(out_k, out_v, offsets, P, sub_bits)


class Received(object):
    """Rows fetched for the partitions this rank owns.  keys/vals are laid out
    source-rank-major, then bucket-major; seg[s][b] = rows from source s for
    local fine bucket b.  rows: the packed buffer keys / vals view, when the rows arrived packed (MapOutput.rows)."""
    __slots__ = ("keys", "vals", "seg", "part_first", "nparts", "sub_bits", "bound", "rows")

    def __init__(self, keys, vals, seg, part_first, nparts, sub_bits, bound=False, rows=None):
        self.keys, self.vals, self.seg = keys, vals, seg
        self.rows = rows
        self.part_first, self.nparts, self.sub_bits = part_first, nparts, sub_bits
        # bound: keys/vals are a whole receive buffer (an upper bound of the rows); the rows actually received are
        # seg.sum() and stay on the device (no host sync on the reduceByKey path)
        self.bound = bound


_LOCAL_ONLY = [0]


class local_only(object):
    """`with shuffle.local_only():` -- the shuffles inside run on THIS rank's rows alone even under torch.distributed
    (the owner-side stage of dpark_b200.engine._routed_shuffle: the rows were already brought to their owner)."""

    def __enter__(self):
        _LOCAL_ONLY[0] += 1

    def __exit__(self, *a):
        _LOCAL_ONLY[0] -= 1


def exchange(mo, group=None):
    """ShuffleFetcher replacement: one alltoallv of the bucket-major buffers
    (torch.distributed all_to_all_single with split sizes == grouped
    ncclSend/ncclRecv over NVLink).  With one rank it is the identity."""
    import torch.distributed as dist
    G = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized() and not _LOCAL_ONLY[0]) else 1
    P, sb = mo.P, mo.sub_bits
    if G == 1:
        seg = (mo.offsets[1:] - mo.offsets[:-1]).unsqueeze(0)
        return Received(mo.keys, mo.vals, seg, 0, P, sb, rows=mo.rows)
    mo = mo.unpacked()
    rank = dist.get_rank(group)
    F = P << sb
    blocks = [b << sb for b in owner_blocks(P, G)]                  # in fine buckets
    counts = (mo.offsets[1:] - mo.offsets[:-1]).contiguous()        # [F] rows I hold per bucket
    all_counts = torch.empty(G * F, dtype=torch.int64, device=counts.device)
    dist.all_gather_into_tensor(all_counts, counts, group=group)    # MapOutputTracker
    all_counts = all_counts.view(G, F)
    host_counts = all_counts.cpu()                                  # split sizes must be known on the host
    send_splits = [int(host_counts[rank, blocks[d]:blocks[d + 1]].sum()) for d in range(G)]
    b0, b1 = blocks[rank], blocks[rank + 1]
    recv_splits = [int(host_counts[s, b0:b1].sum()) for s in range(G)]
    nrecv = sum(recv_splits)
    rk = torch.empty(nrecv, dtype=mo.keys.dtype, device=mo.keys.device)
    dist.all_to_all_single(rk, mo.keys, recv_splits, send_splits, group=group)
    rv = None
    if mo.vals is not None:
        rv = torch.empty(nrecv, dtype=mo.vals.dtype, device=mo.vals.device)
        dist.all_to_all_single(rv, mo.vals, recv_splits, send_splits, group=group)
    seg = all_counts[:, b0:b1].contiguous()
    return Received(rk, rv, seg, b0 >> sb, (b1 - b0) >> sb, sb)


def reduce_side(rx, op, P, thresholds=None):
    """DiskHashMerger._merge over everything received.  Returns
    (keys, vals, part_offsets[nparts+1], counts[nparts]): distinct keys of local
    partition j are keys[part_offsets[j] : part_offsets[j] + counts[j]]."""
    dev = rx.keys.device
    if rx.nparts == 0:
        z = torch.zeros(1, dtype=torch.int64, device=dev)
        return rx.keys[:0], (rx.vals[:0] if rx.vals is not None else None), z, z[:0]
    return nv.combine(rx.keys, rx.vals, op, P, rx.seg.contiguous(), rx.part_first, rx.nparts, thresholds,
                      rx.sub_bits, rows=rx.rows)


RADIX_BITS = 8


def sort_by_key_bits(keys, vals, bits=None):
    """Stable LSD radix sort of (int64 key bits, 8-byte payload) with the multisplit
    passes; digit windows in which all keys agree are skipped."""
    bits = bits or RADIX_BITS
    n = int(keys.numel())
    if n <= 1:
        return keys, vals
    ormask = int(nv.key_or(keys).item()) & 0xFFFFFFFFFFFFFFFF      # tiny host read: which digits differ
    ws = nv.partition_workspace(1 << bits, keys.device)
    src_k, src_v = keys, vals
    dst_k, dst_v = torch.empty_like(keys), (None if vals is None else torch.empty_like(vals))
    spare_k = spare_v = None
    shift = 0
    while shift < 64:
        width = min(bits, 64 - shift)
        if (ormask >> shift) & ((1 << width) - 1):
            nv.radix_pass(src_k, src_v, shift, width, dst_k, dst_v, ws)
            if src_k is keys:      # never write into the caller's buffers
                spare_k, spare_v = torch.empty_like(keys), (None if vals is None else torch.empty_like(vals))
                src_k, src_v, dst_k, dst_v = dst_k, dst_v, spare_k, spare_v
            else:
                src_k, src_v, dst_k, dst_v = dst_k, dst_v, src_k, src_v
        shift += width
    return src_k, src_v


def group_side(rx, P, thresholds=None, key_view=None, row_hash=None):
    """Reduce side of groupByKey (OrderedGroupByDiskHashMerger, dpark/shuffle.py:626-646): a stable sort of the
    received rows by key INSIDE every first-level hash bucket (all rows of a key share a bucket, so no pass over the
    partition id is needed: round 1 sorted the whole buffer by key bits and partitioned it again), then CSR heads.

    The first pass takes the (source rank, bucket) segments as the exchange delivered them and writes bucket-major;
    the later passes run bucket by bucket (`dpk_radix_pass_seg`), one per 8-bit digit in which any two keys differ.
    rx.keys: int64 key bits (float keys: their canonical bits).  thresholds / key_view / row_hash are accepted for
    compatibility and unused (the buckets already are what the partitioner decided on the map side).
    Returns (group_keys, group_starts, ngroups, values, part_offsets[nparts+1]); group g holds
    values[group_starts[g] : group_starts[g+1]], groups are partition-major; part_offsets are the value-row offsets of
    the partitions this rank owns."""
    if row_hash is not None:
        raise NotImplementedError("row-id keys are handled by dpark_b200.grouping")
    dev = rx.keys.device
    seg = rx.seg.contiguous()
    if rx.bound:   # the sort sizes its buffers on the host
        nrecv = int(seg.sum().item())
        rx = Received(rx.keys[:nrecv], None if rx.vals is None else rx.vals[:nrecv], seg, rx.part_first, rx.nparts,
                      rx.sub_bits)
    k, v = rx.keys.view(torch.int64), rx.vals
    n = int(k.numel())
    nsrc, F = int(seg.shape[0]), int(seg.shape[1])
    bucket_rows = seg.sum(0, keepdim=True).contiguous()                 # [1, F]
    if n > 1:
        ormask = int(nv.key_or(k).item()) & 0xFFFFFFFFFFFFFFFF          # tiny host read: which digits differ
        cur = seg
        for shift in range(0, 64, RADIX_BITS):
            if (ormask >> shift) & ((1 << RADIX_BITS) - 1):
                k, v = nv.radix_pass_seg(k, v, shift, RADIX_BITS, cur)
                cur = bucket_rows
        if cur is seg and nsrc > 1:                                     # one key only: still make the rows bucket-major
            k, v = nv.radix_pass_seg(k, v, 0, 1, cur)
    gk, gs, ng = nv.group_heads(k)
    off = torch.zeros(rx.nparts + 1, dtype=torch.int64, device=dev)
    if rx.nparts:
        torch.cumsum(bucket_rows.view(rx.nparts, -1).sum(1), 0, out=off[1:])
    return gk, gs, ng, v, off


def _world(group=None):
    import torch.distributed as dist
    return dist.get_world_size(group) if (dist.is_available() and dist.is_initialized() and not _LOCAL_ONLY[0]) else 1


def check_counts(cnt_h):
    """out_counts of the reduce side on the host: -1 marks a partition whose merge overflowed beyond recovery
    (more distinct keys in one fine bucket than its hash bits can split: dpk_aggregate2.cuh)."""
    if any(c < 0 for c in cnt_h):
        raise nv.NativeError("reduce side: a fine bucket overflowed its shared-memory table beyond the splittable hash "
                             "bits; the partition's result is invalid (dpk_combine out_counts = -1)")


def nan_key_flag(keys):
    """Device flag: the float key column holds a NaN (None for integer keys).  Read by check_nan_flag once the batch's
    result sizes have been read back, so that no extra host sync is needed."""
    return torch.isnan(keys).any() if keys.dtype.is_floating_point else None


def check_nan_flag(flag):
    """TypeError for NaN keys, as the engine raises (join.reject_nan_keys): CPython hashes NaN by identity, so every
    NaN row is a key of its own there, while the device would merge NaNs with equal bits."""
    if flag is not None and bool(flag):
        raise TypeError("NaN keys are not supported (CPython hashes NaN by identity)")


class HostShuffle(object):
    """End-to-end reduceByKey for HOST-resident columns, one batch at a time: the serial form of
    HostShuffleStream (depth 1).  Per call: pinned host -> device copy of every map split, map_side,
    exchange, reduce_side, device -> pinned host copy of every partition's distinct (key, combined)
    rows.  Buffers are allocated once and reused: the views run() returns are valid until the next run().
    Float keys holding a NaN raise TypeError."""

    def __init__(self, n_rows, key_dtype, val_dtype, P, op="sum", splits=8, thresholds=None, group=None,
                 device=None, sub_bits=None, world=1, peer_exchange=None, map_combine=False):
        self.P, self.op, self.splits, self.thresholds, self.group = P, op, splits, thresholds, group
        self.map_combine = map_combine       # merge the local map output before the exchange (hot keys)
        self.peer_exchange = peer_exchange
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        self.n = n_rows
        self.sub_bits = choose_sub_bits(n_rows, P, world) if sub_bits is None else sub_bits
        self.h_keys = torch.empty(n_rows, dtype=key_dtype).pin_memory()
        self.h_vals = torch.empty(n_rows, dtype=val_dtype).pin_memory()
        self.d_keys = torch.empty(n_rows, dtype=key_dtype, device=self.device)
        self.d_vals = torch.empty(n_rows, dtype=val_dtype, device=self.device)
        self.out_keys = None
        self.out_vals = None
        self.h2d_bytes = n_rows * (self.h_keys.element_size() + self.h_vals.element_size())
        self.d2h_bytes = 0

    def _bounds(self):
        per = (self.n + self.splits - 1) // self.splits
        return [(min(self.n, i * per), min(self.n, (i + 1) * per)) for i in range(self.splits)]

    def run(self):
        kc, vc = [], []
        for a, b in self._bounds():
            self.d_keys[a:b].copy_(self.h_keys[a:b], non_blocking=True)
            self.d_vals[a:b].copy_(self.h_vals[a:b], non_blocking=True)
            kc.append(self.d_keys[a:b])
            vc.append(self.d_vals[a:b])
        nan = nan_key_flag(self.d_keys)
        px = self.peer_exchange
        if px is not None and px.mode == "fused" and not self.map_combine:
            from . import peer                 # the scatter kernel stores straight into peer memory
            rx = peer.map_side_push(px, kc, vc, self.P, self.thresholds, self.sub_bits)
        else:
            mo = map_side(kc, vc, self.P, self.thresholds, False, self.sub_bits, unordered=True)
            if self.map_combine:
                mo = combine_map_output(mo, self.op, self.thresholds)
            if px is not None:                 # block push over NVLink peer memory
                from . import peer
                rx = peer.exchange_push(px, mo)
            else:
                rx = exchange(mo, self.group)
        ok, ov, po, cnt = reduce_side(rx, self.op, self.P, self.thresholds)
        po_h, cnt_h = po.cpu().tolist(), cnt.cpu().tolist()      # the one host sync: result sizes
        check_counts(cnt_h)
        if px is not None:
            px.check()
        check_nan_flag(nan)
        nout = sum(cnt_h)
        if self.out_keys is None or self.out_keys.numel() < nout:
            self.out_keys = torch.empty(max(nout, 1), dtype=ok.dtype).pin_memory()
            self.out_vals = torch.empty(max(nout, 1), dtype=ov.dtype).pin_memory()
        res, at = [], 0
        for j in range(rx.nparts):
            a, c = po_h[j], cnt_h[j]
            self.out_keys[at:at + c].copy_(ok[a:a + c], non_blocking=True)
            self.out_vals[at:at + c].copy_(ov[a:a + c], non_blocking=True)
            res.append((rx.part_first + j, self.out_keys[at:at + c], self.out_vals[at:at + c]))
            at += c
        torch.cuda.current_stream().synchronize()
        self.d2h_bytes = nout * (ok.element_size() + ov.element_size())
        return res


class HostShuffleStream(object):
    """Streaming shuffle for back-to-back batches of HOST-resident columns: `depth` batches are in flight on their
    own CUDA streams, so the host->device copy of batch i+1 runs while batch i is reduced and its result is copied
    back (PCIe is full duplex, the copy engines are separate).  Works on one GPU and, under torch.distributed, on
    every rank of the job at once (each slot then owns its PeerExchange: symmetric receive buffers + barrier state,
    so batches in flight never share a receive buffer; all ranks must submit/collect in the same order).

        s = HostShuffleStream(n, torch.int64, torch.int64, P)        # kind="group": groupByKey (CSR result)
        s.submit(h_keys, h_vals)            # pinned host columns of THIS rank; returns immediately
        s.submit(h_keys2, h_vals2)
        parts = s.collect()                 # result of the OLDEST batch for the partitions this rank owns

    reduce: [(partition, keys, combined values)]; group: [(partition, group keys, group starts, values)] with the
    values of group g at values[starts[g]:starts[g+1]] in (map split, position) order.  All pinned-host views of the
    slot's output buffers: valid until that slot is collected again (`depth - 1` further collect() calls).

    Result dtypes.  reduce: keys in the key dtype, values in nv.acc_dtype (int64 or float64).  group: keys int64 for
    integer keys and float64 for float keys (int32 and float32 keys are widened on the device, as the engine's
    group-by does; -0.0 and 0.0 are one key, spelled 0.0), values in the value dtype.

    The copies of h_keys / h_vals run asynchronously on the slot's stream: the caller may rewrite them once that
    batch's collect() has returned, not before.  Float keys holding a NaN make that collect() raise TypeError (the
    slot is free again afterwards).
    """

    class _Slot(object):
        pass

    def __init__(self, n_rows, key_dtype, val_dtype, P, op="sum", splits=8, thresholds=None, device=None,
                 sub_bits=None, depth=2, kind="reduce", peer_mode="push", recv_factor=1.25, group=None):
        if kind not in ("reduce", "group"):
            raise ValueError("kind must be 'reduce' or 'group'")
        self.P, self.op, self.splits, self.thresholds, self.kind, self.group = P, op, splits, thresholds, kind, group
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        self.n = n_rows
        self.world = _world(group)
        self.sub_bits = choose_sub_bits(n_rows, P, self.world) if sub_bits is None else sub_bits
        cap = n_rows if self.world == 1 else int(n_rows * recv_factor) + (1 << 16)
        self.capacity = cap
        ksz = torch.empty(0, dtype=key_dtype).element_size()
        vsz = torch.empty(0, dtype=val_dtype).element_size()
        out_vdt = nv.acc_dtype(val_dtype) if kind == "reduce" else val_dtype
        # group: the radix sort orders int64 key bits, so keys go in widened (float keys as canonical float64)
        wide_kdt = torch.float64 if key_dtype.is_floating_point else torch.int64
        out_kdt = key_dtype if kind == "reduce" else wide_kdt
        self.slots = []
        for _ in range(depth):
            s = self._Slot()
            s.stream = torch.cuda.Stream(device=self.device)
            s.d_keys = torch.empty(n_rows, dtype=key_dtype, device=self.device)
            s.d_vals = torch.empty(n_rows, dtype=val_dtype, device=self.device)
            s.d_wide = None
            if kind == "group" and key_dtype != wide_kdt:
                s.d_wide = torch.empty(n_rows, dtype=wide_kdt, device=self.device)
            s.out_keys = torch.empty(cap, dtype=out_kdt).pin_memory()
            s.out_vals = torch.empty(cap, dtype=out_vdt).pin_memory()
            s.out_starts = torch.empty(cap + 1, dtype=torch.int64).pin_memory() if kind == "group" else None
            s.px = None
            if self.world > 1 and peer_mode is not None:
                from . import peer
                s.px = peer.PeerExchange(cap, out_kdt, val_dtype, self.device, group=group, mode="push")
            s.busy = False
            self.slots.append(s)
        self.next_submit = 0
        self.next_collect = 0
        self.h2d_bytes = n_rows * (ksz + vsz)
        self.d2h_bytes = 0

    def submit(self, h_keys, h_vals):
        s = self.slots[self.next_submit % len(self.slots)]
        if s.busy:
            raise RuntimeError("all %d slots are in flight: collect() first" % len(self.slots))
        self.next_submit += 1
        per = (self.n + self.splits - 1) // self.splits
        bounds = [(min(self.n, i * per), min(self.n, (i + 1) * per)) for i in range(self.splits)]
        with torch.cuda.stream(s.stream):
            for a, b in bounds:
                s.d_keys[a:b].copy_(h_keys[a:b], non_blocking=True)
                s.d_vals[a:b].copy_(h_vals[a:b], non_blocking=True)
            s.nan = nan_key_flag(s.d_keys)
            keys = s.d_keys
            if self.kind == "group":
                if s.d_wide is not None:
                    keys = s.d_wide
                    keys.copy_(s.d_keys)
                if keys.dtype.is_floating_point:
                    keys.add_(0.0)             # -0.0 and 0.0 are one key, spelled 0.0
            kc = [keys[a:b] for a, b in bounds]
            vc = [s.d_vals[a:b] for a, b in bounds]
            mo = map_side(kc, vc, self.P, self.thresholds, False, self.sub_bits, unordered=self.kind == "reduce")
            if s.px is not None:
                from . import peer
                rx = peer.exchange_push(s.px, mo, need_host_count=self.kind == "group")
            else:
                rx = exchange(mo, self.group)
            if self.kind == "reduce":
                s.result = reduce_side(rx, self.op, self.P, self.thresholds)
            else:
                s.result = group_side(rx, self.P, self.thresholds)
            s.nparts, s.part_first = rx.nparts, rx.part_first
        s.busy = True

    def collect(self):
        s = self.slots[self.next_collect % len(self.slots)]
        if not s.busy:
            raise RuntimeError("nothing in flight")
        self.next_collect += 1
        try:
            with torch.cuda.stream(s.stream):
                res = self._collect_reduce(s) if self.kind == "reduce" else self._collect_group(s)
                s.stream.synchronize()
                if s.px is not None:
                    s.px.check()
            check_nan_flag(s.nan)
        finally:
            s.result = None
            s.busy = False
        return res

    def _collect_reduce(self, s):
        ok, ov, po, cnt = s.result
        po_h, cnt_h = po.cpu().tolist(), cnt.cpu().tolist()      # waits for THIS batch only
        check_counts(cnt_h)
        res, at = [], 0
        for j in range(s.nparts):
            a, c = po_h[j], cnt_h[j]
            s.out_keys[at:at + c].copy_(ok[a:a + c], non_blocking=True)
            s.out_vals[at:at + c].copy_(ov[a:a + c], non_blocking=True)
            res.append((s.part_first + j, s.out_keys[at:at + c], s.out_vals[at:at + c]))
            at += c
        self.d2h_bytes = at * (ok.element_size() + ov.element_size())
        return res

    def _collect_group(self, s):
        gk, gs, ng, ov, off = s.result
        G = int(ng.item())                                           # waits for THIS batch only
        off_h = off.cpu().tolist()
        nval = int(ov.numel())
        s.out_keys[:G].copy_(gk[:G].view(s.out_keys.dtype), non_blocking=True)
        s.out_starts[:G + 1].copy_(gs[:G + 1], non_blocking=True)
        s.out_vals[:nval].copy_(ov, non_blocking=True)
        s.stream.synchronize()
        starts = s.out_starts[:G + 1]
        first = torch.searchsorted(starts[:-1].contiguous(), torch.tensor(off_h, dtype=torch.int64)).tolist() if G else \
            [0] * len(off_h)
        res = []
        for j in range(s.nparts):
            g0, g1 = first[j], first[j + 1]
            res.append((s.part_first + j, s.out_keys[g0:g1], s.out_starts[g0:g1 + 1], s.out_vals))
        self.d2h_bytes = G * 8 + (G + 1) * 8 + nval * ov.element_size()
        return res

    def close(self):
        for s in self.slots:
            if s.px is not None:
                s.px.close()
                s.px = None
        self.slots = []


def combine_map_output(mo, op, thresholds=None):
    """Map-side combine: the dict upsert of ShuffleMapTask._run (dpark/task.py:222-226,
    `buckets[i][k] = mergeValue(buckets[i][k], v)`), which the reference always does so that a key
    leaves a map task at most once per reducer.  Here it is an OPTION (reduce_by_key(map_combine=True)):
    with mostly distinct keys it is a wasted merge pass, with hot keys (Zipf, word counts) it shrinks the
    exchange and takes the skew out of it -- every rank sends ONE row per key it holds, so the rank
    owning the hottest key receives G rows for it, not a tenth of the data set.

    The rank's whole map output is merged locally (the reduce-side kernels over all P partitions,
    one "source"), the distinct rows are compacted and partitioned again.  Combining twice with the
    same op is exact for every op the library has (sum/min/max/prod/and/or/xor are associative and
    commutative; float sums are order-free up to the tolerance stated in DESIGN.md §7)."""
    P, sb = mo.P, mo.sub_bits
    seg = (mo.offsets[1:] - mo.offsets[:-1]).unsqueeze(0)
    ok, ov, po, cnt = reduce_side(Received(mo.keys, mo.vals, seg, 0, P, sb, rows=mo.rows), op, P, thresholds)
    po_h, cnt_h = po.cpu().tolist(), cnt.cpu().tolist()           # host read: sizes of the compacted columns
    check_counts(cnt_h)
    keys = torch.cat([ok[a:a + c] for a, c in zip(po_h, cnt_h)])
    vals = torch.cat([ov[a:a + c] for a, c in zip(po_h, cnt_h)])
    return map_side([keys], [vals], P, thresholds, False, sb, unordered=True)


def reduce_by_key(key_chunks, val_chunks, P, op="sum", thresholds=None, group=None, sub_bits=None,
                  map_combine=False):
    """Whole hot path for this rank's map splits.  Returns a list of
    (partition id, keys, vals) for the partitions this rank owns (device tensors)."""
    if sub_bits is None:
        # NOTE under torch.distributed every rank must pass the SAME sub_bits (the bucket layout is exchanged);
        # callers with uneven inputs agree on it first (dpark_b200.engine._device_reduce)
        sub_bits = choose_sub_bits(sum(int(k.numel()) for k in key_chunks), P, _world(group))
    mo = map_side(key_chunks, val_chunks, P, thresholds, False, sub_bits, unordered=True)
    if map_combine:
        mo = combine_map_output(mo, op, thresholds)
    rx = exchange(mo, group)
    ok, ov, po, cnt = reduce_side(rx, op, P, thresholds)
    po_h, cnt_h = po.cpu().tolist(), cnt.cpu().tolist()
    check_counts(cnt_h)
    return [(rx.part_first + j, ok[po_h[j]:po_h[j] + cnt_h[j]], ov[po_h[j]:po_h[j] + cnt_h[j]])
            for j in range(rx.nparts)]
