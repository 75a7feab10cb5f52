"""The exchange over NVLink peer memory: the map side PUSHES.

The reference's reducers PULL every map's bucket over files + HTTP (ShuffleFetcher,
dpark/shuffle.py:309-420).  shuffle.exchange() replaces that by one NCCL alltoallv.  Here every
rank maps its peers' receive buffers into its own address space (torch symmetric memory = cuMem
allocations exchanged between the ranks of one node) and writes into them directly, in one of two
forms:

  exchange_push   (mode "push", default) the map output stays local and bucket-major -- the rows
                  bound for one peer are ONE contiguous block -- and a single launch of
                  dpk_copy_segments pushes every block with full-width stores; the segment table
                  (push_plan) is computed on the device from the gathered counts matrix.
  map_side_push   (mode "fused") dpk_partition_scatter_ptrs: the scatter kernel itself stores each
                  bucket's rows into the owning GPU's buffer while it is partitioning.  No extra
                  HBM pass, but the stores are the short bucket runs of one tile, which NVLink
                  carries poorly (not the default; DESIGN.md section 5).

What remains of the collective is the small all-gather of the counts matrix (the MapOutputTracker)
and ONE stream-ordered barrier per step ("every peer's stores have landed"): the receive buffers are
double-buffered, so the step that overwrites a buffer is two barriers after the step that read it.
Nothing is read back by the host on this path: receive sizes stay on the device (the reduce side takes
them from the segment matrix), and a receive buffer that is too small raises a device flag
(PeerExchange.check(), read together with the result sizes) instead of a per-step host sync.

Layout of a receive buffer = what exchange() delivers: source-rank-major, bucket-major inside.
"""
import torch
import torch.distributed as dist

from . import _native as nv
from .shuffle import Received, owner_blocks


class PeerExchange(object):
    """Symmetric receive buffers (keys + values) of `capacity` rows on every rank, two of each
    (alternating per step)."""

    def __init__(self, capacity, key_dtype, val_dtype, device=None, group=None, mode="push", buffers=2):
        import torch.distributed._symmetric_memory as symm
        if mode not in ("push", "fused"):
            raise ValueError("mode must be 'push' (scatter locally, then block pushes) or 'fused' "
                             "(the scatter kernel stores into peer memory)")
        self.mode = mode
        self.group = group or dist.group.WORLD
        self.rank = dist.get_rank(self.group)
        self.world = dist.get_world_size(self.group)
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        self.capacity = int(capacity)
        self.nbuf = max(1, int(buffers))
        name = self.group.group_name
        self._keys, self._vals, self._hk, self._hv, self._kb, self._vb, self._db = [], [], [], [], [], [], []
        self._pk, self._pv, self._kp, self._vp = [], [], [], []
        for _ in range(self.nbuf):
            k = symm.empty(self.capacity, dtype=key_dtype, device=self.device)
            v = symm.empty(self.capacity, dtype=val_dtype, device=self.device)
            hk, hv = symm.rendezvous(k, name), symm.rendezvous(v, name)
            self._keys.append(k)
            self._vals.append(v)
            self._hk.append(hk)
            self._hv.append(hv)
            self._kb.append(torch.tensor([int(p) for p in hk.buffer_ptrs], dtype=torch.int64, device=self.device))
            self._vb.append(torch.tensor([int(p) for p in hv.buffer_ptrs], dtype=torch.int64, device=self.device))
            self._db.append(torch.cat([self._kb[-1], self._vb[-1]]).contiguous())     # [2][G] for dpk_push_plan
            # every rank's buffers as tensors of THIS process (peer memory mapped over NVLink): targets of copy-engine pushes
            self._pk.append([hk.get_buffer(r, (self.capacity,), key_dtype) for r in range(self.world)])
            self._pv.append([hv.get_buffer(r, (self.capacity,), val_dtype) for r in range(self.world)])
            self._kp.append([int(p) for p in hk.buffer_ptrs])
            self._vp.append([int(p) for p in hv.buffer_ptrs])
        self.step = 0
        self.side = torch.cuda.Stream(device=self.device, priority=-1)     # pushes that overlap the map side
        self.err = torch.zeros(1, dtype=torch.int64, device=self.device)   # max rows any rank needed beyond capacity
        self._closed = False
        self._dump = None
        # SMs an OVERLAPPED push may take (map_exchange_overlapped): the copy kernel is launched on the high-priority
        # side stream as whole-SM CTAs, the multisplit of the next group runs on the SMs that are left
        self.copy_sms = 16
        # shuffle_pipelined: 1 = the pushes are cudaMemcpyAsync calls on the side stream (the GPU's copy engines move the
        # blocks over NVLink while ALL SMs keep computing; costs one small device->host read of the segment tables per
        # step, hidden behind the multisplit); 0 = dpk_copy_segments on copy_sms SMs (nothing read by the host)
        self.copy_engine = 2      # 2 = one cudaMemcpyBatchAsync per (part, group); 1 = one cudaMemcpyAsync per block
        self.side2 = torch.cuda.Stream(device=self.device, priority=-1)
        self._tab_host = None

    # the buffer set of the current step
    @property
    def keys(self):
        return self._keys[self.step % self.nbuf]

    @property
    def vals(self):
        return self._vals[self.step % self.nbuf]

    @property
    def key_base(self):
        return self._kb[self.step % self.nbuf]

    @property
    def val_base(self):
        return self._vb[self.step % self.nbuf]

    @property
    def dst_base(self):
        return self._db[self.step % self.nbuf]

    def barrier(self):
        self._hk[self.step % self.nbuf].barrier()

    def advance(self):
        self.step += 1

    def note_need(self, need_rows):
        """Device-side capacity check: remember by how many rows the largest receive exceeded the buffers."""
        torch.maximum(self.err, (need_rows - self.capacity).reshape(1), out=self.err)

    def check(self):
        """Raise if any step since the last check() needed more rows than the receive buffers hold (one host
        read; call it where the host synchronises anyway, e.g. next to the result sizes)."""
        over = int(self.err.item())
        if over > 0:
            self.err.zero_()
            raise RuntimeError("peer receive buffer too small: a step needed %d rows, capacity %d (results of that "
                               "step are invalid)" % (self.capacity + over, self.capacity))

    def dump(self, rows, with_vals=True):
        """Local columns a fused scatter diverts overflowing buckets into (never read; sized to this rank's rows)."""
        if self._dump is None or self._dump[0].numel() < rows:
            self._dump = (torch.empty(max(rows, 1), dtype=self._keys[0].dtype, device=self.device),
                          torch.empty(max(rows, 1), dtype=self._vals[0].dtype, device=self.device))
        return self._dump[0], (self._dump[1] if with_vals else None)

    def close(self):
        """Drop the symmetric allocations (all ranks must call it)."""
        if not self._closed:
            self._closed = True
            self._keys, self._vals, self._hk, self._hv, self._kb, self._vb, self._db = [], [], [], [], [], [], []
            self._pk, self._pv = [], []


def push_plan(all_counts, blocks, rank):
    """Segment table of one rank's pushes, in rows (pure tensor arithmetic, any device).
    all_counts[s][b] = rows source s holds for fine bucket b; blocks[d]..blocks[d+1] = the buckets
    destination d owns.  Returns (send_first[d], dst_first[d], rows[d], recv_total[d]):
    my block for d starts at row send_first[d] of my bucket-major buffer, holds rows[d] rows, and
    lands at row dst_first[d] of d's receive buffer (source-rank-major: after the blocks of the
    lower ranks); recv_total[d] = rows d receives from everyone."""
    G, F = all_counts.shape
    csum = torch.zeros(G, F + 1, dtype=torch.int64, device=all_counts.device)
    csum[:, 1:] = torch.cumsum(all_counts, 1)
    bidx = torch.tensor(blocks, dtype=torch.int64, device=all_counts.device)
    edge = csum[:, bidx]                                              # [s][d]: first row of d's block at source s
    R = edge[:, 1:] - edge[:, :-1]                                    # rows s sends to d
    src_base = torch.cumsum(R, 0) - R                                 # rows of lower sources inside d's buffer
    return edge[rank, :-1].contiguous(), src_base[rank].contiguous(), R[rank].contiguous(), R.sum(0)


def _landed(seg, capacity):
    """The segment matrix of the rows that land in a receive buffer of `capacity` rows (source-major, bucket-major;
    every push is clamped at the capacity), as dpk_push_plan writes it: a reduce over an overflowed step must not read
    or size anything past the buffer."""
    flat = seg.reshape(-1)
    start = torch.cumsum(flat, 0) - flat
    return torch.minimum(flat, (capacity - start).clamp(min=0)).view(seg.shape).contiguous()


def exchange_push(px, mo, need_host_count=False):
    """shuffle.exchange() over peer memory: the bucket-major map output `mo` stays local, and ONE
    launch of dpk_copy_segments pushes each peer's contiguous block (keys and values) into that
    peer's receive buffer with full-width stores.  The segment table is computed on the device from
    the gathered counts; no host read (unless need_host_count: the group-by reduce side sizes its
    sort buffers on the host).  The returned Received views the WHOLE receive buffer (`bound` rows);
    the rows actually received are what its segment matrix says."""
    G, rank, dev = px.world, px.rank, px.device
    mo = mo.unpacked()     # the pushes move whole column blocks
    P, sb = mo.P, mo.sub_bits
    F = P << sb
    if mo.keys.dtype != px.keys.dtype or (mo.vals is not None and mo.vals.dtype != px.vals.dtype):
        raise TypeError("receive buffers are (%s, %s) but the map output is (%s, %s): allocate the PeerExchange "
                        "with the column dtypes that are exchanged (after a map-side combine the value column "
                        "is the accumulator type)" % (px.keys.dtype, px.vals.dtype, mo.keys.dtype,
                                                      None if mo.vals is None else mo.vals.dtype))
    counts = (mo.offsets[1:] - mo.offsets[:-1]).contiguous()
    all_counts = torch.empty(G * F, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(all_counts, counts, group=px.group)   # the MapOutputTracker
    all_counts = all_counts.view(G, F)
    blocks = [b << sb for b in owner_blocks(P, G)]
    per_block = ((P + G - 1) // G) << sb
    # one launch: segment table of my pushes (clamped to the receive buffers), capacity flag, my segment matrix
    src, dst, nby, seg = nv.push_plan(all_counts, G, per_block, rank, rank, mo.keys, mo.vals,
                                      px.dst_base if mo.vals is not None else px.key_base, px.capacity, px.err)
    nv.copy_segments(src, dst, nby)
    px.barrier()                                                      # every peer's stores have landed
    b0, b1 = blocks[rank], blocks[rank + 1]
    keys, vals = px.keys, (px.vals if mo.vals is not None else None)
    px.advance()                                                      # the next step writes the other buffer set
    if need_host_count:
        nrecv = min(int(seg.sum().item()), px.capacity)
        return Received(keys[:nrecv], None if vals is None else vals[:nrecv], seg, b0 >> sb, (b1 - b0) >> sb, sb)
    return Received(keys, vals, seg, b0 >> sb, (b1 - b0) >> sb, sb, bound=True)


def map_exchange_overlapped(px, key_chunks, val_chunks, P, thresholds=None, sub_bits=0, unordered=True, halves=2):
    """Map side + exchange with the push of one group of map splits running (on a side stream) while the next group is
    still being scattered.  The rank's splits are divided into `halves` contiguous groups, every group gets its own
    bucket-major buffer, and a group's blocks are pushed as soon as its scatter kernel is done; all counts are known
    after the histogram pass, so ONE all-gather describes every group.  In a receive buffer the groups of one source
    rank follow each other in split order, i.e. the layout is still (map split order)-major then bucket-major:
    `Received.seg` simply has G * halves source rows.  Groups whose splits are consecutive slices of one buffer (the
    usual case) take one launch pair each and one dpk_push_plan launch for their segment table.
    Returns the Received view (bound = the whole receive buffer) like exchange_push."""
    from . import shuffle as sh
    G, rank, dev = px.world, px.rank, px.device
    F = P << sub_bits
    M = len(key_chunks)
    H = max(1, min(halves, M))
    has_v = val_chunks[0] is not None
    bounds = [(M * h) // H for h in range(H + 1)]
    gk, gv = [], []
    for h in range(H):
        sel = slice(bounds[h], bounds[h + 1])
        k1 = sh._as_one(key_chunks[sel])
        v1 = sh._as_one(val_chunks[sel]) if has_v else None
        if k1 is None or (has_v and v1 is None) or k1.numel() >= (1 << 31):
            return _map_exchange_overlapped_splits(px, key_chunks, val_chunks, P, thresholds, sub_bits, unordered, H)
        gk.append(k1)
        gv.append(v1)
    counts, wss = [], []
    for k in gk:
        c, ws = nv.partition_count(k, P, thresholds, False, sub_bits, None, None, unordered)
        counts.append(c)
        wss.append(ws)
    gc = torch.stack(counts)                                            # [H, F] rows per group and bucket
    all_counts = torch.empty(G * H * F, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(all_counts, gc.reshape(-1), group=px.group)   # the MapOutputTracker
    all_counts = all_counts.view(G * H, F)                              # source (rank, group) major
    per_block = ((P + G - 1) // G) << sub_bits
    main = torch.cuda.current_stream()
    seg = None
    for h in range(H):
        offsets = torch.zeros(F + 1, dtype=torch.int64, device=dev)
        torch.cumsum(gc[h], 0, out=offsets[1:])
        out_k = torch.empty_like(gk[h])
        out_v = torch.empty_like(gv[h]) if has_v else None
        nv.partition_scatter(gk[h], gv[h], P, offsets, out_k, out_v, wss[h], thresholds, False, sub_bits, None, unordered)
        src, dst, nby, sg = nv.push_plan(all_counts, G, per_block, rank * H + h, rank, out_k, out_v,
                                         px.dst_base if has_v else px.key_base, px.capacity, px.err, want_seg=(h == 0))
        if h == 0:
            seg = sg
        ready = torch.cuda.Event()
        ready.record(main)
        with torch.cuda.stream(px.side):
            px.side.wait_event(ready)
            nv.copy_segments(src, dst, nby, sms=px.copy_sms if h + 1 < H else 0)   # the last push overlaps nothing
            for t in (out_k, out_v, src, dst, nby):
                if t is not None:
                    t.record_stream(px.side)
    main.wait_stream(px.side)
    px.barrier()                                                        # every peer's stores have landed
    blocks = [b << sub_bits for b in owner_blocks(P, G)]
    b0, b1 = blocks[rank], blocks[rank + 1]
    keys, vals = px.keys, (px.vals if has_v else None)
    px.advance()
    return Received(keys, vals, seg, b0 >> sub_bits, (b1 - b0) >> sub_bits, sub_bits, bound=True)


def shuffle_pipelined(px, key_chunks, val_chunks, P, op, thresholds=None, sub_bits=0, groups=2, parts=2):
    """The whole reduceByKey step of one rank with the NVLink transfer hidden behind the kernels on both sides of it.

    Two cuts, both along orders the data already has:
      * the rank's map splits are cut into `groups` (consecutive row ranges), each multisplit into its own bucket-major
        buffer; a group's blocks are pushed (side stream, a few whole SMs: PeerExchange.copy_sms) while the next
        group is being partitioned on the remaining SMs;
      * every destination's block of buckets is cut into `parts` (consecutive partitions: a rank owns `nparts`
        partitions, part q covers partitions [q * nparts / parts, (q + 1) * nparts / parts)); the first parts of ALL
        groups are pushed first, and as soon as they have landed everywhere (one barrier) the reduce side of those
        partitions (dpk_combine) starts while the later parts are still crossing NVLink into their own region of the
        receive buffers.
    The reference's reducers likewise start merging a bucket as soon as its map outputs are fetched while other
    fetches are in flight (ParallelShuffleFetcher, dpark/shuffle.py:365-420).  Nothing is read by the host.

    Needs map splits that are consecutive slices of one buffer per group and nparts divisible into `parts` (else fewer
    parts are used).  Returns [(keys, vals, part_offsets, counts, part_first, nparts)] -- one reduce_side result per
    part, in partition order; a rank that owns no partitions gets one empty part (nparts 0), so that every rank's list
    merges (merge_part_results) into a well-typed result."""
    from . import shuffle as sh
    G, rank, dev = px.world, px.rank, px.device
    F = P << sub_bits
    M = len(key_chunks)
    H = max(1, min(groups, M))
    has_v = val_chunks[0] is not None
    blocks = sh.owner_blocks(P, G)
    per_parts = (P + G - 1) // G                       # partitions per rank (the last ranks may own fewer)
    Q = max(1, min(parts, per_parts))
    while per_parts % Q:
        Q -= 1
    bounds = [(M * h) // H for h in range(H + 1)]
    gk, gv = [], []
    for h in range(H):
        sel = slice(bounds[h], bounds[h + 1])
        k1 = sh._as_one(key_chunks[sel])
        v1 = sh._as_one(val_chunks[sel]) if has_v else None
        if k1 is None or (has_v and v1 is None) or k1.numel() >= (1 << 31):
            raise ValueError("shuffle_pipelined needs every group's map splits to be consecutive slices of one buffer")
        gk.append(k1)
        gv.append(v1)
    counts, wss = [], []
    for k in gk:
        c, ws = nv.partition_count(k, P, thresholds, False, sub_bits, None, None, True)
        counts.append(c)
        wss.append(ws)
    gc = torch.stack(counts)                                            # [H, F] rows per group and bucket
    all_counts = torch.empty(G * H * F, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(all_counts, gc.reshape(-1), group=px.group)   # the MapOutputTracker
    all_counts = all_counts.view(G * H, F)                              # source (rank, group) major
    per_block = per_parts << sub_bits
    region = (px.capacity // Q) & ~15                                   # rows of one part's region in a receive buffer
    dst_base = px.dst_base if has_v else px.key_base
    pad = nv.pipe_pad_rows(G, Q, gk[0].element_size(), gv[0].element_size() if has_v else None)
    main = torch.cuda.current_stream()
    bufs, plans, bases, segs = [], [[None] * H for _ in range(Q)], [], None
    landed = [torch.cuda.Event() for _ in range(Q)]
    ce = bool(px.copy_engine)
    tabs = []
    for h in range(H):
        n_h = int(gk[h].numel())
        out_k = torch.empty(n_h + pad, dtype=gk[h].dtype, device=dev)
        out_v = torch.empty(n_h + pad, dtype=gv[h].dtype, device=dev) if has_v else None
        # one launch: where every bucket of this group goes in the send buffer (blocks padded so that every push is
        # congruent mod 16 bytes to its landing place) + the segment tables of the Q pushes + my own segment matrices
        base, src, dst, nby, sg = nv.pipe_plan(all_counts, G, per_block, Q, region, rank * H + h, rank, out_k, out_v,
                                               dst_base, px.err, want_seg=(h == 0))
        if h == 0:
            segs = sg
        bufs.append((out_k, out_v))
        bases.append(base)
        for q in range(Q):
            plans[q][h] = (src[q], dst[q], nby[q])
        tabs.append(torch.stack([src, dst, nby]))
    tab_ready = None
    if ce:      # the segment tables go to the host while the multisplit kernels run
        ncg = (2 if has_v else 1) * G
        if px._tab_host is None or tuple(px._tab_host.shape) != (H, 3, Q, ncg):
            px._tab_host = torch.empty((H, 3, Q, ncg), dtype=torch.int64).pin_memory()
        px._tab_host.copy_(torch.stack(tabs), non_blocking=True)
        tab_ready = torch.cuda.Event()
        tab_ready.record(main)
    ready = []
    for h in range(H):
        nv.partition_scatter(gk[h], gv[h], P, bases[h], bufs[h][0], bufs[h][1], wss[h], thresholds, False, sub_bits, None, True)
        ev = torch.cuda.Event()
        ev.record(main)
        ready.append(ev)
    kset, vset = px._pk[px.step % px.nbuf], px._pv[px.step % px.nbuf]
    kptr, vptr = px._kp[px.step % px.nbuf], px._vp[px.step % px.nbuf]
    if ce:
        tab_ready.synchronize()
        tab = px._tab_host.numpy()
        ksz = gk[0].element_size()
        vsz = gv[0].element_size() if has_v else 0

    def push(q, h):
        """Part q of group h to every rank (current stream)."""
        if not ce:
            nv.copy_segments(*plans[q][h], sms=px.copy_sms)
            return
        if px.copy_engine == 2:     # one cudaMemcpyBatchAsync for the whole table of this (part, group)
            order = [(rank + 1 + i) % G for i in range(G)]          # staggered: no two ranks start on the same destination
            cols = [c * G + d for d in order for c in range(2 if has_v else 1)]
            nv.memcpy_batch([int(tab[h, 1, q, o]) for o in cols], [int(tab[h, 0, q, o]) for o in cols],
                            [int(tab[h, 2, q, o]) for o in cols])
            return
        out_k, out_v = bufs[h]
        k0 = out_k.data_ptr()
        v0 = out_v.data_ptr() if has_v else 0
        for i in range(G):
            d = (rank + 1 + i) % G
            rows = int(tab[h, 2, q, d]) // ksz
            if rows:
                s0 = (int(tab[h, 0, q, d]) - k0) // ksz
                d0 = (int(tab[h, 1, q, d]) - kptr[d]) // ksz
                kset[d][d0:d0 + rows].copy_(out_k[s0:s0 + rows], non_blocking=True)
                if has_v:
                    s0 = (int(tab[h, 0, q, G + d]) - v0) // vsz
                    d0 = (int(tab[h, 1, q, G + d]) - vptr[d]) // vsz
                    vset[d][d0:d0 + rows].copy_(out_v[s0:s0 + rows], non_blocking=True)

    with torch.cuda.stream(px.side):
        for h in range(H):                               # part 0 of a group leaves while the next group is partitioned
            px.side.wait_event(ready[h])
            push(0, h)
        landed[0].record(px.side)
        for q in range(1, Q):                            # the later parts cross NVLink under the reduce side of the earlier
            for h in range(H):
                push(q, h)
            landed[q].record(px.side)
        for out_k, out_v in bufs:
            out_k.record_stream(px.side)
            if out_v is not None:
                out_v.record_stream(px.side)
        for t in tabs + bases + [t for q in range(Q) for t3 in plans[q] for t in t3]:
            t.record_stream(px.side)
    keys, vals = px.keys, (px.vals if has_v else None)
    first = blocks[rank]
    nparts = blocks[rank + 1] - blocks[rank]
    results = []
    for q in range(Q):
        main.wait_event(landed[q])
        px.barrier()                                     # part q of every peer's pushes has landed here
        p0 = min(nparts, q * (per_parts // Q))
        p1 = min(nparts, (q + 1) * (per_parts // Q))
        if p1 <= p0:
            continue
        seg = segs[q][:, :(p1 - p0) << sub_bits].contiguous()         # [G * H sources, my buckets of part q]
        rk = keys[q * region:(q + 1) * region]
        rv = None if vals is None else vals[q * region:(q + 1) * region]
        ok, ov, po, cnt = nv.combine(rk, rv, op, P, seg, first + p0, p1 - p0, thresholds, sub_bits)
        results.append((ok, ov, po, cnt, first + p0, p1 - p0))
    if not results:   # a rank that owns no partitions (rank * ceil(P / G) >= P): one empty part, typed like the others
        z = torch.zeros(1, dtype=torch.int64, device=dev)
        ev = None if vals is None else torch.empty(0, dtype=nv.acc_dtype(vals.dtype), device=dev)
        results.append((keys[:0], ev, z, z[:0], first, 0))
    px.advance()
    return results


def merge_part_results(results):
    """One (keys, vals, part_offsets, counts) like shuffle.reduce_side from shuffle_pipelined's per-part results
    (copies; for checks and callers that want one buffer -- the pipelined step itself never needs it).  Raises
    NativeError if a part's merge failed (out_counts -1), as every other reduce-side consumer does."""
    from .shuffle import check_counts
    ks, vs, pos, cnts, base = [], [], [], [], 0
    for ok, ov, po, cnt, _, _ in results:
        check_counts(cnt.cpu().tolist())
        n = int(po[-1].item())
        ks.append(ok[:n])
        vs.append(ov[:n])
        pos.append(po[:-1] + base)
        cnts.append(cnt)
        base += n
    dev = ks[0].device
    pos.append(torch.tensor([base], dtype=torch.int64, device=dev))
    return torch.cat(ks), torch.cat(vs), torch.cat(pos), torch.cat(cnts)


def _map_exchange_overlapped_splits(px, key_chunks, val_chunks, P, thresholds=None, sub_bits=0, unordered=True, halves=2):
    """map_exchange_overlapped for splits that are NOT consecutive slices of one buffer (a launch pair per split).
    Map side + exchange with the push of the first half of the map splits running (on a side stream) while the
    second half is still being scattered.  The rank's splits are divided into `halves` contiguous groups, every
    group gets its own bucket-major buffer, and a group's blocks are pushed as soon as its scatter kernels are
    done; all counts are known after the histogram pass, so ONE all-gather describes every group.  In a receive
    buffer the groups of one source rank follow each other in split order, i.e. the layout is still
    (map split order)-major then bucket-major: `Received.seg` simply has G * halves source rows.
    Returns the Received view (bound = the whole receive buffer) like exchange_push."""
    from . import shuffle as sh
    G, rank, dev = px.world, px.rank, px.device
    F = P << sub_bits
    M = len(key_chunks)
    H = max(1, min(halves, M))
    counts, wss = [], []
    for k in key_chunks:
        c, ws = nv.partition_count(k, P, thresholds, False, sub_bits, None, None, unordered)
        counts.append(c)
        wss.append(ws)
    cm = torch.stack(counts)                                            # [M, F]
    bounds = [(M * h) // H for h in range(H + 1)]
    gc = torch.stack([cm[bounds[h]:bounds[h + 1]].sum(0) for h in range(H)])    # [H, F] rows per group and bucket
    all_counts = torch.empty(G * H * F, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(all_counts, gc.reshape(-1).contiguous(), group=px.group)   # the MapOutputTracker
    all_counts = all_counts.view(G * H, F)                              # source (rank, group) major
    blocks = [b << sub_bits for b in owner_blocks(P, G)]
    has_v = val_chunks[0] is not None
    main = torch.cuda.current_stream()
    b0, b1 = blocks[rank], blocks[rank + 1]
    need = None
    for h in range(H):
        src_row = rank * H + h
        send_first, dst_first, rows, recv_total = push_plan(all_counts, blocks, src_row)
        if need is None:
            need = recv_total.max()
            px.note_need(need)
        rows = torch.minimum(rows, (px.capacity - dst_first).clamp_(min=0))
        # this group's bucket-major buffer
        sel = slice(bounds[h], bounds[h + 1])
        n_h = sum(int(k.numel()) for k in key_chunks[sel])
        offsets = torch.zeros(F + 1, dtype=torch.int64, device=dev)
        torch.cumsum(gc[h], 0, out=offsets[1:])
        base = offsets[:-1].unsqueeze(0) + (torch.cumsum(cm[sel], 0) - cm[sel])
        out_k = torch.empty(n_h, dtype=key_chunks[0].dtype, device=dev)
        out_v = torch.empty(n_h, dtype=val_chunks[0].dtype, device=dev) if has_v else None
        for i, m in enumerate(range(bounds[h], bounds[h + 1])):
            nv.partition_scatter(key_chunks[m], val_chunks[m], P, base[i].contiguous(), out_k, out_v, wss[m], thresholds,
                                 False, sub_bits, None, unordered)
        cols = [(out_k.data_ptr(), px.key_base, out_k.element_size())]
        if has_v:
            cols.append((out_v.data_ptr(), px.val_base, out_v.element_size()))
        src = torch.cat([a + send_first * sz for a, _, sz in cols]).contiguous()
        dst = torch.cat([bb + dst_first * sz for _, bb, sz in cols]).contiguous()
        nby = torch.cat([rows * sz for _, _, sz in cols]).contiguous()
        ready = torch.cuda.Event()
        ready.record(main)
        with torch.cuda.stream(px.side):
            px.side.wait_event(ready)
            nv.copy_segments(src, dst, nby)
            for t in (out_k, out_v, src, dst, nby):
                if t is not None:
                    t.record_stream(px.side)
    main.wait_stream(px.side)
    px.barrier()                                                        # every peer's stores have landed
    seg = _landed(all_counts[:, b0:b1], px.capacity)
    keys, vals = px.keys, (px.vals if has_v else None)
    px.advance()
    return Received(keys, vals, seg, b0 >> sub_bits, (b1 - b0) >> sub_bits, sub_bits, bound=True)


def map_side_push(px, key_chunks, val_chunks, P, thresholds=None, sub_bits=0, unordered=True):
    """Map side + exchange in ONE pass over the rows (mode "fused"): the multisplit kernel stores every bucket run of
    a tile straight into the slot of (this rank, bucket) in the owner's receive buffer -- local memory or a peer's
    over NVLink; unordered multisplits (the reduceByKey map side) leave through the TMA (`cp.async.bulk` shared ->
    global, k_part_scatter_bulk in pointer mode), ordered ones (groupByKey) through the round-1 kernel's stores.  No
    bucket-major send buffer, no copy pass.  Nothing is read by the host: the pointer table, the segment matrix and
    the capacity flag come from one small kernel (dpk_fused_plan); a bucket that would overrun its receive buffer
    is diverted to a local dump buffer and PeerExchange.check() reports it.
    Returns the Received view (bound = the whole receive buffer) like exchange_push."""
    from . import shuffle as sh
    G, rank, dev = px.world, px.rank, px.device
    F = P << sub_bits
    has_v = val_chunks[0] is not None
    if len(key_chunks) > 1:   # consecutive slices of one buffer: one launch pair (shuffle.map_side does the same)
        whole_k, whole_v = sh._as_one(key_chunks), (sh._as_one(val_chunks) if has_v else None)
        if whole_k is not None and (not has_v or whole_v is not None) and whole_k.numel() < (1 << 31):
            key_chunks, val_chunks = [whole_k], [whole_v]
    counts, wss = [], []
    for k in key_chunks:
        c, ws = nv.partition_count(k, P, thresholds, False, sub_bits, None, None, unordered)
        counts.append(c)
        wss.append(ws)
    cm = counts[0].unsqueeze(0) if len(counts) == 1 else torch.stack(counts)     # [M, F] rows per chunk and bucket
    mine = counts[0] if len(counts) == 1 else cm.sum(0).contiguous()             # [F]
    all_counts = torch.empty(G * F, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(all_counts, mine, group=px.group)   # the MapOutputTracker
    all_counts = all_counts.view(G, F)
    per_block = ((P + G - 1) // G) << sub_bits
    n_local = sum(int(k.numel()) for k in key_chunks)
    dump_k, dump_v = px.dump(n_local, has_v)
    ksz = key_chunks[0].element_size()
    vsz = val_chunks[0].element_size() if has_v else 0
    kp, vp, seg = nv.fused_plan(all_counts, G, per_block, rank, px.dst_base if has_v else px.key_base, ksz, vsz,
                                px.capacity, dump_k, dump_v, px.err)
    if len(key_chunks) == 1:
        nv.partition_scatter_ptrs(key_chunks[0], val_chunks[0], P, kp, vp, wss[0], thresholds, False, sub_bits, None,
                                  unordered)
    else:
        chunk_off = torch.cumsum(cm, 0) - cm                        # rows of earlier local chunks per bucket
        for m, (k, v) in enumerate(zip(key_chunks, val_chunks)):
            nv.partition_scatter_ptrs(k, v, P, (kp + chunk_off[m] * ksz).contiguous(),
                                      (vp + chunk_off[m] * vsz).contiguous() if has_v else None,
                                      wss[m], thresholds, False, sub_bits, None, unordered)
    px.barrier()                                                    # every peer's stores have landed
    blocks = [b << sub_bits for b in owner_blocks(P, G)]
    b0, b1 = blocks[rank], blocks[rank + 1]
    keys, vals = px.keys, (px.vals if has_v else None)
    px.advance()
    return Received(keys, vals, seg, b0 >> sub_bits, (b1 - b0) >> sub_bits, sub_bits, bound=True)
