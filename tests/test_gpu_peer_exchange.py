"""The NVLink peer-memory exchange (dpark_b200/peer.py) end to end against the oracle, with G ranks simulated on ONE GPU.

Every peer form touches other ranks in two places only: the all-gather of the counts matrix and PeerExchange.barrier().
Everything else is kernels and copies that write to device addresses, and those addresses can as well be G receive
buffers on one GPU.  So G ranks run here as G Python threads of one process:

  * a baton (a lock) lets exactly one rank thread run at a time; a rank hands it over only while it waits inside the
    simulated gather or barrier, so the library's global options (copy_sms, which nv.copy_segments sets and resets)
    never interleave between ranks;
  * peer.dist is replaced by a namespace whose all_gather_into_tensor synchronises the device, deposits a copy of the
    rank's counts, waits for every rank and writes the concatenation in rank order;
  * the simulated barrier synchronises the device, then waits for every rank: after it every push issued before it
    has landed -- the contract of the real, stream-ordered barrier;
  * SimPeerExchange replaces only PeerExchange.__init__ (the symmetric-memory rendezvous) and barrier(); keys, vals,
    the base-address tables, advance, note_need, check and dump are the library's own.  Every rank has its own error
    flag, side streams and pinned segment-table buffer; all ranks share the G x nbuf receive buffers;
  * each receive buffer is allocated with GUARD rows behind its `capacity`.  Before every step every allocation is
    filled with a marker byte, and after every step the guard rows must still hold it, so a push that overruns its
    buffer fails an assertion on memory the test owns.  Marker rows behind the valid ones also stand for the rows of
    an earlier step: a reader that looks past its segment matrix, or at the wrong buffer set, merges them.

Every threading.Barrier has a timeout, and a rank that raises aborts it, so a failure in one rank fails the others
instead of hanging the run.  Real multi-process behaviour (races of the stream-ordered barrier, copy-engine overlap
timing) is out of reach here: scripts/multi_gpu_check.py covers it on a multi-GPU node."""
import threading
import types

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tests.shuffle_cases import REDUCE_VARIANTS, dpk_options, variant_id  # noqa: F401

gpu = pytest.mark.gpu

GUARD = 4096          # rows behind every receive buffer that no push may reach
MARK = 0xA5           # marker byte of every receive-buffer allocation before a step
TIMEOUT = 120.0       # seconds a rank may wait at a simulated collective


def _peer():
    from dpark_b200 import peer
    return peer


# ---------------------------------------------------------------- the simulated world
class _Group(object):
    """What PeerExchange.group is for the simulated collectives: the world and the caller's rank."""

    def __init__(self, world, rank):
        self.world, self.rank = world, rank


class SimWorld(object):
    """G ranks on one GPU: the shared receive buffers, the baton and the collectives."""

    def __init__(self, G, capacity, key_dtype, val_dtype, buffers=2, mode="push"):
        self.G, self.capacity, self.nbuf = G, int(capacity), max(1, int(buffers))
        self.bufs = [[(torch.empty(self.capacity + GUARD, dtype=key_dtype, device="cuda"),
                       torch.empty(self.capacity + GUARD, dtype=val_dtype, device="cuda")) for _ in range(G)]
                     for _ in range(self.nbuf)]
        self.baton = threading.Lock()
        self.bar = None
        self.slots = [None] * G
        self.px = [SimPeerExchange(self, r, mode) for r in range(G)]

    # -- what the ranks call
    def _wait(self):
        self.baton.release()
        try:
            self.bar.wait()
        finally:
            self.baton.acquire()

    def barrier(self):
        torch.cuda.synchronize()
        self._wait()

    def all_gather_into_tensor(self, out, inp, group):
        torch.cuda.synchronize()
        self.slots[group.rank] = inp.detach().reshape(-1).clone()
        torch.cuda.synchronize()
        self._wait()
        out.copy_(torch.cat(self.slots))
        torch.cuda.synchronize()
        self._wait()                     # nobody deposits the next counts before every rank has read these

    # -- what the test calls
    def run(self, fn):
        """[fn(rank) for every rank], each on its own thread, one at a time."""
        self.bar = threading.Barrier(self.G, timeout=TIMEOUT)
        out, err = [None] * self.G, [None] * self.G

        def body(r):
            self.baton.acquire()
            try:
                out[r] = fn(r)
                torch.cuda.synchronize()
            except BaseException as e:   # noqa: B902 -- reported by the main thread
                err[r] = e
                self.bar.abort()
            finally:
                self.baton.release()

        threads = [threading.Thread(target=body, args=(r,), daemon=True) for r in range(self.G)]
        for t in threads:
            t.start()
        for t in threads:
            t.join(TIMEOUT * 4)
        assert not any(t.is_alive() for t in threads), "a simulated rank did not finish"
        real = [e for e in err if e is not None and not isinstance(e, threading.BrokenBarrierError)]
        if real or any(e is not None for e in err):
            raise (real or [e for e in err if e is not None])[0]
        return out

    def fill(self):
        """Every receive-buffer allocation holds the marker (guard rows included)."""
        for bset in self.bufs:
            for pair in bset:
                for t in pair:
                    t.view(torch.uint8).fill_(MARK)

    def check_guards(self):
        torch.cuda.synchronize()
        for b, bset in enumerate(self.bufs):
            for r, pair in enumerate(bset):
                for t in pair:
                    assert bool((t[self.capacity:].view(torch.uint8) == MARK).all()), \
                        "a push wrote past the receive buffer of rank %d (buffer set %d)" % (r, b)


_SIM_CLASS = []


def _sim_peer_exchange_class():
    if _SIM_CLASS:
        return _SIM_CLASS[0]
    peer = _peer()

    class _Sim(peer.PeerExchange):
        """PeerExchange over the simulated world's buffers: __init__ and barrier() replaced, nothing else."""

        def __init__(self, world, rank, mode="push"):
            self.mode = mode
            self.group = _Group(world, rank)
            self.rank, self.world = rank, world.G
            self.device = torch.device("cuda", torch.cuda.current_device())
            self.capacity = world.capacity
            self.nbuf = world.nbuf
            self._keys, self._vals, self._hk, self._hv, self._kb, self._vb, self._db = [], [], [], [], [], [], []
            self._pk, self._pv, self._kp, self._vp = [], [], [], []
            for bset in world.bufs:
                ks = [k[:self.capacity] for k, _ in bset]
                vs = [v[:self.capacity] for _, v in bset]
                self._keys.append(ks[rank])
                self._vals.append(vs[rank])
                self._kp.append([t.data_ptr() for t in ks])
                self._vp.append([t.data_ptr() for t in vs])
                self._kb.append(torch.tensor(self._kp[-1], dtype=torch.int64, device=self.device))
                self._vb.append(torch.tensor(self._vp[-1], dtype=torch.int64, device=self.device))
                self._db.append(torch.cat([self._kb[-1], self._vb[-1]]).contiguous())
                self._pk.append(ks)
                self._pv.append(vs)
            self.step = 0
            self.side = torch.cuda.Stream(device=self.device, priority=-1)
            self.err = torch.zeros(1, dtype=torch.int64, device=self.device)
            self._closed = False
            self._dump = None
            self.copy_sms = 16
            self.copy_engine = 2
            self.side2 = torch.cuda.Stream(device=self.device, priority=-1)
            self._tab_host = None

        def barrier(self):
            self.group.world.barrier()

    _SIM_CLASS.append(_Sim)
    return _Sim


def SimPeerExchange(world, rank, mode="push"):
    return _sim_peer_exchange_class()(world, rank, mode)


def _sim_gather(out, inp, group=None):
    group.world.all_gather_into_tensor(out, inp, group)


@pytest.fixture
def sim(monkeypatch):
    """sim(G, capacity, key_dtype, val_dtype, buffers=2, mode="push") -> SimWorld; peer.dist is the simulated one
    for the test."""
    monkeypatch.setattr(_peer(), "dist", types.SimpleNamespace(all_gather_into_tensor=_sim_gather))
    return SimWorld


# ---------------------------------------------------------------- inputs and the oracle
KDT = {"i64": np.int64, "i32": np.int32, "f64": np.float64}
VDT = {"i64": np.int64, "i32": np.int32, "f32": np.float32, "f64": np.float64}


def make_inputs(G, M, n, kdt="i64", vdt="i64", seed=0, keyspace=3000, hot=None, empty_rank=None, row_ids=False):
    """splits[r] = M (keys, vals) numpy splits of rank r, uneven sizes, one of them empty (index r % M).
    hot = (key, fraction): that share of every rank's rows carries one key.  row_ids: values are global row ids
    (rank-major, then split, then position)."""
    rng = np.random.default_rng(seed)
    splits, base = [], 0
    for r in range(G):
        nr = 0 if r == empty_rank else int(n * (0.6 + 0.8 * rng.random()))
        k = rng.integers(-keyspace, keyspace, nr)
        if hot is not None:
            k[rng.random(nr) < hot[1]] = hot[0]
        k = (k * 0.5).astype(np.float64) if kdt == "f64" else k.astype(KDT[kdt])
        if row_ids:
            v = np.arange(base, base + nr, dtype=np.int64)
        elif vdt in ("f32", "f64"):
            v = rng.standard_normal(nr).astype(VDT[vdt])
        else:
            v = rng.integers(-1000, 1000, nr).astype(VDT[vdt])
        base += nr
        cuts = np.sort(rng.integers(0, nr + 1, M - 1)) if nr else np.zeros(M - 1, dtype=np.int64)
        sizes = list(np.diff(np.concatenate([[0], cuts, [nr]])))
        if M > 1:                           # an empty split: its rows move to the next one
            e = r % M
            sizes[(e + 1) % M] += sizes[e]
            sizes[e] = 0
        at, mine = 0, []
        for s in sizes:
            mine.append((k[at:at + s], v[at:at + s]))
            at += s
        splits.append(mine)
    return splits


def device_chunks(splits_r, consecutive=True):
    """A rank's splits on the device: consecutive slices of one buffer, or one allocation per split."""
    if not consecutive:
        return [torch.from_numpy(np.ascontiguousarray(k)).cuda() for k, _ in splits_r], \
               [torch.from_numpy(np.ascontiguousarray(v)).cuda() for _, v in splits_r]
    k = torch.from_numpy(np.concatenate([k for k, _ in splits_r])).cuda()
    v = torch.from_numpy(np.concatenate([v for _, v in splits_r])).cuda()
    kc, vc, at = [], [], 0
    for sk, _ in splits_r:
        kc.append(k[at:at + len(sk)])
        vc.append(v[at:at + len(sk)])
        at += len(sk)
    return kc, vc


def _bits(a):
    a = np.asarray(a)
    return (a.astype(np.float64) + 0.0).view(np.int64) if a.dtype.kind == "f" else a.astype(np.int64)


def oracle_reduce(splits, P, op, thresholds=None):
    """Per partition (keys, vals) of all ranks' rows, and per partition sum |v| per key for float sums."""
    ks = [k for sp in splits for k, _ in sp if len(k)]
    vs = [v for sp in splits for _, v in sp if len(v)]
    want = orc.reduce_by_key(ks, vs, P, op, thresholds)
    absw = None
    if vs and vs[0].dtype.kind == "f" and op == "sum":
        absw = orc.reduce_by_key(ks, [np.abs(v.astype(np.float64)) for v in vs], P, "sum", thresholds)
    return want, absw


def check_reduced(G, P, per_rank, want, absw):
    """per_rank[r] = (keys, vals, part_offsets, counts) on the host, for the partitions rank r owns."""
    blocks = _peer().owner_blocks(P, G)
    for r in range(G):
        ok, ov, po, cnt = per_rank[r]
        nparts = blocks[r + 1] - blocks[r]
        assert len(po) == nparts + 1 and len(cnt) == nparts, "rank %d" % r
        assert (cnt >= 0).all()
        for j in range(nparts):
            p = blocks[r] + j
            gk, gv = ok[po[j]:po[j] + cnt[j]], ov[po[j]:po[j] + cnt[j]]
            wk, wv = want[p]
            gb, wb = _bits(gk), _bits(wk)
            o1, o2 = np.argsort(gb, kind="stable"), np.argsort(wb, kind="stable")
            assert np.array_equal(gb[o1], wb[o2]), "rank %d partition %d: keys differ" % (r, p)
            if absw is None:
                assert np.array_equal(gv[o1], wv[o2]), "rank %d partition %d: values differ" % (r, p)
            else:
                ak, av = absw[p]
                assert np.array_equal(_bits(ak)[np.argsort(_bits(ak), kind="stable")], wb[o2])
                tol = 1e-9 * av[np.argsort(_bits(ak), kind="stable")]
                assert np.all(np.abs(gv[o1] - wv[o2]) <= tol), "rank %d partition %d: sums differ" % (r, p)


def _host(res):
    ok, ov, po, cnt = res
    return ok.cpu().numpy(), ov.cpu().numpy(), po.cpu().numpy(), cnt.cpu().numpy()


# ---------------------------------------------------------------- the forms
def _form_id(f):
    return "-".join(str(x) for x in f)


FULL_FORMS = ([("push",)]
              + [("overlap", h, c) for h in (1, 2, 3) for c in ("consec", "splits")]
              + [("fused", "one"), ("fused", "splits")]
              + [("pipe", g, q, ce) for g, q in ((1, 1), (2, 2), (3, 4), (4, 1)) for ce in (0, 1, 2)])


def run_form(form, px, splits_r, P, op, thr, sb):
    """One reduceByKey step of one rank in `form`; returns (keys, vals, part_offsets, counts) on the host."""
    peer = _peer()
    from dpark_b200 import shuffle
    kind = form[0]
    consecutive = not (len(form) > 1 and form[-1] == "splits")
    kc, vc = device_chunks(splits_r, consecutive)
    if kind == "pipe":
        _, g, q, ce = form
        px.copy_engine = ce
        parts = peer.shuffle_pipelined(px, kc, vc, P, op, thr, sb, g, q)
        blocks = peer.owner_blocks(P, px.world)
        assert parts and parts[0][4] == blocks[px.rank]
        at = blocks[px.rank]
        for _, _, _, _, first, n in parts:                   # consecutive partition ranges, all owned ones
            assert first == at
            at += n
        assert at == blocks[px.rank + 1]
        return _host(peer.merge_part_results(parts))
    if kind == "push":
        mo = shuffle.map_side(kc, vc, P, thr, False, sb, unordered=True)
        rx = peer.exchange_push(px, mo)
    elif kind == "overlap":
        rx = peer.map_exchange_overlapped(px, kc, vc, P, thr, sb, True, form[1])
    elif kind == "fused":
        rx = peer.map_side_push(px, kc, vc, P, thr, sb)
    else:
        raise ValueError(form)
    return _host(shuffle.reduce_side(rx, op, P, thr))


def run_step(world, form, splits, P, op="sum", thr=None, sb=0):
    world.fill()
    out = world.run(lambda r: run_form(form, world.px[r], splits[r], P, op, thr, sb))
    world.check_guards()
    for px in world.px:
        px.check()
    return out


def _capacity(splits, Q=4):
    total = sum(len(k) for sp in splits for k, _ in sp)
    return Q * total + 1024        # every part's region (capacity / Q) holds everything


# ---------------------------------------------------------------- layout
def _sources(splits, H=1):
    """(keys, row ids) of every source row: rank-major, then the H groups of its splits."""
    out = []
    for sp in splits:
        M = len(sp)
        Hh = max(1, min(H, M))
        bounds = [(M * h) // Hh for h in range(Hh + 1)]
        for h in range(Hh):
            sel = sp[bounds[h]:bounds[h + 1]]
            out.append((np.concatenate([k for k, _ in sel]), np.concatenate([v for _, v in sel])))
    return out


def check_layout(rx, G, rank, sources, P, sb, stable, exact):
    """rx (on the host: keys, vals, seg, part_first, nparts) against the oracle's map tasks of every source row:
    source-major, then partition-major; exact = bit-identical rows in (map split, position) order; else per (source,
    partition) the same rows, and (stable) ascending row ids inside every fine bucket."""
    keys, vals, seg, first, nparts = rx
    blocks = _peer().owner_blocks(P, G)
    S = 1 << sb
    assert first == blocks[rank] and nparts == blocks[rank + 1] - blocks[rank]
    assert seg.shape == (len(sources), nparts << sb)
    at = 0
    for s, (k, v) in enumerate(sources):
        mk, mv, mo = orc.map_task(k, v, P, "sum", None, combine=False) if len(k) else \
            (np.empty(0, np.int64), np.empty(0, np.int64), np.zeros(P + 1, np.int64))
        for j in range(nparts):
            p = first + j
            wk, wv = mk[mo[p]:mo[p + 1]], mv[mo[p]:mo[p + 1]]
            runs = seg[s, j * S:(j + 1) * S]
            n = int(runs.sum())
            assert n == len(wk), "source %d partition %d: %d rows, oracle %d" % (s, p, n, len(wk))
            gk, gv = keys[at:at + n], vals[at:at + n]
            if exact:
                assert np.array_equal(gk, wk) and np.array_equal(gv, wv), "source %d partition %d" % (s, p)
            else:
                o1, o2 = np.argsort(gv), np.argsort(wv)
                assert np.array_equal(gv[o1], wv[o2]) and np.array_equal(gk[o1], wk[o2]), "source %d partition %d" % (s, p)
            if stable:
                r0 = 0
                for c in runs:
                    assert (np.diff(gv[r0:r0 + c]) > 0).all(), "source %d partition %d: a fine bucket lost row order" % (s, p)
                    r0 += c
            at += n
    assert at == int(seg.sum())


LAYOUT_FORMS = [("push", "stable"), ("fused", "stable", "one"), ("fused", "stable", "splits"),
                ("push", "unordered"), ("fused", "unordered", "one"), ("fused", "unordered", "splits"),
                ("overlap", "unordered", "consec"), ("overlap", "unordered", "splits")]


@gpu
@pytest.mark.parametrize("form", LAYOUT_FORMS, ids=_form_id)
@pytest.mark.parametrize("G,P,sb", [(1, 3, 0), (2, 8, 0), (3, 7, 2), (4, 5, 0), (4, 1, 2)])
def test_received_layout_is_what_an_alltoallv_delivers(sim, form, G, P, sb):
    """Each rank's Received: source-rank-major, bucket-major, the rows of the oracle's map task of every source.  A
    stable map side at sub_bits 0 is bit-identical to an alltoallv; with sub-buckets every fine bucket keeps (map
    split, position) order; the unordered forms deliver the same rows per (source, partition) segment."""
    peer = _peer()
    from dpark_b200 import shuffle
    splits = make_inputs(G, 4, 3000, seed=G * 10 + P, keyspace=500, row_ids=True)
    world = sim(G, _capacity(splits, 1), torch.int64, torch.int64)
    kind, order = form[0], form[1]
    stable = order == "stable"
    H = 2 if kind == "overlap" else 1

    def rank_fn(r):
        px = world.px[r]
        kc, vc = device_chunks(splits[r], form[-1] != "splits")
        if kind == "push":
            rx = peer.exchange_push(px, shuffle.map_side(kc, vc, P, None, False, sb, unordered=not stable))
        elif kind == "fused":
            rx = peer.map_side_push(px, kc, vc, P, None, sb, unordered=not stable)
        else:
            rx = peer.map_exchange_overlapped(px, kc, vc, P, None, sb, True, H)
        seg = rx.seg.cpu().numpy()
        n = int(seg.sum())
        return rx.keys[:n].cpu().numpy(), rx.vals[:n].cpu().numpy(), seg, rx.part_first, rx.nparts

    world.fill()
    got = world.run(rank_fn)
    world.check_guards()
    sources = _sources(splits, H)
    for r in range(G):
        check_layout(got[r], G, r, sources, P, sb, stable, exact=stable and sb == 0)


# ---------------------------------------------------------------- reduceByKey, every form
@gpu
@pytest.mark.parametrize("form", FULL_FORMS, ids=_form_id)
@pytest.mark.parametrize("G,P,sb", [(1, 4, 2), (2, 8, 0), (3, 7, 2), (4, 5, 3), (8, 16, 0)])
def test_every_form_reduces_like_the_oracle(sim, monkeypatch, form, G, P, sb):
    """Every peer form, then the reduce side, against orc.reduce_by_key over all ranks' rows: P divisible by G and not
    (P = 5 on 4 ranks: the last rank owns no partition), sub_bits 0 / 2 / 3, uneven map splits with an empty one."""
    peer = _peer()
    splits = make_inputs(G, 4, 4000, seed=1000 + G * 31 + P)
    world = sim(G, _capacity(splits), torch.int64, torch.int64)
    calls = []
    real = peer._map_exchange_overlapped_splits

    def spy(*a, **kw):
        calls.append(1)
        return real(*a, **kw)
    monkeypatch.setattr(peer, "_map_exchange_overlapped_splits", spy)
    got = run_step(world, form, splits, P, "sum", None, sb)
    if form[0] == "overlap":
        assert len(calls) == (G if form[2] == "splits" else 0), "only non-consecutive chunks take the per-split path"
    want, absw = oracle_reduce(splits, P, "sum")
    check_reduced(G, P, got, want, absw)


EDGE_SHAPES = {
    "g1": dict(G=1, P=4, sb=2),
    "g2_sb3": dict(G=2, P=6, sb=3),
    "g3_sb0": dict(G=3, P=9, sb=0),
    "g4_p5": dict(G=4, P=5, sb=2),
    "g4_p1": dict(G=4, P=1, sb=2),
    "g8": dict(G=8, P=16, sb=1),
    "thresholds": dict(G=3, P=4, sb=2, thr=[-300, 0, 250]),
    "empty_rank": dict(G=4, P=8, sb=2, empty_rank=2),
    "hot_key": dict(G=4, P=8, sb=2, hot=(7, 0.8)),
}
EDGE_FORMS = [("push",), ("pipe", 2, 2, 2)]


@gpu
@pytest.mark.parametrize("form", EDGE_FORMS, ids=_form_id)
@pytest.mark.parametrize("shape", list(EDGE_SHAPES))
def test_shape_edges(sim, form, shape):
    """exchange_push and the pipelined 2x2 step on 1 to 8 ranks, P < G and P not divisible by G (ranks that own
    no partition), range-partitioner thresholds, a rank with no rows, and a hot key that sends most rows to one owner."""
    c = EDGE_SHAPES[shape]
    G, P, sb, thr = c["G"], c["P"], c["sb"], c.get("thr")
    splits = make_inputs(G, 4, 3000, seed=list(EDGE_SHAPES).index(shape), keyspace=800, hot=c.get("hot"),
                         empty_rank=c.get("empty_rank"))
    world = sim(G, _capacity(splits), torch.int64, torch.int64)
    got = run_step(world, form, splits, P, "sum", thr, sb)
    want, absw = oracle_reduce(splits, P, "sum", thr)
    check_reduced(G, P, got, want, absw)


DTYPES = [("i64", "i64"), ("i32", "f32"), ("i64", "i32"), ("i32", "i64"), ("f64", "f64")]
TORCH = {"i64": torch.int64, "i32": torch.int32, "f32": torch.float32, "f64": torch.float64}


@gpu
@pytest.mark.parametrize("form", EDGE_FORMS, ids=_form_id)
@pytest.mark.parametrize("op", ["sum", "min", "max"])
@pytest.mark.parametrize("kdt,vdt", DTYPES, ids=["-".join(d) for d in DTYPES])
def test_column_dtypes_and_ops(sim, form, kdt, vdt, op):
    """Key / value widths that differ (the pads of dpk_pipe_plan keep source and landing row congruent mod 16 bytes)
    and every op: integers exact, float sums within 1e-9 * sum |v| per key."""
    G, P, sb = 3, 7, 2
    splits = make_inputs(G, 4, 3000, kdt, vdt, seed=len(kdt + vdt + op) * 7 + (op == "min"), keyspace=600)
    world = sim(G, _capacity(splits), TORCH[kdt], TORCH[vdt])
    got = run_step(world, form, splits, P, op, None, sb)
    want, absw = oracle_reduce(splits, P, op)
    check_reduced(G, P, got, want, absw)


# ---------------------------------------------------------------- consecutive steps on one exchange
STEP_FORMS = [("push",), ("pipe", 2, 2, 2), ("fused", "one"), ("overlap", 2, "consec"), ("pipe", 2, 2, 0)]


def _reduce_variant_id(opts):
    return variant_id(opts) if opts else "default"


@gpu
@pytest.mark.parametrize("variant", REDUCE_VARIANTS, ids=_reduce_variant_id)
@pytest.mark.parametrize("buffers", [1, 2])
def test_consecutive_steps_read_their_own_rows(sim, buffers, variant, dpk_options):
    """Five steps in a row on one exchange object, each with different data and a different form: every step's
    result must be its own oracle's.  With the marker fill this catches a reader of the wrong buffer set, or of rows
    behind the valid ones (pipelined parts hand combine a region longer than its rows), under every reduce variant."""
    dpk_options(variant)
    G, P, sb = 3, 7, 2
    first = make_inputs(G, 4, 3000, seed=500)
    world = sim(G, _capacity(first) * 2, torch.int64, torch.int64, buffers=buffers)
    for i, form in enumerate(STEP_FORMS):
        splits = first if i == 0 else make_inputs(G, 4, 2000 + 700 * i, seed=500 + i, keyspace=300 + 400 * i)
        got = run_step(world, form, splits, P, "sum", None, sb)
        want, absw = oracle_reduce(splits, P, "sum")
        check_reduced(G, P, got, want, absw)
        assert all(px.step == i + 1 for px in world.px)


# ---------------------------------------------------------------- groupByKey
@gpu
@pytest.mark.parametrize("form", ["push", "fused"])
@pytest.mark.parametrize("G,P,sb", [(1, 3, 2), (3, 7, 0), (4, 5, 2)])
def test_group_by_key_keeps_global_row_order(sim, form, G, P, sb):
    """exchange_push(need_host_count=True) and map_side_push(unordered=False), then shuffle.group_side: the values
    are global row ids, and each key's list must equal the oracle's, in (source rank, map split, position) order."""
    peer = _peer()
    from dpark_b200 import shuffle
    splits = make_inputs(G, 4, 3000, seed=70 + G, keyspace=400, row_ids=True)
    world = sim(G, _capacity(splits, 1), torch.int64, torch.int64)

    def rank_fn(r):
        px = world.px[r]
        kc, vc = device_chunks(splits[r], r % 2 == 0)
        if form == "push":
            rx = peer.exchange_push(px, shuffle.map_side(kc, vc, P, None, False, sb), need_host_count=True)
        else:
            rx = peer.map_side_push(px, kc, vc, P, None, sb, unordered=False)
        gk, gs, ng, v, off = shuffle.group_side(rx, P)
        ng = int(ng.item())
        return gk[:ng].cpu().numpy(), gs[:ng + 1].cpu().numpy(), v.cpu().numpy(), off.cpu().numpy()

    world.fill()
    got = world.run(rank_fn)
    world.check_guards()
    ks = [k for sp in splits for k, _ in sp if len(k)]
    vs = [v for sp in splits for _, v in sp if len(v)]
    want = orc.group_by_key(ks, vs, P)
    blocks = peer.owner_blocks(P, G)
    for r in range(G):
        gk, gs, v, off = got[r]
        assert len(off) == blocks[r + 1] - blocks[r] + 1
        for j in range(len(off) - 1):
            p = blocks[r] + j
            sel = np.nonzero((gs[:-1] >= off[j]) & (gs[:-1] < off[j + 1]))[0]
            mine = {int(gk[g]): v[gs[g]:gs[g + 1]].tolist() for g in sel}
            wk, wo, wv = want[p]
            theirs = {int(wk[g]): wv[wo[g]:wo[g + 1]].tolist() for g in range(len(wk))}
            assert mine == theirs, "rank %d partition %d" % (r, p)


# ---------------------------------------------------------------- HostShuffle over the peer exchange
@gpu
@pytest.mark.parametrize("mode", ["push", "fused"])
@pytest.mark.parametrize("G,P", [(2, 8), (3, 5)])
def test_host_shuffle_over_the_peer_exchange(sim, mode, G, P):
    """shuffle.HostShuffle(peer_exchange=px) on every simulated rank, two batches in a row, in both modes."""
    from dpark_b200 import shuffle
    first = make_inputs(G, 1, 5000, seed=900 + G, keyspace=700)
    rng = np.random.default_rng(G)      # the second batch: as many rows per rank (HostShuffle sizes its buffers once)
    second = [[(rng.integers(-300, 300, len(sp[0][0])).astype(np.int64), sp[0][1][::-1].copy())] for sp in first]
    world = sim(G, _capacity(first, 1) * 2, torch.int64, torch.int64, mode=mode)
    hs = [shuffle.HostShuffle(len(sp[0][0]), torch.int64, torch.int64, P, "sum", splits=4, sub_bits=2,
                              peer_exchange=world.px[r]) for r, sp in enumerate(first)]
    for splits in (first, second):
        def rank_fn(r):
            k, v = splits[r][0]
            hs[r].h_keys.copy_(torch.from_numpy(k))
            hs[r].h_vals.copy_(torch.from_numpy(v))
            return [(p, a.numpy().copy(), b.numpy().copy()) for p, a, b in hs[r].run()]

        world.fill()
        got = world.run(rank_fn)
        world.check_guards()
        want, _ = oracle_reduce(splits, P, "sum")
        blocks = shuffle.owner_blocks(P, G)
        for r in range(G):
            assert [p for p, _, _ in got[r]] == list(range(blocks[r], blocks[r + 1]))
            for p, gk, gv in got[r]:
                o1, o2 = np.argsort(gk), np.argsort(want[p][0])
                assert np.array_equal(gk[o1], want[p][0][o2]) and np.array_equal(gv[o1], want[p][1][o2])


# ---------------------------------------------------------------- capacity overflow
def _counts(sources, P):
    """[source][partition] rows."""
    return np.stack([np.bincount(orc.partition_vec(orc.hash_vec(k), P), minlength=P) if len(k) else
                     np.zeros(P, np.int64) for k, _ in sources]).astype(np.int64)


def _landed_push(C, cap):
    flat = C.reshape(-1)
    start = np.cumsum(flat) - flat
    return np.minimum(flat, np.maximum(cap - start, 0)).reshape(C.shape)


def _landed_fused(C, cap):
    flat = C.reshape(-1)
    end = np.cumsum(flat)
    return np.where(end <= cap, flat, 0).reshape(C.shape)


@gpu
@pytest.mark.parametrize("region", [0, 50, 400, 1 << 20])
def test_pipe_plan_segment_matrix_counts_the_rows_that_land(region):
    """dpk_pipe_plan with a region too small for some parts: part q's segment matrix describes exactly the rows that
    land in region q (every source's push is clamped at the region), so combine never reads past the region."""
    from dpark_b200 import _native as nv
    rng = np.random.default_rng(region)
    G, H, Q, P, sb = 3, 2, 2, 12, 1
    F, S = P << sb, G * H
    per_block = ((P + G - 1) // G) << sb
    part_blk = per_block // Q
    counts = rng.integers(0, 40, (S, F)).astype(np.int64)
    base = torch.arange(1, 2 * G + 1, dtype=torch.int64, device="cuda") << 32        # fake receive buffers
    for rank in range(G):
        my = rank * H + 1
        out_k = torch.empty(int(counts[my].sum()) + nv.pipe_pad_rows(G, Q, 8, 4), dtype=torch.int64, device="cuda")
        out_v = torch.empty(out_k.numel(), dtype=torch.float32, device="cuda")
        err = torch.zeros(1, dtype=torch.int64, device="cuda")
        seg = nv.pipe_plan(torch.from_numpy(counts).cuda(), G, per_block, Q, region, my, rank, out_k, out_v, base,
                           err)[4].cpu().numpy()
        for q in range(Q):
            lo = rank * per_block + q * part_blk
            want = _landed_push(counts[:, lo:lo + part_blk], region)
            assert np.array_equal(seg[q], want), "rank %d part %d" % (rank, q)
            assert seg[q].sum() == min(counts[:, lo:lo + part_blk].sum(), region)
        need = max(counts[:, d * per_block + q * part_blk:d * per_block + (q + 1) * part_blk].sum()
                   for d in range(G) for q in range(Q))
        assert int(err.item()) == max(0, need - region)


OVERFLOW_FORMS = [("push",), ("overlap", 2, "consec"), ("overlap", 2, "splits"), ("fused", "one"), ("fused", "splits"),
                  ("pipe", 2, 2, 0), ("pipe", 2, 2, 2)]


@gpu
@pytest.mark.parametrize("form", OVERFLOW_FORMS, ids=_form_id)
def test_capacity_overflow_is_flagged_and_stays_in_bounds(sim, form):
    """A step whose rows do not fit one receive buffer (the pipelined form: one part's region of one rank): nothing
    is written past the buffer, the segment matrix describes only the rows that landed (so the reduce side stays inside
    its buffers), check() raises on every rank (each plan sees every destination's total) and clears the flag, and the
    next step with enough room is right again."""
    peer = _peer()
    G, P, sb = 2, 8, 0
    blocks = peer.owner_blocks(P, G)
    big = make_inputs(G, 4, 6000, seed=41, keyspace=900, hot=(0, 0.5))      # key 0 -> partition 0 on rank 0
    pipe = form[0] == "pipe"
    H = 2 if form[0] == "overlap" else (form[1] if pipe else 1)
    sources = _sources(big, H)
    C = _counts(sources, P)
    if pipe:
        Q = form[2]
        per = (P + G - 1) // G // Q
        part_tot = sorted(((C[:, blocks[d] + q * per:blocks[d] + (q + 1) * per].sum(), d, q)
                           for d in range(G) for q in range(Q)), reverse=True)
        region = ((part_tot[0][0] + part_tot[1][0]) // 2) & ~15
        assert part_tot[1][0] < region < part_tot[0][0]           # exactly one part of one rank overflows
        cap = region * Q
    else:
        recv = sorted(C[:, blocks[d]:blocks[d + 1]].sum() for d in range(G))
        cap = (recv[-1] + recv[-2]) // 2
        assert recv[-2] <= cap < recv[-1]
    world = sim(G, cap, torch.int64, torch.int64)
    from dpark_b200 import shuffle

    def overflow_step(r):
        px = world.px[r]
        kc, vc = device_chunks(big[r], form[-1] != "splits")
        if pipe:
            px.copy_engine = form[3]
            parts = peer.shuffle_pipelined(px, kc, vc, P, "sum", None, sb, form[1], form[2])
            seg_or_po = [(first, po.cpu().numpy(), _host((ok, ov, po, cnt))) for ok, ov, po, cnt, first, _ in parts]
        else:
            if form[0] == "push":
                rx = peer.exchange_push(px, shuffle.map_side(kc, vc, P, None, False, sb, unordered=True))
            elif form[0] == "overlap":
                rx = peer.map_exchange_overlapped(px, kc, vc, P, None, sb, True, H)
            else:
                rx = peer.map_side_push(px, kc, vc, P, None, sb)
            seg_or_po = rx.seg.cpu().numpy()
            mine = C[:, blocks[r]:blocks[r + 1]]
            want = _landed_fused(mine, cap) if form[0] == "fused" else _landed_push(mine, cap)
            assert np.array_equal(seg_or_po, want), "rank %d: the segment matrix must describe the rows that landed" % r
            ok, ov, po, cnt = shuffle.reduce_side(rx, "sum", P)     # in bounds: reads only what seg describes
            assert int(po[-1]) == int(want.sum()) <= cap
        raised = []
        for _ in range(2):
            try:
                px.check()
                raised.append(False)
            except RuntimeError:
                raised.append(True)
        return seg_or_po, raised

    world.fill()
    got = world.run(overflow_step)
    world.check_guards()
    for r in range(G):
        assert got[r][1] == [True, False], "rank %d: check() must raise once, then the flag is clear" % r
    if pipe:
        want, _ = oracle_reduce(big, P, "sum")
        region = cap // form[2]
        per = (P + G - 1) // G // form[2]
        for r in range(G):
            for first, po, res in got[r][0]:
                q = (first - blocks[r]) // per
                landed = _landed_push(C[:, first:first + per], region)
                assert np.array_equal(np.diff(po), landed.sum(0)), "rank %d part %d" % (r, q)
                if np.array_equal(landed, C[:, first:first + per]):    # a part that fit is exact
                    check_reduced(1, per, [res], [want[first + j] for j in range(per)], None)
    # the next step fits, and is right
    small = make_inputs(G, 4, 600, seed=42, keyspace=300)
    got = run_step(world, form, small, P, "sum", None, sb)
    want, absw = oracle_reduce(small, P, "sum")
    check_reduced(G, P, got, want, absw)


# ---------------------------------------------------------------- host-side pieces (no GPU)
def test_merge_part_results_raises_on_a_failed_part():
    """peer.merge_part_results checks the per-part counts like every other reduce-side consumer: a part whose merge
    overflowed (out_counts -1) raises NativeError instead of merging an invalid partition."""
    from dpark_b200 import _native, peer
    a = (torch.tensor([10, 11, 12, 0, 0, 20, 0]), torch.tensor([1, 2, 3, 0, 0, 4, 0]),
         torch.tensor([0, 5, 7]), torch.tensor([3, 1]), 4, 2)
    bad = (torch.tensor([30, 0, 40, 41]), torch.tensor([5, 0, 6, 7]), torch.tensor([0, 2, 4]), torch.tensor([1, -1]), 6, 2)
    with pytest.raises(_native.NativeError):
        peer.merge_part_results([a, bad])
    with pytest.raises(_native.NativeError):
        peer.merge_part_results([bad, a])
    k, v, po, cnt = peer.merge_part_results([a])
    assert po.tolist() == [0, 5, 7] and cnt.tolist() == [3, 1]


def test_merge_part_results_of_a_rank_without_partitions():
    """The one empty part shuffle_pipelined returns on a rank that owns no partitions merges into an empty,
    well-typed result like shuffle.reduce_side's."""
    from dpark_b200 import peer
    z = torch.zeros(1, dtype=torch.int64)
    k, v, po, cnt = peer.merge_part_results([(torch.empty(0, dtype=torch.int32), torch.empty(0, dtype=torch.float64),
                                              z, z[:0], 5, 0)])
    assert k.dtype == torch.int32 and v.dtype == torch.float64 and k.numel() == 0 and v.numel() == 0
    assert po.tolist() == [0] and cnt.tolist() == []


@pytest.mark.parametrize("sizes", [[0, 5, 3], [5, 0, 3], [5, 3, 0], [0, 0, 0], [4]])
def test_consecutive_slices_with_empty_splits_are_one_buffer(sizes):
    """shuffle._as_one (which decides whether map splits take one launch pair, and which shuffle_pipelined needs):
    consecutive slices of one buffer are one tensor even when a split is empty (an empty slice's data_ptr() is not
    its place in the buffer); slices with a gap, out of order or of other buffers are not."""
    from dpark_b200 import shuffle
    buf = torch.arange(20, dtype=torch.int64)[2:]
    at, chunks = 0, []
    for s in sizes:
        chunks.append(buf[at:at + s])
        at += s
    one = shuffle._as_one(chunks)
    assert one is not None and one.tolist() == buf[:at].tolist()
    assert at == 0 or one.data_ptr() == buf.data_ptr()
    if len(sizes) > 1 and sum(sizes):
        assert shuffle._as_one([buf[:2], buf[3:6]]) is None
        assert shuffle._as_one([buf[2:4], buf[:2]]) is None
        assert shuffle._as_one([buf[:2], buf.clone()[2:4]]) is None


@pytest.mark.parametrize("cap", [0, 1, 37, 100, 10 ** 6])
def test_landed_segment_matrix_of_a_clamped_push(cap):
    """peer._landed (the segment matrix of the per-split overlapped push) against a row-by-row walk of the
    source-major, bucket-major receive buffer that stops at the capacity."""
    from dpark_b200 import peer
    rng = np.random.default_rng(cap)
    seg = rng.integers(0, 30, (5, 7)).astype(np.int64)
    seg[1, :] = 0
    want = np.zeros_like(seg)
    row = 0
    for s in range(seg.shape[0]):
        for b in range(seg.shape[1]):
            for _ in range(seg[s, b]):
                if row < cap:
                    want[s, b] += 1
                row += 1
    got = peer._landed(torch.from_numpy(seg), cap).numpy()
    assert np.array_equal(got, want)
    assert np.array_equal(got, _landed_push(seg, cap))
