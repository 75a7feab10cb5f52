"""The operator surface with one driver process per rank (dpark_b200/spmd.py), world_size 2 over gloo on CPU.

What is under test is the SPMD plumbing: split ownership, the lineage walk that makes every rank join a shuffle's
collectives, routing rows to the rank that owns their partition (pickled columns in one all_to_all), sharing results,
accumulators summed over the ranks -- with the GPU stages replaced by oracle-based stand-ins (the kernels need a GPU;
`-m gpu` and scripts/spmd_check.py run the real thing).  Every rank must see exactly what one process computes."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _patch_gpu_stages():
    """Oracle-based stand-ins for the device stages of the routed shuffle."""
    import numpy as np
    from oracle import oracle as orc
    from dpark_b200 import _native as nv
    from dpark_b200 import columnar, engine

    def hash_column(keys):
        return torch.tensor([orc.portable_hash(k) for k in keys], dtype=torch.int64)

    def partition_ids(h, P, thr=None):
        t = None if thr is None else thr.numpy()
        return torch.from_numpy(orc.partition_vec(h.numpy(), P, t))

    def local(kind):
        def run(splits, P, thr, *rest):
            res = engine.ShuffleResult(P)
            buckets = [dict() for _ in range(P)]
            op = rest[0] if kind == "reduce" else None
            f = {"sum": lambda a, b: a + b, "min": min, "max": max}.get(op)
            for c in splits:
                keys = columnar.decode_keys(c.key_kind, c.keys, c.key_offsets, c.key_objs)
                vals = c.objs if c.objs is not None else c.vals.tolist()
                for k, v in zip(keys, vals):
                    b = buckets[orc.get_partition(k, P, thr)]
                    if kind == "group":
                        b.setdefault(k, []).append(v)
                    else:
                        b[k] = f(b[k], v) if k in b else v
            for p, b in enumerate(buckets):
                res.parts[p] = (list(b.keys()), list(b.values()))
            return res
        return run
    columnar._hash_column = hash_column
    nv.partition_ids = partition_ids
    engine._device = lambda: torch.device("cpu")
    engine.TEXT_INGEST = False     # the device tokeniser needs a GPU (tests/test_gpu_textingest.py); rows go through Python here
    engine.ROUTE_EVERYTHING = True
    engine._run_reduce = local("reduce")
    engine._run_group = local("group")


def _job(dc):
    """A little of everything: str-key reduceByKey (wc shape), object-valued groupByKey, a join, an accumulator,
    a co-partitioned cogroup through Bagel."""
    from dpark_b200 import bagel
    out = {}
    words = ["w%d" % (i * 7 % 23) for i in range(400)]
    acc = dc.accumulator(0)

    def one(w):
        acc.add(1)
        return (w, 1)
    out["wc"] = sorted(dc.parallelize(words, 5).map(one).reduceByKey(lambda a, b: a + b, 3).collect())
    out["acc"] = acc.value
    g = dc.parallelize([(i % 7, ("v", i)) for i in range(60)], 4).groupByKey(5)
    out["group"] = sorted((k, list(v)) for k, v in g.collect())
    a = dc.parallelize([(i, i * i) for i in range(20)], 3)
    b = dc.parallelize([(i, str(i)) for i in range(0, 20, 3)], 2)
    out["join"] = sorted(a.join(b, 4).collect())
    out["glom_sizes"] = [len(p) for p in dc.parallelize(words, 5).map(lambda w: (w, 1)).reduceByKey(lambda x, y: x + y, 3)
                         .glom().collect()]
    n = 12

    def compute(vert, msg_sum, agg, step):
        new = 0.15 / n + 0.85 * msg_sum[0] if msg_sum and msg_sum[0] else vert.value
        done = step >= 4
        outbox = [] if done else [(e.target_id, new / len(vert.outEdges)) for e in vert.outEdges]
        return bagel.Vertex(vert.id, new, vert.outEdges, not done), outbox
    verts = dc.parallelize([(i, bagel.Vertex(i, 1.0 / n, [bagel.Edge((i + 1) % n), bagel.Edge((i * 5 + 2) % n)], True))
                            for i in range(n)], 3)
    ranks = bagel.Bagel.run(dc, verts, dc.parallelize([], 3), compute, numSplits=4)
    out["pagerank"] = sorted((k, round(v.value, 12)) for k, v in ranks.collect())
    return out


def _outcome(f):
    try:
        return ("ok", f())
    except Exception as e:
        return (type(e).__name__, str(e))


def _agreed_checks_job(dc):
    """The checks one process makes over the whole input, where no rank's own splits fail them: the int64 sum bound
    (rank 0 holds 2^62 + 1, rank 1 holds 2^62 + 2^62) and a NaN key of a ColumnarRDD in rank 1's split.  Both are
    decided from the descriptors every rank all-gathers before the first collective, so no device stage runs."""
    import numpy as np
    import operator
    from dpark_b200.rdd import ColumnarRDD
    rows = [(7, 2 ** 62), (8, 1), (7, 2 ** 62), (7, 2 ** 62)]
    cols = ColumnarRDD(dc, np.array([1.0, 2.0, 3.0, np.nan]), np.arange(4, dtype=np.int64), 0, bounds=[0, 2, 4])
    return {"sum": _outcome(lambda: dc.parallelize(rows, 2).reduceByKey(operator.add, 3).collect()),
            "nan": _outcome(lambda: cols.reduceByKey(operator.add, 2).collect())}


def _worker(rank, world, port, out_q, job="_job"):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sys.argv = [sys.argv[0]]
    if world > 1:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        _patch_gpu_stages()
        from dpark_b200 import DparkContext
        out_q.put((rank, globals()[job](DparkContext("local"))))
    except Exception as e:                      # surface the failure instead of leaving the other rank waiting
        import traceback
        out_q.put((rank, {"error": "%s\n%s" % (e, traceback.format_exc())}))
    finally:
        if world > 1:
            dist.destroy_process_group()


def _run(world, job="_job"):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q, job)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    return got


def test_two_driver_processes_see_what_one_process_computes():
    one = _run(1)[0]
    two = _run(2)
    for r in two.values():
        assert "error" not in r, r["error"]
    assert one["acc"] == 400 and one["wc"] and one["group"] and one["join"] and len(one["pagerank"]) == 12
    for rank in (0, 1):
        assert two[rank] == one, "rank %d diverged" % rank


def test_whole_input_checks_are_agreed_by_every_rank():
    from dpark_b200 import columnar, engine
    with pytest.raises(OverflowError) as big:          # one process, over both splits
        engine._check_int_sum_range([columnar.ingest_pairs([(7, 2 ** 62), (8, 1)]),
                                     columnar.ingest_pairs([(7, 2 ** 62), (7, 2 ** 62)])], {columnar.VAL_I64}, "sum")
    want = {"sum": ("OverflowError", str(big.value)),
            "nan": ("TypeError", "NaN keys are not supported (CPython hashes NaN by identity)")}
    two = _run(2, "_agreed_checks_job")
    for rank in (0, 1):
        assert "error" not in two[rank], two[rank]["error"]
        assert two[rank] == want, "rank %d" % rank
