"""DparkContext + optParser: the entry points user scripts import
(`from dpark import DparkContext, optParser`, dpark/__init__.py:1-5).

Same names, flags and defaults as the reference (dpark/context.py:103-250,
396-411, 459-519) so scripts like examples/wc.py run unchanged.  The cluster
control plane (Mesos, multiprocess pools, web UI) is out of scope (SURVEY.md §2
rows 7-9): every master string selects the same in-process two-stage plan whose
shuffles run on the local GPU(s).
"""
import logging
import optparse
import os

from .rdd import ColumnarRDD, ParallelCollection, TextFileRDD, UnionRDD

logger = logging.getLogger("dpark")


class _Parser(optparse.OptionParser):
    def _process_args(self, largs, rargs, values):
        # unknown flags are left in args instead of aborting (the reference does the same)
        while rargs:
            try:
                optparse.OptionParser._process_args(self, largs, rargs, values)
            except (optparse.BadOptionError, optparse.AmbiguousOptionError) as e:
                largs.append(e.opt_str)


parser = _Parser(usage="Usage: %prog [options] [args]")


def _add_default_options():
    g = optparse.OptionGroup(parser, "Dpark Options")
    g.add_option("-m", "--master", type="string", default="local",
                 help="local, process, or a cluster master (all run in-process on the local GPUs here)")
    g.add_option("-p", "--parallel", type="int", default=0, help="default parallelism")
    g.add_option("-c", "--cpus", type="float", default=1.0, help="accepted, ignored")
    g.add_option("-M", "--mem", type="string", help="accepted, ignored")
    g.add_option("-g", "--group", type="string", default="", help="accepted, ignored")
    g.add_option("--err", type="float", default=0.0, help="accepted, ignored")
    g.add_option("--checkpoint_dir", type="string", default="", help="accepted, ignored")
    g.add_option("--color", action="store_true")
    g.add_option("--no-color", action="store_false", dest="color")
    g.add_option("--profile", action="store_true", help="print per-kernel CUDA-event times of each shuffle")
    g.add_option("--role", type="string", default="")
    g.add_option("-I", "--image", type="string", help="accepted, ignored")
    g.add_option("-V", "--volumes", type="string", help="accepted, ignored")
    parser.add_option_group(g)
    parser.add_option("-q", "--quiet", action="store_true")
    parser.add_option("-v", "--verbose", action="store_true")


_add_default_options()


def parse_options():
    options, args = parser.parse_args()
    options.logLevel = (options.quiet and logging.ERROR or options.verbose and logging.DEBUG or logging.INFO)
    logging.basicConfig(level=options.logLevel)
    return options


class DparkContext(object):
    """Process-wide singleton, like the reference's @singleton class
    (dpark/context.py:103)."""
    _instance = None
    options = None

    def __new__(cls, master=None):
        if cls._instance is None:
            cls._instance = object.__new__(cls)
            cls._instance._setup(master)
        return cls._instance

    def _setup(self, master):
        self.master = master
        self.initialized = False
        self.started = False
        self.is_local = True
        self.defaultParallelism = 2
        self.defaultMinSplits = 2
        self.nextShuffleId = 0
        self.nextRddId = 0

    def __init__(self, master=None):
        pass

    def init(self):
        if self.initialized:
            return
        cls = self.__class__
        if cls.options is None:
            cls.options = parse_options()
        options = cls.options
        self.master = self.master or options.master
        if options.parallel:
            self.defaultParallelism = options.parallel
        else:
            # LocalScheduler.defaultParallelism() == 2 in the reference (schedule.py:814-829);
            # 'process' defaults to the CPU count
            self.defaultParallelism = 2 if self.master == "local" else (os.cpu_count() or 2)
        self.defaultMinSplits = max(self.defaultParallelism, 2)
        self.initialized = True
        self._join_process_group()

    @staticmethod
    def _join_process_group():
        """Launched under torchrun (WORLD_SIZE > 1): one driver process per GPU, all running this script
        (dpark_b200/spmd.py).  The process group is created here so that user scripts stay unchanged."""
        world = int(os.environ.get("WORLD_SIZE", "1"))
        if world <= 1:
            return
        import torch
        import torch.distributed as dist
        if dist.is_available() and not dist.is_initialized():
            local = int(os.environ.get("LOCAL_RANK", "0"))
            if torch.cuda.is_available():
                from . import shuffle
                shuffle.bind_to_gpu_numa_node(local)
                torch.cuda.set_device(local)
                dist.init_process_group("nccl", device_id=torch.device("cuda", local))
            else:
                dist.init_process_group("gloo")

    @staticmethod
    def setLogLevel(level):
        logging.getLogger("dpark").setLevel(level)

    def newShuffleId(self):
        self.nextShuffleId += 1
        return self.nextShuffleId

    def newRddId(self):
        self.nextRddId += 1
        return self.nextRddId

    # ---------------------------------------------------------------- sources
    def parallelize(self, seq, numSlices=None):
        self.init()
        if numSlices is None:
            numSlices = self.defaultParallelism
        return ParallelCollection(self, seq, numSlices)

    def makeRDD(self, seq, numSlices=None):
        return self.parallelize(seq, numSlices)

    def accumulator(self, init=0, param=None):
        """dpark/context.py:364-365."""
        from .accumulator import Accumulator
        return Accumulator(init, param)

    def parallelizeColumns(self, keys, values, numSlices=None):
        """Extension: a (k, v) RDD from two columns (numpy arrays or torch tensors,
        host or cuda) -- rows never become Python tuples on the way to the shuffle."""
        self.init()
        if numSlices is None:
            numSlices = self.defaultParallelism
        return ColumnarRDD(self, keys, values, numSlices)

    def textFile(self, path, ext="", followLink=True, maxdepth=0, cls=TextFileRDD, *ka, **kws):
        self.init()
        if isinstance(path, (list, tuple)):
            return self.union([self.textFile(p, ext, followLink, maxdepth, cls, *ka, **kws) for p in path])
        path = os.path.realpath(path)
        if os.path.isdir(path):
            paths = []
            for root, dirs, names in os.walk(path, followlinks=followLink):
                if maxdepth > 0:
                    depth = len([f for f in root[len(path):].split("/") if f]) + 1
                    if depth > maxdepth:
                        break
                for n in sorted(names):
                    if n.endswith(ext) and not n.startswith("."):
                        p = os.path.join(root, n)
                        if followLink or not os.path.islink(p):
                            paths.append(p)
                dirs.sort()
                for d in dirs[:]:
                    if d.startswith("."):
                        dirs.remove(d)
            return self.union([cls(self, p, *ka, **kws) for p in paths])
        return cls(self, path, *ka, **kws)

    def textFileColumns(self, path, key=0, value=1, types=(int, int), sep=None, ext="", followLink=True, maxdepth=0,
                        numSplits=None, splitSize=None):
        """Extension: a ColumnarRDD of two numeric fields per line, parsed on the GPU -- split i holds the rows split i
        of textFile(path, ext, followLink, maxdepth, numSplits=..., splitSize=...).map(parse) yields, with
        parse(line) = (types[0](f[key]), types[1](f[value])) for f = line.split(sep).  types: int (int64 column) or
        float (float64).  Built, and its errors raised, here (dpark_b200/textcolumns.py)."""
        self.init()
        from . import textcolumns
        return textcolumns.text_file_columns(self, path, key, value, types, sep, ext, followLink, maxdepth,
                                             numSplits, splitSize)

    def union(self, rdds):
        return UnionRDD(self, rdds)

    # ------------------------------------------------------------------- jobs
    def runJob(self, rdd, func, partitions=None, allowLocal=False):
        """Yields func(iterator) per partition, in partition order
        (dpark/context.py:396-411; dpark/schedule.py:669-672)."""
        self.init()
        self.started = True
        splits = rdd.splits
        if partitions is None:
            partitions = range(len(splits))
        from . import spmd
        rank, world = spmd.rank_world()
        if world == 1:
            for i in partitions:
                yield func(rdd.iterator(splits[i]))
            return
        # one driver process per GPU, all running this script (dpark_b200/spmd.py): every rank joins the lineage's
        # shuffles, computes the partitions it owns, and the per-partition results are shared with all ranks
        partitions = list(partitions)
        spmd.materialize_lineage(rdd)
        n = len(splits)
        mine = [(i, func(rdd.iterator(splits[i]))) for i in partitions if spmd.owner_of(i, n, world) == rank]
        results = {}
        for part in spmd.all_gather_objects(mine):
            results.update(part)
        spmd.sync_accumulators()
        for i in partitions:
            yield results[i]

    def start(self):
        self.init()
        self.started = True

    def stop(self):
        self.started = False

    def clear(self):
        pass

    def __getstate__(self):
        raise ValueError("should not pickle ctx")
