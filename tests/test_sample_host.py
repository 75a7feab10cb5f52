"""The device sample on a CPU: the MT19937 replay of dpk_common.cuh run through tests/samplecheck.cu, twist by twist in
the kernel's three phases, against Python's random.Random and numpy's MT19937 bit generator; the keep rule; which calls
take the device path; the host side of the thresholds (states, the refold of the first digest, the split helpers of
quantiles.skew_thresholds).  The device results themselves are checked in tests/test_gpu_sample.py."""
import ctypes as C
import math
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from dpark_b200 import quantiles, sampling, spmd
from dpark_b200.rdd import ColumnarRDD, SampleRDD, UnionRDD
from tests import cogroup_common as cc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEEDS = [0, 1, 12345, -1, -7, -2 ** 40, 2 ** 32 - 1, 2 ** 32, 2 ** 40, 2 ** 64 + 3, 10 ** 30]
TWISTS = 10


def samplecheck():
    path = os.path.join(ROOT, "tests", "_samplecheck.so")
    if not os.path.exists(path):
        subprocess.call([sys.executable, "-c", "import __graft_entry__ as g; g.build()"], cwd=ROOT)
    if not os.path.exists(path):
        pytest.skip("samplecheck not built")
    L = C.CDLL(path)
    vp, i32, i64, u32, dbl = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_double
    L.smc_state_words.restype = L.smc_phase.restype = L.smc_keep.restype = i32
    L.smc_phase.argtypes = [i32]
    L.smc_temper.restype = u32
    L.smc_temper.argtypes = [u32]
    L.smc_double.restype = dbl
    L.smc_double.argtypes = [u32, u32]
    L.smc_keep.argtypes = [dbl, dbl]
    L.smc_words.argtypes = [vp, i64, vp]
    L.smc_draws.argtypes = [vp, i64, dbl, vp, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _state(seed):
    return np.array(random.Random(seed).getstate()[1][:624], dtype=np.uint32)


def harness_words(L, seed, n):
    out = np.zeros(n, dtype=np.uint32)
    L.smc_words(_p(_state(seed)), n, _p(out))
    return out


def harness_draws(L, seed, n, frac=0.5):
    out, keep = np.zeros(n), np.zeros(n, dtype=np.uint8)
    L.smc_draws(_p(_state(seed)), n, frac, _p(out), _p(keep))
    return out, keep.astype(bool)


def numpy_words(seed, n):
    bg = np.random.MT19937()
    st = bg.state
    st["state"]["key"], st["state"]["pos"] = _state(seed), 624
    bg.state = st
    return bg.random_raw(n).astype(np.uint32)


def test_phases_cover_the_state_in_the_kernel_order():
    L = samplecheck()
    assert L.smc_state_words() == 624
    assert [L.smc_phase(p) for p in range(4)] == [0, 227, 454, 624]


@pytest.mark.parametrize("seed", SEEDS)
def test_words_and_draws_equal_python_and_numpy(seed):
    L = samplecheck()
    n = TWISTS * 624 + 17
    rd = random.Random(seed)
    assert harness_words(L, seed, n).tolist() == [rd.getrandbits(32) for _ in range(n)]
    assert np.array_equal(harness_words(L, seed, n), numpy_words(seed, n))
    rd = random.Random(seed)
    draws, _ = harness_draws(L, seed, TWISTS * 312 + 5)
    assert [x.hex() for x in draws.tolist()] == [rd.random().hex() for _ in range(len(draws))]


def test_the_skew_seeds_of_a_thousand_splits():
    """random.Random(12345 + i) for every split index i < 1000: ten twists against numpy, two against Python."""
    L = samplecheck()
    for i in range(1000):
        seed = 12345 + i
        assert np.array_equal(harness_words(L, seed, TWISTS * 624), numpy_words(seed, TWISTS * 624)), seed
        rd = random.Random(seed)
        draws, _ = harness_draws(L, seed, 2 * 312)
        assert draws.tolist() == [rd.random() for _ in range(len(draws))], seed


def test_tempering_and_double_assembly():
    L = samplecheck()
    rng = np.random.default_rng(0)
    for y in rng.integers(0, 2 ** 32, 1000).tolist() + [0, 1, 2 ** 31, 2 ** 32 - 1]:
        t = y ^ (y >> 11)
        t ^= (t << 7) & 0x9d2c5680
        t ^= (t << 15) & 0xefc60000
        t = (t ^ (t >> 18)) & 0xFFFFFFFF
        assert L.smc_temper(y) == t
    for w0, w1 in [(0, 0), (2 ** 32 - 1, 2 ** 32 - 1), (2 ** 31, 63), (5, 2 ** 32 - 64)]:
        assert L.smc_double(w0, w1) == ((w0 >> 5) * 67108864.0 + (w1 >> 6)) * (1.0 / 9007199254740992.0)
    assert L.smc_double(2 ** 32 - 1, 2 ** 32 - 1) < 1.0


def test_keep_rule_at_the_edges():
    L = samplecheck()
    draws, _ = harness_draws(L, 12345, 5000)
    for u in draws[:50].tolist():
        assert L.smc_keep(u, u) == 1
        assert L.smc_keep(u, math.nextafter(u, -1.0)) == 0
        assert L.smc_keep(u, 0.0) == (u <= 0.0)
        assert L.smc_keep(u, 1.0) == 1 and L.smc_keep(u, 1.5) == 1
        assert L.smc_keep(u, float("nan")) == 0
    assert L.smc_keep(0.0, 0.0) == 1 and L.smc_keep(0.0, -0.0) == 1 and L.smc_keep(0.0, -1e-300) == 0
    frac = draws[123]
    _, keep = harness_draws(L, 12345, 5000, frac)
    rd = random.Random(12345)
    assert keep.tolist() == [rd.random() <= frac for _ in range(5000)]
    for frac in (0.0, 1.0, 1.5, float("nan"), 0.3):
        _, keep = harness_draws(L, 12345, 2000, frac)
        rd = random.Random(12345)
        assert keep.tolist() == [rd.random() <= frac for _ in range(2000)]


def test_int_fractions_compare_as_python_does():
    for frac in (0, 1, 2, -1, -10 ** 400, 10 ** 400, True):
        arg = sampling._frac_arg(frac)
        for u in (0.0, 5e-324, 0.5, 1 - 2 ** -53):
            assert (u <= arg) == (u <= frac)


def test_states_are_the_ones_random_starts_from():
    st = sampling.mt_states(2 ** 40, 3).numpy().view(np.uint32)
    for i in range(3):
        assert st[i].tolist() == list(random.Random(2 ** 40 + i).getstate()[1][:624])
    for bad in (None, "7", (1,)):
        with pytest.raises(TypeError) as e_dev:
            sampling.mt_states(bad, 2)
        with pytest.raises(TypeError) as e_rows:
            random.Random(bad + 0)
        assert str(e_dev.value) == str(e_rows.value)


# ------------------------------------------------------------------------------------------------ path selection
def _col(dc, n=40, kdt=torch.int64, vdt=torch.int64, M=3):
    return dc.parallelizeColumns(torch.arange(n).to(kdt), torch.arange(n).to(vdt), M)


class _Sub(ColumnarRDD):
    pass


def test_which_samples_run_on_the_device(monkeypatch):
    dc = cc.ctx()
    col = _col(dc)
    s = col.sample(0.3)
    assert type(s) is sampling.ColumnarSampleRDD and isinstance(s, SampleRDD)
    assert s.splits is col.splits and s.partitioner is None and s._result is None       # nothing drawn yet
    assert (s.frac, s.withReplacement, s.seed) == (0.3, False, 12345)
    for dt in (torch.int32, torch.int64, torch.float32, torch.float64):
        assert type(_col(dc, kdt=dt, vdt=dt).sample(1)) is sampling.ColumnarSampleRDD
    sub = _Sub(dc, torch.arange(10), torch.arange(10), 2)
    assert type(sub.sample(0.3)) is SampleRDD
    assert type(dc.parallelize(list(zip(range(9), range(9))), 3).sample(0.3)) is SampleRDD
    assert type(col.sample(0.3, True)) is SampleRDD
    assert type(col.sample(0.3, 1)) is SampleRDD
    from fractions import Fraction
    for frac in ("0.3", np.float64(0.3), Fraction(1, 3), None, True):
        assert type(col.sample(frac)) is SampleRDD
    assert type(col.union(col).sample(0.3)) is SampleRDD
    flat = dc.parallelizeColumns(torch.arange(10).view(5, 2), torch.arange(10).view(5, 2), 2)
    assert type(flat.sample(0.3)) is SampleRDD
    u8 = dc.parallelizeColumns(torch.arange(10, dtype=torch.uint8), torch.arange(10), 2)
    assert type(u8.sample(0.3)) is SampleRDD
    monkeypatch.setattr(spmd, "rank_world", lambda: (0, 2))
    assert type(col.sample(0.3)) is SampleRDD


def test_which_thresholds_run_on_the_device(monkeypatch):
    dc = cc.ctx()
    a, b = _col(dc), _col(dc, kdt=torch.float32)
    assert sampling.thresholds_inputs(a, 0.1) == [a]
    assert sampling.thresholds_inputs(a, 2) == [a]
    u = a.union(b, a)
    assert type(u) is UnionRDD and sampling.thresholds_inputs(u, 0.1) == [a, b, a]
    rows = dc.parallelize([(1, 2)], 1)
    assert sampling.thresholds_inputs(a.union(rows), 0.1) is None
    sub = _Sub(dc, torch.arange(10), torch.arange(10), 2)
    assert sampling.thresholds_inputs(sub, 0.1) is None
    assert sampling.thresholds_inputs(a.union(sub), 0.1) is None
    assert sampling.thresholds_inputs(a.map(lambda x: x), 0.1) is None
    assert sampling.thresholds_inputs(a.union(a).union(a), 0.1) is None       # a union of a union: rows, as before
    assert sampling.thresholds_inputs(a, "0.1") is None
    assert sampling.thresholds_inputs(a, np.float64(0.1)) is None
    flat = dc.parallelizeColumns(torch.arange(10).view(5, 2), torch.arange(10).view(5, 2), 2)
    assert sampling.thresholds_inputs(flat, 0.1) is None
    assert sampling.thresholds_inputs(a.union(flat), 0.1) is None
    monkeypatch.setattr(spmd, "rank_world", lambda: (0, 2))
    assert sampling.thresholds_inputs(a, 0.1) is None
    assert sampling.thresholds_inputs(a.union(b), 0.1) is None


def test_partitioners_still_route_through_skew_thresholds(monkeypatch):
    """_combine_partitioner and _cogroup_partitioner call RDD._skew_thresholds as before, with the same arguments."""
    from dpark_b200 import HashPartitioner
    from dpark_b200.rdd import RDD
    dc = cc.ctx()
    a, b = _col(dc), _col(dc, M=2)
    calls = []

    def fake(self, splits, rate):
        calls.append((type(self).__name__, len(self), splits, rate))
        return [1, 2], 3

    monkeypatch.setattr(RDD, "_skew_thresholds", fake)
    assert a._combine_partitioner(5, 0.1) == HashPartitioner(3, thresholds=[1, 2])
    assert a._cogroup_partitioner([b], 5, 0.2) == HashPartitioner(3, thresholds=[1, 2])
    assert calls == [("ColumnarRDD", 3, 5, 0.1), ("UnionRDD", 5, 5, 0.2)]


# ------------------------------------------------------------------------------------------------ thresholds, host side
def _old_skew_thresholds(hash_partitions, splits):
    """quantiles.skew_thresholds as it read before the rule moved into thresholds_of."""
    step = 100. / splits
    marks = [step * i for i in range(1, splits)]
    pcts = quantiles.percentiles_of_partitions(hash_partitions, marks)
    if not pcts:
        return None, splits
    thr = []
    for p in pcts:
        if math.isnan(p):
            continue
        p = int(math.ceil(p))
        if not thr or p > thr[-1]:
            thr.append(p)
    return thr, len(thr) + 1


def test_skew_thresholds_unchanged_by_the_helper_split():
    rnd = random.Random(9)
    cases = [([[], []], 4), ([[5]], 1), ([[5]], 2), ([[], [3, 3, 3]], 7), ([[2 ** 62, -2 ** 62], [0]], 3)]
    for _ in range(30):
        parts = [[rnd.randrange(-2 ** 61, 2 ** 61) for _ in range(rnd.randrange(0, 400))]
                 for _ in range(rnd.randrange(1, 6))]
        cases.append((parts, rnd.choice([2, 3, 7, 64, 1000])))
    for parts, splits in cases:
        assert quantiles.skew_thresholds(parts, splits) == _old_skew_thresholds(parts, splits)
    assert [m / 100. for m in quantiles.skew_marks(64)] == [(100. / 64 * i) / 100. for i in range(1, 64)]


@pytest.mark.parametrize("n", [1, 2, 30, 209, 5000])
def test_refold_of_the_first_digest_is_the_compositions(n):
    """An empty first split: the composition's chain holds E.absorb(d) for the first non-empty digest d, which
    _refold_first writes over d's device slots (CPU tensors stand in for them here)."""
    rnd = random.Random(n)
    vals = [rnd.randrange(-2 ** 61, 2 ** 61) for _ in range(n)]
    d = quantiles.MergingDigest().update(vals)
    d.compress()
    c = len(d.means)
    cm = torch.tensor(d.means + [7.0] * 3, dtype=torch.float64)
    cw = torch.tensor(d.weights + [7.0] * 3, dtype=torch.float64)
    cnt, lohi = torch.tensor([c, 5], dtype=torch.int32), torch.tensor([d.lo, d.hi, 1.0, 2.0], dtype=torch.float64)
    sampling._refold_first((cm, cw, cnt, lohi))
    e = quantiles.MergingDigest()
    e.absorb(quantiles.MergingDigest().update(vals))
    m = int(cnt[0])
    assert m == len(e.means) and cnt[1] == 5
    assert cm[:m].tolist() == e.means and cw[:m].tolist() == e.weights
    assert lohi.tolist() == [e.lo, e.hi, 1.0, 2.0]
    # the composition's percentiles after an empty first split are queried from that refolded chain
    marks = quantiles.skew_marks(16)
    assert quantiles.percentiles_of_partitions([[], vals], marks) == [e.quantile(p / 100.) for p in marks]
