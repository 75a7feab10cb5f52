"""Shared pieces of the shuffle parity tests: the dpk_set_option switches with their defaults, the fixture that sets
them for one test, the variant tables the GPU tests run, and the reduce-side input shapes (the CPU suite checks,
through tests/hostcheck.cu, that each shape reaches the kernel path it is named for)."""
import numpy as np
import pytest

# Every switch dpk_set_option accepts, with its default (documented in include/dpark_b200.h).
DEFAULT_OPTIONS = {
    "reduce_impl": 2, "agg_impl": 1, "agg_cursor": 1, "agg_batched": 0, "agg_ctas": 4, "agg_pipe": 0,
    "agg_wide": 1, "agg_split": 1, "agg_target_rows": 2048, "agg_timing": 0,
    "count_mode": 1, "scatter_bulk": 1, "scatter_threads": 512, "scatter_seg_wide": 1, "scatter_items": 16,
    "scatter_wide_from": 512, "scatter_ptr_bulk": 1, "scatter_ptr_threads": 1024,
    "copy_sms": 0, "copy_tma": 1,
}


@pytest.fixture
def dpk_options():
    """dpk_options({"agg_pipe": 1}) applies switches for the running test; every switch it set goes back to its
    default in teardown, whether the test passed or not."""
    from dpark_b200 import _native
    touched = []

    def apply(opts):
        for name, value in opts.items():
            touched.append(name)
            _native.set_option(name, value)
    yield apply
    for name in touched:
        _native.set_option(name, DEFAULT_OPTIONS[name])


# Reduce side (dpk_combine): every variant must give the oracle's result.
REDUCE_VARIANTS = [
    {},
    {"agg_ctas": 3},
    {"agg_split": 0},
    {"agg_batched": 1},
    {"agg_cursor": 0},
    {"agg_pipe": 1},
    {"agg_pipe": 2},
    {"agg_pipe": 1, "agg_batched": 1},
    {"agg_impl": 0, "agg_wide": 1},
    {"agg_impl": 0, "agg_wide": 0},
    {"reduce_impl": 1},
    {"reduce_impl": 0},
    {"agg_target_rows": 64},
    {"agg_target_rows": 3584},
]

# Map side (dpk_partition*): multisplit kernels and their launch shapes.
MULTISPLIT_VARIANTS = [
    {},
    {"count_mode": 0},
    {"scatter_items": 8},
    {"scatter_bulk": 0},
    {"scatter_threads": 256},
    {"scatter_threads": 1024},
    {"scatter_seg_wide": 0},
    {"scatter_wide_from": 0},
]

# Pointer mode (dpk_partition_scatter_ptrs) and the segment copies (dpk_copy_segments).
POINTER_VARIANTS = [{"scatter_ptr_threads": 512}, {"scatter_ptr_threads": 1024}, {"scatter_ptr_bulk": 0}]
COPY_VARIANTS = [{"copy_tma": 0}, {"copy_tma": 1}]


def variant_id(opts):
    return ",".join("%s=%s" % kv for kv in opts.items()) or "default"


# Second-level split defaults of the reduce side (dpk_combine.cu / dpk_aggregate*.cuh).
AGG_TARGET_ROWS = 2048      # agg_target_rows default
AG2_CAP = 2048              # rows of one staging window of k_smem_aggregate2
AG_LIMIT = 3584             # distinct keys one pass of the round-1 kernel holds


def reduce_shape(name):
    """([(keys, values), ...], P, sub_bits) of a reduce-side input shape: int64 keys and values, one input per run
    (`tiny` has three: n = 0, 1 and 31).  sub_bits None = what shuffle.reduce_by_key chooses."""
    rng = np.random.default_rng(77)
    if name == "distinct":              # mostly distinct keys: every fine bucket fits one window
        n, P, sb = 300_000, 8, None
        k = rng.integers(-2 ** 62, 2 ** 62, n, dtype=np.int64)
        k[: n // 10] = k[n // 10: n // 5]
    elif name == "hot_keys":            # 5 keys hold 6/7 of the rows: fine buckets far above one window
        n, P, sb = 1_000_000, 2, 0
        k = rng.integers(0, 5, n, dtype=np.int64)
        k[::7] = rng.integers(0, 10 ** 6, len(k[::7]))
    elif name == "distinct_overflow":   # more distinct keys per fine bucket than a table holds: hash-disjoint passes
        n, P, sb = 6_000_000, 1, 0
        k = rng.permutation(n).astype(np.int64) * 7919 - 10 ** 9
    elif name == "sentinel_key":        # the key whose bits equal the free-slot marker of the slot tables
        n, P, sb = 200_000, 2, 0
        k = rng.integers(-100, 100, n, dtype=np.int64)
        k[::3] = -2 ** 63
    elif name == "tiny":                # most of the 64 partitions empty
        P, sb = 64, None
        return [(rng.integers(-50, 50, m, dtype=np.int64), rng.integers(-1000, 1000, m, dtype=np.int64))
                for m in (0, 1, 31)], P, sb
    else:
        raise ValueError(name)
    v = rng.integers(-1000, 1000, n, dtype=np.int64)
    return [(k, v)], P, sb


REDUCE_SHAPES = ["distinct", "hot_keys", "distinct_overflow", "sentinel_key", "tiny"]
