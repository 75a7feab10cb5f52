"""ctypes binding of libdpark_b200.so (include/dpark_b200.h).

The CUDA extension is the product: if the library is missing or a tensor is not
on a CUDA device this module raises -- there is no CPU fallback for the shuffle
path.  torch is used only for device memory and streams.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdpark_b200.so")

OK, ERR_INVALID, ERR_UNSUPPORTED, ERR_WORKSPACE, ERR_CUDA = 0, -1, -2, -3, -4
K_HASHED = -1
K_I64, K_I32, K_F64, K_U64, K_F32, K_ROWID = 0, 1, 2, 3, 4, 5
V_I64, V_F64, V_I32, V_F32 = 0, 1, 2, 3
OPS = {"sum": 0, "min": 1, "max": 2, "prod": 3, "and": 4, "or": 5, "xor": 6}
BYTES_SIGNED, STR_UTF8 = 0, 1
MAX_PARTITIONS = 4096

_KEY_KIND = {torch.int64: K_I64, torch.int32: K_I32, torch.float64: K_F64, torch.float32: K_F32}
if hasattr(torch, "uint64"):
    _KEY_KIND[torch.uint64] = K_U64
_VAL_KIND = {torch.int64: V_I64, torch.float64: V_F64, torch.int32: V_I32, torch.float32: V_F32}

# every symbol include/dpark_b200.h declares (tests check the library exports all of them)
EXPORTS = [
    "dpk_abi_version", "dpk_last_error", "dpk_device_info", "dpk_hash_keys", "dpk_hash_bytes",
    "dpk_partition_ids", "dpk_partition_workspace_bytes", "dpk_partition_count",
    "dpk_partition_scatter", "dpk_partition", "dpk_combine_workspace_bytes", "dpk_combine",
    "dpk_launch_count", "dpk_prof_enable", "dpk_prof_count", "dpk_prof_get",
    "dpk_dict_encode_workspace_bytes", "dpk_dict_encode", "dpk_set_option",
    "dpk_key_or", "dpk_radix_pass", "dpk_group_heads_workspace_bytes", "dpk_group_heads", "dpk_gather_i64",
    "dpk_partition_scatter_ptrs", "dpk_copy_segments", "dpk_hash_tuple", "dpk_push_plan", "dpk_push_plan_part", "dpk_pipe_plan", "dpk_fused_plan", "dpk_memcpy_batch",
    "dpk_tokenize_blocks", "dpk_tokenize_count", "dpk_tokenize_emit", "dpk_gather_bytes",
    "dpk_tokenize_utf8_count", "dpk_tokenize_utf8_emit", "dpk_textcols_count", "dpk_textcols_emit", "dpk_textcols_parse",
    "dpk_radix_pass_seg_workspace_bytes", "dpk_radix_pass_seg", "dpk_join_count", "dpk_join_emit",
    "dpk_cogroup_count", "dpk_cogroup_emit", "dpk_topk_lengths", "dpk_topk_round",
    "dpk_bcast_build", "dpk_bcast_probe", "dpk_bcast_emit", "dpk_sort_keys", "dpk_sort_cuts", "dpk_sort_gather",
    "dpk_tdigest_heads", "dpk_tdigest_build", "dpk_tdigest_merge", "dpk_sample_bernoulli",
    "dpk_select_round", "dpk_select_compact", "dpk_select_tiles", "dpk_select_take", "dpk_uniq_insert", "dpk_uniq_emit",
]

_lib = None


class NativeError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "dpark_b200: CUDA extension %s is missing -- build it with "
                "`python -c 'import __graft_entry__ as g; g.build()'` (there is no CPU fallback)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        i64, i32, vp, ci = C.c_int64, C.c_int32, C.c_void_p, C.c_int
        for name in EXPORTS:
            getattr(L, name).restype = ci
        L.dpk_last_error.restype = C.c_char_p
        L.dpk_partition_workspace_bytes.restype = i64
        L.dpk_combine_workspace_bytes.restype = i64
        L.dpk_launch_count.restype = i64
        L.dpk_device_info.argtypes = [vp]
        L.dpk_hash_keys.argtypes = [vp, ci, i64, vp, vp]
        L.dpk_hash_bytes.argtypes = [vp, vp, i64, ci, vp, vp]
        L.dpk_partition_ids.argtypes = [vp, i64, i32, vp, i32, vp, vp]
        L.dpk_hash_tuple.argtypes = [vp, i64, i32, vp, vp]
        L.dpk_partition_workspace_bytes.argtypes = [i64, i32]
        L.dpk_partition_count.argtypes = [vp, ci, vp, i64, i32, vp, i32, i32, vp, vp, i64, vp]
        L.dpk_partition_scatter.argtypes = [vp, ci, vp, vp, i32, i64, i32, vp, i32, i32, vp, vp, vp, vp, i64, vp]
        L.dpk_partition.argtypes = [vp, ci, vp, vp, i32, i64, i32, vp, i32, i32, vp, vp, vp, vp, i64, vp]
        L.dpk_partition_scatter_ptrs.argtypes = [vp, ci, vp, vp, i32, i64, i32, vp, i32, i32, vp, vp, vp, i64, vp]
        L.dpk_copy_segments.argtypes = [vp, vp, vp, i32, vp]
        L.dpk_push_plan.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, C.c_uint64, C.c_uint64, vp, i32, i32, i64, vp, vp, vp, vp, vp, vp]
        L.dpk_push_plan_part.argtypes = [vp, i32, i32, i32, i32, i32, i32, i64, i32, i32, i32, C.c_uint64, C.c_uint64, vp, i32, i32, i64, vp, vp, vp, vp, vp, vp]
        L.dpk_pipe_plan.argtypes = [vp, i32, i32, i32, i32, i32, i64, i32, i32, i32, C.c_uint64, C.c_uint64, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp]
        L.dpk_memcpy_batch.argtypes = [vp, vp, vp, i32, vp]
        L.dpk_fused_plan.argtypes = [vp, i32, i32, i32, i32, i32, vp, i32, i32, i64, C.c_uint64, C.c_uint64, vp, vp, vp, vp, vp]
        L.dpk_tokenize_blocks.restype = i64
        L.dpk_tokenize_blocks.argtypes = [i64]
        L.dpk_tokenize_count.argtypes = [vp, i64, vp, vp, vp]
        L.dpk_tokenize_emit.argtypes = [vp, i64, vp, vp, vp, vp]
        L.dpk_tokenize_utf8_count.argtypes = [vp, i64, vp, vp, vp]
        L.dpk_tokenize_utf8_emit.argtypes = [vp, i64, vp, vp, vp, vp]
        L.dpk_textcols_count.argtypes = [vp, i64, vp, vp, vp]
        L.dpk_textcols_emit.argtypes = [vp, i64, vp, vp, vp]
        L.dpk_textcols_parse.argtypes = [vp, i64, vp, i64, vp, i32, i32, i32, i32, i32, vp, vp, vp, vp]
        L.dpk_gather_bytes.argtypes = [vp, vp, vp, vp, i64, vp, vp, vp]
        L.dpk_combine_workspace_bytes.argtypes = [i64, i32, i32]
        L.dpk_combine.argtypes = [vp, ci, vp, vp, ci, i64, ci, i32, vp, i32, i32, i32, i32, i32, vp, vp, vp, vp,
                                  vp, vp, i64, vp]
        L.dpk_set_option.argtypes = [C.c_char_p, i64]
        L.dpk_key_or.argtypes = [vp, i64, vp, vp]
        L.dpk_gather_i64.argtypes = [vp, vp, i64, vp, vp]
        L.dpk_radix_pass.argtypes = [vp, vp, i32, i64, i32, i32, vp, vp, vp, i64, vp]
        L.dpk_radix_pass_seg_workspace_bytes.restype = i64
        L.dpk_radix_pass_seg_workspace_bytes.argtypes = [i64, i32, i32, i32]
        L.dpk_radix_pass_seg.argtypes = [vp, vp, i32, i64, i32, i32, i32, i32, vp, vp, vp, vp, vp, i64, vp]
        L.dpk_group_heads_workspace_bytes.restype = i64
        L.dpk_group_heads_workspace_bytes.argtypes = [i64]
        L.dpk_group_heads.argtypes = [vp, i64, vp, vp, vp, vp, i64, vp]
        L.dpk_dict_encode_workspace_bytes.restype = i64
        L.dpk_dict_encode_workspace_bytes.argtypes = [i64]
        L.dpk_dict_encode.argtypes = [vp, vp, vp, i64, vp, vp, i64, vp]
        L.dpk_join_count.argtypes = [vp, vp, i64, i64, i32, i32, vp, vp, vp]
        L.dpk_join_emit.argtypes = [vp, vp, vp, vp, vp, i64, i64, vp, i32, vp, i32, i32, i32, i64, vp, vp, vp, vp, vp,
                                    vp]
        L.dpk_cogroup_count.argtypes = [vp, vp, i64, vp, i32, vp, vp, vp]
        L.dpk_cogroup_emit.argtypes = [vp, vp, vp, i64, i64, vp, i32, i64, vp, vp]
        L.dpk_topk_lengths.argtypes = [vp, i64, i32, vp, vp]
        L.dpk_topk_round.argtypes = [vp, vp, i32, i32, vp, i64, i64, vp, i32, i32, vp, vp]
        L.dpk_bcast_build.argtypes = [vp, i64, vp, i64, vp]
        L.dpk_bcast_probe.argtypes = [vp, i32, i64, vp, i64, vp, vp, vp, vp]
        L.dpk_bcast_emit.argtypes = [vp, i32, vp, i32, vp, vp, i64, vp, vp, vp, i32, i64, vp, vp, vp, vp]
        L.dpk_sort_keys.argtypes = [vp, i32, vp, i32, i64, i32, vp, vp, vp, vp, vp]
        L.dpk_sort_cuts.argtypes = [vp, vp, vp, i32, i64, vp, i32, vp, i32, i32, vp, vp]
        L.dpk_sort_gather.argtypes = [vp, i32, vp, i32, vp, i64, vp, vp, vp]
        L.dpk_tdigest_heads.argtypes = [vp, i64, vp, i64, i64, vp, vp]
        L.dpk_tdigest_build.argtypes = [vp, vp, i32, vp, vp, i64, vp, vp, vp, vp, vp, vp, vp]
        L.dpk_tdigest_merge.argtypes = [vp, i64, vp, vp, i64, vp, vp, vp, vp, vp, i32, vp, vp, vp]
        L.dpk_sample_bernoulli.argtypes = [vp, vp, i64, C.c_double, vp, vp, vp]
        L.dpk_select_round.argtypes = [vp, vp, vp, i64, vp, vp, vp]
        L.dpk_select_compact.argtypes = [vp, vp, vp, i64, vp, vp, vp]
        L.dpk_select_tiles.restype = i64
        L.dpk_select_tiles.argtypes = [i64]
        L.dpk_select_take.argtypes = [vp, vp, i64, i64, vp, vp, vp, vp, vp]
        L.dpk_uniq_insert.argtypes = [vp, i32, vp, i32, i64, vp, i64, vp, vp]
        L.dpk_uniq_emit.argtypes = [vp, i64, vp, vp, vp, vp]
        L.dpk_prof_enable.argtypes = [ci]
        L.dpk_prof_get.argtypes = [ci, C.c_char_p, C.POINTER(C.c_float)]
        if L.dpk_abi_version() != 1:
            raise ImportError("dpark_b200: ABI version mismatch")
        _lib = L
        # DPK_OPTIONS="name=value,..." applies dpk_set_option switches at load (A/B runs of whole test suites)
        for item in filter(None, os.environ.get("DPK_OPTIONS", "").split(",")):
            name, _, value = item.partition("=")
            _check(L.dpk_set_option(name.strip().encode(), int(value)))
    return _lib


def _check(rc):
    if rc == OK:
        return
    msg = lib().dpk_last_error().decode("utf-8", "replace")
    if rc == ERR_UNSUPPORTED:
        raise TypeError(msg)
    if rc == ERR_INVALID:
        raise ValueError(msg)
    raise NativeError("dpark_b200 native error %d: %s" % (rc, msg))


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise NativeError("dpark_b200 shuffle kernels need CUDA tensors (no CPU fallback); got %s" % t.device)
        if t is not None and not t.is_contiguous():
            raise ValueError("columns must be contiguous")


def key_kind(t, prehashed=False):
    if prehashed:
        if t.dtype != torch.int64:
            raise TypeError("prehashed keys must be int64")
        return K_HASHED
    try:
        return _KEY_KIND[t.dtype]
    except KeyError:
        raise TypeError("%s is unhashable by portable_hash" % t.dtype)


def val_kind(t):
    try:
        return _VAL_KIND[t.dtype]
    except KeyError:
        raise TypeError("unsupported value dtype %s" % t.dtype)


def _thr(thresholds, device):
    if thresholds is None:
        return None, 0
    if not torch.is_tensor(thresholds):
        thresholds = torch.tensor(list(thresholds), dtype=torch.int64, device=device)
    thresholds = thresholds.to(device=device, dtype=torch.int64).contiguous()
    return thresholds, int(thresholds.numel())


def device_info():
    import numpy as np
    info = np.zeros(4, dtype=np.int32)
    _check(lib().dpk_device_info(info.ctypes.data_as(C.c_void_p)))
    return {"sm_count": int(info[0]), "cc": (int(info[1]), int(info[2])), "l2_mb": int(info[3])}


# ---- a1 / a2 -------------------------------------------------------------------
def hash_keys(keys):
    """portable_hash of a key column (dpark/portable_hash.pyx:51-70)."""
    _need_cuda(keys)
    out = torch.empty(keys.numel(), dtype=torch.int64, device=keys.device)
    _check(lib().dpk_hash_keys(_ptr(keys), key_kind(keys), keys.numel(), _ptr(out), _stream()))
    return out


def hash_bytes(data, offsets, mode):
    _need_cuda(data, offsets)
    n = offsets.numel() - 1
    out = torch.empty(n, dtype=torch.int64, device=offsets.device)
    _check(lib().dpk_hash_bytes(_ptr(data), _ptr(offsets), n, mode, _ptr(out), _stream()))
    return out


def hash_tuple(item_hashes):
    """tuple_hash (dpark/portable_hash.pyx:3-15) of n rows from their items' hashes: int64 tensor [arity, n]."""
    _need_cuda(item_hashes)
    arity, n = int(item_hashes.shape[0]), int(item_hashes.shape[1])
    out = torch.empty(n, dtype=torch.int64, device=item_hashes.device)
    _check(lib().dpk_hash_tuple(_ptr(item_hashes), n, arity, _ptr(out), _stream()))
    return out


def partition_ids(hashes, P, thresholds=None):
    """HashPartitioner.getPartition over a hash column (dpark/dependency.py:229-233)."""
    _need_cuda(hashes)
    thr, nthr = _thr(thresholds, hashes.device)
    out = torch.empty(hashes.numel(), dtype=torch.int32, device=hashes.device)
    _check(lib().dpk_partition_ids(_ptr(hashes), hashes.numel(), P, _ptr(thr), nthr, _ptr(out), _stream()))
    return out


# ---- a4: map side --------------------------------------------------------------
def partition_workspace(nbuckets, device):
    nbytes = lib().dpk_partition_workspace_bytes(0, nbuckets)
    return torch.empty(nbytes, dtype=torch.uint8, device=device)


K_UNORDERED = 0x100   # DPK_K_UNORDERED: rows of a bucket may come out in any order
K_PACKED = 0x200      # DPK_K_PACKED: rows are (key, value) records of one [n, 2] buffer instead of two columns


def packable(keys, vals, prehashed=False):
    """Whether (keys, vals) rows can travel as packed records: values as wide as the keys, hashed keys."""
    return vals is not None and not prehashed and keys.element_size() == vals.element_size()


def packed_views(rows, key_dtype, val_dtype):
    """The key and value columns of a packed [n, 2] row buffer, as strided views."""
    return rows[:, 0], (rows if val_dtype == rows.dtype else rows.view(val_dtype))[:, 1]


def packed_source(keys, vals):
    """The [n, 2] row buffer that keys and vals are the column views of (packed_views), or None."""
    if keys is None or vals is None or keys.dim() != 1 or vals.dim() != 1 or keys.numel() != vals.numel():
        return None
    es = keys.element_size()
    if (vals.element_size() != es or keys.stride() != (2,) or vals.stride() != (2,)
            or vals.data_ptr() != keys.data_ptr() + es or keys.untyped_storage().data_ptr() != vals.untyped_storage().data_ptr()):
        return None
    return keys.as_strided((keys.numel(), 2), (2, 1))


def packed_rows(n, key_dtype, device):
    """An [n, 2] buffer of packed rows (the record alignment is the allocator's)."""
    return torch.empty((n, 2), dtype=key_dtype, device=device)


def _kk(keys, prehashed, row_hash, unordered=False):
    kk = K_ROWID if row_hash is not None else key_kind(keys, prehashed)
    return kk | K_UNORDERED if (unordered and kk >= 0) else kk


def partition_count(keys, P, thresholds=None, prehashed=False, sub_bits=0, ws=None, row_hash=None, unordered=False):
    """Rows per bucket of one chunk; returns (counts[P << sub_bits] int64 device, ws)."""
    _need_cuda(keys, row_hash)
    F = P << sub_bits
    thr, nthr = _thr(thresholds, keys.device)
    if ws is None:
        ws = partition_workspace(F, keys.device)
    counts = torch.empty(F, dtype=torch.int64, device=keys.device)
    _check(lib().dpk_partition_count(_ptr(keys), _kk(keys, prehashed, row_hash, unordered), _ptr(row_hash), keys.numel(), P,
                                     _ptr(thr), nthr,
                                     sub_bits, _ptr(counts), _ptr(ws), ws.numel(), _stream()))
    return counts, ws


def partition_scatter(keys, vals, P, bucket_base, out_keys, out_vals, ws, thresholds=None, prehashed=False,
                      sub_bits=0, row_hash=None, unordered=False):
    """out_vals None with vals given: out_keys is a packed [n, 2] row buffer (packed_rows)."""
    _need_cuda(keys, vals, bucket_base, out_keys, out_vals, ws, row_hash)
    thr, nthr = _thr(thresholds, keys.device)
    vb = 0 if vals is None else vals.element_size()
    kk = _kk(keys, prehashed, row_hash, unordered)
    if vals is not None and out_vals is None:
        kk |= K_PACKED
    _check(lib().dpk_partition_scatter(_ptr(keys), kk, _ptr(row_hash), _ptr(vals), vb,
                                       keys.numel(), P,
                                       _ptr(thr), nthr, sub_bits, _ptr(bucket_base), _ptr(out_keys),
                                       _ptr(out_vals), _ptr(ws), ws.numel(), _stream()))


def partition_scatter_ptrs(keys, vals, P, key_ptrs, val_ptrs, ws, thresholds=None, prehashed=False, sub_bits=0,
                           row_hash=None, unordered=False):
    """Fused scatter + exchange: bucket b of this chunk is written through key_ptrs[b] / val_ptrs[b]
    (device int64 tensors holding absolute device addresses, possibly peer-GPU memory)."""
    _need_cuda(keys, vals, key_ptrs, val_ptrs, ws, row_hash)
    thr, nthr = _thr(thresholds, keys.device)
    vb = 0 if vals is None else vals.element_size()
    _check(lib().dpk_partition_scatter_ptrs(_ptr(keys), _kk(keys, prehashed, row_hash, unordered), _ptr(row_hash), _ptr(vals),
                                            vb, keys.numel(), P, _ptr(thr), nthr, sub_bits, _ptr(key_ptrs),
                                            _ptr(val_ptrs), _ptr(ws), ws.numel(), _stream()))


def copy_segments(src_ptrs, dst_ptrs, nbytes, sms=0):
    """One launch copying nbytes[s] bytes from device address src_ptrs[s] to dst_ptrs[s] (int64 device
    tensors; destinations may be peer-GPU memory): the exchange as block pushes over NVLink.
    sms > 0: the copy runs on that many whole SMs only (dpk_set_option "copy_sms") -- for a push that overlaps
    another kernel."""
    _need_cuda(src_ptrs, dst_ptrs, nbytes)
    if not (src_ptrs.numel() == dst_ptrs.numel() == nbytes.numel()):
        raise ValueError("segment table columns differ in length")
    if sms:
        set_option("copy_sms", int(sms))
    try:
        _check(lib().dpk_copy_segments(_ptr(src_ptrs), _ptr(dst_ptrs), _ptr(nbytes), nbytes.numel(), _stream()))
    finally:
        if sms:
            set_option("copy_sms", 0)


def memcpy_batch(dst_ptrs, src_ptrs, nbytes):
    """Block copies by the copy engines: one cudaMemcpyBatchAsync over HOST lists of device addresses and sizes."""
    n = len(nbytes)
    if not (len(dst_ptrs) == len(src_ptrs) == n):
        raise ValueError("segment table columns differ in length")
    if n == 0:
        return
    U, I = C.c_uint64 * n, C.c_int64 * n
    _check(lib().dpk_memcpy_batch(U(*dst_ptrs), U(*src_ptrs), I(*nbytes), n, _stream()))


def push_plan(all_counts, nranks, per_block, my_src, my_rank, keys, vals, dst_base, capacity, need_over, want_seg=True,
              part=None, dst_row0=0):
    """dpk_push_plan(_part): (src_ptrs, dst_ptrs, nbytes [ncols * nranks], seg [nsrc, own buckets] | None), one launch.
    keys / vals: my bucket-major columns (vals may be None); dst_base: device int64 [ncols * nranks] receive-buffer
    addresses (column-major).  part = (blk_lo, blk_hi): only those buckets of every destination's block, into the
    region of `capacity` rows starting at row dst_row0 of the receive buffers."""
    _need_cuda(all_counts, dst_base, need_over)
    nsrc, F = int(all_counts.shape[0]), int(all_counts.shape[1])
    ncols = 1 if vals is None else 2
    dev = all_counts.device
    lo, hi = (0, per_block) if part is None else part
    src = torch.empty(ncols * nranks, dtype=torch.int64, device=dev)
    dst = torch.empty(ncols * nranks, dtype=torch.int64, device=dev)
    nby = torch.empty(ncols * nranks, dtype=torch.int64, device=dev)
    b0, b1 = min(F, my_rank * per_block + lo), min(F, (my_rank + 1) * per_block, my_rank * per_block + hi)
    seg = torch.empty((nsrc, max(0, b1 - b0)), dtype=torch.int64, device=dev) if want_seg else None
    _check(lib().dpk_push_plan_part(_ptr(all_counts), nsrc, nranks, F, per_block, lo, hi, dst_row0, my_src, my_rank, ncols,
                                    C.c_uint64(keys.data_ptr()), C.c_uint64(0 if vals is None else vals.data_ptr()),
                                    _ptr(dst_base), keys.element_size(), 0 if vals is None else vals.element_size(),
                                    capacity, _ptr(src), _ptr(dst), _ptr(nby), _ptr(need_over), _ptr(seg), _stream()))
    return src, dst, nby, seg


def pipe_plan(all_counts, nranks, per_block, nparts, region_rows, my_src, my_rank, keys, vals, dst_base, need_over,
              want_seg=True):
    """dpk_pipe_plan: (bucket_base[F], src_ptrs, dst_ptrs, nbytes [nparts, ncols * nranks], seg [nparts, nsrc, per_block /
    nparts] | None) for one group of map splits; keys / vals: the group's SEND buffers (allocated with pipe_pad_rows()
    spare rows)."""
    _need_cuda(all_counts, dst_base, need_over, keys, vals)
    nsrc, F = int(all_counts.shape[0]), int(all_counts.shape[1])
    ncols = 1 if vals is None else 2
    dev = all_counts.device
    base = torch.empty(F, dtype=torch.int64, device=dev)
    src = torch.empty((nparts, ncols * nranks), dtype=torch.int64, device=dev)
    dst = torch.empty((nparts, ncols * nranks), dtype=torch.int64, device=dev)
    nby = torch.empty((nparts, ncols * nranks), dtype=torch.int64, device=dev)
    seg = torch.empty((nparts, nsrc, per_block // nparts), dtype=torch.int64, device=dev) if want_seg else None
    _check(lib().dpk_pipe_plan(_ptr(all_counts), nsrc, nranks, F, per_block, nparts, region_rows, my_src, my_rank, ncols,
                               C.c_uint64(keys.data_ptr()), C.c_uint64(0 if vals is None else vals.data_ptr()),
                               _ptr(dst_base), keys.element_size(), 0 if vals is None else vals.element_size(),
                               _ptr(base), _ptr(src), _ptr(dst), _ptr(nby), _ptr(need_over), _ptr(seg), _stream()))
    return base, src, dst, nby, seg


def pipe_pad_rows(nranks, nparts, key_bytes, val_bytes=None):
    """Spare rows a pipelined step's send buffer needs for the congruence pads (dpk_pipe_plan)."""
    return nranks * nparts * (16 // min(key_bytes, val_bytes or key_bytes))


def fused_plan(all_counts, nranks, per_block, my_rank, dst_base, key_bytes, val_bytes, capacity, dump_keys, dump_vals,
               need_over, want_seg=True):
    """dpk_fused_plan: (key_ptrs[F], val_ptrs[F] | None, seg [nranks, own buckets] | None), one launch: where every
    bucket of this rank's map output goes in its owner's receive buffer (see include/dpark_b200.h)."""
    _need_cuda(all_counts, dst_base, need_over, dump_keys, dump_vals)
    G, F = int(all_counts.shape[0]), int(all_counts.shape[1])
    if G != nranks:
        raise ValueError("all_counts has %d source rows for %d ranks" % (G, nranks))
    ncols = 1 if dump_vals is None else 2
    dev = all_counts.device
    kp = torch.empty(F, dtype=torch.int64, device=dev)
    vp_ = torch.empty(F, dtype=torch.int64, device=dev) if ncols == 2 else None
    b0, b1 = min(F, my_rank * per_block), min(F, (my_rank + 1) * per_block)
    seg = torch.empty((G, b1 - b0), dtype=torch.int64, device=dev) if want_seg else None
    _check(lib().dpk_fused_plan(_ptr(all_counts), nranks, F, per_block, my_rank, ncols, _ptr(dst_base), key_bytes,
                                val_bytes if ncols == 2 else 0, capacity, C.c_uint64(dump_keys.data_ptr()),
                                C.c_uint64(0 if dump_vals is None else dump_vals.data_ptr()), _ptr(kp), _ptr(vp_),
                                _ptr(need_over), _ptr(seg), _stream()))
    return kp, vp_, seg


def partition(keys, vals, P, thresholds=None, prehashed=False, sub_bits=0, row_hash=None, unordered=False,
              packed=False):
    """Stable hash-partition of one chunk (ShuffleMapTask._run, dpark/task.py:209-226).
    Returns (out_keys, out_vals, offsets[(P << sub_bits) + 1] int64 device); packed=True (packable rows):
    (rows[n, 2], None, offsets), the rows written as packed records."""
    _need_cuda(keys, vals, row_hash)
    if vals is not None and vals.numel() != keys.numel():
        from .errors import DparkUserFatalError
        raise DparkUserFatalError("ragged pair columns: %d keys, %d values" % (keys.numel(), vals.numel()))
    F = P << sub_bits
    thr, nthr = _thr(thresholds, keys.device)
    ws = partition_workspace(F, keys.device)
    kk = _kk(keys, prehashed, row_hash, unordered)
    if packed:
        if not packable(keys, vals, prehashed):
            raise TypeError("packed rows need hashed keys and values of the same width")
        out_keys, out_vals = packed_rows(keys.numel(), keys.dtype, keys.device), None
        kk |= K_PACKED
    else:
        out_keys = torch.empty_like(keys)
        out_vals = None if vals is None else torch.empty_like(vals)
    offsets = torch.empty(F + 1, dtype=torch.int64, device=keys.device)
    vb = 0 if vals is None else vals.element_size()
    _check(lib().dpk_partition(_ptr(keys), kk, _ptr(row_hash), _ptr(vals), vb,
                               keys.numel(), P,
                               _ptr(thr), nthr, sub_bits, _ptr(out_keys), _ptr(out_vals), _ptr(offsets),
                               _ptr(ws), ws.numel(), _stream()))
    return out_keys, out_vals, offsets


# ---- a9: reduce side -----------------------------------------------------------
def acc_dtype(vals_dtype):
    """Accumulator/output dtype of combine: ints -> int64, floats -> float64
    (the reference adds Python ints / Python floats)."""
    return torch.float64 if vals_dtype in (torch.float32, torch.float64) else torch.int64


def combine(keys, vals, op, P, seg_rows, part_first=0, nparts=None, thresholds=None, sub_bits=0,
            row_hash=None, rows=None):
    """Reduce-side merge (DiskHashMerger._merge, dpark/shuffle.py:600-608) of the
    rows of partitions [part_first, part_first+nparts).  Rows are laid out
    source-major, bucket-major inside; seg_rows: device int64 [nsrc, nparts <<
    sub_bits] rows of local fine bucket b from source s.  Returns (out_keys,
    out_vals, out_offsets[nparts+1], out_counts[nparts]); partition j's distinct
    keys are out[out_offsets[j] : out_offsets[j] + out_counts[j]].  With row_hash
    (the per-row portable_hash column) the keys are representative row ids from
    dict_encode (DPK_K_ROWID).  rows: the packed [n, 2] buffer keys and vals are the column views of (the kernels
    then read one record per row).  Column views of a packed buffer (MapOutput.keys / .vals) are recognised as such
    without it."""
    _need_cuda(seg_rows, row_hash, rows)
    if rows is None:
        rows = packed_source(keys, vals)
    if rows is None:
        _need_cuda(keys, vals)
    if nparts is None:
        nparts = P
    n = keys.numel()
    F = nparts << sub_bits
    if seg_rows.dim() == 1:
        seg_rows = seg_rows.unsqueeze(0)
    nsrc = int(seg_rows.shape[0])
    if seg_rows.shape[1] != F or seg_rows.dtype != torch.int64:
        raise ValueError("seg_rows must be int64[nsrc, %d]" % F)
    bucket_rows = seg_rows
    thr, nthr = _thr(thresholds, keys.device)
    ws_bytes = lib().dpk_combine_workspace_bytes(n, F, nsrc)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=keys.device)
    out_keys = torch.empty(n, dtype=keys.dtype, device=keys.device)
    out_vals = torch.empty(n, dtype=acc_dtype(vals.dtype), device=keys.device)
    out_offsets = torch.empty(nparts + 1, dtype=torch.int64, device=keys.device)
    out_counts = torch.empty(nparts, dtype=torch.int64, device=keys.device)
    kk = key_kind(keys) if row_hash is None else K_ROWID
    src_k, src_v = keys, vals
    if rows is not None:
        if rows.dim() != 2 or rows.shape[1] != 2 or rows.shape[0] != n or keys.element_size() != vals.element_size():
            raise ValueError("rows must be the packed [n, 2] buffer of the key and value columns")
        kk |= K_PACKED
        src_k, src_v = rows, None
    _check(lib().dpk_combine(_ptr(src_k), kk, _ptr(row_hash), _ptr(src_v), val_kind(vals), n, OPS[op], P,
                             _ptr(thr), nthr, sub_bits, part_first, nparts, nsrc, _ptr(bucket_rows), _ptr(out_keys),
                             _ptr(out_vals), _ptr(out_offsets), _ptr(out_counts), _ptr(ws), ws_bytes,
                             _stream()))
    return out_keys, out_vals, out_offsets, out_counts


# ---- variable-length keys ----------------------------------------------------------
def dict_encode(data, offsets, hashes):
    """Representative row id per row: rep[i] == rep[j] <=> the byte strings are equal."""
    _need_cuda(data, offsets, hashes)
    n = offsets.numel() - 1
    ws_bytes = lib().dpk_dict_encode_workspace_bytes(n)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=offsets.device)
    rep = torch.empty(n, dtype=torch.int64, device=offsets.device)
    _check(lib().dpk_dict_encode(_ptr(data), _ptr(offsets), _ptr(hashes), n, _ptr(rep), _ptr(ws), ws_bytes,
                                 _stream()))
    return rep


# ---- f4: device text ingest --------------------------------------------------------
def tokenize(data):
    """Tokens (str.split() without arguments) of an ASCII byte range on the device: (starts, lens, ascii) -- int64
    device tensors in text order; ascii False = the range holds a byte >= 0x80 and must be tokenised by Python
    (starts / lens are None then).  One host read (the token count sizes the outputs)."""
    _need_cuda(data)
    n = int(data.numel())
    dev = data.device
    if n == 0:
        z = torch.zeros(0, dtype=torch.int64, device=dev)
        return z, z.clone(), True
    nb = int(lib().dpk_tokenize_blocks(n))
    counts = torch.empty(nb + 1, dtype=torch.int64, device=dev)   # [nb] = the high-byte flag
    counts[nb] = 0
    _check(lib().dpk_tokenize_count(_ptr(data), n, _ptr(counts), C.c_void_p(counts.data_ptr() + 8 * nb), _stream()))
    incl = torch.cumsum(counts[:nb], 0)
    total, flag = int(incl[-1].item()), int(counts[nb].item())
    if flag & 1:
        return None, None, False
    base = (incl - counts[:nb]).contiguous()
    starts = torch.empty(total, dtype=torch.int64, device=dev)
    lens = torch.empty(total, dtype=torch.int64, device=dev)
    if total:
        _check(lib().dpk_tokenize_emit(_ptr(data), n, _ptr(base), _ptr(starts), _ptr(lens), _stream()))
    return starts, lens, True


def tokenize_utf8(data):
    """Tokens of a UTF-8 byte range on the device, as str.split() without arguments finds them in the decoded text
    (Unicode whitespace): (starts, lens, valid) -- int64 device tensors in text order, each token given by the
    (start, length) of its bytes; valid False = the range is not strict UTF-8, bytes.decode("utf-8") raises on it
    (starts / lens are None then).  One host read, as tokenize."""
    _need_cuda(data)
    n = int(data.numel())
    dev = data.device
    if n == 0:
        z = torch.zeros(0, dtype=torch.int64, device=dev)
        return z, z.clone(), True
    nb = int(lib().dpk_tokenize_blocks(n))
    counts = torch.empty(nb + 1, dtype=torch.int64, device=dev)   # [nb] = the ill-formed flag
    counts[nb] = 0
    _check(lib().dpk_tokenize_utf8_count(_ptr(data), n, _ptr(counts), C.c_void_p(counts.data_ptr() + 8 * nb),
                                         _stream()))
    incl = torch.cumsum(counts[:nb], 0)
    total, flag = int(incl[-1].item()), int(counts[nb].item())
    if flag & 1:
        return None, None, False
    base = (incl - counts[:nb]).contiguous()
    starts = torch.empty(total, dtype=torch.int64, device=dev)
    lens = torch.empty(total, dtype=torch.int64, device=dev)
    if total:
        _check(lib().dpk_tokenize_utf8_emit(_ptr(data), n, _ptr(base), _ptr(starts), _ptr(lens), _stream()))
    return starts, lens, True


def line_starts(data):
    """Every line start of a byte range on the device (byte 0 and each byte after a '\\n', inside the range; a final
    '\\n' opens no line): (starts int64 device tensor in text order, high) -- high True when the range holds a byte
    >= 0x80.  One host read (the line count sizes the output)."""
    _need_cuda(data)
    n = int(data.numel())
    dev = data.device
    if n == 0:
        return torch.zeros(0, dtype=torch.int64, device=dev), False
    nb = int(lib().dpk_tokenize_blocks(n))
    counts = torch.empty(nb + 1, dtype=torch.int64, device=dev)   # [nb] = the high-byte flag
    counts[nb] = 0
    _check(lib().dpk_textcols_count(_ptr(data), n, _ptr(counts), C.c_void_p(counts.data_ptr() + 8 * nb), _stream()))
    incl = torch.cumsum(counts, 0)
    total, flag = int(incl[nb - 1].item()), int(counts[nb].item())
    base = (incl[:nb] - counts[:nb]).contiguous()
    starts = torch.empty(total, dtype=torch.int64, device=dev)
    _check(lib().dpk_textcols_emit(_ptr(data), n, _ptr(base), _ptr(starts), _stream()))
    return starts, bool(flag & 1)


def utf8_valid(data):
    """Is the device byte range strict UTF-8 (what bytes.decode("utf-8") accepts)?  dpk_tokenize_utf8_count's flag."""
    _need_cuda(data)
    n = int(data.numel())
    if n == 0:
        return True
    nb = int(lib().dpk_tokenize_blocks(n))
    counts = torch.zeros(nb + 1, dtype=torch.int64, device=data.device)
    _check(lib().dpk_tokenize_utf8_count(_ptr(data), n, _ptr(counts), C.c_void_p(counts.data_ptr() + 8 * nb),
                                         _stream()))
    return not (int(counts[nb].item()) & 1)


def textcols_parse(data, starts, sep, key, value, key_float, value_float, out_keys=None, out_vals=None, host=None):
    """Fields `key` and `value` of every line of the device byte range (starts from line_starts), parsed as int() or
    float() (dpk_textcols_parse): (keys int64, vals int64, host uint8) device tensors -- float columns hold the float64
    bits -- with host[i] = 1 where Python must parse line i.  sep: None (str.split()) or the separator's UTF-8 bytes as
    a uint8 device tensor."""
    _need_cuda(data, starts, sep)
    m = int(starts.numel())
    dev = data.device
    out_keys = torch.empty(m, dtype=torch.int64, device=dev) if out_keys is None else out_keys
    out_vals = torch.empty(m, dtype=torch.int64, device=dev) if out_vals is None else out_vals
    host = torch.empty(m, dtype=torch.uint8, device=dev) if host is None else host
    kinds = (K_F64 if key_float else K_I64, K_F64 if value_float else K_I64)
    _check(lib().dpk_textcols_parse(_ptr(data), int(data.numel()), _ptr(starts), m, _ptr(sep),
                                    0 if sep is None else int(sep.numel()), key, value, kinds[0], kinds[1],
                                    _ptr(out_keys), _ptr(out_vals), _ptr(host), _stream()))
    return out_keys, out_vals, host


def gather_bytes(data, starts, lens, idx=None):
    """Selected rows made contiguous: (bytes uint8, offsets int64 [m + 1]) with row i = data[starts[r] : starts[r] +
    lens[r]], r = idx[i] (idx None: every row)."""
    _need_cuda(data, starts, lens, idx)
    sel = lens if idx is None else lens[idx]
    m = int(sel.numel())
    off = torch.zeros(m + 1, dtype=torch.int64, device=data.device)
    if m:
        torch.cumsum(sel, 0, out=off[1:])
    out = torch.empty(int(off[-1].item()) if m else 0, dtype=torch.uint8, device=data.device)
    if m and out.numel():
        _check(lib().dpk_gather_bytes(_ptr(data), _ptr(starts), _ptr(lens), _ptr(idx), m, _ptr(off), _ptr(out), _stream()))
    return out, off


# ---- a10: groupByKey reduce side ---------------------------------------------------
def key_or(keys):
    """Device uint64 (as int64 tensor[1]): OR over i of keys[i] ^ keys[0]."""
    _need_cuda(keys)
    out = torch.empty(1, dtype=torch.int64, device=keys.device)
    _check(lib().dpk_key_or(_ptr(keys), keys.numel(), _ptr(out), _stream()))
    return out


def gather_i64(src, idx):
    _need_cuda(src, idx)
    out = torch.empty(idx.numel(), dtype=torch.int64, device=idx.device)
    _check(lib().dpk_gather_i64(_ptr(src), _ptr(idx), idx.numel(), _ptr(out), _stream()))
    return out


def radix_pass(keys, vals, shift, bits, out_keys=None, out_vals=None, ws=None):
    """One stable LSD radix pass over int64 key bits (the multisplit with digit buckets)."""
    _need_cuda(keys, vals)
    if keys.dtype != torch.int64:
        raise TypeError("radix_pass sorts int64 key bits")
    if out_keys is None:
        out_keys = torch.empty_like(keys)
    if out_vals is None and vals is not None:
        out_vals = torch.empty_like(vals)
    if ws is None:
        ws = partition_workspace(1 << bits, keys.device)
    vb = 0 if vals is None else vals.element_size()
    _check(lib().dpk_radix_pass(_ptr(keys), _ptr(vals), vb, keys.numel(), shift, bits, _ptr(out_keys),
                                _ptr(out_vals), _ptr(ws), ws.numel(), _stream()))
    return out_keys, out_vals


def radix_pass_seg(keys, vals, shift, bits, seg_rows, out_keys=None, out_vals=None):
    """One stable radix pass inside every first-level bucket (dpk_radix_pass_seg).  seg_rows: device int64
    [nsrc, nbuckets].  Returns (out_keys, out_vals)."""
    _need_cuda(keys, vals, seg_rows)
    if keys.dtype != torch.int64:
        raise TypeError("radix_pass_seg sorts int64 key bits")
    nsrc, F = int(seg_rows.shape[0]), int(seg_rows.shape[1])
    n = keys.numel()
    if out_keys is None:
        out_keys = torch.empty_like(keys)
    if out_vals is None and vals is not None:
        out_vals = torch.empty_like(vals)
    ws_bytes = lib().dpk_radix_pass_seg_workspace_bytes(n, F, nsrc, bits)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=keys.device)
    fine = torch.empty((F << bits) + 1, dtype=torch.int64, device=keys.device)
    vb = 0 if vals is None else vals.element_size()
    _check(lib().dpk_radix_pass_seg(_ptr(keys), _ptr(vals), vb, n, shift, bits, F, nsrc, _ptr(seg_rows.contiguous()),
                                    _ptr(out_keys), _ptr(out_vals), _ptr(fine), _ptr(ws), ws_bytes, _stream()))
    return out_keys, out_vals


def group_heads(sorted_keys):
    """CSR heads of a key-sorted column: (group_keys[n], starts[n+1], ngroups[1]) device tensors;
    only the first ngroups (+1) entries are meaningful."""
    _need_cuda(sorted_keys)
    n = sorted_keys.numel()
    ws_bytes = lib().dpk_group_heads_workspace_bytes(n)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=sorted_keys.device)
    out_keys = torch.empty(n, dtype=torch.int64, device=sorted_keys.device)
    out_starts = torch.empty(n + 1, dtype=torch.int64, device=sorted_keys.device)
    ng = torch.empty(1, dtype=torch.int64, device=sorted_keys.device)
    _check(lib().dpk_group_heads(_ptr(sorted_keys), n, _ptr(out_keys), _ptr(out_starts), _ptr(ng), _ptr(ws),
                                 ws_bytes, _stream()))
    return out_keys, out_starts, ng


# ---- f1: join expansion -----------------------------------------------------------
def join_count(ids, group_starts, G, nL, keep_left, keep_right):
    """Per group of the tagged union's CSR: (nl[G], out_count[G]) int64 device tensors (dpk_join_count)."""
    _need_cuda(ids, group_starts)
    nl = torch.empty(G, dtype=torch.int64, device=ids.device)
    cnt = torch.empty(G, dtype=torch.int64, device=ids.device)
    _check(lib().dpk_join_count(_ptr(ids), _ptr(group_starts), G, nL, int(keep_left), int(keep_right), _ptr(nl),
                                _ptr(cnt), _stream()))
    return nl, cnt


def join_emit(group_keys, group_starts, ids, nl, out_off, nL, lvals, rvals, keep_left, keep_right, n_out):
    """The joined rows (dpk_join_emit): (keys int64, left, right, left_valid uint8 | None, right_valid uint8 | None);
    values keep their dtypes, a valid column exists only for a side the join kind can miss."""
    _need_cuda(group_keys, group_starts, ids, nl, out_off, lvals, rvals)
    dev = ids.device
    keys = torch.empty(n_out, dtype=torch.int64, device=dev)
    left = torch.empty(n_out, dtype=lvals.dtype, device=dev)
    right = torch.empty(n_out, dtype=rvals.dtype, device=dev)
    lvalid = torch.empty(n_out, dtype=torch.uint8, device=dev) if keep_right else None
    rvalid = torch.empty(n_out, dtype=torch.uint8, device=dev) if keep_left else None
    _check(lib().dpk_join_emit(_ptr(group_keys), _ptr(group_starts), _ptr(ids), _ptr(nl), _ptr(out_off),
                               int(nl.numel()), nL, _ptr(lvals), lvals.element_size(), _ptr(rvals), rvals.element_size(),
                               int(keep_left), int(keep_right), n_out, _ptr(keys), _ptr(left), _ptr(right),
                               _ptr(lvalid), _ptr(rvalid), _stream()))
    return keys, left, right, lvalid, rvalid


def cogroup_count(ids, group_starts, G, bounds):
    """Per input t and group g of the cogroup's CSR (input t owns the ids [bounds[t], bounds[t + 1])): (first, count),
    int64 device tensors [N, G] -- where input t's sub-run of group g starts in ids, and its length (dpk_cogroup_count)."""
    _need_cuda(ids, group_starts, bounds)
    N = int(bounds.numel()) - 1
    first = torch.empty((N, G), dtype=torch.int64, device=ids.device)
    cnt = torch.empty((N, G), dtype=torch.int64, device=ids.device)
    _check(lib().dpk_cogroup_count(_ptr(ids), _ptr(group_starts), G, _ptr(bounds), N, _ptr(first), _ptr(cnt),
                                   _stream()))
    return first, cnt


def cogroup_emit(ids, first, out_off, id_base, vals, n_out):
    """One input's values, per group in its sub-run order (dpk_cogroup_emit): first[G] and out_off[G + 1] are that
    input's rows of cogroup_count's first and of the exclusive scan of its counts; the values keep their dtype."""
    _need_cuda(ids, first, out_off, vals)
    out = torch.empty(n_out, dtype=vals.dtype, device=ids.device)
    _check(lib().dpk_cogroup_emit(_ptr(ids), _ptr(first), _ptr(out_off), int(first.numel()), id_base, _ptr(vals),
                                  vals.element_size(), n_out, _ptr(out), _stream()))
    return out


# ---- f4: topByKey selection ----------------------------------------------------------
TOPK_TILE = 4096      # DPK_TOPK_TILE: candidates per chunk of a round
TOPK_MAX_N = 512      # DPK_TOPK_MAX_N: the largest top_n the rounds take


def topk_lengths(run_starts, top_n):
    """Per run of candidates (run_starts[G + 1]): its length after one round (dpk_topk_lengths), int64 device [G]."""
    _need_cuda(run_starts)
    G = int(run_starts.numel()) - 1
    out = torch.empty(G, dtype=torch.int64, device=run_starts.device)
    _check(lib().dpk_topk_lengths(_ptr(run_starts), G, top_n, _ptr(out), _stream()))
    return out


def topk_round(ids, vals, run_starts, n, out_starts, top_n, reverse):
    """One selection round (dpk_topk_round): candidate i is vals[ids[i]] (ids None: vals[i]) for i < n; out_starts
    [G + 1] is the exclusive scan of topk_lengths.  Returns the next round's candidates in vals' dtype."""
    _need_cuda(ids, vals, run_starts, out_starts)
    out = torch.empty(int(out_starts[-1].item()) if n else 0, dtype=vals.dtype, device=vals.device)
    _check(lib().dpk_topk_round(_ptr(ids), _ptr(vals), vals.element_size(), int(vals.dtype.is_floating_point),
                                _ptr(run_starts), int(run_starts.numel()) - 1, n, _ptr(out_starts), top_n,
                                int(reverse), _ptr(out), _stream()))
    return out


# ---- f5: innerJoin hash table ----------------------------------------------------------
def bcast_slots(G):
    """Slots of the innerJoin table of G keys: the least power of two >= max(2, 2 G) (bcast_slots, dpk_common.cuh)."""
    s = 2
    while s < 2 * G:
        s <<= 1
    return s


def bcast_build(group_keys):
    """The hash table of the distinct normalised keys group_keys[G] (int64 bits): a uint8 device tensor of
    bcast_slots(G) 16-byte slots (dpk_bcast_build)."""
    _need_cuda(group_keys)
    G = int(group_keys.numel())
    S = bcast_slots(G)
    table = torch.full((S * 16,), 0xFF, dtype=torch.uint8, device=group_keys.device)
    _check(lib().dpk_bcast_build(_ptr(group_keys), G, _ptr(table), S, _stream()))
    return table


def bcast_probe(table, keys, group_starts):
    """Every key of the column `keys` (int32 / int64 / float32 / float64, read in place) looked up in bcast_build's
    table: (grp int32, count int64) device tensors -- its group or -1, and group_starts[g + 1] - group_starts[g] or 0
    (dpk_bcast_probe)."""
    _need_cuda(table, keys, group_starts)
    n = int(keys.numel())
    grp = torch.empty(n, dtype=torch.int32, device=keys.device)
    cnt = torch.empty(n, dtype=torch.int64, device=keys.device)
    _check(lib().dpk_bcast_probe(_ptr(keys), _KEY_KIND.get(keys.dtype, -1), n, _ptr(table), int(table.numel()) // 16,
                                 _ptr(group_starts), _ptr(grp), _ptr(cnt), _stream()))
    return grp, cnt


def bcast_emit(keys, lvals, grp, out_off, group_starts, ids, rvals, n_out):
    """The innerJoin rows (dpk_bcast_emit): (keys, left, right) in the dtypes of keys, lvals and rvals; out_off[n + 1]
    is the exclusive scan of bcast_probe's counts."""
    _need_cuda(keys, lvals, grp, out_off, group_starts, ids, rvals)
    dev = keys.device
    ok = torch.empty(n_out, dtype=keys.dtype, device=dev)
    left = torch.empty(n_out, dtype=lvals.dtype, device=dev)
    right = torch.empty(n_out, dtype=rvals.dtype, device=dev)
    _check(lib().dpk_bcast_emit(_ptr(keys), keys.element_size(), _ptr(lvals), lvals.element_size(), _ptr(grp),
                                _ptr(out_off), int(keys.numel()), _ptr(group_starts), _ptr(ids), _ptr(rvals),
                                rvals.element_size(), n_out, _ptr(ok), _ptr(left), _ptr(right), _stream()))
    return ok, left, right


# ---- f6: sort ------------------------------------------------------------------------
def sort_keys(col0, col1, reverse):
    """The order words of one or two order columns (dpk_sort_keys): (w0, w1 | None, ids, nan_flag) int64 / int32 device
    tensors; w0[i] / w1[i] are row i's words, ids = 0..n-1, nan_flag[0] = 1 when an order column holds a NaN."""
    _need_cuda(col0, col1)
    n, dev = int(col0.numel()), col0.device
    w0 = torch.empty(n, dtype=torch.int64, device=dev)
    w1 = torch.empty(n, dtype=torch.int64, device=dev) if col1 is not None else None
    ids = torch.empty(n, dtype=torch.int64, device=dev)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    _check(lib().dpk_sort_keys(_ptr(col0), _KEY_KIND.get(col0.dtype, -1), _ptr(col1),
                               -1 if col1 is None else _KEY_KIND.get(col1.dtype, -1), n, int(reverse), _ptr(w0), _ptr(w1),
                               _ptr(ids), _ptr(flag), _stream()))
    return w0, w1, ids, flag


def sort_cuts(sorted_w0, ids, vals, bounds0, dtype0, bounds1, reverse):
    """The partition starts of the sorted rows (dpk_sort_cuts): int64 device [nbounds + 2], 0 first and n last.  bounds0 /
    bounds1: int64 device tensors of the bounds' widened bits (RangePartitioner.keys order), dtype0 the type of the first
    order column; bounds1 (None unless the order is (k, v)) pairs with the value column vals."""
    _need_cuda(sorted_w0, ids, vals, bounds0, bounds1)
    nb = int(bounds0.numel())
    out = torch.empty(nb + 2, dtype=torch.int64, device=sorted_w0.device)
    _check(lib().dpk_sort_cuts(_ptr(sorted_w0), _ptr(ids), _ptr(vals), _KEY_KIND.get(vals.dtype, -1),
                               int(sorted_w0.numel()), _ptr(bounds0), _KEY_KIND.get(dtype0, -1), _ptr(bounds1), nb,
                               int(reverse), _ptr(out), _stream()))
    return out


def sort_gather(keys, vals, ids):
    """keys[ids], vals[ids] in their own dtypes, bits preserved (dpk_sort_gather)."""
    _need_cuda(keys, vals, ids)
    ok, ov = torch.empty_like(keys), torch.empty_like(vals)
    _check(lib().dpk_sort_gather(_ptr(keys), keys.element_size(), _ptr(vals), vals.element_size(), _ptr(ids),
                                 int(ids.numel()), _ptr(ok), _ptr(ov), _stream()))
    return ok, ov


# ---- f7: percentilesByKey digests ---------------------------------------------------------
TD_CAP = 209          # TD_CAP: the add path folds when buffered values + centroids reach it; a digest's most centroids


def tdigest_heads(ids, group_starts, per):
    """uint8 device [n]: 1 at every row of the group-by's ids that starts a (key, split) segment, split = id // per
    (dpk_tdigest_heads)."""
    _need_cuda(ids, group_starts)
    n = int(ids.numel())
    head = torch.zeros(n, dtype=torch.uint8, device=ids.device)
    _check(lib().dpk_tdigest_heads(_ptr(ids), n, _ptr(group_starts), int(group_starts.numel()) - 1, per, _ptr(head),
                                   _stream()))
    return head


def tdigest_build(ids, vals, seg_starts, seg_off, flag):
    """Every segment's t-digest (dpk_tdigest_build): (means, weights, counts, lohi) device tensors -- segment s holds
    counts[s] centroids at means / weights[seg_off[s]:], lohi[2 s : 2 s + 2] its extreme means.  Sets flag[0] when the
    composition must stand."""
    _need_cuda(ids, vals, seg_starts, seg_off, flag)
    S, dev = int(seg_starts.numel()) - 1, ids.device
    cm = torch.empty(int(ids.numel()), dtype=torch.float64, device=dev)
    cw = torch.empty_like(cm)
    cnt = torch.empty(S, dtype=torch.int32, device=dev)
    lohi = torch.empty(2 * S, dtype=torch.float64, device=dev)
    work = torch.empty(S + 2, dtype=torch.int64, device=dev)
    _check(lib().dpk_tdigest_build(_ptr(ids), _ptr(vals), _KEY_KIND.get(vals.dtype, -1), _ptr(seg_starts),
                                   _ptr(seg_off), S, _ptr(cm), _ptr(cw), _ptr(cnt), _ptr(lohi), _ptr(work), _ptr(flag),
                                   _stream()))
    return cm, cw, cnt, lohi


def tdigest_merge(group_starts, seg_starts, seg_off, digests, qs, flag):
    """quantile(q) of every key's merged digest for every q of the float64 device tensor qs (dpk_tdigest_merge):
    float64 device [G, len(qs)].  digests: tdigest_build's result.  Sets flag[0] when the composition must stand."""
    cm, cw, cnt, lohi = digests
    _need_cuda(group_starts, seg_starts, seg_off, cm, cw, cnt, lohi, qs, flag)
    G, nq = int(group_starts.numel()) - 1, int(qs.numel())
    out = torch.empty((G, nq), dtype=torch.float64, device=group_starts.device)
    _check(lib().dpk_tdigest_merge(_ptr(group_starts), G, _ptr(seg_starts), _ptr(seg_off), int(seg_starts.numel()) - 1,
                                   _ptr(cnt), _ptr(lohi), _ptr(cm), _ptr(cw), _ptr(qs), nq, _ptr(out), _ptr(flag),
                                   _stream()))
    return out


# ---- f8: Bernoulli sample ------------------------------------------------------------------
MT_N = 624            # MT19937's state words


def sample_bernoulli(states, ranges, frac, nrows):
    """SampleRDD's keep rule on the device (dpk_sample_bernoulli): states int32 [S, 624] (the words' bits), ranges
    int64 [S, 2] (row begin, end) -> (ids, counts): int64 device [nrows] holding split i's kept row ids in row order
    from ranges[i, 0] on, and int64 device [S] their numbers."""
    _need_cuda(states, ranges)
    S = int(ranges.shape[0])
    if states.dtype != torch.int32:
        raise TypeError("MT19937 states must be int32 tensors holding the words' bits")
    if tuple(states.shape) != (S, MT_N) or tuple(ranges.shape) != (S, 2) or ranges.dtype != torch.int64:
        raise ValueError("states [S, 624] and ranges [S, 2] int64 expected")
    ids = torch.empty(max(1, nrows), dtype=torch.int64, device=ranges.device)
    counts = torch.zeros(S, dtype=torch.int64, device=ranges.device)
    _check(lib().dpk_sample_bernoulli(_ptr(states), _ptr(ranges), S, float(frac), _ptr(ids), _ptr(counts), _stream()))
    return ids, counts


def gather_columns(keys, vals, ids):
    """keys[ids], vals[ids] in their own dtypes, bits preserved, len(ids) rows (dpk_sort_gather)."""
    _need_cuda(keys, vals, ids)
    n = int(ids.numel())
    ok = torch.empty(n, dtype=keys.dtype, device=keys.device)
    ov = torch.empty(n, dtype=vals.dtype, device=vals.device)
    _check(lib().dpk_sort_gather(_ptr(keys), keys.element_size(), _ptr(vals), vals.element_size(), _ptr(ids), n,
                                 _ptr(ok), _ptr(ov), _stream()))
    return ok, ov


# ---- f9: top / hot select and the uniq table ------------------------------------------------------------------------
SEL_SHIFT0 = 56       # 64 - SEL_BITS: the first digit of a word
SEL_BUCKETS = 256


def select_state(n, m):
    """The select's device state and histogram before the first round (dpk_select_round): rank n among m rows."""
    st = torch.zeros(16, dtype=torch.int64)
    st[1], st[2], st[4] = SEL_SHIFT0, n, m
    hist = torch.zeros(3 * SEL_BUCKETS, dtype=torch.int64)
    hist[2 * SEL_BUCKETS:] = -1
    return st, hist


def select_round(w0, w1, cands, m, state, hist):
    """One MSD radix round of the select over m candidates (cands None: rows 0 .. m-1); updates state (dpk_select_round)."""
    _need_cuda(w0, w1, cands, state, hist)
    _check(lib().dpk_select_round(_ptr(w0), _ptr(w1), _ptr(cands), m, _ptr(state), _ptr(hist), _stream()))


def select_compact(w0, w1, cands, m, state, count):
    """The `count` candidates of the bucket the last round chose, int64 device (dpk_select_compact)."""
    _need_cuda(w0, w1, cands, state)
    out = torch.empty(count, dtype=torch.int64, device=w0.device)
    _check(lib().dpk_select_compact(_ptr(w0), _ptr(w1), _ptr(cands), m, _ptr(state), _ptr(out), _stream()))
    return out


def select_take(w0, w1, take, state):
    """The `take` smallest rows by (w0[, w1], id) once the rounds are done, in row id order (dpk_select_take)."""
    _need_cuda(w0, w1, state)
    n, dev = int(w0.numel()), w0.device
    tiles = int(lib().dpk_select_tiles(n))
    lt = torch.empty(tiles, dtype=torch.int64, device=dev)
    eq = torch.empty(tiles, dtype=torch.int64, device=dev)
    out = torch.empty(take, dtype=torch.int64, device=dev)
    _check(lib().dpk_select_take(_ptr(w0), _ptr(w1), n, take, _ptr(state), _ptr(lt), _ptr(eq), _ptr(out), _stream()))
    return out


def uniq_insert(keys, vals):
    """The distinct-count table of the rows' (k, v) pairs (dpk_uniq_insert): (table, state) -- bcast_slots(n) int64
    slots and int64 [2] whose [0] is 1 when a NaN occurred."""
    _need_cuda(keys, vals)
    n, dev = int(keys.numel()), keys.device
    S = bcast_slots(n)
    table = torch.full((S,), 0x7FFFFFFF, dtype=torch.int64, device=dev)
    state = torch.zeros(2, dtype=torch.int64, device=dev)
    _check(lib().dpk_uniq_insert(_ptr(keys), _KEY_KIND.get(keys.dtype, -1), _ptr(vals), _KEY_KIND.get(vals.dtype, -1), n,
                                 _ptr(table), S, _ptr(state), _stream()))
    return table, state


def uniq_emit(table, state, n):
    """(first, count): int64 device [n] whose first state[1] entries are every distinct pair's first row id and row
    count, in slot order (dpk_uniq_emit)."""
    _need_cuda(table, state)
    first = torch.empty(max(1, n), dtype=torch.int64, device=table.device)
    count = torch.empty(max(1, n), dtype=torch.int64, device=table.device)
    _check(lib().dpk_uniq_emit(_ptr(table), int(table.numel()), _ptr(first), _ptr(count), _ptr(state), _stream()))
    return first, count


def set_option(name, value):
    _check(lib().dpk_set_option(name.encode(), int(value)))


# ---- measurement hooks ---------------------------------------------------------
def launch_count():
    """Kernels launched by the library since load (exact, counted in C)."""
    return int(lib().dpk_launch_count())


def prof_enable(on=True):
    _check(lib().dpk_prof_enable(1 if on else 0))


def prof_collect():
    """[(kernel label, device ms)] for every launch since prof_enable(True)."""
    L = lib()
    out = []
    name = C.create_string_buffer(64)
    ms = C.c_float()
    for i in range(L.dpk_prof_count()):
        _check(L.dpk_prof_get(i, name, C.byref(ms)))
        out.append((name.value.decode(), float(ms.value)))
    return out
