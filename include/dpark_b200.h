/*
 * dpark_b200.h -- C ABI of the H100-native DPark shuffle hot path.
 *
 * The reference (douban/dpark) has NO FFI on this path: the boundary is
 * Python-level (SURVEY.md §8b).  This header is therefore the net-new plugin
 * ABI a maintainer would bind from dpark/task.py and dpark/shuffle.py (see
 * INTEGRATION.md for the ctypes stub).  Every entry point names the reference
 * code it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes; no torch / C++ types.
 *   - every pointer is a DEVICE pointer into caller-owned memory unless the
 *     parameter name starts with `h_`.
 *   - every call takes a cudaStream_t (as void*), is stream-ordered, never
 *     allocates device memory and never synchronises unless stated.
 *   - returns 0 on success, <0 on error (DPK_ERR_*); dpk_last_error() gives a
 *     thread-local message.
 *   - sizes: a single call handles n < 2^31 rows; callers chunk above that.
 */
#ifndef DPARK_B200_H
#define DPARK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DPK_ABI_VERSION 1

typedef void *dpk_stream_t; /* cudaStream_t */

enum {
    DPK_OK = 0,
    DPK_ERR_INVALID = -1,     /* bad argument (NULL pointer, n<0, P<1 ...)            */
    DPK_ERR_UNSUPPORTED = -2, /* unsupported dtype/op/size -> Python TypeError        */
    DPK_ERR_WORKSPACE = -3,   /* workspace too small                                  */
    DPK_ERR_CUDA = -4         /* CUDA runtime error (message in dpk_last_error)       */
};

/* key column kinds.  The hash of each follows dpark/portable_hash.pyx:51-70:
 * ints and floats -> Python's builtin hash(); see dpk_hash_keys. */
enum { DPK_K_I64 = 0, DPK_K_I32 = 1, DPK_K_F64 = 2, DPK_K_U64 = 3, DPK_K_F32 = 4,
       DPK_K_ROWID = 5 /* int64 ids of representative rows; their hash is looked up in key_aux */ };
/* OR-able into key_kind of the dpk_partition* calls (not with -1): the caller does not need the rows
 * of a bucket in input order (reduceByKey merges them anyway; groupByKey does need the order), which
 * lets the multisplit rank rows with one native shared-memory atomic instead of a warp match. */
#define DPK_K_UNORDERED 0x100
/* OR-able into key_kind (not with -1) of dpk_partition / dpk_partition_scatter (values as wide as the keys; not
 * dpk_partition_scatter_ptrs) and of dpk_combine: rows are PACKED records -- key then value, 16 bytes for 8-byte columns, 8 bytes for 4-byte
 * ones -- instead of two columns.  dpk_partition*: the output is packed; out_keys receives the records (aligned to the
 * record size), out_vals is ignored.  dpk_combine: the input is packed; keys points at the records, vals must be
 * NULL and val_kind still names the value type.  Fewer, longer bucket runs in the multisplits and one load per row. */
#define DPK_K_PACKED 0x200
/* value column kinds */
enum { DPK_V_I64 = 0, DPK_V_F64 = 1, DPK_V_I32 = 2, DPK_V_F32 = 3 };
/* combiner ops a reduceByKey(func) lowers to (dpark/rdd.py:543-545 builds
 * Aggregator(identity, func, func); dpark/dependency.py:121-161) */
enum { DPK_OP_SUM = 0, DPK_OP_MIN = 1, DPK_OP_MAX = 2, DPK_OP_PROD = 3,
       DPK_OP_AND = 4, DPK_OP_OR = 5, DPK_OP_XOR = 6 };
/* byte-string key modes for dpk_hash_bytes */
enum { DPK_BYTES_SIGNED = 0,   /* bytes keys: string_hash over signed chars, portable_hash.pyx:17-32 */
       DPK_STR_UTF8 = 1 };     /* str keys stored as UTF-8: unicode_hash over code points, :34-48   */

int dpk_abi_version(void);
const char *dpk_last_error(void);
/* h_info: int32[4] = {sm_count, cc_major, cc_minor, l2_bytes>>20} of the current device */
int dpk_device_info(int32_t *h_info);

/* ---- a1: portable_hash (dpark/portable_hash.pyx:51-70) ------------------- */
/* out_hash[i] = portable_hash(keys[i]); ints: sign(x)*(|x| mod 2^61-1), -1 -> -2;
 * floats: CPython _Py_HashDouble. */
int dpk_hash_keys(const void *keys, int key_kind, int64_t n, int64_t *out_hash,
                  dpk_stream_t stream);
/* variable-length keys: data[offsets[i] .. offsets[i+1]) */
int dpk_hash_bytes(const uint8_t *data, const int64_t *offsets, int64_t n, int mode,
                   int64_t *out_hash, dpk_stream_t stream);

/* ---- a2: HashPartitioner.getPartition (dpark/dependency.py:229-233) ------ */
/* tuple keys (dpark/portable_hash.pyx:3-15, tuple_hash): the hash of row i's tuple from the portable_hash values of
 * its `arity` items, item_hash[a * n + i] (item-major; computed with dpk_hash_keys / dpk_hash_bytes / this function
 * for nested tuples, a constant column 1315925605 for None items, portable_hash.pyx:53-54). */
int dpk_hash_tuple(const int64_t *item_hash, int64_t n, int32_t arity, int64_t *out_hash, dpk_stream_t stream);
/* out_pid[i] = hash[i] floor-mod P, or bisect_right(thresholds, hash[i]) when
 * thresholds != NULL (nthr = P-1 ascending int64 on device). */
int dpk_partition_ids(const int64_t *hash, int64_t n, int32_t P, const int64_t *thresholds,
                      int32_t nthr, int32_t *out_pid, dpk_stream_t stream);

/* ---- a4: map side, ShuffleMapTask._run hash-partition (dpark/task.py:209-226)
 * Stable multisplit of one input chunk into buckets: rows keep their input
 * order inside each bucket (this is what makes ordered groupByKey exact).
 *
 * Buckets: F = P << sub_bits.  Bucket id = partition * 2^sub_bits + sub, where
 * partition = getPartition(key) exactly as the reference and sub is taken from
 * other bits of the key's hash.  sub_bits = 0 gives the reference's P buckets;
 * sub_bits > 0 only refines the layout INSIDE each partition (partition p is the
 * concatenation of its 2^sub_bits sub-buckets) so the reduce-side tables stay
 * L2-resident.  F <= DPK_MAX_PARTITIONS.
 *
 * key_kind = DPK_K_* hashes the key column with portable_hash; key_kind = -1
 * ("prehashed") takes the int64 keys AS the hash; key_kind = DPK_K_ROWID takes
 * int64 row ids (representatives of variable-length keys, dpk_dict_encode) and
 * looks their hash up in key_aux (the column dpk_hash_bytes produced).  key_aux
 * is NULL for every other kind.
 *
 *   ws = dpk_partition_workspace_bytes(n, F)
 *   dpk_partition_count  : out_counts[F] (int64) = rows per bucket of this chunk;
 *                          leaves per-CTA counts in ws for the scatter.
 *   dpk_partition_scatter: writes row i to out_keys/out_vals[bucket_base[b] + rank],
 *                          bucket_base[F] int64 on device (caller-computed from the
 *                          counts of all chunks, so several chunks interleave into
 *                          one bucket-major buffer = the alltoallv send buffer).
 *                          Must follow dpk_partition_count with the same
 *                          (keys, n, P, thresholds, sub_bits, ws).
 *   dpk_partition        : count + exclusive scan + scatter for a single chunk;
 *                          out_offsets[F+1] int64.
 * key width follows key_kind; val_bytes in {0, 4, 8} (0/NULL = keys only).
 */
#define DPK_MAX_PARTITIONS 4096
int64_t dpk_partition_workspace_bytes(int64_t n, int32_t nbuckets);
int dpk_partition_count(const void *keys, int key_kind, const int64_t *key_aux, int64_t n, int32_t P,
                        const int64_t *thresholds, int32_t nthr, int32_t sub_bits,
                        int64_t *out_counts, void *ws, int64_t ws_bytes, dpk_stream_t stream);
int dpk_partition_scatter(const void *keys, int key_kind, const int64_t *key_aux, const void *vals,
                          int32_t val_bytes, int64_t n, int32_t P, const int64_t *thresholds,
                          int32_t nthr, int32_t sub_bits, const int64_t *bucket_base,
                          void *out_keys, void *out_vals, void *ws, int64_t ws_bytes,
                          dpk_stream_t stream);
int dpk_partition(const void *keys, int key_kind, const int64_t *key_aux, const void *vals,
                  int32_t val_bytes, int64_t n, int32_t P, const int64_t *thresholds, int32_t nthr,
                  int32_t sub_bits, void *out_keys, void *out_vals, int64_t *out_offsets, void *ws,
                  int64_t ws_bytes, dpk_stream_t stream);
/* Fused scatter + exchange (replaces the ShuffleFetcher pull, dpark/shuffle.py:309-420, by a
 * push): like dpk_partition_scatter, but bucket b of this chunk is written to the memory at
 * key_dst_ptrs[b] / val_dst_ptrs[b] -- absolute device addresses (uint64, device arrays of F
 * entries) that may point into a PEER GPU's receive buffer mapped over NVLink.  Rows land at
 * element offset (rows of b in this chunk before them), in input order. */
int dpk_partition_scatter_ptrs(const void *keys, int key_kind, const int64_t *key_aux,
                               const void *vals, int32_t val_bytes, int64_t n, int32_t P,
                               const int64_t *thresholds, int32_t nthr, int32_t sub_bits,
                               const uint64_t *key_dst_ptrs, const uint64_t *val_dst_ptrs, void *ws,
                               int64_t ws_bytes, dpk_stream_t stream);
/* The exchange as block pushes (also replaces ShuffleFetcher, dpark/shuffle.py:309-420, and the
 * MapOutputTracker lookup of where each bucket lives, dpark/env.py + dpark/tracker.py): after
 * dpk_partition the rows bound for one peer are ONE contiguous block of the bucket-major buffer.
 * Copies nseg segments in one launch: nbytes[s] bytes from the device address src_ptrs[s] to
 * dst_ptrs[s] (all three are DEVICE arrays, so the table can be computed from the gathered counts
 * without a host sync).  Destinations may be peer-GPU memory mapped over NVLink.  Work items
 * rotate over the segments so that all peers receive at the same time.  nseg <= 1024; addresses
 * and sizes of any alignment (16/8/4/1-byte accesses are chosen per item). */
int dpk_copy_segments(const uint64_t *src_ptrs, const uint64_t *dst_ptrs, const int64_t *nbytes,
                      int32_t nseg, dpk_stream_t stream);
/* The same pushes issued to the GPU's copy engines (no SM is used, so they overlap other kernels at full speed): one
 * cudaMemcpyBatchAsync over a segment table held by the HOST (h_* are host arrays; addresses are device addresses, peer
 * buffers included).  Stream-ordered like everything else; zero-sized segments are skipped. */
int dpk_memcpy_batch(const uint64_t *h_dst_ptrs, const uint64_t *h_src_ptrs, const int64_t *h_nbytes, int32_t count,
                     dpk_stream_t stream);
/* The MapOutputTracker lookup (dpark/shuffle.py:809-826) for the push: from the gathered counts matrix
 * all_counts[nsrc][nbuckets] (device) to the segment table dpk_copy_segments takes, in ONE launch.  Destination d owns
 * the buckets [d * per_block, (d + 1) * per_block); this rank is source row my_src (= my_rank, or my_rank * H + group
 * when every rank sends H groups of map splits).  My bucket-major key / value columns start at the device addresses
 * src_keys / src_vals (ncols = 1: keys only), rank d's receive buffer for column c at dst_base[c * nranks + d] (device
 * array), elements are key_bytes / val_bytes wide.  Writes src_ptrs / dst_ptrs /
 * nbytes [ncols][nranks] (pushes are clamped to `capacity` rows per receive buffer), *need_over = max(*need_over,
 * rows the fullest receive buffer lacks) and, if seg_out != NULL, seg_out[nsrc][own buckets] for dpk_combine: the rows
 * that land in my buffer, so after a clamped push it describes no row past `capacity` (the step's result is invalid,
 * need_over reports it, but the reduce side stays inside its buffers). */
int dpk_push_plan(const int64_t *all_counts, int32_t nsrc, int32_t nranks, int32_t nbuckets, int32_t per_block,
                  int32_t my_src, int32_t my_rank, int32_t ncols, uint64_t src_keys, uint64_t src_vals,
                  const uint64_t *dst_base, int32_t key_bytes, int32_t val_bytes, int64_t capacity, uint64_t *src_ptrs,
                  uint64_t *dst_ptrs, int64_t *nbytes, int64_t *need_over, int64_t *seg_out, dpk_stream_t stream);
/* dpk_push_plan for a PART of every destination's block: the buckets [blk_lo, blk_hi) relative to the block's first
 * bucket, landing in the region of `capacity` rows that starts at row dst_row0 of every receive buffer (seg_out: my own
 * part).  A pipelined shuffle pushes the blocks in parts so that the reduce side (dpk_combine over the part's
 * partitions) runs on the first part while the next is still crossing NVLink. */
int dpk_push_plan_part(const int64_t *all_counts, int32_t nsrc, int32_t nranks, int32_t nbuckets, int32_t per_block,
                       int32_t blk_lo, int32_t blk_hi, int64_t dst_row0, int32_t my_src, int32_t my_rank, int32_t ncols,
                       uint64_t src_keys, uint64_t src_vals, const uint64_t *dst_base, int32_t key_bytes, int32_t val_bytes,
                       int64_t capacity, uint64_t *src_ptrs, uint64_t *dst_ptrs, int64_t *nbytes, int64_t *need_over,
                       int64_t *seg_out, dpk_stream_t stream);
/* The plan of a pipelined shuffle step, one launch per group of map splits: bucket_base[nbuckets] = where the multisplit
 * (dpk_partition_scatter) puts every bucket of this group in the send buffer, and src_ptrs / dst_ptrs / nbytes
 * [nparts][ncols][nranks] = the pushes of part q (the q-th of nparts equal slices of every destination's block of
 * per_block buckets) into region q (region_rows rows, starting at row q * region_rows) of every receive buffer.  In
 * front of every (destination, part) block the send buffer holds up to 16 / min(key_bytes, val_bytes) - 1 pad rows so
 * that source and destination of every push are congruent mod 16 bytes (the copy then runs through the TMA); size it
 * rows + nranks * nparts * (16 / min element size).  seg_out[nparts][nsrc][per_block / nparts]: the segment matrices of
 * my own parts for dpk_combine (the rows that land in each region; columns beyond my last bucket are 0).  need_over as
 * in dpk_push_plan, per region. */
int dpk_pipe_plan(const int64_t *all_counts, int32_t nsrc, int32_t nranks, int32_t nbuckets, int32_t per_block,
                  int32_t nparts, int64_t region_rows, int32_t my_src, int32_t my_rank, int32_t ncols, uint64_t src_keys,
                  uint64_t src_vals, const uint64_t *dst_base, int32_t key_bytes, int32_t val_bytes, int64_t *bucket_base,
                  uint64_t *src_ptrs, uint64_t *dst_ptrs, int64_t *nbytes, int64_t *need_over, int64_t *seg_out,
                  dpk_stream_t stream);
/* The same lookup for the FUSED scatter + exchange (dpk_partition_scatter_ptrs): key_ptrs[b] / val_ptrs[b] (device
 * arrays of nbuckets entries) = the address of the slot of (source my_rank, bucket b) in its owner's receive buffer,
 * laid out source-rank-major then bucket-major exactly as the push delivers it.  A bucket that would end past
 * `capacity` rows of the owner's buffer is pointed into the local dump columns dump_keys / dump_vals (>= this rank's
 * row count) at its local bucket-major offset, and *need_over reports the overflow, so a too-small receive buffer is
 * never overrun; seg_out[nranks][own buckets] (if not NULL) counts the rows that land, 0 for a diverted bucket.
 * nbuckets <= 4096.  Replaces, with dpk_partition_scatter_ptrs, the reducers' pull of every map
 * output over files + HTTP (dpark/shuffle.py:309-420) by stores over NVLink issued by the map-side scatter itself. */
int dpk_fused_plan(const int64_t *all_counts, int32_t nranks, int32_t nbuckets, int32_t per_block, int32_t my_rank,
                   int32_t ncols, const uint64_t *dst_base, int32_t key_bytes, int32_t val_bytes, int64_t capacity,
                   uint64_t dump_keys, uint64_t dump_vals, uint64_t *key_ptrs, uint64_t *val_ptrs, int64_t *need_over,
                   int64_t *seg_out, dpk_stream_t stream);

/* ---- a9: reduce side, DiskHashMerger._merge (dpark/shuffle.py:600-608) ----
 * combined[k] = op(combined[k], v) over the n rows fetched for the nparts reduce
 * partitions [part_first, part_first + nparts) this GPU owns.  Row layout = what
 * the exchange delivers: source-rank-major, and bucket-major inside each source
 * (nsrc = 1 is a plain bucket-major buffer).  seg_rows[nsrc][nparts << sub_bits]
 * (device int64, row-major) = rows of local fine bucket b that came from source
 * s; it locates every segment and sizes one table region per bucket.
 * Outputs: out_offsets[nparts+1] = start
 * of each partition's output range (= row offsets of the partitions),
 * out_counts[nparts] = distinct keys per partition; partition j's result is
 * out_keys/out_vals[out_offsets[j] .. out_offsets[j] + out_counts[j]).  Order
 * inside a partition is unspecified (the reference iterates a dict).
 * Accumulation: I64/I32 values -> int64 (exact while |sum| < 2^63, like the
 * reference's big ints; products wrap mod 2^64, exact while the final product
 * fits); F64/F32 values -> float64 (the reference adds Python floats); out_vals
 * is 8 bytes per row.  out_keys/out_vals hold n entries.
 * Float MIN / MAX are IEEE 754-2019 minimum / maximum: NaN if any of the key's
 * values is NaN, otherwise the usual one with -0.0 < +0.0.  The result does not
 * depend on the merge order, so it is the same on every dpk_set_option setting.
 * n may be an UPPER BOUND of the rows (e.g. the capacity of a receive buffer): every
 * reduce_impl reads only the rows seg_rows describes, so a multi-GPU caller needs no host
 * read of the received row count.
 * Float sums start from -0.0, so a key whose only values are -0.0 sums to -0.0 as in Python.
 * Errors that only the device can see: out_counts[j] == -1 marks a partition whose merge
 * failed -- a fine bucket held more distinct keys than the shared-memory table takes even
 * after splitting it by every spare hash bit (dpk_aggregate2.cuh); nothing is dropped
 * silently, the caller that reads the counts raises (dpark_b200.shuffle.check_counts).
 */
int64_t dpk_combine_workspace_bytes(int64_t n, int32_t nbuckets, int32_t nsrc);
int dpk_combine(const void *keys, int key_kind, const int64_t *key_aux, const void *vals,
                int val_kind, int64_t n, int op, int32_t P, const int64_t *thresholds, int32_t nthr,
                int32_t sub_bits, int32_t part_first, int32_t nparts, int32_t nsrc,
                const int64_t *seg_rows, void *out_keys, void *out_vals, int64_t *out_offsets,
                int64_t *out_counts, void *ws, int64_t ws_bytes, dpk_stream_t stream);
/* Process-wide A/B switches (results are the same for every setting -- the same set of rows per reduce partition,
 * float sums within their rounding; only the speed differs):
 *   "reduce_impl"     2 (default) second-level split + one CTA per fine bucket merging in a
 *                     shared-memory table; 1 = per-bucket tables in HBM, one 8-CTA cluster per bucket;
 *                     0 = three grid-wide passes over global tables
 *   "agg_impl"        1 (default) k_smem_aggregate2: staged rows + 32-bit row-index tags claimed with
 *                     cas.b32; 0 = the round-1 kernel (128-bit {key, accumulator} slots)
 *   "agg_cursor"      1 (default) a fine bucket reserves its output range with one atomicAdd on the
 *                     partition's count (partitions are sets: any order); 0 = chained scan with
 *                     decoupled look-back (fine buckets in order; the order inside one still varies)
 *   "agg_batched"     1 = four rows per thread in flight in the insert phase; 0 (default) = probe loop per row
 *   "agg_ctas"        4 (default) or 3 resident CTAs per SM the merge kernel is compiled for
 *   "agg_pipe"        0 (default); 1 = k_smem_aggregate3 (rows stay in registers, next bucket prefetched: faster on
 *                     duplicate-heavy data, slower on mostly-distinct keys)
 *   "agg_wide"        round-1 kernel only: 1 (default) claim a table slot and deposit the first value with
 *                     one 128-bit shared-memory CAS; 0 = 64-bit key CAS, then an atomic on the accumulator
 *   "agg_target_rows" rows per fine bucket the second-level split aims for (default 2048 = the window)
 *   "count_mode"      1 (default) one shared-memory atomic per row in the histogram pass; 0 = warp
 *                     peer masks + leader update
 *   "scatter_bulk"    1 (default) unordered multisplits (reduceByKey paths, second-level split) run
 *                     k_part_scatter_bulk: one shared atomic per row for the rank, bucket runs leave the
 *                     staged tile through cp.async.bulk (TMA, SASS UBLKCP); 0 = the round-1 kernel
 *   "scatter_threads" 512 (default), 256 or 1024 threads per CTA of the bulk kernel (1024: 8192-row tiles)
 *   "scatter_seg_wide" 1 (default): the segmented (second-level) launches use the 1024-thread form
 *   "scatter_wide_from" 512 (default): bucket count from which plain bulk launches use 8192-row tiles (0 = never)
 *   "scatter_ptr_bulk" 1 (default): unordered pointer-mode scatters (dpk_partition_scatter_ptrs) run the bulk
 *                     kernel; 0 = the round-1 kernel
 *   "scatter_ptr_threads" 1024 (default) or 512 threads per CTA of the bulk kernel in pointer mode
 *   "scatter_items"   round-1 kernel only: 16 (default) or 8 rows per thread and tile
 *   "agg_split"       1 (default): the one-window buckets and the oversized ones take separate launches
 *   "copy_sms"        0 (default) = dpk_copy_segments fills the GPU; n > 0 = it runs on n whole SMs
 *   "copy_tma"        1 (default): copies on a few SMs run through the TMA; 0 = loads and stores
 *   "agg_timing"      0 (default); 1 = debugging aid: the merge kernel prints its per-phase cycle counts */
int dpk_set_option(const char *name, int64_t value);

/* ---- a10: reduce side of groupByKey (dpark/dependency.py:107-118 merged by
 * OrderedGroupByDiskHashMerger, dpark/shuffle.py:626-646): per key the list of
 * its values ordered by (map_id, arrival).  On the device: a STABLE sort of the
 * received rows by key -- LSD radix, each pass the stable multisplit of a4 with
 * bucket = one digit of the raw int64 key bits -- then CSR extraction.
 *   dpk_key_or      : *out_or (device uint64) = OR_i(keys[i] ^ keys[0]); digits where
 *                     it is zero need no pass.
 *   dpk_radix_pass  : one pass, digit = (key >> shift) & (2^bits - 1), bits <= 12;
 *                     ws = dpk_partition_workspace_bytes(n, 1 << bits).
 *   dpk_group_heads : over keys sorted so that equal keys are adjacent: out_keys[g],
 *                     out_starts[g] = first row of group g, out_starts[G] = n,
 *                     *out_ngroups = G (device int64).  out_starts holds n+1 entries.
 */
int dpk_key_or(const int64_t *keys, int64_t n, uint64_t *out_or, dpk_stream_t stream);
/* out[i] = src[idx[i]] (row-id keys: fetch the hash / representative of a moved row) */
int dpk_gather_i64(const int64_t *src, const int64_t *idx, int64_t n, int64_t *out,
                   dpk_stream_t stream);
int dpk_radix_pass(const int64_t *keys, const void *vals, int32_t val_bytes, int64_t n, int32_t shift,
                   int32_t bits, int64_t *out_keys, void *out_vals, void *ws, int64_t ws_bytes,
                   dpk_stream_t stream);
/* One stable radix pass INSIDE every first-level bucket: input source-major, bucket-major (seg_rows[nsrc][nbuckets]
 * device int64: what the exchange delivers; nsrc = 1 once the rows are bucket-major), output bucket-major with every
 * bucket stably split by the digit.  All rows of a key share a bucket, so after the passes over the differing digits
 * every bucket is sorted by key and no pass over the partition id is needed (OrderedGroupByDiskHashMerger,
 * dpark/shuffle.py:626-646).  out_fine_off[(nbuckets << bits) + 1] receives the digit-group boundaries. */
int64_t dpk_radix_pass_seg_workspace_bytes(int64_t n, int32_t nbuckets, int32_t nsrc, int32_t bits);
int dpk_radix_pass_seg(const int64_t *keys, const void *vals, int32_t val_bytes, int64_t n, int32_t shift,
                       int32_t bits, int32_t nbuckets, int32_t nsrc, const int64_t *seg_rows, int64_t *out_keys,
                       void *out_vals, int64_t *out_fine_off, void *ws, int64_t ws_bytes, dpk_stream_t stream);
int64_t dpk_group_heads_workspace_bytes(int64_t n);
int dpk_group_heads(const int64_t *sorted_keys, int64_t n, int64_t *out_keys, int64_t *out_starts,
                    int64_t *out_ngroups, void *ws, int64_t ws_bytes, dpk_stream_t stream);

/* ---- f1: join / leftOuterJoin / rightOuterJoin / outerJoin (dpark/rdd.py:649-676) over columns --------------------
 * Input: the CSR of a groupByKey of the tagged union (dpk_group_heads over the sorted rows): group g's row ids are
 * ids[group_starts[g] .. group_starts[g+1]), where ids < nL are left rows (left value nr. id) and the others right
 * rows (right value nr. id - nL).  Left ids precede right ids inside every group (the group-by is stable and the
 * left rows come first).  keep_left / keep_right: unmatched keys of that side survive, paired with a missing value.
 *   dpk_join_count : out_nl[g] = left rows of group g; out_count[g] = L * R, L = nl ? nl : keep_right,
 *                    R = nr ? nr : keep_left (int64, ngroups entries each).
 *   dpk_join_emit  : out_off[ngroups + 1] = the exclusive scan of out_count (n_out = out_off[ngroups]).  Output row
 *                    out_off[g] + a * R + b of group g: out_keys = group_keys[g] (int64 bits), out_left = left value
 *                    a, out_right = right value b, in the order `for a in left for b in right`.  A missing side
 *                    writes value 0 and valid flag 0; out_lvalid (uint8) is written iff keep_right, out_rvalid iff
 *                    keep_left, and must then be given.  lval_bytes / rval_bytes in {4, 8}, chosen independently; lvals / rvals
 *                    may be NULL when that side has no rows. */
int dpk_join_count(const int64_t *ids, const int64_t *group_starts, int64_t ngroups, int64_t nL, int32_t keep_left,
                   int32_t keep_right, int64_t *out_nl, int64_t *out_count, dpk_stream_t stream);
int dpk_join_emit(const int64_t *group_keys, const int64_t *group_starts, const int64_t *ids, const int64_t *nl,
                  const int64_t *out_off, int64_t ngroups, int64_t nL, const void *lvals, int32_t lval_bytes,
                  const void *rvals, int32_t rval_bytes, int32_t keep_left, int32_t keep_right, int64_t n_out,
                  int64_t *out_keys, void *out_left, void *out_right, uint8_t *out_lvalid, uint8_t *out_rvalid,
                  dpk_stream_t stream);

/* ---- f1: groupWith / cogroup of N inputs (dpark/rdd.py:686-731) over columns ---------------------------------------
 * Input: the same CSR as the join, the ids of input t being [bounds[t], bounds[t+1]) (bounds: device, ninputs + 1
 * entries, ascending).  Inside every group the ids ascend, so input t's rows of the group are one sub-run.
 *   dpk_cogroup_count : out_first[t * ngroups + g] = the position in ids where input t's sub-run of group g starts,
 *                       out_count[t * ngroups + g] = its length (input-major, ninputs * ngroups entries each).
 *   dpk_cogroup_emit  : one input (first = its row of out_first, id_base = its bounds[t]); out_off[ngroups + 1] = the
 *                       exclusive scan of its counts (n_out = out_off[ngroups]).  Output row r of group g
 *                       (out_off[g] <= r < out_off[g+1]) is vals[ids[first[g] + r - out_off[g]] - id_base]: per key
 *                       the input's values in (map split, position) order.  val_bytes in {4, 8}. */
int dpk_cogroup_count(const int64_t *ids, const int64_t *group_starts, int64_t ngroups, const int64_t *bounds,
                      int32_t ninputs, int64_t *out_first, int64_t *out_count, dpk_stream_t stream);
int dpk_cogroup_emit(const int64_t *ids, const int64_t *first, const int64_t *out_off, int64_t ngroups, int64_t id_base,
                     const void *vals, int32_t val_bytes, int64_t n_out, void *out_vals, dpk_stream_t stream);

/* ---- f5: innerJoin (dpark/rdd.py:626-648) of a big column against a small one --------------------------------------
 * The small side's distinct keys go into a hash table; every big row is probed in place and expands to one output row
 * per small row of its key.  Keys are compared as normalised bits: ints widened to int64, floats widened to float64
 * with -0.0 spelled 0.0; a NaN key matches nothing.
 *   dpk_bcast_build : group_keys[ngroups] = the small side's distinct normalised keys (int64 bits, e.g. a group-by's
 *                     group keys), ngroups <= INT32_MAX; table = nslots 16-byte slots, 16-byte aligned, every byte
 *                     0xFF on entry; nslots = the least power of two >= max(2, 2 * ngroups).
 *   dpk_bcast_probe : keys[n] of kind DPK_K_I64 / I32 / F64 / F32, read in place.  out_grp[r] (int32) = the group of
 *                     key r or -1, out_count[r] (int64) = group_starts[g + 1] - group_starts[g], 0 on a miss.
 *   dpk_bcast_emit  : out_off[n + 1] = the exclusive scan of out_count (n_out = out_off[n]).  Output row out_off[r] + j
 *                     of big row r: out_keys = keys[r] (its own bits), out_left = lvals[r], out_right =
 *                     rvals[ids[group_starts[grp[r]] + j]].  key_bytes / lval_bytes / rval_bytes in {4, 8}. */
int dpk_bcast_build(const int64_t *group_keys, int64_t ngroups, void *table, int64_t nslots, dpk_stream_t stream);
int dpk_bcast_probe(const void *keys, int32_t key_kind, int64_t n, const void *table, int64_t nslots,
                    const int64_t *group_starts, int32_t *out_grp, int64_t *out_count, dpk_stream_t stream);
int dpk_bcast_emit(const void *keys, int32_t key_bytes, const void *lvals, int32_t lval_bytes, const int32_t *grp,
                   const int64_t *out_off, int64_t n, const int64_t *group_starts, const int64_t *ids,
                   const void *rvals, int32_t rval_bytes, int64_t n_out, void *out_keys, void *out_left,
                   void *out_right, dpk_stream_t stream);

/* ---- f4: topByKey (dpark/rdd.py:552-594) of a numeric value column ----------------------------------------------------
 * Per key the first top_n values of a stable sort of its values (ascending, or descending with reverse != 0), in rounds
 * over runs of candidates.  Round 1's runs are the group-by's: run_starts = group_starts and candidate i is
 * vals[ids[i]]; later rounds pass ids = NULL and the previous round's output as vals (candidate i is vals[i]).
 *   dpk_topk_lengths : out_len[g] = the length of run g after one round (nruns entries): a run of L <= DPK_TOPK_TILE
 *                      candidates keeps min(top_n, L) -- its answer; a longer one is cut into chunks of DPK_TOPK_TILE
 *                      from its start and keeps the first top_n of every chunk, floor(L / T) * top_n + min(top_n, L % T).
 *   dpk_topk_round   : out_starts[nruns + 1] = the exclusive scan of out_len; writes every chunk's (every short run's)
 *                      first values in order to out_vals.  n = run_starts[nruns].  Equal values keep their candidate
 *                      order; -0.0 and 0.0 compare equal and keep their bits.  Float values must not be NaN.
 *                      val_bytes in {4, 8}, val_float != 0 for IEEE values, 1 <= top_n <= DPK_TOPK_MAX_N.
 * Repeat while the longest run is longer than DPK_TOPK_TILE; then one more round leaves min(top_n, L) values per key. */
#define DPK_TOPK_TILE 4096
#define DPK_TOPK_MAX_N 512
int dpk_topk_lengths(const int64_t *run_starts, int64_t nruns, int32_t top_n, int64_t *out_len, dpk_stream_t stream);
int dpk_topk_round(const int64_t *ids, const void *vals, int32_t val_bytes, int32_t val_float,
                   const int64_t *run_starts, int64_t nruns, int64_t n, const int64_t *out_starts, int32_t top_n,
                   int32_t reverse, void *out_vals, dpk_stream_t stream);

/* ---- f6: sort (dpark/rdd.py:273-287) of a numeric (k, v) column pair --------------------------------------------------
 * One global stable sort by order words, then the range partitions as slices of it.  Columns are read in place, of kind
 * DPK_K_I64 / I32 / F64 / F32.  A value is widened to 64 bits (ints to int64, floats to float64) and its order word is
 * topk_order_key of those bits at width 8, complemented when reverse != 0: unsigned order of the words is the values'
 * order (descending with reverse), -0.0 and 0.0 get one word.  NaN has no word.
 *   dpk_sort_keys   : col0 (kind0) is the first order column, col1 (kind1) the second one or NULL.  out_w0[i] / out_w1[i]
 *                     = the order words of row i (int64 bits), out_ids[i] = i; *nan_flag (device int32) is set to 1 if an
 *                     order column holds a NaN (the caller clears it).  n < 2^31.
 *   dpk_sort_cuts   : sorted_w0[n] = the first order words after the sort, ids[n] the row ids in that order.  bounds0[nbounds]
 *                     = the range bounds' first order values ascending (RangePartitioner.keys), widened bits of kind0's
 *                     type; bounds1 = their second values (the (k, v) order; NULL otherwise), whose rows' second words are
 *                     recomputed from vals[ids[i]] of val_kind.  out_starts[nbounds + 2]: 0, the first row of every
 *                     partition j = 1 .. nbounds, n.  Ascending, partition j starts at the first row whose words are >=
 *                     bound j - 1's; reverse, at the first row whose words are > bound nbounds - j's.
 *   dpk_sort_gather : out_keys[i] = keys[ids[i]], out_vals[i] = vals[ids[i]], key_bytes / val_bytes in {4, 8}. */
int dpk_sort_keys(const void *col0, int32_t kind0, const void *col1, int32_t kind1, int64_t n, int32_t reverse,
                  int64_t *out_w0, int64_t *out_w1, int64_t *out_ids, int32_t *nan_flag, dpk_stream_t stream);
int dpk_sort_cuts(const int64_t *sorted_w0, const int64_t *ids, const void *vals, int32_t val_kind, int64_t n,
                  const int64_t *bounds0, int32_t kind0, const int64_t *bounds1, int32_t nbounds, int32_t reverse,
                  int64_t *out_starts, dpk_stream_t stream);
int dpk_sort_gather(const void *keys, int32_t key_bytes, const void *vals, int32_t val_bytes, const int64_t *ids,
                    int64_t n, void *out_keys, void *out_vals, dpk_stream_t stream);

/* ---- f7: percentilesByKey (dpark/rdd.py:815-850) of a numeric value column ---------------------------------------------
 * Per key and map split the t-digest MergingDigest().update(values) + compress() (dpark_b200/quantiles.py, compression
 * 100), absorbed into the key's first one in split order, then quantile(q) -- bit for bit.  The group-by's CSR gives
 * every key's row ids ids[n] in (split, position) order; the splits are blocks of `per` rows, so row id r lies in split
 * r / per.  A segment is one (key, split) run of ids.
 *   dpk_tdigest_heads : head[n] (uint8, zeroed by the caller) gets 1 at every segment's first row.
 *   dpk_tdigest_build : seg_starts[nseg + 1] = the heads' positions, then n; seg_off[nseg + 1] = the exclusive scan of
 *                       min(segment length, 209).  Segment s's digest: cent_n[s] centroids at cent_m / cent_w[seg_off[s]
 *                       ..] (means, weights), lohi[2 s .. 2 s + 1] = the smallest / largest first / last mean its folds
 *                       met.  val_kind DPK_K_I32 / I64 / F32 / F64, converted as Python's float().  work: nseg + 2
 *                       int64 of scratch.
 *   dpk_tdigest_merge : out[g * nq + j] = quantile(qs[j]) of key g's merged digest (group_starts[ngroups + 1]).
 * Both set *flag (device int32, zeroed by the caller) to nonzero when a value is NaN, a centroid mean comes out NaN or
 * below its predecessor, or a fold would stage more than 418 entries: the results are then void. */
int dpk_tdigest_heads(const int64_t *ids, int64_t n, const int64_t *group_starts, int64_t ngroups, int64_t per,
                      uint8_t *head, dpk_stream_t stream);
int dpk_tdigest_build(const int64_t *ids, const void *vals, int32_t val_kind, const int64_t *seg_starts,
                      const int64_t *seg_off, int64_t nseg, double *cent_m, double *cent_w, int32_t *cent_n,
                      double *lohi, int64_t *work, int32_t *flag, dpk_stream_t stream);
int dpk_tdigest_merge(const int64_t *group_starts, int64_t ngroups, const int64_t *seg_starts, const int64_t *seg_off,
                      int64_t nseg, const int32_t *cent_n, const double *lohi, const double *cent_m,
                      const double *cent_w, const double *qs, int32_t nq, double *out, int32_t *flag,
                      dpk_stream_t stream);

/* ---- f8: Bernoulli sample (dpark/rdd.py:1379-1397 SampleRDD without replacement) ---------------------------------------
 * Split i covers rows [ranges[2 i], ranges[2 i + 1]) and owns the MT19937 state states[624 i .. 624 i + 624), the first
 * 624 words of random.Random(seed + i).getstate()[1] right after seeding (its position is 624).  Row j of the split is
 * kept when the j-th random() of that generator is <= frac (a plain double compare: a NaN frac keeps nothing).
 * out_ids[ranges[2 i] ..] gets split i's kept row ids in row order, out_counts[i] how many there are (device int64). */
int dpk_sample_bernoulli(const uint32_t *states, const int64_t *ranges, int64_t nsplits, double frac,
                         int64_t *out_ids, int64_t *out_counts, dpk_stream_t stream);

/* ---- f9: top, uniq and hot (dpark/rdd.py:383-398) of a numeric (k, v) column pair --------------------------------------
 * Stable select of the n smallest rows by (w0[, w1], row id), w0 / w1 unsigned 64-bit order words (int64 bits, e.g. from
 * dpk_sort_keys; w1 NULL for one word).  state: int64 [16] on the device, set by the caller before the first round to
 * zeros except state[1] = 56 (the first digit's shift), state[2] = n (the rank sought) and state[4] = the row count;
 * hist: int64 [768], zeros in [0, 512) and all ones in [512, 768).
 *   dpk_select_round   : one MSD radix round over the m candidates (cands[m] row ids; NULL: all rows 0 .. m-1): picks the
 *                        8-bit bucket of the state[2]-th smallest.  Afterwards state[4] = the candidates in that bucket,
 *                        state[7] = 1 when the threshold words state[5] / state[6] are exact, state[3] = the rows below
 *                        them.  At most 8 rounds per word.
 *   dpk_select_compact : out_cands[state[4]] = the candidates of the chosen bucket (any order), for the next round.
 *   dpk_select_take    : once state[7] = 1, out_ids[take] = every row below the threshold and the first take - state[3]
 *                        rows equal to it, in row id order (take = the n of the rounds, < n rows).  tile_lt / tile_eq:
 *                        dpk_select_tiles(n) int64 of scratch each.
 * Distinct (k, v) pairs with their counts: a pair is both elements widened (ints to int64, floats to float64) with -0.0
 * spelled 0.0; column kinds DPK_K_I64 / I32 / F64 / F32, read in place.
 *   dpk_uniq_insert : every row into table (nslots = bcast_slots(n) slots of 8 bytes; every int64 slot filled with
 *                     0x7FFFFFFF by the caller).  state: int64 [2], zeroed by the caller; state[0] = 1 when a NaN occurs
 *                     (those rows are left out).
 *   dpk_uniq_emit   : out_first[d] / out_count[d] = the first row id and the row count of every distinct pair, in slot
 *                     order; state[1] = the number of pairs.  out_first / out_count hold at least n entries. */
int dpk_select_round(const int64_t *w0, const int64_t *w1, const int64_t *cands, int64_t m, int64_t *state,
                     int64_t *hist, dpk_stream_t stream);
int dpk_select_compact(const int64_t *w0, const int64_t *w1, const int64_t *cands, int64_t m, int64_t *state,
                       int64_t *out_cands, dpk_stream_t stream);
int64_t dpk_select_tiles(int64_t n);
int dpk_select_take(const int64_t *w0, const int64_t *w1, int64_t n, int64_t take, const int64_t *state,
                    int64_t *tile_lt, int64_t *tile_eq, int64_t *out_ids, dpk_stream_t stream);
int dpk_uniq_insert(const void *keys, int32_t key_kind, const void *vals, int32_t val_kind, int64_t n, void *table,
                    int64_t nslots, int64_t *state, dpk_stream_t stream);
int dpk_uniq_emit(const void *table, int64_t nslots, int64_t *out_first, int64_t *out_count, int64_t *state,
                  dpk_stream_t stream);

/* ---- f4: device text ingest (dpark/rdd.py:1633-1711 TextFileRDD + the tokenising flatMap of examples/wc.py:10-12) ----
 * Tokens of an ASCII byte range that begins and ends on line boundaries = its maximal runs of non-whitespace bytes
 * (str.split() without arguments: ' ', \t \n \v \f \r, \x1c..\x1f).  dpk_tokenize_count writes the number of token
 * starts of every 4096-byte block (dpk_tokenize_blocks(n) entries) and ORs bit 0 into *flags (device) if any byte is
 * >= 0x80 (the caller must then tokenise that range row-wise in Python: Unicode whitespace, decoding errors);
 * dpk_tokenize_emit takes the EXCLUSIVE scan of those counts and writes (start, length) of every token in text order.
 * dpk_gather_bytes makes selected rows contiguous: out[out_off[i] ..) = data[starts[r] .. starts[r] + lens[r]),
 * r = idx ? idx[i] : i -- the (data, offsets) form dpk_hash_bytes / dpk_dict_encode take. */
int64_t dpk_tokenize_blocks(int64_t n);
int dpk_tokenize_count(const uint8_t *data, int64_t n, int64_t *block_counts, int64_t *flags, dpk_stream_t stream);
int dpk_tokenize_emit(const uint8_t *data, int64_t n, const int64_t *block_base, int64_t *starts, int64_t *lens,
                      dpk_stream_t stream);
int dpk_gather_bytes(const uint8_t *data, const int64_t *starts, const int64_t *lens, const int64_t *idx, int64_t m,
                     const int64_t *out_off, uint8_t *out, dpk_stream_t stream);
/* The same pair for UTF-8 text (a range the ASCII pair declines), with the same block counts, scan and outputs.
 * Tokens = maximal runs of code points c with !chr(c).isspace() (Python's whitespace: U+0009..000D, U+001C..0020,
 * U+0085, U+00A0, U+1680, U+2000..200A, U+2028, U+2029, U+202F, U+205F, U+3000), each as the (start, length) of its
 * UTF-8 bytes.  dpk_tokenize_utf8_count ORs bit 0 into *flags if the range is not strict UTF-8 (what
 * bytes.decode("utf-8") rejects: stray continuation bytes, C0, C1, F5..FF, overlong forms, surrogates, values above
 * U+10FFFF, a sequence cut short by the end of the range); the caller must then run no emit and leave the range to
 * the row-wise path, which raises UnicodeDecodeError. */
int dpk_tokenize_utf8_count(const uint8_t *data, int64_t n, int64_t *block_counts, int64_t *flags, dpk_stream_t stream);
int dpk_tokenize_utf8_emit(const uint8_t *data, int64_t n, const int64_t *block_base, int64_t *starts, int64_t *lens,
                           dpk_stream_t stream);

/* ---- f10: numeric text columns (DparkContext.textFileColumns) ---------------------------------------------------------
 * A byte range that starts on a line start; a line ends at the next '\n' or at n, and a final '\n' opens no line.
 *   dpk_textcols_count : per dpk_tokenize_blocks(n) block of 4096 bytes its number of line starts; ORs bit 0 into
 *                        *flags when a byte >= 0x80 occurs (the caller then checks the range with
 *                        dpk_tokenize_utf8_count).
 *   dpk_textcols_emit  : takes the EXCLUSIVE scan of those counts and writes every line start, in text order.
 *   dpk_textcols_parse : per line, fields key and value of line.split() (sep_len == 0) or line.split(sep) (sep[sep_len]
 *                        bytes, UTF-8) parsed as int() (kind DPK_K_I64: out = the int64) or float() (DPK_K_F64: out =
 *                        the float64 bits).  Only [+-]?[0-9]{1,19} within int64, and decimal / exponent / inf /
 *                        infinity / nan ASCII floats whose rounding the conversion decides, with \t \n \v \f \r and
 *                        space stripped, are parsed here; every other line gets host[i] = 1 and zeros, and the caller
 *                        must parse it with Python.
 * None allocates or synchronises. */
int dpk_textcols_count(const uint8_t *data, int64_t n, int64_t *block_counts, int64_t *flags, dpk_stream_t stream);
int dpk_textcols_emit(const uint8_t *data, int64_t n, const int64_t *block_base, int64_t *starts, dpk_stream_t stream);
int dpk_textcols_parse(const uint8_t *data, int64_t n, const int64_t *starts, int64_t nlines, const uint8_t *sep,
                       int32_t sep_len, int32_t key, int32_t value, int32_t key_kind, int32_t value_kind,
                       int64_t *out_keys, int64_t *out_vals, uint8_t *host, dpk_stream_t stream);

/* ---- variable-length keys (str / bytes): key identity on the device ---------
 * The reference's dicts compare keys by value; two different strings may share
 * a portable_hash, so the hash alone cannot be the key.  dpk_dict_encode gives
 * every row the index of a representative row holding an equal byte string
 * (out_rep[i] == out_rep[j]  <=>  key i == key j): an open-addressing table of
 * row indices, probed by hash, verified byte-wise.  The representative ids then
 * go through dpk_combine as DPK_K_ROWID keys with key_aux = hash.
 * hash: the column dpk_hash_bytes produced for the same (data, offsets). */
int64_t dpk_dict_encode_workspace_bytes(int64_t n);
int dpk_dict_encode(const uint8_t *data, const int64_t *offsets, const int64_t *hash, int64_t n,
                    int64_t *out_rep, void *ws, int64_t ws_bytes, dpk_stream_t stream);

/* ---- measurement hooks (SURVEY.md §5 tracing: TaskStats -> CUDA events) -----
 * dpk_launch_count: kernels launched by this library since load.
 * dpk_prof_enable(1): from now on every kernel launch is bracketed by CUDA
 * events on its stream (up to DPK_PROF_MAX launches are kept, later ones are
 * counted but not timed); dpk_prof_enable(0) stops.  dpk_prof_count() = entries
 * kept; dpk_prof_get(i, h_name[64], &h_ms) synchronises entry i's stop event and
 * returns the kernel label and its device time in milliseconds. */
#define DPK_PROF_MAX 4096
int64_t dpk_launch_count(void);
int dpk_prof_enable(int on);
int dpk_prof_count(void);
int dpk_prof_get(int i, char *h_name, float *h_ms);

#ifdef __cplusplus
}
#endif
#endif /* DPARK_B200_H */
