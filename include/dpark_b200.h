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
 * rows the fullest receive buffer lacks) and, if seg_out != NULL, seg_out[nsrc][own buckets] for dpk_combine. */
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
 * my own parts for dpk_combine (columns beyond my last bucket are 0).  need_over as in dpk_push_plan, per region. */
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
 * never overrun.  nbuckets <= 4096.  Replaces, with dpk_partition_scatter_ptrs, the reducers' pull of every map
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
 * reference's big ints); F64/F32 values -> float64 (the reference adds Python
 * floats); out_vals is 8 bytes per row.  out_keys/out_vals hold n entries.
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
