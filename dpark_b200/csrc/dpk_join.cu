// dpk_join.cu -- f1: the expansion step of join / leftOuterJoin / rightOuterJoin / outerJoin (dpark/rdd.py:649-676)
// over the CSR a groupByKey of the tagged union leaves (dpk_group.cu): per key the row ids of its left rows
// (id < nL) followed by those of its right rows, each in (map split, position) order.
//
//   k_join_count : one thread per group; nl[g] by binary search for nL in the group's id run, and the group's
//                  output row count L * R (join_count, dpk_common.cuh).
//   k_join_emit  : load-balanced over OUTPUT rows.  A CTA takes a fixed tile of JN_TILE output rows, finds the groups
//                  the tile spans by binary search on the exclusive scan out_off[G + 1] of the counts, and maps every
//                  row to (group, a, b).  A hot key's L * R rows spread over as many CTAs as they fill; a group with
//                  no output rows occupies no row of any tile.
// Algorithmic bytes of the emit: per output row 8 (key) + LW + RW written (+1 per valid flag), 8 + 8 (the two ids)
// + LW + RW read; the group-level reads (out_off, starts, nl, keys) are per tile, not per row.
//
// groupWith / cogroup of N inputs (dpark/rdd.py:686-731) over the same CSR, input t owning the ids [bounds[t],
// bounds[t + 1]): no cross product, every key's run is split N ways.
//   k_cogroup_count : one thread per group; per input the start of its sub-run (a lower-bound search for bounds[t])
//                     and its length (cogroup_split, dpk_common.cuh).
//   k_cogroup_emit  : one launch per input, load-balanced over that input's output rows with the tile of k_join_emit;
//                     output row r of group g is value ids[first[g] + r - out_off[g]] - id_base.
// Algorithmic bytes of a cogroup emit: per output row 8 (the id) + W read, W written.
//
// innerJoin of a big input against a small one (dpark/rdd.py:626-648), no group-by of the big side:
//   k_bcast_build : one thread per distinct small key; claims a slot of the hash table (BcastSlot, dpk_common.cuh) with
//                   atomicCAS on its group, linear probing, then stores the key bits.
//   k_bcast_probe : one thread per big row, the key column read in place; writes the row's group (or -1) and its
//                   match count.
//   k_bcast_emit  : load-balanced over OUTPUT rows with the tile of k_join_emit, big rows in the role of groups (a
//                   missed row occupies no row of any tile).
// Algorithmic bytes: probe K read, 4 + 8 written per big row; emit per output row K + LW + RW written, K + LW + 8 (the
// id) + RW read.  Table reads are not credited.
#include "dpk_common.cuh"

namespace dpk {

constexpr int JN_THREADS = 256;
constexpr int JN_ITEMS = 8;
constexpr int JN_TILE = JN_THREADS * JN_ITEMS;

__global__ void __launch_bounds__(256)
k_join_count(const int64_t *__restrict__ ids, const int64_t *__restrict__ starts, int64_t G, int64_t nL,
             bool keep_left, bool keep_right, int64_t *__restrict__ out_nl, int64_t *__restrict__ out_count) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const int64_t s = starts[g], len = starts[g + 1] - s;
    const int64_t nl = join_left_rows(ids + s, len, nL);
    out_nl[g] = nl;
    out_count[g] = join_count(nl, len - nl, keep_left, keep_right);
}

// The rows of one CTA of a load-balanced emit: a tile of JN_TILE output rows [i0, i_last], and the groups they fall in,
// g0 .. g0 + span - 1, found by binary search on the exclusive scan off[G + 1] of the groups' row counts.  A tile's
// rows belong to at most JN_TILE groups with rows, but empty groups between them also lie in that range: the offsets
// are staged in shared memory (s_off[JN_TILE + 1]) when they fit, searched in place otherwise.
struct EmitTile {
    const int64_t *off, *s_off;
    int64_t i0, i_last, g0, span;
    bool staged;

    // the group of output row i and that group's first output row
    __device__ __forceinline__ void locate(int64_t i, int64_t *g, int64_t *base) const {
        if (staged) {
            const int64_t j = group_of(s_off, 0, span, i);
            *g = g0 + j;
            *base = s_off[j];
        } else {
            *g = group_of(off, g0, g0 + span, i);
            *base = off[*g];
        }
    }
};

__device__ __forceinline__ EmitTile emit_tile(const int64_t *off, int64_t G, int64_t n_out, int64_t *s_off,
                                              int64_t *s_g) {
    EmitTile t;
    t.off = off;
    t.s_off = s_off;
    t.i0 = (int64_t)blockIdx.x * JN_TILE;
    t.i_last = min(t.i0 + JN_TILE, n_out) - 1;
    // the groups of the tile's first and last rows
    if (threadIdx.x == 0) s_g[0] = group_of(off, 0, G, t.i0);
    if (threadIdx.x == 32) s_g[1] = group_of(off, 0, G, t.i_last);
    __syncthreads();
    t.g0 = s_g[0];
    t.span = s_g[1] - t.g0 + 1;
    t.staged = t.span <= JN_TILE;
    if (t.staged)
        for (int64_t j = threadIdx.x; j <= t.span; j += JN_THREADS) s_off[j] = off[t.g0 + j];
    __syncthreads();
    return t;
}

template <int LW, int RW>
__global__ void __launch_bounds__(JN_THREADS)
k_join_emit(const int64_t *__restrict__ gkeys, const int64_t *__restrict__ starts, const int64_t *__restrict__ ids,
            const int64_t *__restrict__ nls, const int64_t *__restrict__ out_off, int64_t G, int64_t nL,
            const void *__restrict__ lvals, const void *__restrict__ rvals, bool keep_left, int64_t n_out,
            int64_t *__restrict__ out_keys, void *__restrict__ out_left, void *__restrict__ out_right,
            uint8_t *__restrict__ out_lvalid, uint8_t *__restrict__ out_rvalid) {
    typedef typename ValWord<LW>::T LT;
    typedef typename ValWord<RW>::T RT;
    __shared__ int64_t s_off[JN_TILE + 1];
    __shared__ int64_t s_g[2];
    const EmitTile tile = emit_tile(out_off, G, n_out, s_off, s_g);
#pragma unroll 2
    for (int it = 0; it < JN_ITEMS; it++) {
        const int64_t i = tile.i0 + (int64_t)it * JN_THREADS + threadIdx.x;
        if (i > tile.i_last) break;
        int64_t g, base;
        tile.locate(i, &g, &base);
        const int64_t s = starts[g], nl = nls[g], nr = starts[g + 1] - s - nl;
        int64_t a, b;
        join_pair(i - base, nr, keep_left, &a, &b);
        out_keys[i] = gkeys[g];
        LT lv = 0;
        RT rv = 0;
        if (nl > 0) lv = static_cast<const LT *>(lvals)[ids[s + a]];
        if (nr > 0) rv = static_cast<const RT *>(rvals)[ids[s + nl + b] - nL];
        static_cast<LT *>(out_left)[i] = lv;
        static_cast<RT *>(out_right)[i] = rv;
        if (out_lvalid) out_lvalid[i] = nl > 0;
        if (out_rvalid) out_rvalid[i] = nr > 0;
    }
}

typedef void (*EmitFn)(const int64_t *, const int64_t *, const int64_t *, const int64_t *, const int64_t *, int64_t,
                       int64_t, const void *, const void *, bool, int64_t, int64_t *, void *, void *, uint8_t *,
                       uint8_t *);

// cogroup of N inputs: the same CSR split N ways (cogroup_split, dpk_common.cuh); out_first / out_count are
// input-major [ninputs][G]
__global__ void __launch_bounds__(256)
k_cogroup_count(const int64_t *__restrict__ ids, const int64_t *__restrict__ starts, int64_t G,
                const int64_t *__restrict__ bounds, int32_t ninputs, int64_t *__restrict__ out_first,
                int64_t *__restrict__ out_count) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const int64_t s = starts[g];
    cogroup_split(ids, s, starts[g + 1] - s, bounds, ninputs, out_first + g, out_count + g, G);
}

// one input's value runs, load-balanced over its output rows like k_join_emit
template <int W>
__global__ void __launch_bounds__(JN_THREADS)
k_cogroup_emit(const int64_t *__restrict__ ids, const int64_t *__restrict__ first, const int64_t *__restrict__ out_off,
               int64_t G, int64_t id_base, const void *__restrict__ vals, int64_t n_out, void *__restrict__ out_vals) {
    typedef typename ValWord<W>::T T;
    __shared__ int64_t s_off[JN_TILE + 1];
    __shared__ int64_t s_g[2];
    const EmitTile tile = emit_tile(out_off, G, n_out, s_off, s_g);
#pragma unroll 2
    for (int it = 0; it < JN_ITEMS; it++) {
        const int64_t i = tile.i0 + (int64_t)it * JN_THREADS + threadIdx.x;
        if (i > tile.i_last) break;
        int64_t g, base;
        tile.locate(i, &g, &base);
        static_cast<T *>(out_vals)[i] = static_cast<const T *>(vals)[cogroup_source(ids, first[g], base, i, id_base)];
    }
}

// innerJoin: the small side's G distinct keys in a hash table (BcastSlot, dpk_common.cuh), every big row probed in place
__global__ void __launch_bounds__(256)
k_bcast_build(const int64_t *__restrict__ gkeys, int64_t G, BcastSlot *__restrict__ table, uint64_t mask) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    bcast_insert(table, mask, (uint64_t)gkeys[g], (int32_t)g);
}

template <typename K>
__global__ void __launch_bounds__(256)
k_bcast_probe(const K *__restrict__ keys, int64_t n, const BcastSlot *__restrict__ table, uint64_t mask,
              const int64_t *__restrict__ starts, int32_t *__restrict__ out_grp, int64_t *__restrict__ out_count) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    uint64_t kb;
    const int32_t g = bcast_key_bits<K>(keys[r], &kb) ? bcast_find(table, mask, kb) : -1;
    out_grp[r] = g;
    out_count[r] = g < 0 ? 0 : starts[g + 1] - starts[g];
}

// the joined rows, load-balanced over output rows with the join's tile; big row r plays the role of a group: its
// output rows are off[r] .. off[r + 1], one per small row of its key, in ascending small row order (the ids of a
// group-by run ascend).  Six CTAs per SM: 40 registers; left to itself ptxas picks 32 and spills.
template <int KW, int LW, int RW>
__global__ void __launch_bounds__(JN_THREADS, 6)
k_bcast_emit(const void *__restrict__ keys, const void *__restrict__ lvals, const int32_t *__restrict__ grp,
             const int64_t *__restrict__ off, int64_t n, const int64_t *__restrict__ starts,
             const int64_t *__restrict__ ids, const void *__restrict__ rvals, int64_t n_out, void *__restrict__ out_keys,
             void *__restrict__ out_left, void *__restrict__ out_right) {
    typedef typename ValWord<KW>::T KT;
    typedef typename ValWord<LW>::T LT;
    typedef typename ValWord<RW>::T RT;
    __shared__ int64_t s_off[JN_TILE + 1];
    __shared__ int64_t s_g[2];
    const EmitTile tile = emit_tile(off, n, n_out, s_off, s_g);
#pragma unroll 2
    for (int it = 0; it < JN_ITEMS; it++) {
        const int64_t i = tile.i0 + (int64_t)it * JN_THREADS + threadIdx.x;
        if (i > tile.i_last) break;
        int64_t r, base;
        tile.locate(i, &r, &base);
        static_cast<KT *>(out_keys)[i] = static_cast<const KT *>(keys)[r];
        static_cast<LT *>(out_left)[i] = static_cast<const LT *>(lvals)[r];
        static_cast<RT *>(out_right)[i] = static_cast<const RT *>(rvals)[ids[starts[grp[r]] + i - base]];
    }
}

typedef void (*BcastEmitFn)(const void *, const void *, const int32_t *, const int64_t *, int64_t, const int64_t *,
                            const int64_t *, const void *, int64_t, void *, void *, void *);

}  // namespace dpk

using namespace dpk;

extern "C" {

int dpk_join_count(const int64_t *ids, const int64_t *group_starts, int64_t ngroups, int64_t nL, int32_t keep_left,
                   int32_t keep_right, int64_t *out_nl, int64_t *out_count, dpk_stream_t stream) {
    if (ngroups < 0 || nL < 0) return fail(DPK_ERR_INVALID, "ngroups=%lld nL=%lld", (long long)ngroups, (long long)nL);
    if (ngroups == 0) return DPK_OK;
    if (!ids || !group_starts || !out_nl || !out_count) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t blocks = (ngroups + 255) / 256;
    DPK_LAUNCH("join_count", st, k_join_count<<<(unsigned)blocks, 256, 0, st>>>(
        ids, group_starts, ngroups, nL, keep_left != 0, keep_right != 0, out_nl, out_count));
    return DPK_OK;
}

int dpk_join_emit(const int64_t *group_keys, const int64_t *group_starts, const int64_t *ids, const int64_t *nl,
                  const int64_t *out_off, int64_t ngroups, int64_t nL, const void *lvals, int32_t lval_bytes,
                  const void *rvals, int32_t rval_bytes, int32_t keep_left, int32_t keep_right, int64_t n_out,
                  int64_t *out_keys, void *out_left, void *out_right, uint8_t *out_lvalid, uint8_t *out_rvalid,
                  dpk_stream_t stream) {
    if (ngroups < 0 || nL < 0 || n_out < 0)
        return fail(DPK_ERR_INVALID, "ngroups=%lld nL=%lld n_out=%lld", (long long)ngroups, (long long)nL,
                    (long long)n_out);
    if ((lval_bytes != 4 && lval_bytes != 8) || (rval_bytes != 4 && rval_bytes != 8))
        return fail(DPK_ERR_UNSUPPORTED, "value widths %d / %d bytes (4 or 8)", lval_bytes, rval_bytes);
    if (n_out == 0) return DPK_OK;
    // lvals / rvals are read only at rows of a side that has them: an empty column may be NULL (an inner join with
    // output rows has rows on both sides)
    if (!group_keys || !group_starts || !ids || !nl || !out_off || !out_keys || !out_left || !out_right)
        return fail(DPK_ERR_INVALID, "NULL pointer");
    if ((!lvals && nL > 0) || (!rvals && !keep_right && !keep_left))
        return fail(DPK_ERR_INVALID, "NULL value column");
    if ((keep_right && !out_lvalid) || (keep_left && !out_rvalid))
        return fail(DPK_ERR_INVALID, "a side that can be missing needs its valid column");
    if (ngroups == 0) return fail(DPK_ERR_INVALID, "n_out=%lld rows from no group", (long long)n_out);
    static const EmitFn fns[2][2] = {{k_join_emit<4, 4>, k_join_emit<4, 8>}, {k_join_emit<8, 4>, k_join_emit<8, 8>}};
    const EmitFn fn = fns[lval_bytes == 8][rval_bytes == 8];
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t blocks = (n_out + JN_TILE - 1) / JN_TILE;
    DPK_LAUNCH("join_emit", st, fn<<<(unsigned)blocks, JN_THREADS, 0, st>>>(
        group_keys, group_starts, ids, nl, out_off, ngroups, nL, lvals, rvals, keep_left != 0, n_out, out_keys,
        out_left, out_right, keep_right ? out_lvalid : nullptr, keep_left ? out_rvalid : nullptr));
    return DPK_OK;
}

int dpk_cogroup_count(const int64_t *ids, const int64_t *group_starts, int64_t ngroups, const int64_t *bounds,
                      int32_t ninputs, int64_t *out_first, int64_t *out_count, dpk_stream_t stream) {
    if (ngroups < 0 || ninputs < 1)
        return fail(DPK_ERR_INVALID, "ngroups=%lld ninputs=%d", (long long)ngroups, (int)ninputs);
    if (ngroups == 0) return DPK_OK;
    if (!ids || !group_starts || !bounds || !out_first || !out_count) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t blocks = (ngroups + 255) / 256;
    DPK_LAUNCH("cogroup_count", st, k_cogroup_count<<<(unsigned)blocks, 256, 0, st>>>(
        ids, group_starts, ngroups, bounds, ninputs, out_first, out_count));
    return DPK_OK;
}

int dpk_cogroup_emit(const int64_t *ids, const int64_t *first, const int64_t *out_off, int64_t ngroups, int64_t id_base,
                     const void *vals, int32_t val_bytes, int64_t n_out, void *out_vals, dpk_stream_t stream) {
    if (ngroups < 0 || id_base < 0 || n_out < 0)
        return fail(DPK_ERR_INVALID, "ngroups=%lld id_base=%lld n_out=%lld", (long long)ngroups, (long long)id_base,
                    (long long)n_out);
    if (val_bytes != 4 && val_bytes != 8) return fail(DPK_ERR_UNSUPPORTED, "value width %d bytes (4 or 8)", val_bytes);
    if (n_out == 0) return DPK_OK;
    if (!ids || !first || !out_off || !vals || !out_vals) return fail(DPK_ERR_INVALID, "NULL pointer");
    if (ngroups == 0) return fail(DPK_ERR_INVALID, "n_out=%lld rows from no group", (long long)n_out);
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t blocks = (n_out + JN_TILE - 1) / JN_TILE;
    if (val_bytes == 8)
        DPK_LAUNCH("cogroup_emit", st, k_cogroup_emit<8><<<(unsigned)blocks, JN_THREADS, 0, st>>>(
            ids, first, out_off, ngroups, id_base, vals, n_out, out_vals));
    else
        DPK_LAUNCH("cogroup_emit", st, k_cogroup_emit<4><<<(unsigned)blocks, JN_THREADS, 0, st>>>(
            ids, first, out_off, ngroups, id_base, vals, n_out, out_vals));
    return DPK_OK;
}

int dpk_bcast_build(const int64_t *group_keys, int64_t ngroups, void *table, int64_t nslots, dpk_stream_t stream) {
    if (ngroups < 0 || ngroups > INT32_MAX || nslots != (int64_t)bcast_slots(ngroups))
        return fail(DPK_ERR_INVALID, "ngroups=%lld nslots=%lld (want %llu)", (long long)ngroups, (long long)nslots,
                    (unsigned long long)bcast_slots(ngroups < 0 ? 0 : ngroups));
    if (ngroups == 0) return DPK_OK;
    if (!group_keys || !table) return fail(DPK_ERR_INVALID, "NULL pointer");
    if ((uintptr_t)table % sizeof(BcastSlot)) return fail(DPK_ERR_INVALID, "table not 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t blocks = (ngroups + 255) / 256;
    DPK_LAUNCH("bcast_build", st, k_bcast_build<<<(unsigned)blocks, 256, 0, st>>>(
        group_keys, ngroups, static_cast<BcastSlot *>(table), (uint64_t)nslots - 1));
    return DPK_OK;
}

int dpk_bcast_probe(const void *keys, int32_t key_kind, int64_t n, const void *table, int64_t nslots,
                    const int64_t *group_starts, int32_t *out_grp, int64_t *out_count, dpk_stream_t stream) {
    if (n < 0 || nslots < 2 || (nslots & (nslots - 1)))
        return fail(DPK_ERR_INVALID, "n=%lld nslots=%lld (a power of two >= 2)", (long long)n, (long long)nslots);
    if (key_kind != DPK_K_I64 && key_kind != DPK_K_I32 && key_kind != DPK_K_F64 && key_kind != DPK_K_F32)
        return fail(DPK_ERR_UNSUPPORTED, "key kind %d", (int)key_kind);
    if (n == 0) return DPK_OK;
    if (!keys || !table || !group_starts || !out_grp || !out_count) return fail(DPK_ERR_INVALID, "NULL pointer");
    if ((uintptr_t)table % sizeof(BcastSlot)) return fail(DPK_ERR_INVALID, "table not 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    const BcastSlot *t = static_cast<const BcastSlot *>(table);
    const uint64_t mask = (uint64_t)nslots - 1;
    switch (key_kind) {
    case DPK_K_I64:
        DPK_LAUNCH("bcast_probe", st, k_bcast_probe<int64_t><<<blocks, 256, 0, st>>>(
            static_cast<const int64_t *>(keys), n, t, mask, group_starts, out_grp, out_count));
        break;
    case DPK_K_I32:
        DPK_LAUNCH("bcast_probe", st, k_bcast_probe<int32_t><<<blocks, 256, 0, st>>>(
            static_cast<const int32_t *>(keys), n, t, mask, group_starts, out_grp, out_count));
        break;
    case DPK_K_F64:
        DPK_LAUNCH("bcast_probe", st, k_bcast_probe<double><<<blocks, 256, 0, st>>>(
            static_cast<const double *>(keys), n, t, mask, group_starts, out_grp, out_count));
        break;
    default:
        DPK_LAUNCH("bcast_probe", st, k_bcast_probe<float><<<blocks, 256, 0, st>>>(
            static_cast<const float *>(keys), n, t, mask, group_starts, out_grp, out_count));
    }
    return DPK_OK;
}

int dpk_bcast_emit(const void *keys, int32_t key_bytes, const void *lvals, int32_t lval_bytes, const int32_t *grp,
                   const int64_t *out_off, int64_t n, const int64_t *group_starts, const int64_t *ids,
                   const void *rvals, int32_t rval_bytes, int64_t n_out, void *out_keys, void *out_left,
                   void *out_right, dpk_stream_t stream) {
    if (n < 0 || n_out < 0) return fail(DPK_ERR_INVALID, "n=%lld n_out=%lld", (long long)n, (long long)n_out);
    if ((key_bytes != 4 && key_bytes != 8) || (lval_bytes != 4 && lval_bytes != 8) ||
        (rval_bytes != 4 && rval_bytes != 8))
        return fail(DPK_ERR_UNSUPPORTED, "widths %d / %d / %d bytes (4 or 8)", key_bytes, lval_bytes, rval_bytes);
    if (n_out == 0) return DPK_OK;
    if (n == 0) return fail(DPK_ERR_INVALID, "n_out=%lld rows from no big row", (long long)n_out);
    if (!keys || !lvals || !grp || !out_off || !group_starts || !ids || !rvals || !out_keys || !out_left || !out_right)
        return fail(DPK_ERR_INVALID, "NULL pointer");
    static const BcastEmitFn fns[2][2][2] = {
        {{k_bcast_emit<4, 4, 4>, k_bcast_emit<4, 4, 8>}, {k_bcast_emit<4, 8, 4>, k_bcast_emit<4, 8, 8>}},
        {{k_bcast_emit<8, 4, 4>, k_bcast_emit<8, 4, 8>}, {k_bcast_emit<8, 8, 4>, k_bcast_emit<8, 8, 8>}}};
    const BcastEmitFn fn = fns[key_bytes == 8][lval_bytes == 8][rval_bytes == 8];
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t blocks = (n_out + JN_TILE - 1) / JN_TILE;
    DPK_LAUNCH("bcast_emit", st, fn<<<(unsigned)blocks, JN_THREADS, 0, st>>>(
        keys, lvals, grp, out_off, n, group_starts, ids, rvals, n_out, out_keys, out_left, out_right));
    return DPK_OK;
}

}  // extern "C"
