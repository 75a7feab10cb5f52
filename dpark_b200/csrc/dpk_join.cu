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
#include "dpk_common.cuh"

namespace dpk {

constexpr int JN_THREADS = 256;
constexpr int JN_ITEMS = 8;
constexpr int JN_TILE = JN_THREADS * JN_ITEMS;

template <int W> struct ValWord;
template <> struct ValWord<4> { typedef uint32_t T; };
template <> struct ValWord<8> { typedef uint64_t T; };

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

// the last group g in [lo, hi) with off[g] <= i (off[lo] <= i holds); empty groups share their offset with the next
// group, so the answer always has rows
__device__ __forceinline__ int64_t group_of(const int64_t *off, int64_t lo, int64_t hi, int64_t i) {
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (off[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
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
    const int64_t i0 = (int64_t)blockIdx.x * JN_TILE;
    const int64_t i_last = min(i0 + JN_TILE, n_out) - 1;
    // the groups of the tile's first and last rows
    if (threadIdx.x == 0) s_g[0] = group_of(out_off, 0, G, i0);
    if (threadIdx.x == 32) s_g[1] = group_of(out_off, 0, G, i_last);
    __syncthreads();
    const int64_t g0 = s_g[0], span = s_g[1] - g0 + 1;
    // a tile's rows belong to at most JN_TILE groups with rows, but empty groups between them also lie in
    // [g0, g1]: the offsets are staged in shared memory when they fit, searched in place otherwise
    const bool staged = span <= JN_TILE;
    if (staged)
        for (int64_t j = threadIdx.x; j <= span; j += JN_THREADS) s_off[j] = out_off[g0 + j];
    __syncthreads();
#pragma unroll 2
    for (int it = 0; it < JN_ITEMS; it++) {
        const int64_t i = i0 + (int64_t)it * JN_THREADS + threadIdx.x;
        if (i > i_last) break;
        int64_t g, base;
        if (staged) {
            const int64_t j = group_of(s_off, 0, span, i);
            g = g0 + j;
            base = s_off[j];
        } else {
            g = group_of(out_off, g0, g0 + span, i);
            base = out_off[g];
        }
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

}  // extern "C"
