// dpk_topk.cu -- f4: topByKey (dpark/rdd.py:552-594) of a numeric value column over the CSR of the numeric group-by
// (dpk_group.cu: per key its row ids in (map split, position) order).  Per key the first top_n values of a stable sort
// of its values, in rounds over runs of candidates (round 1: the group-by's runs, candidate i = vals[ids[i]]):
//
//   k_topk_lengths : one thread per run; its length after the round (topk_next_len, dpk_common.cuh).  The host scans
//                    them into the next round's run starts.
//   k_topk_round   : a run longer than T = DPK_TOPK_TILE candidates is cut into chunks of T from its start, a shorter run
//                    is one unit.  CTA w takes the units that START in rows [wT, (w + 1)T) (topk_unit): units of
//                    consecutive runs are adjacent, so that is one range of at most 2T rows.  A hot key spreads over as
//                    many CTAs as it has chunks; many small keys share one CTA.  The range is sorted in shared memory by
//                    (unit, order key, index) with a bitonic network, and every unit's first min(top_n, len) values are
//                    written to its place in the next round (topk_unit_out).
//
// Ties: a unit's candidates leave in (order key, index) order and the units in index order, so among equal order keys
// the index order of every round is the (map split, position) order of the values -- the stable sort's tie-break, with
// no positions carried.  After a round every run that was one unit holds its answer; a run of L > T candidates shrinks
// to topk_next_len(L).  The order key drops the sign of -0.0, so the values themselves are re-read when written.
// Algorithmic bytes of round 1: per row 8 (the id) + W (the value) read; per kept value 8 + W read again and W written.
// A later round reads W per candidate.
#include "dpk_common.cuh"

namespace dpk {

constexpr int TK_THREADS = 512;
constexpr int64_t TK_T = DPK_TOPK_TILE;
constexpr int TK_CAP = 2 * DPK_TOPK_TILE;   // rows one CTA can hold
// order keys | (unit << 16 | index) | per run of the CTA: its unit's first row and first output, relative to the CTA's
constexpr int TK_SMEM = TK_CAP * 8 + TK_CAP * 4 + 2 * (DPK_TOPK_TILE + 1) * 2;
static_assert(TK_CAP <= 65536 && DPK_TOPK_TILE + 1 < 65535, "rows and units of a CTA are 16-bit");
static_assert(DPK_TOPK_MAX_N <= DPK_TOPK_TILE, "a full chunk keeps top_n candidates");

__global__ void __launch_bounds__(256)
k_topk_lengths(const int64_t *__restrict__ runs, int64_t G, int32_t top_n, int64_t *__restrict__ out_len) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    out_len[g] = topk_next_len(runs[g + 1] - runs[g], TK_T, top_n);
}

template <int W>
__device__ __forceinline__ uint64_t tk_load(const int64_t *__restrict__ ids, const void *__restrict__ src, int64_t row) {
    return (uint64_t) static_cast<const typename ValWord<W>::T *>(src)[ids ? ids[row] : row];
}

// (unit, order key, index) order; the unit and the index are the high and low halves of the meta word
__device__ __forceinline__ bool tk_before(uint64_t ka, uint32_t ma, uint64_t kb, uint32_t mb) {
    if ((ma >> 16) != (mb >> 16)) return ma < mb;
    return ka < kb || (ka == kb && ma < mb);
}

template <int W>
__global__ void __launch_bounds__(TK_THREADS, 2)
k_topk_round(const int64_t *__restrict__ ids, const void *__restrict__ src, const int64_t *__restrict__ runs,
             int64_t G, int64_t n, const int64_t *__restrict__ out_runs, int32_t top_n, bool is_float, bool reverse,
             void *__restrict__ out) {
    typedef typename ValWord<W>::T T;
    extern __shared__ __align__(16) unsigned char tk_smem[];
    uint64_t *s_key = reinterpret_cast<uint64_t *>(tk_smem);
    uint32_t *s_meta = reinterpret_cast<uint32_t *>(s_key + TK_CAP);
    uint16_t *s_ustart = reinterpret_cast<uint16_t *>(s_meta + TK_CAP);
    uint16_t *s_uout = s_ustart + TK_T + 1;
    __shared__ int64_t s_g[2], s_rng[3];

    const int64_t w = blockIdx.x, w0 = w * TK_T, w1 = min(w0 + TK_T, n);
    // the runs holding the window's first and last rows; every run between them starts inside the window
    if (threadIdx.x == 0) s_g[0] = group_of(runs, 0, G, w0);
    if (threadIdx.x == 32) s_g[1] = group_of(runs, 0, G, w1 - 1);
    __syncthreads();
    const int64_t g_lo = s_g[0], span = s_g[1] - g_lo + 1;
    if (threadIdx.x == 0) {
        // the CTA's rows [A, B) run from its first unit's start to its last unit's end; O = where the first one writes.
        // Only run g_lo can lack a unit here (its chunk in the window may lie past its end); then g_lo + 1 starts inside.
        int64_t u0, u1, j = 0;
        if (!topk_unit(runs[g_lo], runs[g_lo + 1], w, TK_T, &u0, &u1)) j = 1;
        if (j == 1 && span == 1) {
            s_rng[0] = -1;
        } else {
            if (j == 1) topk_unit(runs[g_lo + 1], runs[g_lo + 2], w, TK_T, &u0, &u1);
            s_rng[0] = u0;
            s_rng[2] = topk_unit_out(runs[g_lo + j], u0, out_runs[g_lo + j], TK_T, top_n);
            topk_unit(runs[g_lo + span - 1], runs[g_lo + span], w, TK_T, &u0, &u1);
            s_rng[1] = u1;
        }
    }
    __syncthreads();
    const int64_t A = s_rng[0];
    if (A < 0) return;
    const int64_t O = s_rng[2];
    const int len = (int)(s_rng[1] - A);
    for (int64_t j = threadIdx.x; j < span; j += TK_THREADS) {
        const int64_t g = g_lo + j, s = runs[g];
        int64_t u0, u1;
        if (topk_unit(s, runs[g + 1], w, TK_T, &u0, &u1)) {
            s_ustart[j] = (uint16_t)(u0 - A);
            s_uout[j] = (uint16_t)(topk_unit_out(s, u0, out_runs[g], TK_T, top_n) - O);
        } else {
            s_ustart[j] = 0;      // run g_lo without a unit: no row is looked up as its row
        }
    }
    __syncthreads();
    int np = 1;
    while (np < len) np <<= 1;
    for (int i = threadIdx.x; i < np; i += TK_THREADS) {
        if (i < len) {
            int lo = 0, hi = (int)span;      // the unit of row i: the last one starting at or before it
            while (hi - lo > 1) {
                const int mid = (lo + hi) >> 1;
                if (s_ustart[mid] <= i) lo = mid; else hi = mid;
            }
            s_key[i] = topk_order_key(tk_load<W>(ids, src, A + i), W, is_float, reverse);
            s_meta[i] = ((uint32_t)lo << 16) | (uint32_t)i;
        } else {
            s_key[i] = ~0ull;                // padding sorts after every unit
            s_meta[i] = 0xFFFFFFFFu;
        }
    }
    __syncthreads();
    for (int k = 2; k <= np; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < (np >> 1); t += TK_THREADS) {
                const int a = ((t & ~(j - 1)) << 1) | (t & (j - 1)), b = a + j;
                const uint64_t ka = s_key[a], kb = s_key[b];
                const uint32_t ma = s_meta[a], mb = s_meta[b];
                if ((a & k) == 0 ? tk_before(kb, mb, ka, ma) : tk_before(ka, ma, kb, mb)) {
                    s_key[a] = kb; s_key[b] = ka;
                    s_meta[a] = mb; s_meta[b] = ma;
                }
            }
            __syncthreads();
        }
    }
    // a unit's rows keep their place as a block: sorted position p is rank p - s_ustart[unit] in its unit
    for (int p = threadIdx.x; p < len; p += TK_THREADS) {
        const uint32_t m = s_meta[p];
        const int j = (int)(m >> 16), r = p - (int)s_ustart[j];
        if (r < top_n) static_cast<T *>(out)[O + s_uout[j] + r] = (T)tk_load<W>(ids, src, A + (int64_t)(m & 0xFFFFu));
    }
}

}  // namespace dpk

using namespace dpk;

extern "C" {

int dpk_topk_lengths(const int64_t *run_starts, int64_t nruns, int32_t top_n, int64_t *out_len, dpk_stream_t stream) {
    if (nruns < 0 || top_n < 1 || top_n > DPK_TOPK_MAX_N)
        return fail(DPK_ERR_INVALID, "nruns=%lld top_n=%d (1..%d)", (long long)nruns, (int)top_n, DPK_TOPK_MAX_N);
    if (nruns == 0) return DPK_OK;
    if (!run_starts || !out_len) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t blocks = (nruns + 255) / 256;
    DPK_LAUNCH("topk_lengths", st, k_topk_lengths<<<(unsigned)blocks, 256, 0, st>>>(run_starts, nruns, top_n, out_len));
    return DPK_OK;
}

int dpk_topk_round(const int64_t *ids, const void *vals, int32_t val_bytes, int32_t val_float,
                   const int64_t *run_starts, int64_t nruns, int64_t n, const int64_t *out_starts, int32_t top_n,
                   int32_t reverse, void *out_vals, dpk_stream_t stream) {
    if (nruns < 0 || n < 0 || top_n < 1 || top_n > DPK_TOPK_MAX_N)
        return fail(DPK_ERR_INVALID, "nruns=%lld n=%lld top_n=%d (1..%d)", (long long)nruns, (long long)n, (int)top_n,
                    DPK_TOPK_MAX_N);
    if (val_bytes != 4 && val_bytes != 8) return fail(DPK_ERR_UNSUPPORTED, "value width %d bytes (4 or 8)", val_bytes);
    if (n == 0) return DPK_OK;
    if (nruns == 0) return fail(DPK_ERR_INVALID, "n=%lld candidates in no run", (long long)n);
    if (!vals || !run_starts || !out_starts || !out_vals) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t blocks = (n + TK_T - 1) / TK_T;
    auto fn = val_bytes == 8 ? k_topk_round<8> : k_topk_round<4>;
    DPK_CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, TK_SMEM));
    DPK_LAUNCH("topk_round", st, fn<<<(unsigned)blocks, TK_THREADS, TK_SMEM, st>>>(
        ids, vals, run_starts, nruns, n, out_starts, top_n, val_float != 0, reverse != 0, out_vals));
    return DPK_OK;
}

}  // extern "C"
