// dpk_tdigest.cu -- f7: percentilesByKey (dpark/rdd.py:815-850) of a numeric value column over the CSR of the numeric
// group-by (dpk_group.cu: per key its row ids in (map split, position) order).  The composition builds, per key and map
// split, MergingDigest().update(values) + compress(), and absorbs those digests into the key's first one in split
// order; the kernels build the same digests with the same arithmetic (td_*, dpk_common.cuh):
//
//   k_td_heads       : one thread per row: a row whose split (id / per) differs from its predecessor's, or that starts a
//                      group, starts a segment -- one (key, split) digest.  The host compacts the heads into the segment
//                      starts and scans min(L, TD_CAP) per segment into the compacted centroid scratch.
//   k_td_build_short : one thread per segment of L <= TD_SHORT values: one fold, the buffer insertion-sorted in place in
//                      its scratch.  A longer segment is appended to a device work list.
//   k_td_build_long  : one warp per listed segment, fetched from a device counter: the add path's folds in shared
//                      memory, TD_CAP - C values at a time (C = the centroids so far).  A fold is a stable bitonic sort of
//                      the buffer, a merge with the centroids (ties: the buffer first) by two binary searches per entry,
//                      one lane's pass over the weights that decides which entries open a centroid, and the centroids'
//                      means, one lane per centroid.
//   k_td_merge       : one warp per key: its first segment's digest, then absorb of every further one (a merge of two
//                      sorted lists, ties: the incoming digest first, and one fold), then quantile(q) for every q, one lane
//                      per q.
//
// A NaN value, a NaN or falling centroid mean, or a fold longer than TD_STAGE entries sets *flag: the host then keeps the
// composition, whose answer (or ValueError) alone stands there.
#include "dpk_common.cuh"

namespace dpk {

constexpr int TD_SHORT = 32;      // longest segment one thread builds
constexpr int TD_SORT = 256;      // the buffer's sort width: the least power of two >= TD_CAP
constexpr int TD_WARPS = 4;       // warps per CTA of k_td_build_long and k_td_merge
static_assert(TD_SHORT <= TD_CAP && TD_SORT >= TD_CAP && TD_STAGE + 1 < 32768, "sizes of the staging");

struct TdWarp {
    double cm[TD_STAGE], cw[TD_STAGE];   // the digest's centroids, ascending means
    double xm[TD_STAGE], xw[TD_STAGE];   // one fold's entries in merged order
    double bv[TD_SORT];                  // the add path's buffer, sorted by (value, position)
    int16_t bi[TD_SORT];
    int16_t cs[TD_STAGE + 2];            // the fold's centroid starts
};
constexpr int TD_SMEM = TD_WARPS * (int)sizeof(TdWarp);

__global__ void __launch_bounds__(256)
k_td_heads(const int64_t *__restrict__ ids, int64_t n, const int64_t *__restrict__ gs, int64_t G, int64_t per,
           uint8_t *__restrict__ head) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) {
        if (t > 0 && ids[t] / per != ids[t - 1] / per) head[t] = 1;
    } else if (t < n + G) {
        head[gs[t - n]] = 1;
    }
}

__global__ void __launch_bounds__(256)
k_td_build_short(const int64_t *__restrict__ ids, const void *__restrict__ vals, int32_t kind,
                 const int64_t *__restrict__ ss, const int64_t *__restrict__ so, int64_t S, double *__restrict__ gm,
                 double *__restrict__ gw, int32_t *__restrict__ cnt, double *__restrict__ lohi,
                 unsigned long long *__restrict__ work, int32_t *__restrict__ flag) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const int64_t r0 = ss[s];
    const int L = (int)min(ss[s + 1] - r0, (int64_t)TD_SHORT + 1);
    if (L > TD_SHORT) {
        work[2 + atomicAdd(&work[0], 1ull)] = (unsigned long long)s;
        return;
    }
    double *om = gm + so[s], *ow = gw + so[s];
    bool bad = false;
    for (int i = 0; i < L; i++) {
        const double v = td_value(vals, kind, ids[r0 + i]);
        bad |= v != v;
        om[i] = v;
    }
    td_sort_serial(om, L);
    const int c = td_fold_serial(om, nullptr, L, (double)L, om, ow, &bad);
    cnt[s] = c;
    lohi[2 * s] = om[0];
    lohi[2 * s + 1] = om[c - 1];
    if (bad) atomicOr(flag, 1);
}

// One fold of the n staged entries xm / xw into the centroids cm / cw (*C of them after it); lo / hi as _fold keeps them.
// Returns true (on every lane) when a mean is NaN or falls.
__device__ bool td_warp_fold(TdWarp &w, int n, double total, int lane, int *C, double *lo, double *hi, bool first) {
    int nc = 0;
    if (lane == 0) nc = td_fold_decide(w.xw, n, total, w.cs);
    nc = __shfl_sync(0xFFFFFFFFu, nc, 0);
    __syncwarp();
    for (int c = lane; c < nc; c += 32) td_centroid(w.xm, w.xw, w.cs[c], w.cs[c + 1], &w.cm[c], &w.cw[c]);
    __syncwarp();
    bool ok = true;
    for (int c = lane; c < nc; c += 32) ok &= td_mean_ok(w.cm[c], c ? &w.cm[c - 1] : nullptr);
    *lo = first ? w.cm[0] : td_min(*lo, w.cm[0]);
    *hi = first ? w.cm[nc - 1] : td_max(*hi, w.cm[nc - 1]);
    *C = nc;
    return __any_sync(0xFFFFFFFFu, !ok);
}

__global__ void __launch_bounds__(TD_WARPS * 32)
k_td_build_long(const int64_t *__restrict__ ids, const void *__restrict__ vals, int32_t kind,
                const int64_t *__restrict__ ss, const int64_t *__restrict__ so, double *__restrict__ gm,
                double *__restrict__ gw, int32_t *__restrict__ cnt, double *__restrict__ lohi,
                unsigned long long *__restrict__ work, int32_t *__restrict__ flag) {
    extern __shared__ __align__(16) unsigned char td_smem[];
    TdWarp &w = reinterpret_cast<TdWarp *>(td_smem)[threadIdx.x >> 5];
    const int lane = threadIdx.x & 31;
    const unsigned long long nlong = work[0];
    for (;;) {
        unsigned long long j = 0;
        if (lane == 0) j = atomicAdd(&work[1], 1ull);
        j = __shfl_sync(0xFFFFFFFFu, j, 0);
        if (j >= nlong) return;
        const int64_t s = (int64_t)work[2 + j], r0 = ss[s], L = ss[s + 1] - r0;
        int C = 0;
        double lo = 0.0, hi = 0.0, mw = 0.0;
        bool bad = false;
        for (int64_t pos = 0; pos < L && !bad;) {
            const int B = td_buffer_len(C, L - pos);
            int np = 32;
            while (np < B) np <<= 1;
            bool nan = false;
            for (int t = lane; t < np; t += 32) {
                const double v = t < B ? td_value(vals, kind, ids[r0 + pos + t]) : INFINITY;
                nan |= v != v;
                w.bv[t] = v;
                w.bi[t] = (int16_t)t;          // padding sorts after every value: +inf, and a later position
            }
            if (__any_sync(0xFFFFFFFFu, nan)) { bad = true; break; }
            __syncwarp();
            for (int k = 2; k <= np; k <<= 1) {
                for (int h = k >> 1; h > 0; h >>= 1) {
                    for (int t = lane; t < (np >> 1); t += 32) {
                        const int a = ((t & ~(h - 1)) << 1) | (t & (h - 1)), b = a + h;
                        const double va = w.bv[a], vb = w.bv[b];
                        const int16_t ia = w.bi[a], ib = w.bi[b];
                        const bool b_first = vb < va || (!(va < vb) && ib < ia);
                        if ((a & k) == 0 ? b_first : !b_first) {
                            w.bv[a] = vb; w.bv[b] = va;
                            w.bi[a] = ib; w.bi[b] = ia;
                        }
                    }
                    __syncwarp();
                }
            }
            for (int t = lane; t < B; t += 32) {
                const int p = t + td_count_below(w.cm, C, w.bv[t]);
                w.xm[p] = w.bv[t];
                w.xw[p] = 1.0;
            }
            for (int c = lane; c < C; c += 32) {
                const int p = c + td_count_upto(w.bv, B, w.cm[c]);
                w.xm[p] = w.cm[c];
                w.xw[p] = w.cw[c];
            }
            __syncwarp();
            mw = td_add(mw, (double)B);
            bad = td_warp_fold(w, B + C, mw, lane, &C, &lo, &hi, pos == 0);
            pos += B;
            __syncwarp();
        }
        bad |= C > TD_CAP;
        if (!bad) {
            for (int c = lane; c < C; c += 32) {
                gm[so[s] + c] = w.cm[c];
                gw[so[s] + c] = w.cw[c];
            }
        }
        if (lane == 0) {
            cnt[s] = bad ? 0 : C;
            lohi[2 * s] = lo;
            lohi[2 * s + 1] = hi;
            if (bad) atomicOr(flag, 1);
        }
        __syncwarp();
    }
}

__global__ void __launch_bounds__(TD_WARPS * 32)
k_td_merge(const int64_t *__restrict__ gs, int64_t G, const int64_t *__restrict__ ss, const int64_t *__restrict__ so,
           int64_t S, const int32_t *__restrict__ cnt, const double *__restrict__ lohi, const double *__restrict__ gm,
           const double *__restrict__ gw, const double *__restrict__ qs, int32_t nq, double *__restrict__ out,
           int32_t *__restrict__ flag) {
    extern __shared__ __align__(16) unsigned char td_smem[];
    TdWarp &w = reinterpret_cast<TdWarp *>(td_smem)[threadIdx.x >> 5];
    const int lane = threadIdx.x & 31;
    const int64_t g = (int64_t)blockIdx.x * TD_WARPS + (threadIdx.x >> 5);
    if (g >= G || *(volatile int32_t *)flag) return;       // a segment was not built: the composition stands
    const int64_t s0 = group_of(ss, 0, S + 1, gs[g]), s1 = group_of(ss, 0, S + 1, gs[g + 1]);
    int C = cnt[s0];
    for (int c = lane; c < C; c += 32) {
        w.cm[c] = gm[so[s0] + c];
        w.cw[c] = gw[so[s0] + c];
    }
    double mw = (double)(ss[s0 + 1] - ss[s0]), lo = lohi[2 * s0], hi = lohi[2 * s0 + 1];
    __syncwarp();
    for (int64_t s = s0 + 1; s < s1; s++) {
        const int m = cnt[s];
        if (C + m > TD_STAGE) {
            if (lane == 0) atomicOr(flag, 1);
            return;
        }
        const double *im = gm + so[s], *iw = gw + so[s];
        for (int t = lane; t < m; t += 32) {
            const double x = im[t];
            const int p = t + td_count_below(w.cm, C, x);
            w.xm[p] = x;
            w.xw[p] = iw[t];
        }
        for (int c = lane; c < C; c += 32) {
            const int p = c + td_count_upto(im, m, w.cm[c]);
            w.xm[p] = w.cm[c];
            w.xw[p] = w.cw[c];
        }
        __syncwarp();
        mw = td_add(mw, (double)(ss[s + 1] - ss[s]));
        if (td_warp_fold(w, m + C, mw, lane, &C, &lo, &hi, false)) {
            if (lane == 0) atomicOr(flag, 1);
            return;
        }
        __syncwarp();
    }
    for (int j = lane; j < nq; j += 32) out[g * nq + j] = td_quantile(w.cm, w.cw, C, mw, lo, hi, qs[j]);
}

}  // namespace dpk

using namespace dpk;

extern "C" {

int dpk_tdigest_heads(const int64_t *ids, int64_t n, const int64_t *group_starts, int64_t ngroups, int64_t per,
                      uint8_t *head, dpk_stream_t stream) {
    if (n < 0 || ngroups < 0 || (n > 0 && per < 1))
        return fail(DPK_ERR_INVALID, "n=%lld ngroups=%lld per=%lld", (long long)n, (long long)ngroups, (long long)per);
    if (n == 0) return DPK_OK;
    if (!ids || !group_starts || !head) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t blocks = (n + ngroups + 255) / 256;
    DPK_LAUNCH("tdigest_heads", st, k_td_heads<<<(unsigned)blocks, 256, 0, st>>>(ids, n, group_starts, ngroups, per, head));
    return DPK_OK;
}

int dpk_tdigest_build(const int64_t *ids, const void *vals, int32_t val_kind, const int64_t *seg_starts,
                      const int64_t *seg_off, int64_t nseg, double *cent_m, double *cent_w, int32_t *cent_n,
                      double *lohi, int64_t *work, int32_t *flag, dpk_stream_t stream) {
    if (val_kind != DPK_K_I32 && val_kind != DPK_K_I64 && val_kind != DPK_K_F32 && val_kind != DPK_K_F64)
        return fail(DPK_ERR_UNSUPPORTED, "value kind %d (int32 / int64 / float32 / float64)", val_kind);
    if (nseg < 0) return fail(DPK_ERR_INVALID, "nseg=%lld", (long long)nseg);
    if (nseg == 0) return DPK_OK;
    if (!ids || !vals || !seg_starts || !seg_off || !cent_m || !cent_w || !cent_n || !lohi || !work || !flag)
        return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    unsigned long long *wk = reinterpret_cast<unsigned long long *>(work);
    DPK_CUDA_TRY(cudaMemsetAsync(wk, 0, 2 * sizeof(unsigned long long), st));
    DPK_LAUNCH("tdigest_build_short", st, k_td_build_short<<<(unsigned)((nseg + 255) / 256), 256, 0, st>>>(
        ids, vals, val_kind, seg_starts, seg_off, nseg, cent_m, cent_w, cent_n, lohi, wk, flag));
    DPK_CUDA_TRY(cudaFuncSetAttribute(k_td_build_long, cudaFuncAttributeMaxDynamicSharedMemorySize, TD_SMEM));
    const int64_t ctas = (int64_t)sm_count() * 3;
    DPK_LAUNCH("tdigest_build_long", st, k_td_build_long<<<(unsigned)ctas, TD_WARPS * 32, TD_SMEM, st>>>(
        ids, vals, val_kind, seg_starts, seg_off, cent_m, cent_w, cent_n, lohi, wk, flag));
    return DPK_OK;
}

int dpk_tdigest_merge(const int64_t *group_starts, int64_t ngroups, const int64_t *seg_starts, const int64_t *seg_off,
                      int64_t nseg, const int32_t *cent_n, const double *lohi, const double *cent_m,
                      const double *cent_w, const double *qs, int32_t nq, double *out, int32_t *flag,
                      dpk_stream_t stream) {
    if (ngroups < 0 || nseg < ngroups || nq < 0)
        return fail(DPK_ERR_INVALID, "ngroups=%lld nseg=%lld nq=%d", (long long)ngroups, (long long)nseg, (int)nq);
    if (ngroups == 0) return DPK_OK;
    if (!group_starts || !seg_starts || !seg_off || !cent_n || !lohi || !cent_m || !cent_w || !flag || (nq && (!qs || !out)))
        return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    DPK_CUDA_TRY(cudaFuncSetAttribute(k_td_merge, cudaFuncAttributeMaxDynamicSharedMemorySize, TD_SMEM));
    const int64_t ctas = (ngroups + TD_WARPS - 1) / TD_WARPS;
    DPK_LAUNCH("tdigest_merge", st, k_td_merge<<<(unsigned)ctas, TD_WARPS * 32, TD_SMEM, st>>>(
        group_starts, ngroups, seg_starts, seg_off, nseg, cent_n, lohi, cent_m, cent_w, qs, nq, out, flag));
    return DPK_OK;
}

}  // extern "C"
