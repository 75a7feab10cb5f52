// dpk_sort.cu -- f6: sort (dpark/rdd.py:273-287) of a numeric (k, v) column pair by k, by v or by the tuple (k, v).  The
// rows are sorted once, globally and stably, by 64-bit order words with the group-by's LSD radix passes (dpk_radix_pass);
// the reference's range partitions are then contiguous slices of the sorted rows:
//
//   k_sort_keys   : one pass over the order column(s), each read in its own dtype and widened (ints to int64, floats to
//                   float64): the order word of every row (sort_word, dpk_common.cuh; complemented for reverse), the row
//                   ids 0..n-1, and a flag raised when an order column holds a NaN.
//   k_sort_cuts   : one thread per partition start: a binary search of the bound's words in the sorted words (sort_cut);
//                   the second word of the (k, v) order is recomputed from vals[ids[i]].
//   k_sort_gather : the sorted key and value columns, gathered by id, each in its own width (bits preserved).
//
// Algorithmic bytes: keys pass K (+ V) read, 8 per word + 8 (id) written; gather 8 (id) + K + V read, K + V written per
// row; cuts (P - 1) log2(n) words read, not credited.
#include "dpk_common.cuh"

namespace dpk {

constexpr int SO_THREADS = 256;

__global__ void __launch_bounds__(SO_THREADS)
k_sort_keys(const void *__restrict__ col0, int32_t kind0, const void *__restrict__ col1, int32_t kind1, int64_t n,
            bool reverse, int64_t *__restrict__ w0, int64_t *__restrict__ w1, int64_t *__restrict__ ids,
            int32_t *__restrict__ nan_flag) {
    const bool f0 = sort_kind_float(kind0), f1 = sort_kind_float(kind1);
    bool nan = false;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint64_t b0 = sort_wide_bits(col0, kind0, i);
        nan |= f0 && sort_is_nan(b0);
        w0[i] = (int64_t)sort_word(b0, f0, reverse);
        if (col1) {
            const uint64_t b1 = sort_wide_bits(col1, kind1, i);
            nan |= f1 && sort_is_nan(b1);
            w1[i] = (int64_t)sort_word(b1, f1, reverse);
        }
        ids[i] = i;
    }
    if (__syncthreads_or(nan) && threadIdx.x == 0) *nan_flag = 1;
}

__global__ void __launch_bounds__(SO_THREADS)
k_sort_cuts(const uint64_t *__restrict__ w0, const int64_t *__restrict__ ids, const void *__restrict__ vals,
            int32_t vkind, int64_t n, const uint64_t *__restrict__ bounds0, int32_t kind0,
            const uint64_t *__restrict__ bounds1, int32_t nbounds, bool reverse, int64_t *__restrict__ out_starts) {
    const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j > nbounds + 1) return;
    if (j == 0) { out_starts[0] = 0; return; }
    if (j == nbounds + 1) { out_starts[j] = n; return; }
    const int32_t b = sort_cut_bound(j, nbounds, reverse);
    const uint64_t t0 = sort_word(bounds0[b], sort_kind_float(kind0), reverse);
    const uint64_t t1 = bounds1 ? sort_word(bounds1[b], sort_kind_float(vkind), reverse) : 0;
    out_starts[j] = sort_cut(w0, ids, vals, vkind, n, t0, t1, bounds1 ? 2 : 1, reverse);
}

template <int KW, int VW>
__global__ void __launch_bounds__(SO_THREADS)
k_sort_gather(const void *__restrict__ keys, const void *__restrict__ vals, const int64_t *__restrict__ ids, int64_t n,
              void *__restrict__ out_keys, void *__restrict__ out_vals) {
    typedef typename ValWord<KW>::T K;
    typedef typename ValWord<VW>::T V;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int64_t r = ids[i];
        static_cast<K *>(out_keys)[i] = static_cast<const K *>(keys)[r];
        static_cast<V *>(out_vals)[i] = static_cast<const V *>(vals)[r];
    }
}

static bool so_kind_ok(int32_t kind) {
    return kind == DPK_K_I64 || kind == DPK_K_I32 || kind == DPK_K_F64 || kind == DPK_K_F32;
}

static unsigned so_blocks(int64_t n) {
    int64_t g = (n + SO_THREADS - 1) / SO_THREADS;
    const int64_t cap = (int64_t)sm_count() * 16;
    return (unsigned)(g > cap ? cap : g);
}

}  // namespace dpk

using namespace dpk;

extern "C" {

int dpk_sort_keys(const void *col0, int32_t kind0, const void *col1, int32_t kind1, int64_t n, int32_t reverse,
                  int64_t *out_w0, int64_t *out_w1, int64_t *out_ids, int32_t *nan_flag, dpk_stream_t stream) {
    if (n < 0 || n >= (1ll << 31)) return fail(DPK_ERR_INVALID, "n=%lld (0 .. 2^31 - 1)", (long long)n);
    if (!so_kind_ok(kind0) || (col1 && !so_kind_ok(kind1)))
        return fail(DPK_ERR_UNSUPPORTED, "column kinds %d, %d (int32 / int64 / float32 / float64)", kind0, kind1);
    if (n == 0) return DPK_OK;
    if (!col0 || !out_w0 || !out_ids || !nan_flag || (col1 && !out_w1)) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    DPK_LAUNCH("sort_keys", st, k_sort_keys<<<so_blocks(n), SO_THREADS, 0, st>>>(
        col0, kind0, col1, kind1, n, reverse != 0, out_w0, col1 ? out_w1 : nullptr, out_ids, nan_flag));
    return DPK_OK;
}

int dpk_sort_cuts(const int64_t *sorted_w0, const int64_t *ids, const void *vals, int32_t val_kind, int64_t n,
                  const int64_t *bounds0, int32_t kind0, const int64_t *bounds1, int32_t nbounds, int32_t reverse,
                  int64_t *out_starts, dpk_stream_t stream) {
    if (n < 0 || nbounds < 0 || nbounds >= (1 << 30))
        return fail(DPK_ERR_INVALID, "n=%lld nbounds=%d", (long long)n, (int)nbounds);
    if (!so_kind_ok(kind0) || (bounds1 && !so_kind_ok(val_kind)))
        return fail(DPK_ERR_UNSUPPORTED, "column kinds %d, %d (int32 / int64 / float32 / float64)", kind0, val_kind);
    if (!out_starts || (n && !sorted_w0) || (nbounds && !bounds0) || (bounds1 && n && (!ids || !vals)))
        return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t T = (int64_t)nbounds + 2;
    DPK_LAUNCH("sort_cuts", st, k_sort_cuts<<<(unsigned)((T + SO_THREADS - 1) / SO_THREADS), SO_THREADS, 0, st>>>(
        (const uint64_t *)sorted_w0, ids, vals, val_kind, n, (const uint64_t *)bounds0, kind0,
        (const uint64_t *)bounds1, nbounds, reverse != 0, out_starts));
    return DPK_OK;
}

int dpk_sort_gather(const void *keys, int32_t key_bytes, const void *vals, int32_t val_bytes, const int64_t *ids,
                    int64_t n, void *out_keys, void *out_vals, dpk_stream_t stream) {
    if (n < 0) return fail(DPK_ERR_INVALID, "n < 0");
    if ((key_bytes != 4 && key_bytes != 8) || (val_bytes != 4 && val_bytes != 8))
        return fail(DPK_ERR_UNSUPPORTED, "widths %d, %d bytes (4 or 8)", key_bytes, val_bytes);
    if (n == 0) return DPK_OK;
    if (!keys || !vals || !ids || !out_keys || !out_vals) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    auto fn = key_bytes == 8 ? (val_bytes == 8 ? k_sort_gather<8, 8> : k_sort_gather<8, 4>)
                             : (val_bytes == 8 ? k_sort_gather<4, 8> : k_sort_gather<4, 4>);
    DPK_LAUNCH("sort_gather", st, fn<<<so_blocks(n), SO_THREADS, 0, st>>>(keys, vals, ids, n, out_keys, out_vals));
    return DPK_OK;
}

}  // extern "C"
