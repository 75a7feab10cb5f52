// tests/sortcheck.cu -- runs the sort arithmetic of dpark_b200/csrc/dpk_common.cuh (the __host__ __device__ functions
// dpk_sort.cu's kernels call) on the CPU: widening, order words and the partition cut (with the two-word compare).
// Test-only; not shipped.
#include "dpk_common.cuh"
extern "C" {
uint64_t sc_wide_bits(const void *col, int32_t kind, int64_t i) { return dpk::sort_wide_bits(col, kind, i); }
int32_t sc_is_nan(uint64_t wide_bits) { return dpk::sort_is_nan(wide_bits) ? 1 : 0; }
uint64_t sc_word(uint64_t wide_bits, int32_t is_float, int32_t reverse) {
    return dpk::sort_word(wide_bits, is_float != 0, reverse != 0);
}
// every partition start as k_sort_cuts computes it: out[0] = 0, out[j] for j = 1 .. L, out[L + 1] = n
void sc_cuts(const uint64_t *w0, const int64_t *ids, const void *vals, int32_t vkind, int64_t n, const uint64_t *bounds0,
             int32_t kind0, const uint64_t *bounds1, int32_t L, int32_t reverse, int64_t *out) {
    out[0] = 0;
    out[L + 1] = n;
    for (int32_t j = 1; j <= L; j++) {
        const int32_t b = dpk::sort_cut_bound(j, L, reverse != 0);
        const uint64_t t0 = dpk::sort_word(bounds0[b], dpk::sort_kind_float(kind0), reverse != 0);
        const uint64_t t1 = bounds1 ? dpk::sort_word(bounds1[b], dpk::sort_kind_float(vkind), reverse != 0) : 0;
        out[j] = dpk::sort_cut(w0, ids, vals, vkind, n, t0, t1, bounds1 ? 2 : 1, reverse != 0);
    }
}
}
