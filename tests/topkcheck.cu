// tests/topkcheck.cu -- runs the topByKey arithmetic of dpark_b200/csrc/dpk_common.cuh (the __host__ __device__
// functions dpk_topk.cu calls) on the CPU: the order key, the length rule of a round and the unit a CTA takes of a run.
// Test-only; not shipped.
#include "dpk_common.cuh"
extern "C" {
uint64_t tc_order_key(uint64_t bits, int32_t width, int32_t is_float, int32_t reverse) {
    return dpk::topk_order_key(bits, width, is_float != 0, reverse != 0);
}
int64_t tc_next_len(int64_t L, int64_t T, int64_t top_n) { return dpk::topk_next_len(L, T, top_n); }
int32_t tc_unit(int64_t s, int64_t e, int64_t w, int64_t T, int64_t *u0, int64_t *u1) {
    return dpk::topk_unit(s, e, w, T, u0, u1) ? 1 : 0;
}
int64_t tc_unit_out(int64_t s, int64_t u0, int64_t out_s, int64_t T, int64_t top_n) {
    return dpk::topk_unit_out(s, u0, out_s, T, top_n);
}
int64_t tc_tile(void) { return DPK_TOPK_TILE; }
int64_t tc_max_n(void) { return DPK_TOPK_MAX_N; }
}
