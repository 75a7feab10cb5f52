// tests/cogroupcheck.cu -- runs the cogroup arithmetic of dpark_b200/csrc/dpk_common.cuh (the __host__ __device__
// functions dpk_join.cu calls) on the CPU: the N-way split of a group's id run, output row -> group, and output row ->
// the input row it copies.  Test-only; not shipped.
#include "dpk_common.cuh"
extern "C" {
void cc_cogroup_split(const int64_t *ids, int64_t s, int64_t len, const int64_t *bounds, int32_t ninputs,
                      int64_t *first, int64_t *count, int64_t stride) {
    dpk::cogroup_split(ids, s, len, bounds, ninputs, first, count, stride);
}
int64_t cc_group_of(const int64_t *off, int64_t lo, int64_t hi, int64_t i) { return dpk::group_of(off, lo, hi, i); }
int64_t cc_cogroup_source(const int64_t *ids, int64_t first, int64_t base, int64_t r, int64_t id_base) {
    return dpk::cogroup_source(ids, first, base, r, id_base);
}
}
