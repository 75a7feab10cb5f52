// tests/joincheck.cu -- runs the join arithmetic of dpark_b200/csrc/dpk_common.cuh (the __host__ __device__ functions
// dpk_join.cu calls) on the CPU: the left rows of an id run, the rows of a key, output row -> (left row, right row).
// Test-only; not shipped.
#include "dpk_common.cuh"
extern "C" {
int64_t jc_join_left_rows(const int64_t *run, int64_t len, int64_t nL) { return dpk::join_left_rows(run, len, nL); }
int64_t jc_join_count(int64_t nl, int64_t nr, int keep_left, int keep_right) {
    return dpk::join_count(nl, nr, keep_left != 0, keep_right != 0);
}
void jc_join_pair(int64_t i, int64_t nr, int keep_left, int64_t *a, int64_t *b) {
    dpk::join_pair(i, nr, keep_left != 0, a, b);
}
}
