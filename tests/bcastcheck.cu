// tests/bcastcheck.cu -- runs the innerJoin hash table of dpark_b200/csrc/dpk_common.cuh (the __host__ __device__
// functions dpk_join.cu's build and probe kernels call) on the CPU: key normalisation, slot count, insert and find.
// Test-only; not shipped.
#include "dpk_common.cuh"
extern "C" {
uint64_t bc_slots(int64_t G) { return dpk::bcast_slots(G); }
uint64_t bc_slot(uint64_t kb, uint64_t mask) { return dpk::bcast_slot(kb, mask); }
int32_t bc_bits_i32(int32_t k, uint64_t *kb) { return dpk::bcast_key_bits<int32_t>(k, kb) ? 1 : 0; }
int32_t bc_bits_i64(int64_t k, uint64_t *kb) { return dpk::bcast_key_bits<int64_t>(k, kb) ? 1 : 0; }
int32_t bc_bits_f32(float k, uint64_t *kb) { return dpk::bcast_key_bits<float>(k, kb) ? 1 : 0; }
int32_t bc_bits_f64(double k, uint64_t *kb) { return dpk::bcast_key_bits<double>(k, kb) ? 1 : 0; }
int64_t bc_slot_bytes(void) { return sizeof(dpk::BcastSlot); }
// a table of nslots slots for keys[G] (group g = key g), built one key after the other as k_bcast_build's threads do
void bc_build(const uint64_t *keys, int64_t G, void *table, int64_t nslots) {
    memset(table, 0xFF, nslots * sizeof(dpk::BcastSlot));
    for (int64_t g = 0; g < G; g++)
        dpk::bcast_insert(static_cast<dpk::BcastSlot *>(table), (uint64_t)nslots - 1, keys[g], (int32_t)g);
}
int32_t bc_find(const void *table, int64_t nslots, uint64_t kb) {
    return dpk::bcast_find(static_cast<const dpk::BcastSlot *>(table), (uint64_t)nslots - 1, kb);
}
}
