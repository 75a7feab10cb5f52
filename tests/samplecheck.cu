// tests/samplecheck.cu -- runs the MT19937 replay of dpark_b200/csrc/dpk_common.cuh (the __host__ __device__ functions
// dpk_sample.cu's kernel calls) on the CPU, step for step as the kernel takes it: every twist in its three phases, all
// of a phase's elements computed before any is written, then tempering, the draw's double and the keep rule.  Test-only.
#include <vector>

#include "dpk_common.cuh"

namespace {
void twist_phased(uint32_t *mt) {
    uint32_t v[dpk::MT_N];
    for (int p = 0; p < 3; p++) {
        for (int i = dpk::mt_phase(p); i < dpk::mt_phase(p + 1); i++) v[i] = dpk::mt_twist_elem(mt, i);
        for (int i = dpk::mt_phase(p); i < dpk::mt_phase(p + 1); i++) mt[i] = v[i];
    }
}
}  // namespace

extern "C" {
int32_t smc_state_words(void) { return dpk::MT_N; }
int32_t smc_phase(int32_t p) { return dpk::mt_phase(p); }
uint32_t smc_temper(uint32_t y) { return dpk::mt_temper(y); }
double smc_double(uint32_t w0, uint32_t w1) { return dpk::mt_double(w0, w1); }
int32_t smc_keep(double u, double frac) { return dpk::sample_keep(u, frac) ? 1 : 0; }

// the first n tempered words of the generator whose state right after seeding is state[624] (pos = 624)
void smc_words(const uint32_t *state, int64_t n, uint32_t *out) {
    uint32_t mt[dpk::MT_N];
    for (int i = 0; i < dpk::MT_N; i++) mt[i] = state[i];
    for (int64_t j = 0; j < n; j++) {
        const int k = (int)(j % dpk::MT_N);
        if (k == 0) twist_phased(mt);
        out[j] = dpk::mt_temper(mt[k]);
    }
}

// the first n random() draws, and keep[j] = draw j <= frac
void smc_draws(const uint32_t *state, int64_t n, double frac, double *out, uint8_t *keep) {
    std::vector<uint32_t> w(2 * n);
    smc_words(state, 2 * n, w.data());
    for (int64_t j = 0; j < n; j++) {
        out[j] = dpk::mt_double(w[2 * j], w[2 * j + 1]);
        keep[j] = dpk::sample_keep(out[j], frac) ? 1 : 0;
    }
}
}
