// tests/numparsecheck.cu -- runs the numeric text columns' __host__ __device__ arithmetic (dpark_b200/csrc/dpk_common.cuh
// tc_parse_i64 / tc_parse_f64 / tc_fields / tc_starts16, the per-line step of dpk_strings.cu k_tc_*) on the CPU, so
// that it can be checked against Python's int(), float() and str.split() without a GPU.  Test-only.
#include "dpk_common.cuh"

static const uint64_t POW5[] = {
#include "dpk_pow5.inc"
};

extern "C" {
// the table as compiled, 2 * 651 words
void np_pow5(uint64_t *out) { memcpy(out, POW5, sizeof(POW5)); }

// string i = buf[off[i], off[i + 1]); ok[i] = the device accepts it, out[i] = its int64 value / float64 bits
void np_parse_i64_many(const uint8_t *buf, const int64_t *off, int64_t m, int64_t *out, uint8_t *ok) {
    for (int64_t i = 0; i < m; i++) {
        out[i] = 0;
        ok[i] = dpk::tc_parse_i64(buf, off[i], off[i + 1], &out[i]);
    }
}
void np_parse_f64_many(const uint8_t *buf, const int64_t *off, int64_t m, uint64_t *out, uint8_t *ok) {
    for (int64_t i = 0; i < m; i++) {
        out[i] = 0;
        ok[i] = dpk::tc_parse_f64(buf, off[i], off[i + 1], POW5, &out[i]);
    }
}
// fields k0 and k1 of every line: f[4 i ..] = (b0, e0, b1, e1) relative to the line, ok[i] = enough fields
void np_fields_many(const uint8_t *buf, const int64_t *off, int64_t m, const uint8_t *sep, int32_t sep_len, int32_t k0,
                    int32_t k1, int64_t *f, uint8_t *ok) {
    for (int64_t i = 0; i < m; i++) {
        int64_t g[4] = {0, 0, 0, 0};
        ok[i] = dpk::tc_fields(buf, off[i], off[i + 1], sep, sep_len, k0, k1, g);
        for (int k = 0; k < 4; k++) f[4 * i + k] = ok[i] ? g[k] - off[i] : 0;
    }
}
// k_tc_parse's step for every line: ok[i] = 0 marks a host line
void np_lines_many(const uint8_t *buf, const int64_t *off, int64_t m, const uint8_t *sep, int32_t sep_len, int32_t key,
                   int32_t value, int32_t key_kind, int32_t value_kind, int64_t *k, int64_t *v, uint8_t *ok) {
    for (int64_t i = 0; i < m; i++) {
        k[i] = v[i] = 0;
        ok[i] = dpk::tc_line(buf, off[i], off[i + 1], sep, sep_len, key, value, key_kind, value_kind, POW5, &k[i], &v[i]);
    }
}
// the line starts of data[0, n) as the two kernels find them; returns their number
int64_t np_line_starts(const uint8_t *data, int64_t n, int64_t *starts) {
    int64_t m = 0;
    for (int64_t i0 = 0; i0 < n; i0 += dpk::TK_BYTES) {
        bool hi = false;
        const uint32_t mask = dpk::tc_starts16(data, n, i0, &hi);
        for (int j = 0; j < dpk::TK_BYTES; j++)
            if (mask & (1u << j)) starts[m++] = i0 + j;
    }
    return m;
}
}
