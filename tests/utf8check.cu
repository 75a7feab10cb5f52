// tests/utf8check.cu -- runs the UTF-8 tokeniser's __host__ __device__ arithmetic (dpark_b200/csrc/dpk_common.cuh
// tok8_ws / tok8_seq_ok / tok8_starts16, the per-thread step of dpk_strings.cu k_tok8_count / k_tok8_emit) on the CPU,
// so that it can be checked against Python's str.split() and bytes.decode("utf-8") without a GPU.  Test-only.
#include "dpk_common.cuh"

// one byte range as the two kernels see it: every 16-byte slice's start mask and ill-formed flag, token ends by the
// emit's forward walk; returns the token count, -1 if any slice raised the flag
static int64_t tokenize(const uint8_t *data, int64_t n, int64_t *starts, int64_t *lens) {
    int64_t m = 0;
    bool any_bad = false;
    for (int64_t i0 = 0; i0 < n; i0 += dpk::TK_BYTES) {
        bool bad = false;
        const uint32_t mask = dpk::tok8_starts16(data, n, i0, &bad);
        any_bad |= bad;
        for (int j = 0; j < dpk::TK_BYTES; j++)
            if (mask & (1u << j)) {
                const int64_t b = i0 + j;
                int64_t e = b + 1;
                while (e < n && !dpk::tok8_ws_at(data, n, e)) e++;
                if (starts) {
                    starts[m] = b;
                    lens[m] = e - b;
                }
                m++;
            }
    }
    return any_bad ? -1 : m;
}

extern "C" {
int64_t u8_tokenize(const uint8_t *data, int64_t n, int64_t *starts, int64_t *lens) {
    return tokenize(data, n, starts, lens);
}
// many independent ranges data[begin[i], end[i]) at once: out[i] = u8_tokenize's result for range i
void u8_count_many(const uint8_t *data, const int64_t *begin, const int64_t *end, int64_t m, int64_t *out) {
    for (int64_t i = 0; i < m; i++) out[i] = tokenize(data + begin[i], end[i] - begin[i], nullptr, nullptr);
}
// the whitespace length of the code point at each of the m 3-byte windows c[3 * i ..]
void u8_ws_many(const uint8_t *c, int64_t m, int32_t *out) {
    for (int64_t i = 0; i < m; i++) out[i] = dpk::tok8_ws(c[3 * i], c[3 * i + 1], c[3 * i + 2]);
}
}
