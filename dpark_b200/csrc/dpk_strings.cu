// dpk_strings.cu -- key identity for variable-length keys (str / bytes).
// The reference's per-bucket dicts (dpark/task.py:221-226) and merge dict
// (dpark/shuffle.py:600-608) compare keys by VALUE.  On the device a row's key is
// (data, offsets[i]..offsets[i+1]); k_dict_encode maps every row to the index of a
// representative row with the same bytes, so the fixed-width machinery (partition,
// combine) can run on int64 ids without ever trusting the 64-bit hash as identity.
#include "dpk_common.cuh"

namespace dpk {

__global__ void __launch_bounds__(256)
k_dict_encode(const uint8_t *__restrict__ data, const int64_t *__restrict__ offsets,
              const int64_t *__restrict__ hash, int64_t n, long long *__restrict__ table, uint64_t mask,
              int64_t *__restrict__ rep) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        const int64_t h = hash[i];
        const int64_t b0 = offsets[i];
        const int64_t len = offsets[i + 1] - b0;
        uint64_t slot = mix64((uint64_t)h) & mask;
        int64_t r = i;
        for (;;) {
            long long cur = __ldcg(&table[slot]);
            if (cur < 0) {
                long long prev = (long long)atomicCAS((unsigned long long *)&table[slot], (unsigned long long)-1ll,
                                                      (unsigned long long)i);
                if (prev == -1ll) break;  // this row is the representative
                cur = prev;
            }
            if (hash[cur] == h) {
                const int64_t b1 = offsets[cur];
                if (offsets[cur + 1] - b1 == len) {
                    int64_t j = 0;
                    while (j < len && data[b0 + j] == data[b1 + j]) j++;
                    if (j == len) { r = cur; break; }
                }
            }
            slot = (slot + 1) & mask;
        }
        rep[i] = r;
    }
}

// ---- device text ingest -------------------------------------------------------------------------------------------
// TextFileRDD (dpark/rdd.py:1633-1711) hands out lines, and examples/wc.py splits each with `x.strip().split()`: for
// ASCII text the tokens of a byte range that starts and ends on line boundaries are exactly its maximal runs of
// non-whitespace bytes (newlines are whitespace; str.split() without arguments splits on ' ', \t \n \v \f \r and
// \x1c..\x1f).  Two passes over the bytes: count the token starts per 4096-byte block, then -- after the host-side scan
// of the block counts -- write (start, length) of every token in text order.  A byte >= 0x80 raises `flags` bit 0: the
// caller then leaves the split to the row-wise path (Unicode whitespace and decoding errors are Python's business).
constexpr int TK_THREADS = 256;   // TK_BYTES (16 bytes per thread): dpk_common.cuh
constexpr int TK_CHUNK = TK_THREADS * TK_BYTES;

// tok_ws / tok_starts16 (the per-thread token-start mask) live in dpk_common.cuh: __host__ __device__, so that
// tests/hostcheck.cu can run the same arithmetic on the CPU against Python's str.split()

__global__ void __launch_bounds__(TK_THREADS)
k_tok_count(const uint8_t *__restrict__ data, int64_t n, int64_t *__restrict__ block_counts, unsigned long long *__restrict__ flags) {
    __shared__ int s_w[TK_THREADS / 32];
    const int64_t i0 = ((int64_t)blockIdx.x * TK_THREADS + threadIdx.x) * TK_BYTES;
    bool hi = false;
    const uint32_t m = i0 < n ? tok_starts16(data, n, i0, &hi) : 0u;
    int c = __popc(m);
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = c;
    if (__any_sync(0xffffffffu, hi) && (threadIdx.x & 31) == 0) atomicOr(flags, 1ull);
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < TK_THREADS / 32; w++) t += s_w[w];
        block_counts[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(TK_THREADS)
k_tok_emit(const uint8_t *__restrict__ data, int64_t n, const int64_t *__restrict__ block_base, int64_t *__restrict__ starts,
           int64_t *__restrict__ lens) {
    __shared__ int s_w[TK_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t i0 = ((int64_t)blockIdx.x * TK_THREADS + threadIdx.x) * TK_BYTES;
    bool hi = false;
    uint32_t m = i0 < n ? tok_starts16(data, n, i0, &hi) : 0u;
    const int c = __popc(m);
    int incl = c;
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    int before = 0;
    for (int w = 0; w < warp; w++) before += s_w[w];
    int64_t r = block_base[blockIdx.x] + before + incl - c;
    while (m) {
        const int j = __ffs(m) - 1;
        m &= m - 1;
        const int64_t b = i0 + j;
        int64_t e = b + 1;
        while (e < n && !tok_ws(data[e])) e++;
        starts[r] = b;
        lens[r] = e - b;
        r++;
    }
}

// The same two passes for UTF-8 text (the ranges the ASCII pair declines): TextFileRDD decodes every line with strict
// utf-8, so a range is either well-formed as a whole ('\n' never occurs inside a multi-byte sequence) or the row-wise
// path raises UnicodeDecodeError; whitespace is every code point str.isspace() accepts, 1 to 3 bytes long.
// tok8_starts16 (dpk_common.cuh) classifies the lead bytes of a 16-byte slice and checks their sequences; any
// ill-formed byte raises `flags` bit 0, and the caller then runs no emit.  The emit walks each token to the lead byte of
// the next whitespace code point.
__global__ void __launch_bounds__(TK_THREADS)
k_tok8_count(const uint8_t *__restrict__ data, int64_t n, int64_t *__restrict__ block_counts, unsigned long long *__restrict__ flags) {
    __shared__ int s_w[TK_THREADS / 32];
    const int64_t i0 = ((int64_t)blockIdx.x * TK_THREADS + threadIdx.x) * TK_BYTES;
    bool bad = false;
    const uint32_t m = i0 < n ? tok8_starts16(data, n, i0, &bad) : 0u;
    int c = __popc(m);
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = c;
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(flags, 1ull);
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < TK_THREADS / 32; w++) t += s_w[w];
        block_counts[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(TK_THREADS)
k_tok8_emit(const uint8_t *__restrict__ data, int64_t n, const int64_t *__restrict__ block_base, int64_t *__restrict__ starts,
            int64_t *__restrict__ lens) {
    __shared__ int s_w[TK_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t i0 = ((int64_t)blockIdx.x * TK_THREADS + threadIdx.x) * TK_BYTES;
    bool bad = false;
    uint32_t m = i0 < n ? tok8_starts16(data, n, i0, &bad) : 0u;
    const int c = __popc(m);
    int incl = c;
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    int before = 0;
    for (int w = 0; w < warp; w++) before += s_w[w];
    int64_t r = block_base[blockIdx.x] + before + incl - c;
    while (m) {
        const int j = __ffs(m) - 1;
        m &= m - 1;
        const int64_t b = i0 + j;
        int64_t e = b + 1;
        while (e < n && !tok8_ws_at(data, n, e)) e++;
        starts[r] = b;
        lens[r] = e - b;
        r++;
    }
}

// ---- numeric text columns (textFileColumns) ----------------------------------------------------------------------------
// k_tc_count / k_tc_emit: the line starts of a byte range in the tokenisers' layout (16 bytes per thread, 4096-byte
// blocks, block counts, the host-side scan, then every start in text order); the count pass also ORs bit 0 into
// `flags` when a byte >= 0x80 occurs, so that the UTF-8 check runs only on such ranges.  k_tc_parse: one thread per
// line finds the key and value fields and parses them (tc_line, dpk_common.cuh), or marks the line for the host.
// The powers of five live in global memory and are read through L1: lanes index them divergently.
__device__ const uint64_t g_tc_pow5[] = {
#include "dpk_pow5.inc"
};

__global__ void __launch_bounds__(TK_THREADS)
k_tc_count(const uint8_t *__restrict__ data, int64_t n, int64_t *__restrict__ block_counts, unsigned long long *__restrict__ flags) {
    __shared__ int s_w[TK_THREADS / 32];
    const int64_t i0 = ((int64_t)blockIdx.x * TK_THREADS + threadIdx.x) * TK_BYTES;
    bool hi = false;
    const uint32_t m = i0 < n ? tc_starts16(data, n, i0, &hi) : 0u;
    int c = __popc(m);
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = c;
    if (__any_sync(0xffffffffu, hi) && (threadIdx.x & 31) == 0) atomicOr(flags, 1ull);
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < TK_THREADS / 32; w++) t += s_w[w];
        block_counts[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(TK_THREADS)
k_tc_emit(const uint8_t *__restrict__ data, int64_t n, const int64_t *__restrict__ block_base, int64_t *__restrict__ starts) {
    __shared__ int s_w[TK_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t i0 = ((int64_t)blockIdx.x * TK_THREADS + threadIdx.x) * TK_BYTES;
    bool hi = false;
    uint32_t m = i0 < n ? tc_starts16(data, n, i0, &hi) : 0u;
    const int c = __popc(m);
    int incl = c;
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    int before = 0;
    for (int w = 0; w < warp; w++) before += s_w[w];
    int64_t r = block_base[blockIdx.x] + before + incl - c;
    while (m) {
        const int j = __ffs(m) - 1;
        m &= m - 1;
        starts[r++] = i0 + j;
    }
}

// line i = data[starts[i], the next '\n' or n); out_keys / out_vals get int64 values or float64 bits, host[i] = 1
// (and zeros in the outputs) when the host must parse the line
__global__ void __launch_bounds__(256)
k_tc_parse(const uint8_t *__restrict__ data, int64_t n, const int64_t *__restrict__ starts, int64_t nlines,
           const uint8_t *__restrict__ sep, int32_t sep_len, int32_t key, int32_t value, int32_t key_kind,
           int32_t value_kind, int64_t *__restrict__ out_keys, int64_t *__restrict__ out_vals, uint8_t *__restrict__ host) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nlines) return;
    const int64_t b = starts[i];
    const int64_t e = i + 1 < nlines ? starts[i + 1] - 1 : (data[n - 1] == '\n' ? n - 1 : n);
    int64_t k = 0, v = 0;
    const bool ok = tc_line(data, b, e, sep, sep_len, key, value, key_kind, value_kind, g_tc_pow5, &k, &v);
    out_keys[i] = ok ? k : 0;
    out_vals[i] = ok ? v : 0;
    host[i] = ok ? 0 : 1;
}

// out[out_off[i] .. out_off[i] + lens[row]) = data[starts[row] ..), row = idx ? idx[i] : i  (token bytes made contiguous:
// the (data, offsets) form dpk_hash_bytes / dpk_dict_encode take; or the bytes of the distinct keys for the host)
__global__ void __launch_bounds__(256)
k_gather_bytes(const uint8_t *__restrict__ data, const int64_t *__restrict__ starts, const int64_t *__restrict__ lens,
               const int64_t *__restrict__ idx, int64_t m, const int64_t *__restrict__ out_off, uint8_t *__restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < m; i += stride) {
        const int64_t row = idx ? idx[i] : i;
        const uint8_t *src = data + starts[row];
        uint8_t *dst = out + out_off[i];
        const int64_t len = lens[row];
        for (int64_t j = 0; j < len; j++) dst[j] = src[j];
    }
}

static inline int64_t dict_slots(int64_t n) {
    int64_t s = 1024;
    while (s < 2 * n) s <<= 1;
    return s;
}

}  // namespace dpk

using namespace dpk;

extern "C" {

int64_t dpk_tokenize_blocks(int64_t n) { return n <= 0 ? 0 : (n + TK_CHUNK - 1) / TK_CHUNK; }

int dpk_tokenize_count(const uint8_t *data, int64_t n, int64_t *block_counts, int64_t *flags, dpk_stream_t stream) {
    if (n < 0) return fail(DPK_ERR_INVALID, "n=%lld < 0", (long long)n);
    if (n == 0) return DPK_OK;
    if (!data || !block_counts || !flags) return fail(DPK_ERR_INVALID, "NULL pointer");
    const int64_t nb = dpk_tokenize_blocks(n);
    if (nb >= ((int64_t)1 << 31)) return fail(DPK_ERR_INVALID, "text of %lld bytes is too long for one launch", (long long)n);
    cudaStream_t st = (cudaStream_t)stream;
    DPK_LAUNCH("tok_count", st, k_tok_count<<<(int)nb, TK_THREADS, 0, st>>>(data, n, block_counts, (unsigned long long *)flags));
    return DPK_OK;
}

int dpk_tokenize_emit(const uint8_t *data, int64_t n, const int64_t *block_base, int64_t *starts, int64_t *lens,
                      dpk_stream_t stream) {
    if (n < 0) return fail(DPK_ERR_INVALID, "n=%lld < 0", (long long)n);
    if (n == 0) return DPK_OK;
    if (!data || !block_base || !starts || !lens) return fail(DPK_ERR_INVALID, "NULL pointer");
    const int64_t nb = dpk_tokenize_blocks(n);
    if (nb >= ((int64_t)1 << 31)) return fail(DPK_ERR_INVALID, "text of %lld bytes is too long for one launch", (long long)n);
    cudaStream_t st = (cudaStream_t)stream;
    DPK_LAUNCH("tok_emit", st, k_tok_emit<<<(int)nb, TK_THREADS, 0, st>>>(data, n, block_base, starts, lens));
    return DPK_OK;
}

int dpk_tokenize_utf8_count(const uint8_t *data, int64_t n, int64_t *block_counts, int64_t *flags, dpk_stream_t stream) {
    if (n < 0) return fail(DPK_ERR_INVALID, "n=%lld < 0", (long long)n);
    if (n == 0) return DPK_OK;
    if (!data || !block_counts || !flags) return fail(DPK_ERR_INVALID, "NULL pointer");
    const int64_t nb = dpk_tokenize_blocks(n);
    if (nb >= ((int64_t)1 << 31)) return fail(DPK_ERR_INVALID, "text of %lld bytes is too long for one launch", (long long)n);
    cudaStream_t st = (cudaStream_t)stream;
    DPK_LAUNCH("tok8_count", st, k_tok8_count<<<(int)nb, TK_THREADS, 0, st>>>(data, n, block_counts, (unsigned long long *)flags));
    return DPK_OK;
}

int dpk_tokenize_utf8_emit(const uint8_t *data, int64_t n, const int64_t *block_base, int64_t *starts, int64_t *lens,
                           dpk_stream_t stream) {
    if (n < 0) return fail(DPK_ERR_INVALID, "n=%lld < 0", (long long)n);
    if (n == 0) return DPK_OK;
    if (!data || !block_base || !starts || !lens) return fail(DPK_ERR_INVALID, "NULL pointer");
    const int64_t nb = dpk_tokenize_blocks(n);
    if (nb >= ((int64_t)1 << 31)) return fail(DPK_ERR_INVALID, "text of %lld bytes is too long for one launch", (long long)n);
    cudaStream_t st = (cudaStream_t)stream;
    DPK_LAUNCH("tok8_emit", st, k_tok8_emit<<<(int)nb, TK_THREADS, 0, st>>>(data, n, block_base, starts, lens));
    return DPK_OK;
}

int dpk_textcols_count(const uint8_t *data, int64_t n, int64_t *block_counts, int64_t *flags, dpk_stream_t stream) {
    if (n < 0) return fail(DPK_ERR_INVALID, "n=%lld < 0", (long long)n);
    if (n == 0) return DPK_OK;
    if (!data || !block_counts || !flags) return fail(DPK_ERR_INVALID, "NULL pointer");
    const int64_t nb = dpk_tokenize_blocks(n);
    if (nb >= ((int64_t)1 << 31)) return fail(DPK_ERR_INVALID, "text of %lld bytes is too long for one launch", (long long)n);
    cudaStream_t st = (cudaStream_t)stream;
    DPK_LAUNCH("tc_count", st, k_tc_count<<<(int)nb, TK_THREADS, 0, st>>>(data, n, block_counts, (unsigned long long *)flags));
    return DPK_OK;
}

int dpk_textcols_emit(const uint8_t *data, int64_t n, const int64_t *block_base, int64_t *starts, dpk_stream_t stream) {
    if (n < 0) return fail(DPK_ERR_INVALID, "n=%lld < 0", (long long)n);
    if (n == 0) return DPK_OK;
    if (!data || !block_base || !starts) return fail(DPK_ERR_INVALID, "NULL pointer");
    const int64_t nb = dpk_tokenize_blocks(n);
    if (nb >= ((int64_t)1 << 31)) return fail(DPK_ERR_INVALID, "text of %lld bytes is too long for one launch", (long long)n);
    cudaStream_t st = (cudaStream_t)stream;
    DPK_LAUNCH("tc_emit", st, k_tc_emit<<<(int)nb, TK_THREADS, 0, st>>>(data, n, block_base, starts));
    return DPK_OK;
}

int dpk_textcols_parse(const uint8_t *data, int64_t n, const int64_t *starts, int64_t nlines, const uint8_t *sep,
                       int32_t sep_len, int32_t key, int32_t value, int32_t key_kind, int32_t value_kind,
                       int64_t *out_keys, int64_t *out_vals, uint8_t *host, dpk_stream_t stream) {
    if (n < 0 || nlines < 0 || nlines > n) return fail(DPK_ERR_INVALID, "n=%lld nlines=%lld", (long long)n, (long long)nlines);
    if (sep_len < 0 || key < 0 || value < 0) return fail(DPK_ERR_INVALID, "sep_len=%d key=%d value=%d", sep_len, key, value);
    if ((key_kind != DPK_K_I64 && key_kind != DPK_K_F64) || (value_kind != DPK_K_I64 && value_kind != DPK_K_F64))
        return fail(DPK_ERR_UNSUPPORTED, "column kinds %d, %d (DPK_K_I64 / DPK_K_F64)", key_kind, value_kind);
    if (nlines == 0) return DPK_OK;
    if (!data || !starts || (sep_len && !sep) || !out_keys || !out_vals || !host) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    DPK_LAUNCH("tc_parse", st, k_tc_parse<<<(unsigned)((nlines + 255) / 256), 256, 0, st>>>(
        data, n, starts, nlines, sep, sep_len, key, value, key_kind, value_kind, out_keys, out_vals, host));
    return DPK_OK;
}

int dpk_gather_bytes(const uint8_t *data, const int64_t *starts, const int64_t *lens, const int64_t *idx, int64_t m,
                     const int64_t *out_off, uint8_t *out, dpk_stream_t stream) {
    if (m < 0) return fail(DPK_ERR_INVALID, "m=%lld < 0", (long long)m);
    if (m == 0) return DPK_OK;
    if (!data || !starts || !lens || !out_off || !out) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    int64_t g = (m + 255) / 256, cap = (int64_t)sm_count() * 16;
    if (g > cap) g = cap;
    DPK_LAUNCH("gather_bytes", st, k_gather_bytes<<<(int)g, 256, 0, st>>>(data, starts, lens, idx, m, out_off, out));
    return DPK_OK;
}

int64_t dpk_dict_encode_workspace_bytes(int64_t n) { return dict_slots(n < 0 ? 0 : n) * 8; }

int dpk_dict_encode(const uint8_t *data, const int64_t *offsets, const int64_t *hash, int64_t n,
                    int64_t *out_rep, void *ws, int64_t ws_bytes, dpk_stream_t stream) {
    if (n < 0 || n >= ((int64_t)1 << 31)) return fail(DPK_ERR_INVALID, "n=%lld out of range [0, 2^31)", (long long)n);
    if (n == 0) return DPK_OK;
    if (!offsets || !hash || !out_rep || !ws) return fail(DPK_ERR_INVALID, "NULL pointer");
    const int64_t slots = dict_slots(n);
    if (ws_bytes < slots * 8) return fail(DPK_ERR_WORKSPACE, "workspace needs %lld B, got %lld", (long long)(slots * 8), (long long)ws_bytes);
    cudaStream_t st = (cudaStream_t)stream;
    DPK_CUDA_TRY(cudaMemsetAsync(ws, 0xff, (size_t)slots * 8, st));
    int64_t g = (n + 255) / 256, cap = (int64_t)sm_count() * 16;
    if (g > cap) g = cap;
    DPK_LAUNCH("dict_encode", st, k_dict_encode<<<(int)g, 256, 0, st>>>(data, offsets, hash, n, (long long *)ws,
                                                                       (uint64_t)(slots - 1), out_rep));
    return DPK_OK;
}

}  // extern "C"
