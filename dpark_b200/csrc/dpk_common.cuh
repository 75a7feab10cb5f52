// dpk_common.cuh -- shared pieces of the H100 shuffle kernels: error plumbing,
// the portable_hash device functions (a1) and the partitioner functor (a2).
// Hash/partition functions are __host__ __device__ so tests/hostcheck can run
// the very same code on the CPU against the oracle without a GPU.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <string.h>
#include <math.h>

#include "dpark_b200.h"

#define DPK_HD __host__ __device__ __forceinline__

namespace dpk {

// ------------------------------------------------------------------ errors
extern thread_local char g_err[512];
int fail(int code, const char *fmt, ...);
#define DPK_CUDA_TRY(expr)                                                        \
    do {                                                                          \
        cudaError_t _e = (expr);                                                  \
        if (_e != cudaSuccess)                                                    \
            return dpk::fail(DPK_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,        \
                             cudaGetErrorString(_e), __FILE__, __LINE__);         \
    } while (0)
#define DPK_LAUNCH_CHECK() DPK_CUDA_TRY(cudaGetLastError())

int sm_count();
extern int g_scatter_items;  // dpk_partition.cu, rows per thread and tile of the scatter (16 or 8)
extern int g_count_mode;  // dpk_partition.cu, A/B switch of the histogram pass
extern int g_scatter_threads;  // dpk_partition.cu, CTA size of the bulk multisplit (256 or 512)
extern int g_scatter_seg_wide;  // dpk_partition.cu
extern int g_scatter_wide_from, g_copy_sms, g_copy_tma;  // dpk_partition.cu / dpk_peer.cu
extern int g_scatter_ptr_bulk, g_scatter_ptr_threads;  // dpk_partition.cu, pointer mode (fused scatter + exchange)
extern int g_scatter_bulk;  // dpk_partition.cu, 1 = unordered multisplits use the TMA bulk-store kernel

// every kernel launch goes through DPK_LAUNCH: counts it and, when profiling
// is on, brackets it with CUDA events on the launching stream.
struct ProfScope {
    int idx;
    cudaStream_t st;
    ProfScope(const char *label, cudaStream_t s);
    ~ProfScope();
};
#define DPK_LAUNCH(label, st, ...)              \
    do {                                        \
        {                                       \
            dpk::ProfScope _ps(label, st);      \
            __VA_ARGS__;                        \
        }                                       \
        DPK_LAUNCH_CHECK();                     \
    } while (0)

// ------------------------------------------------------------- a1: hashing
constexpr uint64_t kPyMod = (1ull << 61) - 1;  // CPython _PyHASH_MODULUS

// hash(int) for an int64 value -- dpark/portable_hash.pyx:61-62 (CPython
// long_hash: sign * (|x| mod 2^61-1); -1 -> -2).
DPK_HD int64_t hash_i64(int64_t x) {
    if ((uint64_t)x < kPyMod) return x;                      // 0 <= x < 2^61-1 hashes to itself (the common case)
    uint64_t a = x < 0 ? 0ull - (uint64_t)x : (uint64_t)x;  // |INT64_MIN| = 2^63 ok
    uint64_t r = (a & kPyMod) + (a >> 61);                   // hi <= 4
    if (r >= kPyMod) r -= kPyMod;
    int64_t h = x < 0 ? -(int64_t)r : (int64_t)r;
    return h == -1 ? -2 : h;
}
DPK_HD int64_t hash_u64(uint64_t a) {
    uint64_t r = (a & kPyMod) + (a >> 61);                   // hi <= 7
    if (r >= kPyMod) r -= kPyMod;
    return (int64_t)r;
}
// hash(float) -- CPython _Py_HashDouble (NaN unsupported: hashed by identity there)
DPK_HD int64_t hash_f64(double v) {
    if (isinf(v)) return v > 0 ? 314159 : -314159;
    if (v != v) return 0;
    int e;
    double m = frexp(v, &e);
    bool neg = m < 0;
    if (neg) m = -m;
    uint64_t x = 0;
    while (m != 0.0) {
        x = ((x << 28) & kPyMod) | (x >> (61 - 28));
        m *= 268435456.0;
        e -= 28;
        uint64_t y = (uint64_t)m;
        m -= (double)y;
        x += y;
        if (x >= kPyMod) x -= kPyMod;
    }
    e = e >= 0 ? e % 61 : 61 - 1 - ((-1 - e) % 61);
    x = ((x << e) & kPyMod) | (x >> (61 - e));
    int64_t h = neg ? -(int64_t)x : (int64_t)x;
    return h == -1 ? -2 : h;
}

template <typename T> struct KeyHash;
template <> struct KeyHash<int64_t> { static DPK_HD int64_t of(int64_t k) { return hash_i64(k); } };
template <> struct KeyHash<int32_t> { static DPK_HD int64_t of(int32_t k) { return hash_i64((int64_t)k); } };
template <> struct KeyHash<uint64_t> { static DPK_HD int64_t of(uint64_t k) { return hash_u64(k); } };
template <> struct KeyHash<double> { static DPK_HD int64_t of(double k) { return hash_f64(k); } };
template <> struct KeyHash<float> { static DPK_HD int64_t of(float k) { return hash_f64((double)k); } };

// string_hash over signed chars -- dpark/portable_hash.pyx:17-32
DPK_HD int64_t hash_bytes_signed(const uint8_t *s, int64_t len) {
    if (len == 0) return 0;
    uint64_t value = (uint64_t)(int64_t)(int8_t)s[0] << 7;
    for (int64_t i = 0; i < len; i++)
        value = (1000003ull * value) ^ (uint64_t)(int64_t)(int8_t)s[i];
    value ^= (uint64_t)len;
    return (int64_t)value == -1 ? -2 : (int64_t)value;
}
// unicode_hash over the code points of a UTF-8 encoded str -- portable_hash.pyx:34-48
DPK_HD int64_t hash_utf8_codepoints(const uint8_t *s, int64_t nbytes) {
    if (nbytes == 0) return 0;
    uint64_t value = 0;
    int64_t ncp = 0, i = 0;
    while (i < nbytes) {
        uint32_t c = s[i], cp;
        int extra;
        if (c < 0x80) { cp = c; extra = 0; }
        else if (c < 0xE0) { cp = c & 0x1F; extra = 1; }
        else if (c < 0xF0) { cp = c & 0x0F; extra = 2; }
        else { cp = c & 0x07; extra = 3; }
        for (int j = 1; j <= extra && i + j < nbytes; j++) cp = (cp << 6) | (s[i + j] & 0x3F);
        i += extra + 1;
        if (ncp == 0) value = (uint64_t)cp << 7;
        value = (1000003ull * value) ^ (uint64_t)cp;
        ncp++;
    }
    value ^= (uint64_t)ncp;
    return (int64_t)value == -1 ? -2 : (int64_t)value;
}

// tuple_hash -- dpark/portable_hash.pyx:3-15 over the portable_hash values of the items (item_hash[a * stride + i] is
// item a of row i); int64 wraparound like the Cython code.  An empty tuple hashes to 0x345678 + 97531.
DPK_HD int64_t hash_tuple_items(const int64_t *item_hash, int64_t stride, int64_t i, int32_t arity) {
    uint64_t mul = 1000003ull, value = 0x345678ull;
    int64_t l = arity;
    for (int32_t a = 0; a < arity; a++) {
        l -= 1;
        value = (value ^ (uint64_t)item_hash[(int64_t)a * stride + i]) * mul;
        mul += (uint64_t)(82520 + l * 2);
    }
    value += 97531ull;
    return (int64_t)value == -1 ? -2 : (int64_t)value;
}

// ------------------------------------------------- a2: HashPartitioner functor
// getPartition = portable_hash(key) floor-mod P, or bisect_right(thresholds, h)
// (dpark/dependency.py:229-233).  floor-mod by an arbitrary P without a 64-bit
// divide: power-of-two mask, else multiply-high by a precomputed magic
// (round-up method, Granlund-Montgomery / libdivide "branchfree" form).
struct PartFn {
    int32_t P;
    int32_t mode;  // 0: P==1, 1: power of two, 2: magic, 3: thresholds
    uint64_t magic;
    int32_t shift;
    int32_t nthr;
    const int64_t *thresholds;
    // fine buckets: each reduce partition is split into 2^sub_bits sub-buckets by
    // other bits of the key's hash (an internal layout detail -- partition p still
    // owns exactly the keys the reference gives it; its rows are the concatenation
    // of its sub-buckets).  Sub-buckets bound the reduce-side table working set so
    // it stays resident in the 50 MB L2.
    int32_t sub_bits;
    // DPK_K_ROWID keys: per-row portable_hash column the multisplit looks the hash up in
    const int64_t *row_hash;

    DPK_HD int32_t nbuckets() const { return P << sub_bits; }
    // bucket id = partition * 2^sub_bits + sub, sub a function of the hash only
    // (equal keys -> equal hash -> same bucket)
    DPK_HD int32_t bucket(int64_t h) const {
        // mode 4 (radix pass of the group-by sort): digit `shift` of the raw key bits, P = 2^bits
        if (mode == 4) return (int32_t)(((uint64_t)h >> shift) & (uint64_t)(P - 1));
        // mode 5 (second-level split on the reduce side): the P = 2^k bits of the same mixed
        // hash that follow the first-level sub-bucket bits (shift = 32 - sub_bits_1 - k)
        if (mode == 5) return P == 1 ? 0 : (int32_t)((mixed(h) >> shift) & (uint32_t)(P - 1));
        int32_t p = (*this)(h);
        if (sub_bits == 0) return p;
        return (p << sub_bits) | (int32_t)(mixed(h) >> (32 - sub_bits));
    }
    // 32 well-mixed bits of the hash for the LAYOUT-ONLY sub-bucket levels (first level: the top sub_bits
    // bits, second level: the bits below them; at most 12 + 10).  Both halves of the hash enter through
    // odd multipliers, then the lowbias32 finaliser; five 32-bit multiplies/xorshifts instead of the two
    // 64-bit multiplies of a splitmix step (the multisplit kernels are issue-bound, DESIGN.md section 4).
    static DPK_HD uint32_t mixed(int64_t h) {
        uint32_t x = (uint32_t)(uint64_t)h * 0x9E3779B1u + (uint32_t)((uint64_t)h >> 32) * 0x85EBCA77u;
        x ^= x >> 16; x *= 0x21F0AAADu;
        x ^= x >> 15; x *= 0x735A2D97u;
        x ^= x >> 15;
        return x;
    }

    DPK_HD int32_t operator()(int64_t h) const {
        if (mode == 1) return (int32_t)((uint64_t)h & (uint64_t)(P - 1));  // two's complement == floor-mod
        if (mode == 2) {
            uint64_t a = h < 0 ? 0ull - (uint64_t)h : (uint64_t)h;
#ifdef __CUDA_ARCH__
            uint64_t q = __umul64hi(magic, a);
#else
            uint64_t q = (uint64_t)(((unsigned __int128)magic * a) >> 64);
#endif
            uint64_t t = ((a - q) >> 1) + q;
            q = t >> shift;
            uint32_t r = (uint32_t)(a - q * (uint64_t)P);
            return h < 0 ? (r ? P - (int32_t)r : 0) : (int32_t)r;
        }
        if (mode == 3) {
            int32_t lo = 0, hi = nthr;
            while (lo < hi) {
                int32_t mid = (lo + hi) >> 1;
                if (h < thresholds[mid]) hi = mid; else lo = mid + 1;
            }
            return lo;
        }
        return 0;
    }
};
// host: build the functor (thresholds is a device pointer, only stored)
int make_partfn(int32_t P, const int64_t *thresholds, int32_t nthr, int32_t sub_bits, PartFn *out);

// Segmented multisplit (dpk_partition.cu), used by the reduce side: every first-level
// bucket b (rows in nsrc segments seg_start/seg_rows[s][b] of the input) is split into
// fine.nbuckets() fine buckets; output rows are bucket-major then fine-bucket-major and
// fine_off[F1 * S2 + 1] delimits the fine buckets.  keys/vals: device; st-ordered.
int64_t seg_multisplit_ws_bytes(int64_t n, int32_t F1, int32_t S2, int32_t nsrc);
int seg_multisplit(const void *keys, int key_kind, const void *vals, int32_t val_bytes, int64_t n,
                   const PartFn &fine, int32_t F1, int32_t nsrc, const int64_t *seg_start,
                   const int64_t *seg_rows, void *out_keys, void *out_vals, int64_t *fine_off, void *ws,
                   int64_t ws_bytes, cudaStream_t st, bool stable = false);

// murmur3 fmix64 -- slot hash for the reduce-side tables in HBM (implementations 0/1; not part of the
// reference semantics; only spreads keys over table slots)
DPK_HD uint64_t mix64(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull;
    return x ^ (x >> 33);
}
// 32-bit slot hash of 64 key bits for the shared-memory merge (implementation 2): independent of
// PartFn::mixed (all rows of a fine bucket agree in those bits), murmur3 fmix32 after folding the halves
DPK_HD uint32_t slot_hash32(uint64_t kb) {
    uint32_t x = (uint32_t)kb * 0xCC9E2D51u + (uint32_t)(kb >> 32) * 0x1B873593u + 0x7F4A7C15u;
    x ^= x >> 16; x *= 0x85EBCA6Bu;
    x ^= x >> 13; x *= 0xC2B2AE35u;
    x ^= x >> 16;
    return x;
}

// Second-level split of the reduce side (dpk_combine.cu, implementation 2): every one of the F first-level buckets
// of n rows is split 2^sb2 ways (PartFn mode 5) until the average fine bucket holds at most target_rows rows
// (dpk_set_option "agg_target_rows"), at most 2^AG_MAX_SB2 ways.
constexpr int AG_MAX_SB2 = 10;
DPK_HD int choose_sb2(int64_t n, int32_t F, int target_rows) {
    int sb2 = 0;
    while (sb2 < AG_MAX_SB2 && n / ((int64_t)F << sb2) > target_rows) sb2++;
    return sb2;
}
// the functor of that split: fine bucket = the 2^sb2 bits of mixed(hash) below the first level's sub_bits
DPK_HD PartFn fine_partfn(const PartFn &first, int sb2) {
    PartFn fine = first;
    fine.mode = 5; fine.P = 1 << sb2; fine.shift = 32 - first.sub_bits - sb2; fine.sub_bits = 0;
    return fine;
}

// ------------------------------------------------------------- f4: tokeniser arithmetic (dpk_strings.cu)
// str.split() without arguments on ASCII text: whitespace = ' ', \t \n \v \f \r, \x1c..\x1f
constexpr int TK_BYTES = 16;   // bytes per thread
__host__ __device__ __forceinline__ bool tok_ws(uint8_t c) { return c == 0x20 || (c >= 0x09 && c <= 0x0d) || (c >= 0x1c && c <= 0x1f); }

// bit j of the result: a token starts at byte i0 + j; *hi |= any byte >= 0x80
__host__ __device__ __forceinline__ uint32_t tok_starts16(const uint8_t *__restrict__ data, int64_t n, int64_t i0, bool *hi) {
    uint8_t c[TK_BYTES];
    if (i0 + TK_BYTES <= n && (((uintptr_t)(data + i0)) & 15u) == 0) {
        const uint4 q = *reinterpret_cast<const uint4 *>(data + i0);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < TK_BYTES; j++) c[j] = (uint8_t)(w[j >> 2] >> ((j & 3) * 8));
    } else {
#pragma unroll
        for (int j = 0; j < TK_BYTES; j++) c[j] = i0 + j < n ? data[i0 + j] : (uint8_t)0x20;
    }
    bool prev_ws = i0 == 0 ? true : tok_ws(data[i0 - 1]);
    uint32_t m = 0;
    bool h = false;
#pragma unroll
    for (int j = 0; j < TK_BYTES; j++) {
        const bool ws = tok_ws(c[j]);
        h |= c[j] >= 0x80;
        if (!ws && prev_ws) m |= 1u << j;
        prev_ws = ws;
    }
    *hi = h;
    return m;
}


}  // namespace dpk
