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
// pack: PK_OUT = write packed rows (out_keys: PackedRow array, out_vals unused), PK_IN = read packed rows (keys:
// PackedRow array, vals unused); both need key and value columns of the same width.
int64_t seg_multisplit_ws_bytes(int64_t n, int32_t F1, int32_t S2, int32_t nsrc);
int seg_multisplit(const void *keys, int key_kind, const void *vals, int32_t val_bytes, int64_t n,
                   const PartFn &fine, int32_t F1, int32_t nsrc, const int64_t *seg_start,
                   const int64_t *seg_rows, void *out_keys, void *out_vals, int64_t *fine_off, void *ws,
                   int64_t ws_bytes, cudaStream_t st, bool stable = false, int pack = 0);

// Packed shuffle rows (DPK_K_PACKED): one record per row, key then value, for key and value columns of the same
// width -- 16-byte records for 8-byte columns, 8-byte records for 4-byte ones.  A multisplit that writes records stores
// one bucket run per bucket instead of one per column, and a reader fetches a row with one load.
constexpr int PK_OUT = 1, PK_IN = 2;
template <typename KeyT, typename ValT>
struct __align__(2 * sizeof(KeyT)) PackedRow {
    KeyT k;
    ValT v;
};

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

// a value column of 4- or 8-byte elements moved as raw words (the join / cogroup emits, the topByKey rounds)
template <int W> struct ValWord;
template <> struct ValWord<4> { typedef uint32_t T; };
template <> struct ValWord<8> { typedef uint64_t T; };

// ------------------------------------------------------------- f1: join arithmetic (dpk_join.cu; tests/joincheck.cu
// runs the same functions on the CPU)
// A group's id run ids[0 .. len) holds its left rows (ids < nL) before its right rows: the map side is a stable
// multisplit, the radix passes are stable and the left splits come first.  So the left count is a binary search (the
// lower bound of nL: the ids below it).
DPK_HD int64_t join_left_rows(const int64_t *run, int64_t len, int64_t nL) {
    int64_t lo = 0, hi = len;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (run[mid] < nL) lo = mid + 1; else hi = mid;
    }
    return lo;
}
// rows a side contributes to the cross product: its own rows, or one None row when it has none and the OTHER side's
// unmatched keys are kept (dpark_b200/rdd.py _join: `if not left and keep_right: left = [None]`)
DPK_HD int64_t join_side(int64_t n, bool keep_other) { return n > 0 ? n : (keep_other ? 1 : 0); }
DPK_HD int64_t join_count(int64_t nl, int64_t nr, bool keep_left, bool keep_right) {
    return join_side(nl, keep_right) * join_side(nr, keep_left);
}
// output row i of a group -> (a, b): left row a, right row b, `for a in left for b in right`
DPK_HD void join_pair(int64_t i, int64_t nr, bool keep_left, int64_t *a, int64_t *b) {
    const int64_t R = join_side(nr, keep_left);
    *a = i / R;
    *b = i - *a * R;
}
// the last group g in [lo, hi) with off[g] <= i (off[lo] <= i holds): the group of output row i given the exclusive
// scan off of the groups' row counts.  Empty groups share their offset with the next group, so the answer always has
// rows.  The load-balanced emits of the join and the cogroup map their rows to groups with it.
DPK_HD int64_t group_of(const int64_t *off, int64_t lo, int64_t hi, int64_t i) {
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (off[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
}

// ------------------------------------------------------------- f1: cogroup arithmetic (dpk_join.cu; tests/cogroupcheck.cu
// runs the same functions on the CPU)
// Input t of a cogroup owns the row ids [bounds[t], bounds[t + 1]).  A group's id run ids[s .. s + len) is ascending in
// input order, so input t's sub-run starts where the ids below bounds[t] end: one lower-bound search per boundary.
// Writes first[t * stride] (absolute position in ids) and count[t * stride] for t < ninputs.
DPK_HD void cogroup_split(const int64_t *ids, int64_t s, int64_t len, const int64_t *bounds, int32_t ninputs,
                          int64_t *first, int64_t *count, int64_t stride) {
    int64_t lo = join_left_rows(ids + s, len, bounds[0]);
    for (int32_t t = 0; t < ninputs; t++) {
        const int64_t hi = join_left_rows(ids + s, len, bounds[t + 1]);
        first[t * stride] = s + lo;
        count[t * stride] = hi - lo;
        lo = hi;
    }
}
// output row r of one input, in the group that starts at output row base and whose sub-run starts at ids[first]: the
// input's own row number (its values column is indexed from 0, its ids from id_base)
DPK_HD int64_t cogroup_source(const int64_t *ids, int64_t first, int64_t base, int64_t r, int64_t id_base) {
    return ids[first + r - base] - id_base;
}

// ------------------------------------------------------------- f4: topByKey arithmetic (dpk_topk.cu; tests/topkcheck.cu
// runs the same functions on the CPU)
// The low `width` bytes of a value (int, or IEEE float when is_float) -> a word whose unsigned order is the value's
// order, complemented for reverse: ints flip the sign bit; floats map -0.0 to +0.0 (they compare equal in Python), then
// flip the sign bit of positives and every bit of negatives.  NaN has no place in this order; callers keep it out.
DPK_HD uint64_t topk_order_key(uint64_t bits, int32_t width, bool is_float, bool reverse) {
    const uint64_t mask = width == 8 ? ~0ull : 0xFFFFFFFFull, sign = width == 8 ? 1ull << 63 : 1ull << 31;
    bits &= mask;
    uint64_t k;
    if (!is_float) {
        k = bits ^ sign;
    } else {
        if (bits == sign) bits = 0;
        k = (bits & sign) ? (~bits & mask) : (bits | sign);
    }
    return reverse ? (~k & mask) : k;
}
// A run of L candidates after one round with tile T: its full chunks of T keep top_n each, the rest min(top_n, rest).
// A run of L <= T is one unit and keeps min(top_n, L), its answer (top_n <= T).
DPK_HD int64_t topk_next_len(int64_t L, int64_t T, int64_t top_n) {
    const int64_t rest = L % T;
    return L / T * top_n + (rest < top_n ? rest : top_n);
}
// The unit of run [s, e) that CTA w takes: units are the run's chunks [s + cT, min(e, s + (c + 1)T)), and a CTA takes the
// units that start in its window of rows [wT, (w + 1)T).  A window holds at most one chunk start of a run.  Returns
// false when the run has none there; a CTA's units lie in [wT, (w + 2)T).
DPK_HD bool topk_unit(int64_t s, int64_t e, int64_t w, int64_t T, int64_t *u0, int64_t *u1) {
    const int64_t w0 = w * T;
    const int64_t a = s >= w0 ? s : s + (w0 - s + T - 1) / T * T;
    if (a >= w0 + T || a >= e) return false;
    *u0 = a;
    *u1 = e < a + T ? e : a + T;
    return true;
}
// where the unit starting at row u0 of the run that starts at s writes: the run's next-round start out_s plus top_n per
// full chunk before it
DPK_HD int64_t topk_unit_out(int64_t s, int64_t u0, int64_t out_s, int64_t T, int64_t top_n) {
    return out_s + (u0 - s) / T * top_n;
}

// ------------------------------------------------------------- f5: innerJoin hash table (dpk_join.cu; tests/bcastcheck.cu
// runs the same functions on the CPU)
// The small side's distinct keys in an open-addressing table of 2^k >= 2 G slots, linear probing.  A slot is 16 bytes so
// that a probe step is one aligned load; grp = -1 marks an empty slot (the caller fills the table with 0xFF bytes).
struct __align__(16) BcastSlot {
    uint64_t key;   // normalised key bits (bcast_key_bits)
    int32_t grp;    // the key's group, -1 = empty
    int32_t pad;
};
// A key as the table holds it: ints widened to int64, floats widened to float64 with -0.0 spelled 0.0 (Python's dict
// finds 0.0 under -0.0).  False for NaN, which no dict lookup finds.
template <typename T> DPK_HD bool bcast_key_bits(T k, uint64_t *kb) {
    *kb = (uint64_t)(int64_t)k;
    return true;
}
template <> DPK_HD bool bcast_key_bits<double>(double k, uint64_t *kb) {
    if (k != k) return false;
    if (k == 0.0) k = 0.0;
    memcpy(kb, &k, sizeof k);
    return true;
}
template <> DPK_HD bool bcast_key_bits<float>(float k, uint64_t *kb) { return bcast_key_bits<double>((double)k, kb); }
// slots of a table of G keys: the least power of two >= 2 G (at most half full, so a probe ends at an empty slot)
DPK_HD uint64_t bcast_slots(int64_t G) {
    uint64_t s = 2;
    while (s < 2 * (uint64_t)G) s <<= 1;
    return s;
}
// a key's first slot: all 64 bits mixed (mix64), not portable_hash, which is the identity on small ints and would put
// keys that differ only above the mask into one slot run
DPK_HD uint64_t bcast_slot(uint64_t kb, uint64_t mask) { return mix64(kb) & mask; }
DPK_HD uint64_t bcast_next(uint64_t s, uint64_t mask) { return (s + 1) & mask; }
// claims the first empty slot of kb's probe sequence for group g; the keys are distinct, so no slot is compared
DPK_HD void bcast_insert(BcastSlot *table, uint64_t mask, uint64_t kb, int32_t g) {
    for (uint64_t s = bcast_slot(kb, mask);; s = bcast_next(s, mask)) {
#ifdef __CUDA_ARCH__
        const int32_t old = atomicCAS(&table[s].grp, -1, g);
#else
        const int32_t old = table[s].grp;
        if (old == -1) table[s].grp = g;
#endif
        if (old == -1) {
            table[s].key = kb;
            return;
        }
    }
}
// kb's group, or -1 when its probe sequence reaches an empty slot first
DPK_HD int32_t bcast_find(const BcastSlot *table, uint64_t mask, uint64_t kb) {
    for (uint64_t s = bcast_slot(kb, mask);; s = bcast_next(s, mask)) {
        const BcastSlot e = table[s];
        if (e.grp < 0) return -1;
        if (e.key == kb) return e.grp;
    }
}

// ------------------------------------------------------------- f6: sort arithmetic (dpk_sort.cu; tests/sortcheck.cu runs the
// same functions on the CPU)
// Element i of a column of kind DPK_K_I32 / I64 / F32 / F64 widened to 64 bits: ints to int64, floats to float64 (both
// exact and order-keeping, and the values Python sees), returned as the bit pattern.
DPK_HD bool sort_kind_float(int32_t kind) { return kind == DPK_K_F32 || kind == DPK_K_F64; }
DPK_HD uint64_t sort_wide_bits(const void *col, int32_t kind, int64_t i) {
    if (kind == DPK_K_I32) return (uint64_t)(int64_t) static_cast<const int32_t *>(col)[i];
    if (kind == DPK_K_F32) {
        const double d = (double)static_cast<const float *>(col)[i];
        uint64_t b;
        memcpy(&b, &d, sizeof b);
        return b;
    }
    return static_cast<const uint64_t *>(col)[i];
}
DPK_HD bool sort_is_nan(uint64_t wide_bits) { return (wide_bits & ~(1ull << 63)) > 0x7FF0000000000000ull; }
// The 64-bit order word of a widened value: topk_order_key at width 8, complemented for reverse.
DPK_HD uint64_t sort_word(uint64_t wide_bits, bool is_float, bool reverse) {
    return topk_order_key(wide_bits, 8, is_float, reverse);
}
// Lexicographic order of rows of nw (1 or 2) order words: -1, 0 or 1.
DPK_HD int sort_cmp(uint64_t a0, uint64_t a1, uint64_t b0, uint64_t b1, int32_t nw) {
    if (a0 != b0) return a0 < b0 ? -1 : 1;
    if (nw == 1 || a1 == b1) return 0;
    return a1 < b1 ? -1 : 1;
}
// Partition j >= 1 of L + 1 starts at the bound sorted_bounds[sort_cut_bound(j, L, reverse)]: getPartition is the number
// of bounds <= key ascending, the number of bounds > key for reverse.
DPK_HD int32_t sort_cut_bound(int32_t j, int32_t L, bool reverse) { return reverse ? L - j : j - 1; }
// Where that partition starts among n rows sorted by their order words: the first row >= the bound's words (lower
// bound; ascending), or > them (upper bound; reverse, whose words are complemented).  Row i's first word is w0[i]; with
// nw = 2 its second word is computed from vals[ids[i]] (the value column of kind vkind).
DPK_HD int64_t sort_cut(const uint64_t *w0, const int64_t *ids, const void *vals, int32_t vkind, int64_t n, uint64_t t0,
                        uint64_t t1, int32_t nw, bool reverse) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        const uint64_t m1 = nw == 2 ? sort_word(sort_wide_bits(vals, vkind, ids[mid]), sort_kind_float(vkind), reverse) : 0;
        const int c = sort_cmp(w0[mid], m1, t0, t1, nw);
        if (reverse ? c <= 0 : c < 0) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// ------------------------------------------------------------- f7: t-digest arithmetic (dpk_tdigest.cu; tests/tdigestcheck.cu
// runs the same functions on the CPU).  dpark_b200/quantiles.py operation for operation: every sum, product and
// quotient is rounded on its own in Python's order (the __d*_rn intrinsics are never contracted into an FMA), and min /
// max are Python's, which keep the first argument unless the second compares strictly below / above it.
constexpr int TD_CAP = 209;            // capacity - 1 = 2 * ceil(100) + 10 - 1: a full buffer plus the centroids
constexpr int TD_STAGE = 2 * TD_CAP;   // the longest fold the kernels stage; a longer one keeps the composition
constexpr double TD_COMPRESSION = 100.0;
DPK_HD double td_add(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
DPK_HD double td_sub(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
DPK_HD double td_mul(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
DPK_HD double td_div(double a, double b) {
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}
DPK_HD double td_min(double a, double b) { return b < a ? b : a; }
DPK_HD double td_max(double a, double b) { return b > a ? b : a; }
// Element i of a value column of kind DPK_K_I32 / I64 / F32 / F64 as Python's float(x): ints round to nearest.
DPK_HD double td_value(const void *col, int32_t kind, int64_t i) {
    if (kind == DPK_K_I32) return (double)static_cast<const int32_t *>(col)[i];
    if (kind == DPK_K_I64) return (double)static_cast<const int64_t *>(col)[i];
    if (kind == DPK_K_F32) return (double)static_cast<const float *>(col)[i];
    return static_cast<const double *>(col)[i];
}
// zz <= q * (1 - q) with q = a / total, the quotient rounded as Python rounds it (0 <= a <= total; r = 1 / total).  The
// product with the reciprocal lies within 3 ulp of 1 of the quotient, so q * (1 - q) moves by less than 1e-15; outside a
// band of 4e-15 around zz the answer is settled without the division.
DPK_HD bool td_within(double zz, double a, double total, double r) {
    const double qa = td_mul(a, r), d = td_sub(zz, td_mul(qa, td_sub(1.0, qa)));
    if (d > 4e-15) return false;
    if (d < -4e-15) return true;
    const double q = td_div(a, total);
    return zz <= td_mul(q, td_sub(1.0, q));
}
// _fold's scale test: does the next entry (weight w) join the open centroid (weight W), `done` the weight before it?
DPK_HD bool td_fuses(double W, double w, double done, double total, double norm, double r) {
    const double fused = td_add(W, w), z = td_mul(fused, norm), zz = td_mul(z, z);
    return td_within(zz, done, total, r) && td_within(zz, td_add(done, fused), total, r);
}
DPK_HD double td_norm(double total) { return td_div(TD_COMPRESSION, td_mul(M_PI, total)); }
// out_m[-1] + (ms[i] - out_m[-1]) * ws[i] / out_w[-1], W the centroid's weight with w already added
DPK_HD double td_mean_step(double m, double x, double w, double W) {
    return td_add(m, td_div(td_mul(td_sub(x, m), w), W));
}
// A fold's first pass, over its n entries' weights in merged order: which entries open a centroid.  The scale test reads
// weights only, so the means follow per centroid (td_centroid).  cstart[c] = the first entry of centroid c, cstart[count]
// = n; returns the count.
DPK_HD int td_fold_decide(const double *xw, int n, double total, int16_t *cstart) {
    if (n == 0) return 0;
    const double norm = td_norm(total), r = td_div(1.0, total);
    double W = xw[0], done = 0.0;
    int c = 0;
    cstart[0] = 0;
    for (int i = 1; i < n; i++) {
        if (td_fuses(W, xw[i], done, total, norm, r)) {
            W = td_add(W, xw[i]);
        } else {
            done = td_add(done, W);
            W = xw[i];
            cstart[++c] = (int16_t)i;
        }
    }
    cstart[c + 1] = (int16_t)n;
    return c + 1;
}
// The mean and weight of the centroid made of entries [s, e) (xw == NULL: every weight 1)
DPK_HD void td_centroid(const double *xm, const double *xw, int s, int e, double *m, double *W) {
    double mm = xm[s], ww = xw ? xw[s] : 1.0;
    for (int i = s + 1; i < e; i++) {
        const double w = xw ? xw[i] : 1.0;
        ww = td_add(ww, w);
        mm = td_mean_step(mm, xm[i], w, ww);
    }
    *m = mm;
    *W = ww;
}
// A centroid mean the next fold can take: not NaN and not below its predecessor.  Means of finite values never fall
// (each is a rounded point between its first and last entry); a NaN (inf - inf) or an overflowed x - m has no answer
// but the composition's.
DPK_HD bool td_mean_ok(double m, const double *prev) { return prev ? m >= *prev : m == m; }
// The whole fold in one pass (the two passes above interleaved) for one thread: centroids to (om, ow), which may alias
// (xm, xw) since centroid c is written after entry c is read.  *bad is set as by td_mean_ok.  Returns the count.
DPK_HD int td_fold_serial(const double *xm, const double *xw, int n, double total, double *om, double *ow, bool *bad) {
    if (n == 0) return 0;
    const double norm = td_norm(total), r = td_div(1.0, total);
    double m = xm[0], W = xw ? xw[0] : 1.0, done = 0.0, prev = 0.0;
    int c = 0;
    for (int i = 1; i < n; i++) {
        const double w = xw ? xw[i] : 1.0, x = xm[i];
        if (td_fuses(W, w, done, total, norm, r)) {
            W = td_add(W, w);
            m = td_mean_step(m, x, w, W);
        } else {
            *bad |= !td_mean_ok(m, c ? &prev : nullptr);
            om[c] = m; ow[c] = W; prev = m; c++;
            done = td_add(done, W);
            m = x; W = w;
        }
    }
    *bad |= !td_mean_ok(m, c ? &prev : nullptr);
    om[c] = m; ow[c] = W;
    return c + 1;
}
// Stable insertion sort of a short buffer by value (-0.0 and 0.0 compare equal and keep their order)
DPK_HD void td_sort_serial(double *v, int n) {
    for (int i = 1; i < n; i++) {
        const double x = v[i];
        int j = i;
        while (j > 0 && x < v[j - 1]) { v[j] = v[j - 1]; j--; }
        v[j] = x;
    }
}
// Merged order of a fold: incoming entries (sorted) before old centroids (sorted) among equal means.  Incoming entry x
// lands at its index + the old means below x; old mean y at its index + the incoming means <= y.
DPK_HD int td_count_below(const double *v, int n, double x) {      // entries < x
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (v[mid] < x) lo = mid + 1; else hi = mid; }
    return lo;
}
DPK_HD int td_count_upto(const double *v, int n, double x) {       // entries <= x
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (!(x < v[mid])) lo = mid + 1; else hi = mid; }
    return lo;
}
// Entries one buffer takes before the add path folds: len(buf) + len(centroids) reaches TD_CAP first (at least one, as
// MergingDigest.add appends after a compress that may leave TD_CAP centroids)
DPK_HD int td_buffer_len(int C, int64_t left) {
    const int64_t b = C < TD_CAP ? TD_CAP - C : 1;
    return (int)(left < b ? left : b);
}
DPK_HD double td_between(double x1, double w1, double x2, double w2) {
    const double lo = td_min(x1, x2), hi = td_max(x1, x2);
    return td_max(lo, td_min(hi, td_div(td_add(td_mul(x1, w1), td_mul(x2, w2)), td_add(w1, w2))));
}
// MergingDigest.quantile(q) of a compressed digest: c centroids, merged weight mw, lo / hi the extreme means seen
DPK_HD double td_quantile(const double *ms, const double *ws, int c, double mw, double lo, double hi, double q) {
    if (c == 0) return NAN;
    if (c == 1) return ms[0];
    const double target = td_mul(q, mw);
    if (target < td_div(ws[0], 2.0)) return td_add(lo, td_mul(td_div(td_mul(2.0, target), ws[0]), td_sub(ms[0], lo)));
    double seen = td_div(ws[0], 2.0);
    for (int i = 0; i < c - 1; i++) {
        const double end = td_add(seen, td_div(td_add(ws[i], ws[i + 1]), 2.0));
        if (end > target) return td_between(ms[i], td_sub(end, target), ms[i + 1], td_sub(target, seen));
        seen = end;
    }
    const double left = td_sub(td_sub(target, mw), td_div(ws[c - 1], 2.0));
    return td_between(ms[c - 1], left, hi, td_sub(td_div(ws[c - 1], 2.0), left));
}

// ------------------------------------------------------------- f8: Bernoulli sample (dpk_sample.cu; tests/samplecheck.cu
// runs the same functions on the CPU).  SampleRDD keeps row j of split i when the j-th random.Random(seed + i).random()
// is <= frac.  That generator is CPython's MT19937 (Modules/_randommodule.c): exact integer arithmetic, replayed here
// word for word from the 624-word state random.Random(seed + i).getstate() holds right after seeding (pos = 624, so the
// first draw twists).  A twist rewrites mt[0..624) in index order; it runs in three phases whose elements depend only on
// words of earlier phases or not yet rewritten ones:
//   [0, 227)   : mt[i + 1] and mt[i + 397], all old;
//   [227, 454) : mt[i + 1] old, mt[i - 227] from phase 1;
//   [454, 624) : mt[i + 1] old except the new mt[0] for i = 623, mt[i - 227] from phase 2.
// Within a phase element i reads the old mt[i + 1] that element i + 1 rewrites, so every read precedes every write.
constexpr int MT_N = 624, MT_M = 397;
constexpr int MT_DRAWS = MT_N / 2;     // random() takes two words; a twist yields 312 draws and no pair straddles two
DPK_HD int mt_phase(int p) { return p < 3 ? p * (MT_N - MT_M) : MT_N; }   // phase p covers [mt_phase(p), mt_phase(p + 1))
DPK_HD uint32_t mt_twist_elem(const uint32_t *mt, int i) {
    const uint32_t y = (mt[i] & 0x80000000u) | (mt[i + 1 == MT_N ? 0 : i + 1] & 0x7fffffffu);
    const int far = i + MT_M < MT_N ? i + MT_M : i + MT_M - MT_N;
    return mt[far] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}
DPK_HD uint32_t mt_temper(uint32_t y) {
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    return y ^ (y >> 18);
}
// random_random: (a * 2^26 + b) / 2^53 with a = w0 >> 5, b = w1 >> 6.  Every step is exact (a * 2^26 + b < 2^53), so a
// contracted FMA gives the same double.
DPK_HD double mt_double(uint32_t w0, uint32_t w1) {
    return ((double)(w0 >> 5) * 67108864.0 + (double)(w1 >> 6)) * (1.0 / 9007199254740992.0);
}
// rd.random() <= frac as Python compares two floats: a NaN frac keeps nothing
DPK_HD bool sample_keep(double u, double frac) { return u <= frac; }

// ------------------------------------------------------------- f9: top / hot select and the uniq table (dpk_select.cu;
// tests/selectcheck.cu runs the same functions on the CPU)
// The n smallest rows by (w0[, w1], row id) of unsigned 64-bit order words (sort_word), found by an MSD radix select:
// each round takes one 8-bit digit of the current word over the candidates, picks the bucket holding the need-th
// smallest, and keeps that bucket's rows as the next candidates.  Per bucket the round also ORs and ANDs the words, so
// the bits in which the bucket's rows differ are known: the next digit starts at the highest of them, and when none is
// left the word of the threshold row is exact.  A round therefore fixes at least 8 more bits or finishes a word: at most
// 8 rounds per word.
constexpr int SEL_BITS = 8, SEL_BUCKETS = 1 << SEL_BITS;
DPK_HD uint32_t sel_digit(uint64_t w, int32_t shift) { return (uint32_t)(w >> shift) & (SEL_BUCKETS - 1); }
// the bucket that holds the need-th smallest (1 <= need <= sum of hist): the first b with hist[0..b] >= need;
// *below = hist[0..b), the candidates in lower buckets
DPK_HD int32_t sel_bucket(const int64_t *hist, int64_t need, int64_t *below) {
    int64_t cum = 0;
    int32_t b = 0;
    for (; b < SEL_BUCKETS - 1 && cum + hist[b] < need; b++) cum += hist[b];
    *below = cum;
    return b;
}
// the next round's shift given the bits below the current digit in which the chosen bucket's rows differ (nonzero):
// the digit whose top bit is the highest of them, clamped at bit 0
DPK_HD int32_t sel_next_shift(uint64_t diff) {
    int32_t hb = 63;
    while (!((diff >> hb) & 1)) hb--;
    return hb >= SEL_BITS - 1 ? hb - (SEL_BITS - 1) : 0;
}
// (w0, w1) against the threshold (t0, t1) with nw words: < 0 below, 0 equal, > 0 above (sort_cmp)
DPK_HD int sel_cmp(uint64_t w0, uint64_t w1, uint64_t t0, uint64_t t1, int32_t nw) { return sort_cmp(w0, w1, t0, t1, nw); }
// The select state (int64 [SEL_STATE]): the current word and digit shift, the rank sought among the candidates, the
// rows already below the threshold, the chosen bucket's size, the threshold words, done, and the rule the chosen
// bucket's rows match (word, mask, value: (w & mask) == value); ST_OUT is the compaction's counter.
enum { ST_WORD, ST_SHIFT, ST_NEED, ST_BELOW, ST_COUNT, ST_T0, ST_T1, ST_DONE, ST_MWORD, ST_MMASK, ST_MVAL, ST_OUT,
       SEL_STATE = 16 };
// One round's decision from its histogram hist[3 * SEL_BUCKETS] (counts, ORs, ANDs of the candidates' words per
// bucket); clears the histogram for the next round (ANDs to all ones).
DPK_HD void sel_pick(int64_t *st, uint64_t *hist, int32_t nw) {
    int64_t below;
    const int32_t b = sel_bucket(reinterpret_cast<const int64_t *>(hist), st[ST_NEED], &below);
    const int32_t wi = (int32_t)st[ST_WORD], shift = (int32_t)st[ST_SHIFT];
    // the candidates agree on the bits above the digit (earlier rounds), so the bucket's rows agree on every bit >= shift
    const uint64_t hi = ~0ull << shift;
    const uint64_t orb = hist[SEL_BUCKETS + b], andb = hist[2 * SEL_BUCKETS + b];
    const uint64_t diff = (orb ^ andb) & ~hi;
    st[ST_BELOW] += below;
    st[ST_NEED] -= below;
    st[ST_COUNT] = (int64_t)hist[b];
    st[ST_MWORD] = wi;
    st[ST_T0 + wi] = (int64_t)andb;                      // exact once diff is 0; its bits >= shift are final already
    if (diff == 0) {                                     // the bucket's rows agree on the whole word
        st[ST_MMASK] = (int64_t)~0ull;
        if (wi + 1 < nw) {
            st[ST_WORD] = wi + 1;
            st[ST_SHIFT] = 64 - SEL_BITS;
        } else {
            st[ST_DONE] = 1;
        }
    } else {
        st[ST_MMASK] = (int64_t)hi;
        st[ST_SHIFT] = sel_next_shift(diff);
    }
    st[ST_MVAL] = (int64_t)(andb & (uint64_t)st[ST_MMASK]);
    st[ST_OUT] = 0;
    for (int j = 0; j < SEL_BUCKETS; j++) {
        hist[j] = 0;
        hist[SEL_BUCKETS + j] = 0;
        hist[2 * SEL_BUCKETS + j] = ~0ull;
    }
}

// uniq: a row's (k, v) pair as the distinct table compares it.  Each element widened as Python sees it (sort_wide_bits:
// ints to int64, floats to float64) and, for floats, -0.0 spelled 0.0 (Python's dict finds (0.0, v) under (-0.0, v)).
// False for a NaN in either element, which no dict lookup finds (the caller raises).  An int column and a float column
// never share a table, so int bits and float bits never meet.
DPK_HD uint64_t uniq_canon(uint64_t wide_bits, bool is_float) {
    return is_float && wide_bits == (1ull << 63) ? 0ull : wide_bits;
}
DPK_HD bool uniq_pair_bits(const void *keys, int32_t kkind, const void *vals, int32_t vkind, int64_t i, uint64_t *kb,
                           uint64_t *vb) {
    const bool fk = sort_kind_float(kkind), fv = sort_kind_float(vkind);
    const uint64_t a = sort_wide_bits(keys, kkind, i), b = sort_wide_bits(vals, vkind, i);
    *kb = uniq_canon(a, fk);
    *vb = uniq_canon(b, fv);
    return !((fk && sort_is_nan(a)) || (fv && sort_is_nan(b)));
}
// The table: bcast_slots(n) slots of {owner, count}, linear probing.  owner is UNIQ_EMPTY or the id of a row holding
// the slot's pair -- the pair lives in the input columns, never in the table, so a claim is one 32-bit CAS and nothing
// is published after it.  Race-free: an owner goes only from UNIQ_EMPTY to a row id and then to smaller ids of rows
// with the same pair, and claims are never undone, so every row of a pair stops at the same slot (the first one of its
// probe sequence that is empty or holds the pair when reached) and the final owner is the pair's first row.
constexpr int32_t UNIQ_EMPTY = 0x7FFFFFFF;     // above every row id (n < 2^31 - 1 rows)
struct __align__(8) UniqSlot {
    int32_t owner;
    uint32_t count;
};
// a pair's first slot: both words mixed (mix64), the value word first so (a, b) and (b, a) part
DPK_HD uint64_t uniq_slot(uint64_t kb, uint64_t vb, uint64_t mask) { return mix64(kb ^ mix64(vb + 0x9E3779B97F4A7C15ull)) & mask; }
// Row i (pair kb, vb) into the table: claim the first empty slot of its probe sequence, or join the slot whose owner
// row holds the same pair.  On the device the claim is a CAS and the join an atomicMin / atomicAdd.
DPK_HD void uniq_insert_row(UniqSlot *table, uint64_t mask, const void *keys, int32_t kkind, const void *vals,
                            int32_t vkind, int32_t i, uint64_t kb, uint64_t vb) {
    for (uint64_t s = uniq_slot(kb, vb, mask);; s = (s + 1) & mask) {
#ifdef __CUDA_ARCH__
        int32_t o = *reinterpret_cast<volatile int32_t *>(&table[s].owner);
        if (o == UNIQ_EMPTY) {
            o = atomicCAS(&table[s].owner, UNIQ_EMPTY, i);
            if (o == UNIQ_EMPTY) {
                atomicAdd(&table[s].count, 1u);
                return;
            }
        }
#else
        const int32_t o = table[s].owner;
        if (o == UNIQ_EMPTY) {
            table[s].owner = i;
            table[s].count = 1;
            return;
        }
#endif
        uint64_t ok, ov;
        uniq_pair_bits(keys, kkind, vals, vkind, o, &ok, &ov);
        if (ok == kb && ov == vb) {
#ifdef __CUDA_ARCH__
            if (i < o) atomicMin(&table[s].owner, i);
            atomicAdd(&table[s].count, 1u);
#else
            if (i < o) table[s].owner = i;
            table[s].count++;
#endif
            return;
        }
    }
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

// ------------------------------------------------------------- f4: UTF-8 tokeniser arithmetic (dpk_strings.cu k_tok8_*)
// str.split() without arguments on text decoded with strict utf-8: whitespace = the code points c with
// chr(c).isspace(): U+0009..000D, U+001C..0020, U+0085, U+00A0, U+1680, U+2000..200A, U+2028, U+2029, U+202F, U+205F,
// U+3000 -- UTF-8 forms of 1, 2 or 3 bytes, each beginning with a lead byte, so none matches from the middle of
// another code point.  A token = a maximal run of non-whitespace code points.

// length of the whitespace code point whose UTF-8 form begins c0 c1 c2; 0: the code point there is not whitespace
__host__ __device__ __forceinline__ int tok8_ws(uint32_t c0, uint32_t c1, uint32_t c2) {
    if (c0 < 0x80) return tok_ws((uint8_t)c0) ? 1 : 0;
    if (c0 == 0xC2) return (c1 == 0x85 || c1 == 0xA0) ? 2 : 0;                   // U+0085, U+00A0
    const uint32_t v = (c0 << 16) | (c1 << 8) | c2;
    const bool w = v == 0xE19A80u || v == 0xE38080u                               // U+1680, U+3000
                   || (v >= 0xE28080u && v <= 0xE2808Au)                         // U+2000..200A
                   || v == 0xE280A8u || v == 0xE280A9u || v == 0xE280AFu || v == 0xE2819Fu;   // U+2028 2029 202F 205F
    return w ? 3 : 0;
}

// is a whitespace code point's form at data[i] (bytes past n read as 0x00, which matches none)
__host__ __device__ __forceinline__ bool tok8_ws_at(const uint8_t *__restrict__ data, int64_t n, int64_t i) {
    const uint32_t c0 = data[i];
    if (c0 < 0x80) return tok_ws((uint8_t)c0);
    const uint32_t c1 = i + 1 < n ? data[i + 1] : 0u, c2 = i + 2 < n ? data[i + 2] : 0u;
    return tok8_ws(c0, c1, c2) != 0;
}

// the sequence length a byte announces: 1 ASCII, 0 continuation (10xxxxxx), 2 / 3 / 4 by its high bits
__host__ __device__ __forceinline__ int tok8_len(uint32_t c) { return c < 0x80 ? 1 : c < 0xC0 ? 0 : c < 0xE0 ? 2 : c < 0xF0 ? 3 : 4; }

// strict UTF-8 (Unicode Table 3-7, what bytes.decode("utf-8") accepts): does the lead byte c0 begin a well-formed
// sequence with the bytes c1 c2 c3 after it?  Rejects C0, C1 and F5..FF, overlong 3- and 4-byte forms (E0 80..9F,
// F0 80..8F), surrogates (ED A0..BF), values above U+10FFFF (F4 90..BF) and a missing continuation byte.
__host__ __device__ __forceinline__ bool tok8_seq_ok(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
    const bool k2 = (c2 & 0xC0u) == 0x80u, k3 = (c3 & 0xC0u) == 0x80u;
    const uint32_t lo = c0 == 0xE0 ? 0xA0u : c0 == 0xF0 ? 0x90u : 0x80u;          // second byte's range
    const uint32_t hi = c0 == 0xED ? 0x9Fu : c0 == 0xF4 ? 0x8Fu : 0xBFu;
    const bool k1 = c1 >= lo && c1 <= hi;
    if (c0 < 0x80) return true;
    if (c0 < 0xC2) return false;                                                   // continuation, or overlong C0 / C1
    if (c0 < 0xE0) return k1;
    if (c0 < 0xF0) return k1 && k2;
    if (c0 < 0xF5) return k1 && k2 && k3;
    return false;
}

// The per-thread step of k_tok8_count / k_tok8_emit over data[i0, i0 + 16): bit j of the result = a token starts at
// byte i0 + j (a non-whitespace code point's lead byte after a whitespace code point or at byte 0); *bad = some byte
// of the slice is ill-formed: a lead byte that does not begin a well-formed sequence inside [0, n), or a
// continuation byte that no lead byte at most 3 bytes before it announces (with every lead byte checked, that is a
// continuation byte outside any sequence).  Reads 3 bytes before the slice (the whitespace code point that may end
// just before it, the lead of a sequence running into it) and 3 after (the sequences that begin in it).
__host__ __device__ __forceinline__ uint32_t tok8_starts16(const uint8_t *__restrict__ data, int64_t n, int64_t i0, bool *bad) {
    uint8_t c[3 + TK_BYTES + 3];                     // c[k] = data[i0 - 3 + k], 0x00 outside [0, n)
    if (i0 >= 4 && i0 + TK_BYTES + 4 <= n && (((uintptr_t)(data + i0)) & 15u) == 0) {
        const uint32_t b = *reinterpret_cast<const uint32_t *>(data + i0 - 4);
        const uint4 q = *reinterpret_cast<const uint4 *>(data + i0);
        const uint32_t a = *reinterpret_cast<const uint32_t *>(data + i0 + TK_BYTES);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int k = 0; k < 3; k++) c[k] = (uint8_t)(b >> ((k + 1) * 8));
#pragma unroll
        for (int j = 0; j < TK_BYTES; j++) c[3 + j] = (uint8_t)(w[j >> 2] >> ((j & 3) * 8));
#pragma unroll
        for (int k = 0; k < 3; k++) c[3 + TK_BYTES + k] = (uint8_t)(a >> (k * 8));
    } else {
#pragma unroll
        for (int k = 0; k < 3 + TK_BYTES + 3; k++) {
            const int64_t i = i0 - 3 + k;
            c[k] = i >= 0 && i < n ? data[i] : (uint8_t)0;
        }
    }
    // l1 / l2 / l3: tok8_ws at the 1st / 2nd / 3rd byte before the current one; a whitespace code point ends just
    // before byte j exactly when l1 == 1, l2 == 2 or l3 == 3
    int l3 = tok8_ws(c[0], c[1], c[2]), l2 = tok8_ws(c[1], c[2], c[3]), l1 = tok8_ws(c[2], c[3], c[4]);
    uint32_t m = 0;
    bool b = false;
#pragma unroll
    for (int j = 0; j < TK_BYTES; j++) {
        const int k = 3 + j;
        const int l0 = tok8_ws(c[k], c[k + 1], c[k + 2]);
        if (i0 + j < n) {
            const bool lead = (c[k] & 0xC0u) != 0x80u;
            if (lead) {
                b |= !tok8_seq_ok(c[k], c[k + 1], c[k + 2], c[k + 3]);
                if (l0 == 0 && (i0 + j == 0 || l1 == 1 || l2 == 2 || l3 == 3)) m |= 1u << j;
            } else {
                b |= !(tok8_len(c[k - 1]) >= 2 || tok8_len(c[k - 2]) >= 3 || tok8_len(c[k - 3]) >= 4);
            }
        }
        l3 = l2;
        l2 = l1;
        l1 = l0;
    }
    *bad = b;
    return m;
}

// ------------------------------------------------------------- f10: numeric text columns (dpk_strings.cu k_tc_*;
// tests/numparsecheck.cu runs the same arithmetic on the CPU).  Every line either gets its final values here or is
// marked for the host, which runs Python's own line.split(sep) / int() / float() on it.  Accepted (ASCII only, after
// stripping \t \n \v \f \r and space -- what int() and float() strip; \x1c..\x1f they do not):
//   int   [+-]?[0-9]{1,19} whose value fits int64
//   float [+-]? digits with at most one '.' and at least one digit, then optionally [eE][+-]?[0-9]+; or inf, infinity,
//         nan in any case
// Everything else -- '_', a byte >= 0x80, more digits, a malformed or missing field -- goes to the host.

// bit j of the result: a line starts at byte i0 + j (byte 0, or the byte after a '\n', inside [0, n)); *hi |= any
// byte of the slice >= 0x80
__host__ __device__ __forceinline__ uint32_t tc_starts16(const uint8_t *__restrict__ data, int64_t n, int64_t i0, bool *hi) {
    uint8_t c[TK_BYTES];
    if (i0 + TK_BYTES <= n && (((uintptr_t)(data + i0)) & 15u) == 0) {
        const uint4 q = *reinterpret_cast<const uint4 *>(data + i0);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < TK_BYTES; j++) c[j] = (uint8_t)(w[j >> 2] >> ((j & 3) * 8));
    } else {
#pragma unroll
        for (int j = 0; j < TK_BYTES; j++) c[j] = i0 + j < n ? data[i0 + j] : (uint8_t)0;
    }
    bool after_nl = i0 == 0 || data[i0 - 1] == '\n';
    uint32_t m = 0;
    bool h = false;
#pragma unroll
    for (int j = 0; j < TK_BYTES; j++) {
        if (after_nl && i0 + j < n) m |= 1u << j;
        after_nl = c[j] == '\n';
        h |= c[j] >= 0x80;
    }
    *hi = h;
    return m;
}

// what int() and float() strip among ASCII bytes
__host__ __device__ __forceinline__ bool tc_space(uint32_t c) { return c == 0x20 || (c >= 0x09 && c <= 0x0d); }

__host__ __device__ __forceinline__ bool tc_digit(uint32_t c) { return c - '0' < 10u; }

__host__ __device__ __forceinline__ uint64_t tc_ld(const uint64_t *p) {
#ifdef __CUDA_ARCH__
    return __ldg(reinterpret_cast<const unsigned long long *>(p));
#else
    return *p;
#endif
}

__host__ __device__ __forceinline__ int tc_clz64(uint64_t x) {
#ifdef __CUDA_ARCH__
    return __clzll((long long)x);
#else
    return __builtin_clzll(x);
#endif
}

__host__ __device__ __forceinline__ void tc_mul128(uint64_t a, uint64_t b, uint64_t *hi, uint64_t *lo) {
#ifdef __CUDA_ARCH__
    *hi = __umul64hi(a, b);
    *lo = a * b;
#else
    const unsigned __int128 p = (unsigned __int128)a * b;
    *hi = (uint64_t)(p >> 64);
    *lo = (uint64_t)p;
#endif
}

// [*b, *e) without the strippable bytes at either end
__host__ __device__ __forceinline__ void tc_trim(const uint8_t *__restrict__ s, int64_t *b, int64_t *e) {
    while (*b < *e && tc_space(s[*b])) ++*b;
    while (*e > *b && tc_space(s[*e - 1])) --*e;
}

// int(s[b, e)) when the device grammar accepts it and the value fits int64
__host__ __device__ __forceinline__ bool tc_parse_i64(const uint8_t *__restrict__ s, int64_t b, int64_t e, int64_t *out) {
    tc_trim(s, &b, &e);
    bool neg = false;
    if (b < e && (s[b] == '+' || s[b] == '-')) neg = s[b++] == '-';
    if (e - b < 1 || e - b > 19) return false;
    uint64_t v = 0;                                  // 19 digits stay below 2^64
    for (int64_t p = b; p < e; p++) {
        const uint32_t d = (uint32_t)s[p] - '0';
        if (d >= 10u) return false;
        v = v * 10 + d;
    }
    if (v > (neg ? (1ull << 63) : (1ull << 63) - 1)) return false;
    *out = (int64_t)(neg ? 0 - v : v);
    return true;
}

// Eisel-Lemire (Lemire 2021, "Number parsing at a gigabyte per second", section 5): the binary64 bits (sign clear)
// nearest to w * 10^q, w != 0 a 64-bit decimal significand.  pow5 = dpk_pow5.inc (2 words per q in [-342, 308]).
// False: the truncated 128-bit product cannot decide the rounding.
__host__ __device__ __forceinline__ bool tc_eisel_lemire(int64_t q, uint64_t w, const uint64_t *__restrict__ pow5,
                                                         uint64_t *bits) {
    if (q < -342) { *bits = 0; return true; }
    if (q > 308) { *bits = 0x7FF0000000000000ull; return true; }
    const int lz = tc_clz64(w);
    w <<= lz;
    const int idx = 2 * (int)(q + 342);
    uint64_t hi, lo;
    tc_mul128(w, tc_ld(pow5 + idx), &hi, &lo);
    if ((hi & 0x1FF) == 0x1FF) {                     // the 9 bits below the 55 kept are all ones: refine
        uint64_t hi2, lo2;
        tc_mul128(w, tc_ld(pow5 + idx + 1), &hi2, &lo2);
        lo += hi2;
        if (hi2 > lo) hi++;
        if ((hi & 0x1FF) == 0x1FF && lo == ~0ull) return false;   // the product's error could still carry into hi
    }
    const int upper = (int)(hi >> 63);
    const int shift = upper + 9;
    uint64_t m = hi >> shift;
    int32_t p2 = (int32_t)(((217706 * (int32_t)q) >> 16) + 63) + upper - lz + 1023;   // floor(q log2(10)) + 63 + ...
    if (p2 <= 0) {                                   // subnormal, or below the least subnormal
        if (-p2 + 1 >= 64) { *bits = 0; return true; }
        m >>= -p2 + 1;
        m += m & 1;
        m >>= 1;
        *bits = m | ((uint64_t)(m < (1ull << 52) ? 0 : 1) << 52);
        return true;
    }
    // an exact halfway case can only occur for q in [-4, 23]: round it to even
    if (lo <= 1 && q >= -4 && q <= 23 && (m & 3) == 1 && (m << shift) == hi) m &= ~1ull;
    m += m & 1;
    m >>= 1;
    if (m >= (2ull << 52)) { m = 1ull << 52; p2++; }
    m &= ~(1ull << 52);
    if (p2 >= 0x7FF) { *bits = 0x7FF0000000000000ull; return true; }
    *bits = m | ((uint64_t)p2 << 52);
    return true;
}

// does s[b, e) spell `word` (lower case) in any case
__host__ __device__ __forceinline__ bool tc_word(const uint8_t *__restrict__ s, int64_t b, int64_t e, const char *word, int len) {
    if (e - b != len) return false;
    for (int k = 0; k < len; k++)
        if ((s[b + k] | 0x20) != (uint8_t)word[k]) return false;
    return true;
}

// the bits of float(s[b, e)) when the device grammar accepts it and the conversion can decide its rounding
__host__ __device__ __forceinline__ bool tc_parse_f64(const uint8_t *__restrict__ s, int64_t b, int64_t e,
                                                      const uint64_t *__restrict__ pow5, uint64_t *out) {
    tc_trim(s, &b, &e);
    uint64_t sign = 0;
    if (b < e && (s[b] == '+' || s[b] == '-')) sign = s[b++] == '-' ? 1ull << 63 : 0;
    if (b >= e) return false;
    if ((s[b] | 0x20) == 'i' || (s[b] | 0x20) == 'n') {
        if (tc_word(s, b, e, "inf", 3) || tc_word(s, b, e, "infinity", 8)) { *out = sign | 0x7FF0000000000000ull; return true; }
        if (tc_word(s, b, e, "nan", 3)) { *out = sign | 0x7FF8000000000000ull; return true; }
        return false;
    }
    // w = the first 19 significant digits, q = the decimal exponent of its last one; dropped = a nonzero digit
    // past those 19
    uint64_t w = 0;
    int nd = 0;
    int64_t q = 0;
    bool dropped = false, any = false;
    for (; b < e && tc_digit(s[b]); b++) {
        const uint32_t d = s[b] - '0';
        any = true;
        if (nd == 0 && d == 0) continue;
        if (nd < 19) { w = w * 10 + d; nd++; } else { q++; dropped |= d != 0; }
    }
    if (b < e && s[b] == '.') {
        for (b++; b < e && tc_digit(s[b]); b++) {
            const uint32_t d = s[b] - '0';
            any = true;
            if (nd == 0 && d == 0) { q--; continue; }
            if (nd < 19) { w = w * 10 + d; nd++; q--; } else { dropped |= d != 0; }
        }
    }
    if (!any) return false;
    if (b < e && (s[b] | 0x20) == 'e') {
        b++;
        bool eneg = false;
        if (b < e && (s[b] == '+' || s[b] == '-')) eneg = s[b++] == '-';
        if (b >= e || !tc_digit(s[b])) return false;
        int64_t x = 0;
        for (; b < e && tc_digit(s[b]); b++) x = x < 1000000000000ll ? x * 10 + (s[b] - '0') : x;   // saturates far
        q += eneg ? -x : x;                                                                           // outside 10^308
    }
    if (b != e) return false;
    if (w == 0) { *out = sign; return true; }
    if (!dropped && q >= -22 && q <= 22 && w <= (1ull << 53)) {       // exact operands, one correctly rounded op
        double p = 1.0;
        for (int64_t k = q < 0 ? -q : q; k > 0; k--) p *= 10.0;        // 10^k, k <= 22, is exact
        const double v = q < 0 ? (double)w / p : (double)w * p;
        uint64_t vb;
        memcpy(&vb, &v, 8);
        *out = sign | vb;
        return true;
    }
    uint64_t lo;
    if (!tc_eisel_lemire(q, w, pow5, &lo)) return false;
    if (dropped) {                                   // the value lies in (w, w + 1) * 10^q: both ends must agree
        uint64_t hi;
        if (!tc_eisel_lemire(q, w + 1, pow5, &hi) || hi != lo) return false;
    }
    *out = sign | lo;
    return true;
}

// The fields k0 and k1 of the line s[b, e) as [f[0], f[1]) and [f[2], f[3]): line.split() (sep_len == 0: maximal runs
// of non-whitespace code points, tok8_ws) or line.split(sep) (the matches of sep[0, sep_len) from left to right,
// without overlap).  Walks no further than field max(k0, k1); false when the line has fewer fields.
__host__ __device__ __forceinline__ int tc_ws_len(const uint8_t *__restrict__ s, int64_t p, int64_t e) {
    const uint32_t c0 = s[p];
    if (c0 < 0x80) return tok_ws((uint8_t)c0) ? 1 : 0;
    return tok8_ws(c0, p + 1 < e ? s[p + 1] : 0u, p + 2 < e ? s[p + 2] : 0u);
}

__host__ __device__ __forceinline__ bool tc_fields(const uint8_t *__restrict__ s, int64_t b, int64_t e,
                                                   const uint8_t *__restrict__ sep, int32_t sep_len, int32_t k0,
                                                   int32_t k1, int64_t *f) {
    const int32_t last = k0 > k1 ? k0 : k1;
    int64_t p = b;
    for (int32_t fi = 0;; fi++) {
        int64_t fb, fe;
        bool more;
        if (sep_len == 0) {
            for (int l; p < e && (l = tc_ws_len(s, p, e)) != 0;) p += l;
            if (p >= e) return false;
            fb = p;
            while (p < e && tc_ws_len(s, p, e) == 0) p++;
            fe = p;
            more = true;
        } else {
            fb = p;
            const uint8_t s0 = sep[0];
            for (; p + sep_len <= e; p++) {
                if (s[p] != s0) continue;
                int32_t k = 1;
                while (k < sep_len && s[p + k] == sep[k]) k++;
                if (k == sep_len) break;
            }
            more = p + sep_len <= e;
            fe = more ? p : e;
            p = more ? p + sep_len : e;
        }
        if (fi == k0) { f[0] = fb; f[1] = fe; }
        if (fi == k1) { f[2] = fb; f[3] = fe; }
        if (fi == last) return true;
        if (!more) return false;
    }
}

// one line s[b, e): its key and value (int64 or float64 bits by kind DPK_K_I64 / DPK_K_F64); false = a host line
__host__ __device__ __forceinline__ bool tc_parse_field(const uint8_t *__restrict__ s, int64_t b, int64_t e, int32_t kind,
                                                        const uint64_t *__restrict__ pow5, int64_t *out) {
    if (kind == DPK_K_I64) return tc_parse_i64(s, b, e, out);
    uint64_t bits;
    if (!tc_parse_f64(s, b, e, pow5, &bits)) return false;
    *out = (int64_t)bits;
    return true;
}

__host__ __device__ __forceinline__ bool tc_line(const uint8_t *__restrict__ s, int64_t b, int64_t e,
                                                 const uint8_t *__restrict__ sep, int32_t sep_len, int32_t key,
                                                 int32_t value, int32_t key_kind, int32_t value_kind,
                                                 const uint64_t *__restrict__ pow5, int64_t *k, int64_t *v) {
    int64_t f[4];
    return tc_fields(s, b, e, sep, sep_len, key, value, f) && tc_parse_field(s, f[0], f[1], key_kind, pow5, k)
           && tc_parse_field(s, f[2], f[3], value_kind, pow5, v);
}


}  // namespace dpk
