// dpk_select.cu -- f9: top (dpark/rdd.py:387-394), uniq and hot (dpark/rdd.py:383-398) of a numeric (k, v) column pair.
//
//   k_sel_hist / k_sel_pick / k_sel_compact : one round of the MSD radix select (sel_*, dpk_common.cuh) over the
//       candidates: an 8-bit digit histogram with per-bucket OR / AND of the words (warp-aggregated: lanes with one digit
//       add once, lanes whose word equals the leader's skip the OR / AND); one thread's sel_pick; the chosen bucket's
//       candidates appended with one atomic per warp (their order is free: only histograms read them).
//   k_sel_tiles / k_sel_scan / k_sel_write : the stable compaction once the threshold T is exact.  Per 1024-row tile the
//       rows below / equal to T are counted, one block scans the tile counts, and each tile ranks its rows by warp
//       ballots in row order: a row below T goes to (rows below T before it) + min(rows equal to T before it, n - below).
//   k_uniq_insert / k_uniq_emit : the distinct table (uniq_insert_row; race-free by its owner rule, see there), then
//       every occupied slot's (owner, count).  A NaN in either element sets state[0] and the row is left out.
//
// Algorithmic bytes: a round 8 (word) + 8 (candidate id) read per candidate, compaction 8 written per kept candidate;
// the stable compaction 8 per word per row, read twice; insert K + V per row (the owner's pair and the slot are random
// reads, not credited); emit 8 per slot read, 16 per distinct pair written.
#include "dpk_common.cuh"

namespace dpk {

constexpr int SEL_THREADS = 256;
constexpr int SEL_WARPS = SEL_THREADS / 32;
constexpr int SEL_TILE = 4 * SEL_THREADS;     // rows per tile of the stable compaction
constexpr int SEL_SCAN_THREADS = 1024;
constexpr unsigned FULL = 0xFFFFFFFFu;

__global__ void __launch_bounds__(SEL_THREADS)
k_sel_hist(const uint64_t *__restrict__ w0, const uint64_t *__restrict__ w1, const int64_t *__restrict__ cands,
           int64_t m, const int64_t *__restrict__ st, unsigned long long *__restrict__ hist) {
    __shared__ unsigned long long sc[SEL_BUCKETS], so[SEL_BUCKETS], sa[SEL_BUCKETS];
    for (int b = threadIdx.x; b < SEL_BUCKETS; b += SEL_THREADS) { sc[b] = 0; so[b] = 0; sa[b] = ~0ull; }
    __syncthreads();
    const uint64_t *w = st[ST_WORD] ? w1 : w0;
    const int32_t shift = (int32_t)st[ST_SHIFT];
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * SEL_THREADS;
    for (int64_t base = (int64_t)blockIdx.x * SEL_THREADS + (threadIdx.x & ~31); base < m; base += stride) {
        const int64_t i = base + lane;
        const bool valid = i < m;
        uint64_t x = 0;
        uint32_t d = 0xFFFFFFFFu;
        if (valid) {
            x = w[cands ? cands[i] : i];
            d = sel_digit(x, shift);
        }
        const unsigned grp = __match_any_sync(FULL, d);
        const int leader = __ffs(grp) - 1;
        const uint64_t lx = __shfl_sync(FULL, x, leader);
        if (valid) {
            if (lane == leader) atomicAdd(&sc[d], (unsigned long long)__popc(grp));
            if (lane == leader || x != lx) {
                atomicOr(&so[d], (unsigned long long)x);
                atomicAnd(&sa[d], (unsigned long long)x);
            }
        }
    }
    __syncthreads();
    for (int b = threadIdx.x; b < SEL_BUCKETS; b += SEL_THREADS) {
        if (!sc[b]) continue;
        atomicAdd(&hist[b], sc[b]);
        atomicOr(&hist[SEL_BUCKETS + b], so[b]);
        atomicAnd(&hist[2 * SEL_BUCKETS + b], sa[b]);
    }
}

// one thread: the state is written by this kernel, read by the next ones and once per round by the host
__global__ void k_sel_pick(int64_t *__restrict__ st, unsigned long long *__restrict__ hist, int32_t nw) {
    sel_pick(st, reinterpret_cast<uint64_t *>(hist), nw);
}

__global__ void __launch_bounds__(SEL_THREADS)
k_sel_compact(const uint64_t *__restrict__ w0, const uint64_t *__restrict__ w1, const int64_t *__restrict__ cands,
              int64_t m, int64_t *__restrict__ st, int64_t *__restrict__ out) {
    const uint64_t *w = st[ST_MWORD] ? w1 : w0;
    const uint64_t mask = (uint64_t)st[ST_MMASK], val = (uint64_t)st[ST_MVAL];
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * SEL_THREADS;
    for (int64_t base = (int64_t)blockIdx.x * SEL_THREADS + (threadIdx.x & ~31); base < m; base += stride) {
        const int64_t i = base + lane;
        int64_t id = 0;
        bool keep = false;
        if (i < m) {
            id = cands ? cands[i] : i;
            keep = (w[id] & mask) == val;
        }
        const unsigned bal = __ballot_sync(FULL, keep);
        unsigned long long at = 0;
        if (lane == 0 && bal) at = atomicAdd(reinterpret_cast<unsigned long long *>(&st[ST_OUT]), (unsigned long long)__popc(bal));
        at = __shfl_sync(FULL, at, 0);
        if (keep) out[at + __popc(bal & ((1u << lane) - 1u))] = id;
    }
}

__device__ __forceinline__ int sel_row_cmp(const uint64_t *w0, const uint64_t *w1, int64_t i, uint64_t t0, uint64_t t1) {
    return sel_cmp(w0[i], w1 ? w1[i] : 0, t0, t1, w1 ? 2 : 1);
}

__global__ void __launch_bounds__(SEL_THREADS)
k_sel_tiles(const uint64_t *__restrict__ w0, const uint64_t *__restrict__ w1, int64_t n,
            const int64_t *__restrict__ st, int64_t *__restrict__ tile_lt, int64_t *__restrict__ tile_eq) {
    __shared__ int wl[SEL_WARPS], we[SEL_WARPS];
    const uint64_t t0 = (uint64_t)st[ST_T0], t1 = (uint64_t)st[ST_T1];
    const int64_t tile = blockIdx.x;
    int lt = 0, eq = 0;
#pragma unroll
    for (int j = 0; j < SEL_TILE / SEL_THREADS; j++) {
        const int64_t i = tile * SEL_TILE + j * SEL_THREADS + threadIdx.x;
        if (i < n) {
            const int c = sel_row_cmp(w0, w1, i, t0, t1);
            lt += c < 0;
            eq += c == 0;
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        lt += __shfl_xor_sync(FULL, lt, o);
        eq += __shfl_xor_sync(FULL, eq, o);
    }
    if ((threadIdx.x & 31) == 0) { wl[threadIdx.x >> 5] = lt; we[threadIdx.x >> 5] = eq; }
    __syncthreads();
    if (threadIdx.x == 0) {
        int a = 0, e = 0;
        for (int w = 0; w < SEL_WARPS; w++) { a += wl[w]; e += we[w]; }
        tile_lt[tile] = a;
        tile_eq[tile] = e;
    }
}

// exclusive scan in place of two arrays of len entries (one block: each thread a contiguous chunk, then a block scan
// of the chunk sums)
__global__ void __launch_bounds__(SEL_SCAN_THREADS)
k_sel_scan(int64_t *__restrict__ a, int64_t *__restrict__ b, int64_t len) {
    __shared__ int64_t sa[SEL_SCAN_THREADS], sb[SEL_SCAN_THREADS];
    const int t = threadIdx.x;
    const int64_t per = (len + SEL_SCAN_THREADS - 1) / SEL_SCAN_THREADS;
    const int64_t lo = t * per < len ? t * per : len, hi = lo + per < len ? lo + per : len;
    int64_t x = 0, y = 0;
    for (int64_t i = lo; i < hi; i++) { x += a[i]; y += b[i]; }
    sa[t] = x;
    sb[t] = y;
    __syncthreads();
    for (int o = 1; o < SEL_SCAN_THREADS; o <<= 1) {     // Hillis-Steele, inclusive
        const int64_t px = t >= o ? sa[t - o] : 0, py = t >= o ? sb[t - o] : 0;
        __syncthreads();
        sa[t] += px;
        sb[t] += py;
        __syncthreads();
    }
    x = sa[t] - x;
    y = sb[t] - y;
    for (int64_t i = lo; i < hi; i++) {
        const int64_t ca = a[i], cb = b[i];
        a[i] = x;
        b[i] = y;
        x += ca;
        y += cb;
    }
}

__global__ void __launch_bounds__(SEL_THREADS)
k_sel_write(const uint64_t *__restrict__ w0, const uint64_t *__restrict__ w1, int64_t n, int64_t take,
            const int64_t *__restrict__ st, const int64_t *__restrict__ lt_off, const int64_t *__restrict__ eq_off,
            int64_t *__restrict__ out) {
    __shared__ int wl[SEL_WARPS], we[SEL_WARPS];
    const uint64_t t0 = (uint64_t)st[ST_T0], t1 = (uint64_t)st[ST_T1];
    const int64_t tile = blockIdx.x, take_eq = take - st[ST_BELOW];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned before_me = (1u << lane) - 1u;
    int64_t lt_base = lt_off[tile], eq_base = eq_off[tile];
    for (int j = 0; j < SEL_TILE / SEL_THREADS; j++) {
        const int64_t i = tile * SEL_TILE + j * SEL_THREADS + threadIdx.x;
        const int c = i < n ? sel_row_cmp(w0, w1, i, t0, t1) : 1;
        const unsigned bl = __ballot_sync(FULL, c < 0), be = __ballot_sync(FULL, c == 0);
        if (lane == 0) { wl[warp] = __popc(bl); we[warp] = __popc(be); }
        __syncthreads();
        int pl = 0, pe = 0, tl = 0, te = 0;
#pragma unroll
        for (int w = 0; w < SEL_WARPS; w++) {
            pl += w < warp ? wl[w] : 0;
            pe += w < warp ? we[w] : 0;
            tl += wl[w];
            te += we[w];
        }
        const int64_t lt_rank = lt_base + pl + __popc(bl & before_me), eq_rank = eq_base + pe + __popc(be & before_me);
        if (c < 0) out[lt_rank + (eq_rank < take_eq ? eq_rank : take_eq)] = i;
        else if (c == 0 && eq_rank < take_eq) out[lt_rank + eq_rank] = i;
        lt_base += tl;
        eq_base += te;
        __syncthreads();                                 // wl / we are rewritten in the next step
    }
}

__global__ void __launch_bounds__(SEL_THREADS)
k_uniq_insert(const void *__restrict__ keys, int32_t kkind, const void *__restrict__ vals, int32_t vkind, int64_t n,
              UniqSlot *__restrict__ table, uint64_t mask, int64_t *__restrict__ st) {
    bool nan = false;
    const int64_t stride = (int64_t)gridDim.x * SEL_THREADS;
    for (int64_t i = (int64_t)blockIdx.x * SEL_THREADS + threadIdx.x; i < n; i += stride) {
        uint64_t kb, vb;
        if (!uniq_pair_bits(keys, kkind, vals, vkind, i, &kb, &vb)) {
            nan = true;
            continue;
        }
        uniq_insert_row(table, mask, keys, kkind, vals, vkind, (int32_t)i, kb, vb);
    }
    if (__syncthreads_or(nan) && threadIdx.x == 0) st[0] = 1;
}

__global__ void __launch_bounds__(SEL_THREADS)
k_uniq_emit(const UniqSlot *__restrict__ table, int64_t nslots, int64_t *__restrict__ out_first,
            int64_t *__restrict__ out_count, int64_t *__restrict__ st) {
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * SEL_THREADS;
    for (int64_t base = (int64_t)blockIdx.x * SEL_THREADS + (threadIdx.x & ~31); base < nslots; base += stride) {
        const int64_t s = base + lane;
        UniqSlot e = {UNIQ_EMPTY, 0};
        if (s < nslots) e = table[s];
        const bool keep = e.owner != UNIQ_EMPTY;
        const unsigned bal = __ballot_sync(FULL, keep);
        unsigned long long at = 0;
        if (lane == 0 && bal) at = atomicAdd(reinterpret_cast<unsigned long long *>(&st[1]), (unsigned long long)__popc(bal));
        at = __shfl_sync(FULL, at, 0);
        if (keep) {
            const int64_t p = (int64_t)at + __popc(bal & ((1u << lane) - 1u));
            out_first[p] = e.owner;
            out_count[p] = e.count;
        }
    }
}

static bool sel_kind_ok(int32_t kind) {
    return kind == DPK_K_I64 || kind == DPK_K_I32 || kind == DPK_K_F64 || kind == DPK_K_F32;
}

static unsigned sel_blocks(int64_t n) {
    int64_t g = (n + SEL_THREADS - 1) / SEL_THREADS;
    const int64_t cap = (int64_t)sm_count() * 16;
    return (unsigned)(g < 1 ? 1 : g > cap ? cap : g);
}

}  // namespace dpk

using namespace dpk;

extern "C" {

int dpk_select_round(const int64_t *w0, const int64_t *w1, const int64_t *cands, int64_t m, int64_t *state,
                     int64_t *hist, dpk_stream_t stream) {
    if (m <= 0 || m >= (1ll << 31)) return fail(DPK_ERR_INVALID, "m=%lld (1 .. 2^31 - 1 candidates)", (long long)m);
    if (!w0 || !state || !hist) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    DPK_LAUNCH("select_hist", st, k_sel_hist<<<sel_blocks(m), SEL_THREADS, 0, st>>>(
        (const uint64_t *)w0, (const uint64_t *)w1, cands, m, state, (unsigned long long *)hist));
    DPK_LAUNCH("select_pick", st, k_sel_pick<<<1, 1, 0, st>>>(state, (unsigned long long *)hist, w1 ? 2 : 1));
    return DPK_OK;
}

int dpk_select_compact(const int64_t *w0, const int64_t *w1, const int64_t *cands, int64_t m, int64_t *state,
                       int64_t *out_cands, dpk_stream_t stream) {
    if (m <= 0 || m >= (1ll << 31)) return fail(DPK_ERR_INVALID, "m=%lld (1 .. 2^31 - 1 candidates)", (long long)m);
    if (!w0 || !state || !out_cands) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    DPK_LAUNCH("select_compact", st, k_sel_compact<<<sel_blocks(m), SEL_THREADS, 0, st>>>(
        (const uint64_t *)w0, (const uint64_t *)w1, cands, m, state, out_cands));
    return DPK_OK;
}

int64_t dpk_select_tiles(int64_t n) { return n <= 0 ? 0 : (n + SEL_TILE - 1) / SEL_TILE; }

int dpk_select_take(const int64_t *w0, const int64_t *w1, int64_t n, int64_t take, const int64_t *state,
                    int64_t *tile_lt, int64_t *tile_eq, int64_t *out_ids, dpk_stream_t stream) {
    if (n <= 0 || n >= (1ll << 31) || take <= 0 || take > n)
        return fail(DPK_ERR_INVALID, "n=%lld take=%lld (1 <= take <= n < 2^31)", (long long)n, (long long)take);
    if (!w0 || !state || !tile_lt || !tile_eq || !out_ids) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t tiles = dpk_select_tiles(n);
    DPK_LAUNCH("select_tiles", st, k_sel_tiles<<<(unsigned)tiles, SEL_THREADS, 0, st>>>(
        (const uint64_t *)w0, (const uint64_t *)w1, n, state, tile_lt, tile_eq));
    DPK_LAUNCH("select_scan", st, k_sel_scan<<<1, SEL_SCAN_THREADS, 0, st>>>(tile_lt, tile_eq, tiles));
    DPK_LAUNCH("select_write", st, k_sel_write<<<(unsigned)tiles, SEL_THREADS, 0, st>>>(
        (const uint64_t *)w0, (const uint64_t *)w1, n, take, state, tile_lt, tile_eq, out_ids));
    return DPK_OK;
}

int dpk_uniq_insert(const void *keys, int32_t key_kind, const void *vals, int32_t val_kind, int64_t n, void *table,
                    int64_t nslots, int64_t *state, dpk_stream_t stream) {
    if (n < 0 || n >= (1ll << 31) - 1) return fail(DPK_ERR_INVALID, "n=%lld (0 .. 2^31 - 2)", (long long)n);
    if (!sel_kind_ok(key_kind) || !sel_kind_ok(val_kind))
        return fail(DPK_ERR_UNSUPPORTED, "column kinds %d, %d (int32 / int64 / float32 / float64)", key_kind, val_kind);
    if (nslots != (int64_t)bcast_slots(n))
        return fail(DPK_ERR_INVALID, "nslots=%lld (want %llu)", (long long)nslots, (unsigned long long)bcast_slots(n));
    if (n == 0) return DPK_OK;
    if (!keys || !vals || !table || !state) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    DPK_LAUNCH("uniq_insert", st, k_uniq_insert<<<sel_blocks(n), SEL_THREADS, 0, st>>>(
        keys, key_kind, vals, val_kind, n, (UniqSlot *)table, (uint64_t)nslots - 1, state));
    return DPK_OK;
}

int dpk_uniq_emit(const void *table, int64_t nslots, int64_t *out_first, int64_t *out_count, int64_t *state,
                  dpk_stream_t stream) {
    if (nslots < 2 || (nslots & (nslots - 1))) return fail(DPK_ERR_INVALID, "nslots=%lld (a power of two)", (long long)nslots);
    if (!table || !out_first || !out_count || !state) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    DPK_LAUNCH("uniq_emit", st, k_uniq_emit<<<sel_blocks(nslots), SEL_THREADS, 0, st>>>(
        (const UniqSlot *)table, nslots, out_first, out_count, state));
    return DPK_OK;
}

}  // extern "C"
