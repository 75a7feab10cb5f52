// dpk_partition.cu -- map side of the shuffle: ShuffleMapTask._run's
// hash-partition (dpark/task.py:209-226, dpark/dependency.py:229-233) as a
// STABLE multisplit of a columnar chunk into P bucket-major ranges.
//
// Data layout in HBM: struct-of-arrays.  keys[n], vals[n] in; out_keys[*],
// out_vals[*] bucket-major (bucket p occupies [base[p], base[p]+count[p])), rows
// of a bucket in input order.  The bucket-major buffer IS the alltoallv send
// buffer (buckets owned by one peer are adjacent).
//
// Kernels (HBM-bound integer work, no tensor cores):
//   k_part_count   : each CTA owns one contiguous row range of the grid, hashes keys, counts rows per
//                    bucket (warp-private shared-memory histograms) -> tile_counts[P][T].
//   k_part_scan    : per bucket, exclusive scan over the T CTAs.
//   k_part_scatter : each CTA re-reads its range tile by tile (4096 rows): fused hash -> bucket ->
//                    rank inside the tile -> block multisplit in shared memory -> run-wise coalesced
//                    stores to HBM.  Ranking is STABLE by default (warp match + leader: rows of a bucket
//                    stay in input order, what groupByKey and the LSD radix passes need) or, with
//                    DPK_K_UNORDERED, one native shared-memory atomic per row (reduceByKey paths).
// Modes of the same kernels: plain (one chunk of rows -> bucket-major output), pointer (every bucket has
// its own destination address, possibly peer-GPU memory: dpk_partition_scatter_ptrs), segmented (the grid
// runs over a device-built chunk table and splits every first-level bucket again: seg_multisplit, the
// first stage of the reduce side), radix digit (dpk_radix_pass).
// Algorithmic bytes: 2*(K+V) per row (read once, write once); this two-pass form re-reads K once more
// for the histogram (not credited).
#include "dpk_common.cuh"

namespace dpk {

constexpr int PT_THREADS = 256;
constexpr int PT_WARPS = PT_THREADS / 32;
constexpr int PT_ITEMS = 16;
constexpr int PT_TILE = PT_THREADS * PT_ITEMS;  // 4096 rows per tile
constexpr int PT_COUNT_PRIV = 1024;             // k_part_count: warp-private histograms up to this many buckets

struct NoVal {};

// dpk_set_option("count_mode"): 1 (default) = one shared-memory atomic per row into a warp-private
// histogram; 0 = warp peer mask + leader update (slower: 0.83 vs 0.34 ms per 1e8 rows on an H100, C2 map side)
int g_count_mode = 1;
int g_scatter_items = 16;
// dpk_set_option("scatter_bulk"): 1 (default) = unordered multisplits run k_part_scatter_bulk (CTA-wide
// shared-memory ranking + TMA bulk stores of the staged bucket runs); 0 = the round-1 kernel (A/B switch)
int g_scatter_bulk = 1;
int g_scatter_threads = 512;
int g_scatter_seg_wide = 1;
// dpk_set_option("scatter_ptr_bulk"): 1 (default) = the fused scatter + exchange (pointer mode) runs the TMA bulk-store
// kernel for unordered multisplits; 0 = the round-1 kernel (per-thread 8-byte stores over NVLink).
// dpk_set_option("scatter_ptr_threads"): CTA size of the bulk kernel in pointer mode: 1024 (default; 8192-row tiles: the
// bucket runs that cross NVLink are twice as long) or 512
int g_scatter_wide_from = 512;   // dpk_set_option("scatter_wide_from"): bucket count from which plain launches use 8192-row tiles (0 = never)
int g_scatter_ptr_bulk = 1;
int g_scatter_ptr_threads = 1024;   // dpk_set_option("scatter_seg_wide"): segmented launches use the 1024-thread / 8192-row form

// Segmented mode (second-level split on the reduce side): the grid runs over a
// device-resident chunk table instead of equal row ranges; every chunk lies inside
// one first-level bucket and is split by OTHER hash bits into f.nbuckets() fine
// buckets.  Counts / offsets are chunk-major [chunk][bucket].  All pointers null =
// plain mode.
struct SegTab {
    const int64_t *cbeg, *cend;     // row range of chunk c
    const int32_t *ctotal;          // number of chunks (device)
    int32_t *chunk_counts;          // [chunk][F]   (count kernel writes)
    const int64_t *chunk_off;       // [chunk][F]   absolute output position (scatter kernel reads)
    // Pointer mode (fused scatter + exchange): bucket b of this chunk is written to the memory at
    // key_ptrs[b] / val_ptrs[b] -- absolute device addresses, which may be peer-GPU memory mapped
    // over NVLink -- at element offset (rows of b in earlier CTAs of this chunk) + rank.
    const uint64_t *key_ptrs, *val_ptrs;
    // rows of a bucket may come out in any order (DPK_K_UNORDERED): cheaper ranking in the scatter
    int unordered;
};

struct Plan {
    int32_t T;  // CTAs (row ranges, or the chunk-table upper bound in segmented mode)
    int64_t L;  // rows per CTA, multiple of PT_TILE
    SegTab seg;
    const char *label_count = nullptr, *label_scatter = nullptr;  // profiling labels (default: part_* / seg_*)
    int pack = 0;   // PK_IN | PK_OUT: packed rows in / out (same-width key and value columns)
};

static Plan make_plan(int64_t n) {
    Plan pl;
    pl.seg = SegTab{nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0};
    // CTA c owns the tiles [c*tiles/T, (c+1)*tiles/T): contiguous (stability), evenly spread
    // (every CTA gets floor or ceil of tiles/T), T a multiple of the SM count when there is
    // enough work.  pl.L carries the TOTAL tile count.
    int64_t tiles = (n + PT_TILE - 1) / PT_TILE;
    if (tiles < 1) tiles = 1;
    int64_t maxT = (int64_t)sm_count() * 8;
    pl.T = (int32_t)(tiles < maxT ? tiles : maxT);
    pl.L = tiles;
    return pl;
}

static inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

// workspace: int32 tile_counts[P][Tmax] | int64 totals[P] | int64 offsets[P+1]
static int64_t ws_counts_bytes(int32_t P) { return align_up((int64_t)P * sm_count() * 8 * 4, 256); }
static int64_t ws_total_bytes(int32_t P) {
    return ws_counts_bytes(P) + align_up((int64_t)P * 8, 256) + align_up((int64_t)(P + 1) * 8, 256);
}

// PRE: 0 = portable_hash of the key column, 1 = the int64 key IS the hash
// (prehashed / radix digits), 2 = the key is a row id and its hash is looked up
// in f.row_hash (DPK_K_ROWID, variable-length keys)
template <typename KeyT, int PRE>
__device__ __forceinline__ int64_t key_hash(KeyT k, const PartFn &f) {
    if constexpr (PRE == 1) return (int64_t)k;
    else if constexpr (PRE == 2) return __ldg(&f.row_hash[(int64_t)k]);
    else return KeyHash<KeyT>::of(k);
}

// Lanes of the warp holding the same bucket id, built from one ballot per bit of the id
// (nbits <= 13, warp-uniform).  Only used by the histogram pass's count_mode 0; the scatter
// kernel keeps MATCH.ANY (one instruction instead of one ballot per bit).
__device__ __forceinline__ unsigned warp_peers(int id, int nbits) {
    unsigned peers = 0xffffffffu;
#pragma unroll
    for (int b = 0; b < 13; b++) {
        if (b < nbits) {
            const unsigned set = __ballot_sync(0xffffffffu, (id >> b) & 1);
            peers &= ((id >> b) & 1) ? set : ~set;
        }
    }
    return peers;
}

// exclusive scan of one int per thread over the 256-thread CTA; returns the
// exclusive prefix, *total gets the CTA sum.  s_warp: >= PT_WARPS ints.
template <int NW = PT_WARPS>
__device__ __forceinline__ int block_excl_scan(int v, int *s_warp, int *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += t;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    int base = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < NW; w++) {
        int t = s_warp[w];
        if (w < warp) base += t;
        tot += t;
    }
    __syncthreads();
    *total = tot;
    return base + inc - v;
}

// ------------------------------------------------------------------ count
// PIN: the rows are packed records (key then a value of the key's width): the key of row i is element 2 * i
template <typename KeyT, int PRE, bool PIN = false>
__global__ void __launch_bounds__(PT_THREADS)
k_part_count(const KeyT *__restrict__ keys, int64_t n, int64_t L, PartFn f,
             int32_t *__restrict__ tile_counts, int32_t T, SegTab seg, int count_mode) {
    // Histograms: up to PT_COUNT_PRIV buckets every warp owns a private histogram and its
    // match leader updates it with a plain read-modify-write (shared-memory atomics per
    // lane were the bound of this kernel); beyond that one CTA histogram
    // with atomics.  s_cnt: [PT_WARPS][P] or [P].
    extern __shared__ int32_t s_cnt[];
    const int P = f.nbuckets();
    if (seg.cbeg != nullptr && (int)blockIdx.x >= *seg.ctotal) return;
    const bool priv = P <= PT_COUNT_PRIV;
    const int nhist = priv ? PT_WARPS * P : P;
    for (int p = threadIdx.x; p < nhist; p += PT_THREADS) s_cnt[p] = 0;
    __syncthreads();
    const int64_t beg = seg.cbeg ? seg.cbeg[blockIdx.x] : ((int64_t)blockIdx.x * L / T) * PT_TILE;
    const int64_t end = seg.cbeg ? seg.cend[blockIdx.x] : min(n, ((int64_t)(blockIdx.x + 1) * L / T) * PT_TILE);
    const int lane = threadIdx.x & 31;
    int32_t *wh = s_cnt + (priv ? (threadIdx.x >> 5) * P : 0);
    constexpr int U = 8;
    int64_t i0 = beg;
    if (count_mode == 1) {
        // full blocks of 2048 rows: no bounds predicates (the kernel is issue-bound: hash + one atomic per row)
        for (; i0 + (int64_t)PT_THREADS * U <= end; i0 += (int64_t)PT_THREADS * U) {
            KeyT k[U];
#pragma unroll
            for (int u = 0; u < U; u++) k[u] = keys[(i0 + (int64_t)u * PT_THREADS + threadIdx.x) * (PIN ? 2 : 1)];
#pragma unroll
            for (int u = 0; u < U; u++) atomicAdd(&wh[f.bucket(key_hash<KeyT, PRE>(k[u], f))], 1);
        }
    }
    for (; i0 < end; i0 += (int64_t)PT_THREADS * U) {
        KeyT k[U];
        bool ok[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            int64_t i = i0 + (int64_t)u * PT_THREADS + threadIdx.x;
            ok[u] = i < end;
            k[u] = ok[u] ? keys[i * (PIN ? 2 : 1)] : KeyT(0);
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            int pid = ok[u] ? f.bucket(key_hash<KeyT, PRE>(k[u], f)) : -1;
            if (count_mode == 1) {  // one shared-memory atomic per row, no warp matching
                if (ok[u]) atomicAdd(&wh[pid], 1);
                continue;
            }
            unsigned m = warp_peers(pid, 32 - __clz(P));
            if (priv) {
                if (ok[u] && lane == __ffs(m) - 1) wh[pid] += __popc(m);
                __syncwarp();  // the next round's leader may be another lane touching the same counter
            } else {
                if (ok[u] && lane == __ffs(m) - 1) atomicAdd(&s_cnt[pid], __popc(m));
            }
        }
    }
    __syncthreads();
    if (priv) {  // fold the warp histograms into the first one
        for (int p = threadIdx.x; p < P; p += PT_THREADS) {
            int t = 0;
#pragma unroll
            for (int w = 0; w < PT_WARPS; w++) t += s_cnt[w * P + p];
            s_cnt[p] = t;
        }
        __syncthreads();
    }
    if (seg.cbeg) {
        for (int p = threadIdx.x; p < P; p += PT_THREADS) seg.chunk_counts[(int64_t)blockIdx.x * P + p] = s_cnt[p];
    } else {
        for (int p = threadIdx.x; p < P; p += PT_THREADS) tile_counts[(int64_t)p * T + blockIdx.x] = s_cnt[p];
    }
}

// one CTA per bucket: exclusive scan of its T per-CTA counts, total -> totals[p]
__global__ void __launch_bounds__(PT_THREADS)
k_part_scan(int32_t *__restrict__ tile_counts, int32_t T, int64_t *__restrict__ totals) {
    __shared__ int s_warp[PT_WARPS];
    int32_t *row = tile_counts + (int64_t)blockIdx.x * T;
    const int E = (T + PT_THREADS - 1) / PT_THREADS;
    const int b = threadIdx.x * E;
    int sum = 0;
    for (int i = b; i < min(b + E, T); i++) sum += row[i];
    int tot;
    int run = block_excl_scan(sum, s_warp, &tot);
    for (int i = b; i < min(b + E, T); i++) {
        int t = row[i];
        row[i] = run;
        run += t;
    }
    if (threadIdx.x == 0) totals[blockIdx.x] = (int64_t)tot;
}

// single CTA: offsets[0..P] = exclusive scan of totals (int64)
__global__ void __launch_bounds__(PT_THREADS)
k_part_offsets(const int64_t *__restrict__ totals, int32_t P, int64_t *__restrict__ offsets) {
    __shared__ long long s_part[PT_THREADS];
    const int E = (P + PT_THREADS - 1) / PT_THREADS;
    const int b = threadIdx.x * E;
    long long sum = 0;
    for (int i = b; i < min(b + E, P); i++) sum += totals[i];
    s_part[threadIdx.x] = sum;
    __syncthreads();
    long long base = 0;
    for (int t = 0; t < (int)threadIdx.x; t++) base += s_part[t];
    for (int i = b; i < min(b + E, P); i++) {
        offsets[i] = base;
        base += totals[i];
    }
    if (b < P && min(b + E, P) == P) offsets[P] = base;
    if (P == 0 && threadIdx.x == 0) offsets[0] = 0;
}

// ---------------------------------------------------------------- scatter
struct ScatterSmem {
    int64_t key_off, val_off, pid_off, gpos_off, tstart_off, tcount_off, whist_off, kptr_off, vptr_off, total;
};
static ScatterSmem scatter_smem(int kb, int vb, int32_t P, bool ptr_mode, int tile) {
    ScatterSmem s;
    int64_t o = 0;
    s.key_off = o; o += align_up((int64_t)tile * kb, 16);
    s.val_off = o; o += align_up((int64_t)tile * vb, 16);
    s.gpos_off = o; o += align_up((int64_t)P * 8, 16);
    s.tstart_off = o; o += align_up((int64_t)P * 4, 16);
    s.tcount_off = o; o += align_up((int64_t)P * 4, 16);
    s.pid_off = o; o += align_up((int64_t)tile * 2, 16);
    s.whist_off = o; o += align_up((int64_t)PT_WARPS * P * 2, 16);
    s.kptr_off = o; if (ptr_mode) o += align_up((int64_t)P * 8, 16);
    s.vptr_off = o; if (ptr_mode) o += align_up((int64_t)P * 8, 16);
    s.total = o;
    return s;
}

// ITEMS rows per thread and tile: 16 (4096-row tiles, 2 CTAs per SM) or 8 (2048-row tiles, half the
// registers and shared memory, 4 CTAs per SM -- more warps to hide the phase barriers; bucket runs
// inside a tile are half as long).  The CTA's row range comes from the plan in PT_TILE units either way.
// PK (PK_IN | PK_OUT bits, plain and segmented destinations only): rows are read from / written as packed records.
template <typename KeyT, typename ValT, int PRE, int ITEMS, int PK = 0>
__global__ void __launch_bounds__(PT_THREADS, ITEMS == 16 ? 2 : 4)
k_part_scatter(const KeyT *__restrict__ keys, const ValT *__restrict__ vals, int64_t n, int64_t L,
               PartFn f, const int32_t *__restrict__ tile_off, int32_t T,
               const int64_t *__restrict__ bucket_base, KeyT *__restrict__ out_keys,
               ValT *__restrict__ out_vals, ScatterSmem lay, SegTab seg) {
    constexpr bool HAS_VAL = !std::is_same<ValT, NoVal>::value;
    using Rec = PackedRow<KeyT, ValT>;
    constexpr int TILE = PT_THREADS * ITEMS;
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int s_warp[PT_WARPS];
    KeyT *s_key = reinterpret_cast<KeyT *>(smem + lay.key_off);
    ValT *s_val = reinterpret_cast<ValT *>(smem + lay.val_off);
    int64_t *s_gpos = reinterpret_cast<int64_t *>(smem + lay.gpos_off);   // global pos of next row of bucket p
    int32_t *s_tstart = reinterpret_cast<int32_t *>(smem + lay.tstart_off);
    int32_t *s_tcount = reinterpret_cast<int32_t *>(smem + lay.tcount_off);
    uint16_t *s_pid = reinterpret_cast<uint16_t *>(smem + lay.pid_off);
    uint16_t *s_whist = reinterpret_cast<uint16_t *>(smem + lay.whist_off);  // [PT_WARPS][P]

    const int P = f.nbuckets();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned lt_mask = (1u << lane) - 1u;
    if (seg.cbeg != nullptr && (int)blockIdx.x >= *seg.ctotal) return;
    const int64_t beg = seg.cbeg ? seg.cbeg[blockIdx.x] : ((int64_t)blockIdx.x * L / T) * PT_TILE;
    const int64_t end = seg.cbeg ? seg.cend[blockIdx.x] : min(n, ((int64_t)(blockIdx.x + 1) * L / T) * PT_TILE);

    uint64_t *s_kptr = reinterpret_cast<uint64_t *>(smem + lay.kptr_off);
    uint64_t *s_vptr = reinterpret_cast<uint64_t *>(smem + lay.vptr_off);
    if (seg.key_ptrs) {
        for (int p = threadIdx.x; p < P; p += PT_THREADS) {
            s_gpos[p] = (int64_t)tile_off[(int64_t)p * T + blockIdx.x];
            s_kptr[p] = seg.key_ptrs[p];
            if constexpr (HAS_VAL) s_vptr[p] = seg.val_ptrs[p];
        }
    } else if (seg.cbeg) {
        for (int p = threadIdx.x; p < P; p += PT_THREADS) s_gpos[p] = seg.chunk_off[(int64_t)blockIdx.x * P + p];
    } else {
        for (int p = threadIdx.x; p < P; p += PT_THREADS)
            s_gpos[p] = bucket_base[p] + (int64_t)tile_off[(int64_t)p * T + blockIdx.x];
    }

    const int E = (P + PT_THREADS - 1) / PT_THREADS;  // buckets per thread in the scan

    for (int64_t tile = beg; tile < end; tile += TILE) {
        const int rows = (int)min((int64_t)TILE, end - tile);
        for (int i = threadIdx.x; i < PT_WARPS * P; i += PT_THREADS) s_whist[i] = 0;

        // ---- load: warp w owns rows [w*512, w*512+512) of the tile, item j = 32 consecutive rows
        KeyT k[ITEMS];
        ValT v[ITEMS];
        const int64_t wbase = tile + (int64_t)warp * (32 * ITEMS) + lane;
        if constexpr ((PK & PK_IN) != 0) {
#pragma unroll
            for (int j = 0; j < ITEMS; j++) {
                int64_t idx = wbase + j * 32;
                k[j] = KeyT(0);
                if (idx < end) {
                    const Rec r = reinterpret_cast<const Rec *>(keys)[idx];
                    k[j] = r.k;
                    v[j] = r.v;
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < ITEMS; j++) {
                int64_t idx = wbase + j * 32;
                k[j] = idx < end ? keys[idx] : KeyT(0);
            }
        }
        if constexpr (HAS_VAL && (PK & PK_IN) == 0) {
#pragma unroll
            for (int j = 0; j < ITEMS; j++) {
                int64_t idx = wbase + j * 32;
                if (idx < end) v[j] = vals[idx];
            }
        }
        __syncthreads();  // whist zeroed; previous tile's copy-out done with the staging buffers

        // ---- warp-level ranks (stable: lanes in order, items in order)
        uint16_t pid[ITEMS], rank[ITEMS];
        uint16_t *wh = s_whist + warp * P;
#pragma unroll
        for (int j = 0; j < ITEMS; j++) {
            const bool ok = (wbase + j * 32) < end;
            const int p = ok ? f.bucket(key_hash<KeyT, PRE>(k[j], f)) : P;  // P = "no row"
            if (seg.unordered) {
                // rows may be permuted inside a bucket (reduceByKey does not care): the rank inside the
                // warp's share of the bucket is whatever one native 32-bit atomic on the packed pair of
                // 16-bit counters returns -- no warp match, no leader, no __syncwarp
                pid[j] = (uint16_t)p;
                if (ok) {
                    const unsigned old = atomicAdd(reinterpret_cast<unsigned *>(wh) + (p >> 1), (p & 1) ? 0x10000u : 1u);
                    rank[j] = (uint16_t)((p & 1) ? (old >> 16) : (old & 0xffffu));
                }
                continue;
            }
            // peers with the same bucket: one MATCH.ANY instead of a ballot per bucket bit
            const unsigned m = __match_any_sync(0xffffffffu, p);
            int base = 0;
            if (ok) base = wh[p];
            __syncwarp();
            pid[j] = (uint16_t)p;
            rank[j] = (uint16_t)(base + __popc(m & lt_mask));
            if (ok && lane == __ffs(m) - 1) wh[p] = (uint16_t)(base + __popc(m));
            __syncwarp();
        }
        __syncthreads();

        // ---- per bucket: exclusive scan over the 8 warps, tile count
        for (int p = threadIdx.x; p < P; p += PT_THREADS) {
            int run = 0;
#pragma unroll
            for (int w = 0; w < PT_WARPS; w++) {
                int t = s_whist[w * P + p];
                s_whist[w * P + p] = (uint16_t)run;
                run += t;
            }
            s_tcount[p] = run;
        }
        __syncthreads();
        // ---- exclusive scan of tile counts over buckets -> start of each bucket's run in the tile
        {
            const int b = threadIdx.x * E;
            int sum = 0;
            for (int i = b; i < min(b + E, P); i++) sum += s_tcount[i];
            int tot;
            int run = block_excl_scan(sum, s_warp, &tot);
            for (int i = b; i < min(b + E, P); i++) {
                s_tstart[i] = run;
                run += s_tcount[i];
            }
        }
        __syncthreads();

        // ---- place rows at their sorted position in the staging tile
#pragma unroll
        for (int j = 0; j < ITEMS; j++) {
            const int p = pid[j];
            if (p < P) {
                const int pos = s_tstart[p] + s_whist[warp * P + p] + rank[j];
                s_key[pos] = k[j];
                if constexpr (HAS_VAL) s_val[pos] = v[j];
                s_pid[pos] = (uint16_t)p;
            }
        }
        __syncthreads();

        // ---- copy out: consecutive threads -> consecutive addresses inside each bucket run
        for (int i = threadIdx.x; i < rows; i += PT_THREADS) {
            const int p = s_pid[i];
            const int64_t dst = s_gpos[p] + (int64_t)(i - s_tstart[p]);
            if constexpr ((PK & PK_OUT) != 0) {
                reinterpret_cast<Rec *>(out_keys)[dst] = Rec{s_key[i], s_val[i]};
            } else if (seg.key_ptrs) {  // pointer mode: the bucket's destination may be a peer GPU
                reinterpret_cast<KeyT *>(s_kptr[p])[dst] = s_key[i];
                if constexpr (HAS_VAL) reinterpret_cast<ValT *>(s_vptr[p])[dst] = s_val[i];
            } else {
                out_keys[dst] = s_key[i];
                if constexpr (HAS_VAL) out_vals[dst] = s_val[i];
            }
        }
        __syncthreads();
        for (int p = threadIdx.x; p < P; p += PT_THREADS) s_gpos[p] += s_tcount[p];
        // (next iteration's first __syncthreads orders this against later reads)
    }
}


// ------------------------------------------------- scatter, TMA bulk-store form
// Unordered multisplit of one tile at a time (reduceByKey paths: the order of rows inside a bucket is not
// observable).  Differences to k_part_scatter:
//   * rank = the value ONE native shared-memory atomic on the tile's bucket counter returns (ATOMS.ADD,
//     far cheaper than MATCH.ANY at random addresses): no warp
//     histograms, no scan over warps, one block barrier less per tile;
//   * the staged tile leaves through the TMA: every bucket run is written with cp.async.bulk
//     (shared -> global, UBLKCP.G.S) instead of the per-thread LDS + STG.64 copy-out: it costs the SM one
//     instruction per run instead of two per row.
//     Bulk copies need 16-byte aligned addresses and sizes on both sides: the staging position of a run is
//     shifted by up to 16/size-1 elements so that it has the same alignment phase as its destination, and the
//     unaligned head/tail elements of a run (at most 16/size-1 each) are stored by the issuing thread;
//   * the next tile's rows are loaded into the (now free) registers right after the placement, so their DRAM
//     latency overlaps the barrier, the bulk-store issue and the counter reset.
// Per tile: rank -> barrier -> aligned scan of the 256..1024 tile counts -> barrier -> placement ->
// fence.proxy.async -> barrier -> bulk stores (asynchronous; their shared-memory reads are awaited with
// cp.async.bulk.wait_group.read right before the next placement).
struct BulkSmem {
    int64_t key_off, val_off, gpos_off, cnt_off, sk_off, sv_off, vd_off, total;
    int32_t key_slots, val_slots;
};
static BulkSmem bulk_smem(int kb, int vb, int32_t P, int tile, bool ptr_mode = false) {
    BulkSmem s;
    int64_t o = 0;
    const int padk = 16 / kb - 1, padv = vb ? 16 / vb - 1 : 0;
    s.key_slots = tile + P * padk;
    s.val_slots = vb ? tile + P * padv : 0;
    s.key_off = o; o += align_up((int64_t)s.key_slots * kb, 128);
    s.val_off = o; o += align_up((int64_t)s.val_slots * vb, 128);
    s.gpos_off = o; o += align_up((int64_t)P * 8, 16);
    s.cnt_off = o; o += align_up((int64_t)P * 4 * 2, 16);    // two alternating count arrays
    s.sk_off = o; o += align_up((int64_t)P * 4, 16);
    s.sv_off = o; o += align_up((int64_t)P * 4, 16);
    s.vd_off = o; if (ptr_mode && vb) o += align_up((int64_t)P * 8, 16);   // pointer mode: value slot - key slot, in elements
    s.total = o;
    return s;
}

__device__ __forceinline__ void bulk_store_s2g(void *gdst, uint32_t ssrc, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(ssrc), "r"(bytes) : "memory");
}

// copy-out of one bucket run of one column: [head: plain stores][aligned middle: one bulk store][tail: plain]
template <typename T>
__device__ __forceinline__ void flush_run(T *__restrict__ out, int64_t g, const T *s_col, uint32_t s_col_addr, int s0, int cnt) {
    constexpr int A = 16 / (int)sizeof(T);
    T *dst = out + g;
    int head = (int)(((16u - (uint32_t)((uintptr_t)dst & 15u)) & 15u) / (uint32_t)sizeof(T));
    if (head > cnt) head = cnt;
    const int mid = ((cnt - head) / A) * A;
    for (int i = 0; i < head; i++) dst[i] = s_col[s0 + i];
    if (mid) bulk_store_s2g(dst + head, s_col_addr + (uint32_t)(s0 + head) * (uint32_t)sizeof(T), (uint32_t)mid * (uint32_t)sizeof(T));
    for (int i = head + mid; i < cnt; i++) dst[i] = s_col[s0 + i];
}

// bucket function specialised at compile time for the configurations the hot paths use (the generic PartFn::bucket
// walks a chain of uniform branches per row; the kernel is issue-bound):
//   FMODE 1: P a power of two (or 1), any sub_bits: (h & (P-1)) << sub_bits | top sub_bits bits of mixed(h)
//   FMODE 2: second-level split (PartFn mode 5): bits of mixed(h) below the first-level ones
//   FMODE 0: anything else (thresholds, magic divide, radix digits)
template <int FMODE>
__device__ __forceinline__ int bucket_of(const PartFn &f, int64_t h) {
    if constexpr (FMODE == 1) {
        const uint32_t sub = (uint32_t)(((uint64_t)PartFn::mixed(h) << f.sub_bits) >> 32);   // top sub_bits bits (0 when sub_bits == 0)
        return (int)((((uint32_t)h & (uint32_t)(f.P - 1)) << f.sub_bits) | sub);
    } else if constexpr (FMODE == 2) {
        return (int)((PartFn::mixed(h) >> f.shift) & (uint32_t)(f.P - 1));
    } else {
        return f.bucket(h);
    }
}

// PK (PK_IN | PK_OUT bits, not with PTRS): rows are read from / staged and written as packed records.  A packed tile is
// one array of records: every bucket run leaves with ONE bulk store, issued by one thread per bucket, and with 16-byte
// records every run starts and ends on a 16-byte boundary (no head or tail stores).
template <typename KeyT, typename ValT, int PRE, int NT, int FMODE, bool PTRS = false, int PK = 0>
__global__ void __launch_bounds__(NT, NT == 1024 ? 1 : 2)
k_part_scatter_bulk(const KeyT *__restrict__ keys, const ValT *__restrict__ vals, int64_t n, int64_t L,
                    PartFn f, const int32_t *__restrict__ tile_off, int32_t T,
                    const int64_t *__restrict__ bucket_base, KeyT *__restrict__ out_keys,
                    ValT *__restrict__ out_vals, BulkSmem lay, SegTab seg) {
    constexpr bool HAS_VAL = !std::is_same<ValT, NoVal>::value;
    // 256 threads x 16 rows or 512 x 8 (twice the resident warps) on 4096-row tiles, two CTAs per SM; 1024 x 8 on
    // 8192-row tiles, one CTA per SM (bucket runs twice as long, half the barriers and scans per row)
    constexpr int ITEMS = NT == 256 ? 16 : 8;
    constexpr int TILE = NT * ITEMS;
    constexpr int NW = NT / 32;
    constexpr int AK = 16 / (int)sizeof(KeyT);
    constexpr int AV = HAS_VAL ? 16 / (int)sizeof(typename std::conditional<HAS_VAL, ValT, int64_t>::type) : 1;
    constexpr bool PIN = (PK & PK_IN) != 0, POUT = (PK & PK_OUT) != 0;
    using Rec = PackedRow<KeyT, ValT>;
    constexpr int AR = 16 / (int)sizeof(Rec);
    static_assert(PK == 0 || (HAS_VAL && !PTRS && sizeof(KeyT) == sizeof(ValT)), "packed rows: same-width key and value, plain or segmented mode");
    extern __shared__ __align__(128) unsigned char smem_bulk[];
    unsigned char *smem = smem_bulk;
    __shared__ int s_warp[NW];
    KeyT *s_key = reinterpret_cast<KeyT *>(smem + lay.key_off);
    ValT *s_val = reinterpret_cast<ValT *>(smem + lay.val_off);
    Rec *s_rec = reinterpret_cast<Rec *>(smem + lay.key_off);                 // POUT: the staging tile holds records
    Rec *out_rec = reinterpret_cast<Rec *>(out_keys);
    int64_t *s_gpos = reinterpret_cast<int64_t *>(smem + lay.gpos_off);
    uint32_t *s_cnt = reinterpret_cast<uint32_t *>(smem + lay.cnt_off);      // [2][P]
    int32_t *s_sk = reinterpret_cast<int32_t *>(smem + lay.sk_off);          // start of bucket p's key run in the staging tile
    int32_t *s_sv = reinterpret_cast<int32_t *>(smem + lay.sv_off);
    // Pointer mode (PTRS: fused scatter + exchange, seg.key_ptrs != nullptr; out_keys == out_vals == nullptr): s_gpos[p] is
    // the ABSOLUTE element index (address / sizeof(KeyT)) of the next key slot of bucket p -- in this GPU's memory or in
    // a peer's receive buffer mapped over NVLink -- and s_vd[p] the distance, in elements, from there to the value slot
    // (address / sizeof(ValT) - address / sizeof(KeyT)): the bucket runs of a tile leave through the TMA straight into
    // the buffer their reducer reads.
    constexpr bool ptrs = PTRS;
    int64_t *s_vd = reinterpret_cast<int64_t *>(smem + lay.vd_off);
    const uint32_t key_addr = (uint32_t)__cvta_generic_to_shared(s_key);
    const uint32_t val_addr = (uint32_t)__cvta_generic_to_shared(s_val);

    const int P = f.nbuckets();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (seg.cbeg != nullptr && (int)blockIdx.x >= *seg.ctotal) return;
    const int64_t beg = seg.cbeg ? seg.cbeg[blockIdx.x] : ((int64_t)blockIdx.x * L / T) * PT_TILE;
    const int64_t end = seg.cbeg ? seg.cend[blockIdx.x] : min(n, ((int64_t)(blockIdx.x + 1) * L / T) * PT_TILE);
    if (seg.cbeg) {
        for (int p = threadIdx.x; p < P; p += NT) s_gpos[p] = seg.chunk_off[(int64_t)blockIdx.x * P + p];
    } else if constexpr (PTRS) {
        for (int p = threadIdx.x; p < P; p += NT) {
            const int64_t ke = (int64_t)(seg.key_ptrs[p] / sizeof(KeyT));
            s_gpos[p] = ke + (int64_t)tile_off[(int64_t)p * T + blockIdx.x];
            if constexpr (HAS_VAL) s_vd[p] = (int64_t)(seg.val_ptrs[p] / sizeof(ValT)) - ke;
        }
    } else {
        for (int p = threadIdx.x; p < P; p += NT)
            s_gpos[p] = bucket_base[p] + (int64_t)tile_off[(int64_t)p * T + blockIdx.x];
    }
    for (int p = threadIdx.x; p < 2 * P; p += NT) s_cnt[p] = 0;
    const int E = (P + NT - 1) / NT;  // buckets per thread in the scan

    KeyT k[ITEMS];
    ValT v[ITEMS];
    // rows of the tile this thread holds: row j of warp w's lane l = tile + w * 32 * ITEMS + j * 32 + l
    auto load_tile = [&](int64_t tile) {
        if constexpr (PIN) {   // one 8- or 16-byte load per row
            const Rec *rp = reinterpret_cast<const Rec *>(keys) + tile + warp * (32 * ITEMS) + lane;
            const int left = (int)min((int64_t)TILE, end - tile) - warp * (32 * ITEMS) - lane;
#pragma unroll
            for (int j = 0; j < ITEMS; j++) {
                k[j] = KeyT(0);
                if (j * 32 < left) {
                    const Rec r = rp[j * 32];
                    k[j] = r.k;
                    v[j] = r.v;
                }
            }
            return;
        }
        const KeyT *kp = keys + tile + warp * (32 * ITEMS) + lane;
        if (tile + TILE <= end) {
#pragma unroll
            for (int j = 0; j < ITEMS; j++) k[j] = kp[j * 32];
            if constexpr (HAS_VAL) {
                const ValT *vp = vals + tile + warp * (32 * ITEMS) + lane;
#pragma unroll
                for (int j = 0; j < ITEMS; j++) v[j] = vp[j * 32];
            }
        } else {
            const int left = (int)(end - tile) - warp * (32 * ITEMS) - lane;   // rows from this thread's first row to the end
#pragma unroll
            for (int j = 0; j < ITEMS; j++) k[j] = j * 32 < left ? kp[j * 32] : KeyT(0);
            if constexpr (HAS_VAL) {
                const ValT *vp = vals + tile + warp * (32 * ITEMS) + lane;
#pragma unroll
                for (int j = 0; j < ITEMS; j++)
                    if (j * 32 < left) v[j] = vp[j * 32];
            }
        }
    };
    if (beg < end) load_tile(beg);
    __syncthreads();  // s_gpos, s_cnt initialised

    int par = 0;
    for (int64_t tile = beg; tile < end; tile += TILE, par ^= 1) {
        uint32_t *cnt = s_cnt + par * P;
        // ---- rank: one shared-memory atomic per row on the tile's bucket counter
        uint32_t pr[ITEMS];  // bucket << 16 | rank inside the tile (both < 2^16: P <= 4096, TILE = 4096)
        if (tile + TILE <= end) {   // full tile: no bounds predicates
#pragma unroll
            for (int j = 0; j < ITEMS; j++) {
                const int p = bucket_of<FMODE>(f, key_hash<KeyT, PRE>(k[j], f));
                pr[j] = ((uint32_t)p << 16) | atomicAdd(&cnt[p], 1u);
            }
        } else {
            const int left = (int)(end - tile) - warp * (32 * ITEMS) - lane;
#pragma unroll
            for (int j = 0; j < ITEMS; j++) {
                pr[j] = 0xffffffffu;
                if (j * 32 < left) {
                    const int p = bucket_of<FMODE>(f, key_hash<KeyT, PRE>(k[j], f));
                    pr[j] = ((uint32_t)p << 16) | atomicAdd(&cnt[p], 1u);
                }
            }
        }
        // the previous tile's bulk stores must have read the staging tile before it is overwritten
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        __syncthreads();  // (A) counts final

        // ---- starts of the bucket runs in the staging tile: exclusive scan of the counts, every run shifted
        //      so that it has the alignment phase of its destination
        {
            const int b = threadIdx.x * E;
            int sum = 0;
            for (int i = b; i < min(b + E, P); i++) sum += (int)cnt[i];
            int tot;
            int run = block_excl_scan<NW>(sum, s_warp, &tot);
            for (int i = b; i < min(b + E, P); i++) {
                const int64_t g = s_gpos[i];
                if constexpr (POUT) {
                    const uint32_t gr = (uint32_t)(((uintptr_t)(out_rec + g)) / sizeof(Rec));
                    const int baser = run + i * (AR - 1);
                    s_sk[i] = baser + (int)((gr - (uint32_t)baser) & (uint32_t)(AR - 1));
                    run += (int)cnt[i];
                    continue;
                }
                const uint32_t gk = (uint32_t)(((uintptr_t)(out_keys + g)) / sizeof(KeyT));
                const int basek = run + i * (AK - 1);
                s_sk[i] = basek + (int)((gk - (uint32_t)basek) & (uint32_t)(AK - 1));
                if constexpr (HAS_VAL) {
                    const uint32_t gv = (uint32_t)(((uintptr_t)(out_vals + (ptrs ? g + s_vd[i] : g))) / sizeof(ValT));
                    const int basev = run + i * (AV - 1);
                    s_sv[i] = basev + (int)((gv - (uint32_t)basev) & (uint32_t)(AV - 1));
                }
                run += (int)cnt[i];
            }
        }
        __syncthreads();  // (B)

        // ---- placement (rows past the end carry bucket 0xffff)
#pragma unroll
        for (int j = 0; j < ITEMS; j++) {
            const int p = (int)(pr[j] >> 16), r = (int)(pr[j] & 0xffffu);
            if (p != 0xffff) {
                if constexpr (POUT) {
                    s_rec[s_sk[p] + r] = Rec{k[j], v[j]};
                } else {
                    s_key[s_sk[p] + r] = k[j];
                    if constexpr (HAS_VAL) s_val[s_sv[p] + r] = v[j];
                }
            }
        }
        // registers are free: fetch the next tile now, its latency hides behind the barrier and the copy-out
        if (tile + TILE < end) load_tile(tile + TILE);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the TMA
        __syncthreads();  // (C)

        // ---- copy-out: bucket runs leave through the TMA.  With values, lane pairs share a bucket (even lane: key
        //      run, odd lane: value run) so that every thread issues at most one bulk store per round: the issue
        //      rate of one thread bounds the bulk-store rate below 512-byte runs (scripts/microbench/smem_ops.cu).
        //      Packed records: one run per bucket, one thread per bucket.
        if constexpr (POUT) {
            const uint32_t rec_addr = key_addr;
            for (int p = threadIdx.x; p < P; p += NT) {
                const int c = (int)cnt[p];
                if (c) {
                    const int64_t g = s_gpos[p];
                    flush_run<Rec>(out_rec, g, s_rec, rec_addr, s_sk[p], c);
                    s_gpos[p] = g + c;
                    cnt[p] = 0;
                }
            }
        } else if constexpr (HAS_VAL) {
            for (int q0 = 0; q0 < 2 * P; q0 += NT) {
                const int q = q0 + (int)threadIdx.x;
                const int p = q >> 1;
                const bool on = q < 2 * P;
                const int c = on ? (int)cnt[p] : 0;
                const int64_t g = on ? s_gpos[p] : 0;
                if (c) {
                    if (q & 1) flush_run<ValT>(out_vals, ptrs ? g + s_vd[p] : g, s_val, val_addr, s_sv[p], c);
                    else flush_run<KeyT>(out_keys, g, s_key, key_addr, s_sk[p], c);
                }
                __syncwarp();   // both lanes of the pair have read the count and the position
                if (c && !(q & 1)) {
                    s_gpos[p] = g + c;
                    cnt[p] = 0;  // this array is used again two tiles from now (barriers A..C of the next tile in between)
                }
            }
        } else {
            for (int p = threadIdx.x; p < P; p += NT) {
                const int c = (int)cnt[p];
                if (c) {
                    const int64_t g = s_gpos[p];
                    flush_run<KeyT>(out_keys, g, s_key, key_addr, s_sk[p], c);
                    s_gpos[p] = g + c;
                    cnt[p] = 0;
                }
            }
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // all stores complete before the CTA's shared memory goes away
}

// ------------------------------------------------------------ host dispatch
template <typename KeyT, int PRE>
static int launch_count(const void *keys, int64_t n, const Plan &pl, const PartFn &f,
                        int32_t *tile_counts, cudaStream_t st) {
    size_t sh = (size_t)f.nbuckets() * sizeof(int32_t) * (f.nbuckets() <= PT_COUNT_PRIV ? PT_WARPS : 1);
    auto kern = (pl.pack & PK_IN) ? k_part_count<KeyT, PRE, true> : k_part_count<KeyT, PRE, false>;
    DPK_LAUNCH(pl.label_count ? pl.label_count : (pl.seg.cbeg ? "seg_count" : "part_count"), st, kern<<<pl.T, PT_THREADS, sh, st>>>((const KeyT *)keys, n, pl.L, f, tile_counts, pl.T, pl.seg, g_count_mode));
    return DPK_OK;
}

static int dispatch_count(const void *keys, int key_kind, int64_t n, const Plan &pl, const PartFn &f,
                          int32_t *tile_counts, cudaStream_t st) {
    if (key_kind >= 0) key_kind &= ~DPK_K_PACKED;                   // nor about the layout the scatter writes
    if (key_kind >= DPK_K_UNORDERED) key_kind -= DPK_K_UNORDERED;  // the histogram does not care about order
    switch (key_kind) {
    case -1: return launch_count<int64_t, true>(keys, n, pl, f, tile_counts, st);
    case DPK_K_I64: return launch_count<int64_t, false>(keys, n, pl, f, tile_counts, st);
    case DPK_K_I32: return launch_count<int32_t, false>(keys, n, pl, f, tile_counts, st);
    case DPK_K_F64: return launch_count<double, false>(keys, n, pl, f, tile_counts, st);
    case DPK_K_U64: return launch_count<uint64_t, false>(keys, n, pl, f, tile_counts, st);
    case DPK_K_F32: return launch_count<float, false>(keys, n, pl, f, tile_counts, st);
    case DPK_K_ROWID:
        if (!f.row_hash) return fail(DPK_ERR_INVALID, "DPK_K_ROWID needs key_aux (the per-row hash column)");
        return launch_count<int64_t, 2>(keys, n, pl, f, tile_counts, st);
    }
    return fail(DPK_ERR_UNSUPPORTED, "key kind %d is unhashable by portable_hash", key_kind);
}

template <typename KeyT, typename ValT, int PRE, int ITEMS>
static int launch_scatter_items(const void *keys, const void *vals, int64_t n, const Plan &pl, const PartFn &f,
                                const int32_t *tile_off, const int64_t *bucket_base, void *out_keys,
                                void *out_vals, cudaStream_t st) {
    constexpr int vb = std::is_same<ValT, NoVal>::value ? 0 : (int)sizeof(ValT);
    ScatterSmem lay = scatter_smem((int)sizeof(KeyT), vb, f.nbuckets(), pl.seg.key_ptrs != nullptr, PT_THREADS * ITEMS);
    auto kern = k_part_scatter<KeyT, ValT, PRE, ITEMS>;
    if constexpr (vb == (int)sizeof(KeyT) && ITEMS == 16) {
        if (pl.pack == PK_OUT) kern = k_part_scatter<KeyT, ValT, PRE, ITEMS, PK_OUT>;
        else if (pl.pack == PK_IN) kern = k_part_scatter<KeyT, ValT, PRE, ITEMS, PK_IN>;
        else if (pl.pack == (PK_IN | PK_OUT)) kern = k_part_scatter<KeyT, ValT, PRE, ITEMS, PK_IN | PK_OUT>;
    }
    if (lay.total > 227 * 1024)
        return fail(DPK_ERR_UNSUPPORTED, "%d buckets need %lld B of shared memory", f.nbuckets(), (long long)lay.total);
    DPK_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lay.total));
    DPK_LAUNCH(pl.label_scatter ? pl.label_scatter : (pl.seg.cbeg ? "seg_scatter" : "part_scatter"), st,
               kern<<<pl.T, PT_THREADS, (size_t)lay.total, st>>>((const KeyT *)keys, (const ValT *)vals, n, pl.L, f,
                                                                tile_off, pl.T, bucket_base, (KeyT *)out_keys,
                                                                (ValT *)out_vals, lay, pl.seg));
    return DPK_OK;
}

template <typename KeyT, typename ValT, int PRE>
static int launch_scatter_bulk(const void *keys, const void *vals, int64_t n, const Plan &pl, const PartFn &f,
                               const int32_t *tile_off, const int64_t *bucket_base, void *out_keys,
                               void *out_vals, cudaStream_t st) {
    constexpr int vb = std::is_same<ValT, NoVal>::value ? 0 : (int)sizeof(ValT);
    if constexpr (vb == (int)sizeof(KeyT)) {
        if (pl.pack) {
            // packed rows: 8192-row tiles (1024 threads) always -- a tile of records takes the shared memory of a tile of
            // two columns and its runs are one bulk store each.  Packed input only comes from the reduce side, whose
            // fine bucket function is the second-level split (FMODE 2).
            const int fmode = f.mode == 5 ? 2 : ((f.mode == 0 || f.mode == 1) ? 1 : 0);
            BulkSmem lay = bulk_smem(2 * (int)sizeof(KeyT), 0, f.nbuckets(), 8192);
            auto kern = fmode == 2 ? k_part_scatter_bulk<KeyT, ValT, PRE, 1024, 2, false, PK_OUT>
                      : fmode == 1 ? k_part_scatter_bulk<KeyT, ValT, PRE, 1024, 1, false, PK_OUT>
                                   : k_part_scatter_bulk<KeyT, ValT, PRE, 1024, 0, false, PK_OUT>;
            if (pl.pack & PK_IN) {
                if (fmode != 2) return fail(DPK_ERR_UNSUPPORTED, "packed input needs the second-level split");
                kern = (pl.pack & PK_OUT) ? k_part_scatter_bulk<KeyT, ValT, PRE, 1024, 2, false, PK_IN | PK_OUT>
                                          : k_part_scatter_bulk<KeyT, ValT, PRE, 1024, 2, false, PK_IN>;
                if (!(pl.pack & PK_OUT)) lay = bulk_smem((int)sizeof(KeyT), vb, f.nbuckets(), 8192);
            }
            DPK_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lay.total));
            DPK_LAUNCH(pl.label_scatter ? pl.label_scatter : (pl.seg.cbeg ? "seg_scatter" : "part_scatter"), st,
                       kern<<<pl.T, 1024, (size_t)lay.total, st>>>((const KeyT *)keys, (const ValT *)vals, n, pl.L, f,
                                                                  tile_off, pl.T, bucket_base, (KeyT *)out_keys,
                                                                  (ValT *)out_vals, lay, pl.seg));
            return DPK_OK;
        }
    }
    // dpk_set_option("scatter_threads"): 512 (default; 8 rows per thread, 4096-row tiles, 2 CTAs per SM), 256 (16 rows
    // per thread) or 1024 (8192-row tiles, 1 CTA per SM)
    int nt = g_scatter_threads;
    if (nt == 512 && pl.seg.cbeg != nullptr && g_scatter_seg_wide) nt = 1024;   // second-level split, H100 C2: 1.33 vs 1.83 ms
    // rows of 4-byte columns: a 4096-row tile's bucket runs are 64 bytes, where the bulk stores are issue-bound (not
    // measured apart on the H100: at C4's sizes the bucket-count rule below selects 8192-row tiles anyway)
    if (nt == 512 && g_scatter_seg_wide && sizeof(KeyT) <= 4 && (vb == 0 || vb <= 4)) nt = 1024;
    // from 512 buckets up a 4096-row tile's runs are 64 bytes even for 8-byte rows: on an H100 4.33 ms (4096-row
    // tiles) against 2.71 ms (8192-row tiles) per 1e8 (int64,int64) rows at 512 buckets
    if (nt == 512 && g_scatter_wide_from > 0 && f.nbuckets() >= g_scatter_wide_from) nt = 1024;
    const bool ptr_mode = pl.seg.key_ptrs != nullptr;
    if (ptr_mode && nt == 512 && g_scatter_ptr_threads == 1024) nt = 1024;
    if (nt == 1024 && bulk_smem((int)sizeof(KeyT), vb, f.nbuckets(), 8192, ptr_mode).total > 220 * 1024) nt = 512;
    BulkSmem lay = bulk_smem((int)sizeof(KeyT), vb, f.nbuckets(), nt == 1024 ? 8192 : PT_TILE, ptr_mode);
    const int fmode = f.mode == 5 ? 2 : ((f.mode == 0 || f.mode == 1) ? 1 : 0);
    if (ptr_mode) {   // fused scatter + exchange: only the map-side bucket functions occur
        auto kp = nt == 1024 ? (fmode == 1 ? k_part_scatter_bulk<KeyT, ValT, PRE, 1024, 1, true> : k_part_scatter_bulk<KeyT, ValT, PRE, 1024, 0, true>)
                             : (fmode == 1 ? k_part_scatter_bulk<KeyT, ValT, PRE, 512, 1, true> : k_part_scatter_bulk<KeyT, ValT, PRE, 512, 0, true>);
        if (nt != 512 && nt != 1024) return fail(DPK_ERR_UNSUPPORTED, "pointer mode needs 512- or 1024-thread CTAs");
        DPK_CUDA_TRY(cudaFuncSetAttribute(kp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lay.total));
        DPK_LAUNCH(pl.label_scatter ? pl.label_scatter : "part_scatter", st,
                   kp<<<pl.T, nt, (size_t)lay.total, st>>>((const KeyT *)keys, (const ValT *)vals, n, pl.L, f, tile_off, pl.T,
                                                          bucket_base, (KeyT *)out_keys, (ValT *)out_vals, lay, pl.seg));
        return DPK_OK;
    }
    auto kern = nt == 1024 ? (fmode == 2 ? k_part_scatter_bulk<KeyT, ValT, PRE, 1024, 2> :
                              fmode == 1 ? k_part_scatter_bulk<KeyT, ValT, PRE, 1024, 1> : k_part_scatter_bulk<KeyT, ValT, PRE, 1024, 0>)
              : nt == 512 ? (fmode == 2 ? k_part_scatter_bulk<KeyT, ValT, PRE, 512, 2> :
                             fmode == 1 ? k_part_scatter_bulk<KeyT, ValT, PRE, 512, 1> : k_part_scatter_bulk<KeyT, ValT, PRE, 512, 0>)
                          : k_part_scatter_bulk<KeyT, ValT, PRE, 256, 0>;
    DPK_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lay.total));
    DPK_LAUNCH(pl.label_scatter ? pl.label_scatter : (pl.seg.cbeg ? "seg_scatter" : "part_scatter"), st,
               kern<<<pl.T, nt, (size_t)lay.total, st>>>((const KeyT *)keys, (const ValT *)vals, n, pl.L, f,
                                                                tile_off, pl.T, bucket_base, (KeyT *)out_keys,
                                                                (ValT *)out_vals, lay, pl.seg));
    return DPK_OK;
}

template <typename KeyT, typename ValT, int PRE>
static int launch_scatter(const void *keys, const void *vals, int64_t n, const Plan &pl_in, const PartFn &f,
                          const int32_t *tile_off, const int64_t *bucket_base, void *out_keys,
                          void *out_vals, cudaStream_t st) {
    Plan pl = pl_in;
    if (pl.seg.unordered == 2) {  // unordered + plain/segmented destination: the TMA bulk-store kernel
        constexpr int vb = std::is_same<ValT, NoVal>::value ? 0 : (int)sizeof(ValT);
        const bool fits = (pl.pack & PK_OUT) ? bulk_smem(2 * (int)sizeof(KeyT), 0, f.nbuckets(), 8192).total <= 220 * 1024
                        : pl.pack ? bulk_smem((int)sizeof(KeyT), vb, f.nbuckets(), 8192).total <= 220 * 1024
                                  : bulk_smem((int)sizeof(KeyT), vb, f.nbuckets(), PT_TILE, pl.seg.key_ptrs != nullptr).total <= 110 * 1024;
        if (fits)
            return launch_scatter_bulk<KeyT, ValT, PRE>(keys, vals, n, pl, f, tile_off, bucket_base, out_keys, out_vals, st);
        pl.seg.unordered = (f.nbuckets() % 2 == 0) ? 1 : 0;  // too many buckets for two resident CTAs: the round-1 kernel
    }
    // dpk_set_option("scatter_items"): 16 or 8 rows per thread and tile (A/B switch; packed rows: 16)
    if (g_scatter_items == 8 && !pl.pack)
        return launch_scatter_items<KeyT, ValT, PRE, 8>(keys, vals, n, pl, f, tile_off, bucket_base, out_keys, out_vals, st);
    return launch_scatter_items<KeyT, ValT, PRE, 16>(keys, vals, n, pl, f, tile_off, bucket_base, out_keys, out_vals, st);
}

template <typename KeyT, int PRE>
static int dispatch_val(const void *keys, const void *vals, int32_t val_bytes, int64_t n, const Plan &pl,
                        const PartFn &f, const int32_t *tile_off, const int64_t *bucket_base,
                        void *out_keys, void *out_vals, cudaStream_t st) {
    if (pl.pack) {
        if (vals == nullptr && !(pl.pack & PK_IN)) return fail(DPK_ERR_INVALID, "packed rows need a value column");
        if (val_bytes != (int)sizeof(KeyT)) return fail(DPK_ERR_UNSUPPORTED, "packed rows need values as wide as the keys (%d B), got %d B", (int)sizeof(KeyT), val_bytes);
        if (pl.seg.key_ptrs) return fail(DPK_ERR_UNSUPPORTED, "packed rows are not written through pointer tables");
        if (((pl.pack & PK_OUT) && ((uintptr_t)out_keys % (2 * sizeof(KeyT)))) || ((pl.pack & PK_IN) && ((uintptr_t)keys % (2 * sizeof(KeyT)))))
            return fail(DPK_ERR_INVALID, "packed rows must be aligned to their %d-byte size", 2 * (int)sizeof(KeyT));
    }
    if ((vals == nullptr && !(pl.pack & PK_IN)) || val_bytes == 0)
        return launch_scatter<KeyT, NoVal, PRE>(keys, nullptr, n, pl, f, tile_off, bucket_base, out_keys, nullptr, st);
    if (val_bytes == 8)
        return launch_scatter<KeyT, int64_t, PRE>(keys, vals, n, pl, f, tile_off, bucket_base, out_keys, out_vals, st);
    if (val_bytes == 4)
        return launch_scatter<KeyT, int32_t, PRE>(keys, vals, n, pl, f, tile_off, bucket_base, out_keys, out_vals, st);
    return fail(DPK_ERR_UNSUPPORTED, "val_bytes must be 0, 4 or 8, got %d", val_bytes);
}

static int dispatch_scatter(const void *keys, int key_kind, const void *vals, int32_t val_bytes, int64_t n,
                            const Plan &pl_in, const PartFn &f, const int32_t *tile_off,
                            const int64_t *bucket_base, void *out_keys, void *out_vals, cudaStream_t st) {
    Plan pl = pl_in;
    if (key_kind >= 0 && (key_kind & DPK_K_PACKED)) {  // packed output
        key_kind &= ~DPK_K_PACKED;
        pl.pack |= PK_OUT;
    }
    if (key_kind >= DPK_K_UNORDERED) {  // caller does not need input order inside a bucket
        key_kind -= DPK_K_UNORDERED;
        if (f.nbuckets() % 2 == 0) pl.seg.unordered = 1;  // packed 16-bit counter pairs need an even bucket count
        if (g_scatter_bulk && (pl.seg.key_ptrs == nullptr || g_scatter_ptr_bulk)) pl.seg.unordered = 2;
    } else if (pl.seg.unordered && g_scatter_bulk && pl.seg.key_ptrs == nullptr) {
        pl.seg.unordered = 2;  // segmented mode (reduce side): never ordered
    }
    // the scatter only moves bits: 8-byte keys share the int64/uint64/double code
    // paths for hashing, so dispatch on the hash kind
    switch (key_kind) {
    case -1: return dispatch_val<int64_t, true>(keys, vals, val_bytes, n, pl, f, tile_off, bucket_base, out_keys, out_vals, st);
    case DPK_K_I64: return dispatch_val<int64_t, false>(keys, vals, val_bytes, n, pl, f, tile_off, bucket_base, out_keys, out_vals, st);
    case DPK_K_I32: return dispatch_val<int32_t, false>(keys, vals, val_bytes, n, pl, f, tile_off, bucket_base, out_keys, out_vals, st);
    case DPK_K_F64: return dispatch_val<double, false>(keys, vals, val_bytes, n, pl, f, tile_off, bucket_base, out_keys, out_vals, st);
    case DPK_K_U64: return dispatch_val<uint64_t, false>(keys, vals, val_bytes, n, pl, f, tile_off, bucket_base, out_keys, out_vals, st);
    case DPK_K_F32: return dispatch_val<float, false>(keys, vals, val_bytes, n, pl, f, tile_off, bucket_base, out_keys, out_vals, st);
    case DPK_K_ROWID:
        if (!f.row_hash) return fail(DPK_ERR_INVALID, "DPK_K_ROWID needs key_aux (the per-row hash column)");
        return dispatch_val<int64_t, 2>(keys, vals, val_bytes, n, pl, f, tile_off, bucket_base, out_keys, out_vals, st);
    }
    return fail(DPK_ERR_UNSUPPORTED, "key kind %d is unhashable by portable_hash", key_kind);
}

static int check_common(const void *keys, int64_t n, int32_t P, int32_t sub_bits, void *ws, int64_t ws_bytes) {
    if (n < 0 || n >= ((int64_t)1 << 31)) return fail(DPK_ERR_INVALID, "n=%lld out of range [0, 2^31)", (long long)n);
    if (P < 1 || sub_bits < 0 || sub_bits > 12 || ((int64_t)P << sub_bits) > DPK_MAX_PARTITIONS)
        return fail(DPK_ERR_UNSUPPORTED, "P=%d (x 2^%d sub-buckets) out of range [1, %d]", P, sub_bits, DPK_MAX_PARTITIONS);
    P <<= sub_bits;
    if (n > 0 && !keys) return fail(DPK_ERR_INVALID, "keys is NULL");
    if (!ws || ws_bytes < ws_total_bytes(P)) return fail(DPK_ERR_WORKSPACE, "workspace needs %lld B, got %lld", (long long)ws_total_bytes(P), (long long)ws_bytes);
    return DPK_OK;
}

// ---------------------------------------------------- segmented multisplit
constexpr int SEG_CHUNK_TILES = 4;
constexpr int64_t SEG_CHUNK = (int64_t)SEG_CHUNK_TILES * PT_TILE;  // rows per chunk

static inline int64_t seg_max_chunks(int64_t n, int32_t F1, int32_t nsrc) {
    return n / SEG_CHUNK + (int64_t)F1 * nsrc + 1;
}

// single CTA: chunk table + bucket-major row offsets from the segment matrix
__global__ void __launch_bounds__(PT_THREADS)
k_seg_plan(const int64_t *__restrict__ seg_start, const int64_t *__restrict__ seg_rows, int32_t nsrc, int32_t F1,
           int64_t *__restrict__ brow_off, int64_t *__restrict__ cfirst, int64_t *__restrict__ cbeg,
           int64_t *__restrict__ cend, int32_t *__restrict__ ctotal) {
    __shared__ long long s_rows[PT_THREADS], s_chunks[PT_THREADS];
    const int E = (F1 + PT_THREADS - 1) / PT_THREADS;
    const int b0 = threadIdx.x * E, b1 = min(b0 + E, F1);
    long long rows = 0, chunks = 0;
    for (int b = b0; b < b1; b++)
        for (int s = 0; s < nsrc; s++) {
            long long r = seg_rows[(int64_t)s * F1 + b];
            rows += r;
            chunks += (r + SEG_CHUNK - 1) / SEG_CHUNK;
        }
    s_rows[threadIdx.x] = rows;
    s_chunks[threadIdx.x] = chunks;
    __syncthreads();
    long long rbase = 0, cbase = 0;
    for (int t = 0; t < (int)threadIdx.x; t++) { rbase += s_rows[t]; cbase += s_chunks[t]; }
    for (int b = b0; b < b1; b++) {
        brow_off[b] = rbase;
        cfirst[b] = cbase;
        for (int s = 0; s < nsrc; s++) {
            const long long r0 = seg_start[(int64_t)s * F1 + b], r = seg_rows[(int64_t)s * F1 + b];
            for (long long o = 0; o < r; o += SEG_CHUNK) {
                cbeg[cbase] = r0 + o;
                cend[cbase] = r0 + min(r, o + SEG_CHUNK);
                cbase++;
            }
            rbase += r;
        }
    }
    if (b0 < F1 && b1 == F1) { brow_off[F1] = rbase; cfirst[F1] = cbase; *ctotal = (int32_t)cbase; }
    if (F1 == 0 && threadIdx.x == 0) { brow_off[0] = 0; cfirst[0] = 0; *ctotal = 0; }
}

// one CTA per first-level bucket: fine-bucket offsets and per-chunk output positions
__global__ void __launch_bounds__(PT_THREADS)
k_seg_scan(const int32_t *__restrict__ chunk_counts, const int64_t *__restrict__ cfirst,
           const int64_t *__restrict__ brow_off, int32_t F1, int32_t S2, int64_t *__restrict__ chunk_off,
           int64_t *__restrict__ fine_off) {
    extern __shared__ int32_t s_tot[];  // [S2] totals, then exclusive bases
    __shared__ int s_warp[PT_WARPS];
    const int b = blockIdx.x;
    const int64_t c0 = cfirst[b], c1 = cfirst[b + 1];
    for (int p = threadIdx.x; p < S2; p += PT_THREADS) {
        int t = 0;
        for (int64_t c = c0; c < c1; c++) t += chunk_counts[c * S2 + p];
        s_tot[p] = t;
    }
    __syncthreads();
    const int E = (S2 + PT_THREADS - 1) / PT_THREADS;
    const int p0 = threadIdx.x * E, p1 = min(p0 + E, S2);
    int sum = 0;
    for (int p = p0; p < p1; p++) sum += s_tot[p];
    int tot;
    int run = block_excl_scan(sum, s_warp, &tot);
    for (int p = p0; p < p1; p++) {
        int t = s_tot[p];
        s_tot[p] = run;
        run += t;
    }
    __syncthreads();
    const int64_t base = brow_off[b];
    for (int p = threadIdx.x; p < S2; p += PT_THREADS) {
        int64_t pos = base + s_tot[p];
        fine_off[(int64_t)b * S2 + p] = pos;
        for (int64_t c = c0; c < c1; c++) {
            chunk_off[c * S2 + p] = pos;
            pos += chunk_counts[c * S2 + p];
        }
    }
    if (b == F1 - 1 && threadIdx.x == 0) fine_off[(int64_t)F1 * S2] = brow_off[F1];
}

int64_t seg_multisplit_ws_bytes(int64_t n, int32_t F1, int32_t S2, int32_t nsrc) {
    const int64_t maxc = seg_max_chunks(n, F1, nsrc);
    return align_up((int64_t)(F1 + 1) * 8, 256) * 2 + 256 + align_up(maxc * 8, 256) * 2 +
           align_up(maxc * S2 * 4, 256) + align_up(maxc * S2 * 8, 256);
}

int seg_multisplit(const void *keys, int key_kind, const void *vals, int32_t val_bytes, int64_t n,
                   const PartFn &fine, int32_t F1, int32_t nsrc, const int64_t *seg_start,
                   const int64_t *seg_rows, void *out_keys, void *out_vals, int64_t *fine_off, void *ws,
                   int64_t ws_bytes, cudaStream_t st, bool stable, int pack) {
    const int32_t S2 = fine.nbuckets();
    if (ws_bytes < seg_multisplit_ws_bytes(n, F1, S2, nsrc)) return fail(DPK_ERR_WORKSPACE, "segmented multisplit workspace too small");
    const int64_t maxc = seg_max_chunks(n, F1, nsrc);
    char *w = (char *)ws;
    int64_t *brow_off = (int64_t *)w; w += align_up((int64_t)(F1 + 1) * 8, 256);
    int64_t *cfirst = (int64_t *)w; w += align_up((int64_t)(F1 + 1) * 8, 256);
    int32_t *ctotal = (int32_t *)w; w += 256;
    int64_t *cbeg = (int64_t *)w; w += align_up(maxc * 8, 256);
    int64_t *cend = (int64_t *)w; w += align_up(maxc * 8, 256);
    int32_t *chunk_counts = (int32_t *)w; w += align_up(maxc * S2 * 4, 256);
    int64_t *chunk_off = (int64_t *)w;
    DPK_LAUNCH("seg_plan", st, k_seg_plan<<<1, PT_THREADS, 0, st>>>(seg_start, seg_rows, nsrc, F1, brow_off, cfirst, cbeg, cend, ctotal));
    Plan pl;
    pl.T = (int32_t)maxc;
    pl.L = 0;
    // the reduce side never needs the order of rows inside a fine bucket
    pl.seg = SegTab{cbeg, cend, ctotal, chunk_counts, chunk_off, nullptr, nullptr, (S2 % 2 == 0) ? 1 : (g_scatter_bulk ? 2 : 0)};
    pl.pack = pack;
    if (stable) {   // radix passes of the group-by: rows of a fine bucket keep their order (warp-match ranking)
        pl.seg.unordered = 0;
        pl.label_count = "radix_count";
        pl.label_scatter = "radix_scatter";
    }
    int rc = DPK_OK;
    if (n > 0) {
        rc = dispatch_count(keys, key_kind, n, pl, fine, nullptr, st);
        if (rc) return rc;
    }
    DPK_LAUNCH("seg_scan", st, k_seg_scan<<<F1, PT_THREADS, (size_t)S2 * 4, st>>>(chunk_counts, cfirst, brow_off, F1, S2, chunk_off, fine_off));
    if (n > 0) rc = dispatch_scatter(keys, key_kind, vals, val_bytes, n, pl, fine, nullptr, nullptr, out_keys, out_vals, st);
    return rc;
}

}  // namespace dpk

using namespace dpk;

extern "C" {

int64_t dpk_partition_workspace_bytes(int64_t n, int32_t nbuckets) {
    (void)n;
    if (nbuckets < 1) nbuckets = 1;
    return ws_total_bytes(nbuckets);
}

int dpk_partition_count(const void *keys, int key_kind, const int64_t *key_aux, int64_t n, int32_t P,
                        const int64_t *thresholds, int32_t nthr, int32_t sub_bits, int64_t *out_counts,
                        void *ws, int64_t ws_bytes, dpk_stream_t stream) {
    int rc = check_common(keys, n, P, sub_bits, ws, ws_bytes);
    if (rc) return rc;
    if (!out_counts) return fail(DPK_ERR_INVALID, "out_counts is NULL");
    PartFn f;
    rc = make_partfn(P, thresholds, nthr, sub_bits, &f);
    if (rc) return rc;
    f.row_hash = key_aux;
    const int32_t F = f.nbuckets();
    cudaStream_t st = (cudaStream_t)stream;
    int32_t *tile_counts = (int32_t *)ws;
    Plan pl = make_plan(n);
    if (n == 0) {
        DPK_CUDA_TRY(cudaMemsetAsync(tile_counts, 0, (size_t)F * pl.T * 4, st));
    } else {
        rc = dispatch_count(keys, key_kind, n, pl, f, tile_counts, st);
        if (rc) return rc;
    }
    DPK_LAUNCH("part_scan", st, k_part_scan<<<F, PT_THREADS, 0, st>>>(tile_counts, pl.T, out_counts));
    return DPK_OK;
}

int dpk_partition_scatter(const void *keys, int key_kind, const int64_t *key_aux, const void *vals,
                          int32_t val_bytes, int64_t n, int32_t P, const int64_t *thresholds, int32_t nthr,
                          int32_t sub_bits,
                          const int64_t *bucket_base, void *out_keys, void *out_vals, void *ws,
                          int64_t ws_bytes, dpk_stream_t stream) {
    int rc = check_common(keys, n, P, sub_bits, ws, ws_bytes);
    if (rc) return rc;
    if (n == 0) return DPK_OK;
    if (!bucket_base || !out_keys) return fail(DPK_ERR_INVALID, "NULL pointer");
    PartFn f;
    rc = make_partfn(P, thresholds, nthr, sub_bits, &f);
    if (rc) return rc;
    f.row_hash = key_aux;
    Plan pl = make_plan(n);
    return dispatch_scatter(keys, key_kind, vals, val_bytes, n, pl, f, (const int32_t *)ws, bucket_base,
                            out_keys, out_vals, (cudaStream_t)stream);
}

int dpk_partition(const void *keys, int key_kind, const int64_t *key_aux, const void *vals, int32_t val_bytes,
                  int64_t n, int32_t P, const int64_t *thresholds, int32_t nthr, int32_t sub_bits, void *out_keys, void *out_vals,
                  int64_t *out_offsets, void *ws, int64_t ws_bytes, dpk_stream_t stream) {
    int rc = check_common(keys, n, P, sub_bits, ws, ws_bytes);
    if (rc) return rc;
    if (!out_offsets) return fail(DPK_ERR_INVALID, "out_offsets is NULL");
    const int32_t F = P << sub_bits;
    int64_t *totals = (int64_t *)((char *)ws + ws_counts_bytes(F));
    rc = dpk_partition_count(keys, key_kind, key_aux, n, P, thresholds, nthr, sub_bits, totals, ws, ws_bytes, stream);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    DPK_LAUNCH("part_offsets", st, k_part_offsets<<<1, PT_THREADS, 0, st>>>(totals, F, out_offsets));
    return dpk_partition_scatter(keys, key_kind, key_aux, vals, val_bytes, n, P, thresholds, nthr, sub_bits, out_offsets,
                                 out_keys, out_vals, ws, ws_bytes, stream);
}

// Fused scatter + exchange: like dpk_partition_scatter, but bucket b is written through
// key_dst_ptrs[b] / val_dst_ptrs[b] (absolute device addresses, device arrays of F entries): the
// caller points each bucket at its slot in the owning GPU's receive buffer (peer memory mapped over
// NVLink, or local memory), so the rows land where the reducer reads them and no separate
// alltoallv pass over HBM is needed.  Must follow dpk_partition_count with the same arguments.
int dpk_partition_scatter_ptrs(const void *keys, int key_kind, const int64_t *key_aux, const void *vals,
                               int32_t val_bytes, int64_t n, int32_t P, const int64_t *thresholds, int32_t nthr,
                               int32_t sub_bits, const uint64_t *key_dst_ptrs, const uint64_t *val_dst_ptrs,
                               void *ws, int64_t ws_bytes, dpk_stream_t stream) {
    int rc = check_common(keys, n, P, sub_bits, ws, ws_bytes);
    if (rc) return rc;
    if (n == 0) return DPK_OK;
    if (!key_dst_ptrs || (vals && val_bytes && !val_dst_ptrs)) return fail(DPK_ERR_INVALID, "NULL pointer table");
    PartFn f;
    rc = make_partfn(P, thresholds, nthr, sub_bits, &f);
    if (rc) return rc;
    f.row_hash = key_aux;
    Plan pl = make_plan(n);
    pl.seg.key_ptrs = key_dst_ptrs;
    pl.seg.val_ptrs = val_dst_ptrs;
    return dispatch_scatter(keys, key_kind, vals, val_bytes, n, pl, f, (const int32_t *)ws, nullptr, nullptr, nullptr,
                            (cudaStream_t)stream);
}

// first row of segment (s, b) in a source-major, bucket-major buffer: single CTA
__global__ void __launch_bounds__(PT_THREADS)
k_seg_starts(const int64_t *__restrict__ seg_rows, int32_t nsrc, int32_t F, int64_t *__restrict__ seg_start) {
    __shared__ long long s_part[PT_THREADS];
    __shared__ long long s_carry;
    const int E = (F + PT_THREADS - 1) / PT_THREADS;
    const int b0 = threadIdx.x * E, b1 = min(b0 + E, F);
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int s = 0; s < nsrc; s++) {
        long long mine = 0;
        for (int b = b0; b < b1; b++) mine += seg_rows[(int64_t)s * F + b];
        s_part[threadIdx.x] = mine;
        __syncthreads();
        long long base = s_carry, tot = 0;
        for (int t = 0; t < PT_THREADS; t++) {
            if (t < (int)threadIdx.x) base += s_part[t];
            tot += s_part[t];
        }
        for (int b = b0; b < b1; b++) {
            seg_start[(int64_t)s * F + b] = base;
            base += seg_rows[(int64_t)s * F + b];
        }
        __syncthreads();
        if (threadIdx.x == 0) s_carry += tot;
        __syncthreads();
    }
}

int64_t dpk_radix_pass_seg_workspace_bytes(int64_t n, int32_t nbuckets, int32_t nsrc, int32_t bits) {
    if (n < 0) n = 0;
    if (nbuckets < 1) nbuckets = 1;
    if (nsrc < 1) nsrc = 1;
    return align_up((int64_t)nbuckets * nsrc * 8, 256) + seg_multisplit_ws_bytes(n, nbuckets, 1 << bits, nsrc);
}

// One stable LSD radix pass INSIDE every first-level bucket (the group-by's reduce side sorts each hash bucket by
// its key bits independently -- all rows of a key are in one bucket -- so no pass over the partition id is needed
// afterwards): the input is source-major, bucket-major (seg_rows[nsrc][nbuckets], what the exchange delivers; nsrc = 1
// for the later passes), the output is bucket-major with every bucket stably split by the digit `shift` (bits wide) of
// the raw key bits.  out_fine_off[nbuckets << bits + 1] delimits the digit groups (optional, may be NULL... it is
// always written into the workspace; pass a buffer to keep it).
int dpk_radix_pass_seg(const int64_t *keys, const void *vals, int32_t val_bytes, int64_t n, int32_t shift, int32_t bits,
                       int32_t nbuckets, int32_t nsrc, const int64_t *seg_rows, int64_t *out_keys, void *out_vals,
                       int64_t *out_fine_off, void *ws, int64_t ws_bytes, dpk_stream_t stream) {
    if (bits < 1 || bits > 10 || shift < 0 || shift > 63) return fail(DPK_ERR_INVALID, "bad radix digit shift=%d bits=%d", shift, bits);
    if (n < 0 || n >= ((int64_t)1 << 31)) return fail(DPK_ERR_INVALID, "n=%lld out of range [0, 2^31)", (long long)n);
    if (nbuckets < 1 || nsrc < 1 || !seg_rows || !out_fine_off || !ws) return fail(DPK_ERR_INVALID, "bad segment description");
    if (n > 0 && (!keys || !out_keys)) return fail(DPK_ERR_INVALID, "NULL pointer");
    if (ws_bytes < dpk_radix_pass_seg_workspace_bytes(n, nbuckets, nsrc, bits)) return fail(DPK_ERR_WORKSPACE, "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    int64_t *seg_start = (int64_t *)ws;
    void *ws2 = (char *)ws + align_up((int64_t)nbuckets * nsrc * 8, 256);
    DPK_LAUNCH("seg_starts", st, k_seg_starts<<<1, PT_THREADS, 0, st>>>(seg_rows, nsrc, nbuckets, seg_start));
    PartFn f;
    f.P = 1 << bits; f.mode = 4; f.magic = 0; f.shift = shift; f.nthr = 0; f.thresholds = nullptr; f.sub_bits = 0;
    f.row_hash = nullptr;
    return seg_multisplit(keys, -1, vals, val_bytes, n, f, nbuckets, nsrc, seg_start, seg_rows, out_keys, out_vals,
                          out_fine_off, ws2, ws_bytes - align_up((int64_t)nbuckets * nsrc * 8, 256), st, true);
}

// One stable LSD radix pass over int64 key bits: the same multisplit with the
// bucket = digit `shift` (bits wide) of the raw key.  groupByKey's reduce side is
// a stable sort by key built from these passes (dpk_group.cu).
int dpk_radix_pass(const int64_t *keys, const void *vals, int32_t val_bytes, int64_t n, int32_t shift,
                   int32_t bits, int64_t *out_keys, void *out_vals, void *ws, int64_t ws_bytes,
                   dpk_stream_t stream) {
    if (bits < 1 || bits > 12 || shift < 0 || shift > 63)
        return fail(DPK_ERR_INVALID, "bad radix digit shift=%d bits=%d", shift, bits);
    const int32_t F = 1 << bits;
    int rc = check_common(keys, n, F, 0, ws, ws_bytes);
    if (rc) return rc;
    if (n == 0) return DPK_OK;
    if (!out_keys) return fail(DPK_ERR_INVALID, "NULL pointer");
    PartFn f;
    f.P = F; f.mode = 4; f.magic = 0; f.shift = shift; f.nthr = 0; f.thresholds = nullptr; f.sub_bits = 0;
    f.row_hash = nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    int32_t *tile_counts = (int32_t *)ws;
    int64_t *totals = (int64_t *)((char *)ws + ws_counts_bytes(F));
    int64_t *offsets = (int64_t *)((char *)totals + align_up((int64_t)F * 8, 256));
    Plan pl = make_plan(n);
    pl.label_count = "radix_count";
    pl.label_scatter = "radix_scatter";
    rc = dispatch_count(keys, -1, n, pl, f, tile_counts, st);
    if (rc) return rc;
    DPK_LAUNCH("part_scan", st, k_part_scan<<<F, PT_THREADS, 0, st>>>(tile_counts, pl.T, totals));
    DPK_LAUNCH("part_offsets", st, k_part_offsets<<<1, PT_THREADS, 0, st>>>(totals, F, offsets));
    return dispatch_scatter(keys, -1, vals, val_bytes, n, pl, f, tile_counts, offsets, out_keys, out_vals, st);
}

}  // extern "C"
