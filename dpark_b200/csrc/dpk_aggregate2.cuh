// dpk_aggregate2.cuh -- reduce-side implementation 2, final stage, round-2 form (included by
// dpk_combine.cu after dpk_aggregate.cuh; the round-1 kernel k_smem_aggregate stays selectable with
// dpk_set_option("agg_impl", 0) as the A/B baseline and parity cross-check).
//
// One CTA merges one fine bucket (~1.5 k rows after the second-level split) at a time.  What changed
// (scripts/microbench/smem_ops.cu measures the shared-memory primitives this rests on):
//
//   * The rows of the bucket are STAGED in shared memory (key bits + accumulator, 8 B each, row-linear),
//     and the hash table holds only a 32-bit TAG per slot: staged row index + 1 of the row that claimed
//     the slot (0 = free).  A claim is one atom.shared.cas.b32 (instead of the round-1 128-bit
//     {key, accumulator} claim), no key value is reserved as "empty" marker
//     (no side slot), and the claiming row's staged value IS the key's accumulator: rows that claim
//     (97.7 % of C2's rows) touch no accumulator at all; later rows of a key compare with the claimer's
//     staged key and add into its staged accumulator with native shared atomics.
//   * Output positions come from the claim ballots (row-index order: coalesced stores), summed per warp
//     and item into 64 counters that warp 0 scans while it does the decoupled look-back; no claim list,
//     no atomic on a CTA-wide counter.  The distinct rows are written from registers (key) and the
//     staged accumulator (conflict-free linear LDS).
//   * The tag table (16 KB) is cleared with 128-bit stores instead of one random reset per claimed row.
//   * 48 KB of shared memory per CTA instead of 72: four CTAs per SM.
//
// Buckets that do not fit one staging window (more than AG2_CAP rows: hot keys) take the general path:
// windows of rows are staged behind the RESIDENT distinct rows found so far (claimed rows are compacted
// to the front and re-tagged after every window), so a bucket of any size with up to ~AG2_CAP distinct
// keys is one pass; more distinct keys than that split the bucket into hash-disjoint passes (m, r).
// Splitting stops at AG2_MAX_M; a bucket that still overflows marks its partition as failed
// (out_counts[p] = -1, surfaced as DPK error by the caller) instead of dropping rows silently.
#pragma once

constexpr int AG2_THREADS = 256;
constexpr int AG2_WARPS = AG2_THREADS / 32;
constexpr int AG2_TAGS = 4096;
constexpr int AG2_CAP = 2048;                       // staged rows per window
constexpr int AG2_ITEMS = AG2_CAP / AG2_THREADS;    // 8 rows per thread and window
constexpr int AG2_GEN_ITEMS = 4;                    // general path: rows per thread and window (register pressure)
constexpr uint32_t AG2_IDX_MASK = 0xfffu;            // low tag bits: staged row index + 1 (<= AG2_CAP = 2^11)
constexpr int AG2_MINW = 256;                       // a window smaller than this is not worth a round: split the pass
constexpr int AG2_MAX_M = 1 << 16;                  // hash-disjoint passes use hash bits 12..27
constexpr int AG2_STACK = 40;

struct Ag2Shared {
    int fb, sp, overflow, nres;
    unsigned long long excl;
    int next_fb[2];                          // ticket of the next fine bucket (prefetched), by iteration parity
    long long next_r0[2], next_r1[2];        // ... and its row range
    int wcnt[AG2_ITEMS * AG2_WARPS];   // claims per (item, warp), then their exclusive prefix
    int total;
    int stack_m[AG2_STACK], stack_r[AG2_STACK];
};

__device__ __forceinline__ uint32_t sm_ld_u32(uint32_t a) {
    uint32_t v;
    asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t sm_cas_u32(uint32_t a, uint32_t cmp, uint32_t val) {
    uint32_t old;
    asm volatile("atom.shared.cas.b32 %0, [%1], %2, %3;" : "=r"(old) : "r"(a), "r"(cmp), "r"(val) : "memory");
    return old;
}
__device__ __forceinline__ long long sm_ld_s64(uint32_t a) {
    long long v;
    asm volatile("ld.volatile.shared.b64 %0, [%1];" : "=l"(v) : "r"(a) : "memory");
    return v;
}

// Insert the staged rows [lo, hi) of the window (staged index = lo + j * THREADS + tid) into the tag table.
// Returns the bit mask of the items this thread claimed.  Per item the claim ballot gives the number of claims
// of the warp (lane j keeps item j's count in *lane_cnt) and this lane's rank among them (8 bits per item in
// offs[2]); SLOTS: remember the slot of every claimed item (12 bits each in slots[3]) for re-tagging.
// (m, r): hash-disjoint pass filter.  Whole warps run the loop together (ballots).
template <typename AccT, bool SLOTS, int NI>
__device__ __forceinline__ unsigned ag2_insert(int lo, int hi, int m, int r, int op, uint32_t tag_base, uint32_t key_base,
                                               uint32_t acc_base, long long *s_acc, uint32_t (&offs)[2], int *lane_cnt,
                                               uint32_t (&slots)[3]) {
    unsigned mine = 0;
    const int lane = threadIdx.x & 31;
    const unsigned lt = (1u << lane) - 1u;
    offs[0] = offs[1] = 0;
    if constexpr (SLOTS) slots[0] = slots[1] = slots[2] = 0;
    int lc = 0;
#pragma unroll
    for (int j = 0; j < NI; j++) {
        const int idx = lo + j * AG2_THREADS + (int)threadIdx.x;
        bool claimed = false;
        if (idx < hi) {
            const long long k = sm_ld_s64(key_base + (uint32_t)idx * 8u);
            const uint32_t hs = slot_hash32((uint64_t)k);
            if (m == 1 || (int)((hs >> 12) & (uint32_t)(m - 1)) == r) {
                uint32_t h = hs & (AG2_TAGS - 1);
                // tag = 20 fingerprint bits of the slot hash | staged row index + 1: a slot owned by another key is
                // recognised from the tag alone (no key load, no 64-bit compare) except for one in 2^20 collisions
                const uint32_t fp = hs & ~(uint32_t)AG2_IDX_MASK;
                for (;;) {
                    uint32_t t = sm_ld_u32(tag_base + h * 4u);
                    if (t == 0u) {
                        t = sm_cas_u32(tag_base + h * 4u, 0u, fp | ((uint32_t)idx + 1u));
                        if (t == 0u) { claimed = true; break; }
                    }
                    if ((t & ~(uint32_t)AG2_IDX_MASK) == fp) {
                        const uint32_t o = (t & AG2_IDX_MASK) - 1u;
                        if (sm_ld_s64(key_base + o * 8u) == k) {   // a row of the same key owns the slot: add into its accumulator
                            const long long mv = sm_ld_s64(acc_base + (uint32_t)idx * 8u);
                            if constexpr (std::is_same<AccT, double>::value)
                                sm_apply<double>(op, acc_base + o * 8u, s_acc + o, __longlong_as_double(mv));
                            else
                                sm_apply<int64_t>(op, acc_base + o * 8u, s_acc + o, (int64_t)mv);
                            break;
                        }
                    }
                    h = (h + 1u) & (AG2_TAGS - 1);
                }
                if constexpr (SLOTS) {
                    if (claimed) {   // 12 bits per item: items 0..7 at bit 12*j of the 96-bit word slots[0..2]
                        const int bit = 12 * j;
                        slots[bit >> 5] |= h << (bit & 31);
                        if ((bit & 31) > 20) slots[(bit >> 5) + 1] |= h >> (32 - (bit & 31));
                    }
                }
            }
        }
        const unsigned cmj = __ballot_sync(0xffffffffu, claimed);
        if (lane == j) lc = __popc(cmj);
        offs[j >> 2] |= (uint32_t)__popc(cmj & lt) << (8 * (j & 3));
        if (claimed) mine |= 1u << j;
    }
    *lane_cnt = lc;
    return mine;
}
// Fast-path form of ag2_insert (one window, one pass, no slots): the items are taken four at a time and the common
// case -- the home slot is free and the claim succeeds -- is issued as independent instruction groups (4 key loads,
// 4 hashes, 4 tag loads, 4 claims) instead of four dependent probe loops; only rows that met an occupied slot enter
// the probe loop.  (ncu r02a: the loop form spent 11 % of its samples on branch resolution and 21 % on fixed-latency
// and shared-memory dependencies with one row in flight per thread.)
template <typename AccT, int NI>
__device__ __forceinline__ unsigned ag2_insert_batched(int n, int op, uint32_t tag_base, uint32_t key_base, uint32_t acc_base,
                                                       long long *s_acc, uint32_t (&offs)[2], int *lane_cnt) {
    static_assert(NI % 4 == 0, "items are taken four at a time");
    unsigned mine = 0;
    const int lane = threadIdx.x & 31;
    const unsigned lt = (1u << lane) - 1u;
    offs[0] = offs[1] = 0;
    int lc = 0;
#pragma unroll
    for (int g = 0; g < NI; g += 4) {
        long long k[4];
        uint32_t h[4], t[4];
        bool claimed[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int idx = (g + u) * AG2_THREADS + (int)threadIdx.x;
            k[u] = idx < n ? sm_ld_s64(key_base + (uint32_t)idx * 8u) : 0ll;
        }
        uint32_t fpb[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {   // (slot hash, fingerprint)
            const uint32_t hs = slot_hash32((uint64_t)k[u]);
            h[u] = hs & (AG2_TAGS - 1);
            fpb[u] = hs & ~(uint32_t)AG2_IDX_MASK;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int idx = (g + u) * AG2_THREADS + (int)threadIdx.x;
            t[u] = idx < n ? sm_ld_u32(tag_base + h[u] * 4u) : 0xffffffffu;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int idx = (g + u) * AG2_THREADS + (int)threadIdx.x;
            claimed[u] = false;
            if (t[u] == 0u) {
                t[u] = sm_cas_u32(tag_base + h[u] * 4u, 0u, fpb[u] | ((uint32_t)idx + 1u));
                claimed[u] = t[u] == 0u;
            }
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int idx = (g + u) * AG2_THREADS + (int)threadIdx.x;
            if (idx < n && !claimed[u]) {   // the home slot belongs to another row: same key -> add, else probe on
                uint32_t hh = h[u], tt = t[u];
                for (;;) {
                    if (tt == 0u) {
                        tt = sm_cas_u32(tag_base + hh * 4u, 0u, fpb[u] | ((uint32_t)idx + 1u));
                        if (tt == 0u) { claimed[u] = true; break; }
                    }
                    if ((tt & ~(uint32_t)AG2_IDX_MASK) == fpb[u]) {
                        const uint32_t o = (tt & AG2_IDX_MASK) - 1u;
                        if (sm_ld_s64(key_base + o * 8u) == k[u]) {
                            const long long mv = sm_ld_s64(acc_base + (uint32_t)idx * 8u);
                            if constexpr (std::is_same<AccT, double>::value)
                                sm_apply<double>(op, acc_base + o * 8u, s_acc + o, __longlong_as_double(mv));
                            else
                                sm_apply<int64_t>(op, acc_base + o * 8u, s_acc + o, (int64_t)mv);
                            break;
                        }
                    }
                    hh = (hh + 1u) & (AG2_TAGS - 1);
                    tt = sm_ld_u32(tag_base + hh * 4u);
                }
            }
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int j = g + u;
            const unsigned cmj = __ballot_sync(0xffffffffu, claimed[u]);
            if (lane == j) lc = __popc(cmj);
            offs[j >> 2] |= (uint32_t)__popc(cmj & lt) << (8 * (j & 3));
            if (claimed[u]) mine |= 1u << j;
        }
    }
    *lane_cnt = lc;
    return mine;
}

__device__ __forceinline__ int ag2_off(const uint32_t (&offs)[2], int j) { return (int)((offs[j >> 2] >> (8 * (j & 3))) & 0xffu); }
__device__ __forceinline__ uint32_t ag2_slot(const uint32_t (&slots)[3], int j) {
    const int bit = 12 * j;
    uint32_t v = slots[bit >> 5] >> (bit & 31);
    if ((bit & 31) > 20) v |= slots[(bit >> 5) + 1] << (32 - (bit & 31));
    return v & 0xfffu;
}

// CURSOR = true (default): the output range of a fine bucket inside its partition is reserved with ONE
// atomicAdd on the partition's count (the buckets of a partition come out in any order: a reduce partition is a
// set).  CURSOR = false: the round-1 scheme, a chained scan with decoupled look-back over fb_state[] (fine buckets in
// order; the rows inside one still come in run-to-run varying order, as the unordered multisplits deliver them).
// With hundreds of resident CTAs all finishing equal-sized buckets in lockstep, the look-back waits for the SLOWEST of its nearest predecessors every time, and a wider look-back window does not help; the atomic costs a fixed L2 round trip, no waiting on other CTAs, and lifts the
// in-order requirement, so the next ticket and its row range are prefetched a bucket ahead.
// PACKED: the fine buckets are packed records (keys: PackedRow array, vals unused) -- one load per row
template <typename KeyT, typename ValT, typename AccT, int MINB, bool CURSOR, bool BATCHED, bool FAST_ONLY = false,
          bool PACKED = false>
__global__ void __launch_bounds__(AG2_THREADS, MINB)
k_smem_aggregate2(const KeyT *__restrict__ keys, const ValT *__restrict__ vals, int op,
                  const int64_t *__restrict__ fine_off, int32_t nfine, int32_t fine_per_part,
                  const int64_t *__restrict__ part_offsets, KeyT *__restrict__ out_keys,
                  int64_t *__restrict__ out_vals, long long *__restrict__ out_counts,
                  unsigned long long *__restrict__ fb_state, int *__restrict__ work_counter,
                  int *__restrict__ part_err, const int *__restrict__ bucket_list, const int *__restrict__ bucket_count,
                  long long *__restrict__ phase_cycles, int *__restrict__ big_list = nullptr, int *__restrict__ big_count = nullptr) {
    // FAST_ONLY (CURSOR only): this instance contains the one-window path alone -- the general path's live state cost
    // the hot loop registers (r02f: 244 B of spills per thread at 64 registers, 0.3 GB of local-memory traffic per
    // launch) -- and appends oversized buckets to big_list for a second launch of the full kernel in list mode
    // phase_cycles != nullptr (dpk_set_option("agg_timing", 1), debugging): thread 0 adds the cycles between the
    // phase boundaries of every fast-path bucket: [0] top..rows loaded+staged (S), [1] S..inserts done (B),
    // [2] B..output range known (D), [3] D..write-out issued, [4] write-out..next top (A), [5] buckets
    long long tstamp = 0;
    auto stamp = [&](int k) {
        if (phase_cycles != nullptr && threadIdx.x == 0) {
            const long long now = clock64();
            if (k >= 0) atomicAdd(reinterpret_cast<unsigned long long *>(&phase_cycles[k]), (unsigned long long)(now - tstamp));
            tstamp = now;
        }
    };
    // bucket_list != nullptr (CURSOR only): the tickets index a list of fine buckets (the oversized ones
    // k_smem_aggregate3 left behind) instead of all nfine buckets
    const int nwork = bucket_list ? *bucket_count : nfine;
    auto bucket_of_ticket = [&](int t) { return bucket_list ? bucket_list[t] : t; };
    extern __shared__ __align__(16) long long s_dyn2[];  // [TAGS] u32 tags | [CAP] key bits | [CAP] accumulators
    uint32_t *s_tag = reinterpret_cast<uint32_t *>(s_dyn2);
    long long *s_key = s_dyn2 + AG2_TAGS / 2;
    long long *s_acc = s_key + AG2_CAP;
    const uint32_t tag_base = (uint32_t)__cvta_generic_to_shared(s_tag);
    const uint32_t key_base = (uint32_t)__cvta_generic_to_shared(s_key);
    const uint32_t acc_base = (uint32_t)__cvta_generic_to_shared(s_acc);
    __shared__ Ag2Shared sh;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    auto clear_tags = [&]() {
        uint4 *t4 = reinterpret_cast<uint4 *>(s_tag);
#pragma unroll
        for (int i = 0; i < AG2_TAGS / 4 / AG2_THREADS; i++) t4[i * AG2_THREADS + threadIdx.x] = make_uint4(0, 0, 0, 0);
    };
    // stage the rows [g0, g0 + w) of the input at staged indices [at, at + w); between its loads and its stores
    // thread 0 runs `between` (the ticket prefetch: its L2 round trip overlaps the row loads)
    auto stage = [&](int64_t g0, int w, int at, auto ni_tag, auto between) {
        constexpr int NI = decltype(ni_tag)::value;
        KeyT kr[NI];
        ValT vr[NI];
#pragma unroll
        for (int j = 0; j < NI; j++) {
            const int i = j * AG2_THREADS + (int)threadIdx.x;
            if (i < w) {
                if constexpr (PACKED) {
                    const PackedRow<KeyT, ValT> r = reinterpret_cast<const PackedRow<KeyT, ValT> *>(keys)[g0 + i];
                    kr[j] = r.k;
                    vr[j] = r.v;
                } else {
                    kr[j] = keys[g0 + i];
                    vr[j] = vals[g0 + i];
                }
            }
        }
        between();
#pragma unroll
        for (int j = 0; j < NI; j++) {
            const int i = j * AG2_THREADS + (int)threadIdx.x;
            if (i < w) {
                s_key[at + i] = key_bits<KeyT>(kr[j]);
                if constexpr (std::is_same<AccT, double>::value) s_acc[at + i] = __double_as_longlong((double)vr[j]);
                else s_acc[at + i] = (long long)vr[j];
            }
        }
    };
    auto nothing = []() {};
    // warp 0: exclusive prefix of the (item, warp) claim counts in place, total -> sh.total
    auto scan_claims = [&]() {
        constexpr int N = AG2_ITEMS * AG2_WARPS;   // 64
        int a = sh.wcnt[lane], b = sh.wcnt[lane + 32];
        int ia = a, ib = b;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            int ta = __shfl_up_sync(0xffffffffu, ia, d), tb = __shfl_up_sync(0xffffffffu, ib, d);
            if (lane >= d) { ia += ta; ib += tb; }
        }
        const int suma = __shfl_sync(0xffffffffu, ia, 31);
        sh.wcnt[lane] = ia - a;
        sh.wcnt[lane + 32] = suma + ib - b;
        if (lane == 31) sh.total = suma + ib;
        static_assert(N == 64, "scan_claims handles 64 counters");
    };

    clear_tags();
    if (threadIdx.x == 0) {
        const int t = atomicAdd(work_counter, 1);
        sh.next_fb[0] = t < nwork ? bucket_of_ticket(t) : nfine;
        if (t < nwork) { const int b = bucket_of_ticket(t); sh.next_r0[0] = fine_off[b]; sh.next_r1[0] = fine_off[b + 1]; }
    }
    for (int it = 0;; it++) {
        __syncthreads();                                            // (A) also: previous write-out and tag clear finished
        stamp(it ? 4 : -1);
        const int fb = sh.next_fb[it & 1];
        if (fb >= nfine) break;
        const int64_t r0 = sh.next_r0[it & 1], r1 = sh.next_r1[it & 1];
        const int p = fb / fine_per_part;
        const int first_fb = p * fine_per_part;
        const bool last_fb = fb == first_fb + fine_per_part - 1;
        const int64_t pbase = part_offsets[p];
        uint32_t offs[2], slots[3];
        int lane_cnt;
        // next ticket: taken while this bucket's rows are in flight (CURSOR: any order is fine; look-back: the ticket
        // must not be taken before this bucket is published, so it is taken at the end instead)
        int nt = 0;
        long long nr0 = 0, nr1 = 0;
        auto prefetch_ticket = [&]() {
            if (CURSOR && threadIdx.x == 0) nt = atomicAdd(work_counter, 1);
        };
        auto prefetch_range = [&]() {
            if (CURSOR && threadIdx.x == 0) {
                const int b = nt < nwork ? bucket_of_ticket(nt) : nfine;
                sh.next_fb[(it + 1) & 1] = b;
                if (b < nfine) { nr0 = fine_off[b]; nr1 = fine_off[b + 1]; }
            }
        };
        auto publish_range = [&]() {   // before a barrier that precedes (A) of the next iteration
            if (threadIdx.x == 0) {
                if (!CURSOR) {   // (look-back mode never runs in list mode)
                    nt = atomicAdd(work_counter, 1);
                    sh.next_fb[(it + 1) & 1] = nt;
                    if (nt < nfine) { nr0 = fine_off[nt]; nr1 = fine_off[nt + 1]; }
                }
                sh.next_r0[(it + 1) & 1] = nr0;
                sh.next_r1[(it + 1) & 1] = nr1;
            }
        };

        if (r1 - r0 <= AG2_CAP) {
            // ================= fast path: the whole bucket is one window, one pass
            const int n = (int)(r1 - r0);
            stage(r0, n, 0, std::integral_constant<int, AG2_ITEMS>(), prefetch_ticket);
            prefetch_range();
            __syncthreads();                                        // (S) rows staged
            stamp(0);
            const unsigned mine = BATCHED ? ag2_insert_batched<AccT, AG2_ITEMS>(n, op, tag_base, key_base, acc_base, s_acc, offs, &lane_cnt)
                                          : ag2_insert<AccT, false, AG2_ITEMS>(0, n, 1, 0, op, tag_base, key_base, acc_base, s_acc, offs, &lane_cnt, slots);
            if (lane < AG2_ITEMS) sh.wcnt[lane * AG2_WARPS + warp] = lane_cnt;
            if (CURSOR) publish_range();
            __syncthreads();                                        // (B) inserts done, claim counts written
            stamp(1);
            if (warp == 0) {
                scan_claims();
                __syncwarp();
                const unsigned long long cnt = (unsigned long long)sh.total;
                if constexpr (CURSOR) {
                    if (lane == 0) sh.excl = atomicAdd(reinterpret_cast<unsigned long long *>(&out_counts[p]), cnt);
                } else {
                    if (lane == 0) atomicExch(&fb_state[fb], AG_FLAG_AGG | cnt);
                    const unsigned long long e = ag_look_back(fb_state, first_fb, fb);
                    if (lane == 0) {
                        sh.excl = e;
                        atomicExch(&fb_state[fb], AG_FLAG_INC | (e + cnt));
                        if (last_fb) out_counts[p] = *(volatile int *)&part_err[p] ? -1ll : (long long)(e + cnt);
                    }
                }
            } else {
                clear_tags();   // 7 warps x 4 x 16 B per thread cover 14 KB; warp 0 clears its share after the barrier
            }
            if (!CURSOR) publish_range();
            __syncthreads();                                        // (D) offsets known
            stamp(2);
            const int64_t obase = pbase + (int64_t)sh.excl;
#pragma unroll
            for (int j = 0; j < AG2_ITEMS; j++) {
                if (mine & (1u << j)) {
                    const int idx = j * AG2_THREADS + (int)threadIdx.x;
                    const int64_t o = obase + sh.wcnt[j * AG2_WARPS + warp] + ag2_off(offs, j);
                    out_keys[o] = key_from_bits<KeyT>(s_key[idx]);
                    out_vals[o] = s_acc[idx];
                }
            }
            if (warp == 0) clear_tags();
            stamp(3);
            if (phase_cycles != nullptr && threadIdx.x == 0) atomicAdd(reinterpret_cast<unsigned long long *>(&phase_cycles[5]), 1ull);
            continue;  // barrier (A) of the next iteration orders the reads and the clear before the next staging
        }

        if constexpr (FAST_ONLY) {
            if (threadIdx.x == 0) big_list[atomicAdd(big_count, 1)] = fb;
            prefetch_ticket();
            prefetch_range();
            publish_range();
            continue;
        }
        // ================= general path: windows behind resident distinct rows, hash-disjoint passes on overflow
        prefetch_ticket();
        prefetch_range();
        unsigned long long written = 0, excl = 0;  // uniform
        bool have_excl = false, failed = false;
        if (threadIdx.x == 0) { sh.stack_m[0] = 1; sh.stack_r[0] = 0; sh.sp = 1; }
        __syncthreads();
        while (sh.sp > 0) {
            const int m = sh.stack_m[sh.sp - 1], r = sh.stack_r[sh.sp - 1];
            __syncthreads();
            if (threadIdx.x == 0) { sh.sp--; sh.overflow = 0; sh.nres = 0; }
            __syncthreads();
            int64_t cursor = r0;
            int nres = 0;
            bool ok = true;
            while (cursor < r1) {
                const int room = AG2_CAP - nres;
                if (room < AG2_MINW) { ok = false; break; }          // too many distinct keys for one pass
                const int w = (int)min((int64_t)min(room, AG2_GEN_ITEMS * AG2_THREADS), r1 - cursor);
                stage(cursor, w, nres, std::integral_constant<int, AG2_GEN_ITEMS>(), nothing);
                __syncthreads();
                const unsigned mine = ag2_insert<AccT, true, AG2_GEN_ITEMS>(nres, nres + w, m, r, op, tag_base, key_base, acc_base, s_acc, offs, &lane_cnt, slots);
                if (lane < AG2_ITEMS) sh.wcnt[lane * AG2_WARPS + warp] = lane_cnt;
                __syncthreads();
                // compact the claimed rows behind the residents and re-tag their slots
                long long kv[AG2_GEN_ITEMS], av[AG2_GEN_ITEMS];
#pragma unroll
                for (int j = 0; j < AG2_GEN_ITEMS; j++)
                    if (mine & (1u << j)) {
                        kv[j] = s_key[nres + j * AG2_THREADS + (int)threadIdx.x];
                        av[j] = s_acc[nres + j * AG2_THREADS + (int)threadIdx.x];
                    }
                if (warp == 0) scan_claims();
                __syncthreads();
#pragma unroll
                for (int j = 0; j < AG2_GEN_ITEMS; j++) {
                    if (mine & (1u << j)) {
                        const int ni = nres + sh.wcnt[j * AG2_WARPS + warp] + ag2_off(offs, j);
                        s_key[ni] = kv[j];
                        s_acc[ni] = av[j];
                        const uint32_t sl = ag2_slot(slots, j);
                        s_tag[sl] = (s_tag[sl] & ~(uint32_t)AG2_IDX_MASK) | ((uint32_t)ni + 1u);
                    }
                }
                nres += sh.total;
                cursor += w;
                __syncthreads();
            }
            if (!ok) {  // uniform: split this pass in two, or give up (error flag) when the hash bits are used up
                if (m * 2 <= AG2_MAX_M && sh.sp + 2 <= AG2_STACK) {
                    if (threadIdx.x == 0) {
                        sh.stack_m[sh.sp] = m * 2; sh.stack_r[sh.sp] = r; sh.sp++;
                        sh.stack_m[sh.sp] = m * 2; sh.stack_r[sh.sp] = r + m; sh.sp++;
                    }
                } else {
                    failed = true;
                }
                clear_tags();
                __syncthreads();
                continue;
            }
            if constexpr (CURSOR) {
                if (threadIdx.x == 0)
                    sh.excl = atomicAdd(reinterpret_cast<unsigned long long *>(&out_counts[p]), (unsigned long long)nres);
                __syncthreads();
                excl = sh.excl;
                written = 0;
            } else if (!have_excl) {  // multi-pass buckets publish only their inclusive value, at the end
                if (warp == 0) {
                    const unsigned long long e = ag_look_back(fb_state, first_fb, fb);
                    if (lane == 0) sh.excl = e;
                }
                __syncthreads();
                excl = sh.excl;
                have_excl = true;
            }
            const int64_t obase = pbase + (int64_t)(excl + written);
            for (int i = threadIdx.x; i < nres; i += AG2_THREADS) {
                out_keys[obase + i] = key_from_bits<KeyT>(s_key[i]);
                out_vals[obase + i] = s_acc[i];
            }
            written += (unsigned long long)nres;
            clear_tags();
            __syncthreads();
        }
        if (warp == 0) {
            if constexpr (CURSOR) {
                if (lane == 0 && failed) atomicExch(&part_err[p], 1);
            } else {
                unsigned long long e = have_excl ? excl : ag_look_back(fb_state, first_fb, fb);
                if (lane == 0) {
                    if (failed) { atomicExch(&part_err[p], 1); __threadfence(); }
                    atomicExch(&fb_state[fb], AG_FLAG_INC | (e + written));
                    if (last_fb) out_counts[p] = (failed || *(volatile int *)&part_err[p]) ? -1ll : (long long)(e + written);
                }
            }
        }
        publish_range();
    }
}

// CURSOR mode: mark the partitions whose merge failed (out_counts = -1), after the merge kernel
__global__ void k_agg_finalize(const int *__restrict__ part_err, long long *__restrict__ out_counts, int32_t nparts) {
    for (int p = threadIdx.x; p < nparts; p += blockDim.x)
        if (part_err[p]) out_counts[p] = -1;
}
