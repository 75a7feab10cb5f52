// dpk_peer.cu -- the exchange step of the shuffle as a PUSH over NVLink peer memory.
//
// The reference's reducers pull every map's bucket over files + HTTP (ShuffleFetcher,
// dpark/shuffle.py:309-420).  After the map-side multisplit the rows bound for one peer GPU
// are one contiguous block of the bucket-major buffer (buckets owned by a peer are adjacent),
// so the exchange is G block copies per column.  k_copy_segments moves all of them in ONE
// launch: a segment table (source address, destination address, bytes) built on the device
// from the gathered bucket counts -- no host sync -- and a grid of 4 CTAs per SM that walks
// 32 KB work items ROUND-ROBIN over the segments, so every peer link carries traffic at the
// same time (a segment-after-segment order would aim all GPUs at the same peer).
// Destinations are plain device addresses: this GPU's memory or a peer's receive buffer mapped
// into this address space (torch symmetric memory = cuMem allocations exchanged on one node).
//
// Algorithmic bytes: (K+V) per row read locally + (K+V) per row stored through NVLink; the
// bound is the NVLink egress/ingress of one GPU (H100 SXM data sheet: 450 GB/s per direction), not HBM.
#include <cstring>
#include "dpk_common.cuh"

namespace dpk {

constexpr int CP_THREADS = 256;
constexpr int CP_WIDE_THREADS = 1024;
constexpr int CP_WIDE_SMEM = 160 * 1024;   // claimed, unused: one wide copy CTA owns its SM
// dpk_set_option("copy_sms"): 0 (default) = dpk_copy_segments fills the GPU (4 CTAs of 256 threads per SM); n > 0 = n
// CTAs of 1024 threads that each claim a whole SM (by their shared-memory request), so that a copy launched first on a
// high-priority stream leaves the other SMs to the kernel it overlaps with.  A push over NVLink is bound by the links
// (450 GB/s per direction per GPU on the H100 data sheet), which a few SMs' load/store bandwidth covers.
int g_copy_sms = 0;
constexpr int CP_MAX_SEG = 1024;
constexpr int64_t CP_ITEM = 32768;  // bytes per work item

template <typename T, int NT>
__device__ __forceinline__ void copy_item(const unsigned char *__restrict__ s, unsigned char *__restrict__ d,
                                          int64_t bytes) {
    const T *sp = reinterpret_cast<const T *>(s);
    T *dp = reinterpret_cast<T *>(d);
    const int n = (int)(bytes / (int64_t)sizeof(T));
    int i = threadIdx.x;
    for (; i + 3 * NT < n; i += 4 * NT) {  // 4 independent loads in flight per thread
        const T a = sp[i], b = sp[i + NT], c = sp[i + 2 * NT], e = sp[i + 3 * NT];
        dp[i] = a;
        dp[i + NT] = b;
        dp[i + 2 * NT] = c;
        dp[i + 3 * NT] = e;
    }
    for (; i < n; i += NT) dp[i] = sp[i];
}

template <int NT, int64_t ITEM>
__global__ void __launch_bounds__(NT)
k_copy_segments(const uint64_t *__restrict__ src_ptrs, const uint64_t *__restrict__ dst_ptrs,
                const int64_t *__restrict__ nbytes, int32_t nseg) {
    constexpr int CP_THREADS = NT;
    constexpr int64_t CP_ITEM = ITEM;
    __shared__ long long s_max;
    if (threadIdx.x == 0) s_max = 0;
    __syncthreads();
    long long mine = 0;
    for (int s = threadIdx.x; s < nseg; s += CP_THREADS) mine = max(mine, (long long)nbytes[s]);
    if (mine > 0) atomicMax(&s_max, mine);
    __syncthreads();
    const int64_t items_per_seg = ((int64_t)s_max + CP_ITEM - 1) / CP_ITEM;
    const int64_t total = items_per_seg * nseg;
    for (int64_t w = blockIdx.x; w < total; w += gridDim.x) {
        const int seg = (int)(w % nseg);
        const int64_t off = (w / nseg) * CP_ITEM;
        const int64_t len = nbytes[seg];
        if (off >= len) continue;
        const int64_t bytes = min(CP_ITEM, len - off);
        const uint64_t sa = src_ptrs[seg] + (uint64_t)off, da = dst_ptrs[seg] + (uint64_t)off;
        const unsigned align = (unsigned)((sa | da | (uint64_t)bytes) & 15u);
        const unsigned char *s = reinterpret_cast<const unsigned char *>(sa);
        unsigned char *d = reinterpret_cast<unsigned char *>(da);
        if (align == 0) copy_item<uint4, NT>(s, d, bytes);
        else if ((align & 7u) == 0) copy_item<uint2, NT>(s, d, bytes);
        else if ((align & 3u) == 0) copy_item<uint32_t, NT>(s, d, bytes);
        else copy_item<unsigned char, NT>(s, d, bytes);
    }
}

// ---- the same copy driven by the TMA --------------------------------------------------------------------------------
// A push that overlaps the multisplit of the next group or the merge of the previous part should take as few SMs as
// possible.  Moving the bytes with loads and stores needs tens of whole SMs to fill the links (how many has not been
// measured on H100s); here ONE thread per CTA streams 32 KB chunks through a
// shared-memory ring with bulk async copies (`cp.async.bulk` global -> shared completing on an mbarrier, then shared ->
// global, i.e. into the peer's buffer): 160 KB in flight per SM without occupying its issue slots or registers.
// Bulk copies need 16-byte aligned addresses and sizes: a segment whose source and destination are congruent mod 16
// is split into [head < 16 B][aligned middle][tail < 16 B] (head and tail by plain byte copies); any other segment takes
// the load/store path (dpk_pipe_plan lays the send buffer out so that every push is congruent).
constexpr int TC_THREADS = 128;
constexpr int TC_STAGES = 6;
constexpr int TC_CHUNK = 32768;
constexpr int TC_SMEM = TC_STAGES * TC_CHUNK;     // 192 KB: also makes the CTA the only one on its SM
int g_copy_tma = 1;   // dpk_set_option("copy_tma"): limited-SM copies (copy_sms > 0) use the TMA ring (1) or loads/stores (0)

__global__ void __launch_bounds__(TC_THREADS)
k_copy_segments_tma(const uint64_t *__restrict__ src_ptrs, const uint64_t *__restrict__ dst_ptrs,
                    const int64_t *__restrict__ nbytes, int32_t nseg) {
    extern __shared__ __align__(128) unsigned char tc_ring[];
    __shared__ __align__(8) unsigned long long tc_bar[TC_STAGES];
    __shared__ long long s_max;
    const uint32_t ring = (uint32_t)__cvta_generic_to_shared(tc_ring);
    const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(&tc_bar[0]);
    if (threadIdx.x == 0) {
        s_max = 0;
        for (int i = 0; i < TC_STAGES; i++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar0 + 8 * i));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    long long mine = 0;
    for (int s = threadIdx.x; s < nseg; s += TC_THREADS) mine = max(mine, (long long)nbytes[s]);
    if (mine > 0) atomicMax(&s_max, mine);
    __syncthreads();
    const int64_t items_per_seg = ((int64_t)s_max + TC_CHUNK - 1) / TC_CHUNK;
    const int64_t total = items_per_seg * nseg;
    // (1) heads and tails of the congruent segments, and whole incongruent segments, by plain accesses
    for (int seg = blockIdx.x * TC_THREADS + threadIdx.x; seg < nseg; seg += gridDim.x * TC_THREADS) {
        const int64_t len = nbytes[seg];
        const uint64_t sa = src_ptrs[seg], da = dst_ptrs[seg];
        if (len <= 0 || ((sa ^ da) & 15u)) continue;
        int64_t head = (int64_t)((16u - (unsigned)(sa & 15u)) & 15u);
        if (head > len) head = len;
        const int64_t mid = ((len - head) >> 4) << 4;
        const unsigned char *sp = reinterpret_cast<const unsigned char *>(sa);
        unsigned char *dp = reinterpret_cast<unsigned char *>(da);
        for (int64_t i = 0; i < head; i++) dp[i] = sp[i];
        for (int64_t i = head + mid; i < len; i++) dp[i] = sp[i];
    }
    for (int64_t w = blockIdx.x; w < total; w += gridDim.x) {
        const int seg = (int)(w % nseg);
        const int64_t off = (w / nseg) * TC_CHUNK;
        const int64_t len = nbytes[seg];
        const uint64_t sa = src_ptrs[seg], da = dst_ptrs[seg];
        if (off >= len || ((sa ^ da) & 15u) == 0) continue;
        const int64_t bytes = min((int64_t)TC_CHUNK, len - off);
        const unsigned align = (unsigned)(((sa + off) | (da + off) | (uint64_t)bytes) & 15u);
        const unsigned char *sp = reinterpret_cast<const unsigned char *>(sa + off);
        unsigned char *dp = reinterpret_cast<unsigned char *>(da + off);
        if ((align & 7u) == 0) copy_item<uint2, TC_THREADS>(sp, dp, bytes);
        else if ((align & 3u) == 0) copy_item<uint32_t, TC_THREADS>(sp, dp, bytes);
        else copy_item<unsigned char, TC_THREADS>(sp, dp, bytes);
    }
    // (2) the aligned middles through the ring: one thread, TC_STAGES - 1 chunk loads in flight
    if (threadIdx.x != 0) return;
    struct Item { uint64_t sa, da; uint32_t bytes; };
    auto fetch = [&](int64_t &w, Item &it) -> bool {
        for (; w < total; w += gridDim.x) {
            const int seg = (int)(w % nseg);
            const int64_t off = (w / nseg) * TC_CHUNK;
            const int64_t len = nbytes[seg];
            if (len <= 0) continue;
            const uint64_t sa = src_ptrs[seg], da = dst_ptrs[seg];
            if ((sa ^ da) & 15u) continue;
            int64_t head = (int64_t)((16u - (unsigned)(sa & 15u)) & 15u);
            if (head > len) head = len;
            const int64_t mid = ((len - head) >> 4) << 4;
            if (off >= mid) continue;
            it.sa = sa + (uint64_t)(head + off);
            it.da = da + (uint64_t)(head + off);
            it.bytes = (uint32_t)min((int64_t)TC_CHUNK, mid - off);
            return true;
        }
        return false;
    };
    int64_t wl = blockIdx.x, wst = blockIdx.x;
    int nl = 0, nst = 0;
    Item it;
    auto issue_load = [&](const Item &x, int k) {
        const uint32_t b = bar0 + 8 * (k % TC_STAGES), dst = ring + (uint32_t)(k % TC_STAGES) * TC_CHUNK;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(x.bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(dst), "l"(x.sa), "r"(x.bytes), "r"(b) : "memory");
    };
    while (nl < TC_STAGES - 1 && fetch(wl, it)) {
        issue_load(it, nl++);
        wl += gridDim.x;
    }
    while (nst < nl) {
        fetch(wst, it);        // the descriptor of item nst again (same walk as the load cursor)
        wst += gridDim.x;
        const uint32_t b = bar0 + 8 * (nst % TC_STAGES), par = (uint32_t)((nst / TC_STAGES) & 1);
        unsigned done = 0;
        while (!done)
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                         : "=r"(done) : "r"(b), "r"(par) : "memory");
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                     ::"l"(it.da), "r"(ring + (uint32_t)(nst % TC_STAGES) * TC_CHUNK), "r"(it.bytes) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        nst++;
        // store k = nst - 1 was just issued; the next load is item k + TC_STAGES - 1, whose stage was last read by store
        // k - 1: at most the newest store group may still be reading
        Item nx;
        if (fetch(wl, nx)) {
            asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
            issue_load(nx, nl++);
            wl += gridDim.x;
        }
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// One launch instead of ~20 small tensor operations on the host side of every step: from the gathered counts matrix
// (the MapOutputTracker) to the segment table of this rank's pushes, the rows every rank will receive and the segment
// matrix of this rank's own partitions.  Single CTA; G <= 64 ranks, any F.
//   all_counts[S][F]   rows source s holds for fine bucket b (S = G sources, or G * H when a rank sends H groups)
//   my_src             this rank's source row (rank, or rank * H + group)
//   per_blk            fine buckets per destination block (ceil(P / G) << sub_bits); destination d owns
//                      [d * per_blk, min(F, (d + 1) * per_blk))
//   blk_lo, blk_hi     the part of every destination's block this push covers, [blk_lo, blk_hi) relative to the block's
//                      first bucket (0, per_blk = the whole block; a pipelined shuffle pushes a block in parts so that the
//                      reduce side can start on the first part while the second is still crossing NVLink)
//   dst_row0           first row of this part's region in every receive buffer; `capacity` = rows of the region
//   src0/src1, dst_base[c][G], elem0/elem1   column c (keys, values): address of my bucket-major buffer, of every
//                      rank's receive buffer, element size
// Outputs: src_ptrs / dst_ptrs / nbytes [ncols][G] (clamped so that nothing is written past `capacity` rows of the
// region), need_over = max(need_over, max_d rows d receives - capacity), seg_out[S][blk_hi - blk_lo clipped to F]
// (the segment matrix of my own part: the rows that land in my region, so that a reduce over an overflowed step never
// reads or sizes anything past `capacity` rows; that step's result is invalid and need_over says so).
__global__ void __launch_bounds__(256)
k_push_plan(const int64_t *__restrict__ all_counts, int32_t S, int32_t G, int32_t F, int32_t per_blk, int32_t blk_lo,
            int32_t blk_hi, int64_t dst_row0, int32_t my_src, int32_t my_rank, int32_t ncols, uint64_t src0, uint64_t src1,
            const uint64_t *__restrict__ dst_base, int32_t elem0, int32_t elem1, int64_t capacity,
            uint64_t *__restrict__ src_ptrs, uint64_t *__restrict__ dst_ptrs, int64_t *__restrict__ nbytes,
            long long *__restrict__ need_over, int64_t *__restrict__ seg_out) {
    extern __shared__ long long s_pp[];
    long long *s_R = s_pp;              // [S][G] rows source s sends to destination d in this part
    long long *s_T = s_pp + S * G;      // [G] rows of destination d's WHOLE block in my buffer
    long long *s_P = s_T + G;           // [G] rows of d's block in my buffer that lie before blk_lo
    for (int i = threadIdx.x; i < S * G; i += blockDim.x) {
        const int s = i / G, d = i % G;
        const int b0 = min(F, d * per_blk + blk_lo), b1 = min(F, min((d + 1) * per_blk, d * per_blk + blk_hi));
        long long r = 0;
        for (int b = b0; b < b1; b++) r += all_counts[(int64_t)s * F + b];
        s_R[i] = r;
    }
    for (int i = threadIdx.x; i < 2 * G; i += blockDim.x) {
        const int d = i % G;
        const int b0 = min(F, d * per_blk), b1 = i < G ? min(F, (d + 1) * per_blk) : min(F, d * per_blk + blk_lo);
        long long r = 0;
        for (int b = b0; b < b1; b++) r += all_counts[(int64_t)my_src * F + b];
        (i < G ? s_T : s_P)[d] = r;
    }
    __syncthreads();
    if (threadIdx.x < G) {
        const int d = threadIdx.x;
        long long send_first = s_P[d], dst_first = 0, total = 0;
        for (int dd = 0; dd < d; dd++) send_first += s_T[dd];
        for (int s = 0; s < S; s++) {
            if (s < my_src) dst_first += s_R[s * G + d];
            total += s_R[s * G + d];
        }
        long long rows = s_R[my_src * G + d];
        const long long room = capacity - dst_first;
        if (rows > room) rows = room > 0 ? room : 0;
        for (int c = 0; c < ncols; c++) {
            const long long e = c ? elem1 : elem0;
            src_ptrs[c * G + d] = (c ? src1 : src0) + (uint64_t)(send_first * e);
            dst_ptrs[c * G + d] = dst_base[c * G + d] + (uint64_t)((dst_row0 + dst_first) * e);
            nbytes[c * G + d] = rows * e;
        }
        if (total > capacity) atomicMax(need_over, total - capacity);
    }
    if (seg_out) {   // the rows that LAND here: source s's push is clamped at `capacity` rows of the region
        const int b0 = min(F, my_rank * per_blk + blk_lo), b1 = min(F, min((my_rank + 1) * per_blk, my_rank * per_blk + blk_hi));
        const int fo = b1 - b0;
        for (int s = threadIdx.x; s < S; s += blockDim.x) {
            long long at = 0;                                  // row of source s's first row in my region
            for (int t = 0; t < s; t++) at += s_R[t * G + my_rank];
            for (int j = 0; j < fo; j++) {
                const long long c = all_counts[(int64_t)s * F + b0 + j];
                seg_out[(int64_t)s * fo + j] = max(0LL, min(c, capacity - at));
                at += c;
            }
        }
    }
}

// The plan of a PIPELINED shuffle step (dpark_b200.peer.shuffle_pipelined), one launch per group of map splits: where the
// multisplit puts every bucket of this group in the send buffer, and the segment tables of the Q pushes (part q of every
// destination's block -> region q of that destination's receive buffer).  The send buffer is bucket-major with up to
// `align_rows - 1` pad rows in front of every (destination, part) block, chosen so that the block starts at a row
// congruent (mod align_rows = 16 bytes / smallest element) to the row it lands on in the receive region: source and
// destination of every push are then congruent mod 16 bytes and the whole block moves through the TMA
// (k_copy_segments_tma).  The send buffer needs rows(my_src) + G * Q * (align_rows - 1) rows.
//   all_counts[S][F], per_blk, my_src, my_rank: as in k_push_plan;  part_blk = buckets per part (per_blk / Q);
//   region = rows of one part's region in a receive buffer (part q starts at row q * region)
// Outputs: bucket_base[F] (row of bucket b's first row in the send buffer), src_ptrs / dst_ptrs / nbytes [Q][ncols][G],
// need_over, seg_out[Q][S][part_blk] (own part columns, the rows that land in region q; clipped columns hold 0) if not
// NULL.  Single CTA.
__global__ void __launch_bounds__(256)
k_pipe_plan(const int64_t *__restrict__ all_counts, int32_t S, int32_t G, int32_t F, int32_t per_blk, int32_t Q,
            int32_t part_blk, int64_t region, int32_t align_rows, int32_t my_src, int32_t my_rank, int32_t ncols,
            uint64_t src0, uint64_t src1, const uint64_t *__restrict__ dst_base, int32_t elem0, int32_t elem1,
            int64_t *__restrict__ bucket_base, uint64_t *__restrict__ src_ptrs, uint64_t *__restrict__ dst_ptrs,
            int64_t *__restrict__ nbytes, long long *__restrict__ need_over, int64_t *__restrict__ seg_out) {
    extern __shared__ long long s_pl[];
    long long *s_R = s_pl;                         // [Q][S][G] rows source s sends to destination d in part q
    long long *s_first = s_R + (int64_t)Q * S * G;  // [G][Q] first row of block (d, q) in my send buffer
    long long *s_mine = s_first + G * Q;           // [F] my rows per bucket
    for (int i = threadIdx.x; i < Q * S * G; i += blockDim.x) {
        const int q = i / (S * G), s = (i / G) % S, d = i % G;
        const int b0 = min(F, d * per_blk + q * part_blk), b1 = min(F, min((d + 1) * per_blk, d * per_blk + (q + 1) * part_blk));
        long long r = 0;
        for (int b = b0; b < b1; b++) r += all_counts[(int64_t)s * F + b];
        s_R[i] = r;
    }
    for (int b = threadIdx.x; b < F; b += blockDim.x) s_mine[b] = all_counts[(int64_t)my_src * F + b];
    __syncthreads();
    if (threadIdx.x == 0) {   // G * Q <= 512 blocks, laid out in (destination, part) order with congruence pads
        long long pos = 0;
        for (int d = 0; d < G; d++)
            for (int q = 0; q < Q; q++) {
                long long dst_first = 0, total = 0;
                for (int s = 0; s < S; s++) {
                    const long long r = s_R[((int64_t)q * S + s) * G + d];
                    if (s < my_src) dst_first += r;
                    total += r;
                }
                long long rows = s_R[((int64_t)q * S + my_src) * G + d];
                const long long landing = (long long)q * region + dst_first;
                pos += ((landing - pos) % align_rows + align_rows) % align_rows;
                s_first[d * Q + q] = pos;
                const long long room = region - dst_first;
                long long push = rows;
                if (push > room) push = room > 0 ? room : 0;
                for (int c = 0; c < ncols; c++) {
                    const long long e = c ? elem1 : elem0;
                    const int o = (q * ncols + c) * G + d;
                    src_ptrs[o] = (c ? src1 : src0) + (uint64_t)(pos * e);
                    dst_ptrs[o] = dst_base[c * G + d] + (uint64_t)(landing * e);
                    nbytes[o] = push * e;
                }
                if (total > region) atomicMax(need_over, total - region);
                pos += rows;
            }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < G * Q; i += blockDim.x) {   // bucket bases inside every block
        const int d = i / Q, q = i % Q;
        const int b0 = min(F, d * per_blk + q * part_blk), b1 = min(F, min((d + 1) * per_blk, d * per_blk + (q + 1) * part_blk));
        long long run = s_first[i];
        for (int b = b0; b < b1; b++) {
            bucket_base[b] = run;
            run += s_mine[b];
        }
    }
    if (seg_out) {   // the rows that LAND here: every push into region q is clamped at `region` rows
        for (int i = threadIdx.x; i < Q * S; i += blockDim.x) {
            const int q = i / S, s = i % S;
            long long at = 0;                                  // row of source s's first row in region q
            for (int t = 0; t < s; t++) at += s_R[((int64_t)q * S + t) * G + my_rank];
            for (int j = 0; j < part_blk; j++) {
                const int b = my_rank * per_blk + q * part_blk + j;
                const long long c = (b < F && b < (my_rank + 1) * per_blk) ? all_counts[(int64_t)s * F + b] : 0;
                seg_out[(int64_t)i * part_blk + j] = max(0LL, min(c, region - at));
                at += c;
            }
        }
    }
}

// The plan of the FUSED scatter + exchange (dpk_partition_scatter_ptrs): for every fine bucket b of this rank's map
// output the address its rows go to -- the slot of (source = this rank, bucket b) in the OWNER's receive buffer, layout
// source-rank-major then bucket-major exactly as the push form delivers it -- plus this rank's segment matrix and the
// capacity flag.  A bucket that would end past `capacity` rows of its receive buffer is pointed at a local dump buffer
// instead (dump0/dump1: >= this rank's row count; position = the bucket's local bucket-major offset), so a too-small
// buffer can never be overrun; need_over reports it, and the segment matrix counts such a bucket as 0 rows (it
// describes what landed).  Single CTA; G <= 64 ranks, F <= 4096 buckets.
__global__ void __launch_bounds__(256)
k_fused_plan(const int64_t *__restrict__ all_counts, int32_t G, int32_t F, int32_t per_blk, int32_t my_rank, int32_t ncols,
             const uint64_t *__restrict__ dst_base, int32_t elem0, int32_t elem1, int64_t capacity, uint64_t dump0,
             uint64_t dump1, uint64_t *__restrict__ key_ptrs, uint64_t *__restrict__ val_ptrs,
             long long *__restrict__ need_over, int64_t *__restrict__ seg_out) {
    extern __shared__ long long s_fp[];
    long long *s_R = s_fp;             // [G][G] rows source s sends to destination d
    long long *s_mine = s_fp + G * G;  // [F] my rows per bucket
    for (int i = threadIdx.x; i < G * G; i += blockDim.x) {
        const int s = i / G, d = i % G;
        const int b0 = min(F, d * per_blk), b1 = min(F, (d + 1) * per_blk);
        long long r = 0;
        for (int b = b0; b < b1; b++) r += all_counts[(int64_t)s * F + b];
        s_R[i] = r;
    }
    for (int b = threadIdx.x; b < F; b += blockDim.x) s_mine[b] = all_counts[(int64_t)my_rank * F + b];
    __syncthreads();
    if (threadIdx.x < G) {
        const int d = threadIdx.x;
        long long dst_first = 0, total = 0, local_first = 0;
        for (int dd = 0; dd < d; dd++) local_first += s_R[my_rank * G + dd];
        for (int s = 0; s < G; s++) {
            if (s < my_rank) dst_first += s_R[s * G + d];
            total += s_R[s * G + d];
        }
        const int b0 = min(F, d * per_blk), b1 = min(F, (d + 1) * per_blk);
        long long run = 0;
        for (int b = b0; b < b1; b++) {
            const long long c = s_mine[b];
            const bool fits = dst_first + run + c <= capacity;
            key_ptrs[b] = fits ? dst_base[d] + (uint64_t)((dst_first + run) * elem0) : dump0 + (uint64_t)((local_first + run) * elem0);
            if (ncols > 1)
                val_ptrs[b] = fits ? dst_base[G + d] + (uint64_t)((dst_first + run) * elem1)
                                   : dump1 + (uint64_t)((local_first + run) * elem1);
            run += c;
        }
        if (total > capacity) atomicMax(need_over, total - capacity);
    }
    if (seg_out) {   // the rows that LAND here: a bucket diverted to its source's dump counts 0
        const int b0 = min(F, my_rank * per_blk), b1 = min(F, (my_rank + 1) * per_blk), fo = b1 - b0;
        for (int s = threadIdx.x; s < G; s += blockDim.x) {
            long long at = 0;                                  // row of source s's first row in my buffer
            for (int t = 0; t < s; t++) at += s_R[t * G + my_rank];
            for (int j = 0; j < fo; j++) {
                const long long c = all_counts[(int64_t)s * F + b0 + j];
                seg_out[(int64_t)s * fo + j] = at + c <= capacity ? c : 0;
                at += c;
            }
        }
    }
}

}  // namespace dpk

using namespace dpk;

extern "C" int dpk_fused_plan(const int64_t *all_counts, int32_t nranks, int32_t nbuckets, int32_t per_block, int32_t my_rank,
                              int32_t ncols, const uint64_t *dst_base, int32_t key_bytes, int32_t val_bytes, int64_t capacity,
                              uint64_t dump_keys, uint64_t dump_vals, uint64_t *key_ptrs, uint64_t *val_ptrs,
                              int64_t *need_over, int64_t *seg_out, dpk_stream_t stream) {
    if (nranks < 1 || nranks > 64 || nbuckets < 1 || nbuckets > 4096 || ncols < 1 || ncols > 2 || per_block < 0 ||
        my_rank < 0 || my_rank >= nranks)
        return fail(DPK_ERR_INVALID, "bad fused plan shape: %d ranks, %d buckets, %d columns", nranks, nbuckets, ncols);
    if (!all_counts || !dst_base || !key_ptrs || (ncols > 1 && !val_ptrs) || !need_over || !dump_keys || (ncols > 1 && !dump_vals))
        return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t sh = ((size_t)nranks * nranks + nbuckets) * sizeof(long long);
    DPK_CUDA_TRY(cudaFuncSetAttribute(k_fused_plan, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh));
    DPK_LAUNCH("fused_plan", st, k_fused_plan<<<1, 256, sh, st>>>(all_counts, nranks, nbuckets, per_block, my_rank, ncols, dst_base,
                                                               key_bytes, val_bytes, capacity, dump_keys, dump_vals, key_ptrs,
                                                               val_ptrs, (long long *)need_over, seg_out));
    return DPK_OK;
}

extern "C" int dpk_push_plan_part(const int64_t *all_counts, int32_t nsrc, int32_t nranks, int32_t nbuckets, int32_t per_block,
                                  int32_t blk_lo, int32_t blk_hi, int64_t dst_row0, int32_t my_src, int32_t my_rank, int32_t ncols,
                                  uint64_t src_keys, uint64_t src_vals, const uint64_t *dst_base, int32_t key_bytes,
                                  int32_t val_bytes, int64_t capacity, uint64_t *src_ptrs, uint64_t *dst_ptrs, int64_t *nbytes,
                                  int64_t *need_over, int64_t *seg_out, dpk_stream_t stream) {
    if (nranks < 1 || nranks > 64 || nsrc < nranks || nsrc > 4096 || ncols < 1 || ncols > 2 || per_block < 0)
        return fail(DPK_ERR_INVALID, "bad push plan shape: %d sources, %d ranks, %d columns", nsrc, nranks, ncols);
    if (blk_lo < 0 || blk_hi < blk_lo || blk_hi > per_block || dst_row0 < 0)
        return fail(DPK_ERR_INVALID, "bad push plan part [%d, %d) of %d buckets, region row %lld", blk_lo, blk_hi, per_block,
                    (long long)dst_row0);
    if (!all_counts || !dst_base || !src_ptrs || !dst_ptrs || !nbytes || !need_over)
        return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t sh = ((size_t)nsrc * nranks + 2 * (size_t)nranks) * sizeof(long long);
    if (sh > 48 * 1024) return fail(DPK_ERR_UNSUPPORTED, "push plan: %d x %d sources x ranks exceed shared memory", nsrc, nranks);
    DPK_LAUNCH("push_plan", st, k_push_plan<<<1, 256, sh, st>>>(all_counts, nsrc, nranks, nbuckets, per_block, blk_lo, blk_hi, dst_row0,
                                                             my_src, my_rank, ncols, src_keys, src_vals, dst_base, key_bytes, val_bytes,
                                                             capacity, src_ptrs, dst_ptrs, nbytes, (long long *)need_over, seg_out));
    return DPK_OK;
}

extern "C" int dpk_push_plan(const int64_t *all_counts, int32_t nsrc, int32_t nranks, int32_t nbuckets, int32_t per_block,
                             int32_t my_src, int32_t my_rank, int32_t ncols, uint64_t src_keys, uint64_t src_vals,
                             const uint64_t *dst_base, int32_t key_bytes, int32_t val_bytes, int64_t capacity, uint64_t *src_ptrs,
                             uint64_t *dst_ptrs, int64_t *nbytes, int64_t *need_over, int64_t *seg_out,
                             dpk_stream_t stream) {
    return dpk_push_plan_part(all_counts, nsrc, nranks, nbuckets, per_block, 0, per_block, 0, my_src, my_rank, ncols, src_keys,
                              src_vals, dst_base, key_bytes, val_bytes, capacity, src_ptrs, dst_ptrs, nbytes, need_over, seg_out,
                              stream);
}

extern "C" int dpk_pipe_plan(const int64_t *all_counts, int32_t nsrc, int32_t nranks, int32_t nbuckets, int32_t per_block,
                             int32_t nparts, int64_t region_rows, int32_t my_src, int32_t my_rank, int32_t ncols,
                             uint64_t src_keys, uint64_t src_vals, const uint64_t *dst_base, int32_t key_bytes,
                             int32_t val_bytes, int64_t *bucket_base, uint64_t *src_ptrs, uint64_t *dst_ptrs, int64_t *nbytes,
                             int64_t *need_over, int64_t *seg_out, dpk_stream_t stream) {
    if (nranks < 1 || nranks > 64 || nsrc < nranks || nsrc > 4096 || ncols < 1 || ncols > 2 || per_block < 1 ||
        nbuckets < 1 || nbuckets > 4096 || nparts < 1 || nparts > 8 || per_block % nparts || region_rows < 0)
        return fail(DPK_ERR_INVALID, "bad pipe plan shape: %d sources, %d ranks, %d buckets, %d per block in %d parts", nsrc, nranks,
                    nbuckets, per_block, nparts);
    if (!all_counts || !dst_base || !bucket_base || !src_ptrs || !dst_ptrs || !nbytes || !need_over)
        return fail(DPK_ERR_INVALID, "NULL pointer");
    if ((key_bytes != 4 && key_bytes != 8) || (ncols > 1 && val_bytes != 4 && val_bytes != 8))
        return fail(DPK_ERR_UNSUPPORTED, "element sizes %d / %d", key_bytes, val_bytes);
    const int min_elem = ncols > 1 && val_bytes < key_bytes ? val_bytes : key_bytes;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t sh = ((size_t)nparts * nsrc * nranks + (size_t)nranks * nparts + nbuckets) * sizeof(long long);
    if (sh > 200 * 1024) return fail(DPK_ERR_UNSUPPORTED, "pipe plan: %d parts x %d sources x %d ranks exceed shared memory", nparts, nsrc, nranks);
    DPK_CUDA_TRY(cudaFuncSetAttribute(k_pipe_plan, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh));
    DPK_LAUNCH("pipe_plan", st, k_pipe_plan<<<1, 256, sh, st>>>(all_counts, nsrc, nranks, nbuckets, per_block, nparts, per_block / nparts,
                                                             region_rows, 16 / min_elem, my_src, my_rank, ncols, src_keys, src_vals,
                                                             dst_base, key_bytes, val_bytes, bucket_base, src_ptrs, dst_ptrs, nbytes,
                                                             (long long *)need_over, seg_out));
    return DPK_OK;
}

// The same block pushes handed to the GPU's COPY ENGINES: one cudaMemcpyBatchAsync for a whole segment table that the HOST
// holds (sizes read back from dpk_pipe_plan's tables while the multisplit runs).  The engines move the blocks over NVLink
// without occupying a single SM, so a push issued this way overlaps the multisplit of the next group and the merge of the
// previous part at their full speed; the batch call costs one driver round trip instead of one per block.
extern "C" int dpk_memcpy_batch(const uint64_t *h_dst_ptrs, const uint64_t *h_src_ptrs, const int64_t *h_nbytes, int32_t count,
                                dpk_stream_t stream) {
    if (count < 0 || count > 1024) return fail(DPK_ERR_INVALID, "count=%d out of range [0, 1024]", count);
    if (count == 0) return DPK_OK;
    if (!h_dst_ptrs || !h_src_ptrs || !h_nbytes) return fail(DPK_ERR_INVALID, "NULL pointer");
    void *dsts[1024], *srcs[1024];     // 24 KB of stack: a step pushes 2 columns x (ranks <= 64) blocks per call
    size_t sizes[1024];
    size_t m = 0;
    for (int i = 0; i < count; i++) {
        if (h_nbytes[i] < 0) return fail(DPK_ERR_INVALID, "negative size in segment %d", i);
        if (h_nbytes[i] == 0) continue;
        dsts[m] = reinterpret_cast<void *>(h_dst_ptrs[i]);
        srcs[m] = reinterpret_cast<void *>(h_src_ptrs[i]);
        sizes[m] = (size_t)h_nbytes[i];
        m++;
    }
    if (m == 0) return DPK_OK;
    cudaMemcpyAttributes attr;
    memset(&attr, 0, sizeof(attr));
    attr.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
    size_t attr_idx = 0, fail_idx = 0;
    cudaError_t e = cudaMemcpyBatchAsync(dsts, srcs, sizes, m, &attr, &attr_idx, 1, &fail_idx, (cudaStream_t)stream);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        // a driver without the batch entry point (or the legacy stream): one call per block
        for (size_t i = 0; i < m; i++)
            DPK_CUDA_TRY(cudaMemcpyAsync(dsts[i], srcs[i], sizes[i], cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    }
    return DPK_OK;
}

extern "C" int dpk_copy_segments(const uint64_t *src_ptrs, const uint64_t *dst_ptrs, const int64_t *nbytes,
                                 int32_t nseg, dpk_stream_t stream) {
    if (nseg < 0 || nseg > CP_MAX_SEG)
        return fail(DPK_ERR_INVALID, "nseg=%d out of range [0, %d]", nseg, CP_MAX_SEG);
    if (nseg == 0) return DPK_OK;
    if (!src_ptrs || !dst_ptrs || !nbytes) return fail(DPK_ERR_INVALID, "segment table is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    if (g_copy_sms > 0 && g_copy_tma) {   // a few whole SMs, one TMA-issuing thread each
        DPK_CUDA_TRY(cudaFuncSetAttribute(k_copy_segments_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
        DPK_LAUNCH("copy_segments", st, k_copy_segments_tma<<<g_copy_sms, TC_THREADS, TC_SMEM, st>>>(src_ptrs, dst_ptrs, nbytes, nseg));
        return DPK_OK;
    }
    if (g_copy_sms > 0) {   // a few whole SMs (the rest stay free for the kernel this copy overlaps with)
        auto kern = k_copy_segments<CP_WIDE_THREADS, 4 * CP_ITEM>;
        DPK_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, CP_WIDE_SMEM));
        DPK_LAUNCH("copy_segments", st, kern<<<g_copy_sms, CP_WIDE_THREADS, CP_WIDE_SMEM, st>>>(src_ptrs, dst_ptrs, nbytes, nseg));
        return DPK_OK;
    }
    DPK_LAUNCH("copy_segments", st,
               (k_copy_segments<CP_THREADS, CP_ITEM><<<sm_count() * 4, CP_THREADS, 0, st>>>(src_ptrs, dst_ptrs, nbytes, nseg)));
    return DPK_OK;
}
