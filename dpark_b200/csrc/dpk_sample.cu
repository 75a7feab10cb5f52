// dpk_sample.cu -- f8: the Bernoulli sample of SampleRDD (dpark/rdd.py:1379-1397) over row ranges: row j of split i is
// kept when the j-th random.Random(seed + i).random() is <= frac.  A split's draws are one sequential MT19937 chain
// (mt_*, dpk_common.cuh), so one CTA walks one split:
//
//   k_sample_bernoulli : per twist, the 624-word state in shared memory is rewritten in its three barrier-separated
//                        phases (each element's inputs read into registers before any thread writes); then thread
//                        t < 312 tempers words 2t and 2t + 1 into row base + t's draw, and a block scan (warp ballots,
//                        one word per warp) writes the kept row ids in row order at the split's own begin.
//
// Host reads: the S per-split counts.
#include "dpk_common.cuh"

namespace dpk {

constexpr int SMP_THREADS = 320;                 // >= MT_DRAWS and >= every phase's length
constexpr int SMP_WARPS = SMP_THREADS / 32;
static_assert(SMP_THREADS >= MT_DRAWS && SMP_THREADS >= MT_N - MT_M, "one element per thread");

__global__ void __launch_bounds__(SMP_THREADS)
k_sample_bernoulli(const uint32_t *__restrict__ states, const int64_t *__restrict__ ranges, double frac,
                   int64_t *__restrict__ out_ids, int64_t *__restrict__ counts) {
    __shared__ uint32_t mt[MT_N];
    __shared__ int wcnt[SMP_WARPS];
    const int64_t s = blockIdx.x;
    const int64_t begin = ranges[2 * s], end = ranges[2 * s + 1];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    for (int i = t; i < MT_N; i += SMP_THREADS) mt[i] = states[s * MT_N + i];
    __syncthreads();
    int64_t kept = 0;
    for (int64_t base = begin; base < end; base += MT_DRAWS) {
#pragma unroll
        for (int p = 0; p < 3; p++) {
            const int i = mt_phase(p) + t;
            const bool mine = i < mt_phase(p + 1);
            const uint32_t v = mine ? mt_twist_elem(mt, i) : 0u;
            __syncthreads();
            if (mine) mt[i] = v;
            __syncthreads();
        }
        bool keep = false;
        if (t < MT_DRAWS && base + t < end)
            keep = sample_keep(mt_double(mt_temper(mt[2 * t]), mt_temper(mt[2 * t + 1])), frac);
        const unsigned bal = __ballot_sync(0xFFFFFFFFu, keep);
        if (lane == 0) wcnt[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < SMP_WARPS; w++) {
            const int c = wcnt[w];
            before += w < warp ? c : 0;
            total += c;
        }
        if (keep) out_ids[begin + kept + before + __popc(bal & ((1u << lane) - 1u))] = base + t;
        kept += total;
        // wcnt is rewritten only after the next twist's barriers, which every thread reaches after reading it here
    }
    if (t == 0) counts[s] = kept;
}

}  // namespace dpk

using namespace dpk;

extern "C" {

int dpk_sample_bernoulli(const uint32_t *states, const int64_t *ranges, int64_t nsplits, double frac,
                         int64_t *out_ids, int64_t *out_counts, dpk_stream_t stream) {
    if (nsplits < 0 || nsplits > 0x7fffffffLL) return fail(DPK_ERR_INVALID, "nsplits=%lld", (long long)nsplits);
    if (nsplits == 0) return DPK_OK;
    if (!states || !ranges || !out_ids || !out_counts) return fail(DPK_ERR_INVALID, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    DPK_LAUNCH("sample_bernoulli", st, k_sample_bernoulli<<<(unsigned)nsplits, SMP_THREADS, 0, st>>>(
        states, ranges, frac, out_ids, out_counts));
    return DPK_OK;
}

}  // extern "C"
