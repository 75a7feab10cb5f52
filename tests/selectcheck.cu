// tests/selectcheck.cu -- runs the select and distinct-table arithmetic of dpark_b200/csrc/dpk_common.cuh (the
// __host__ __device__ functions dpk_select.cu's kernels call) on the CPU, round for round as the kernels take it: the
// histogram with per-bucket OR / AND over the candidates, sel_pick, the compaction by the match rule, then the stable
// take in row order and a stable sort of the taken rows by their words; and the distinct table filled row by row.
// Test-only.
#include <algorithm>
#include <vector>

#include "dpk_common.cuh"

extern "C" {
uint32_t slc_digit(uint64_t w, int32_t shift) { return dpk::sel_digit(w, shift); }
int32_t slc_bucket(const int64_t *hist, int64_t need, int64_t *below) { return dpk::sel_bucket(hist, need, below); }
int32_t slc_next_shift(uint64_t diff) { return dpk::sel_next_shift(diff); }

// the n smallest of m rows by (w0[, w1], id) (w1 NULL: one word) into out_ids[n], in that order; returns the number of
// radix rounds, or a negative number when they exceed 8 per word or a bucket count disagrees with the compaction
int32_t slc_select(const uint64_t *w0, const uint64_t *w1, int64_t m, int64_t n, int64_t *out_ids) {
    using namespace dpk;
    const int32_t nw = w1 ? 2 : 1;
    int64_t st[SEL_STATE] = {0};
    st[ST_SHIFT] = 64 - SEL_BITS;
    st[ST_NEED] = n;
    st[ST_COUNT] = m;
    std::vector<uint64_t> hist(3 * SEL_BUCKETS, 0);
    for (int b = 0; b < SEL_BUCKETS; b++) hist[2 * SEL_BUCKETS + b] = ~0ull;
    std::vector<int64_t> cands(m);
    for (int64_t i = 0; i < m; i++) cands[i] = i;
    int32_t rounds = 0;
    if (n < m) {
        for (;;) {
            const uint64_t *w = st[ST_WORD] ? w1 : w0;
            for (int64_t c : cands) {
                const uint32_t d = sel_digit(w[c], (int32_t)st[ST_SHIFT]);
                hist[d]++;
                hist[SEL_BUCKETS + d] |= w[c];
                hist[2 * SEL_BUCKETS + d] &= w[c];
            }
            sel_pick(st, hist.data(), nw);
            if (++rounds > 8 * nw) return -1;
            if (st[ST_DONE]) break;
            const uint64_t *mw = st[ST_MWORD] ? w1 : w0;
            std::vector<int64_t> next;
            for (int64_t c : cands)
                if ((mw[c] & (uint64_t)st[ST_MMASK]) == (uint64_t)st[ST_MVAL]) next.push_back(c);
            if ((int64_t)next.size() != st[ST_COUNT]) return -2;
            cands.swap(next);
        }
    }
    std::vector<int64_t> taken;
    if (n >= m) {
        for (int64_t i = 0; i < m; i++) taken.push_back(i);
    } else {
        const int64_t take_eq = n - st[ST_BELOW];
        int64_t eq = 0;
        for (int64_t i = 0; i < m; i++) {
            const int c = sel_cmp(w0[i], w1 ? w1[i] : 0, (uint64_t)st[ST_T0], (uint64_t)st[ST_T1], nw);
            if (c < 0 || (c == 0 && eq++ < take_eq)) taken.push_back(i);
        }
        if ((int64_t)taken.size() != n) return -3;
    }
    std::stable_sort(taken.begin(), taken.end(), [&](int64_t a, int64_t b) {
        return sel_cmp(w0[a], w1 ? w1[a] : 0, w0[b], w1 ? w1[b] : 0, nw) < 0;
    });
    for (size_t j = 0; j < taken.size(); j++) out_ids[j] = taken[j];
    return rounds;
}

// the distinct pairs of n rows: out_first[d] / out_count[d] in slot order; returns d, or -1 for a NaN
int64_t slc_uniq(const void *keys, int32_t kkind, const void *vals, int32_t vkind, int64_t n, int64_t *out_first,
                 int64_t *out_count) {
    using namespace dpk;
    const uint64_t S = bcast_slots(n);
    std::vector<UniqSlot> table(S, UniqSlot{UNIQ_EMPTY, 0});
    for (int64_t i = 0; i < n; i++) {
        uint64_t kb, vb;
        if (!uniq_pair_bits(keys, kkind, vals, vkind, i, &kb, &vb)) return -1;
        uniq_insert_row(table.data(), S - 1, keys, kkind, vals, vkind, (int32_t)i, kb, vb);
    }
    int64_t d = 0;
    for (uint64_t s = 0; s < S; s++) {
        if (table[s].owner == UNIQ_EMPTY) continue;
        out_first[d] = table[s].owner;
        out_count[d] = table[s].count;
        d++;
    }
    return d;
}
}
