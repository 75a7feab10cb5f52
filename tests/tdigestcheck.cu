// tests/tdigestcheck.cu -- runs the t-digest arithmetic of dpark_b200/csrc/dpk_common.cuh (the __host__ __device__
// functions dpk_tdigest.cu's kernels call) on the CPU, step for step as the kernels take it: segments of at most
// TD_SHORT values in one serial fold, longer ones buffer by buffer (stable sort, merge with the centroids by the two
// counts, the weights' pass, the centroids' means), then per key the absorb chain and the quantiles.  Test-only.
#include <vector>

#include "dpk_common.cuh"

namespace {
constexpr int TD_SHORT = 32;     // dpk_tdigest.cu

// the staged fold of k_td_build_long / k_td_merge: xm / xw (n entries) -> cm / cw; false when a mean is NaN or falls
bool staged_fold(const double *xm, const double *xw, int n, double total, double *cm, double *cw, int *C, double *lo,
                 double *hi, bool first) {
    int16_t cs[dpk::TD_STAGE + 2];
    const int nc = dpk::td_fold_decide(xw, n, total, cs);
    bool ok = true;
    for (int c = 0; c < nc; c++) {
        dpk::td_centroid(xm, xw, cs[c], cs[c + 1], &cm[c], &cw[c]);
        ok &= dpk::td_mean_ok(cm[c], c ? &cm[c - 1] : nullptr);
    }
    *lo = first ? cm[0] : dpk::td_min(*lo, cm[0]);
    *hi = first ? cm[nc - 1] : dpk::td_max(*hi, cm[nc - 1]);
    *C = nc;
    return ok;
}
}  // namespace

extern "C" {
int32_t tdc_cap(void) { return dpk::TD_CAP; }
int32_t tdc_short(void) { return TD_SHORT; }
double tdc_value(const void *col, int32_t kind, int64_t i) { return dpk::td_value(col, kind, i); }

// dpk_tdigest_build on the CPU; returns the flag (1 = the composition stands)
int32_t tdc_build(const int64_t *ids, const void *vals, int32_t kind, const int64_t *ss, const int64_t *so, int64_t S,
                  double *gm, double *gw, int32_t *cnt, double *lohi) {
    int32_t flag = 0;
    std::vector<double> bv(dpk::TD_CAP), cm(dpk::TD_STAGE), cw(dpk::TD_STAGE), xm(dpk::TD_STAGE), xw(dpk::TD_STAGE);
    for (int64_t s = 0; s < S; s++) {
        const int64_t r0 = ss[s], L = ss[s + 1] - r0;
        bool bad = false;
        if (L <= TD_SHORT) {
            double *om = gm + so[s], *ow = gw + so[s];
            for (int i = 0; i < L; i++) {
                om[i] = dpk::td_value(vals, kind, ids[r0 + i]);
                bad |= om[i] != om[i];
            }
            dpk::td_sort_serial(om, (int)L);
            const int c = dpk::td_fold_serial(om, nullptr, (int)L, (double)L, om, ow, &bad);
            cnt[s] = c;
            lohi[2 * s] = om[0];
            lohi[2 * s + 1] = om[c - 1];
        } else {
            int C = 0;
            double lo = 0.0, hi = 0.0, mw = 0.0;
            for (int64_t pos = 0; pos < L && !bad;) {
                const int B = dpk::td_buffer_len(C, L - pos);
                for (int t = 0; t < B; t++) {
                    bv[t] = dpk::td_value(vals, kind, ids[r0 + pos + t]);
                    bad |= bv[t] != bv[t];
                }
                if (bad) break;
                dpk::td_sort_serial(bv.data(), B);
                for (int t = 0; t < B; t++) {
                    const int p = t + dpk::td_count_below(cm.data(), C, bv[t]);
                    xm[p] = bv[t];
                    xw[p] = 1.0;
                }
                for (int c = 0; c < C; c++) {
                    const int p = c + dpk::td_count_upto(bv.data(), B, cm[c]);
                    xm[p] = cm[c];
                    xw[p] = cw[c];
                }
                mw = dpk::td_add(mw, (double)B);
                bad = !staged_fold(xm.data(), xw.data(), B + C, mw, cm.data(), cw.data(), &C, &lo, &hi, pos == 0);
                pos += B;
            }
            bad |= C > dpk::TD_CAP;
            for (int c = 0; c < C && !bad; c++) {
                gm[so[s] + c] = cm[c];
                gw[so[s] + c] = cw[c];
            }
            cnt[s] = bad ? 0 : C;
            lohi[2 * s] = lo;
            lohi[2 * s + 1] = hi;
        }
        if (bad) flag = 1;
    }
    return flag;
}

// dpk_tdigest_merge on the CPU; returns the flag
int32_t tdc_merge(const int64_t *gs, int64_t G, const int64_t *ss, const int64_t *so, int64_t S, const int32_t *cnt,
                  const double *lohi, const double *gm, const double *gw, const double *qs, int32_t nq, double *out) {
    std::vector<double> cm(dpk::TD_STAGE), cw(dpk::TD_STAGE), xm(dpk::TD_STAGE), xw(dpk::TD_STAGE);
    for (int64_t g = 0; g < G; g++) {
        const int64_t s0 = dpk::group_of(ss, 0, S + 1, gs[g]), s1 = dpk::group_of(ss, 0, S + 1, gs[g + 1]);
        int C = cnt[s0];
        for (int c = 0; c < C; c++) {
            cm[c] = gm[so[s0] + c];
            cw[c] = gw[so[s0] + c];
        }
        double mw = (double)(ss[s0 + 1] - ss[s0]), lo = lohi[2 * s0], hi = lohi[2 * s0 + 1];
        for (int64_t s = s0 + 1; s < s1; s++) {
            const int m = cnt[s];
            if (C + m > dpk::TD_STAGE) return 1;
            const double *im = gm + so[s], *iw = gw + so[s];
            for (int t = 0; t < m; t++) {
                const int p = t + dpk::td_count_below(cm.data(), C, im[t]);
                xm[p] = im[t];
                xw[p] = iw[t];
            }
            for (int c = 0; c < C; c++) {
                const int p = c + dpk::td_count_upto(im, m, cm[c]);
                xm[p] = cm[c];
                xw[p] = cw[c];
            }
            mw = dpk::td_add(mw, (double)(ss[s + 1] - ss[s]));
            if (!staged_fold(xm.data(), xw.data(), m + C, mw, cm.data(), cw.data(), &C, &lo, &hi, false)) return 1;
        }
        for (int j = 0; j < nq; j++) out[g * nq + j] = dpk::td_quantile(cm.data(), cw.data(), C, mw, lo, hi, qs[j]);
    }
    return 0;
}

// one fold of n entries in merged order (MergingDigest._fold with total = the merged weight after it), as one thread
// runs it; returns the centroid count, *bad as td_mean_ok
int32_t tdc_fold_serial(const double *xm, const double *xw, int32_t n, double total, double *om, double *ow,
                        int32_t *bad) {
    bool b = false;
    const int c = dpk::td_fold_serial(xm, xw, n, total, om, ow, &b);
    *bad = b ? 1 : 0;
    return c;
}
double tdc_quantile(const double *ms, const double *ws, int32_t c, double mw, double lo, double hi, double q) {
    return dpk::td_quantile(ms, ws, c, mw, lo, hi, q);
}
}
