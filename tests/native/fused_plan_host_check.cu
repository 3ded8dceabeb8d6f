// Host build of the fused block's stream planner (csrc/nfb_fused_plan.h) for tests/test_fused_plan_host.py: the masks
// in, the slice ownership, step table and record halves out.
#include "../../normalizing-flows_b200/csrc/nfb_fused_plan.h"

// m_init null: unmasked net; m_hid null: no hidden-to-hidden GEMM masks.  recs: 5 values per half (gemm, row0, nrows,
// kc, off_hi) and off_lo in recs_lo.  Returns the number of steps, or -1 when an output array is too small.
extern "C" int fused_plan_host_check(int H, int n_in, int T, int n_hidden, const float* m_init, const float* m_hid,
                                     const float* m_fin, int* own, long long* bytes, int max_steps, nfb::FusedStep* steps,
                                     int max_recs, long long* recs, long long* recs_lo, int* n_recs) {
    const int fpc = 2, n_chunks = ((T + fpc - 1) / fpc + 1) & ~1;   // as nfb_api.cu build_fused
    const nfb::FusedNeeds nd = nfb::fused_needs(H, n_in, T, fpc, n_chunks, m_init, m_hid, m_fin);
    const nfb::FusedPlan P = nfb::plan_fused(nd, n_hidden, fpc * 24);
    for (int i = 0; i < 4; ++i) own[i] = P.own[i / 2][i % 2];
    *bytes = (long long)P.bytes;
    if ((int)P.steps.size() > max_steps) return -1;
    for (size_t i = 0; i < P.steps.size(); ++i) steps[i] = P.steps[i];
    int n = 0;
    for (size_t g = 0; g < P.recs.size(); ++g)
        for (const nfb::FusedRec& r : P.recs[g]) {
            if (n == max_recs) return -1;
            long long* o = recs + 5 * n;
            o[0] = (long long)g; o[1] = r.row0; o[2] = r.nrows; o[3] = r.kc; o[4] = (long long)r.off_hi;
            recs_lo[n++] = (long long)r.off_lo;
        }
    *n_recs = n;
    return (int)P.steps.size();
}
