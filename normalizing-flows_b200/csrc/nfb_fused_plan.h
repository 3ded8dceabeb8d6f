// nfb_fused_plan.h -- layout of a fused spline block's packed weight stream (host code, no CUDA): which [64 x 64] blocks
// of the conditioner's matrices are non-zero, which consumer warpgroup of the fused kernel (nfb_fused_rqs.cu) owns which
// output slice of the hidden GEMMs, the step table the kernel walks and the records the packer (nfb_api.cu) fills.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <utility>
#include <vector>

namespace nfb {

// One weight record of the packed stream: a W_hi tile followed by its W_lo twin.  A tile stacks up to two [8 n8 x 64]
// halves, one per consumer warpgroup (warpgroup 0's, then warpgroup 1's); a record with one half (kStepHalf) holds it
// at offset 0.  Each warpgroup multiplies its half with its own A-operand K-chunk and reads its own (kc, flags) pair;
// the records of one of its output slices are consecutive, and the records come in the order the kernel consumes them
// (LU map, hidden GEMMs, final-layer chunks).
enum { kStepFirst = 1,    // first record of the warpgroup's slice: overwrites the accumulator
       kStepLast = 2,     // last record of the warpgroup's slice: the slice's epilogue follows
       kStepQuad = 4,     // four products (W_lo A_lo as well): the LU map, which transforms z itself
       kStepSkip = 8,     // the record has no half for this warpgroup, or an all-zero one (MADE mask): no products
       kStepHalf = 16,    // the record carries one half only, at offset 0
       kStepSlabShift = 5 };  // bits 5-6: trailing K = 16 slabs of the half that are all zero (MADE mask): no products
struct alignas(8) FusedStep {
    uint16_t bytes16;     // record size / 16
    uint8_t n8;           // rows of a half / 8 (MMA N / 8)
    uint8_t kc, flags;    // warpgroup 0: A-operand K-chunk, kStep*
    uint8_t kc1, flags1;  // warpgroup 1
    uint8_t pad_;
};
static_assert(sizeof(FusedStep) == 8, "the kernel loads a step as one uint2");

// one half of a record: rows [row0, row0 + nrows) of a GEMM's effective matrix, K-chunk kc, at these stream offsets
struct FusedRec { int row0, nrows, kc; size_t off_hi, off_lo; };

// Which [64 x 64] blocks of a fused block's matrices are non-zero, with the hidden units sorted by MADE degree so that
// every masked matrix is block-triangular (nets/made.py:57-76 degree rules).  Unmasked nets: every block.
struct FusedNeeds {
    std::vector<int> perm;        // sorted position -> hidden unit (identity for unmasked nets)
    int ns = 0, n_chunks = 0;     // 64-column slices of the hidden width; final-layer chunks
    std::vector<uint8_t> hidden;  // [ns][ns]: output slice j, K-chunk kc of the hidden-to-hidden GEMMs
    std::vector<uint8_t> fin;     // [n_chunks][ns]: final-layer chunk c, K-chunk kc: 1 + the last K = 16 slab with a
                                  // non-zero (the hidden units are sorted by degree, so the needed slabs are a prefix)
};

// m_init [H x n_in], m_hid [H x H] (all hidden masks share the structure; null: none), m_fin [T*23 x H]: the MADE masks
// (m_init null: unmasked net).  Final-layer chunk c holds features [fpc c, fpc c + fpc), 24 rows each (23 parameters +
// 1 pad).
inline FusedNeeds fused_needs(int H, int n_in, int T, int fpc, int n_chunks, const float* m_init, const float* m_hid,
                              const float* m_fin) {
    FusedNeeds nd;
    const int ns = H / 64, crow = fpc * 24;
    nd.ns = ns;
    nd.n_chunks = n_chunks;
    nd.perm.resize(H);
    for (int i = 0; i < H; ++i) nd.perm[i] = i;
    const bool masked = m_init != nullptr;
    if (masked) {
        std::vector<int> deg(H, 0);  // row sum of the input mask = number of inputs a unit may see = its degree
        for (int i = 0; i < H; ++i) for (int j = 0; j < n_in; ++j) deg[i] += m_init[(size_t)i * n_in + j] != 0.f;
        std::stable_sort(nd.perm.begin(), nd.perm.end(), [&](int x, int y) { return deg[x] < deg[y]; });
    }
    const std::vector<int>& perm = nd.perm;
    nd.hidden.assign((size_t)ns * ns, 1);
    if (masked && m_hid)
        for (int j = 0; j < ns; ++j)
            for (int kc = 0; kc < ns; ++kc) {
                bool any = false;
                for (int i = 64 * j; i < 64 * j + 64 && !any; ++i)
                    for (int k = kc * 64; k < kc * 64 + 64; ++k)
                        if (m_hid[(size_t)perm[i] * H + perm[k]] != 0.f) { any = true; break; }
                nd.hidden[(size_t)j * ns + kc] = any;
            }
    nd.fin.assign((size_t)n_chunks * ns, 4);
    if (masked)
        for (int c = 0; c < n_chunks; ++c)
            for (int kc = 0; kc < ns; ++kc) {
                int last = 0;
                for (int i = 0; i < crow; ++i) {
                    const int t = fpc * c + i / 24, q = i % 24;
                    if (t >= T || q >= 23) continue;
                    for (int k = kc * 64 + 16 * last; k < kc * 64 + 64; ++k)
                        if (m_fin[(size_t)(t * 23 + q) * H + perm[k]] != 0.f) last = (k - kc * 64) / 16 + 1;
                }
                nd.fin[(size_t)c * ns + kc] = (uint8_t)last;
            }
    return nd;
}

struct FusedPlan {
    int own[2][2];                            // hidden output slices of each consumer warpgroup, in order; -1: none
    std::vector<FusedStep> steps;             // hidden GEMMs 0 .. n_hidden - 1, then the final-layer chunk pairs
    std::vector<std::vector<FusedRec>> recs;  // [n_hidden + 1]: the halves of each GEMM's records
    size_t bytes = 0;                         // size of the stream
};

// The (slice, K-chunk) blocks one warpgroup multiplies in a hidden GEMM of kcs K-chunks: its slices in order, each
// slice's non-zero K-chunks ascending (the accumulation order is part of the validated numerics).  K-chunk 0 is always
// kept, so that every slice has a first record that initialises its accumulator.
inline std::vector<std::pair<int, int>> fused_blocks(const int (&own)[2], int kcs, const FusedNeeds& nd) {
    std::vector<std::pair<int, int>> b;
    for (int q = 0; q < 2; ++q)
        if (own[q] >= 0)
            for (int kc = 0; kc < kcs; ++kc)
                if (kc == 0 || nd.hidden[(size_t)own[q] * nd.ns + kc]) b.emplace_back(own[q], kc);
    return b;
}

// Hidden GEMMs: record i carries block i of each warpgroup's list; when one list is longer, its extra records carry
// that warpgroup's half alone, and the other warpgroup passes them as skipped records at the end of its last slice (a
// warpgroup without a slice, H = 64, passes every record as one slice with no products).  The slice ownership is
// shared by every GEMM of the block (the residual stream stays in the owner's registers) and is chosen to minimise the
// records: each warpgroup owns at most ceil(ns / 2) slices (the residual stream has 2 x 32 registers per thread), and
// the contiguous split {0 .. ceil(ns/2) - 1} / {ceil(ns/2) .. ns - 1} wins ties, so an unmasked net streams the same
// records as a plain split.  The streamed halves are exactly the non-zero blocks whatever the ownership; balancing the
// two lists leaves no record with an all-zero half.
// Final layer: record c carries chunk 2c for warpgroup 0 and 2c + 1 for warpgroup 1 on the union of their K-chunks; a
// K-chunk only one of them reaches is skipped by the other, and the all-zero trailing K = 16 slabs of a half (the last
// K-chunk a chunk's features reach) are skipped by its warpgroup.  Zero weights add exact zeros: skipping their
// products leaves every accumulator bit as it was.
inline FusedPlan plan_fused(const FusedNeeds& nd, int n_hidden, int crow) {
    const int ns = nd.ns, half = (ns + 1) / 2;
    FusedPlan P;
    auto make_own = [&](unsigned m, int (&o)[2][2]) {  // bit j of m set: warpgroup 1 owns slice j
        int n[2] = {0, 0};
        o[0][0] = o[0][1] = o[1][0] = o[1][1] = -1;
        for (int j = 0; j < ns; ++j) {
            const int w = (m >> j) & 1u;
            if (n[w] == half) return false;
            o[w][n[w]++] = j;
        }
        return true;
    };
    auto records = [&](const int (&o)[2][2]) {
        size_t r = 0;
        for (int ph = 0; ph < n_hidden; ++ph) {
            const int kcs = ph == 0 ? 1 : ns;
            r += std::max(fused_blocks(o[0], kcs, nd).size(), fused_blocks(o[1], kcs, nd).size());
        }
        return r;
    };
    const unsigned all = (1u << ns) - 1u, contiguous = all & ~((1u << half) - 1u);
    make_own(contiguous, P.own);
    size_t best = records(P.own);
    for (unsigned m = 0; m <= all; ++m) {
        int o[2][2];
        if (!make_own(m, o)) continue;
        const size_t r = records(o);
        if (r < best) {
            best = r;
            std::copy(&o[0][0], &o[0][0] + 4, &P.own[0][0]);
        }
    }

    P.recs.resize(n_hidden + 1);
    size_t off = 0;
    for (int ph = 0; ph < n_hidden; ++ph) {
        const bool onto = ph > 0 && (ph & 1) == 0;  // second GEMM of a residual block: h += ..., no first record
        const int kcs = ph == 0 ? 1 : ns;
        const std::vector<std::pair<int, int>> b[2] = {fused_blocks(P.own[0], kcs, nd), fused_blocks(P.own[1], kcs, nd)};
        const size_t n = std::max(b[0].size(), b[1].size());
        for (size_t i = 0; i < n; ++i) {
            uint8_t kc[2], fl[2];
            const bool both = i < b[0].size() && i < b[1].size();
            const int tot = both ? 128 : 64;
            size_t o = 0;
            for (int w = 0; w < 2; ++w) {
                const auto& L = b[w];
                if (i < L.size()) {
                    const bool first = i == 0 || L[i - 1].first != L[i].first;
                    const bool last = i + 1 == L.size() ? i + 1 == n : L[i + 1].first != L[i].first;
                    kc[w] = (uint8_t)L[i].second;
                    fl[w] = (uint8_t)((first && !onto ? kStepFirst : 0) | (last ? kStepLast : 0));
                    P.recs[ph].push_back(FusedRec{64 * L[i].first, 64, L[i].second, off + o, off + (size_t)tot * 128 + o});
                    o += (size_t)64 * 128;
                } else {
                    kc[w] = 0;
                    fl[w] = (uint8_t)(kStepSkip | (i + 1 == n ? kStepLast : 0));
                }
                if (!both) fl[w] |= kStepHalf;
            }
            P.steps.push_back(FusedStep{(uint16_t)(tot * 16), 8, kc[0], fl[0], kc[1], fl[1], 0});
            off += (size_t)tot * 256;
        }
    }
    for (int c = 0; c + 1 < nd.n_chunks; c += 2) {
        const uint8_t* na = &nd.fin[(size_t)c * ns];
        const uint8_t* nb = &nd.fin[(size_t)(c + 1) * ns];
        std::vector<int> kcs;
        for (int kc = 0; kc < ns; ++kc)
            if (kc == 0 || na[kc] || nb[kc]) kcs.push_back(kc);
        const int tot = 2 * crow;
        // (K-chunk 0 of a chunk with no non-zero in it: all four slabs, as the first record must initialise the accumulator)
        auto half_flags = [&](int kc, uint8_t need, int fl) {
            if (kc > 0 && !need) return (uint8_t)(fl | kStepSkip);
            return (uint8_t)(fl | ((need ? 4 - need : 0) << kStepSlabShift));
        };
        for (size_t i = 0; i < kcs.size(); ++i) {
            const int kc = kcs[i];
            const int fl = (i == 0 ? kStepFirst : 0) | (i + 1 == kcs.size() ? kStepLast : 0);
            P.steps.push_back(FusedStep{(uint16_t)(tot * 16), (uint8_t)(crow / 8), (uint8_t)kc, half_flags(kc, na[kc], fl),
                                        (uint8_t)kc, half_flags(kc, nb[kc], fl), 0});
            P.recs[n_hidden].push_back(FusedRec{c * crow, crow, kc, off, off + (size_t)tot * 128});
            P.recs[n_hidden].push_back(FusedRec{(c + 1) * crow, crow, kc, off + (size_t)crow * 128,
                                                off + (size_t)(tot + crow) * 128});
            off += (size_t)tot * 256;
        }
    }
    P.bytes = off;
    return P;
}

}  // namespace nfb
