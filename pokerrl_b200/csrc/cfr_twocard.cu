// Level-synchronous public-tree sweeps for TWO-HOLE-CARD games (Hold'em family, range R = C(deck,2) = 1326) - sm_90a.
//
// The reference has no working value path for these games (ValueFiller.py:18-19 and PublicTree.py:193-203 are
// one-card only); the arithmetic here is the generalisation stated in SURVEY.md appendix A and restated in float64 by
// oracle/cfr2_numpy.py: blocker-aware fold / showdown values, board deals that zero blocked hands, board-weighted chance
// sums with optional suit-isomorphism symmetrisation.  Everything else (regrets, regret matching, averaging, BR) is the
// same statement as the one-card sweeps (cfr_levels.cu), evaluated in float32.
//
// Mapping: one THREAD per (node, hand) with hands contiguous -> every row access is a fully coalesced 5.3 KB stream;
// node structure loads are warp-uniform (broadcast).  Terminal rows are evaluated by one CTA per terminal node:
//   fold      T - cs[c1] - cs[c2] + r[h]                 (52 per-card sums, deterministic)
//   showdown  O(R) via the board's strength order: scatter by sorted position, block scan, strictly-weaker /
//             strictly-stronger mass from group boundaries, minus a ~100-term blocker correction per hand
// instead of the O(R^2) sign-matrix product: these rows are HBM-bound, the dense 1326x1326 contraction (tensor cores)
// would only add work - see DESIGN.md §6.
// Each operation (reach, decision nodes with the CFR rules, showdown steps) is written once as a device body; the
// record-based kernels (*_v2, terminal2_kernel_v3) and the record-free ones differ only in how they read a node's
// structure (16-byte records or pointer chains) and the board's tables (packed hand records or separate tables).
#include <cuda_runtime.h>
#include <vector>
#include <stdint.h>

#include "pokerrl_b200.h"
#include "prl_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kVecThreads = 128;  // row kernels: 128 threads x 4 hands
constexpr int kTermThreads = 256;
constexpr int kRowStride = 53;     // n_deck - 1 hands per card row + 1, +1 padding against bank conflicts
constexpr int kChanceChunk = 128;  // children summed per block in the first stage of a chance-node reduction

struct Ctx2 {
    prl_tree_t T;
    prl_buffers_t B;
    int lo, n;       // first work-list entry of this launch, number of entries
    int mask;        // seats to process
    int mode[2];     // strategy source per seat
    int algo, upd_p, iter, delay;
    float m_old, m_new;  // CFR+ averaging weights of this iteration (CFRPlus.py:68-73), computed on the host
};

__device__ __forceinline__ const float* strat_table(const Ctx2& c, int m) {
    return (m == PRL_STRAT_F32) ? c.B.strat : (const float*)c.B.avg;
}

// ---- four hands per thread: rows are read / written as float4 (ld is a multiple of 4, rows are 16-byte aligned) -------
struct F4 {
    float v[4];
};
__device__ __forceinline__ F4 ld4(const float* p) {
    const float4 q = *reinterpret_cast<const float4*>(p);
    return F4{{q.x, q.y, q.z, q.w}};
}
__device__ __forceinline__ void st4(float* p, const F4& a) {
    *reinterpret_cast<float4*>(p) = make_float4(a.v[0], a.v[1], a.v[2], a.v[3]);
}
__device__ __forceinline__ F4 splat(float x) { return F4{{x, x, x, x}}; }

// probabilities of the action leading to the child in table row `slot` for hands h0..h0+3 (rows fs..fs+A-1 belong to
// one decision node)
__device__ __forceinline__ F4 strat4(const Ctx2& c, int m, int slot, int fs, int A, int h0) {
    const size_t ld = c.T.ld;
    if (m == PRL_STRAT_UNIFORM64) return splat(1.0f / (float)A);
    if (m == PRL_STRAT_AVG_SUM) {  // reach-weighted sums, normalised on the fly (LinearCFR.py:64-71)
        const float* tab = (const float*)c.B.avg;
        F4 tot = splat(0.0f), mine = splat(0.0f);
        for (int j = 0; j < A; ++j) {
            const F4 x = ld4(tab + (size_t)(fs + j) * ld + h0);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                tot.v[i] += x.v[i];
                if (fs + j == slot) mine.v[i] = x.v[i];
            }
        }
        F4 s;
#pragma unroll
        for (int i = 0; i < 4; ++i) s.v[i] = (tot.v[i] == 0.0f) ? 1.0f / (float)A : mine.v[i] / tot.v[i];
        return s;
    }
    return ld4(strat_table(c, m) + (size_t)slot * ld + h0);
}

__device__ __forceinline__ bool hand_blocked(const prl_tree_t& T, int h, unsigned long long bmask) {
    const int c1 = T.hand_cards[2 * h], c2 = T.hand_cards[2 * h + 1];
    return ((bmask >> c1) | (bmask >> c2)) & 1ull;
}

// ------------------------------------------------------------------------------------------------ CFR rules
// regret matching of one node's rows: a row's positive regret over the node's positive regret mass, uniform where that
// mass is 0
struct RegretMatch {
    F4 ssum, inv;
    float uni;
    __device__ __forceinline__ RegretMatch(const F4& pos_mass, int A) : ssum(pos_mass), uni(1.0f / (float)A) {
#pragma unroll
        for (int i = 0; i < 4; ++i) inv.v[i] = (ssum.v[i] > 0.0f) ? 1.0f / ssum.v[i] : 0.0f;
    }
    __device__ __forceinline__ F4 operator()(const F4& r) const {
        F4 st;
#pragma unroll
        for (int i = 0; i < 4; ++i) st.v[i] = (ssum.v[i] > 0.0f) ? fmaxf(r.v[i], 0.0f) * inv.v[i] : uni;
        return st;
    }
};

// average-strategy update of table row ap from the row's strategy s and the child's reach r.  PRED: PCFR+, whose average is
// DCFR's reach-weighted sum with weight w_t.
template <bool PRED>
__device__ __forceinline__ void avg_update(const Ctx2& c, float* ap, const F4& s, const F4& r) {
    if (!PRED && c.algo == PRL_ALGO_CFR_PLUS) {  // CFRPlus.py:65-87 (float table)
        if (c.iter >= c.delay) {
            F4 a = ld4(ap);
#pragma unroll
            for (int i = 0; i < 4; ++i) a.v[i] = c.m_old * a.v[i] + c.m_new * s.v[i];
            st4(ap, a);
        }
    } else {
        F4 a = ld4(ap);
        const float w = (c.algo == PRL_ALGO_LINEAR) ? (float)(c.iter + 1)                  // LinearCFR.py:56-61
                        : (PRED || c.algo == PRL_ALGO_DCFR) ? c.B.dcfr[3 * (size_t)c.iter + 2] : 1.0f;
#pragma unroll
        for (int i = 0; i < 4; ++i) a.v[i] = a.v[i] + r.v[i] * w;  // VanillaCFR.py:57-62
        st4(ap, a);
    }
}

// ------------------------------------------------------------------------------------------------ reach (top-down)
// reach rows of node n for hands h0..h0+3 (StrategyFiller.py:118-146 generalised).  Structure of n: parent par, n's table
// row `slot`, first table row fs of its siblings, kind pk and fan-out A of the parent (read only when par >= 0).
template <bool UPDATE_AVG, bool PRED = false>
__device__ __forceinline__ void reach_rows(const Ctx2& c, int n, int h0, int par, int slot, int fs, int pk, int A) {
    const int ld = c.T.ld, R = c.T.n_range;
    const size_t N = (size_t)c.T.n_nodes;
#pragma unroll 1
    for (int q = 0; q < 2; ++q) {
        if (!(c.mask & (1 << q))) continue;
        float* reach_q = c.B.reach + (size_t)q * N * ld;
        F4 r;
        if (par < 0) {  // PublicTree.py:122-124; a sub-game root that already shows a board zeroes the blocked hands
            const int b = c.T.board[n];
            const unsigned long long bm = (b >= 0) ? c.T.board_mask[b] : 0ull;
#pragma unroll
            for (int i = 0; i < 4; ++i) r.v[i] = (h0 + i < R && !hand_blocked(c.T, h0 + i, bm)) ? 1.0f / (float)R : 0.0f;
        } else {
            const F4 rp = ld4(reach_q + (size_t)par * ld + h0);
            if (pk == PRL_KIND_CHANCE) {  // the deal multiplies both rows and zeroes hands holding a board card
                const int b = c.T.board[n];
                const unsigned long long bm = c.T.board_mask[b];
                const float pr = c.T.board_prob[b];
#pragma unroll
                for (int i = 0; i < 4; ++i) r.v[i] = (h0 + i < R && !hand_blocked(c.T, h0 + i, bm)) ? rp.v[i] * pr : 0.0f;
            } else if (pk == q) {
                const F4 s = strat4(c, c.mode[q], slot, fs, A, h0);
#pragma unroll
                for (int i = 0; i < 4; ++i) r.v[i] = s.v[i] * rp.v[i];
                if (UPDATE_AVG && q == c.upd_p) avg_update<PRED>(c, (float*)c.B.avg + (size_t)slot * ld + h0, s, r);
            } else {
                r = rp;
            }
        }
        st4(reach_q + (size_t)n * ld + h0, r);
    }
}

// block x = child node n of the level, thread = four hands; structure through the parent -> first_child -> slot chain
template <bool UPDATE_AVG, bool PRED = false>
__global__ void __launch_bounds__(kVecThreads) reach2_kernel(const Ctx2 c) {
    const int n = c.lo + blockIdx.x;
    const int h0 = 4 * (blockIdx.y * blockDim.x + threadIdx.x);
    if (h0 >= c.T.n_range) return;
    const int par = c.T.parent[n];
    int fs = 0, pk = 0, A = 0;  // a root has no parent to read
    if (par >= 0) {
        fs = c.T.slot[c.T.first_child[par]];
        pk = c.T.kind[par];
        A = c.T.n_children[par];
    }
    reach_rows<UPDATE_AVG, PRED>(c, n, h0, par, c.T.slot[n], fs, pk, A);
}

// ---- v2 row kernels: one CTA per node (ceil(R / 4) threads rounded up to a warp), node structure from ONE 16-byte
// record instead of a chain of dependent loads (parent -> first_child[parent] -> slot[...] -> rows)
constexpr int kRowThreadsMax = 352;  // 1326 hands / 4 per thread = 332 -> 11 warps

// node_rec2[n] = {parent, slot of n, first slot of the parent's children, kind(parent) | n_children(parent) << 8}
template <bool UPDATE_AVG, bool PRED = false>
__global__ void __launch_bounds__(kRowThreadsMax, 4) reach2_kernel_v2(const Ctx2 c) {
    const int n = c.lo + blockIdx.x;
    const int h0 = 4 * threadIdx.x;
    if (h0 >= c.T.n_range) return;
    const int4 rec = reinterpret_cast<const int4*>(c.T.node_rec2)[n];
    reach_rows<UPDATE_AVG, PRED>(c, n, h0, rec.x, rec.y, rec.z, rec.w & 0xff, rec.w >> 8);
}

// ------------------------------------------------------------------------------------------------ decision nodes (bottom-up)
// regrets + regret matching of the seat's own node with the A child rows held in registers (each row is loaded once);
// same operations in the same order as the loops of value_rows -> identical results.  PRED: PCFR+'s regret, and regret
// matching of its prediction max(R_new + d, 0)
template <int A, bool PRED>
__device__ __forceinline__ F4 own_node_update(const Ctx2& c, int fs, int h0, const float* ecol) {
    const size_t ld = c.T.ld;
    float* rcol = c.B.regret + (size_t)fs * ld + h0;
    float* scol = c.B.strat + (size_t)fs * ld + h0;
    F4 e[A], rg[A];
#pragma unroll
    for (int k = 0; k < A; ++k) e[k] = ld4(ecol + (size_t)k * ld);
#pragma unroll
    for (int k = 0; k < A; ++k) rg[k] = ld4(rcol + (size_t)k * ld);
    F4 v = splat(0.0f);
#pragma unroll
    for (int k = 0; k < A; ++k) {
        const F4 s = ld4(scol + (size_t)k * ld);  // the seat's current strategy (PRL_STRAT_F32)
#pragma unroll
        for (int i = 0; i < 4; ++i) v.v[i] += s.v[i] * e[k].v[i];
    }
    F4 ssum = splat(0.0f);
    if constexpr (PRED) {  // each row's regrets are stored as soon as they are known; rg[k] then holds the prediction
#pragma unroll
        for (int k = 0; k < A; ++k) {
            F4 pr;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float d = e[k].v[i] - v.v[i];
                rg[k].v[i] = prl::pcfr_regret(d, rg[k].v[i]);
                pr.v[i] = prl::pcfr_prediction(rg[k].v[i], d);
                ssum.v[i] += pr.v[i];
            }
            st4(rcol + (size_t)k * ld, rg[k]);
            rg[k] = pr;
        }
        const RegretMatch rm(ssum, A);
#pragma unroll
        for (int k = 0; k < A; ++k) st4(scol + (size_t)k * ld, rm(rg[k]));
        return v;
    }
    const prl::RegretW w = prl::regret_w(c);
#pragma unroll
    for (int k = 0; k < A; ++k) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            rg[k].v[i] = prl::regret_step(c.algo, e[k].v[i] - v.v[i], rg[k].v[i], w);
            ssum.v[i] += fmaxf(rg[k].v[i], 0.0f);
        }
    }
    const RegretMatch rm(ssum, A);
#pragma unroll
    for (int k = 0; k < A; ++k) {
        st4(rcol + (size_t)k * ld, rg[k]);
        st4(scol + (size_t)k * ld, rm(rg[k]));
    }
    return v;
}

// ValueFiller.py:80-93 + _CFRBase.py:146-185 + regret matching of decision node n for hands h0..h0+3, given its
// structure: first child fc, first table row fs of the children, kind, fan-out A.  REG_ROWS: the updating seat's own
// node with fan-out 2..4 takes the register-resident own_node_update.  PRED: the update is PCFR+'s.
template <bool WITH_BR, bool UPDATE, bool REG_ROWS, bool PRED = false>
__device__ __forceinline__ void value_rows(const Ctx2& c, int n, int fc, int fs, int kind, int A, int h0) {
    const int ld = c.T.ld;
    const size_t N = (size_t)c.T.n_nodes;
#pragma unroll 1
    for (int p = 0; p < 2; ++p) {
        if (!(c.mask & (1 << p))) continue;
        float* ev_p = c.B.ev + (size_t)p * N * ld;
        float* evbr_p = WITH_BR ? c.B.ev_br + (size_t)p * N * ld : nullptr;
        const float* ecol = ev_p + (size_t)fc * ld + h0;
        F4 v = splat(0.0f), vbr = splat(0.0f);
        if (kind != p) {  // the other seat acts: sums over children
            for (int k = 0; k < A; ++k) {
                const F4 e = ld4(ecol + (size_t)k * ld);
#pragma unroll
                for (int i = 0; i < 4; ++i) v.v[i] += e.v[i];
            }
            if (WITH_BR)
                for (int k = 0; k < A; ++k) {
                    const F4 e = ld4(evbr_p + (size_t)(fc + k) * ld + h0);
#pragma unroll
                    for (int i = 0; i < 4; ++i) vbr.v[i] += e.v[i];
                }
        } else if (REG_ROWS && UPDATE && p == c.upd_p && A >= 2 && A <= 4 && c.mode[p] == PRL_STRAT_F32) {
            if (A == 2) v = own_node_update<2, PRED>(c, fs, h0, ecol);
            else if (A == 3) v = own_node_update<3, PRED>(c, fs, h0, ecol);
            else v = own_node_update<4, PRED>(c, fs, h0, ecol);
        } else {
            const int m = c.mode[p];
            for (int k = 0; k < A; ++k) {
                const F4 e = ld4(ecol + (size_t)k * ld);
                const F4 s = strat4(c, m, fs + k, fs, A, h0);
#pragma unroll
                for (int i = 0; i < 4; ++i) v.v[i] += s.v[i] * e.v[i];
            }
            if (WITH_BR) {
                vbr = ld4(evbr_p + (size_t)fc * ld + h0);
                for (int k = 1; k < A; ++k) {
                    const F4 e = ld4(evbr_p + (size_t)(fc + k) * ld + h0);
#pragma unroll
                    for (int i = 0; i < 4; ++i) vbr.v[i] = fmaxf(vbr.v[i], e.v[i]);
                }
            }
            if (UPDATE && p == c.upd_p) {  // any fan-out: rows re-read from L1 / L2
                float* rcol = c.B.regret + (size_t)fs * ld + h0;
                float* scol = c.B.strat + (size_t)fs * ld + h0;
                const prl::RegretW w = prl::regret_w(c);
                F4 ssum = splat(0.0f);
                for (int k = 0; k < A; ++k) {  // pass A: positive regret mass (new regrets are recomputed in pass B)
                    const F4 e = ld4(ecol + (size_t)k * ld), rg = ld4(rcol + (size_t)k * ld);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        if constexpr (PRED) {
                            const float d = e.v[i] - v.v[i];
                            ssum.v[i] += prl::pcfr_prediction(prl::pcfr_regret(d, rg.v[i]), d);
                        } else {
                            ssum.v[i] += fmaxf(prl::regret_step(c.algo, e.v[i] - v.v[i], rg.v[i], w), 0.0f);
                        }
                    }
                }
                const RegretMatch rm(ssum, A);
                for (int k = 0; k < A; ++k) {  // pass B: store regrets and the regret-matching strategy
                    const F4 e = ld4(ecol + (size_t)k * ld);
                    F4 rg = ld4(rcol + (size_t)k * ld);
                    if constexpr (PRED) {
                        F4 pr;
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const float d = e.v[i] - v.v[i];
                            rg.v[i] = prl::pcfr_regret(d, rg.v[i]);
                            pr.v[i] = prl::pcfr_prediction(rg.v[i], d);
                        }
                        st4(rcol + (size_t)k * ld, rg);
                        st4(scol + (size_t)k * ld, rm(pr));
                    } else {
#pragma unroll
                        for (int i = 0; i < 4; ++i) rg.v[i] = prl::regret_step(c.algo, e.v[i] - v.v[i], rg.v[i], w);
                        st4(rcol + (size_t)k * ld, rg);
                        st4(scol + (size_t)k * ld, rm(rg));
                    }
                }
            }
        }
        st4(ev_p + (size_t)n * ld + h0, v);
        if (WITH_BR) st4(evbr_p + (size_t)n * ld + h0, vbr);
    }
}

// block x = work-list entry t -> decision node n, thread = four hands; structure through order / first_child / slot
template <bool WITH_BR, bool UPDATE, bool PRED = false>
__global__ void __launch_bounds__(kVecThreads) value2_kernel(const Ctx2 c) {
    const int h0 = 4 * (blockIdx.y * blockDim.x + threadIdx.x);
    if (h0 >= c.T.n_range) return;
    const int n = c.T.order[c.lo + blockIdx.x];
    const int kind = c.T.kind[n], fc = c.T.first_child[n], A = c.T.n_children[n];
    value_rows<WITH_BR, UPDATE, false, PRED>(c, n, fc, c.T.slot[fc], kind, A, h0);
}

// work_rec2[t] = {node, first child, first slot of the children, kind | n_children << 8} of work-list entry t
template <bool WITH_BR, bool UPDATE, bool PRED = false>
__global__ void __launch_bounds__(kRowThreadsMax, 3) value2_kernel_v2(const Ctx2 c) {
    const int h0 = 4 * threadIdx.x;
    if (h0 >= c.T.n_range) return;
    const int4 rec = reinterpret_cast<const int4*>(c.T.work_rec2)[c.lo + blockIdx.x];
    value_rows<WITH_BR, UPDATE, true, PRED>(c, rec.x, rec.y, rec.z, rec.w & 0xff, rec.w >> 8, h0);
}

// ------------------------------------------------------------------------------------------------ chance nodes (bottom-up)
// stage 1: block (chance entry j, chunk) sums board_mult * child rows of its chunk -> workspace[arr][j][chunk][h]
// stage 2: thread (j, h): sums the chunks in order -> workspace W[arr][j][h]
// stage 3: thread (j, h): ev[n][h] = sum over suit permutations of W (or W itself) - DESIGN.md §6
// arr = 2 * seat + (0: ev, 1: ev_br)
struct ChanceGeom {
    int n_chance, max_chunks;
    size_t w_off;  // float offset of the W vectors inside the workspace
};

__device__ __forceinline__ const float* node_array(const Ctx2& c, int arr) {
    const size_t stride = (size_t)c.T.n_nodes * c.T.ld;
    return ((arr & 1) ? c.B.ev_br : c.B.ev) + (size_t)(arr >> 1) * stride;
}

__global__ void __launch_bounds__(kThreads) chance_partial_kernel(const Ctx2 c, const ChanceGeom g, const int n_arr_mask) {
    const int j = blockIdx.x / g.max_chunks, chunk = blockIdx.x % g.max_chunks;
    const int n = c.T.order[c.lo + j];
    const int fc = c.T.first_child[n], A = c.T.n_children[n];
    const int k0 = chunk * kChanceChunk, k1 = min(A, k0 + kChanceChunk);
    if (k0 >= A) return;
    const int ld = c.T.ld;
    float* ws = (float*)c.B.workspace;
    for (int arr = 0; arr < 4; ++arr) {
        if (!(n_arr_mask & (1 << arr))) continue;
        const float* src = node_array(c, arr);
        float* dst = ws + (((size_t)arr * g.n_chance + j) * g.max_chunks + chunk) * ld;
        for (int h = threadIdx.x; h < c.T.n_range; h += blockDim.x) {
            float acc = 0.0f;
            for (int k = k0; k < k1; ++k) acc += c.T.board_mult[c.T.board[fc + k]] * src[(size_t)(fc + k) * ld + h];
            dst[h] = acc;
        }
    }
}

__global__ void __launch_bounds__(kThreads) chance_sum_kernel(const Ctx2 c, const ChanceGeom g, const int n_arr_mask) {
    const int ld = c.T.ld;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int j = (int)(idx / ld), h = (int)(idx % ld);
    if (j >= g.n_chance || h >= c.T.n_range) return;
    const int n = c.T.order[c.lo + j];
    const int chunks = (c.T.n_children[n] + kChanceChunk - 1) / kChanceChunk;
    float* ws = (float*)c.B.workspace;
    for (int arr = 0; arr < 4; ++arr) {
        if (!(n_arr_mask & (1 << arr))) continue;
        const float* src = ws + (((size_t)arr * g.n_chance + j) * g.max_chunks) * ld + h;
        float acc = 0.0f;
        for (int k = 0; k < chunks; ++k) acc += src[(size_t)k * ld];
        ws[g.w_off + ((size_t)arr * g.n_chance + j) * ld + h] = acc;
    }
}

__global__ void __launch_bounds__(kThreads) chance_final_kernel(const Ctx2 c, const ChanceGeom g, const int n_arr_mask) {
    const int ld = c.T.ld;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int j = (int)(idx / ld), h = (int)(idx % ld);
    if (j >= g.n_chance || h >= c.T.n_range) return;
    const int n = c.T.order[c.lo + j];
    const float* ws = (const float*)c.B.workspace;
    for (int arr = 0; arr < 4; ++arr) {
        if (!(n_arr_mask & (1 << arr))) continue;
        const float* W = ws + g.w_off + ((size_t)arr * g.n_chance + j) * ld;
        float v;
        if (c.T.n_sym > 1) {
            v = 0.0f;
            for (int s = 0; s < c.T.n_sym; ++s) v += W[c.T.sym_perm[(size_t)s * c.T.n_range + h]];
        } else {
            v = W[h];
        }
        const_cast<float*>(node_array(c, arr))[(size_t)n * ld + h] = v;
    }
}

// ------------------------------------------------------------------------------------------------ terminals (bottom-up)
// hand index of the unordered pair (a, b), a != b, in LUT order (c1 < c2 lexicographic)
__device__ __forceinline__ int pair_index(int a, int b, int n_deck) {
    const int c1 = min(a, b), c2 = max(a, b);
    return c1 * (2 * n_deck - 1 - c1) / 2 + (c2 - c1 - 1);
}

__device__ __forceinline__ float block_sum(float v, float* red /* >= 32 floats */) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) red[w] = v;
    __syncthreads();
    float t = (l < (blockDim.x >> 5)) ? red[l] : 0.0f;
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    return t;  // every thread holds the total (fixed reduction order: deterministic)
}

// one CTA per terminal node; ValueFiller.py:34-62, 103-158 generalised (SURVEY.md appendix A)
//
// v2: same arithmetic with fewer instructions and barriers per terminal row
//   - card rows are scanned by QUADS (4 lanes x <= 16 consecutive row entries, sequential in registers, then a 2-step
//     quad scan) instead of one warp per row: 52 rows fit one pass of 208 threads
//   - every prefix array is stored CENTRED,  E[i] = (mass of the i weakest) - total / 2,  so that
//     (strictly weaker) - (strictly stronger) = E[gs] + E[ge]  without loading the totals
//   - the scatter into strength order happens while the row is loaded; fold rows skip scans, showdown rows skip the sum
//   - optional packed per-hand record (prl_tree_t.board_hand_rec): {gs, ge, 4 offsets into the card-row prefix array}
//     in one 16-byte load instead of five narrow ones
constexpr int kSegMax = 16;  // row entries per quad lane: ceil((n_deck - 1) / 4) <= 16
constexpr int kSeg52 = 13;   // ceil((52 - 1) / 4): a 52-card deck, the only one terminal2_kernel_v3 is built for

// ---- steps 2a, 2b and 3 of a showdown row over the CTA's shared arrays: ro[R] opponent reach row, srt[R + 1] reach in
// strength order, rp[n_deck][kRowStride] card-row prefix sums
// 2a. centred prefix sums of every card row in strength order: rp[c][i] = mass of the i weakest live hands holding card
//     c, minus half the row's mass.  Quad lane qj scans entries [qj * seg, qj * seg + seg) in registers, seg <= SEG.
template <int SEG>
__device__ __forceinline__ void card_row_prefix(float* rp, const float* ro, const int16_t* row_order, int n_deck, int seg) {
    const int row_len = n_deck - 1;
    const int qj = threadIdx.x & 3;
    for (int base = 0; base < n_deck; base += blockDim.x >> 2) {
        const int cc = base + (threadIdx.x >> 2);
        const bool live = cc < n_deck;
        float inc[SEG];
        float run = 0.0f;
#pragma unroll
        for (int i = 0; i < SEG; ++i) {
            const int idx = qj * seg + i;
            float v = 0.0f;
            if (live && i < seg && idx < row_len) {
                const int hh = row_order[cc * row_len + idx];
                if (hh >= 0) v = ro[hh];
            }
            run += v;
            inc[i] = run;
        }
        float sc = run;  // inclusive scan over the quad
        float t = __shfl_up_sync(0xffffffffu, sc, 1, 4);
        if (qj >= 1) sc += t;
        t = __shfl_up_sync(0xffffffffu, sc, 2, 4);
        if (qj >= 2) sc += t;
        const float half = 0.5f * __shfl_sync(0xffffffffu, sc, 3, 4);
        const float off = (sc - run) - half;
        if (live) {
            float* row = rp + cc * kRowStride;
            if (qj == 0) row[0] = -half;
#pragma unroll
            for (int i = 0; i < SEG; ++i) {
                const int idx = qj * seg + i;
                if (i < seg && idx < row_len) row[idx + 1] = off + inc[i];
            }
        }
    }
}

// 2b. centred exclusive prefix sums over srt[0..R], in place (each thread owns a contiguous segment, then a block scan;
//     wsum holds the warp totals).  srt[] must be published before the call; it is published again on return.
__device__ __forceinline__ void centred_scan(float* srt, float* wsum, int R) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
    const int per = (R + 1 + blockDim.x - 1) / blockDim.x;
    const int i0 = threadIdx.x * per, i1 = min(R + 1, i0 + per);
    float loc = 0.0f;
    for (int i = i0; i < i1; ++i) loc += srt[i];
    float incw = loc;  // inclusive scan of the per-thread sums within the warp
    for (int o = 1; o < 32; o <<= 1) {
        const float t = __shfl_up_sync(0xffffffffu, incw, o);
        if (lane >= o) incw += t;
    }
    if (lane == 31) wsum[warp] = incw;
    __syncthreads();
    float before = 0.0f, total = 0.0f;  // every thread adds the warp totals itself (fixed order)
    for (int w = 0; w < n_warps; ++w) {
        const float x = wsum[w];
        if (w < warp) before += x;
        total += x;
    }
    float run = (incw - loc) + before - 0.5f * total;
    for (int i = i0; i < i1; ++i) {
        const float x = srt[i];
        srt[i] = run;
        run += x;
    }
    __syncthreads();
}

// 3. per hand: (weaker - stronger) mass over all live hands minus the same over the two card rows of the hand (the hands
//    that share a card with it; the hand itself ties with itself and drops out), read through the packed hand records
//    of the board
template <bool WITH_BR>
__device__ __forceinline__ void showdown_from_records(const uint4* rec, const float* srt, const float* rp, float scale, int R,
                                                      float* ev_p, float* evbr_p) {
    for (int h = threadIdx.x; h < R; h += blockDim.x) {
        const uint4 q = rec[h];  // int16 x 8: gs, ge, c1 row + lt, c1 row + le, c2 row + lt, c2 row + le, 0, 0
        const int gs = (int)(short)(q.x & 0xffffu);
        float v = 0.0f;
        if (gs >= 0) {
            const float all = srt[gs] + srt[q.x >> 16];
            const float rows = (rp[q.y & 0xffffu] + rp[q.y >> 16]) + (rp[q.z & 0xffffu] + rp[q.z >> 16]);
            v = (all - rows) * scale;
        }
        ev_p[h] = v;
        if (WITH_BR) evbr_p[h] = v;
    }
}

// one CTA per terminal node; ValueFiller.py:34-62, 103-158 generalised (SURVEY.md appendix A)
//
// v2: same arithmetic with fewer instructions and barriers per terminal row
//   - card rows are scanned by QUADS (4 lanes x <= 16 consecutive row entries, sequential in registers, then a 2-step
//     quad scan) instead of one warp per row: 52 rows fit one pass of 208 threads
//   - every prefix array is stored CENTRED,  E[i] = (mass of the i weakest) - total / 2,  so that
//     (strictly weaker) - (strictly stronger) = E[gs] + E[ge]  without loading the totals
//   - the scatter into strength order happens while the row is loaded; fold rows skip scans, showdown rows skip the sum
//   - optional packed per-hand record (prl_tree_t.board_hand_rec): {gs, ge, 4 offsets into the card-row prefix array}
//     in one 16-byte load instead of five narrow ones
template <bool WITH_BR>
__global__ void __launch_bounds__(kTermThreads) terminal2_kernel(const Ctx2 c) {
    extern __shared__ float smem[];
    const int R = c.T.n_range, ld = c.T.ld, n_deck = c.T.n_deck;
    float* ro = smem;                      // [R]      opponent reach row
    float* srt = ro + R;                   // [R + 1]  reach in strength order, then its centred exclusive prefix sums
    float* red = srt + R + 1;              // [32]
    float* wsum = red + 32;                // [kTermThreads / 32]
    float* rp = wsum + kTermThreads / 32;  // [n_deck][kRowStride] centred prefix sums of every card row (fold: [n_deck] sums)
    const int n = c.T.order[c.lo + blockIdx.x];
    const int kind = c.T.kind[n];
    const int b = c.T.board[n];
    const size_t N = (size_t)c.T.n_nodes;
    const float scale = c.T.eq_const * c.T.pot[n] * 0.5f;
    const bool fold = kind == PRL_KIND_FOLD;
    const int row_len = n_deck - 1, seg = (row_len + 3) >> 2;
    const int qj = threadIdx.x & 3;
#pragma unroll 1
    for (int p = 0; p < 2; ++p) {
        if (!(c.mask & (1 << p))) continue;
        const float* ro_g = c.B.reach + ((size_t)(1 - p) * N + n) * ld;
        float* ev_p = c.B.ev + ((size_t)p * N + n) * ld;
        float* evbr_p = WITH_BR ? c.B.ev_br + ((size_t)p * N + n) * ld : nullptr;
        __syncthreads();  // shared arrays are reused by the second seat
        if (fold) {
            float part = 0.0f;
            for (int h = threadIdx.x; h < R; h += blockDim.x) {
                const float r = ro_g[h];
                ro[h] = r;
                part += r;
            }
            const float T = block_sum(part, red);  // includes the barrier that publishes ro[]
            // per-card sums: quad lane qj adds entries [qj * seg, qj * seg + seg) of the card's row
            for (int base = 0; base < n_deck; base += blockDim.x >> 2) {
                const int cc = base + (threadIdx.x >> 2);
                float run = 0.0f;
                if (cc < n_deck) {
                    for (int i = 0; i < seg; ++i) {
                        const int idx = qj * seg + i;
                        if (idx < row_len) run += ro[pair_index(cc, idx + (idx >= cc), n_deck)];
                    }
                }
                run += __shfl_xor_sync(0xffffffffu, run, 1);
                run += __shfl_xor_sync(0xffffffffu, run, 2);
                if (cc < n_deck && qj == 0) rp[cc] = run;
            }
            __syncthreads();
            const float sgn = (c.T.acted_last[n] == p) ? -scale : scale;
            const unsigned long long bmask = (b >= 0) ? c.T.board_mask[b] : 0ull;
            for (int h = threadIdx.x; h < R; h += blockDim.x) {
                const int c1 = c.T.hand_cards[2 * h], c2 = c.T.hand_cards[2 * h + 1];
                float v = (T - rp[c1] - rp[c2] + ro[h]) * sgn;
                if (((bmask >> c1) | (bmask >> c2)) & 1ull) v = 0.0f;
                ev_p[h] = v;
                if (WITH_BR) evbr_p[h] = v;
            }
            continue;
        }
        // ---- showdown on a complete board (strength tables exist)
        const int16_t* pos_tab = c.T.board_pos + (size_t)b * R;
        const int16_t* row_order = c.T.board_row_order + (size_t)b * n_deck * row_len;
        for (int i = threadIdx.x; i <= R; i += blockDim.x) srt[i] = 0.0f;
        __syncthreads();
        // 1. load the row, scattering it into strength order (pos is a permutation of the live hands: deterministic)
        for (int h = threadIdx.x; h < R; h += blockDim.x) {
            const float r = ro_g[h];
            const int ps = pos_tab[h];
            ro[h] = r;
            if (ps >= 0) srt[ps] = r;
        }
        __syncthreads();
        card_row_prefix<kSegMax>(rp, ro, row_order, n_deck, seg);
        centred_scan(srt, wsum, R);
        if (c.T.board_hand_rec) {
            showdown_from_records<WITH_BR>(reinterpret_cast<const uint4*>(c.T.board_hand_rec) + (size_t)b * R, srt, rp,
                                           scale, R, ev_p, evbr_p);
        } else {  // 3. through the separate strength and card-row position tables
            const int16_t* gs_tab = c.T.board_gs + (size_t)b * R;
            const int16_t* ge_tab = c.T.board_ge + (size_t)b * R;
            const uchar4* row_pos = reinterpret_cast<const uchar4*>(c.T.board_row_pos) + (size_t)b * R;
            for (int h = threadIdx.x; h < R; h += blockDim.x) {
                const int gs = gs_tab[h];
                float v = 0.0f;
                if (gs >= 0) {
                    const int ge = ge_tab[h];
                    const int c1 = c.T.hand_cards[2 * h], c2 = c.T.hand_cards[2 * h + 1];
                    const uchar4 q = row_pos[h];  // {weaker in row c1, weaker in row c2, weaker-or-equal c1, c2}
                    const float* r1 = rp + c1 * kRowStride;
                    const float* r2 = rp + c2 * kRowStride;
                    const float all = srt[gs] + srt[ge];
                    const float rows = (r1[q.x] + r1[q.z]) + (r2[q.y] + r2[q.w]);
                    v = (all - rows) * scale;
                }
                ev_p[h] = v;
                if (WITH_BR) evbr_p[h] = v;
            }
        }
    }
}

// v3: showdown rows only, with the v2 arithmetic and every input of a row STAGED IN SHARED MEMORY BY ASYNCHRONOUS COPIES
// (cp.async): the opponent's reach row and the board's three tables (strength positions, card-row orders, packed hand
// records) are requested together right after ONE structure load (work_rec2), so a terminal row pays two dependent global
// latencies (record -> everything) instead of five (order -> node fields -> reach row -> row orders -> hand records).
__device__ __forceinline__ void cp_async4(void* dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}
__host__ __device__ inline size_t up16(size_t x) { return (x + 15) & ~(size_t)15; }

// shared-memory carve-up of terminal2_kernel_v3 (byte offsets, every region 16-byte aligned)
struct TermSmem {
    size_t rec, ro, roword, pos, srt, red, wsum, rp, total;
    __host__ __device__ TermSmem(int R, int n_deck) {
        rec = 0;
        ro = rec + up16((size_t)R * 16);
        roword = ro + up16((size_t)R * 4);
        pos = roword + up16((size_t)n_deck * (n_deck - 1) * 2);
        srt = pos + up16((size_t)R * 2);
        red = srt + up16((size_t)(R + 1) * 4);
        wsum = red + 32 * 4;
        rp = wsum + up16((kTermThreads / 32) * 4);
        total = rp + up16((size_t)n_deck * kRowStride * 4);
    }
};

// work_rec2 entry of a TERMINAL work-list entry: {node, board id, pot (float bits), kind | (acted_last & 0xff) << 8}.
// Fold rows come first among the terminals of a level and go to fold2_kernel; this kernel is launched on the showdown
// rows after them, so its fold branch is never taken.  The branch stays: without it nvcc schedules the showdown path
// differently, and the kernel measured 434 instead of 419 us per launch (hulh, 12 turns, H100 80GB HBM3 at 400 W).
template <bool WITH_BR>
__global__ void __launch_bounds__(kTermThreads) terminal2_kernel_v3(const Ctx2 c) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int R = c.T.n_range, ld = c.T.ld, n_deck = c.T.n_deck;
    const TermSmem L(R, n_deck);
    uint4* rec_s = reinterpret_cast<uint4*>(smem_raw + L.rec);     // [R]   packed hand records of the board
    float* ro = reinterpret_cast<float*>(smem_raw + L.ro);         // [R]   opponent reach row
    int16_t* roword_s = reinterpret_cast<int16_t*>(smem_raw + L.roword);  // [n_deck][n_deck - 1] card rows in strength order
    int16_t* pos_s = reinterpret_cast<int16_t*>(smem_raw + L.pos); // [R]   position in strength order
    float* srt = reinterpret_cast<float*>(smem_raw + L.srt);       // [R + 1]
    float* red = reinterpret_cast<float*>(smem_raw + L.red);       // [32]
    float* wsum = reinterpret_cast<float*>(smem_raw + L.wsum);     // [kTermThreads / 32]
    float* rp = reinterpret_cast<float*>(smem_raw + L.rp);         // [n_deck][kRowStride]
    const int4 w = reinterpret_cast<const int4*>(c.T.work_rec2)[c.lo + blockIdx.x];
    const int n = w.x, b = w.y, kind = w.w & 0xff, acted_last = (w.w >> 8) & 0xff;
    const bool fold = kind == PRL_KIND_FOLD;
    const int qj = threadIdx.x & 3;
    const size_t N = (size_t)c.T.n_nodes;
    const float scale = c.T.eq_const * __int_as_float(w.z) * 0.5f;
    const int row_len = n_deck - 1;
    if (!fold) {  // the board's tables do not depend on the seat: requested once, consumed after the first wait
        const uint4* rec_g = reinterpret_cast<const uint4*>(c.T.board_hand_rec) + (size_t)b * R;
        for (int h = threadIdx.x; h < R; h += blockDim.x) cp_async16(rec_s + h, rec_g + h);
        const int32_t* ro_g32 = reinterpret_cast<const int32_t*>(c.T.board_row_order + (size_t)b * n_deck * row_len);
        for (int i = threadIdx.x; i < n_deck * row_len / 2; i += blockDim.x)
            cp_async4(reinterpret_cast<int32_t*>(roword_s) + i, ro_g32 + i);
        const int32_t* pos_g32 = reinterpret_cast<const int32_t*>(c.T.board_pos + (size_t)b * R);
        for (int i = threadIdx.x; i < R / 2; i += blockDim.x) cp_async4(reinterpret_cast<int32_t*>(pos_s) + i, pos_g32 + i);
    }
#pragma unroll 1
    for (int p = 0; p < 2; ++p) {
        if (!(c.mask & (1 << p))) continue;
        const float* ro_g = c.B.reach + ((size_t)(1 - p) * N + n) * ld;
        float* ev_p = c.B.ev + ((size_t)p * N + n) * ld;
        float* evbr_p = WITH_BR ? c.B.ev_br + ((size_t)p * N + n) * ld : nullptr;
        __syncthreads();  // shared arrays are reused by the second seat
        if (fold) {  // not reached (see above)
            float part = 0.0f;
            for (int h = threadIdx.x; h < R; h += blockDim.x) {
                const float r = ro_g[h];
                ro[h] = r;
                part += r;
            }
            const float T = block_sum(part, red);  // includes the barrier that publishes ro[]
            for (int base = 0; base < n_deck; base += blockDim.x >> 2) {
                const int cc = base + (threadIdx.x >> 2);
                float run = 0.0f;
                if (cc < n_deck) {
                    for (int i = 0; i < kSeg52; ++i) {
                        const int idx = qj * kSeg52 + i;
                        if (idx < row_len) run += ro[pair_index(cc, idx + (idx >= cc), n_deck)];
                    }
                }
                run += __shfl_xor_sync(0xffffffffu, run, 1);
                run += __shfl_xor_sync(0xffffffffu, run, 2);
                if (cc < n_deck && qj == 0) rp[cc] = run;
            }
            __syncthreads();
            const float sgn = (acted_last == p) ? -scale : scale;
            const unsigned long long bmask = (b >= 0) ? c.T.board_mask[b] : 0ull;
            for (int h = threadIdx.x; h < R; h += blockDim.x) {
                const int c1 = c.T.hand_cards[2 * h], c2 = c.T.hand_cards[2 * h + 1];
                float v = (T - rp[c1] - rp[c2] + ro[h]) * sgn;
                if (((bmask >> c1) | (bmask >> c2)) & 1ull) v = 0.0f;
                ev_p[h] = v;
                if (WITH_BR) evbr_p[h] = v;
            }
            continue;
        }
        // the reach row joins the outstanding table copies; 16-byte chunks, 4-byte tail
        for (int i = threadIdx.x; i < R / 4; i += blockDim.x) cp_async16(ro + 4 * i, ro_g + 4 * i);
        for (int h = (R & ~3) + threadIdx.x; h < R; h += blockDim.x) cp_async4(ro + h, ro_g + h);
        for (int i = threadIdx.x; i <= R; i += blockDim.x) srt[i] = 0.0f;
        cp_async_wait_all();
        __syncthreads();
        // 1. scatter into strength order (pos is a permutation of the live hands: deterministic)
        for (int h = threadIdx.x; h < R; h += blockDim.x) {
            const int ps = pos_s[h];
            if (ps >= 0) srt[ps] = ro[h];
        }
        card_row_prefix<kSeg52>(rp, ro, roword_s, n_deck, kSeg52);  // reads ro[] only: no barrier needed after the scatter yet
        __syncthreads();  // srt[] scattered
        centred_scan(srt, wsum, R);
        showdown_from_records<WITH_BR>(rec_s, srt, rp, scale, R, ev_p, evbr_p);
    }
}

// Fold rows on their own (generation 4): no board tables, 7 KB of shared memory.  The per-card sums use the
// lexicographic layout of the range itself - hands (c, x > c) are the contiguous segment ro[base(c) ..], hands (r < c, c)
// sit at ro[base(r) + c - r - 1] - instead of index arithmetic per element: thread (card c, quarter j) adds every fourth
// term of both parts in a fixed order, four partials per card are combined in a fixed order.
constexpr int kFoldThreads = 256;  // 64 card slots x 4 quarters
inline size_t fold_smem(const prl_tree_t& T) { return sizeof(float) * ((size_t)((T.n_range + 3) & ~3) + 256 + 64 + 32 + 64); }

template <bool WITH_BR>
__global__ void __launch_bounds__(kFoldThreads) fold2_kernel(const Ctx2 c) {
    extern __shared__ float fsm[];
    const int R = c.T.n_range, ld = c.T.ld, n_deck = c.T.n_deck;
    float* ro = fsm;                       // [R]  opponent reach row
    float* part = ro + ((R + 3) & ~3);     // [4][64] partial per-card sums
    float* cs = part + 256;                // [64] per-card sums; +inf for cards on the board
    float* red = cs + 64;                  // [32]
    int* base_s = reinterpret_cast<int*>(red + 32);  // [64] first range index of the hands (c, x > c)
    const int4 w = reinterpret_cast<const int4*>(c.T.work_rec2)[c.lo + blockIdx.x];
    const int n = w.x, b = w.y, acted_last = (w.w >> 8) & 0xff;
    const size_t N = (size_t)c.T.n_nodes;
    const float scale = c.T.eq_const * __int_as_float(w.z) * 0.5f;
    const unsigned long long bmask = (b >= 0) ? c.T.board_mask[b] : 0ull;
    const int cc = threadIdx.x & 63, j = threadIdx.x >> 6;
    if (threadIdx.x < 64) base_s[threadIdx.x] = threadIdx.x * (2 * n_deck - 1 - threadIdx.x) / 2;
    const unsigned short* hc = reinterpret_cast<const unsigned short*>(c.T.hand_cards);
#pragma unroll 1
    for (int p = 0; p < 2; ++p) {
        if (!(c.mask & (1 << p))) continue;
        const float* ro_g = c.B.reach + ((size_t)(1 - p) * N + n) * ld;
        float* ev_p = c.B.ev + ((size_t)p * N + n) * ld;
        float* evbr_p = WITH_BR ? c.B.ev_br + ((size_t)p * N + n) * ld : nullptr;
        __syncthreads();  // shared arrays are reused by the second seat
        float psum = 0.0f;
        for (int h = threadIdx.x; h < R; h += blockDim.x) {
            const float r = ro_g[h];
            ro[h] = r;
            psum += r;
        }
        const float T = block_sum(psum, red);  // includes the barriers that publish ro[] and base_s[]
        float acc = 0.0f;
        if (cc < n_deck) {
            for (int r = j; r < cc; r += 4) acc += ro[base_s[r] + cc - r - 1];          // hands (r, cc), r < cc
            const int b0 = base_s[cc];
            for (int k = j; k < n_deck - 1 - cc; k += 4) acc += ro[b0 + k];             // hands (cc, cc + 1 + k)
        }
        part[j * 64 + cc] = acc;
        __syncthreads();
        if (threadIdx.x < 64) {
            const float v = (part[threadIdx.x] + part[64 + threadIdx.x]) + (part[128 + threadIdx.x] + part[192 + threadIdx.x]);
            cs[threadIdx.x] = ((bmask >> threadIdx.x) & 1ull) ? __int_as_float(0x7f800000) : v;
        }
        __syncthreads();
        const float sgn = (acted_last == p) ? -scale : scale;
        for (int h = threadIdx.x; h < R; h += blockDim.x) {
            const unsigned cards = hc[h];  // {c1, c2} as two bytes
            const float e = T - cs[cards & 0xffu] - cs[cards >> 8] + ro[h];  // -inf for a hand holding a board card
            const float v = (e > -3.0e38f) ? e * sgn : 0.0f;
            ev_p[h] = v;
            if (WITH_BR) evbr_p[h] = v;
        }
    }
}

// ---- strength-order tables of complete boards: gs = # live hands strictly weaker, ge = # live hands weaker or equal,
//      pos = unique position in strength order (ties by hand index); -1 for hands blocked by the board
__global__ void __launch_bounds__(256) board_order_kernel(const int32_t* __restrict__ ranks, int n_boards, int R,
                                                          int16_t* gs, int16_t* ge, int16_t* pos) {
    extern __shared__ int srk[];
    const int b = blockIdx.x;
    for (int h = threadIdx.x; h < R; h += blockDim.x) srk[h] = ranks[(size_t)b * R + h];
    __syncthreads();
    for (int h = threadIdx.x; h < R; h += blockDim.x) {
        const int r = srk[h];
        int lt = 0, le = 0, tie_before = 0;
        if (r >= 0) {
            for (int j = 0; j < R; ++j) {
                const int q = srk[j];
                if (q < 0) continue;
                lt += q < r;
                le += q <= r;
                tie_before += (q == r) && (j < h);
            }
        }
        gs[(size_t)b * R + h] = (int16_t)(r >= 0 ? lt : -1);
        ge[(size_t)b * R + h] = (int16_t)(r >= 0 ? le : -1);
        pos[(size_t)b * R + h] = (int16_t)(r >= 0 ? lt + tie_before : -1);
    }
}

// ---- card-row tables of complete boards: for every card c the live hands containing c in strength order
//      (row_order[b][c][i], -1 padded) and, per hand, how many hands of its two card rows are strictly weaker /
//      weaker-or-equal (row_pos[b][h] = {lt(c1), lt(c2), le(c1), le(c2)})
__global__ void __launch_bounds__(256) board_rows_kernel(const int16_t* __restrict__ gs, int n_boards, int R, int n_deck,
                                                         int16_t* row_order, uint8_t* row_pos) {
    extern __shared__ short sgs[];
    const int b = blockIdx.x;
    const int row_len = n_deck - 1;
    for (int h = threadIdx.x; h < R; h += blockDim.x) sgs[h] = gs[(size_t)b * R + h];
    for (int i = threadIdx.x; i < n_deck * row_len; i += blockDim.x) row_order[(size_t)b * n_deck * row_len + i] = -1;
    __syncthreads();
    for (int i = threadIdx.x; i < n_deck * row_len; i += blockDim.x) {
        const int cc = i / row_len, j = i % row_len;
        const int x = j + (j >= cc);
        const int h = pair_index(cc, x, n_deck);
        const int g = sgs[h];
        if (g < 0) continue;
        int lt = 0, le = 0, tie_before = 0;
        for (int j2 = 0; j2 < row_len; ++j2) {
            const int g2 = sgs[pair_index(cc, j2 + (j2 >= cc), n_deck)];
            if (g2 < 0) continue;
            lt += g2 < g;
            le += g2 <= g;
            tie_before += (g2 == g) && (j2 < j);
        }
        row_order[(size_t)b * n_deck * row_len + cc * row_len + lt + tie_before] = (int16_t)h;
        const int k = (cc == min(cc, x)) ? 0 : 1;  // is cc the first (smaller) or second card of the hand?
        row_pos[((size_t)b * R + h) * 4 + k] = (uint8_t)lt;
        row_pos[((size_t)b * R + h) * 4 + 2 + k] = (uint8_t)le;
    }
}

// root exploitability: sum_h reach[p][0][h] * (ev_br - ev)[p][0][h]  (ValueFiller.py:95-101), double accumulation
__global__ void root_exploitability2_kernel(prl_tree_t T, prl_buffers_t B, float* out) {
    __shared__ double red[256];
    const size_t N = (size_t)T.n_nodes;
    for (int p = 0; p < 2; ++p) {
        const float* ev = B.ev + (size_t)p * N * T.ld;
        const float* evbr = B.ev_br + (size_t)p * N * T.ld;
        const float* reach = B.reach + (size_t)p * N * T.ld;
        double s = 0.0;
        for (int h = threadIdx.x; h < T.n_range; h += blockDim.x) s += (double)reach[h] * ((double)evbr[h] - (double)ev[h]);
        red[threadIdx.x] = s;
        __syncthreads();
        for (int o = 128; o > 0; o >>= 1) {
            if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
            __syncthreads();
        }
        if (threadIdx.x == 0) out[p] = (float)red[0];
        __syncthreads();
    }
}

inline unsigned blocks_for(long long threads) { return (unsigned)((threads + kThreads - 1) / kThreads); }

int check_tree2(const prl_tree_t* t) {
    if (!t || !t->level_start || !t->order || !t->level_nonterm || !t->level_ndec)
        return prl::fail("prl(two-card): level_start / order / level_nonterm / level_ndec missing");
    if (!t->hand_cards || !t->board_mask || !t->board_prob || !t->board_mult || !t->board_row_order || !t->board_row_pos ||
        !t->board_complete)
        return prl::fail("prl(two-card): hand_cards / board tables missing");
    if (t->n_deck - 1 > 64 || t->n_deck - 1 >= kRowStride) return prl::fail("prl(two-card): deck too large for the card-row scans");
    if (t->n_sym > 1 && !t->sym_perm) return prl::fail("prl(two-card): sym_perm missing");
    if (t->ld % 4 || t->ld < t->n_range) return prl::fail("prl(two-card): ld must be a multiple of 4 (float4 rows) and >= n_range");
    return 0;
}

size_t term_smem(const prl_tree_t& T) {
    return sizeof(float) * ((size_t)2 * T.n_range + 1 + 64 + 32 + kTermThreads / 32 + 1 + (size_t)T.n_deck * kRowStride);
}

// threads of the one-CTA-per-node row kernels (0: range too wide, use the tiled v1 kernels)
inline int row_threads(const prl_tree_t& T) {
    const int t = (((T.n_range + 3) / 4) + 31) & ~31;
    return t <= kRowThreadsMax ? t : 0;
}

// one level of the reach sweep: c.lo / c.n set by the caller
void launch_reach_level(const Ctx2& c, bool update_avg, cudaStream_t s) {
    const prl_tree_t& T = c.T;
    const int rt = row_threads(T);
    const bool pred = update_avg && c.algo == PRL_ALGO_PCFR_PLUS;
    if (T.node_rec2 && rt) {
        if (pred) reach2_kernel_v2<true, true><<<c.n, rt, 0, s>>>(c);
        else if (update_avg) reach2_kernel_v2<true><<<c.n, rt, 0, s>>>(c);
        else reach2_kernel_v2<false><<<c.n, rt, 0, s>>>(c);
    } else {
        const dim3 g((unsigned)c.n, (unsigned)((T.n_range + 4 * kVecThreads - 1) / (4 * kVecThreads)));
        if (pred) reach2_kernel<true, true><<<g, kVecThreads, 0, s>>>(c);
        else if (update_avg) reach2_kernel<true><<<g, kVecThreads, 0, s>>>(c);
        else reach2_kernel<false><<<g, kVecThreads, 0, s>>>(c);
    }
    prl::count_launch();
}

void reach_sweep2(Ctx2 c, bool update_avg, cudaStream_t s) {
    const prl_tree_t& T = c.T;
    for (int d = 0; d < T.n_levels; ++d) {
        c.lo = (int)T.level_start[d];
        c.n = (int)(T.level_start[d + 1] - T.level_start[d]);
        if (c.n == 0) continue;
        launch_reach_level(c, update_avg, s);
    }
}

// levels d_hi .. d_lo (bottom-up).  chance_phase: 0 = whole levels; 1 = everything except the final stage of the chance
// reduction (the per-node sums W stay in the workspace, e.g. to be all-reduced across GPUs); 2 = only that final stage
int value_levels2(Ctx2 c, bool with_br, bool update, int d_hi, int d_lo, int chance_phase, cudaStream_t s) {
    const prl_tree_t& T = c.T;
    // the opt-in for > 48 KB of dynamic shared memory is a PER-DEVICE function attribute: (re)applied on every call
    const size_t tsm = term_smem(T);
    cudaFuncSetAttribute(terminal2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tsm);
    cudaFuncSetAttribute(terminal2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tsm);
    // terminal rows: fold rows and showdown rows in their own kernels (packed records, cp.async staging, 52-card decks); the
    // record-free kernel is the fallback for callers that pass NULL records or another deck size
    const bool packed = T.work_rec2 && T.board_hand_rec && !(T.n_range & 1) && T.level_nfold && T.n_deck <= 64 &&
                        ((T.n_deck - 1 + 3) >> 2) == kSeg52;
    const TermSmem tl(T.n_range, T.n_deck);
    cudaFuncSetAttribute(terminal2_kernel_v3<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tl.total);
    cudaFuncSetAttribute(terminal2_kernel_v3<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tl.total);
    int arr_mask = 0;
    for (int p = 0; p < 2; ++p)
        if (c.mask & (1 << p)) arr_mask |= (1 << (2 * p)) | (with_br ? (2 << (2 * p)) : 0);
    // all-in showdowns before the deal (last among the terminals of their level): their inputs - the opponent's reach rows -
    // are complete before the sweep starts, so all of them are evaluated up front by the dense tensor-core product
    if (T.level_nallin && chance_phase != 2) {
        int n_in_range = 0, first = 0;
        for (int d = 0; d < T.n_levels; ++d) {
            if (d >= d_lo && d <= d_hi) n_in_range += (int)T.level_nallin[d];
        }
        if (n_in_range > 0 && (!T.allin_tiles || !T.allin_partial || !T.allin_nodes || !T.allin_pot))
            return prl::fail("prl(two-card): all-in terminals need allin_nodes / allin_pot / allin_tiles / allin_partial");
        const size_t N = (size_t)T.n_nodes, ld = (size_t)T.ld;
        std::vector<int> todo;  // indices into allin_nodes of the nodes of the level range
        for (int d = 0; d < T.n_levels; ++d) {
            const int na = (int)T.level_nallin[d];
            if (d >= d_lo && d <= d_hi)
                for (int k = 0; k < na; ++k) todo.push_back(first + k);
            first += na;
        }
        std::vector<char> done(todo.size(), 0);
        for (size_t i0 = 0; i0 < todo.size(); ++i0) {  // one product per public board (nodes on a board share their tiles)
            if (done[i0]) continue;
            const void* tiles = T.allin_tiles[todo[i0]];
            std::vector<const float*> xr;
            std::vector<float*> yr, y2r;
            std::vector<float> sc;
            for (size_t i = i0; i < todo.size(); ++i) {
                if (done[i] || T.allin_tiles[todo[i]] != tiles) continue;
                done[i] = 1;
                const size_t node = (size_t)T.allin_nodes[todo[i]];
                for (int p = 0; p < 2; ++p) {
                    if (!(c.mask & (1 << p))) continue;
                    xr.push_back(c.B.reach + ((size_t)(1 - p) * N + node) * ld);
                    yr.push_back(c.B.ev + ((size_t)p * N + node) * ld);
                    y2r.push_back(with_br ? c.B.ev_br + ((size_t)p * N + node) * ld : nullptr);
                    sc.push_back(T.eq_const * T.allin_pot[todo[i]] * 0.5f);  // ValueFiller.py:160-175 with K, pot / 2
                }
            }
            if (xr.empty()) continue;
            if (int e = prl_allin_values(tiles, T.n_range, xr.data(), yr.data(), y2r.data(), sc.data(), (int)xr.size(),
                                         T.allin_partial, (prl_stream_t)s))
                return e;
        }
    }
    for (int d = d_hi; d >= d_lo; --d) {
        const int lo = (int)T.level_start[d], n_all = (int)(T.level_start[d + 1] - T.level_start[d]);
        const int n_dec = (int)T.level_ndec[d], n_nonterm = (int)T.level_nonterm[d];
        const int n_chance = n_nonterm - n_dec;
        const int n_term = n_all - n_nonterm - (T.level_nallin ? (int)T.level_nallin[d] : 0);  // fold + showdown rows
        if (n_term > 0 && chance_phase != 2) {
            c.lo = lo + n_nonterm;
            c.n = n_term;
            if (packed) {  // fold rows (first among the terminals of a level) and showdown rows launched apart
                const int n_fold = (int)T.level_nfold[d];
                if (n_fold > 0) {
                    c.n = n_fold;
                    if (with_br) fold2_kernel<true><<<n_fold, kFoldThreads, fold_smem(T), s>>>(c);
                    else fold2_kernel<false><<<n_fold, kFoldThreads, fold_smem(T), s>>>(c);
                    prl::count_launch();
                }
                if (n_term > n_fold) {
                    c.lo = lo + n_nonterm + n_fold;
                    c.n = n_term - n_fold;
                    if (with_br) terminal2_kernel_v3<true><<<c.n, kTermThreads, tl.total, s>>>(c);
                    else terminal2_kernel_v3<false><<<c.n, kTermThreads, tl.total, s>>>(c);
                    prl::count_launch();
                }
            } else {
                if (with_br) terminal2_kernel<true><<<n_term, kTermThreads, tsm, s>>>(c);
                else terminal2_kernel<false><<<n_term, kTermThreads, tsm, s>>>(c);
                prl::count_launch();
            }
        }
        if (n_dec > 0 && chance_phase != 2) {
            c.lo = lo;
            c.n = n_dec;
            const int rt = row_threads(T);
            const bool pred = update && c.algo == PRL_ALGO_PCFR_PLUS;
            if (T.work_rec2 && rt) {
                if (pred) value2_kernel_v2<false, true, true><<<n_dec, rt, 0, s>>>(c);
                else if (update) value2_kernel_v2<false, true><<<n_dec, rt, 0, s>>>(c);
                else if (with_br) value2_kernel_v2<true, false><<<n_dec, rt, 0, s>>>(c);
                else value2_kernel_v2<false, false><<<n_dec, rt, 0, s>>>(c);
            } else {
                const dim3 g((unsigned)n_dec, (unsigned)((T.n_range + 4 * kVecThreads - 1) / (4 * kVecThreads)));
                if (pred) value2_kernel<false, true, true><<<g, kVecThreads, 0, s>>>(c);
                else if (update) value2_kernel<false, true><<<g, kVecThreads, 0, s>>>(c);
                else if (with_br) value2_kernel<true, false><<<g, kVecThreads, 0, s>>>(c);
                else value2_kernel<false, false><<<g, kVecThreads, 0, s>>>(c);
            }
            prl::count_launch();
        }
        if (n_chance > 0) {
            c.lo = lo + n_dec;
            c.n = n_chance;
            ChanceGeom g;
            g.n_chance = n_chance;
            g.max_chunks = (T.max_chance_children + kChanceChunk - 1) / kChanceChunk;
            g.w_off = (size_t)4 * n_chance * g.max_chunks * T.ld;
            const size_t need = (g.w_off + (size_t)4 * n_chance * T.ld) * sizeof(float);
            if (!c.B.workspace || c.B.workspace_bytes < need) return prl::fail("prl(two-card): workspace too small for the chance reduction");
            if (chance_phase != 2) {
                chance_partial_kernel<<<n_chance * g.max_chunks, kThreads, 0, s>>>(c, g, arr_mask);
                chance_sum_kernel<<<blocks_for((long long)n_chance * T.ld), kThreads, 0, s>>>(c, g, arr_mask);
                prl::count_launch();
                prl::count_launch();
            }
            if (chance_phase != 1) {
                chance_final_kernel<<<blocks_for((long long)n_chance * T.ld), kThreads, 0, s>>>(c, g, arr_mask);
                prl::count_launch();
            }
        }
    }
    return 0;
}

int value_sweep2(Ctx2 c, bool with_br, bool update, cudaStream_t s) {
    return value_levels2(c, with_br, update, c.T.n_levels - 1, 0, 0, s);
}

}  // namespace

// entry points used by the dispatchers in cfr_levels.cu when tree->n_hole == 2
namespace prl2 {

int reach_pass(const prl_tree_t* tree, const prl_buffers_t* buf, int player_mask, const int* mode, cudaStream_t s) {
    if (int e = check_tree2(tree)) return e;
    Ctx2 c{*tree, *buf, 0, 0, player_mask, {mode[0], mode[1]}, 0, -1, 0, 0, 0.0f, 1.0f};
    reach_sweep2(c, false, s);
    return prl::check(cudaGetLastError(), "prl_reach_pass(two-card)");
}

int value_pass(const prl_tree_t* tree, const prl_buffers_t* buf, int player_mask, int with_br, const int* mode,
               cudaStream_t s) {
    if (int e = check_tree2(tree)) return e;
    Ctx2 c{*tree, *buf, 0, 0, player_mask, {mode[0], mode[1]}, 0, -1, 0, 0, 0.0f, 1.0f};
    if (int e = value_sweep2(c, with_br != 0, false, s)) return e;
    return prl::check(cudaGetLastError(), "prl_value_pass(two-card)");
}

int root_exploitability(const prl_tree_t* tree, const prl_buffers_t* buf, float* out, cudaStream_t s) {
    root_exploitability2_kernel<<<1, 256, 0, s>>>(*tree, *buf, out);
    prl::count_launch();
    return prl::check(cudaGetLastError(), "prl_root_exploitability(two-card)");
}

int cfr_sweep(const prl_tree_t* tree, const prl_buffers_t* buf, int algo, int p, int iter, int delay, const int* mode,
              int which, cudaStream_t s) {
    if (int e = check_tree2(tree)) return e;
    if (p < 0 || p > 1) return prl::fail("prl_cfr_sweep(two-card): bad p");
    if (int e = prl::check_algo(algo, buf->dcfr, true, "prl_cfr_sweep(two-card)")) return e;
    Ctx2 c{*tree, *buf, 0, 0, 1 << p, {mode[0], mode[1]}, algo, p, iter, delay, 0.0f, 1.0f};
    prl::cfrp_weights(iter, delay, &c.m_old, &c.m_new);
    if (which & 1)
        if (int e = value_sweep2(c, false, true, s)) return e;
    if (which & 2) {
        c.mode[p] = PRL_STRAT_F32;
        reach_sweep2(c, true, s);
    }
    return prl::check(cudaGetLastError(), "prl_cfr_sweep(two-card)");
}

}  // namespace prl2

// Bottom-up value sweep over tree levels level_hi .. level_lo only (two-card trees), with the chance reduction optionally
// split around an external all-reduce of the per-chance-node sums (see include/pokerrl_b200.h).
extern "C" int prl_value_levels(const prl_tree_t* tree, const prl_buffers_t* buf, int player_mask, int with_br, int algo,
                                int upd_p, int iter, int delay, const int* strat_mode, int level_hi, int level_lo,
                                int chance_phase, prl_stream_t stream) {
    if (!tree || tree->n_hole != 2) return prl::fail("prl_value_levels: two-card trees only");
    if (int e = check_tree2(tree)) return e;
    if (level_hi >= tree->n_levels || level_lo < 0 || level_hi < level_lo) return prl::fail("prl_value_levels: bad level range");
    if (with_br && algo >= 0) return prl::fail("prl_value_levels: the update sweep does not compute best responses");
    if (algo >= 0)
        if (int e = prl::check_algo(algo, buf->dcfr, true, "prl_value_levels")) return e;
    Ctx2 c{*tree, *buf, 0, 0, player_mask, {strat_mode[0], strat_mode[1]}, algo < 0 ? 0 : algo, algo < 0 ? -1 : upd_p, iter, delay, 0.0f, 1.0f};
    if (int e = value_levels2(c, with_br != 0, algo >= 0, level_hi, level_lo, chance_phase, (cudaStream_t)stream)) return e;
    return prl::check(cudaGetLastError(), "prl_value_levels");
}

// Top-down reach sweep of seat p with the average-strategy update of p's nodes (second half of prl_cfr_half_iteration).
extern "C" int prl_reach_update(const prl_tree_t* tree, const prl_buffers_t* buf, int algo, int p, int iter, int delay,
                                prl_stream_t stream) {
    if (!tree || tree->n_hole != 2) return prl::fail("prl_reach_update: two-card trees only");
    const int mode[2] = {PRL_STRAT_F32, PRL_STRAT_F32};
    return prl2::cfr_sweep(tree, buf, algo, p, iter, delay, mode, 2, (cudaStream_t)stream);
}

extern "C" int prl_board_order_tables(const int32_t* ranks, int n_boards, int n_range, int n_deck, int16_t* gs,
                                      int16_t* ge, int16_t* pos, int16_t* row_order, uint8_t* row_pos,
                                      prl_stream_t stream) {
    if (n_boards <= 0) return 0;
    board_order_kernel<<<n_boards, 256, sizeof(int) * n_range, (cudaStream_t)stream>>>(ranks, n_boards, n_range, gs, ge, pos);
    board_rows_kernel<<<n_boards, 256, sizeof(short) * n_range, (cudaStream_t)stream>>>(gs, n_boards, n_range, n_deck,
                                                                                      row_order, row_pos);
    prl::count_launch();
    prl::count_launch();
    return prl::check(cudaGetLastError(), "prl_board_order_tables");
}

// Top-down reach sweep restricted to tree levels level_lo..level_hi (the rows of level_lo - 1 must be current); with
// algo >= 0 it also applies the average-strategy update of seat p's nodes whose children lie in the range.
extern "C" int prl_reach_levels(const prl_tree_t* tree, const prl_buffers_t* buf, int player_mask, int algo, int upd_p, int iter,
                                int delay, const int* strat_mode, int level_lo, int level_hi, prl_stream_t stream) {
    if (!tree || tree->n_hole != 2) return prl::fail("prl_reach_levels: two-card trees only");
    if (int e = check_tree2(tree)) return e;
    if (level_lo < 0 || level_hi >= tree->n_levels || level_lo > level_hi) return prl::fail("prl_reach_levels: bad level range");
    if (algo >= 0)
        if (int e = prl::check_algo(algo, buf->dcfr, true, "prl_reach_levels")) return e;
    Ctx2 c{*tree, *buf, 0, 0, player_mask, {strat_mode[0], strat_mode[1]}, algo < 0 ? 0 : algo, algo < 0 ? -1 : upd_p, iter, delay, 0.0f, 1.0f};
    prl::cfrp_weights(iter, delay, &c.m_old, &c.m_new);
    const prl_tree_t& T = c.T;
    for (int d = level_lo; d <= level_hi; ++d) {
        c.lo = (int)T.level_start[d];
        c.n = (int)(T.level_start[d + 1] - T.level_start[d]);
        if (c.n == 0) continue;
        launch_reach_level(c, algo >= 0, (cudaStream_t)stream);
    }
    return prl::check(cudaGetLastError(), "prl_reach_levels");
}

// Batched StrategyFiller._fill_with_agent_policy (StrategyFiller.py:88-116): the agent answered for ALL decision nodes at
// once - probs[d][h][a] over the env's N_ACTIONS - and table row `slot` (child of decision node dec_of_slot[slot], reached by
// discrete action action_of_slot[slot]) takes probs[dec][.][action] (the reference's `agent_strat[:, allowed_actions]`, :111).
namespace {
__global__ void gather_agent_policy_kernel(const float* __restrict__ probs, int n_actions, const int32_t* __restrict__ dec_of_slot,
                                           const int32_t* __restrict__ action_of_slot, int n_range, int ld, float* __restrict__ out) {
    const int slot = blockIdx.x;
    const float* src = probs + (size_t)dec_of_slot[slot] * n_range * n_actions + action_of_slot[slot];
    float* dst = out + (size_t)slot * ld;
    for (int h = threadIdx.x; h < ld; h += blockDim.x) dst[h] = (h < n_range) ? src[(size_t)h * n_actions] : 0.0f;
}
}  // namespace

extern "C" int prl_gather_agent_policy(const float* probs, int n_actions, const int32_t* dec_of_slot, const int32_t* action_of_slot,
                                       int n_slots, int n_range, int ld, float* out, prl_stream_t stream) {
    if (n_slots <= 0) return 0;
    if (!probs || !dec_of_slot || !action_of_slot || !out || ld < n_range) return prl::fail("prl_gather_agent_policy: bad arguments");
    gather_agent_policy_kernel<<<n_slots, 256, 0, (cudaStream_t)stream>>>(probs, n_actions, dec_of_slot, action_of_slot, n_range, ld, out);
    prl::count_launch();
    return prl::check(cudaGetLastError(), "prl_gather_agent_policy");
}
