// Level-synchronous public-tree sweeps for tabular CFR / best response, one-hole-card games (sm_90a).
//
// Mapping: ONE LANE PER (NODE, HAND); a warp holds 32 / R whole nodes (5 for Leduc's R = 6, 1 for BigLeduc's R = 24),
// taken from a per-level work list sorted by node kind (no divergence).  Nodes of one depth are contiguous, children of
// a node are contiguous and children groups of adjacent nodes are adjacent, so a warp reads / writes contiguous runs of
// rows.  All per-node structure comes from ONE 16-byte record (`prl_tree_t.meta`, LDG.128) so that the dependent chain
// of a lane is: work-list entry -> record -> {children / table elements, requested together} -> stores; rows of a node
// are exchanged between its lanes with group-masked warp shuffles.
//
// These sweeps are HBM/L2-bound vector work (no GEMM shape anywhere): what matters is coalescing, memory-level
// parallelism and launch count - not tensor cores.
//
// Arithmetic contract: every expression is evaluated in the reference's dtype and operation order
// (oracle/cfr_numpy.py and oracle/cfr_oracle.c are pinned bit-for-bit against the reference); a sum over a row of hands
// follows np.sum, which is pairwise from 8 elements on (numpy_sum).  This translation unit is compiled with
// -fmad=false so that no multiply-add is contracted; the reference (numpy) never fuses.
//
// Reference statements restated here (paths under PokerRL/):
//   reach pass      game/_/tree/_/StrategyFiller.py:118-146, 148-169
//   value pass      game/_/tree/_/ValueFiller.py:21-101, terminals :103-175
//   regrets         cfr/_CFRBase.py:146-185, cfr/CFRPlus.py:37-41, cfr/LinearCFR.py:27-31, cfr/VanillaCFR.py:26-30
//   regret matching cfr/CFRPlus.py:43-63, cfr/LinearCFR.py:33-51, cfr/VanillaCFR.py:32-52
//   averaging       cfr/CFRPlus.py:65-87, cfr/LinearCFR.py:53-76, cfr/VanillaCFR.py:54-77
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdlib.h>
#include <stdint.h>

#include "pokerrl_b200.h"
#include "prl_common.cuh"

namespace cg = cooperative_groups;

// two-hole-card sweeps (cfr_twocard.cu)
namespace prl2 {
int reach_pass(const prl_tree_t*, const prl_buffers_t*, int player_mask, const int* mode, cudaStream_t);
int value_pass(const prl_tree_t*, const prl_buffers_t*, int player_mask, int with_br, const int* mode, cudaStream_t);
int root_exploitability(const prl_tree_t*, const prl_buffers_t*, float* out, cudaStream_t);
int cfr_sweep(const prl_tree_t*, const prl_buffers_t*, int algo, int p, int iter, int delay, const int* mode, int which,
              cudaStream_t);
}  // namespace prl2

namespace {

constexpr int kThreads = 128;
constexpr int kChunk = 4;  // children whose rows are loaded together before use
constexpr int kPThreads = 512;  // persistent kernels: ONE 512-thread block per SM keeps the grid barrier small

struct Ctx {
    prl_tree_t T;
    prl_buffers_t B;
    int lo, hi;       // node range of this level
    int mask;         // seats to process
    int mode[2];      // strategy source per seat
    int algo, upd_p, iter, delay, avg_f64;  // CFR update parameters
};

// ---- packed node record (see prl_pack_node_meta) ----------------------------------------------------------------
struct Meta {
    int first_child, first_slot;
    float pot;
    int kind, acted_last, board, n_children;
};

__device__ __forceinline__ Meta load_meta(const prl_tree_t& T, int n) {
    const int4 q = __ldg(reinterpret_cast<const int4*>(T.meta) + n);
    Meta m;
    m.first_child = q.x;
    m.first_slot = q.y;
    m.pot = __int_as_float(q.z);
    const unsigned w = (unsigned)q.w;
    m.kind = w & 0xF;
    m.acted_last = (int)((w >> 4) & 0x3) - 2;
    m.board = (int)((w >> 8) & 0xFF) - 1;
    m.n_children = (int)(w >> 16);
    return m;
}

__global__ void pack_meta_kernel(prl_tree_t T, int4* out) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= T.n_nodes) return;
    const int fc = T.first_child[n];
    const int k = T.kind[n];
    int4 q;
    q.x = fc;
    q.y = (k <= PRL_KIND_P1 && fc >= 0) ? T.slot[fc] : -1;
    q.z = __float_as_int(T.pot[n]);
    const unsigned nc = (unsigned)T.n_children[n];
    q.w = (int)((unsigned)k | ((unsigned)(T.acted_last[n] + 2) << 4) | ((unsigned)(T.board[n] + 1) << 8) | (nc << 16));
    out[n] = q;
}

// ---- lane mapping -------------------------------------------------------------------------------------------------
// One LANE per (node, hand): a warp holds NPW = 32 / R whole nodes (5 for Leduc's R = 6, lanes 30-31 idle; 1 for R = 24).
// All per-lane state is scalar, the dependent chain of a lane is  work-list entry -> node record -> {children /
// table elements, all issued together} -> stores, and the rows of a node are exchanged with group-masked shuffles.
template <int R>
struct LaneMap {
    static constexpr int NPW = 32 / R;
    int g, h, base;
    unsigned gmask;
    __device__ __forceinline__ LaneMap() {
        const int lane = threadIdx.x & 31;
        g = lane / R;
        h = lane - g * R;
        base = g * R;
        gmask = ((R >= 32) ? 0xffffffffu : ((1u << R) - 1u)) << base;
    }
};

__host__ __device__ __forceinline__ int groups_of(int nodes, int npw) { return (nodes + npw - 1) / npw; }

__device__ __forceinline__ bool mode_is_f32(int m) { return m == PRL_STRAT_F32 || m == PRL_STRAT_AVG_F32; }

// strategy probability of child k (row fs + k) for hand h in double, for the float64 sources
__device__ __forceinline__ double strat_f64(const Ctx& c, int m, int fs, int k, int A, int h) {
    const int ld = c.T.ld;
    if (m == PRL_STRAT_UNIFORM64) return 1.0 / (double)A;  // StrategyFiller.py:61-62
    if (m == PRL_STRAT_AVG_F64) return ((const double*)c.B.avg)[(size_t)(fs + k) * ld + h];
    // PRL_STRAT_AVG_SUM: float sums / float division, promoted to double (LinearCFR.py:64-71)
    const float* tab = (const float*)c.B.avg;
    float tot = tab[(size_t)fs * ld + h];
    for (int j = 1; j < A; ++j) tot = tot + tab[(size_t)(fs + j) * ld + h];
    if (tot == 0.0f) return 1.0 / (double)A;
    return (double)(tab[(size_t)(fs + k) * ld + h] / tot);
}

// float sum of x(0) .. x(n - 1) in numpy's order (np.sum of a float32 row: pairwise_sum in
// numpy/_core/src/umath/loops_utils.h.src, restated in oracle/pairwise_sum.py), for 1 <= n <= 128 and n <= NMAX.
// Fewer than 8 elements are added in order.  From 8 on, 8 interleaved partial sums r[j] = x(j) + x(j + 8) + ... run
// over the first n - n % 8 elements and are combined as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)); the last
// n % 8 elements follow in order.  numpy also adds the total to the identity +0.0, which only turns a total of -0.0
// into +0.0; that add is left out.  With NMAX < 8 (Leduc's rows of 6) only the sequential loop is compiled.
template <int NMAX, class F>
__device__ __forceinline__ float numpy_sum(const int n, F x) {
    if constexpr (NMAX >= 8) {
        if (n >= 8) {
            float r[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) r[j] = x(j);
            int i = 8;
            for (; i < n - n % 8; i += 8) {
#pragma unroll
                for (int j = 0; j < 8; ++j) r[j] = r[j] + x(i + j);
            }
            float s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
            for (; i < n; ++i) s = s + x(i);
            return s;
        }
    }
    float s = 0.0f;
    for (int i = 0; i < n; ++i) {
        const float e = x(i);
        s = (i == 0) ? e : s + e;
    }
    return s;
}

// hand rank of card h on board card b (game_rules.py:68-75); NS = N_SUITS (compile time)
template <int NS>
__device__ __forceinline__ int card_rank(int h, int b, int pair_bonus) {
    const int r = h / NS;
    return (b / NS == r) ? pair_bonus + r : r;
}

// ------------------------------------------------------------------------------------------------ reach (top-down)
// Lane = (parent node of level d, hand); writes element h of the reach rows of the children (level d+1).
template <int R, bool UPDATE_AVG>
__device__ __forceinline__ void reach_group(const Ctx& c, const int lo, const int hi, const int grp) {
    const LaneMap<R> L;
    const int t = lo + grp * LaneMap<R>::NPW + L.g;
    if (L.g >= LaneMap<R>::NPW || t >= hi) return;
    const int h = L.h;
    const int n = __ldg(c.T.order + t);
    const Meta m = load_meta(c.T, n);
    const size_t N = (size_t)c.T.n_nodes;
    const int ld = c.T.ld;
    const int A = m.n_children, fc = m.first_child;
#pragma unroll 1
    for (int q = 0; q < 2; ++q) {
        if (!(c.mask & (1 << q))) continue;
        float* reach_q = c.B.reach + (size_t)q * N * ld;
        float r;
        if (n == 0) {  // PublicTree.py:122-124
            r = (float)(1.0 / (double)R);
            reach_q[h] = r;
        } else {
            if (fc < 0) continue;
            r = reach_q[(size_t)n * ld + h];
        }
        if (fc < 0) continue;
        float* out = reach_q + (size_t)fc * ld + h;
        if (m.kind == PRL_KIND_CHANCE) {  // StrategyFiller.py:137-140, 159-166 (child k deals card k)
            const float cp = (float)(1.0 / (double)(c.T.n_deck - 2));
            for (int k = 0; k < A; ++k) out[(size_t)k * ld] = r * ((h == k) ? 0.0f : cp);
        } else if (m.kind == q) {  // StrategyFiller.py:129-134
            const int md = c.mode[q];
            const int fs = m.first_slot;
            if (mode_is_f32(md)) {
                const float* tab = ((md == PRL_STRAT_F32) ? c.B.strat : (const float*)c.B.avg) + (size_t)fs * ld + h;
                const bool upd = UPDATE_AVG && q == c.upd_p;
                double m_old = 0.0, m_new = 1.0;
                if (upd && c.algo == PRL_ALGO_CFR_PLUS) {  // CFRPlus.py:68-73
                    const long long cw = ((long long)c.iter * (c.iter + 1) - (long long)c.delay * (c.delay + 1)) / 2;
                    const long long nw = (long long)c.iter - c.delay + 1;
                    m_old = (double)cw / (double)(cw + nw);
                    m_new = (double)nw / (double)(cw + nw);
                }
                const bool avg_f32 = upd && !(c.algo == PRL_ALGO_CFR_PLUS && (c.avg_f64 || c.iter < c.delay));
                const bool avg_f64 = upd && c.algo == PRL_ALGO_CFR_PLUS && c.avg_f64 && c.iter >= c.delay;
                float* avf = (float*)c.B.avg + (size_t)fs * ld + h;
                double* avd = (double*)c.B.avg + (size_t)fs * ld + h;
                const float w = (float)(c.iter + 1);
                for (int k0 = 0; k0 < A; k0 += kChunk) {  // loads of a chunk first, then the stores
                    float s[kChunk], av[kChunk];
                    double ad[kChunk];
#pragma unroll
                    for (int j = 0; j < kChunk; ++j) {
                        if (k0 + j < A) {
                            s[j] = tab[(size_t)(k0 + j) * ld];
                            if (avg_f32) av[j] = avf[(size_t)(k0 + j) * ld];
                            if (avg_f64) ad[j] = avd[(size_t)(k0 + j) * ld];
                        }
                    }
#pragma unroll
                    for (int j = 0; j < kChunk; ++j) {
                        if (k0 + j < A) {
                            const float x = s[j] * r;
                            out[(size_t)(k0 + j) * ld] = x;
                            if (avg_f64) {
                                avd[(size_t)(k0 + j) * ld] = m_old * ad[j] + m_new * (double)s[j];
                            } else if (avg_f32) {
                                float a;
                                if (c.algo == PRL_ALGO_CFR_PLUS) a = (float)m_old * av[j] + (float)m_new * s[j];
                                else if (c.algo == PRL_ALGO_LINEAR) a = av[j] + x * w;  // LinearCFR.py:56-61
                                else a = av[j] + x;                                      // VanillaCFR.py:57-62
                                avf[(size_t)(k0 + j) * ld] = a;
                            }
                        }
                    }
                }
            } else {
                for (int k = 0; k < A; ++k) out[(size_t)k * ld] = (float)(strat_f64(c, md, fs, k, A, h) * (double)r);
            }
        } else {  // the other seat acts: reach of q is copied down
            for (int k = 0; k < A; ++k) out[(size_t)k * ld] = r;
        }
    }
}

// ------------------------------------------------------------------------------------------------ terminals
// equity of hand h at a showdown on board card b against the opponent row ro[] (ValueFiller.py:140-155): sequential
// float += / -= over opponent hands in ascending order
template <int R, int NS>
__device__ __forceinline__ float showdown_equity(const float (&ro)[R], int h, int b, int pair_bonus) {
    const int rh = card_rank<NS>(h, b, pair_bonus);
    float e = 0.0f;
#pragma unroll
    for (int j = 0; j < R; ++j) {
        const int rj = card_rank<NS>(j, b, pair_bonus);
        const bool live = (j != h) && (h != b) && (j != b);
        if (live && rh > rj) e = e + ro[j];
        else if (live && rh < rj) e = e - ro[j];
    }
    return e;
}

template <int R, int NS>
__device__ __forceinline__ float terminal_value(const Ctx& c, const Meta& m, int n, int p, const LaneMap<R>& L) {
    const int h = L.h;
    const float mine = c.B.reach[((size_t)(1 - p) * c.T.n_nodes + n) * c.T.ld + h];  // opponent reach of MY hand index
    float ro[R];  // the whole opponent row, gathered from the lanes of this node
#pragma unroll
    for (int j = 0; j < R; ++j) ro[j] = __shfl_sync(L.gmask, mine, L.base + j);
    const float K = (float)((double)c.T.n_deck / (double)(c.T.n_deck - 1));  // ValueFiller.py:19
    float eq;
    if (m.kind == PRL_KIND_FOLD) {  // ValueFiller.py:103-125 (np.sum over the opponent's hands)
        const float s = numpy_sum<R>(R, [&](int j) { return ro[j]; });
        eq = s - mine;
        if (m.acted_last == p) eq = -eq;
        eq = eq * K;
    } else if (m.kind == PRL_KIND_SHOWDOWN) {  // ValueFiller.py:127-158
        eq = showdown_equity<R, NS>(ro, h, m.board, c.T.pair_bonus) * K;
    } else {  // all-in before the board card: ValueFiller.py:160-175
        eq = 0.0f;
        for (int bb = 0; bb < c.T.n_deck; ++bb) eq = eq + showdown_equity<R, NS>(ro, h, bb, c.T.pair_bonus) * K;
        eq = eq / (float)(c.T.n_deck - 2);
    }
    if (h == m.board) eq = 0.0f;  // ValueFiller.py:57-59
    return eq * m.pot / 2.0f;     // ValueFiller.py:61
}

// children elements combined in child order (sum, or max for the best response), loads issued chunk-wise up front
template <bool MAX>
__device__ __forceinline__ float fold_children(const float* __restrict__ col, int ld, int A) {
    float v = 0.0f;
    for (int k0 = 0; k0 < A; k0 += kChunk) {
        float e[kChunk];
#pragma unroll
        for (int j = 0; j < kChunk; ++j)
            if (k0 + j < A) e[j] = col[(size_t)(k0 + j) * ld];
#pragma unroll
        for (int j = 0; j < kChunk; ++j) {
            if (k0 + j < A) {
                if (k0 + j == 0) v = e[j];
                else v = MAX ? fmaxf(v, e[j]) : v + e[j];
            }
        }
    }
    return v;
}

__device__ __forceinline__ float regret_step(int algo, float d, float old, float w) {
    if (algo == PRL_ALGO_CFR_PLUS) return fmaxf(d + old, 0.0f);  // CFRPlus.py:37-41
    if (algo == PRL_ALGO_LINEAR) return w * d + old;             // LinearCFR.py:27-31
    return d + old;                                              // VanillaCFR.py:26-30
}

// Seat p acts at this node and is being updated, A children (compile time): node value with the current strategy,
// regret update (_CFRBase.py:146-185) and regret matching (CFRPlus.py:43-63 and siblings).  Everything the lane needs
// is requested before the first use; returns the node value.
template <int A>
__device__ __forceinline__ float update_own(const Ctx& c, int md, const float* __restrict__ ecol, int fs, int h) {
    const int ld = c.T.ld;
    float* rcol = c.B.regret + (size_t)fs * ld + h;
    float* scol = c.B.strat + (size_t)fs * ld + h;
    const bool f32 = mode_is_f32(md);
    const float* tab = ((md == PRL_STRAT_AVG_F32) ? (const float*)c.B.avg : c.B.strat) + (size_t)fs * ld + h;
    float e[A], rg[A], sg[A];
#pragma unroll
    for (int k = 0; k < A; ++k) {
        e[k] = ecol[k * ld];
        rg[k] = rcol[k * ld];
        sg[k] = f32 ? tab[k * ld] : 0.0f;
    }
    float v;
    if (f32) {
        v = sg[0] * e[0];
#pragma unroll
        for (int k = 1; k < A; ++k) v = v + sg[k] * e[k];
    } else {
        double acc = strat_f64(c, md, fs, 0, A, h) * (double)e[0];
#pragma unroll
        for (int k = 1; k < A; ++k) acc = acc + strat_f64(c, md, fs, k, A, h) * (double)e[k];
        v = (float)acc;
    }
    const float w = (float)(c.iter + 1);
    float ssum = 0.0f;
#pragma unroll
    for (int k = 0; k < A; ++k) {
        rg[k] = regret_step(c.algo, e[k] - v, rg[k], w);
        const float rp = fmaxf(rg[k], 0.0f);
        ssum = (k == 0) ? rp : ssum + rp;
    }
    const float uni = (float)(1.0 / (double)A);
    const float den = (ssum > 0.0f) ? ssum : 1.0f;  // keeps div.rn off its slow path when the positive mass is 0
#pragma unroll
    for (int k = 0; k < A; ++k) {
        rcol[k * ld] = rg[k];
        const float q = fmaxf(rg[k], 0.0f) / den;
        scol[k * ld] = (ssum > 0.0f) ? q : uni;
    }
    return v;
}

// ------------------------------------------------------------------------------------------------ value (bottom-up)
// Lane = (node of level d, hand); reads element h of its children's rows (level d+1).
template <int R, int NS, bool WITH_BR, bool UPDATE>
__device__ __forceinline__ void value_group(const Ctx& c, const int lo, const int hi, const int grp) {
    constexpr int kRegA = 8;  // children of an updated node kept in registers (wider nodes stream)
    const LaneMap<R> L;
    const int t = lo + grp * LaneMap<R>::NPW + L.g;
    if (L.g >= LaneMap<R>::NPW || t >= hi) return;
    const int h = L.h;
    const int n = __ldg(c.T.order + t);
    const Meta m = load_meta(c.T, n);
    const size_t N = (size_t)c.T.n_nodes;
    const int ld = c.T.ld;
    const int A = m.n_children, fc = m.first_child;
#pragma unroll 1
    for (int p = 0; p < 2; ++p) {
        if (!(c.mask & (1 << p))) continue;
        float* ev_p = c.B.ev + (size_t)p * N * ld;
        float* evbr_p = WITH_BR ? c.B.ev_br + (size_t)p * N * ld : nullptr;
        float v, vbr = 0.0f;
        if (m.kind >= PRL_KIND_FOLD) {
            v = terminal_value<R, NS>(c, m, n, p, L);
            vbr = v;
        } else if (m.kind == PRL_KIND_CHANCE || m.kind != p) {
            // chance node, or the other seat acts: plain sums over children (ValueFiller.py:76-78, 88-90)
            v = fold_children<false>(ev_p + (size_t)fc * ld + h, ld, A);
            if (WITH_BR) vbr = fold_children<false>(evbr_p + (size_t)fc * ld + h, ld, A);
        } else {
            // seat p acts here (ValueFiller.py:87, 91)
            const int fs = m.first_slot;
            const int md = c.mode[p];
            const float* ecol = ev_p + (size_t)fc * ld + h;
            if (WITH_BR) vbr = fold_children<true>(evbr_p + (size_t)fc * ld + h, ld, A);
            const bool upd = UPDATE && p == c.upd_p;
            if (upd && A <= kRegA) {
                // warps are uniform in A (work list sorted by kind, n_children): jump to the exactly-unrolled variant
                switch (A) {
                    case 1: v = update_own<1>(c, md, ecol, fs, h); break;
                    case 2: v = update_own<2>(c, md, ecol, fs, h); break;
                    case 3: v = update_own<3>(c, md, ecol, fs, h); break;
                    case 4: v = update_own<4>(c, md, ecol, fs, h); break;
                    case 5: v = update_own<5>(c, md, ecol, fs, h); break;
                    case 6: v = update_own<6>(c, md, ecol, fs, h); break;
                    case 7: v = update_own<7>(c, md, ecol, fs, h); break;
                    default: v = update_own<8>(c, md, ecol, fs, h); break;
                }
            } else {
                if (mode_is_f32(md)) {
                    const float* tab = ((md == PRL_STRAT_F32) ? c.B.strat : (const float*)c.B.avg) + (size_t)fs * ld + h;
                    v = 0.0f;
                    for (int k0 = 0; k0 < A; k0 += kChunk) {
                        float s[kChunk], e[kChunk];
#pragma unroll
                        for (int j = 0; j < kChunk; ++j) {
                            if (k0 + j < A) {
                                s[j] = tab[(size_t)(k0 + j) * ld];
                                e[j] = ecol[(size_t)(k0 + j) * ld];
                            }
                        }
#pragma unroll
                        for (int j = 0; j < kChunk; ++j)
                            if (k0 + j < A) v = (k0 + j == 0) ? s[j] * e[j] : v + s[j] * e[j];
                    }
                } else {
                    double acc = 0.0;
                    for (int k = 0; k < A; ++k) {
                        const double sk = strat_f64(c, md, fs, k, A, h);
                        acc = (k == 0) ? sk * (double)ecol[(size_t)k * ld] : acc + sk * (double)ecol[(size_t)k * ld];
                    }
                    v = (float)acc;
                }
                if (upd) {  // wide node: stream (regrets are recomputed in the second loop instead of re-read)
                    float* rcol = c.B.regret + (size_t)fs * ld + h;
                    float* scol = c.B.strat + (size_t)fs * ld + h;
                    const float w = (float)(c.iter + 1);
                    float ssum = 0.0f;
                    for (int k = 0; k < A; ++k) {
                        const float rp = fmaxf(regret_step(c.algo, ecol[(size_t)k * ld] - v, rcol[(size_t)k * ld], w), 0.0f);
                        ssum = (k == 0) ? rp : ssum + rp;
                    }
                    const float uni = (float)(1.0 / (double)A);
                    const float den = (ssum > 0.0f) ? ssum : 1.0f;
                    for (int k = 0; k < A; ++k) {
                        const float r = regret_step(c.algo, ecol[(size_t)k * ld] - v, rcol[(size_t)k * ld], w);
                        rcol[(size_t)k * ld] = r;
                        const float q = fmaxf(r, 0.0f) / den;
                        scol[(size_t)k * ld] = (ssum > 0.0f) ? q : uni;
                    }
                }
            }
        }
        ev_p[(size_t)n * ld + h] = v;
        if (WITH_BR) evbr_p[(size_t)n * ld + h] = vbr;
    }
}

// ---- one launch per level (any tree size): one warp per group of NPW nodes --------------------------------------------
template <int R, bool UPDATE_AVG>
__global__ void __launch_bounds__(kThreads) reach_level_kernel(const Ctx c) {
    const int grp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (grp < groups_of(c.hi - c.lo, LaneMap<R>::NPW)) reach_group<R, UPDATE_AVG>(c, c.lo, c.hi, grp);
}

template <int R, int NS, bool WITH_BR, bool UPDATE>
__global__ void __launch_bounds__(kThreads) value_level_kernel(const Ctx c) {
    const int grp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (grp < groups_of(c.hi - c.lo, LaneMap<R>::NPW)) value_group<R, NS, WITH_BR, UPDATE>(c, c.lo, c.hi, grp);
}

// ---- persistent cooperative kernels: whole sweeps / iterations in ONE launch, grid barrier between levels ------------
// (one launch instead of 4 x n_levels per iteration: no launch gaps, instruction cache stays warm, L1 is invalidated by
// the gpu-scope fence inside grid.sync())
constexpr int kMaxLevels = 40;
struct Levels {
    int n_levels;
    int start[kMaxLevels + 1];
    int nonterm[kMaxLevels];
    unsigned long long* timeline;  // optional (prl_debug_set_timeline): %globaltimer after every grid barrier
};

__device__ __forceinline__ void stamp(const Levels& lv, int& slot) {
    if (lv.timeline && blockIdx.x == 0 && threadIdx.x == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
        lv.timeline[slot] = t;
    }
    ++slot;
}

// root exploitability of seat p (ValueFiller.py:95-101): np.sum over hands of ev_br * reach - ev * reach; NMAX bounds
// T.n_range (see numpy_sum)
template <int NMAX>
__device__ __forceinline__ void root_exploitability(const prl_tree_t& T, const prl_buffers_t& B, int p, float* out) {
    const size_t N = (size_t)T.n_nodes;
    const float* ev = B.ev + (size_t)p * N * T.ld;
    const float* evbr = B.ev_br + (size_t)p * N * T.ld;
    const float* reach = B.reach + (size_t)p * N * T.ld;
    out[p] = numpy_sum<NMAX>(T.n_range, [&](int h) { return evbr[h] * reach[h] - ev[h] * reach[h]; });
}

// THREADS: block size = threads per SM (one block per SM): 512 at 128 registers per thread.  A 1024-thread / 64-register
// instantiation was no faster on the B_5 tree and was removed.
template <int R, int NS, int THREADS>
__global__ void __launch_bounds__(THREADS, 1) cfr_iterations_kernel(Ctx c, const Levels lv, const int n_iters) {
    cg::grid_group grid = cg::this_grid();
    // warp w of block b takes 32-entry chunk (w * gridDim + b) of the kind-sorted work list: consecutive chunks go to
    // different SMs, so every SM sees the same mix of node kinds (no per-kind load imbalance at the grid barrier)
    const int gwarp = (threadIdx.x >> 5) * gridDim.x + blockIdx.x;
    const int nwarps = gridDim.x * (blockDim.x >> 5);
    constexpr int NPW = LaneMap<R>::NPW;
    const int last = lv.n_levels > 1 ? lv.n_levels - 1 : 1;
    int ts = 0;
    stamp(lv, ts);
    for (int it = 0; it < n_iters; ++it) {
        for (int p = 0; p < 2; ++p) {  // _CFRBase.py:123-128
            c.mask = 1 << p;
            c.upd_p = p;
            for (int d = lv.n_levels - 1; d >= 0; --d) {
                const int lo = lv.start[d], hi = lv.start[d + 1], ng = groups_of(hi - lo, NPW);
                for (int grp = gwarp; grp < ng; grp += nwarps) value_group<R, NS, false, true>(c, lo, hi, grp);
                grid.sync();
                stamp(lv, ts);
            }
            c.mode[p] = PRL_STRAT_F32;
            for (int d = 0; d < last; ++d) {
                const int lo = lv.start[d], hi = lo + lv.nonterm[d], ng = groups_of(hi - lo, NPW);
                for (int grp = gwarp; grp < ng; grp += nwarps) reach_group<R, true>(c, lo, hi, grp);
                grid.sync();
                stamp(lv, ts);
            }
        }
        c.iter += 1;
    }
}

template <int R, int NS>
__global__ void __launch_bounds__(kPThreads, 1) evaluate_kernel(Ctx c, const Levels lv, const int do_reach, float* out) {
    cg::grid_group grid = cg::this_grid();
    const int gwarp = (threadIdx.x >> 5) * gridDim.x + blockIdx.x;
    const int nwarps = gridDim.x * (blockDim.x >> 5);
    constexpr int NPW = LaneMap<R>::NPW;
    const int last = lv.n_levels > 1 ? lv.n_levels - 1 : 1;
    c.mask = 3;
    c.upd_p = -1;
    if (do_reach) {
        for (int d = 0; d < last; ++d) {
            const int lo = lv.start[d], hi = lo + lv.nonterm[d], ng = groups_of(hi - lo, NPW);
            for (int grp = gwarp; grp < ng; grp += nwarps) reach_group<R, false>(c, lo, hi, grp);
            grid.sync();
        }
    }
    for (int d = lv.n_levels - 1; d >= 0; --d) {
        const int lo = lv.start[d], hi = lv.start[d + 1], ng = groups_of(hi - lo, NPW);
        for (int grp = gwarp; grp < ng; grp += nwarps) value_group<R, NS, true, false>(c, lo, hi, grp);
        grid.sync();
    }
    if (blockIdx.x == 0 && threadIdx.x < 2) root_exploitability<R>(c.T, c.B, threadIdx.x, out);
}

// root exploitability (ValueFiller.py:95-101) of both seats, one thread each; ranges of up to 128 hands
__global__ void root_exploitability_kernel(prl_tree_t T, prl_buffers_t B, float* out) {
    const int p = threadIdx.x;
    if (p >= 2) return;
    root_exploitability<128>(T, B, p, out);
}

// one warp per group of `npw` nodes
inline unsigned grid_for(int n_nodes, int npw) {
    const long long threads = 32LL * groups_of(n_nodes, npw);
    return (unsigned)((threads + kThreads - 1) / kThreads);
}

#define PRL_LAUNCH(kernel, nodes, npw, stream, ...)                              \
    do {                                                                         \
        kernel<<<grid_for(nodes, npw), kThreads, 0, (stream)>>>(__VA_ARGS__);    \
        prl::count_launch();                                                     \
    } while (0)

int check_tree(const prl_tree_t* t) {
    if (!t || !t->level_start) return prl::fail("prl: null tree / level_start");
    if (t->n_hole != 1) return prl::fail("prl: these sweeps serve one-hole-card games (n_hole == 1)");
    if (!t->meta) return prl::fail("prl: tree.meta is NULL (call prl_pack_node_meta once after uploading the tree)");
    if (!t->order || !t->level_nonterm) return prl::fail("prl: tree.order / level_nonterm missing");
    if (t->n_suits != 2 || (t->n_range != 6 && t->n_range != 24) || t->n_deck != t->n_range)
        return prl::fail("prl: one-card kernels are instantiated for Leduc (R=6) and BigLeduc (R=24), 2 suits");
    return 0;
}

template <int R>
void launch_reach(const Ctx& c, int nodes, bool update_avg, cudaStream_t s) {
    if (update_avg) PRL_LAUNCH((reach_level_kernel<R, true>), nodes, LaneMap<R>::NPW, s, c);
    else PRL_LAUNCH((reach_level_kernel<R, false>), nodes, LaneMap<R>::NPW, s, c);
}

template <int R>
void launch_value(const Ctx& c, int nodes, bool with_br, bool update, cudaStream_t s) {
    if (update) PRL_LAUNCH((value_level_kernel<R, 2, false, true>), nodes, LaneMap<R>::NPW, s, c);
    else if (with_br) PRL_LAUNCH((value_level_kernel<R, 2, true, false>), nodes, LaneMap<R>::NPW, s, c);
    else PRL_LAUNCH((value_level_kernel<R, 2, false, false>), nodes, LaneMap<R>::NPW, s, c);
}

void reach_sweep(Ctx c, bool update_avg, cudaStream_t s) {
    const prl_tree_t& T = c.T;
    const int last = T.n_levels > 1 ? T.n_levels - 1 : 1;  // parents of level d write level d+1; leaves write nothing
    for (int d = 0; d < last; ++d) {
        c.lo = (int)T.level_start[d];
        c.hi = c.lo + (int)T.level_nonterm[d];  // the work list puts terminals last: they have nothing to push down
        if (c.hi == c.lo) continue;
        if (T.n_range == 6) launch_reach<6>(c, c.hi - c.lo, update_avg, s);
        else launch_reach<24>(c, c.hi - c.lo, update_avg, s);
    }
}

void value_sweep(Ctx c, bool with_br, bool update, cudaStream_t s) {
    const prl_tree_t& T = c.T;
    for (int d = T.n_levels - 1; d >= 0; --d) {
        c.lo = (int)T.level_start[d];
        c.hi = (int)T.level_start[d + 1];
        if (c.hi == c.lo) continue;
        if (T.n_range == 6) launch_value<6>(c, c.hi - c.lo, with_br, update, s);
        else launch_value<24>(c, c.hi - c.lo, with_br, update, s);
    }
}

}  // namespace

extern "C" int prl_pack_node_meta(const prl_tree_t* tree, void* out_meta, prl_stream_t stream) {
    if (!tree || !out_meta) return prl::fail("prl_pack_node_meta: null argument");
    if (tree->n_hole == 1 && tree->n_deck > 254) return prl::fail("prl_pack_node_meta: deck too large");
    pack_meta_kernel<<<(tree->n_nodes + 255) / 256, 256, 0, (cudaStream_t)stream>>>(*tree, (int4*)out_meta);
    prl::count_launch();
    return prl::check(cudaGetLastError(), "prl_pack_node_meta");
}

extern "C" int prl_reach_pass(const prl_tree_t* tree, const prl_buffers_t* buf, int player_mask, const int* strat_mode,
                              prl_stream_t stream) {
    if (tree && tree->n_hole == 2) return prl2::reach_pass(tree, buf, player_mask, strat_mode, (cudaStream_t)stream);
    if (int e = check_tree(tree)) return e;
    Ctx c{*tree, *buf, 0, 0, player_mask, {strat_mode[0], strat_mode[1]}, 0, -1, 0, 0, 0};
    reach_sweep(c, false, (cudaStream_t)stream);
    return prl::check(cudaGetLastError(), "prl_reach_pass");
}

extern "C" int prl_value_pass(const prl_tree_t* tree, const prl_buffers_t* buf, int player_mask, int with_br,
                              const int* strat_mode, prl_stream_t stream) {
    if (with_br && !buf->ev_br) return prl::fail("prl_value_pass: with_br needs ev_br");
    if (tree && tree->n_hole == 2) return prl2::value_pass(tree, buf, player_mask, with_br, strat_mode, (cudaStream_t)stream);
    if (int e = check_tree(tree)) return e;
    Ctx c{*tree, *buf, 0, 0, player_mask, {strat_mode[0], strat_mode[1]}, 0, -1, 0, 0, 0};
    value_sweep(c, with_br != 0, false, (cudaStream_t)stream);
    return prl::check(cudaGetLastError(), "prl_value_pass");
}

extern "C" int prl_root_exploitability(const prl_tree_t* tree, const prl_buffers_t* buf, float* out_expl,
                                       prl_stream_t stream) {
    if (!buf->ev_br) return prl::fail("prl_root_exploitability needs ev_br");
    if (tree->n_hole == 2) return prl2::root_exploitability(tree, buf, out_expl, (cudaStream_t)stream);
    root_exploitability_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(*tree, *buf, out_expl);
    prl::count_launch();
    return prl::check(cudaGetLastError(), "prl_root_exploitability");
}

extern "C" int prl_cfr_sweep(const prl_tree_t* tree, const prl_buffers_t* buf, int algo, int p, int iter, int delay,
                             int avg_f64, const int* strat_mode, int which, prl_stream_t stream) {
    if (tree && tree->n_hole == 2) {
        if (avg_f64) return prl::fail("two-card games keep the average in float32");
        return prl2::cfr_sweep(tree, buf, algo, p, iter, delay, strat_mode, which, (cudaStream_t)stream);
    }
    if (int e = check_tree(tree)) return e;
    if (p < 0 || p > 1 || algo < 0 || algo > 2) return prl::fail("prl_cfr_sweep: bad p / algo");
    if (algo != PRL_ALGO_CFR_PLUS && avg_f64) return prl::fail("avg_f64 only applies to CFR+");
    Ctx c{*tree, *buf, 0, 0, 1 << p, {strat_mode[0], strat_mode[1]}, algo, p, iter, delay, avg_f64};
    if (which & 1) value_sweep(c, false, true, (cudaStream_t)stream);
    if (which & 2) {
        c.mode[p] = PRL_STRAT_F32;  // p's strategy now lives in the float table
        reach_sweep(c, true, (cudaStream_t)stream);
    }
    return prl::check(cudaGetLastError(), "prl_cfr_sweep");
}

namespace {

unsigned long long* g_timeline = nullptr;

int make_levels(const prl_tree_t* T, Levels* lv) {
    lv->timeline = g_timeline;
    if (T->n_levels > kMaxLevels) return prl::fail("prl: tree deeper than the persistent kernels support");
    lv->n_levels = T->n_levels;
    for (int d = 0; d <= T->n_levels; ++d) lv->start[d] = (int)T->level_start[d];
    for (int d = 0; d < T->n_levels; ++d) lv->nonterm[d] = (int)T->level_nonterm[d];
    return 0;
}

// co-resident grid for a cooperative launch of `kernel` (cached per kernel and device)
template <typename K>
int coop_grid(K kernel, int* grid, int threads = kPThreads) {
    static int cached[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 64 && cached[dev] && threads == kPThreads) { *grid = cached[dev]; return 0; }
    int per_sm = 0, sms = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return prl::check(e, "cooperative occupancy query");
    if (per_sm < 1) return prl::fail("prl: persistent kernel does not fit on an SM");
    *grid = sms;  // one block per SM
    if (dev < 64 && threads == kPThreads) cached[dev] = *grid;
    return 0;
}

template <int R>
int launch_iterations(Ctx& c, Levels& lv, int n_iters, cudaStream_t s) {
    int grid = 0;
    void* args[] = {&c, &lv, &n_iters};
    if (int e = coop_grid(cfr_iterations_kernel<R, 2, kPThreads>, &grid)) return e;
    prl::count_launch();
    return prl::check(cudaLaunchCooperativeKernel((void*)cfr_iterations_kernel<R, 2, kPThreads>, dim3(grid), dim3(kPThreads), args, 0, s),
                      "prl_cfr_iterations");
}

template <int R>
int launch_evaluate(Ctx& c, Levels& lv, int do_reach, float* out, cudaStream_t s) {
    int grid = 0;
    if (int e = coop_grid(evaluate_kernel<R, 2>, &grid)) return e;
    void* args[] = {&c, &lv, &do_reach, &out};
    prl::count_launch();
    return prl::check(cudaLaunchCooperativeKernel((void*)evaluate_kernel<R, 2>, dim3(grid), dim3(kPThreads), args, 0, s),
                      "prl_evaluate");
}

}  // namespace

extern "C" void prl_debug_set_timeline(void* device_u64_buffer) { g_timeline = (unsigned long long*)device_u64_buffer; }

extern "C" int prl_cfr_iterations(const prl_tree_t* tree, const prl_buffers_t* buf, int algo, int iter0, int n_iters,
                                  int delay, int avg_f64, const int* strat_mode, prl_stream_t stream) {
    if (tree && tree->n_hole == 2) {  // the big trees of the two-card games are bandwidth-bound: plain per-level launches
        if (avg_f64) return prl::fail("two-card games keep the average in float32");
        int mode[2] = {strat_mode[0], strat_mode[1]};
        for (int it = 0; it < n_iters; ++it)
            for (int p = 0; p < 2; ++p) {
                if (int e = prl2::cfr_sweep(tree, buf, algo, p, iter0 + it, delay, mode, 3, (cudaStream_t)stream)) return e;
                mode[p] = PRL_STRAT_F32;
            }
        return 0;
    }
    if (int e = check_tree(tree)) return e;
    if (algo < 0 || algo > 2 || n_iters < 0) return prl::fail("prl_cfr_iterations: bad algo / n_iters");
    if (algo != PRL_ALGO_CFR_PLUS && avg_f64) return prl::fail("avg_f64 only applies to CFR+");
    if (n_iters == 0) return 0;
    Ctx c{*tree, *buf, 0, 0, 0, {strat_mode[0], strat_mode[1]}, algo, 0, iter0, delay, avg_f64};
    Levels lv;
    if (int e = make_levels(tree, &lv)) return e;
    return tree->n_range == 6 ? launch_iterations<6>(c, lv, n_iters, (cudaStream_t)stream)
                              : launch_iterations<24>(c, lv, n_iters, (cudaStream_t)stream);
}

extern "C" int prl_evaluate(const prl_tree_t* tree, const prl_buffers_t* buf, const int* strat_mode, int do_reach,
                            float* out_expl, prl_stream_t stream) {
    if (!buf->ev_br || !out_expl) return prl::fail("prl_evaluate needs ev_br and out_expl");
    if (tree && tree->n_hole == 2) {
        if (do_reach)
            if (int e = prl2::reach_pass(tree, buf, 3, strat_mode, (cudaStream_t)stream)) return e;
        if (int e = prl2::value_pass(tree, buf, 3, 1, strat_mode, (cudaStream_t)stream)) return e;
        return prl2::root_exploitability(tree, buf, out_expl, (cudaStream_t)stream);
    }
    if (int e = check_tree(tree)) return e;
    Ctx c{*tree, *buf, 0, 0, 3, {strat_mode[0], strat_mode[1]}, 0, -1, 0, 0, 0};
    Levels lv;
    if (int e = make_levels(tree, &lv)) return e;
    return tree->n_range == 6 ? launch_evaluate<6>(c, lv, do_reach, out_expl, (cudaStream_t)stream)
                              : launch_evaluate<24>(c, lv, do_reach, out_expl, (cudaStream_t)stream);
}

extern "C" int prl_cfr_half_iteration(const prl_tree_t* tree, const prl_buffers_t* buf, int algo, int p, int iter,
                                      int delay, int avg_f64, const int* strat_mode, prl_stream_t stream) {
    return prl_cfr_sweep(tree, buf, algo, p, iter, delay, avg_f64, strat_mode, 3, stream);
}
