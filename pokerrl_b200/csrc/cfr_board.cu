// Board-resident CFR+ sweeps for two-hole-card games with ONE chance layer (Flop5Holdem, PokerRL/game/games.py:222-254) - sm_90a.
//
// The level-synchronous sweeps (cfr_twocard.cu) spill every node vector of every board subtree to HBM: 186 GB per
// iteration against 40 GB of regret / average tables.  Here ONE persistent CTA walks whole (board, seat)
// units: the 15-node post-deal subtree of a board lives in registers / shared memory, HBM sees only
//     opponent regret rows (strategy by regret matching)  ->  reach of the opponent, top-down        (P1)
//     9 terminal rows (5 showdown + 4 fold) evaluated together in shared memory                      (P2)
//     own regret + average rows read, updated, written; the board's root value accumulated into the
//     chance-node sum as 64-bit FIXED POINT (exactly associative: any grouping over CTAs / GPUs gives
//     the same bits)                                                                                 (P3)
// Rows of a board's table are stored in the board's STRENGTH ORDER and hold only the 1081 hands that do not collide
// with the board (stride 1088 floats instead of 1326 natural-order entries): showdown prefix sums run over consecutive
// addresses, blocked hands cost nothing, 18 % fewer bytes.  The per-board index tables (15 KB: packed per-hand record,
// hand ids, card rows) are staged by cp.async.bulk (TMA 1-D bulk copies) completing on mbarriers, the next board's tables
// in flight while the current board computes.
//
// Arithmetic follows the reference statements generalised to two-card hands (SURVEY.md appendix A; float64 restatement
// in oracle/cfr2_oracle.c): reach StrategyFiller.py:118-146, 159-166; fold / showdown values ValueFiller.py:103-158;
// value backup :64-93; regrets _CFRBase.py:146-185 + CFRPlus.py:37-41; regret matching CFRPlus.py:43-63; averaging
// CFRPlus.py:65-87.  The strategy is never stored: it is a pure function of the regret rows (CFRPlus.py:49-58).
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>

#include "pokerrl_b200.h"
#include "prl_common.cuh"

namespace {

// ---- geometry of a 52-card deck with a complete 5-card board
constexpr int kDeck = 52;
constexpr int kBoardCards = 5;
constexpr int kLiveCards = kDeck - kBoardCards;            // 47
constexpr int kLive = kLiveCards * (kLiveCards - 1) / 2;   // 1081 hands that hold no board card
constexpr int kLdb = 1088;                                  // row stride (floats) of the strength-ordered tables
constexpr int kRowLen = kLiveCards - 1;                     // 46 live hands hold a given live card
constexpr int kRowPad = 48;                                 // card rows padded to 4 lanes x 12 entries
constexpr int kRowSeg = 12;
constexpr int kErStride = kLiveCards;                       // centred prefix array of a card row: entries 0..46
constexpr int kZeroSlot = kLive + 1;                        // S[v][1082] is always 0 (target of the row padding)
constexpr int kRange = 1326;

// per-board table blob (bytes): packed records, hand ids, card rows
constexpr int kRecBytes = kLdb * 8;                         // uint64 per strength position
constexpr int kShBytes = kLdb * 2;                          // int16 hand id per strength position
constexpr int kRowIdxBytes = kLiveCards * kRowPad * 2;      // int16 strength position per card-row entry
constexpr int kBlobA = kRecBytes + kShBytes;                // 10 880 B, needed by P1 and P3
constexpr int kBlobBytes = kBlobA + kRowIdxBytes;           // 15 392 B
static_assert(kBlobA % 16 == 0 && kRowIdxBytes % 16 == 0, "bulk copies move multiples of 16 bytes");

// instrumentation switch, off in the library (tools/build_variants.py stamps builds it on)
#ifndef PRL_BV_STAMPS
#define PRL_BV_STAMPS 0      // 1 = phase stamps: clock64() at the unit start and B1-B5 of sampled units (tools/board_phases.py)
#endif
// tried and removed: five-warp / one-warp-per-vector scans, the single-warp stage spread over nine warps, the third P3 pass
// spread over all warps, two positions requested a unit ahead, all three positions requested a unit ahead, chance sums by
// load + add + store, card-major card-row prefix arrays, row totals summed in double per element, the bare MUFU.RCP, fold
// row sums gathered in the update forms, all rows of the next board prefetched at the top of an update unit (DESIGN §6.1)

constexpr int kThreads = 384;  // 12 warps; 3 strength positions per thread (3 * 384 = 1152 >= 1081: 94 % of the lanes busy)
constexpr int kWarps = kThreads / 32;

// ---- compiled shapes of the post-deal subtree (breadth-first; Flop5Holdem with pot-size raises).  The host checks the game's
//      abstract tree against these arrays and picks the shape it matches.
// per-node tables packed 4 bits per node (value + 1): a lookup is a shift, never a local-memory array
struct Nodes15 {
    int v[15];
};
constexpr unsigned long long pack_nodes(Nodes15 t) {
    unsigned long long r = 0;
    for (int i = 0; i < 15; ++i) r |= (unsigned long long)(t.v[i] + 1) << (4 * i);
    return r;
}
constexpr int unpack_node(unsigned long long t, int i) { return (int)((t >> (4 * i)) & 0xF) - 1; }

// what every shape derives from its four node arrays (SH::N, kKind, kParent, kFirstChild, kNChildren)
template <class SH>
struct ShapeOps {
    static constexpr int kind(int i) { return unpack_node(SH::kKind, i); }
    static constexpr int parent(int i) { return unpack_node(SH::kParent, i); }
    static constexpr int first_child(int i) { return unpack_node(SH::kFirstChild, i); }
    static constexpr int n_children(int i) { return unpack_node(SH::kNChildren, i); }
    // index of terminal i among the showdown / fold vectors
    static constexpr int vec_index(int i) {
        int n = 0;
        for (int k = 0; k < i; ++k) n += (kind(k) == kind(i));
        return n;
    }
    static constexpr int count(int k) {
        int n = 0;
        for (int i = 0; i < SH::N; ++i) n += (kind(i) == k);
        return n;
    }
    // table rows of one board: the rows of seat 0's decision nodes first, then seat 1's, children in breadth-first order
    static constexpr int rows_of_seat(int p) {
        int n = 0;
        for (int i = 1; i < SH::N; ++i) n += (kind(parent(i)) == p);
        return n;
    }
    static constexpr int row_of(int c) {  // c = child of a decision node
        const int p = kind(parent(c));
        int n = (p == 0) ? 0 : rows_of_seat(0);
        for (int k = 1; k < c; ++k) n += (kind(parent(k)) == p);
        return n;
    }
    // decision nodes, ascending local id (the columns of prl_board_policy_query's out_index)
    static constexpr int n_dec() {
        int n = 0;
        for (int i = 0; i < SH::N; ++i) n += (kind(i) <= 1 && n_children(i) > 0);
        return n;
    }
    static constexpr int dec_node(int d) {
        int n = 0;
        for (int i = 0; i < SH::N; ++i)
            if (kind(i) <= 1 && n_children(i) > 0 && n++ == d) return i;
        return -1;
    }
};

// Stacks of 901 chips and more: the flop bet, the pot-size raise and the all-in re-raise all fit.
// fold_coef: reach of the OPPONENT of seat P at fold terminal f as a combination of its reach at the showdown terminals
// (strategies sum to one, own nodes copy the reach): x_fold[f] = sum_v fold_coef(P, f, v) * x_sd[v].  Every linear functional
// of the fold vectors (their card-row sums) follows from the showdown vectors' at no cost.  tools/fold_relations.py derives
// the tables of both shapes.
struct ShapeFHP : ShapeOps<ShapeFHP> {
    static constexpr int N = 15;
    static constexpr unsigned long long kKind = pack_nodes({{1, 0, 0, 4, 1, 3, 4, 1, 3, 4, 0, 3, 4, 3, 4}});
    static constexpr unsigned long long kParent = pack_nodes({{-1, 0, 0, 1, 1, 2, 2, 2, 4, 4, 4, 7, 7, 10, 10}});
    static constexpr unsigned long long kFirstChild = pack_nodes({{1, 3, 5, -1, 8, -1, -1, 11, -1, -1, 13, -1, -1, -1, -1}});
    static constexpr unsigned long long kNChildren = pack_nodes({{2, 2, 3, 0, 3, 0, 0, 2, 0, 0, 2, 0, 0, 0, 0}});
    static constexpr int n_sd = 5, n_fold = 4;
    static constexpr int rows = 14;
    static constexpr int fold_coef(int P, int f, int v) {
        constexpr int c[2][4][5] = {{{0, 1, 0, 0, 0}, {1, 0, -1, 0, -1}, {0, 1, 0, -1, 0}, {0, 0, 0, 0, 1}},
                                    {{1, -1, 1, -1, 0}, {0, 0, 1, 0, 0}, {0, 0, 0, 1, 0}, {0, 0, 1, 0, -1}}};
        return c[P][f][v];
    }
};

// Stacks of 301 to 900 chips: the flop's pot-size bet is all-in, so the player facing it may only fold or call.
struct ShapeFHPShort : ShapeOps<ShapeFHPShort> {
    static constexpr int N = 9;
    static constexpr unsigned long long kKind = pack_nodes({{1, 0, 0, 4, 1, 3, 4, 3, 4}});
    static constexpr unsigned long long kParent = pack_nodes({{-1, 0, 0, 1, 1, 2, 2, 4, 4}});
    static constexpr unsigned long long kFirstChild = pack_nodes({{1, 3, 5, -1, 7, -1, -1, -1, -1}});
    static constexpr unsigned long long kNChildren = pack_nodes({{2, 2, 2, 0, 2, 0, 0, 0, 0}});
    static constexpr int n_sd = 3, n_fold = 2;
    static constexpr int rows = 8;
    static constexpr int fold_coef(int P, int f, int v) {
        constexpr int c[2][2][3] = {{{0, 1, 0}, {1, 0, -1}}, {{1, -1, 1}, {0, 0, 1}}};
        return c[P][f][v];
    }
};

template <class SH>
constexpr bool shape_consistent() {
    return SH::count(4) == SH::n_sd && SH::count(3) == SH::n_fold && SH::rows_of_seat(0) + SH::rows_of_seat(1) == SH::rows &&
           SH::N <= 15 && SH::n_fold % 2 == 0;  // P2a splits the fold vectors evenly over two groups
}
static_assert(shape_consistent<ShapeFHP>() && shape_consistent<ShapeFHPShort>(), "shape");

template <int I, int N, class F>
__device__ __forceinline__ void static_for(F&& f) {
    if constexpr (I < N) {
        f(std::integral_constant<int, I>{});
        static_for<I + 1, N>(f);
    }
}
template <int I, int N, class F>
__device__ __forceinline__ void static_for_down(F&& f) {  // N-1 .. I
    if constexpr (I < N) {
        f(std::integral_constant<int, N - 1>{});
        static_for_down<I, N - 1>(f);
    }
}

// ---- shared memory carve-up of the sweep (bytes; ShapeFHP: 9 terminal vectors, 5 of them showdowns, 4 folds)
constexpr int kErVec = kLiveCards * kErStride;                              // 2209 floats per showdown vector
template <class SH>
struct SweepSmem {
    static constexpr int kNVec = SH::n_sd + SH::n_fold;                     // terminal vectors
    static constexpr int kSOff = 0;                                         // float S[kNVec][1088]
    static constexpr int kErOff = kSOff + kNVec * kLdb * 4;                 // float Er[n_sd][47*47]
    static constexpr int kErBytes = ((SH::n_sd * kErVec * 4) + 15) & ~15;
    static constexpr int kBlobOff = kErOff + kErBytes;                      // 2 x (rec + hand ids)
    static constexpr int kRowIdxOff = kBlobOff + 2 * kBlobA;                // card rows (single buffer)
    static constexpr int kCsOff = kRowIdxOff + kRowIdxBytes;                // float cs[n_fold][48] per-card sums of the fold vectors
    static constexpr int kCsdOff = kCsOff + SH::n_fold * kRowPad * 4;       // double csd[n_fold][48]: the same sums before rounding
    static constexpr int kMiscOff = kCsdOff + SH::n_fold * kRowPad * 8;     // double wsum[n_sd][16], wexc[n_sd][16]; float tf[8]
    static constexpr int kMiscBytes = (SH::n_sd * 16 + SH::n_sd * 16) * 8 + 8 * 4;
    static constexpr int kRowTotOff = kMiscOff + kMiscBytes;                // double rowtot[n_sd][48]: card-row totals of the showdown vectors
    static constexpr int kRowTotBytes = SH::n_sd * kRowPad * 8;
    static constexpr int kBarOff = kRowTotOff + kRowTotBytes;               // 3 mbarriers
    static constexpr int kSmemBytes = kBarOff + 32;                         // 3 mbarriers, then DCFR's {a_t, b_t}
    static_assert(kBlobOff % 16 == 0 && kRowIdxOff % 16 == 0 && kCsdOff % 8 == 0 && kMiscOff % 8 == 0 && kRowTotOff % 8 == 0 &&
                      kBarOff % 8 == 0, "alignment");
    static_assert(2 * (kSmemBytes + 1024) <= 233472, "two CTAs per SM (228 KB of shared memory per H100 SM)");
    static_assert(SH::n_fold <= 8, "tf[8]");
};

struct SweepArgs {
    prl_board_game_t g;
    const float* trunk_reach_opp;  // natural order row of the opponent's reach at the chance node
    int iter, delay;
    float m_old, m_new;            // CFRPlus.py:68-73
    int pair;                      // CFR+ update: 1 = the seat's pending averaging step is applied before this iteration's
    float m_old_due, m_new_due;    // the pending step's weights
    int src_own, src_opp;          // evaluation: 0 = regret matching of `regret`, 1 = `avg` rows as they are (CFR+ average),
                                   // 2 = `avg` rows normalised (reach-weighted sums of Vanilla / Linear CFR, LinearCFR.py:64-71)
    float rw;                      // weight of the instantaneous regret: 1, Linear CFR iter + 1 (LinearCFR.py:27-28)
    const float* disc;             // DEFER: DCFR's {a_t, b_t} of this iteration (device), nullptr: no discount
    float defer_w;                 // DEFER: weight of the opponent's pending average-strategy contribution (0: none)
    double fx_scale;               // 2^frac_bits
    float sc[16];                  // terminal n: K * pot / 2, negated where the seat of this sweep is the folder
};

// ---- PTX helpers: mbarrier + 1-D bulk copy global -> shared (TMA) + bulk L2 prefetch, sm_90+
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void bulk_prefetch_l2(const void* src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!ok);
}
__device__ __forceinline__ void fence_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- phase stamps (PRL_BV_STAMPS builds only): thread 0 of CTA b < kStampCtas records, for its units it = 0, kStampEvery,
//      2 kStampEvery, ... (kStampUnits of them), clock64() at the unit start (slot 0) and right after B1 .. B5 (slots 1-5), the
//      SM id (slot 6) and it (slot 7).  prl_board_stamps copies the records out and clears them.
#if PRL_BV_STAMPS
constexpr int kStampCtas = 512, kStampUnits = 16, kStampEvery = 32, kStampSlots = 8;
__device__ long long g_stamps[kStampCtas * kStampUnits * kStampSlots];
#endif
__device__ __forceinline__ void stamp(int it, int slot) {
#if PRL_BV_STAMPS
    if (threadIdx.x == 0 && blockIdx.x < kStampCtas && it % kStampEvery == 0 && it / kStampEvery < kStampUnits) {
        long long* r = g_stamps + ((size_t)blockIdx.x * kStampUnits + it / kStampEvery) * kStampSlots;
        r[slot] = clock64();
        if (slot == 0) {
            unsigned smid;
            asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
            r[6] = smid;
            r[7] = it;
        }
    }
#endif
}

// strategy of one decision node from its table rows: regret matching (CFRPlus.py:43-63; the regrets of Vanilla / Linear
// CFR are clipped first, LinearCFR.py:33-51) or the rows as they are (CFR+ average strategy)
template <int A>
__device__ __forceinline__ void node_strategy(const float (&g)[A], int src, float (&s)[A]) {
    if (src == 1) {
#pragma unroll
        for (int a = 0; a < A; ++a) s[a] = g[a];
        return;
    }
    float sum = 0.0f;
#pragma unroll
    for (int a = 0; a < A; ++a) {
        s[a] = fmaxf(g[a], 0.0f);
        sum += s[a];
    }
    const bool pos = sum > 0.0f;
    // reciprocal = MUFU.RCP + one Newton step (<= 1 ulp, no range-check branch; sums below 1e-37 cannot occur: regrets are
    // chip amounts times probabilities)
    const float sm = fmaxf(sum, 1e-37f);
    float inv;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv) : "f"(sm));
    inv = fmaf(inv, fmaf(-sm, inv, 1.0f), inv);
    inv = pos ? inv : 0.0f;
    const float uni = pos ? 0.0f : 1.0f / (float)A;  // CFRPlus.py:53-58: uniform where no regret is positive
#pragma unroll
    for (int a = 0; a < A; ++a) s[a] = fmaf(s[a], inv, uni);
}

// one CFR+ averaging step (CFRPlus.py:65-87), avg = m_old * avg + m_new * s, rounded as nvcc contracted the plain expression
// (FMUL of m_new * s, then FFMA): a step applied a sweep later or by the flush kernel gives the same bits
__device__ __forceinline__ float avg_step(float m_old, float avg, float m_new, float s) {
    return __fmaf_rn(m_old, avg, __fmul_rn(m_new, s));
}

__device__ __forceinline__ float ld_stream(const float* p) { return __ldcs(p); }
__device__ __forceinline__ void st_stream(float* p, float v) { __stcs(p, v); }

// =====================================================================================================================
// The sweep kernel.  P = seat whose values are computed; EVAL = false: CFR+ update of seat P (regrets, average);
// EVAL = true: values and best-response values of seat P under the strategies selected by src_own / src_opp.
// Table rows of board j: [j][SH::rows][1088] floats, rows SH::row_of(child); everything a unit touches is contiguous.
// =====================================================================================================================
// DEFER (Vanilla / Linear CFR, update form): regrets are not clipped, and the average is the reach-weighted SUM of
// strategies (VanillaCFR.py:54-60, LinearCFR.py:53-59) with the seat's reach under its NEW strategy - which includes its
// new trunk reach, known only after this seat's trunk update.  The contribution of seat q's update is therefore added
// during the NEXT sweep that walks q's rows anyway: P1 of the other seat's sweep computes exactly q's strategy and reach
// at every node (defer_w = its weight).  P1ONLY: nothing but that (flush before an evaluation of the average strategy).
// AVG (CFR+ update form): false = the average rows are neither read nor written - this iteration's averaging step, if any, is
// left pending.  The strategy of the step of iteration t is regret matching of the regrets the sweep of t wrote, which the
// seat's next sweep reads and matches for its value backup anyway: there (a.pair) the pending step is applied to the loaded
// average right before this iteration's, one read and one write of the average rows for two steps.
// PRED (PCFR+ update form, DEFER family): every strategy is regret matching of the prediction rows G.pred.  P3 loads the own
// regret rows and the own prediction rows (in the registers the paired form gives its average rows), takes the strategy from
// the predictions and writes R = max(d + R, 0), then Q = max(R + d, 0).  The average is DEFER's reach-weighted sum (defer_w =
// w_t).  PCFR+'s evaluation and flush run the EVAL / P1ONLY forms on a copy of the descriptor whose `regret` is `pred`.
// RNR (restricted Nash response; Johanson, Zinkevich & Bowling, NIPS 2007): the opponent is a mixture of a fixed model
// (probability G.rnr_p) and a free strategy.  The values of seat P are linear in the opponent's reach, so the mixture only
// changes what P1 writes into S: kRnrMix adds G.rnr_p times the model's showdown reach G.rnr_reach[j][v] (trunk reach and deal
// included; the caller scales trunk_reach_opp by 1 - rnr_p) and takes the fold terminals' share through SH::fold_coef, which
// holds for any opponent whose rows sum to one.  CFR+ update forms (the exploiter's update) and the evaluation form (the
// exploitation of the model, with rnr_p = 1 and a zero trunk_reach_opp).  kRnrOut: P1 only, the opponent's strategy = the rows
// of `avg` as they are (the model), its showdown reach written to G.rnr_reach instead of S.
// BREX (evaluation form): the best response is exported as well - at each of seat P's decision nodes P3 writes, per strength
// position, 1.0f to the G.br_out row of the FIRST child whose br equals the node's maximum (np.argmax's rule; the maximum is
// the fmaxf chain the value backup takes anyway) and 0.0f to the node's other rows; the padding positions kLive .. kLdb - 1 of
// P's rows are written as 0.  The opponent's rows of G.br_out are never touched.
constexpr int kRnrMix = 1, kRnrOut = 2;
template <class SH, int P, bool EVAL, bool DEFER = false, bool P1ONLY = false, bool AVG = true, bool PRED = false, int RNR = 0,
          bool BREX = false>
__global__ void __launch_bounds__(kThreads, 2) board_sweep_kernel(const SweepArgs a) {
    static_assert(!(EVAL && DEFER) && (!P1ONLY || DEFER || RNR == kRnrOut) && (AVG || (!EVAL && !DEFER)), "variants");
    static_assert(!PRED || (DEFER && !P1ONLY), "PRED is an update form of the DEFER family");
    static_assert(RNR == 0 || (!DEFER && !PRED && (RNR == kRnrOut) == P1ONLY && (RNR == kRnrMix || !EVAL)), "RNR forms");
    static_assert(!BREX || (EVAL && RNR == 0), "BREX is an export of the plain evaluation form");
    using M = SweepSmem<SH>;
    constexpr int NSD = SH::n_sd, NF = SH::n_fold;
    extern __shared__ __align__(128) unsigned char smem[];
    float* S = reinterpret_cast<float*>(smem + M::kSOff);
    float* Er = reinterpret_cast<float*>(smem + M::kErOff);
    float* cs = reinterpret_cast<float*>(smem + M::kCsOff);
    double* csd = reinterpret_cast<double*>(smem + M::kCsdOff);
    double* wsum = reinterpret_cast<double*>(smem + M::kMiscOff);  // [NSD][16] warp totals of the main scans
    double* wexc = wsum + NSD * 16;                                 // [NSD][16] exclusive prefix of the warp totals - total / 2
    float* tf = reinterpret_cast<float*>(wexc + NSD * 16);          // [8]       totals of the fold vectors
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + M::kBarOff);  // [0], [1]: blob A buffers; [2]: card rows
    const int16_t* rowidx = reinterpret_cast<const int16_t*>(smem + M::kRowIdxOff);
    double* rowtot = reinterpret_cast<double*>(smem + M::kRowTotOff);  // [NSD][48]
    // kLin: card-row sums of the fold vectors from the showdown vectors' row totals (linearity), update forms only:
    constexpr bool kLin = !EVAL;  // evaluation may read average-strategy rows, which sum to one only up to rounding

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const prl_board_game_t& G = a.g;
    const int nb = G.n_boards;
    constexpr int OPP = 1 - P;
    constexpr int ROWS = SH::rows;
    constexpr int OWN0 = (P == 0) ? 0 : SH::rows_of_seat(0);      // first table row of the seat / of the opponent
    constexpr int OPP0 = (P == 0) ? SH::rows_of_seat(0) : 0;
    constexpr int NOWN = SH::rows_of_seat(P), NOPP = SH::rows_of_seat(OPP);
    constexpr size_t kBoardFloats = (size_t)ROWS * kLdb;
    const unsigned char* blob_g = reinterpret_cast<const unsigned char*>(G.tables);
    // tables the two seats' strategies come from (evaluation: regret matching of `regret` or the rows of `avg`)
    const float* tab_opp = PRED ? G.pred : (RNR == kRnrOut || (EVAL && a.src_opp >= 1)) ? G.avg : G.regret;
    const float* tab_own = (EVAL && a.src_own >= 1) ? G.avg : G.regret;
    const int asis_opp = (RNR == kRnrOut || (EVAL && a.src_opp == 1)) ? 1 : 0, asis_own = (EVAL && a.src_own == 1) ? 1 : 0;
    constexpr size_t kRnrFloats = (size_t)SH::n_sd * kLdb;  // G.rnr_reach per board
    const bool do_avg = !EVAL && !DEFER && AVG && a.iter >= a.delay;
    const bool pair = do_avg && a.pair;
    const bool defer_now = DEFER && a.defer_w != 0.0f;
    // DCFR's {a_t, b_t} (DEFER with a.disc only) in the 8 spare bytes after the three mbarriers: read from shared memory where
    // they are used, so that they occupy no register across the board loop (the DEFER form is at the register cap)
    float* disc = reinterpret_cast<float*>(smem + M::kBarOff + 3 * sizeof(uint64_t));
    const bool read_avg = do_avg && (pair ? a.m_old_due : a.m_old) != 0.0f;  // the first step applied reads the stored average

    // private chance-sum accumulators of this CTA (global, L2-resident): [2][kRange] int64
    long long* wp = reinterpret_cast<long long*>(G.w_private) + (size_t)blockIdx.x * 2 * kRange;
    for (int h = tid; h < 2 * kRange; h += kThreads) wp[h] = 0;
    for (int v = 0; v < M::kNVec; ++v)
        for (int i = kLive + tid; i < kLdb; i += kThreads) S[v * kLdb + i] = 0.0f;  // incl. the always-zero slot
    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        mbar_init(&bars[2], 1);
        fence_async_shared();
        if (DEFER && a.disc) {
            disc[0] = a.disc[0];
            disc[1] = a.disc[1];
        }
    }
    __syncthreads();
    int j = blockIdx.x;
    // rows of board jj into L2 ahead of their use (one bulk prefetch per contiguous piece; nothing waits on them)
    auto prefetch_rows = [&](int jj) {
        bulk_prefetch_l2(tab_opp + (size_t)jj * kBoardFloats + (size_t)OPP0 * kLdb, NOPP * kLdb * 4);
        bulk_prefetch_l2(tab_own + (size_t)jj * kBoardFloats + (size_t)OWN0 * kLdb, NOWN * kLdb * 4);
        if (read_avg) bulk_prefetch_l2(G.avg + (size_t)jj * kBoardFloats + (size_t)OWN0 * kLdb, NOWN * kLdb * 4);
        if (defer_now) bulk_prefetch_l2(G.avg + (size_t)jj * kBoardFloats + (size_t)OPP0 * kLdb, NOPP * kLdb * 4);
        if constexpr (RNR == kRnrMix) bulk_prefetch_l2(G.rnr_reach + (size_t)jj * kRnrFloats, kRnrFloats * 4);
    };
    // Update forms: each stream one phase ahead of its first use, so that a CTA holds about one board's rows in L2, not two -
    // two boards of the paired form (264 CTAs x (2 x 91 KB read + 61 KB stored)) overflow the 50 MB L2 of an H100, and rows
    // evicted before their use are fetched twice.  The evaluation form stores nothing and fits two boards deep (31 MB): it
    // keeps the whole-unit lead (measured: the phase schedule slowed it by 4 %).
    constexpr bool kPfPhase = !EVAL;
    // rows first read in P1: the next unit's opponent rows (DEFER: and the opponent's average rows), prefetched at B2 ...
    auto prefetch_opp = [&](int jj) {
        bulk_prefetch_l2(tab_opp + (size_t)jj * kBoardFloats + (size_t)OPP0 * kLdb, NOPP * kLdb * 4);
        if (defer_now) bulk_prefetch_l2(G.avg + (size_t)jj * kBoardFloats + (size_t)OPP0 * kLdb, NOPP * kLdb * 4);
        if constexpr (RNR == kRnrMix) bulk_prefetch_l2(G.rnr_reach + (size_t)jj * kRnrFloats, kRnrFloats * 4);  // P1 only reads them
    };
    // ... rows first read in P3: this unit's own rows (paired form: and the average rows), prefetched at B1 to load behind P2
    auto prefetch_own = [&](int jj) {
        bulk_prefetch_l2(tab_own + (size_t)jj * kBoardFloats + (size_t)OWN0 * kLdb, NOWN * kLdb * 4);
        if (read_avg) bulk_prefetch_l2(G.avg + (size_t)jj * kBoardFloats + (size_t)OWN0 * kLdb, NOWN * kLdb * 4);
        if constexpr (PRED) bulk_prefetch_l2(G.pred + (size_t)jj * kBoardFloats + (size_t)OWN0 * kLdb, NOWN * kLdb * 4);
    };
    if (tid == 0 && j < nb) {  // first board's tables
        mbar_expect_tx(&bars[0], kBlobA);
        bulk_g2s(smem + M::kBlobOff, blob_g + (size_t)j * kBlobBytes, kBlobA, &bars[0]);
        if (!P1ONLY) {
            mbar_expect_tx(&bars[2], kRowIdxBytes);
            bulk_g2s(smem + M::kRowIdxOff, blob_g + (size_t)j * kBlobBytes + kBlobA, kRowIdxBytes, &bars[2]);
        }
        if constexpr (kPfPhase) prefetch_opp(j);
        else prefetch_rows(j);
    }

    // P1 inputs of the thread's three strength positions (opponent rows + trunk reach).  Only the first position is
    // requested one unit ahead (8 registers live across the unit's last barrier - 24 spilled to local memory and made the
    // warp wait for the loads there); the other two are requested inside P1, one position ahead of their use.
    float p1_g[NOPP], p1_x0;
    auto p1_load_k = [&](int jj, const int16_t* sh_jj, int k, float (&g)[NOPP], float& x0) {
        // lanes past the last hand read the last hand's values (never used): unconditional loads keep the arrays in registers
        const int i = min(tid + k * kThreads, kLive - 1);
        const float* rows = tab_opp + (size_t)jj * kBoardFloats + (size_t)OPP0 * kLdb + i;
#pragma unroll
        for (int r = 0; r < NOPP; ++r) g[r] = ld_stream(rows + (size_t)r * kLdb);
        x0 = __ldg(a.trunk_reach_opp + sh_jj[i]);
    };
    auto p1_load = [&](int jj, const int16_t* sh_jj) { p1_load_k(jj, sh_jj, 0, p1_g, p1_x0); };

    for (int it = 0; j < nb; j += gridDim.x, ++it) {
        const int buf = it & 1;
        const unsigned char* blob = smem + M::kBlobOff + buf * kBlobA;
        const uint64_t* rec = reinterpret_cast<const uint64_t*>(blob);
        const int16_t* sh = reinterpret_cast<const int16_t*>(blob + kRecBytes);
        const int jn = j + gridDim.x;
        stamp(it, 0);
        if (tid == 0 && jn < nb) {  // next board: records + hand ids into the other buffer (free since the last barrier), rows into L2
            mbar_expect_tx(&bars[buf ^ 1], kBlobA);
            bulk_g2s(smem + M::kBlobOff + (buf ^ 1) * kBlobA, blob_g + (size_t)jn * kBlobBytes, kBlobA, &bars[buf ^ 1]);
            if constexpr (!kPfPhase) prefetch_rows(jn);
        }
        const float prob = __ldg(G.board_prob + j);
        if (it == 0) {
            mbar_wait(&bars[buf], 0);
            p1_load(j, sh);
        }

        // ------------------------------------------------------------------------------------------ P1: reach, top-down
        // x[i] = reach of the OPPONENT at local node i (StrategyFiller.py:118-146); terminal rows go to S in strength order.
        // The rows were requested before the previous unit's last barrier (p1_load): their latency is off this path.
        auto p1_hand = [&](int k, const float (&gk)[NOPP], float x0k) {
            const int i = tid + k * kThreads;
            if (i < kLive) {
                float x[SH::N];
                x[0] = x0k * prob;  // the deal (StrategyFiller.py:137-140); blocked hands are not stored at all
                float fm[RNR == kRnrMix ? NSD : 1];  // kRnrMix: the model's showdown reach of this hand
                if constexpr (RNR == kRnrMix) {
#pragma unroll
                    for (int v = 0; v < NSD; ++v) fm[v] = ld_stream(G.rnr_reach + (size_t)j * kRnrFloats + (size_t)v * kLdb + i);
                }
                static_for<0, SH::N>([&](auto I) {
                    constexpr int n = decltype(I)::value;
                    constexpr int A = SH::n_children(n);
                    if constexpr (SH::kind(n) <= 1) {
                        constexpr int fc = SH::first_child(n);
                        if constexpr (SH::kind(n) == OPP) {
                            constexpr int r0 = SH::row_of(fc);  // the node's children own rows r0 .. r0 + A - 1
                            float gg[A], s[A];
#pragma unroll
                            for (int c = 0; c < A; ++c) gg[c] = gk[r0 - OPP0 + c];
                            node_strategy<A>(gg, asis_opp, s);
#pragma unroll
                            for (int c = 0; c < A; ++c) x[fc + c] = x[n] * s[c];
                            if constexpr (DEFER) {
                                if (defer_now) {  // avg_strat_sum += strategy * reach * weight (VanillaCFR.py:56-59, LinearCFR.py:55-58)
                                    float* arow = G.avg + (size_t)j * kBoardFloats + i;
#pragma unroll
                                    for (int c = 0; c < A; ++c) {
                                        float* ap = arow + (size_t)(r0 + c) * kLdb;
                                        st_stream(ap, __fadd_rn(ld_stream(ap), __fmul_rn(x[fc + c], a.defer_w)));
                                    }
                                }
                            }
                        } else {
#pragma unroll
                            for (int c = 0; c < A; ++c) x[fc + c] = x[n];
                        }
                    } else if constexpr (SH::kind(n) == 4) {
                        constexpr int v = SH::vec_index(n);
                        if constexpr (RNR == kRnrOut) st_stream(G.rnr_reach + (size_t)j * kRnrFloats + (size_t)v * kLdb + i, x[n]);
                        else if constexpr (RNR == kRnrMix) S[v * kLdb + i] = __fmaf_rn(G.rnr_p, fm[v], x[n]);
                        else S[v * kLdb + i] = x[n];
                    } else if constexpr (RNR == kRnrMix) {  // the model's fold reach: x_fold[f] = sum_v fold_coef * x_sd[v]
                        constexpr int f = SH::vec_index(n);
                        float m = 0.0f;
                        static_for<0, NSD>([&](auto V) {
                            constexpr int cf = SH::fold_coef(P, f, decltype(V)::value);
                            if constexpr (cf > 0) m = __fadd_rn(m, fm[decltype(V)::value]);
                            else if constexpr (cf < 0) m = __fsub_rn(m, fm[decltype(V)::value]);
                        });
                        S[(NSD + f) * kLdb + i] = __fmaf_rn(G.rnr_p, m, x[n]);
                    } else if constexpr (RNR != kRnrOut) {
                        S[(NSD + SH::vec_index(n)) * kLdb + i] = x[n];
                    }
                });
            }
        };
        {
            float gB[NOPP], gC[NOPP], xB = 0.0f, xC = 0.0f;
            p1_load_k(j, sh, 1, gB, xB);
            p1_hand(0, p1_g, p1_x0);
            p1_load_k(j, sh, 2, gC, xC);
            p1_hand(1, gB, xB);
            p1_hand(2, gC, xC);
        }
        __syncthreads();  // B1: S complete
        stamp(it, 1);
        if (kPfPhase && tid == 0) {
            if constexpr (P1ONLY) {  // no P2 / P3: the next unit's opponent rows right away
                if (jn < nb) prefetch_opp(jn);
            } else {
                prefetch_own(j);
            }
        }
        if constexpr (!P1ONLY) {

        // ------------------------------------------------------------------------------------------ P2a: card rows
        // quad (live card lc, lane q): entries [12 q, 12 q + 12) of the card's row in strength order.  Showdown vectors:
        // centred exclusive prefix sums Er[v][lc][k] = (mass of the k weakest hands holding the card) - half the row's mass;
        // fold vectors: the row's mass cs[f][lc].  Two groups of 47 quads share the terminal vectors (ShapeFHP: SD 0-2 + fold
        // 0-1 | SD 3-4 + fold 2-3; ShapeFHPShort: SD 0-1 + fold 0 | SD 2 + fold 1); the other threads start on the main scans,
        // which only read S as well.
        mbar_wait(&bars[2], it & 1);
        float a0[NSD], a1[NSD], a2[NSD];
        double pre[NSD];
        constexpr int kQuadThreads = kLiveCards * 4;  // 188
        constexpr int kSdSplit = (NSD + 1) / 2, kFoldSplit = NF / 2;  // first vector of the second group
        if (warp < (2 * kQuadThreads + 31) / 32) {   // whole warps (the quad shuffles name every lane)
            const int grp = (tid >= kQuadThreads) ? 1 : 0;
            const int t = tid - grp * kQuadThreads;
            const bool row_live = t < kQuadThreads;
            const int lc = row_live ? (t >> 2) : (kLiveCards - 1), q = tid & 3;
            const unsigned qmask = 0xFu << (lane & 28);  // the two groups run different trip counts: shuffles name the quad only
            const uint2* rp = reinterpret_cast<const uint2*>(rowidx + lc * kRowPad + q * kRowSeg);
            const uint2 w0 = rp[0], w1 = rp[1], w2 = rp[2];
            const unsigned pk[6] = {w0.x, w0.y, w1.x, w1.y, w2.x, w2.y};
            int idx[kRowSeg];
#pragma unroll
            for (int e = 0; e < kRowSeg; ++e) idx[e] = (pk[e >> 1] >> ((e & 1) * 16)) & 0xffffu;
            const int v_lo = grp ? kSdSplit : 0, v_hi = grp ? NSD : kSdSplit;
#pragma unroll 1
            for (int v = v_lo; v < v_hi; ++v) {
                const float* Sv = S + v * kLdb;
                float inc[kRowSeg];
                float run = 0.0f;
#pragma unroll
                for (int e = 0; e < kRowSeg; ++e) {
                    inc[e] = run;
                    run += Sv[idx[e]];
                }
                if constexpr (kLin) {
                    // the row's total in double (the fold vectors' row sums derive from these): a lane's 12 terms summed in
                    // float, only the quad reduction in double (measured: +1 %, parity unchanged at <= 1.6e-7)
                    double drun = (double)run;
                    drun += __shfl_xor_sync(qmask, drun, 1, 4);
                    drun += __shfl_xor_sync(qmask, drun, 2, 4);
                    if (row_live && q == 0) rowtot[v * kRowPad + lc] = drun;
                }
                float sc = run;  // inclusive scan over the quad
                float tt = __shfl_up_sync(qmask, sc, 1, 4);
                if (q >= 1) sc += tt;
                tt = __shfl_up_sync(qmask, sc, 2, 4);
                if (q >= 2) sc += tt;
                const float half = 0.5f * __shfl_sync(qmask, sc, 3, 4);
                const float off = (sc - run) - half;
                float* row = Er + v * kErVec + q * kRowSeg * kErStride + lc;  // entry-major: Er[v][k][card]
#pragma unroll
                for (int e = 0; e < kRowSeg; ++e)
                    if (row_live && q * kRowSeg + e < kErStride) row[e * kErStride] = off + inc[e];
            }
#pragma unroll 1
            for (int f = kFoldSplit * grp; f < (kLin ? 0 : kFoldSplit * grp + kFoldSplit); ++f) {  // kLin: nothing to gather for the fold vectors
                const float* Sv = S + (NSD + f) * kLdb;
                double run = 0.0;  // double: the fold value subtracts these sums from the total (cancellation)
#pragma unroll
                for (int e = 0; e < kRowSeg; ++e) run += (double)Sv[idx[e]];
                run += __shfl_xor_sync(qmask, run, 1, 4);
                run += __shfl_xor_sync(qmask, run, 2, 4);
                if (row_live && q == 0) csd[f * kRowPad + lc] = run;
            }
        }
        __syncwarp();
        // ------------------------------------------------------------------------------------------ P2b: main scans, part 1
        // centred exclusive prefix sums over the strength order: E[k] = (mass of the k weakest hands) - total / 2, k = 0 ..
        // 1081, sums in double (the showdown value is a difference of two prefixes).
        // Thread t owns positions 3t .. 3t+2.
        {
            const int b0 = 3 * tid;
#pragma unroll
            for (int v = 0; v < NSD; ++v) {
                const float* Sv = S + v * kLdb;
                a0[v] = (b0 < kLive) ? Sv[b0] : 0.0f;
                a1[v] = (b0 + 1 < kLive) ? Sv[b0 + 1] : 0.0f;
                a2[v] = (b0 + 2 < kLive) ? Sv[b0 + 2] : 0.0f;
                const double loc = ((double)a0[v] + (double)a1[v]) + (double)a2[v];
                double incw = loc;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const double tt = __shfl_up_sync(0xffffffffu, incw, o);
                    if (lane >= o) incw += tt;
                }
                pre[v] = incw - loc;  // exclusive within the warp
                if (lane == 31) wsum[v * 16 + warp] = incw;
            }
        }
        // P3 inputs of the first strength position: requested here, consumed after the prefix sums are written back
        const float mult = __ldg(G.board_mult + j);
        const double fx = (double)mult * a.fx_scale;
        const float* own_rows = tab_own + (size_t)j * kBoardFloats + (size_t)OWN0 * kLdb;
        float* reg_rows = G.regret + (size_t)j * kBoardFloats + (size_t)OWN0 * kLdb;
        float* avg_rows = G.avg + (size_t)j * kBoardFloats + (size_t)OWN0 * kLdb;
        float* pred_rows = PRED ? G.pred + (size_t)j * kBoardFloats + (size_t)OWN0 * kLdb : nullptr;  // PRED: own predictions
        auto p3_pos = [&](int k) -> int { return tid + k * kThreads; };  // strength position of the thread's k-th hand of P3
        float gA[NOWN], aA[NOWN], gB[NOWN], aB[NOWN];
        auto p3_load = [&](int k, float (&g)[NOWN], float (&av)[NOWN]) {
            const int i = min(p3_pos(k), kLive - 1);  // unconditional (see p1_load_k)
#pragma unroll
            for (int r = 0; r < NOWN; ++r) g[r] = ld_stream(own_rows + (size_t)r * kLdb + i);
#pragma unroll
            for (int r = 0; r < NOWN; ++r) av[r] = 0.0f;
            if (read_avg) {
#pragma unroll
                for (int r = 0; r < NOWN; ++r) av[r] = ld_stream(avg_rows + (size_t)r * kLdb + i);
            }
            if constexpr (PRED) {  // the own prediction rows ride in the average's registers
#pragma unroll
                for (int r = 0; r < NOWN; ++r) av[r] = ld_stream(pred_rows + (size_t)r * kLdb + i);
            }
        };
        p3_load(0, gA, aA);
        __syncthreads();  // B2: card rows done, S may be overwritten, the row table may be replaced
        stamp(it, 2);
        if (tid == 0 && jn < nb) {
            mbar_expect_tx(&bars[2], kRowIdxBytes);
            bulk_g2s(smem + M::kRowIdxOff, blob_g + (size_t)jn * kBlobBytes + kBlobA, kRowIdxBytes, &bars[2]);
            if constexpr (kPfPhase) prefetch_opp(jn);
        }
        // card-row sums cs[f][card] and total tf[f] of fold vector f (total = half the sum of its card rows): from the gathered
        // sums csd, or - kLin - as the combination SH::fold_coef of the showdown vectors' row totals
        auto fold_finish = [&](auto F) {
            constexpr int f = decltype(F)::value;
            double c0 = 0.0, c1 = 0.0;
            if constexpr (kLin) {
                static_for<0, NSD>([&](auto V) {
                    constexpr int v = decltype(V)::value;
                    constexpr int cf = SH::fold_coef(P, f, v);
                    if constexpr (cf != 0) {
                        const double r0 = (lane < kLiveCards) ? rowtot[v * kRowPad + lane] : 0.0;
                        const double r1 = (lane + 32 < kLiveCards) ? rowtot[v * kRowPad + lane + 32] : 0.0;
                        c0 = (cf > 0) ? c0 + r0 : c0 - r0;
                        c1 = (cf > 0) ? c1 + r1 : c1 - r1;
                    }
                });
            } else {
                c0 = (lane < kLiveCards) ? csd[f * kRowPad + lane] : 0.0;
                c1 = (lane + 32 < kLiveCards) ? csd[f * kRowPad + lane + 32] : 0.0;
            }
            double s2 = c0 + c1;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
            if (lane == 0) tf[f] = (float)(0.5 * s2);
            if (lane < kLiveCards) cs[f * kRowPad + lane] = (float)c0;  // float copies for the per-hand epilogue
            if (lane + 32 < kLiveCards) cs[f * kRowPad + lane + 32] = (float)c1;
        };
        {
            auto warp_totals_scan = [&](int v) {  // exclusive scan of the 12 warp totals of vector v
                const double w = (lane < kWarps) ? wsum[v * 16 + lane] : 0.0;
                double sc = w;
#pragma unroll
                for (int o = 1; o < 16; o <<= 1) {
                    const double tt = __shfl_up_sync(0xffffffffu, sc, o);
                    if (lane >= o) sc += tt;
                }
                const double total = __shfl_sync(0xffffffffu, sc, kWarps - 1);
                if (lane < kWarps) wexc[v * 16 + lane] = (sc - w) - 0.5 * total;
            };
            if (warp == 0) {
#pragma unroll
                for (int v = 0; v < NSD; ++v) warp_totals_scan(v);
            } else if (warp == 1) {
                static_for<0, NF>([&](auto F) { fold_finish(F); });
            }
            __syncthreads();  // B3
            stamp(it, 3);
            const int b0 = 3 * tid;
#pragma unroll
            for (int v = 0; v < NSD; ++v) {
                float* Sv = S + v * kLdb;
                double run = pre[v] + wexc[v * 16 + warp];
                if (b0 <= kLive) Sv[b0] = (float)run;
                run += (double)a0[v];
                if (b0 + 1 <= kLive) Sv[b0 + 1] = (float)run;
                run += (double)a1[v];
                if (b0 + 2 <= kLive) Sv[b0 + 2] = (float)run;
            }
        }
        __syncthreads();  // B4: prefix arrays complete
        stamp(it, 4);

        // ------------------------------------------------------------------------------------------ P3: values, bottom-up
        auto p3_hand = [&](int k, const float (&gown)[NOWN], float (&av)[NOWN]) {
            const int i = p3_pos(k);
            const uint64_t w = rec[i];
            const int hand = sh[i];
            long long* wacc = wp + hand;
            const int gs = (int)(w & 0x7ffu), ge = (int)((w >> 11) & 0x7ffu);
            const int lc1 = (int)((w >> 22) & 0x3fu), lc2 = (int)((w >> 28) & 0x3fu);
            const int k1 = (int)((w >> 34) & 0x3fu), t1 = (int)((w >> 40) & 0x3fu), k2 = (int)((w >> 46) & 0x3fu), t2 = (int)((w >> 52) & 0x3fu);
            const int o1 = k1 * kErStride + lc1, o1e = o1 + t1 * kErStride;
            const int o2 = k2 * kErStride + lc2, o2e = o2 + t2 * kErStride;
            float e[SH::N], br[EVAL ? SH::N : 1];
            // terminal rows (ValueFiller.py:103-158): ev = equity * K * pot / 2, the folder loses
            static_for<0, SH::N>([&](auto I) {
                constexpr int n = decltype(I)::value;
                if constexpr (SH::kind(n) == 4) {
                    constexpr int v = SH::vec_index(n);
                    const float* Ev = S + v * kLdb;
                    const float* Rv = Er + v * kErVec;
                    const float all = Ev[gs] + Ev[ge];
                    const float rows = (Rv[o1] + Rv[o1e]) + (Rv[o2] + Rv[o2e]);
                    e[n] = (all - rows) * a.sc[n];
                    if constexpr (EVAL) br[n] = e[n];
                } else if constexpr (SH::kind(n) == 3) {
                    constexpr int f = SH::vec_index(n);
                    const float mass = ((tf[f] - cs[f * kRowPad + lc1]) - cs[f * kRowPad + lc2]) + S[(NSD + f) * kLdb + i];
                    e[n] = mass * a.sc[n];
                    if constexpr (EVAL) br[n] = e[n];
                }
            });
            // decision nodes, deepest first (ValueFiller.py:64-93); regrets / matching / average at P's nodes
            static_for_down<0, SH::N>([&](auto I) {
                constexpr int n = decltype(I)::value;
                constexpr int A = SH::n_children(n);
                if constexpr (SH::kind(n) <= 1) {
                    constexpr int fc = SH::first_child(n);
                    if constexpr (SH::kind(n) == OPP) {
                        float v = e[fc];
#pragma unroll
                        for (int c = 1; c < A; ++c) v += e[fc + c];
                        e[n] = v;
                        if constexpr (EVAL) {
                            float b = br[fc];
#pragma unroll
                            for (int c = 1; c < A; ++c) b += br[fc + c];
                            br[n] = b;
                        }
                    } else {
                        constexpr int r0 = SH::row_of(fc) - OWN0;  // rows r0 .. r0 + A - 1 of the seat's block
                        float g[A], s[A];
#pragma unroll
                        for (int c = 0; c < A; ++c) g[c] = gown[r0 + c];
                        if constexpr (PRED) {  // PCFR+: the strategy from the predictions
                            float q[A];
#pragma unroll
                            for (int c = 0; c < A; ++c) q[c] = av[r0 + c];
                            node_strategy<A>(q, 0, s);
                        } else {
                            node_strategy<A>(g, asis_own, s);
                        }
                        if (pair) {  // s = the pending step's strategy: matching of the same regret rows, same statements
#pragma unroll
                            for (int c = 0; c < A; ++c) av[r0 + c] = avg_step(a.m_old_due, av[r0 + c], a.m_new_due, s[c]);
                        }
                        float v = s[0] * e[fc];
#pragma unroll
                        for (int c = 1; c < A; ++c) v += s[c] * e[fc + c];
                        e[n] = v;
                        if constexpr (EVAL) {
                            float b = br[fc];
#pragma unroll
                            for (int c = 1; c < A; ++c) b = fmaxf(b, br[fc + c]);
                            br[n] = b;
                            if constexpr (BREX) {  // one-hot rows of the first child whose br is the maximum
                                float* xrow = G.br_out + (size_t)j * kBoardFloats + (size_t)SH::row_of(fc) * kLdb + i;
                                bool found = false;
#pragma unroll
                                for (int c = 0; c < A; ++c) {
                                    const bool pick = !found && br[fc + c] == b;
                                    found = found || pick;
                                    st_stream(xrow + (size_t)c * kLdb, pick ? 1.0f : 0.0f);
                                }
                            }
                        } else {
                            if constexpr (PRED) {  // PCFR+: R = max(d + R, 0) (CFRPlus.py:37-41), then Q = max(R + d, 0)
#pragma unroll
                                for (int c = 0; c < A; ++c) {
                                    const float d = e[fc + c] - v;
                                    g[c] = fmaxf(d + g[c], 0.0f);
                                    st_stream(reg_rows + (size_t)(r0 + c) * kLdb + i, g[c]);
                                    st_stream(pred_rows + (size_t)(r0 + c) * kLdb + i, fmaxf(g[c] + d, 0.0f));
                                }
                            } else {
#pragma unroll
                            for (int c = 0; c < A; ++c) {
                                if constexpr (DEFER) {  // VanillaCFR.py:26-27, LinearCFR.py:27-28
                                    g[c] = __fadd_rn(__fmul_rn(a.rw, e[fc + c] - v), g[c]);
                                    // DCFR: the new sum times a_t where it is positive, else b_t
                                    if (a.disc) g[c] = __fmul_rn(g[c], (g[c] > 0.0f) ? disc[0] : disc[1]);
                                } else g[c] = fmaxf((e[fc + c] - v) + g[c], 0.0f);                          // CFRPlus.py:37-41
                            }
                            if constexpr (!DEFER) node_strategy<A>(g, 0, s);
#pragma unroll
                            for (int c = 0; c < A; ++c) st_stream(reg_rows + (size_t)(r0 + c) * kLdb + i, g[c]);
                            if (do_avg) {  // CFRPlus.py:65-87 (not reach-weighted)
#pragma unroll
                                for (int c = 0; c < A; ++c)
                                    st_stream(avg_rows + (size_t)(r0 + c) * kLdb + i, avg_step(a.m_old, av[r0 + c], a.m_new, s[c]));
                            }
                            }  // !PRED
                        }
                    }
                }
            });
            // the board's contribution to its parent's sum (ValueFiller.py:76-78), 64-bit fixed point: fire-and-forget 64-bit RED
            // into the CTA's private vector, nothing to wait for
            atomicAdd(reinterpret_cast<unsigned long long*>(wacc), (unsigned long long)__double2ll_rn((double)e[0] * fx));
            if constexpr (EVAL)
                atomicAdd(reinterpret_cast<unsigned long long*>(wacc + kRange), (unsigned long long)__double2ll_rn((double)br[0] * fx));
        };
        // software pipeline over the thread's three strength positions: the next position's rows are in flight while the
        // current one is evaluated (position 0 was requested before the prefix sums were written back)
        p3_load(1, gB, aB);
        p3_hand(0, gA, aA);
        p3_load(2, gA, aA);
        if (p3_pos(1) < kLive) p3_hand(1, gB, aB);
        if (p3_pos(2) < kLive) p3_hand(2, gA, aA);
        if constexpr (BREX) {  // the padding positions of the seat's exported rows
            if (tid < kLdb - kLive)
#pragma unroll
                for (int r = 0; r < NOWN; ++r) st_stream(G.br_out + (size_t)j * kBoardFloats + (size_t)(OWN0 + r) * kLdb + kLive + tid, 0.0f);
        }
        }  // !P1ONLY
        // next unit's P1 inputs: requested before the barrier below, consumed after it (the other table buffer is long there)
        if (jn < nb) {
            mbar_wait(&bars[buf ^ 1], ((it + 1) >> 1) & 1);
            p1_load(jn, reinterpret_cast<const int16_t*>(smem + M::kBlobOff + (buf ^ 1) * kBlobA + kRecBytes));
        }
        __syncthreads();  // B5: S / Er / tables of this board are free
        stamp(it, 5);
    }
    // merge into the device-wide sums (integer adds: exact in any order)
    __syncthreads();
    unsigned long long* wt = reinterpret_cast<unsigned long long*>(G.w_total) + (EVAL ? 2 * P * kRange : 0);  // eval: [seat][ev, ev_br]
    for (int h = tid; h < (EVAL ? 2 : 1) * kRange; h += kThreads) {
        const long long v = __ldcg(wp + h);  // L2: where the REDs landed
        if (v != 0) atomicAdd(wt + h, (unsigned long long)v);
    }
}

// A pending CFR+ averaging step of seat P on its own (before the average is read or exported): the strategy from the seat's
// regret rows, which no sweep has changed since the step's iteration, by the statements of board_sweep_kernel.  One CTA per
// board; hands that hold a board card (positions >= kLive) are never written, as in the sweep.
template <class SH, int P>
__global__ void __launch_bounds__(256) avg_flush_kernel(float* __restrict__ regret, float* __restrict__ avg, float m_old, float m_new) {
    constexpr size_t kBoardFloats = (size_t)SH::rows * kLdb;
    const float* reg_b = regret + (size_t)blockIdx.x * kBoardFloats;
    float* avg_b = avg + (size_t)blockIdx.x * kBoardFloats;
    for (int i = threadIdx.x; i < kLive; i += blockDim.x) {
        static_for<0, SH::N>([&](auto I) {
            constexpr int n = decltype(I)::value;
            if constexpr (SH::kind(n) == P) {
                constexpr int A = SH::n_children(n), r0 = SH::row_of(SH::first_child(n));
                float g[A], s[A];
#pragma unroll
                for (int c = 0; c < A; ++c) g[c] = ld_stream(reg_b + (size_t)(r0 + c) * kLdb + i);
                node_strategy<A>(g, 0, s);
#pragma unroll
                for (int c = 0; c < A; ++c) {
                    float* ap = avg_b + (size_t)(r0 + c) * kLdb + i;
                    st_stream(ap, avg_step(m_old, (m_old != 0.0f) ? ld_stream(ap) : 0.0f, m_new, s[c]));
                }
            }
        });
    }
}

// =====================================================================================================================
// Per-board tables from the hand strengths (prl_hand_rank_boards): strength order, packed records, card rows.
// One CTA per board.  blob layout: uint64 rec[1088] | int16 hand[1088] | int16 rowidx[47][48]
//   rec[s] (s = strength position, ties ordered by hand id): bits 0-10 gs (# strictly weaker), 11-21 ge (# weaker or equal),
//          22-27 / 28-33 compact index of the hand's first / second card among the 47 live cards, 34-39 # hands of the first
//          card's row strictly weaker, 40-45 # tied in that row (incl. the hand itself), 46-51 / 52-57 same for the second card
// =====================================================================================================================
__global__ void __launch_bounds__(256) board_tables_kernel(const int32_t* __restrict__ ranks, const uint64_t* __restrict__ board_mask,
                                                           const int8_t* __restrict__ hand_cards, int n_boards,
                                                           unsigned char* __restrict__ out) {
    __shared__ int srk[kRange];
    __shared__ short spos[kRange], sgs[kRange], sge[kRange];
    const int b = blockIdx.x;
    const uint64_t bm = board_mask[b];
    unsigned char* blob = out + (size_t)b * kBlobBytes;
    uint64_t* rec = reinterpret_cast<uint64_t*>(blob);
    int16_t* sh = reinterpret_cast<int16_t*>(blob + kRecBytes);
    int16_t* rowidx = reinterpret_cast<int16_t*>(blob + kBlobA);
    for (int h = threadIdx.x; h < kRange; h += blockDim.x) srk[h] = ranks[(size_t)b * kRange + h];
    for (int i = threadIdx.x; i < kLdb; i += blockDim.x) {
        rec[i] = 0;
        sh[i] = 0;
    }
    for (int i = threadIdx.x; i < kLiveCards * kRowPad; i += blockDim.x) rowidx[i] = (int16_t)kZeroSlot;
    __syncthreads();
    for (int h = threadIdx.x; h < kRange; h += blockDim.x) {
        const int r = srk[h];
        int lt = 0, le = 0, tb = 0;
        if (r >= 0) {
            for (int q = 0; q < kRange; ++q) {
                const int x = srk[q];
                if (x < 0) continue;
                lt += x < r;
                le += x <= r;
                tb += (x == r) && (q < h);
            }
        }
        sgs[h] = (short)(r >= 0 ? lt : -1);
        sge[h] = (short)(r >= 0 ? le : -1);
        spos[h] = (short)(r >= 0 ? lt + tb : -1);
    }
    __syncthreads();
    // card rows: item (card c, other card x)
    for (int it = threadIdx.x; it < kDeck * (kDeck - 1); it += blockDim.x) {
        const int c = it / (kDeck - 1), xr = it % (kDeck - 1);
        const int x = xr + (xr >= c);
        if (((bm >> c) | (bm >> x)) & 1ull) continue;
        const int c1 = min(c, x), c2 = max(c, x);
        const int h = c1 * (2 * kDeck - 1 - c1) / 2 + (c2 - c1 - 1);
        const int g = sgs[h], ps = spos[h];
        int lt = 0, le = 0, kpos = 0;
        for (int y = 0; y < kDeck; ++y) {
            if (y == c || ((bm >> y) & 1ull)) continue;
            const int d1 = min(c, y), d2 = max(c, y);
            const int h2 = d1 * (2 * kDeck - 1 - d1) / 2 + (d2 - d1 - 1);
            const int g2 = sgs[h2];
            lt += g2 < g;
            le += g2 <= g;
            kpos += spos[h2] < ps;
        }
        const int lc = c - __popcll(bm & ((1ull << c) - 1ull));
        rowidx[lc * kRowPad + kpos] = (int16_t)ps;
        // this card's fields of the hand's record (first card = the smaller id)
        const uint64_t fld = ((uint64_t)lc) << (c == c1 ? 22 : 28) | ((uint64_t)lt) << (c == c1 ? 34 : 46) |
                             ((uint64_t)(le - lt)) << (c == c1 ? 40 : 52);
        atomicOr(reinterpret_cast<unsigned long long*>(rec + ps), (unsigned long long)fld);
    }
    __syncthreads();
    for (int h = threadIdx.x; h < kRange; h += blockDim.x) {
        const int ps = spos[h];
        if (ps < 0) continue;
        sh[ps] = (int16_t)h;
        atomicOr(reinterpret_cast<unsigned long long*>(rec + ps),
                 (unsigned long long)((uint64_t)sgs[h] | ((uint64_t)sge[h] << 11)));
    }
}

// chance-node rows from the fixed-point sums: out[a][h] = 2^-frac * sum over the suit permutations s of W[a][s(h)]
// (integer sum: exact), or W[a][h] itself without isomorphism (DESIGN.md: suit symmetrisation)
__global__ void board_collect_kernel(const long long* __restrict__ w_total, int n_arr, const int16_t* __restrict__ sym_perm,
                                     int n_sym, double inv_scale, float* __restrict__ out, int ld) {
    const int h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= kRange) return;
    for (int a = 0; a < n_arr; ++a) {
        long long s = 0;
        if (n_sym > 1) {
            for (int q = 0; q < n_sym; ++q) s += w_total[(size_t)a * kRange + sym_perm[(size_t)q * kRange + h]];
        } else {
            s = w_total[(size_t)a * kRange + h];
        }
        out[(size_t)a * ld + h] = (float)((double)s * inv_scale);
    }
}

// strength-ordered rows <-> natural-order rows of ONE table (interfaces to the level engine, checkpoints, agents)
__global__ void board_permute_kernel(const unsigned char* __restrict__ tables, int n_boards, int rows_per_board,
                                     const int64_t* __restrict__ row_src, const int64_t* __restrict__ row_dst, float* sorted_tab,
                                     float* natural_tab, int ld, int to_natural) {
    // block = (board j, row r of the board); row_src[r] / row_dst[r]: row index on board 0 and stride per board packed
    const int j = blockIdx.x / rows_per_board, r = blockIdx.x % rows_per_board;
    const int16_t* sh = reinterpret_cast<const int16_t*>(tables + (size_t)j * kBlobBytes + kRecBytes);
    float* srow = sorted_tab + ((size_t)row_src[2 * r] + (size_t)j * row_src[2 * r + 1]) * kLdb;
    float* nrow = natural_tab + ((size_t)row_dst[2 * r] + (size_t)j * row_dst[2 * r + 1]) * ld;
    if (to_natural) {
        for (int h = threadIdx.x; h < ld; h += blockDim.x) nrow[h] = 0.0f;
        __syncthreads();
        for (int i = threadIdx.x; i < kLive; i += blockDim.x) nrow[sh[i]] = srow[i];
    } else {
        for (int i = threadIdx.x; i < kLive; i += blockDim.x) srow[i] = nrow[sh[i]];
    }
}

// =====================================================================================================================
// An agent's answers from its strength-ordered tables, for boards it may hold only as suit-isomorphism classes.  One CTA per
// query board: canonical key -> class (binary search over the agent's sorted keys) -> out[d][h][action] in natural hand
// order for the board's decision nodes.  The canonical key is the minimum over the 24 suit permutations s of the sorted cards
// s(c) = rank * 4 + s[suit] packed base 64 (holdem_boards.canonical_boards); the permutation used is the FIRST minimal one in
// itertools.permutations order, since a class's rows are suit-symmetric only up to rounding.  Hand h on the query board is
// answered by the class's row entry of hand s(h) on the representative.
// =====================================================================================================================
__constant__ int8_t c_suit_perm[24][4] = {
    {0, 1, 2, 3}, {0, 1, 3, 2}, {0, 2, 1, 3}, {0, 2, 3, 1}, {0, 3, 1, 2}, {0, 3, 2, 1}, {1, 0, 2, 3}, {1, 0, 3, 2},
    {1, 2, 0, 3}, {1, 2, 3, 0}, {1, 3, 0, 2}, {1, 3, 2, 0}, {2, 0, 1, 3}, {2, 0, 3, 1}, {2, 1, 0, 3}, {2, 1, 3, 0},
    {2, 3, 0, 1}, {2, 3, 1, 0}, {3, 0, 1, 2}, {3, 0, 2, 1}, {3, 1, 0, 2}, {3, 1, 2, 0}, {3, 2, 0, 1}, {3, 2, 1, 0}};


__device__ __forceinline__ int hand_index(int c1, int c2) {  // c1 < c2, LUT_HOLE_CARDS_2_IDX order
    return c1 * (2 * kDeck - 1 - c1) / 2 + (c2 - c1 - 1);
}

// out_index[q][d], d < SH::n_dec(): the shape's decision nodes in ascending local id (SH::dec_node)
template <class SH>
__global__ void __launch_bounds__(256) policy_query_kernel(const float* __restrict__ rows, const long long* __restrict__ keys,
                                                           const int16_t* __restrict__ pos_hand, int n_cls, int iso,
                                                           const int8_t* __restrict__ boards, const int32_t* __restrict__ out_index,
                                                           unsigned long long act, int n_actions, float* __restrict__ out,
                                                           int* __restrict__ miss) {
    __shared__ short s_pos[kRange];  // hand on the representative -> strength position
    __shared__ long long s_key[24];
    __shared__ int s_perm, s_cls;
    constexpr int kNDec = SH::n_dec();
    const int q = blockIdx.x, tid = threadIdx.x;
    int cards[kBoardCards];
    uint64_t bm = 0;
#pragma unroll
    for (int k = 0; k < kBoardCards; ++k) {
        cards[k] = boards[(size_t)q * kBoardCards + k];
        bm |= 1ull << cards[k];
    }
    if (tid < 24) {
        const int s = iso ? tid : 0;
        int m[kBoardCards];
#pragma unroll
        for (int k = 0; k < kBoardCards; ++k) m[k] = (cards[k] >> 2) * 4 + c_suit_perm[s][cards[k] & 3];
#pragma unroll
        for (int i = 1; i < kBoardCards; ++i)
#pragma unroll
            for (int j = i; j > 0; --j)
                if (m[j] < m[j - 1]) {
                    const int t = m[j];
                    m[j] = m[j - 1];
                    m[j - 1] = t;
                }
        long long key = 0;
#pragma unroll
        for (int k = 0; k < kBoardCards; ++k) key = key * 64 + m[k];
        s_key[tid] = key;
    }
    __syncthreads();
    if (tid == 0) {
        int best = 0;
        if (iso)
            for (int s = 1; s < 24; ++s)
                if (s_key[s] < s_key[best]) best = s;  // strict: the first minimal permutation
        const long long k = s_key[best];
        int lo = 0, hi = n_cls;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (keys[mid] < k) lo = mid + 1;
            else hi = mid;
        }
        s_perm = best;
        s_cls = (lo < n_cls && keys[lo] == k) ? lo : -1;
        if (s_cls < 0) atomicExch(miss, 1);
    }
    for (int h = tid; h < kRange; h += blockDim.x) s_pos[h] = -1;
    __syncthreads();
    const int cls = s_cls, sp = s_perm;
    if (cls >= 0)
        for (int i = tid; i < kLive; i += blockDim.x) s_pos[pos_hand[(size_t)cls * kLive + i]] = (short)i;
    __syncthreads();
    const float* crow = rows + (size_t)(cls < 0 ? 0 : cls) * SH::rows * kLdb;
    for (int h = tid; h < kRange; h += blockDim.x) {
        int c1 = 0;
        while (hand_index(c1 + 1, c1 + 2) <= h) ++c1;  // first card: the largest c1 whose hands start at or before h
        const int c2 = h - hand_index(c1, c1 + 1) + c1 + 1;
        int pos = -1;
        if (cls >= 0 && !(((bm >> c1) | (bm >> c2)) & 1ull)) {
            const int m1 = (c1 >> 2) * 4 + c_suit_perm[sp][c1 & 3], m2 = (c2 >> 2) * 4 + c_suit_perm[sp][c2 & 3];
            pos = s_pos[hand_index(min(m1, m2), max(m1, m2))];
        }
#pragma unroll
        for (int d = 0; d < kNDec; ++d) {
            const int oi = out_index[(size_t)q * kNDec + d];
            if (oi < 0) continue;
            float* o = out + ((size_t)oi * kRange + h) * n_actions;
            for (int a = 0; a < n_actions; ++a) o[a] = 0.0f;
            if (pos < 0) continue;  // blocked hand (or a board the agent does not hold): all zero
            const int n = SH::dec_node(d), fc = SH::first_child(n);
            for (int c = fc; c < fc + SH::n_children(n); ++c)
                o[(act >> (4 * c)) & 0xF] = crow[(size_t)SH::row_of(c) * kLdb + pos];
        }
    }
}

// =====================================================================================================================
// The pre-deal trunk in ONE launch (one CTA): chance-node rows from the fixed-point sums (integer sum over the suit
// permutations), fold terminals, value backup, and - update form - regrets / matching / average of seat p's trunk nodes and
// its new reach rows; evaluation form: values + best response of both seats and the root exploitability.  Same statements as
// the level kernels (ValueFiller.py:64-125, CFRPlus.py:37-87, StrategyFiller.py:118-146) on <= 8 nodes in natural hand order.
// =====================================================================================================================
constexpr int kTrunkThreads = 1024;

__device__ __forceinline__ float trunk_sigma(const prl_trunk_t& t, int src, int fs, int c, int A, int h) {
    if (src == PRL_STRAT_UNIFORM64) return 1.0f / (float)A;
    if (src == PRL_STRAT_AVG_SUM) {  // reach-weighted sums, normalised on the fly (LinearCFR.py:64-71, VanillaCFR.py:65-72)
        float tot = 0.0f;
        for (int k = 0; k < A; ++k) tot += t.avg[(size_t)(fs + k) * t.ld + h];
        return (tot == 0.0f) ? 1.0f / (float)A : t.avg[(size_t)(fs + c) * t.ld + h] / tot;
    }
    const float* tab = (src == PRL_STRAT_F32) ? t.strat : t.avg;
    return tab[(size_t)(fs + c) * t.ld + h];
}

// peers != NULL: the cross-GPU sum is done HERE - every rank's fixed-point vector sits in symmetric (peer-mapped) memory and
// is read over NVLink with coalesced 8-byte loads, rank 0 .. n_peers-1 in order (integers: any order gives the same bits),
// into w_scratch; the caller has placed a cross-rank barrier between the sweep kernels and this launch.
// PRED (PCFR+ update): regrets max(d + R, 0), stored strategy = regret matching of max(R + d, 0), average += s * reach * w_t
// with w_t = disc[2] (no discount)
// RNR (restricted Nash response, t.reach_model): update form, the opponent's reach at the fold terminals is the mixture
// (1 - rnr_p) * free + rnr_p * model; evaluation form, out_expl[2 + p] / out_expl[4 + p] = the root value / best-response
// value of seat p as well
template <bool EVAL, bool PRED = false, bool RNR = false>
__global__ void __launch_bounds__(kTrunkThreads) trunk_kernel(const prl_trunk_t t, const long long* __restrict__ w_total,
                                                              const long long* const* __restrict__ peers, int n_peers,
                                                              long long peer_offset, long long* __restrict__ w_scratch,
                                                              const int16_t* __restrict__ sym_perm, int n_sym, double inv_scale,
                                                              int p_upd, int iter, int delay, float m_old, float m_new, int algo,
                                                              float rw, const float* __restrict__ disc, float* out_expl) {
    __shared__ float ro[kRange + 2];
    __shared__ float cs[64];
    __shared__ float red[32];
    __shared__ double dred[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t N = (size_t)t.n_buf_nodes, ld = (size_t)t.ld;
    const int seat_lo = EVAL ? 0 : p_upd, seat_hi = EVAL ? 1 : p_upd;
    if (peers != nullptr) {
        for (int i = tid; i < (EVAL ? 4 : 1) * kRange; i += kTrunkThreads) {
            long long s = 0;
            for (int r = 0; r < n_peers; ++r) s += peers[r][peer_offset + i];
            w_scratch[i] = s;
        }
        __syncthreads();
        w_total = w_scratch;
    }
    // 1. the chance node's rows
    for (int p = seat_lo; p <= seat_hi; ++p)
        for (int k = 0; k < (EVAL ? 2 : 1); ++k) {
            const long long* W = w_total + (size_t)(EVAL ? (2 * p + k) : 0) * kRange;
            float* dst = (k ? t.ev_br : t.ev) + ((size_t)p * N + t.chance_node) * ld;
            for (int h = tid; h < kRange; h += kTrunkThreads) {
                long long s = 0;
                if (n_sym > 1) {
                    for (int q = 0; q < n_sym; ++q) s += W[sym_perm[(size_t)q * kRange + h]];
                } else {
                    s = W[h];
                }
                dst[h] = (float)((double)s * inv_scale);
            }
        }
    // 2. fold terminals (no board): ValueFiller.py:103-113 for two-card hands
    for (int n = 0; n < t.n_nodes; ++n) {
        if (t.kind[n] != PRL_KIND_FOLD) continue;
        for (int p = seat_lo; p <= seat_hi; ++p) {
            const float* rg = t.reach + ((size_t)(1 - p) * N + n) * ld;
            __syncthreads();
            float part = 0.0f;
            for (int h = tid; h < kRange; h += kTrunkThreads) {
                float r = rg[h];
                if constexpr (RNR && !EVAL)
                    r = __fmaf_rn(t.rnr_p, t.reach_model[((size_t)(1 - p) * N + n) * ld + h], __fmul_rn(1.0f - t.rnr_p, r));
                ro[h] = r;
                part += r;
            }
            for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
            if (lane == 0) red[warp] = part;
            __syncthreads();
            float T = 0.0f;
            for (int w = 0; w < kTrunkThreads / 32; ++w) T += red[w];
            if (tid < kDeck) {  // per-card sums over the lexicographic range layout, fixed order
                float acc = 0.0f;
                const int c = tid;
                for (int r = 0; r < c; ++r) acc += ro[r * (2 * kDeck - 1 - r) / 2 + c - r - 1];
                const int b0 = c * (2 * kDeck - 1 - c) / 2;
                for (int k = 0; k < kDeck - 1 - c; ++k) acc += ro[b0 + k];
                cs[c] = acc;
            }
            __syncthreads();
            const float sc = t.eq_const * t.pot[n] * 0.5f * ((t.acted_last[n] == p) ? -1.0f : 1.0f);
            float* e = t.ev + ((size_t)p * N + n) * ld;
            float* b = t.ev_br + ((size_t)p * N + n) * ld;
            for (int h = tid; h < kRange; h += kTrunkThreads) {
                const float v = (T - cs[t.hand_cards[2 * h]] - cs[t.hand_cards[2 * h + 1]] + ro[h]) * sc;
                e[h] = v;
                if (EVAL) b[h] = v;
            }
        }
    }
    __syncthreads();
    // 3. decision nodes bottom-up, per hand (children have larger ids); 4. regrets / matching / average; 5. reach of seat p
    double ex[2] = {0.0, 0.0}, root_ev[2] = {0.0, 0.0}, root_br[2] = {0.0, 0.0};
    for (int h = tid; h < kRange; h += kTrunkThreads) {
        for (int n = t.n_nodes - 1; n >= 0; --n) {
            const int k = t.kind[n];
            if (k > PRL_KIND_P1) continue;
            const int A = t.n_children[n], fc = t.first_child[n], fs = t.first_slot[n];
            for (int p = seat_lo; p <= seat_hi; ++p) {
                float* ev_p = t.ev + (size_t)p * N * ld;
                float* br_p = t.ev_br + (size_t)p * N * ld;
                float v = 0.0f, b = 0.0f;
                if (k != p) {
                    for (int c = 0; c < A; ++c) v += ev_p[(size_t)(fc + c) * ld + h];
                    if (EVAL)
                        for (int c = 0; c < A; ++c) b += br_p[(size_t)(fc + c) * ld + h];
                } else {
                    for (int c = 0; c < A; ++c) v += trunk_sigma(t, t.mode[p], fs, c, A, h) * ev_p[(size_t)(fc + c) * ld + h];
                    if (EVAL) {
                        b = br_p[(size_t)fc * ld + h];
                        for (int c = 1; c < A; ++c) b = fmaxf(b, br_p[(size_t)(fc + c) * ld + h]);
                    } else if (PRED) {  // PCFR+: the predictions go through `strat`, then are normalised in place
                        float ssum = 0.0f;
                        for (int c = 0; c < A; ++c) {
                            float* rg = t.regret + (size_t)(fs + c) * ld + h;
                            const float d = ev_p[(size_t)(fc + c) * ld + h] - v;
                            const float r = fmaxf(d + *rg, 0.0f);
                            const float q = fmaxf(r + d, 0.0f);
                            *rg = r;
                            t.strat[(size_t)(fs + c) * ld + h] = q;
                            ssum += q;
                        }
                        const float inv = (ssum > 0.0f) ? 1.0f / ssum : 0.0f;
                        for (int c = 0; c < A; ++c) {
                            float* st = t.strat + (size_t)(fs + c) * ld + h;
                            *st = (ssum > 0.0f) ? *st * inv : 1.0f / (float)A;
                        }
                    } else {  // CFRPlus.py:37-63; VanillaCFR.py:26-52 / LinearCFR.py:27-51: weighted, unclipped, matching on the positive part
                        float ssum = 0.0f;
                        for (int c = 0; c < A; ++c) {
                            float* rg = t.regret + (size_t)(fs + c) * ld + h;
                            const float d = ev_p[(size_t)(fc + c) * ld + h] - v;
                            float r = (algo == PRL_ALGO_CFR_PLUS) ? fmaxf(d + *rg, 0.0f) : __fadd_rn(__fmul_rn(rw, d), *rg);
                            if (disc) r = __fmul_rn(r, (r > 0.0f) ? disc[0] : disc[1]);  // DCFR: a_t / b_t
                            *rg = r;
                            ssum += fmaxf(r, 0.0f);
                        }
                        const float inv = (ssum > 0.0f) ? 1.0f / ssum : 0.0f;
                        for (int c = 0; c < A; ++c) {
                            const float r = fmaxf(t.regret[(size_t)(fs + c) * ld + h], 0.0f);
                            t.strat[(size_t)(fs + c) * ld + h] = (ssum > 0.0f) ? r * inv : 1.0f / (float)A;
                        }
                    }
                }
                ev_p[(size_t)n * ld + h] = v;
                if (EVAL) br_p[(size_t)n * ld + h] = b;
            }
        }
        if (EVAL) {
            for (int p = 0; p < 2; ++p)  // ValueFiller.py:95-101 at the root
            {
                ex[p] += (double)t.reach[((size_t)p * N) * ld + h] *
                         ((double)t.ev_br[((size_t)p * N) * ld + h] - (double)t.ev[((size_t)p * N) * ld + h]);
                if constexpr (RNR) {
                    root_ev[p] += (double)t.reach[((size_t)p * N) * ld + h] * (double)t.ev[((size_t)p * N) * ld + h];
                    root_br[p] += (double)t.reach[((size_t)p * N) * ld + h] * (double)t.ev_br[((size_t)p * N) * ld + h];
                }
            }
        } else {
            const int p = p_upd;
            float* rp = t.reach + (size_t)p * N * ld;
            for (int n = 0; n < t.n_nodes; ++n) {  // StrategyFiller.py:118-146 with the new strategy; average CFRPlus.py:65-87
                const int k = t.kind[n];
                if (k > PRL_KIND_P1) continue;
                const int A = t.n_children[n], fc = t.first_child[n], fs = t.first_slot[n];
                const float r = rp[(size_t)n * ld + h];
                for (int c = 0; c < A; ++c) {
                    float s = 1.0f;
                    if (k == p) {
                        s = t.strat[(size_t)(fs + c) * ld + h];
                        float* a = t.avg + (size_t)(fs + c) * ld + h;
                        if (PRED) *a = __fadd_rn(*a, __fmul_rn(__fmul_rn(s, r), disc[2]));  // PCFR+: weight w_t
                        else if (algo != PRL_ALGO_CFR_PLUS)  // VanillaCFR.py:56-59, LinearCFR.py:55-58; DCFR: weight w_t
                            *a = __fadd_rn(*a, __fmul_rn(__fmul_rn(s, r), disc ? disc[2] : rw));
                        else if (iter >= delay) *a = m_old * (*a) + m_new * s;
                    }
                    rp[(size_t)(fc + c) * ld + h] = s * r;
                }
            }
        }
    }
    if (EVAL) {
        for (int p = 0; p < 2; ++p) {
            double v = ex[p];
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            __syncthreads();
            if (lane == 0) dred[warp] = v;
            __syncthreads();
            if (tid == 0) {
                double s = 0.0;
                for (int w = 0; w < kTrunkThreads / 32; ++w) s += dred[w];
                out_expl[p] = (float)s;
            }
        }
        if constexpr (RNR) {
            for (int q = 0; q < 4; ++q) {
                double v = (q < 2) ? root_ev[q] : root_br[q - 2];
                for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                __syncthreads();
                if (lane == 0) dred[warp] = v;
                __syncthreads();
                if (tid == 0) {
                    double s = 0.0;
                    for (int w = 0; w < kTrunkThreads / 32; ++w) s += dred[w];
                    out_expl[2 + q] = (float)s;
                }
            }
        }
    }
}

template <class SH>
bool shape_matches(const prl_board_game_t* g) {
    if (g->n_local != SH::N) return false;
    for (int i = 0; i < SH::N; ++i)
        if (g->kind[i] != SH::kind(i) || g->parent[i] != SH::parent(i) || g->first_child[i] != SH::first_child(i) ||
            g->n_children[i] != SH::n_children(i))
            return false;
    return true;
}

// the table layout the kernel compiles in: row(i, j) = j * SH::rows + row_of(i)
template <class SH>
bool layout_matches(const prl_board_game_t* g) {
    for (int i = 1; i < SH::N; ++i)
        if (g->row0[i] != SH::row_of(i) || g->row_m[i] != SH::rows) return false;
    return true;
}

// f(SH{}) for the compiled shape whose kind / parent / first_child / n_children the descriptor holds; kNoShape if none does
constexpr int kNoShape = -1000;
template <class F>
int with_shape(const prl_board_game_t* g, F&& f) {
    if (!g) return kNoShape;
    if (shape_matches<ShapeFHP>(g)) return f(ShapeFHP{});
    if (shape_matches<ShapeFHPShort>(g)) return f(ShapeFHPShort{});
    return kNoShape;
}

int default_grid() {
    static int cached[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (!cached[dev]) {
        int sms = 132;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cached[dev] = 2 * sms;
    }
    return cached[dev];
}

template <class SH, int P, bool EVAL, bool DEFER = false, bool P1ONLY = false, bool AVG = true, bool PRED = false, int RNR = 0,
          bool BREX = false>
int launch_sweep(const SweepArgs& a, int grid, cudaStream_t s) {
    auto kern = board_sweep_kernel<SH, P, EVAL, DEFER, P1ONLY, AVG, PRED, RNR, BREX>;
    constexpr int kSmemBytes = SweepSmem<SH>::kSmemBytes;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);  // per device: set every time
    if (e != cudaSuccess) return prl::check(e, "prl_board_sweep: shared memory opt-in");
    kern<<<grid, kThreads, kSmemBytes, s>>>(a);
    prl::count_launch();
    return 0;
}

}  // namespace

extern "C" int prl_board_layout(const prl_board_game_t* shape, int32_t* out) {
    int n_local = 0;
    if (shape) {
        n_local = with_shape(shape, [](auto sh) { return decltype(sh)::N; });
        if (n_local == kNoShape) return prl::fail("prl_board_layout: the post-deal subtree has no compiled shape");
    }
    out[0] = kLive;
    out[1] = kLdb;
    out[2] = kBlobBytes;
    out[3] = kRecBytes;            // offset of the hand ids inside a board's blob
    out[4] = kBlobA;               // offset of the card rows
    out[5] = kLiveCards;
    out[6] = kRowPad;
    out[7] = n_local;
    return 0;
}

extern "C" int prl_board_grid(void) { return default_grid(); }

extern "C" int prl_board_rows(const prl_board_game_t* shape, int32_t* row_of, int32_t* rows_per_board) {
    const int rc = with_shape(shape, [&](auto sh) {
        using SH = decltype(sh);
        for (int i = 0; i < 16; ++i) row_of[i] = (i >= 1 && i < SH::N) ? SH::row_of(i) : -1;
        *rows_per_board = SH::rows;
        return 0;
    });
    return rc == kNoShape ? prl::fail("prl_board_rows: the post-deal subtree has no compiled shape") : rc;
}

extern "C" int prl_board_shape_ok(const prl_board_game_t* g) {
    return with_shape(g, [](auto) { return 1; }) == 1 ? 1 : 0;
}

extern "C" int prl_board_build_tables(const int32_t* ranks, const uint64_t* board_mask, const int8_t* hand_cards, int n_boards,
                                      void* blob, prl_stream_t stream) {
    if (n_boards <= 0) return 0;
    board_tables_kernel<<<n_boards, 256, 0, (cudaStream_t)stream>>>(ranks, board_mask, hand_cards, n_boards, (unsigned char*)blob);
    prl::count_launch();
    return prl::check(cudaGetLastError(), "prl_board_build_tables");
}

// CFR+ update, averaging mode: due = iteration of the seat's pending averaging step (-1: none), now = 1: this iteration's step is
// written, 0: it is left pending.  Today's form (-1, 1), deferred (-1, 0), paired (due, 1).
static int board_sweep(const prl_board_game_t* g, int p, int eval, int src_own, int src_opp, const float* trunk_reach_opp, int iter,
                       int delay, int algo, float defer_w, int p1_only, int due, int now, prl_stream_t stream) {
    if (int e = prl::check_algo(algo, g->dcfr, !eval && !p1_only, "prl_board_sweep")) return e;
    const bool pred = algo == PRL_ALGO_PCFR_PLUS;
    if (pred && !g->pred) return prl::fail("prl_board_sweep: PCFR+ needs the prediction table g->pred");
    const bool defer = !eval && algo != PRL_ALGO_CFR_PLUS;
    const bool rnr = g->rnr_reach != nullptr;
    if (rnr && algo != PRL_ALGO_CFR_PLUS) return prl::fail("prl_board_sweep: the restricted Nash response is a CFR+ form");
    if (rnr && !(g->rnr_p >= 0.0f && g->rnr_p <= 1.0f)) return prl::fail("prl_board_sweep: rnr_p must be in [0, 1]");
    const bool brex = g->br_out != nullptr;
    if (brex && (!eval || p1_only || rnr))
        return prl::fail("prl_board_sweep: br_out is written by the evaluation sweep without a restricted Nash response only");
    if (p1_only && !defer && !rnr)
        return prl::fail("prl_board_sweep: p1_only is the average flush of Vanilla / Linear CFR or the model reach of a restricted "
                         "Nash response");
    const int layout_ok = with_shape(g, [&](auto sh) { return layout_matches<decltype(sh)>(g) ? 1 : 0; });
    if (layout_ok == kNoShape) return prl::fail("prl_board_sweep: the post-deal subtree has no compiled shape");
    if (g->n_range != kRange || g->n_deck != kDeck) return prl::fail("prl_board_sweep: 52-card deck / 1326 hands only");
    if (!layout_ok) return prl::fail("prl_board_sweep: row0 / row_m must be the board-major layout of prl_board_rows");
    if (p < 0 || p > 1) return prl::fail("prl_board_sweep: bad seat");
    if (!g->tables || !g->regret || !g->avg || !g->w_private || !g->w_total || !trunk_reach_opp)
        return prl::fail("prl_board_sweep: missing buffers");
    const bool step = now && iter >= delay;  // this iteration's averaging step is written
    if (due != -1 && (due < delay || !step))
        return prl::fail("prl_board_sweep: a pending averaging step (iteration >= delay) is written with this iteration's");
    cudaStream_t s = (cudaStream_t)stream;
    const int grid = g->grid > 0 ? g->grid : default_grid();
    SweepArgs a;
    a.g = *g;
    // PCFR+'s strategies are regret matching of the predictions: the evaluation and the flush read them where the other
    // algorithms read their regrets (their instantiations unchanged); the update form (PRED) reads both tables
    if (pred && (eval || p1_only)) a.g.regret = g->pred;
    a.trunk_reach_opp = trunk_reach_opp;
    a.iter = iter;
    a.delay = delay;
    prl::cfrp_weights(iter, delay, &a.m_old, &a.m_new);
    a.pair = due >= 0;
    a.m_old_due = a.m_new_due = 0.0f;
    if (a.pair) prl::cfrp_weights(due, delay, &a.m_old_due, &a.m_new_due);
    a.src_own = src_own;
    a.src_opp = src_opp;
    a.rw = prl::regret_weight(algo, iter);
    a.disc = prl::dcfr_row(algo, g->dcfr, iter, !eval && !p1_only);
    a.defer_w = defer ? defer_w : 0.0f;
    a.fx_scale = (double)(1ull << g->frac_bits);
    for (int n = 0; n < 16; ++n) {
        const bool folder = n < g->n_local && g->kind[n] == PRL_KIND_FOLD && g->acted_last[n] == p;
        a.sc[n] = (n < g->n_local) ? g->eq_const * g->pot[n] * 0.5f * (folder ? -1.0f : 1.0f) : 0.0f;
    }
    if (p1_only) {
        const int rc1 = with_shape(g, [&](auto sh) {
            using SH = decltype(sh);
            if (rnr) return (p == 0) ? launch_sweep<SH, 0, false, false, true, false, false, kRnrOut>(a, grid, s)
                                     : launch_sweep<SH, 1, false, false, true, false, false, kRnrOut>(a, grid, s);
            return (p == 0) ? launch_sweep<SH, 0, false, true, true>(a, grid, s) : launch_sweep<SH, 1, false, true, true>(a, grid, s);
        });
        return rc1 ? rc1 : prl::check(cudaGetLastError(), "prl_board_sweep(flush)");
    }
    {   // the sums this launch produces: update -> w_total[0]; evaluation of seat p -> w_total[2p], w_total[2p + 1]
        char* base = reinterpret_cast<char*>(g->w_total) + (eval ? sizeof(long long) * 2 * p * kRange : 0);
        if (int e = prl::check(cudaMemsetAsync(base, 0, sizeof(long long) * (eval ? 2 : 1) * kRange, s), "prl_board_sweep: memset")) return e;
    }
    const int rc = with_shape(g, [&](auto sh) {
        using SH = decltype(sh);
        if (eval && rnr) return (p == 0) ? launch_sweep<SH, 0, true, false, false, true, false, kRnrMix>(a, grid, s)
                                         : launch_sweep<SH, 1, true, false, false, true, false, kRnrMix>(a, grid, s);
        if (eval && brex) return (p == 0) ? launch_sweep<SH, 0, true, false, false, true, false, 0, true>(a, grid, s)
                                          : launch_sweep<SH, 1, true, false, false, true, false, 0, true>(a, grid, s);
        if (eval) return (p == 0) ? launch_sweep<SH, 0, true>(a, grid, s) : launch_sweep<SH, 1, true>(a, grid, s);
        if (rnr && step) return (p == 0) ? launch_sweep<SH, 0, false, false, false, true, false, kRnrMix>(a, grid, s)
                                         : launch_sweep<SH, 1, false, false, false, true, false, kRnrMix>(a, grid, s);
        if (rnr) return (p == 0) ? launch_sweep<SH, 0, false, false, false, false, false, kRnrMix>(a, grid, s)
                                 : launch_sweep<SH, 1, false, false, false, false, false, kRnrMix>(a, grid, s);
        if (pred) return (p == 0) ? launch_sweep<SH, 0, false, true, false, true, true>(a, grid, s)
                                  : launch_sweep<SH, 1, false, true, false, true, true>(a, grid, s);
        if (defer) return (p == 0) ? launch_sweep<SH, 0, false, true>(a, grid, s) : launch_sweep<SH, 1, false, true>(a, grid, s);
        if (step) return (p == 0) ? launch_sweep<SH, 0, false>(a, grid, s) : launch_sweep<SH, 1, false>(a, grid, s);
        return (p == 0) ? launch_sweep<SH, 0, false, false, false, false>(a, grid, s)
                        : launch_sweep<SH, 1, false, false, false, false>(a, grid, s);
    });
    if (rc) return rc;
    return prl::check(cudaGetLastError(), "prl_board_sweep");
}

extern "C" int prl_board_sweep(const prl_board_game_t* g, int p, int eval, int src_own, int src_opp, const float* trunk_reach_opp,
                               int iter, int delay, int algo, float defer_w, int p1_only, prl_stream_t stream) {
    return board_sweep(g, p, eval, src_own, src_opp, trunk_reach_opp, iter, delay, algo, defer_w, p1_only, -1, 1, stream);
}

extern "C" int prl_board_update_cfrp(const prl_board_game_t* g, int p, const float* trunk_reach_opp, int iter, int delay, int due,
                                     int now, prl_stream_t stream) {
    return board_sweep(g, p, 0, 0, 0, trunk_reach_opp, iter, delay, PRL_ALGO_CFR_PLUS, 0.0f, 0, due, now, stream);
}

extern "C" int prl_board_avg_flush(const prl_board_game_t* g, int p, int due, int delay, prl_stream_t stream) {
    const int layout_ok = with_shape(g, [&](auto sh) { return layout_matches<decltype(sh)>(g) ? 1 : 0; });
    if (layout_ok != 1) return prl::fail("prl_board_avg_flush: not a compiled shape / layout");
    if (p < 0 || p > 1) return prl::fail("prl_board_avg_flush: bad seat");
    if (due < delay) return prl::fail("prl_board_avg_flush: no averaging step before iteration delay");
    if (!g->regret || !g->avg) return prl::fail("prl_board_avg_flush: missing buffers");
    if (g->n_boards <= 0) return 0;
    float m_old, m_new;
    prl::cfrp_weights(due, delay, &m_old, &m_new);
    cudaStream_t s = (cudaStream_t)stream;
    with_shape(g, [&](auto sh) {
        using SH = decltype(sh);
        if (p == 0) avg_flush_kernel<SH, 0><<<g->n_boards, 256, 0, s>>>(g->regret, g->avg, m_old, m_new);
        else avg_flush_kernel<SH, 1><<<g->n_boards, 256, 0, s>>>(g->regret, g->avg, m_old, m_new);
        return 0;
    });
    prl::count_launch();
    return prl::check(cudaGetLastError(), "prl_board_avg_flush");
}

#if PRL_BV_STAMPS
// phase stamps of the last board_sweep_kernel launch (see stamp()): out[kStampCtas][kStampUnits][kStampSlots] int64, then cleared;
// shape[3] = the three dimensions.  Exported by PRL_BV_STAMPS builds only.
extern "C" int prl_board_stamps(int64_t* out, int32_t* shape) {
    shape[0] = kStampCtas;
    shape[1] = kStampUnits;
    shape[2] = kStampSlots;
    if (int e = prl::check(cudaMemcpyFromSymbol(out, g_stamps, sizeof(g_stamps)), "prl_board_stamps: copy")) return e;
    static const long long zeros[kStampCtas * kStampUnits * kStampSlots] = {};
    return prl::check(cudaMemcpyToSymbol(g_stamps, zeros, sizeof(g_stamps)), "prl_board_stamps: clear");
}
#endif

extern "C" int prl_board_collect(const prl_board_game_t* g, int n_arr, const int16_t* sym_perm, int n_sym, float* out, int ld,
                                 prl_stream_t stream) {
    if (!g || n_arr < 1 || n_arr > 4) return prl::fail("prl_board_collect: bad arguments");
    board_collect_kernel<<<(kRange + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const long long*>(g->w_total), n_arr, sym_perm, n_sym, 1.0 / (double)(1ull << g->frac_bits), out, ld);
    prl::count_launch();
    return prl::check(cudaGetLastError(), "prl_board_collect");
}

extern "C" int prl_board_permute(const prl_board_game_t* g, int rows_per_board, const int64_t* row_src, const int64_t* row_dst,
                                 float* sorted_tab, float* natural_tab, int ld, int to_natural, prl_stream_t stream) {
    if (g && with_shape(g, [](auto) { return 0; }) == kNoShape)
        return prl::fail("prl_board_permute: the post-deal subtree has no compiled shape");
    if (!g || g->n_boards <= 0 || rows_per_board <= 0) return 0;
    board_permute_kernel<<<g->n_boards * rows_per_board, 256, 0, (cudaStream_t)stream>>>(
        (const unsigned char*)g->tables, g->n_boards, rows_per_board, row_src, row_dst, sorted_tab, natural_tab, ld, to_natural);
    prl::count_launch();
    return prl::check(cudaGetLastError(), "prl_board_permute");
}

extern "C" int prl_board_policy_query(const prl_board_game_t* shape, const float* rows, const int64_t* keys, const int16_t* pos_hand,
                                      int n_cls, int iso, const int8_t* boards, int n_boards, const int32_t* out_index,
                                      uint64_t actions, int n_actions, float* out, int32_t* miss, prl_stream_t stream) {
    if (with_shape(shape, [](auto) { return 0; }) == kNoShape)
        return prl::fail("prl_board_policy_query: the post-deal subtree has no compiled shape");
    if (n_boards <= 0) return 0;
    if (!rows || !keys || !pos_hand || n_cls <= 0 || !boards || !out_index || !out || !miss)
        return prl::fail("prl_board_policy_query: missing buffers");
    if (n_actions < 1 || n_actions > 16) return prl::fail("prl_board_policy_query: 1..16 actions");
    const int rc = with_shape(shape, [&](auto sh) {
        using SH = decltype(sh);
        for (int c = 1; c < SH::N; ++c)
            if (SH::kind(SH::parent(c)) <= 1 && (int)((actions >> (4 * c)) & 0xF) >= n_actions)
                return prl::fail("prl_board_policy_query: an action id is out of range");
        policy_query_kernel<SH><<<n_boards, 256, 0, (cudaStream_t)stream>>>(rows, reinterpret_cast<const long long*>(keys), pos_hand,
                                                                            n_cls, iso, boards, out_index, (unsigned long long)actions,
                                                                            n_actions, out, reinterpret_cast<int*>(miss));
        return 0;
    });
    if (rc) return rc;
    prl::count_launch();
    return prl::check(cudaGetLastError(), "prl_board_policy_query");
}

// Trunk of seat p's half-iteration (eval == 0) or of an evaluation of both seats (eval != 0) in one launch; see prl_trunk_t.
extern "C" int prl_board_trunk(const prl_board_game_t* g, const prl_trunk_t* t, int eval, int p, int n_sym, const int16_t* sym_perm,
                               int iter, int delay, float* out_expl, const int64_t* const* peers, int n_peers,
                               int64_t peer_offset, int64_t* w_scratch, int algo, prl_stream_t stream) {
    if (int e = prl::check_algo(algo, g ? g->dcfr : nullptr, !eval, "prl_board_trunk")) return e;
    if (!g || !t || t->n_nodes < 1 || t->n_nodes > 8) return prl::fail("prl_board_trunk: 1..8 trunk nodes");
    const float rw = prl::regret_weight(algo, iter);
    const bool pred = algo == PRL_ALGO_PCFR_PLUS && !eval;  // PCFR+ update: w_t from the factor table, no discount
    const float* disc = pred ? g->dcfr + 3 * (size_t)iter : prl::dcfr_row(algo, g->dcfr, iter, !eval);
    if (with_shape(g, [](auto) { return 0; }) == kNoShape) return prl::fail("prl_board_trunk: the post-deal subtree has no compiled shape");
    if (t->n_range != kRange || g->n_deck != kDeck) return prl::fail("prl_board_trunk: 52-card deck / 1326 hands only");
    if (eval && !out_expl) return prl::fail("prl_board_trunk: out_expl missing");
    for (int n = 0; n < t->n_nodes; ++n)
        if (t->kind[n] == PRL_KIND_SHOWDOWN || t->kind[n] == PRL_KIND_SHOWDOWN_ALLIN)
            return prl::fail("prl_board_trunk: showdowns before the deal are not supported");
    float m_old, m_new;
    prl::cfrp_weights(iter, delay, &m_old, &m_new);
    const double inv_scale = 1.0 / (double)(1ull << g->frac_bits);
    const long long* w = reinterpret_cast<const long long*>(g->w_total);
    if (peers && (n_peers < 1 || !w_scratch)) return prl::fail("prl_board_trunk: peer sum needs n_peers >= 1 and w_scratch");
    const long long* const* pp = reinterpret_cast<const long long* const*>(peers);
    long long* ws = reinterpret_cast<long long*>(w_scratch);
    const bool rnr = t->reach_model != nullptr;
    if (rnr && (algo != PRL_ALGO_CFR_PLUS || !(t->rnr_p >= 0.0f && t->rnr_p <= 1.0f)))
        return prl::fail("prl_board_trunk: the restricted Nash response is a CFR+ form with rnr_p in [0, 1]");
    if (rnr)
        (eval ? trunk_kernel<true, false, true> : trunk_kernel<false, false, true>)<<<1, kTrunkThreads, 0, (cudaStream_t)stream>>>(
            *t, w, pp, n_peers, (long long)peer_offset, ws, sym_perm, n_sym, inv_scale, eval ? -1 : p, iter, delay, m_old, m_new, algo,
            rw, disc, out_expl);
    else if (eval)
        trunk_kernel<true><<<1, kTrunkThreads, 0, (cudaStream_t)stream>>>(*t, w, pp, n_peers, (long long)peer_offset, ws, sym_perm, n_sym,
                                                                       inv_scale, -1, iter, delay, m_old, m_new, algo, rw, disc, out_expl);
    else if (pred)
        trunk_kernel<false, true><<<1, kTrunkThreads, 0, (cudaStream_t)stream>>>(*t, w, pp, n_peers, (long long)peer_offset, ws, sym_perm,
                                                                              n_sym, inv_scale, p, iter, delay, m_old, m_new, algo, rw, disc,
                                                                              out_expl);
    else
        trunk_kernel<false><<<1, kTrunkThreads, 0, (cudaStream_t)stream>>>(*t, w, pp, n_peers, (long long)peer_offset, ws, sym_perm, n_sym,
                                                                        inv_scale, p, iter, delay, m_old, m_new, algo, rw, disc, out_expl);
    prl::count_launch();
    return prl::check(cudaGetLastError(), "prl_board_trunk");
}
