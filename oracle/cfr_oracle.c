/*
 * CPU restatement (plain C) of the reference's tabular CFR / public-tree value path.  TEST INFRASTRUCTURE ONLY:
 * used by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs; never linked into or
 * called from the product library.
 *
 * Parity status: PINNED.  tests/test_oracle_c.py checks this file bit-for-bit against fixtures produced by running
 * the reference itself (oracle/gen_golden_cfr.py), exactly like oracle/cfr_numpy.py.
 *
 * It walks the same depth-sorted arrays as the product (`prl_tree_t` / `prl_buffers_t` from include/pokerrl_b200.h,
 * here with HOST pointers) level by level; every float expression keeps the reference's dtype and operation order
 * (compile with -ffp-contract=off).  OpenMP over the nodes of a level gives the multi-threaded CPU baseline.
 *
 * Reference statements (paths under PokerRL/):
 *   reach      game/_/tree/_/StrategyFiller.py:118-146, 148-169      value   game/_/tree/_/ValueFiller.py:21-175
 *   regrets    cfr/_CFRBase.py:146-185 + cfr/{CFRPlus.py:37-41,LinearCFR.py:27-31,VanillaCFR.py:26-30}
 *   matching   cfr/CFRPlus.py:43-63, LinearCFR.py:33-51, VanillaCFR.py:32-52
 *   averaging  cfr/CFRPlus.py:65-87, LinearCFR.py:53-76, VanillaCFR.py:54-77
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "pokerrl_b200.h"

#ifdef _OPENMP
#include <omp.h>
#endif

/* number of host threads used by the level loops (0 = OpenMP default); returns the count in effect */
int orc_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
    return omp_get_max_threads();
#else
    (void)n;
    return 1;
#endif
}

typedef struct {
    const prl_tree_t* T;
    const prl_buffers_t* B;
    int mask, mode[2];
    int algo, upd_p, iter, delay, avg_f64;
} ctx_t;

static int is_f32(int m) { return m == PRL_STRAT_F32 || m == PRL_STRAT_AVG_F32; }

static float strat_f32(const ctx_t* c, int m, int slot, int h) {
    const float* tab = (m == PRL_STRAT_F32) ? c->B->strat : (const float*)c->B->avg;
    return tab[(size_t)slot * c->T->ld + h];
}

static double strat_f64(const ctx_t* c, int m, int slot, int fs, int A, int h) {
    const int ld = c->T->ld;
    if (m == PRL_STRAT_UNIFORM64) return 1.0 / (double)A; /* StrategyFiller.py:61-62 */
    if (m == PRL_STRAT_AVG_F64) return ((const double*)c->B->avg)[(size_t)slot * ld + h];
    const float* tab = (const float*)c->B->avg; /* LinearCFR.py:64-71 */
    float s = tab[(size_t)fs * ld + h];
    for (int k = 1; k < A; ++k) s = s + tab[(size_t)(fs + k) * ld + h];
    if (s == 0.0f) return 1.0 / (double)A;
    return (double)(tab[(size_t)slot * ld + h] / s);
}

/* np.sum's order over a contiguous float32 row of n >= 1 elements: numpy's pairwise_sum (loops_utils.h.src), restated
 * in oracle/pairwise_sum.py.  Fewer than 8 elements in order; up to 128, 8 interleaved partial sums combined as
 * ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the last n % 8 elements in order; above 128, the two halves split at
 * n/2 rounded down to a multiple of 8.  np.sum adds the total to +0.0, which only changes the sign of a -0.0 total;
 * that add is left out, as in the kernels. */
float orc_pairwise_sum(const float* a, int n) {
    if (n < 8) {
        float s = a[0];
        for (int i = 1; i < n; ++i) s = s + a[i];
        return s;
    }
    if (n <= 128) {
        float r[8];
        for (int j = 0; j < 8; ++j) r[j] = a[j];
        int i = 8;
        for (; i < n - n % 8; i += 8)
            for (int j = 0; j < 8; ++j) r[j] = r[j] + a[i + j];
        float s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
        for (; i < n; ++i) s = s + a[i];
        return s;
    }
    int n2 = n / 2;
    n2 -= n2 % 8;
    return orc_pairwise_sum(a, n2) + orc_pairwise_sum(a + n2, n - n2);
}

static int leduc_rank(const prl_tree_t* T, int h, int b) { /* game_rules.py:68-75 */
    int r = h / T->n_suits;
    return (b / T->n_suits == r) ? T->pair_bonus + r : r;
}

/* ------------------------------------------------------------------------------------------ reach, one node */
static void reach_node(const ctx_t* c, int n, int update_avg) {
    const prl_tree_t* T = c->T;
    const int R = T->n_range, ld = T->ld;
    const size_t N = (size_t)T->n_nodes;
    const int par = T->parent[n];
    for (int q = 0; q < 2; ++q) {
        if (!(c->mask & (1 << q))) continue;
        float* reach_q = c->B->reach + (size_t)q * N * ld;
        for (int h = 0; h < R; ++h) {
            float r;
            if (par < 0) {
                r = (float)(1.0 / (double)R); /* PublicTree.py:122-124 */
            } else {
                const float rp = reach_q[(size_t)par * ld + h];
                const int pk = T->kind[par];
                if (pk == PRL_KIND_CHANCE) { /* StrategyFiller.py:137-140, 159-166 */
                    const float cp = (h == T->board[n]) ? 0.0f : (float)(1.0 / (double)(T->n_deck - 2));
                    r = rp * cp;
                } else if (pk == q) { /* StrategyFiller.py:129-134 */
                    const int slot = T->slot[n];
                    const int m = c->mode[q];
                    if (is_f32(m)) {
                        const float s = strat_f32(c, m, slot, h);
                        r = s * rp;
                        if (update_avg && q == c->upd_p) {
                            if (c->algo == PRL_ALGO_CFR_PLUS) { /* CFRPlus.py:65-87 */
                                if (c->iter >= c->delay) {
                                    const long long cw = ((long long)c->iter * (c->iter + 1) -
                                                          (long long)c->delay * (c->delay + 1)) / 2;
                                    const long long nw = (long long)c->iter - c->delay + 1;
                                    const double m_old = (double)cw / (double)(cw + nw);
                                    const double m_new = (double)nw / (double)(cw + nw);
                                    if (c->avg_f64) {
                                        double* a = (double*)c->B->avg + (size_t)slot * ld + h;
                                        *a = m_old * (*a) + m_new * (double)s;
                                    } else {
                                        float* a = (float*)c->B->avg + (size_t)slot * ld + h;
                                        *a = (float)m_old * (*a) + (float)m_new * s;
                                    }
                                }
                            } else { /* VanillaCFR.py:57-62, LinearCFR.py:56-61 */
                                float contrib = r;
                                if (c->algo == PRL_ALGO_LINEAR) contrib = contrib * (float)(c->iter + 1);
                                float* a = (float*)c->B->avg + (size_t)slot * ld + h;
                                *a = *a + contrib;
                            }
                        }
                    } else {
                        const int fs = T->slot[T->first_child[par]];
                        r = (float)(strat_f64(c, m, slot, fs, T->n_children[par], h) * (double)rp);
                    }
                } else {
                    r = rp;
                }
            }
            reach_q[(size_t)n * ld + h] = r;
        }
    }
}

/* ------------------------------------------------------------------------------------------ terminals */
static float showdown_row(const prl_tree_t* T, const float* ro, int h, int b) { /* ValueFiller.py:140-155 */
    float eq = 0.0f;
    if (h != b) {
        const int rh = leduc_rank(T, h, b);
        for (int j = 0; j < T->n_range; ++j) {
            if (j == h || j == b) continue;
            const int rj = leduc_rank(T, j, b);
            if (rh > rj) eq = eq + ro[j];
            else if (rh < rj) eq = eq - ro[j];
        }
    }
    return eq;
}

static float terminal_equity(const ctx_t* c, int n, int h, int p, int kind) {
    const prl_tree_t* T = c->T;
    const int R = T->n_range, ld = T->ld;
    const float* ro = c->B->reach + ((size_t)(1 - p) * T->n_nodes + n) * ld;
    const float K = (float)((double)T->n_deck / (double)(T->n_deck - 1)); /* ValueFiller.py:19 */
    const int b = T->board[n];
    float eq;
    if (kind == PRL_KIND_FOLD) { /* ValueFiller.py:103-125 (np.sum over the opponent's hands) */
        eq = orc_pairwise_sum(ro, R) - ro[h];
        if (T->acted_last[n] == p) eq = -eq;
        eq = eq * K;
    } else if (kind == PRL_KIND_SHOWDOWN) { /* ValueFiller.py:127-158 */
        eq = showdown_row(T, ro, h, b) * K;
    } else { /* ValueFiller.py:160-175 */
        eq = 0.0f;
        for (int bb = 0; bb < T->n_deck; ++bb) eq = eq + showdown_row(T, ro, h, bb) * K;
        eq = eq / (float)(T->n_deck - 2);
    }
    if (h == b) eq = 0.0f; /* ValueFiller.py:57-59 */
    return eq;
}

/* ------------------------------------------------------------------------------------------ value, one node */
static void value_node(const ctx_t* c, int n, int with_br, int update) {
    const prl_tree_t* T = c->T;
    const int R = T->n_range, ld = T->ld;
    const size_t N = (size_t)T->n_nodes;
    const int kind = T->kind[n], fc = T->first_child[n], A = T->n_children[n];
    for (int p = 0; p < 2; ++p) {
        if (!(c->mask & (1 << p))) continue;
        float* ev_p = c->B->ev + (size_t)p * N * ld;
        float* evbr_p = with_br ? c->B->ev_br + (size_t)p * N * ld : NULL;
        for (int h = 0; h < R; ++h) {
            float v, vbr = 0.0f;
            if (kind >= PRL_KIND_FOLD) {
                v = terminal_equity(c, n, h, p, kind) * T->pot[n] / 2.0f; /* ValueFiller.py:61 */
                vbr = v;
            } else if (kind == PRL_KIND_CHANCE || kind != p) { /* ValueFiller.py:76-78, 88-90 */
                v = ev_p[(size_t)fc * ld + h];
                for (int k = 1; k < A; ++k) v = v + ev_p[(size_t)(fc + k) * ld + h];
                if (with_br) {
                    vbr = evbr_p[(size_t)fc * ld + h];
                    for (int k = 1; k < A; ++k) vbr = vbr + evbr_p[(size_t)(fc + k) * ld + h];
                }
            } else { /* ValueFiller.py:87, 91 */
                const int fs = T->slot[fc];
                const int m = c->mode[p];
                if (is_f32(m)) {
                    v = strat_f32(c, m, fs, h) * ev_p[(size_t)fc * ld + h];
                    for (int k = 1; k < A; ++k) v = v + strat_f32(c, m, fs + k, h) * ev_p[(size_t)(fc + k) * ld + h];
                } else {
                    double acc = strat_f64(c, m, fs, fs, A, h) * (double)ev_p[(size_t)fc * ld + h];
                    for (int k = 1; k < A; ++k)
                        acc = acc + strat_f64(c, m, fs + k, fs, A, h) * (double)ev_p[(size_t)(fc + k) * ld + h];
                    v = (float)acc;
                }
                if (with_br) {
                    vbr = evbr_p[(size_t)fc * ld + h];
                    for (int k = 1; k < A; ++k) vbr = fmaxf(vbr, evbr_p[(size_t)(fc + k) * ld + h]);
                }
                if (update && p == c->upd_p) {
                    float* reg = c->B->regret;
                    float* st = c->B->strat;
                    const float w = (float)(c->iter + 1);
                    float s = 0.0f;
                    for (int k = 0; k < A; ++k) {
                        const size_t off = (size_t)(fs + k) * ld + h;
                        const float d = ev_p[(size_t)(fc + k) * ld + h] - v;
                        float r;
                        if (c->algo == PRL_ALGO_CFR_PLUS) r = fmaxf(d + reg[off], 0.0f);
                        else if (c->algo == PRL_ALGO_LINEAR) r = w * d + reg[off];
                        else r = d + reg[off];
                        reg[off] = r;
                        const float rp = fmaxf(r, 0.0f);
                        s = (k == 0) ? rp : s + rp;
                    }
                    const float uni = (float)(1.0 / (double)A);
                    for (int k = 0; k < A; ++k) {
                        const size_t off = (size_t)(fs + k) * ld + h;
                        st[off] = (s > 0.0f) ? fmaxf(reg[off], 0.0f) / s : uni;
                    }
                }
            }
            ev_p[(size_t)n * ld + h] = v;
            if (with_br) evbr_p[(size_t)n * ld + h] = vbr;
        }
    }
}

/* ------------------------------------------------------------------------------------------ passes */
static void reach_levels(const ctx_t* c, int update_avg) {
    const prl_tree_t* T = c->T;
    for (int d = 0; d < T->n_levels; ++d) {
        const int lo = (int)T->level_start[d], hi = (int)T->level_start[d + 1];
#pragma omp parallel for schedule(static)
        for (int n = lo; n < hi; ++n) reach_node(c, n, update_avg);
    }
}

static void value_levels(const ctx_t* c, int with_br, int update) {
    const prl_tree_t* T = c->T;
    for (int d = T->n_levels - 1; d >= 0; --d) {
        const int lo = (int)T->level_start[d], hi = (int)T->level_start[d + 1];
#pragma omp parallel for schedule(static)
        for (int n = lo; n < hi; ++n) value_node(c, n, with_br, update);
    }
}

int orc_reach_pass(const prl_tree_t* tree, const prl_buffers_t* buf, int player_mask, const int* strat_mode) {
    ctx_t c = {tree, buf, player_mask, {strat_mode[0], strat_mode[1]}, 0, -1, 0, 0, 0};
    reach_levels(&c, 0);
    return 0;
}

int orc_value_pass(const prl_tree_t* tree, const prl_buffers_t* buf, int player_mask, int with_br,
                   const int* strat_mode) {
    ctx_t c = {tree, buf, player_mask, {strat_mode[0], strat_mode[1]}, 0, -1, 0, 0, 0};
    value_levels(&c, with_br, 0);
    return 0;
}

int orc_root_exploitability(const prl_tree_t* T, const prl_buffers_t* B, float* out) { /* ValueFiller.py:95-101 */
    const size_t N = (size_t)T->n_nodes;
    for (int p = 0; p < 2; ++p) {
        const float* ev = B->ev + (size_t)p * N * T->ld;
        const float* evbr = B->ev_br + (size_t)p * N * T->ld;
        const float* reach = B->reach + (size_t)p * N * T->ld;
        float e[T->n_range];
        for (int h = 0; h < T->n_range; ++h) e[h] = evbr[h] * reach[h] - ev[h] * reach[h];
        out[p] = orc_pairwise_sum(e, T->n_range); /* np.sum(node.epsilon, axis=1) */
    }
    return 0;
}

/* _CFRBase.py:123-128 for one seat p */
int orc_cfr_half_iteration(const prl_tree_t* tree, const prl_buffers_t* buf, int algo, int p, int iter, int delay,
                           int avg_f64, const int* strat_mode) {
    ctx_t c = {tree, buf, 1 << p, {strat_mode[0], strat_mode[1]}, algo, p, iter, delay, avg_f64};
    value_levels(&c, 0, 1);
    c.mode[p] = PRL_STRAT_F32;
    reach_levels(&c, 1);
    return 0;
}
