/*
 * CPU restatement (plain C, float64, OpenMP) of the tabular CFR / value / best-response path for TWO-HOLE-CARD games.
 * TEST INFRASTRUCTURE ONLY: used by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs; never linked into or called from the product library.
 *
 * Parity status: the reference cannot run Hold'em trees (ValueFiller.py:18-19, PublicTree.py:193-203), so there is no
 * reference `node.ev` to compare with.  This file is pinned (tests/test_oracle_twocard_rows.py, tests/test_oracle_cfr2_c.py)
 *   - on its terminal rows against tests/golden/twocard_rows.npz: brute-force O(R^2) float64 evaluation of
 *     ValueFiller.py:103-158 generalised per SURVEY.md appendix A, with hand strengths produced by the reference's own
 *     lib_hand_eval.so (oracle/gen_golden_twocard.py), and
 *   - on whole sweeps / iterations against oracle/cfr2_numpy.py (dense sign matrices), which reproduces the reference's
 *     one-card values in the one-card limit (tests/test_oracle_cfr2.py).
 *
 * Same statements as oracle/cfr2_numpy.py, level by level over the flat tree (reach StrategyFiller.py:118-146, 148-169;
 * values + BR ValueFiller.py:21-101; regrets _CFRBase.py:146-185 with CFRPlus.py:37-41 / LinearCFR.py:27-31 /
 * VanillaCFR.py:26-30; matching CFRPlus.py:43-63; averaging CFRPlus.py:65-87 / LinearCFR.py:53-76 / VanillaCFR.py:54-77),
 * but the showdown row is evaluated in O(R) by ONE SWEEP OVER THE HANDS IN STRENGTH ORDER with running per-card sums
 * (the textbook serial formulation - deliberately a different algorithm from the CUDA kernels' parallel prefix scans):
 *     win[h]  = (mass of strictly weaker live hands) - (same restricted to hands holding c1(h)) - (... holding c2(h))
 *     lose[h] likewise from the strong end;  eq[h] = K * (win[h] - lose[h]);  ties add 0 (ValueFiller.py:151-155).
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

enum { K_P0 = 0, K_P1 = 1, K_CHANCE = 2, K_FOLD = 3, K_SHOWDOWN = 4, K_SHOWDOWN_ALLIN = 5 };
enum { ALGO_VANILLA = 0, ALGO_CFR_PLUS = 1, ALGO_LINEAR = 2 };

typedef struct {
    int32_t n_nodes, n_levels, n_slots, R, n_deck, n_boards, n_sym, pad;
    const int64_t* level_start; /* [n_levels + 1] */
    const int32_t* parent;
    const int32_t* first_child;
    const int32_t* n_children;
    const int32_t* slot;       /* table row of a node as child of a decision node */
    const int32_t* board;      /* global board id of the node, -1 = none */
    const int8_t* kind;
    const int8_t* acted_last;
    const double* pot;
    const int8_t* hand_cards;  /* [R][2] */
    const int32_t* board_ranks;  /* [n_boards][R]; -1 = hand holds a board card (or board incomplete) */
    const uint8_t* board_blocked; /* [n_boards][R] */
    const double* board_prob;
    const double* board_mult;
    const int16_t* sym_perm;   /* [n_sym][R] or NULL */
    int32_t* board_order;      /* [n_boards][R] scratch: live hands in ascending strength (filled by orc2_prepare) */
    int32_t* board_nlive;      /* [n_boards] */
    double K;
    double* reach; /* [n_nodes][2][R] */
    double* ev;
    double* ev_br;
    double* regret; /* [n_slots][R] */
    double* strat;
    double* avg;    /* CFR+: average strategy; Vanilla / Linear: reach-weighted sums */
} orc2_t;

int orc2_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
    return omp_get_max_threads();
#else
    (void)n;
    return 1;
#endif
}

/* ---- sort the live hands of one board by strength (ties keep hand order) */
typedef struct { int32_t rank, hand; } rk_t;
static int cmp_rk(const void* a, const void* b) {
    const rk_t* x = (const rk_t*)a; const rk_t* y = (const rk_t*)b;
    if (x->rank != y->rank) return x->rank < y->rank ? -1 : 1;
    return x->hand < y->hand ? -1 : (x->hand > y->hand);
}
static int sort_board(const int32_t* ranks, int R, int32_t* order) {
    rk_t* tmp = (rk_t*)malloc(sizeof(rk_t) * (size_t)R);
    int n = 0;
    for (int h = 0; h < R; ++h)
        if (ranks[h] >= 0) { tmp[n].rank = ranks[h]; tmp[n].hand = h; ++n; }
    qsort(tmp, (size_t)n, sizeof(rk_t), cmp_rk);
    for (int i = 0; i < n; ++i) order[i] = tmp[i].hand;
    free(tmp);
    return n;
}

void orc2_prepare(orc2_t* t) {
#pragma omp parallel for schedule(dynamic, 16)
    for (int b = 0; b < t->n_boards; ++b)
        t->board_nlive[b] = sort_board(t->board_ranks + (size_t)b * t->R, t->R, t->board_order + (size_t)b * t->R);
}

/* ---- terminal rows (unit pot: the caller multiplies by pot / 2); ro = opponent reach, out[h] for every hand */
void orc2_fold_row(int R, int n_deck, const int8_t* hc, const uint8_t* blocked, const double* ro, double K, double* out) {
    double cs[64];
    double T = 0.0;
    for (int c = 0; c < n_deck; ++c) cs[c] = 0.0;
    for (int h = 0; h < R; ++h) {
        T += ro[h];
        cs[hc[2 * h]] += ro[h];
        cs[hc[2 * h + 1]] += ro[h];
    }
    for (int h = 0; h < R; ++h)
        out[h] = (blocked && blocked[h]) ? 0.0 : K * (T - cs[hc[2 * h]] - cs[hc[2 * h + 1]] + ro[h]);
}

void orc2_showdown_row(int R, int n_deck, const int8_t* hc, const int32_t* ranks, const int32_t* order, int n_live,
                       const double* ro, double K, double* out) {
    double cs[64], tot;
    for (int h = 0; h < R; ++h) out[h] = 0.0;
    /* weak -> strong: mass of strictly weaker compatible hands */
    tot = 0.0;
    for (int c = 0; c < n_deck; ++c) cs[c] = 0.0;
    for (int i = 0; i < n_live;) {
        int j = i;
        while (j < n_live && ranks[order[j]] == ranks[order[i]]) ++j;
        for (int k = i; k < j; ++k) {
            const int h = order[k];
            out[h] += tot - cs[hc[2 * h]] - cs[hc[2 * h + 1]];
        }
        for (int k = i; k < j; ++k) {
            const int h = order[k];
            tot += ro[h];
            cs[hc[2 * h]] += ro[h];
            cs[hc[2 * h + 1]] += ro[h];
        }
        i = j;
    }
    /* strong -> weak: minus the mass of strictly stronger compatible hands */
    tot = 0.0;
    for (int c = 0; c < n_deck; ++c) cs[c] = 0.0;
    for (int i = n_live - 1; i >= 0;) {
        int j = i;
        while (j >= 0 && ranks[order[j]] == ranks[order[i]]) --j;
        for (int k = i; k > j; --k) {
            const int h = order[k];
            out[h] -= tot - cs[hc[2 * h]] - cs[hc[2 * h + 1]];
        }
        for (int k = i; k > j; --k) {
            const int h = order[k];
            tot += ro[h];
            cs[hc[2 * h]] += ro[h];
            cs[hc[2 * h + 1]] += ro[h];
        }
        i = j;
    }
    for (int h = 0; h < R; ++h) out[h] *= K;
}

#define ROW(arr, n, p) ((arr) + ((size_t)(n) * 2 + (p)) * (size_t)t->R)

/* ---- strategies */
void orc2_fill_uniform(orc2_t* t) {
    for (int n = 0; n < t->n_nodes; ++n) {
        if (t->kind[n] > K_P1 || t->n_children[n] == 0) continue;
        const int A = t->n_children[n], fs = t->slot[t->first_child[n]];
        for (int a = 0; a < A; ++a)
            for (int h = 0; h < t->R; ++h) t->strat[(size_t)(fs + a) * t->R + h] = 1.0 / (double)A;
    }
}

/* ---- top-down reach of both seats; use_avg: strategies come from `avg` (the caller normalised it) */
void orc2_reach(orc2_t* t, const double* strat) {
    const int R = t->R;
    for (int p = 0; p < 2; ++p)
        for (int h = 0; h < R; ++h) {
            double r = 1.0 / (double)R; /* PublicTree.py:122-124 */
            if (t->board[0] >= 0 && t->board_blocked[(size_t)t->board[0] * R + h]) r = 0.0;
            ROW(t->reach, 0, p)[h] = r;
        }
    for (int d = 0; d + 1 < t->n_levels; ++d) {
        const int lo = (int)t->level_start[d], hi = (int)t->level_start[d + 1];
#pragma omp parallel for schedule(dynamic, 64)
        for (int n = lo; n < hi; ++n) {
            const int A = t->n_children[n];
            if (A == 0) continue;
            const int fc = t->first_child[n], k = t->kind[n];
            for (int a = 0; a < A; ++a) {
                const int c = fc + a;
                for (int p = 0; p < 2; ++p) {
                    const double* src = ROW(t->reach, n, p);
                    double* dst = ROW(t->reach, c, p);
                    if (k == K_CHANCE) { /* StrategyFiller.py:137-140, 159-166 */
                        const int b = t->board[c];
                        const uint8_t* bl = t->board_blocked + (size_t)b * R;
                        const double pr = t->board_prob[b];
                        for (int h = 0; h < R; ++h) dst[h] = bl[h] ? 0.0 : src[h] * pr;
                    } else if (k == p) { /* StrategyFiller.py:129-134 */
                        const double* s = strat + (size_t)t->slot[c] * R;
                        for (int h = 0; h < R; ++h) dst[h] = s[h] * src[h];
                    } else {
                        memcpy(dst, src, sizeof(double) * (size_t)R);
                    }
                }
            }
        }
    }
}

/* ---- bottom-up values (+ best response if with_br) of the seats in mask (ValueFiller.py:21-101); fills ev / ev_br.
 * The reference always evaluates both seats with BR (mask 3, with_br 1); the lean form is what a CFR half-iteration needs.
 * orc2_values_levels sweeps levels d_hi .. 0 only and, if keep_chance, leaves the chance nodes' rows as the caller set them:
 * the trunk of a game whose chance-node rows were summed elsewhere (oracle/cfr2_chunked.py). */
void orc2_values_levels(orc2_t* t, const double* strat, int mask, int with_br, int d_hi, int keep_chance) {
    const int R = t->R;
    for (int d = d_hi; d >= 0; --d) {
        const int lo = (int)t->level_start[d], hi = (int)t->level_start[d + 1];
#pragma omp parallel for schedule(dynamic, 16)
        for (int n = lo; n < hi; ++n) {
            const int k = t->kind[n], A = t->n_children[n], fc = t->first_child[n];
            if (k >= K_FOLD) {
                const int b = t->board[n];
                const double half_pot = t->pot[n] / 2.0;
                for (int p = 0; p < 2; ++p) {
                    if (!(mask & (1 << p))) continue;
                    const double* ro = ROW(t->reach, n, 1 - p);
                    double* e = ROW(t->ev, n, p);
                    if (k == K_FOLD) {
                        orc2_fold_row(R, t->n_deck, t->hand_cards, b >= 0 ? t->board_blocked + (size_t)b * R : NULL, ro,
                                      t->K, e);
                        const double sgn = (t->acted_last[n] == p) ? -half_pot : half_pot; /* ValueFiller.py:112,124 */
                        for (int h = 0; h < R; ++h) e[h] *= sgn;
                    } else {
                        orc2_showdown_row(R, t->n_deck, t->hand_cards, t->board_ranks + (size_t)b * R,
                                          t->board_order + (size_t)b * R, t->board_nlive[b], ro, t->K, e);
                        for (int h = 0; h < R; ++h) e[h] *= half_pot;
                    }
                    if (with_br) memcpy(ROW(t->ev_br, n, p), e, sizeof(double) * (size_t)R);
                }
                continue;
            }
            if (k == K_CHANCE) { /* ValueFiller.py:76-78 with board weights; suit symmetrisation (DESIGN.md) */
                if (keep_chance) continue;
                double* w = (double*)malloc(sizeof(double) * (size_t)R * 2);
                for (int p = 0; p < 2; ++p)
                    for (int br = 0; br < (with_br ? 2 : 1); ++br) {
                        if (!(mask & (1 << p))) continue;
                        double* arr = br ? t->ev_br : t->ev;
                        double* acc = w;
                        for (int h = 0; h < R; ++h) acc[h] = 0.0;
                        for (int a = 0; a < A; ++a) {
                            const double m = t->board_mult[t->board[fc + a]];
                            const double* src = ROW(arr, fc + a, p);
                            for (int h = 0; h < R; ++h) acc[h] += m * src[h];
                        }
                        double* dst = ROW(arr, n, p);
                        if (t->n_sym > 1) {
                            for (int h = 0; h < R; ++h) {
                                double s = 0.0;
                                for (int q = 0; q < t->n_sym; ++q) s += acc[t->sym_perm[(size_t)q * R + h]];
                                dst[h] = s;
                            }
                        } else {
                            memcpy(dst, acc, sizeof(double) * (size_t)R);
                        }
                    }
                free(w);
                continue;
            }
            const int fs = t->slot[fc];
            for (int q = 0; q < 2; ++q) {
                if (!(mask & (1 << q))) continue;
                double* evq = ROW(t->ev, n, q);
                double* brq = ROW(t->ev_br, n, q);
                for (int h = 0; h < R; ++h) {
                    double v = 0.0, b = (q == k) ? -INFINITY : 0.0;
                    for (int a = 0; a < A; ++a) {
                        const double e = ROW(t->ev, fc + a, q)[h];
                        v += (q == k) ? strat[(size_t)(fs + a) * R + h] * e : e;
                        if (with_br) {
                            const double x = ROW(t->ev_br, fc + a, q)[h];
                            if (q == k) b = (x > b) ? x : b; else b += x;
                        }
                    }
                    evq[h] = v;
                    if (with_br) brq[h] = b;
                }
            }
        }
    }
}

void orc2_values(orc2_t* t, const double* strat, int mask, int with_br) {
    orc2_values_levels(t, strat, mask, with_br, t->n_levels - 1, 0);
}

/* strategy = regret matching of the stored regrets at every decision node (CFRPlus.py:43-63) */
void orc2_regret_match(orc2_t* t) {
    const int R = t->R;
#pragma omp parallel for schedule(dynamic, 64)
    for (int n = 0; n < t->n_nodes; ++n) {
        if (t->kind[n] > K_P1 || t->n_children[n] == 0) continue;
        const int A = t->n_children[n], fs = t->slot[t->first_child[n]];
        for (int h = 0; h < R; ++h) {
            double s = 0.0;
            for (int a = 0; a < A; ++a) s += fmax(t->regret[(size_t)(fs + a) * R + h], 0.0);
            for (int a = 0; a < A; ++a) {
                const double r = fmax(t->regret[(size_t)(fs + a) * R + h], 0.0);
                t->strat[(size_t)(fs + a) * R + h] = (s > 0.0) ? r / s : 1.0 / (double)A;
            }
        }
    }
}

/* root exploitability per seat (ValueFiller.py:95-101) */
void orc2_exploitability(const orc2_t* t, double* out) {
    for (int p = 0; p < 2; ++p) {
        double s = 0.0;
        for (int h = 0; h < t->R; ++h) s += (ROW(t->ev_br, 0, p)[h] - ROW(t->ev, 0, p)[h]) * ROW(t->reach, 0, p)[h];
        out[p] = s;
    }
}

/* regret update + regret matching at seat p's nodes (needs ev under the pre-update profile) */
void orc2_regret_update(orc2_t* t, int p, int algo, int iter) {
    const int R = t->R;
#pragma omp parallel for schedule(dynamic, 64)
    for (int n = 0; n < t->n_nodes; ++n) {
        if (t->kind[n] != p || t->n_children[n] == 0) continue;
        const int A = t->n_children[n], fc = t->first_child[n], fs = t->slot[fc];
        const double* evn = ROW(t->ev, n, p);
        for (int h = 0; h < R; ++h) {
            double s = 0.0;
            for (int a = 0; a < A; ++a) {
                const double dlt = ROW(t->ev, fc + a, p)[h] - evn[h];
                double* rg = t->regret + (size_t)(fs + a) * R + h;
                double r;
                if (algo == ALGO_CFR_PLUS) r = fmax(dlt + *rg, 0.0);       /* CFRPlus.py:37-41 */
                else if (algo == ALGO_LINEAR) r = (double)(iter + 1) * dlt + *rg; /* LinearCFR.py:27-31 */
                else r = dlt + *rg;                                          /* VanillaCFR.py:26-30 */
                *rg = r;
                s += fmax(r, 0.0);
            }
            for (int a = 0; a < A; ++a) { /* CFRPlus.py:43-63 */
                const double r = fmax(t->regret[(size_t)(fs + a) * R + h], 0.0);
                t->strat[(size_t)(fs + a) * R + h] = (s > 0.0) ? r / s : 1.0 / (double)A;
            }
        }
    }
}

/* average-strategy update of seat p's nodes (reach must be current under the new strategy) */
void orc2_avg_update(orc2_t* t, int p, int algo, int iter, int delay) {
    const int R = t->R;
    double m_old = 0.0, m_new = 1.0;
    if (algo == ALGO_CFR_PLUS && iter > delay) { /* CFRPlus.py:68-73 */
        const double cw = 0.5 * ((double)iter * (iter + 1) - (double)delay * (delay + 1));
        const double nw = (double)iter - delay + 1;
        m_old = cw / (cw + nw);
        m_new = nw / (cw + nw);
    }
    if (algo == ALGO_CFR_PLUS && iter < delay) return;
#pragma omp parallel for schedule(dynamic, 64)
    for (int n = 0; n < t->n_nodes; ++n) {
        if (t->kind[n] != p || t->n_children[n] == 0) continue;
        const int A = t->n_children[n], fs = t->slot[t->first_child[n]];
        const double* rp = ROW(t->reach, n, p);
        for (int a = 0; a < A; ++a) {
            double* av = t->avg + (size_t)(fs + a) * R;
            const double* s = t->strat + (size_t)(fs + a) * R;
            for (int h = 0; h < R; ++h) {
                if (algo == ALGO_CFR_PLUS) av[h] = m_old * av[h] + m_new * s[h];
                else av[h] += s[h] * rp[h] * (algo == ALGO_LINEAR ? (double)(iter + 1) : 1.0);
            }
        }
    }
}

/* out[slot][h] = normalised average strategy (LinearCFR.py:64-71: uniform where the sum is 0); CFR+: copy of avg */
void orc2_average_strategy(const orc2_t* t, int algo, double* out) {
    const int R = t->R;
    if (algo == ALGO_CFR_PLUS) {
        memcpy(out, t->avg, sizeof(double) * (size_t)t->n_slots * R);
        return;
    }
#pragma omp parallel for schedule(dynamic, 64)
    for (int n = 0; n < t->n_nodes; ++n) {
        if (t->kind[n] > K_P1 || t->n_children[n] == 0) continue;
        const int A = t->n_children[n], fs = t->slot[t->first_child[n]];
        for (int h = 0; h < R; ++h) {
            double s = 0.0;
            for (int a = 0; a < A; ++a) s += t->avg[(size_t)(fs + a) * R + h];
            for (int a = 0; a < A; ++a)
                out[(size_t)(fs + a) * R + h] = (s == 0.0) ? 1.0 / (double)A : t->avg[(size_t)(fs + a) * R + h] / s;
        }
    }
}
