// Shared by the pokerrl_b200 CUDA library: error reporting for the C ABI, and the CFR algorithms' rules on the host (entry
// points) and in the level sweeps (cfr_levels.cu and cfr_twocard.cu compile them with their own flags).
#pragma once
#include <cuda_runtime.h>

#include "pokerrl_b200.h"

namespace prl {
// Stores `msg` for prl_last_error() and returns a non-zero status.
int fail(const char* msg);
// cudaSuccess -> 0; otherwise records "<where>: <cuda error string>" and returns the CUDA error code.
int check(cudaError_t e, const char* where);
// counts kernel launches issued by this library (prl_launch_count())
void count_launch();

// 0 if `algo` is a PRL_ALGO_* code and, where the call updates, DCFR / PCFR+ have the factor table; otherwise fails naming
// `where`
int check_algo(int algo, const float* dcfr, bool updates, const char* where);
// CFR+'s averaging weights of iteration iter (CFRPlus.py:68-73): (0, 1) at iter == delay, whose step copies the strategy
// (and below delay, which has no step)
inline void cfrp_weights(int iter, int delay, float* m_old, float* m_new) {
    const double cw = 0.5 * ((double)iter * (iter + 1) - (double)delay * (delay + 1));
    const double nw = (double)iter - delay + 1;
    *m_old = (iter > delay) ? (float)(cw / (cw + nw)) : 0.0f;
    *m_new = (iter > delay) ? (float)(nw / (cw + nw)) : 1.0f;
}
// weight of iteration iter's instantaneous regret: Linear CFR's iter + 1, otherwise 1
inline float regret_weight(int algo, int iter) { return (algo == PRL_ALGO_LINEAR) ? (float)(iter + 1) : 1.0f; }
// DCFR's factor row {a_t, b_t, w_t} of iteration iter in `dcfr` where the call updates (nullptr otherwise: no discount)
inline const float* dcfr_row(int algo, const float* dcfr, int iter, bool updates) {
    return (algo == PRL_ALGO_DCFR && updates) ? dcfr + 3 * (size_t)iter : nullptr;
}

// the level sweeps' regret update of iteration c.iter (Ctx: a sweep context with algo, iter and B, the prl_buffers_t):
// Linear CFR's weight iter + 1, DCFR's discounts of positive / negative sums
struct RegretW {
    float w, a, b;
};
template <typename Ctx>
__device__ __forceinline__ RegretW regret_w(const Ctx& c) {
    RegretW r{(float)(c.iter + 1), 1.0f, 1.0f};
    if (c.algo == PRL_ALGO_DCFR) {
        r.a = c.B.dcfr[3 * (size_t)c.iter];
        r.b = c.B.dcfr[3 * (size_t)c.iter + 1];
    }
    return r;
}

// new regret of one (row, hand) from the instantaneous regret d = v(child) - v(node) and the stored regret
__device__ __forceinline__ float regret_step(int algo, float d, float old, const RegretW& w) {
    if (algo == PRL_ALGO_CFR_PLUS) return fmaxf(d + old, 0.0f);  // CFRPlus.py:37-41
    if (algo == PRL_ALGO_LINEAR) return w.w * d + old;           // LinearCFR.py:27-31
    if (algo == PRL_ALGO_DCFR) {                                 // discounted after this iteration's regret is added
        const float x = d + old;
        return x * ((x > 0.0f) ? w.a : w.b);
    }
    return d + old;                                              // VanillaCFR.py:26-30
}

// PCFR+ (the level sweeps' PRED instantiations): the regret is CFR+'s, r_new = max(d + R_old, 0), and regret matching reads
// the prediction max(r_new + d, 0) - the last instantaneous regret added to the new regret - instead of r_new
__device__ __forceinline__ float pcfr_regret(float d, float old) { return fmaxf(d + old, 0.0f); }
__device__ __forceinline__ float pcfr_prediction(float r_new, float d) { return fmaxf(r_new + d, 0.0f); }
}  // namespace prl
