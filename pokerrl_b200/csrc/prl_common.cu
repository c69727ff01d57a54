// Error reporting, ABI version and the algorithm check for the pokerrl_b200 C ABI (include/pokerrl_b200.h).
#include <stdio.h>
#include <string.h>

#include "pokerrl_b200.h"
#include "prl_common.cuh"

namespace {
thread_local char g_err[512] = "";
unsigned long long g_launches = 0;
}

namespace prl {
int fail(const char* msg) {
    strncpy(g_err, msg, sizeof(g_err) - 1);
    g_err[sizeof(g_err) - 1] = 0;
    return -1;
}
int check(cudaError_t e, const char* where) {
    if (e == cudaSuccess) return 0;
    snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
    return (int)e;
}
void count_launch() { ++g_launches; }

int check_algo(int algo, const float* dcfr, bool updates, const char* where) {
    char msg[256];
    if (algo < PRL_ALGO_VANILLA || algo > PRL_ALGO_PCFR_PLUS) snprintf(msg, sizeof(msg), "%s: bad algo %d", where, algo);
    else if (updates && algo == PRL_ALGO_DCFR && !dcfr) snprintf(msg, sizeof(msg), "%s: DCFR needs the factor table dcfr", where);
    else if (updates && algo == PRL_ALGO_PCFR_PLUS && !dcfr)
        snprintf(msg, sizeof(msg), "%s: PCFR+ needs the weight table dcfr (w_t in column 2)", where);
    else return 0;
    return fail(msg);
}
}  // namespace prl

extern "C" int prl_abi_version(void) { return PRL_ABI_VERSION; }
extern "C" const char* prl_last_error(void) { return g_err; }
extern "C" unsigned long long prl_launch_count(void) { return g_launches; }
