// C shim around openrl_b200/csrc/orl_deep_core.h with a DiagGaussian head, for the CPU test (g++ -O2 -shared -fPIC).
#include "orl_deep_core.h"
using namespace orl_deep;

extern "C" {
int shim_gauss_param_count(int d, int n) { return deep_offsets(d, n, true).total; }
int shim_gauss_logstd_offset(int d, int n) { return logstd_offset(deep_offsets(d, n, true)); }
int shim_gauss_tape_width() { return tape_width(true); }
int shim_gauss_dls_field() { return TS_DLS; }

// rows independent forwards (value, mean) and the backward tape rows from dL/dvalue and dL/dmean; the rows' dL/dlogstd
// go into the TS_DLS field, zero beyond n, as share_fwdbwd_kernel writes them
void shim_gauss_rows(const float* P, int d, int n, int act, int rows, const float* X, float* values, float* means,
                     const float* dvalue, const float* dmean, const float* dlogstd, float* tape) {
    const Offsets o = deep_offsets(d, n, true);
    const int W = tape_width(true);
    for (int r = 0; r < rows; ++r) {
        Save sv;
        float* tp = tape + (size_t)r * W;
        deep_forward(P, o, act, X + r * d, values + r, means + r * n, &sv, tp);
        deep_backward(P, o, act, sv, dvalue[r], dmean + r * n, tp);
        for (int j = 0; j < 8; ++j) tp[TS_DLS + j] = j < n ? dlogstd[r * n + j] : 0.f;
    }
}
}
