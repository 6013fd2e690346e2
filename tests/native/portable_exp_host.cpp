// Host build of the device exp (csrc/portable_exp.h) for the CPU test-suite; compiled with -ffp-contract=off, as the kernels
// are compiled with -fmad=false.
#include "portable_exp.h"
using namespace b200flow;

extern "C" void pexp_batch(const double* x, int64_t n, double* out) {
    for (int64_t i = 0; i < n; ++i) out[i] = portable_exp(x[i]);
}
