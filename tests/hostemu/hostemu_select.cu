// hostemu_select.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.  Never linked into librpt_b200.so, never loaded by rpt_b200/*:
// only tests/test_denoise_select.py builds and loads it (`make hostemu`, tests/hostemu/_build/libhostemu_select.so).
//
// The selection's per-pixel functions (select.h) compiled for the host and run as select.cu's kernels run them: m_k,
// and one level's smoothing and update.  -ffp-contract=off, as the device's -fmad=false.  The demodulation and the
// passes are halves.h's, emulated by libhostemu_halves.so.
#include "../../rpt_b200/csrc/select.h"

using namespace rptb;

extern "C" {

// select_m_kernel on n pixels: m (n).
void hostemu_select_m(const double* ik, const double* Uk, const double* i0, const double* u0, const double* albedo, uint64_t n, double eps_a,
                      double* m) {
    for (uint64_t p = 0; p < n; p++) m[p] = select_m(ik + 3 * p, Uk + 3 * p, i0 + 3 * p, u0 + 3 * p, albedo + 3 * p, eps_a);
}

// select_level_kernel at every pixel for level k: best (3 per pixel), best_M, level updated in place.
void hostemu_select_level(const double* m, const double* ik, const double* albedo, const double* sums, const uint32_t* counts, uint32_t width,
                          uint32_t height, uint32_t k, double eps_a, double* best, double* best_M, uint8_t* level) {
#pragma omp parallel for schedule(static)
    for (int64_t y = 0; y < (int64_t)height; y++)
        for (uint32_t x = 0; x < width; x++) {
            const size_t p = (size_t)y * width + x;
            select_level(m, ik, albedo, sums, counts, width, height, x, (uint32_t)y, k, eps_a, best + 3 * p, best_M + p, level + p);
        }
}

}  // extern "C"
