// hostemu_cross.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.  Never linked into librpt_b200.so, never loaded by rpt_b200/*:
// only tests/test_denoise_cross.py builds and loads it (`make hostemu`, tests/hostemu/_build/libhostemu_cross.so).
//
// The cross-filtered denoiser's per-pixel functions (cross.h) compiled for the host and run as cross.cu's kernels run
// them: the demodulation of the halves, m_k, one level's argmin step and one level's blend.  -ffp-contract=off, as the
// device's -fmad=false.  The chains' passes are halves.h's, emulated by libhostemu_halves.so.
#include "../../rpt_b200/csrc/cross.h"

using namespace rptb;

extern "C" {

// cross_demodulate_kernel on n pixels: iA (3n), vA (n), iB (3n), vB (n).
void hostemu_cross_demodulate(const double* sums, const double* m2, const double* half, const uint32_t* counts, uint64_t n,
                              const double* albedo, double eps_a, double* iA, double* vA, double* iB, double* vB) {
    for (uint64_t p = 0; p < n; p++)
        cross_demodulate(sums + 3 * p, half + 3 * p, m2[p], counts[p], albedo + 3 * p, eps_a, iA + 3 * p, vA + p, iB + 3 * p, vB + p);
}

// cross_m_kernel on n pixels: m (n).
void hostemu_cross_m(const double* XA, const double* XB, const double* iA0, const double* iB0, const double* vA, const double* vB,
                     const uint32_t* counts, const double* albedo, uint64_t n, double eps_a, double* m) {
    for (uint64_t p = 0; p < n; p++)
        m[p] = cross_m(XA + 3 * p, XB + 3 * p, iA0 + 3 * p, iB0 + 3 * p, vA[p], vB[p], counts[p], albedo + 3 * p, eps_a);
}

// cross_level_kernel at every pixel for level k: best_M, level updated in place.
void hostemu_cross_level(const double* m, uint32_t width, uint32_t height, uint32_t k, double* best_M, uint8_t* level) {
    for (uint32_t y = 0; y < height; y++)
        for (uint32_t x = 0; x < width; x++) {
            const size_t p = (size_t)y * width + x;
            cross_level(m, width, height, x, y, k, best_M + p, level + p);
        }
}

// cross_blend_kernel at every pixel for level k: out (3 per pixel), M_hat updated in place.
void hostemu_cross_blend(const uint8_t* level, const double* m, const double* XA, const double* XB, const double* sums, const uint32_t* counts,
                         const double* albedo, uint32_t width, uint32_t height, uint32_t k, double eps_a, double* out, double* M_hat) {
#pragma omp parallel for schedule(static)
    for (int64_t y = 0; y < (int64_t)height; y++)
        for (uint32_t x = 0; x < width; x++) {
            const size_t p = (size_t)y * width + x;
            cross_blend(level, m, XA, XB, sums, counts, albedo, width, height, x, (uint32_t)y, k, eps_a, out + 3 * p, M_hat + p);
        }
}

}  // extern "C"
