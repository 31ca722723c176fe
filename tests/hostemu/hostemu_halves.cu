// hostemu_halves.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.  Never linked into librpt_b200.so, never loaded by rpt_b200/*:
// only tests/test_halves.py builds and loads it (`make hostemu`, tests/hostemu/_build/libhostemu_halves.so).
//
// The error estimate's per-pixel functions (halves.h) compiled for the host and run as halves.cu's kernels run them:
// the demodulation with u, one a-trous pass with u, and E.  -ffp-contract=off, as the device's -fmad=false.
#include "../../rpt_b200/csrc/halves.h"

using namespace rptb;

extern "C" {

// halves_demodulate_kernel on n pixels: col (3n), var (n), u (3n).
void hostemu_halves_demodulate(const double* sums, const double* m2, const double* half, const uint32_t* counts, uint64_t n,
                               const double* albedo, double eps_a, double* col, double* var, double* u) {
    for (uint64_t p = 0; p < n; p++) {
        denoise_demodulate(sums + 3 * p, m2[p], counts[p], albedo + 3 * p, eps_a, col + 3 * p, var + p);
        halves_u(sums + 3 * p, half + 3 * p, counts[p], albedo + 3 * p, eps_a, u + 3 * p);
    }
}

// One pass (halves_pixel at every pixel) with step h.
void hostemu_halves_pass(const double* col, const double* var, const double* u, const double* nrm, const double* depth, const double* albedo,
                         uint32_t width, uint32_t height, uint32_t h, const rptb_denoise* d, double* out_col, double* out_var, double* out_u) {
#pragma omp parallel for schedule(static)
    for (int64_t y = 0; y < (int64_t)height; y++)
        for (uint32_t x = 0; x < width; x++) {
            const size_t p = (size_t)y * width + x;
            halves_pixel(col, var, u, nrm, depth, albedo, width, height, x, (uint32_t)y, h, *d, out_col + 3 * p, out_var + p, out_u + 3 * p);
        }
}

// One plain pass (denoise_pixel at every pixel), for the bit-for-bit comparison with halves_pixel's colour and variance.
void hostemu_halves_plain_pass(const double* col, const double* var, const double* nrm, const double* depth, const double* albedo,
                               uint32_t width, uint32_t height, uint32_t h, const rptb_denoise* d, double* out_col, double* out_var) {
    for (uint32_t y = 0; y < height; y++)
        for (uint32_t x = 0; x < width; x++) {
            const size_t p = (size_t)y * width + x;
            denoise_pixel(col, var, nrm, depth, albedo, width, height, x, y, h, *d, out_col + 3 * p, out_var + p);
        }
}

// E (halves_error) at every pixel from the last pass's U.
void hostemu_halves_error(const double* U, const double* albedo, uint32_t width, uint32_t height, double eps_a, double* E) {
    for (uint32_t y = 0; y < height; y++)
        for (uint32_t x = 0; x < width; x++) E[(size_t)y * width + x] = halves_error(U, albedo, width, height, x, y, eps_a);
}

}  // extern "C"
