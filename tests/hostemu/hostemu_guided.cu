// hostemu_guided.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.  Never linked into librpt_b200.so, never loaded by rpt_b200/*:
// only tests/test_guided.py builds and loads it (`make hostemu`, tests/hostemu/_build/libhostemu_guided.so).
//
// The guided criterion's per-pixel and per-slot functions (guided.h) compiled for the host, on top of the denoiser's
// emulation (hostemu_denoise.cu, included whole: its demodulation and passes give the planes the criterion reads).  Same
// switches as hostemu.cu.
#include "../../rpt_b200/csrc/guided.h"
#include "hostemu_denoise.cu"

extern "C" {

// guided_active at each of n row-major pixels: counts, the last pass's col (3 per pixel) and var, albedo (3 per pixel).
// out: 1 where the pixel takes the next entry.
void hostemu_guided_pixels(const uint32_t* counts, const double* col, const double* var, const double* albedo, uint64_t n, double eps_a,
                           const rptb_adaptive* crit, uint8_t* out) {
    for (uint64_t p = 0; p < n; p++) out[p] = guided_active(counts[p], col + 3 * p, albedo + 3 * p, eps_a, var[p], *crit) ? 1u : 0u;
}

// guided_slot at every slot of part (index, count)'s `tiles` owned tiles, as guided_mark_kernel runs it: mask (tiles*128),
// flags (tiles*4, one per 8x4 warp block that has an active slot); returns the active slots.
uint64_t hostemu_guided_part(const double* col, const double* var, const double* albedo, const uint32_t* counts, uint32_t width,
                             uint32_t height, uint32_t index, uint32_t count, uint32_t tiles, double eps_a, const rptb_adaptive* crit,
                             uint8_t* mask, uint8_t* flags) {
    uint64_t active = 0;
    for (uint32_t k = 0; k < tiles; k++)
        for (uint32_t w = 0; w < 4; w++) {
            bool any = false;
            for (uint32_t l = 0; l < 32; l++) {
                const uint32_t j = w * 32u + l;
                const bool on = guided_slot(col, var, albedo, counts, width, height, index, count, k, j, eps_a, *crit);
                mask[(uint64_t)k * 128u + j] = on ? 1u : 0u;
                any = any || on;
                active += on ? 1u : 0u;
            }
            flags[(uint64_t)k * 4u + w] = any ? 1u : 0u;
        }
    return active;
}

}  // extern "C"
