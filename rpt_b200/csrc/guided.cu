// guided.cu -- which pixels a guided adaptive call renders (rptb_sample_into_guided).  Compiled with -fmad=false, so
// guided_active (guided.h) rounds every product and sum on its own, as the host emulation and numpy do.
//
// The filter has run over the gathered row-major state on parts[0]'s device (denoise.cu, launch_denoise_passes).  Per
// buffer part, one CTA per owned 16x8 tile maps each compact slot to its pixel, evaluates the test there, and writes the
// part's pixel mask and one flag per 8x4 warp block, and counts the active pixels -- what adaptive_mark_kernel writes,
// so the part's select, list render and masked accumulate run unchanged (adaptive.cu, api.cu).
#include "guided.h"

namespace rptb {

__global__ void __launch_bounds__(128) guided_mark_kernel(const double* __restrict__ col, const double* __restrict__ var,
                                                          const double* __restrict__ albedo, const uint32_t* __restrict__ counts,
                                                          uint32_t width, uint32_t height, uint32_t index, uint32_t count,
                                                          double eps_a, const rptb_adaptive crit, uint8_t* __restrict__ mask,
                                                          uint8_t* __restrict__ flags, unsigned long long* __restrict__ active_pixels) {
    const uint32_t k = blockIdx.x, j = threadIdx.x;
    const bool on = guided_slot(col, var, albedo, counts, width, height, index, count, k, j, eps_a, crit);
    mask[(uint64_t)k * 128u + j] = on ? 1u : 0u;
    const unsigned votes = __ballot_sync(0xffffffffu, on);
    if ((j & 31u) == 0) {
        flags[(uint64_t)k * 4u + (j >> 5)] = votes != 0u ? 1u : 0u;
        if (votes) atomicAdd(active_pixels, (unsigned long long)__popc(votes));
    }
}

// The mask (tiles*128) and flags (tiles*4) of part (index, count) and its active pixel count, which is zeroed first.
cudaError_t launch_guided_mark(const double* col, const double* var, const double* albedo, const uint32_t* counts, uint32_t width,
                               uint32_t height, uint32_t index, uint32_t count, uint32_t tiles, double eps_a, const rptb_adaptive& crit,
                               uint8_t* mask, uint8_t* flags, unsigned long long* active_pixels, cudaStream_t stream) {
    const cudaError_t e = cudaMemsetAsync(active_pixels, 0, sizeof(unsigned long long), stream);
    if (e != cudaSuccess || tiles == 0) return e;
    guided_mark_kernel<<<tiles, 128, 0, stream>>>(col, var, albedo, counts, width, height, index, count, eps_a, crit, mask, flags,
                                                  active_pixels);
    return cudaGetLastError();
}

}  // namespace rptb
