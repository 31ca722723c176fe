// halves.cu -- the error estimate of the denoised image from two half buffers (rptb_buffer_denoise_error,
// rptb_sample_into_guided_error).  Compiled with -fmad=false: halves.h rounds every operation on its own, as its host
// emulation and tests/halves_ref.py do.
//
// Everything runs on parts[0]'s device over the gathered row-major state (api.cu), like the denoiser (denoise.cu): one
// kernel demodulates the colour and variance and forms u, one per a-trous pass carries colour, variance and u through
// the filter's weights (ping-pong planes), and one forms E.  One thread per pixel.  The selection of each pixel's pass
// count (select.cu) runs the demodulation and the passes through the same launchers.
#include <cuda_runtime.h>

#include "halves.h"

namespace rptb {

__global__ void halves_demodulate_kernel(const double* __restrict__ sums, const double* __restrict__ m2, const double* __restrict__ half,
                                         const uint32_t* __restrict__ counts, uint64_t npix, const double* __restrict__ albedo,
                                         double eps_a, double* __restrict__ col, double* __restrict__ var, double* __restrict__ u) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npix) return;
    denoise_demodulate(sums + 3 * p, m2[p], counts[p], albedo + 3 * p, eps_a, col + 3 * p, var + p);
    halves_u(sums + 3 * p, half + 3 * p, counts[p], albedo + 3 * p, eps_a, u + 3 * p);
}

__global__ void __launch_bounds__(256) halves_pass_kernel(const double* __restrict__ col, const double* __restrict__ var,
                                                          const double* __restrict__ u, const double* __restrict__ nrm,
                                                          const double* __restrict__ depth, const double* __restrict__ albedo,
                                                          uint32_t width, uint32_t height, uint32_t h, const rptb_denoise d,
                                                          double* __restrict__ out_col, double* __restrict__ out_var,
                                                          double* __restrict__ out_u) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    const size_t p = (size_t)y * width + x;
    halves_pixel(col, var, u, nrm, depth, albedo, width, height, x, y, h, d, out_col + 3 * p, out_var + p, out_u + 3 * p);
}

__global__ void halves_error_kernel(const double* __restrict__ U, const double* __restrict__ albedo, uint32_t width, uint32_t height,
                                    double eps_a, double* __restrict__ E) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    E[(size_t)y * width + x] = halves_error(U, albedo, width, height, x, y, eps_a);
}

// The demodulation with u: col, var, u (level 0 of the filter) from sums / m2 / half / counts.
void launch_halves_demodulate(const double* sums, const double* m2, const double* half, const uint32_t* counts, const double* albedo,
                              uint32_t width, uint32_t height, double eps_a, double* col, double* var, double* u, cudaStream_t stream) {
    const uint64_t npix = (uint64_t)width * height;
    halves_demodulate_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, stream>>>(sums, m2, half, counts, npix, albedo, eps_a, col, var, u);
}

// Pass k (step 2^k) with u, from col / var / u into out_col / out_var / out_u.
void launch_halves_pass(const double* col, const double* var, const double* u, const double* nrm, const double* depth, const double* albedo,
                        uint32_t width, uint32_t height, uint32_t k, const rptb_denoise& d, double* out_col, double* out_var, double* out_u,
                        cudaStream_t stream) {
    const dim3 block(32, 8), grid2((width + 31) / 32, (height + 7) / 8);
    halves_pass_kernel<<<grid2, block, 0, stream>>>(col, var, u, nrm, depth, albedo, width, height, 1u << k, d, out_col, out_var, out_u);
}

// The filter with the estimate: sums / m2 / half / counts and the resolved features in; d.iterations (> 0) passes over the
// ping-pong planes col[2], var[2], u[2]; E (width*height) out.  *out_col: the plane holding the last pass's i' (what the
// guided mark remodulates for m').  *launches: kernels enqueued.
cudaError_t launch_halves_error(const double* sums, const double* m2, const double* half, const uint32_t* counts, const double* nrm,
                                const double* depth, const double* albedo, uint32_t width, uint32_t height, const rptb_denoise& d,
                                double* const col[2], double* const var[2], double* const u[2], double* E, const double** out_col,
                                cudaStream_t stream, uint32_t* launches) {
    launch_halves_demodulate(sums, m2, half, counts, albedo, width, height, d.albedo_eps, col[0], var[0], u[0], stream);
    const dim3 block(32, 8), grid2((width + 31) / 32, (height + 7) / 8);
    uint32_t cur = 0;
    for (uint32_t k = 0; k < d.iterations; k++, cur ^= 1u)
        launch_halves_pass(col[cur], var[cur], u[cur], nrm, depth, albedo, width, height, k, d, col[cur ^ 1u], var[cur ^ 1u], u[cur ^ 1u],
                           stream);
    halves_error_kernel<<<grid2, block, 0, stream>>>(u[cur], albedo, width, height, d.albedo_eps, E);
    *out_col = col[cur];
    *launches = 2u + d.iterations;
    return cudaGetLastError();
}

}  // namespace rptb
