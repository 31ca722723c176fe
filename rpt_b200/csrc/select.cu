// select.cu -- the per-pixel choice of the filter's pass count from a half-buffer estimate of each level's error
// (rptb_buffer_denoise_select).  Compiled with -fmad=false: select.h rounds every operation on its own, as its host
// emulation and tests/select_ref.py do.
//
// Everything runs on parts[0]'s device over the gathered row-major state (api.cu), like the error estimate (halves.cu),
// whose demodulation and pass kernels it runs unchanged.  The demodulated level 0 (i_0, v_0, u_0) keeps planes of its
// own; the passes ping-pong between two other sets.  After the demodulation and after each pass, one kernel forms m_k
// and one smooths it into M_k and updates each pixel's best colour, M and level in place.  One thread per pixel.
#include <cuda_runtime.h>

#include "select.h"

namespace rptb {

void launch_halves_demodulate(const double* sums, const double* m2, const double* half, const uint32_t* counts, const double* albedo,
                              uint32_t width, uint32_t height, double eps_a, double* col, double* var, double* u, cudaStream_t stream);
void launch_halves_pass(const double* col, const double* var, const double* u, const double* nrm, const double* depth, const double* albedo,
                        uint32_t width, uint32_t height, uint32_t k, const rptb_denoise& d, double* out_col, double* out_var, double* out_u,
                        cudaStream_t stream);

__global__ void select_m_kernel(const double* __restrict__ ik, const double* __restrict__ Uk, const double* __restrict__ i0,
                                const double* __restrict__ u0, const double* __restrict__ albedo, uint64_t npix, double eps_a,
                                double* __restrict__ m) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npix) return;
    m[p] = select_m(ik + 3 * p, Uk + 3 * p, i0 + 3 * p, u0 + 3 * p, albedo + 3 * p, eps_a);
}

__global__ void select_level_kernel(const double* __restrict__ m, const double* __restrict__ ik, const double* __restrict__ albedo,
                                    const double* __restrict__ sums, const uint32_t* __restrict__ counts, uint32_t width, uint32_t height,
                                    uint32_t k, double eps_a, double* __restrict__ best, double* __restrict__ best_M,
                                    uint8_t* __restrict__ level) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    const size_t p = (size_t)y * width + x;
    select_level(m, ik, albedo, sums, counts, width, height, x, y, k, eps_a, best + 3 * p, best_M + p, level + p);
}

// The selection: sums / m2 / half / counts and the resolved features in.  col[0], var[0], u[0]: level 0's planes;
// col[1..2], var[1..2], u[1..2]: the passes' ping-pong planes; m: m_k (width*height).  Out: best (width*height*3) the
// chosen level's c', best_M (width*height) its M, level (width*height) the chosen level.  d.iterations > 0.
// *launches: kernels enqueued.
cudaError_t launch_denoise_select(const double* sums, const double* m2, const double* half, const uint32_t* counts, const double* nrm,
                                  const double* depth, const double* albedo, uint32_t width, uint32_t height, const rptb_denoise& d,
                                  double* const col[3], double* const var[3], double* const u[3], double* m, double* best, double* best_M,
                                  uint8_t* level, cudaStream_t stream, uint32_t* launches) {
    const uint64_t npix = (uint64_t)width * height;
    const unsigned grid1 = (unsigned)((npix + 255) / 256);
    const dim3 block(32, 8), grid2((width + 31) / 32, (height + 7) / 8);
    const double eps_a = d.albedo_eps;
    launch_halves_demodulate(sums, m2, half, counts, albedo, width, height, eps_a, col[0], var[0], u[0], stream);
    select_m_kernel<<<grid1, 256, 0, stream>>>(col[0], u[0], col[0], u[0], albedo, npix, eps_a, m);
    select_level_kernel<<<grid2, block, 0, stream>>>(m, col[0], albedo, sums, counts, width, height, 0u, eps_a, best, best_M, level);
    uint32_t cur = 0;
    for (uint32_t k = 0; k < d.iterations; k++) {
        const uint32_t next = cur == 1u ? 2u : 1u;
        launch_halves_pass(col[cur], var[cur], u[cur], nrm, depth, albedo, width, height, k, d, col[next], var[next], u[next], stream);
        cur = next;
        select_m_kernel<<<grid1, 256, 0, stream>>>(col[cur], u[cur], col[0], u[0], albedo, npix, eps_a, m);
        select_level_kernel<<<grid2, block, 0, stream>>>(m, col[cur], albedo, sums, counts, width, height, k + 1u, eps_a, best, best_M,
                                                         level);
    }
    *launches = 3u + 3u * d.iterations;
    return cudaGetLastError();
}

}  // namespace rptb
