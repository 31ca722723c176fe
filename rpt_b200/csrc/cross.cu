// cross.cu -- the cross-filtered denoiser with a smoothed selection map (rptb_buffer_denoise_cross).  Compiled with
// -fmad=false: cross.h rounds every operation on its own, as its host emulation and tests/cross_ref.py do.
//
// Everything runs on parts[0]'s device over the gathered row-major state (api.cu), like the selection (select.cu).  One
// kernel demodulates the two halves into level 0's planes, which are kept; each pass runs halves_pass_kernel once per
// chain (guide A carrying X_B, guide B carrying X_A), ping-ponging between two other sets of planes.  The call sweeps
// the chains twice.  The first sweep forms m_k after every level and keeps each pixel's running argmin (k*, best M_k).
// The blend needs k* over each pixel's 5x5 neighbourhood before it can weigh any level, so the second sweep runs the
// same chains again from level 0's planes and, after every level, forms m_k once more and adds beta_k O_k and beta_k M_k.
// So the memory does not grow with the pass count: two ping-pong sets and level 0 (36 doubles a pixel) against 3
// doubles a pixel per level to keep every O_k.  One thread per pixel.
#include <cuda_runtime.h>

#include "cross.h"

namespace rptb {

void launch_halves_pass(const double* col, const double* var, const double* u, const double* nrm, const double* depth, const double* albedo,
                        uint32_t width, uint32_t height, uint32_t k, const rptb_denoise& d, double* out_col, double* out_var, double* out_u,
                        cudaStream_t stream);

__global__ void cross_demodulate_kernel(const double* __restrict__ sums, const double* __restrict__ m2, const double* __restrict__ half,
                                        const uint32_t* __restrict__ counts, uint64_t npix, const double* __restrict__ albedo, double eps_a,
                                        double* __restrict__ iA, double* __restrict__ vA, double* __restrict__ iB, double* __restrict__ vB) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npix) return;
    cross_demodulate(sums + 3 * p, half + 3 * p, m2[p], counts[p], albedo + 3 * p, eps_a, iA + 3 * p, vA + p, iB + 3 * p, vB + p);
}

__global__ void cross_m_kernel(const double* __restrict__ XA, const double* __restrict__ XB, const double* __restrict__ iA0,
                               const double* __restrict__ iB0, const double* __restrict__ vA, const double* __restrict__ vB,
                               const uint32_t* __restrict__ counts, const double* __restrict__ albedo, uint64_t npix, double eps_a,
                               double* __restrict__ m) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npix) return;
    m[p] = cross_m(XA + 3 * p, XB + 3 * p, iA0 + 3 * p, iB0 + 3 * p, vA[p], vB[p], counts[p], albedo + 3 * p, eps_a);
}

__global__ void cross_level_kernel(const double* __restrict__ m, uint32_t width, uint32_t height, uint32_t k, double* __restrict__ best_M,
                                   uint8_t* __restrict__ level) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    const size_t p = (size_t)y * width + x;
    cross_level(m, width, height, x, y, k, best_M + p, level + p);
}

__global__ void cross_blend_kernel(const uint8_t* __restrict__ level, const double* __restrict__ m, const double* __restrict__ XA,
                                   const double* __restrict__ XB, const double* __restrict__ sums, const uint32_t* __restrict__ counts,
                                   const double* __restrict__ albedo, uint32_t width, uint32_t height, uint32_t k, double eps_a,
                                   double* __restrict__ out, double* __restrict__ M_hat) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    const size_t p = (size_t)y * width + x;
    cross_blend(level, m, XA, XB, sums, counts, albedo, width, height, x, y, k, eps_a, out + 3 * p, M_hat + p);
}

// The cross-filtered denoiser: sums / m2 / half / counts and the resolved features in.  set[0]: level 0's planes, whose
// payloads are the other chain's colours (set[0].XB == set[0].colB, set[0].XA == set[0].colA); set[1..2]: the passes'
// ping-pong planes; m: m_k (width*height); best_M (width*height): the first sweep's best M, then M^.  Out: out
// (width*height*3) the blended colour, M_hat (== best_M) and level (width*height) k*.  d.iterations > 0.  *launches: kernels
// enqueued.
cudaError_t launch_denoise_cross(const double* sums, const double* m2, const double* half, const uint32_t* counts, const double* nrm,
                                 const double* depth, const double* albedo, uint32_t width, uint32_t height, const rptb_denoise& d,
                                 const CrossSet set[3], double* m, double* best_M, double* out, uint8_t* level, cudaStream_t stream,
                                 uint32_t* launches) {
    const uint64_t npix = (uint64_t)width * height;
    const unsigned grid1 = (unsigned)((npix + 255) / 256);
    const dim3 block(32, 8), grid2((width + 31) / 32, (height + 7) / 8);
    const double eps_a = d.albedo_eps;
    const CrossSet& s0 = set[0];
    cross_demodulate_kernel<<<grid1, 256, 0, stream>>>(sums, m2, half, counts, npix, albedo, eps_a, s0.colA, s0.varA, s0.colB, s0.varB);
    for (uint32_t sweep = 0; sweep < 2; sweep++) {
        uint32_t cur = 0;
        for (uint32_t k = 0; k <= d.iterations; k++) {
            if (k > 0) {
                const uint32_t next = cur == 1u ? 2u : 1u;
                const CrossSet &a = set[cur], &b = set[next];
                launch_halves_pass(a.colA, a.varA, a.XB, nrm, depth, albedo, width, height, k - 1u, d, b.colA, b.varA, b.XB, stream);
                launch_halves_pass(a.colB, a.varB, a.XA, nrm, depth, albedo, width, height, k - 1u, d, b.colB, b.varB, b.XA, stream);
                cur = next;
            }
            const CrossSet& c = set[cur];
            cross_m_kernel<<<grid1, 256, 0, stream>>>(c.XA, c.XB, s0.colA, s0.colB, s0.varA, s0.varB, counts, albedo, npix, eps_a, m);
            if (sweep == 0)
                cross_level_kernel<<<grid2, block, 0, stream>>>(m, width, height, k, best_M, level);
            else
                cross_blend_kernel<<<grid2, block, 0, stream>>>(level, m, c.XA, c.XB, sums, counts, albedo, width, height, k, eps_a, out,
                                                                best_M);
        }
    }
    *launches = 1u + 2u * (2u + 4u * d.iterations);
    return cudaGetLastError();
}

}  // namespace rptb
