// denoise.cu -- the device Buffer's feature planes and its edge-avoiding a-trous denoiser (rptb_buffer_features,
// rptb_buffer_denoise).  Compiled with -fmad=false: denoise.h rounds every operation on its own, as its host emulation
// and tests/denoise_ref.py do.
//
// Everything runs on parts[0]'s device over the gathered row-major state (api.cu): one kernel resolves the feature
// planes, one demodulates, one per a-trous pass (ping-pong colour and variance planes), one remodulates.  One thread per
// pixel; the tap loop reads its 25 neighbours straight from global memory (the planes of a 1920x1080 image fit in L2).
#include <cuda_runtime.h>

#include "denoise.h"
#include "planes.h"

namespace rptb {

__global__ void features_resolve_kernel(const double* __restrict__ sn, const double* __restrict__ sa, const double* __restrict__ hits,
                                        const double* __restrict__ sz, uint64_t npix, double rays, double* __restrict__ nrm,
                                        double* __restrict__ depth, double* __restrict__ albedo, double* __restrict__ frac) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npix) return;
    double f;
    features_resolve(hits[p], sn + 3 * p, sz[p], sa + 3 * p, rays, nrm + 3 * p, depth + p, albedo + 3 * p, &f);
    frac[p] = f;
}

__global__ void denoise_demodulate_kernel(const double* __restrict__ sums, const double* __restrict__ m2,
                                          const uint32_t* __restrict__ counts, uint64_t npix,
                                          const double* __restrict__ albedo, double eps_a, double* __restrict__ col,
                                          double* __restrict__ var) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npix) return;
    denoise_demodulate(sums + 3 * p, m2[p], counts[p], albedo + 3 * p, eps_a, col + 3 * p, var + p);
}

__global__ void __launch_bounds__(256) denoise_pass_kernel(const double* __restrict__ col, const double* __restrict__ var,
                                                           const double* __restrict__ nrm, const double* __restrict__ depth,
                                                           const double* __restrict__ albedo, uint32_t width, uint32_t height,
                                                           uint32_t h, const rptb_denoise d,
                                                           double* __restrict__ out_col, double* __restrict__ out_var) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    const size_t p = (size_t)y * width + x;
    denoise_pixel(col, var, nrm, depth, albedo, width, height, x, y, h, d, out_col + 3 * p, out_var + p);
}

// c' = i * (a + eps_a); iterations == 0 (identity): c = S / n, the value Buffer::image divides out
__global__ void denoise_finish_kernel(const double* __restrict__ col, const double* __restrict__ albedo, double eps_a,
                                      const double* __restrict__ sums, const uint32_t* __restrict__ counts, uint64_t npix,
                                      double* __restrict__ out) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npix) return;
    for (int k = 0; k < 3; k++)
        out[3 * p + k] = col ? col[3 * p + k] * (albedo[3 * p + k] + eps_a) : sums[3 * p + k] / (double)counts[p];
}

cudaError_t launch_features_resolve(const FeaturePlanes& f, uint64_t npix, double rays, const Aov& out, cudaStream_t stream) {
    features_resolve_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, stream>>>(f.n, f.a, f.h, f.z, npix, rays, out.normal, out.depth,
                                                                               out.albedo, out.frac);
    return cudaGetLastError();
}

// The filter without its remodulation: demodulate, then d.iterations passes (none: the demodulated planes themselves).
// col[2] / var[2]: the ping-pong planes; *out_col / *out_var: which of them holds the last pass's i' and v' (the
// variance of the denoised value, rptb_buffer_denoise_variance; what a guided adaptive call tests).  *launches:
// kernels enqueued.
cudaError_t launch_denoise_passes(const double* sums, const double* m2, const uint32_t* counts, const double* nrm, const double* depth,
                                  const double* albedo, uint32_t width, uint32_t height, const rptb_denoise& d, double* const col[2],
                                  double* const var[2], const double** out_col, const double** out_var, cudaStream_t stream,
                                  uint32_t* launches) {
    const uint64_t npix = (uint64_t)width * height;
    denoise_demodulate_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, stream>>>(sums, m2, counts, npix, albedo, d.albedo_eps, col[0],
                                                                                  var[0]);
    const dim3 block(32, 8), grid2((width + 31) / 32, (height + 7) / 8);
    uint32_t cur = 0;
    for (uint32_t k = 0; k < d.iterations; k++, cur ^= 1u)
        denoise_pass_kernel<<<grid2, block, 0, stream>>>(col[cur], var[cur], nrm, depth, albedo, width, height, 1u << k, d, col[cur ^ 1u],
                                                         var[cur ^ 1u]);
    *out_col = col[cur];
    *out_var = var[cur];
    *launches = 1u + d.iterations;
    return cudaGetLastError();
}

// The whole filter: sums / m2 / counts and the resolved features in, c' (width*height*3) out.
// col[2] / var[2]: the ping-pong planes.  *launches: kernels enqueued.
cudaError_t launch_denoise(const double* sums, const double* m2, const uint32_t* counts, const double* nrm,
                           const double* depth, const double* albedo, uint32_t width, uint32_t height, const rptb_denoise& d,
                           double* const col[2], double* const var[2], double* out, cudaStream_t stream, uint32_t* launches) {
    const uint64_t npix = (uint64_t)width * height;
    const unsigned grid = (unsigned)((npix + 255) / 256);
    if (d.iterations == 0) {
        denoise_finish_kernel<<<grid, 256, 0, stream>>>(nullptr, albedo, d.albedo_eps, sums, counts, npix, out);
        *launches = 1;
        return cudaGetLastError();
    }
    const double *icol, *ivar;
    const cudaError_t e = launch_denoise_passes(sums, m2, counts, nrm, depth, albedo, width, height, d, col, var, &icol, &ivar, stream,
                                                launches);
    if (e != cudaSuccess) return e;
    denoise_finish_kernel<<<grid, 256, 0, stream>>>(icol, albedo, d.albedo_eps, sums, counts, npix, out);
    (*launches)++;
    return cudaGetLastError();
}

}  // namespace rptb
