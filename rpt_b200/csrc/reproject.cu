// reproject.cu -- rptb_buffer_reproject on the device: one thread per destination pixel runs reproject_pixel
// (reproject.h) over the gathered row-major state of both buffers on parts[0]'s device, and the result goes back to each
// destination part's compact tile-major layout.  Compiled with -fmad=false: reproject.h rounds every operation on its own,
// as its host emulation and tests/reproject_ref.py do.
//
// Also the per-pixel minimum of a buffer's counts, which image / variance / denoise of a reprojected buffer check.
#include <cuda_runtime.h>

#include "reproject.h"
#include "tile.h"

namespace rptb {

__global__ void __launch_bounds__(256) reproject_kernel(const ReprojectView dv, const ReprojectView sv, const ReprojectSource s,
                                                        const double* __restrict__ dnrm, const double* __restrict__ ddepth,
                                                        const double* __restrict__ dfrac, const rptb_reproject prm,
                                                        double* __restrict__ sums, double* __restrict__ m2,
                                                        uint32_t* __restrict__ counts, unsigned long long* __restrict__ reused) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t npix = (uint64_t)dv.width * dv.height;
    uint32_t n = 0;
    if (p < npix) {
        const uint32_t x = (uint32_t)(p % dv.width), y = (uint32_t)(p / dv.width);
        n = reproject_pixel(dv, sv, s, x, y, dnrm + 3 * p, ddepth[p], dfrac[p], prm, sums + 3 * p, m2 + p);
        counts[p] = n;
    }
    if (reused) {  // every lane reaches the ballot: no early return above
        const unsigned got = __ballot_sync(0xffffffffu, n > 0u);
        if ((threadIdx.x & 31u) == 0u && got) atomicAdd(reused, (unsigned long long)__popc(got));
    }
}

// The row-major planes of the whole image -> the compact tiles of replica `shard_index` of `shard_count` (the inverse of
// film.cu's buffer_scatter_kernel).  Elements past a ragged edge are zeroed, as a fresh buffer holds them.  Null counts
// planes (the feature sums, which have none) are skipped.
__global__ void buffer_compact_kernel(const double* __restrict__ row_sums, const double* __restrict__ row_m2,
                                      const uint32_t* __restrict__ row_counts, uint64_t nelem, uint32_t width, uint32_t height,
                                      uint32_t shard_index, uint32_t shard_count, double* __restrict__ sums, double* __restrict__ m2,
                                      uint32_t* __restrict__ counts) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nelem) return;
    const int64_t p = tile_pixel(width, height, shard_index + (uint32_t)(e >> 7) * shard_count, (uint32_t)(e & 127u));
    sums[3 * e] = p < 0 ? 0.0 : row_sums[3 * p];
    sums[3 * e + 1] = p < 0 ? 0.0 : row_sums[3 * p + 1];
    sums[3 * e + 2] = p < 0 ? 0.0 : row_sums[3 * p + 2];
    m2[e] = p < 0 ? 0.0 : row_m2[p];
    if (counts) counts[e] = p < 0 ? 0u : row_counts[p];
}

// *out = min(*out, counts[0..npix)); the caller sets *out to UINT32_MAX first.
__global__ void __launch_bounds__(256) buffer_min_count_kernel(const uint32_t* __restrict__ counts, uint64_t npix, uint32_t* out) {
    uint32_t m = 0xFFFFFFFFu;
    for (uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += (uint64_t)gridDim.x * blockDim.x)
        m = counts[p] < m ? counts[p] : m;
    m = __reduce_min_sync(0xffffffffu, m);
    if ((threadIdx.x & 31u) == 0u) atomicMin(out, m);
}

cudaError_t launch_reproject(const ReprojectView& dv, const ReprojectView& sv, const ReprojectSource& s, const double* dnrm,
                             const double* ddepth, const double* dfrac, const rptb_reproject& prm, double* sums, double* m2,
                             uint32_t* counts, unsigned long long* reused, cudaStream_t stream) {
    const uint64_t npix = (uint64_t)dv.width * dv.height;
    reproject_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, stream>>>(dv, sv, s, dnrm, ddepth, dfrac, prm, sums, m2, counts, reused);
    return cudaGetLastError();
}

cudaError_t launch_buffer_compact(const double* row_sums, const double* row_m2, const uint32_t* row_counts, uint64_t nelem,
                                  uint32_t width, uint32_t height, uint32_t shard_index, uint32_t shard_count, double* sums,
                                  double* m2, uint32_t* counts, cudaStream_t stream) {
    if (nelem == 0) return cudaSuccess;
    buffer_compact_kernel<<<(unsigned)((nelem + 255) / 256), 256, 0, stream>>>(row_sums, row_m2, row_counts, nelem, width, height,
                                                                             shard_index, shard_count, sums, m2, counts);
    return cudaGetLastError();
}

cudaError_t launch_buffer_min_count(const uint32_t* counts, uint64_t npix, uint32_t* out, cudaStream_t stream) {
    cudaError_t e = cudaMemsetAsync(out, 0xFF, sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    uint64_t blocks = (npix + 255) / 256;
    if (blocks > 1024) blocks = 1024;
    buffer_min_count_kernel<<<(unsigned)blocks, 256, 0, stream>>>(counts, npix, out);
    return cudaGetLastError();
}

}  // namespace rptb
