// reproject.cu -- rptb_buffer_reproject and rptb_buffer_reproject_shard on the device: one thread per element of a
// destination part's compact tiles runs reproject_slot (reproject.h) against the source's gathered row-major state and
// writes the part's colour planes in place.  Compiled with -fmad=false: reproject.h rounds every operation on its own,
// as its host emulation and tests/reproject_ref.py do.
//
// rptb_buffer_reproject_merge / _merge_shard: the same, but each thread merges the history into the element's fresh
// colour planes in place when reproject_merge accepts it, and counts reused and rejected pixels.
//
// Also the per-pixel minimum of a buffer's counts, which image / variance / denoise of a reprojected buffer check.
#include <cuda_runtime.h>

#include "reproject.h"

namespace rptb {

__global__ void __launch_bounds__(256) reproject_part_kernel(const ReprojectView dv, const ReprojectView sv, const ReprojectSource s,
                                                             const FeaturePlanes f, double rays, uint32_t index, uint32_t count,
                                                             uint64_t nelem, const rptb_reproject prm, double* __restrict__ sums,
                                                             double* __restrict__ m2, uint32_t* __restrict__ counts,
                                                             unsigned long long* __restrict__ reused) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t n = 0;
    if (e < nelem) {
        n = reproject_slot(dv, sv, s, f, rays, index, count, e, prm, sums + 3 * e, m2 + e);
        counts[e] = n;
    }
    if (reused) {  // every lane reaches the ballot: no early return above
        const unsigned got = __ballot_sync(0xffffffffu, n > 0u);
        if ((threadIdx.x & 31u) == 0u && got) atomicAdd(reused, (unsigned long long)__popc(got));
    }
}

// tally[0] += the warp's reused pixels, tally[1] += its rejected ones (verdicts of reproject_merge: 1, 2).
__device__ __forceinline__ void merge_tally(int verdict, unsigned long long* tally) {
    const unsigned reused = __ballot_sync(0xffffffffu, verdict == 1), rejected = __ballot_sync(0xffffffffu, verdict == 2);
    if ((threadIdx.x & 31u) == 0u) {
        if (reused) atomicAdd(tally, (unsigned long long)__popc(reused));
        if (rejected) atomicAdd(tally + 1, (unsigned long long)__popc(rejected));
    }
}

__global__ void __launch_bounds__(256) reproject_merge_part_kernel(const ReprojectView dv, const ReprojectView sv, const ReprojectSource s,
                                                                   const FeaturePlanes f, double rays, uint32_t index, uint32_t count,
                                                                   uint64_t nelem, const rptb_reproject prm, double gamma,
                                                                   double* __restrict__ sums, double* __restrict__ m2,
                                                                   uint32_t* __restrict__ counts, unsigned long long* __restrict__ tally) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int verdict = 0;
    if (e < nelem) verdict = reproject_merge_slot(dv, sv, s, f, rays, index, count, e, prm, gamma, sums + 3 * e, m2 + e, counts + e);
    if (tally) merge_tally(verdict, tally);  // every lane reaches the ballots: no early return above
}

// *out = min(*out, counts[0..npix)); the caller sets *out to UINT32_MAX first.
__global__ void __launch_bounds__(256) buffer_min_count_kernel(const uint32_t* __restrict__ counts, uint64_t npix, uint32_t* out) {
    uint32_t m = 0xFFFFFFFFu;
    for (uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += (uint64_t)gridDim.x * blockDim.x)
        m = counts[p] < m ? counts[p] : m;
    m = __reduce_min_sync(0xffffffffu, m);
    if ((threadIdx.x & 31u) == 0u) atomicMin(out, m);
}

cudaError_t launch_reproject_part(const ReprojectView& dv, const ReprojectView& sv, const ReprojectSource& s, const FeaturePlanes& f,
                                  double rays, uint32_t index, uint32_t count, uint64_t nelem, const rptb_reproject& prm, double* sums,
                                  double* m2, uint32_t* counts, unsigned long long* reused, cudaStream_t stream) {
    if (nelem == 0) return cudaSuccess;
    reproject_part_kernel<<<(unsigned)((nelem + 255) / 256), 256, 0, stream>>>(dv, sv, s, f, rays, index, count, nelem, prm, sums, m2,
                                                                               counts, reused);
    return cudaGetLastError();
}

cudaError_t launch_reproject_merge_part(const ReprojectView& dv, const ReprojectView& sv, const ReprojectSource& s,
                                        const FeaturePlanes& f, double rays, uint32_t index, uint32_t count, uint64_t nelem,
                                        const rptb_reproject& prm, double gamma, double* sums, double* m2, uint32_t* counts,
                                        unsigned long long* tally, cudaStream_t stream) {
    if (nelem == 0) return cudaSuccess;
    reproject_merge_part_kernel<<<(unsigned)((nelem + 255) / 256), 256, 0, stream>>>(dv, sv, s, f, rays, index, count, nelem, prm, gamma,
                                                                                     sums, m2, counts, tally);
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
