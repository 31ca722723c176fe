// film.cu -- film resolve on the device ("next" row N1 of SURVEY section 8f).
//
// Replaces Buffer::image -> get_filtered_color -> color_bytes
// (ekzhang/rpt src/buffer.rs:43-56,75-93, src/color.rs:17-23): box filter of radius r
// over the per-pixel sample sums (every pixel holds `nbatches` equally weighted
// entries), then clamp, gamma 1/2.2 and a truncating cast to u8.  Computed in f64 and
// summed in the reference's order (x outer, y inner), so the bytes match the CPU
// restatement exactly.
//
// The device-resident Buffer (rptb_buffer, src/buffer.rs:6-93) keeps those sums on the GPU: every entry is added
// there by buffer_accumulate_kernel, together with a streaming (Welford) variance and the pixel's entry count, and
// film_resolve_counted_kernel reads them.
#include <cuda_runtime.h>
#include <stdint.h>

#include "planes.h"
#include "tile.h"

namespace rptb {

// One output pixel.  COUNTED: pixel q holds counts[q] entries (the device Buffer), else every pixel nbatches (the host
// Buffer, and a denoised image).
template <bool COUNTED>
__device__ __forceinline__ void film_resolve_pixel(const double* __restrict__ sums, uint32_t nbatches,
                                                   const uint32_t* __restrict__ counts, uint32_t width, uint32_t height,
                                                   uint32_t radius, uint8_t* __restrict__ out, uint32_t x, uint32_t y) {
    double c0 = 0.0, c1 = 0.0, c2 = 0.0;
    unsigned long long count = 0;
    const uint32_t i0 = x >= radius ? x - radius : 0u;  // saturating_sub
    const uint32_t j0 = y >= radius ? y - radius : 0u;
    const uint64_t i1 = (uint64_t)x + radius, j1 = (uint64_t)y + radius;
    for (uint64_t i = i0; i <= i1 && i < width; i++)
        for (uint64_t j = j0; j <= j1 && j < height; j++) {
            const double* p = sums + 3 * (j * width + i);
            c0 += p[0];
            c1 += p[1];
            c2 += p[2];
            if (COUNTED) count += counts[j * width + i];
            else count += nbatches;
        }
    const double n = (double)count;
    const double c[3] = {c0 / n, c1 / n, c2 / n};
    uint8_t* o = out + 3 * ((size_t)y * width + x);
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const double v = fmin(fmax(c[k], 0.0), 1.0);
        o[k] = (uint8_t)(pow(v, 1.0 / 2.2) * 255.0);  // `as u8` truncates
    }
}

__global__ void film_resolve_kernel(const double* __restrict__ sums, uint32_t nbatches, uint32_t width,
                                    uint32_t height, uint32_t radius, uint8_t* __restrict__ out) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    film_resolve_pixel<false>(sums, nbatches, nullptr, width, height, radius, out, x, y);
}

// get_filtered_color over per-pixel entry counts (src/buffer.rs:75-93: it divides by the entries in the window)
__global__ void film_resolve_counted_kernel(const double* __restrict__ sums, const uint32_t* __restrict__ counts, uint32_t width,
                                            uint32_t height, uint32_t radius, uint8_t* __restrict__ out) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    film_resolve_pixel<true>(sums, 0u, counts, width, height, radius, out, x, y);
}

__global__ void convert_f64_f32_kernel(const double* __restrict__ in, float* __restrict__ out, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (float)in[i];
}

// Buffer::variance (src/buffer.rs:59-73): per pixel, the sample variance (n - 1) of its `nbatches`
// entries summed over the three channels; block-reduced and added to *out_sum (the caller divides by
// the pixel count).  The block partials are added with atomics, so the last bits depend on the order.
__global__ void film_variance_kernel(const double* __restrict__ batches, uint32_t nbatches, uint64_t npixels,
                                     double* __restrict__ out_sum) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    double v = 0.0;
    if (p < npixels) {
        double mean[3] = {0.0, 0.0, 0.0};
        for (uint32_t b = 0; b < nbatches; b++)
            for (int k = 0; k < 3; k++) mean[k] += batches[((size_t)b * npixels + p) * 3 + k];
        for (int k = 0; k < 3; k++) mean[k] /= (double)nbatches;
        double ss = 0.0;
        for (uint32_t b = 0; b < nbatches; b++)
            for (int k = 0; k < 3; k++) {
                const double d = batches[((size_t)b * npixels + p) * 3 + k] - mean[k];
                ss += d * d;
            }
        v = ss / ((double)nbatches - 1.0);
    }
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __shared__ double warp_sum[8];
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (unsigned w = 0; w < blockDim.x / 32; w++) s += warp_sum[w];
        atomicAdd(out_sum, s);
    }
}

// ---- the device-resident Buffer (rptb_buffer) ---------------------------------------------------------------------
// A replica holds its own 16x8 tiles in the compact tile-major layout of rptb_tile_pixel: element e = k*128 + j is
// pixel j of the k-th owned tile, sums[3e..3e+3) its running per-channel sum, m2[e] its Welford M2 summed over the
// channels and counts[e] its number of entries (pixels may hold different numbers: adaptive sampling).

// Entry n of one pixel into its running sums s[0..3) and M2 *m.  The sum is added in entry order, so it is the
// sequential sum np.sum(batches, axis=0) computes; M2 takes the mean from the sums before and after the entry:
// M2 += sum_c (x_c - S_old,c/(n-1)) * (x_c - S_new,c/n); the first entry is the sum, and its M2 is zero.  Written
// without a branch on n, so that the loads of the old state do not wait for the load of n.
__device__ __forceinline__ void welford_add(double x0, double x1, double x2, uint32_t n, double* __restrict__ s,
                                            double* __restrict__ m) {
    const double o0 = s[0], o1 = s[1], o2 = s[2], om = *m;
    const double n0 = o0 + x0, n1 = o1 + x1, n2 = o2 + x2;
    const double a = (double)(n - 1), b = (double)n;
    const double dm = (x0 - o0 / a) * (x0 - n0 / b) + (x1 - o1 / a) * (x1 - n1 / b) + (x2 - o2 / a) * (x2 - n2 / b);
    const bool first = n == 1;
    s[0] = first ? x0 : n0;
    s[1] = first ? x1 : n1;
    s[2] = first ? x2 : n2;
    *m = first ? 0.0 : om + dm;
}

// HALVES (a buffer with halves, planes.h): entry k = counts[e] (the count before the add) also goes into half[3e..3e+3)
// when k is odd, added in entry order.
template <class T, bool ROWMAJOR, bool HALVES>
__global__ void buffer_accumulate_kernel(const T* __restrict__ in, const uint8_t* __restrict__ mask, uint64_t nelem,
                                         uint32_t width, uint32_t height, uint32_t shard_index, uint32_t shard_count,
                                         double* __restrict__ sums, double* __restrict__ m2, uint32_t* __restrict__ counts,
                                         double* __restrict__ half) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nelem) return;
    if (mask && !mask[e]) return;
    const T* src = in + 3 * e;
    if (ROWMAJOR) {
        const int64_t p = tile_pixel(width, height, shard_index + (uint32_t)(e >> 7) * shard_count, (uint32_t)(e & 127u));
        if (p < 0) return;
        src = in + 3 * p;
    }
    const uint32_t k = counts[e];
    const double x0 = (double)src[0], x1 = (double)src[1], x2 = (double)src[2];
    welford_add(x0, x1, x2, k + 1u, sums + 3 * e, m2 + e);
    counts[e] = k + 1u;
    if constexpr (HALVES) {
        if (k & 1u) {
            half[3 * e] = half[3 * e] + x0;
            half[3 * e + 1] = half[3 * e + 1] + x1;
            half[3 * e + 2] = half[3 * e + 2] + x2;
        }
    }
}

// Element `from` of every plane k < NP present in both sets (planes.h) -> element `to` of dst; from < 0 writes zeros.
// Every value is loaded before any is stored, so the loads of all planes are in flight together.  NP is HALF unless
// the sets hold HALF (launch_buffer_move): the kernels that move the other planes alone keep the registers and the
// instructions they have without it.
template <int NP>
__device__ __forceinline__ void move_planes(const PlaneSet& src, const PlaneSet& dst, int64_t from, uint64_t to) {
    unsigned long long v[NP][3];
#pragma unroll
    for (int k = 0; k < NP; k++) {
        const PlaneShape s = plane_shape(k);
        if (!src.p[k] || !dst.p[k] || from < 0) continue;
        for (uint32_t j = 0; j < s.values; j++)
            v[k][j] = s.bytes == 8 ? ((const unsigned long long*)src.p[k])[s.values * from + j] : ((const uint32_t*)src.p[k])[s.values * from + j];
    }
#pragma unroll
    for (int k = 0; k < NP; k++) {
        const PlaneShape s = plane_shape(k);
        if (!src.p[k] || !dst.p[k]) continue;
        for (uint32_t j = 0; j < s.values; j++) {
            const unsigned long long x = from < 0 ? 0ull : v[k][j];
            if (s.bytes == 8) ((unsigned long long*)dst.p[k])[s.values * to + j] = x;
            else ((uint32_t*)dst.p[k])[s.values * to + j] = (uint32_t)x;
        }
    }
}

// The compact tiles of replica `shard_index` of `shard_count` -> the row-major planes of the whole image.
template <int NP>
__global__ void buffer_scatter_kernel(const PlaneSet src, const PlaneSet dst, uint64_t nelem, uint32_t width, uint32_t height,
                                      uint32_t shard_index, uint32_t shard_count) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nelem) return;
    const int64_t p = tile_pixel(width, height, shard_index + (uint32_t)(e >> 7) * shard_count, (uint32_t)(e & 127u));
    if (p >= 0) move_planes<NP>(src, dst, e, p);
}

// The inverse: the row-major planes -> the compact tiles.  Elements past a ragged edge are zeroed, as a fresh buffer
// holds them.
template <int NP>
__global__ void buffer_compact_kernel(const PlaneSet src, const PlaneSet dst, uint64_t nelem, uint32_t width, uint32_t height,
                                      uint32_t shard_index, uint32_t shard_count) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nelem) return;
    move_planes<NP>(src, dst, tile_pixel(width, height, shard_index + (uint32_t)(e >> 7) * shard_count, (uint32_t)(e & 127u)), e);
}

// Buffer::variance from the row-major M2 and counts: the sum over pixels of M2/(n-1), each pixel with its own n (a
// pixel with one entry gives 0/0: NaN, as the reference's variance does), in a fixed order and without atomics, so
// the bits do not depend on the run or on how many devices rendered.  Block b sums pixels [b*CHUNK, (b+1)*CHUNK):
// thread t its pixels t, t+256, ... in order, then a fixed tree; one block then reduces the block partials the same way.
constexpr uint32_t kVarThreads = 256, kVarChunk = kVarThreads * 16;

__device__ __forceinline__ double block_sum_fixed(double v) {
    __shared__ double sh[kVarThreads];
    sh[threadIdx.x] = v;
    __syncthreads();
    for (uint32_t s = kVarThreads / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
        __syncthreads();
    }
    return sh[0];
}

__global__ void __launch_bounds__(kVarThreads) buffer_variance_partial_kernel(const double* __restrict__ m2,
                                                                              const uint32_t* __restrict__ counts,
                                                                              uint64_t npixels, double* __restrict__ partial) {
    const uint64_t base = (uint64_t)blockIdx.x * kVarChunk;
    double v = 0.0;
    for (uint32_t i = threadIdx.x; i < kVarChunk; i += kVarThreads)
        if (base + i < npixels) v += m2[base + i] / ((double)counts[base + i] - 1.0);
    const double s = block_sum_fixed(v);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

__global__ void __launch_bounds__(kVarThreads) buffer_variance_final_kernel(const double* __restrict__ partial, uint32_t nblocks,
                                                                            double* __restrict__ out_sum) {
    double v = 0.0;
    for (uint32_t i = threadIdx.x; i < nblocks; i += kVarThreads) v += partial[i];
    const double s = block_sum_fixed(v);
    if (threadIdx.x == 0) *out_sum = s;
}

// half: the HALF plane of a buffer with halves (buffer_accumulate_kernel's HALVES), else null.
cudaError_t launch_buffer_accumulate(const float* in32, const double* in64, bool rowmajor, const uint8_t* mask, uint64_t nelem,
                                     uint32_t width, uint32_t height, uint32_t shard_index, uint32_t shard_count, double* sums,
                                     double* m2, uint32_t* counts, double* half, cudaStream_t stream) {
    if (nelem == 0) return cudaSuccess;
    const unsigned grid = (unsigned)((nelem + 255) / 256);
    if (in32) {
        const auto k = half ? buffer_accumulate_kernel<float, false, true> : buffer_accumulate_kernel<float, false, false>;
        k<<<grid, 256, 0, stream>>>(in32, mask, nelem, width, height, shard_index, shard_count, sums, m2, counts, half);
    } else {
        const auto k = rowmajor ? (half ? buffer_accumulate_kernel<double, true, true> : buffer_accumulate_kernel<double, true, false>)
                                : (half ? buffer_accumulate_kernel<double, false, true> : buffer_accumulate_kernel<double, false, false>);
        k<<<grid, 256, 0, stream>>>(in64, mask, nelem, width, height, shard_index, shard_count, sums, m2, counts, half);
    }
    return cudaGetLastError();
}

uint32_t buffer_variance_blocks(uint64_t npixels) { return (uint32_t)((npixels + kVarChunk - 1) / kVarChunk); }

// *out_sum = sum over pixels of m2[p] / (counts[p] - 1); `partial` holds buffer_variance_blocks(npixels) doubles.
cudaError_t launch_buffer_variance_sum(const double* m2, const uint32_t* counts, uint64_t npixels, double* partial,
                                       double* out_sum, cudaStream_t stream) {
    const uint32_t nb = buffer_variance_blocks(npixels);
    buffer_variance_partial_kernel<<<nb, kVarThreads, 0, stream>>>(m2, counts, npixels, partial);
    buffer_variance_final_kernel<<<1, kVarThreads, 0, stream>>>(partial, nb, out_sum);
    return cudaGetLastError();
}

cudaError_t launch_film_resolve_counted(const double* sums, const uint32_t* counts, uint32_t width, uint32_t height,
                                        uint32_t radius, uint8_t* out, cudaStream_t stream) {
    const dim3 block(32, 8), grid((width + 31) / 32, (height + 7) / 8);
    film_resolve_counted_kernel<<<grid, block, 0, stream>>>(sums, counts, width, height, radius, out);
    return cudaGetLastError();
}

// `compact`: row-major src -> compact dst (buffer_compact_kernel), else compact src -> row-major dst.
cudaError_t launch_buffer_move(bool compact, const PlaneSet& src, const PlaneSet& dst, uint64_t nelem, uint32_t width, uint32_t height,
                               uint32_t shard_index, uint32_t shard_count, cudaStream_t stream) {
    if (nelem == 0) return cudaSuccess;
    const unsigned grid = (unsigned)((nelem + 255) / 256);
    const bool half = src.p[HALF] && dst.p[HALF];
    if (compact)
        (half ? buffer_compact_kernel<NPLANES> : buffer_compact_kernel<HALF>)<<<grid, 256, 0, stream>>>(src, dst, nelem, width, height,
                                                                                                       shard_index, shard_count);
    else
        (half ? buffer_scatter_kernel<NPLANES> : buffer_scatter_kernel<HALF>)<<<grid, 256, 0, stream>>>(src, dst, nelem, width, height,
                                                                                                       shard_index, shard_count);
    return cudaGetLastError();
}

cudaError_t launch_film_variance(const double* batches, uint32_t nbatches, uint64_t npixels, double* out_sum,
                                 cudaStream_t stream) {
    film_variance_kernel<<<(unsigned)((npixels + 255) / 256), 256, 0, stream>>>(batches, nbatches, npixels, out_sum);
    return cudaGetLastError();
}

cudaError_t launch_film_resolve(const double* sums, uint32_t nbatches, uint32_t width, uint32_t height,
                                uint32_t radius, uint8_t* out, cudaStream_t stream) {
    const dim3 block(32, 8), grid((width + 31) / 32, (height + 7) / 8);
    film_resolve_kernel<<<grid, block, 0, stream>>>(sums, nbatches, width, height, radius, out);
    return cudaGetLastError();
}

cudaError_t launch_convert_f64_to_f32(const double* in, float* out, size_t n, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    convert_f64_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(in, out, n);
    return cudaGetLastError();
}

}  // namespace rptb
