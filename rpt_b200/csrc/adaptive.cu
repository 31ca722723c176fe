// adaptive.cu -- which pixels an adaptive call renders (rptb_sample_into_adaptive).  Compiled with -fmad=false, so
// adaptive_active (adaptive.h) rounds every product and sum on its own, as the host emulation and numpy do.
//
// Per buffer part (one replica's owned 16x8 tiles, compact tile-major as in film.cu): one kernel evaluates every pixel,
// writes the pixel mask and one flag per 8x4 warp block, and counts the active pixels; an order-preserving select
// (CUB DeviceSelect::Flagged, deterministic) then writes the ids k*4 + w of the flagged blocks and their number -- the
// RenderList the list-scheduled render takes.  Nothing is read back to the host.
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include "adaptive.h"
#include "tile.h"

namespace rptb {

__global__ void __launch_bounds__(128) adaptive_mark_kernel(const double* __restrict__ sums, const double* __restrict__ m2,
                                                            const uint32_t* __restrict__ counts, uint32_t width, uint32_t height,
                                                            uint32_t shard_index, uint32_t shard_count, const rptb_adaptive crit,
                                                            uint8_t* __restrict__ mask, uint8_t* __restrict__ flags,
                                                            unsigned long long* __restrict__ active_pixels) {
    const uint32_t k = blockIdx.x, j = threadIdx.x;
    const uint64_t e = (uint64_t)k * 128u + j;
    // pixel j of owned tile k; the slots past a ragged edge are never active
    bool on = false;
    if (tile_pixel(width, height, shard_index + k * shard_count, j) >= 0)
        on = adaptive_active(counts[e], sums[3 * e], sums[3 * e + 1], sums[3 * e + 2], m2[e], crit);
    mask[e] = on ? 1u : 0u;
    const unsigned votes = __ballot_sync(0xffffffffu, on);
    if ((j & 31u) == 0) {
        flags[(uint64_t)k * 4u + (j >> 5)] = votes != 0u ? 1u : 0u;
        if (votes) atomicAdd(active_pixels, (unsigned long long)__popc(votes));
    }
}

size_t adaptive_temp_bytes(uint32_t tiles) {
    size_t bytes = 0;
    cub::DeviceSelect::Flagged(nullptr, bytes, cub::CountingInputIterator<uint32_t>(0u), (const uint8_t*)nullptr,
                               (uint32_t*)nullptr, (uint32_t*)nullptr, (int)(tiles * 4u));
    return bytes;
}

// The ids of the flagged warp blocks of marked flags (tiles*4) and their number *len.
cudaError_t launch_adaptive_list(const uint8_t* flags, uint32_t tiles, uint32_t* ids, uint32_t* len, void* temp, size_t temp_bytes,
                                 cudaStream_t stream) {
    if (tiles == 0) return cudaMemsetAsync(len, 0, sizeof(uint32_t), stream);
    return cub::DeviceSelect::Flagged(temp, temp_bytes, cub::CountingInputIterator<uint32_t>(0u), flags, ids, len, (int)(tiles * 4u),
                                      stream);
}

// mask: tiles*128, flags / ids: tiles*4, *len: listed blocks, *active_pixels: pixels that take the entry.
cudaError_t launch_adaptive_select(const double* sums, const double* m2, const uint32_t* counts, uint32_t tiles, uint32_t width,
                                   uint32_t height, uint32_t shard_index, uint32_t shard_count, const rptb_adaptive& crit,
                                   uint8_t* mask, uint8_t* flags, uint32_t* ids, uint32_t* len, unsigned long long* active_pixels,
                                   void* temp, size_t temp_bytes, cudaStream_t stream) {
    cudaError_t e = cudaMemsetAsync(active_pixels, 0, sizeof(unsigned long long), stream);
    if (e != cudaSuccess) return e;
    if (tiles) {
        adaptive_mark_kernel<<<tiles, 128, 0, stream>>>(sums, m2, counts, width, height, shard_index, shard_count, crit, mask, flags,
                                                        active_pixels);
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return launch_adaptive_list(flags, tiles, ids, len, temp, temp_bytes, stream);
}

}  // namespace rptb
