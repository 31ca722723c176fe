// delta.cu -- the delta exchange of a shard buffer (delta.h): the export's compaction and copy, and the import's scatter.
// Compiled with -fmad=false like its neighbours; it only moves values, so every double arrives with its bits.
//
// Export: an order-preserving select (CUB DeviceSelect::Flagged, deterministic) lists the compact slots the part's mask
// marks -- exactly the pixels its last adaptive or guided call accumulated -- straight into the block's slot plane, then
// one thread per listed pixel copies its sums, M2 and count.  Import: one launch over every block's capacity; thread
// (b, i) writes element i of block b into a one-part whole buffer, and threads past block b's pixel count exit.  A halves
// block's kernels move HALF too; the plain kernels keep it out, so they keep the registers and instructions they had
// before halves blocks existed.
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include "delta.h"

namespace rptb {

__global__ void __launch_bounds__(256) delta_export_kernel(DeltaPlanes d, uint32_t pixels, const double* __restrict__ sums,
                                                           const double* __restrict__ m2, const uint32_t* __restrict__ counts) {
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    if (i < pixels) delta_export_one(d, i, sums, m2, counts);
}

__global__ void __launch_bounds__(256) delta_import_kernel(const char* __restrict__ blocks, uint32_t shard_count, uint32_t capacity,
                                                           double* __restrict__ sums, double* __restrict__ m2,
                                                           uint32_t* __restrict__ counts) {
    const uint64_t t = (uint64_t)blockIdx.x * 256u + threadIdx.x;
    const uint32_t b = (uint32_t)(t / capacity), i = (uint32_t)(t % capacity);
    if (b >= shard_count) return;
    const char* block = blocks + b * delta_bytes(capacity);
    if (i >= ((const DeltaHeader*)block)->pixels) return;
    delta_import_one(delta_planes(block, capacity), i, b, shard_count, sums, m2, counts);
}

__global__ void __launch_bounds__(256) delta_export_halves_kernel(DeltaHalvesPlanes d, uint32_t pixels, const double* __restrict__ sums,
                                                                  const double* __restrict__ m2, const uint32_t* __restrict__ counts,
                                                                  const double* __restrict__ half) {
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    if (i < pixels) delta_export_halves_one(d, i, sums, m2, counts, half);
}

__global__ void __launch_bounds__(256) delta_import_halves_kernel(const char* __restrict__ blocks, uint32_t shard_count, uint32_t capacity,
                                                                  double* __restrict__ sums, double* __restrict__ m2,
                                                                  uint32_t* __restrict__ counts, double* __restrict__ half) {
    const uint64_t t = (uint64_t)blockIdx.x * 256u + threadIdx.x;
    const uint32_t b = (uint32_t)(t / capacity), i = (uint32_t)(t % capacity);
    if (b >= shard_count) return;
    const char* block = blocks + b * delta_bytes_halves(capacity);
    if (i >= ((const DeltaHeader*)block)->pixels) return;
    delta_import_halves_one(delta_halves_planes(block, capacity), i, b, shard_count, sums, m2, counts, half);
}

size_t delta_temp_bytes(uint64_t nelem) {
    size_t bytes = 0;
    cub::DeviceSelect::Flagged(nullptr, bytes, cub::CountingInputIterator<uint32_t>(0u), (const uint8_t*)nullptr, (uint32_t*)nullptr,
                               (uint32_t*)nullptr, (int)nelem);
    return bytes;
}

// The block's planes for the `pixels` slots of mask (nelem) that are set; *selected receives their number again.  half:
// the part's HALF plane, for a halves block (delta_bytes_halves), else null.
cudaError_t launch_delta_export(const uint8_t* mask, uint64_t nelem, const double* sums, const double* m2, const uint32_t* counts,
                                const double* half, void* block, uint32_t capacity, uint32_t pixels, uint32_t* selected, void* temp,
                                size_t temp_bytes, cudaStream_t stream) {
    if (nelem == 0 || pixels == 0) return cudaSuccess;
    const DeltaPlanes d = delta_planes(block, capacity);
    cudaError_t e = cub::DeviceSelect::Flagged(temp, temp_bytes, cub::CountingInputIterator<uint32_t>(0u), mask, d.slots, selected,
                                               (int)nelem, stream);
    if (e != cudaSuccess) return e;
    if (half)
        delta_export_halves_kernel<<<(pixels + 255u) / 256u, 256, 0, stream>>>(delta_halves_planes(block, capacity), pixels, sums, m2,
                                                                               counts, half);
    else
        delta_export_kernel<<<(pixels + 255u) / 256u, 256, 0, stream>>>(d, pixels, sums, m2, counts);
    return cudaGetLastError();
}

// The shard_count blocks of capacity `capacity` at `blocks` (checked by the caller) into a one-part whole buffer's planes.
// half: the buffer's HALF plane, for halves blocks, else null.
cudaError_t launch_delta_import(const void* blocks, uint32_t shard_count, uint32_t capacity, double* sums, double* m2, uint32_t* counts,
                                double* half, cudaStream_t stream) {
    const uint64_t threads = (uint64_t)shard_count * capacity;
    if (threads == 0) return cudaSuccess;
    const unsigned grid = (unsigned)((threads + 255u) / 256u);
    if (half)
        delta_import_halves_kernel<<<grid, 256, 0, stream>>>((const char*)blocks, shard_count, capacity, sums, m2, counts, half);
    else
        delta_import_kernel<<<grid, 256, 0, stream>>>((const char*)blocks, shard_count, capacity, sums, m2, counts);
    return cudaGetLastError();
}

}  // namespace rptb
