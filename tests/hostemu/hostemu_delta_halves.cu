// hostemu_delta_halves.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.  Never linked into librpt_b200.so, never loaded by
// rpt_b200/*: only tests/test_hostemu_delta_halves.py builds and loads it (`make hostemu`,
// tests/hostemu/_build/libhostemu_delta_halves.so).
//
// The halves delta block's per-element functions (delta.h) compiled for the host and run as delta_export_halves_kernel
// and delta_import_halves_kernel run them: the export over a block whose slot list is already written, the import over
// every element of every block.
#include "../../rpt_b200/csrc/delta.h"

using namespace rptb;

extern "C" {

uint64_t hostemu_delta_halves_bytes(uint32_t capacity) { return delta_bytes_halves(capacity); }

// Writes the header's pixel count and, for the slots the block already lists, their state and HALF from a part's
// compact planes.
void hostemu_delta_halves_export(void* block, uint32_t capacity, uint32_t pixels, const double* sums, const double* m2,
                                 const uint32_t* counts, const double* half) {
    DeltaHeader* h = (DeltaHeader*)block;
    h->pixels = pixels;
    h->capacity = capacity;
    const DeltaHalvesPlanes d = delta_halves_planes(block, capacity);
    for (uint32_t i = 0; i < pixels; i++) delta_export_halves_one(d, i, sums, m2, counts, half);
}

// Element i of every halves block b of shard_count (block b holds shard b), i below the block header's pixel count,
// into a one-part whole buffer's planes.
void hostemu_delta_halves_import(const void* blocks, uint32_t shard_count, uint32_t capacity, double* sums, double* m2,
                                 uint32_t* counts, double* half) {
    for (uint32_t b = 0; b < shard_count; b++) {
        const char* block = (const char*)blocks + b * delta_bytes_halves(capacity);
        const uint32_t pixels = ((const DeltaHeader*)block)->pixels;
        for (uint32_t i = 0; i < pixels; i++)
            delta_import_halves_one(delta_halves_planes(block, capacity), i, b, shard_count, sums, m2, counts, half);
    }
}

}  // extern "C"
