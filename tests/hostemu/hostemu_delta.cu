// hostemu_delta.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.  Never linked into librpt_b200.so, never loaded by rpt_b200/*:
// only tests/test_hostemu_delta.py builds and loads it (`make hostemu`, tests/hostemu/_build/libhostemu_delta.so).
//
// The delta exchange's per-element functions (delta.h) compiled for the host and run as delta_export_kernel and
// delta_import_kernel run them: the export over a block whose slot list is already written, the import over every
// element of every block.
#include <cstring>

#include "../../rpt_b200/csrc/delta.h"

using namespace rptb;

extern "C" {

uint64_t hostemu_delta_bytes(uint32_t capacity) { return delta_bytes(capacity); }

// Writes the header's pixel count and, for the slots the block already lists, their state from a part's compact planes.
void hostemu_delta_export(void* block, uint32_t capacity, uint32_t pixels, const double* sums, const double* m2, const uint32_t* counts) {
    DeltaHeader* h = (DeltaHeader*)block;
    h->pixels = pixels;
    h->capacity = capacity;
    const DeltaPlanes d = delta_planes(block, capacity);
    for (uint32_t i = 0; i < pixels; i++) delta_export_one(d, i, sums, m2, counts);
}

// Element i of every block b of shard_count (block b holds shard b), i below the block header's pixel count, into a
// one-part whole buffer's planes.
void hostemu_delta_import(const void* blocks, uint32_t shard_count, uint32_t capacity, double* sums, double* m2, uint32_t* counts) {
    for (uint32_t b = 0; b < shard_count; b++) {
        const char* block = (const char*)blocks + b * delta_bytes(capacity);
        const uint32_t pixels = ((const DeltaHeader*)block)->pixels;
        for (uint32_t i = 0; i < pixels; i++) delta_import_one(delta_planes(block, capacity), i, b, shard_count, sums, m2, counts);
    }
}

// delta_whole_slot for n slots of shard (index, count).
void hostemu_delta_whole_slots(uint32_t index, uint32_t count, const uint32_t* slots, uint64_t n, uint64_t* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = delta_whole_slot(index, count, slots[i]);
}

}  // extern "C"
