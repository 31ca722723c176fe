// delta.h -- the delta exchange block of a shard buffer (rptb_buffer_export_delta / rptb_buffer_import_deltas), one set of
// functions for the device (delta.cu) and the host emulation (tests/hostemu/hostemu_delta.cu).
//
// A delta block carries the pixels a shard's last adaptive or guided call changed, with their complete new state, so
// that every rank can bring its gathered whole buffer up to date in place instead of gathering every shard's full block
// (DESIGN.md section 6f).  For a capacity m, the same on every rank: a header of kDeltaHeaderBytes, then
//     sums    3m doubles
//     m2      m doubles
//     counts  m uint32
//     slots   m uint32   the shard's compact slot of each pixel, ascending
// 256 + 40 m bytes, so every plane and the next block start 8-byte aligned.  A shard with halves
// (rptb_buffer_create_shard_halves; its header's flags hold kShardHalves) appends
//     half    3m doubles  the sums of each pixel's odd entries (the HALF plane, planes.h)
// at 256 + 40 m: 256 + 64 m bytes, with the prefix laid out as above.  Only the header's `pixels` entries of each plane
// are written.
#pragma once
#include "../../include/rpt_b200.h"
#include "tile.h"

namespace rptb {

constexpr uint32_t kDeltaMagic = 0x544c4544u;  // "DELT"
constexpr uint64_t kDeltaHeaderBytes = 256;

// A CameraRecord (api.cu) in an exchange header: its state, and the camera when the state is ONE (zero otherwise).
struct ShardCamera {
    uint32_t state, _pad;
    rptb_camera cam;
};

// A buffer's state as both exchange headers carry it, at the same offset: its entry calls, flags (kShardReprojected and
// kShardHalves, api.cu), feature rays per pixel and cameras.  Every byte is written (shard_camera zeroes what a state leaves unused),
// so two states are the same when their bytes are.
struct BlockState {
    uint32_t entries, flags;
    uint64_t feature_rays;
    ShardCamera entry_cam, feat_cam;
};

// The header of a delta block.  `s` is the shard's state after the call, and entries_before its entry count before it
// (rptb_buffer_import_deltas derives the rest of the state before the call from `s`).
struct DeltaHeader {
    uint32_t magic, width, height, shard_index, shard_count, entries_before;
    BlockState s;
    uint32_t pixels, capacity;
};
static_assert(sizeof(DeltaHeader) <= kDeltaHeaderBytes, "the delta header outgrew its slot");
static_assert(offsetof(DeltaHeader, s) == 24, "the state sits where the shard header's does");
static_assert(offsetof(DeltaHeader, pixels) == 248, "distributed.DELTA_PIXELS_AT");

RPTB_HD uint64_t delta_bytes(uint32_t capacity) { return kDeltaHeaderBytes + 40ull * capacity; }
RPTB_HD uint64_t delta_bytes_halves(uint32_t capacity) { return kDeltaHeaderBytes + 64ull * capacity; }

// The planes of the block at `block`, of capacity m.
struct DeltaPlanes {
    double* sums;
    double* m2;
    uint32_t* counts;
    uint32_t* slots;
};
RPTB_HD DeltaPlanes delta_planes(const void* block, uint32_t m) {
    char* b = (char*)block + kDeltaHeaderBytes;
    return {(double*)b, (double*)(b + 24ull * m), (uint32_t*)(b + 32ull * m), (uint32_t*)(b + 36ull * m)};
}

// Export, element i: copies the state of the shard's compact slot d.slots[i] from its planes into the block.
RPTB_HD void delta_export_one(const DeltaPlanes& d, uint32_t i, const double* __restrict__ sums, const double* __restrict__ m2,
                              const uint32_t* __restrict__ counts) {
    const uint64_t s = d.slots[i];
    d.sums[3ull * i] = sums[3 * s];
    d.sums[3ull * i + 1] = sums[3 * s + 1];
    d.sums[3ull * i + 2] = sums[3 * s + 2];
    d.m2[i] = m2[s];
    d.counts[i] = counts[s];
}

// Slot s of shard (index, count) is lane s % 128 of its owned tile s / 128, i.e. of tile index + (s / 128) * count: compact
// slot tile * 128 + lane of a one-part whole buffer, which owns every tile in order.
RPTB_HD uint64_t delta_whole_slot(uint32_t index, uint32_t count, uint32_t s) {
    return ((uint64_t)index + (uint64_t)(s >> 7) * count) * 128u + (s & 127u);
}

// Import, element i of the block of shard (index, count): writes its state in place into a one-part whole buffer's planes.
RPTB_HD void delta_import_one(const DeltaPlanes& d, uint32_t i, uint32_t index, uint32_t count, double* __restrict__ sums,
                              double* __restrict__ m2, uint32_t* __restrict__ counts) {
    const uint64_t e = delta_whole_slot(index, count, d.slots[i]);
    sums[3 * e] = d.sums[3ull * i];
    sums[3 * e + 1] = d.sums[3ull * i + 1];
    sums[3 * e + 2] = d.sums[3ull * i + 2];
    m2[e] = d.m2[i];
    counts[e] = d.counts[i];
}

// The planes of a halves block at `block`, of capacity m: the plain block's, then HALF.
struct DeltaHalvesPlanes {
    DeltaPlanes d;
    double* half;
};
RPTB_HD DeltaHalvesPlanes delta_halves_planes(const void* block, uint32_t m) {
    return {delta_planes(block, m), (double*)((char*)block + kDeltaHeaderBytes + 40ull * m)};
}

// delta_export_one, and the slot's HALF.
RPTB_HD void delta_export_halves_one(const DeltaHalvesPlanes& d, uint32_t i, const double* __restrict__ sums,
                                     const double* __restrict__ m2, const uint32_t* __restrict__ counts,
                                     const double* __restrict__ half) {
    delta_export_one(d.d, i, sums, m2, counts);
    const uint64_t s = d.d.slots[i];
    d.half[3ull * i] = half[3 * s];
    d.half[3ull * i + 1] = half[3 * s + 1];
    d.half[3ull * i + 2] = half[3 * s + 2];
}

// delta_import_one, and the element's HALF.
RPTB_HD void delta_import_halves_one(const DeltaHalvesPlanes& d, uint32_t i, uint32_t index, uint32_t count,
                                     double* __restrict__ sums, double* __restrict__ m2, uint32_t* __restrict__ counts,
                                     double* __restrict__ half) {
    delta_import_one(d.d, i, index, count, sums, m2, counts);
    const uint64_t e = delta_whole_slot(index, count, d.d.slots[i]);
    half[3 * e] = d.half[3ull * i];
    half[3 * e + 1] = d.half[3ull * i + 1];
    half[3 * e + 2] = d.half[3ull * i + 2];
}

}  // namespace rptb
