// tile.h -- the compact tile-major layout of a replica's pixels (rptb_tile_pixel), for the device Buffer (film.cu),
// adaptive sampling's mark kernel (adaptive.cu) and the C ABI (api.cu).
//
// The image is cut into 16x8 tiles, row-major; replica `shard_index` of `shard_count` owns the tiles
// shard_index + k*shard_count.  Element j of a tile is lane j & 31 of warp j >> 5, and each warp covers one 8x4 block:
// warps 0 and 1 side by side on top, 2 and 3 below them.
#pragma once
#include "vec.cuh"

namespace rptb {

// Pixel (y*width + x) of element j of tile `tile`, or -1 past a ragged edge.
RPTB_HD int64_t tile_pixel(uint32_t width, uint32_t height, uint32_t tile, uint32_t j) {
    const uint32_t tiles_x = (width + 15u) / 16u;
    const uint32_t tx = tile % tiles_x, ty = tile / tiles_x;
    const uint32_t warp = j >> 5, lane = j & 31u;
    const uint32_t x = tx * 16u + (warp & 1u) * 8u + (lane & 7u), y = ty * 8u + (warp >> 1) * 4u + (lane >> 3);
    if (x >= width || y >= height) return -1;
    return (int64_t)y * width + x;
}

}  // namespace rptb
