// hostemu_list.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.  Never linked into librpt_b200.so, never loaded by rpt_b200/*:
// only tests/test_adaptive.py builds and loads it (`make hostemu`, tests/hostemu/_build/libhostemu_list.so).
//
// Adaptive sampling's device code compiled for the host, on top of the host emulation of hostemu.cu (included whole, so
// its scenes, warp policy and dispatch are the ones used here): the list-scheduled megakernel (render_list_kernel, the
// F_LIST variants through pick_render_list) and the convergence test (adaptive.h).  Same switches as hostemu.cu.
#include <limits>

#include "../../rpt_b200/csrc/adaptive.h"
#include "hostemu.cu"

namespace {

// render_list_kernel's grid (FEAT has F_LIST): entry 4b + w of the list goes to warp w of block b, as on the device.
template <class R, int MAXD, bool STATS, int FEAT>
void run_grid_list(const SceneView<R>& sv, const RenderArgs<R>& a, const RenderList& list) {
    const int64_t nblocks = (int64_t)a.ntiles_mine * a.ngroups;
#pragma omp parallel for schedule(dynamic, 1)
    for (int64_t b = 0; b < nblocks; b++) {
        const uint32_t bx = (uint32_t)(b % a.ntiles_mine), by = (uint32_t)(b / a.ntiles_mine);
        for (uint32_t t = 0; t < (uint32_t)RENDER_THREADS; t++) render_thread_list<R, MAXD, STATS, FEAT, HostLane>(sv, a, list, bx, by, t);
    }
    if (a.nchunks > 1) {
#pragma omp parallel for schedule(static)
        for (int64_t bx = 0; bx < (int64_t)a.ntiles_mine; bx++)
            for (uint32_t t = 0; t < (uint32_t)RENDER_THREADS; t++) resolve_chunks_list_thread<R>(a, list, (uint32_t)bx, t);
    }
}

// launch_render_list_impl's dispatch.  Returns the FEAT it ran (F_LIST included), -1 if that variant is not compiled.
template <class R>
int run_render_list(const SceneView<R>& sv, const RenderArgs<R>& a, const RenderList& list, int stats, int features) {
    using List = std::conditional_t<M<R>::literal, RenderListVariantsF64, RenderListVariantsF32>;
    const Variant v = pick_render_list(features, stats, M<R>::literal, a.max_bounces);
    if (!visit(List{}, v, [&](auto t) { using T = decltype(t); run_grid_list<R, T::maxd, T::stats, T::feat>(sv, a, list); })) return -1;
    return v.feat;
}

}  // namespace

extern "C" {

// The list-scheduled megakernel (render_list_kernel) over the pixels pixel_mask (width*height bytes, row-major) sets:
// the mask and the warp-block list are built the way adaptive.cu builds them (blocks with an active pixel, in tile-major
// order), and out_rgb gets the render's pixels and NaN wherever nothing was written.  Same contract as hostemu_render
// otherwise (the slot engine always; no ext_bvh).  Returns the FEAT bits that ran (F_LIST included), or -1.
int hostemu_render_list(const hostemu_scene* s, const rptb_camera* cam, const rptb_render_params* p, const uint8_t* pixel_mask,
                        double* out_rgb, rptb_stats* stats) {
    if (!s || !cam || !p || !pixel_mask || !out_rgb || p->width == 0 || p->height == 0 || p->iterations == 0 ||
        p->max_bounces > MAX_BOUNCES_SUPPORTED)
        return -1;
    auto run = [&](auto tag, const auto& sv, int features) -> int {
        using R = decltype(tag);
        RenderArgs<R> a;
        fill_args(cam, p, a);
        const size_t nvals = (size_t)p->width * p->height * 3;
        std::vector<R> out(nvals, std::numeric_limits<R>::quiet_NaN());
        std::vector<double> partial;
        if (a.nchunks > 1) partial.assign((size_t)a.nchunks * a.ntiles_mine * RENDER_THREADS * 3, 0.0);
        std::vector<uint8_t> mask((size_t)a.ntiles_mine * RENDER_THREADS, 0);
        std::vector<uint32_t> ids;
        for (uint32_t k = 0; k < a.ntiles_mine; k++) {
            const uint32_t tile = a.shard_index + k * a.shard_count, tx = tile % a.tiles_x, ty = tile / a.tiles_x;
            for (uint32_t w = 0; w < 4u; w++) {
                bool any = false;
                for (uint32_t lane = 0; lane < 32u; lane++) {
                    const uint32_t x = tx * TILE_W + (w & 1u) * 8u + (lane & 7u), y = ty * TILE_H + (w >> 1) * 4u + (lane >> 3);
                    const bool on = x < a.width && y < a.height && pixel_mask[(size_t)y * a.width + x] != 0;
                    mask[(size_t)k * RENDER_THREADS + w * 32u + lane] = on ? 1u : 0u;
                    any = any || on;
                }
                if (any) ids.push_back(k * 4u + w);
            }
        }
        const uint32_t len = (uint32_t)ids.size();
        const RenderList list = {ids.data(), &len, mask.data()};
        DeviceCounters counters;
        std::memset(&counters, 0, sizeof(counters));
        a.out = out.data();
        a.partial = partial.empty() ? nullptr : partial.data();
        a.counters = &counters;
        const int feat = a.ntiles_mine > 0 ? run_render_list<R>(sv, a, list, (int)p->collect_stats, features) : -1;
        for (size_t i = 0; i < nvals; i++) out_rgb[i] = (double)out[i];
        if (stats) {
            std::memset(stats, 0, sizeof(*stats));
            stats->segments = counters.segments; stats->rays = counters.rays;
            stats->engine = RPTB_ENGINE_MEGAKERNEL;
        }
        return feat;
    };
    if (p->precision == RPTB_PRECISION_F64) return run(0.0, s->v64, s->features);
    return run(0.0f, s->v32, (s->features & F_EXT) ? s->features & ~(int)F_BVH : s->features);
}

// The adaptive criterion (adaptive.h) on n pixels: out[i] = 1 iff pixel i (counts[i], sums[3i..3i+3), m2[i]) is active.
void hostemu_adaptive_active(const uint32_t* counts, const double* sums, const double* m2, uint64_t n, const rptb_adaptive* crit,
                             uint8_t* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = adaptive_active(counts[i], sums[3 * i], sums[3 * i + 1], sums[3 * i + 2], m2[i], *crit) ? 1u : 0u;
}

}  // extern "C"
