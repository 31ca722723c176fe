// hostemu_reproject_part.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.  Never linked into librpt_b200.so, never loaded by
// rpt_b200/*: `make hostemu` links it into tests/hostemu/_build/libhostemu_reproject.so next to hostemu_reproject.cu,
// and only tests/test_shard_reproject.py calls it.
//
// The reprojection into a shard buffer's compact tiles (reproject_slot, reproject.h) compiled for the host, with the
// same switches as hostemu.cu.  Its own translation unit: it needs reproject.h alone, not the emulated scenes.
#include <cstdint>

#include "../../rpt_b200/csrc/reproject.h"

using namespace rptb;

extern "C" {

// reproject_slot at every element of the compact tiles of shard `index` of `count` of a dw x dh view through dcam, as
// reproject_part_kernel runs it: nelem elements (the shard's tiles * 128), whose feature sums dfeat are laid out as
// feature_planes(dfeat, nelem) over `rays` camera rays.  The source as hostemu_reproject's.  Writes out_sums (3 per
// element), out_m2, out_counts in element order, and *out_reused, the elements with a count > 0.
void hostemu_reproject_part(const rptb_camera* dcam, uint32_t dw, uint32_t dh, uint32_t index, uint32_t count, double* dfeat,
                            uint64_t nelem, double rays, const rptb_camera* scam, uint32_t sw, uint32_t sh, const double* ssums,
                            const double* sm2, const uint32_t* scounts, const double* snrm, const double* sdepth, const double* sfrac,
                            const rptb_reproject* prm, double* out_sums, double* out_m2, uint32_t* out_counts, uint64_t* out_reused) {
    const ReprojectView dv = reproject_view(*dcam, dw, dh), sv = reproject_view(*scam, sw, sh);
    const ReprojectSource s = {ssums, sm2, scounts, snrm, sdepth, sfrac};
    const FeaturePlanes f = feature_planes(dfeat, nelem);
    uint64_t reused = 0;
#pragma omp parallel for schedule(static) reduction(+ : reused)
    for (int64_t e = 0; e < (int64_t)nelem; e++) {
        out_counts[e] = reproject_slot(dv, sv, s, f, rays, index, count, (uint64_t)e, *prm, out_sums + 3 * e, out_m2 + e);
        reused += out_counts[e] > 0u;
    }
    *out_reused = reused;
}

}  // extern "C"
