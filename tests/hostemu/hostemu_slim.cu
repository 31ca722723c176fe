// hostemu_slim.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.  Never linked into librpt_b200.so, never loaded by rpt_b200/*:
// only tests/test_render_budget_slim.py builds and loads it (`make hostemu`, tests/hostemu/_build/libhostemu_slim.so).
//
// The host emulation of hostemu.cu (included whole: same scenes, warp policy and dispatch) plus what a render given no
// counters runs: the packed-table F_NOCOUNT twins, whose lane is slimmer (integrator.cuh, slim_lane) -- status / dead
// / depth in one word, the run of samples in two.  hostemu.cu always passes counters, so it never picks those twins.
#include "hostemu.cu"

extern "C" {

// Renderer::sample through the variant launch_render_impl picks for a render given no counters (pick_render with
// counters = false), f32 only.  Returns the FEAT it ran, -1 on bad params or a variant that is not compiled.
int hostemu_render_silent(const hostemu_scene* s, const rptb_camera* cam, const rptb_render_params* p, double* out_rgb) {
    if (!s || !cam || !p || !out_rgb || p->width == 0 || p->height == 0 || p->iterations == 0 ||
        p->max_bounces > MAX_BOUNCES_SUPPORTED || p->precision == RPTB_PRECISION_F64)
        return -1;
    RenderArgs<float> a;
    fill_args(cam, p, a);
    const size_t nvals = (size_t)p->width * p->height * 3;
    std::vector<float> out(nvals, 0.0f);
    std::vector<double> partial;
    if (a.nchunks > 1) partial.assign((size_t)a.nchunks * a.ntiles_mine * RENDER_THREADS * 3, 0.0);
    a.out = out.data();
    a.partial = partial.empty() ? nullptr : partial.data();
    a.counters = nullptr;
    const Variant v = pick_render(s->features, (int)p->collect_stats, false, a.max_bounces, false);
    if (a.ntiles_mine > 0 &&
        !visit(RenderVariantsF32{}, v, [&](auto t) { using T = decltype(t); run_grid<float, T::maxd, T::stats, T::feat>(s->v32, a); }))
        return -1;
    for (size_t i = 0; i < nvals; i++) out_rgb[i] = (double)out[i];
    return v.feat;
}

}  // extern "C"
