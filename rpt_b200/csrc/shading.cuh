// shading.cuh -- BSDF evaluation / sampling, light sampling, environment lookup.
//
// Reference functions restated (ekzhang/rpt @815b21c):
//   Material::bsdf                   src/material.rs:125-210
//   Material::sample_f               src/material.rs:224-313
//   local_to_world                   src/material.rs:316-324
//   Light::illuminate                src/light.rs:23-47
//   Sphere::sample                   src/shape/sphere.rs:52-64
//   Cube::sample                     src/shape/cube.rs:74-87
//   KdTree::sample / Triangle::sample src/kdtree.rs:138-143, src/shape/mesh.rs:84-98
//   Transformed::sample              src/shape.rs:139-150
//   Hdri::get_color                  src/environment.rs:25-52
//
// f64 keeps the reference's expressions verbatim.  f32 evaluates the same
// functions in forms that survive single precision:
//   * 1 - (n.h)^2 is taken from |n x h|^2: with roughness 1e-4 (examples/glass.rs)
//     the Beckmann exponent divides that difference by 1e-8, so the cancellation
//     in "nh2 - 1.0" would be fatal in f32;
//   * theta = atan(sqrt(-m^2 ln U)) followed by sin_cos becomes
//     cos^2 = 1/(1 + tan^2), sin^2 = 1 - cos^2 (identical values, no atan/sincos,
//     and finite at U = 0);
//   * exp/log/divide use the SFU approximations (ex2/lg2/rcp), |rel err| ~ 1e-6.
#pragma once
#include "geometry.cuh"
#include "rng.cuh"

namespace rptb {

template <class R>
RPTB_D Vec3<R> lerp3(Vec3<R> a, Vec3<R> b, R t) { return a * ((R)1 - t) + b * t; }  // glm::lerp / mix

template <class R>
RPTB_D Vec3<R> mat_color(const MaterialRec<R>& m) { return {m.color[0], m.color[1], m.color[2]}; }

// sin^2 and cos^2 of the angle between unit vectors n and h
template <class R>
RPTB_D void sincos2(Vec3<R> n, Vec3<R> h, R& s2, R& c2) {
    const R c = dot(n, h);
    c2 = c * c;
    if (M<R>::literal) s2 = (R)1 - c2;
    else s2 = length2(cross(n, h));
}

// Beckmann D as written in bsdf(): exp((nh2 - 1)/(m2 nh2)) / (pi m2 nh2^2)
template <class R>
RPTB_D R beckmann_d(R m2, Vec3<R> n, Vec3<R> h) {
    R s2, nh2;
    sincos2(n, h, s2, nh2);
    if (M<R>::literal) return M<R>::exp((nh2 - (R)1) / (m2 * nh2)) / (m2 * M<R>::pi() * nh2 * nh2);
    return M<R>::div(M<R>::exp(-M<R>::div(s2, m2 * nh2)), m2 * M<R>::pi() * nh2 * nh2);
}

template <class R>
RPTB_D Vec3<R> fresnel_f0(const MaterialRec<R>& m) {
    const R r = (m.index - (R)1) / (m.index + (R)1);
    const R f0 = r * r;
    return lerp3(mk(f0, f0, f0), mat_color(m), m.metallic);
}

// Material::bsdf (material.rs:125-210)
template <class R, int FEAT = F_ALL>
RPTB_D Vec3<R> bsdf(const MaterialRec<R>& m, Vec3<R> n, Vec3<R> wo, Vec3<R> wi) {
    const R n_dot_wi = dot(n, wi);
    const R n_dot_wo = dot(n, wo);
    const bool wi_outside = !M<R>::signbit(n_dot_wi);
    const bool wo_outside = !M<R>::signbit(n_dot_wo);
    const Vec3<R> one = mk((R)1, (R)1, (R)1);
    constexpr bool TR = (FEAT & F_TRANSP) != 0;  // false: every material of the scene is opaque
    if ((!TR || !m.transparent) && (!wi_outside || !wo_outside)) return mk((R)0, (R)0, (R)0);
    const R m2 = m.roughness * m.roughness;
    if (!TR || wi_outside == wo_outside) {
        const Vec3<R> h = M<R>::normalize(wi + wo);
        const R wo_dot_h = dot(wo, h);
        const R n_dot_h = dot(n, h);
        const R d = beckmann_d(m2, n, h);
        Vec3<R> f;
        if (TR && !wi_outside && M<R>::sqrt((R)1 - wo_dot_h * wo_dot_h) * m.index > (R)1) {
            f = one;  // total internal reflection
        } else {
            const Vec3<R> f0 = fresnel_f0(m);
            f = f0 + (one - f0) * pow5((R)1 - wo_dot_h);
        }
        R g = M<R>::min(n_dot_wi * n_dot_h, n_dot_wo * n_dot_h);
        g = ((R)2 * g) / wo_dot_h;
        g = M<R>::min(g, (R)1);
        const Vec3<R> specular = (d * f) * g / ((R)4 * n_dot_wo * n_dot_wi);
        if (TR && m.transparent) return specular;
        const Vec3<R> diffuse = cmul(one - f, mat_color(m)) / M<R>::pi();
        return specular + diffuse;
    } else {
        const R eta_t = wo_outside ? m.index : (R)1 / m.index;
        const Vec3<R> h = M<R>::normalize(wi * eta_t + wo);
        const R wi_dot_h = dot(wi, h);
        const R wo_dot_h = dot(wo, h);
        const R n_dot_h = dot(n, h);
        const R d = beckmann_d(m2, n, h);
        const Vec3<R> f0 = fresnel_f0(m);
        const Vec3<R> f = f0 + (one - f0) * pow5((R)1 - M<R>::abs(wi_dot_h));
        R g = M<R>::min(M<R>::abs(n_dot_wi * n_dot_h), M<R>::abs(n_dot_wo * n_dot_h));
        g = ((R)2 * g) / M<R>::abs(wo_dot_h);
        g = M<R>::min(g, (R)1);
        const R denom = eta_t * wi_dot_h + wo_dot_h;
        const Vec3<R> btdf =
            M<R>::abs(wi_dot_h * wo_dot_h / (n_dot_wi * n_dot_wo)) * ((d * (one - f)) * g / (denom * denom));
        return cmul(btdf, mat_color(m));
    }
}

template <class R>
struct Frame {  // columns (ns, nss, n) of local_to_world
    Vec3<R> ns, nss, n;
    RPTB_D Vec3<R> apply(R x, R y, R z) const { return ns * x + nss * y + n * z; }
};
template <class R>
RPTB_D Frame<R> local_to_world(Vec3<R> n) {
    Frame<R> f;
    f.ns = M<R>::isnormal(n.x) ? M<R>::normalize(mk(n.y, -n.x, (R)0)) : M<R>::normalize(mk((R)0, -n.z, n.y));
    f.nss = cross(n, f.ns);
    f.n = n;
    return f;
}

// PIT sample of the Beckmann microfacet angle (material.rs:247-250): one draw
template <class R, class RNG>
RPTB_D void beckmann_angle(R m2, RNG& rng, R& sin_t, R& cos_t) {
    const R u = rng.gen();
    if (M<R>::literal) {
        const double theta = atan(sqrt(m2 * -log((double)u)));
        sin_t = (R)sin(theta);
        cos_t = (R)cos(theta);
    } else {
        const R tan2 = m2 * -M<R>::log(u);         // +inf at u = 0
        const R c2 = M<R>::rcp((R)1 + tan2);       // 0 at u = 0
        cos_t = M<R>::sqrt(c2);
        sin_t = M<R>::sqrt(M<R>::max((R)1 - c2, (R)0));
    }
}

// PIT sample of the Beckmann microfacet normal (material.rs:244-254)
template <class R, class RNG>
RPTB_D Vec3<R> beckmann_sample(R m2, Vec3<R> n, RNG& rng) {
    R sin_t, cos_t;
    beckmann_angle(m2, rng, sin_t, cos_t);
    R x, y;
    unit_circle(rng, x, y);
    return local_to_world(n).apply(x * sin_t, y * sin_t, cos_t);
}

// p = 1/(pi m^2 cos^3) exp(-tan^2/m^2)  (material.rs:256-262)
template <class R>
RPTB_D R beckmann_pdf(R m2, Vec3<R> n, Vec3<R> h) {
    if (M<R>::literal) {
        const R cos_t = M<R>::abs(dot(h, n));
        const R sin_t = M<R>::sqrt((R)1 - cos_t * cos_t);
        const R tn = sin_t / cos_t;
        return ((R)1 / (M<R>::pi() * m2 * (cos_t * (cos_t * cos_t)))) * M<R>::exp(-(tn * tn) / m2);
    }
    R s2, c2;
    sincos2(n, h, s2, c2);
    const R cos_t = M<R>::sqrt(c2);
    return M<R>::div(M<R>::exp(-M<R>::div(s2, c2 * m2)), M<R>::pi() * m2 * cos_t * c2);
}

// Material::sample_f (material.rs:224-313).  Returns false for `None` (TIR ends the path).
//
// The lobes are sampled in one pass.  The Beckmann lobes (reflection, and transmission on a transparent material) draw
// the microfacet angle and then a UnitCircle pair, the diffuse lobe draws a UnitDisc pair; both are rejection from
// [-1,1]^2 and differ only in accepting `< 1` or `<= 1`, so one loop serves both and a warp whose lanes chose different
// lobes runs it once, for as many tries as its slowest lane needs, instead of once per lobe.  One frame maps the local
// sample to world space.  Every lane takes the draws, in the order, and the source arithmetic of rng.cuh's unit_circle /
// unit_disc and of the lobes written one after the other.  The compiler may still fuse multiply-adds differently in the
// two forms, so the rounding is a property of each kernel and not of the source: the Cornell and glass images at the
// bench size are bit-identical to the two-loop form's; the F_BVH kernels keep that form (below).
template <class R, int FEAT = F_ALL, class RNG>
RPTB_D bool sample_f(const MaterialRec<R>& m, Vec3<R> n, Vec3<R> wo, RNG& rng, Vec3<R>& wi_out, R& pdf_out) {
    constexpr bool TR = (FEAT & F_TRANSP) != 0;
    const R m2 = m.roughness * m.roughness;
    const R r0 = (m.index - (R)1) / (m.index + (R)1);
    const R f0 = r0 * r0;
    R f = ((R)1 - m.metallic) * f0 + m.metallic * ((m.color[0] + m.color[1] + m.color[2]) / (R)3);
    f = f * ((R)1 - (R)0.2) + (R)1 * (R)0.2;  // glm::mix_scalar(f, 1.0, 0.2)
    const R wo_dot_n = dot(wo, n);
    const R eta_t = wo_dot_n > (R)0 ? m.index : (R)1 / m.index;

    Vec3<R> wi;
    if constexpr ((FEAT & F_BVH) != 0) {
        // The kernels that traverse a BVH keep the lobes one after the other.  With the one-pass form their compiled
        // rounding differed from this form's (the dragon proxy's image changed in ~1 % of its pixels at 1024 spp); the
        // instruction that differs has not been found, and these kernels were not faster with it.
        if (gen_bool(rng, f)) {
            const Vec3<R> h = beckmann_sample(m2, n, rng);
            wi = -(wo - ((R)2 * dot(h, wo)) * h);  // -glm::reflect_vec(wo, h)
        } else if (!TR || !m.transparent) {
            R x, y;
            unit_disc(rng, x, y);
            const R z = M<R>::sqrt(M<R>::literal ? ((R)1 - x * x - y * y) : M<R>::max((R)1 - x * x - y * y, (R)0));
            wi = local_to_world(n).apply(x, y, z);
        } else {
            const Vec3<R> h = beckmann_sample(m2, n, rng);
            const R cos_to = dot(h, wo);
            const Vec3<R> wo_perp = wo - h * cos_to;
            const Vec3<R> wi_perp = -wo_perp / eta_t;
            const R sin2_ti = length2(wi_perp);
            if (sin2_ti > (R)1) return false;
            const R cos_ti = M<R>::sqrt((R)1 - sin2_ti);
            wi = (-signum(cos_to) * cos_ti) * h + wi_perp;
        }
    } else {
        const bool reflect = gen_bool(rng, f);
        const bool beckmann = reflect || (TR && m.transparent);  // else the diffuse lobe
        R sin_t = (R)0, cos_t = (R)0;
        if (beckmann) beckmann_angle(m2, rng, sin_t, cos_t);
        R x1, x2, sum;
        while (true) {  // UnitCircle (beckmann) or UnitDisc
            x1 = uniform_pm1<R>(rng);
            x2 = uniform_pm1<R>(rng);
            sum = x1 * x1 + x2 * x2;
            if (beckmann ? sum < (R)1 : sum <= (R)1) break;
        }
        R lx, ly, lz;
        if (beckmann) {  // von Neumann's map of the pair onto the circle, scaled to the microfacet angle
            const R diff = x1 * x1 - x2 * x2;
            lx = diff / sum * sin_t;
            ly = (R)2 * x1 * x2 / sum * sin_t;
            lz = cos_t;
        } else {
            lx = x1;
            ly = x2;
            lz = M<R>::sqrt(M<R>::literal ? ((R)1 - x1 * x1 - x2 * x2) : M<R>::max((R)1 - x1 * x1 - x2 * x2, (R)0));
        }
        const Vec3<R> v = local_to_world(n).apply(lx, ly, lz);  // beckmann: the microfacet normal h; diffuse: wi

        if (reflect) {
            wi = -(wo - ((R)2 * dot(v, wo)) * v);  // -glm::reflect_vec(wo, h)
        } else if (!TR || !m.transparent) {
            wi = v;
        } else {
            const R cos_to = dot(v, wo);
            const Vec3<R> wo_perp = wo - v * cos_to;
            const Vec3<R> wi_perp = -wo_perp / eta_t;
            const R sin2_ti = length2(wi_perp);
            if (sin2_ti > (R)1) return false;
            const R cos_ti = M<R>::sqrt((R)1 - sin2_ti);
            wi = (-signum(cos_to) * cos_ti) * v + wi_perp;
        }
    }

    R p = (R)0;
    {
        const Vec3<R> h = M<R>::normalize(wi + wo);
        const R p_h = beckmann_pdf(m2, n, h);
        p += f * p_h / ((R)4 * M<R>::abs(dot(h, wo)));
    }
    const R wi_dot_n = dot(wi, n);
    if (!TR || !m.transparent) {
        p += ((R)1 - f) * M<R>::max(wi_dot_n, (R)0) * ((R)1 / M<R>::pi());
    } else if (M<R>::signbit(wo_dot_n) != M<R>::signbit(wi_dot_n)) {
        const Vec3<R> h = M<R>::normalize(wi * eta_t + wo);
        const R p_h = beckmann_pdf(m2, n, h);
        const R h_dot_wo = dot(h, wo);
        const R h_dot_wi = dot(h, wi);
        const R den = eta_t * h_dot_wi + h_dot_wo;
        const R jacobian = M<R>::abs(h_dot_wo) / (den * den);
        p += ((R)1 - f) * p_h * jacobian;
    }
    wi_out = wi;
    pdf_out = p;
    return true;
}

// ------------------------------------------------------------- light shapes ---
// Shape::sample of the light's object -> (point, normal, pdf per unit area)
template <class R, int FEAT = F_ALL, class RNG>
RPTB_D void shape_sample(const SceneView<R>& sv, const ObjectRec<R>& ob, Vec3<R> target, RNG& rng, Vec3<R>& v,
                         Vec3<R>& n, R& p) {
    if (ob.has_transform) target = xform_point(ob.inv, target);  // shape.rs:140
    bool done = false;
    if constexpr ((FEAT & F_MONO) != 0)
        if (ob.kind == SHAPE_MONOMIAL) {  // monomial_surface.rs:107-122: a point of the RIM (UnitCircle), either side
            R x, z;
            unit_circle(rng, x, z);
            const R height = ob.plane_v;
            const R r2 = x * x + z * z;
            v = mk(x, height * M<R>::pow(r2, ob.plane_n[0] / (R)2), z);
            n = M<R>::normalize(mk(height * (R)4 * x * r2, (R)-1, height * (R)4 * z * r2));
            if (rng.coin()) n = -n;
            p = (R)1 / ((R)2 * (R)6.3406654362);
            done = true;
        }
    if constexpr ((FEAT & F_GROUP) != 0)
        if (ob.kind == SHAPE_GROUP) {  // KdTree::sample, kdtree.rs:138-143: uniform child, pdf / num
            const GroupRec<R>& g = sv.groups[ob.mesh];
            const uint32_t index = (uint32_t)uniform_usize(rng, (uint64_t)g.nchildren);
            shape_sample<R, FEAT & ~F_GROUP>(sv, g.children[index], target, rng, v, n, p);
            p = p / (R)g.nchildren;
            done = true;
        }
    if (!done) switch (ob.kind) {
        case SHAPE_SPHERE: {  // sphere.rs:52-64
            R x, y;
            unit_disc(rng, x, y);
            const R z = M<R>::sqrt(M<R>::literal ? ((R)1 - x * x - y * y) : M<R>::max((R)1 - x * x - y * y, (R)0));
            const Vec3<R> tn = M<R>::normalize(target);
            const Vec3<R> n1 =
                M<R>::isnormal(tn.x) ? M<R>::normalize(mk(tn.y, -tn.x, (R)0)) : M<R>::normalize(mk((R)0, -tn.z, tn.y));
            const Vec3<R> n2 = cross(n1, tn);
            const Vec3<R> pt = x * n1 + y * n2 + z * tn;
            v = pt;
            n = pt;
            p = z * ((R)1 / M<R>::pi());
            break;
        }
        case SHAPE_CUBE: {  // cube.rs:74-87
            const R a = rng.gen() - (R)0.5;
            const R b = rng.gen() - (R)0.5;
            switch ((int)uniform_usize(rng, 6)) {
                case 0: v = mk(a, b, (R)0.5); n = mk((R)0, (R)0, (R)1); break;
                case 1: v = mk(a, b, (R)-0.5); n = mk((R)0, (R)0, (R)-1); break;
                case 2: v = mk(a, (R)0.5, b); n = mk((R)0, (R)1, (R)0); break;
                case 3: v = mk(a, (R)-0.5, b); n = mk((R)0, (R)-1, (R)0); break;
                case 4: v = mk((R)0.5, a, b); n = mk((R)1, (R)0, (R)0); break;
                default: v = mk((R)-0.5, a, b); n = mk((R)-1, (R)0, (R)0); break;
            }
            p = (R)1 / (R)6;
            break;
        }
        case SHAPE_MESH: {  // kdtree.rs:138-143 (uniform pick) + mesh.rs:84-98
            const MeshRec<R>& m = sv.meshes[ob.mesh];
            const uint32_t num = m.ntris;
            const uint32_t index = (uint32_t)uniform_usize(rng, (uint64_t)num);
            R u = rng.gen();
            R w_ = rng.gen();
            while (u + w_ > (R)1) {
                u = rng.gen();
                w_ = rng.gen();
            }
            const R vv = w_;  // reference names: u, v, w = 1 - u - v
            const R w = (R)1 - u - vv;
            const R* q = m.verts + 9 * (size_t)index;
            const R* qn = m.norms + 9 * (size_t)index;
            const Vec3<R> v1 = {q[0], q[1], q[2]}, v2 = {q[3], q[4], q[5]}, v3 = {q[6], q[7], q[8]};
            const Vec3<R> n1 = {qn[0], qn[1], qn[2]}, n2 = {qn[3], qn[4], qn[5]}, n3 = {qn[6], qn[7], qn[8]};
            const R area = (R)0.5 * M<R>::sqrt(length2(cross(v2 - v1, v3 - v1)));
            v = u * v1 + vv * v2 + w * v3;
            n = M<R>::normalize(u * n1 + vv * n2 + w * n3);
            p = ((R)1 / area) / (R)num;
            break;
        }
        default:  // Plane::sample is unimplemented!() in the reference (plane.rs:34-36)
            v = n = mk((R)NAN, (R)NAN, (R)NAN);
            p = (R)NAN;
    }
    if (ob.has_transform) {  // shape.rs:142-149
        const Vec3<R> new_normal = M<R>::normalize(xform3(ob.nrm, n));
        const R parallelepiped_height = dot(xform_dir(ob.fwd, n), new_normal);
        const R parallelepiped_base = ob.det / parallelepiped_height;
        v = xform_point(ob.fwd, v);
        n = new_normal;
        p = p / parallelepiped_base;
    }
}

// How many draws Light::illuminate typically takes (a hint for the generator's refill, rng.cuh): none for point and
// directional lights; UnitDisc for a sphere (2 per try), index + rejection pairs for a mesh, 3 for a cube, more below a group.
template <class R>
RPTB_D uint32_t light_draws_hint(const LightRec<R>& l) {
    if (l.kind != LIGHT_OBJECT) return 0u;
    switch (l.object.kind) {
        case SHAPE_SPHERE: return 4u;
        case SHAPE_CUBE: return 3u;
        case SHAPE_MESH: return 5u;
        default: return 6u;
    }
}

// Light::illuminate (light.rs:23-47) for the non-ambient kinds
template <class R, int FEAT = F_ALL, class RNG>
RPTB_D void illuminate(const SceneView<R>& sv, const LightRec<R>& l, Vec3<R> pos, RNG& rng, Vec3<R>& intensity,
                       Vec3<R>& wi, R& dist) {
    const Vec3<R> color = {l.color[0], l.color[1], l.color[2]};
    if (l.kind == LIGHT_POINT) {
        const Vec3<R> disp = mk(l.vec[0], l.vec[1], l.vec[2]) - pos;
        const R len = M<R>::sqrt(length2(disp));
        intensity = color / (len * len);
        wi = disp / len;
        dist = len;
    } else if (l.kind == LIGHT_DIRECTIONAL) {
        intensity = color;
        wi = -M<R>::normalize(mk(l.vec[0], l.vec[1], l.vec[2]));
        dist = M<R>::inf();
    } else {
        Vec3<R> v, n;
        R p;
        shape_sample<R, FEAT>(sv, l.object, pos, rng, v, n, p);
        const Vec3<R> disp = v - pos;
        const R len = M<R>::sqrt(length2(disp));
        const R cosine = M<R>::max(-dot(disp, n), (R)0) / len;
        const R surface_area = M<R>::max(cosine, (R)0) / (len * len);
        intensity = mk(l.radiance[0], l.radiance[1], l.radiance[2]) * surface_area / p;
        // f32: a UnitDisc draw exactly on the rim (x^2 + y^2 == 1, probability ~1e-7 with 24-bit
        // uniforms, ~1e-16 in f64) gives z = 0 -> pdf 0 and cosine 0 -> 0/0.  Its weight is 0.
        if (!M<R>::literal && !(p > (R)0)) intensity = mk((R)0, (R)0, (R)0);
        wi = disp / len;
        dist = len;
    }
}

// Environment::get_color (environment.rs:25-52,72-77); the unclamped x0+1 / y0+1 of the
// reference is clamped (SURVEY Appendix A #15).
template <class R>
RPTB_D Vec3<R> env_texel(const EnvRec<R>& e, uint32_t x, uint32_t y) {
    x = min(x, e.width - 1);
    y = min(y, e.height - 1);
    if (M<R>::literal) {
        const double* p = e.texels_f64 + 3 * ((size_t)y * e.width + x);
        return mk((R)p[0], (R)p[1], (R)p[2]);
    }
    const float4 t = ldg(e.texels_f4 + (size_t)y * e.width + x);
    return mk((R)t.x, (R)t.y, (R)t.z);
}
template <class R, int FEAT = F_ALL>
RPTB_D Vec3<R> env_color(const EnvRec<R>& e, Vec3<R> dir_in) {
    if (!(FEAT & F_HDRI) || e.kind == 0) return mk(e.color[0], e.color[1], e.color[2]);
    const Vec3<R> dir = M<R>::normalize(dir_in);
    R azimuth, polar;
    if (M<R>::literal) {
        azimuth = (R)(atan2((double)dir.z, (double)dir.x) + 3.14159265358979323846264338327950288);
        polar = (R)acos((double)dir.y);
    } else {
        azimuth = (R)(atan2f((float)dir.z, (float)dir.x) + 3.14159265358979323846f);
        polar = (R)acosf(fminf(fmaxf((float)dir.y, -1.0f), 1.0f));
    }
    const R x = azimuth / ((R)2 * M<R>::pi()) * (R)(e.width - 1);
    const R y = polar / M<R>::pi() * (R)(e.height - 1);
    const uint32_t x0 = min((uint32_t)x, e.width - 1);
    const uint32_t y0 = min((uint32_t)y, e.height - 1);
    const R ax = x - (R)x0;
    const R ay = y - (R)y0;
    return lerp3(lerp3(env_texel(e, x0, y0), env_texel(e, x0 + 1, y0), ax),
                 lerp3(env_texel(e, x0, y0 + 1), env_texel(e, x0 + 1, y0 + 1), ax), ay);
}

}  // namespace rptb
