// rpt.hpp -- header-only C++ host mirror of rpt's public builder API over the C ABI of
// rpt_b200.h, for compiled hosts (the reference is a compiled Rust crate; its Rust side
// here is never compiled, see INTEGRATION.md).  Same names and argument meaning as:
//
//   Scene / SceneAdd            src/scene.rs:7-41        Object            src/object.rs:10-32
//   Material::{diffuse,...}     src/material.rs:28-106   Light             src/light.rs:7-19
//   Camera::{look_at,focus}     src/camera.rs:8-61       Transformable     src/shape.rs:179-284
//   sphere/plane/cube/polygon   src/shape.rs:286-313     Renderer          src/renderer.rs:18-115
//   Buffer / Filter             src/buffer.rs:6-108      hex_color         src/color.rs:10-15
//
// Everything below Renderer::sample (src/renderer.rs:117-129) runs in librpt_b200.so.
#pragma once
#include <array>
#include <cmath>
#include <cstdint>
#include <fstream>
#include <functional>
#include <memory>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "rpt_b200.h"

namespace rpt {

struct Vec3 {
    double x = 0, y = 0, z = 0;
};
inline Vec3 vec3(double x, double y, double z) { return Vec3{x, y, z}; }
inline Vec3 operator-(Vec3 a, Vec3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
inline Vec3 operator*(Vec3 a, double s) { return {a.x * s, a.y * s, a.z * s}; }
inline double dot(Vec3 a, Vec3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
inline Vec3 cross(Vec3 a, Vec3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
inline Vec3 normalize(Vec3 a) { const double l = std::sqrt(dot(a, a)); return {a.x / l, a.y / l, a.z / l}; }
using Color = Vec3;

inline Color hex_color(uint32_t x) {  // src/color.rs:10-15
    auto ch = [](uint32_t v) { return std::pow((double)(v & 0xff) / 255.0, 2.2); };
    return {ch(x >> 16), ch(x >> 8), ch(x)};
}

// ---- 4x4 column-major transforms (glm::translate / scale / rotate) ------------------------
struct Mat4 {
    std::array<double, 16> m{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    Mat4 operator*(const Mat4& b) const {
        Mat4 r;
        for (int c = 0; c < 4; c++)
            for (int row = 0; row < 4; row++) {
                double s = 0;
                for (int k = 0; k < 4; k++) s += m[k * 4 + row] * b.m[c * 4 + k];
                r.m[c * 4 + row] = s;
            }
        return r;
    }
    static Mat4 translate(Vec3 v) { Mat4 r; r.m[12] = v.x; r.m[13] = v.y; r.m[14] = v.z; return r; }
    static Mat4 scale(Vec3 v) { Mat4 r; r.m[0] = v.x; r.m[5] = v.y; r.m[10] = v.z; return r; }
    static Mat4 rotate(double angle, Vec3 axis) {
        const Vec3 a = normalize(axis);
        const double c = std::cos(angle), s = std::sin(angle), t = 1 - c;
        Mat4 r;
        r.m[0] = c + a.x * a.x * t;        r.m[4] = a.x * a.y * t - a.z * s;  r.m[8] = a.x * a.z * t + a.y * s;
        r.m[1] = a.y * a.x * t + a.z * s;  r.m[5] = c + a.y * a.y * t;        r.m[9] = a.y * a.z * t - a.x * s;
        r.m[2] = a.z * a.x * t - a.y * s;  r.m[6] = a.z * a.y * t + a.x * s;  r.m[10] = c + a.z * a.z * t;
        return r;
    }
};

// ---- shapes (src/shape.rs) ------------------------------------------------------------------
struct Mesh {  // KdTree<Triangle>; the tree is built by the library when `nodes` stays null
    std::vector<double> tris;  // 18 doubles per triangle: v1 v2 v3 n1 n2 n3
};

struct Shape {
    uint32_t kind = RPTB_SHAPE_SPHERE;
    Vec3 plane_normal;
    double plane_value = 0;
    std::shared_ptr<Mesh> mesh;                           // MESH; copies of a Shape share it (Arc<Mesh>)
    double monomial_height = 0, monomial_exp = 4;           // MONOMIAL
    std::shared_ptr<std::vector<Shape>> children;           // GROUP: KdTree<Box<dyn Bounded>>::objects
    bool has_transform = false;
    Mat4 matrix;
    // Transformable: chaining composes, new * self.transform (src/shape.rs:234-284)
    Shape transform(const Mat4& t) const { Shape s = *this; s.matrix = t * (has_transform ? matrix : Mat4()); s.has_transform = true; return s; }
    Shape translate(Vec3 v) const { return transform(Mat4::translate(v)); }
    Shape scale(Vec3 v) const { return transform(Mat4::scale(v)); }
    Shape rotate(double a, Vec3 axis) const { return transform(Mat4::rotate(a, axis)); }
    Shape rotate_x(double a) const { return rotate(a, {1, 0, 0}); }
    Shape rotate_y(double a) const { return rotate(a, {0, 1, 0}); }
    Shape rotate_z(double a) const { return rotate(a, {0, 0, 1}); }
};
inline Shape sphere() { return Shape{}; }
inline Shape cube() { Shape s; s.kind = RPTB_SHAPE_CUBE; return s; }
inline Shape plane(Vec3 normal, double value) { Shape s; s.kind = RPTB_SHAPE_PLANE; s.plane_normal = normal; s.plane_value = value; return s; }
inline Shape monomial_surface(double height, double exp) {  // src/shape.rs:292-294
    Shape s; s.kind = RPTB_SHAPE_MONOMIAL; s.monomial_height = height; s.monomial_exp = exp; return s;
}
// KdTree::new(objects) over whole Bounded shapes (src/kdtree.rs:108-119): spheres, cubes, monomial surfaces and
// meshes, bare or transformed -- the kd-tree of kd-trees of examples/fractal_teapots.rs.  The library builds the tree.
inline Shape KdTree(std::vector<Shape> objects) {
    for (const Shape& c : objects)
        if (c.kind == RPTB_SHAPE_PLANE || c.kind == RPTB_SHAPE_GROUP) throw std::invalid_argument("rpt::KdTree: child is not a supported Bounded shape");
    Shape s; s.kind = RPTB_SHAPE_GROUP; s.children = std::make_shared<std::vector<Shape>>(std::move(objects)); return s;
}
inline Shape polygon(const std::vector<Vec3>& v) {  // triangle fan, src/shape.rs:307-313
    Shape s;
    s.kind = RPTB_SHAPE_MESH;
    s.mesh = std::make_shared<Mesh>();
    for (size_t i = 1; i + 1 < v.size(); i++) {
        const Vec3 n = normalize(cross(v[i] - v[0], v[i + 1] - v[0]));
        for (Vec3 p : {v[0], v[i], v[i + 1]}) { s.mesh->tris.push_back(p.x); s.mesh->tris.push_back(p.y); s.mesh->tris.push_back(p.z); }
        for (int k = 0; k < 3; k++) { s.mesh->tris.push_back(n.x); s.mesh->tris.push_back(n.y); s.mesh->tris.push_back(n.z); }
    }
    return s;
}

// ---- material (src/material.rs:7-106) ----------------------------------------------------------
struct Material {
    Color color = hex_color(0xff0000);
    double index = 1.5, roughness = 0.5, metallic = 0.0, emittance = 0.0;
    bool transparent = false;
    static Material diffuse(Color c) { return {c, 1.5, 1.0, 0.0, 0.0, false}; }
    static Material specular(Color c, double r) { return {c, 1.5, r, 0.0, 0.0, false}; }
    static Material clear(double index, double r) { return {{1, 1, 1}, index, r, 0.0, 0.0, true}; }
    static Material transparent_(Color c, double index, double r) { return {c, index, r, 0.0, 0.0, true}; }
    static Material metallic_(Color c, double r) { return {c, 1.5, r, 1.0, 0.0, false}; }
    static Material light(Color c, double e) { return {c, 1.0, 1.0, 0.0, e, false}; }
};

struct Object {  // Object::new(shape).material(m)
    Shape shape;
    Material mat;
    explicit Object(Shape s) : shape(std::move(s)) {}
    Object material(Material m) && { mat = m; return std::move(*this); }
    Object material(Material m) const& { Object o = *this; o.mat = m; return o; }
};

// ---- mesh ingestion (src/io.rs:27-360); the parsing itself is the library's ----------------------
namespace detail {
inline std::string slurp(const std::string& path) {
    std::ifstream f(path, std::ios::binary);
    if (!f) throw std::runtime_error("rpt: cannot open " + path);
    std::ostringstream ss;
    ss << f.rdbuf();
    return ss.str();
}
inline Shape mesh_shape(const double* tris, uint64_t first, uint64_t n) {
    Shape s;
    s.kind = RPTB_SHAPE_MESH;
    s.mesh = std::make_shared<Mesh>();
    s.mesh->tris.assign(tris + 18 * first, tris + 18 * (first + n));
    return s;
}
}  // namespace detail

inline Shape load_obj(const std::string& path) {  // src/io.rs:27-73
    const std::string text = detail::slurp(path);
    double* tris = nullptr;
    uint64_t n = 0;
    if (rptb_parse_obj(text.data(), text.size(), &tris, &n) != 0) throw std::runtime_error(rptb_last_error());
    Shape s = detail::mesh_shape(tris, 0, n);
    rptb_free_triangles(tris);
    return s;
}

inline Shape load_stl(const std::string& path) {  // src/io.rs:260-287
    const std::string data = detail::slurp(path);
    double* tris = nullptr;
    uint64_t n = 0;
    if (rptb_parse_stl(data.data(), data.size(), &tris, &n) != 0) throw std::runtime_error(rptb_last_error());
    Shape s = detail::mesh_shape(tris, 0, n);
    rptb_free_triangles(tris);
    return s;
}

inline std::vector<Object> load_obj_with_mtl(const std::string& obj_path, const std::string& mtl_path) {  // src/io.rs:83-149
    const std::string obj = detail::slurp(obj_path), mtl = detail::slurp(mtl_path);
    rptb_obj_groups_out out;
    if (rptb_parse_obj_mtl(obj.data(), obj.size(), mtl.data(), mtl.size(), &out) != 0) throw std::runtime_error(rptb_last_error());
    std::vector<Object> objects;
    for (uint64_t g = 0; g < out.ngroups; g++) {
        const rptb_material& m = out.groups[g].material;
        Object o(detail::mesh_shape(out.tris, out.groups[g].first_tri, out.groups[g].ntris));
        o.mat = Material{{m.color[0], m.color[1], m.color[2]}, m.index, m.roughness, m.metallic, m.emittance, m.transparent != 0};
        objects.push_back(std::move(o));
    }
    rptb_free_obj_groups(&out);
    return objects;
}

struct Light {  // src/light.rs:7-19
    uint32_t kind;
    Color color;
    Vec3 vec;
    std::shared_ptr<rpt::Object> object;
    static Light Point(Color c, Vec3 location) { return {RPTB_LIGHT_POINT, c, location, nullptr}; }
    static Light Ambient(Color c) { return {RPTB_LIGHT_AMBIENT, c, {}, nullptr}; }
    static Light Directional(Color c, Vec3 dir) { return {RPTB_LIGHT_DIRECTIONAL, c, dir, nullptr}; }
    static Light Object(rpt::Object o) { return {RPTB_LIGHT_OBJECT, {}, {}, std::make_shared<rpt::Object>(std::move(o))}; }
};

struct Scene {  // src/scene.rs:7-41
    std::vector<Object> objects;
    std::vector<Light> lights;
    Color environment{0, 0, 0};
    void add(Object o) { objects.push_back(std::move(o)); }
    void add(Light l) { lights.push_back(std::move(l)); }
};

struct Camera {  // src/camera.rs:8-61
    Vec3 eye{0, 0, 10}, direction{0, 0, -1}, up{0, 1, 0};
    double fov = 0.52359877559829887, aperture = 0, focal_distance = 0;
    static Camera look_at(Vec3 eye, Vec3 center, Vec3 up, double fov) {
        Camera c;
        c.eye = eye;
        c.direction = normalize(center - eye);
        c.up = normalize(up - c.direction * dot(up, c.direction));
        c.fov = fov;
        return c;
    }
    Camera focus(Vec3 focal_point, double aperture_) const {
        Camera c = *this;
        c.focal_distance = dot(focal_point - eye, direction);
        c.aperture = aperture_;
        return c;
    }
};

struct Filter {
    uint32_t radius = 0;
    static Filter Box(uint32_t r) { return Filter{r}; }
};

// Buffer: one equally weighted entry per pixel per add_samples (src/buffer.rs:6-93)
class Buffer {
public:
    Buffer(uint32_t w, uint32_t h, Filter f = {}) : width_(w), height_(h), filter_(f), sums_((size_t)w * h * 3, 0.0) {}
    void add_samples(const std::vector<double>& rgb) {
        if (rgb.size() != sums_.size()) throw std::invalid_argument("Invalid sample dimension");
        for (size_t i = 0; i < rgb.size(); i++) sums_[i] += rgb[i];
        batches_++;
    }
    std::vector<uint8_t> image(int device = 0) const {  // Buffer::image on the device
        std::vector<uint8_t> out(sums_.size());
        if (rptb_film_resolve(sums_.data(), batches_, width_, height_, filter_.radius, device, out.data()) != RPTB_OK)
            throw std::runtime_error(rptb_last_error());
        return out;
    }
    uint32_t batches() const { return batches_; }

private:
    uint32_t width_, height_;
    Filter filter_;
    std::vector<double> sums_;
    uint32_t batches_ = 0;
};

// Renderer (src/renderer.rs:18-115); `sample` is the seam into the CUDA library.
class Renderer {
public:
    Renderer(const Scene& scene, Camera camera) : scene_(scene), camera_(camera) {}
    ~Renderer() { if (handle_) rptb_scene_destroy(handle_); }
    Renderer(const Renderer&) = delete;
    Renderer& width(uint32_t v) { width_ = v; return *this; }
    Renderer& height(uint32_t v) { height_ = v; return *this; }
    Renderer& exposure_value(double v) { ev_ = v; return *this; }
    Renderer& filter(Filter f) { filter_ = f; return *this; }
    Renderer& max_bounces(uint32_t v) { max_bounces_ = v; return *this; }
    Renderer& num_samples(uint32_t v) { num_samples_ = v; return *this; }
    Renderer& seed(uint64_t v) { seed_ = v; return *this; }
    Renderer& device(int d) { device_ = d; ngpus_ = 1; return *this; }
    // Renderer::sample fans out over GPUs 0..n-1 behind the same call (rptb_scene_create_multi); the image is
    // bit-identical for any n.  The reference's fan-out is rayon over rows inside `sample` (src/renderer.rs:118-127).
    Renderer& gpus(int n) { ngpus_ = n < 1 ? 1 : n; device_ = 0; return *this; }

    std::vector<uint8_t> render() {  // :96-100
        Buffer buffer(width_, height_, filter_);
        sample(num_samples_, buffer);
        return buffer.image(device_);
    }
    void iterative_render(uint32_t interval, const std::function<void(uint32_t, const Buffer&)>& cb) {  // :103-115
        Buffer buffer(width_, height_, filter_);
        uint32_t iteration = 0;
        while (iteration < num_samples_) {
            const uint32_t steps = std::min(num_samples_ - iteration, interval);
            sample(steps, buffer);
            iteration += steps;
            cb(iteration, buffer);
        }
    }
    void sample(uint32_t iterations, Buffer& buffer) {  // :117-129
        ensure_scene();
        rptb_render_params p{};
        p.width = width_; p.height = height_; p.iterations = iterations; p.max_bounces = max_bounces_;
        p.exposure_value = ev_; p.seed = seed_; p.first_sample = next_sample_; p.shard_count = 1;
        rptb_camera c{};
        const Vec3* src[3] = {&camera_.eye, &camera_.direction, &camera_.up};
        double* dst[3] = {c.eye, c.direction, c.up};
        for (int i = 0; i < 3; i++) { dst[i][0] = src[i]->x; dst[i][1] = src[i]->y; dst[i][2] = src[i]->z; }
        c.fov = camera_.fov; c.aperture = camera_.aperture; c.focal_distance = camera_.focal_distance;
        std::vector<double> colors((size_t)width_ * height_ * 3);
        if (rptb_render_samples(handle_, &c, &p, colors.data(), &stats) != RPTB_OK) throw std::runtime_error(rptb_last_error());
        next_sample_ += iterations;
        buffer.add_samples(colors);
    }
    rptb_stats stats{};

private:
    static rptb_material to_c(const Material& m) {
        rptb_material r{};
        r.color[0] = m.color.x; r.color[1] = m.color.y; r.color[2] = m.color.z;
        r.index = m.index; r.roughness = m.roughness; r.metallic = m.metallic; r.emittance = m.emittance;
        r.transparent = m.transparent ? 1u : 0u;
        return r;
    }
    void ensure_scene() {
        if (handle_) return;
        std::vector<rptb_material> mats;
        std::vector<rptb_mesh> meshes;
        std::vector<const Mesh*> mesh_ids;                       // one rptb_mesh per distinct Mesh (instancing)
        std::vector<rptb_group> groups;
        std::vector<std::unique_ptr<std::vector<rptb_object>>> group_children;  // owned until rptb_scene_create returns
        std::function<rptb_object(const Shape&)> to_shape = [&](const Shape& sh) {
            rptb_object r{};
            r.kind = sh.kind;
            r.has_transform = sh.has_transform ? 1u : 0u;
            const Mat4 m = sh.has_transform ? sh.matrix : Mat4();
            for (int i = 0; i < 16; i++) r.transform[i] = m.m[i];
            r.plane_normal[0] = sh.plane_normal.x; r.plane_normal[1] = sh.plane_normal.y; r.plane_normal[2] = sh.plane_normal.z;
            r.plane_value = sh.plane_value;
            r.monomial_height = sh.monomial_height;
            r.monomial_exp = sh.monomial_exp;
            if (sh.kind == RPTB_SHAPE_MESH) {
                size_t k = 0;
                while (k < mesh_ids.size() && mesh_ids[k] != sh.mesh.get()) k++;
                if (k == mesh_ids.size()) {
                    rptb_mesh cm{};
                    cm.tris = sh.mesh->tris.data();
                    cm.ntris = sh.mesh->tris.size() / 18;
                    meshes.push_back(cm);
                    mesh_ids.push_back(sh.mesh.get());
                }
                r.mesh = (uint32_t)k;
            }
            if (sh.kind == RPTB_SHAPE_GROUP) {
                auto kids = std::make_unique<std::vector<rptb_object>>();
                for (const Shape& c : *sh.children) kids->push_back(to_shape(c));
                rptb_group g{};
                g.children = kids->data();
                g.nchildren = kids->size();
                r.mesh = (uint32_t)groups.size();
                groups.push_back(g);
                group_children.push_back(std::move(kids));
            }
            return r;
        };
        auto to_object = [&](const Object& o) {
            rptb_object r = to_shape(o.shape);
            r.material = (uint32_t)mats.size();
            mats.push_back(to_c(o.mat));
            return r;
        };
        std::vector<rptb_object> objs;
        for (const Object& o : scene_.objects) objs.push_back(to_object(o));
        std::vector<rptb_light> lights;
        for (const Light& l : scene_.lights) {
            rptb_light r{};
            r.kind = l.kind;
            r.color[0] = l.color.x; r.color[1] = l.color.y; r.color[2] = l.color.z;
            r.vec[0] = l.vec.x; r.vec[1] = l.vec.y; r.vec[2] = l.vec.z;
            if (l.kind == RPTB_LIGHT_OBJECT) r.object = to_object(*l.object);
            lights.push_back(r);
        }
        rptb_scene_desc d{};
        d.materials = mats.data(); d.nmaterials = (uint32_t)mats.size();
        d.meshes = meshes.data(); d.nmeshes = (uint32_t)meshes.size();
        d.objects = objs.data(); d.nobjects = (uint32_t)objs.size();
        d.lights = lights.data(); d.nlights = (uint32_t)lights.size();
        d.groups = groups.data(); d.ngroups = (uint32_t)groups.size();
        d.environment.kind = RPTB_ENV_COLOR;
        d.environment.color[0] = scene_.environment.x; d.environment.color[1] = scene_.environment.y; d.environment.color[2] = scene_.environment.z;
        const int rc = ngpus_ > 1 ? rptb_scene_create_multi(&d, nullptr, ngpus_, &handle_) : rptb_scene_create(&d, device_, &handle_);
        if (rc != RPTB_OK) throw std::runtime_error(rptb_last_error());
    }

    const Scene& scene_;
    Camera camera_;
    uint32_t width_ = 800, height_ = 600, max_bounces_ = 0, num_samples_ = 1;  // :46-57
    double ev_ = 0.0;
    Filter filter_;
    uint64_t seed_ = 0, next_sample_ = 0;
    int device_ = 0, ngpus_ = 1;
    rptb_scene* handle_ = nullptr;
};

}  // namespace rpt
