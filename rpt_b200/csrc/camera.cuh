// camera.cuh -- the camera ray of one sample, shared by every kernel that starts a path or a primary ray.
#pragma once
#include "scene_dev.cuh"
#include "rng.cuh"

namespace rptb {

// Renderer::get_color's jitter and Camera::cast_ray (src/renderer.rs:137-139, src/camera.rs:64-81) for the pixel whose
// normalised centre is (xn, yn), dim = max(width, height): draws dx, dy, then unit_disc when the aperture is open, in
// that order, from `rng` (already at the sample's stream).  Gives the origin and the unit direction.
template <class R, class RNG>
RPTB_D void camera_ray(const CameraRec<R>& cam, R xn, R yn, R dim, RNG& rng, Vec3<R>& ro, Vec3<R>& rd) {
    const R dx = gen_range(rng, (R)-1 / dim, (R)1 / dim);
    const R dy = gen_range(rng, (R)-1 / dim, (R)1 / dim);
    const Vec3<R> eye = {cam.eye[0], cam.eye[1], cam.eye[2]};
    const Vec3<R> cdir = {cam.direction[0], cam.direction[1], cam.direction[2]};
    const Vec3<R> cup = {cam.up[0], cam.up[1], cam.up[2]};
    const Vec3<R> cright = {cam.right[0], cam.right[1], cam.right[2]};
    const R cx = xn + dx, cy = yn + dy;
    Vec3<R> origin = eye;
    Vec3<R> new_dir = cam.d * cdir + cx * cright + cy * cup;
    if (cam.aperture > (R)0) {
        const Vec3<R> focal_point = origin + M<R>::normalize(new_dir) * cam.focal_distance;
        R ax, ay;
        unit_disc(rng, ax, ay);
        origin = origin + (ax * cright + ay * cup) * cam.aperture;
        new_dir = focal_point - origin;
    }
    ro = origin;
    rd = M<R>::normalize(new_dir);
}

}  // namespace rptb
