// The camera model on the device, both ways: pixel -> camera-space direction (camera_dir, the ray caster of
// camera.cu) and world point -> continuous pixel and ray parameter (project_point, and project_to_pixel for the
// TSDF fusion and the view counts of mesh.cu).
// One copy, included by both units; each is compiled with -fmad=false, so the fp32 rounding is the same in both.
#pragma once

#include "common.cuh"

namespace mnrf {

template <typename T> struct Vec3 { T x, y, z; };
using V3 = Vec3<float>;

template <typename T>
__device__ __forceinline__ Vec3<T> mat3_vec(const T* __restrict__ m, int ld, Vec3<T> v) {
  Vec3<T> r;
  r.x = m[0] * v.x + m[1] * v.y + m[2] * v.z;
  r.y = m[ld] * v.x + m[ld + 1] * v.y + m[ld + 2] * v.z;
  r.z = m[2 * ld] * v.x + m[2 * ld + 1] * v.y + m[2 * ld + 2] * v.z;
  return r;
}

__device__ __forceinline__ void undistort(const mnrf_camera_desc& d, float xd, float yd, float& xo, float& yo) {
  float x = xd, y = yd;
  const float k1 = d.k1, k2 = d.k2, k3 = d.k3, k4 = d.k4, p1 = d.p1, p2 = d.p2;
  for (int it = 0; it < d.undistort_iters; ++it) {
    const float r = x * x + y * y;
    const float dd = 1.0f + r * (k1 + r * (k2 + r * (k3 + r * k4)));
    const float fx = dd * x + 2.f * p1 * x * y + p2 * (r + 2.f * x * x) - xd;
    const float fy = dd * y + 2.f * p2 * x * y + p1 * (r + 2.f * y * y) - yd;
    const float d_r = k1 + r * (2.0f * k2 + r * (3.0f * k3 + r * 4.0f * k4));
    const float d_x = 2.0f * x * d_r;
    const float d_y = 2.0f * y * d_r;
    const float fx_x = dd + d_x * x + 2.0f * p1 * y + 6.0f * p2 * x;
    const float fx_y = d_y * x + 2.0f * p1 * x + 2.0f * p2 * y;
    const float fy_x = d_x * y + 2.0f * p2 * y + 2.0f * p1 * x;
    const float fy_y = dd + d_y * y + 2.0f * p2 * x + 6.0f * p1 * y;
    const float den = fy_x * fx_y - fx_x * fy_y;
    const float xn = fx * fy_y - fy * fx_y;
    const float yn = fy * fx_x - fx * fy_x;
    const bool ok = fabsf(den) > d.undistort_eps;
    x = x + (ok ? xn / den : 0.f);
    y = y + (ok ? yn / den : 0.f);
  }
  xo = x; yo = y;
}

// camera-space direction of pixel centre (px, py): inverse intrinsics, undistortion, fisheye,
// OpenCV -> OpenGL flip.  The fisheye's sin(theta) / theta is taken as its limit 1 on the optical axis (theta = 0,
// the centre pixel of an odd-sized image with cx = W / 2), where the reference divides 0 by 0.
__device__ __forceinline__ V3 camera_dir(const mnrf_camera_desc& d, const float* __restrict__ p2c, float px, float py) {
  V3 v = mat3_vec(p2c, 3, V3{px + 0.5f, py + 0.5f, 1.0f});
  if (d.has_distortion) {
    float x, y;
    undistort(d, v.x, v.y, x, y);
    v = V3{x, y, 1.0f};
  }
  if (d.camtype == MNRF_CAM_FISHEYE) {
    float theta = sqrtf(v.x * v.x + v.y * v.y);
    theta = fminf(3.14159274101257324f, theta);
    const float s = theta > 0.f ? sinf(theta) / theta : 1.0f;
    v = V3{v.x * s, v.y * s, cosf(theta)};
  }
  return V3{v.x, -v.y, -v.z};
}

// The inverse of camera_dir composed with the camera pose: world point p -> continuous pixel (u, v) and the
// parameter t with p = origin + t * direction(pixel).  w2c: world-to-camera [3, 4] (OpenGL axes), c2p:
// camera-to-pixel [3, 3] (the inverse of pixtocam).  Steps: pose, OpenGL -> OpenCV flip, the pinhole divide or the
// fisheye angle theta = atan2(r, z) (the undistorted point is (x, y) theta / r), the forward radial-tangential
// polynomial (the residual `undistort` solves), the intrinsics.  t is the OpenCV depth for a perspective camera
// (its directions have z = -1) and |q| for a fisheye (unit directions).  Pixel centres sit at +0.5, so the pixel is
// (floor(u), floor(v)).  Returns false when the point has no pixel: behind a perspective camera, or on the optical
// axis behind a fisheye (theta = pi).
__device__ __forceinline__ bool project_point(const mnrf_camera_desc& d, const float* __restrict__ w2c,
                                              const float* __restrict__ c2p, V3 p, float& u, float& v, float& t) {
  V3 q = mat3_vec(w2c, 4, p);
  q = V3{q.x + w2c[3], -(q.y + w2c[7]), -(q.z + w2c[11])};
  float x, y;
  if (d.camtype == MNRF_CAM_FISHEYE) {
    const float r = sqrtf(q.x * q.x + q.y * q.y);
    t = sqrtf(r * r + q.z * q.z);
    if (r == 0.f) {
      if (!(q.z > 0.f)) return false;
      x = 0.f; y = 0.f;
    } else {
      const float s = atan2f(r, q.z) / r;
      x = q.x * s; y = q.y * s;
    }
  } else {
    if (!(q.z > 0.f)) return false;
    t = q.z;
    x = q.x / q.z; y = q.y / q.z;
  }
  if (d.has_distortion) {
    const float k1 = d.k1, k2 = d.k2, k3 = d.k3, k4 = d.k4, p1 = d.p1, p2 = d.p2;
    const float r = x * x + y * y;
    const float dd = 1.0f + r * (k1 + r * (k2 + r * (k3 + r * k4)));
    const float xd = dd * x + 2.f * p1 * x * y + p2 * (r + 2.f * x * x);
    const float yd = dd * y + 2.f * p2 * x * y + p1 * (r + 2.f * y * y);
    x = xd; y = yd;
  }
  const V3 h = mat3_vec(c2p, 3, V3{x, y, 1.0f});
  u = h.x / h.z;
  v = h.y / h.z;
  return true;
}

// Whether world point p lands on a width x height image: project_point succeeds and its pixel (px, py) =
// (floor(u), floor(v)) lies in [0, width) x [0, height).  The one rule both the TSDF fusion and the view counts of
// mesh.cu use; t is project_point's ray parameter.
__device__ __forceinline__ bool project_to_pixel(const mnrf_camera_desc& d, const float* __restrict__ w2c,
                                                 const float* __restrict__ c2p, V3 p, int width, int height,
                                                 int& px, int& py, float& t) {
  float u, v;
  if (!project_point(d, w2c, c2p, p, u, v, t)) return false;
  if (!(u >= 0.f && u < (float)width && v >= 0.f && v < (float)height)) return false;
  px = (int)floorf(u);     // u < width and v < height: in range
  py = (int)floorf(v);
  return true;
}

}  // namespace mnrf
