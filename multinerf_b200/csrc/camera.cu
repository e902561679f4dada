// Pixel -> ray generation on the device: one thread per ray.
//
// Also the equirectangular panorama camera (camera_utils.cast_spherical_rays camera_utils.py:716-763,
// datasets.py:486-492): spherical_rays_kernel, one thread per pixel, in fp64 -- see there.
//
// Replaces (reference file:line): camera_utils.pixels_to_rays camera_utils.py:522-636,
// _compute_residual_and_jacobian :427-475, _radial_and_tangential_undistort :478-513,
// convert_to_ndc :32-97 and the per-ray camera gather of cast_ray_batch :639-688 -- the
// `xnp=jnp` path of train_utils.py:266-268 (Config.cast_rays_in_train_step).
// HBM-bound: reads 12 B (pixel + camera index; the camera matrices stay in L1/L2), writes 48 B
// per ray.  Compiled without FMA contraction so the fp32 rounding follows the reference's
// unfused elementwise graph.  The camera model itself (camera_dir) is in camera.cuh, shared with the TSDF fusion
// of mesh.cu.
#include "camera.cuh"

namespace mnrf {

// mip-NeRF cone radius from the distances to the dx / dy neighbours: the std of a unit box is 1/sqrt(12)
constexpr double kSqrt12 = 3.4641016151377544;
template <typename T>
__device__ __forceinline__ T cone_radius(T dx_norm, T dy_norm) {
  return (T(0.5) * (dx_norm + dy_norm)) * T(2) / T(kSqrt12);
}

// convert_to_ndc: returns the NDC origin; `dir` is overwritten with the NDC direction
__device__ __forceinline__ V3 to_ndc(const mnrf_camera_desc& d, V3 o, V3& dir) {
  const float t = -(d.ndc_near + o.z) / dir.z;
  o = V3{o.x + t * dir.x, o.y + t * dir.y, o.z + t * dir.z};
  const float xm = 1.0f / d.ndc_p02, ym = 1.0f / d.ndc_p12;
  const V3 o_ndc{xm * o.x / o.z, ym * o.y / o.z, -1.0f};
  const V3 inf_ndc{xm * dir.x / dir.z, ym * dir.y / dir.z, 1.0f};
  dir = V3{inf_ndc.x - o_ndc.x, inf_ndc.y - o_ndc.y, inf_ndc.z - o_ndc.z};
  return o_ndc;
}

template <typename T>
__device__ __forceinline__ T dist3(Vec3<T> a, Vec3<T> b) {
  const T x = a.x - b.x, y = a.y - b.y, z = a.z - b.z;
  return sqrt(x * x + y * y + z * z);
}

__global__ void __launch_bounds__(256)
pixels_to_rays_kernel(mnrf_camera_desc d, const int32_t* __restrict__ pix_x, const int32_t* __restrict__ pix_y,
                      const int32_t* __restrict__ cam_idx, const float* __restrict__ pixtocams,
                      const float* __restrict__ camtoworlds, float* __restrict__ origins,
                      float* __restrict__ directions, float* __restrict__ viewdirs,
                      float* __restrict__ radii, float* __restrict__ imageplane) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < d.num_rays; i += gridDim.x * blockDim.x) {
    int cam = (d.num_cameras > 1 && cam_idx) ? cam_idx[i] : 0;
    cam = min(max(cam, 0), d.num_cameras - 1);
    const float* p2c = pixtocams + (size_t)cam * 9;
    const float* c2w = camtoworlds + (size_t)cam * 12;
    const int xi = pix_x[i], yi = pix_y[i];
    const V3 c0 = camera_dir(d, p2c, (float)xi, (float)yi);
    const V3 cx = camera_dir(d, p2c, (float)(xi + 1), (float)yi);
    const V3 cy = camera_dir(d, p2c, (float)xi, (float)(yi + 1));
    V3 dir = mat3_vec(c2w, 4, c0);
    V3 dx = mat3_vec(c2w, 4, cx);
    V3 dy = mat3_vec(c2w, 4, cy);
    V3 o{c2w[3], c2w[7], c2w[11]};
    const float n = sqrtf(dir.x * dir.x + dir.y * dir.y + dir.z * dir.z);
    const V3 vd{dir.x / n, dir.y / n, dir.z / n};
    float dx_norm, dy_norm;
    if (!d.has_ndc) {
      dx_norm = dist3(dx, dir);
      dy_norm = dist3(dy, dir);
    } else {
      const V3 o_dx = to_ndc(d, o, dx);
      const V3 o_dy = to_ndc(d, o, dy);
      o = to_ndc(d, o, dir);
      dx_norm = dist3(o_dx, o);
      dy_norm = dist3(o_dy, o);
    }
    origins[3 * i + 0] = o.x; origins[3 * i + 1] = o.y; origins[3 * i + 2] = o.z;
    directions[3 * i + 0] = dir.x; directions[3 * i + 1] = dir.y; directions[3 * i + 2] = dir.z;
    viewdirs[3 * i + 0] = vd.x; viewdirs[3 * i + 1] = vd.y; viewdirs[3 * i + 2] = vd.z;
    radii[i] = cone_radius(dx_norm, dy_norm);
    imageplane[2 * i + 0] = c0.x; imageplane[2 * i + 1] = c0.y;
  }
}

// Node k of numpy's linspace(0, stop, n + 1): k * (stop / n), with the last node exactly `stop`.
__device__ __forceinline__ double linspace_node(int64_t k, int32_t n, double stop) {
  return k == n ? stop : (double)k * (stop / n);
}

// World direction of the sphere node (theta, phi): R [-sin(phi) sin(theta), cos(phi), sin(phi) cos(theta)]
__device__ __forceinline__ Vec3<double> sphere_dir(const double* __restrict__ c2w, double theta, double phi) {
  double st, ct, sp, cp;
  sincos(theta, &st, &ct);
  sincos(phi, &sp, &cp);
  return mat3_vec(c2w, 4, Vec3<double>{-sp * st, cp, sp * ct});
}

// One panorama pixel per thread.  Pixel (x, y) looks along grid node (x, y) -- no half-pixel offset -- and its
// radius comes from the differences to nodes (x+1, y) and (x, y+1).  The reference computes all of this in
// float64; so does the kernel, rounding to fp32 only at the store: the radii are differences of nearly equal
// unit vectors, and in fp32 they would lose most of their digits at panorama widths.
// 48 B written per ray, nothing read (the pose is in the descriptor); four fp64 sincos per thread.
__global__ void __launch_bounds__(256)
spherical_rays_kernel(mnrf_spherical_desc d, float* __restrict__ origins, float* __restrict__ directions,
                      float* __restrict__ viewdirs, float* __restrict__ radii, float* __restrict__ imageplane) {
  const int64_t n = (int64_t)d.height * d.width;
  const double two_pi = 2.0 * 3.141592653589793;     // 2 * np.pi
  const double pi = 3.141592653589793;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t y = i / d.width, x = i - y * d.width;
    const double th0 = linspace_node(x, d.width, two_pi), th1 = linspace_node(x + 1, d.width, two_pi);
    const double ph0 = linspace_node(y, d.height, pi), ph1 = linspace_node(y + 1, d.height, pi);
    const Vec3<double> dir = sphere_dir(d.camtoworld, th0, ph0);
    const Vec3<double> dx = sphere_dir(d.camtoworld, th1, ph0);
    const Vec3<double> dy = sphere_dir(d.camtoworld, th0, ph1);
    const float r = (float)cone_radius(dist3(dx, dir), dist3(dy, dir));
    const float o[3] = {(float)d.camtoworld[3], (float)d.camtoworld[7], (float)d.camtoworld[11]};
    const float v[3] = {(float)dir.x, (float)dir.y, (float)dir.z};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      origins[3 * i + c] = o[c];
      directions[3 * i + c] = v[c];
      viewdirs[3 * i + c] = v[c];
    }
    radii[i] = r;
    imageplane[2 * i + 0] = 0.f; imageplane[2 * i + 1] = 0.f;
  }
}

}  // namespace mnrf

extern "C" int mnrf_spherical_rays(const mnrf_spherical_desc* d, float* origins, float* directions,
                                   float* viewdirs, float* radii, float* imageplane, mnrf_stream stream) {
  using namespace mnrf;
  set_error("");
  MNRF_CHECK(d && origins && directions && viewdirs && radii && imageplane, "mnrf_spherical_rays: null pointer");
  MNRF_CHECK(d->height >= 1 && d->width >= 1, "mnrf_spherical_rays: height and width must be >= 1");
  const int64_t blocks = ((int64_t)d->height * d->width + 255) / 256;
  const int64_t maxb = (int64_t)mnrf_num_sms() * 8;
  spherical_rays_kernel<<<(int)(blocks < maxb ? blocks : maxb), 256, 0, (cudaStream_t)stream>>>(
      *d, origins, directions, viewdirs, radii, imageplane);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_pixels_to_rays(const mnrf_camera_desc* d, const int32_t* pix_x, const int32_t* pix_y,
                                   const int32_t* cam_idx, const float* pixtocams, const float* camtoworlds,
                                   float* origins, float* directions, float* viewdirs, float* radii,
                                   float* imageplane, mnrf_stream stream) {
  using namespace mnrf;
  set_error("");
  if (d && d->num_rays == 0) return 0;            // nothing to do (and empty tensors carry null pointers)
  MNRF_CHECK(d && pix_x && pix_y && pixtocams && camtoworlds && origins && directions && viewdirs && radii &&
             imageplane, "mnrf_pixels_to_rays: null pointer");
  MNRF_CHECK(d->num_cameras >= 1, "mnrf_pixels_to_rays: num_cameras must be >= 1");
  MNRF_CHECK(d->num_cameras == 1 || cam_idx, "mnrf_pixels_to_rays: cam_idx is required with several cameras");
  MNRF_CHECK(d->camtype == MNRF_CAM_PERSPECTIVE || d->camtype == MNRF_CAM_FISHEYE,
             "mnrf_pixels_to_rays: camtype must be perspective or fisheye");
  MNRF_CHECK(!d->has_distortion || d->undistort_iters >= 0, "mnrf_pixels_to_rays: undistort_iters < 0");
  if (d->num_rays == 0) return 0;
  int blocks = ceil_div(d->num_rays, 256);
  const int maxb = mnrf_num_sms() * 8;
  if (blocks > maxb) blocks = maxb;
  pixels_to_rays_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(*d, pix_x, pix_y, cam_idx, pixtocams,
                                                                  camtoworlds, origins, directions, viewdirs,
                                                                  radii, imageplane);
  MNRF_LAUNCH_CHECK();
  return 0;
}
