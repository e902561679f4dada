// Marching cubes on an fp32 scalar grid [nz, ny, nx]: a point is inside when its value is above `level`.
//
// Point p = (z * ny + y) * nx + x owns the grid edges that leave it along +x, +y and +z (edge id 3 p + axis), and,
// when it is not on the upper face of any axis, the cell whose lowest corner it is (cell id p).  Two phases:
//   count: per edge a cut flag, per cell its triangle count (0 for points that start no cell);
//   emit:  given inclusive scans of both, one vertex per cut edge at the linear crossing, stored at the edge's
//          rank among the cut edges, and each cell's triangles at its rank, in case-table order.
// Vertices and triangles are therefore ordered by edge and cell id, and the output does not depend on scheduling.
// The case table (mc_tables.cuh, tools/gen_mc_tables.py) pairs the cut edges of each face from the face's corners
// alone, so the two cells that share a face agree on it: the mesh is closed and consistently wound wherever the
// level set stays off the grid boundary.
// A third pass (mc_normals_kernel), run after emit with the same scan, writes one unit normal per vertex, also at the
// edge's rank.
// A NaN grid point is unobserved: a cell with a NaN corner has no triangles, an edge with a NaN end is not cut, and an
// edge is cut only if a cell it borders has eight observed corners, so every vertex belongs to a face.  On a grid
// without NaN the output is what it was before unobserved points existed.
//
// Also the TSDF fusion of rendered depth maps (tsdf_integrate_kernel): one thread per grid point, its running
// truncated signed distance, weight and colour sums held in registers across every view of a launch.
//
// And the two passes of mesh cleaning: connected components by union-find (uf_*_kernel) and the number of views
// each vertex lands in (points_view_count_kernel).
#include <algorithm>

#include <cuda/atomic>

#include "camera.cuh"
#include "mc_tables.cuh"

namespace mnrf {

constexpr int kMcMaxDim = 1024;

struct McGrid {
  int nx, ny, nz;
  int64_t n;          // points
  float level;
};

__device__ __forceinline__ void mc_coords(const McGrid& g, int64_t p, int& x, int& y, int& z) {
  const int64_t row = p / g.nx;
  x = (int)(p - row * g.nx);
  z = (int)(row / g.ny);
  y = (int)(row - (int64_t)z * g.ny);
}

__device__ __forceinline__ int64_t mc_stride(const McGrid& g, int axis) {
  return axis == 0 ? 1 : axis == 1 ? (int64_t)g.nx : (int64_t)g.nx * g.ny;
}

// inside pattern of the cell whose lowest corner is p: bit i = corner (i & 1, i >> 1 & 1, i >> 2 & 1)
__device__ __forceinline__ int mc_case(const McGrid& g, const float* __restrict__ f, int64_t p) {
  const int64_t sy = g.nx, sz = (int64_t)g.nx * g.ny;
  int c = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    c |= (__ldg(f + p + (i & 1) + (i >> 1 & 1) * sy + (i >> 2 & 1) * sz) > g.level) << i;
  return c;
}

// mc_case, and whether all eight corners are observed (not NaN)
__device__ __forceinline__ int mc_case(const McGrid& g, const float* __restrict__ f, int64_t p, bool& observed) {
  const int64_t sy = g.nx, sz = (int64_t)g.nx * g.ny;
  int c = 0;
  bool nan = false;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float v = __ldg(f + p + (i & 1) + (i >> 1 & 1) * sy + (i >> 2 & 1) * sz);
    c |= (v > g.level) << i;
    nan |= isnan(v);
  }
  observed = !nan;
  return c;
}

// Whether the edge leaving point p = (c[0], c[1], c[2]) along `axis` borders a cell with eight observed corners,
// other than the cell whose lowest corner is p (the caller knows that one): the cells whose lowest corners are p
// moved down by one along either or both of the other two axes.
__device__ __forceinline__ bool mc_edge_other_cell_observed(const McGrid& g, const float* __restrict__ f, int64_t p,
                                                            const int c[3], const int dim[3], int axis) {
  const int b0 = axis == 0 ? 1 : 0, b1 = axis == 2 ? 1 : 2;
  for (int j = 1; j < 4; ++j) {
    const int l0 = c[b0] - (j & 1), l1 = c[b1] - (j >> 1);
    if (l0 < 0 || l0 + 1 >= dim[b0] || l1 < 0 || l1 + 1 >= dim[b1]) continue;
    bool observed;
    mc_case(g, f, p - (j & 1) * mc_stride(g, b0) - (j >> 1) * mc_stride(g, b1), observed);
    if (observed) return true;
  }
  return false;
}

// global id of edge e of the cell at p: e runs along axis e / 4 from the corner whose two other coordinates are the
// bits of e % 4, lower axis first
__device__ __forceinline__ int64_t mc_edge_id(const McGrid& g, int64_t p, int e) {
  const int axis = e >> 2, j = e & 3;
  const int a0 = axis == 0 ? 1 : 0, a1 = axis == 2 ? 1 : 2;
  return 3 * (p + (j & 1) * mc_stride(g, a0) + (j >> 1) * mc_stride(g, a1)) + axis;
}

__global__ void __launch_bounds__(256)
mc_count_kernel(McGrid g, const float* __restrict__ f, uint8_t* __restrict__ edge_cut, uint8_t* __restrict__ cell_tris) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < g.n; p += (int64_t)gridDim.x * blockDim.x) {
    int x, y, z;
    mc_coords(g, p, x, y, z);
    const float f0 = __ldg(f + p);
    const bool in0 = f0 > g.level;
    const int c[3] = {x, y, z};
    const int dim[3] = {g.nx, g.ny, g.nz};
    const bool cell = x + 1 < g.nx && y + 1 < g.ny && z + 1 < g.nz;
    bool observed = false;
    const int cs = cell ? mc_case(g, f, p, observed) : 0;
    // the cell at p borders all three edges of p: only where it is missing or unobserved do the other cells count
    const bool cell_ok = cell && observed;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      bool cut = false;
      if (c[a] + 1 < dim[a]) {
        const float f1 = __ldg(f + p + mc_stride(g, a));
        cut = (f1 > g.level) != in0 && !isnan(f0) && !isnan(f1) &&
              (cell_ok || mc_edge_other_cell_observed(g, f, p, c, dim, a));
      }
      edge_cut[3 * p + a] = cut;
    }
    cell_tris[p] = cell_ok ? kMcNumTris[cs] : 0;
  }
}

__global__ void __launch_bounds__(256)
mc_emit_kernel(McGrid g, const float* __restrict__ f, const uint8_t* __restrict__ edge_cut,
               const uint8_t* __restrict__ cell_tris, const int64_t* __restrict__ edge_scan,
               const int64_t* __restrict__ tri_scan, float* __restrict__ vertices, int32_t* __restrict__ faces) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < g.n; p += (int64_t)gridDim.x * blockDim.x) {
    int x, y, z;
    mc_coords(g, p, x, y, z);
    const float f0 = __ldg(f + p);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (!edge_cut[3 * p + a]) continue;
      const float f1 = __ldg(f + p + mc_stride(g, a));
      const float t = (g.level - f0) / (f1 - f0);     // f1 != f0: exactly one end is above the level
      float* v = vertices + 3 * (edge_scan[3 * p + a] - 1);
      v[0] = (float)x + (a == 0 ? t : 0.f);
      v[1] = (float)y + (a == 1 ? t : 0.f);
      v[2] = (float)z + (a == 2 ? t : 0.f);
    }
    const int nt = cell_tris[p];
    if (nt == 0) continue;
    const int cs = mc_case(g, f, p);
    int32_t* tri = faces + 3 * (tri_scan[p] - nt);
    for (int i = 0; i < 3 * nt; ++i) tri[i] = (int32_t)(edge_scan[mc_edge_id(g, p, kMcTris[cs][i])] - 1);
  }
}

// Gradient of the grid at point p = (x, y, z): central differences, one-sided on the grid boundary and next to an
// unobserved (NaN) neighbour.  Returns false when both neighbours along an axis are missing or unobserved.
__device__ __forceinline__ bool mc_grad(const McGrid& g, const float* __restrict__ f, int64_t p, int x, int y, int z,
                                        float grad[3]) {
  const int c[3] = {x, y, z};
  const int dim[3] = {g.nx, g.ny, g.nz};
  const float f0 = __ldg(f + p);
  bool ok = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int64_t s = mc_stride(g, a);
    const float fm = c[a] > 0 ? __ldg(f + p - s) : NAN;
    const float fp = c[a] + 1 < dim[a] ? __ldg(f + p + s) : NAN;
    if (!isnan(fm) && !isnan(fp)) grad[a] = 0.5f * (fp - fm);
    else if (!isnan(fp)) grad[a] = fp - f0;
    else if (!isnan(fm)) grad[a] = f0 - fm;
    else { grad[a] = 0.f; ok = false; }
  }
  return ok;
}

// One unit normal per cut edge, at the edge's rank (the index of its vertex): -grad / |grad| with the gradients of
// the edge's two ends interpolated at the vertex's t.  The gradient is scaled by its largest component before it is
// squared, so no finite gradient overflows; a zero or non-finite one gives the edge's direction from its inside end
// to its outside end.
__global__ void __launch_bounds__(256)
mc_normals_kernel(McGrid g, const float* __restrict__ f, const uint8_t* __restrict__ edge_cut,
                  const int64_t* __restrict__ edge_scan, float* __restrict__ normals) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < g.n; p += (int64_t)gridDim.x * blockDim.x) {
    int x, y, z;
    mc_coords(g, p, x, y, z);
    const float f0 = __ldg(f + p);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (!edge_cut[3 * p + a]) continue;
      const int64_t q = p + mc_stride(g, a);
      const float f1 = __ldg(f + q);
      const float t = (g.level - f0) / (f1 - f0);     // as mc_emit_kernel
      float g0[3], g1[3], n[3];
      const bool ok = mc_grad(g, f, p, x, y, z, g0) & mc_grad(g, f, q, x + (a == 0), y + (a == 1), z + (a == 2), g1);
#pragma unroll
      for (int i = 0; i < 3; ++i) n[i] = g0[i] + t * (g1[i] - g0[i]);
      const float m = fmaxf(fabsf(n[0]), fmaxf(fabsf(n[1]), fabsf(n[2])));
      if (ok && m > 0.f && isfinite(m)) {
#pragma unroll
        for (int i = 0; i < 3; ++i) n[i] = n[i] / m;
        const float len = sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
#pragma unroll
        for (int i = 0; i < 3; ++i) n[i] = -n[i] / len;
      } else {
        const float dir = f0 > g.level ? 1.f : -1.f;   // inside end first: +axis when the lower end is inside
#pragma unroll
        for (int i = 0; i < 3; ++i) n[i] = i == a ? dir : 0.f;
      }
      float* o = normals + 3 * (edge_scan[3 * p + a] - 1);
      o[0] = n[0];
      o[1] = n[1];
      o[2] = n[2];
    }
  }
}

// ---------------------------------------------------------------------------------------------------- TSDF fusion
struct TsdfArgs {
  mnrf_camera_desc cam;
  int nx, ny, nz;
  int64_t n;
  double x0, y0, z0, h;
  int num_views, height, width;
  float tau;
  const float* w2c;      // [K, 3, 4]
  const float* c2p;      // [K or 1, 3, 3]
  int64_t c2p_stride;    // 9 or 0
  const float* depth;    // [K, H, W]
  const float* acc;      // [K, H, W]
  const float* rgb;      // [K, H, W, 3] or null
  float* tsdf;
  float* weight;
  float* color_sum;      // [n, 3] or null (with rgb)
  float* color_weight;
};

// Grid point p = lo + h (x, y, z), rounded to fp32 from fp64 as mesh.density_grid does.  For each view in order:
// skip it when the point has no pixel, lands off the image or on a non-finite depth; d = depth - t where the pixel's
// acc >= 0.5 (its median distance is a surface) and +inf otherwise (the median sits at `far`: seen-through space);
// skip it when d < -tau (occluded); else fold min(d, tau) / tau into the running mean and, when |d| <= tau, the
// pixel's colour into the colour sums.  No atomics: the state of a point depends on the views and their order only,
// not on how they are split into launches.  Per point and view: 8 B of depth and acc (+ 12 B of rgb) gathered from
// L2; per point: 8 B (+ 16 B) of state read and written once.
template <bool kColor>
__global__ void __launch_bounds__(256)
tsdf_integrate_kernel(const TsdfArgs a) {
  const float tau = a.tau;
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < a.n; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = p / a.nx;
    const int x = (int)(p - row * a.nx);
    const int z = (int)(row / a.ny);
    const int y = (int)(row - (int64_t)z * a.ny);
    const V3 pt{(float)(a.x0 + (double)x * a.h), (float)(a.y0 + (double)y * a.h), (float)(a.z0 + (double)z * a.h)};
    float s = a.tsdf[p], w = a.weight[p];
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, cw = 0.f;
    if (kColor) {
      c0 = a.color_sum[3 * p]; c1 = a.color_sum[3 * p + 1]; c2 = a.color_sum[3 * p + 2];
      cw = a.color_weight[p];
    }
    for (int k = 0; k < a.num_views; ++k) {
      int px, py;
      float t;
      if (!project_to_pixel(a.cam, a.w2c + 12 * (int64_t)k, a.c2p + a.c2p_stride * k, pt, a.width, a.height, px, py,
                            t))
        continue;
      const int64_t i = ((int64_t)k * a.height + py) * a.width + px;
      const float dep = __ldg(a.depth + i);
      if (!isfinite(dep)) continue;
      const float d = __ldg(a.acc + i) >= 0.5f ? dep - t : INFINITY;
      if (d < -tau) continue;
      s = (w * s + fminf(d, tau) / tau) / (w + 1.f);
      w = w + 1.f;
      if (kColor && fabsf(d) <= tau) {
        c0 = c0 + __ldg(a.rgb + 3 * i);
        c1 = c1 + __ldg(a.rgb + 3 * i + 1);
        c2 = c2 + __ldg(a.rgb + 3 * i + 2);
        cw = cw + 1.f;
      }
    }
    a.tsdf[p] = s;
    a.weight[p] = w;
    if (kColor) {
      a.color_sum[3 * p] = c0; a.color_sum[3 * p + 1] = c1; a.color_sum[3 * p + 2] = c2;
      a.color_weight[p] = cw;
    }
  }
}

// ------------------------------------------------------------------------------------------ mesh cleaning
// Connected components of a triangle mesh by union-find on `parent` (the labels array): initialise parent[v] = v;
// hook every face's edges; compress.  A root is only ever hooked under a smaller root, and path halving only moves a
// parent to one of its ancestors, so parent[v] <= v always and each root is its component's minimum vertex: after
// compression every label is that minimum, whatever the thread schedule.  Loads of parent go through relaxed
// device-scope atomics so that no thread keeps a stale copy across the loop of find; the halving stores of the hook
// pass are relaxed stores.  A non-root never becomes a root again, so a halving store never overwrites a hook.
using ParentRef = cuda::atomic_ref<int, cuda::thread_scope_device>;

__device__ __forceinline__ int uf_find(int* parent, int x) {
  while (true) {
    const int p = ParentRef(parent[x]).load(cuda::memory_order_relaxed);
    if (p == x) return x;
    const int gp = ParentRef(parent[p]).load(cuda::memory_order_relaxed);
    if (gp == p) return p;
    ParentRef(parent[x]).store(gp, cuda::memory_order_relaxed);      // path halving: gp is an ancestor of x
    x = gp;
  }
}

__device__ __forceinline__ void uf_union(int* parent, int a, int b) {
  while (true) {
    a = uf_find(parent, a);
    b = uf_find(parent, b);
    if (a == b) return;
    if (a < b) { const int s = a; a = b; b = s; }
    if (atomicCAS(parent + a, a, b) == a) return;     // a was still a root: hooked under b; else retry from find
  }
}

__global__ void __launch_bounds__(256) uf_init_kernel(int32_t n, int* __restrict__ parent) {
  for (int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; v < n; v += (int64_t)gridDim.x * blockDim.x)
    parent[v] = (int)v;
}

// one thread per face: its edges (v0, v1) and (v0, v2) join all three corners
__global__ void __launch_bounds__(256) uf_hook_kernel(int64_t num_faces, const int32_t* __restrict__ faces,
                                                      int* parent) {
  for (int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; f < num_faces;
       f += (int64_t)gridDim.x * blockDim.x) {
    const int v0 = __ldg(faces + 3 * f), v1 = __ldg(faces + 3 * f + 1), v2 = __ldg(faces + 3 * f + 2);
    uf_union(parent, v0, v1);
    uf_union(parent, v0, v2);
  }
}

// Each label becomes its root.  The walk makes no halving stores: one could land on a vertex whose thread has
// already stored its root and put back a non-root ancestor.  The only stores of this pass are roots.
__global__ void __launch_bounds__(256) uf_compress_kernel(int32_t n, int* parent) {
  for (int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; v < n; v += (int64_t)gridDim.x * blockDim.x) {
    int x = (int)v;
    for (int p; (p = ParentRef(parent[x]).load(cuda::memory_order_relaxed)) != x;) x = p;
    ParentRef(parent[v]).store(x, cuda::memory_order_relaxed);
  }
}

struct ViewCountArgs {
  mnrf_camera_desc cam;
  int64_t n;
  const float* points;   // [n, 3]
  int num_views, height, width;
  const float* w2c;      // [K, 3, 4]
  const float* c2p;      // [K or 1, 3, 3]
  int64_t c2p_stride;    // 9 or 0
  int32_t* counts;
};

// One thread per point: the number of views whose image it lands on (project_to_pixel, the rule of the fusion).
__global__ void __launch_bounds__(256) points_view_count_kernel(const ViewCountArgs a) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < a.n; p += (int64_t)gridDim.x * blockDim.x) {
    const V3 pt{__ldg(a.points + 3 * p), __ldg(a.points + 3 * p + 1), __ldg(a.points + 3 * p + 2)};
    int c = 0;
    for (int k = 0; k < a.num_views; ++k) {
      int px, py;
      float t;
      c += project_to_pixel(a.cam, a.w2c + 12 * (int64_t)k, a.c2p + a.c2p_stride * k, pt, a.width, a.height, px, py,
                            t);
    }
    a.counts[p] = c;
  }
}

}  // namespace mnrf

extern "C" int mnrf_marching_cubes(int32_t phase, int32_t nx, int32_t ny, int32_t nz, const float* grid, float level,
                                   uint8_t* edge_cut, uint8_t* cell_tris, const int64_t* edge_scan,
                                   const int64_t* tri_scan, float* vertices, int32_t* faces, mnrf_stream stream) {
  using namespace mnrf;
  MNRF_CHECK(phase == MNRF_MC_COUNT || phase == MNRF_MC_EMIT, "mnrf_marching_cubes: unknown phase %d", phase);
  MNRF_CHECK(nx >= 2 && ny >= 2 && nz >= 2 && nx <= kMcMaxDim && ny <= kMcMaxDim && nz <= kMcMaxDim,
             "mnrf_marching_cubes: grid %d x %d x %d (nz x ny x nx), each side must be in [2, %d]", nz, ny, nx,
             kMcMaxDim);
  MNRF_CHECK(grid && edge_cut && cell_tris, "mnrf_marching_cubes: null pointer");
  if (phase == MNRF_MC_EMIT)
    MNRF_CHECK(edge_scan && tri_scan && vertices && faces, "mnrf_marching_cubes: null pointer (emit)");
  const McGrid g{nx, ny, nz, (int64_t)nx * ny * nz, level};
  const int blocks = (int)std::min<int64_t>((g.n + 255) / 256, (int64_t)mnrf_num_sms() * 16);
  if (phase == MNRF_MC_COUNT) {
    mc_count_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(g, grid, edge_cut, cell_tris);
  } else {
    mc_emit_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(g, grid, edge_cut, cell_tris, edge_scan, tri_scan,
                                                             vertices, faces);
  }
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_mc_normals(int32_t nx, int32_t ny, int32_t nz, const float* grid, float level,
                               const uint8_t* edge_cut, const int64_t* edge_scan, float* normals, mnrf_stream stream) {
  using namespace mnrf;
  MNRF_CHECK(nx >= 2 && ny >= 2 && nz >= 2 && nx <= kMcMaxDim && ny <= kMcMaxDim && nz <= kMcMaxDim,
             "mnrf_mc_normals: grid %d x %d x %d (nz x ny x nx), each side must be in [2, %d]", nz, ny, nx, kMcMaxDim);
  MNRF_CHECK(grid && edge_cut && edge_scan && normals, "mnrf_mc_normals: null pointer");
  const McGrid g{nx, ny, nz, (int64_t)nx * ny * nz, level};
  const int blocks = (int)std::min<int64_t>((g.n + 255) / 256, (int64_t)mnrf_num_sms() * 16);
  mc_normals_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(g, grid, edge_cut, edge_scan, normals);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_tsdf_integrate(const mnrf_camera_desc* cam, int32_t nx, int32_t ny, int32_t nz, double x0,
                                   double y0, double z0, double h, int32_t num_views, int32_t height, int32_t width,
                                   const float* worldtocams, const float* camtopixs, const float* depth,
                                   const float* acc, const float* rgb, float tau, float* tsdf, float* weight,
                                   float* color_sum, float* color_weight, mnrf_stream stream) {
  using namespace mnrf;
  set_error("");
  MNRF_CHECK(cam, "mnrf_tsdf_integrate: null camera descriptor");
  MNRF_CHECK(nx >= 2 && ny >= 2 && nz >= 2 && nx <= kMcMaxDim && ny <= kMcMaxDim && nz <= kMcMaxDim,
             "mnrf_tsdf_integrate: grid %d x %d x %d (nz x ny x nx), each side must be in [2, %d]", nz, ny, nx,
             kMcMaxDim);
  MNRF_CHECK(num_views >= 0 && height >= 1 && width >= 1, "mnrf_tsdf_integrate: %d views of %d x %d pixels",
             num_views, height, width);
  MNRF_CHECK(cam->camtype == MNRF_CAM_PERSPECTIVE || cam->camtype == MNRF_CAM_FISHEYE,
             "mnrf_tsdf_integrate: camtype must be perspective or fisheye");
  MNRF_CHECK(!cam->has_ndc, "mnrf_tsdf_integrate: NDC cameras are not supported");
  MNRF_CHECK(cam->num_cameras == 1 || cam->num_cameras == num_views,
             "mnrf_tsdf_integrate: num_cameras = %d camera-to-pixel matrices for %d views", cam->num_cameras,
             num_views);
  MNRF_CHECK(tau > 0.f && isfinite(tau) && h > 0.0 && isfinite(h), "mnrf_tsdf_integrate: tau %g, h %g", tau, h);
  MNRF_CHECK(tsdf && weight, "mnrf_tsdf_integrate: null state pointer");
  MNRF_CHECK(!rgb == !color_sum && !color_sum == !color_weight,
             "mnrf_tsdf_integrate: rgb, color_sum and color_weight go together");
  if (num_views == 0) return 0;
  MNRF_CHECK(worldtocams && camtopixs && depth && acc, "mnrf_tsdf_integrate: null view pointer");
  TsdfArgs a{*cam, nx, ny, nz, (int64_t)nx * ny * nz, x0, y0, z0, h, num_views, height, width, tau,
             worldtocams, camtopixs, cam->num_cameras == 1 ? 0 : 9, depth, acc, rgb, tsdf, weight, color_sum,
             color_weight};
  const int blocks = (int)std::min<int64_t>((a.n + 255) / 256, (int64_t)mnrf_num_sms() * 16);
  if (rgb)
    tsdf_integrate_kernel<true><<<blocks, 256, 0, (cudaStream_t)stream>>>(a);
  else
    tsdf_integrate_kernel<false><<<blocks, 256, 0, (cudaStream_t)stream>>>(a);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_mesh_components(int32_t num_vertices, int64_t num_faces, const int32_t* faces, int32_t* labels,
                                    mnrf_stream stream) {
  using namespace mnrf;
  set_error("");
  MNRF_CHECK(num_vertices >= 0 && num_faces >= 0, "mnrf_mesh_components: %d vertices, %lld faces", num_vertices,
             (long long)num_faces);
  MNRF_CHECK(num_faces == 0 || num_vertices > 0, "mnrf_mesh_components: %lld faces on no vertices",
             (long long)num_faces);
  if (num_vertices == 0) return 0;
  MNRF_CHECK(labels && (faces || num_faces == 0), "mnrf_mesh_components: null pointer");
  const int cap = mnrf_num_sms() * 16;
  const int vblocks = (int)std::min<int64_t>((num_vertices + 255) / 256, cap);
  uf_init_kernel<<<vblocks, 256, 0, (cudaStream_t)stream>>>(num_vertices, labels);
  if (num_faces > 0) {
    const int fblocks = (int)std::min<int64_t>((num_faces + 255) / 256, cap);
    uf_hook_kernel<<<fblocks, 256, 0, (cudaStream_t)stream>>>(num_faces, faces, labels);
  }
  uf_compress_kernel<<<vblocks, 256, 0, (cudaStream_t)stream>>>(num_vertices, labels);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_points_view_count(const mnrf_camera_desc* cam, int64_t n, const float* points, int32_t num_views,
                                      int32_t height, int32_t width, const float* worldtocams,
                                      const float* camtopixs, int32_t* counts, mnrf_stream stream) {
  using namespace mnrf;
  set_error("");
  MNRF_CHECK(cam, "mnrf_points_view_count: null camera descriptor");
  MNRF_CHECK(n >= 0 && num_views >= 0 && height >= 1 && width >= 1,
             "mnrf_points_view_count: %lld points, %d views of %d x %d pixels", (long long)n, num_views, height,
             width);
  MNRF_CHECK(cam->camtype == MNRF_CAM_PERSPECTIVE || cam->camtype == MNRF_CAM_FISHEYE,
             "mnrf_points_view_count: camtype must be perspective or fisheye");
  MNRF_CHECK(!cam->has_ndc, "mnrf_points_view_count: NDC cameras are not supported");
  MNRF_CHECK(cam->num_cameras == 1 || cam->num_cameras == num_views,
             "mnrf_points_view_count: num_cameras = %d camera-to-pixel matrices for %d views", cam->num_cameras,
             num_views);
  if (n == 0) return 0;
  MNRF_CHECK(points && counts, "mnrf_points_view_count: null point or count pointer");
  MNRF_CHECK(num_views == 0 || (worldtocams && camtopixs), "mnrf_points_view_count: null view pointer");
  const ViewCountArgs a{*cam, n, points, num_views, height, width, worldtocams, camtopixs,
                        cam->num_cameras == 1 ? 0 : 9, counts};
  const int blocks = (int)std::min<int64_t>((n + 255) / 256, (int64_t)mnrf_num_sms() * 16);
  points_view_count_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(a);
  MNRF_LAUNCH_CHECK();
  return 0;
}
