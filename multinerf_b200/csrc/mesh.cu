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
// With kContract, the grid lies in the contracted space of an unbounded scene (coord.contract): each point is
// projected at its world preimage, and its signed distance is measured in contracted space.  uncontract_kernel maps
// the vertices and normals of a mesh extracted there back to world space.
//
// And the two passes of mesh cleaning: connected components by union-find (uf_*_kernel) and the number of views
// each vertex lands in (points_view_count_kernel); mesh simplification by quadric edge collapse (qem_*_kernel); and
// the texture atlas of a mesh: its per-face charts and one surface sample per texel (tex_*_kernel).
#include <algorithm>
#include <cmath>

#include <cuda/atomic>

#include "camera.cuh"
#include "contract.cuh"
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
//
// kContract: the grid points p lie in contracted space.  A point with |p| >= 2 has no world preimage and is left
// untouched (weight 0: unobserved).  Otherwise x = inv_contract(p) is projected; the pixel's surface point on the ray
// through x is s = o + (x - o) depth / t (o: the camera centre of w2c), and d = sign(depth - t) |contract(s) - p|,
// the distance in contracted space, with tau in contracted units.
template <bool kColor, bool kContract = false>
__global__ void __launch_bounds__(256)
tsdf_integrate_kernel(const TsdfArgs a) {
  const float tau = a.tau;
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < a.n; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = p / a.nx;
    const int x = (int)(p - row * a.nx);
    const int z = (int)(row / a.ny);
    const int y = (int)(row - (int64_t)z * a.ny);
    const V3 pt{(float)(a.x0 + (double)x * a.h), (float)(a.y0 + (double)y * a.h), (float)(a.z0 + (double)z * a.h)};
    V3 pw = pt;
    if (kContract) {
      if (!(pt.x * pt.x + pt.y * pt.y + pt.z * pt.z < 4.f)) continue;
      const float zc[3] = {pt.x, pt.y, pt.z};
      float xw[3];
      inv_contract_point(zc, xw);
      if (!(isfinite(xw[0]) && isfinite(xw[1]) && isfinite(xw[2]))) continue;     // |p| rounds to 2
      pw = V3{xw[0], xw[1], xw[2]};
    }
    float s = a.tsdf[p], w = a.weight[p];
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, cw = 0.f;
    if (kColor) {
      c0 = a.color_sum[3 * p]; c1 = a.color_sum[3 * p + 1]; c2 = a.color_sum[3 * p + 2];
      cw = a.color_weight[p];
    }
    for (int k = 0; k < a.num_views; ++k) {
      int px, py;
      float t;
      if (!project_to_pixel(a.cam, a.w2c + 12 * (int64_t)k, a.c2p + a.c2p_stride * k, pw, a.width, a.height, px, py,
                            t))
        continue;
      const int64_t i = ((int64_t)k * a.height + py) * a.width + px;
      const float dep = __ldg(a.depth + i);
      if (!isfinite(dep)) continue;
      float d;
      if (!kContract) {
        d = __ldg(a.acc + i) >= 0.5f ? dep - t : INFINITY;
      } else if (__ldg(a.acc + i) >= 0.5f) {
        const float* m = a.w2c + 12 * (int64_t)k;
        const float f = dep / t;
        const float xw[3] = {pw.x, pw.y, pw.z};
        float sp[3], sc[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const float o = -(m[j] * m[3] + m[4 + j] * m[7] + m[8 + j] * m[11]);     // o = -R^T t
          sp[j] = o + (xw[j] - o) * f;
        }
        contract_point(sp, sc);
        const float e0 = sc[0] - pt.x, e1 = sc[1] - pt.y, e2 = sc[2] - pt.z;
        const float dist = sqrtf(e0 * e0 + e1 * e1 + e2 * e2);
        d = dep >= t ? dist : -dist;
      } else {
        d = INFINITY;
      }
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

// Contracted mesh -> world: x = inv_contract(p) per point and, with normals, the unit world normal J(x) n of each
// contracted level-set normal n (a gradient's pullback through y = contract(x), J symmetric).  J n is scaled by its
// largest component before it is squared, as mc_normals_kernel scales; a zero or non-finite J n (n zero, or |p| so
// close to 2 that x overflows) falls back to n itself, then to (0, 0, 1).
__device__ __forceinline__ bool unit_normal(float v[3]) {
  const float m = fmaxf(fabsf(v[0]), fmaxf(fabsf(v[1]), fabsf(v[2])));
  if (!(m > 0.f && isfinite(m))) return false;
#pragma unroll
  for (int i = 0; i < 3; ++i) v[i] = v[i] / m;
  const float len = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
#pragma unroll
  for (int i = 0; i < 3; ++i) v[i] = v[i] / len;
  return true;
}

__global__ void __launch_bounds__(256)
uncontract_kernel(int64_t n, const float* __restrict__ points, const float* __restrict__ normals,
                  float* __restrict__ world_points, float* __restrict__ world_normals) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float z[3] = {points[3 * i], points[3 * i + 1], points[3 * i + 2]};
    float x[3];
    inv_contract_point(z, x);
#pragma unroll
    for (int j = 0; j < 3; ++j) world_points[3 * i + j] = x[j];
    if (!normals) continue;
    float s, q, xh[3], nw[3];
    contract_jacobian(x, s, q, xh);
    const float nc[3] = {normals[3 * i], normals[3 * i + 1], normals[3 * i + 2]};
    contract_jacobian_apply(s, q, xh, nc, nw);
    if (!unit_normal(nw)) {
      nw[0] = nc[0]; nw[1] = nc[1]; nw[2] = nc[2];
      if (!unit_normal(nw)) { nw[0] = 0.f; nw[1] = 0.f; nw[2] = 1.f; }
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) world_normals[3 * i + j] = nw[j];
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

// ------------------------------------------------------------------------------------- mesh simplification
// Parallel greedy quadric edge collapse (Garland and Heckbert 1997) in rounds; mesh.simplify_mesh drives it and
// tests/mesh_simplify_ref.py restates every kernel below in numpy.  All geometry is fp64 in registers (positions are
// stored fp32, quadrics fp64) and the unit is compiled with -fmad=false, so each expression rounds exactly as its
// numpy restatement, operation by operation: keep both in the same order.  The only atomics are atomicOr of
// constant flag bits and atomicMin of 64-bit keys, whose results do not depend on their order.
// A quadric is 10 fp64 values: (aa, ab, ac, ad, bb, bc, bd, cc, cd, dd) of w (a, b, c, d)^T (a, b, c, d).
constexpr double kBoundaryWeight = 1000.0;    // boundary-edge planes, times |e|^2
constexpr double kDetRel = 1e-10;             // |det A| <= kDetRel max|A_ij|^3: A is near-singular
constexpr int kMaxValence = 24;               // faces at a vertex; edges at a vertex with more are never collapsed
constexpr int kFlagBoundary = 1, kFlagNonManifold = 2;

struct D3 {
  double x, y, z;
};

__device__ __forceinline__ D3 ld_pos(const float* __restrict__ v, int i) {
  return D3{(double)v[3 * (int64_t)i], (double)v[3 * (int64_t)i + 1], (double)v[3 * (int64_t)i + 2]};
}
__device__ __forceinline__ D3 sub(D3 a, D3 b) { return D3{a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ double dot(D3 a, D3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ D3 cross(D3 a, D3 b) {
  return D3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}

// q += w (a, b, c, d)^T (a, b, c, d), each product as w * (a * b)
__device__ __forceinline__ void add_plane(double q[10], double a, double b, double c, double d, double w) {
  q[0] = q[0] + w * (a * a); q[1] = q[1] + w * (a * b); q[2] = q[2] + w * (a * c); q[3] = q[3] + w * (a * d);
  q[4] = q[4] + w * (b * b); q[5] = q[5] + w * (b * c); q[6] = q[6] + w * (b * d);
  q[7] = q[7] + w * (c * c); q[8] = q[8] + w * (c * d); q[9] = q[9] + w * (d * d);
}

// The unit normal of the plane through p0, p1, p2 (from (p1 - p0) x (p2 - p0)) and twice the triangle's area;
// false when the area is 0.
__device__ __forceinline__ bool face_plane(D3 p0, D3 p1, D3 p2, D3& u, double& len) {
  const D3 n = cross(sub(p1, p0), sub(p2, p0));
  len = sqrt(dot(n, n));
  if (!(len > 0.0)) return false;
  u = D3{n.x / len, n.y / len, n.z / len};
  return true;
}

// v^T Q v of the homogeneous point (v, 1)
__device__ __forceinline__ double quadric_eval(const double q[10], D3 v) {
  return v.x * (q[0] * v.x + 2.0 * (q[1] * v.y + q[2] * v.z + q[3])) + v.y * (q[4] * v.y + 2.0 * (q[5] * v.z + q[6])) +
         v.z * (q[7] * v.z + 2.0 * q[8]) + q[9];
}

__device__ __forceinline__ D3 round_f32(D3 v) {
  return D3{(double)__double2float_rn(v.x), (double)__double2float_rn(v.y), (double)__double2float_rn(v.z)};
}

__device__ __forceinline__ bool has_corner(const int32_t* __restrict__ faces, int f, int v) {
  const int64_t o = 3 * (int64_t)f;
  return faces[o] == v || faces[o + 1] == v || faces[o + 2] == v;
}

struct QemArgs {
  int32_t nv;
  int64_t nf, ne, nb;
  float* vertices;          // [nv, 3]
  int32_t* faces;           // [nf, 3]
  double* quadrics;         // [nv, 10]
  float* normals;           // [nv, 3] or null
  const int32_t* edges;     // [ne, 2]: (a, b), a < b, sorted
  const int64_t* edge_off;  // [ne + 1]: faces of edge e at edge_face[edge_off[e], edge_off[e + 1])
  const int32_t* edge_face;
  const int64_t* vf_off;    // [nv + 1]: faces at v at vf_face[vf_off[v], vf_off[v + 1]), ascending
  const int32_t* vf_face;
  const int32_t* bnd_edges; // [nb, 2]: the boundary edges, in edge order
  const int32_t* bnd_face;  // [nb]: the one face of each
  const int64_t* vb_off;    // [nv + 1]: boundary edges at v at vb_edge[vb_off[v], vb_off[v + 1]), ascending
  const int32_t* vb_edge;
  int32_t* flags;           // [nv]
  uint64_t* keys;           // [ne]
  float* positions;         // [ne, 3]
  uint64_t* vmin;           // [nv]
  uint64_t* rmin;           // [nv]
  uint8_t* selected;        // [ne]
  const uint8_t* collapse;  // [ne]
  uint8_t* face_alive;      // [nf]
};

#define QEM_LOOP(i, n) for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < (n); \
                            i += (int64_t)gridDim.x * blockDim.x)

// Per vertex: the area-weighted planes of its faces in face order, then the boundary-edge planes of its boundary
// edges in edge order.  A boundary edge's plane contains the edge and is perpendicular to its face.
__global__ void __launch_bounds__(256) qem_quadrics_kernel(const QemArgs a) {
  QEM_LOOP(v, a.nv) {
    double q[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int64_t k = a.vf_off[v]; k < a.vf_off[v + 1]; ++k) {
      const int64_t f = a.vf_face[k];
      const D3 p0 = ld_pos(a.vertices, a.faces[3 * f]);
      D3 u;
      double len;
      if (!face_plane(p0, ld_pos(a.vertices, a.faces[3 * f + 1]), ld_pos(a.vertices, a.faces[3 * f + 2]), u, len))
        continue;
      add_plane(q, u.x, u.y, u.z, -dot(u, p0), 0.5 * len);
    }
    for (int64_t k = a.vb_off[v]; k < a.vb_off[v + 1]; ++k) {
      const int64_t e = a.vb_edge[k], f = a.bnd_face[e];
      D3 u;
      double len;
      if (!face_plane(ld_pos(a.vertices, a.faces[3 * f]), ld_pos(a.vertices, a.faces[3 * f + 1]),
                      ld_pos(a.vertices, a.faces[3 * f + 2]), u, len))
        continue;
      const D3 x = ld_pos(a.vertices, a.bnd_edges[2 * e]);
      const D3 ev = sub(ld_pos(a.vertices, a.bnd_edges[2 * e + 1]), x);
      const D3 m = cross(ev, u);
      const double ml = sqrt(dot(m, m));
      if (!(ml > 0.0)) continue;
      const D3 mu{m.x / ml, m.y / ml, m.z / ml};
      add_plane(q, mu.x, mu.y, mu.z, -dot(mu, x), kBoundaryWeight * dot(ev, ev));
    }
    for (int i = 0; i < 10; ++i) a.quadrics[10 * v + i] = q[i];
  }
}

__global__ void __launch_bounds__(256) qem_flags_kernel(const QemArgs a) {
  QEM_LOOP(e, a.ne) {
    const int64_t c = a.edge_off[e + 1] - a.edge_off[e];
    const int bit = c == 1 ? kFlagBoundary : c > 2 ? kFlagNonManifold : 0;
    if (bit) {
      atomicOr(a.flags + a.edges[2 * e], bit);
      atomicOr(a.flags + a.edges[2 * e + 1], bit);
    }
  }
}

// Whether moving corner `from` of face f to p keeps the face's orientation: the new normal is not zero, and where
// the old one is not zero, their dot product is positive.
__device__ __forceinline__ bool keeps_orientation(const QemArgs& a, int64_t f, int from, D3 p) {
  const int v0 = a.faces[3 * f], v1 = a.faces[3 * f + 1], v2 = a.faces[3 * f + 2];
  const D3 c0 = ld_pos(a.vertices, v0), c1 = ld_pos(a.vertices, v1), c2 = ld_pos(a.vertices, v2);
  const D3 d0 = v0 == from ? p : c0, d1 = v1 == from ? p : c1, d2 = v2 == from ? p : c2;
  const D3 n = cross(sub(c1, c0), sub(c2, c0));
  const D3 m = cross(sub(d1, d0), sub(d2, d0));
  if (m.x == 0.0 && m.y == 0.0 && m.z == 0.0) return false;
  if (n.x == 0.0 && n.y == 0.0 && n.z == 0.0) return true;
  return dot(m, n) > 0.0;
}

// Whether a face at v has x as a corner: x is a neighbour of v
__device__ __forceinline__ bool star_has(const QemArgs& a, int v, int x) {
  for (int64_t k = a.vf_off[v]; k < a.vf_off[v + 1]; ++k)
    if (has_corner(a.faces, a.vf_face[k], x)) return true;
  return false;
}

// Per edge (a, b): the position and cost of its collapse and, when it may be collapsed, its key.  (256, 1): at the
// default bound ptxas caps the kernel at 80 registers and spills.
__global__ void __launch_bounds__(256, 1) qem_cost_kernel(const QemArgs a) {
  QEM_LOOP(e, a.ne) {
    const int va = a.edges[2 * e], vb = a.edges[2 * e + 1];
    double q[10];
    for (int i = 0; i < 10; ++i) q[i] = a.quadrics[10 * (int64_t)va + i] + a.quadrics[10 * (int64_t)vb + i];
    const D3 pa = ld_pos(a.vertices, va), pb = ld_pos(a.vertices, vb);
    // the minimiser of v^T Q v: A v = -(q3, q6, q8) by cofactors
    const double c00 = q[4] * q[7] - q[5] * q[5], c01 = q[5] * q[2] - q[1] * q[7], c02 = q[1] * q[5] - q[4] * q[2];
    const double c11 = q[0] * q[7] - q[2] * q[2], c12 = q[1] * q[2] - q[0] * q[5], c22 = q[0] * q[4] - q[1] * q[1];
    const double det = q[0] * c00 + q[1] * c01 + q[2] * c02;
    const double s = fmax(fmax(fmax(fabs(q[0]), fabs(q[1])), fmax(fabs(q[2]), fabs(q[4]))), fmax(fabs(q[5]), fabs(q[7])));
    const D3 mid{(pa.x + pb.x) * 0.5, (pa.y + pb.y) * 0.5, (pa.z + pb.z) * 0.5};
    const D3 ev = sub(pb, pa);
    bool solved = fabs(det) > kDetRel * (s * s * s);
    D3 p;
    double cost;
    if (solved) {
      const D3 x{-(c00 * q[3] + c01 * q[6] + c02 * q[8]) / det, -(c01 * q[3] + c11 * q[6] + c12 * q[8]) / det,
                 -(c02 * q[3] + c12 * q[6] + c22 * q[8]) / det};
      const D3 dm = sub(x, mid);
      solved = dot(dm, dm) <= dot(ev, ev);
      if (solved) {
        p = round_f32(x);
        cost = quadric_eval(q, p);
      }
    }
    if (!solved) {   // the cheapest of a, b and the midpoint, ties to the earlier
      p = pa;
      cost = quadric_eval(q, pa);
      const double cb = quadric_eval(q, pb);
      if (cb < cost) { p = pb; cost = cb; }
      const D3 pm = round_f32(mid);
      const double cm = quadric_eval(q, pm);
      if (cm < cost) { p = pm; cost = cm; }
    }
    cost = cost > 0.0 ? cost : 0.0;
    a.positions[3 * e] = (float)p.x;
    a.positions[3 * e + 1] = (float)p.y;
    a.positions[3 * e + 2] = (float)p.z;

    uint64_t key = ~0ull;
    const int64_t s0 = a.edge_off[e], nfe = a.edge_off[e + 1] - s0;
    const int fl = a.flags[va] | a.flags[vb];
    const int64_t da = a.vf_off[va + 1] - a.vf_off[va], db = a.vf_off[vb + 1] - a.vf_off[vb];
    bool ok = (nfe == 1 || nfe == 2) && !(fl & kFlagNonManifold) &&
              !(nfe == 2 && (a.flags[va] & kFlagBoundary) && (a.flags[vb] & kFlagBoundary)) && da <= kMaxValence &&
              db <= kMaxValence && da + db - nfe > nfe;
    // the apexes of the edge's faces
    int apex0 = -1, apex1 = -1;
    for (int j = 0; ok && j < nfe; ++j) {
      const int64_t f = a.edge_face[s0 + j];
      for (int i = 0; i < 3; ++i) {
        const int v = a.faces[3 * f + i];
        if (v != va && v != vb) (j == 0 ? apex0 : apex1) = v;
      }
    }
    // link condition: every common neighbour of a and b is an apex, and no faces (a, x, y) and (b, x, y) both exist
    for (int64_t k = a.vf_off[va]; ok && k < a.vf_off[va + 1]; ++k) {
      const int64_t f = a.vf_face[k];
      int x = -1, y = -1;
      bool with_b = false;
      for (int i = 0; i < 3; ++i) {
        const int v = a.faces[3 * f + i];
        if (v == vb) with_b = true;
        else if (v != va) (x < 0 ? x : y) = v;
      }
      if (x >= 0 && x != apex0 && x != apex1 && star_has(a, vb, x)) ok = false;
      if (y >= 0 && y != apex0 && y != apex1 && star_has(a, vb, y)) ok = false;
      if (!ok || with_b || y < 0) continue;
      for (int64_t l = a.vf_off[vb]; ok && l < a.vf_off[vb + 1]; ++l) {
        const int g = a.vf_face[l];
        if (has_corner(a.faces, g, x) && has_corner(a.faces, g, y)) ok = false;
      }
      if (ok) ok = keeps_orientation(a, f, va, p);
    }
    for (int64_t k = a.vf_off[vb]; ok && k < a.vf_off[vb + 1]; ++k) {
      const int64_t f = a.vf_face[k];
      if (!has_corner(a.faces, (int)f, va)) ok = keeps_orientation(a, f, vb, p);
    }
    if (ok) key = (uint64_t)__float_as_uint(__double2float_rn(cost)) << 32 | (uint64_t)e;
    a.keys[e] = key;
  }
}

__global__ void __launch_bounds__(256) qem_vmin_kernel(const QemArgs a) {
  QEM_LOOP(e, a.ne) {
    const uint64_t k = a.keys[e];
    if (k == ~0ull) continue;
    atomicMin((unsigned long long*)a.vmin + a.edges[2 * e], (unsigned long long)k);
    atomicMin((unsigned long long*)a.vmin + a.edges[2 * e + 1], (unsigned long long)k);
  }
}

// fmin[f] = min of vmin over f's corners, folded straight into rmin of each corner
__global__ void __launch_bounds__(256) qem_rmin_kernel(const QemArgs a) {
  QEM_LOOP(f, a.nf) {
    const int v0 = a.faces[3 * f], v1 = a.faces[3 * f + 1], v2 = a.faces[3 * f + 2];
    const uint64_t m = min(a.vmin[v0], min(a.vmin[v1], a.vmin[v2]));
    if (m == ~0ull) continue;
    atomicMin((unsigned long long*)a.rmin + v0, (unsigned long long)m);
    atomicMin((unsigned long long*)a.rmin + v1, (unsigned long long)m);
    atomicMin((unsigned long long*)a.rmin + v2, (unsigned long long)m);
  }
}

__global__ void __launch_bounds__(256) qem_select_kernel(const QemArgs a) {
  QEM_LOOP(e, a.ne) {
    const uint64_t k = a.keys[e];
    a.selected[e] = k != ~0ull && a.rmin[a.edges[2 * e]] == k && a.rmin[a.edges[2 * e + 1]] == k;
  }
}

// Per collapsed edge (a, b), a < b: a moves to the edge's position and takes Q_a + Q_b and the blended normal; the
// edge's faces die; b becomes a in its other faces.  Collapsed edges have disjoint stars, so nothing races.
__global__ void __launch_bounds__(256) qem_apply_kernel(const QemArgs a) {
  QEM_LOOP(e, a.ne) {
    if (!a.collapse[e]) continue;
    const int va = a.edges[2 * e], vb = a.edges[2 * e + 1];
    const D3 p{(double)a.positions[3 * e], (double)a.positions[3 * e + 1], (double)a.positions[3 * e + 2]};
    if (a.normals) {
      const D3 pa = ld_pos(a.vertices, va), ev = sub(ld_pos(a.vertices, vb), pa);
      const double el2 = dot(ev, ev);
      double t = el2 > 0.0 ? dot(sub(p, pa), ev) / el2 : 0.0;
      t = fmin(fmax(t, 0.0), 1.0);
      const D3 na = ld_pos(a.normals, va), nb = ld_pos(a.normals, vb);
      const D3 n{(1.0 - t) * na.x + t * nb.x, (1.0 - t) * na.y + t * nb.y, (1.0 - t) * na.z + t * nb.z};
      const double len = sqrt(dot(n, n));
      if (len > 0.0) {
        a.normals[3 * (int64_t)va] = (float)(n.x / len);
        a.normals[3 * (int64_t)va + 1] = (float)(n.y / len);
        a.normals[3 * (int64_t)va + 2] = (float)(n.z / len);
      }
    }
    a.vertices[3 * (int64_t)va] = (float)p.x;
    a.vertices[3 * (int64_t)va + 1] = (float)p.y;
    a.vertices[3 * (int64_t)va + 2] = (float)p.z;
    for (int i = 0; i < 10; ++i)
      a.quadrics[10 * (int64_t)va + i] = a.quadrics[10 * (int64_t)va + i] + a.quadrics[10 * (int64_t)vb + i];
    for (int64_t k = a.edge_off[e]; k < a.edge_off[e + 1]; ++k) a.face_alive[a.edge_face[k]] = 0;
    for (int64_t k = a.vf_off[vb]; k < a.vf_off[vb + 1]; ++k) {
      const int64_t f = a.vf_face[k];
      if (has_corner(a.faces, (int)f, va)) continue;
      for (int i = 0; i < 3; ++i)
        if (a.faces[3 * f + i] == vb) a.faces[3 * f + i] = va;
    }
  }
}

// ------------------------------------------------------------------------------------------- texture atlas
// Per-face charts, two faces per square cell of c x c texels, cells row-major in rows of n (mesh.bake_texture; the
// layout is restated in tests/mesh_texture_ref.py).  Cell k holds faces 2k (A) and 2k + 1 (B).  In the cell's texel
// units (texel (i, j) centred at (i + 0.5, j + 0.5)) each face is a right isosceles triangle with its corners on
// texel centres: corner 0 at o, corner 1 at o + (d, 0), corner 2 at o + (0, d), with o = (0.5, 0.5), d = c - 3 for A
// and o = (c - 0.5, c - 0.5), d = -(c - 2) for B.  Texel (i, j) belongs to A when i + j + 2 <= c, else to B (to A
// when the cell has no B).  A bilinear sample inside A (u + v <= c - 2) reads texels with i + j < u + v + 1 <= c - 1,
// all A's; one inside B (u + v >= c + 1) reads texels with i + j > u + v - 3 >= c - 2, all B's.  So no sample of a
// face at mip level 0 reads another face's texel.
struct TexAtlas {
  int64_t nf;
  int n, c, size;
};

// The chart of face f: its cell's first texel (x0, y0) in the atlas, and o, d in the cell's texel units
__device__ __forceinline__ void tex_chart(const TexAtlas& a, int64_t f, int& x0, int& y0, float& o, float& d) {
  const int64_t k = f >> 1;
  x0 = (int)(k % a.n) * a.c;
  y0 = (int)(k / a.n) * a.c;
  o = f & 1 ? (float)a.c - 0.5f : 0.5f;
  d = f & 1 ? (float)(2 - a.c) : (float)(a.c - 3);
}

// The face that owns texel (i, j) of cell k
__device__ __forceinline__ int64_t tex_owner(const TexAtlas& a, int64_t k, int i, int j) {
  return 2 * k + (i + j + 2 > a.c && 2 * k + 1 < a.nf);
}

__device__ __forceinline__ V3 tex_ld3(const float* __restrict__ p, int i) {
  return V3{__ldg(p + 3 * (int64_t)i), __ldg(p + 3 * (int64_t)i + 1), __ldg(p + 3 * (int64_t)i + 2)};
}

// v / max|v_i| / |v / max|v_i||, so no finite v overflows or underflows; false when v is zero or not finite
__device__ __forceinline__ bool tex_unit(V3& v) {
  const float m = fmaxf(fabsf(v.x), fmaxf(fabsf(v.y), fabsf(v.z)));
  if (!(m > 0.f) || !isfinite(m)) return false;
  v = V3{v.x / m, v.y / m, v.z / m};
  const float len = sqrtf(v.x * v.x + v.y * v.y + v.z * v.z);
  v = V3{v.x / len, v.y / len, v.z / len};
  return true;
}

__global__ void __launch_bounds__(256) tex_uv_kernel(const TexAtlas a, float* __restrict__ uv) {
  for (int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; f < a.nf; f += (int64_t)gridDim.x * blockDim.x) {
    int x0, y0;
    float o, d;
    tex_chart(a, f, x0, y0, o, d);
    float* q = uv + 6 * f;
    q[0] = (float)x0 + o;     q[1] = (float)y0 + o;
    q[2] = (float)x0 + o + d; q[3] = (float)y0 + o;
    q[4] = (float)x0 + o;     q[5] = (float)y0 + o + d;
  }
}

// One thread per texel t of the used cells, cell-major, row-major within a cell: its owner's barycentrics at the
// texel centre, clamped to the triangle (the nearest point of the chart), then the surface point and the unit
// interpolated vertex normal (the face's normal when that is zero, (0, 0, 1) when the face has no area).
__global__ void __launch_bounds__(256)
tex_raster_kernel(const TexAtlas a, int64_t num_texels, const float* __restrict__ vertices,
                  const int32_t* __restrict__ faces, const float* __restrict__ vnormals,
                  int32_t* __restrict__ texel_index, float* __restrict__ points, float* __restrict__ normals) {
  const int cc = a.c * a.c;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < num_texels;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = t / cc;
    const int r = (int)(t - k * cc), j = r / a.c, i = r - j * a.c;
    const int64_t f = tex_owner(a, k, i, j);
    int x0, y0;
    float o, d;
    tex_chart(a, f, x0, y0, o, d);
    float fa = fmaxf(((float)i + 0.5f - o) / d, 0.f), fb = fmaxf(((float)j + 0.5f - o) / d, 0.f);
    if (fa + fb > 1.f) {
      fa = fminf(fmaxf((fa - fb + 1.f) * 0.5f, 0.f), 1.f);
      fb = 1.f - fa;
    }
    const float w0 = 1.f - fa - fb;
    const int v0 = __ldg(faces + 3 * f), v1 = __ldg(faces + 3 * f + 1), v2 = __ldg(faces + 3 * f + 2);
    const V3 p0 = tex_ld3(vertices, v0), p1 = tex_ld3(vertices, v1), p2 = tex_ld3(vertices, v2);
    const V3 n0 = tex_ld3(vnormals, v0), n1 = tex_ld3(vnormals, v1), n2 = tex_ld3(vnormals, v2);
    V3 n{w0 * n0.x + fa * n1.x + fb * n2.x, w0 * n0.y + fa * n1.y + fb * n2.y, w0 * n0.z + fa * n1.z + fb * n2.z};
    if (!tex_unit(n)) {
      const V3 e1{p1.x - p0.x, p1.y - p0.y, p1.z - p0.z}, e2{p2.x - p0.x, p2.y - p0.y, p2.z - p0.z};
      n = V3{e1.y * e2.z - e1.z * e2.y, e1.z * e2.x - e1.x * e2.z, e1.x * e2.y - e1.y * e2.x};
      if (!tex_unit(n)) n = V3{0.f, 0.f, 1.f};
    }
    texel_index[t] = (y0 + j) * a.size + x0 + i;
    float* pt = points + 3 * t;
    pt[0] = w0 * p0.x + fa * p1.x + fb * p2.x;
    pt[1] = w0 * p0.y + fa * p1.y + fb * p2.y;
    pt[2] = w0 * p0.z + fa * p1.z + fb * p2.z;
    float* nt = normals + 3 * t;
    nt[0] = n.x;
    nt[1] = n.y;
    nt[2] = n.z;
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

namespace mnrf {
namespace {
// Both TSDF entry points: checks (messages under `name`) and the launch of the kContract instance.
template <bool kContract>
int tsdf_integrate(const char* name, const mnrf_camera_desc* cam, int32_t nx, int32_t ny, int32_t nz, double x0,
                   double y0, double z0, double h, int32_t num_views, int32_t height, int32_t width,
                   const float* worldtocams, const float* camtopixs, const float* depth, const float* acc,
                   const float* rgb, float tau, float* tsdf, float* weight, float* color_sum, float* color_weight,
                   mnrf_stream stream) {
  set_error("");
  MNRF_CHECK(cam, "%s: null camera descriptor", name);
  MNRF_CHECK(nx >= 2 && ny >= 2 && nz >= 2 && nx <= kMcMaxDim && ny <= kMcMaxDim && nz <= kMcMaxDim,
             "%s: grid %d x %d x %d (nz x ny x nx), each side must be in [2, %d]", name, nz, ny, nx, kMcMaxDim);
  MNRF_CHECK(num_views >= 0 && height >= 1 && width >= 1, "%s: %d views of %d x %d pixels", name,
             num_views, height, width);
  MNRF_CHECK(cam->camtype == MNRF_CAM_PERSPECTIVE || cam->camtype == MNRF_CAM_FISHEYE,
             "%s: camtype must be perspective or fisheye", name);
  MNRF_CHECK(!cam->has_ndc, "%s: NDC cameras are not supported", name);
  MNRF_CHECK(cam->num_cameras == 1 || cam->num_cameras == num_views,
             "%s: num_cameras = %d camera-to-pixel matrices for %d views", name, cam->num_cameras, num_views);
  MNRF_CHECK(tau > 0.f && isfinite(tau) && h > 0.0 && isfinite(h), "%s: tau %g, h %g", name, tau, h);
  MNRF_CHECK(tsdf && weight, "%s: null state pointer", name);
  MNRF_CHECK(!rgb == !color_sum && !color_sum == !color_weight,
             "%s: rgb, color_sum and color_weight go together", name);
  if (num_views == 0) return 0;
  MNRF_CHECK(worldtocams && camtopixs && depth && acc, "%s: null view pointer", name);
  TsdfArgs a{*cam, nx, ny, nz, (int64_t)nx * ny * nz, x0, y0, z0, h, num_views, height, width, tau,
             worldtocams, camtopixs, cam->num_cameras == 1 ? 0 : 9, depth, acc, rgb, tsdf, weight, color_sum,
             color_weight};
  const int blocks = (int)std::min<int64_t>((a.n + 255) / 256, (int64_t)mnrf_num_sms() * 16);
  if (rgb)
    tsdf_integrate_kernel<true, kContract><<<blocks, 256, 0, (cudaStream_t)stream>>>(a);
  else
    tsdf_integrate_kernel<false, kContract><<<blocks, 256, 0, (cudaStream_t)stream>>>(a);
  MNRF_LAUNCH_CHECK();
  return 0;
}
}  // namespace
}  // namespace mnrf

extern "C" int mnrf_tsdf_integrate(const mnrf_camera_desc* cam, int32_t nx, int32_t ny, int32_t nz, double x0,
                                   double y0, double z0, double h, int32_t num_views, int32_t height, int32_t width,
                                   const float* worldtocams, const float* camtopixs, const float* depth,
                                   const float* acc, const float* rgb, float tau, float* tsdf, float* weight,
                                   float* color_sum, float* color_weight, mnrf_stream stream) {
  return mnrf::tsdf_integrate<false>("mnrf_tsdf_integrate", cam, nx, ny, nz, x0, y0, z0, h, num_views, height,
                                    width, worldtocams, camtopixs, depth, acc, rgb, tau, tsdf, weight,
                                    color_sum, color_weight, stream);
}

extern "C" int mnrf_tsdf_integrate_contracted(const mnrf_camera_desc* cam, int32_t nx, int32_t ny, int32_t nz,
                                              double x0, double y0, double z0, double h, int32_t num_views,
                                              int32_t height, int32_t width, const float* worldtocams,
                                              const float* camtopixs, const float* depth, const float* acc,
                                              const float* rgb, float tau, float* tsdf, float* weight,
                                              float* color_sum, float* color_weight, mnrf_stream stream) {
  return mnrf::tsdf_integrate<true>("mnrf_tsdf_integrate_contracted", cam, nx, ny, nz, x0, y0, z0, h, num_views,
                                    height, width, worldtocams, camtopixs, depth, acc, rgb, tau, tsdf, weight,
                                    color_sum, color_weight, stream);
}

extern "C" int mnrf_mesh_uncontract(int64_t n, const float* points, const float* normals, float* world_points,
                                    float* world_normals, mnrf_stream stream) {
  using namespace mnrf;
  set_error("");
  MNRF_CHECK(n >= 0, "mnrf_mesh_uncontract: %lld points", (long long)n);
  MNRF_CHECK(!normals == !world_normals, "mnrf_mesh_uncontract: normals and world_normals go together");
  if (n == 0) return 0;
  MNRF_CHECK(points && world_points, "mnrf_mesh_uncontract: null pointer");
  const int blocks = (int)std::min<int64_t>((n + 255) / 256, (int64_t)mnrf_num_sms() * 16);
  uncontract_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(n, points, normals, world_points, world_normals);
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

namespace {
int qem_blocks(int64_t n) { return (int)std::min<int64_t>((n + 255) / 256, (int64_t)mnrf_num_sms() * 16); }
}  // namespace

extern "C" int mnrf_mesh_quadrics(int32_t num_vertices, int64_t num_faces, const float* vertices,
                                  const int32_t* faces, const int64_t* vf_off, const int32_t* vf_face,
                                  int64_t num_boundary, const int32_t* boundary_edges, const int32_t* boundary_face,
                                  const int64_t* vb_off, const int32_t* vb_edge, double* quadrics,
                                  mnrf_stream stream) {
  using namespace mnrf;
  set_error("");
  MNRF_CHECK(num_vertices >= 0 && num_faces >= 0 && num_boundary >= 0,
             "mnrf_mesh_quadrics: %d vertices, %lld faces, %lld boundary edges", num_vertices, (long long)num_faces,
             (long long)num_boundary);
  if (num_vertices == 0) return 0;
  MNRF_CHECK(vertices && vf_off && vb_off && quadrics && (faces && vf_face || num_faces == 0) &&
             (boundary_edges && boundary_face && vb_edge || num_boundary == 0),
             "mnrf_mesh_quadrics: null pointer");
  QemArgs a{};
  a.nv = num_vertices; a.nf = num_faces; a.nb = num_boundary;
  a.vertices = const_cast<float*>(vertices); a.faces = const_cast<int32_t*>(faces); a.quadrics = quadrics;
  a.vf_off = vf_off; a.vf_face = vf_face; a.bnd_edges = boundary_edges; a.bnd_face = boundary_face;
  a.vb_off = vb_off; a.vb_edge = vb_edge;
  qem_quadrics_kernel<<<qem_blocks(num_vertices), 256, 0, (cudaStream_t)stream>>>(a);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_mesh_edge_cost(int32_t num_vertices, int64_t num_faces, int64_t num_edges, const float* vertices,
                                   const int32_t* faces, const double* quadrics, const int32_t* edges,
                                   const int64_t* edge_off, const int32_t* edge_face, const int64_t* vf_off,
                                   const int32_t* vf_face, int32_t* flags, uint64_t* keys, float* positions,
                                   mnrf_stream stream) {
  using namespace mnrf;
  set_error("");
  MNRF_CHECK(num_vertices >= 0 && num_faces >= 0 && num_edges >= 0 && num_edges <= (int64_t)UINT32_MAX,
             "mnrf_mesh_edge_cost: %d vertices, %lld faces, %lld edges (at most 2^32 - 1)", num_vertices,
             (long long)num_faces, (long long)num_edges);
  if (num_edges == 0) return 0;
  MNRF_CHECK(num_vertices > 0 && num_faces > 0, "mnrf_mesh_edge_cost: edges without vertices or faces");
  MNRF_CHECK(vertices && faces && quadrics && edges && edge_off && edge_face && vf_off && vf_face && flags && keys &&
             positions, "mnrf_mesh_edge_cost: null pointer");
  QemArgs a{};
  a.nv = num_vertices; a.nf = num_faces; a.ne = num_edges;
  a.vertices = const_cast<float*>(vertices); a.faces = const_cast<int32_t*>(faces);
  a.quadrics = const_cast<double*>(quadrics); a.edges = edges; a.edge_off = edge_off; a.edge_face = edge_face;
  a.vf_off = vf_off; a.vf_face = vf_face; a.flags = flags; a.keys = keys; a.positions = positions;
  MNRF_CUDA(cudaMemsetAsync(flags, 0, sizeof(int32_t) * (size_t)num_vertices, (cudaStream_t)stream));
  qem_flags_kernel<<<qem_blocks(num_edges), 256, 0, (cudaStream_t)stream>>>(a);
  qem_cost_kernel<<<qem_blocks(num_edges), 256, 0, (cudaStream_t)stream>>>(a);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_mesh_collapse_select(int32_t num_vertices, int64_t num_faces, int64_t num_edges,
                                         const int32_t* faces, const int32_t* edges, const uint64_t* keys,
                                         uint64_t* vmin, uint64_t* rmin, uint8_t* selected, mnrf_stream stream) {
  using namespace mnrf;
  set_error("");
  MNRF_CHECK(num_vertices >= 0 && num_faces >= 0 && num_edges >= 0 && num_edges <= (int64_t)UINT32_MAX,
             "mnrf_mesh_collapse_select: %d vertices, %lld faces, %lld edges (at most 2^32 - 1)", num_vertices,
             (long long)num_faces, (long long)num_edges);
  if (num_edges == 0) return 0;
  MNRF_CHECK(num_vertices > 0 && num_faces > 0, "mnrf_mesh_collapse_select: edges without vertices or faces");
  MNRF_CHECK(faces && edges && keys && vmin && rmin && selected, "mnrf_mesh_collapse_select: null pointer");
  QemArgs a{};
  a.nv = num_vertices; a.nf = num_faces; a.ne = num_edges;
  a.faces = const_cast<int32_t*>(faces); a.edges = edges; a.keys = const_cast<uint64_t*>(keys);
  a.vmin = vmin; a.rmin = rmin; a.selected = selected;
  const cudaStream_t s = (cudaStream_t)stream;
  MNRF_CUDA(cudaMemsetAsync(vmin, 0xff, sizeof(uint64_t) * (size_t)num_vertices, s));
  MNRF_CUDA(cudaMemsetAsync(rmin, 0xff, sizeof(uint64_t) * (size_t)num_vertices, s));
  qem_vmin_kernel<<<qem_blocks(num_edges), 256, 0, s>>>(a);
  qem_rmin_kernel<<<qem_blocks(num_faces), 256, 0, s>>>(a);
  qem_select_kernel<<<qem_blocks(num_edges), 256, 0, s>>>(a);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_mesh_collapse_apply(int32_t num_vertices, int64_t num_faces, int64_t num_edges,
                                        const uint8_t* collapse, const int32_t* edges, const int64_t* edge_off,
                                        const int32_t* edge_face, const int64_t* vf_off, const int32_t* vf_face,
                                        const float* positions, float* vertices, double* quadrics, float* normals,
                                        int32_t* faces, uint8_t* face_alive, mnrf_stream stream) {
  using namespace mnrf;
  set_error("");
  MNRF_CHECK(num_vertices >= 0 && num_faces >= 0 && num_edges >= 0 && num_edges <= (int64_t)UINT32_MAX,
             "mnrf_mesh_collapse_apply: %d vertices, %lld faces, %lld edges (at most 2^32 - 1)", num_vertices,
             (long long)num_faces, (long long)num_edges);
  if (num_faces == 0) return 0;
  MNRF_CHECK(num_vertices > 0, "mnrf_mesh_collapse_apply: faces without vertices");
  MNRF_CHECK(faces && face_alive && (num_edges == 0 || collapse && edges && edge_off && edge_face && vf_off &&
                                     vf_face && positions && vertices && quadrics),
             "mnrf_mesh_collapse_apply: null pointer");
  const cudaStream_t s = (cudaStream_t)stream;
  MNRF_CUDA(cudaMemsetAsync(face_alive, 1, (size_t)num_faces, s));
  if (num_edges == 0) return 0;
  QemArgs a{};
  a.nv = num_vertices; a.nf = num_faces; a.ne = num_edges;
  a.collapse = collapse; a.edges = edges; a.edge_off = edge_off; a.edge_face = edge_face; a.vf_off = vf_off;
  a.vf_face = vf_face; a.positions = const_cast<float*>(positions); a.vertices = vertices; a.quadrics = quadrics;
  a.normals = normals; a.faces = faces; a.face_alive = face_alive;
  qem_apply_kernel<<<qem_blocks(num_edges), 256, 0, s>>>(a);
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_mesh_texture_raster(int32_t num_vertices, int64_t num_faces, const float* vertices,
                                        const int32_t* faces, const float* normals, int32_t size, float* uv,
                                        int32_t* texel_index, float* points, float* texel_normals,
                                        mnrf_stream stream) {
  using namespace mnrf;
  set_error("");
  MNRF_CHECK(num_vertices >= 0 && num_faces >= 0, "mnrf_mesh_texture_raster: %d vertices, %lld faces", num_vertices,
             (long long)num_faces);
  MNRF_CHECK(size >= 4 && size <= 16384, "mnrf_mesh_texture_raster: texture size %d, want [4, 16384]", size);
  if (num_faces == 0) return 0;
  const int64_t cells = (num_faces + 1) / 2;
  int64_t n = (int64_t)std::sqrt((double)cells);
  while (n * n < cells) ++n;
  while (n > 1 && (n - 1) * (n - 1) >= cells) --n;
  const int64_t c = size / n;
  MNRF_CHECK(c >= 4, "mnrf_mesh_texture_raster: %lld faces do not fit a %d x %d atlas (%lld texels per cell, want >= "
             "4; it holds at most %lld faces)", (long long)num_faces, size, size, (long long)c,
             2 * (long long)(size / 4) * (size / 4));
  MNRF_CHECK(num_vertices > 0 && vertices && faces && normals && uv && texel_index && points && texel_normals,
             "mnrf_mesh_texture_raster: null pointer or no vertices");
  const TexAtlas a{num_faces, (int)n, (int)c, size};
  const int64_t num_texels = cells * c * c;
  const int cap = mnrf_num_sms() * 16;
  const cudaStream_t s = (cudaStream_t)stream;
  tex_uv_kernel<<<(int)std::min<int64_t>((num_faces + 255) / 256, cap), 256, 0, s>>>(a, uv);
  tex_raster_kernel<<<(int)std::min<int64_t>((num_texels + 255) / 256, cap), 256, 0, s>>>(
      a, num_texels, vertices, faces, normals, texel_index, points, texel_normals);
  MNRF_LAUNCH_CHECK();
  return 0;
}
