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
#include <algorithm>

#include "common.cuh"
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
    const bool in0 = __ldg(f + p) > g.level;
    const int c[3] = {x, y, z};
    const int dim[3] = {g.nx, g.ny, g.nz};
#pragma unroll
    for (int a = 0; a < 3; ++a)
      edge_cut[3 * p + a] = c[a] + 1 < dim[a] && ((__ldg(f + p + mc_stride(g, a)) > g.level) != in0);
    const bool cell = x + 1 < g.nx && y + 1 < g.ny && z + 1 < g.nz;
    cell_tris[p] = cell ? kMcNumTris[mc_case(g, f, p)] : 0;
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

// Gradient of the grid at point p = (x, y, z): central differences, one-sided on the grid boundary
__device__ __forceinline__ void mc_grad(const McGrid& g, const float* __restrict__ f, int64_t p, int x, int y, int z,
                                        float grad[3]) {
  const int c[3] = {x, y, z};
  const int dim[3] = {g.nx, g.ny, g.nz};
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int64_t s = mc_stride(g, a);
    if (c[a] == 0) grad[a] = __ldg(f + p + s) - __ldg(f + p);
    else if (c[a] == dim[a] - 1) grad[a] = __ldg(f + p) - __ldg(f + p - s);
    else grad[a] = 0.5f * (__ldg(f + p + s) - __ldg(f + p - s));
  }
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
      mc_grad(g, f, p, x, y, z, g0);
      mc_grad(g, f, q, x + (a == 0), y + (a == 1), z + (a == 2), g1);
#pragma unroll
      for (int i = 0; i < 3; ++i) n[i] = g0[i] + t * (g1[i] - g0[i]);
      const float m = fmaxf(fabsf(n[0]), fmaxf(fabsf(n[1]), fabsf(n[2])));
      if (m > 0.f && isfinite(m)) {
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
