// Closest-hit ray casting into a triangle mesh (mesh evaluation, multinerf_b200/mesh.py): a linear BVH over the
// faces (Karras 2012), built in three phases with no host synchronisation inside, and one thread per ray tracing it.
//
// Build (mnrf_mesh_bvh):
//   boxes: per face, its fp32 min/max box and the centroid ((v0 + v1) + v2) / 3;
//   keys:  given the centroid bounds (a device reduction by the caller), the 30-bit Morton code of each centroid on
//          1024 cells per axis, key = morton << 32 | face, unique even when every centroid is the same;
//   tree:  given the keys sorted ascending, the Karras topology (one thread per internal node), then the boxes fitted
//          bottom-up by one thread per leaf: the second child to arrive at a node (atomic arrival counter, zeroed in
//          the same call, a fence between writing a box and counting the arrival) carries on to the parent.
// Node layout: internal node i (0 = root) holds both children's boxes, so one 64-byte load tests both:
//   floats [0, 6) left box (lo xyz, hi xyz), [6, 12) right box, [12, 14) the child indices as int32, [14, 16) zero.
// Node index c < F - 1 is internal; c >= F - 1 is leaf c - (F - 1), in key order, whose face is leaf_face[leaf].
// Boxes are min/max of vertex coordinates, so no rounding happens anywhere in the build.
//
// Trace (mnrf_mesh_trace): depth-first with a fixed stack, nearer child first; slab tests whose far bound is widened
// by 1 + 2 gamma(3) (Ize 2013), the watertight ray/triangle test of Woop, Benthin and Wald (JCGT 2013), with the edge
// functions recomputed in fp64 when one of them is exactly 0.  Among the faces tested, the closest hit is the least
// (t, face), and the traversal is a fixed function of the tree, so the result is deterministic for a given mesh.  A
// box is skipped when its fp32 entry distance exceeds the best t; that distance is not widened downward, so where two
// faces' t tie exactly (or lie within rounding of a box entry), a different tree -- the same faces in another order --
// can settle on the other face.
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace mnrf {

namespace {

constexpr int kBvhStack = 64;
// 1 + 2 gamma(3), gamma(n) = n eps / (1 - n eps), eps = 2^-24: 1.00000035762793 rounded up to the next float,
// 1 + 4 * 2^-23 (the float nearest 1.0000004 is 1 + 3 * 2^-23, just below it)
constexpr float kIzeWiden = 1.0000005f;

__device__ __forceinline__ uint32_t expand_bits10(uint32_t v) {
  v = (v | (v << 16)) & 0x030000FFu;
  v = (v | (v << 8)) & 0x0300F00Fu;
  v = (v | (v << 4)) & 0x030C30C3u;
  v = (v | (v << 2)) & 0x09249249u;
  return v;
}

// cell of c in [lo, hi] along one axis: floor((c - lo) / (hi - lo) * 1024) clamped to [0, 1023] (0 for a flat axis)
__device__ __forceinline__ uint32_t morton_cell(float c, float lo, float hi) {
  const float ext = __fsub_rn(hi, lo);
  float t = ext > 0.f ? __fdiv_rn(__fsub_rn(c, lo), ext) : 0.f;
  t = t >= 0.f ? (t <= 1.f ? t : 1.f) : 0.f;                  // also maps NaN to 0
  return min((uint32_t)__fmul_rn(t, 1024.f), 1023u);
}

__global__ void __launch_bounds__(256) bvh_boxes_kernel(int64_t num_faces, const float* __restrict__ vertices,
                                                        const int32_t* __restrict__ faces, float* __restrict__ boxes,
                                                        float* __restrict__ centroids) {
  for (int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; f < num_faces;
       f += (int64_t)gridDim.x * blockDim.x) {
    float p[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int64_t v = faces[3 * f + k];
#pragma unroll
      for (int a = 0; a < 3; ++a) p[k][a] = vertices[3 * v + a];
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      boxes[6 * f + a] = fminf(fminf(p[0][a], p[1][a]), p[2][a]);
      boxes[6 * f + 3 + a] = fmaxf(fmaxf(p[0][a], p[1][a]), p[2][a]);
      centroids[3 * f + a] = __fdiv_rn(__fadd_rn(__fadd_rn(p[0][a], p[1][a]), p[2][a]), 3.f);
    }
  }
}

__global__ void __launch_bounds__(256) bvh_keys_kernel(int64_t num_faces, const float* __restrict__ centroids,
                                                       const float* __restrict__ bounds, int64_t* __restrict__ keys) {
  for (int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; f < num_faces;
       f += (int64_t)gridDim.x * blockDim.x) {
    uint32_t m = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a)
      m |= expand_bits10(morton_cell(centroids[3 * f + a], bounds[a], bounds[3 + a])) << (2 - a);
    keys[f] = (int64_t)(((uint64_t)m << 32) | (uint64_t)f);
  }
}

// length of the common prefix of keys i and j, -1 when j lies outside [0, n)
__device__ __forceinline__ int bvh_delta(const int64_t* __restrict__ keys, int64_t n, int64_t i, int64_t j) {
  if (j < 0 || j >= n) return -1;
  return __clzll(keys[i] ^ keys[j]);      // keys are unique: the xor is never 0
}

__global__ void __launch_bounds__(256) bvh_topology_kernel(int64_t n, const int64_t* __restrict__ keys,
                                                           float* __restrict__ nodes, int32_t* __restrict__ parent) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n - 1; i += (int64_t)gridDim.x * blockDim.x) {
    const int d = bvh_delta(keys, n, i, i + 1) > bvh_delta(keys, n, i, i - 1) ? 1 : -1;
    const int dmin = bvh_delta(keys, n, i, i - d);
    int64_t lmax = 2;
    while (bvh_delta(keys, n, i, i + lmax * d) > dmin) lmax *= 2;      // lmax <= 2 n
    int64_t l = 0;
    for (int64_t t = lmax / 2; t >= 1; t /= 2)
      if (bvh_delta(keys, n, i, i + (l + t) * d) > dmin) l += t;
    const int64_t j = i + l * d;
    const int dnode = bvh_delta(keys, n, i, j);
    int64_t s = 0, t = l;
    do {
      t = (t + 1) / 2;
      if (bvh_delta(keys, n, i, i + (s + t) * d) > dnode) s += t;
    } while (t > 1);
    const int64_t gamma = i + s * d + min(d, 0);
    const int32_t left = (int32_t)(min(i, j) == gamma ? (n - 1) + gamma : gamma);
    const int32_t right = (int32_t)(max(i, j) == gamma + 1 ? (n - 1) + gamma + 1 : gamma + 1);
    int32_t* node = reinterpret_cast<int32_t*>(nodes + 16 * i);
    node[12] = left;
    node[13] = right;
    node[14] = 0;
    node[15] = 0;
    parent[left] = (int32_t)i;
    parent[right] = (int32_t)i;
    if (i == 0) parent[0] = -1;
  }
}

// One thread per leaf climbs toward the root; the second child to arrive at a node fits its box and carries on.
__global__ void __launch_bounds__(256) bvh_refit_kernel(int64_t n, const int64_t* __restrict__ sorted_keys,
                                                        const float* __restrict__ face_boxes,
                                                        int32_t* __restrict__ leaf_face, const int32_t* parent,
                                                        int32_t* counters, float* nodes) {
  for (int64_t leaf = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; leaf < n;
       leaf += (int64_t)gridDim.x * blockDim.x) {
    const int32_t face = (int32_t)(sorted_keys[leaf] & 0xffffffffll);
    leaf_face[leaf] = face;
    float box[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) box[k] = face_boxes[6 * (int64_t)face + k];
    int32_t node = (int32_t)((n - 1) + leaf);
    while (true) {
      const int32_t p = parent[node];
      if (p < 0) break;                                       // node is the root
      float* pn = nodes + 16 * (int64_t)p;
      const int slot = reinterpret_cast<const int32_t*>(pn)[12] == node ? 0 : 1;
#pragma unroll
      for (int k = 0; k < 6; ++k) __stcg(pn + 6 * slot + k, box[k]);
      __threadfence();
      if (atomicAdd(counters + p, 1) == 0) break;              // the sibling's thread fits p
      __threadfence();
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        box[k] = fminf(__ldcg(pn + k), __ldcg(pn + 6 + k));
        box[3 + k] = fmaxf(__ldcg(pn + 3 + k), __ldcg(pn + 9 + k));
      }
      node = p;
    }
  }
}

struct TraceArgs {
  int64_t num_rays, num_faces;
  const float* origins;
  const float* directions;
  const float* near;
  const float* far;
  const float4* nodes;
  const int32_t* leaf_face;
  const float* vertices;
  const int32_t* faces;
  int32_t* hit_face;
  float* hit_t;
  float* hit_bary;
  int32_t* error_flag;
};

// entry parameter of the ray into box [lo, hi], or +inf when it misses [t0, t1] (far bound widened, Ize 2013).  A
// 0 * inf slab (origin on a plane, direction along it) is NaN and dropped by fminf / fmaxf: the ray lies in the
// slab's closure, so dropping it keeps the test conservative.
__device__ __forceinline__ float slab(const float* o, const float* inv, float lx, float ly, float lz, float hx,
                                      float hy, float hz, float t0, float t1) {
  const float ax = __fmul_rn(__fsub_rn(lx, o[0]), inv[0]), bx = __fmul_rn(__fsub_rn(hx, o[0]), inv[0]);
  const float ay = __fmul_rn(__fsub_rn(ly, o[1]), inv[1]), by = __fmul_rn(__fsub_rn(hy, o[1]), inv[1]);
  const float az = __fmul_rn(__fsub_rn(lz, o[2]), inv[2]), bz = __fmul_rn(__fsub_rn(hz, o[2]), inv[2]);
  const float tn = fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fmaxf(fminf(az, bz), t0));
  const float tf = fminf(fminf(fmaxf(ax, bx), fmaxf(ay, by)), fmaxf(az, bz));
  return tn <= fminf(__fmul_rn(tf, kIzeWiden), t1) ? tn : INFINITY;
}

struct Shear {
  int kx, ky, kz;
  float sx, sy, sz;
  float ox, oy, oz;           // the origin's components along kx, ky, kz
};

// Woop, Benthin and Wald 2013.  Returns true with (t, b1, b2) when the ray hits face f with near <= t <= best
// interval [t0, t1]; b1, b2 are the barycentrics of corners 1 and 2.
__device__ __forceinline__ bool hit_triangle(const TraceArgs& a, const Shear& s, int32_t f, float t0, float t1,
                                             float& t, float& b1, float& b2) {
  float ax[3], ay[3], az[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float* p = a.vertices + 3 * (int64_t)__ldg(a.faces + 3 * (int64_t)f + k);
    const float rx = __fsub_rn(__ldg(p + s.kx), s.ox);
    const float ry = __fsub_rn(__ldg(p + s.ky), s.oy);
    const float rz = __fsub_rn(__ldg(p + s.kz), s.oz);
    ax[k] = __fsub_rn(rx, __fmul_rn(s.sx, rz));
    ay[k] = __fsub_rn(ry, __fmul_rn(s.sy, rz));
    az[k] = __fmul_rn(s.sz, rz);
  }
  // U, V, W: edge functions of the edges opposite corners 0, 1, 2
  float u = __fsub_rn(__fmul_rn(ax[2], ay[1]), __fmul_rn(ay[2], ax[1]));
  float v = __fsub_rn(__fmul_rn(ax[0], ay[2]), __fmul_rn(ay[0], ax[2]));
  float w = __fsub_rn(__fmul_rn(ax[1], ay[0]), __fmul_rn(ay[1], ax[0]));
  if (u == 0.f || v == 0.f || w == 0.f) {
    u = (float)__dsub_rn(__dmul_rn(ax[2], ay[1]), __dmul_rn(ay[2], ax[1]));
    v = (float)__dsub_rn(__dmul_rn(ax[0], ay[2]), __dmul_rn(ay[0], ax[2]));
    w = (float)__dsub_rn(__dmul_rn(ax[1], ay[0]), __dmul_rn(ay[1], ax[0]));
  }
  if ((u < 0.f || v < 0.f || w < 0.f) && (u > 0.f || v > 0.f || w > 0.f)) return false;
  const float det = __fadd_rn(__fadd_rn(u, v), w);
  if (det == 0.f) return false;
  const float tt = __fadd_rn(__fadd_rn(__fmul_rn(u, az[0]), __fmul_rn(v, az[1])), __fmul_rn(w, az[2]));
  const float rcp = __fdiv_rn(1.f, det);
  t = __fmul_rn(tt, rcp);
  if (!(t >= t0 && t <= t1)) return false;
  b1 = __fmul_rn(v, rcp);
  b2 = __fmul_rn(w, rcp);
  return true;
}

__global__ void __launch_bounds__(128) trace_kernel(const TraceArgs a) {
  const int64_t internal = a.num_faces - 1;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < a.num_rays;
       r += (int64_t)gridDim.x * blockDim.x) {
    float o[3], d[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      o[k] = a.origins[3 * r + k];
      d[k] = a.directions[3 * r + k];
    }
    const float t0 = a.near[r];
    float best = a.far[r];
    int32_t best_face = -1;
    float best_b1 = 0.f, best_b2 = 0.f;
    const bool valid = isfinite(o[0]) && isfinite(o[1]) && isfinite(o[2]) && isfinite(d[0]) && isfinite(d[1]) &&
                       isfinite(d[2]) && (d[0] != 0.f || d[1] != 0.f || d[2] != 0.f) && !isnan(t0) &&
                       !isnan(best) && t0 <= best;
    if (valid) {
      float inv[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) inv[k] = __fdiv_rn(1.f, d[k]);
      Shear s;
      const float adx = fabsf(d[0]), ady = fabsf(d[1]), adz = fabsf(d[2]);
      s.kz = adx >= ady ? (adx >= adz ? 0 : 2) : (ady >= adz ? 1 : 2);
      s.kx = s.kz == 2 ? 0 : s.kz + 1;
      s.ky = s.kx == 2 ? 0 : s.kx + 1;
      const auto pick = [&](int k) { return k == 0 ? d[0] : k == 1 ? d[1] : d[2]; };
      if (pick(s.kz) < 0.f) {
        const int tmp = s.kx;
        s.kx = s.ky;
        s.ky = tmp;
      }
      s.sx = __fdiv_rn(pick(s.kx), pick(s.kz));
      s.sy = __fdiv_rn(pick(s.ky), pick(s.kz));
      s.sz = __fdiv_rn(1.f, pick(s.kz));
      s.ox = s.kx == 0 ? o[0] : s.kx == 1 ? o[1] : o[2];
      s.oy = s.ky == 0 ? o[0] : s.ky == 1 ? o[1] : o[2];
      s.oz = s.kz == 0 ? o[0] : s.kz == 1 ? o[1] : o[2];

      int32_t stack_node[kBvhStack];
      float stack_t[kBvhStack];
      int sp = 0;
      int32_t node = 0;                                       // the root; a leaf when F = 1
      while (true) {
        if (node >= internal) {
          const int32_t f = __ldg(a.leaf_face + (node - internal));
          float t, b1, b2;
          if (hit_triangle(a, s, f, t0, best, t, b1, b2) && (t < best || best_face < 0 || f < best_face)) {
            best = t;
            best_face = f;
            best_b1 = b1;
            best_b2 = b2;
          }
        } else {
          const float4 q0 = __ldg(a.nodes + 4 * (int64_t)node), q1 = __ldg(a.nodes + 4 * (int64_t)node + 1);
          const float4 q2 = __ldg(a.nodes + 4 * (int64_t)node + 2), q3 = __ldg(a.nodes + 4 * (int64_t)node + 3);
          const float tl = slab(o, inv, q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, t0, best);
          const float tr = slab(o, inv, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, t0, best);
          const int32_t cl = __float_as_int(q3.x), cr = __float_as_int(q3.y);
          const bool hl = tl != INFINITY, hr = tr != INFINITY;
          if (hl && hr) {
            if (sp == kBvhStack) {                            // cannot happen for depth <= 63; never write past it
              atomicOr(a.error_flag, 1);
              best_face = -1;
              break;
            }
            const bool left_first = tl <= tr;
            stack_node[sp] = left_first ? cr : cl;
            stack_t[sp] = left_first ? tr : tl;
            ++sp;
            node = left_first ? cl : cr;
            continue;
          }
          if (hl || hr) {
            node = hl ? cl : cr;
            continue;
          }
        }
        // next deferred node that may still hold a hit no later than the best
        bool found = false;
        while (sp > 0) {
          --sp;
          if (stack_t[sp] <= best) {
            node = stack_node[sp];
            found = true;
            break;
          }
        }
        if (!found) break;
      }
    }
    a.hit_face[r] = best_face;
    a.hit_t[r] = best_face >= 0 ? best : INFINITY;
    a.hit_bary[2 * r] = best_face >= 0 ? best_b1 : 0.f;
    a.hit_bary[2 * r + 1] = best_face >= 0 ? best_b2 : 0.f;
  }
}

int grid_blocks(int64_t n, int threads) {
  return (int)std::min<int64_t>((n + threads - 1) / threads, (int64_t)mnrf_num_sms() * 16);
}

}  // namespace

}  // namespace mnrf

extern "C" int mnrf_mesh_bvh(int32_t phase, int32_t num_vertices, int64_t num_faces, const float* vertices,
                             const int32_t* faces, float* face_boxes, float* centroids, const float* centroid_bounds,
                             int64_t* keys, const int64_t* sorted_keys, float* nodes, int32_t* parent,
                             int32_t* leaf_face, int32_t* counters, mnrf_stream stream) {
  using namespace mnrf;
  set_error("");
  MNRF_CHECK(phase == MNRF_BVH_BOXES || phase == MNRF_BVH_KEYS || phase == MNRF_BVH_TREE,
             "mnrf_mesh_bvh: unknown phase %d", phase);
  MNRF_CHECK(num_vertices > 0 && num_faces >= 1 && num_faces < (int64_t(1) << 30),
             "mnrf_mesh_bvh: %d vertices, %lld faces", num_vertices, (long long)num_faces);
  const cudaStream_t st = (cudaStream_t)stream;
  const int blocks = grid_blocks(num_faces, 256);
  if (phase == MNRF_BVH_BOXES) {
    MNRF_CHECK(vertices && faces && face_boxes && centroids, "mnrf_mesh_bvh: null pointer (boxes)");
    bvh_boxes_kernel<<<blocks, 256, 0, st>>>(num_faces, vertices, faces, face_boxes, centroids);
  } else if (phase == MNRF_BVH_KEYS) {
    MNRF_CHECK(centroids && centroid_bounds && keys, "mnrf_mesh_bvh: null pointer (keys)");
    bvh_keys_kernel<<<blocks, 256, 0, st>>>(num_faces, centroids, centroid_bounds, keys);
  } else {
    MNRF_CHECK(num_faces >= 2, "mnrf_mesh_bvh: %lld faces: a tree needs 2 or more", (long long)num_faces);
    MNRF_CHECK(face_boxes && sorted_keys && nodes && parent && leaf_face && counters,
               "mnrf_mesh_bvh: null pointer (tree)");
    MNRF_CUDA(cudaMemsetAsync(counters, 0, sizeof(int32_t) * (num_faces - 1), st));
    bvh_topology_kernel<<<grid_blocks(num_faces - 1, 256), 256, 0, st>>>(num_faces, sorted_keys, nodes, parent);
    bvh_refit_kernel<<<blocks, 256, 0, st>>>(num_faces, sorted_keys, face_boxes, leaf_face, parent, counters, nodes);
  }
  MNRF_LAUNCH_CHECK();
  return 0;
}

extern "C" int mnrf_mesh_trace(int64_t num_rays, const float* origins, const float* directions, const float* near,
                               const float* far, int64_t num_faces, const float* nodes, const int32_t* leaf_face,
                               const float* vertices, const int32_t* faces, int32_t* hit_face, float* hit_t,
                               float* hit_bary, int32_t* error_flag, mnrf_stream stream) {
  using namespace mnrf;
  set_error("");
  MNRF_CHECK(num_rays >= 0 && num_faces >= 1 && num_faces < (int64_t(1) << 30),
             "mnrf_mesh_trace: %lld rays, %lld faces", (long long)num_rays, (long long)num_faces);
  if (num_rays == 0) return 0;
  MNRF_CHECK(origins && directions && near && far && leaf_face && vertices && faces && hit_face && hit_t &&
                 hit_bary && error_flag && (nodes || num_faces == 1),
             "mnrf_mesh_trace: null pointer");
  MNRF_CHECK(((uintptr_t)nodes & 15) == 0, "mnrf_mesh_trace: nodes must be 16-byte aligned");
  TraceArgs a{num_rays, num_faces, origins, directions, near, far, reinterpret_cast<const float4*>(nodes),
              leaf_face, vertices, faces, hit_face, hit_t, hit_bary, error_flag};
  trace_kernel<<<grid_blocks(num_rays, 128), 128, 0, (cudaStream_t)stream>>>(a);
  MNRF_LAUNCH_CHECK();
  return 0;
}
