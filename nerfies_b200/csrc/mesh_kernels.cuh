// Marching cubes on a density grid: an indexed, watertight, oriented triangle mesh of the surface
// {value > level}, with no atomics, so that two calls on one grid write bitwise-equal meshes.
//   classify_kernel     per grid point: crossing flags of its three edges, case and triangle count of
//                       its cube
//   (CUB)               int64 total of the triangle counts; exclusive scans of the edge flags (vertex
//                       ids) and of the triangle counts (face offsets), in place
//   finish_counts_kernel  the two totals into the caller's counts
//   vertex_kernel       one vertex per crossing edge: interpolated position and normal
//   face_kernel         each cube's triangles from the case table, in table order
// The case table is derived below from one rule at compile time (derive_wide_table); DESIGN.md §5.5e
// describes the rule, the layout and the workspace.
#pragma once
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>

#include "../../include/nerfies_b200.h"

namespace nfb {
namespace mesh {

constexpr int kMaxSide = 1024;
constexpr int kThreads = 256;

// ---------------------------------------------------------------------------------------------
// Cube geometry.  Corner c sits at offset (c & 1, c >> 1 & 1, c >> 2 & 1) from the cube's lowest
// grid point.  Edge e = 4 * axis + r runs along `axis` from corner edge_corner(e); r = u + 2 v, where
// u and v are that corner's coordinates along the other two axes, the lower axis first.
// ---------------------------------------------------------------------------------------------
__host__ __device__ constexpr int other_axis(int axis, int which) {   // which 0: lower, 1: higher
  return which == 0 ? (axis == 0 ? 1 : 0) : (axis == 2 ? 1 : 2);
}
__host__ __device__ constexpr int edge_corner(int e) {
  const int axis = e >> 2;
  return ((e & 1) << other_axis(axis, 0)) | (((e >> 1) & 1) << other_axis(axis, 1));
}
__host__ __device__ constexpr bool share_face(int e0, int e1) {     // face = 2 * axis + side
  const int f0a = 2 * other_axis(e0 >> 2, 0) + (e0 & 1), f0b = 2 * other_axis(e0 >> 2, 1) + ((e0 >> 1) & 1);
  const int f1a = 2 * other_axis(e1 >> 2, 0) + (e1 & 1), f1b = 2 * other_axis(e1 >> 2, 1) + ((e1 >> 1) & 1);
  return f0a == f1a || f0a == f1b || f0b == f1a || f0b == f1b;
}
__host__ __device__ constexpr int edge_between(int c0, int c1) {      // c0, c1 differ in one bit
  const int bit = c0 ^ c1, axis = bit == 1 ? 0 : bit == 2 ? 1 : 2;
  const int lo = c0 & c1;
  return 4 * axis + ((lo >> other_axis(axis, 0)) & 1) + 2 * ((lo >> other_axis(axis, 1)) & 1);
}

// ---------------------------------------------------------------------------------------------
// Case table.  For case bits (bit c set <=> corner c inside) and each of the six faces, walk the
// face's corners counter-clockwise as seen from outside the cube.  Every maximal run of consecutive
// inside corners is entered through one crossing edge and left through another; it gives the segment
// entry -> exit.  A face with two inside corners on a diagonal has two runs of one corner each, so
// each inside corner is cut off separately.  Each crossing edge lies on two faces, which traverse it
// in opposite directions, so it ends one segment and starts another: the segments chain into closed
// loops.  Each loop is fan-triangulated from the first vertex (in loop order from its lowest edge)
// whose diagonals all cross the cube's interior, none lying in a face.  A cube sharing a face sees
// the same four corners and the same runs, traversed the other way round: the mesh is closed and
// every triangle is counter-clockwise seen from outside (from lower density).
// ---------------------------------------------------------------------------------------------
constexpr int kWideTriangles = 10;     // a loop of all 12 edges would give 10

struct WideTable {
  int count[256];
  int edge[256][3 * kWideTriangles];
  int max_triangles;
  bool no_apex;              // some loop has no vertex whose fan keeps every diagonal off the faces
};

constexpr WideTable derive_wide_table() {
  WideTable t{};
  for (int cs = 0; cs < 256; ++cs) {
    int next[12] = {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1};
    for (int f = 0; f < 6; ++f) {
      const int axis = f >> 1, side = f & 1;
      const int b = (axis + 1) % 3, c = (axis + 2) % 3;    // e_b x e_c = e_axis
      const int uv[4][2] = {{0, 0}, {1, 0}, {1, 1}, {0, 1}};   // counter-clockwise seen from +e_axis
      int ring[4] = {0, 0, 0, 0};
      for (int q = 0; q < 4; ++q) {
        const int k = side ? q : 3 - q;                    // seen from outside: reversed on the low side
        ring[q] = (side << axis) | (uv[k][0] << b) | (uv[k][1] << c);
      }
      for (int q = 0; q < 4; ++q) {
        const int u = ring[q], v = ring[(q + 1) & 3];
        if (((cs >> u) & 1) || !((cs >> v) & 1)) continue;  // not an entry (outside -> inside)
        for (int r = 1; r < 4; ++r) {                      // the run's exit: first inside -> outside
          const int x = ring[(q + r) & 3], y = ring[(q + r + 1) & 3];
          if (((cs >> x) & 1) && !((cs >> y) & 1)) {
            next[edge_between(u, v)] = edge_between(x, y);
            break;
          }
        }
      }
    }
    bool seen[12] = {};
    int n = 0;
    for (int e0 = 0; e0 < 12; ++e0) {
      if (next[e0] < 0 || seen[e0]) continue;
      int loop[12] = {}, len = 0;
      for (int e = e0; !seen[e]; e = next[e]) {
        seen[e] = true;
        loop[len++] = e;
      }
      // The fan's apex: the first loop vertex none of whose diagonals joins two edges of one cube
      // face.  Such a diagonal would lie in the face, where the neighbouring cube can draw it too.
      int apex = -1;
      for (int s = 0; s < len && apex < 0; ++s) {
        bool ok = true;
        for (int i = 2; i + 1 < len; ++i) ok = ok && !share_face(loop[s], loop[(s + i) % len]);
        if (ok) apex = s;
      }
      if (apex < 0) {
        t.no_apex = true;
        apex = 0;
      }
      for (int i = 1; i + 1 < len; ++i) {
        t.edge[cs][3 * n] = loop[apex];
        t.edge[cs][3 * n + 1] = loop[(apex + i) % len];
        t.edge[cs][3 * n + 2] = loop[(apex + i + 1) % len];
        ++n;
      }
    }
    t.count[cs] = n;
    if (n > t.max_triangles) t.max_triangles = n;
  }
  return t;
}

constexpr WideTable kWideTable = derive_wide_table();
constexpr int kMaxTriangles = kWideTable.max_triangles;
static_assert(kMaxTriangles > 0 && kMaxTriangles <= kWideTriangles, "case table derivation");
static_assert(!kWideTable.no_apex, "a loop whose every fan puts a diagonal on a cube face");

struct CaseTable {
  unsigned char count[256];
  unsigned char edge[256][3 * kMaxTriangles];
};

constexpr CaseTable narrow_table() {
  CaseTable t{};
  for (int cs = 0; cs < 256; ++cs) {
    t.count[cs] = (unsigned char)kWideTable.count[cs];
    for (int i = 0; i < 3 * kWideTable.count[cs]; ++i) t.edge[cs][i] = (unsigned char)kWideTable.edge[cs][i];
  }
  return t;
}

constexpr CaseTable kCaseTable = narrow_table();
__constant__ CaseTable c_case_table = kCaseTable;

// ---------------------------------------------------------------------------------------------
// Kernels.  Grid point p = (k * ny + j) * nx + i; the edge of axis a starting at p is edge a * n + p
// (n = nx * ny * nz), and the cube whose lowest corner is p is cube p.  Points on the high border
// start no edge along that axis and no cube: their flags and counts are 0.
// ---------------------------------------------------------------------------------------------
struct MeshArgs {
  const float* grid;
  int nx, ny, nz;
  long long n;
  float level;
  float origin[3], spacing[3];
  unsigned* edge_ids;        // (3n + 1): flags, then their exclusive scan = vertex ids
  unsigned* tri_offsets;     // (n + 1): triangle counts, then their exclusive scan = face offsets
  long long* totals;         // [vertices, faces]
  float* vertices;           // (V, 3)
  float* normals;            // (V, 3), nullable
  int* faces;                // (F, 3)
};

__device__ __forceinline__ bool is_inside(float v, float level) { return v > level; }   // NaN: outside

__device__ __forceinline__ void grid_coords(const MeshArgs& a, long long p, int* c) {
  const long long q = p / a.nx;
  c[0] = (int)(p - q * a.nx);
  c[1] = (int)(q % a.ny);
  c[2] = (int)(q / a.ny);
}

__device__ __forceinline__ long long corner_offset(const MeshArgs& a, int corner) {
  return (corner & 1) + ((corner >> 1) & 1) * (long long)a.nx + ((corner >> 2) & 1) * (long long)a.nx * a.ny;
}

__device__ __forceinline__ int cube_case(const MeshArgs& a, long long p) {
  int cs = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) cs |= (int)is_inside(__ldg(a.grid + p + corner_offset(a, c)), a.level) << c;
  return cs;
}

__global__ void __launch_bounds__(kThreads) classify_kernel(const MeshArgs a) {
  const long long p = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (p == 0) {
    a.edge_ids[3 * a.n] = 0;
    a.tri_offsets[a.n] = 0;
  }
  if (p >= a.n) return;
  int c[3];
  grid_coords(a, p, c);
  const bool in0 = is_inside(__ldg(a.grid + p), a.level);
  const int dims[3] = {a.nx, a.ny, a.nz};
  const long long stride[3] = {1, a.nx, (long long)a.nx * a.ny};
#pragma unroll
  for (int axis = 0; axis < 3; ++axis) {
    unsigned flag = 0;
    if (c[axis] + 1 < dims[axis]) flag = in0 != is_inside(__ldg(a.grid + p + stride[axis]), a.level);
    a.edge_ids[axis * a.n + p] = flag;
  }
  const bool cube = c[0] + 1 < a.nx && c[1] + 1 < a.ny && c[2] + 1 < a.nz;
  a.tri_offsets[p] = cube ? c_case_table.count[cube_case(a, p)] : 0u;
}

__global__ void finish_counts_kernel(const MeshArgs a, long long* counts_out) {
  a.totals[0] = a.edge_ids[3 * a.n];
  counts_out[0] = a.totals[0];
  counts_out[1] = a.totals[1];
  counts_out[2] = a.edge_ids[a.n];          // first vertex on a y-edge
  counts_out[3] = a.edge_ids[2 * a.n];      // first vertex on a z-edge
}

// Central difference along each axis, one-sided on the border, over the spacing.
__device__ __forceinline__ void gradient(const MeshArgs& a, long long p, const int* c, float* g) {
  const int dims[3] = {a.nx, a.ny, a.nz};
  const long long stride[3] = {1, a.nx, (long long)a.nx * a.ny};
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const bool lo = c[d] > 0, hi = c[d] + 1 < dims[d];
    const float vp = __ldg(a.grid + p + (hi ? stride[d] : 0));
    const float vm = __ldg(a.grid + p - (lo ? stride[d] : 0));
    const float h = (lo && hi) ? __fmul_rn(2.f, a.spacing[d]) : a.spacing[d];
    g[d] = __fdiv_rn(__fsub_rn(vp, vm), h);
  }
}

// Vertex of a crossing edge from p0 (value v0) to p1 (value v1), each coordinate in this order:
//   t = (level - v0) / (v1 - v0)            (t = 0.5 when v0 or v1 is NaN)
//   x0 = origin + float(index) * spacing,   x1 likewise at index + 1 along the edge's axis
//   x = x0 + t * (x1 - x0)                  (x = x0 across the edge)
// every operation rounded once (no fused multiply-add).
__global__ void __launch_bounds__(kThreads) vertex_kernel(const MeshArgs a) {
  const long long e = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (e >= 3 * a.n) return;
  const unsigned id = a.edge_ids[e];
  if (a.edge_ids[e + 1] == id) return;
  const int axis = (int)(e / a.n);
  const long long p = e - axis * a.n;
  int c[3];
  grid_coords(a, p, c);
  const long long stride = axis == 0 ? 1 : axis == 1 ? (long long)a.nx : (long long)a.nx * a.ny;
  const float v0 = __ldg(a.grid + p), v1 = __ldg(a.grid + p + stride);
  float t = __fdiv_rn(__fsub_rn(a.level, v0), __fsub_rn(v1, v0));
  if (isnan(v0) || isnan(v1)) t = 0.5f;
  float* out = a.vertices + 3ll * id;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float x0 = __fadd_rn(a.origin[d], __fmul_rn((float)c[d], a.spacing[d]));
    if (d != axis) {
      out[d] = x0;
    } else {
      const float x1 = __fadd_rn(a.origin[d], __fmul_rn((float)(c[d] + 1), a.spacing[d]));
      out[d] = __fadd_rn(x0, __fmul_rn(t, __fsub_rn(x1, x0)));
    }
  }
  if (!a.normals) return;
  // Outward normal: minus the gradient interpolated between the edge's endpoints, normalised.
  float g0[3], g1[3], g[3];
  gradient(a, p, c, g0);
  const int c1[3] = {c[0] + (axis == 0), c[1] + (axis == 1), c[2] + (axis == 2)};
  gradient(a, p + stride, c1, g1);
  float len2 = 0.f;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    g[d] = g0[d] + t * (g1[d] - g0[d]);
    len2 += g[d] * g[d];
  }
  const float inv = len2 > 0.f && isfinite(len2) ? -rsqrtf(len2) : 0.f;
  float* nrm = a.normals + 3ll * id;
#pragma unroll
  for (int d = 0; d < 3; ++d) nrm[d] = inv != 0.f ? g[d] * inv : 0.f;
}

__global__ void __launch_bounds__(kThreads) face_kernel(const MeshArgs a) {
  const long long p = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (p >= a.n) return;
  const unsigned first = a.tri_offsets[p];
  const unsigned count = a.tri_offsets[p + 1] - first;
  if (count == 0) return;
  const int cs = cube_case(a, p);
  int* out = a.faces + 3ll * first;
  for (unsigned i = 0; i < 3 * count; ++i) {
    const int e = c_case_table.edge[cs][i];
    out[i] = (int)a.edge_ids[(e >> 2) * a.n + p + corner_offset(a, edge_corner(e))];
  }
}

}  // namespace mesh
}  // namespace nfb
