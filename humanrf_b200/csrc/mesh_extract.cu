// Marching cubes over a (G+1)^3 fp32 lattice (include/humanrf_b200.h, hrf_marching_cubes_*).  The lattice is cut into
// bricks of kBrick consecutive vertices (linear index x + (G+1) (y + (G+1) z)); vertex v owns the lattice edges from v
// along +x, +y, +z and, when x, y, z < G, the cube whose lower corner it is.  A three-phase scan over the bricks gives
// every vertex and face its place without atomics, so two runs write identical bytes:
//   mc_count_kernel : per brick, the number of crossing edges (mesh vertices) and of triangles
//   mc_scan_kernel  : one CTA, exclusive scan of the brick totals (int64) -> brick offsets, counts[2] = {V, F}
//   -- the caller reads counts[2] and sizes the outputs --
//   mc_vertex_kernel: per brick, block scan of the vertex counts -> vertex ids (kept in the workspace for the faces),
//                     positions, normals
//   mc_face_kernel  : per brick, block scan of the triangle counts -> faces, from the case table in __constant__
// The case table is generated once per device on the host from the face rule (mc_build_table).
#include <math.h>

#include <mutex>
#include <vector>

#include "common.cuh"

namespace hrf {

constexpr int kMcThreads = 256;
constexpr int kMcRounds = 8;
constexpr int64_t kBrick = (int64_t)kMcThreads * kMcRounds;   // lattice vertices per brick
constexpr int kMcMaxTri = 5;                                  // the face rule never needs more (checked when generated)
constexpr int kMcScanThreads = 1024;

__constant__ uint8_t c_mc_ntri[256];
__constant__ uint8_t c_mc_tri[256][3 * kMcMaxTri];

// ------------------------------------------------------------------------------------------------- case table (host)
// Corner c = a + 2b + 4d sits at (a, b, d).  Cube edge e = 4 * axis + idx runs along `axis` from its lower corner, whose
// two other coordinates are (idx & 1, idx >> 1) in axis order.
static void edge_corners(int e, int* lo, int* hi) {
  const int axis = e >> 2, idx = e & 3;
  int p[3] = {0, 0, 0};
  int o = 0;
  for (int a = 0; a < 3; ++a)
    if (a != axis) p[a] = o++ == 0 ? (idx & 1) : (idx >> 1);
  *lo = p[0] + 2 * p[1] + 4 * p[2];
  p[axis] = 1;
  *hi = p[0] + 2 * p[1] + 4 * p[2];
}

static int corner_coord(int c, int a) { return (c >> a) & 1; }

// Face rule: on a face with two crossing edges they are joined; with four (ambiguous), the two edges at each inside
// corner are joined, so inside corners are never connected across a face.  Segment A -> B is oriented so that
// (mid B - mid A) x (inside corner of A - mid A) points into the cube; the loops then wind counter-clockwise seen from
// the outside.  Loops start at their smallest unused crossing edge, in ascending order, and are fan-triangulated from
// their first vertex (in loop order) whose diagonals join no two edges of a common cube face (such a diagonal could be
// drawn by the neighbouring cube too).
static bool mc_build_table(uint8_t* ntri, uint8_t (*tri)[3 * kMcMaxTri]) {
  int lo[12], hi[12];
  for (int e = 0; e < 12; ++e) edge_corners(e, &lo[e], &hi[e]);
  auto mid = [&](int e, int a) { return 0.5 * (corner_coord(lo[e], a) + corner_coord(hi[e], a)); };
  auto on_face = [&](int e, int ax, int side) { return (e >> 2) != ax && corner_coord(lo[e], ax) == side; };
  auto share_face = [&](int e, int f) {
    for (int ax = 0; ax < 3; ++ax)
      for (int side = 0; side < 2; ++side)
        if (on_face(e, ax, side) && on_face(f, ax, side)) return true;
    return false;
  };
  for (int cs = 0; cs < 256; ++cs) {
    bool cross[12];
    int nxt[12];
    for (int e = 0; e < 12; ++e) {
      cross[e] = ((cs >> lo[e]) & 1) != ((cs >> hi[e]) & 1);
      nxt[e] = -1;
    }
    for (int ax = 0; ax < 3; ++ax)
      for (int side = 0; side < 2; ++side) {
        int fe[4], nf = 0, fc[4], nc = 0;
        for (int e = 0; e < 12; ++e)
          if (on_face(e, ax, side)) {
            fe[nf++] = e;
            if (cross[e]) fc[nc++] = e;
          }
        int seg[2][2], ns = 0;
        if (nc == 2) {
          seg[0][0] = fc[0], seg[0][1] = fc[1], ns = 1;
        } else if (nc == 4) {
          for (int c = 0; c < 8; ++c) {
            if (corner_coord(c, ax) != side || !((cs >> c) & 1)) continue;
            int k = 0;
            for (int q = 0; q < 4; ++q)
              if (lo[fe[q]] == c || hi[fe[q]] == c) seg[ns][k++] = fe[q];
            ++ns;
          }
        }
        for (int s = 0; s < ns; ++s) {
          int a = seg[s][0], b = seg[s][1];
          const int ca = ((cs >> lo[a]) & 1) ? lo[a] : hi[a];
          double u[3], w[3];
          for (int q = 0; q < 3; ++q) u[q] = mid(b, q) - mid(a, q), w[q] = corner_coord(ca, q) - mid(a, q);
          const double cr[3] = {u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0]};
          const double d = cr[ax] * (2 * side - 1);
          if (d == 0.0) return false;
          if (d > 0) std::swap(a, b);
          if (nxt[a] != -1) return false;
          nxt[a] = b;
        }
      }
    bool used[12] = {};
    int nt = 0;
    for (int e = 0; e < 12; ++e) {
      if (!cross[e] || used[e]) continue;
      int loop[12], n = 0;
      for (int x = e;;) {
        if (n == 12 || x < 0) return false;
        loop[n++] = x;
        used[x] = true;
        x = nxt[x];
        if (x == e) break;
      }
      int r = 0;
      for (; r < n; ++r) {
        bool ok = true;
        for (int i = 2; i < n - 1; ++i) ok = ok && !share_face(loop[r], loop[(r + i) % n]);
        if (ok) break;
      }
      if (r == n) return false;
      for (int i = 1; i < n - 1; ++i) {
        if (nt == kMcMaxTri) return false;
        tri[cs][3 * nt] = (uint8_t)loop[r], tri[cs][3 * nt + 1] = (uint8_t)loop[(r + i) % n];
        tri[cs][3 * nt + 2] = (uint8_t)loop[(r + i + 1) % n];
        ++nt;
      }
    }
    ntri[cs] = (uint8_t)nt;
  }
  return true;
}

// Uploads the table to the current device once.
static int mc_upload_table() {
  static std::mutex mu;
  static std::vector<int> done;
  int dev = 0;
  HRF_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  if (dev < (int)done.size() && done[dev]) return 0;
  static uint8_t ntri[256], tri[256][3 * kMcMaxTri];
  static const bool ok = mc_build_table(ntri, tri);
  HRF_REQUIRE(ok, "marching-cubes case table generation failed");
  HRF_CUDA(cudaMemcpyToSymbol(c_mc_ntri, ntri, sizeof(ntri)));
  HRF_CUDA(cudaMemcpyToSymbol(c_mc_tri, tri, sizeof(tri)));
  if (dev >= (int)done.size()) done.resize(dev + 1, 0);
  done[dev] = 1;
  return 0;
}

// ------------------------------------------------------------------------------------------------------ device side
struct McGrid {
  const float* sig;
  int G;
  float level;
  int64_t n;   // (G+1)^3
};

__device__ __forceinline__ bool mc_inside(const McGrid& g, int64_t v) { return __ldg(g.sig + v) >= g.level; }

// Lattice coordinates of vertex v ((G+1)^3 <= 1025^3 fits 32 bits).
__device__ __forceinline__ void mc_coords(const McGrid& g, int64_t v, int* x, int* y, int* z) {
  const uint32_t Gp = (uint32_t)g.G + 1u, vu = (uint32_t)v, yz = vu / Gp;
  *x = (int)(vu - yz * Gp), *y = (int)(yz % Gp), *z = (int)(yz / Gp);
}

// Crossing bits (x, y, z) of the lattice edges vertex v owns.
__device__ __forceinline__ int mc_edge_bits(const McGrid& g, int64_t v) {
  const int64_t Gp = g.G + 1;
  int x, y, z;
  mc_coords(g, v, &x, &y, &z);
  const bool in0 = mc_inside(g, v);
  int b = 0;
  if (x < g.G && mc_inside(g, v + 1) != in0) b |= 1;
  if (y < g.G && mc_inside(g, v + Gp) != in0) b |= 2;
  if (z < g.G && mc_inside(g, v + Gp * Gp) != in0) b |= 4;
  return b;
}

// Case (bit k = corner k inside) of the cube whose lower corner is v, or -1 when v has no cube.
__device__ __forceinline__ int mc_case(const McGrid& g, int64_t v) {
  const int64_t Gp = g.G + 1;
  int x, y, z;
  mc_coords(g, v, &x, &y, &z);
  if (x >= g.G || y >= g.G || z >= g.G) return -1;
  int c = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) c |= (int)mc_inside(g, v + (k & 1) + ((k >> 1) & 1) * Gp + (k >> 2) * Gp * Gp) << k;
  return c;
}

__device__ __forceinline__ int mc_ntri(int cs) { return cs < 0 ? 0 : (int)c_mc_ntri[cs]; }

// Exclusive block scan of one int per thread; *total = the block's sum.  smem: kMcThreads / 32 ints.
__device__ __forceinline__ int mc_block_scan(int x, int* smem, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int s = x;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, s, d);
    if (lane >= d) s += y;
  }
  if (lane == 31) smem[warp] = s;
  __syncthreads();
  int before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < kMcThreads / 32; ++w) {
    const int t = smem[w];
    if (w < warp) before += t;
    all += t;
  }
  __syncthreads();
  *total = all;
  return before + s - x;
}

__global__ void __launch_bounds__(kMcThreads) mc_count_kernel(const McGrid g, int32_t* __restrict__ brick_v,
                                                             int32_t* __restrict__ brick_f) {
  __shared__ int red[2][kMcThreads / 32];
  const int64_t base = (int64_t)blockIdx.x * kBrick;
  int nv = 0, nf = 0;
  for (int r = 0; r < kMcRounds; ++r) {
    const int64_t v = base + r * kMcThreads + threadIdx.x;
    if (v < g.n) {
      nv += __popc(mc_edge_bits(g, v));
      nf += mc_ntri(mc_case(g, v));
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    nv += __shfl_xor_sync(0xffffffffu, nv, d);
    nf += __shfl_xor_sync(0xffffffffu, nf, d);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[0][warp] = nv, red[1][warp] = nf;
  __syncthreads();
  if (threadIdx.x == 0) {
    int sv = 0, sf = 0;
    for (int w = 0; w < kMcThreads / 32; ++w) sv += red[0][w], sf += red[1][w];
    brick_v[blockIdx.x] = sv;
    brick_f[blockIdx.x] = sf;
  }
}

// One CTA: thread t scans a contiguous run of bricks serially; the runs are joined by a block scan.
__global__ void __launch_bounds__(kMcScanThreads) mc_scan_kernel(const int32_t* __restrict__ brick_v,
                                                                const int32_t* __restrict__ brick_f, int64_t nb,
                                                                int64_t* __restrict__ off_v, int64_t* __restrict__ off_f,
                                                                int64_t* __restrict__ counts) {
  __shared__ long long sv[kMcScanThreads], sf[kMcScanThreads];
  const int t = threadIdx.x;
  const int64_t per = (nb + kMcScanThreads - 1) / kMcScanThreads;
  const int64_t b0 = (int64_t)t * per, b1 = b0 + per < nb ? b0 + per : nb;
  long long av = 0, af = 0;
  for (int64_t b = b0; b < b1; ++b) av += brick_v[b], af += brick_f[b];
  sv[t] = av, sf[t] = af;
  __syncthreads();
  for (int d = 1; d < kMcScanThreads; d <<= 1) {   // Hillis-Steele inclusive scan
    const long long xv = t >= d ? sv[t - d] : 0, xf = t >= d ? sf[t - d] : 0;
    __syncthreads();
    sv[t] += xv, sf[t] += xf;
    __syncthreads();
  }
  long long ov = sv[t] - av, of = sf[t] - af;
  for (int64_t b = b0; b < b1; ++b) {
    off_v[b] = ov, off_f[b] = of;
    ov += brick_v[b], of += brick_f[b];
  }
  if (t == kMcScanThreads - 1) counts[0] = sv[t], counts[1] = sf[t];
}

// d sigma / d axis at lattice vertex v (coordinate c along that axis, stride st): central differences, one-sided at the
// lattice border.
__device__ __forceinline__ float mc_grad(const McGrid& g, int64_t v, int c, int64_t st) {
  if (c == 0) return __fsub_rn(__ldg(g.sig + v + st), __ldg(g.sig + v));
  if (c == g.G) return __fsub_rn(__ldg(g.sig + v), __ldg(g.sig + v - st));
  return __fmul_rn(__fsub_rn(__ldg(g.sig + v + st), __ldg(g.sig + v - st)), 0.5f);
}

__global__ void __launch_bounds__(kMcThreads) mc_vertex_kernel(const McGrid g, const int64_t* __restrict__ off_v,
                                                              int64_t cap_v, int32_t* __restrict__ vid,
                                                              float* __restrict__ verts, float* __restrict__ normals) {
  __shared__ int scan_smem[kMcThreads / 32];
  const int64_t base = (int64_t)blockIdx.x * kBrick;
  int64_t next = off_v[blockIdx.x];
  const int64_t Gp = g.G + 1;
  const float Gf = (float)g.G;
  for (int r = 0; r < kMcRounds; ++r) {
    const int64_t v = base + r * kMcThreads + threadIdx.x;
    const int bits = v < g.n ? mc_edge_bits(g, v) : 0;
    int total;
    const int pre = mc_block_scan(__popc(bits), scan_smem, &total);
    int64_t id = next + pre;
    next += total;
    if (v >= g.n) continue;
    vid[v] = (int32_t)id;   // first vertex of v (the caller guarantees V <= INT32_MAX)
    if (bits == 0) continue;
    int c[3];
    mc_coords(g, v, &c[0], &c[1], &c[2]);
    const int64_t st[3] = {1, Gp, Gp * Gp};
    const float s0 = __ldg(g.sig + v);
    float p[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) p[a] = __fsub_rn(__fdiv_rn((float)c[a], Gf), 0.5f);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (!((bits >> a) & 1)) continue;
      if (id < cap_v) {
        const float s1 = __ldg(g.sig + v + st[a]);
        const float t = __fdiv_rn(__fsub_rn(g.level, s0), __fsub_rn(s1, s0));
        float q[3] = {p[0], p[1], p[2]};
        q[a] = __fsub_rn(__fdiv_rn(__fadd_rn((float)c[a], t), Gf), 0.5f);
        verts[3 * id] = q[0], verts[3 * id + 1] = q[1], verts[3 * id + 2] = q[2];
        if (normals != nullptr) {
          float n[3];
#pragma unroll
          for (int b = 0; b < 3; ++b) {
            const float g0 = mc_grad(g, v, c[b], st[b]);
            const int c1 = c[b] + (b == a ? 1 : 0);
            const float g1 = mc_grad(g, v + st[a], c1, st[b]);
            n[b] = -__fadd_rn(g0, __fmul_rn(t, __fsub_rn(g1, g0)));
          }
          const float m = fmaxf(fabsf(n[0]), fmaxf(fabsf(n[1]), fabsf(n[2])));
          if (m > 0.f) {
#pragma unroll
            for (int b = 0; b < 3; ++b) n[b] = __fdiv_rn(n[b], m);
            const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(n[0], n[0]), __fmul_rn(n[1], n[1])),
                                                   __fmul_rn(n[2], n[2])));
#pragma unroll
            for (int b = 0; b < 3; ++b) n[b] = __fdiv_rn(n[b], len);
          } else {
            n[0] = n[1] = n[2] = 0.f;
          }
          normals[3 * id] = n[0], normals[3 * id + 1] = n[1], normals[3 * id + 2] = n[2];
        }
      }
      ++id;
    }
  }
}

// Mesh vertex of cube edge e of the cube whose lower corner is v: owner = lower corner of the edge; its id = the
// owner's first vertex + the number of its crossing edges along lower axes.
__device__ __forceinline__ int32_t mc_edge_vertex(const McGrid& g, const int32_t* __restrict__ vid, int64_t v, int x,
                                                  int y, int e) {
  const int64_t Gp = g.G + 1;
  const int axis = e >> 2, idx = e & 3;
  const int ox = axis == 0 ? 0 : (idx & 1);
  const int oy = axis == 1 ? 0 : (axis == 0 ? (idx & 1) : (idx >> 1));
  const int oz = axis == 2 ? 0 : (idx >> 1);
  const int64_t w = v + ox + oy * Gp + oz * Gp * Gp;
  int32_t id = __ldg(vid + w);
  if (axis > 0) {   // the owner's crossing edges along lower axes come first
    const bool in0 = mc_inside(g, w);
    if (x + ox < g.G && mc_inside(g, w + 1) != in0) ++id;
    if (axis == 2 && y + oy < g.G && mc_inside(g, w + Gp) != in0) ++id;
  }
  return id;
}

__global__ void __launch_bounds__(kMcThreads) mc_face_kernel(const McGrid g, const int64_t* __restrict__ off_f,
                                                            const int32_t* __restrict__ vid, int64_t cap_f,
                                                            int32_t* __restrict__ faces) {
  __shared__ int scan_smem[kMcThreads / 32];
  const int64_t base = (int64_t)blockIdx.x * kBrick;
  int64_t next = off_f[blockIdx.x];
  for (int r = 0; r < kMcRounds; ++r) {
    const int64_t v = base + r * kMcThreads + threadIdx.x;
    const int cs = v < g.n ? mc_case(g, v) : -1;
    const int nt = mc_ntri(cs);
    int total;
    const int pre = mc_block_scan(nt, scan_smem, &total);
    const int64_t first = next + pre;
    next += total;
    int x = 0, y = 0, z = 0;
    if (nt > 0) mc_coords(g, v, &x, &y, &z);
    for (int k = 0; k < nt; ++k) {
      const int64_t fid = first + k;
      if (fid >= cap_f) break;
#pragma unroll
      for (int q = 0; q < 3; ++q) faces[3 * fid + q] = mc_edge_vertex(g, vid, v, x, y, c_mc_tri[cs][3 * k + q]);
    }
  }
}

static int64_t mc_bricks(int G) {
  const int64_t gp = (int64_t)G + 1;
  return (gp * gp * gp + kBrick - 1) / kBrick;
}

}  // namespace hrf

using namespace hrf;

// workspace: brick totals (2 x int32) and offsets (2 x int64) per brick, then the per-vertex first-vertex ids
extern "C" int64_t hrf_marching_cubes_workspace_bytes(int grid_resolution) {
  if (grid_resolution < 1 || grid_resolution > 1024) return 0;
  const int64_t gp = (int64_t)grid_resolution + 1;
  const int64_t nb = mc_bricks(grid_resolution);
  return ((24 * nb + 255) / 256) * 256 + 4 * gp * gp * gp;
}

static int mc_check(const float* lattice, int G, float level, void* workspace) {
  HRF_REQUIRE(lattice != nullptr && workspace != nullptr, "null argument");
  HRF_REQUIRE(G >= 1 && G <= 1024, "grid resolution must be in [1, 1024] ((G+1)^3 int32 vertex ids)");
  HRF_REQUIRE(isfinite(level), "iso-level must be finite");
  return mc_upload_table();
}

extern "C" int hrf_marching_cubes_count(const float* lattice, int grid_resolution, float level, int64_t* counts,
                                        void* workspace, void* stream) {
  if (int rc = mc_check(lattice, grid_resolution, level, workspace)) return rc;
  HRF_REQUIRE(counts != nullptr, "null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t nb = mc_bricks(grid_resolution);
  char* ws = reinterpret_cast<char*>(workspace);
  int64_t* off_v = reinterpret_cast<int64_t*>(ws);
  int64_t* off_f = off_v + nb;
  int32_t* brick_v = reinterpret_cast<int32_t*>(off_f + nb);
  int32_t* brick_f = brick_v + nb;
  const int64_t gp = (int64_t)grid_resolution + 1;
  const McGrid g{lattice, grid_resolution, level, gp * gp * gp};
  mc_count_kernel<<<(unsigned)nb, kMcThreads, 0, st>>>(g, brick_v, brick_f);
  HRF_CHECK_LAUNCH();
  mc_scan_kernel<<<1, kMcScanThreads, 0, st>>>(brick_v, brick_f, nb, off_v, off_f, counts);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_marching_cubes_emit(const float* lattice, int grid_resolution, float level, int64_t num_vertices,
                                       int64_t num_faces, float* vertices, float* normals, int32_t* faces,
                                       void* workspace, void* stream) {
  if (int rc = mc_check(lattice, grid_resolution, level, workspace)) return rc;
  HRF_REQUIRE(num_vertices >= 0 && num_vertices <= INT32_MAX && num_faces >= 0,
              "vertex count must fit the int32 face indices");
  HRF_REQUIRE((vertices != nullptr || num_vertices == 0) && (faces != nullptr || num_faces == 0), "null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t nb = mc_bricks(grid_resolution);
  char* ws = reinterpret_cast<char*>(workspace);
  int64_t* off_v = reinterpret_cast<int64_t*>(ws);
  int64_t* off_f = off_v + nb;
  int32_t* vid = reinterpret_cast<int32_t*>(ws + ((24 * nb + 255) / 256) * 256);
  const int64_t gp = (int64_t)grid_resolution + 1;
  const McGrid g{lattice, grid_resolution, level, gp * gp * gp};
  mc_vertex_kernel<<<(unsigned)nb, kMcThreads, 0, st>>>(g, off_v, num_vertices, vid, vertices, normals);
  HRF_CHECK_LAUNCH();
  if (num_faces > 0) {
    mc_face_kernel<<<(unsigned)nb, kMcThreads, 0, st>>>(g, off_f, vid, num_faces, faces);
    HRF_CHECK_LAUNCH();
  }
  return 0;
}
