// Triangle rasterisation of a mesh into a camera-z depth map, a coverage mask and a face-id map (what the ActorsHQ
// toolbox's OpenGL mesh renderer writes), and depth / mask scores of a rendered depth map against such a reference.
// Contract: include/humanrf_b200.h, hrf_rasterize_mesh and hrf_depth_metrics; DESIGN.md §3.12.
// hrf_rasterize_mesh launches, in stream order, none synchronising with the host:
//   init_kernel    : keys = ~0, hits = 0, error = 0, skipped = 0;
//   vertex_kernel  : one thread per vertex: camera point, fixed-point pixel coordinates and camera z (fp64);
//   setup_kernel   : one thread per face: index check, skip rules, clipped bounding box, chunk count
//                    ceil(box pixels / kChunk) (0 for a face that draws nothing);
//   CUB exclusive sum of the chunk counts (int64);
//   raster_kernel  : persistent; each thread walks work items (face, chunk of <= kChunk box pixels), finding an item's
//                    face by binary search over the sum; coverage by exact int64 edge functions, fp64 depth, and a
//                    64-bit atomicMin of (z bits << 32 | face) per pixel;
//   resolve_kernel : keys -> z, mask, face.
// hrf_depth_metrics: metrics_kernel (fp64 / int64 sums per CTA) and finish_kernel (one CTA folds them in a fixed order).
// The only atomics are integer min / add / or: two calls write identical bytes.
#include <algorithm>

#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace hrf {
namespace {

constexpr int kThreads = 256;
constexpr int kChunk = 32;                     // box pixels per work item
constexpr int kRasterCtasPerSm = 8;
constexpr int kBadVertex = INT32_MIN;          // vertex record x of a vertex behind near or beyond +-2^21 pixels
constexpr double kMaxFixed = 536870912.0;      // 2^21 pixels in 8-bit fixed point
constexpr unsigned long long kEmptyKey = ~0ull;
constexpr int kMaxTaus = 8;
constexpr int kMetricPixels = 8;               // pixels per thread of metrics_kernel
constexpr int kCounts = 5;                     // n, |P|, |R|, |P and R|, |P or R|

struct __align__(16) VRec {
  int x, y;      // rint(256 u), rint(256 v); x = kBadVertex when the vertex is skipped
  double z;      // camera z
};

struct __align__(16) FRec {
  int x[3], y[3];   // fixed-point vertices, in the face's own order
  int x0, y0;       // first pixel of the clipped bounding box
  int bw, bh;       // its width and height in pixels
  double z[3];
};

struct Proj {
  double m[12];     // world -> camera, row-major 3x4
  double fx, fy, cx, cy, near;
};

__global__ void init_kernel(unsigned long long* __restrict__ keys, int64_t n, int32_t* __restrict__ hits,
                            int32_t* __restrict__ error, long long* __restrict__ skipped) {
  const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
  if (i < n) {
    keys[i] = kEmptyKey;
    if (hits) hits[i] = 0;
  }
  if (i == 0) *error = 0, *skipped = 0;
}

// X = ((m00 x + m01 y) + m02 z) + m03 (likewise Y, Z); u = (fxW X) / Z + cxW, v = (fyH Y) / Z + cyH; every operation
// rounded to nearest on its own.
__global__ void __launch_bounds__(kThreads) vertex_kernel(const float* __restrict__ verts, int64_t nv, Proj pr,
                                                          VRec* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
  if (i >= nv) return;
  const double p[3] = {(double)__ldg(verts + 3 * i), (double)__ldg(verts + 3 * i + 1), (double)__ldg(verts + 3 * i + 2)};
  double c[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double* m = pr.m + 4 * r;
    c[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[0], p[0]), __dmul_rn(m[1], p[1])), __dmul_rn(m[2], p[2])), m[3]);
  }
  const double u = __dadd_rn(__ddiv_rn(__dmul_rn(pr.fx, c[0]), c[2]), pr.cx);
  const double v = __dadd_rn(__ddiv_rn(__dmul_rn(pr.fy, c[1]), c[2]), pr.cy);
  const double us = __dmul_rn(u, 256.0), vs = __dmul_rn(v, 256.0);      // exact
  VRec o;
  o.z = c[2];
  // comparisons are false for NaN: a non-finite vertex is skipped too
  if (c[2] >= pr.near && c[2] <= 1.7976931348623157e308 && fabs(us) <= kMaxFixed && fabs(vs) <= kMaxFixed) {
    o.x = (int)rint(us), o.y = (int)rint(vs);
  } else {
    o.x = kBadVertex, o.y = 0;
  }
  out[i] = o;
}

// twice the signed area: (b - a) x (c - a), |coordinates| <= 2^29 so both products stay below 2^60
__device__ __forceinline__ long long area2(int ax, int ay, int bx, int by, int cx, int cy) {
  return (long long)(bx - ax) * (long long)(cy - ay) - (long long)(by - ay) * (long long)(cx - ax);
}

// One thread per face: index check (error bit 0), skip rule (skipped), zero area, clipped box; chunk count.
__global__ void __launch_bounds__(kThreads) setup_kernel(const int32_t* __restrict__ faces, int nf, int64_t nv,
                                                         const VRec* __restrict__ vrec, int width, int height,
                                                         FRec* __restrict__ frec, long long* __restrict__ chunks,
                                                         int32_t* __restrict__ error, long long* __restrict__ skipped) {
  const int f = blockIdx.x * kThreads + threadIdx.x;
  unsigned bad = 0, skip = 0;
  if (f < nf) {
    long long count = 0;
    const int i0 = __ldg(faces + 3 * (int64_t)f), i1 = __ldg(faces + 3 * (int64_t)f + 1),
              i2 = __ldg(faces + 3 * (int64_t)f + 2);
    if (i0 < 0 || i1 < 0 || i2 < 0 || i0 >= nv || i1 >= nv || i2 >= nv) {
      bad = 1;
    } else {
      const VRec a = vrec[i0], b = vrec[i1], c = vrec[i2];
      if (a.x == kBadVertex || b.x == kBadVertex || c.x == kBadVertex) {
        skip = 1;
      } else if (area2(a.x, a.y, b.x, b.y, c.x, c.y) != 0) {
        // pixels i with 256 i + 128 in [lo, hi]: ceil((lo - 128) / 256) .. floor((hi - 128) / 256) (>> floors)
        const int x_lo = max((min(min(a.x, b.x), c.x) + 127) >> 8, 0);
        const int x_hi = min((max(max(a.x, b.x), c.x) - 128) >> 8, width - 1);
        const int y_lo = max((min(min(a.y, b.y), c.y) + 127) >> 8, 0);
        const int y_hi = min((max(max(a.y, b.y), c.y) - 128) >> 8, height - 1);
        if (x_lo <= x_hi && y_lo <= y_hi) {
          FRec r;
          r.x[0] = a.x, r.x[1] = b.x, r.x[2] = c.x, r.y[0] = a.y, r.y[1] = b.y, r.y[2] = c.y;
          r.x0 = x_lo, r.y0 = y_lo, r.bw = x_hi - x_lo + 1, r.bh = y_hi - y_lo + 1;
          r.z[0] = a.z, r.z[1] = b.z, r.z[2] = c.z;
          frec[f] = r;
          count = ((long long)r.bw * r.bh + kChunk - 1) / kChunk;
        }
      }
    }
    chunks[f] = count;
  }
  bad = __reduce_or_sync(0xffffffffu, bad);
  const unsigned nskip = __reduce_add_sync(0xffffffffu, skip);
  if ((threadIdx.x & 31) == 0) {
    if (bad) atomicOr(error, 1);
    if (nskip) atomicAdd(reinterpret_cast<unsigned long long*>(skipped), (unsigned long long)nskip);
  }
}

// Tie rule for a sample on an oriented edge of direction d (E = 0): inside when d.y > 0, or d.y = 0 and d.x < 0.  It
// equals moving the sample by an infinitesimal (-1, -eps), so P(d) != P(-d) and a closed fan covers its centre once.
__device__ __forceinline__ bool tie_inside(long long dx, long long dy) { return dy > 0 || (dy == 0 && dx < 0); }

__global__ void __launch_bounds__(kThreads) raster_kernel(const FRec* __restrict__ frec,
                                                          const long long* __restrict__ P,
                                                          const long long* __restrict__ chunks, int nf, int width,
                                                          double near, double far, unsigned long long* __restrict__ keys,
                                                          int32_t* __restrict__ hits) {
  const long long total = nf > 0 ? P[nf - 1] + chunks[nf - 1] : 0;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long t = blockIdx.x * (long long)kThreads + threadIdx.x; t < total; t += stride) {
    int lo = 0, hi = nf;                     // P[lo] <= t, and P[hi] > t or hi = nf
    while (hi - lo > 1) {
      const int mid = lo + ((hi - lo) >> 1);
      if (__ldg(P + mid) <= t) lo = mid; else hi = mid;
    }
    const int f = lo;
    const FRec r = frec[f];
    long long A = area2(r.x[0], r.y[0], r.x[1], r.y[1], r.x[2], r.y[2]);
    const long long sg = A < 0 ? -1 : 1;
    A *= sg;
    const double Ad = __ll2double_rn(A);
    // edge k runs from vertex k+1 to vertex k+2: E_k(s) = d_k x (s - v_{k+1}), times the sign of A
    long long dx[3], dy[3];
    bool tie[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int a = (k + 1) % 3, b = (k + 2) % 3;
      dx[k] = (long long)(r.x[b] - r.x[a]), dy[k] = (long long)(r.y[b] - r.y[a]);
      tie[k] = tie_inside(sg * dx[k], sg * dy[k]);
    }
    const long long first = (t - __ldg(P + f)) * kChunk;
    const long long end = min(first + kChunk, (long long)r.bw * r.bh);
    for (long long p = first; p < end; ++p) {
      const int py = r.y0 + (int)(p / r.bw), px = r.x0 + (int)(p % r.bw);
      const long long sx = 256ll * px + 128, sy = 256ll * py + 128;
      long long E[3];
      bool inside = true;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int a = (k + 1) % 3;
        E[k] = sg * (dx[k] * (sy - r.y[a]) - dy[k] * (sx - r.x[a]));
        inside = inside && (E[k] > 0 || (E[k] == 0 && tie[k]));
      }
      if (!inside) continue;
      const int64_t pix = (int64_t)py * width + px;
      if (hits) atomicAdd(hits + pix, 1);
      const double b0 = __ddiv_rn(__ll2double_rn(E[0]), Ad), b1 = __ddiv_rn(__ll2double_rn(E[1]), Ad),
                   b2 = __ddiv_rn(__ll2double_rn(E[2]), Ad);
      const double s = __dadd_rn(__dadd_rn(__ddiv_rn(b0, r.z[0]), __ddiv_rn(b1, r.z[1])), __ddiv_rn(b2, r.z[2]));
      const float z = __double2float_rn(__ddiv_rn(1.0, s));
      const double zd = (double)z;
      if (zd >= near && zd <= far)
        atomicMin(keys + pix, ((unsigned long long)__float_as_uint(z) << 32) | (unsigned)f);
    }
  }
}

__global__ void __launch_bounds__(kThreads) resolve_kernel(const unsigned long long* __restrict__ keys, int64_t n,
                                                           float* __restrict__ z, uint8_t* __restrict__ mask,
                                                           int32_t* __restrict__ face) {
  const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i];
  const bool hit = k != kEmptyKey;
  z[i] = hit ? __uint_as_float((unsigned)(k >> 32)) : 0.0f;
  mask[i] = hit ? 255 : 0;
  if (face) face[i] = hit ? (int32_t)(unsigned)k : -1;
}

// ------------------------------------------------------------------------------------------------------- depth scores
struct DSlot {
  double sum[4];                        // sum d, sum |d|, sum d^2, sum |d| / ref
  long long count[kCounts + kMaxTaus];  // n, |P|, |R|, |P and R|, |P or R|, then #{|d| <= tau_i}
};

struct DTaus {
  double t[kMaxTaus];
  int n;
};

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// CTA b reads pixels b * kThreads * kMetricPixels + j * kThreads + threadIdx.x, j = 0 .. kMetricPixels - 1, in that
// order; the warp sums (xor butterfly) and the CTA's eight warps (in order) make its slot.
__global__ void __launch_bounds__(kThreads) metrics_kernel(const float* __restrict__ pred_z,
                                                           const uint8_t* __restrict__ pred_mask,
                                                           const float* __restrict__ ref_z,
                                                           const uint8_t* __restrict__ ref_mask, int64_t n, DTaus taus,
                                                           DSlot* __restrict__ slots, int32_t* __restrict__ error) {
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  int c[kCounts + kMaxTaus];
#pragma unroll
  for (int k = 0; k < kCounts + kMaxTaus; ++k) c[k] = 0;
  unsigned bad = 0;
  const int64_t base = blockIdx.x * (int64_t)(kThreads * kMetricPixels) + threadIdx.x;
#pragma unroll
  for (int j = 0; j < kMetricPixels; ++j) {
    const int64_t i = base + j * kThreads;
    if (i >= n) break;
    const bool pm = pred_mask[i] != 0, rm = ref_mask[i] != 0;
    c[1] += pm, c[2] += rm, c[3] += pm && rm, c[4] += pm || rm;
    if (!(pm && rm)) continue;
    ++c[0];
    const float pz = pred_z[i], rz = ref_z[i];
    const float inf = __int_as_float(0x7f800000);
    if (!(pz > 0.0f && pz < inf && rz > 0.0f && rz < inf)) {
      bad = 1;
      continue;
    }
    const double d = __dsub_rn((double)pz, (double)rz), ad = fabs(d);
    s[0] = __dadd_rn(s[0], d), s[1] = __dadd_rn(s[1], ad), s[2] = __dadd_rn(s[2], __dmul_rn(d, d));
    s[3] = __dadd_rn(s[3], __ddiv_rn(ad, (double)rz));
#pragma unroll
    for (int k = 0; k < kMaxTaus; ++k) c[kCounts + k] += (k < taus.n && ad <= taus.t[k]) ? 1 : 0;
  }
  __shared__ double s_s[kThreads / 32][4];
  __shared__ int s_c[kThreads / 32][kCounts + kMaxTaus];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 4; ++k) s[k] = warp_sum(s[k]);
#pragma unroll
  for (int k = 0; k < kCounts + kMaxTaus; ++k) c[k] = __reduce_add_sync(0xffffffffu, c[k]);
  bad = __reduce_or_sync(0xffffffffu, bad);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) s_s[warp][k] = s[k];
#pragma unroll
    for (int k = 0; k < kCounts + kMaxTaus; ++k) s_c[warp][k] = c[k];
    if (bad) atomicOr(error, 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    DSlot o;
    for (int k = 0; k < 4; ++k) o.sum[k] = 0.0;
    for (int k = 0; k < kCounts + kMaxTaus; ++k) o.count[k] = 0;
    for (int w = 0; w < kThreads / 32; ++w) {
      for (int k = 0; k < 4; ++k) o.sum[k] += s_s[w][k];
      for (int k = 0; k < kCounts + kMaxTaus; ++k) o.count[k] += s_c[w][k];
    }
    slots[blockIdx.x] = o;
  }
}

__global__ void __launch_bounds__(kThreads) metrics_init_kernel(int32_t* __restrict__ error) { *error = 0; }

__global__ void __launch_bounds__(kThreads) metrics_finish_kernel(const DSlot* __restrict__ slots, int num_slots,
                                                                        int num_taus, const int32_t* __restrict__ error,
                                                                        double* __restrict__ out,
                                                                        long long* __restrict__ counts) {
  constexpr int kC = kCounts + kMaxTaus;
  __shared__ double s_s[kThreads / 32][4];
  __shared__ long long s_c[kThreads / 32][kC];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  long long c[kC];
#pragma unroll
  for (int k = 0; k < kC; ++k) c[k] = 0;
  for (int i = tid; i < num_slots; i += kThreads) {
    const DSlot& o = slots[i];
#pragma unroll
    for (int k = 0; k < 4; ++k) s[k] += o.sum[k];
#pragma unroll
    for (int k = 0; k < kC; ++k) c[k] += o.count[k];
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) s[k] = warp_sum(s[k]);
#pragma unroll
  for (int k = 0; k < kC; ++k) c[k] = warp_sum(c[k]);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) s_s[warp][k] = s[k];
#pragma unroll
    for (int k = 0; k < kC; ++k) s_c[warp][k] = c[k];
  }
  __syncthreads();
  if (tid != 0) return;
  double sum[4] = {0.0, 0.0, 0.0, 0.0};
  long long cnt[kC];
#pragma unroll
  for (int k = 0; k < kC; ++k) cnt[k] = 0;
  for (int w = 0; w < kThreads / 32; ++w) {
#pragma unroll
    for (int k = 0; k < 4; ++k) sum[k] += s_s[w][k];
#pragma unroll
    for (int k = 0; k < kC; ++k) cnt[k] += s_c[w][k];
  }
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  const bool valid = *error == 0 && cnt[0] > 0;
  const double nb = (double)cnt[0];
  out[0] = valid ? sum[0] / nb : nan;
  out[1] = valid ? sum[1] / nb : nan;
  out[2] = valid ? sqrt(sum[2] / nb) : nan;
  out[3] = valid ? sum[3] / nb : nan;
#pragma unroll
  for (int k = 0; k < kC; ++k)
    if (k < kCounts + num_taus) counts[k] = cnt[k];
}

template <typename T>
T* carve(char*& p, int64_t count) {
  T* r = reinterpret_cast<T*>(p);
  p += (count * (int64_t)sizeof(T) + 255) & ~int64_t(255);
  return r;
}

struct Layout {
  VRec* vrec;
  FRec* frec;
  long long *chunks, *P;
  unsigned long long* keys;
  void* cub_temp;
  size_t cub_bytes;
  int64_t total;
};

Layout layout(void* base, int64_t nv, int64_t nf, int64_t pixels) {
  char* p = reinterpret_cast<char*>(base);
  Layout l;
  l.vrec = carve<VRec>(p, nv);
  l.frec = carve<FRec>(p, nf);
  l.chunks = carve<long long>(p, nf);
  l.P = carve<long long>(p, nf);
  l.keys = carve<unsigned long long>(p, pixels);
  l.cub_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, l.cub_bytes, (const long long*)nullptr, (long long*)nullptr,
                                (int)std::max<int64_t>(nf, 1));
  l.cub_temp = carve<char>(p, (int64_t)l.cub_bytes);
  l.total = p - reinterpret_cast<char*>(base);
  return l;
}

unsigned blocks(int64_t n) { return (unsigned)std::max<int64_t>((n + kThreads - 1) / kThreads, 1); }

int64_t metric_slots(int64_t n) { return std::max<int64_t>((n + kThreads * kMetricPixels - 1) / (kThreads * kMetricPixels), 1); }

}  // namespace
}  // namespace hrf

using namespace hrf;

extern "C" int64_t hrf_rasterize_mesh_workspace_bytes(int64_t num_vertices, int64_t num_faces, int width, int height) {
  if (num_vertices < 0 || num_faces < 0 || num_faces >= (int64_t)1 << 31 || width < 1 || height < 1 ||
      (int64_t)width * height >= (int64_t)1 << 31)
    return 0;
  return layout(nullptr, num_vertices, num_faces, (int64_t)width * height).total;
}

extern "C" int hrf_rasterize_mesh(const float* vertices, int64_t num_vertices, const int32_t* faces, int64_t num_faces,
                                  const double* world2cam, double fxW, double fyH, double cxW, double cyH, int width,
                                  int height, double near, double far, float* z, uint8_t* mask, int32_t* face,
                                  int32_t* hits, int32_t* error, int64_t* skipped, void* workspace, void* stream) {
  HRF_REQUIRE(world2cam && z && mask && error && skipped && workspace, "null argument");
  HRF_REQUIRE(num_faces >= 0 && num_faces < (int64_t)1 << 31, "face count outside [0, 2^31)");
  HRF_REQUIRE(num_vertices >= 0, "negative vertex count");
  HRF_REQUIRE((vertices || num_vertices == 0) && (faces || num_faces == 0), "null mesh array");
  HRF_REQUIRE(width >= 1 && height >= 1 && (int64_t)width * height < (int64_t)1 << 31,
              "image size must be at least 1x1 and below 2^31 pixels");
  HRF_REQUIRE(near > 0.0 && far >= near && far <= 1.7976931348623157e308, "need 0 < near <= far < inf");
  HRF_REQUIRE(reinterpret_cast<uintptr_t>(workspace) % 256 == 0, "workspace must be 256-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int nf = (int)num_faces;
  const int64_t pixels = (int64_t)width * height;
  Layout l = layout(workspace, num_vertices, nf, pixels);
  Proj pr;
  for (int k = 0; k < 12; ++k) pr.m[k] = world2cam[k];
  pr.fx = fxW, pr.fy = fyH, pr.cx = cxW, pr.cy = cyH, pr.near = near;

  init_kernel<<<blocks(pixels), kThreads, 0, st>>>(l.keys, pixels, hits, error, reinterpret_cast<long long*>(skipped));
  HRF_CHECK_LAUNCH();
  if (num_vertices > 0) {
    vertex_kernel<<<blocks(num_vertices), kThreads, 0, st>>>(vertices, num_vertices, pr, l.vrec);
    HRF_CHECK_LAUNCH();
  }
  if (nf > 0) {
    setup_kernel<<<blocks(nf), kThreads, 0, st>>>(faces, nf, num_vertices, l.vrec, width, height, l.frec, l.chunks,
                                                  error, reinterpret_cast<long long*>(skipped));
    HRF_CHECK_LAUNCH();
    size_t bytes = l.cub_bytes;
    HRF_CUDA(cub::DeviceScan::ExclusiveSum(l.cub_temp, bytes, l.chunks, l.P, nf, st));
    raster_kernel<<<(unsigned)(sm_count() * kRasterCtasPerSm), kThreads, 0, st>>>(l.frec, l.P, l.chunks, nf, width,
                                                                                   near, far, l.keys, hits);
    HRF_CHECK_LAUNCH();
  }
  resolve_kernel<<<blocks(pixels), kThreads, 0, st>>>(l.keys, pixels, z, mask, face);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int64_t hrf_depth_metrics_workspace_bytes(int64_t num_pixels) {
  if (num_pixels < 1 || num_pixels >= (int64_t)1 << 31) return 0;
  return metric_slots(num_pixels) * (int64_t)sizeof(DSlot);
}

extern "C" int hrf_depth_metrics(const float* pred_z, const uint8_t* pred_mask, const float* ref_z,
                                 const uint8_t* ref_mask, int64_t num_pixels, const double* taus, int num_taus,
                                 double* out, int64_t* counts, int32_t* error, void* workspace, void* stream) {
  HRF_REQUIRE(pred_z && pred_mask && ref_z && ref_mask && out && counts && error && workspace, "null argument");
  HRF_REQUIRE(num_pixels >= 1 && num_pixels < (int64_t)1 << 31, "pixel count outside [1, 2^31)");
  HRF_REQUIRE(num_taus >= 0 && num_taus <= kMaxTaus && (taus || num_taus == 0), "at most 8 thresholds");
  HRF_REQUIRE(reinterpret_cast<uintptr_t>(workspace) % 16 == 0, "workspace must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  DTaus tv{};
  tv.n = num_taus;
  for (int k = 0; k < num_taus; ++k) tv.t[k] = taus[k];
  const int num_slots = (int)metric_slots(num_pixels);
  DSlot* slots = reinterpret_cast<DSlot*>(workspace);
  metrics_init_kernel<<<1, 1, 0, st>>>(error);
  HRF_CHECK_LAUNCH();
  metrics_kernel<<<num_slots, kThreads, 0, st>>>(pred_z, pred_mask, ref_z, ref_mask, num_pixels, tv, slots, error);
  HRF_CHECK_LAUNCH();
  metrics_finish_kernel<<<1, kThreads, 0, st>>>(slots, num_slots, num_taus, error, out,
                                                      reinterpret_cast<long long*>(counts));
  HRF_CHECK_LAUNCH();
  return 0;
}
