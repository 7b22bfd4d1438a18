// Surface distances between two triangle meshes, one direction per call: points sampled on a source mesh S by area,
// each queried against a target mesh T for the closest point on its surface.  Contract: include/humanrf_b200.h,
// hrf_mesh_distance; DESIGN.md §3.11.  Launches, in stream order, none synchronising with the host:
//   init_kernel          : zero the header (area maxima, centroid box, error word);
//   prep_kernel (S, T)   : one thread per face: index check, area vector n, eligibility, unit normal, area; the largest
//                          area and (T) the centroid box are raised with integer atomics (order-independent);
//   weight_kernel (S)    : q_f = floor(area_f / area_max * 2^32) as uint64, then a CUB exclusive sum gives P;
//   sample_kernel        : one thread per sample: splitmix64 draws, binary search in P, barycentric point; sort keys
//                          (face << 32 | k), sorted by CUB so that neighbouring queries start on neighbouring faces;
//   morton_kernel (T)    : (30-bit Morton code of the centroid << 32) | face id, sorted by CUB;
//   leaf_kernel (T)      : gathers 4 consecutive sorted triangles per leaf and their box; refit_kernel: one tree level
//                          per launch, bottom-up;
//   query_kernel         : one thread per sample: stack traversal of the implicit tree, nearer child first, exact
//                          tie rule; per-sample outputs and fp64 / int64 per-CTA partial sums;
//   finish_kernel        : one CTA folds the partial sums in a fixed order.
// Every fold is in a fixed order and the only atomics are integer max / min / or: two calls write identical bytes.
#include <algorithm>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace hrf {
namespace {

constexpr int kThreads = 256;
constexpr int kFinishThreads = 1024;
constexpr int kMaxTaus = 8;
constexpr int kLeafSize = 4;
constexpr int kStack = 32;                              // tree depth <= 29 for F < 2^31
constexpr uint64_t kNoFaceKey = (1ull << 62) - 1;       // sorts after every eligible key (morton < 2^30, id < 2^31)
constexpr int kKeyBits = 62;

struct Header {
  uint32_t amax_bits[2];   // largest eligible area of S (0) and T (1), as float bits (positive floats order as ints)
  uint32_t box[6];         // T's centroid box: ordered-int min x, y, z (init ~0), max x, y, z (init 0)
};

struct Slot {
  double sum_d, sum_d2, sum_n;
  long long count[kMaxTaus];
};

struct Taus {
  float t[kMaxTaus];
  int n;
};

__device__ __forceinline__ uint32_t ordered(float x) {
  const uint32_t u = __float_as_uint(x);
  return u ^ ((u >> 31) ? 0xffffffffu : 0x80000000u);
}
__device__ __forceinline__ float unordered(uint32_t e) {
  return __uint_as_float(e ^ ((e >> 31) ? 0x80000000u : 0xffffffffu));
}

__device__ __forceinline__ float3 sub3(float3 a, float3 b) {
  return make_float3(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z));
}
// ((x.x y.x + x.y y.y) + x.z y.z), every product and sum rounded on its own
__device__ __forceinline__ float dot3(float3 a, float3 b) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z));
}
// a + s b per component
__device__ __forceinline__ float3 axpy3(float3 a, float s, float3 b) {
  return make_float3(__fadd_rn(a.x, __fmul_rn(s, b.x)), __fadd_rn(a.y, __fmul_rn(s, b.y)),
                     __fadd_rn(a.z, __fmul_rn(s, b.z)));
}
// xy - zw
__device__ __forceinline__ float det2(float x, float y, float z, float w) {
  return __fsub_rn(__fmul_rn(x, y), __fmul_rn(z, w));
}

__device__ __forceinline__ float3 load_vertex(const float* __restrict__ v, int i) {
  return make_float3(__ldg(v + 3 * (int64_t)i), __ldg(v + 3 * (int64_t)i + 1), __ldg(v + 3 * (int64_t)i + 2));
}

// Squared distance from p to triangle abc: Ericson, Real-Time Collision Detection §5.1.5 (Voronoi regions of the three
// vertices, three edges and the face, tested in that book's order), in fp32 with every operation rounded on its own;
// the closest point is then clamped per component into the triangle's bounding box (a no-op in exact arithmetic, and
// it keeps q finite and inside the box the tree's bounds cover).  tests/geometry_oracle.py restates it op for op.
__device__ __forceinline__ float point_triangle_d2(float3 p, float3 a, float3 b, float3 c) {
  const float3 ab = sub3(b, a), ac = sub3(c, a), ap = sub3(p, a);
  const float d1 = dot3(ab, ap), d2 = dot3(ac, ap);
  float3 q;
  if (d1 <= 0.0f && d2 <= 0.0f) {
    q = a;
  } else {
    const float3 bp = sub3(p, b);
    const float d3 = dot3(ab, bp), d4 = dot3(ac, bp);
    if (d3 >= 0.0f && d4 <= d3) {
      q = b;
    } else {
      const float vc = det2(d1, d4, d3, d2);
      if (vc <= 0.0f && d1 >= 0.0f && d3 <= 0.0f) {
        q = axpy3(a, __fdiv_rn(d1, __fsub_rn(d1, d3)), ab);
      } else {
        const float3 cp = sub3(p, c);
        const float d5 = dot3(ab, cp), d6 = dot3(ac, cp);
        if (d6 >= 0.0f && d5 <= d6) {
          q = c;
        } else {
          const float vb = det2(d5, d2, d1, d6);
          if (vb <= 0.0f && d2 >= 0.0f && d6 <= 0.0f) {
            q = axpy3(a, __fdiv_rn(d2, __fsub_rn(d2, d6)), ac);
          } else {
            const float va = det2(d3, d6, d5, d4);
            const float e43 = __fsub_rn(d4, d3), e56 = __fsub_rn(d5, d6);
            if (va <= 0.0f && e43 >= 0.0f && e56 >= 0.0f) {
              q = axpy3(b, __fdiv_rn(e43, __fadd_rn(e43, e56)), sub3(c, b));
            } else {
              const float denom = __fdiv_rn(1.0f, __fadd_rn(__fadd_rn(va, vb), vc));
              q = axpy3(axpy3(a, __fmul_rn(vb, denom), ab), __fmul_rn(vc, denom), ac);
            }
          }
        }
      }
    }
  }
  // fmaxf / fminf return the non-NaN operand, so a NaN coordinate becomes the box's bound
  q.x = fminf(fmaxf(q.x, fminf(fminf(a.x, b.x), c.x)), fmaxf(fmaxf(a.x, b.x), c.x));
  q.y = fminf(fmaxf(q.y, fminf(fminf(a.y, b.y), c.y)), fmaxf(fmaxf(a.y, b.y), c.y));
  q.z = fminf(fmaxf(q.z, fminf(fminf(a.z, b.z), c.z)), fmaxf(fmaxf(a.z, b.z), c.z));
  const float3 e = sub3(p, q);
  return dot3(e, e);
}

// A lower bound on point_triangle_d2(p, .) for every triangle inside the box [lo, hi]: the box distance with every
// operation rounded down, less the rounding of point_triangle_d2's own subtraction and dot product (a relative 5 * 2^-24,
// covered by 2^-20, and an absolute 1e-30 for underflow).  An empty box (lo = +inf) gives +inf.
__device__ __forceinline__ float box_lower_bound(float3 p, float4 lo, float4 hi) {
  const float gx = fmaxf(fmaxf(__fsub_rd(lo.x, p.x), __fsub_rd(p.x, hi.x)), 0.0f);
  const float gy = fmaxf(fmaxf(__fsub_rd(lo.y, p.y), __fsub_rd(p.y, hi.y)), 0.0f);
  const float gz = fmaxf(fmaxf(__fsub_rd(lo.z, p.z), __fsub_rd(p.z, hi.z)), 0.0f);
  const float s = __fadd_rd(__fadd_rd(__fmul_rd(gx, gx), __fmul_rd(gy, gy)), __fmul_rd(gz, gz));
  return __fsub_rd(__fmul_rd(s, 0.99999904632568359375f), 1e-30f);
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void init_kernel(Header* __restrict__ h, int32_t* __restrict__ error) {
  const int t = threadIdx.x;
  if (t < 2) h->amax_bits[t] = 0;
  if (t < 3) h->box[t] = 0xffffffffu, h->box[3 + t] = 0;
  if (t == 0) *error = 0;
}

// One thread per face.  info[f] = (n / |n|, area) for an eligible face (0 < |n|^2 < inf, indices in [0, V)), all zero
// otherwise.  With box != nullptr (the target) the eligible centroids' box is raised too.
__global__ void __launch_bounds__(kThreads) prep_kernel(const float* __restrict__ verts, int64_t nv,
                                                        const int32_t* __restrict__ faces, int nf,
                                                        float4* __restrict__ info, uint32_t* __restrict__ amax_bits,
                                                        int32_t* __restrict__ error, int error_bit,
                                                        uint32_t* __restrict__ box) {
  const int f = blockIdx.x * kThreads + threadIdx.x;
  uint32_t amax = 0, bad = 0;
  uint32_t bmin[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, bmax[3] = {0, 0, 0};
  if (f < nf) {
    const int i0 = __ldg(faces + 3 * (int64_t)f), i1 = __ldg(faces + 3 * (int64_t)f + 1),
              i2 = __ldg(faces + 3 * (int64_t)f + 2);
    float4 o = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (i0 < 0 || i1 < 0 || i2 < 0 || i0 >= nv || i1 >= nv || i2 >= nv) {
      bad = 1;
    } else {
      const float3 a = load_vertex(verts, i0), b = load_vertex(verts, i1), c = load_vertex(verts, i2);
      const float3 e1 = sub3(b, a), e2 = sub3(c, a);
      const float3 n = make_float3(det2(e1.y, e2.z, e1.z, e2.y), det2(e1.z, e2.x, e1.x, e2.z),
                                   det2(e1.x, e2.y, e1.y, e2.x));
      const float nn = dot3(n, n);
      if (nn > 0.0f && nn < __int_as_float(0x7f800000)) {
        const float len = __fsqrt_rn(nn);
        o = make_float4(__fdiv_rn(n.x, len), __fdiv_rn(n.y, len), __fdiv_rn(n.z, len), __fmul_rn(0.5f, len));
        amax = __float_as_uint(o.w);
        if (box) {
          const float cx = __fadd_rn(__fadd_rn(a.x, b.x), c.x), cy = __fadd_rn(__fadd_rn(a.y, b.y), c.y),
                      cz = __fadd_rn(__fadd_rn(a.z, b.z), c.z);
          bmin[0] = bmax[0] = ordered(cx), bmin[1] = bmax[1] = ordered(cy), bmin[2] = bmax[2] = ordered(cz);
        }
      }
    }
    info[f] = o;
  }
  amax = __reduce_max_sync(0xffffffffu, amax);
  bad = __reduce_or_sync(0xffffffffu, bad);
  if ((threadIdx.x & 31) == 0) {
    if (amax) atomicMax(amax_bits, amax);
    if (bad) atomicOr(error, error_bit);
  }
  if (box) {
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      bmin[q] = __reduce_min_sync(0xffffffffu, bmin[q]);
      bmax[q] = __reduce_max_sync(0xffffffffu, bmax[q]);
    }
    if ((threadIdx.x & 31) == 0 && bmax[0]) {
#pragma unroll
      for (int q = 0; q < 3; ++q) atomicMin(box + q, bmin[q]), atomicMax(box + 3 + q, bmax[q]);
    }
  }
}

// q_f = floor(area_f / area_max * 2^32) with the division in fp64 (exact multiply by 2^32); 0 for ineligible faces.
__global__ void __launch_bounds__(kThreads) weight_kernel(const float4* __restrict__ info, int nf,
                                                          const uint32_t* __restrict__ amax_bits,
                                                          uint64_t* __restrict__ q) {
  const int f = blockIdx.x * kThreads + threadIdx.x;
  if (f >= nf) return;
  const float area = info[f].w;
  const double amax = (double)__uint_as_float(*amax_bits);
  q[f] = area > 0.0f ? (uint64_t)floor(__dmul_rn(__ddiv_rn((double)area, amax), 4294967296.0)) : 0ull;
}

__device__ __forceinline__ uint64_t total_weight(const uint64_t* __restrict__ P, const uint64_t* __restrict__ q, int nf) {
  return nf > 0 ? P[nf - 1] + q[nf - 1] : 0ull;
}

// One thread per sample k: x_j = splitmix64(seed * 2^40 + 3k + j); face f with P_f <= mulhi(x_0, Q) < P_f + q_f;
// u1, u2 = top 24 bits of x_1, x_2 times 2^-24; r = sqrt(u1); p = (1 - r) v0 + r (1 - u2) v1 + (r u2) v2.
__global__ void __launch_bounds__(kThreads) sample_kernel(const float* __restrict__ verts,
                                                          const int32_t* __restrict__ faces, int nf,
                                                          const uint64_t* __restrict__ P,
                                                          const uint64_t* __restrict__ q, int n, uint64_t seed,
                                                          float4* __restrict__ samples, uint64_t* __restrict__ keys,
                                                          float* __restrict__ points_out,
                                                          int32_t* __restrict__ faces_out) {
  const int k = blockIdx.x * kThreads + threadIdx.x;
  if (k >= n) return;
  const uint64_t Q = total_weight(P, q, nf);
  float4 s;
  int face = -1;
  if (Q == 0) {
    const float nan = __int_as_float(0x7fc00000);
    s = make_float4(nan, nan, nan, __int_as_float(-1));
  } else {
    const uint64_t base = seed * (1ull << 40) + 3ull * (uint64_t)k;
    const uint64_t x0 = splitmix64(base), x1 = splitmix64(base + 1), x2 = splitmix64(base + 2);
    const uint64_t t = __umul64hi(x0, Q);
    int lo = 0, hi = nf;                   // P[lo] <= t, and P[hi] > t or hi = nf
    while (hi - lo > 1) {
      const int mid = lo + ((hi - lo) >> 1);
      if (P[mid] <= t) lo = mid; else hi = mid;
    }
    face = lo;
    const float u1 = __fmul_rn((float)(uint32_t)(x1 >> 40), 5.9604644775390625e-8f);
    const float u2 = __fmul_rn((float)(uint32_t)(x2 >> 40), 5.9604644775390625e-8f);
    const float r = __fsqrt_rn(u1);
    const float w0 = __fsub_rn(1.0f, r), w1 = __fmul_rn(r, __fsub_rn(1.0f, u2)), w2 = __fmul_rn(r, u2);
    const float3 a = load_vertex(verts, __ldg(faces + 3 * (int64_t)face)),
                 b = load_vertex(verts, __ldg(faces + 3 * (int64_t)face + 1)),
                 c = load_vertex(verts, __ldg(faces + 3 * (int64_t)face + 2));
    s = make_float4(__fadd_rn(__fadd_rn(__fmul_rn(w0, a.x), __fmul_rn(w1, b.x)), __fmul_rn(w2, c.x)),
                    __fadd_rn(__fadd_rn(__fmul_rn(w0, a.y), __fmul_rn(w1, b.y)), __fmul_rn(w2, c.y)),
                    __fadd_rn(__fadd_rn(__fmul_rn(w0, a.z), __fmul_rn(w1, b.z)), __fmul_rn(w2, c.z)),
                    __int_as_float(face));
  }
  samples[k] = s;
  keys[k] = ((uint64_t)(uint32_t)face << 32) | (uint32_t)k;      // Q = 0: face -1 sorts last, order unchanged
  if (points_out) points_out[3 * (int64_t)k] = s.x, points_out[3 * (int64_t)k + 1] = s.y, points_out[3 * (int64_t)k + 2] = s.z;
  if (faces_out) faces_out[k] = face;
}

__device__ __forceinline__ uint32_t spread10(uint32_t x) {     // 10 bits -> every third of 30
  x &= 0x3ffu;
  x = (x | (x << 16)) & 0x030000ffu;
  x = (x | (x << 8)) & 0x0300f00fu;
  x = (x | (x << 4)) & 0x030c30c3u;
  x = (x | (x << 2)) & 0x09249249u;
  return x;
}

// Key of face f: (Morton code of its centroid in the centroid box, 10 bits per axis) << 32 | f; kNoFaceKey when
// ineligible.  The codes only order the leaves: any order gives the same query results.
__global__ void __launch_bounds__(kThreads) morton_kernel(const float* __restrict__ verts,
                                                          const int32_t* __restrict__ faces, int nf,
                                                          const float4* __restrict__ info,
                                                          const uint32_t* __restrict__ box, uint64_t* __restrict__ keys) {
  const int f = blockIdx.x * kThreads + threadIdx.x;
  if (f >= nf) return;
  if (!(info[f].w > 0.0f)) {
    keys[f] = kNoFaceKey;
    return;
  }
  const float3 a = load_vertex(verts, __ldg(faces + 3 * (int64_t)f)), b = load_vertex(verts, __ldg(faces + 3 * (int64_t)f + 1)),
               c = load_vertex(verts, __ldg(faces + 3 * (int64_t)f + 2));
  const float cen[3] = {__fadd_rn(__fadd_rn(a.x, b.x), c.x), __fadd_rn(__fadd_rn(a.y, b.y), c.y),
                        __fadd_rn(__fadd_rn(a.z, b.z), c.z)};
  uint32_t code = 0;
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const float lo = unordered(box[q]), hi = unordered(box[3 + q]);
    const float ext = hi - lo;
    const float u = ext > 0.0f ? fminf(fmaxf((cen[q] - lo) / ext, 0.0f), 1.0f) : 0.0f;
    code |= spread10((uint32_t)(u * 1023.0f)) << (2 - q);
  }
  keys[f] = ((uint64_t)code << 32) | (uint32_t)f;
}

// One thread per leaf j of the Lp: sorted slots 4j .. 4j+3 (those < nf) are gathered as 3 float4 each, (a, face id),
// (b, 0), (c, 0), face id -1 for a slot without an eligible face; the leaf's box is written at node Lp + j.
__global__ void __launch_bounds__(kThreads) leaf_kernel(const float* __restrict__ verts,
                                                        const int32_t* __restrict__ faces, int nf,
                                                        const uint64_t* __restrict__ sorted, int num_leaves,
                                                        float4* __restrict__ tris, float4* __restrict__ node_lo,
                                                        float4* __restrict__ node_hi) {
  const int j = blockIdx.x * kThreads + threadIdx.x;
  if (j >= num_leaves) return;
  const float inf = __int_as_float(0x7f800000);
  float4 lo = make_float4(inf, inf, inf, 0.0f), hi = make_float4(-inf, -inf, -inf, 0.0f);
#pragma unroll
  for (int s = kLeafSize * j; s < kLeafSize * j + kLeafSize; ++s) {
    if (s >= nf) break;
    const uint64_t key = sorted[s];
    if (key == kNoFaceKey) {
      tris[3 * (int64_t)s] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(-1));
      continue;
    }
    const int f = (int)(uint32_t)key;
    const float3 v[3] = {load_vertex(verts, __ldg(faces + 3 * (int64_t)f)), load_vertex(verts, __ldg(faces + 3 * (int64_t)f + 1)),
                         load_vertex(verts, __ldg(faces + 3 * (int64_t)f + 2))};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      tris[3 * (int64_t)s + i] = make_float4(v[i].x, v[i].y, v[i].z, i == 0 ? __int_as_float(f) : 0.0f);
      lo.x = fminf(lo.x, v[i].x), lo.y = fminf(lo.y, v[i].y), lo.z = fminf(lo.z, v[i].z);
      hi.x = fmaxf(hi.x, v[i].x), hi.y = fmaxf(hi.y, v[i].y), hi.z = fmaxf(hi.z, v[i].z);
    }
  }
  node_lo[num_leaves + j] = lo;
  node_hi[num_leaves + j] = hi;
}

// Nodes [first, 2 first) of the heap-ordered tree (children of i at 2i, 2i + 1): the union of the children's boxes.
__global__ void __launch_bounds__(kThreads) refit_kernel(int first, float4* __restrict__ node_lo,
                                                         float4* __restrict__ node_hi) {
  const int i = first + blockIdx.x * kThreads + threadIdx.x;
  if (i >= 2 * first) return;
  const float4 l0 = node_lo[2 * i], l1 = node_lo[2 * i + 1], h0 = node_hi[2 * i], h1 = node_hi[2 * i + 1];
  node_lo[i] = make_float4(fminf(l0.x, l1.x), fminf(l0.y, l1.y), fminf(l0.z, l1.z), 0.0f);
  node_hi[i] = make_float4(fmaxf(h0.x, h1.x), fmaxf(h0.y, h1.y), fmaxf(h0.z, h1.z), 0.0f);
}

// One thread per sample, in the order of the sorted (face, k) keys.  best = min over eligible target faces of
// point_triangle_d2, ties to the lowest face id; a node is skipped only when its lower bound is strictly above best.
__global__ void __launch_bounds__(kThreads) query_kernel(const float4* __restrict__ samples,
                                                         const uint64_t* __restrict__ order, int n,
                                                         const float4* __restrict__ src_info,
                                                         const float4* __restrict__ tgt_info,
                                                         const float4* __restrict__ tris, int nf_tgt,
                                                         const float4* __restrict__ node_lo,
                                                         const float4* __restrict__ node_hi, int num_leaves,
                                                         const uint32_t* __restrict__ tgt_amax_bits, Taus taus,
                                                         Slot* __restrict__ slots, float* __restrict__ dist_out,
                                                         int32_t* __restrict__ closest_out) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  double sd = 0.0, sd2 = 0.0, sn = 0.0;
  int cnt[kMaxTaus];
#pragma unroll
  for (int t = 0; t < kMaxTaus; ++t) cnt[t] = 0;
  if (i < n) {
    const int k = (int)(uint32_t)order[i];
    const float4 s = samples[k];
    const int src_face = __float_as_int(s.w);
    float d = __int_as_float(0x7fc00000);
    int best_id = -1;
    if (src_face >= 0 && *tgt_amax_bits != 0) {      // a target without eligible faces: nothing to visit
      const float3 p = make_float3(s.x, s.y, s.z);
      float best = __int_as_float(0x7f800000);
      int bid = 0x7fffffff;
      int stack[kStack];
      float stack_lb[kStack];
      int sp = 0;
      stack[sp] = 1, stack_lb[sp] = 0.0f, ++sp;
      while (sp > 0) {
        --sp;
        const int node = stack[sp];
        if (stack_lb[sp] > best) continue;
        if (node >= num_leaves) {
          const int s0 = kLeafSize * (node - num_leaves);
#pragma unroll
          for (int j = 0; j < kLeafSize; ++j) {
            if (s0 + j >= nf_tgt) break;
            const float4 ta = __ldg(tris + 3 * (int64_t)(s0 + j));
            const int f = __float_as_int(ta.w);
            if (f < 0) break;                               // ineligible slots sort after every eligible one
            const float4 tb = __ldg(tris + 3 * (int64_t)(s0 + j) + 1), tc = __ldg(tris + 3 * (int64_t)(s0 + j) + 2);
            const float d2 = point_triangle_d2(p, make_float3(ta.x, ta.y, ta.z), make_float3(tb.x, tb.y, tb.z),
                                               make_float3(tc.x, tc.y, tc.z));
            if (d2 < best || (d2 == best && f < bid)) best = d2, bid = f;
          }
        } else {
          const int c0 = 2 * node;
          const float lb0 = box_lower_bound(p, __ldg(node_lo + c0), __ldg(node_hi + c0));
          const float lb1 = box_lower_bound(p, __ldg(node_lo + c0 + 1), __ldg(node_hi + c0 + 1));
          const bool first0 = lb0 <= lb1;
          const int near = first0 ? c0 : c0 + 1, far = first0 ? c0 + 1 : c0;
          const float lbn = first0 ? lb0 : lb1, lbf = first0 ? lb1 : lb0;
          if (!(lbf > best)) stack[sp] = far, stack_lb[sp] = lbf, ++sp;
          if (!(lbn > best)) stack[sp] = near, stack_lb[sp] = lbn, ++sp;
        }
      }
      d = __fsqrt_rn(best);
      if (bid != 0x7fffffff) {
        best_id = bid;
        const float4 ns = src_info[src_face], nt = tgt_info[bid];
        const float nterm = fabsf(__fadd_rn(__fadd_rn(__fmul_rn(ns.x, nt.x), __fmul_rn(ns.y, nt.y)),
                                            __fmul_rn(ns.z, nt.z)));
        sd = (double)d, sd2 = (double)d * (double)d, sn = (double)nterm;
#pragma unroll
        for (int t = 0; t < kMaxTaus; ++t) cnt[t] = (t < taus.n && d <= taus.t[t]) ? 1 : 0;
      }
    }
    if (dist_out) dist_out[k] = d;
    if (closest_out) closest_out[k] = best_id;
  }
  // fixed-order CTA reduction into the CTA's slot
  __shared__ double s_d[kThreads / 32][3];
  __shared__ int s_c[kThreads / 32][kMaxTaus];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  sd = warp_sum(sd), sd2 = warp_sum(sd2), sn = warp_sum(sn);
#pragma unroll
  for (int t = 0; t < kMaxTaus; ++t) cnt[t] = __reduce_add_sync(0xffffffffu, cnt[t]);
  if (lane == 0) {
    s_d[warp][0] = sd, s_d[warp][1] = sd2, s_d[warp][2] = sn;
#pragma unroll
    for (int t = 0; t < kMaxTaus; ++t) s_c[warp][t] = cnt[t];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    Slot o{0.0, 0.0, 0.0, {0, 0, 0, 0, 0, 0, 0, 0}};
    for (int w = 0; w < kThreads / 32; ++w) {
      o.sum_d += s_d[w][0], o.sum_d2 += s_d[w][1], o.sum_n += s_d[w][2];
      for (int t = 0; t < kMaxTaus; ++t) o.count[t] += s_c[w][t];
    }
    slots[blockIdx.x] = o;
  }
}

__global__ void __launch_bounds__(kFinishThreads) finish_kernel(const Slot* __restrict__ slots, int num_slots, int n,
                                                                int num_taus, const uint64_t* __restrict__ P_src,
                                                                const uint64_t* __restrict__ q_src, int nf_src,
                                                                const uint32_t* __restrict__ amax_bits,
                                                                const int32_t* __restrict__ error,
                                                                double* __restrict__ out, long long* __restrict__ counts) {
  __shared__ double s_d[kFinishThreads / 32][3];
  __shared__ long long s_c[kFinishThreads / 32][kMaxTaus];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double d[3] = {0.0, 0.0, 0.0};
  long long c[kMaxTaus];
#pragma unroll
  for (int t = 0; t < kMaxTaus; ++t) c[t] = 0;
  for (int i = tid; i < num_slots; i += kFinishThreads) {
    const Slot& s = slots[i];
    d[0] += s.sum_d, d[1] += s.sum_d2, d[2] += s.sum_n;
#pragma unroll
    for (int t = 0; t < kMaxTaus; ++t) c[t] += s.count[t];
  }
#pragma unroll
  for (int q = 0; q < 3; ++q) d[q] = warp_sum(d[q]);
#pragma unroll
  for (int t = 0; t < kMaxTaus; ++t) c[t] = warp_sum(c[t]);
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < 3; ++q) s_d[warp][q] = d[q];
#pragma unroll
    for (int t = 0; t < kMaxTaus; ++t) s_c[warp][t] = c[t];
  }
  __syncthreads();
  if (tid != 0) return;
  double sum[3] = {0.0, 0.0, 0.0};
  long long cnt[kMaxTaus] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int w = 0; w < kFinishThreads / 32; ++w) {
    for (int q = 0; q < 3; ++q) sum[q] += s_d[w][q];
    for (int t = 0; t < kMaxTaus; ++t) cnt[t] += s_c[w][t];
  }
  // a target without eligible faces leaves amax_bits[1] at 0
  const bool valid = *error == 0 && total_weight(P_src, q_src, nf_src) != 0 && amax_bits[1] != 0;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  for (int q = 0; q < 3; ++q) out[q] = valid ? sum[q] / (double)n : nan;
  for (int t = 0; t < num_taus; ++t) counts[t] = valid ? cnt[t] : -1;
}

template <typename T>
T* carve(char*& p, int64_t count) {
  T* r = reinterpret_cast<T*>(p);
  p += (count * (int64_t)sizeof(T) + 255) & ~int64_t(255);
  return r;
}

int num_leaves_of(int64_t nf) {            // power of two >= ceil(nf / 4), at least 1
  int64_t l = 1;
  while (l * kLeafSize < nf) l <<= 1;
  return (int)l;
}

size_t cub_temp_bytes(int64_t nf_src, int64_t nf_tgt, int64_t n) {
  size_t scan = 0, sort_t = 0, sort_n = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, scan, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)std::max<int64_t>(nf_src, 1));
  cub::DeviceRadixSort::SortKeys(nullptr, sort_t, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                 (int)std::max<int64_t>(nf_tgt, 1), 0, kKeyBits);
  cub::DeviceRadixSort::SortKeys(nullptr, sort_n, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                 (int)std::max<int64_t>(n, 1), 0, 64);
  return std::max(scan, std::max(sort_t, sort_n));
}

struct Layout {
  Header* header;
  float4* src_info;
  uint64_t *q, *P;
  float4* tgt_info;
  uint64_t *keys_in, *keys_out;
  float4* tris;
  float4 *node_lo, *node_hi;
  float4* samples;
  uint64_t *order_in, *order_out;
  Slot* slots;
  void* cub_temp;
  size_t cub_bytes;
  int64_t total;
};

Layout layout(void* base, int64_t nf_src, int64_t nf_tgt, int64_t n) {
  char* p = reinterpret_cast<char*>(base);
  Layout l;
  const int leaves = num_leaves_of(nf_tgt);
  l.header = carve<Header>(p, 1);
  l.src_info = carve<float4>(p, nf_src);
  l.q = carve<uint64_t>(p, nf_src);
  l.P = carve<uint64_t>(p, nf_src);
  l.tgt_info = carve<float4>(p, nf_tgt);
  l.keys_in = carve<uint64_t>(p, nf_tgt);
  l.keys_out = carve<uint64_t>(p, nf_tgt);
  l.tris = carve<float4>(p, 3 * nf_tgt);
  l.node_lo = carve<float4>(p, 2 * (int64_t)leaves);
  l.node_hi = carve<float4>(p, 2 * (int64_t)leaves);
  l.samples = carve<float4>(p, n);
  l.order_in = carve<uint64_t>(p, n);
  l.order_out = carve<uint64_t>(p, n);
  l.slots = carve<Slot>(p, (n + kThreads - 1) / kThreads);
  l.cub_bytes = cub_temp_bytes(nf_src, nf_tgt, n);
  l.cub_temp = carve<char>(p, (int64_t)l.cub_bytes);
  l.total = p - reinterpret_cast<char*>(base);
  return l;
}

unsigned blocks(int64_t n) { return (unsigned)std::max<int64_t>((n + kThreads - 1) / kThreads, 1); }

}  // namespace
}  // namespace hrf

using namespace hrf;

extern "C" int64_t hrf_mesh_distance_workspace_bytes(int64_t num_src_faces, int64_t num_tgt_faces, int64_t num_samples,
                                                     int num_taus) {
  if (num_src_faces < 0 || num_tgt_faces < 0 || num_src_faces >= (int64_t)1 << 31 ||
      num_tgt_faces >= (int64_t)1 << 31 || num_samples < 1 || num_samples >= (int64_t)1 << 31 || num_taus < 0 ||
      num_taus > kMaxTaus)
    return 0;
  return layout(nullptr, num_src_faces, num_tgt_faces, num_samples).total;
}

extern "C" int hrf_mesh_distance(const float* src_vertices, int64_t num_src_vertices, const int32_t* src_faces,
                                 int64_t num_src_faces, const float* tgt_vertices, int64_t num_tgt_vertices,
                                 const int32_t* tgt_faces, int64_t num_tgt_faces, int64_t num_samples, uint64_t seed,
                                 const float* taus, int num_taus, double* out, int64_t* counts, int32_t* error,
                                 float* points, int32_t* sample_faces, float* distances, int32_t* closest_faces,
                                 void* workspace, void* stream) {
  HRF_REQUIRE(out && error && workspace, "null argument");
  HRF_REQUIRE(num_src_faces >= 0 && num_src_faces < (int64_t)1 << 31 && num_tgt_faces >= 0 &&
                  num_tgt_faces < (int64_t)1 << 31, "face count outside [0, 2^31)");
  HRF_REQUIRE(num_samples >= 1 && num_samples < (int64_t)1 << 31, "sample count outside [1, 2^31)");
  HRF_REQUIRE(num_src_vertices >= 0 && num_tgt_vertices >= 0, "negative vertex count");
  HRF_REQUIRE((src_vertices || num_src_vertices == 0) && (src_faces || num_src_faces == 0) &&
                  (tgt_vertices || num_tgt_vertices == 0) && (tgt_faces || num_tgt_faces == 0), "null mesh array");
  HRF_REQUIRE(num_taus >= 0 && num_taus <= kMaxTaus && (taus || num_taus == 0) && (counts || num_taus == 0),
              "at most 8 thresholds");
  HRF_REQUIRE(reinterpret_cast<uintptr_t>(workspace) % 256 == 0, "workspace must be 256-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int fs = (int)num_src_faces, ft = (int)num_tgt_faces, n = (int)num_samples;
  Layout l = layout(workspace, fs, ft, n);
  Taus tv{};
  tv.n = num_taus;
  for (int t = 0; t < num_taus; ++t) tv.t[t] = taus[t];
  const int leaves = num_leaves_of(ft);

  init_kernel<<<1, 32, 0, st>>>(l.header, error);
  HRF_CHECK_LAUNCH();
  // source: eligibility, weights, CDF, samples, sorted query order
  if (fs > 0) {
    prep_kernel<<<blocks(fs), kThreads, 0, st>>>(src_vertices, num_src_vertices, src_faces, fs, l.src_info,
                                                 &l.header->amax_bits[0], error, 1, nullptr);
    HRF_CHECK_LAUNCH();
    weight_kernel<<<blocks(fs), kThreads, 0, st>>>(l.src_info, fs, &l.header->amax_bits[0], l.q);
    HRF_CHECK_LAUNCH();
    size_t bytes = l.cub_bytes;
    HRF_CUDA(cub::DeviceScan::ExclusiveSum(l.cub_temp, bytes, l.q, l.P, fs, st));
  }
  sample_kernel<<<blocks(n), kThreads, 0, st>>>(src_vertices, src_faces, fs, l.P, l.q, n, seed, l.samples, l.order_in,
                                                points, sample_faces);
  HRF_CHECK_LAUNCH();
  {
    size_t bytes = l.cub_bytes;
    HRF_CUDA(cub::DeviceRadixSort::SortKeys(l.cub_temp, bytes, l.order_in, l.order_out, n, 0, 64, st));
  }
  // target: eligibility, Morton order, leaves, refit
  if (ft > 0) {
    prep_kernel<<<blocks(ft), kThreads, 0, st>>>(tgt_vertices, num_tgt_vertices, tgt_faces, ft, l.tgt_info,
                                                 &l.header->amax_bits[1], error, 2, l.header->box);
    HRF_CHECK_LAUNCH();
    morton_kernel<<<blocks(ft), kThreads, 0, st>>>(tgt_vertices, tgt_faces, ft, l.tgt_info, l.header->box, l.keys_in);
    HRF_CHECK_LAUNCH();
    size_t bytes = l.cub_bytes;
    HRF_CUDA(cub::DeviceRadixSort::SortKeys(l.cub_temp, bytes, l.keys_in, l.keys_out, ft, 0, kKeyBits, st));
  }
  leaf_kernel<<<blocks(leaves), kThreads, 0, st>>>(tgt_vertices, tgt_faces, ft, l.keys_out, leaves, l.tris, l.node_lo,
                                                   l.node_hi);
  HRF_CHECK_LAUNCH();
  for (int first = leaves >> 1; first >= 1; first >>= 1) {
    refit_kernel<<<blocks(first), kThreads, 0, st>>>(first, l.node_lo, l.node_hi);
    HRF_CHECK_LAUNCH();
  }
  const int num_slots = (int)blocks(n);
  query_kernel<<<num_slots, kThreads, 0, st>>>(l.samples, l.order_out, n, l.src_info, l.tgt_info, l.tris, ft, l.node_lo,
                                               l.node_hi, leaves, &l.header->amax_bits[1], tv, l.slots, distances, closest_faces);
  HRF_CHECK_LAUNCH();
  finish_kernel<<<1, kFinishThreads, 0, st>>>(l.slots, num_slots, n, num_taus, l.P, l.q, fs, l.header->amax_bits,
                                              error, out, reinterpret_cast<long long*>(counts));
  HRF_CHECK_LAUNCH();
  return 0;
}
