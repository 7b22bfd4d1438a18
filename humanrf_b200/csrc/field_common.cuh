// Device code shared by the forward and backward radiance-field kernels: sample loading,
// multi-resolution hash-grid gathers (tcnn grid.h semantics), vector lerps
// (tensor_composition.cu:30-45), shared-memory operand layouts for wgmma.
#pragma once
#include "common.cuh"

namespace hrf {

constexpr int kTile = 128;              // samples per CTA tile == threads per CTA == one warpgroup
constexpr uint32_t kPrimeY = 2654435761u;  // tcnn coherent_prime_hash
constexpr uint32_t kPrimeZ = 805459861u;

// Byte offsets of the packed bf16 weight blob (K-major no-swizzle core-matrix layout,
// element (n,k) of W[N,K] at ((k/8)*(N/8) + n/8)*128 + (n%8)*16 + (k%8)*2).
constexpr uint32_t kWSig1 = 0;       // sigma  W1 [64,32]
constexpr uint32_t kWSig2 = 4096;    // sigma  W2 [16,64]
constexpr uint32_t kWCol1 = 6144;    // colour W1 [64,K], K = 32 | 48
__host__ __device__ constexpr uint32_t w_col2(int K) { return kWCol1 + 128u * (uint32_t)K; }   // colour W2 [64,64]
__host__ __device__ constexpr uint32_t w_col3(int K) { return w_col2(K) + 8192u; }             // colour W3 [16,64]
__host__ __device__ constexpr uint32_t w_blob_bytes(int K) { return w_col3(K) + 2048u; }       // 20480 | 22528
constexpr uint32_t kWBlobBytesMax = HRF_MLP_BLOB_BYTES;
// row-major fp32 gradient buffer offsets (elements)
constexpr int kGSig1 = 0, kGSig2 = 2048, kGCol1 = 3072;  // colour W2 at 3072 + 64*K, colour W3 4096 later (K = 32 | 48)

// A-operand tile: 128 rows x K bf16, K-major SWIZZLE_NONE: element (r,k) at
// (k/8)*kAChunk + (r/8)*128 + (r%8)*16 + (k%8)*2   -> LBO = kAChunk (K direction), SBO = 128 (M direction).
constexpr uint32_t kAChunk = (kTile / 8) * 128;  // 2048

__device__ __forceinline__ uint32_t a_row_off(int r) { return (uint32_t)(r >> 3) * 128u + (uint32_t)(r & 7) * 16u; }
__device__ __forceinline__ uint32_t w_off(int n, int k, int N) {
  return (uint32_t)((k >> 3) * (N >> 3) + (n >> 3)) * 128u + (uint32_t)(n & 7) * 16u + (uint32_t)(k & 7) * 2u;
}

// Optional early-stop schedule of the density-only pass (see field_fwd.cu).
struct EarlyStop {
  const int32_t* ray_offsets;      // [R+1] first sample of each ray; NULL disables the schedule
  int64_t num_rays;
  float* ray_depth;                // [R] accumulated optical depth sum(sigma*step) of the finished chunks (zeroed)
  unsigned long long* counter;     // work-item counter (zeroed)
  const int32_t* max_chunks;       // device scalar: ceil(max samples per ray / 128)
  float step, stop_depth;
};

// Optional compositing epilogue of the forward kernel (inference): see field_fwd.cu.
struct Composite {
  const int32_t* ray_offsets;   // [R+1] first sample of each ray (samples sorted by ray); NULL disables the epilogue
  const float* background;      // [R,3] or NULL
  float* color;                 // [R,3]
  float* wsum;                  // [R]
  float* partial;               // [tiles][2][8]: (optical depth, C.r, C.g, C.b, W) of the ray segments cut by a tile border
  float step;
};

struct FieldArgs {
  hrf_field f;
  hrf_samples s;
  EarlyStop es;
  Composite comp;
  float* sigma;
  uint32_t* geo;   // bf16 [N,16] viewed as u32 pairs
  float* rgb;
  uint4* feat;     // bf16 [N,32] composed features (optional output)
  uint32_t* egrid; // bf16x2 [16*4][N] per-grid interpolated features (optional output, for the backward scatter)
  const uint4* feat_in;       // bf16 [M,32] composed features of an earlier pass (kFromFeat kernels: no encode)
  const int32_t* feat_index;  // row of feat_in per sample, or NULL (identity)
  int mode;
};

// Live number of samples: the device scalar of a sync-free pipeline (bounded by the capacity), or the host value.
__device__ __forceinline__ int64_t live_samples(const hrf_samples& s) {
  if (s.num_samples_dev == nullptr) return s.num_samples;
  const int64_t n = *reinterpret_cast<const volatile int64_t*>(s.num_samples_dev);
  return n < s.num_samples ? (n < 0 ? 0 : n) : s.num_samples;
}

struct Sample {
  float x, y, z, t;        // normalised coordinates in [0,1] (positions + 0.5, local time)
  const hrf_segment* seg;  // segment descriptor (NULL for padding threads)
};
// View direction and camera row of a sample.  Loaded separately, AFTER the gather phase, so that these four values do
// not occupy registers during the 512-gather loop (the re-read hits L1/L2).
struct View {
  float dx, dy, dz;
  int cam;                 // camera row of the embedding table, or -1 (zeros: evaluation / no embedding)
};

__device__ __forceinline__ Sample load_sample(const hrf_field& f, const hrf_samples& s, int64_t i, int64_t n_live) {
  Sample o;
  o.seg = nullptr;
  o.x = o.y = o.z = o.t = 0.f;
  if (i >= n_live) return o;
  int frame;
  float px, py, pz;
  if (s.ray_origins != nullptr) {
    // volume_rendering.py:66-69 : positions = origins[ri] + t * dirs[ri]  (mul, then add: two roundings)
    const int64_t r = __ldg(s.ray_indices + i);
    const float t = __ldg(s.sample_distances + i);
    const float* ro = s.ray_origins + 3 * r;
    const float* rd = s.ray_directions + 3 * r;
    px = __fadd_rn(__ldg(ro), __fmul_rn(t, __ldg(rd)));
    py = __fadd_rn(__ldg(ro + 1), __fmul_rn(t, __ldg(rd + 1)));
    pz = __fadd_rn(__ldg(ro + 2), __fmul_rn(t, __ldg(rd + 2)));
    frame = __ldg(s.ray_frame_numbers + r);
  } else {
    px = __ldg(s.positions + 3 * i), py = __ldg(s.positions + 3 * i + 1), pz = __ldg(s.positions + 3 * i + 2);
    frame = __ldg(s.frame_numbers + i);
  }
  // humanrf.py:175 : positions + 0.5 ; :176 normalised local frame number
  o.x = __fadd_rn(px, 0.5f), o.y = __fadd_rn(py, 0.5f), o.z = __fadd_rn(pz, 0.5f);
  int sg = -1;
  if (frame >= 0 && frame < f.lut_size) {
    sg = __ldg(f.frame_to_segment + frame);
    o.t = __ldg(f.frame_to_tlocal + frame);
  }
  if (sg >= 0 && sg < f.num_segments) o.seg = f.segments + sg;
  return o;
}

__device__ __forceinline__ View load_view(const hrf_field& f, const hrf_samples& s, int64_t i, int64_t n_live) {
  View v;
  v.dx = v.dy = v.dz = 0.f;
  v.cam = -1;
  if (i >= n_live) return v;
  const bool want_cam = s.use_camera_embeddings && f.camera_embeddings != nullptr;
  if (s.ray_origins != nullptr) {
    const int64_t r = __ldg(s.ray_indices + i);
    const float* rd = s.ray_directions + 3 * r;
    v.dx = __ldg(rd), v.dy = __ldg(rd + 1), v.dz = __ldg(rd + 2);
    if (want_cam && s.ray_camera_numbers != nullptr) v.cam = __ldg(s.ray_camera_numbers + r);
  } else {
    if (s.directions != nullptr)
      v.dx = __ldg(s.directions + 3 * i), v.dy = __ldg(s.directions + 3 * i + 1), v.dz = __ldg(s.directions + 3 * i + 2);
    if (want_cam && s.camera_numbers != nullptr) v.cam = __ldg(s.camera_numbers + i);
  }
  if (v.cam < 0 || v.cam >= f.num_cameras) v.cam = -1;
  return v;
}

struct Cell {
  uint32_t g;
  float f;
};
__device__ __forceinline__ Cell to_cell(float scale, float v) {
  // tcnn pos_fract: pos = fmaf(scale, x, 0.5); grid = (uint32_t)(int)floorf(pos); frac = pos - floor
  const float p = __fmaf_rn(scale, v, 0.5f);
  const float fl = floorf(p);
  Cell c;
  c.g = (uint32_t)(int)fl;
  c.f = p - fl;
  return c;
}

static __device__ __noinline__ uint32_t slow_mod(uint32_t v, uint32_t size) { return size != 0u ? v % size : 0u; }

// Eight corner indices of one level (tcnn grid_index): dense x + y*res + z*res^2, or the
// coherent prime hash, both reduced modulo the level's hashmap size.
__device__ __forceinline__ void corner_indices(bool hashed, uint32_t res, uint32_t size, Cell a, Cell b, Cell c,
                                               uint32_t idx[8]) {
  if (hashed) {
    const uint32_t m = size - 1u;  // hashed levels always have size == 2^log2T
    const uint32_t b0 = b.g * kPrimeY, b1 = (b.g + 1u) * kPrimeY;
    const uint32_t c0 = c.g * kPrimeZ, c1 = (c.g + 1u) * kPrimeZ;
#pragma unroll
    for (int k = 0; k < 8; ++k)
      idx[k] = (((k & 1) ? a.g + 1u : a.g) ^ ((k & 2) ? b1 : b0) ^ ((k & 4) ? c1 : c0)) & m;
  } else {
    const uint32_t r2 = res * res;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      uint32_t v = ((k & 1) ? a.g + 1u : a.g) + ((k & 2) ? b.g + 1u : b.g) * res + ((k & 4) ? c.g + 1u : c.g) * r2;
      // v % size.  A dense level has res^3 <= size and, for a position inside [0,1], v <= res^3 + res^2 + res < 2 size,
      // so one subtraction settles it without inlining a 32-bit division at each of the 32 corners (that division was
      // 654 of the forward kernel's 3 336 SASS instructions, and the kernel is instruction-cache sensitive).  Positions
      // outside the unit cube (reachable through QueryInput) take the cold, out-of-line modulo: constant time, as tcnn.
      if (v >= size) {
        v -= size;
        if (v >= size) v = slow_mod(v, size);
      }
      idx[k] = v;
    }
  }
}
__device__ __forceinline__ void corner_weights(Cell a, Cell b, Cell c, float w[8]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    float v = (k & 1) ? a.f : 1.f - a.f;   // weight = 1; weight *= ... per dim, in dim order
    v *= (k & 2) ? b.f : 1.f - b.f;
    v *= (k & 4) ? c.f : 1.f - c.f;
    w[k] = v;
  }
}

// Trilinear gather of one level of one grid -> 2 features (fp32 blend of bf16 entries).
__device__ __forceinline__ float2 gather_level(const uint32_t* __restrict__ tab, bool hashed, uint32_t res,
                                               uint32_t size, Cell a, Cell b, Cell c) {
  uint32_t idx[8], raw[8];
  float w[8];
  corner_indices(hashed, res, size, a, b, c, idx);
#pragma unroll
  for (int k = 0; k < 8; ++k) raw[k] = __ldg(tab + idx[k]);
  corner_weights(a, b, c, w);
  float2 acc = make_float2(0.f, 0.f);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    acc.x = __fmaf_rn(w[k], bf16_lo(raw[k]), acc.x);
    acc.y = __fmaf_rn(w[k], bf16_hi(raw[k]), acc.y);
  }
  return acc;
}

// 1-D lerp taps into `vectors` (tensor_composition.cu:37-45)
struct VecTap {
  uint32_t o0, o1;  // element offsets of row i0 / i1 inside vectors[axis]
  float frac;
};
__device__ __forceinline__ VecTap make_tap(float coord, int vec_res, int axis) {
  const float c = __fmaf_rn(coord, (float)vec_res, -0.5f);
  const float fl = floorf(c);
  VecTap t;
  t.frac = c - fl;
  const int i0 = (int)fmaxf(fl, 0.f);
  const int i1 = (int)fminf(fl + 1.f, (float)(vec_res - 1));
  t.o0 = ((uint32_t)axis * (uint32_t)vec_res + (uint32_t)min(max(i0, 0), vec_res - 1)) * HRF_N_FEATURES;
  t.o1 = ((uint32_t)axis * (uint32_t)vec_res + (uint32_t)min(max(i1, 0), vec_res - 1)) * HRF_N_FEATURES;
  return t;
}
__device__ __forceinline__ float2 lerp_tap(const float* __restrict__ vec, const VecTap& t, int feat) {
  const float2 v0 = __ldg(reinterpret_cast<const float2*>(vec + t.o0 + feat));
  const float2 v1 = __ldg(reinterpret_cast<const float2*>(vec + t.o1 + feat));
  return make_float2(v0.x + t.frac * (v1.x - v0.x), v0.y + t.frac * (v1.y - v0.y));
}

// The same taps as row indices, and their lerp through the TRANSPOSED copy vectors_t[axis][level][row][2] when the segment
// has one (hrf_segment.vectors_t): the lanes of a warp are consecutive samples of a ray, i.e. neighbouring rows -- in
// `vectors` ([axis][row][32]) every row is its own 128-byte line (15-26 lines per load instruction at the finest
// resolution), in the transposed copy 16 rows share a line.  Same fp32 values, same arithmetic.
struct RowTap2 {
  uint32_t i0, i1;
  float frac;
};
__device__ __forceinline__ RowTap2 make_row_tap2(float coord, int vec_res) {
  const float c = __fmaf_rn(coord, (float)vec_res, -0.5f);
  const float fl = floorf(c);
  RowTap2 t;
  t.frac = c - fl;
  t.i0 = (uint32_t)min(max((int)fmaxf(fl, 0.f), 0), vec_res - 1);
  t.i1 = (uint32_t)min(max((int)fminf(fl + 1.f, (float)(vec_res - 1)), 0), vec_res - 1);
  return t;
}
// base = vectors_t + (axis*16 + level) * vec_res * 2  (stride 2)   or   vectors + axis * vec_res * 32 + 2 * level  (stride 32)
__device__ __forceinline__ float2 lerp_row_tap(const float* __restrict__ base, uint32_t stride, const RowTap2& t) {
  const float2 v0 = __ldg(reinterpret_cast<const float2*>(base + t.i0 * stride));
  const float2 v1 = __ldg(reinterpret_cast<const float2*>(base + t.i1 * stride));
  return make_float2(v0.x + t.frac * (v1.x - v0.x), v0.y + t.frac * (v1.y - v0.y));
}

// Degree-4 real spherical harmonics of the view direction (tcnn SphericalHarmonics on (d+1)/2).
__device__ __forceinline__ void sh4(float dx, float dy, float dz, float* o) {
  const float x = ((dx + 1.f) * 0.5f) * 2.f - 1.f, y = ((dy + 1.f) * 0.5f) * 2.f - 1.f,
              z = ((dz + 1.f) * 0.5f) * 2.f - 1.f;
  const float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
  o[0] = 0.28209479177387814f;
  o[1] = -0.48860251190291987f * y;
  o[2] = 0.48860251190291987f * z;
  o[3] = -0.48860251190291987f * x;
  o[4] = 1.0925484305920792f * xy;
  o[5] = -1.0925484305920792f * yz;
  o[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
  o[7] = -1.0925484305920792f * xz;
  o[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
  o[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2);
  o[10] = 2.8906114426405538f * xy * z;
  o[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2);
  o[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
  o[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2);
  o[14] = 1.4453057213202769f * z * (x2 - y2);
  o[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
}

// Colour-net input row (humanrf.py:192-206 + tcnn Composite[SH(4) on 3 dims, Identity] padded with 1.0):
// [SH 0..15 | geo 16..30 | camera embedding 31..30+E | 1.0 ...] as bf16, K = 32 (E = 0) or 48.
__device__ __forceinline__ void write_color_input(const hrf_field& f, unsigned char* abuf, uint32_t roff, const View& s,
                                                  const float* o /* sigma-net output, o[1..15] = geo */) {
  float sh[16];
  sh4(s.dx, s.dy, s.dz, sh);
  const int E = f.camera_embedding_dim;
  const float* emb = (s.cam >= 0) ? f.camera_embeddings + (size_t)s.cam * E : nullptr;
  auto tail = [&](int j) -> float {  // feature j >= 31
    const int e = j - 31;
    return e < E ? (emb != nullptr ? __ldg(emb + e) : 0.f) : 1.0f;
  };
  *reinterpret_cast<uint4*>(abuf + 0 * kAChunk + roff) = make_uint4(
      pack_bf16x2(sh[0], sh[1]), pack_bf16x2(sh[2], sh[3]), pack_bf16x2(sh[4], sh[5]), pack_bf16x2(sh[6], sh[7]));
  *reinterpret_cast<uint4*>(abuf + 1 * kAChunk + roff) = make_uint4(
      pack_bf16x2(sh[8], sh[9]), pack_bf16x2(sh[10], sh[11]), pack_bf16x2(sh[12], sh[13]), pack_bf16x2(sh[14], sh[15]));
  *reinterpret_cast<uint4*>(abuf + 2 * kAChunk + roff) = make_uint4(
      pack_bf16x2(o[1], o[2]), pack_bf16x2(o[3], o[4]), pack_bf16x2(o[5], o[6]), pack_bf16x2(o[7], o[8]));
  *reinterpret_cast<uint4*>(abuf + 3 * kAChunk + roff) = make_uint4(
      pack_bf16x2(o[9], o[10]), pack_bf16x2(o[11], o[12]), pack_bf16x2(o[13], o[14]), pack_bf16x2(o[15], tail(31)));
  if (f.color_in_width == 48) {
    *reinterpret_cast<uint4*>(abuf + 4 * kAChunk + roff) = make_uint4(
        pack_bf16x2(tail(32), tail(33)), pack_bf16x2(tail(34), tail(35)), pack_bf16x2(tail(36), tail(37)),
        pack_bf16x2(tail(38), tail(39)));
    *reinterpret_cast<uint4*>(abuf + 5 * kAChunk + roff) = make_uint4(
        pack_bf16x2(tail(40), tail(41)), pack_bf16x2(tail(42), tail(43)), pack_bf16x2(tail(44), tail(45)),
        pack_bf16x2(tail(46), tail(47)));
  }
}

// Encode one sample (4 grids x 16 levels, composed with the vector lerps) and write the 32
// bf16 features of row `row` into the K-major A tile at `abuf` (shared memory).
// If `egrid` is not NULL the per-grid interpolated features e_k (before composition) are also stored, bf16x2, as
// egrid[(level*4 + grid) * n + i]: the backward scatter needs them for the vector gradients and then does not have
// to gather the tables a second time.
// kLevelUnroll = 4 keeps four levels' gathers in flight per thread; 2 / 1 shrink the unrolled code.  The forward kernel
// runs fastest with 1 (it was instruction-cache bound at 4: 117 KB of SASS), see launch_field_forward.
template <bool kSaveGrid = false, int kLevelUnroll = 4>
__device__ __forceinline__ void encode_to_smem(const hrf_field& f, const Sample& s, unsigned char* abuf, int row,
                                               uint32_t* egrid = nullptr, int64_t i = 0, int64_t n = 0) {
  const uint32_t roff = a_row_off(row);
  if (s.seg == nullptr) {
#pragma unroll
    for (int kg = 0; kg < 4; ++kg) *reinterpret_cast<uint4*>(abuf + kg * kAChunk + roff) = make_uint4(0, 0, 0, 0);
    return;
  }
  const hrf_segment* sg = s.seg;
  const uint32_t* g0 = sg->grid[0];
  const uint32_t* g1 = sg->grid[1];
  const uint32_t* g2 = sg->grid[2];
  const uint32_t* g3 = sg->grid[3];
  const uint32_t hmask = sg->hashed_mask;
  const RowTap2 tx = make_row_tap2(s.x, f.vec_res), ty = make_row_tap2(s.y, f.vec_res), tz = make_row_tap2(s.z, f.vec_res),
                tt = make_row_tap2(s.t, f.vec_res);
  const bool vt = sg->vectors_t != nullptr;
  const float* vbase = vt ? sg->vectors_t : sg->vectors;
  const uint32_t vstride = vt ? 2u : (uint32_t)HRF_N_FEATURES;
  const uint32_t vaxis = (uint32_t)f.vec_res * (vt ? 2u * HRF_N_LEVELS : (uint32_t)HRF_N_FEATURES);   // elements per axis
  const uint32_t vlevel = vt ? 2u * (uint32_t)f.vec_res : 2u;                                            // elements per level
  auto one_level = [&](int l) -> uint32_t {
    const float scale = f.level_scale[l];
    const uint32_t res = f.level_res[l];
    const uint32_t off = sg->level_offset[l];
    const uint32_t size = sg->level_size[l];
    const bool hashed = (hmask >> l) & 1u;
    const Cell cx = to_cell(scale, s.x), cy = to_cell(scale, s.y), cz = to_cell(scale, s.z), ct = to_cell(scale, s.t);
    // decomposition4d.py:126-129 : xyz, xyt, yzt, xzt
    const float2 e0 = gather_level(g0 + off, hashed, res, size, cx, cy, cz);
    const float2 e1 = gather_level(g1 + off, hashed, res, size, cx, cy, ct);
    const float2 e2 = gather_level(g2 + off, hashed, res, size, cy, cz, ct);
    const float2 e3 = gather_level(g3 + off, hashed, res, size, cx, cz, ct);
    const float* vl = vbase + (uint32_t)l * vlevel;
    const float2 vx = lerp_row_tap(vl, vstride, tx), vy = lerp_row_tap(vl + vaxis, vstride, ty),
                 vz = lerp_row_tap(vl + 2u * vaxis, vstride, tz), vt_ = lerp_row_tap(vl + 3u * vaxis, vstride, tt);
    // tensor_composition.cu:49-52 : xyz*v_t + xyt*v_z + yzt*v_x + xzt*v_y
    const float o0 = e0.x * vt_.x + e1.x * vz.x + e2.x * vx.x + e3.x * vy.x;
    const float o1 = e0.y * vt_.y + e1.y * vz.y + e2.y * vx.y + e3.y * vy.y;
    if (kSaveGrid && egrid != nullptr) {
      uint32_t* eg = egrid + (size_t)(4 * l) * n + i;
      eg[0] = pack_bf16x2(e0.x, e0.y);
      eg[n] = pack_bf16x2(e1.x, e1.y);
      eg[2 * n] = pack_bf16x2(e2.x, e2.y);
      eg[3 * n] = pack_bf16x2(e3.x, e3.y);
    }
    return pack_bf16x2(o0, o1);
  };
  if constexpr (kLevelUnroll == 4) {
#pragma unroll 1
    for (int kg = 0; kg < 4; ++kg) {
      uint32_t pk[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) pk[j] = one_level(kg * 4 + j);
      *reinterpret_cast<uint4*>(abuf + kg * kAChunk + roff) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    }
  } else {
#pragma unroll kLevelUnroll
    for (int l = 0; l < HRF_N_LEVELS; ++l)
      *reinterpret_cast<uint32_t*>(abuf + (l >> 2) * kAChunk + roff + (l & 3) * 4) = one_level(l);
  }
}

// A 128-row tile is two m64 wgmma operands: rows 64h..64h+63 start 8 row groups of 128 bytes later per half.
constexpr uint32_t kAHalf = 8u * 128u;

// Issue one dense layer D[128,N] = A[128,K] * W[N,K]^T on the tensor cores (all 128 threads): rows 0-63 accumulate
// into d[0, N/2), rows 64-127 into d[N/2, N).  kHalf = 0 | 1 issues the rows of that half only, into d[0, N/2).
template <int N, int K, int kHalf = -1>
__device__ __forceinline__ void mma_layer(float* d, uint32_t a_addr, uint32_t w_addr) {
  constexpr uint32_t b_lbo = (uint32_t)(N >> 3) * 128u;
#pragma unroll
  for (int k = 0; k < K / 16; ++k) {
    const uint64_t bd = make_smem_desc(w_addr + (uint32_t)k * 2u * b_lbo, b_lbo, 128u);
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (kHalf < 0 || h == kHalf)
        wgmma_bf16<N>(d + (kHalf < 0 ? h * (N / 2) : 0),
                      make_smem_desc(a_addr + h * kAHalf + (uint32_t)k * 2u * kAChunk, kAChunk, 128u), bd, k > 0 ? 1u : 0u);
  }
}

// An MMA round: mma_begin() publishes the operand tiles written with ordinary stores to the tensor cores; after
// mma_end() every MMA of the round has completed, so its operand tiles may be overwritten.
__device__ __forceinline__ void mma_begin() {
  fence_proxy_async_smem();
  __syncthreads();
  wgmma_fence();
}
__device__ __forceinline__ void mma_end() {
  wgmma_commit();
  wgmma_wait_all();
  __syncthreads();
}

// Tile row and column of accumulator register q of this thread in half h of a 128-row result (see wgmma_bf16).
__device__ __forceinline__ int frag_row(int h, int q) {
  return 64 * h + 16 * (int)(threadIdx.x >> 5) + (int)((threadIdx.x & 31) >> 2) + 8 * ((q >> 1) & 1);
}
__device__ __forceinline__ int frag_col(int q) { return 8 * (q >> 2) + 2 * (int)(threadIdx.x & 3) + (q & 1); }

// relu(D[128,64]) -> bf16 K-major tile (K = 64): the A operand of the next layer.  kHalf as in mma_layer.
template <int kHalf = -1>
__device__ __forceinline__ void frag_store_relu64(unsigned char* buf, const float* d) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int q = 0; q < 32; q += 2) {
      if (kHalf >= 0 && h != kHalf) continue;
      const int r = frag_row(h, q), c = frag_col(q), j = (kHalf < 0 ? h * 32 : 0) + q;
      *reinterpret_cast<uint32_t*>(buf + (c >> 3) * kAChunk + a_row_off(r) + (c & 7) * 2) =
          pack_bf16x2(fmaxf(d[j], 0.f), fmaxf(d[j + 1], 0.f));
    }
}

// fp32 staging of columns [kC0, kC0 + kW) of D[128,N] (kW a power of two >= 4) so that thread r can read row r:
// row-major, the 16-byte groups of a row XOR-swizzled by the row so that neither the fragment stores nor the row
// reads pile onto a few banks.
template <int kW>
__device__ __forceinline__ int stage_off(int r, int c) {
  constexpr int mask = (kW / 4 < 8 ? kW / 4 : 8) - 1;
  return r * kW + ((((c >> 2) ^ (r & mask))) << 2) + (c & 3);
}
template <int N, int kW, int kC0 = 0>
__device__ __forceinline__ void frag_stage(float* st, const float* d) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int q = 0; q < N / 2; q += 2) {
      const int c = frag_col(q) - kC0;
      if (c >= 0 && c < kW)
        *reinterpret_cast<float2*>(st + stage_off<kW>(frag_row(h, q), c)) = make_float2(d[h * (N / 2) + q], d[h * (N / 2) + q + 1]);
    }
}
template <int kW>
__device__ __forceinline__ void stage_read_row(const float* st, float* v) {
  const int r = threadIdx.x;
#pragma unroll
  for (int g = 0; g < kW / 4; ++g) {
    const float4 x = *reinterpret_cast<const float4*>(st + stage_off<kW>(r, 4 * g));
    v[4 * g] = x.x, v[4 * g + 1] = x.y, v[4 * g + 2] = x.z, v[4 * g + 3] = x.w;
  }
}

// Gradient of the TIME rows of `vectors` (grid xyz, tensor_composition.cu:49-52,109-111).  Every sample of a ray has the
// same two rows and a batch holds a handful of frames (max_num_frames_per_batch, run_args.py:101): a whole scatter launch
// adds into ~16 rows x 16 levels, i.e. a few 128-byte lines, and same-line REDs serialise in one L2 slice (which made the
// scatter time depend on which frames a batch had drawn until these adds were combined).
// The lanes of a warp walk about one ray: sum the lanes that hold the same row, one RED per distinct row and warp.
// `key` identifies the row (0xffffffff: nothing to add), `addr` is the same for equal keys.  All 32 lanes must call.
__device__ __forceinline__ void warp_combine_red2(uint32_t key, float* addr, float s0, float s1) {
  const int lane = threadIdx.x & 31;
  uint32_t rem = __ballot_sync(0xffffffffu, key != 0xffffffffu);
  while (rem != 0u) {                                // (warp-uniform)
    const int leader = __ffs(rem) - 1;
    const uint32_t k = __shfl_sync(0xffffffffu, key, leader);
    const bool mine = key == k;
    float t0 = mine ? s0 : 0.f, t1 = mine ? s1 : 0.f;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      t0 += __shfl_xor_sync(0xffffffffu, t0, d);
      t1 += __shfl_xor_sync(0xffffffffu, t1, d);
    }
    if (lane == leader) asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(t0), "f"(t1));
    rem &= ~__ballot_sync(0xffffffffu, mine);
  }
}

}  // namespace hrf
