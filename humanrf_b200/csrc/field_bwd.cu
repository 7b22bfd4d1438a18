// Fused backward of the HumanRF radiance field for sm_90a (autograd of humanrf.py:158-208).
// Per 128-sample tile (thread r = sample r = operand row r; the CTA is one warpgroup):
//   1. forward recompute of both MLPs from the saved composed features (or a re-encode),
//      keeping every activation tile in shared memory (bf16, K-major core-matrix layout);
//   2. MLP backward on the tensor cores (wgmma).  The SAME shared-memory tiles serve three roles by
//      switching descriptors only:  K-major A operand of the forward / dgrad GEMMs, and
//      MN-major A / B operands of the wgrad GEMMs (contraction over the 128 samples).  The
//      packed forward weight blob is re-used as the MN-major B operand of the dgrad GEMMs.
//      Weight-gradient accumulators (M=64 each, 88 registers a thread) live in registers for the whole
//      persistent CTA and are flushed once with fp32 atomics;
//   3. d(composed features) goes to a level-major [16][N] workspace; a second, high-occupancy kernel
//      (grid_scatter_kernel: thread = (sample, level)) re-gathers the 4x8 corners (needed for the vector
//      gradients) and issues red.global.add.v2.f32 into the fp32 table gradients, with warp-combined adds
//      for the time axis.  (One fused kernel was latency-bound at its low occupancy.)
#include <cstddef>
#include <cstdlib>

#include "field_common.cuh"

namespace hrf {

struct __align__(1024) BwdSmem {
  unsigned char w[kWBlobBytesMax];
  unsigned char feat[kTile * 32 * 2];  // composed features            (A32)
  unsigned char cin[kTile * 48 * 2];   // colour-net input              (A32 / A48)
  unsigned char hs[kTile * 64 * 2];    // sigma hidden, then d(hidden)  (A64)
  unsigned char h1[kTile * 64 * 2];    // colour hidden 1, then its gradient, then dFeat staging
  unsigned char h2[kTile * 64 * 2];    // colour hidden 2, then its gradient, then d(colour input) staging
  unsigned char g3[kTile * 16 * 2];    // d(colour pre-activation)  [128,16]
  unsigned char gs[kTile * 16 * 2];    // colour-net output staging, then d(sigma-net output) [128,16]
  uint64_t bar_w;
};

struct BwdArgs {
  hrf_field f;
  hrf_samples s;
  const hrf_segment_grads* seg_grads;
  const float* d_sigma;
  const float* d_rgb;
  const float* d_geo;    // [N,15] gradient of the geometry features, or NULL
  const uint4* feat_in;  // bf16 [M,32] saved by a forward pass, or NULL (re-encode)
  const int32_t* feat_index;  // row of feat_in per sample, or NULL (identity)
  float* d_mlp;
  float* d_emb;   // camera-embedding gradient [num_cameras, E] or NULL
  float2* dfeat;  // [16][N] float2 workspace: d(composed features)
  float4* pos4;   // [N] normalised (x,y,z,t) of every sample, for grid_scatter_kernel
  uint8_t* seg8;  // [N] segment index (255 = no segment)
};

// D[128,Nin] = G[128,Kout] * W[Kout,Nin]  : A = gradient tile (K-major), B = forward blob read MN-major
template <int Nin, int Kout>
__device__ __forceinline__ void issue_dgrad(float* d, uint32_t g_addr, uint32_t w_addr) {
  constexpr uint32_t b_sbo = (uint32_t)(Kout >> 3) * 128u;
#pragma unroll
  for (int k = 0; k < Kout / 16; ++k) {
    const uint64_t bd = make_smem_desc(w_addr + (uint32_t)k * 256u, 128u, b_sbo);
#pragma unroll
    for (int h = 0; h < 2; ++h)
      wgmma_bf16<Nin, 0, 1>(d + h * (Nin / 2), make_smem_desc(g_addr + h * kAHalf + (uint32_t)k * 2u * kAChunk, kAChunk, 128u),
                            bd, k > 0 ? 1u : 0u);
  }
}
// D[64,N] += X^T[64,128] * Y[128,N] : both tiles read MN-major, contraction over the 128 samples
template <int N>
__device__ __forceinline__ void issue_wgrad(float* d, uint32_t x_addr, uint32_t y_addr) {
#pragma unroll
  for (int k = 0; k < kTile / 16; ++k) {
    const uint64_t ad = make_smem_desc(x_addr + (uint32_t)k * 256u, 128u, kAChunk);
    const uint64_t bd = make_smem_desc(y_addr + (uint32_t)k * 256u, 128u, kAChunk);
    wgmma_bf16<N, 1, 1>(d, ad, bd, 1u);
  }
}

// in place: the tile holds relu(h) (bf16, K = 64); replace it by D * (h > 0) (bf16), D[128,64] in fragments
__device__ __forceinline__ void frag_relu_backward64(unsigned char* buf, const float* d) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int q = 0; q < 32; q += 2) {
      const int r = frag_row(h, q), c = frag_col(q);
      uint32_t* p = reinterpret_cast<uint32_t*>(buf + (c >> 3) * kAChunk + a_row_off(r) + (c & 7) * 2);
      const uint32_t a = *p;
      const float lo = (a & 0x7fffu) != 0u && !(a & 0x8000u) ? d[h * 32 + q] : 0.f;
      const float hi = (a & 0x7fff0000u) != 0u && !(a & 0x80000000u) ? d[h * 32 + q + 1] : 0.f;
      *p = pack_bf16x2(lo, hi);
    }
}

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}
__device__ __forceinline__ void red_add2(float* addr, float a, float b) {
  // no return value wanted: the vector RED, not the ATOM the float2 atomicAdd intrinsic compiles to
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// Flush of an M = 64 weight-gradient fragment D (kRegs registers): dst[m * ld + c] += D[m][c] for c < n, the two
// adjacent columns a thread holds as one 8-byte RED when dst is 8-byte aligned.
template <int kRegs>
__device__ __forceinline__ void flush_rows(float* dst, int ld, const float* acc, int n, bool v2ok) {
#pragma unroll
  for (int q = 0; q < kRegs; q += 2) {
    const int m = frag_row(0, q), c = frag_col(q);
    if (c < n) {
      if (v2ok) red_add2(dst + m * ld + c, acc[q], acc[q + 1]);
      else atomicAdd(dst + m * ld + c, acc[q]), atomicAdd(dst + m * ld + c + 1, acc[q + 1]);
    }
  }
}
// Transposed flush of an M = 64, N = 16 fragment: dst[c * 64 + m] += D[m][c].
__device__ __forceinline__ void flush_cols(float* dst, const float* acc) {
#pragma unroll
  for (int q = 0; q < 8; ++q) atomicAdd(dst + frag_col(q) * 64 + frag_row(0, q), acc[q]);
}

// Moving to the neighbouring cell along one axis (bit kBit of the corner number) keeps the face the two cells share:
// the 4 corners that leave are flushed, the 4 shared ones slide to the opposite plane with their accumulators.
template <int kBit>
__device__ __forceinline__ void shift_corners(int d, float* gtab, uint32_t (&idx)[8], float (&ax)[8], float (&ay)[8]) {
  const bool up = d > 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    if (q & kBit) continue;
    const int lo = q, hi = q | kBit;
    const float dx = up ? ax[lo] : ax[hi], dy = up ? ay[lo] : ay[hi];   // the corner that leaves
    const uint32_t di = up ? idx[lo] : idx[hi];
    if (dx != 0.f || dy != 0.f) red_add2(gtab + 2 * (size_t)di, dx, dy);
    const float kx = up ? ax[hi] : ax[lo], ky = up ? ay[hi] : ay[lo];   // the corner that stays
    const uint32_t ki = up ? idx[hi] : idx[lo];
    ax[lo] = up ? kx : 0.f, ay[lo] = up ? ky : 0.f;
    ax[hi] = up ? 0.f : kx, ay[hi] = up ? 0.f : ky;
    idx[lo] = ki, idx[hi] = ki;   // (the vacated slot holds a zero accumulator; all indices are recomputed after the shifts)
  }
}

// Table / vector gradient scatter (tcnn kernel_grid_backward + compose_tensors_backward,
// tensor_composition.cu:57-118) as a separate high-occupancy kernel.
//   thread = (chunk of kChunk consecutive samples, level, grid): blockIdx.y = level * grid_count + (grid - grid_first).
// Consecutive samples of a ray are 4e-4 apart, so at most levels they stay in the same grid cell for several
// samples: the thread keeps the cell's 8 corner indices / values in registers, accumulates w*g per corner while
// the cell does not change and issues the 8 vector REDs once per RUN of samples (not once per sample).  The
// same run-length trick applies to the vector taps (the time tap never changes along a ray).  This cuts both
// the L2 atomics and the gathers by the run length (about 80 samples at level 0, 1.2 at level 15) with no
// shuffles.  Each grid pairs with exactly one vector axis (xyz<->t, xyt<->z, yzt<->x, xzt<->y), so the
// (level, grid) threads are independent.
constexpr int kChunkDefault = 16;  // samples per thread (HRF_SCATTER_CHUNK overrides)

struct ScatterArgs {
  hrf_field f;
  hrf_samples s;
  const hrf_segment_grads* seg_grads;
  const float2* dfeat;  // [16 levels][N] float2, written by field_backward_kernel
  const float4* pos4;   // [N] (x,y,z,t), written by field_backward_kernel
  const uint8_t* seg8;  // [N]
  const uint32_t* egrid;  // bf16x2 [16*4][egrid_stride] per-grid features saved by a forward pass, or NULL (re-gather the tables)
  const int32_t* feat_index;  // column of sample i inside egrid, or NULL (identity)
  int64_t egrid_stride;
  int chunk;                   // consecutive samples per thread
  int tapstage;                // staged kernel: 1 = stage the interpolated vector values too (HRF_SCATTER_TAPSTAGE)
  int carry;                   // 1: carry the accumulators of corners shared with the previous cell (HRF_SCATTER_CARRY=0 disables)
  int grid_first, grid_count;  // this launch covers grids [grid_first, grid_first + grid_count) of xyz, xyt, yzt, xzt
};

__global__ void __launch_bounds__(256, 3) grid_scatter_kernel(const __grid_constant__ ScatterArgs a) {
  const hrf_field& f = a.f;
  const int64_t n = live_samples(a.s);
  const int64_t ns = a.s.num_samples;   // row length of the level-major workspace
  const int kChunk = a.chunk;
  const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * kChunk;
  if (i0 >= n) return;
  const int l = (int)blockIdx.y / a.grid_count, k = a.grid_first + (int)blockIdx.y % a.grid_count;
  const int axis = (k == 0) ? 3 : (k == 1) ? 2 : (k == 2) ? 0 : 1;  // vector axis paired with grid k
  const float scale = f.level_scale[l];
  const uint32_t res = f.level_res[l];
  const float2* __restrict__ dfl = a.dfeat + (size_t)l * ns;

  // state of the current run
  const hrf_segment* cur_seg = nullptr;
  uint32_t ca = 0xffffffffu, cb = 0, cc = 0;  // current cell
  uint32_t idx[8], raw[8];
  float accx[8], accy[8];
  float* gtab = nullptr;
  // vector-tap run
  uint32_t to0 = 0xffffffffu, to1 = 0;
  float* gvec = nullptr;
  float va0 = 0.f, va1 = 0.f, vb0 = 0.f, vb1 = 0.f;
#pragma unroll
  for (int q = 0; q < 8; ++q) accx[q] = accy[q] = 0.f, idx[q] = raw[q] = 0u;

  auto flush_cell = [&]() {
    if (gtab != nullptr) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        if (accx[q] != 0.f || accy[q] != 0.f) red_add2(gtab + 2 * (size_t)idx[q], accx[q], accy[q]);
        accx[q] = accy[q] = 0.f;
      }
    }
  };
  auto flush_tap = [&]() {
    if (gvec != nullptr && to0 != 0xffffffffu) {
      if (va0 != 0.f || va1 != 0.f) red_add2(gvec + to0 + 2 * l, va0, va1);
      if (vb0 != 0.f || vb1 != 0.f) red_add2(gvec + to1 + 2 * l, vb0, vb1);
    }
    va0 = va1 = vb0 = vb1 = 0.f;
  };

  const int cnt = (int)((n - i0) < kChunk ? (n - i0) : kChunk);
#pragma unroll 1
  for (int j = 0; j < cnt; ++j) {
    const int64_t i = i0 + j;
    const uint32_t sgi = a.seg8[i];
    if (sgi == 255u) continue;
    const float4 p4 = __ldg(a.pos4 + i);   // (the ray -> position chain was resolved once, in field_backward_kernel)
    Sample s;
    s.x = p4.x, s.y = p4.y, s.z = p4.z, s.t = p4.w;
    s.seg = f.segments + sgi;
    const float2 dO = __ldg(dfl + i);
    const float c0 = (k == 2) ? s.y : s.x;                       // grid coordinates (decomposition4d.py:126-129)
    const float c1 = (k == 0 || k == 1) ? s.y : s.z;
    const float c2 = (k == 0) ? s.z : s.t;
    const float cv = (axis == 0) ? s.x : (axis == 1) ? s.y : (axis == 2) ? s.z : s.t;
    const Cell A = to_cell(scale, c0), B = to_cell(scale, c1), C = to_cell(scale, c2);
    if (s.seg != cur_seg || A.g != ca || B.g != cb || C.g != cc) {  // new cell: flush the run, fetch the corners
      const int dA = (int)(A.g - ca), dB = (int)(B.g - cb), dC = (int)(C.g - cc);
      if (a.carry && s.seg == cur_seg && dA >= -1 && dA <= 1 && dB >= -1 && dB <= 1 && dC >= -1 && dC <= 1) {
        // neighbouring cell (the usual case along a ray at the fine levels): only the corners that leave are flushed
        if (dA != 0) shift_corners<1>(dA, gtab, idx, accx, accy);
        if (dB != 0) shift_corners<2>(dB, gtab, idx, accx, accy);
        if (dC != 0) shift_corners<4>(dC, gtab, idx, accx, accy);
      } else {
        flush_cell();
      }
      const hrf_segment* sg = s.seg;
      const uint32_t off = sg->level_offset[l];
      corner_indices((sg->hashed_mask >> l) & 1u, res, sg->level_size[l], A, B, C, idx);
      if (a.egrid == nullptr) {
        const uint32_t* tab = sg->grid[k] + off;
#pragma unroll
        for (int q = 0; q < 8; ++q) raw[q] = __ldg(tab + idx[q]);
      }
      if (sg != cur_seg) {
        flush_tap();
        to0 = 0xffffffffu;
        gvec = a.seg_grads[(int)(sg - f.segments)].vectors;
      }
      gtab = a.seg_grads[(int)(sg - f.segments)].grid[k] + 2 * (size_t)off;
      cur_seg = sg, ca = A.g, cb = B.g, cc = C.g;
    }
    const VecTap tp = make_tap(cv, f.vec_res, axis);
    const float2 v = lerp_tap(s.seg->vectors, tp, 2 * l);
    float w[8];
    corner_weights(A, B, C, w);
    const float gx = v.x * dO.x, gy = v.y * dO.y;
    float ex = 0.f, ey = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      accx[q] = __fmaf_rn(w[q], gx, accx[q]);
      accy[q] = __fmaf_rn(w[q], gy, accy[q]);
    }
    if (a.egrid != nullptr) {  // interpolated grid features saved by the forward
      const uint32_t ev = __ldg(a.egrid + (size_t)(4 * l + k) * a.egrid_stride + (a.feat_index != nullptr ? (int64_t)__ldg(a.feat_index + i) : i));
      ex = bf16_lo(ev), ey = bf16_hi(ev);
    } else {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        ex = __fmaf_rn(w[q], bf16_lo(raw[q]), ex);
        ey = __fmaf_rn(w[q], bf16_hi(raw[q]), ey);
      }
    }
    // d vectors[axis][i0/i1][2l..2l+1] = e_k * dOut * (1-frac | frac)   (tensor_composition.cu:109-111)
    if (tp.o0 != to0 || tp.o1 != to1) {
      flush_tap();
      to0 = tp.o0, to1 = tp.o1;
    }
    const float dx = ex * dO.x, dy = ey * dO.y;
    va0 = __fmaf_rn(dx, 1.f - tp.frac, va0), va1 = __fmaf_rn(dy, 1.f - tp.frac, va1);
    vb0 = __fmaf_rn(dx, tp.frac, vb0), vb1 = __fmaf_rn(dy, tp.frac, vb1);
  }
  flush_cell();
  flush_tap();
}

// ---- staged variant (the default) --------------------------------------------------------------------------------
// grid_scatter_kernel reads its per-sample inputs with a stride of `chunk` samples between lanes, so every 32-byte
// sector is fetched for 16 / 8 / 4 / 1 useful bytes and the ~400 KB of streams per SM thrash L1.
// Here a CTA of 128 threads owns 1024 consecutive samples: positions and segment ids are staged in shared memory
// once with coalesced loads and re-used for kStLevels levels; per level the d(feature) row and the saved grid
// features are staged the same way.  Each thread then walks its 8 consecutive samples out of shared memory
// (per-thread rows padded by one element: conflict-free) with the same run-length / shared-corner accumulation.
constexpr int kStThreads = 128, kStChunk = 8, kStSamples = kStThreads * kStChunk, kStLevels = 4, kStRow = kStChunk + 1;

struct __align__(16) StagedSmem {
  float4 pos[kStThreads * kStRow];
  float2 df[kStThreads * kStRow];
  uint32_t eg[kStThreads * kStRow];
  uint8_t seg[kStSamples];
  float2 vv[kStThreads * kStRow];  // only with tap staging (the dynamic allocation stops before it otherwise)
};
constexpr int kStSmemBase = (int)offsetof(StagedSmem, vv), kStSmemTaps = (int)sizeof(StagedSmem);

__global__ void __launch_bounds__(kStThreads, 6) grid_scatter_staged_kernel(const __grid_constant__ ScatterArgs a) {
  extern __shared__ __align__(16) unsigned char staged_raw[];
  StagedSmem& sm = *reinterpret_cast<StagedSmem*>(staged_raw);
  const hrf_field& f = a.f;
  const int64_t n = live_samples(a.s);
  const int64_t ns = a.s.num_samples;   // row length of the level-major workspace
  const int64_t base = (int64_t)blockIdx.x * kStSamples;
  if (base >= n) return;
  const int tid = threadIdx.x;
  const int k = a.grid_first + (int)blockIdx.y % a.grid_count;
  const int l0 = ((int)blockIdx.y / a.grid_count) * kStLevels;
  const int axis = (k == 0) ? 3 : (k == 1) ? 2 : (k == 2) ? 0 : 1;  // vector axis paired with grid k
  const int valid = (int)((n - base) < kStSamples ? (n - base) : kStSamples);

  for (int s = tid; s < kStSamples; s += kStThreads) {
    const bool ok = s < valid;
    sm.pos[(s >> 3) * kStRow + (s & 7)] = ok ? __ldg(a.pos4 + base + s) : make_float4(0.f, 0.f, 0.f, 0.f);
    sm.seg[s] = ok ? a.seg8[base + s] : (uint8_t)255;
  }

  const int row = tid * kStRow;
  const int cnt = min(max(valid - tid * kStChunk, 0), kStChunk);
#pragma unroll 1
  for (int li = 0; li < kStLevels; ++li) {
    const int l = l0 + li;
    __syncthreads();  // the previous level's readers are done with df / eg
    {
      const float2* __restrict__ dfl = a.dfeat + (size_t)l * ns + base;
      for (int s = tid; s < valid; s += kStThreads) sm.df[(s >> 3) * kStRow + (s & 7)] = __ldg(dfl + s);
      if (a.egrid != nullptr) {
        const uint32_t* __restrict__ eg = a.egrid + (size_t)(4 * l + k) * a.egrid_stride;
        if (a.feat_index == nullptr) {
          for (int s = tid; s < valid; s += kStThreads) sm.eg[(s >> 3) * kStRow + (s & 7)] = __ldg(eg + base + s);
        } else {   // survivors of a pruning pass: their columns in the candidates' buffer (mostly consecutive)
          for (int s = tid; s < valid; s += kStThreads)
            sm.eg[(s >> 3) * kStRow + (s & 7)] = __ldg(eg + __ldg(a.feat_index + base + s));
        }
      }
      if (a.tapstage) {
        // the interpolated vector value of every sample, fetched here with 8 independent taps in flight per thread:
        // the run loop below then has no global load on its critical path (ncu: long-scoreboard was the top stall)
#pragma unroll
        for (int r = 0; r < kStChunk; ++r) {
          const int s = tid + r * kStThreads;
          float2 v = make_float2(0.f, 0.f);
          const uint32_t sgi = sm.seg[s];
          if (sgi != 255u) {
            const float4 p4 = sm.pos[(s >> 3) * kStRow + (s & 7)];
            const float cv = (axis == 0) ? p4.x : (axis == 1) ? p4.y : (axis == 2) ? p4.z : p4.w;
            v = lerp_tap(f.segments[sgi].vectors, make_tap(cv, f.vec_res, axis), 2 * l);
          }
          sm.vv[(s >> 3) * kStRow + (s & 7)] = v;
        }
      }
    }
    __syncthreads();
    const float scale = f.level_scale[l];
    const uint32_t res = f.level_res[l];

    // state of the current run
    uint32_t cur_sgi = 255u;
    const hrf_segment* sg = nullptr;
    uint32_t ca = 0xffffffffu, cb = 0, cc = 0;  // current cell
    uint32_t idx[8], raw[8];
    float accx[8], accy[8];
    float* gtab = nullptr;
    const uint32_t* tab = nullptr;
    const float* vecs = nullptr;
    uint32_t lsize = 0;
    bool hashed = false;
    // vector-tap run
    uint32_t to0 = 0xffffffffu, to1 = 0;
    float* gvec = nullptr;
    float2 tv0 = make_float2(0.f, 0.f), tv1 = make_float2(0.f, 0.f);
    float va0 = 0.f, va1 = 0.f, vb0 = 0.f, vb1 = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) accx[q] = accy[q] = 0.f, idx[q] = raw[q] = 0u;

    auto flush_cell = [&]() {
      if (gtab != nullptr) {
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          if (accx[q] != 0.f || accy[q] != 0.f) red_add2(gtab + 2 * (size_t)idx[q], accx[q], accy[q]);
          accx[q] = accy[q] = 0.f;
        }
      }
    };
    auto flush_tap = [&]() {
      if (gvec != nullptr && to0 != 0xffffffffu) {
        if (va0 != 0.f || va1 != 0.f) red_add2(gvec + to0 + 2 * l, va0, va1);
        if (vb0 != 0.f || vb1 != 0.f) red_add2(gvec + to1 + 2 * l, vb0, vb1);
      }
      va0 = va1 = vb0 = vb1 = 0.f;
    };

#pragma unroll 1
    for (int j = 0; j < cnt; ++j) {
      const uint32_t sgi = sm.seg[tid * kStChunk + j];
      if (sgi == 255u) continue;
      const float4 p4 = sm.pos[row + j];
      const float2 dO = sm.df[row + j];
      const float c0 = (k == 2) ? p4.y : p4.x;                       // grid coordinates (decomposition4d.py:126-129)
      const float c1 = (k == 0 || k == 1) ? p4.y : p4.z;
      const float c2 = (k == 0) ? p4.z : p4.w;
      const float cv = (axis == 0) ? p4.x : (axis == 1) ? p4.y : (axis == 2) ? p4.z : p4.w;
      const Cell A = to_cell(scale, c0), B = to_cell(scale, c1), C = to_cell(scale, c2);
      const bool new_seg = sgi != cur_sgi;
      if (new_seg || A.g != ca || B.g != cb || C.g != cc) {  // new cell: flush what leaves, fetch the corners
        const int dA = (int)(A.g - ca), dB = (int)(B.g - cb), dC = (int)(C.g - cc);
        if (a.carry && !new_seg && dA >= -1 && dA <= 1 && dB >= -1 && dB <= 1 && dC >= -1 && dC <= 1) {
          if (dA != 0) shift_corners<1>(dA, gtab, idx, accx, accy);
          if (dB != 0) shift_corners<2>(dB, gtab, idx, accx, accy);
          if (dC != 0) shift_corners<4>(dC, gtab, idx, accx, accy);
        } else {
          flush_cell();
        }
        if (new_seg) {  // per-segment constants of this level
          flush_tap();
          to0 = 0xffffffffu;
          sg = f.segments + sgi;
          const uint32_t off = sg->level_offset[l];
          lsize = sg->level_size[l];
          hashed = ((sg->hashed_mask >> l) & 1u) != 0u;
          tab = sg->grid[k] + off;
          vecs = sg->vectors;
          gvec = a.seg_grads[sgi].vectors;
          gtab = a.seg_grads[sgi].grid[k] + 2 * (size_t)off;
          cur_sgi = sgi;
        }
        corner_indices(hashed, res, lsize, A, B, C, idx);
        if (a.egrid == nullptr) {
#pragma unroll
          for (int q = 0; q < 8; ++q) raw[q] = __ldg(tab + idx[q]);
        }
        ca = A.g, cb = B.g, cc = C.g;
      }
      const VecTap tp = make_tap(cv, f.vec_res, axis);
      if (tp.o0 != to0 || tp.o1 != to1) {  // new tap pair: flush its gradient run, fetch the two rows once
        flush_tap();
        to0 = tp.o0, to1 = tp.o1;
        if (!a.tapstage) {
          tv0 = __ldg(reinterpret_cast<const float2*>(vecs + to0 + 2 * l));
          tv1 = __ldg(reinterpret_cast<const float2*>(vecs + to1 + 2 * l));
        }
      }
      const float2 v = a.tapstage ? sm.vv[row + j]
                                  : make_float2(tv0.x + tp.frac * (tv1.x - tv0.x), tv0.y + tp.frac * (tv1.y - tv0.y));
      float w[8];
      corner_weights(A, B, C, w);
      const float gx = v.x * dO.x, gy = v.y * dO.y;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        accx[q] = __fmaf_rn(w[q], gx, accx[q]);
        accy[q] = __fmaf_rn(w[q], gy, accy[q]);
      }
      float ex = 0.f, ey = 0.f;
      if (a.egrid != nullptr) {  // interpolated grid features saved by the forward
        const uint32_t ev = sm.eg[row + j];
        ex = bf16_lo(ev), ey = bf16_hi(ev);
      } else {
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          ex = __fmaf_rn(w[q], bf16_lo(raw[q]), ex);
          ey = __fmaf_rn(w[q], bf16_hi(raw[q]), ey);
        }
      }
      // d vectors[axis][i0/i1][2l..2l+1] = e_k * dOut * (1-frac | frac)   (tensor_composition.cu:109-111)
      const float dx = ex * dO.x, dy = ey * dO.y;
      va0 = __fmaf_rn(dx, 1.f - tp.frac, va0), va1 = __fmaf_rn(dy, 1.f - tp.frac, va1);
      vb0 = __fmaf_rn(dx, tp.frac, vb0), vb1 = __fmaf_rn(dy, tp.frac, vb1);
    }
    flush_cell();
    flush_tap();
  }
}

// kLevelUnroll: levels unrolled in the re-encode loop (only taken when the forward's features were not saved)
template <int kLevelUnroll = 4>
__global__ void __launch_bounds__(kTile, 2) field_backward_kernel(const __grid_constant__ BwdArgs args) {
  extern __shared__ unsigned char smem_raw[];
  BwdSmem& sm = *reinterpret_cast<BwdSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x;
  const hrf_field& f = args.f;
  const uint32_t roff = a_row_off(tid);

  if (tid == 0) {
    mbar_init(&sm.bar_w, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(&sm.bar_w, w_blob_bytes(f.color_in_width));
    tma_load_1d(sm.w, f.mlp_blob, w_blob_bytes(f.color_in_width), &sm.bar_w);
  }
  const uint32_t wbase = smem_u32(sm.w);
  const uint32_t a_feat = smem_u32(sm.feat), a_cin = smem_u32(sm.cin), a_hs = smem_u32(sm.hs),
                 a_h1 = smem_u32(sm.h1), a_h2 = smem_u32(sm.h2), a_g3 = smem_u32(sm.g3), a_gs = smem_u32(sm.gs);
  bool weights_ready = false, have_acc = false;
  // weight-gradient accumulators, M = 64 wgmma fragments (see wgmma_bf16), summed over every tile of the CTA
  float gw1s[16], gw2s[8], gw1c[24], gw2c[32], gw3c[8];   // dW1s [64 out,32 in], dW2s^T [64 in,16 out],
#pragma unroll                                             // dW1c [64 out,K1 in], dW2c [64,64], dW3c^T [64 in,16 out]
  for (int q = 0; q < 32; ++q) {
    if (q < 16) gw1s[q] = 0.f;
    if (q < 8) gw2s[q] = 0.f, gw3c[q] = 0.f;
    if (q < 24) gw1c[q] = 0.f;
    gw2c[q] = 0.f;
  }
  const int K1 = f.color_in_width;

  const int64_t n = live_samples(args.s);
  const int64_t ns = args.s.num_samples;   // row length of the level-major workspace
  const int64_t num_tiles = (n + kTile - 1) / kTile;
  for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int64_t i = tile * kTile + tid;
    const bool valid = i < n;
    const Sample s = load_sample(f, args.s, i, n);
    if (valid) {
      args.pos4[i] = make_float4(s.x, s.y, s.z, s.t);
      args.seg8[i] = s.seg != nullptr ? (uint8_t)(s.seg - f.segments) : (uint8_t)255;
    }
    if (args.feat_in != nullptr) {
      const int64_t row = !(valid && s.seg != nullptr) ? -1 : (args.feat_index != nullptr ? (int64_t)__ldg(args.feat_index + i) : i);
#pragma unroll
      for (int kg = 0; kg < 4; ++kg)
        *reinterpret_cast<uint4*>(sm.feat + kg * kAChunk + roff) =
            row >= 0 ? __ldg(args.feat_in + row * 4 + kg) : make_uint4(0, 0, 0, 0);
    } else {
      encode_to_smem<false, kLevelUnroll>(f, s, sm.feat, tid);
    }
    // Everything else this tile will read from global memory is requested here, before the ten MMA rounds: each round
    // ends in asm statements that clobber memory, so the compiler cannot move a later load above them, and at 8 warps
    // per SM a load issued where its value is needed is a fully exposed round trip.
    const View vw = load_view(f, args.s, i, n);
    float up_sigma = 0.f, up_rgb[3] = {0.f, 0.f, 0.f};
    if (valid) {
      if (args.d_sigma != nullptr) up_sigma = __ldg(args.d_sigma + i);
      if (args.d_rgb != nullptr) up_rgb[0] = __ldg(args.d_rgb + 3 * i), up_rgb[1] = __ldg(args.d_rgb + 3 * i + 1), up_rgb[2] = __ldg(args.d_rgb + 3 * i + 2);
    }
    if (!weights_ready) {
      mbar_wait(&sm.bar_w, 0);
      weights_ready = true;
    }
    float d[64], o[16];
    // ---------------- forward recompute ----------------
    mma_begin();
    mma_layer<64, 32>(d, a_feat, wbase + kWSig1);
    mma_end();
    wgmma_fence_regs<64>(d);
    frag_store_relu64(sm.hs, d);
    mma_begin();
    mma_layer<16, 64>(d, a_hs, wbase + kWSig2);
    mma_end();
    wgmma_fence_regs<16>(d);
    frag_stage<16, 16>(reinterpret_cast<float*>(sm.h1), d);   // h1 is written by the next round only
    __syncthreads();
    stage_read_row<16>(reinterpret_cast<const float*>(sm.h1), o);
    const float h0 = o[0];
    write_color_input(f, sm.cin, roff, vw, o);
    mma_begin();
    if (K1 == 48) mma_layer<64, 48>(d, a_cin, wbase + kWCol1);
    else mma_layer<64, 32>(d, a_cin, wbase + kWCol1);
    mma_end();
    wgmma_fence_regs<64>(d);
    frag_store_relu64(sm.h1, d);
    mma_begin();
    mma_layer<64, 64>(d, a_h1, wbase + w_col2(K1));
    mma_end();
    wgmma_fence_regs<64>(d);
    frag_store_relu64(sm.h2, d);
    mma_begin();
    mma_layer<16, 64>(d, a_h2, wbase + w_col3(K1));
    mma_end();
    wgmma_fence_regs<16>(d);
    frag_stage<16, 4>(reinterpret_cast<float*>(sm.gs), d);    // colour pre-activation 0..2; gs is written much later
    __syncthreads();
    stage_read_row<4>(reinterpret_cast<const float*>(sm.gs), o);

    // ---------------- backward ----------------
    {  // d(colour pre-activation) = d_rgb * rgb * (1 - rgb), cols 3..15 = 0
      float d3[3] = {0.f, 0.f, 0.f};
      if (valid && args.d_rgb != nullptr) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float r = 1.f / (1.f + __expf(-o[c]));
          d3[c] = up_rgb[c] * r * (1.f - r);
        }
      }
      *reinterpret_cast<uint4*>(sm.g3 + 0 * kAChunk + roff) =
          make_uint4(pack_bf16x2(d3[0], d3[1]), pack_bf16x2(d3[2], 0.f), 0u, 0u);
      *reinterpret_cast<uint4*>(sm.g3 + 1 * kAChunk + roff) = make_uint4(0u, 0u, 0u, 0u);
    }
    wgmma_fence_regs<8>(gw3c);
    mma_begin();
    issue_wgrad<16>(gw3c, a_h2, a_g3);                          // dW3c^T += H2^T dO3
    issue_dgrad<64, 16>(d, a_g3, wbase + w_col3(K1));           // dH2 = dO3 W3c
    mma_end();
    wgmma_fence_regs<8>(gw3c);
    wgmma_fence_regs<64>(d);
    frag_relu_backward64(sm.h2, d);
    wgmma_fence_regs<32>(gw2c);
    mma_begin();
    issue_wgrad<64>(gw2c, a_h2, a_h1);                          // dW2c += dH2^T H1
    issue_dgrad<64, 64>(d, a_h2, wbase + w_col2(K1));           // dH1 = dH2 W2c
    mma_end();
    wgmma_fence_regs<32>(gw2c);
    wgmma_fence_regs<64>(d);
    frag_relu_backward64(sm.h1, d);
    wgmma_fence_regs<24>(gw1c);
    mma_begin();
    if (K1 == 48) {
      issue_wgrad<48>(gw1c, a_h1, a_cin);                       // dW1c += dH1^T Cin
      issue_dgrad<48, 64>(d, a_h1, wbase + kWCol1);             // dCin = dH1 W1c
    } else {
      issue_wgrad<32>(gw1c, a_h1, a_cin);
      issue_dgrad<32, 64>(d, a_h1, wbase + kWCol1);
    }
    mma_end();
    wgmma_fence_regs<24>(gw1c);
    wgmma_fence_regs<48>(d);
    {
      // colour-input columns 16..47 (geometry features, camera embedding) staged in h2, free since the last round
      float dc[48];
      if (K1 == 48) frag_stage<48, 32, 16>(reinterpret_cast<float*>(sm.h2), d);
      else frag_stage<32, 32, 16>(reinterpret_cast<float*>(sm.h2), d);
      __syncthreads();
      stage_read_row<32>(reinterpret_cast<const float*>(sm.h2), dc + 16);
      if (args.d_emb != nullptr && vw.cam >= 0) {  // d(camera embedding): colour-input features 31..30+E
        const int E = f.camera_embedding_dim;
#pragma unroll
        for (int e = 0; e < HRF_MAX_CAMERA_EMBEDDING_DIM; ++e)
          if (e < E) atomicAdd(args.d_emb + (size_t)vw.cam * E + e, dc[31 + e]);
      }
      // d(sigma-net output): col 0 from the density (truncated_exp backward, activation.py:21), 1..15 = d geo: what the
      // colour net sends back plus the caller's own gradient of QueryOutput.geometry_features (humanrf.py:185-186)
      if (args.d_geo != nullptr && valid) {
#pragma unroll
        for (int j = 0; j < HRF_GEO_DIM; ++j) dc[16 + j] += __ldg(args.d_geo + i * HRF_GEO_DIM + j);
      }
      float dh0 = 0.f;
      if (valid && args.d_sigma != nullptr)
        dh0 = up_sigma * f.density_scale * __expf(fminf(fmaxf(h0, -15.f), 15.f));
      *reinterpret_cast<uint4*>(sm.gs + 0 * kAChunk + roff) = make_uint4(
          pack_bf16x2(dh0, dc[16]), pack_bf16x2(dc[17], dc[18]), pack_bf16x2(dc[19], dc[20]), pack_bf16x2(dc[21], dc[22]));
      *reinterpret_cast<uint4*>(sm.gs + 1 * kAChunk + roff) = make_uint4(
          pack_bf16x2(dc[23], dc[24]), pack_bf16x2(dc[25], dc[26]), pack_bf16x2(dc[27], dc[28]), pack_bf16x2(dc[29], dc[30]));
    }
    wgmma_fence_regs<8>(gw2s);
    mma_begin();
    issue_wgrad<16>(gw2s, a_hs, a_gs);                          // dW2s^T += Hs^T dOs
    issue_dgrad<64, 16>(d, a_gs, wbase + kWSig2);               // dHs = dOs W2s
    mma_end();
    wgmma_fence_regs<8>(gw2s);
    wgmma_fence_regs<64>(d);
    frag_relu_backward64(sm.hs, d);
    wgmma_fence_regs<16>(gw1s);
    mma_begin();
    issue_wgrad<32>(gw1s, a_hs, a_feat);                        // dW1s += dHs^T feat
    issue_dgrad<32, 64>(d, a_hs, wbase + kWSig1);               // dFeat = dHs W1s
    mma_end();
    wgmma_fence_regs<16>(gw1s);
    wgmma_fence_regs<32>(d);
    have_acc = true;
    {
      // d(composed features) -> global, level-major [16][N] float2 (coalesced here and in grid_scatter_kernel)
      float df[32];
      frag_stage<32, 32>(reinterpret_cast<float*>(sm.h1), d);   // h1 is free until the next tile's recompute
      __syncthreads();
      stage_read_row<32>(reinterpret_cast<const float*>(sm.h1), df);
      if (valid) {
#pragma unroll
        for (int l = 0; l < 16; ++l) args.dfeat[(size_t)l * ns + i] = make_float2(df[2 * l], df[2 * l + 1]);
      }
    }
  }

  if (!weights_ready) mbar_wait(&sm.bar_w, 0);
  // ---------------- flush the weight-gradient accumulators ----------------
  if (have_acc && args.d_mlp != nullptr) {
    // Every CTA adds its 11 264 partial sums into the same 44 KB at the same moment (persistent CTAs finish together):
    // the two adjacent columns a thread holds go out as one 8-byte RED where the destination row is contiguous.
    const bool v2ok = (reinterpret_cast<uintptr_t>(args.d_mlp) & 7u) == 0;
    const int gcol2 = kGCol1 + 64 * K1, gcol3 = gcol2 + 4096;
    flush_rows<16>(args.d_mlp + kGSig1, 32, gw1s, 32, v2ok);
    flush_cols(args.d_mlp + kGSig2, gw2s);
    flush_rows<24>(args.d_mlp + kGCol1, K1, gw1c, K1, v2ok);
    flush_rows<32>(args.d_mlp + gcol2, 64, gw2c, 64, v2ok);
    flush_cols(args.d_mlp + gcol3, gw3c);
  }
}

}  // namespace hrf

using namespace hrf;

extern "C" int hrf_field_backward_mlp(const hrf_field* f, const hrf_samples* s, const float* d_sigma, const float* d_rgb,
                                      const float* d_geo, const void* feat_bf16, const int32_t* feat_index, float* d_mlp,
                                      float* d_camera_embeddings, void* workspace, void* stream) {
  HRF_REQUIRE(f != nullptr && s != nullptr, "null argument");
  HRF_REQUIRE(f->num_segments < 255, "at most 254 temporal segments");
  if (s->num_samples == 0) return 0;
  HRF_REQUIRE(workspace != nullptr, "hrf_field_backward needs a workspace of 160 bytes per sample");
  HRF_REQUIRE(d_sigma != nullptr || d_rgb != nullptr || d_geo != nullptr, "no upstream gradient given");
  if (s->ray_origins == nullptr) {
    HRF_REQUIRE(s->positions && s->frame_numbers, "query form needs positions and frame numbers");
    HRF_REQUIRE(d_rgb == nullptr || s->directions, "radiance gradients need directions");
  }
  BwdArgs a;
  a.f = *f;
  a.s = *s;
  a.seg_grads = nullptr;
  a.d_sigma = d_sigma;
  a.d_rgb = d_rgb;
  a.d_geo = d_geo;
  a.feat_in = reinterpret_cast<const uint4*>(feat_bf16);
  a.feat_index = feat_bf16 != nullptr ? feat_index : nullptr;
  a.d_mlp = d_mlp;
  a.d_emb = d_camera_embeddings;
  a.dfeat = reinterpret_cast<float2*>(workspace);
  a.pos4 = reinterpret_cast<float4*>(reinterpret_cast<char*>(workspace) + 128 * (size_t)s->num_samples);
  a.seg8 = reinterpret_cast<uint8_t*>(reinterpret_cast<char*>(workspace) + 144 * (size_t)s->num_samples);
  const int64_t tiles = (s->num_samples + kTile - 1) / kTile;
  const int smem = (int)sizeof(BwdSmem) + 1024;
  const int64_t max_ctas = (int64_t)sm_count() * 2;
  const int grid = (int)(tiles < max_ctas ? tiles : max_ctas);
  // HRF_BWD_UNROLL=1: experiment for round 2 (the forward gained 19 % from the smaller loop; this kernel is 155 KB of SASS)
  static const bool compact = [] { const char* e = getenv("HRF_BWD_UNROLL"); return e && e[0] == '1'; }();
  if (compact) {
    HRF_CUDA(cudaFuncSetAttribute(field_backward_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    field_backward_kernel<1><<<grid, kTile, smem, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  } else {
    HRF_CUDA(cudaFuncSetAttribute(field_backward_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    field_backward_kernel<4><<<grid, kTile, smem, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  }
  HRF_CHECK_LAUNCH();
  return 0;
}

int hrf_launch_scatter_v2(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads, const void* grid_feat_bf16,
                          const int32_t* feat_index, int64_t grid_feat_stride, const void* workspace, int grid_first, int grid_count,
                          cudaStream_t st);   // scatter_v2.cu
int hrf_launch_scatter_v3(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads, const void* grid_feat_bf16,
                          const int32_t* feat_index, int64_t grid_feat_stride, const void* workspace, int grid_first, int grid_count,
                          cudaStream_t st);   // scatter_v3.cu
int hrf_launch_scatter_v4(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads, const void* grid_feat_bf16,
                          const int32_t* feat_index, int64_t grid_feat_stride, const void* workspace, int grid_first, int grid_count,
                          cudaStream_t st);   // scatter_v4.cu
int hrf_launch_scatter_v5(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads, const void* grid_feat_bf16,
                          const int32_t* feat_index, int64_t grid_feat_stride, const void* workspace, int grid_first, int grid_count,
                          cudaStream_t st);   // scatter_v5.cu
#ifndef HRF_SCATTER_DEFAULT
#define HRF_SCATTER_DEFAULT 5   // the fastest generation on the train bench on an H100 (DESIGN.md section 3.3)
#endif

extern "C" int hrf_field_backward_tables(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads,
                                         const void* grid_feat_bf16, const int32_t* feat_index, int64_t grid_feat_stride,
                                         const void* workspace, int grid_first, int grid_count, void* stream) {
  HRF_REQUIRE(f != nullptr && s != nullptr && seg_grads != nullptr, "null argument");
  HRF_REQUIRE(grid_first >= 0 && grid_count >= 1 && grid_first + grid_count <= 4, "grids are 0..3 (xyz, xyt, yzt, xzt)");
  if (s->num_samples == 0) return 0;
  HRF_REQUIRE(workspace != nullptr, "needs the workspace hrf_field_backward_mlp filled");
  // HRF_SCATTER = 5 | 4 | 3 | 2 | 1 (read per call: the tests switch it): scatter_v5.cu ... scatter_v2.cu, the
  // first-generation kernels below.  All stay built: each is the others' cross-check in tests/test_scatter_gpu.py.
  const int gen = [] { const char* e = getenv("HRF_SCATTER"); const int v = e ? atoi(e) : HRF_SCATTER_DEFAULT; return (v >= 1 && v <= 5) ? v : HRF_SCATTER_DEFAULT; }();
  if (gen == 5)
    return hrf_launch_scatter_v5(f, s, seg_grads, grid_feat_bf16, feat_index, grid_feat_stride, workspace, grid_first, grid_count,
                                 reinterpret_cast<cudaStream_t>(stream));
  if (gen == 4)
    return hrf_launch_scatter_v4(f, s, seg_grads, grid_feat_bf16, feat_index, grid_feat_stride, workspace, grid_first, grid_count,
                                 reinterpret_cast<cudaStream_t>(stream));
  if (gen == 3)
    return hrf_launch_scatter_v3(f, s, seg_grads, grid_feat_bf16, feat_index, grid_feat_stride, workspace, grid_first, grid_count,
                                 reinterpret_cast<cudaStream_t>(stream));
  if (gen == 2)
    return hrf_launch_scatter_v2(f, s, seg_grads, grid_feat_bf16, feat_index, grid_feat_stride, workspace, grid_first, grid_count,
                                 reinterpret_cast<cudaStream_t>(stream));
  ScatterArgs sa;
  sa.f = *f;
  sa.s = *s;
  sa.seg_grads = seg_grads;
  sa.dfeat = reinterpret_cast<const float2*>(workspace);
  sa.pos4 = reinterpret_cast<const float4*>(reinterpret_cast<const char*>(workspace) + 128 * (size_t)s->num_samples);
  sa.seg8 = reinterpret_cast<const uint8_t*>(reinterpret_cast<const char*>(workspace) + 144 * (size_t)s->num_samples);
  sa.egrid = reinterpret_cast<const uint32_t*>(grid_feat_bf16);
  sa.feat_index = grid_feat_bf16 != nullptr ? feat_index : nullptr;
  sa.egrid_stride = grid_feat_stride > 0 ? grid_feat_stride : s->num_samples;
  sa.grid_first = grid_first;
  sa.grid_count = grid_count;
  const int kChunk = [] { const char* e = getenv("HRF_SCATTER_CHUNK"); const int v = e ? atoi(e) : 0; return v > 0 ? v : kChunkDefault; }();
  sa.chunk = kChunk;
  const int kCarry = [] { const char* e = getenv("HRF_SCATTER_CARRY"); return (e && e[0] == '0') ? 0 : 1; }();
  sa.carry = kCarry;
  const bool staged = [] { const char* e = getenv("HRF_SCATTER_STAGED"); return !(e && e[0] == '0'); }();
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  sa.tapstage = [] { const char* e = getenv("HRF_SCATTER_TAPSTAGE"); return (e && e[0] == '1') ? 1 : 0; }();
  if (staged) {
    const int64_t blocks = (s->num_samples + kStSamples - 1) / kStSamples;
    const int smem = sa.tapstage ? kStSmemTaps : kStSmemBase;
    grid_scatter_staged_kernel<<<dim3((unsigned)blocks, (HRF_N_LEVELS / kStLevels) * grid_count), kStThreads, smem, st>>>(sa);
  } else {
    const int64_t chunks = (s->num_samples + kChunk - 1) / kChunk;
    grid_scatter_kernel<<<dim3((unsigned)((chunks + 255) / 256), HRF_N_LEVELS * grid_count), 256, 0, st>>>(sa);
  }
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_field_backward(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads,
                                  const float* d_sigma, const float* d_rgb, const float* d_geo, const void* feat_bf16,
                                  const void* grid_feat_bf16, const int32_t* feat_index, int64_t grid_feat_stride,
                                  float* d_mlp, float* d_camera_embeddings, void* workspace, void* stream) {
  HRF_REQUIRE(seg_grads != nullptr, "null argument");
  if (int rc = hrf_field_backward_mlp(f, s, d_sigma, d_rgb, d_geo, feat_bf16, feat_index, d_mlp, d_camera_embeddings, workspace,
                                      stream))
    return rc;
  return hrf_field_backward_tables(f, s, seg_grads, grid_feat_bf16, feat_index, grid_feat_stride, workspace, 0, 4, stream);
}
