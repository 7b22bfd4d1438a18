// Table / vector gradient scatter, fourth generation (replaces tcnn kernel_grid_backward + compose_tensors_backward,
// tensor_composition.cu:57-118).  Same arithmetic as scatter_v3.cu; the change is OCCUPANCY.
//
// v3 looks latency-bound (few eligible warps per scheduler and cycle): 96 registers per thread (8 table indices + 16 accumulators + run state) allow 5 CTAs x 4 warps per SM, and
// three attempts to hide the remaining latencies inside a thread (prefetching, cp.async double buffering, shared-memory
// descriptors) changed nothing.  Here the 8 parity slots of a sample chunk are split over TWO threads: warps 0-3 of a
// 256-thread CTA own the slots whose third-axis vertex is even, warps 4-7 the odd ones (4 indices + 8 accumulators each).
// Warp w and warp w+4 walk the same 256 samples out of the same shared-memory rows; they stage them together (half the
// rows each) and meet at a 64-thread named barrier.  The vector-row gradient belongs to the even half (it needs the
// whole per-grid feature, which the saved egrid provides); when the tables are re-gathered instead, each half adds its
// partial blend.
#include <cstddef>
#include <cstdlib>

#include "field_common.cuh"

namespace hrf {

constexpr int kV4Threads = 256, kV4Chunk = 8, kV4Samples = 128 * kV4Chunk, kV4Levels = 8, kV4Row = kV4Chunk + 1;

struct ScatterV4Args {
  hrf_field f;
  hrf_samples s;
  const hrf_segment_grads* seg_grads;
  const float2* dfeat;        // [16 levels][stride] float2, written by field_backward_kernel
  const float4* pos4;         // [N] (x,y,z,t)
  const uint8_t* seg8;        // [N]
  const uint32_t* egrid;      // bf16x2 [16*4][egrid_stride] per-grid features of a forward pass, or NULL (re-gather)
  const int32_t* feat_index;  // column of sample i inside egrid, or NULL
  int64_t egrid_stride;
  int grid_first, grid_count;
};

struct __align__(16) V4Smem {
  float4 pos[128 * kV4Row];
  float2 df[128 * kV4Row];
  uint32_t eg[128 * kV4Row];
  uint8_t seg[kV4Samples];
};

__device__ __forceinline__ void red2v4(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b));
}
// The two warps that share 256 samples meet here.  Barrier ids 0..3 as IMMEDIATES: with a register operand ptxas reserves
// all 16 hardware barriers for the CTA (one CTA per SM); 4 per CTA x 4 CTAs is exactly what an SM has.  (__syncthreads,
// which is barrier 0, is not used in this kernel.)
__device__ __forceinline__ void pair_sync(int pair) {
  switch (pair) {
    case 0: asm volatile("bar.sync 0, 64;" ::: "memory"); break;
    case 1: asm volatile("bar.sync 1, 64;" ::: "memory"); break;
    case 2: asm volatile("bar.sync 2, 64;" ::: "memory"); break;
    default: asm volatile("bar.sync 3, 64;" ::: "memory"); break;
  }
}

struct RowTap4 {
  uint32_t i0, i1;
  float frac;
};
__device__ __forceinline__ RowTap4 make_row_tap4(float coord, int vec_res) {
  const float c = __fmaf_rn(coord, (float)vec_res, -0.5f);
  const float fl = floorf(c);
  RowTap4 t;
  t.frac = c - fl;
  t.i0 = (uint32_t)min(max((int)fmaxf(fl, 0.f), 0), vec_res - 1);
  t.i1 = (uint32_t)min(max((int)fminf(fl + 1.f, (float)(vec_res - 1)), 0), vec_res - 1);
  return t;
}

// Table entries of the 4 vertices of a cell whose third-axis vertex has parity kZ, in parity-slot order (slot bit 0 = parity
// of the first-axis vertex, bit 1 = of the second-axis vertex).  hashed: tcnn's coherent prime hash; dense: one
// conditional subtraction (cell inside the grid, see corner_indices).
template <int kZ>
__device__ __forceinline__ void slot_indices4(Cell A, Cell B, Cell C, bool hashed, uint32_t mulY, uint32_t mulZ, uint32_t hmask,
                                              uint32_t lsize, uint32_t (&v)[4]) {
  const uint32_t nx0 = (A.g + 1u) & ~1u, nx1 = A.g | 1u;
  const uint32_t ny0 = ((B.g + 1u) & ~1u) * mulY, ny1 = (B.g | 1u) * mulY;
  const uint32_t nz = (kZ ? (C.g | 1u) : ((C.g + 1u) & ~1u)) * mulZ;
  if (hashed) {
#pragma unroll
    for (int q = 0; q < 4; ++q) v[q] = (((q & 1) ? nx1 : nx0) ^ ((q & 2) ? ny1 : ny0) ^ nz) & hmask;
  } else {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t t = ((q & 1) ? nx1 : nx0) + ((q & 2) ? ny1 : ny0) + nz;
      v[q] = t >= lsize ? t - lsize : t;
    }
  }
}

// cold path: a sample outside a dense level's grid (all 8 corners, the forward's general index wrap); even half only
template <bool kGather>
__device__ __noinline__ void scatter_sample_slow4(const uint32_t* tab, float* gtab, float* gvec, const float* vecs, bool hashed,
                                                  uint32_t res, uint32_t lsize, Cell A, Cell B, Cell C, VecTap tp, int l, float2 dO,
                                                  uint32_t ev) {
  uint32_t idx[8];
  float w[8];
  corner_indices(hashed, res, lsize, A, B, C, idx);
  corner_weights(A, B, C, w);
  const float2 v0 = __ldg(reinterpret_cast<const float2*>(vecs + tp.o0 + 2 * l)), v1 = __ldg(reinterpret_cast<const float2*>(vecs + tp.o1 + 2 * l));
  const float gx = (v0.x + tp.frac * (v1.x - v0.x)) * dO.x, gy = (v0.y + tp.frac * (v1.y - v0.y)) * dO.y;
  float ex = bf16_lo(ev), ey = bf16_hi(ev);
  if (kGather) {
    ex = ey = 0.f;
    for (int q = 0; q < 8; ++q) {
      const uint32_t r = __ldg(tab + idx[q]);
      ex = __fmaf_rn(w[q], bf16_lo(r), ex), ey = __fmaf_rn(w[q], bf16_hi(r), ey);
    }
  }
  for (int q = 0; q < 8; ++q) red2v4(gtab + 2 * (size_t)idx[q], w[q] * gx, w[q] * gy);
  const float dx = ex * dO.x, dy = ey * dO.y;
  red2v4(gvec + tp.o0 + 2 * l, dx * (1.f - tp.frac), dy * (1.f - tp.frac));
  red2v4(gvec + tp.o1 + 2 * l, dx * tp.frac, dy * tp.frac);
}

// kGrid: 0 xyz, 1 xyt, 2 yzt, 3 xzt (decomposition4d.py:126-129); its vector axis is t, z, x, y (tensor_composition.cu:49-52)
template <int kGrid, bool kGather, int kZ>
__device__ __forceinline__ void scatter_levels4(const ScatterV4Args& a, V4Smem& sm, int l0, int64_t base, int valid) {
  const hrf_field& f = a.f;
  const int tid = threadIdx.x & 127;          // position inside the half (same samples in both halves)
  const int pair = tid >> 5, lane = tid & 31;
  const int64_t ns = a.s.num_samples;
  constexpr int kAxis = (kGrid == 0) ? 3 : (kGrid == 1) ? 2 : (kGrid == 2) ? 0 : 1;
  constexpr bool kVec = kGather || kZ == 0;   // who accumulates the vector-row gradient
  const int row = tid * kV4Row;
  const int cnt = min(max(valid - tid * kV4Chunk, 0), kV4Chunk);
  const int w0 = (tid & ~31) * kV4Chunk;
  constexpr int kHalf = kV4Chunk / 2, r0 = kZ * kHalf;   // this warp stages rows r0 .. r0+3 of the pair's 8
  int32_t col4[kHalf];
  if (!kGather) {
#pragma unroll
    for (int r = 0; r < kHalf; ++r) {
      const int s = w0 + lane + 32 * (r0 + r);
      col4[r] = s < valid ? (a.feat_index == nullptr ? (int32_t)(base + s) : __ldg(a.feat_index + base + s)) : -1;
    }
  }
#pragma unroll 1
  for (int li = 0; li < kV4Levels; ++li) {
    const int l = l0 + li;
    pair_sync(pair);  // both warps are done with the previous level's df / eg
    {
      const float2* __restrict__ dfl = a.dfeat + (size_t)l * ns + base;
      float2 d4[kHalf];
#pragma unroll
      for (int r = 0; r < kHalf; ++r) {
        const int s = w0 + lane + 32 * (r0 + r);
        d4[r] = s < valid ? __ldg(dfl + s) : make_float2(0.f, 0.f);
      }
      uint32_t e4[kHalf];
      if (!kGather) {
        const uint32_t* __restrict__ eg = a.egrid + (size_t)(4 * l + kGrid) * a.egrid_stride;
#pragma unroll
        for (int r = 0; r < kHalf; ++r) e4[r] = col4[r] >= 0 ? __ldg(eg + col4[r]) : 0u;
      }
#pragma unroll
      for (int r = 0; r < kHalf; ++r) {
        const int s = w0 + lane + 32 * (r0 + r);
        sm.df[(s >> 3) * kV4Row + (s & 7)] = d4[r];
        if (!kGather) sm.eg[(s >> 3) * kV4Row + (s & 7)] = e4[r];
      }
    }
    pair_sync(pair);
    const float scale = f.level_scale[l];
    const uint32_t res = f.level_res[l];

    uint32_t cur_sgi = 255u;
    uint32_t idx[4], raw[4];
    float accx[4], accy[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) accx[q] = accy[q] = 0.f, idx[q] = 0u, raw[q] = 0u;
    float* gtab = nullptr;
    float* gvec = nullptr;
    const uint32_t* tab = nullptr;
    const float* vecs = nullptr;
    uint32_t lsize = 1u, mulY = 0u, mulZ = 0u, hmask = 0u, vstride = 2u;
    bool hashed = false;
    uint32_t to0 = 0u, to1 = 0u;
    float va0 = 0.f, va1 = 0.f, vb0 = 0.f, vb1 = 0.f;
    uint32_t slow_mask = 0u;

#pragma unroll 1
    for (int j = 0; j < cnt; ++j) {
      const uint32_t sgi = sm.seg[tid * kV4Chunk + j];
      if (sgi == 255u) continue;                       // sample without a temporal segment: no gradient
      const float4 p4 = sm.pos[row + j];
      const float2 dO = sm.df[row + j];
      const float c0 = (kGrid == 2) ? p4.y : p4.x;
      const float c1 = (kGrid == 0 || kGrid == 1) ? p4.y : p4.z;
      const float c2 = (kGrid == 0) ? p4.z : p4.w;
      const float cv = (kAxis == 0) ? p4.x : (kAxis == 1) ? p4.y : (kAxis == 2) ? p4.z : p4.w;
      const RowTap4 tp = make_row_tap4(cv, f.vec_res);
      const Cell A = to_cell(scale, c0), B = to_cell(scale, c1), C = to_cell(scale, c2);
      if (sgi != cur_sgi) {                             // (rare) new temporal segment: flush everything, new constants
        if (gtab != nullptr) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            red2v4(gtab + 2 * (size_t)idx[q], accx[q], accy[q]);
            accx[q] = accy[q] = 0.f;
          }
          if (kVec) {
            red2v4(gvec + to0 * HRF_N_FEATURES, va0, va1);
            red2v4(gvec + to1 * HRF_N_FEATURES, vb0, vb1);
            va0 = va1 = vb0 = vb1 = 0.f;
          }
        }
        const hrf_segment* sg = f.segments + sgi;
        const uint32_t off = sg->level_offset[l];
        lsize = sg->level_size[l];
        hashed = ((sg->hashed_mask >> l) & 1u) != 0u;
        mulY = hashed ? kPrimeY : res;
        mulZ = hashed ? kPrimeZ : res * res;
        hmask = hashed ? lsize - 1u : 0xffffffffu;
        tab = sg->grid[kGrid] + off;
        vstride = sg->vectors_t != nullptr ? 2u : (uint32_t)HRF_N_FEATURES;
        vecs = sg->vectors_t != nullptr ? sg->vectors_t + (size_t)(kAxis * HRF_N_LEVELS + l) * f.vec_res * 2
                                        : sg->vectors + (size_t)kAxis * f.vec_res * HRF_N_FEATURES + 2 * l;
        gvec = a.seg_grads[sgi].vectors + (size_t)kAxis * f.vec_res * HRF_N_FEATURES + 2 * l;
        gtab = a.seg_grads[sgi].grid[kGrid] + 2 * (size_t)off;
        // start the runs AT this sample (nothing to flush below, no "slot is empty" test on the hot path)
        to0 = tp.i0, to1 = tp.i1;
        if (hashed || (A.g < res && B.g < res && C.g < res)) {
          slot_indices4<kZ>(A, B, C, hashed, mulY, mulZ, hmask, lsize, idx);
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) idx[q] = 0u;       // (out-of-grid sample: any valid entry; it only ever receives +0)
        }
        if (kGather) {
#pragma unroll
          for (int q = 0; q < 4; ++q) raw[q] = __ldg(tab + idx[q]);
        }
        cur_sgi = sgi;
      }
      uint32_t ev = 0u;
      if (!kGather && kZ == 0) ev = sm.eg[row + j];
      if (!hashed && (A.g >= res || B.g >= res || C.g >= res)) {   // outside a dense grid (never for samples inside the AABB)
        slow_mask |= 1u << j;
        continue;
      }
      // vector rows of this sample (tensor_composition.cu:37-45): both halves need the lerped value v
      const float2 tv0 = __ldg(reinterpret_cast<const float2*>(vecs + tp.i0 * vstride));
      const float2 tv1 = __ldg(reinterpret_cast<const float2*>(vecs + tp.i1 * vstride));
      if (kVec && (tp.i0 != to0 || tp.i1 != to1)) {    // a new tap pair flushes the vector-gradient run
        red2v4(gvec + to0 * HRF_N_FEATURES, va0, va1);
        red2v4(gvec + to1 * HRF_N_FEATURES, vb0, vb1);
        va0 = va1 = vb0 = vb1 = 0.f;
        to0 = tp.i0, to1 = tp.i1;
      }
      // the 4 vertex indices of this half in parity-slot order; a slot whose index changed is flushed and re-keyed
      uint32_t nidx[4];
      slot_indices4<kZ>(A, B, C, hashed, mulY, mulZ, hmask, lsize, nidx);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (nidx[q] != idx[q]) {
          red2v4(gtab + 2 * (size_t)idx[q], accx[q], accy[q]);
          accx[q] = accy[q] = 0.f;
          idx[q] = nidx[q];
          if (kGather) raw[q] = __ldg(tab + nidx[q]);
        }
      }
      // corner weights in slot order: slot bit 0 <-> even vertex = the LOWER corner iff the cell coordinate is even
      const float ax = (A.g & 1u) ? A.f : 1.f - A.f, bx = (A.g & 1u) ? 1.f - A.f : A.f;
      const float ay = (B.g & 1u) ? B.f : 1.f - B.f, by = (B.g & 1u) ? 1.f - B.f : B.f;
      const float wz = ((C.g & 1u) != 0u) == (kZ == 0) ? C.f : 1.f - C.f;   // even vertex (kZ 0): upper corner iff the cell is odd
      float w[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) w[q] = (((q & 1) ? bx : ax) * ((q & 2) ? by : ay)) * wz;   // same product order as corner_weights
      const float2 v = make_float2(tv0.x + tp.frac * (tv1.x - tv0.x), tv0.y + tp.frac * (tv1.y - tv0.y));
      const float gx = v.x * dO.x, gy = v.y * dO.y;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        accx[q] = __fmaf_rn(w[q], gx, accx[q]);
        accy[q] = __fmaf_rn(w[q], gy, accy[q]);
      }
      if (kVec) {
        float ex = 0.f, ey = 0.f;
        if (!kGather) {
          ex = bf16_lo(ev), ey = bf16_hi(ev);
        } else {   // this half's share of the blend; the other half adds its own
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            ex = __fmaf_rn(w[q], bf16_lo(raw[q]), ex);
            ey = __fmaf_rn(w[q], bf16_hi(raw[q]), ey);
          }
        }
        // d vectors[axis][i0/i1][2l..2l+1] = e_k * dOut * (1-frac | frac)   (tensor_composition.cu:109-111)
        const float dx = ex * dO.x, dy = ey * dO.y;
        va0 = __fmaf_rn(dx, 1.f - tp.frac, va0), va1 = __fmaf_rn(dy, 1.f - tp.frac, va1);
        vb0 = __fmaf_rn(dx, tp.frac, vb0), vb1 = __fmaf_rn(dy, tp.frac, vb1);
      }
    }
    if (gtab != nullptr) {
#pragma unroll
      for (int q = 0; q < 4; ++q) red2v4(gtab + 2 * (size_t)idx[q], accx[q], accy[q]);
      if (kVec && kAxis != 3) {
        red2v4(gvec + to0 * HRF_N_FEATURES, va0, va1);
        red2v4(gvec + to1 * HRF_N_FEATURES, vb0, vb1);
      }
    }
    if (kVec && kAxis == 3) {   // grid xyz: the vector axis is time, a few hot rows: summed across the warp first (field_common.cuh)
      warp_combine_red2(gtab != nullptr ? ((cur_sgi << 24) | to0) : 0xffffffffu, gvec + to0 * HRF_N_FEATURES, va0, va1);
      warp_combine_red2(gtab != nullptr ? ((cur_sgi << 24) | to1) : 0xffffffffu, gvec + to1 * HRF_N_FEATURES, vb0, vb1);
    }
    if (kZ == 0 && slow_mask != 0u) {   // cold: samples outside a dense level's grid, all 8 corners, even half only
      for (int j = 0; j < cnt; ++j) {
        if (!((slow_mask >> j) & 1u)) continue;
        const uint32_t sgi = sm.seg[tid * kV4Chunk + j];
        const float4 p4 = sm.pos[row + j];
        const float c0 = (kGrid == 2) ? p4.y : p4.x, c1 = (kGrid == 0 || kGrid == 1) ? p4.y : p4.z, c2 = (kGrid == 0) ? p4.z : p4.w;
        const float cv = (kAxis == 0) ? p4.x : (kAxis == 1) ? p4.y : (kAxis == 2) ? p4.z : p4.w;
        const hrf_segment* sg = f.segments + sgi;
        const uint32_t off = sg->level_offset[l];
        scatter_sample_slow4<kGather>(sg->grid[kGrid] + off, a.seg_grads[sgi].grid[kGrid] + 2 * (size_t)off, a.seg_grads[sgi].vectors,
                                      sg->vectors, ((sg->hashed_mask >> l) & 1u) != 0u, res, sg->level_size[l], to_cell(scale, c0),
                                      to_cell(scale, c1), to_cell(scale, c2), make_tap(cv, f.vec_res, kAxis), l, sm.df[row + j],
                                      kGather ? 0u : sm.eg[row + j]);
      }
    }
  }
}

template <int kGrid, bool kGather>
__device__ __forceinline__ void scatter_halves(const ScatterV4Args& a, V4Smem& sm, int l0, int64_t base, int valid) {
  if (threadIdx.x < 128) scatter_levels4<kGrid, kGather, 0>(a, sm, l0, base, valid);   // (uniform per warp)
  else scatter_levels4<kGrid, kGather, 1>(a, sm, l0, base, valid);
}

template <bool kGather>
__global__ void __launch_bounds__(kV4Threads, 4) grid_scatter_v4_kernel(const __grid_constant__ ScatterV4Args a) {
  extern __shared__ __align__(16) unsigned char v4_raw[];
  V4Smem& sm = *reinterpret_cast<V4Smem*>(v4_raw);
  const int64_t n = live_samples(a.s);
  const int64_t base = (int64_t)blockIdx.x * kV4Samples;
  if (base >= n) return;
  const int k = a.grid_first + (int)blockIdx.y % a.grid_count;
  const int l0 = ((int)blockIdx.y / a.grid_count) * kV4Levels;
  const int valid = (int)((n - base) < kV4Samples ? (n - base) : kV4Samples);
  {   // positions / segment ids of the 256 samples a warp pair walks: each warp of the pair stages half the rows
    const int tid = threadIdx.x & 127, lane = tid & 31, w0 = (tid & ~31) * kV4Chunk, r0 = (threadIdx.x >> 7) * (kV4Chunk / 2);
#pragma unroll
    for (int r = 0; r < kV4Chunk / 2; ++r) {
      const int s = w0 + lane + 32 * (r0 + r);
      const bool ok = s < valid;
      sm.pos[(s >> 3) * kV4Row + (s & 7)] = ok ? __ldg(a.pos4 + base + s) : make_float4(0.f, 0.f, 0.f, 0.f);
      sm.seg[s] = ok ? a.seg8[base + s] : (uint8_t)255;
    }
  }
  if (k == 0) scatter_halves<0, kGather>(a, sm, l0, base, valid);       // (k is uniform over the CTA)
  else if (k == 1) scatter_halves<1, kGather>(a, sm, l0, base, valid);
  else if (k == 2) scatter_halves<2, kGather>(a, sm, l0, base, valid);
  else scatter_halves<3, kGather>(a, sm, l0, base, valid);
}

}  // namespace hrf

using namespace hrf;

// called from hrf_field_backward_tables (field_bwd.cu); HRF_SCATTER=4
int hrf_launch_scatter_v4(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads, const void* grid_feat_bf16,
                          const int32_t* feat_index, int64_t grid_feat_stride, const void* workspace, int grid_first, int grid_count,
                          cudaStream_t st) {
  HRF_REQUIRE(f->vec_res < (1 << 24), "the scatter keys vector rows in 24 bits");
  ScatterV4Args a;
  a.f = *f;
  a.s = *s;
  a.seg_grads = seg_grads;
  a.dfeat = reinterpret_cast<const float2*>(workspace);
  a.pos4 = reinterpret_cast<const float4*>(reinterpret_cast<const char*>(workspace) + 128 * (size_t)s->num_samples);
  a.seg8 = reinterpret_cast<const uint8_t*>(reinterpret_cast<const char*>(workspace) + 144 * (size_t)s->num_samples);
  a.egrid = reinterpret_cast<const uint32_t*>(grid_feat_bf16);
  a.feat_index = grid_feat_bf16 != nullptr ? feat_index : nullptr;
  a.egrid_stride = grid_feat_stride > 0 ? grid_feat_stride : s->num_samples;
  a.grid_first = grid_first;
  a.grid_count = grid_count;
  const int64_t blocks = (s->num_samples + kV4Samples - 1) / kV4Samples;
  const dim3 grid((unsigned)blocks, (HRF_N_LEVELS / kV4Levels) * grid_count);
  const int smem = (int)sizeof(V4Smem);
  if (grid_feat_bf16 != nullptr) grid_scatter_v4_kernel<false><<<grid, kV4Threads, smem, st>>>(a);
  else grid_scatter_v4_kernel<true><<<grid, kV4Threads, smem, st>>>(a);
  HRF_CHECK_LAUNCH();
  return 0;
}
