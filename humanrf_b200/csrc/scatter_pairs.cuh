// The lane-pair walk of the table / vector gradient scatter (scatter_v5.cu, scatter_v6.cu): what one warp does for one
// (level, grid) over the 128 samples it has staged in shared memory.  v5 and v6 differ only in what a CTA covers and how
// it stages its inputs.
//
// Consecutive samples of a ray mostly stay in the same cell or step into a neighbouring one, so the walk accumulates
// w * g per vertex over a run of samples and issues one RED per run, not per sample.  The accumulators are PARITY SLOTS:
// indexed not by corner offset (dx, dy, dz) but by the parity of the vertex coordinate on each axis.  A cell [g, g+1]
// holds exactly one even and one odd vertex per axis, so
//   * when the ray steps into the neighbouring cell along an axis, the vertex the two cells share keeps its slot and its
//     accumulator (that is the shared-corner carry), and the vertex that enters has the parity of the one that leaves,
//     so it takes over that slot.  "Flush and zero the slots whose table index changed" is the whole carry: no data
//     moves between slots, and jumps and new rays need no special case;
//   * "index changed" is one integer compare per slot and a flush is a predicated RED; the corner weights are computed
//     in slot order directly (two selects per axis).  The per-sample step is straight-line code, with no divergent
//     branch for the runs.
// The 8 slots of a sample are split over the two lanes of a pair by the parity of the first-axis vertex (scatter_v5.cu).
#pragma once

#include <cstddef>

#include "field_common.cuh"

namespace hrf {

constexpr int kV5Threads = 256, kV5Chunk = 8, kV5Chunks = kV5Threads / 2, kV5Samples = kV5Chunks * kV5Chunk,
              kV5Row = kV5Chunk + 1, kV5WarpSamples = 16 * kV5Chunk, kV5Stage = kV5WarpSamples / 32;

struct ScatterV5Args {
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

__device__ __forceinline__ void red2v5(float* addr, float a, float b) {
  // No "memory" clobber: the scatter never reads the gradient buffers, and the clobber would pin every load of the next
  // step behind this step's REDs.
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b));
}

// Table entries of the 4 vertices of a cell whose FIRST-axis vertex has parity p, in parity-slot order (slot bit 0 = parity
// of the second-axis vertex, bit 1 = of the third-axis vertex).  hashed: tcnn's coherent prime hash; dense: one
// conditional subtraction (cell inside the grid, see corner_indices).
__device__ __forceinline__ void slot_indices5(uint32_t p, Cell A, Cell B, Cell C, bool hashed, uint32_t mulY, uint32_t mulZ,
                                              uint32_t hmask, uint32_t lsize, uint32_t (&v)[4]) {
  const uint32_t nx = p ? (A.g | 1u) : ((A.g + 1u) & ~1u);
  const uint32_t ny0 = ((B.g + 1u) & ~1u) * mulY, ny1 = (B.g | 1u) * mulY;
  const uint32_t nz0 = ((C.g + 1u) & ~1u) * mulZ, nz1 = (C.g | 1u) * mulZ;
  if (hashed) {
#pragma unroll
    for (int q = 0; q < 4; ++q) v[q] = (nx ^ ((q & 1) ? ny1 : ny0) ^ ((q & 2) ? nz1 : nz0)) & hmask;
  } else {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t t = nx + ((q & 1) ? ny1 : ny0) + ((q & 2) ? nz1 : nz0);   // < 2 * lsize (see corner_indices)
      v[q] = t >= lsize ? t - lsize : t;
    }
  }
}

// cold path: a sample outside a dense level's grid (all 8 corners, the forward's general index wrap); even lane only
template <bool kGather>
__device__ __noinline__ void scatter_sample_slow5(const uint32_t* tab, float* gtab, float* gvec, const float* vecs, bool hashed,
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
  for (int q = 0; q < 8; ++q) red2v5(gtab + 2 * (size_t)idx[q], w[q] * gx, w[q] * gy);
  const float dx = ex * dO.x, dy = ey * dO.y;
  red2v5(gvec + tp.o0 + 2 * l, dx * (1.f - tp.frac), dy * (1.f - tp.frac));
  red2v5(gvec + tp.o1 + 2 * l, dx * tp.frac, dy * tp.frac);
}

// Level l of grid kGrid over the warp's staged samples.  Smem has pos / df / eg in rows of kV5Row per chunk of 8 samples
// and seg per sample; the caller has staged df (and eg unless kGather) for (l, kGrid) and passed a __syncwarp.
// kGrid: 0 xyz, 1 xyt, 2 yzt, 3 xzt (decomposition4d.py:126-129); its vector axis is t, z, x, y (tensor_composition.cu:49-52)
template <int kGrid, bool kGather, class Smem>
__device__ __forceinline__ void scatter_level_pairs(const ScatterV5Args& a, const Smem& sm, int l) {
  const hrf_field& f = a.f;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t p = (uint32_t)lane & 1u;          // parity of the first-axis vertex this lane owns; tap row it owns
  const int ch = warp * 16 + (lane >> 1);          // the chunk of 8 consecutive samples the lane pair walks
  constexpr int kAxis = (kGrid == 0) ? 3 : (kGrid == 1) ? 2 : (kGrid == 2) ? 0 : 1;
  const int row = ch * kV5Row;
  const float scale = f.level_scale[l];
  const uint32_t res = f.level_res[l];

  uint32_t cur_sgi = 255u;
  uint32_t idx[4], raw[4];      // table entry of the vertex each of this lane's parity slots holds, its bf16x2 value
  float accx[4], accy[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) accx[q] = accy[q] = 0.f, idx[q] = 0u, raw[q] = 0u;
  float* gtab = nullptr;
  float* gvec = nullptr;
  const uint32_t* tab = nullptr;
  const float* vecs = nullptr;
  uint32_t lsize = 1u, mulY = 0u, mulZ = 0u, hmask = 0u, vstride = 2u;
  bool hashed = false;
  uint32_t to = 0u;             // the tap row of the vector axis this lane accumulates for (i0 on even lanes, i1 on odd)
  float va0 = 0.f, va1 = 0.f;
  uint32_t slow_mask = 0u;

  // Uniform trip count: every lane of the warp reaches the pair shuffle of every step (slots past `valid` carry segment
  // id 255 and do nothing).  `ok` and all branches below are the same in both lanes of a pair.
#pragma unroll 1
  for (int j = 0; j < kV5Chunk; ++j) {
    const uint32_t sgi = sm.seg[ch * kV5Chunk + j];
    bool ok = sgi != 255u;                           // 255: no temporal segment / past the end: no gradient
    uint32_t changed = 0u;
    uint32_t nidx[4] = {0u, 0u, 0u, 0u};
    Cell A{0u, 0.f}, B{0u, 0.f}, C{0u, 0.f};
    RowTap2 tp{0u, 0u, 0.f};
    float2 dO = make_float2(0.f, 0.f);
    if (ok) {
      const float4 p4 = sm.pos[row + j];
      dO = sm.df[row + j];
      const float c0 = (kGrid == 2) ? p4.y : p4.x;
      const float c1 = (kGrid == 0 || kGrid == 1) ? p4.y : p4.z;
      const float c2 = (kGrid == 0) ? p4.z : p4.w;
      const float cv = (kAxis == 0) ? p4.x : (kAxis == 1) ? p4.y : (kAxis == 2) ? p4.z : p4.w;
      tp = make_row_tap2(cv, f.vec_res);
      A = to_cell(scale, c0), B = to_cell(scale, c1), C = to_cell(scale, c2);
      if (sgi != cur_sgi) {                           // (rare) new temporal segment: flush everything, new constants
        if (gtab != nullptr) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            red2v5(gtab + 2 * (size_t)idx[q], accx[q], accy[q]);
            accx[q] = accy[q] = 0.f;
          }
          red2v5(gvec + to * HRF_N_FEATURES, va0, va1);
          va0 = va1 = 0.f;
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
        to = p ? tp.i1 : tp.i0;
        if (hashed || (A.g < res && B.g < res && C.g < res)) {
          slot_indices5(p, A, B, C, hashed, mulY, mulZ, hmask, lsize, idx);
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) idx[q] = 0u;     // (out-of-grid sample: any valid entry; it only ever receives +0)
        }
        if (kGather) {
#pragma unroll
          for (int q = 0; q < 4; ++q) raw[q] = __ldg(tab + idx[q]);
        }
        cur_sgi = sgi;
      }
      if (!hashed && (A.g >= res || B.g >= res || C.g >= res)) {   // outside a dense grid (never for samples inside the AABB)
        slow_mask |= 1u << j;
        ok = false;
      } else {
        slot_indices5(p, A, B, C, hashed, mulY, mulZ, hmask, lsize, nidx);
#pragma unroll
        for (int q = 0; q < 4; ++q) changed |= (nidx[q] != idx[q]) ? (1u << q) : 0u;
      }
    }
    // a slot is flushed by BOTH lanes of the pair when either lane's entry changed: the two entries (first-axis
    // neighbours, same 128-byte line 15 times out of 16) travel in one RED instruction
    const uint32_t flush = changed | __shfl_xor_sync(0xffffffffu, changed, 1);
    float ex = 0.f, ey = 0.f;
    float w[4] = {0.f, 0.f, 0.f, 0.f};
    if (ok) {
      // vector rows of this sample (tensor_composition.cu:37-45): both lanes need the lerped value v
      const float2 tv0 = __ldg(reinterpret_cast<const float2*>(vecs + tp.i0 * vstride));
      const float2 tv1 = __ldg(reinterpret_cast<const float2*>(vecs + tp.i1 * vstride));
      const uint32_t trow = p ? tp.i1 : tp.i0;
      if (trow != to) {                               // a new tap row flushes this lane's vector-gradient run
        red2v5(gvec + to * HRF_N_FEATURES, va0, va1);
        va0 = va1 = 0.f;
        to = trow;
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if ((flush >> q) & 1u) {
          red2v5(gtab + 2 * (size_t)idx[q], accx[q], accy[q]);
          accx[q] = accy[q] = 0.f;
          if (kGather) {
            if (nidx[q] != idx[q]) raw[q] = __ldg(tab + nidx[q]);
          }
          idx[q] = nidx[q];
        }
      }
      // corner weights in slot order: even vertex = the LOWER corner iff the cell coordinate is even
      const float wx = ((A.g & 1u) != 0u) == (p == 0u) ? A.f : 1.f - A.f;   // even vertex (p 0): upper corner iff the cell is odd
      const float ay = (B.g & 1u) ? B.f : 1.f - B.f, by = (B.g & 1u) ? 1.f - B.f : B.f;
      const float az = (C.g & 1u) ? C.f : 1.f - C.f, bz = (C.g & 1u) ? 1.f - C.f : C.f;
#pragma unroll
      for (int q = 0; q < 4; ++q) w[q] = (wx * ((q & 1) ? by : ay)) * ((q & 2) ? bz : az);   // same product order as corner_weights
      const float2 v = make_float2(tv0.x + tp.frac * (tv1.x - tv0.x), tv0.y + tp.frac * (tv1.y - tv0.y));
      const float gx = v.x * dO.x, gy = v.y * dO.y;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        accx[q] = __fmaf_rn(w[q], gx, accx[q]);
        accy[q] = __fmaf_rn(w[q], gy, accy[q]);
      }
      if (!kGather) {
        const uint32_t ev = sm.eg[row + j];
        ex = bf16_lo(ev), ey = bf16_hi(ev);
      } else {   // this lane's share of the blend
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          ex = __fmaf_rn(w[q], bf16_lo(raw[q]), ex);
          ey = __fmaf_rn(w[q], bf16_hi(raw[q]), ey);
        }
      }
    }
    if (kGather) {   // the other lane's share (uniform: every lane shuffles)
      ex += __shfl_xor_sync(0xffffffffu, ex, 1);
      ey += __shfl_xor_sync(0xffffffffu, ey, 1);
    }
    if (ok) {
      // d vectors[axis][i0 | i1][2l..2l+1] = e_k * dOut * (1-frac | frac)   (tensor_composition.cu:109-111)
      const float tw = p ? tp.frac : 1.f - tp.frac;
      va0 = __fmaf_rn(ex * dO.x, tw, va0), va1 = __fmaf_rn(ey * dO.y, tw, va1);
    }
  }
  if (gtab != nullptr) {
#pragma unroll
    for (int q = 0; q < 4; ++q) red2v5(gtab + 2 * (size_t)idx[q], accx[q], accy[q]);
    if (kAxis != 3) red2v5(gvec + to * HRF_N_FEATURES, va0, va1);
  }
  if (kAxis == 3)   // grid xyz: the vector axis is time, a few hot rows: summed across the warp first (field_common.cuh)
    warp_combine_red2(gtab != nullptr ? ((cur_sgi << 24) | to) : 0xffffffffu, gvec + to * HRF_N_FEATURES, va0, va1);
  if (p == 0u && slow_mask != 0u) {   // cold: samples outside a dense level's grid, all 8 corners, even lane only
    for (int j = 0; j < kV5Chunk; ++j) {
      if (!((slow_mask >> j) & 1u)) continue;
      const uint32_t sgi = sm.seg[ch * kV5Chunk + j];
      const float4 p4 = sm.pos[row + j];
      const float c0 = (kGrid == 2) ? p4.y : p4.x, c1 = (kGrid == 0 || kGrid == 1) ? p4.y : p4.z, c2 = (kGrid == 0) ? p4.z : p4.w;
      const float cv = (kAxis == 0) ? p4.x : (kAxis == 1) ? p4.y : (kAxis == 2) ? p4.z : p4.w;
      const hrf_segment* sg = f.segments + sgi;
      const uint32_t off = sg->level_offset[l];
      scatter_sample_slow5<kGather>(sg->grid[kGrid] + off, a.seg_grads[sgi].grid[kGrid] + 2 * (size_t)off, a.seg_grads[sgi].vectors,
                                    sg->vectors, ((sg->hashed_mask >> l) & 1u) != 0u, res, sg->level_size[l], to_cell(scale, c0),
                                    to_cell(scale, c1), to_cell(scale, c2), make_tap(cv, f.vec_res, kAxis), l, sm.df[row + j],
                                    kGather ? 0u : sm.eg[row + j]);
    }
  }
}

}  // namespace hrf
