// Table / vector gradient scatter, second generation (replaces tcnn kernel_grid_backward + compose_tensors_backward,
// tensor_composition.cu:57-118, like grid_scatter_staged_kernel in field_bwd.cu, which it supersedes as the default).
//
// Why: the staged kernel issues several times the warp instructions converged code needs per (sample, level, grid)
// item, and its RED instructions run with about a quarter of the lanes active: the run-length logic ("new cell? shift the shared corners, flush the ones that leave") is a data-dependent
// branch per lane, and at the middle levels some lane of the warp takes it at almost every step.
//
// Here the per-sample step is STRAIGHT-LINE code.  The 8 accumulator slots of a thread are not indexed by corner
// offset (dx,dy,dz) but by the PARITY of the vertex coordinates: slot bit a = parity of the vertex coordinate on axis
// a.  A cell [g, g+1] always holds exactly one even and one odd vertex per axis, so
//   * when the ray steps into the neighbouring cell along an axis, the vertex the two cells share keeps its slot (and
//     its accumulator: this IS the shared-corner carry), and the vertex that enters has the parity of the one that
//     leaves, i.e. it replaces it in the same slots: "flush and zero the slots whose vertex changed" is all there is
//     to do, with no data movement between slots and no special case for jumps or new rays;
//   * "vertex changed" is one integer compare per slot (new table index vs the slot's); flushes are predicated REDs;
//     the corner weights are computed directly in slot order (two selects per axis).
// Same number of REDs as the carried run-length scheme (about 2 per (sample, level, grid)), none of its divergence.
#include <cstddef>
#include <cstdlib>

#include "field_common.cuh"

namespace hrf {

constexpr int kV2Threads = 128, kV2Chunk = 8, kV2Samples = kV2Threads * kV2Chunk, kV2Levels = 4, kV2Row = kV2Chunk + 1;

struct ScatterV2Args {
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

struct __align__(16) V2Smem {
  float4 pos[kV2Threads * kV2Row];
  float2 df[kV2Threads * kV2Row];
  uint32_t eg[kV2Threads * kV2Row];
  uint8_t seg[kV2Samples];
};

__device__ __forceinline__ void red2(float* addr, float a, float b) {
  // (no "memory" clobber: the gradient buffers are never read in this kernel, and the clobber would pin every load of
  //  the next step behind the REDs of this one)
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b));
}
// Table entries of the 8 vertices of a cell in parity-slot order (slot bit a = parity of the vertex coordinate on axis a).
// hashed: tcnn's coherent prime hash; dense: x + y res + z res^2, one conditional subtraction (cell inside the grid).
__device__ __forceinline__ void slot_indices(Cell A, Cell B, Cell C, bool hashed, uint32_t mulY, uint32_t mulZ, uint32_t hmask,
                                             uint32_t lsize, uint32_t (&v)[8]) {
  const uint32_t nx0 = (A.g + 1u) & ~1u, nx1 = A.g | 1u;                   // even / odd vertex on each axis
  const uint32_t ny0 = ((B.g + 1u) & ~1u) * mulY, ny1 = (B.g | 1u) * mulY;
  const uint32_t nz0 = ((C.g + 1u) & ~1u) * mulZ, nz1 = (C.g | 1u) * mulZ;
  if (hashed) {   // (uniform over the warp unless the 32 x 8 samples straddle temporal segments of different sizes)
#pragma unroll
    for (int q = 0; q < 8; ++q) v[q] = (((q & 1) ? nx1 : nx0) ^ ((q & 2) ? ny1 : ny0) ^ ((q & 4) ? nz1 : nz0)) & hmask;
  } else {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const uint32_t t = ((q & 1) ? nx1 : nx0) + ((q & 2) ? ny1 : ny0) + ((q & 4) ? nz1 : nz0);   // < 2 * lsize (see corner_indices)
      v[q] = t >= lsize ? t - lsize : t;
    }
  }
}

// A sample whose cell lies outside a DENSE level's grid (a position outside the unit cube: only reachable through the
// QueryInput API, never through ray batches inside the AABB): the forward wraps its indices with the general modulo
// (corner_indices); the straight-line step below assumes one conditional subtraction.  Such samples take this cold,
// out-of-line path: 8 direct REDs with exactly the forward's indices, and the two vector-row REDs.
template <bool kGather>
__device__ __noinline__ void scatter_sample_slow(const uint32_t* tab, float* gtab, float* gvec, const float* vecs, bool hashed,
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
  for (int q = 0; q < 8; ++q) red2(gtab + 2 * (size_t)idx[q], w[q] * gx, w[q] * gy);
  const float dx = ex * dO.x, dy = ey * dO.y;
  red2(gvec + tp.o0 + 2 * l, dx * (1.f - tp.frac), dy * (1.f - tp.frac));
  red2(gvec + tp.o1 + 2 * l, dx * tp.frac, dy * tp.frac);
}

// kGrid: 0 xyz, 1 xyt, 2 yzt, 3 xzt (decomposition4d.py:126-129); its vector axis is t, z, x, y (tensor_composition.cu:49-52)
template <int kGrid, bool kGather>
__device__ __forceinline__ void scatter_levels(const ScatterV2Args& a, V2Smem& sm, int l0, int64_t base, int valid) {
  const hrf_field& f = a.f;
  const int tid = threadIdx.x;
  const int64_t ns = a.s.num_samples;
  constexpr int kAxis = (kGrid == 0) ? 3 : (kGrid == 1) ? 2 : (kGrid == 2) ? 0 : 1;
  const int row = tid * kV2Row;
  const int cnt = min(max(valid - tid * kV2Chunk, 0), kV2Chunk);
#pragma unroll 1
  for (int li = 0; li < kV2Levels; ++li) {
    const int l = l0 + li;
    __syncthreads();  // the previous level's readers are done with df / eg
    {
      const float2* __restrict__ dfl = a.dfeat + (size_t)l * ns + base;
      for (int s = tid; s < valid; s += kV2Threads) sm.df[(s >> 3) * kV2Row + (s & 7)] = __ldg(dfl + s);
      if (!kGather) {
        const uint32_t* __restrict__ eg = a.egrid + (size_t)(4 * l + kGrid) * a.egrid_stride;
        if (a.feat_index == nullptr) {
          for (int s = tid; s < valid; s += kV2Threads) sm.eg[(s >> 3) * kV2Row + (s & 7)] = __ldg(eg + base + s);
        } else {
          for (int s = tid; s < valid; s += kV2Threads)
            sm.eg[(s >> 3) * kV2Row + (s & 7)] = __ldg(eg + __ldg(a.feat_index + base + s));
        }
      }
    }
    __syncthreads();
    const float scale = f.level_scale[l];
    const uint32_t res = f.level_res[l];

    uint32_t cur_sgi = 255u;
    uint32_t idx[8], raw[8];      // table entry of the vertex each parity slot holds, its bf16x2 value
    float accx[8], accy[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) accx[q] = accy[q] = 0.f, idx[q] = 0xffffffffu, raw[q] = 0u;
    float* gtab = nullptr;
    float* gvec = nullptr;
    const uint32_t* tab = nullptr;
    const float* vecs = nullptr;
    uint32_t lsize = 1u, mulY = 0u, mulZ = 0u, hmask = 0u;
    bool hashed = false;
    uint32_t to0 = 0u, to1 = 0u;          // current tap rows (valid once gtab != nullptr)
    float va0 = 0.f, va1 = 0.f, vb0 = 0.f, vb1 = 0.f;
    uint32_t slow_mask = 0u;

#pragma unroll 1
    for (int j = 0; j < cnt; ++j) {
      const uint32_t sgi = sm.seg[tid * kV2Chunk + j];
      if (sgi == 255u) continue;                       // sample without a temporal segment: no gradient
      const float4 p4 = sm.pos[row + j];
      const float2 dO = sm.df[row + j];
      const float c0 = (kGrid == 2) ? p4.y : p4.x;
      const float c1 = (kGrid == 0 || kGrid == 1) ? p4.y : p4.z;
      const float c2 = (kGrid == 0) ? p4.z : p4.w;
      const float cv = (kAxis == 0) ? p4.x : (kAxis == 1) ? p4.y : (kAxis == 2) ? p4.z : p4.w;
      const VecTap tp = make_tap(cv, f.vec_res, kAxis);
      const Cell A = to_cell(scale, c0), B = to_cell(scale, c1), C = to_cell(scale, c2);
      if (sgi != cur_sgi) {                             // (rare) new temporal segment: flush everything, new constants
        if (gtab != nullptr) {
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            red2(gtab + 2 * (size_t)idx[q], accx[q], accy[q]);
            accx[q] = accy[q] = 0.f;
          }
          red2(gvec + to0, va0, va1);
          red2(gvec + to1, vb0, vb1);
          va0 = va1 = vb0 = vb1 = 0.f;
        }
        const hrf_segment* sg = f.segments + sgi;
        const uint32_t off = sg->level_offset[l];
        lsize = sg->level_size[l];
        hashed = ((sg->hashed_mask >> l) & 1u) != 0u;
        mulY = hashed ? kPrimeY : res;
        mulZ = hashed ? kPrimeZ : res * res;
        hmask = hashed ? lsize - 1u : 0xffffffffu;
        tab = sg->grid[kGrid] + off;
        vecs = sg->vectors + 2 * l;                    // (this level's feature pair of every row)
        gvec = a.seg_grads[sgi].vectors + 2 * l;
        gtab = a.seg_grads[sgi].grid[kGrid] + 2 * (size_t)off;
        // start the runs AT this sample: its own vertices / taps are the current ones, so the step below finds nothing to
        // flush (the accumulators are zero) and the hot path needs no "slot is empty" test
        to0 = tp.o0, to1 = tp.o1;
        if (hashed || (A.g < res && B.g < res && C.g < res)) {
          slot_indices(A, B, C, hashed, mulY, mulZ, hmask, lsize, idx);
        } else {
#pragma unroll
          for (int q = 0; q < 8; ++q) idx[q] = 0u;       // (out-of-grid sample: any valid entry; it only ever receives +0)
        }
        if (kGather) {
#pragma unroll
          for (int q = 0; q < 8; ++q) raw[q] = __ldg(tab + idx[q]);
        }
        cur_sgi = sgi;
      }
      uint32_t ev = 0u;
      if (!kGather) ev = sm.eg[row + j];
      if (!hashed && (A.g >= res || B.g >= res || C.g >= res)) {   // outside a dense grid (never for samples inside the AABB):
        slow_mask |= 1u << j;                                       // handled after the loop, out of line (keeps the call, and
        continue;                                                   // what it does to register allocation, out of the hot loop)
      }
      // ---- vector tap of this sample (tensor_composition.cu:37-45); a new tap pair flushes the gradient run.  The two
      // rows are fetched every step (L1 hits, issued here, consumed after the index work below): no stall on them.
      if (tp.o0 != to0 || tp.o1 != to1) {
        red2(gvec + to0, va0, va1);
        red2(gvec + to1, vb0, vb1);
        va0 = va1 = vb0 = vb1 = 0.f;
        to0 = tp.o0, to1 = tp.o1;
      }
      const float2 tv0 = __ldg(reinterpret_cast<const float2*>(vecs + tp.o0));
      const float2 tv1 = __ldg(reinterpret_cast<const float2*>(vecs + tp.o1));
      // ---- cell -> the 8 vertex indices in parity-slot order; a slot whose index changed is flushed and re-keyed
      // (two different vertices that hash to the same entry keep accumulating into one slot: same table entry anyway)
      uint32_t nidx[8];
      slot_indices(A, B, C, hashed, mulY, mulZ, hmask, lsize, nidx);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        if (nidx[q] != idx[q]) {
          red2(gtab + 2 * (size_t)idx[q], accx[q], accy[q]);
          accx[q] = accy[q] = 0.f;
          idx[q] = nidx[q];
          if (kGather) raw[q] = __ldg(tab + nidx[q]);
        }
      }
      // ---- corner weights in slot order: slot bit 0 <-> even vertex = the LOWER corner iff the cell coordinate is even
      const float ax = (A.g & 1u) ? A.f : 1.f - A.f, bx = (A.g & 1u) ? 1.f - A.f : A.f;   // even-vertex / odd-vertex weight, x
      const float ay = (B.g & 1u) ? B.f : 1.f - B.f, by = (B.g & 1u) ? 1.f - B.f : B.f;
      const float az = (C.g & 1u) ? C.f : 1.f - C.f, bz = (C.g & 1u) ? 1.f - C.f : C.f;
      float w[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) w[q] = (((q & 1) ? bx : ax) * ((q & 2) ? by : ay)) * ((q & 4) ? bz : az);   // same product order as corner_weights
      const float2 v = make_float2(tv0.x + tp.frac * (tv1.x - tv0.x), tv0.y + tp.frac * (tv1.y - tv0.y));
      const float gx = v.x * dO.x, gy = v.y * dO.y;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        accx[q] = __fmaf_rn(w[q], gx, accx[q]);
        accy[q] = __fmaf_rn(w[q], gy, accy[q]);
      }
      float ex = 0.f, ey = 0.f;
      if (!kGather) {
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
    if (gtab != nullptr) {
#pragma unroll
      for (int q = 0; q < 8; ++q) red2(gtab + 2 * (size_t)idx[q], accx[q], accy[q]);
      red2(gvec + to0, va0, va1);
      red2(gvec + to1, vb0, vb1);
    }
    if (slow_mask != 0u) {   // cold: samples outside a dense level's grid, one by one with the forward's general index wrap
      for (int j = 0; j < cnt; ++j) {
        if (!((slow_mask >> j) & 1u)) continue;
        const uint32_t sgi = sm.seg[tid * kV2Chunk + j];
        const float4 p4 = sm.pos[row + j];
        const float c0 = (kGrid == 2) ? p4.y : p4.x, c1 = (kGrid == 0 || kGrid == 1) ? p4.y : p4.z, c2 = (kGrid == 0) ? p4.z : p4.w;
        const float cv = (kAxis == 0) ? p4.x : (kAxis == 1) ? p4.y : (kAxis == 2) ? p4.z : p4.w;
        const hrf_segment* sg = f.segments + sgi;
        const uint32_t off = sg->level_offset[l];
        scatter_sample_slow<kGather>(sg->grid[kGrid] + off, a.seg_grads[sgi].grid[kGrid] + 2 * (size_t)off, a.seg_grads[sgi].vectors,
                                     sg->vectors, ((sg->hashed_mask >> l) & 1u) != 0u, res, sg->level_size[l], to_cell(scale, c0),
                                     to_cell(scale, c1), to_cell(scale, c2), make_tap(cv, f.vec_res, kAxis), l, sm.df[row + j],
                                     kGather ? 0u : sm.eg[row + j]);
      }
    }
  }
}

template <bool kGather, int kCtas>
__global__ void __launch_bounds__(kV2Threads, kCtas) grid_scatter_v2_kernel(const __grid_constant__ ScatterV2Args a) {
  extern __shared__ __align__(16) unsigned char v2_raw[];
  V2Smem& sm = *reinterpret_cast<V2Smem*>(v2_raw);
  const int64_t n = live_samples(a.s);
  const int64_t base = (int64_t)blockIdx.x * kV2Samples;
  if (base >= n) return;
  const int tid = threadIdx.x;
  const int k = a.grid_first + (int)blockIdx.y % a.grid_count;
  const int l0 = ((int)blockIdx.y / a.grid_count) * kV2Levels;
  const int valid = (int)((n - base) < kV2Samples ? (n - base) : kV2Samples);
  for (int s = tid; s < kV2Samples; s += kV2Threads) {
    const bool ok = s < valid;
    sm.pos[(s >> 3) * kV2Row + (s & 7)] = ok ? __ldg(a.pos4 + base + s) : make_float4(0.f, 0.f, 0.f, 0.f);
    sm.seg[s] = ok ? a.seg8[base + s] : (uint8_t)255;
  }
  if (k == 0) scatter_levels<0, kGather>(a, sm, l0, base, valid);       // (k is uniform over the CTA)
  else if (k == 1) scatter_levels<1, kGather>(a, sm, l0, base, valid);
  else if (k == 2) scatter_levels<2, kGather>(a, sm, l0, base, valid);
  else scatter_levels<3, kGather>(a, sm, l0, base, valid);
}

}  // namespace hrf

using namespace hrf;

// called from hrf_field_backward_tables (field_bwd.cu)
int hrf_launch_scatter_v2(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads, const void* grid_feat_bf16,
                          const int32_t* feat_index, int64_t grid_feat_stride, const void* workspace, int grid_first, int grid_count,
                          cudaStream_t st) {
  ScatterV2Args a;
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
  const int64_t blocks = (s->num_samples + kV2Samples - 1) / kV2Samples;
  const dim3 grid((unsigned)blocks, (HRF_N_LEVELS / kV2Levels) * grid_count);
  const int smem = (int)sizeof(V2Smem);
  // CTAs per SM: 6 (80 registers, a few spilled words) or 5 (96 registers, no spills): HRF_SCATTER_CTAS
  const int ctas = [] { const char* e = getenv("HRF_SCATTER_CTAS"); return (e && e[0] == '5') ? 5 : 6; }();
  if (grid_feat_bf16 != nullptr) {
    if (ctas == 5) grid_scatter_v2_kernel<false, 5><<<grid, kV2Threads, smem, st>>>(a);
    else grid_scatter_v2_kernel<false, 6><<<grid, kV2Threads, smem, st>>>(a);
  } else {
    if (ctas == 5) grid_scatter_v2_kernel<true, 5><<<grid, kV2Threads, smem, st>>>(a);
    else grid_scatter_v2_kernel<true, 6><<<grid, kV2Threads, smem, st>>>(a);
  }
  HRF_CHECK_LAUNCH();
  return 0;
}
