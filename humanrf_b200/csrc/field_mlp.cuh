// Shared-memory layout and MLP layers of the fused field kernels (the forward in field_fwd.cu, the occupancy bake in
// occupancy_bake.cu): one warpgroup runs each dense layer of a 128-row tile on wgmma, thread r owning row r.
#pragma once
#include <stddef.h>

#include "field_common.cuh"

namespace hrf {

// One activation buffer serves every layer: a layer's output tile is written over its input tile, which is safe
// because each thread writes only after the wgmma wait and the CTA barrier that follow the MMA that read the old tile.
// The same buffer stages the fp32 outputs of the 16-wide layers so that every thread can read its row.
// The weight blob comes LAST and only its used part is requested as dynamic shared memory (20 KB without camera
// embeddings), so 5 CTAs/SM leave part of the 228 KB of shared memory and L1 to the L1 cache for the gathers.
struct __align__(128) FwdSmem {
  unsigned char a[kTile * 64 * 2];    // A tile: K = 32 layout in the first 8 KB, or K = 64 layout (hidden activations)
  uint64_t bar_w;                     // weights landed
  // early-stop schedule: the current work item, published by thread 0
  int64_t item_start, item_end;
  int32_t item_ray, item_skip;
  __align__(128) unsigned char w[kWBlobBytesMax];   // packed weights (TMA bulk copy, once per CTA)
};

// fp32 CUDA-core version of one dense layer (the debug path, tests only): every thread computes its row's N outputs.
template <int N, int K>
__device__ __forceinline__ void simt_layer(FwdSmem& sm, const unsigned char* abuf, uint32_t woff, float* v) {
  const int tid = threadIdx.x;
  __syncthreads();
  const uint32_t roff = a_row_off(tid);
  float in[K];
#pragma unroll
  for (int k = 0; k < K; k += 2) {
    const uint32_t u = *reinterpret_cast<const uint32_t*>(abuf + (k >> 3) * kAChunk + roff + (k & 7) * 2);
    in[k] = bf16_lo(u), in[k + 1] = bf16_hi(u);
  }
#pragma unroll 4
  for (int n = 0; n < N; ++n) {
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < K; k += 2) {
      const uint32_t u = *reinterpret_cast<const uint32_t*>(sm.w + woff + w_off(n, k, N));
      acc = __fmaf_rn(in[k], bf16_lo(u), acc);
      acc = __fmaf_rn(in[k + 1], bf16_hi(u), acc);
    }
    v[n] = acc;
  }
  __syncthreads();
}

// relu -> bf16 -> K-major A tile with K = 64
__device__ __forceinline__ void store_hidden(unsigned char* hbuf, int row, const float* v) {
  const uint32_t roff = a_row_off(row);
#pragma unroll
  for (int kg = 0; kg < 8; ++kg) {
    uint4 q;
    q.x = pack_bf16x2(fmaxf(v[kg * 8 + 0], 0.f), fmaxf(v[kg * 8 + 1], 0.f));
    q.y = pack_bf16x2(fmaxf(v[kg * 8 + 2], 0.f), fmaxf(v[kg * 8 + 3], 0.f));
    q.z = pack_bf16x2(fmaxf(v[kg * 8 + 4], 0.f), fmaxf(v[kg * 8 + 5], 0.f));
    q.w = pack_bf16x2(fmaxf(v[kg * 8 + 6], 0.f), fmaxf(v[kg * 8 + 7], 0.f));
    *reinterpret_cast<uint4*>(hbuf + kg * kAChunk + roff) = q;
  }
}

// One dense layer with 16 outputs; every thread ends up with its row's outputs in v[].  kSimt == true is the fp32
// CUDA-core debug path (tests only).  On return the A tile is free for the next operands.
template <bool kSimt, int K>
__device__ __forceinline__ void run_layer16(FwdSmem& sm, uint32_t woff, float* v) {
  if constexpr (!kSimt) {
    float d[16];
    mma_begin();
    mma_layer<16, K>(d, smem_u32(sm.a), smem_u32(sm.w + woff));
    mma_end();
    wgmma_fence_regs<16>(d);
    float* st = reinterpret_cast<float*>(sm.a);
    frag_stage<16, 16>(st, d);
    __syncthreads();
    stage_read_row<16>(st, v);
    __syncthreads();
  } else {
    simt_layer<16, K>(sm, sm.a, woff, v);
  }
}

// One hidden layer with 64 outputs: relu -> bf16 written over the A tile, the K = 64 operand of the next layer.
// One 64-row half at a time: the halves read and write disjoint rows of the tile, and 32 accumulators a thread
// instead of 64 keep the kernel within the 96 registers of 5 CTAs per SM without spilling.
template <bool kSimt, int K>
__device__ __forceinline__ void run_hidden(FwdSmem& sm, uint32_t woff) {
  if constexpr (!kSimt) {
    float d[32];
    mma_begin();
    mma_layer<64, K, 0>(d, smem_u32(sm.a), smem_u32(sm.w + woff));
    mma_end();
    wgmma_fence_regs<32>(d);
    frag_store_relu64<0>(sm.a, d);
    mma_begin();
    mma_layer<64, K, 1>(d, smem_u32(sm.a), smem_u32(sm.w + woff));
    mma_end();
    wgmma_fence_regs<32>(d);
    frag_store_relu64<1>(sm.a, d);
  } else {
    float v[64];
    simt_layer<64, K>(sm, sm.a, woff, v);
    store_hidden(sm.a, threadIdx.x, v);
  }
}

}  // namespace hrf
