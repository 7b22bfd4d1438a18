// Table / vector gradient scatter, fifth generation (replaces tcnn kernel_grid_backward + compose_tensors_backward,
// tensor_composition.cu:57-118).  Its walk (scatter_pairs.cuh) is shaped by what ONE RED INSTRUCTION carries to the L2.
//
// When a thread owns all vertices of its sample, the 32 lanes of a RED instruction address 32 unrelated cells: one L2
// request of one sector per lane.  But the two vertices of a cell that differ in the FIRST axis are neighbours in the
// table (tcnn's hash multiplies the first axis by 1; a dense level is x-major): 15 times out of 16 they lie in the same
// 128-byte line.  Here the 8 parity slots of a sample chunk are split over the two lanes of a LANE PAIR by the parity of
// the first-axis vertex, and the pair flushes a slot TOGETHER (when either lane's entry changed): both entries leave in
// the same RED instruction and share one L2 request.  A lane that flushes early only splits its sum in two adds.
// The vector-row gradient is split the same way: the even lane owns tap row i0, the odd lane row i1.
// A CTA covers 1024 samples, one grid and half of the levels.  scatter_v6.cu walks the same way over a different CTA
// shape and is the one the train step runs; this kernel is its reference in the tests.  DESIGN.md section 3.3 has the
// measurements against the earlier generations.
#include <cstdlib>

#include "scatter_pairs.cuh"

namespace hrf {

constexpr int kV5Levels = 8;

struct __align__(16) V5Smem {
  float4 pos[kV5Chunks * kV5Row];
  float2 df[kV5Chunks * kV5Row];
  uint32_t eg[kV5Chunks * kV5Row];
  uint8_t seg[kV5Samples];
};

// kGrid: 0 xyz, 1 xyt, 2 yzt, 3 xzt (decomposition4d.py:126-129); its vector axis is t, z, x, y (tensor_composition.cu:49-52)
template <int kGrid, bool kGather>
__device__ __forceinline__ void scatter_levels5(const ScatterV5Args& a, V5Smem& sm, int l0, int64_t base, int valid) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t ns = a.s.num_samples;
  const int w0 = warp * kV5WarpSamples;            // the warp stages the 128 samples its own lanes walk
  int32_t col4[kV5Stage];                          // columns of this lane's staging slots inside egrid (same for every level)
  if (!kGather) {
#pragma unroll
    for (int r = 0; r < kV5Stage; ++r) {
      const int s = w0 + lane + 32 * r;
      col4[r] = s < valid ? (a.feat_index == nullptr ? (int32_t)(base + s) : __ldg(a.feat_index + base + s)) : -1;
    }
  }
#pragma unroll 1
  for (int li = 0; li < kV5Levels; ++li) {
    const int l = l0 + li;
    __syncwarp();  // this warp's lanes are done with the previous level's df / eg
    {
      const float2* __restrict__ dfl = a.dfeat + (size_t)l * ns + base;
      float2 d4[kV5Stage];
#pragma unroll
      for (int r = 0; r < kV5Stage; ++r) {
        const int s = w0 + lane + 32 * r;
        d4[r] = s < valid ? __ldg(dfl + s) : make_float2(0.f, 0.f);
      }
      uint32_t e4[kV5Stage];
      if (!kGather) {
        const uint32_t* __restrict__ eg = a.egrid + (size_t)(4 * l + kGrid) * a.egrid_stride;
#pragma unroll
        for (int r = 0; r < kV5Stage; ++r) e4[r] = col4[r] >= 0 ? __ldg(eg + col4[r]) : 0u;
      }
#pragma unroll
      for (int r = 0; r < kV5Stage; ++r) {
        const int s = w0 + lane + 32 * r;
        sm.df[(s >> 3) * kV5Row + (s & 7)] = d4[r];
        if (!kGather) sm.eg[(s >> 3) * kV5Row + (s & 7)] = e4[r];
      }
    }
    __syncwarp();
    scatter_level_pairs<kGrid, kGather>(a, sm, l);
  }
}

template <bool kGather>
__global__ void __launch_bounds__(kV5Threads, 4) grid_scatter_v5_kernel(const __grid_constant__ ScatterV5Args a) {
  extern __shared__ __align__(16) unsigned char v5_raw[];
  V5Smem& sm = *reinterpret_cast<V5Smem*>(v5_raw);
  const int64_t n = live_samples(a.s);
  const int64_t base = (int64_t)blockIdx.x * kV5Samples;
  if (base >= n) return;
  const int k = a.grid_first + (int)blockIdx.y % a.grid_count;
  const int l0 = ((int)blockIdx.y / a.grid_count) * kV5Levels;
  const int valid = (int)((n - base) < kV5Samples ? (n - base) : kV5Samples);
  {   // positions / segment ids of the 128 samples this warp's lanes walk (warp-private: no block barrier anywhere)
    const int lane = threadIdx.x & 31, w0 = (threadIdx.x >> 5) * kV5WarpSamples;
#pragma unroll
    for (int r = 0; r < kV5Stage; ++r) {
      const int s = w0 + lane + 32 * r;
      const bool ok = s < valid;
      sm.pos[(s >> 3) * kV5Row + (s & 7)] = ok ? __ldg(a.pos4 + base + s) : make_float4(0.f, 0.f, 0.f, 0.f);
      sm.seg[s] = ok ? a.seg8[base + s] : (uint8_t)255;
    }
  }
  if (k == 0) scatter_levels5<0, kGather>(a, sm, l0, base, valid);       // (k is uniform over the CTA)
  else if (k == 1) scatter_levels5<1, kGather>(a, sm, l0, base, valid);
  else if (k == 2) scatter_levels5<2, kGather>(a, sm, l0, base, valid);
  else scatter_levels5<3, kGather>(a, sm, l0, base, valid);
}

}  // namespace hrf

using namespace hrf;

// called from hrf_field_backward_tables (field_bwd.cu); HRF_SCATTER=5
int hrf_launch_scatter_v5(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads, const void* grid_feat_bf16,
                          const int32_t* feat_index, int64_t grid_feat_stride, const void* workspace, int grid_first, int grid_count,
                          cudaStream_t st) {
  HRF_REQUIRE(f->vec_res < (1 << 24), "scatter v5 keys vector rows in 24 bits");
  ScatterV5Args a;
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
  const int64_t blocks = (s->num_samples + kV5Samples - 1) / kV5Samples;
  const dim3 grid((unsigned)blocks, (HRF_N_LEVELS / kV5Levels) * grid_count);
  const int smem = (int)sizeof(V5Smem);
  if (grid_feat_bf16 != nullptr) grid_scatter_v5_kernel<false><<<grid, kV5Threads, smem, st>>>(a);
  else grid_scatter_v5_kernel<true><<<grid, kV5Threads, smem, st>>>(a);
  HRF_CHECK_LAUNCH();
  return 0;
}
