// Table / vector gradient scatter, sixth generation: v5's lane-pair walk (scatter_pairs.cuh) unchanged; the change is
// what a CTA covers, i.e. how often the per-sample inputs stream in from HBM.
//
// v5 launches one CTA per (1024 samples, grid, half of the levels), sample blocks fastest: the GPU streams over all
// survivors 8 times and every pass re-reads positions, segment ids and the d(feature) row that is the same for all 4
// grids (about 900 B per sample in all).  The slices are far apart in launch order (one slice's d(features) alone is
// 61 MB at the bench's 950 k survivors), so a re-read is a DRAM read, not an L2 hit.
// Here a CTA owns 1024 samples and a GROUP of kV6Levels levels for every grid of the launch: positions, segment ids and
// egrid columns are staged once per CTA, each level's d(feature) row once, then the grids are walked one after another,
// staging only that grid's saved features: 552 B per sample with groups of 2 levels.  The price is the L2 working set:
// the gradient tables of 4 grids x kV6Levels levels are hot at once (2 MB per hashed level at log2T = 18).  With 2 levels
// that is 16 MB, as much as v5's fine half of one grid; 4 levels (32 MB) and 8 levels (64 MB) lose more in the L2 than
// they save in the stream (DESIGN.md section 3.3).
#include <cstdlib>

#include "scatter_pairs.cuh"

namespace hrf {

constexpr int kV6Levels = 2;   // levels per CTA (DESIGN.md section 3.3: 2 / 4 / 8 measured)
static_assert(HRF_N_LEVELS % kV6Levels == 0, "level groups tile the levels");

struct __align__(16) V6Smem {
  float4 pos[kV5Chunks * kV5Row];
  float2 df[kV5Chunks * kV5Row];
  uint32_t eg[kV5Chunks * kV5Row];
  int32_t col[kV5Samples];   // column of each staged sample inside egrid (-1 past the end), read at every (level, grid)
  uint8_t seg[kV5Samples];
};

template <bool kGather>
__global__ void __launch_bounds__(kV5Threads, 4) grid_scatter_v6_kernel(const __grid_constant__ ScatterV5Args a) {
  extern __shared__ __align__(16) unsigned char v6_raw[];
  V6Smem& sm = *reinterpret_cast<V6Smem*>(v6_raw);
  const int64_t n = live_samples(a.s);
  const int64_t base = (int64_t)blockIdx.x * kV5Samples;
  if (base >= n) return;
  const int64_t ns = a.s.num_samples;
  const int l0 = (int)blockIdx.y * kV6Levels;
  const int valid = (int)((n - base) < kV5Samples ? (n - base) : kV5Samples);
  // Staging is warp-private as in v5 (no block barrier anywhere): the warp stages the 128 samples its own lanes walk.
  const int lane = threadIdx.x & 31, w0 = (threadIdx.x >> 5) * kV5WarpSamples;
#pragma unroll
  for (int r = 0; r < kV5Stage; ++r) {
    const int s = w0 + lane + 32 * r;
    const bool ok = s < valid;
    sm.pos[(s >> 3) * kV5Row + (s & 7)] = ok ? __ldg(a.pos4 + base + s) : make_float4(0.f, 0.f, 0.f, 0.f);
    sm.seg[s] = ok ? a.seg8[base + s] : (uint8_t)255;
    if (!kGather) sm.col[s] = ok ? (a.feat_index == nullptr ? (int32_t)(base + s) : __ldg(a.feat_index + base + s)) : -1;
  }
#pragma unroll 1
  for (int li = 0; li < kV6Levels; ++li) {
    const int l = l0 + li;
#pragma unroll 1
    for (int k = a.grid_first; k < a.grid_first + a.grid_count; ++k) {
      __syncwarp();  // this warp's lanes are done with the previous walk's df / eg
      float2 d4[kV5Stage];
      const bool first = k == a.grid_first;   // the level's d(feature) row is staged once, for all grids
      if (first) {
        const float2* __restrict__ dfl = a.dfeat + (size_t)l * ns + base;
#pragma unroll
        for (int r = 0; r < kV5Stage; ++r) {
          const int s = w0 + lane + 32 * r;
          d4[r] = s < valid ? __ldg(dfl + s) : make_float2(0.f, 0.f);
        }
      }
      uint32_t e4[kV5Stage];
      if (!kGather) {
        const uint32_t* __restrict__ eg = a.egrid + (size_t)(4 * l + k) * a.egrid_stride;
#pragma unroll
        for (int r = 0; r < kV5Stage; ++r) {
          const int32_t c = sm.col[w0 + lane + 32 * r];
          e4[r] = c >= 0 ? __ldg(eg + c) : 0u;
        }
      }
#pragma unroll
      for (int r = 0; r < kV5Stage; ++r) {
        const int s = w0 + lane + 32 * r;
        if (first) sm.df[(s >> 3) * kV5Row + (s & 7)] = d4[r];
        if (!kGather) sm.eg[(s >> 3) * kV5Row + (s & 7)] = e4[r];
      }
      __syncwarp();
      if (k == 0) scatter_level_pairs<0, kGather>(a, sm, l);   // (k is uniform over the CTA)
      else if (k == 1) scatter_level_pairs<1, kGather>(a, sm, l);
      else if (k == 2) scatter_level_pairs<2, kGather>(a, sm, l);
      else scatter_level_pairs<3, kGather>(a, sm, l);
    }
  }
}

}  // namespace hrf

using namespace hrf;

// called from hrf_field_backward_tables (field_bwd.cu); HRF_SCATTER=6
int hrf_launch_scatter_v6(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads, const void* grid_feat_bf16,
                          const int32_t* feat_index, int64_t grid_feat_stride, const void* workspace, int grid_first, int grid_count,
                          cudaStream_t st) {
  HRF_REQUIRE(f->vec_res < (1 << 24), "scatter v6 keys vector rows in 24 bits");
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
  const dim3 grid((unsigned)blocks, HRF_N_LEVELS / kV6Levels);   // sample blocks fastest: one level group's tables hot at a time
  const int smem = (int)sizeof(V6Smem);
  if (grid_feat_bf16 != nullptr) grid_scatter_v6_kernel<false><<<grid, kV5Threads, smem, st>>>(a);
  else grid_scatter_v6_kernel<true><<<grid, kV5Threads, smem, st>>>(a);
  HRF_CHECK_LAUNCH();
  return 0;
}
