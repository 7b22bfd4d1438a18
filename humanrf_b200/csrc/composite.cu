// Per-ray transmittance scans, visibility pruning and alpha compositing for sm_90a.
// Replaces the nerfacc 0.3.1 calls of humanrf/volume_rendering.py:75-84,123-145
// (render_visibility, render_weight_from_density, accumulate_along_rays) and their backward.
// One warp owns one ray; transmittance is a warp-shuffle prefix scan with a running carry,
// so no scan-by-key over the whole batch, no atomics, no [N]-sized intermediates.
#include "common.cuh"

namespace hrf {

__device__ __forceinline__ float warp_incl_sum(float v, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v += t;
  }
  return v;
}
__device__ __forceinline__ float warp_incl_prod(float v, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v *= t;
  }
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

__global__ void ray_offsets_kernel(const int64_t* __restrict__ ri, int64_t n, int64_t num_rays,
                                   int32_t* __restrict__ off) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r > num_rays) return;
  int64_t lo = 0, hi = n;  // lower_bound(ri, r)
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (__ldg(ri + mid) < r) lo = mid + 1;
    else hi = mid;
  }
  off[r] = (int32_t)lo;
}

// render_visibility (nerfacc 0.3.1): T_i = prod_{j<i} (1 - alpha_j); keep = T>=eps & alpha>=thre.
__global__ void __launch_bounds__(256) visibility_kernel(const float* __restrict__ sigma,
                                                         const int32_t* __restrict__ ray_off, int64_t num_rays,
                                                         float step, float eps, float thre,
                                                         uint8_t* __restrict__ keep, int32_t* __restrict__ kept_counts) {
  const int lane = threadIdx.x & 31;
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= num_rays) return;
  const int b = ray_off[r], e = ray_off[r + 1];
  float carry = 1.f;
  int count = 0;
  for (int i0 = b; i0 < e; i0 += 32) {
    const int i = i0 + lane;
    const bool in = i < e;
    // volume_rendering.py:76 : alphas = 1 - exp(-density * step)
    const float alpha = in ? 1.f - expf(-sigma[i] * step) : 0.f;
    const float om = 1.f - alpha;
    const float incl = warp_incl_prod(om, lane);
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 1.f;
    const float T = carry * excl;
    const bool k = in && (T >= eps) && (alpha >= thre);
    if (in) keep[i] = k ? 1 : 0;
    count += __popc(__ballot_sync(0xffffffffu, k));
    carry *= __shfl_sync(0xffffffffu, incl, 31);
  }
  if (lane == 0) kept_counts[r] = count;
}

// single-CTA exclusive scan of int32 counts -> offsets[n+1]; total also to counters[0]
// (`in` and `out` may be the same buffer -- hrf_prune scans its counts in place -- so neither is __restrict__)
__global__ void __launch_bounds__(1024) scan_i32_kernel(const int32_t* in, int64_t n, int32_t* out,
                                                        int64_t* __restrict__ counters) {
  __shared__ int warp_tot[32];
  __shared__ int carry;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int64_t base = 0; base < n; base += 1024) {
    const int64_t i = base + tid;
    const int c = (i < n) ? in[i] : 0;
    int s = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += t;
    }
    if (lane == 31) warp_tot[wid] = s;
    __syncthreads();
    if (wid == 0) {
      const int t = warp_tot[lane];
      int a = t;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, a, d);
        if (lane >= d) a += u;
      }
      warp_tot[lane] = a - t;
    }
    __syncthreads();
    const int wo = warp_tot[wid], cr = carry;
    if (i < n) out[i] = cr + wo + s - c;
    __syncthreads();
    if (tid == 1023) carry = cr + wo + s;
    __syncthreads();
  }
  if (tid == 0) {
    out[n] = carry;
    if (counters != nullptr) counters[0] = carry;
  }
}

// in-place-safe compaction of the kept samples (volume_rendering.py:83-84); warp per ray
__global__ void __launch_bounds__(256) prune_compact_kernel(const uint8_t* __restrict__ keep,
                                                            const float* __restrict__ dist,
                                                            const int32_t* __restrict__ ray_off,
                                                            const int32_t* __restrict__ kept_off, int64_t num_rays,
                                                            float* __restrict__ out_dist, int64_t* __restrict__ out_ri,
                                                            int32_t* __restrict__ out_src) {
  const int lane = threadIdx.x & 31;
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= num_rays) return;
  const int b = ray_off[r], e = ray_off[r + 1];
  int base = kept_off[r];
  for (int i0 = b; i0 < e; i0 += 32) {
    const int i = i0 + lane;
    const bool k = (i < e) && keep[i];
    const uint32_t m = __ballot_sync(0xffffffffu, k);
    if (k) {
      const int pos = base + __popc(m & ((1u << lane) - 1u));
      out_dist[pos] = dist[i];
      out_ri[pos] = r;
      if (out_src != nullptr) out_src[pos] = i;
    }
    base += __popc(m);
  }
}

// render_weight_from_density + accumulate_along_rays (+ background blend, volume_rendering.py:144-145)
__global__ void __launch_bounds__(256) composite_fwd_kernel(const float* __restrict__ sigma,
                                                            const float* __restrict__ rgb,
                                                            const float* __restrict__ dist,
                                                            const int32_t* __restrict__ ray_off, int64_t num_rays,
                                                            float step, const float* __restrict__ bg,
                                                            float* __restrict__ color, float* __restrict__ wsum,
                                                            float* __restrict__ weights) {
  const int lane = threadIdx.x & 31;
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= num_rays) return;
  const int b = ray_off[r], e = ray_off[r + 1];
  float carry = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f, ws = 0.f;
  for (int i0 = b; i0 < e; i0 += 32) {
    const int i = i0 + lane;
    const bool in = i < e;
    float sdt = 0.f;
    if (in) {
      const float t = dist[i];
      sdt = sigma[i] * __fsub_rn(__fadd_rn(t, step), t);  // sigmas * (t_ends - t_starts)
    }
    const float incl = warp_incl_sum(sdt, lane);
    const float excl = carry + (incl - sdt);
    const float w = in ? __expf(-excl) * (1.f - __expf(-sdt)) : 0.f;
    if (in) {
      if (weights != nullptr) weights[i] = w;
      c0 += w * rgb[3 * i], c1 += w * rgb[3 * i + 1], c2 += w * rgb[3 * i + 2];
      ws += w;
    }
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
  c0 = warp_sum(c0), c1 = warp_sum(c1), c2 = warp_sum(c2), ws = warp_sum(ws);
  if (lane == 0) {
    if (bg != nullptr) {
      const float k = 1.f - ws;
      c0 += bg[3 * r] * k, c1 += bg[3 * r + 1] * k, c2 += bg[3 * r + 2] * k;
    }
    color[3 * r] = c0, color[3 * r + 1] = c1, color[3 * r + 2] = c2;
    wsum[r] = ws;
  }
}

// Backward: with g_i = dC . rgb_i + (dWsum - dC . bg),
//   d(sigma_k*dt_k) = g_k T_k (1 - alpha_k) - sum_{i>k} g_i w_i ,  d rgb_i = w_i dC.
__global__ void __launch_bounds__(256) composite_bwd_kernel(const float* __restrict__ sigma,
                                                            const float* __restrict__ rgb,
                                                            const float* __restrict__ dist,
                                                            const int32_t* __restrict__ ray_off, int64_t num_rays,
                                                            float step, const float* __restrict__ bg,
                                                            const float* __restrict__ dcolor,
                                                            const float* __restrict__ dwsum,
                                                            float* __restrict__ dsigma, float* __restrict__ drgb) {
  const int lane = threadIdx.x & 31;
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= num_rays) return;
  const int b = ray_off[r], e = ray_off[r + 1];
  const float d0 = dcolor[3 * r], d1 = dcolor[3 * r + 1], d2 = dcolor[3 * r + 2];
  float gw = dwsum != nullptr ? dwsum[r] : 0.f;
  if (bg != nullptr) gw -= d0 * bg[3 * r] + d1 * bg[3 * r + 1] + d2 * bg[3 * r + 2];
  // pass 1: total of g_i w_i
  float carry = 0.f, total = 0.f;
  for (int i0 = b; i0 < e; i0 += 32) {
    const int i = i0 + lane;
    const bool in = i < e;
    float sdt = 0.f, g = 0.f;
    if (in) {
      const float t = dist[i];
      sdt = sigma[i] * __fsub_rn(__fadd_rn(t, step), t);
      g = d0 * rgb[3 * i] + d1 * rgb[3 * i + 1] + d2 * rgb[3 * i + 2] + gw;
    }
    const float incl = warp_incl_sum(sdt, lane);
    const float excl = carry + (incl - sdt);
    if (in) total += g * __expf(-excl) * (1.f - __expf(-sdt));
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
  total = warp_sum(total);
  // pass 2: gradients
  carry = 0.f;
  float pref = 0.f;  // sum_{i<chunk} g_i w_i
  for (int i0 = b; i0 < e; i0 += 32) {
    const int i = i0 + lane;
    const bool in = i < e;
    float sdt = 0.f, g = 0.f, dt = 0.f;
    if (in) {
      const float t = dist[i];
      dt = __fsub_rn(__fadd_rn(t, step), t);
      sdt = sigma[i] * dt;
      g = d0 * rgb[3 * i] + d1 * rgb[3 * i + 1] + d2 * rgb[3 * i + 2] + gw;
    }
    const float incl = warp_incl_sum(sdt, lane);
    const float excl = carry + (incl - sdt);
    const float T = __expf(-excl), ea = __expf(-sdt);
    const float w = in ? T * (1.f - ea) : 0.f;
    const float gwv = g * w;
    const float gincl = warp_incl_sum(gwv, lane);
    if (in) {
      const float suffix = total - (pref + gincl);  // sum_{i>k} g_i w_i
      dsigma[i] = (g * T * ea - suffix) * dt;
      if (drgb != nullptr) drgb[3 * i] = w * d0, drgb[3 * i + 1] = w * d1, drgb[3 * i + 2] = w * d2;
    }
    pref += __shfl_sync(0xffffffffu, gincl, 31);
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
}

}  // namespace hrf

using namespace hrf;

static inline unsigned warp_grid(int64_t rays) { return (unsigned)((rays * 32 + 255) / 256); }

extern "C" int hrf_ray_offsets(const int64_t* ray_indices, int64_t num_samples, int64_t num_rays, int32_t* ray_offsets,
                               void* stream) {
  HRF_REQUIRE(num_samples < (1ll << 31), "more than 2^31 samples per batch is not supported");
  ray_offsets_kernel<<<(unsigned)((num_rays + 1 + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      ray_indices, num_samples, num_rays, ray_offsets);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_prune(const float* sigma, const float* sample_distances, const int64_t* ray_indices,
                         const int32_t* ray_offsets, int64_t num_rays, float step, float early_stop_eps,
                         float alpha_thre, uint8_t* keep_mask, int32_t* kept_offsets, float* out_distances,
                         int64_t* out_ray_indices, int32_t* out_source_index, int64_t* counters, void* stream) {
  (void)ray_indices;
  HRF_REQUIRE(kept_offsets != nullptr && counters != nullptr, "null workspace");  // keep_mask may be NULL only for N == 0
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (num_rays == 0) {
    HRF_CUDA(cudaMemsetAsync(counters, 0, sizeof(int64_t), st));
    return 0;
  }
  // kept_offsets doubles as the per-ray count buffer before the scan (scan is in-place safe)
  visibility_kernel<<<warp_grid(num_rays), 256, 0, st>>>(sigma, ray_offsets, num_rays, step, early_stop_eps,
                                                         alpha_thre, keep_mask, kept_offsets);
  HRF_CHECK_LAUNCH();
  scan_i32_kernel<<<1, 1024, 0, st>>>(kept_offsets, num_rays, kept_offsets, counters);
  HRF_CHECK_LAUNCH();
  if (out_distances != nullptr) {
    prune_compact_kernel<<<warp_grid(num_rays), 256, 0, st>>>(keep_mask, sample_distances, ray_offsets, kept_offsets,
                                                              num_rays, out_distances, out_ray_indices, out_source_index);
    HRF_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int hrf_composite_forward(const float* sigma, const float* rgb, const float* sample_distances,
                                     const int32_t* ray_offsets, int64_t num_rays, float step, const float* background,
                                     float* color, float* weights_sum, float* weights, void* stream) {
  if (num_rays == 0) return 0;
  composite_fwd_kernel<<<warp_grid(num_rays), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      sigma, rgb, sample_distances, ray_offsets, num_rays, step, background, color, weights_sum, weights);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_composite_backward(const float* sigma, const float* rgb, const float* sample_distances,
                                      const int32_t* ray_offsets, int64_t num_rays, float step, const float* background,
                                      const float* d_color, const float* d_weights_sum, float* d_sigma, float* d_rgb,
                                      void* stream) {
  if (num_rays == 0) return 0;
  composite_bwd_kernel<<<warp_grid(num_rays), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      sigma, rgb, sample_distances, ray_offsets, num_rays, step, background, d_color, d_weights_sum, d_sigma, d_rgb);
  HRF_CHECK_LAUNCH();
  return 0;
}
