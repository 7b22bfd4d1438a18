// Gradients of the ray form's inputs from the per-sample position and direction gradients (hrf_ray_gradients).
//
// The ray form evaluates sample i of ray r at p_i = o_r + t_i d_r with view direction d_r (volume_rendering.py:66-72).
// With dpos_i = dL/dp_i (hrf_field_position_grad) and ddir_i = dL/d(view direction)_i (hrf_field_backward_mlp_dirs):
//   d_o[r] = sum_i dpos_i
//   d_d[r] = sum_i (t_i dpos_i + ddir_i)
//   d_t[i] = dpos_i . d_r
// One warp per ray: lane l sums samples lo + l, lo + l + 32, ... in order, then a fixed butterfly combines the lanes.
// No atomics and a fixed order, so two runs write identical bytes.
#include "common.cuh"

namespace hrf {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(256) ray_gradients_kernel(const float* __restrict__ d_positions,
                                                            const float* __restrict__ d_directions,
                                                            const float* __restrict__ sample_distances,
                                                            const float* __restrict__ ray_directions,
                                                            const int32_t* __restrict__ ray_offsets, int64_t num_rays,
                                                            float* __restrict__ d_origins, float* __restrict__ d_ray_directions,
                                                            float* __restrict__ d_sample_distances) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= num_rays) return;
  const int64_t lo = __ldg(ray_offsets + r), hi = __ldg(ray_offsets + r + 1);
  const float dx = __ldg(ray_directions + 3 * r), dy = __ldg(ray_directions + 3 * r + 1), dz = __ldg(ray_directions + 3 * r + 2);
  float ox = 0.f, oy = 0.f, oz = 0.f, ex = 0.f, ey = 0.f, ez = 0.f;
  for (int64_t i = lo + lane; i < hi; i += 32) {
    const float px = __ldg(d_positions + 3 * i), py = __ldg(d_positions + 3 * i + 1), pz = __ldg(d_positions + 3 * i + 2);
    const float t = __ldg(sample_distances + i);
    ox += px, oy += py, oz += pz;
    float vx = t * px, vy = t * py, vz = t * pz;
    if (d_directions != nullptr)
      vx += __ldg(d_directions + 3 * i), vy += __ldg(d_directions + 3 * i + 1), vz += __ldg(d_directions + 3 * i + 2);
    ex += vx, ey += vy, ez += vz;
    if (d_sample_distances != nullptr) d_sample_distances[i] = px * dx + py * dy + pz * dz;
  }
  ox = warp_sum(ox), oy = warp_sum(oy), oz = warp_sum(oz);
  ex = warp_sum(ex), ey = warp_sum(ey), ez = warp_sum(ez);
  if (lane == 0) {
    d_origins[3 * r] = ox, d_origins[3 * r + 1] = oy, d_origins[3 * r + 2] = oz;
    d_ray_directions[3 * r] = ex, d_ray_directions[3 * r + 1] = ey, d_ray_directions[3 * r + 2] = ez;
  }
}

}  // namespace hrf

using namespace hrf;

extern "C" int hrf_ray_gradients(const float* d_positions, const float* d_directions, const float* sample_distances,
                                 const float* ray_directions, const int32_t* ray_offsets, int64_t num_rays, float* d_origins,
                                 float* d_ray_directions, float* d_sample_distances, void* stream) {
  HRF_REQUIRE(num_rays >= 0, "negative ray count");
  if (num_rays == 0) return 0;
  HRF_REQUIRE(d_origins != nullptr && d_ray_directions != nullptr, "null output");
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (d_positions == nullptr && sample_distances == nullptr) {
    // a batch without samples (every ray missed or was pruned; empty tensors have no storage): every ray gets zeros
    HRF_CUDA(cudaMemsetAsync(d_origins, 0, 3 * sizeof(float) * (size_t)num_rays, st));
    HRF_CUDA(cudaMemsetAsync(d_ray_directions, 0, 3 * sizeof(float) * (size_t)num_rays, st));
    return 0;
  }
  HRF_REQUIRE(d_positions != nullptr && sample_distances != nullptr && ray_directions != nullptr && ray_offsets != nullptr,
              "null input");
  const int64_t blocks = (num_rays * 32 + 255) / 256;
  ray_gradients_kernel<<<(unsigned)blocks, 256, 0, st>>>(
      d_positions, d_directions, sample_distances, ray_directions, ray_offsets, num_rays, d_origins, d_ray_directions,
      d_sample_distances);
  HRF_CHECK_LAUNCH();
  return 0;
}
