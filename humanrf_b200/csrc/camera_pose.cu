// Per-camera pose refinement inside the fused train step (hrf_camera_pose_grad, hrf_camera_pose_step).
//
// Camera c carries an increment (omega_c, tau_c): R' = exp([omega_c]x) R and c' = c + tau_c, in normalised scene units.
// A ray r of camera c was sampled from the tables of the current increment, so o_r = c_c + tau_c and
// d_r = exp([omega_c]x) d0_r.  With g_o, g_d the per-ray gradients of hrf_ray_gradients:
//   dL/dtau_c   = sum_{r in c} g_o[r]
//   dL/domega_c = J_l(omega_c)^T sum_{r in c} (d_r x g_d[r])
//   J_l(w) = I + (1 - cos t)/t^2 [w]x + (t - sin t)/t^3 [w]x^2,  t = |w|
// (the left Jacobian of SO(3): exp([w + e]x) = exp([J_l(w) e]x) exp([w]x) to first order in e).
//
// hrf_camera_pose_grad, two launches, no float atomics:
//   pose_partials_kernel : block b sums a contiguous range of rays.  Each warp takes 32-ray tiles of the range in turn;
//                          in a tile the lanes of one camera are found with __match_any_sync and summed by a fixed tree
//                          whose shape depends only on their lane positions, and the lowest lane adds the sum to the
//                          warp's own per-camera slot in shared memory (one writer per camera per tile).  The warps'
//                          slots are then added in warp order into the block's partial record per camera.
//   pose_finish_kernel   : one thread per camera adds the blocks' partials in block order and applies J_l^T (float64).
// The block count depends on R alone, so the order of every addition is fixed by the batch: two runs write identical
// bytes.
//
// hrf_camera_pose_step, one single-CTA launch: Adam for every camera that had rays and is not fixed, the camera's
// sampler tables rebuilt in float64 from the base tables and rounded once, then the pool slots' copies.
#include "common.cuh"

namespace hrf {

constexpr int kPoseWarps = 4;
constexpr int kPoseThreads = 32 * kPoseWarps;
constexpr int kPoseMaxBlocks = 256;
constexpr int kPoseRaysPerBlock = 2048;        // a block sums at least this many rays before more blocks are used
constexpr int kPoseMaxCameras = 1024;

struct PoseSlot {                              // 32 bytes: 6 sums, the ray count, padding
  float v[6];
  int n;
  int pad;
};

__host__ __device__ inline int pose_blocks(int64_t num_rays) {
  const int64_t b = (num_rays + kPoseRaysPerBlock - 1) / kPoseRaysPerBlock;
  return (int)(b < kPoseMaxBlocks ? b : kPoseMaxBlocks);
}

// Sum of x over the lanes of `peers` (this lane included), left in the lowest lane of `peers`.  A tree over the peers'
// ranks: round k adds the partial 2^k ranks up.  Every lane of the warp runs every round.
template <int N>
__device__ __forceinline__ void reduce_peers(unsigned peers, float (&x)[N]) {
  const int lane = threadIdx.x & 31;
  int rank = __popc(peers & ((1u << lane) - 1u));
  unsigned above = peers & ~((2u << lane) - 1u);
  while (__any_sync(0xffffffffu, above != 0)) {
    const int next = __ffs(above);                     // 1-based; 0 = none
    const int src = next ? next - 1 : lane;
#pragma unroll
    for (int k = 0; k < N; ++k) {
      const float t = __shfl_sync(0xffffffffu, x[k], src);
      if (next) x[k] += t;
    }
    above &= __ballot_sync(0xffffffffu, (rank & 1) == 0);
    rank >>= 1;
  }
}

__global__ void __launch_bounds__(kPoseThreads) pose_partials_kernel(
    const float* __restrict__ d_origins, const float* __restrict__ d_ray_directions,
    const float* __restrict__ ray_directions, const int32_t* __restrict__ camera_numbers, int64_t num_rays,
    int num_cameras, int64_t rays_per_block, PoseSlot* __restrict__ partials, int32_t* __restrict__ error) {
  extern __shared__ PoseSlot acc[];                    // [kPoseWarps][num_cameras]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < kPoseWarps * num_cameras; i += kPoseThreads) {
#pragma unroll
    for (int k = 0; k < 6; ++k) acc[i].v[k] = 0.f;
    acc[i].n = 0;
  }
  __syncthreads();
  const int64_t lo = (int64_t)blockIdx.x * rays_per_block;
  const int64_t hi = min(lo + rays_per_block, num_rays);
  PoseSlot* mine = acc + warp * num_cameras;
  unsigned bad = 0;
  for (int64_t base = lo + 32 * warp; base < hi; base += 32 * kPoseWarps) {
    const int64_t r = base + lane;
    int cam = -1;
    float x[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (r < hi) {
      const int c = __ldg(camera_numbers + r);
      if (c >= 0 && c < num_cameras) {
        cam = c;
        const float dx = __ldg(ray_directions + 3 * r), dy = __ldg(ray_directions + 3 * r + 1),
                    dz = __ldg(ray_directions + 3 * r + 2);
        const float gx = __ldg(d_ray_directions + 3 * r), gy = __ldg(d_ray_directions + 3 * r + 1),
                    gz = __ldg(d_ray_directions + 3 * r + 2);
        x[0] = dy * gz - dz * gy, x[1] = dz * gx - dx * gz, x[2] = dx * gy - dy * gx;
        x[3] = __ldg(d_origins + 3 * r), x[4] = __ldg(d_origins + 3 * r + 1), x[5] = __ldg(d_origins + 3 * r + 2);
      } else {
        bad = 1;
      }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, cam);
    reduce_peers<6>(peers, x);
    if (cam >= 0 && lane == __ffs(peers) - 1) {
#pragma unroll
      for (int k = 0; k < 6; ++k) mine[cam].v[k] += x[k];
      mine[cam].n += __popc(peers);
    }
    __syncwarp();
  }
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(error, 1);
  __syncthreads();
  for (int c = threadIdx.x; c < num_cameras; c += kPoseThreads) {
    PoseSlot s = acc[c];
    for (int w = 1; w < kPoseWarps; ++w) {
      const PoseSlot& t = acc[w * num_cameras + c];
#pragma unroll
      for (int k = 0; k < 6; ++k) s.v[k] += t.v[k];
      s.n += t.n;
    }
    partials[(int64_t)blockIdx.x * num_cameras + c] = s;
  }
}

// sin(t)/t, (1 - cos t)/t^2, (t - sin t)/t^3 at t^2 = th2; Taylor series below t = 1e-2 (truncation < 1e-17 relative).
__device__ __forceinline__ void so3_coeffs(double th2, double& a, double& b, double& c) {
  if (th2 < 1e-4) {
    a = 1.0 - th2 / 6.0 * (1.0 - th2 / 20.0 * (1.0 - th2 / 42.0));
    b = 0.5 * (1.0 - th2 / 12.0 * (1.0 - th2 / 30.0 * (1.0 - th2 / 56.0)));
    c = (1.0 - th2 / 20.0 * (1.0 - th2 / 42.0 * (1.0 - th2 / 72.0))) / 6.0;
  } else {
    const double th = sqrt(th2), s = sin(th), co = cos(th);
    a = s / th, b = (1.0 - co) / th2, c = (th - s) / (th2 * th);
  }
}

// I + p [w]x + q [w]x^2, row-major.
__device__ __forceinline__ void so3_matrix(const double w[3], double p, double q, double m[9]) {
  const double K[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double k2 = K[3 * i] * K[j] + K[3 * i + 1] * K[3 + j] + K[3 * i + 2] * K[6 + j];
      m[3 * i + j] = (i == j ? 1.0 : 0.0) + p * K[3 * i + j] + q * k2;
    }
}

__global__ void __launch_bounds__(128) pose_finish_kernel(const PoseSlot* __restrict__ partials, int num_blocks,
                                                          int num_cameras, const double* __restrict__ omega,
                                                          float* __restrict__ pose_grad, int32_t* __restrict__ ray_count) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= num_cameras) return;
  float s[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  int n = 0;
  for (int b = 0; b < num_blocks; ++b) {
    const PoseSlot& p = partials[(int64_t)b * num_cameras + c];
#pragma unroll
    for (int k = 0; k < 6; ++k) s[k] += p.v[k];
    n += p.n;
  }
  const double w[3] = {omega[3 * c], omega[3 * c + 1], omega[3 * c + 2]};
  double a, b, cc, J[9];
  so3_coeffs(w[0] * w[0] + w[1] * w[1] + w[2] * w[2], a, b, cc);
  so3_matrix(w, b, cc, J);
#pragma unroll
  for (int j = 0; j < 3; ++j)     // (J^T s)_j = sum_i J[i][j] s_i
    pose_grad[6 * c + j] = (float)(J[j] * (double)s[0] + J[3 + j] * (double)s[1] + J[6 + j] * (double)s[2]);
#pragma unroll
  for (int j = 3; j < 6; ++j) pose_grad[6 * c + j] = s[j];
  ray_count[c] = n;
}

__global__ void __launch_bounds__(256) pose_step_kernel(hrf_camera_poses p, const float* __restrict__ pose_grad,
                                                        const int32_t* __restrict__ ray_count,
                                                        const int32_t* __restrict__ error, double lr, double beta1,
                                                        double beta2, double eps) {
  if (error != nullptr && *error != 0) return;
  for (int c = threadIdx.x; c < p.num_cameras; c += blockDim.x) {
    if (ray_count[c] == 0 || p.fixed[c] != 0) continue;
    const int step = p.step[c] + 1;
    p.step[c] = step;
    const double bc1 = 1.0 - pow(beta1, (double)step), bc2s = sqrt(1.0 - pow(beta2, (double)step));
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const double g = (double)pose_grad[6 * c + k];
      const double m = beta1 * p.exp_avg[6 * c + k] + (1.0 - beta1) * g;
      const double v = beta2 * p.exp_avg_sq[6 * c + k] + (1.0 - beta2) * g * g;
      p.exp_avg[6 * c + k] = m, p.exp_avg_sq[6 * c + k] = v;
      double* q = k < 3 ? p.omega + 3 * c + k : p.tau + 3 * c + k - 3;
      *q -= lr / bc1 * (m / (sqrt(v) / bc2s + eps));   // torch.optim.Adam
    }
    // table: (exp([w]x) M)^T with M = T^T, T the base table: T'[i][j] = sum_k R[j][k] T[i][k]
    const double w[3] = {p.omega[3 * c], p.omega[3 * c + 1], p.omega[3 * c + 2]};
    double a, b, cc, R[9], T[9];
    so3_coeffs(w[0] * w[0] + w[1] * w[1] + w[2] * w[2], a, b, cc);
    so3_matrix(w, a, b, R);
#pragma unroll
    for (int i = 0; i < 9; ++i) T[i] = (double)p.base_inverse_krs[9 * c + i];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j)
        p.inverse_krs[9 * c + 3 * i + j] =
            (float)(R[3 * j] * T[3 * i] + R[3 * j + 1] * T[3 * i + 1] + R[3 * j + 2] * T[3 * i + 2]);
#pragma unroll
    for (int k = 0; k < 3; ++k) p.camera_origins[3 * c + k] = (float)((double)p.base_camera_origins[3 * c + k] + p.tau[3 * c + k]);
  }
  __syncthreads();                // the per-camera tables written above are visible to the whole block
  for (int s = threadIdx.x; s < p.num_slots; s += blockDim.x) {
    const int c = p.slot_camera_numbers[s];
    if (c < 0 || c >= p.num_cameras) continue;
#pragma unroll
    for (int i = 0; i < 9; ++i) p.slot_inverse_krs[9 * s + i] = p.inverse_krs[9 * c + i];
#pragma unroll
    for (int k = 0; k < 3; ++k) p.slot_camera_origins[3 * s + k] = p.camera_origins[3 * c + k];
  }
}

}  // namespace hrf

using namespace hrf;

extern "C" int64_t hrf_camera_pose_grad_workspace_bytes(int num_cameras) {
  if (num_cameras < 1 || num_cameras > kPoseMaxCameras) return -1;
  return (int64_t)kPoseMaxBlocks * num_cameras * (int64_t)sizeof(PoseSlot);
}

extern "C" int hrf_camera_pose_grad(const float* d_origins, const float* d_ray_directions, const float* ray_directions,
                                    const int32_t* camera_numbers, int64_t num_rays, const double* omega, int num_cameras,
                                    float* pose_grad, int32_t* ray_count, int32_t* error, void* workspace, void* stream) {
  HRF_REQUIRE(num_rays >= 0 && num_rays < ((int64_t)1 << 31), "ray count outside [0, 2^31)");
  HRF_REQUIRE(num_cameras >= 1 && num_cameras <= kPoseMaxCameras, "camera count outside [1, 1024]");
  HRF_REQUIRE(omega != nullptr && pose_grad != nullptr && ray_count != nullptr && error != nullptr, "null argument");
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int blocks = pose_blocks(num_rays);
  if (blocks > 0) {
    HRF_REQUIRE(d_origins != nullptr && d_ray_directions != nullptr && ray_directions != nullptr &&
                    camera_numbers != nullptr && workspace != nullptr,
                "null input");
    const size_t smem = (size_t)kPoseWarps * num_cameras * sizeof(PoseSlot);
    if (smem > 48 * 1024)     // more than 384 cameras
      HRF_CUDA(cudaFuncSetAttribute(pose_partials_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t per_block = (num_rays + blocks - 1) / blocks;
    pose_partials_kernel<<<blocks, kPoseThreads, smem, st>>>(d_origins, d_ray_directions, ray_directions, camera_numbers,
                                                             num_rays, num_cameras, per_block,
                                                             reinterpret_cast<PoseSlot*>(workspace), error);
    HRF_CHECK_LAUNCH();
  }
  pose_finish_kernel<<<(num_cameras + 127) / 128, 128, 0, st>>>(reinterpret_cast<const PoseSlot*>(workspace), blocks,
                                                                num_cameras, omega, pose_grad, ray_count);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_camera_pose_step(const hrf_camera_poses* poses, const float* pose_grad, const int32_t* ray_count,
                                    const int32_t* error, double lr, double beta1, double beta2, double eps,
                                    void* stream) {
  HRF_REQUIRE(poses != nullptr && pose_grad != nullptr && ray_count != nullptr, "null argument");
  const hrf_camera_poses& p = *poses;
  HRF_REQUIRE(p.num_cameras >= 1 && p.num_cameras <= kPoseMaxCameras, "camera count outside [1, 1024]");
  HRF_REQUIRE(p.num_slots >= 0, "negative slot count");
  HRF_REQUIRE(p.omega && p.tau && p.exp_avg && p.exp_avg_sq && p.step && p.fixed && p.base_inverse_krs &&
                  p.base_camera_origins && p.inverse_krs && p.camera_origins,
              "null camera table");
  HRF_REQUIRE(p.num_slots == 0 || (p.slot_inverse_krs && p.slot_camera_origins && p.slot_camera_numbers),
              "null slot table");
  pose_step_kernel<<<1, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p, pose_grad, ray_count, error, lr, beta1,
                                                                          beta2, eps);
  HRF_CHECK_LAUNCH();
  return 0;
}
