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
//
// Intrinsics (hrf_camera_calib_grad, hrf_camera_calib_step, DESIGN.md §3.15): camera c also carries alpha_c (log focal
// scales) and beta_c (principal-point offsets in units of the base focal length), u' = ((x0 - bx) e^-ax, (y0 - by) e^-ay, 1)
// for the base camera coordinates (x0, y0, 1) of a pixel, d = R' u' / |u'| with R' = exp([omega]x) R.  With
// q = R'^T d_r = u' / |u'| and h = R'^T (g_d - d_r (d_r . g_d)), dL/du' = q_z h, so
//   dL/dalpha_x = -sum_r q_x h_x,   dL/dbeta_x = -e^-alpha_x sum_r q_z h_x   (same for y)
// needs only d_r, g_d and R'_c.  The same two launches sum the four extra terms beside the pose's six: the pose columns
// take the same lane tree and block order, so they are bit-identical to hrf_camera_pose_grad's.
//
// Data parallel (hrf_camera_pose_step_ranks, hrf_camera_calib_step_ranks, DESIGN.md §3.16): one single-CTA launch per rank
// reduces the W ranks' gradient records in rank order and runs the same per-camera step (camera_step_body) and slot copy
// as the single-rank kernels.
#include <type_traits>

#include "camera_common.cuh"

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
struct CalibSlot {                             // 48 bytes: the pose's 6 sums, the intrinsics' 4, the ray count, padding
  float v[10];
  int n;
  int pad;
};

__host__ __device__ inline int pose_blocks(int64_t num_rays) {
  const int64_t b = (num_rays + kPoseRaysPerBlock - 1) / kPoseRaysPerBlock;
  return (int)(b < kPoseMaxBlocks ? b : kPoseMaxBlocks);
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


// pose_partials_kernel with the four intrinsics terms (CalibSlot).  The pose terms are formed by the same expressions
// and summed by the same tree in the same order, so the pose columns are bit-identical to pose_partials_kernel's.
__global__ void __launch_bounds__(kPoseThreads) calib_partials_kernel(
    const float* __restrict__ d_origins, const float* __restrict__ d_ray_directions,
    const float* __restrict__ ray_directions, const int32_t* __restrict__ camera_numbers,
    const float* __restrict__ rotations, int64_t num_rays, int num_cameras, int64_t rays_per_block,
    CalibSlot* __restrict__ partials, int32_t* __restrict__ error) {
  extern __shared__ CalibSlot cacc[];                    // [kPoseWarps][num_cameras]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < kPoseWarps * num_cameras; i += kPoseThreads) {
#pragma unroll
    for (int k = 0; k < 10; ++k) cacc[i].v[k] = 0.f;
    cacc[i].n = 0;
  }
  __syncthreads();
  const int64_t lo = (int64_t)blockIdx.x * rays_per_block;
  const int64_t hi = min(lo + rays_per_block, num_rays);
  CalibSlot* mine = cacc + warp * num_cameras;
  unsigned bad = 0;
  for (int64_t base = lo + 32 * warp; base < hi; base += 32 * kPoseWarps) {
    const int64_t r = base + lane;
    int cam = -1;
    float x[10] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
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
        // q = R'^T d, h = R'^T (g_d - d (d . g_d)) (x, y only); the terms q_x h_x, q_y h_y, q_z h_x, q_z h_y
        const float* Rc = rotations + 9 * c;
        float Rm[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) Rm[i] = __ldg(Rc + i);
        const float dg = dx * gx + dy * gy + dz * gz;
        const float px = gx - dx * dg, py = gy - dy * dg, pz = gz - dz * dg;
        const float qx = Rm[0] * dx + Rm[3] * dy + Rm[6] * dz, qy = Rm[1] * dx + Rm[4] * dy + Rm[7] * dz,
                    qz = Rm[2] * dx + Rm[5] * dy + Rm[8] * dz;
        const float hx = Rm[0] * px + Rm[3] * py + Rm[6] * pz, hy = Rm[1] * px + Rm[4] * py + Rm[7] * pz;
        x[6] = qx * hx, x[7] = qy * hy, x[8] = qz * hx, x[9] = qz * hy;
      } else {
        bad = 1;
      }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, cam);
    reduce_peers<10>(peers, x);
    if (cam >= 0 && lane == __ffs(peers) - 1) {
#pragma unroll
      for (int k = 0; k < 10; ++k) mine[cam].v[k] += x[k];
      mine[cam].n += __popc(peers);
    }
    __syncwarp();
  }
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(error, 1);
  __syncthreads();
  for (int c = threadIdx.x; c < num_cameras; c += kPoseThreads) {
    CalibSlot s = cacc[c];
    for (int w = 1; w < kPoseWarps; ++w) {
      const CalibSlot& t = cacc[w * num_cameras + c];
#pragma unroll
      for (int k = 0; k < 10; ++k) s.v[k] += t.v[k];
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

// One thread per camera: the blocks' partials in block order, then J_l^T (float64).  kCalib also writes
// intrinsics_grad [C,4] = (-s6, -s7, -e^-alpha_x s8, -e^-alpha_y s9) (float64 before the rounding).
template <bool kCalib>
__device__ __forceinline__ void pose_finish_body(const std::conditional_t<kCalib, CalibSlot, PoseSlot>* __restrict__ partials,
                                                 int num_blocks, int num_cameras, const double* __restrict__ omega,
                                                 const double* __restrict__ alpha, float* __restrict__ pose_grad,
                                                 float* __restrict__ intrinsics_grad, int32_t* __restrict__ ray_count) {
  using Slot = std::conditional_t<kCalib, CalibSlot, PoseSlot>;
  constexpr int kSums = kCalib ? 10 : 6;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= num_cameras) return;
  float s[kSums];
#pragma unroll
  for (int k = 0; k < kSums; ++k) s[k] = 0.f;
  int n = 0;
  for (int b = 0; b < num_blocks; ++b) {
    const Slot& p = partials[(int64_t)b * num_cameras + c];
#pragma unroll
    for (int k = 0; k < kSums; ++k) s[k] += p.v[k];
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
  if constexpr (kCalib) {
    intrinsics_grad[4 * c] = -s[6];
    intrinsics_grad[4 * c + 1] = -s[7];
    intrinsics_grad[4 * c + 2] = (float)(-exp(-alpha[2 * c]) * (double)s[8]);
    intrinsics_grad[4 * c + 3] = (float)(-exp(-alpha[2 * c + 1]) * (double)s[9]);
  }
  ray_count[c] = n;
}

__global__ void __launch_bounds__(128) pose_finish_kernel(const PoseSlot* __restrict__ partials, int num_blocks,
                                                          int num_cameras, const double* __restrict__ omega,
                                                          float* __restrict__ pose_grad, int32_t* __restrict__ ray_count) {
  pose_finish_body<false>(partials, num_blocks, num_cameras, omega, nullptr, pose_grad, nullptr, ray_count);
}

__global__ void __launch_bounds__(128) calib_finish_kernel(const CalibSlot* __restrict__ partials, int num_blocks,
                                                           int num_cameras, const double* __restrict__ omega,
                                                           const double* __restrict__ alpha, float* __restrict__ pose_grad,
                                                           float* __restrict__ intrinsics_grad,
                                                           int32_t* __restrict__ ray_count) {
  pose_finish_body<true>(partials, num_blocks, num_cameras, omega, alpha, pose_grad, intrinsics_grad, ray_count);
}

// Adam on camera c's (omega, tau) at lr and, with kCalib, on its (alpha, beta) at lr_intrinsics with the same step
// counter; then its table and origin (and with kCalib its rotation) in float64, rounded once.  grad(k) is the camera's
// gradient entry k in float64: 0..5 the pose, 6..9 the intrinsics.  Every step kernel runs this for a camera it moves.
//
// Without intrinsics the table is (exp([w]x) M)^T with M = T^T, T the base table: T'[i][j] = sum_k R[j][k] T[i][k].
// With them it is (exp([omega]x) M0 B)^T in float64, rounded once.  B = K0 A K0^-1 acts on the base table's rows:
// T'0 = e^-ax T0, T'1 = e^-ay T1, T'2 = T2 + B02 T0 + B12 T1 with B02 = -cx0 expm1(-ax) - fx0 bx e^-ax.  A zero B02 / B12
// is not added, so alpha = beta = 0 gives M0 exactly (signed zeros included) and the table equals the pose-only one bit
// for bit.  The current rotation exp([omega]x) R is rewritten for the next hrf_camera_calib_grad.
template <bool kCalib, class Grad>
__device__ __forceinline__ void camera_step_body(const hrf_camera_poses& p, const hrf_camera_intrinsics& q, int c,
                                                 Grad grad, double lr, double lr_intrinsics, double beta1, double beta2,
                                                 double eps) {
  const int step = p.step[c] + 1;
  p.step[c] = step;
  const double bc1 = 1.0 - pow(beta1, (double)step), bc2s = sqrt(1.0 - pow(beta2, (double)step));
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    double* x = k < 3 ? p.omega + 3 * c + k : p.tau + 3 * c + k - 3;
    adam_update(grad(k), p.exp_avg[6 * c + k], p.exp_avg_sq[6 * c + k], *x, lr / bc1, bc2s, beta1, beta2, eps);
  }
  if constexpr (kCalib) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      double* x = k < 2 ? q.alpha + 2 * c + k : q.beta + 2 * c + k - 2;
      adam_update(grad(6 + k), q.exp_avg[4 * c + k], q.exp_avg_sq[4 * c + k], *x, lr_intrinsics / bc1, bc2s, beta1, beta2,
                  eps);
    }
  }
  const double w[3] = {p.omega[3 * c], p.omega[3 * c + 1], p.omega[3 * c + 2]};
  double a, b, cc, R[9], T[9];
  so3_coeffs(w[0] * w[0] + w[1] * w[1] + w[2] * w[2], a, b, cc);
  so3_matrix(w, a, b, R);
  if constexpr (kCalib) {
    const double ax = q.alpha[2 * c], ay = q.alpha[2 * c + 1], bx = q.beta[2 * c], by = q.beta[2 * c + 1];
    const double fx0 = q.base_intrinsics[4 * c], fy0 = q.base_intrinsics[4 * c + 1];
    const double cx0 = q.base_intrinsics[4 * c + 2], cy0 = q.base_intrinsics[4 * c + 3];
    const double ex = exp(-ax), ey = exp(-ay);
    const double b02 = -cx0 * expm1(-ax) - fx0 * bx * ex, b12 = -cy0 * expm1(-ay) - fy0 * by * ey;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double t0 = (double)p.base_inverse_krs[9 * c + k], t1 = (double)p.base_inverse_krs[9 * c + 3 + k];
      double t2 = (double)p.base_inverse_krs[9 * c + 6 + k];
      if (b02 != 0.0) t2 += b02 * t0;
      if (b12 != 0.0) t2 += b12 * t1;
      T[k] = t0 * ex, T[3 + k] = t1 * ey, T[6 + k] = t2;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 9; ++i) T[i] = (double)p.base_inverse_krs[9 * c + i];
  }
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      p.inverse_krs[9 * c + 3 * i + j] =
          (float)(R[3 * j] * T[3 * i] + R[3 * j + 1] * T[3 * i + 1] + R[3 * j + 2] * T[3 * i + 2]);
#pragma unroll
  for (int k = 0; k < 3; ++k) p.camera_origins[3 * c + k] = (float)((double)p.base_camera_origins[3 * c + k] + p.tau[3 * c + k]);
  if constexpr (kCalib) {
    const double* Rb = q.base_rotations + 9 * c;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j)
        q.rotations[9 * c + 3 * i + j] = (float)(R[3 * i] * Rb[j] + R[3 * i + 1] * Rb[3 + j] + R[3 * i + 2] * Rb[6 + j]);
  }
}

// Every pool slot that holds a camera copies that camera's tables.  The caller has synchronised the block after the
// per-camera tables were written.
__device__ __forceinline__ void slot_copy_body(const hrf_camera_poses& p) {
  for (int s = threadIdx.x; s < p.num_slots; s += blockDim.x) {
    const int c = p.slot_camera_numbers[s];
    if (c < 0 || c >= p.num_cameras) continue;
#pragma unroll
    for (int i = 0; i < 9; ++i) p.slot_inverse_krs[9 * s + i] = p.inverse_krs[9 * c + i];
#pragma unroll
    for (int k = 0; k < 3; ++k) p.slot_camera_origins[3 * s + k] = p.camera_origins[3 * c + k];
  }
}

__global__ void __launch_bounds__(256) pose_step_kernel(hrf_camera_poses p, const float* __restrict__ pose_grad,
                                                        const int32_t* __restrict__ ray_count,
                                                        const int32_t* __restrict__ error, double lr, double beta1,
                                                        double beta2, double eps) {
  if (error != nullptr && *error != 0) return;
  const hrf_camera_intrinsics none{};
  for (int c = threadIdx.x; c < p.num_cameras; c += blockDim.x) {
    if (ray_count[c] == 0 || p.fixed[c] != 0) continue;
    camera_step_body<false>(p, none, c, [&](int k) { return (double)pose_grad[6 * c + k]; }, lr, 0.0, beta1, beta2, eps);
  }
  __syncthreads();                // the per-camera tables written above are visible to the whole block
  slot_copy_body(p);
}

// hrf_camera_calib_step: pose_step_kernel's Adam and origin for (omega, tau), Adam at lr_intrinsics for (alpha, beta)
// with the same step counter, then the table with the intrinsics and the rotation (camera_step_body<true>).
__global__ void __launch_bounds__(256) calib_step_kernel(hrf_camera_poses p, hrf_camera_intrinsics q,
                                                         const float* __restrict__ pose_grad,
                                                         const float* __restrict__ intrinsics_grad,
                                                         const int32_t* __restrict__ ray_count,
                                                         const int32_t* __restrict__ error, double lr,
                                                         double lr_intrinsics, double beta1, double beta2, double eps) {
  if (error != nullptr && *error != 0) return;
  for (int c = threadIdx.x; c < p.num_cameras; c += blockDim.x) {
    if (ray_count[c] == 0 || p.fixed[c] != 0) continue;
    camera_step_body<true>(p, q, c,
                           [&](int k) { return k < 6 ? (double)pose_grad[6 * c + k] : (double)intrinsics_grad[4 * c + k - 6]; },
                           lr, lr_intrinsics, beta1, beta2, eps);
  }
  __syncthreads();                // the per-camera tables written above are visible to the whole block
  slot_copy_body(p);
}

// The data-parallel step (hrf_camera_pose_step_ranks / hrf_camera_calib_step_ranks, DESIGN.md §3.16), one CTA on every
// rank over the same W records (header: the record layout).
//   1. Any rank's error word set: nothing is written; a rank that sees bit 0 (a bad camera number) in ANOTHER rank's
//      word sets bit 1 of its own sticky word.  Bit 0 is only written by the gradient kernels, which every rank's
//      barrier orders before this kernel, so every rank takes the same decision even while a peer sets its bit 1.
//   2. The records are staged into shared memory, one record word per thread and step, coalesced: the gradient entry
//      as (sum over r = 0..W-1 in rank order of (double)grad_r) / W, the camera's touched flag as the OR of the ray
//      counts.  At W = 1 the entry is (double)grad_0 exactly: the single-rank kernels' input.
//   3. Every touched camera that is not fixed takes camera_step_body, then the slots are copied.
constexpr int kRankStepThreads = 384;

template <bool kCalib>
__global__ void __launch_bounds__(kRankStepThreads) step_ranks_kernel(hrf_camera_poses p, hrf_camera_intrinsics q,
                                                                      hrf_camera_grad_records rec, int32_t* error,
                                                                      double lr, double lr_intrinsics, double beta1,
                                                                      double beta2, double eps) {
  extern __shared__ double sgrad[];                    // [C][10] reduced gradients, then int32 touched [C]
  const int C = p.num_cameras, W = rec.world;
  int any = 0, peer_bad = 0;
#pragma unroll
  for (int r = 0; r < HRF_DP_MAX_WORLD; ++r) {
    if (r < W) {
      const int e = reinterpret_cast<const int32_t*>(rec.record[r])[11 * C];
      any |= e;
      if (r != rec.rank) peer_bad |= e & 1;
    }
  }
  if (any != 0) {
    if (threadIdx.x == 0 && peer_bad != 0) atomicOr(error, 2);
    return;
  }
  int* touched = reinterpret_cast<int*>(sgrad + 10 * C);
  constexpr int kSums = kCalib ? 10 : 6;
  const int n_sums = kSums * C;
  for (int i = threadIdx.x; i < n_sums + C; i += blockDim.x) {
    const int word = i < n_sums ? i : 10 * C + (i - n_sums);      // pose [6C] | intrinsics [4C] | ray counts [C]
    uint32_t v[HRF_DP_MAX_WORLD];
#pragma unroll
    for (int r = 0; r < HRF_DP_MAX_WORLD; ++r)
      if (r < W) v[r] = reinterpret_cast<const uint32_t*>(rec.record[r])[word];
    if (i < n_sums) {
      double s = (double)__uint_as_float(v[0]);
#pragma unroll
      for (int r = 1; r < HRF_DP_MAX_WORLD; ++r)
        if (r < W) s += (double)__uint_as_float(v[r]);
      const int c = i < 6 * C ? i / 6 : (i - 6 * C) / 4, k = i < 6 * C ? i % 6 : 6 + (i - 6 * C) % 4;
      sgrad[10 * c + k] = s / (double)W;
    } else {
      uint32_t seen = 0;
#pragma unroll
      for (int r = 0; r < HRF_DP_MAX_WORLD; ++r)
        if (r < W) seen |= v[r];
      touched[i - n_sums] = seen != 0;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    if (touched[c] == 0 || p.fixed[c] != 0) continue;
    camera_step_body<kCalib>(p, q, c, [&](int k) { return sgrad[10 * c + k]; }, lr, lr_intrinsics, beta1, beta2, eps);
  }
  __syncthreads();                // the per-camera tables written above are visible to the whole block
  slot_copy_body(p);
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

extern "C" int64_t hrf_camera_calib_grad_workspace_bytes(int num_cameras) {
  if (num_cameras < 1 || num_cameras > kPoseMaxCameras) return -1;
  return (int64_t)kPoseMaxBlocks * num_cameras * (int64_t)sizeof(CalibSlot);
}

extern "C" int hrf_camera_calib_grad(const float* d_origins, const float* d_ray_directions, const float* ray_directions,
                                     const int32_t* camera_numbers, int64_t num_rays, const double* omega,
                                     const double* alpha, const float* rotations, int num_cameras, float* pose_grad,
                                     float* intrinsics_grad, int32_t* ray_count, int32_t* error, void* workspace,
                                     void* stream) {
  HRF_REQUIRE(num_rays >= 0 && num_rays < ((int64_t)1 << 31), "ray count outside [0, 2^31)");
  HRF_REQUIRE(num_cameras >= 1 && num_cameras <= kPoseMaxCameras, "camera count outside [1, 1024]");
  HRF_REQUIRE(omega != nullptr && alpha != nullptr && pose_grad != nullptr && intrinsics_grad != nullptr &&
                  ray_count != nullptr && error != nullptr,
              "null argument");
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int blocks = pose_blocks(num_rays);
  if (blocks > 0) {
    HRF_REQUIRE(d_origins != nullptr && d_ray_directions != nullptr && ray_directions != nullptr &&
                    camera_numbers != nullptr && rotations != nullptr && workspace != nullptr,
                "null input");
    const size_t smem = (size_t)kPoseWarps * num_cameras * sizeof(CalibSlot);
    if (smem > 48 * 1024)     // more than 256 cameras
      HRF_CUDA(cudaFuncSetAttribute(calib_partials_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t per_block = (num_rays + blocks - 1) / blocks;
    calib_partials_kernel<<<blocks, kPoseThreads, smem, st>>>(d_origins, d_ray_directions, ray_directions,
                                                              camera_numbers, rotations, num_rays, num_cameras,
                                                              per_block, reinterpret_cast<CalibSlot*>(workspace), error);
    HRF_CHECK_LAUNCH();
  }
  calib_finish_kernel<<<(num_cameras + 127) / 128, 128, 0, st>>>(reinterpret_cast<const CalibSlot*>(workspace), blocks,
                                                                 num_cameras, omega, alpha, pose_grad, intrinsics_grad,
                                                                 ray_count);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_camera_calib_step(const hrf_camera_poses* poses, const hrf_camera_intrinsics* intrinsics,
                                     const float* pose_grad, const float* intrinsics_grad, const int32_t* ray_count,
                                     const int32_t* error, double lr, double lr_intrinsics, double beta1, double beta2,
                                     double eps, void* stream) {
  HRF_REQUIRE(poses != nullptr && intrinsics != nullptr && pose_grad != nullptr && intrinsics_grad != nullptr &&
                  ray_count != nullptr,
              "null argument");
  const hrf_camera_poses& p = *poses;
  const hrf_camera_intrinsics& q = *intrinsics;
  HRF_REQUIRE(p.num_cameras >= 1 && p.num_cameras <= kPoseMaxCameras, "camera count outside [1, 1024]");
  HRF_REQUIRE(p.num_slots >= 0, "negative slot count");
  HRF_REQUIRE(p.omega && p.tau && p.exp_avg && p.exp_avg_sq && p.step && p.fixed && p.base_inverse_krs &&
                  p.base_camera_origins && p.inverse_krs && p.camera_origins,
              "null camera table");
  HRF_REQUIRE(q.alpha && q.beta && q.exp_avg && q.exp_avg_sq && q.base_intrinsics && q.base_rotations && q.rotations,
              "null intrinsics table");
  HRF_REQUIRE(p.num_slots == 0 || (p.slot_inverse_krs && p.slot_camera_origins && p.slot_camera_numbers),
              "null slot table");
  calib_step_kernel<<<1, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p, q, pose_grad, intrinsics_grad, ray_count,
                                                                           error, lr, lr_intrinsics, beta1, beta2, eps);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int64_t hrf_camera_grad_record_bytes(int num_cameras) {
  if (num_cameras < 1 || num_cameras > kPoseMaxCameras) return -1;
  return (int64_t)(11 * num_cameras + 1) * 4;
}

static int step_ranks(bool calib, const hrf_camera_poses* poses, const hrf_camera_intrinsics* intrinsics,
                      const hrf_camera_grad_records* records, int32_t* error, double lr, double lr_intrinsics,
                      double beta1, double beta2, double eps, void* stream) {
  HRF_REQUIRE(poses != nullptr && records != nullptr && error != nullptr, "null argument");
  const hrf_camera_poses& p = *poses;
  const hrf_camera_grad_records& rec = *records;
  HRF_REQUIRE(p.num_cameras >= 1 && p.num_cameras <= kPoseMaxCameras, "camera count outside [1, 1024]");
  HRF_REQUIRE(p.num_slots >= 0, "negative slot count");
  HRF_REQUIRE(rec.world >= 1 && rec.world <= HRF_DP_MAX_WORLD, "world size outside [1, 8]");
  HRF_REQUIRE(rec.rank >= 0 && rec.rank < rec.world, "rank outside [0, world)");
  for (int r = 0; r < rec.world; ++r) HRF_REQUIRE(rec.record[r] != nullptr, "null gradient record");
  HRF_REQUIRE(p.omega && p.tau && p.exp_avg && p.exp_avg_sq && p.step && p.fixed && p.base_inverse_krs &&
                  p.base_camera_origins && p.inverse_krs && p.camera_origins,
              "null camera table");
  HRF_REQUIRE(p.num_slots == 0 || (p.slot_inverse_krs && p.slot_camera_origins && p.slot_camera_numbers),
              "null slot table");
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t smem = (size_t)p.num_cameras * (10 * sizeof(double) + sizeof(int));
  if (calib) {
    HRF_REQUIRE(intrinsics != nullptr, "null argument");
    const hrf_camera_intrinsics& q = *intrinsics;
    HRF_REQUIRE(q.alpha && q.beta && q.exp_avg && q.exp_avg_sq && q.base_intrinsics && q.base_rotations && q.rotations,
                "null intrinsics table");
    if (smem > 48 * 1024)     // more than 585 cameras
      HRF_CUDA(cudaFuncSetAttribute(step_ranks_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    step_ranks_kernel<true><<<1, kRankStepThreads, smem, st>>>(p, q, rec, error, lr, lr_intrinsics, beta1, beta2, eps);
  } else {
    if (smem > 48 * 1024)
      HRF_CUDA(cudaFuncSetAttribute(step_ranks_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    step_ranks_kernel<false><<<1, kRankStepThreads, smem, st>>>(p, hrf_camera_intrinsics{}, rec, error, lr, 0.0, beta1,
                                                                beta2, eps);
  }
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_camera_pose_step_ranks(const hrf_camera_poses* poses, const hrf_camera_grad_records* records,
                                          int32_t* error, double lr, double beta1, double beta2, double eps,
                                          void* stream) {
  return step_ranks(false, poses, nullptr, records, error, lr, 0.0, beta1, beta2, eps, stream);
}

extern "C" int hrf_camera_calib_step_ranks(const hrf_camera_poses* poses, const hrf_camera_intrinsics* intrinsics,
                                           const hrf_camera_grad_records* records, int32_t* error, double lr,
                                           double lr_intrinsics, double beta1, double beta2, double eps, void* stream) {
  return step_ranks(true, poses, intrinsics, records, error, lr, lr_intrinsics, beta1, beta2, eps, stream);
}
