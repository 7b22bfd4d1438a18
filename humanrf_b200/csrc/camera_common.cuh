// Device functions shared by the per-camera calibration kernels (camera_pose.cu, camera_response.cu): the lane tree of
// the deterministic per-camera reduction and the float64 Adam update with its roundings spelled out.
#pragma once

#include "common.cuh"

namespace hrf {

// Sum of x over the lanes of `peers` (this lane included), left in the lowest lane of `peers`.  A tree over the peers'
// ranks: round k adds the partial 2^k ranks up.  Every lane of the warp runs every round.
template <int N, typename T>
__device__ __forceinline__ void reduce_peers(unsigned peers, T (&x)[N]) {
  const int lane = threadIdx.x & 31;
  int rank = __popc(peers & ((1u << lane) - 1u));
  unsigned above = peers & ~((2u << lane) - 1u);
  while (__any_sync(0xffffffffu, above != 0)) {
    const int next = __ffs(above);                     // 1-based; 0 = none
    const int src = next ? next - 1 : lane;
#pragma unroll
    for (int k = 0; k < N; ++k) {
      const T t = __shfl_sync(0xffffffffu, x[k], src);
      if (next) x[k] += t;
    }
    above &= __ballot_sync(0xffffffffu, (rank & 1) == 0);
    rank >>= 1;
  }
}

// The response of one channel: color + em (color - (1 - w) bg) + w b, with a zero em or b not added (so that em = b = 0
// returns color bit for bit).  The loss kernel, hrf_camera_response_apply and
// the error map's per-ray error (error_map.cu) share it.
__device__ __forceinline__ float respond(float color, float w, float bg, float em, float b, float& fg) {
  fg = __fmaf_rn(-(1.f - w), bg, color);
  float pred = color;
  if (em != 0.f) pred = __fmaf_rn(em, fg, pred);
  if (b != 0.f) pred = __fmaf_rn(w, b, pred);
  return pred;
}

// One torch.optim.Adam update of x: m = b1 m + (1 - b1) g, v = b2 v + (1 - b2) g g, x -= lr / bc1 * m / (sqrt(v) / bc2s + eps)
// in float64, every rounding spelled out.  Left to the compiler, which products are fused into an FMA depends on the
// kernel around the update, and every step kernel must give the same bits from the same gradient.
__device__ __forceinline__ void adam_update(double g, double& m_io, double& v_io, double& x, double lr_bc1, double bc2s,
                                            double beta1, double beta2, double eps) {
  const double m = __fma_rn(m_io, beta1, __dmul_rn(1.0 - beta1, g));
  const double v = __fma_rn(v_io, beta2, __dmul_rn(__dmul_rn(1.0 - beta2, g), g));
  m_io = m, v_io = v;
  x = __fma_rn(-lr_bc1, m / (sqrt(v) / bc2s + eps), x);
}

}  // namespace hrf
