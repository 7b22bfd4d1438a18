// Per-camera colour response refined with the field in the fused train step (hrf_train_loss_response,
// hrf_camera_response_step, hrf_camera_response_step_ranks, hrf_camera_response_apply; DESIGN.md §3.17), and the
// held-out fit of a camera's response against a frozen model (hrf_response_fit_accumulate, hrf_response_fit_solve; §3.18).
//
// Camera c carries a per-channel log gain gamma_c and offset b_c.  With fg = color - (1 - w) bg the ray's foreground
// (w = weights_sum, bg the trainer's random background, never seen by a camera):
//   pred = color + expm1(gamma) fg + w b          (= e^gamma fg + w b + (1 - w) bg)
//   dpred/dcolor = e^gamma,  dpred/dw = expm1(gamma) bg + b,  dpred/dgamma = e^gamma fg,  dpred/db = w
// The loss kernel reads the response table [C,6] = ((float)expm1(gamma), (float)b) that the step kernels write, and
// takes g = 1 + em in fp32.  A channel whose em and b are both zero adds nothing to pred or d_wsum: at identity pred is
// color bit for bit, g = 1 exactly, and the kernel writes hrf_train_loss's d_color and d_wsum (signed zeros included).
//
// hrf_train_loss_response, two launches, no float atomics in the sums:
//   response_loss_kernel   : block b covers a contiguous range of 256-ray chunks.  Per chunk, warp w takes the 32-ray
//                            tiles w and w + 4; each ray's loss, d_color and d_wsum are computed as train_loss_kernel
//                            computes them, and the chunk's loss is summed by train_loss_kernel's tree (the warp
//                            butterfly, then ((t0 + t4) + (t2 + t6)) + ((t1 + t5) + (t3 + t7)) over the tiles) and added
//                            with one atomicAdd: the loss takes the same addends as hrf_train_loss's.  The per-camera
//                            terms (d_pred fg, d_pred w) go through the pose kernels' lane tree (__match_any_sync,
//                            reduce_peers) into the warp's slot, and the warps' slots are added in warp order into the
//                            block's partial.
//   response_finish_kernel : one thread per camera adds the blocks' partials in block order in float64 and multiplies
//                            the gamma columns by g = 1 + em.
// The block count, min(ceil(R / 2048), 256), depends on R alone, so two runs write identical bytes.
#include <atomic>

#include "camera_common.cuh"

namespace hrf {

constexpr int kRespWarps = 4;
constexpr int kRespThreads = 32 * kRespWarps;
constexpr int kRespChunk = 256;                // rays per loss addend, train_loss_kernel's block size
constexpr int kRespMaxBlocks = 256;
constexpr int kRespRaysPerBlock = 2048;        // a block covers at least this many rays before more blocks are used
constexpr int kRespMaxCameras = 1024;

struct ResponseSlot {                          // 32 bytes: sum d_pred fg (rgb), sum d_pred w (rgb), the ray count, padding
  float v[6];
  int n;
  int pad;
};

__host__ __device__ inline int response_blocks(int64_t num_rays) {
  const int64_t b = (num_rays + kRespRaysPerBlock - 1) / kRespRaysPerBlock;
  return (int)(b < kRespMaxBlocks ? b : kRespMaxBlocks);
}

__global__ void __launch_bounds__(kRespThreads) response_loss_kernel(
    const float* __restrict__ color, const float* __restrict__ wsum, const float* __restrict__ rgba,
    const float* __restrict__ bg, const int32_t* __restrict__ camera_numbers, const float* __restrict__ table,
    int64_t num_rays, int num_cameras, int64_t rays_per_block, float delta, float bce_w,
    const float* __restrict__ scale_dev, float* __restrict__ d_color, float* __restrict__ d_wsum,
    float* __restrict__ loss_out, ResponseSlot* __restrict__ partials, int32_t* __restrict__ error) {
  extern __shared__ ResponseSlot racc[];               // [kRespWarps][num_cameras]
  __shared__ float chunk_loss[2][kRespWarps];          // by chunk parity: one barrier per chunk
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < kRespWarps * num_cameras; i += kRespThreads) {
#pragma unroll
    for (int k = 0; k < 6; ++k) racc[i].v[k] = 0.f;
    racc[i].n = 0;
  }
  __syncthreads();
  const float scale = scale_dev != nullptr ? __ldg(scale_dev) : 1.f;
  const float inv3r = 1.f / (3.f * (float)num_rays), invr = 1.f / (float)num_rays;
  const int64_t lo = (int64_t)blockIdx.x * rays_per_block;
  const int64_t hi = min(lo + rays_per_block, num_rays);
  ResponseSlot* mine = racc + warp * num_cameras;
  unsigned bad = 0;
  int parity = 0;
  for (int64_t chunk = lo; chunk < hi; chunk += kRespChunk, parity ^= 1) {
    float tile_loss[2];
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int64_t r = chunk + 32 * (warp + kRespWarps * half) + lane;
      int cam = -1;
      float x[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      float loss = 0.f;
      if (r < hi) {
        const int c = __ldg(camera_numbers + r);
        float em[3] = {0.f, 0.f, 0.f}, off[3] = {0.f, 0.f, 0.f};
        if (c >= 0 && c < num_cameras) {
          cam = c;
#pragma unroll
          for (int k = 0; k < 3; ++k) em[k] = __ldg(table + 6 * c + k), off[k] = __ldg(table + 6 * c + 3 + k);
        } else {
          bad = 1;                                     // the ray takes the identity and stays out of the sums
        }
        const float m = rgba[4 * r + 3];
        const float w = wsum[r];
        float dresp = 0.f;
        bool any = false;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          float fg;
          const float col = color[3 * r + k], b = bg[3 * r + k];
          const float pred = respond(col, w, b, em[k], off[k], fg);
          // train_loss_kernel's expressions on pred
          const float gt = rgba[4 * r + k] * m + b * (1.f - m);
          const float xk = pred - gt, ax = fabsf(xk);
          const bool quad = ax < delta;
          loss += (quad ? 0.5f * xk * xk : delta * (ax - 0.5f * delta)) * inv3r;
          const float dpred = (quad ? xk : copysignf(delta, xk)) * inv3r * scale;
          d_color[3 * r + k] = dpred * (1.f + em[k]);
          if (em[k] != 0.f || off[k] != 0.f) {
            dresp = any ? __fmaf_rn(dpred, __fmaf_rn(em[k], b, off[k]), dresp) : __fmul_rn(dpred, __fmaf_rn(em[k], b, off[k]));
            any = true;
          }
          x[k] = __fmul_rn(dpred, fg);
          x[3 + k] = __fmul_rn(dpred, w);
        }
        const float pc = fminf(fmaxf(w, 0.f), 1.f);
        loss += -(m * logf(pc + 1e-10f) + (1.f - m) * logf(1.f - pc + 1e-10f)) * invr * bce_w;
        const float dpc = -(m / (pc + 1e-10f) - (1.f - m) / (1.f - pc + 1e-10f));
        const float dw = (w >= 0.f && w <= 1.f) ? dpc * invr * bce_w * scale : 0.f;
        d_wsum[r] = any ? __fadd_rn(dw, dresp) : dw;
        if (cam < 0) {
#pragma unroll
          for (int k = 0; k < 6; ++k) x[k] = 0.f;
        }
      }
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, d);
      tile_loss[half] = loss;
      const unsigned peers = __match_any_sync(0xffffffffu, cam);
      reduce_peers<6>(peers, x);
      if (cam >= 0 && lane == __ffs(peers) - 1) {
#pragma unroll
        for (int k = 0; k < 6; ++k) mine[cam].v[k] += x[k];
        mine[cam].n += __popc(peers);
      }
      __syncwarp();
    }
    if (lane == 0) chunk_loss[parity][warp] = tile_loss[0] + tile_loss[1];
    __syncthreads();
    if (threadIdx.x == 0 && loss_out != nullptr) {
      const float* t = chunk_loss[parity];
      atomicAdd(loss_out, (t[0] + t[2]) + (t[1] + t[3]));
    }
  }
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(error, 1);
  __syncthreads();
  for (int c = threadIdx.x; c < num_cameras; c += kRespThreads) {
    ResponseSlot s = racc[c];
    for (int w = 1; w < kRespWarps; ++w) {
      const ResponseSlot& t = racc[w * num_cameras + c];
#pragma unroll
      for (int k = 0; k < 6; ++k) s.v[k] += t.v[k];
      s.n += t.n;
    }
    partials[(int64_t)blockIdx.x * num_cameras + c] = s;
  }
}

// One thread per camera: the blocks' partials in block order (float64), the gamma columns times g = 1 + em.
__global__ void __launch_bounds__(128) response_finish_kernel(const ResponseSlot* __restrict__ partials, int num_blocks,
                                                              int num_cameras, const float* __restrict__ table,
                                                              float* __restrict__ response_grad,
                                                              int32_t* __restrict__ ray_count) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= num_cameras) return;
  double s[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  int n = 0;
  for (int b = 0; b < num_blocks; ++b) {
    const ResponseSlot& p = partials[(int64_t)b * num_cameras + c];
#pragma unroll
    for (int k = 0; k < 6; ++k) s[k] += (double)p.v[k];
    n += p.n;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) response_grad[6 * c + k] = (float)(s[k] * (1.0 + (double)table[6 * c + k]));
#pragma unroll
  for (int k = 3; k < 6; ++k) response_grad[6 * c + k] = (float)s[k];
  ray_count[c] = n;
}

// Camera c's table row (expm1(gamma), b) from its float64 parameters, rounded once: what the loss kernel reads.
__device__ __forceinline__ void response_table_row(const hrf_camera_responses& p, int c) {
#pragma unroll
  for (int k = 0; k < 3; ++k) p.table[6 * c + k] = (float)expm1(p.params[6 * c + k]);
#pragma unroll
  for (int k = 3; k < 6; ++k) p.table[6 * c + k] = (float)p.params[6 * c + k];
}

// Adam on camera c's (gamma, b) in float64 (adam_update), then its table row.
template <class Grad>
__device__ __forceinline__ void response_step_body(const hrf_camera_responses& p, int c, Grad grad, double lr,
                                                   double beta1, double beta2, double eps) {
  const int step = p.step[c] + 1;
  p.step[c] = step;
  const double bc1 = 1.0 - pow(beta1, (double)step), bc2s = sqrt(1.0 - pow(beta2, (double)step));
#pragma unroll
  for (int k = 0; k < 6; ++k)
    adam_update(grad(k), p.exp_avg[6 * c + k], p.exp_avg_sq[6 * c + k], p.params[6 * c + k], lr / bc1, bc2s, beta1,
                beta2, eps);
  response_table_row(p, c);
}

__global__ void __launch_bounds__(128) response_table_kernel(hrf_camera_responses p) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < p.num_cameras) response_table_row(p, c);
}

__global__ void __launch_bounds__(256) response_step_kernel(hrf_camera_responses p, const float* __restrict__ grad,
                                                            const int32_t* __restrict__ ray_count,
                                                            const int32_t* __restrict__ error, double lr, double beta1,
                                                            double beta2, double eps) {
  if (error != nullptr && *error != 0) return;
  for (int c = threadIdx.x; c < p.num_cameras; c += blockDim.x) {
    if (ray_count[c] == 0 || p.fixed[c] != 0) continue;
    response_step_body(p, c, [&](int k) { return (double)grad[6 * c + k]; }, lr, beta1, beta2, eps);
  }
}

// The data-parallel step: the pose kernels' step_ranks_kernel scheme on the response record [grad 6C | count C | error].
//   1. Any rank's error word set: nothing is written; a rank that sees bit 0 in ANOTHER rank's word sets bit 1 of its own.
//   2. The records are staged into shared memory, one word per thread and step: the gradient entry as (sum over
//      r = 0..W-1 in rank order of (double)grad_r) / W, the touched flag as the OR of the ray counts.  At W = 1 the
//      entry is (double)grad_0 exactly: response_step_kernel's input.
//   3. Every touched camera that is not fixed takes response_step_body.
constexpr int kRespRankThreads = 384;

__global__ void __launch_bounds__(kRespRankThreads) response_step_ranks_kernel(hrf_camera_responses p,
                                                                               hrf_camera_grad_records rec,
                                                                               int32_t* error, double lr, double beta1,
                                                                               double beta2, double eps) {
  extern __shared__ double rgrad[];                    // [C][6] reduced gradients, then int32 touched [C]
  const int C = p.num_cameras, W = rec.world;
  int any = 0, peer_bad = 0;
#pragma unroll
  for (int r = 0; r < HRF_DP_MAX_WORLD; ++r) {
    if (r < W) {
      const int e = reinterpret_cast<const int32_t*>(rec.record[r])[7 * C];
      any |= e;
      if (r != rec.rank) peer_bad |= e & 1;
    }
  }
  if (any != 0) {
    if (threadIdx.x == 0 && peer_bad != 0) atomicOr(error, 2);
    return;
  }
  int* touched = reinterpret_cast<int*>(rgrad + 6 * C);
  for (int i = threadIdx.x; i < 7 * C; i += blockDim.x) {
    uint32_t v[HRF_DP_MAX_WORLD];
#pragma unroll
    for (int r = 0; r < HRF_DP_MAX_WORLD; ++r)
      if (r < W) v[r] = reinterpret_cast<const uint32_t*>(rec.record[r])[i];
    if (i < 6 * C) {
      double s = (double)__uint_as_float(v[0]);
#pragma unroll
      for (int r = 1; r < HRF_DP_MAX_WORLD; ++r)
        if (r < W) s += (double)__uint_as_float(v[r]);
      rgrad[i] = s / (double)W;
    } else {
      uint32_t seen = 0;
#pragma unroll
      for (int r = 0; r < HRF_DP_MAX_WORLD; ++r)
        if (r < W) seen |= v[r];
      touched[i - 6 * C] = seen != 0;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    if (touched[c] == 0 || p.fixed[c] != 0) continue;
    response_step_body(p, c, [&](int k) { return rgrad[6 * c + k]; }, lr, beta1, beta2, eps);
  }
}

__global__ void __launch_bounds__(256) response_apply_kernel(float* __restrict__ color, const float* __restrict__ alpha,
                                                             int64_t num_pixels, const float* __restrict__ row,
                                                             const float* __restrict__ background) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= num_pixels) return;
  const float w = alpha[i];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float fg;
    color[3 * i + k] = respond(color[3 * i + k], w, __ldg(background + k), __ldg(row + k), __ldg(row + 3 + k), fg);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Held-out response fit (hrf_response_fit_accumulate, hrf_response_fit_solve; DESIGN.md §3.18).  Per camera and channel
// the gain g and offset b minimising sum (g f + a b - y/255)^2 + lambda n ((g - 1)^2 + b^2) over the fit pixels, from
// the moments row [n, S_aa, per channel: S_ff, S_fa, S_fy, S_ay, S_yy] (y the 8-bit colour as an integer).  Every
// addend is exact in float64 (fp32 x fp32, fp32 x u8, u8 x u8), so the sums' only rounding is the summation itself.
constexpr int kFitRow = 17;
constexpr int kFitThreads = 256;
constexpr int kFitPixelsPerBlock = 2048;
constexpr int kFitMaxBlocks = 1024;

__host__ __device__ inline int fit_blocks(int64_t num_pixels) {
  const int64_t b = (num_pixels + kFitPixelsPerBlock - 1) / kFitPixelsPerBlock;
  return (int)(b < kFitMaxBlocks ? b : kFitMaxBlocks);
}

// Grid-stride over the pixels (the grid depends on P alone), a thread's sums in pixel order, the warp butterfly, then
// the warps in order: one partial row per block.
__global__ void __launch_bounds__(kFitThreads) response_fit_partials_kernel(
    const float* __restrict__ color, const float* __restrict__ alpha, const uint8_t* __restrict__ gt,
    const uint8_t* __restrict__ mask, int64_t num_pixels, double* __restrict__ partials) {
  __shared__ double warp_rows[kFitThreads / 32][kFitRow];
  double s[kFitRow];
#pragma unroll
  for (int e = 0; e < kFitRow; ++e) s[e] = 0.0;
  const int64_t stride = (int64_t)gridDim.x * kFitThreads;
  for (int64_t i = (int64_t)blockIdx.x * kFitThreads + threadIdx.x; i < num_pixels; i += stride) {
    if (__ldg(mask + i) == 0) continue;
    const double a = (double)__ldg(alpha + i);
    s[0] += 1.0;
    s[1] += a * a;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double f = (double)__ldg(color + 3 * i + k), y = (double)__ldg(gt + 3 * i + k);
      s[2 + 5 * k] += f * f;
      s[3 + 5 * k] += f * a;
      s[4 + 5 * k] += f * y;
      s[5 + 5 * k] += a * y;
      s[6 + 5 * k] += y * y;
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int e = 0; e < kFitRow; ++e) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s[e] += __shfl_xor_sync(0xffffffffu, s[e], d);
  }
  if (lane == 0) {
#pragma unroll
    for (int e = 0; e < kFitRow; ++e) warp_rows[warp][e] = s[e];
  }
  __syncthreads();
  if (threadIdx.x < kFitRow) {
    double t = warp_rows[0][threadIdx.x];
#pragma unroll
    for (int w = 1; w < kFitThreads / 32; ++w) t += warp_rows[w][threadIdx.x];
    partials[(int64_t)blockIdx.x * kFitRow + threadIdx.x] = t;
  }
}

// One warp: entry e of the blocks' partials in block order, then added into the camera's row.  A camera outside
// [0, C) sets the error word and writes nothing.
__global__ void __launch_bounds__(32) response_fit_finish_kernel(const double* __restrict__ partials, int num_blocks,
                                                                 int camera, int num_cameras,
                                                                 double* __restrict__ moments,
                                                                 int32_t* __restrict__ error) {
  if (camera < 0 || camera >= num_cameras) {
    if (threadIdx.x == 0) atomicOr(error, 1);
    return;
  }
  const int e = threadIdx.x;
  if (e >= kFitRow || num_blocks == 0) return;
  double t = partials[e];
#pragma unroll 8
  for (int b = 1; b < num_blocks; ++b) t += partials[(int64_t)b * kFitRow + e];
  moments[(int64_t)camera * kFitRow + e] += t;
}

// The 2x2 ridge system of one channel by Cramer's rule, every operation rounded as written (no contraction), so that
// a float64 restatement in the same order gives the same bits.  Returns (g, b); the data SSE at the identity and at
// (g, b) come from the moments.
struct FitChannel {
  double g, b, sse_identity, sse_fit;
};

__device__ __forceinline__ FitChannel fit_channel(double n, double saa, const double* m, double lambda) {
  const double inv255 = 1.0 / 255.0;
  const double sff = m[0], sfa = m[1], sfy = __dmul_rn(m[2], inv255), say = __dmul_rn(m[3], inv255);
  const double syy = __dmul_rn(__dmul_rn(m[4], inv255), inv255);
  const double ln = __dmul_rn(lambda, n);
  const double a11 = __dadd_rn(sff, ln), a22 = __dadd_rn(saa, ln), r1 = __dadd_rn(sfy, ln);
  const double det = __dsub_rn(__dmul_rn(a11, a22), __dmul_rn(sfa, sfa));
  FitChannel o;
  o.g = __ddiv_rn(__dsub_rn(__dmul_rn(r1, a22), __dmul_rn(sfa, say)), det);
  o.b = __ddiv_rn(__dsub_rn(__dmul_rn(a11, say), __dmul_rn(sfa, r1)), det);
  // sum (f - y)^2 and sum (g f + a b - y)^2, expanded
  o.sse_identity = __dadd_rn(__dsub_rn(sff, __dmul_rn(2.0, sfy)), syy);
  double q = __dmul_rn(__dmul_rn(o.g, o.g), sff);
  q = __dadd_rn(q, __dmul_rn(__dmul_rn(o.b, o.b), saa));
  q = __dadd_rn(q, __dmul_rn(__dmul_rn(2.0, __dmul_rn(o.g, o.b)), sfa));
  q = __dsub_rn(q, __dmul_rn(__dmul_rn(2.0, o.g), sfy));
  q = __dsub_rn(q, __dmul_rn(__dmul_rn(2.0, o.b), say));
  o.sse_fit = __dadd_rn(q, syy);
  return o;
}

constexpr int kFitSolveThreads = 256;

// One CTA.  Pass 1: every listed camera's three systems, its report and status.  Pass 2, only when every listed camera
// succeeded: gamma = log g and b into params, then the camera's table row (the step kernels' expression).
__global__ void __launch_bounds__(kFitSolveThreads) response_fit_solve_kernel(
    hrf_camera_responses p, const double* __restrict__ moments, const int32_t* __restrict__ cameras, int K,
    double lambda, double min_pixels, double* __restrict__ report, int32_t* __restrict__ status) {
  int failed = 0;
  for (int k = threadIdx.x; k < K; k += kFitSolveThreads) {
    const int c = cameras[k];
    double* rep = report + 8 * (int64_t)k;
    int st = HRF_FIT_OK;
    if (c < 0 || c >= p.num_cameras) {
      st = HRF_FIT_BAD_CAMERA;
#pragma unroll
      for (int j = 0; j < 7; ++j) rep[j] = 0.0;
    } else {
      const double* row = moments + (int64_t)c * kFitRow;
      const double n = row[0];
      rep[0] = n;
      if (n < min_pixels) st = HRF_FIT_TOO_FEW_PIXELS;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const FitChannel o = fit_channel(n, row[1], row + 2 + 5 * ch, lambda);
        rep[1 + ch] = o.sse_identity;
        rep[4 + ch] = o.sse_fit;
        if (st == HRF_FIT_OK && !(isfinite(o.g) && isfinite(o.b))) st = HRF_FIT_NOT_FINITE;
        if (st == HRF_FIT_OK && !(o.g > 0.0)) st = HRF_FIT_GAIN_NOT_POSITIVE;
      }
    }
    rep[7] = (double)st;
    status[k] = st;
    failed |= st != HRF_FIT_OK;
  }
  if (__syncthreads_or(failed)) return;
  for (int k = threadIdx.x; k < K; k += kFitSolveThreads) {
    const int c = cameras[k];
    const double* row = moments + (int64_t)c * kFitRow;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const FitChannel o = fit_channel(row[0], row[1], row + 2 + 5 * ch, lambda);
      p.params[6 * c + ch] = log(o.g);
      p.params[6 * c + 3 + ch] = o.b;
    }
    response_table_row(p, c);
  }
}

// Raises a kernel's dynamic shared-memory limit to `bytes` once per device (bit d of `done`), not on every call: the
// attribute belongs to the device's context, and the loss kernel runs on every train step.
static int opt_in_smem_once(std::atomic<uint64_t>& done, const void* kernel, int bytes) {
  int dev = 0;
  HRF_CUDA(cudaGetDevice(&dev));
  const uint64_t bit = dev < 64 ? (uint64_t)1 << dev : 0;
  if (bit != 0 && (done.load(std::memory_order_acquire) & bit) != 0) return 0;
  HRF_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done.fetch_or(bit, std::memory_order_release);
  return 0;
}

}  // namespace hrf

using namespace hrf;

extern "C" int64_t hrf_train_loss_response_workspace_bytes(int num_cameras) {
  if (num_cameras < 1 || num_cameras > kRespMaxCameras) return -1;
  return (int64_t)kRespMaxBlocks * num_cameras * (int64_t)sizeof(ResponseSlot);
}

extern "C" int64_t hrf_camera_response_record_bytes(int num_cameras) {
  if (num_cameras < 1 || num_cameras > kRespMaxCameras) return -1;
  return (int64_t)(7 * num_cameras + 1) * 4;
}

extern "C" int hrf_train_loss_response(const float* color, const float* weights_sum, const float* rgba,
                                       const float* background, const int32_t* camera_numbers, int64_t num_rays,
                                       const float* response_table, int num_cameras, float huber_delta,
                                       float bce_weight, const float* loss_scale_dev, float* d_color,
                                       float* d_weights_sum, float* loss_out, float* response_grad, int32_t* ray_count,
                                       int32_t* error, void* workspace, void* stream) {
  HRF_REQUIRE(num_rays >= 0 && num_rays < ((int64_t)1 << 31), "ray count outside [0, 2^31)");
  HRF_REQUIRE(num_cameras >= 1 && num_cameras <= kRespMaxCameras, "camera count outside [1, 1024]");
  HRF_REQUIRE(response_table != nullptr && response_grad != nullptr && ray_count != nullptr && error != nullptr,
              "null argument");
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int blocks = response_blocks(num_rays);
  if (blocks > 0) {
    HRF_REQUIRE(color && weights_sum && rgba && background && camera_numbers && d_color && d_weights_sum && workspace,
                "null input");
    const size_t smem = (size_t)kRespWarps * num_cameras * sizeof(ResponseSlot);
    if (smem > 48 * 1024) {   // more than 384 cameras: the limit is raised once, to what 1024 cameras take
      static std::atomic<uint64_t> done{0};
      const int rc = opt_in_smem_once(done, reinterpret_cast<const void*>(response_loss_kernel),
                                      (int)(kRespWarps * kRespMaxCameras * sizeof(ResponseSlot)));
      if (rc != 0) return rc;
    }
    const int64_t chunks = (num_rays + kRespChunk - 1) / kRespChunk;
    const int64_t per_block = (chunks + blocks - 1) / blocks * kRespChunk;
    response_loss_kernel<<<blocks, kRespThreads, smem, st>>>(
        color, weights_sum, rgba, background, camera_numbers, response_table, num_rays, num_cameras, per_block,
        huber_delta, bce_weight, loss_scale_dev, d_color, d_weights_sum, loss_out,
        reinterpret_cast<ResponseSlot*>(workspace), error);
    HRF_CHECK_LAUNCH();
  }
  response_finish_kernel<<<(num_cameras + 127) / 128, 128, 0, st>>>(reinterpret_cast<const ResponseSlot*>(workspace),
                                                                    blocks, num_cameras, response_table, response_grad,
                                                                    ray_count);
  HRF_CHECK_LAUNCH();
  return 0;
}

static bool responses_valid(const hrf_camera_responses& p) {
  return p.params && p.exp_avg && p.exp_avg_sq && p.step && p.fixed && p.table;
}

extern "C" int hrf_camera_response_step(const hrf_camera_responses* responses, const float* response_grad,
                                        const int32_t* ray_count, const int32_t* error, double lr, double beta1,
                                        double beta2, double eps, void* stream) {
  HRF_REQUIRE(responses != nullptr && response_grad != nullptr && ray_count != nullptr, "null argument");
  const hrf_camera_responses& p = *responses;
  HRF_REQUIRE(p.num_cameras >= 1 && p.num_cameras <= kRespMaxCameras, "camera count outside [1, 1024]");
  HRF_REQUIRE(responses_valid(p), "null response table");
  response_step_kernel<<<1, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p, response_grad, ray_count, error, lr,
                                                                              beta1, beta2, eps);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_camera_response_step_ranks(const hrf_camera_responses* responses,
                                              const hrf_camera_grad_records* records, int32_t* error, double lr,
                                              double beta1, double beta2, double eps, void* stream) {
  HRF_REQUIRE(responses != nullptr && records != nullptr && error != nullptr, "null argument");
  const hrf_camera_responses& p = *responses;
  const hrf_camera_grad_records& rec = *records;
  HRF_REQUIRE(p.num_cameras >= 1 && p.num_cameras <= kRespMaxCameras, "camera count outside [1, 1024]");
  HRF_REQUIRE(responses_valid(p), "null response table");
  HRF_REQUIRE(rec.world >= 1 && rec.world <= HRF_DP_MAX_WORLD, "world size outside [1, 8]");
  HRF_REQUIRE(rec.rank >= 0 && rec.rank < rec.world, "rank outside [0, world)");
  for (int r = 0; r < rec.world; ++r) HRF_REQUIRE(rec.record[r] != nullptr, "null gradient record");
  const size_t smem = (size_t)p.num_cameras * (6 * sizeof(double) + sizeof(int));
  if (smem > 48 * 1024) {     // more than 945 cameras: the limit is raised once, to what 1024 cameras take
    static std::atomic<uint64_t> done{0};
    const int rc = opt_in_smem_once(done, reinterpret_cast<const void*>(response_step_ranks_kernel),
                                    (int)(kRespMaxCameras * (6 * sizeof(double) + sizeof(int))));
    if (rc != 0) return rc;
  }
  response_step_ranks_kernel<<<1, kRespRankThreads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      p, rec, error, lr, beta1, beta2, eps);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_camera_response_write_table(const hrf_camera_responses* responses, void* stream) {
  HRF_REQUIRE(responses != nullptr, "null argument");
  const hrf_camera_responses& p = *responses;
  HRF_REQUIRE(p.num_cameras >= 1 && p.num_cameras <= kRespMaxCameras, "camera count outside [1, 1024]");
  HRF_REQUIRE(p.params != nullptr && p.table != nullptr, "null response table");
  response_table_kernel<<<(p.num_cameras + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int64_t hrf_response_fit_workspace_bytes(int64_t num_pixels) {
  if (num_pixels < 0) return -1;
  const int blocks = fit_blocks(num_pixels);
  return (int64_t)(blocks > 0 ? blocks : 1) * kFitRow * (int64_t)sizeof(double);
}

extern "C" int hrf_response_fit_accumulate(const float* color, const float* alpha, const uint8_t* gt,
                                           const uint8_t* mask, int64_t num_pixels, int camera, int num_cameras,
                                           double* moments, int32_t* error, void* workspace, void* stream) {
  HRF_REQUIRE(num_pixels >= 0, "negative pixel count");
  HRF_REQUIRE(num_cameras >= 1 && num_cameras <= kRespMaxCameras, "camera count outside [1, 1024]");
  HRF_REQUIRE(moments != nullptr && error != nullptr, "null argument");
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const bool valid = camera >= 0 && camera < num_cameras;
  const int blocks = valid ? fit_blocks(num_pixels) : 0;
  if (blocks > 0) {
    HRF_REQUIRE(color && alpha && gt && mask && workspace, "null input");
    response_fit_partials_kernel<<<blocks, kFitThreads, 0, st>>>(color, alpha, gt, mask, num_pixels,
                                                                 reinterpret_cast<double*>(workspace));
    HRF_CHECK_LAUNCH();
  }
  if (blocks > 0 || !valid) {
    response_fit_finish_kernel<<<1, 32, 0, st>>>(reinterpret_cast<const double*>(workspace), blocks, camera,
                                                 num_cameras, moments, error);
    HRF_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int hrf_response_fit_solve(const hrf_camera_responses* responses, const double* moments,
                                      const int32_t* cameras, int num_listed, double lambda, double min_pixels,
                                      double* report, int32_t* status, void* stream) {
  HRF_REQUIRE(responses != nullptr, "null argument");
  const hrf_camera_responses& p = *responses;
  HRF_REQUIRE(p.num_cameras >= 1 && p.num_cameras <= kRespMaxCameras, "camera count outside [1, 1024]");
  HRF_REQUIRE(p.params != nullptr && p.table != nullptr, "null response table");
  HRF_REQUIRE(num_listed >= 0 && num_listed <= kRespMaxCameras, "listed camera count outside [0, 1024]");
  HRF_REQUIRE(lambda >= 0.0, "negative ridge");
  if (num_listed == 0) return 0;
  HRF_REQUIRE(moments && cameras && report && status, "null argument");
  response_fit_solve_kernel<<<1, kFitSolveThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      p, moments, cameras, num_listed, lambda, min_pixels, report, status);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_camera_response_apply(float* color, const float* alpha, int64_t num_pixels,
                                         const float* response_table, int camera, int num_cameras,
                                         const float* background, void* stream) {
  HRF_REQUIRE(num_pixels >= 0, "negative pixel count");
  HRF_REQUIRE(num_cameras >= 1 && num_cameras <= kRespMaxCameras, "camera count outside [1, 1024]");
  HRF_REQUIRE(camera >= 0 && camera < num_cameras, "camera outside [0, num_cameras)");
  HRF_REQUIRE(response_table != nullptr && background != nullptr, "null argument");
  if (num_pixels == 0) return 0;
  HRF_REQUIRE(color != nullptr && alpha != nullptr, "null image");
  response_apply_kernel<<<(unsigned)((num_pixels + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      color, alpha, num_pixels, response_table + 6 * (int64_t)camera, background);
  HRF_CHECK_LAUNCH();
  return 0;
}
