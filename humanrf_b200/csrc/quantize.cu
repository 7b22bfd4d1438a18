// 8-bit hash tables for inference (HRF_TABLE_INT8X2, DESIGN.md §3.19): per (grid, level, feature) slice a symmetric scale
// chosen from a fixed list of clip ratios by the least squared reconstruction error, the int8 codes, and the scales
// folded into the vectors.  Every rounding is pinned (_rn intrinsics, no contraction) so that tests/quant_oracle.py
// reproduces scales, codes and folded vectors bit for bit.
#include "common.cuh"

namespace hrf {

constexpr int kQuantThreads = 512;
__constant__ float kClip[HRF_QUANT_CLIPS] = {1.0f, 0.9f, 0.8f, 0.7f, 0.6f, 0.5f, 0.4f, 0.3f};

struct QuantGrids {
  const float* master[4];
  uint32_t level_offset[HRF_N_LEVELS];
  uint32_t level_size[HRF_N_LEVELS];
};

__device__ __forceinline__ float quant_scale(float c, float absmax) { return __fdiv_rn(__fmul_rn(c, absmax), 127.f); }
__device__ __forceinline__ int quant_code(float x, float s) {
  if (s == 0.f) return 0;
  return (int)fminf(fmaxf(rintf(__fdiv_rn(x, s)), -127.f), 127.f);
}

// Deterministic block reductions: a fixed xor tree inside each warp, then the warps in index order.
template <class T, class Op>
__device__ __forceinline__ T block_reduce(T v, T* sm, Op op) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, d));
  const int w = threadIdx.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sm[w] = v;
  __syncthreads();
  T r = sm[0];
  for (int i = 1; i < kQuantThreads / 32; ++i) r = op(r, sm[i]);
  return r;
}

// Pass one: one CTA per (grid, level) = two slices.  The first loop reads the level's fp32 masters from HBM for the
// absmax; the second walks the same bytes again (at most 4 MB per level, resident in the L2) for the error of every
// candidate.  Per-thread float64 partials in a fixed element order, then block_reduce: the result does not depend on
// scheduling.
__global__ void __launch_bounds__(kQuantThreads) quant_select_kernel(const __grid_constant__ QuantGrids g, float* scale,
                                                                    int32_t* clip, double* sq_err, int32_t* status) {
  __shared__ double smd[kQuantThreads / 32];
  __shared__ float smf[kQuantThreads / 32];
  __shared__ int smi[kQuantThreads / 32];
  const int grid = blockIdx.x / HRF_N_LEVELS, level = blockIdx.x % HRF_N_LEVELS;
  const float2* x = reinterpret_cast<const float2*>(g.master[grid]) + g.level_offset[level];
  const uint32_t n = g.level_size[level];
  float m0 = 0.f, m1 = 0.f;
  int bad = 0;
  for (uint32_t e = threadIdx.x; e < n; e += kQuantThreads) {
    const float2 v = __ldg(x + e);
    bad |= !isfinite(v.x) || !isfinite(v.y);
    m0 = fmaxf(m0, fabsf(v.x));
    m1 = fmaxf(m1, fabsf(v.y));
  }
  auto fmax_op = [](float a, float b) { return fmaxf(a, b); };
  auto or_op = [](int a, int b) { return a | b; };
  m0 = block_reduce(m0, smf, fmax_op);
  m1 = block_reduce(m1, smf, fmax_op);
  bad = block_reduce(bad, smi, or_op);
  const int slice = grid * HRF_N_LEVELS + level;
  if (bad) {
    if (threadIdx.x == 0) status[slice] = 1;
    return;
  }
  float s0[HRF_QUANT_CLIPS], s1[HRF_QUANT_CLIPS];
  double e0[HRF_QUANT_CLIPS], e1[HRF_QUANT_CLIPS];
#pragma unroll
  for (int c = 0; c < HRF_QUANT_CLIPS; ++c) {
    s0[c] = quant_scale(kClip[c], m0), s1[c] = quant_scale(kClip[c], m1);
    e0[c] = e1[c] = 0.0;
  }
  for (uint32_t e = threadIdx.x; e < n; e += kQuantThreads) {
    const float2 v = __ldg(x + e);
#pragma unroll
    for (int c = 0; c < HRF_QUANT_CLIPS; ++c) {
      const double d0 = __dsub_rn((double)v.x, __dmul_rn((double)s0[c], (double)quant_code(v.x, s0[c])));
      const double d1 = __dsub_rn((double)v.y, __dmul_rn((double)s1[c], (double)quant_code(v.y, s1[c])));
      e0[c] = __dadd_rn(e0[c], __dmul_rn(d0, d0));
      e1[c] = __dadd_rn(e1[c], __dmul_rn(d1, d1));
    }
  }
  auto add_op = [](double a, double b) { return __dadd_rn(a, b); };
#pragma unroll
  for (int c = 0; c < HRF_QUANT_CLIPS; ++c) {
    e0[c] = block_reduce(e0[c], smd, add_op);
    e1[c] = block_reduce(e1[c], smd, add_op);
  }
  if (threadIdx.x == 0) {
    int b0 = 0, b1 = 0;
    for (int c = 1; c < HRF_QUANT_CLIPS; ++c) {   // strictly less: a tie keeps the larger ratio (earlier in the list)
      if (e0[c] < e0[b0]) b0 = c;
      if (e1[c] < e1[b1]) b1 = c;
    }
    scale[2 * slice] = s0[b0], scale[2 * slice + 1] = s1[b1];
    clip[2 * slice] = b0, clip[2 * slice + 1] = b1;
    for (int c = 0; c < HRF_QUANT_CLIPS; ++c)
      sq_err[(2 * slice) * HRF_QUANT_CLIPS + c] = e0[c], sq_err[(2 * slice + 1) * HRF_QUANT_CLIPS + c] = e1[c];
    status[slice] = 0;
  }
}

struct QuantCodes {
  uint16_t* codes[4];
};

// Pass two: blockIdx.y = grid * 16 + level, the x blocks stride over the level's entries.
__global__ void __launch_bounds__(256) quant_write_kernel(const __grid_constant__ QuantGrids g,
                                                          const __grid_constant__ QuantCodes out,
                                                          const float* __restrict__ scale) {
  const int grid = blockIdx.y / HRF_N_LEVELS, level = blockIdx.y % HRF_N_LEVELS;
  const uint32_t off = g.level_offset[level], n = g.level_size[level];
  const float2* x = reinterpret_cast<const float2*>(g.master[grid]) + off;
  uint16_t* q = out.codes[grid] + off;
  const float s0 = __ldg(scale + 2 * blockIdx.y), s1 = __ldg(scale + 2 * blockIdx.y + 1);
  for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
    const float2 v = __ldg(x + e);
    q[e] = (uint16_t)(((uint32_t)quant_code(v.x, s0) & 0xffu) | (((uint32_t)quant_code(v.y, s1) & 0xffu) << 8));
  }
}

// vectors [4][VR][32]: axis a = x, y, z, t is composed with grid yzt, xzt, xyt, xyz (tensor_composition.cu:49-52:
// xyz*v_t + xyt*v_z + yzt*v_x + xzt*v_y).
__global__ void __launch_bounds__(256) quant_fold_kernel(const float* __restrict__ v, const float* __restrict__ scale,
                                                         int64_t n, int vec_res, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int j = (int)(i & 31);
  const int a = (int)((i >> 5) / vec_res);
  const int grid = a == 0 ? 2 : a == 1 ? 3 : a == 2 ? 1 : 0;
  out[i] = __fmul_rn(__ldg(scale + grid * 2 * HRF_N_LEVELS + j), __ldg(v + i));
}

static int quant_grids(const float* const* masters, const uint32_t* level_offset, const uint32_t* level_size,
                       QuantGrids& g) {
  HRF_REQUIRE(masters != nullptr && level_offset != nullptr && level_size != nullptr, "null argument");
  for (int k = 0; k < 4; ++k) {
    HRF_REQUIRE(masters[k] != nullptr, "null master table");
    g.master[k] = masters[k];
  }
  for (int l = 0; l < HRF_N_LEVELS; ++l) g.level_offset[l] = level_offset[l], g.level_size[l] = level_size[l];
  return 0;
}

}  // namespace hrf

using namespace hrf;

extern "C" int hrf_quantize_tables_select(const float* const* masters, const uint32_t* level_offset,
                                          const uint32_t* level_size, int segment, float* scale, int32_t* clip,
                                          double* sq_err, int32_t* status, void* stream) {
  QuantGrids g;
  if (int rc = quant_grids(masters, level_offset, level_size, g)) return rc;
  HRF_REQUIRE(scale != nullptr && clip != nullptr && sq_err != nullptr && status != nullptr, "null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  quant_select_kernel<<<4 * HRF_N_LEVELS, kQuantThreads, 0, st>>>(g, scale, clip, sq_err, status);
  HRF_CHECK_LAUNCH();
  int32_t host[4 * HRF_N_LEVELS];
  HRF_CUDA(cudaMemcpyAsync(host, status, sizeof(host), cudaMemcpyDeviceToHost, st));
  HRF_CUDA(cudaStreamSynchronize(st));
  static const char* kGrid[4] = {"xyz", "xyt", "yzt", "xzt"};
  for (int i = 0; i < 4 * HRF_N_LEVELS; ++i)
    if (host[i] != 0) {
      set_error("non-finite master parameter in segment " + std::to_string(segment) + ", grid " +
                std::to_string(i / HRF_N_LEVELS) + " (" + kGrid[i / HRF_N_LEVELS] + "), level " +
                std::to_string(i % HRF_N_LEVELS));
      return -1;
    }
  return 0;
}

extern "C" int hrf_quantize_tables_write(const float* const* masters, const uint32_t* level_offset,
                                         const uint32_t* level_size, const float* scale, void* const* codes,
                                         void* stream) {
  QuantGrids g;
  if (int rc = quant_grids(masters, level_offset, level_size, g)) return rc;
  HRF_REQUIRE(scale != nullptr && codes != nullptr, "null argument");
  QuantCodes q;
  uint32_t max_size = 1;
  for (int k = 0; k < 4; ++k) {
    HRF_REQUIRE(codes[k] != nullptr, "null code table");
    q.codes[k] = reinterpret_cast<uint16_t*>(codes[k]);
  }
  for (int l = 0; l < HRF_N_LEVELS; ++l) max_size = level_size[l] > max_size ? level_size[l] : max_size;
  const dim3 blocks((unsigned)((max_size + 255) / 256 < 1024 ? (max_size + 255) / 256 : 1024), 4 * HRF_N_LEVELS);
  quant_write_kernel<<<blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(g, q, scale);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_quantize_fold_vectors(const float* vectors, const float* scale, int vec_res, float* folded,
                                         void* stream) {
  HRF_REQUIRE(vectors != nullptr && scale != nullptr && folded != nullptr && vec_res > 0, "bad argument");
  const int64_t n = (int64_t)4 * vec_res * HRF_N_FEATURES;
  quant_fold_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(vectors, scale, n,
                                                                                                    vec_res, folded);
  HRF_CHECK_LAUNCH();
  return 0;
}
