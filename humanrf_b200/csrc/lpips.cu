// LPIPS (lpips.LPIPS(net="alex", version="0.1"), normalize=True) of one image pair over a ROI, the score
// actorshq/evaluation/evaluate.py:66-73 reports.  Contract: include/humanrf_b200.h, hrf_lpips.  Launches, in order, with
// no host synchronisation (every grid is sized from the full image; CTAs read the ROI on the device and exit outside it):
//   input_kernel  : ROI crop of both images -> 2v - 1 -> (x - shift) / scale -> tf32, NHWC with a zero 4th channel;
//   conv_kernel   : AlexNet's five convolutions as implicit GEMMs on TF32 wgmma (M = output pixels of both images,
//                   N = output channels, K = (ky, kx, cin)), bias + ReLU + tf32 rounding in the epilogue;
//   pool_kernel   : the two exact 3x3 / 2 max-pools;
//   tail_kernel   : per layer and pixel, unit-normalise both feature vectors, dot lin with their squared difference, and
//                   fold a CTA's pixels in fp64 into its own slot;
//   finish_kernel : one CTA folds the slots in a fixed order into the five spatial means and their sum.
// Weights are packed once by pack_kernel: [Cout][Kpad] fp32, K-major with k = (ky * KS + kx) * Cin + c (conv1's Cin
// padded to 4), Kpad = K rounded up to 32 with zeros, every value rounded to tf32.  That layout is known only here.
#include <algorithm>

#include "common.cuh"

namespace hrf {
namespace {

constexpr int kMinRoi = 31;                        // pool2 is empty below 31 pixels
constexpr int kTensors = 8;                        // input, conv1, pool1, conv2, pool2, conv3, conv4, conv5
constexpr int kChannels[kTensors] = {4, 64, 64, 192, 192, 384, 256, 256};
constexpr int kBM = 128, kBK = 32, kStages = 4;    // conv CTA tile: 128 pixels (two warpgroups) x BN channels x 32 k
constexpr int kConvThreads = 256;
constexpr int kTailWarps = 8, kTailPixPerWarp = 4, kTailPix = kTailWarps * kTailPixPerWarp;
constexpr int kFinishThreads = 1024;
constexpr int64_t kAlign = 256;

struct ConvShape {
  int cin, cout, ks, stride, pad;
  __host__ __device__ constexpr int k() const { return ks * ks * cin; }
  __host__ __device__ constexpr int kpad() const { return (k() + kBK - 1) / kBK * kBK; }
};
__host__ __device__ constexpr ConvShape conv_shape(int l) {   // conv1's 3 input channels padded to 4
  return l == 0   ? ConvShape{4, 64, 11, 4, 2}
         : l == 1 ? ConvShape{64, 192, 5, 1, 2}
         : l == 2 ? ConvShape{192, 384, 3, 1, 1}
         : l == 3 ? ConvShape{384, 256, 3, 1, 1}
                  : ConvShape{256, 256, 3, 1, 1};
}
__host__ __device__ constexpr int torch_cin(int l) { return l == 0 ? 3 : conv_shape(l).cin; }
// the LPIPS layers are the five ReLU outputs: tensors 1, 3, 5, 6, 7
__host__ __device__ constexpr int layer_tensor(int l) { return l < 2 ? 2 * l + 1 : l + 3; }

__host__ __device__ constexpr int64_t packed_offset(int l) {   // in floats
  int64_t o = 0;
  for (int i = 0; i < l; ++i) o += (int64_t)conv_shape(i).cout * conv_shape(i).kpad();
  return o;
}

// Heights and widths of the eight tensors for a w x h crop (0 where a layer would be empty).
struct Dims {
  int h[kTensors], w[kTensors];
};
__host__ __device__ inline int conv1_out(int x) { return x >= 7 ? (x - 7) / 4 + 1 : 0; }
__host__ __device__ inline int pool_out(int x) { return x >= 3 ? (x - 3) / 2 + 1 : 0; }
__host__ __device__ inline Dims make_dims(int w, int h) {
  Dims d;
  d.w[0] = w, d.h[0] = h;
  d.w[1] = conv1_out(w), d.h[1] = conv1_out(h);
  d.w[2] = d.w[3] = pool_out(d.w[1]), d.h[2] = d.h[3] = pool_out(d.h[1]);
  d.w[4] = pool_out(d.w[3]), d.h[4] = pool_out(d.h[3]);
  for (int t = 5; t < kTensors; ++t) d.w[t] = d.w[4], d.h[t] = d.h[4];
  return d;
}

struct Roi {
  int x, y, w, h;
  bool valid;
};
// A NULL roi is the whole image.  Valid: at least 31 x 31 and inside the image; otherwise no kernel does anything and
// the score is NaN.
__device__ __forceinline__ Roi read_roi(const int32_t* roi, int W, int H) {
  Roi r{0, 0, W, H, false};
  if (roi) r.x = __ldg(roi), r.y = __ldg(roi + 1), r.w = __ldg(roi + 2), r.h = __ldg(roi + 3);
  r.valid = r.w >= kMinRoi && r.h >= kMinRoi && r.x >= 0 && r.y >= 0 && r.x <= W - r.w && r.y <= H - r.h;
  return r;
}

// Workspace layout for a W x H image: tensor t at tensor_offset(t), [2][h_t][w_t][C_t] fp32 for the ROI's dims, then
// the tail's fp64 slots, layer l's at slot_offset(l).
struct Layout {
  int64_t tensor[kTensors + 1];
  int64_t slots[6];   // in doubles, relative to tensor[kTensors]
};
Layout make_layout(int W, int H) {
  const Dims d = make_dims(W, H);
  Layout L;
  L.tensor[0] = 0;
  for (int t = 0; t < kTensors; ++t) {
    const int64_t bytes = 2 * (int64_t)d.h[t] * d.w[t] * kChannels[t] * 4;
    L.tensor[t + 1] = L.tensor[t] + (bytes + kAlign - 1) / kAlign * kAlign;
  }
  L.slots[0] = 0;
  for (int l = 0; l < 5; ++l) {
    const int t = layer_tensor(l);
    L.slots[l + 1] = L.slots[l] + ((int64_t)d.h[t] * d.w[t] + kTailPix - 1) / kTailPix;
  }
  return L;
}

// ---- packing ---------------------------------------------------------------------------------------------------------
struct ConvWeights {
  const float* w[5];   // torchvision OIHW
};

__global__ void pack_kernel(ConvWeights src, float* __restrict__ packed) {
  const int64_t total = packed_offset(5);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int l = 0;
    while (l < 4 && i >= packed_offset(l + 1)) ++l;
    const ConvShape s = conv_shape(l);
    const int64_t j = i - packed_offset(l);
    const int n = (int)(j / s.kpad()), k = (int)(j % s.kpad());
    float v = 0.0f;
    if (k < s.k()) {
      const int c = k % s.cin, t = k / s.cin, kx = t % s.ks, ky = t / s.ks;
      const float* w = l == 0 ? src.w[0] : l == 1 ? src.w[1] : l == 2 ? src.w[2] : l == 3 ? src.w[3] : src.w[4];
      if (c < torch_cin(l)) v = w[(((int64_t)n * torch_cin(l) + c) * s.ks + ky) * s.ks + kx];
    }
    packed[i] = tf32_rna(v);
  }
}

// ---- input -----------------------------------------------------------------------------------------------------------
// lpips' ScalingLayer constants, as the fp32 values of its literals
__device__ __forceinline__ float scaled(float v, int c) {
  const float shift = c == 0 ? -.030f : c == 1 ? -.088f : -.188f;
  const float scale = c == 0 ? .458f : c == 1 ? .448f : .450f;
  const float x = __fsub_rn(__fmul_rn(2.0f, v), 1.0f);
  return tf32_rna(__fdiv_rn(__fsub_rn(x, shift), scale));
}

__global__ void __launch_bounds__(256) input_kernel(const void* __restrict__ pred, const void* __restrict__ gt,
                                                    int dtype, int W, int H, const int32_t* __restrict__ roi,
                                                    float4* __restrict__ out) {
  const Roi r = read_roi(roi, W, H);
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, n = (int64_t)r.w * r.h;
  if (!r.valid || i >= n) return;
  const int img = blockIdx.y, y = (int)(i / r.w), x = (int)(i % r.w);
  const int64_t p = 3 * ((int64_t)(r.y + y) * W + (r.x + x));
  float v[3];
  if (dtype == 0) {
    const uint8_t* s = static_cast<const uint8_t*>(img ? gt : pred) + p;
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = __fdiv_rn((float)__ldg(s + c), 255.0f);
  } else {
    const float* s = static_cast<const float*>(img ? gt : pred) + p;
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = __ldg(s + c);
  }
  out[img * n + i] = make_float4(scaled(v[0], 0), scaled(v[1], 1), scaled(v[2], 2), 0.0f);
}

// ---- convolution -----------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void wgmma_wait_one() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

template <int BN>
constexpr int conv_smem_bytes() { return kStages * (kBM + BN) * kBK * 4; }

// Shared-memory stage: A [128 rows][32 k], then B [BN rows][32 k], both K-major without swizzle: core matrix (kq, g)
// (rows 8g..8g+7, k 4kq..4kq+3) at (kq * rows / 8 + g) * 128 bytes.
template <int L, int BN>
__global__ void __launch_bounds__(kConvThreads, 1) conv_kernel(const float* __restrict__ in,
                                                                const float* __restrict__ packed,
                                                                const float* __restrict__ bias, float* __restrict__ out,
                                                                const int32_t* __restrict__ roi, int W, int H) {
  constexpr ConvShape s = conv_shape(L);
  constexpr int Cin = s.cin, Cout = s.cout, KS = s.ks, K = s.k(), Kpad = s.kpad(), KT = Kpad / kBK;
  constexpr int tin = L == 0 ? 0 : L == 1 ? 2 : L == 2 ? 4 : L + 2, tout = layer_tensor(L);
  constexpr uint32_t kABytes = kBM * kBK * 4, kBBytes = BN * kBK * 4, kStageBytes = kABytes + kBBytes;
  constexpr uint32_t kALbo = (kBM / 8) * 128, kBLbo = (BN / 8) * 128;
  extern __shared__ __align__(128) uint8_t smem[];

  const Roi r = read_roi(roi, W, H);
  if (!r.valid) return;
  const Dims d = make_dims(r.w, r.h);
  const int hi = d.h[tin], wi = d.w[tin], ho = d.h[tout], wo = d.w[tout];
  const int M = 2 * ho * wo, m0 = blockIdx.x * kBM, n0 = blockIdx.y * BN;
  if (m0 >= M) return;

  const int tid = threadIdx.x, row = tid & (kBM - 1), kq0 = tid >> 7;
  const int m = m0 + row;
  const bool mvalid = m < M;
  const int img = mvalid ? m / (ho * wo) : 0, rem = mvalid ? m - img * ho * wo : 0;
  const int iy0 = (rem / wo) * s.stride - s.pad, ix0 = (rem % wo) * s.stride - s.pad;
  const float* in_img = in + (int64_t)img * hi * wi * Cin;
  const uint32_t sbase = smem_u32(smem);

  auto load_stage = [&](int kt, int slot) {
    const uint32_t sa = sbase + slot * kStageBytes, sb = sa + kABytes;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int kq = kq0 + 2 * i, k = kt * kBK + 4 * kq;
      const int c = k % Cin, t = k / Cin, kx = t % KS, ky = t / KS;
      const int iy = iy0 + ky, ix = ix0 + kx;
      const bool ok = mvalid && k < K && iy >= 0 && iy < hi && ix >= 0 && ix < wi;
      const float* src = ok ? in_img + ((int64_t)iy * wi + ix) * Cin + c : in;
      cp_async16(sa + (kq * (kBM / 8) + (row >> 3)) * 128 + (row & 7) * 16, src, ok ? 16u : 0u);
    }
#pragma unroll
    for (int j = tid; j < BN * (kBK / 4); j += kConvThreads) {
      const int n = j % BN, kq = j / BN;
      cp_async16(sb + (kq * (BN / 8) + (n >> 3)) * 128 + (n & 7) * 16,
                 packed + (int64_t)(n0 + n) * Kpad + kt * kBK + 4 * kq, 16u);
    }
  };

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
  const int wg = tid >> 7;

  load_stage(0, 0);
  cp_async_commit();
  if (KT > 1) load_stage(1, 1);
  cp_async_commit();
  for (int kt = 0; kt < KT; ++kt) {
    // stage kt has landed for every thread, and every warpgroup has retired its MMAs of stage kt - 2 (waited for below
    // in iteration kt - 1), whose slot the load of stage kt + 2 reuses
    cp_async_wait<1>();
    fence_proxy_async_smem();
    __syncthreads();
    if (kt + 2 < KT) load_stage(kt + 2, (kt + 2) % kStages);
    cp_async_commit();
    const uint32_t sa = sbase + (kt % kStages) * kStageBytes + wg * 8 * 128, sb = sbase + (kt % kStages) * kStageBytes + kABytes;
    wgmma_fence();
#pragma unroll
    for (int k8 = 0; k8 < kBK / 8; ++k8)
      wgmma_tf32<BN>(acc, make_smem_desc(sa + 2 * k8 * kALbo, kALbo, 128), make_smem_desc(sb + 2 * k8 * kBLbo, kBLbo, 128), 1);
    wgmma_commit();
    wgmma_wait_one();
  }
  wgmma_wait_all();
  wgmma_fence_regs<BN / 2>(acc);

  // epilogue: register 4j + 2h + e is row 16 warp + lane / 4 + 8h, column 8j + 2 (lane % 4) + e of the warpgroup's tile
  const int lane = tid & 31, warp = (tid >> 5) & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int mo = m0 + 64 * wg + 16 * warp + (lane >> 2) + 8 * h;
    if (mo >= M) continue;
    float* o = out + (int64_t)mo * Cout + n0 + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const float2 b = __ldg(reinterpret_cast<const float2*>(bias + n0 + 8 * j + 2 * (lane & 3)));
      const float v0 = tf32_rna(fmaxf(__fadd_rn(acc[4 * j + 2 * h], b.x), 0.0f));
      const float v1 = tf32_rna(fmaxf(__fadd_rn(acc[4 * j + 2 * h + 1], b.y), 0.0f));
      *reinterpret_cast<float2*>(o + 8 * j) = make_float2(v0, v1);
    }
  }
}

// ---- max-pool 3x3 / 2 ------------------------------------------------------------------------------------------------
template <int C, int tin>
__global__ void __launch_bounds__(256) pool_kernel(const float4* __restrict__ in, float4* __restrict__ out,
                                                   const int32_t* __restrict__ roi, int W, int H) {
  const Roi r = read_roi(roi, W, H);
  if (!r.valid) return;
  const Dims d = make_dims(r.w, r.h);
  const int hi = d.h[tin], wi = d.w[tin], ho = d.h[tin + 1], wo = d.w[tin + 1];
  constexpr int C4 = C / 4;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * (int64_t)ho * wo * C4) return;
  const int c = (int)(i % C4);
  const int64_t p = i / C4;
  const int ox = (int)(p % wo), oy = (int)(p / wo % ho), img = (int)(p / ((int64_t)wo * ho));
  const float4* base = in + (((int64_t)img * hi + 2 * oy) * wi + 2 * ox) * C4 + c;
  float4 m = __ldg(base);
#pragma unroll
  for (int dy = 0; dy < 3; ++dy)
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) {
      const float4 v = __ldg(base + ((int64_t)dy * wi + dx) * C4);
      m.x = fmaxf(m.x, v.x), m.y = fmaxf(m.y, v.y), m.z = fmaxf(m.z, v.z), m.w = fmaxf(m.w, v.w);
    }
  out[i] = m;
}

// ---- tail ------------------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One warp per pixel: lane handles channels lane + 32 i.  Both images go through the same arithmetic, so swapping them
// swaps n0 and n1 exactly and (f0 - f1)^2 is unchanged: the score is symmetric bit for bit.
template <int C, int t>
__global__ void __launch_bounds__(kTailWarps * 32) tail_kernel(const float* __restrict__ feat, const float* __restrict__ lin,
                                                                const int32_t* __restrict__ roi, int W, int H,
                                                                double* __restrict__ slots) {
  const Roi r = read_roi(roi, W, H);
  if (!r.valid) return;
  const Dims d = make_dims(r.w, r.h);
  const int64_t P = (int64_t)d.h[t] * d.w[t];
  if ((int64_t)blockIdx.x * kTailPix >= P) return;
  constexpr int kPer = C / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float l[kPer];
#pragma unroll
  for (int i = 0; i < kPer; ++i) l[i] = __ldg(lin + lane + 32 * i);
  double acc = 0.0;
  for (int q = 0; q < kTailPixPerWarp; ++q) {
    const int64_t p = (int64_t)blockIdx.x * kTailPix + warp * kTailPixPerWarp + q;
    if (p >= P) break;
    const float* f0 = feat + p * C;
    const float* f1 = feat + (P + p) * C;
    float y0[kPer], y1[kPer], s0 = 0.0f, s1 = 0.0f;
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
      y0[i] = __ldg(f0 + lane + 32 * i), y1[i] = __ldg(f1 + lane + 32 * i);
      s0 = __fmaf_rn(y0[i], y0[i], s0), s1 = __fmaf_rn(y1[i], y1[i], s1);
    }
    s0 = warp_sum(s0), s1 = warp_sum(s1);
    const float n0 = __fadd_rn(__fsqrt_rn(s0), 1e-10f), n1 = __fadd_rn(__fsqrt_rn(s1), 1e-10f);
    float v = 0.0f;
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
      const float e = __fsub_rn(__fdiv_rn(y0[i], n0), __fdiv_rn(y1[i], n1));
      v = __fmaf_rn(l[i], __fmul_rn(e, e), v);
    }
    acc += (double)warp_sum(v);
  }
  __shared__ double s_acc[kTailWarps];
  if (lane == 0) s_acc[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double o = 0.0;
    for (int i = 0; i < kTailWarps; ++i) o += s_acc[i];
    slots[blockIdx.x] = o;
  }
}

struct SlotOffsets {
  int64_t o[6];
};

__global__ void __launch_bounds__(kFinishThreads) finish_kernel(const double* __restrict__ slots, SlotOffsets so,
                                                                const int32_t* __restrict__ roi, int W, int H,
                                                                double* __restrict__ out) {
  __shared__ double s_d[kFinishThreads / 32];
  const Roi r = read_roi(roi, W, H);
  if (!r.valid) {
    if (threadIdx.x == 0) out[0] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  const Dims d = make_dims(r.w, r.h);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double total = 0.0;
  for (int l = 0; l < 5; ++l) {
    const int t = layer_tensor(l);
    const int64_t P = (int64_t)d.h[t] * d.w[t], n = (P + kTailPix - 1) / kTailPix;
    double a = 0.0;
    for (int64_t i = tid; i < n; i += kFinishThreads) a += slots[so.o[l] + i];
    a = warp_sum(a);
    __syncthreads();
    if (lane == 0) s_d[warp] = a;
    __syncthreads();
    if (tid == 0) {
      double sum = 0.0;
      for (int i = 0; i < kFinishThreads / 32; ++i) sum += s_d[i];
      total += sum / (double)P;
    }
  }
  if (tid == 0) out[0] = total;
}

template <int L, int BN>
int launch_conv(const float* in, const float* packed, const float* bias, float* out, const int32_t* roi, int W, int H,
                int64_t max_pixels, cudaStream_t st) {
  constexpr int smem = conv_smem_bytes<BN>();
  HRF_CUDA(cudaFuncSetAttribute(conv_kernel<L, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const dim3 grid((unsigned)((2 * max_pixels + kBM - 1) / kBM), conv_shape(L).cout / BN);
  conv_kernel<L, BN><<<grid, kConvThreads, smem, st>>>(in, packed + packed_offset(L), bias, out, roi, W, H);
  HRF_CHECK_LAUNCH();
  return 0;
}

template <int C, int tin>
int launch_pool(const float* in, float* out, const Dims& dmax, const int32_t* roi, int W, int H,
                cudaStream_t st) {
  const int64_t n = 2 * (int64_t)dmax.h[tin + 1] * dmax.w[tin + 1] * (C / 4);
  pool_kernel<C, tin><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float4*>(in),
                                                                    reinterpret_cast<float4*>(out), roi, W, H);
  HRF_CHECK_LAUNCH();
  return 0;
}

template <int C, int t>
int launch_tail(const float* feat, const float* lin, int64_t num_slots, const int32_t* roi, int W, int H,
                double* slots, cudaStream_t st) {
  tail_kernel<C, t><<<(unsigned)num_slots, kTailWarps * 32, 0, st>>>(feat, lin, roi, W, H, slots);
  HRF_CHECK_LAUNCH();
  return 0;
}

#define HRF_TRY(expr)            \
  do {                           \
    const int _rc = (expr);      \
    if (_rc != 0) return _rc;    \
  } while (0)

}  // namespace
}  // namespace hrf

using namespace hrf;

extern "C" int64_t hrf_lpips_packed_bytes(void) { return packed_offset(5) * (int64_t)sizeof(float); }

extern "C" int hrf_lpips_pack_weights(const float* const* conv_w, void* packed, void* stream) {
  HRF_REQUIRE(conv_w && packed, "null argument");
  ConvWeights w;
  for (int l = 0; l < 5; ++l) {
    HRF_REQUIRE(conv_w[l], "null conv weight");
    w.w[l] = conv_w[l];
  }
  HRF_REQUIRE(reinterpret_cast<uintptr_t>(packed) % 16 == 0, "packed weights must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t n = packed_offset(5);
  pack_kernel<<<(unsigned)std::min<int64_t>((n + 255) / 256, (int64_t)sm_count() * 8), 256, 0, st>>>(
      w, static_cast<float*>(packed));
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int64_t hrf_lpips_workspace_bytes(int width, int height) {
  if (width <= 0 || height <= 0) return 0;
  const Layout L = make_layout(width, height);
  return L.tensor[kTensors] + L.slots[5] * (int64_t)sizeof(double);
}

extern "C" int hrf_lpips(const hrf_lpips_weights* weights, const void* pred, const void* gt, int dtype, int width,
                         int height, const int32_t* roi, double* out, void* workspace, void* stream) {
  HRF_REQUIRE(weights && weights->packed && pred && gt && out && workspace, "null argument");
  for (int l = 0; l < 5; ++l) HRF_REQUIRE(weights->bias[l] && weights->lin[l], "null bias or lin weight");
  HRF_REQUIRE(dtype == 0 || dtype == 1, "dtype must be 0 (uint8) or 1 (float32)");
  HRF_REQUIRE(width > 0 && height > 0 && (int64_t)width * height * 3 < (int64_t)1 << 31, "bad image size");
  HRF_REQUIRE(reinterpret_cast<uintptr_t>(workspace) % kAlign == 0, "workspace must be 256-byte aligned");
  HRF_REQUIRE(reinterpret_cast<uintptr_t>(weights->packed) % 16 == 0, "packed weights must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const Layout L = make_layout(width, height);
  char* ws = static_cast<char*>(workspace);
  float* t[kTensors];
  for (int i = 0; i < kTensors; ++i) t[i] = reinterpret_cast<float*>(ws + L.tensor[i]);
  double* slots = reinterpret_cast<double*>(ws + L.tensor[kTensors]);
  SlotOffsets so;
  for (int l = 0; l < 6; ++l) so.o[l] = L.slots[l];
  if (width >= kMinRoi && height >= kMinRoi) {   // otherwise no ROI is valid: only the finish pass runs
    const Dims dmax = make_dims(width, height);
    const float* pk = static_cast<const float*>(weights->packed);
    const int64_t npix = (int64_t)width * height;
    input_kernel<<<dim3((unsigned)((npix + 255) / 256), 2), 256, 0, st>>>(pred, gt, dtype, width, height, roi,
                                                                          reinterpret_cast<float4*>(t[0]));
    HRF_CHECK_LAUNCH();
    HRF_TRY((launch_conv<0, 64>(t[0], pk, weights->bias[0], t[1], roi, width, height, (int64_t)dmax.h[1] * dmax.w[1], st)));
    HRF_TRY((launch_pool<64, 1>(t[1], t[2], dmax, roi, width, height, st)));
    HRF_TRY((launch_conv<1, 64>(t[2], pk, weights->bias[1], t[3], roi, width, height, (int64_t)dmax.h[3] * dmax.w[3], st)));
    HRF_TRY((launch_pool<192, 3>(t[3], t[4], dmax, roi, width, height, st)));
    HRF_TRY((launch_conv<2, 128>(t[4], pk, weights->bias[2], t[5], roi, width, height, (int64_t)dmax.h[5] * dmax.w[5], st)));
    HRF_TRY((launch_conv<3, 128>(t[5], pk, weights->bias[3], t[6], roi, width, height, (int64_t)dmax.h[6] * dmax.w[6], st)));
    HRF_TRY((launch_conv<4, 128>(t[6], pk, weights->bias[4], t[7], roi, width, height, (int64_t)dmax.h[7] * dmax.w[7], st)));
    HRF_TRY((launch_tail<64, 1>(t[1], weights->lin[0], L.slots[1] - L.slots[0], roi, width, height, slots + L.slots[0], st)));
    HRF_TRY((launch_tail<192, 3>(t[3], weights->lin[1], L.slots[2] - L.slots[1], roi, width, height, slots + L.slots[1], st)));
    HRF_TRY((launch_tail<384, 5>(t[5], weights->lin[2], L.slots[3] - L.slots[2], roi, width, height, slots + L.slots[2], st)));
    HRF_TRY((launch_tail<256, 6>(t[6], weights->lin[3], L.slots[4] - L.slots[3], roi, width, height, slots + L.slots[3], st)));
    HRF_TRY((launch_tail<256, 7>(t[7], weights->lin[4], L.slots[5] - L.slots[4], roi, width, height, slots + L.slots[4], st)));
  }
  finish_kernel<<<1, kFinishThreads, 0, st>>>(slots, so, roi, width, height, out);
  HRF_CHECK_LAUNCH();
  return 0;
}
