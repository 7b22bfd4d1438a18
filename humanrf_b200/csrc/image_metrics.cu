// Image scores of the ActorsHQ evaluation (actorshq/evaluation/evaluate.py:76-85,117-125) on 8-bit RGB images: the mask's
// bounding rectangle (cv2.boundingRect), a PSNR over the masked pixels and scikit-image's SSIM over that rectangle.
// Contract: include/humanrf_b200.h, hrf_image_metrics.  Three launches, no host synchronisation:
//   roi_kernel    : min / max of the masked pixels' coordinates, folded with integer atomicMax into the workspace header;
//   tile_kernel   : one CTA per 64x16 pixel tile, skipped when the tile misses the ROI.  It stages its pixels and a
//                   3-pixel halo of both images in shared memory (only bytes inside the ROI are read), forms the 7x7
//                   window sums separably with sliding sums (exact int32), evaluates S in fp64 for every window lying
//                   wholly inside the ROI and writes its partial sums to its own slot;
//   finish_kernel : one CTA folds the slots in a fixed order and writes out / roi.  Two calls write identical bytes.
#include <algorithm>

#include "common.cuh"

namespace hrf {
namespace {

constexpr int kTX = 64, kTY = 16, kR = 3;          // tile of window centres, window radius
constexpr int kSH = kTY + 2 * kR;                  // staged rows (22)
constexpr int kRowWords = 56;                      // 3 * (kTX + 6) bytes + up to 3 bytes of alignment on either side <= 216
constexpr int kThreads = 256;
constexpr int kSegs = 8;                           // horizontal pass: 8 runs of 8 window columns per staged row
constexpr int kRowsPerThread = kTY / (kThreads / kTX);   // vertical pass: 4 window rows per thread
constexpr int kFinishThreads = 1024;
constexpr int64_t kSlotOffset = 64;                // workspace: uint32 box[4], then the per-tile slots

// 49^2 C1 and 48*49 C2, C1 = (0.01 * 255)^2, C2 = (0.03 * 255)^2 (skimage's K1, K2 with data_range 255)
constexpr double kK1 = 2401.0 * (0.01 * 255.0) * (0.01 * 255.0);
constexpr double kK2 = 2352.0 * (0.03 * 255.0) * (0.03 * 255.0);

struct Slot {
  double ssim[3];        // sum of S over the tile's valid windows, per channel
  long long sse;         // sum over the tile's masked pixels of sum_c (p_c - g_c)^2
  int32_t masked;        // masked pixels of the tile
  int32_t windows;       // valid windows of the tile
};
static_assert(sizeof(Slot) == 40, "slot layout");

// Box in the workspace header, all four zero-initialised and raised with atomicMax:
// box[0] = max(W - x), box[1] = max(H - y), box[2] = max(x + 1), box[3] = max(y + 1) over the masked pixels.
struct Roi {
  int x0, y0, x1, y1;    // inclusive; x1 < x0 when the mask is empty
};
__device__ __forceinline__ Roi read_roi(const uint32_t* box, int W, int H) {
  return Roi{W - (int)box[0], H - (int)box[1], (int)box[2] - 1, (int)box[3] - 1};
}

__device__ __forceinline__ uint32_t warp_max(uint32_t v) { return __reduce_max_sync(0xffffffffu, v); }

__global__ void __launch_bounds__(kThreads) roi_kernel(const uint8_t* __restrict__ mask, int W, int H,
                                                       uint32_t* __restrict__ box) {
  // 16-byte chunks of the aligned-down range: bytes outside [0, W*H) share an aligned chunk with a mask byte and are
  // skipped by index.
  const uintptr_t p0 = reinterpret_cast<uintptr_t>(mask), a0 = p0 & ~uintptr_t(15);
  const int64_t n = (int64_t)W * H;
  const int64_t lead = (int64_t)(p0 - a0), nchunks = (lead + n + 15) / 16;
  uint32_t m[4] = {0, 0, 0, 0};
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nchunks; k += (int64_t)gridDim.x * blockDim.x) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(a0) + k);
    if ((v.x | v.y | v.z | v.w) == 0) continue;
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    const int64_t i0 = 16 * k - lead;                   // mask index of the chunk's first byte
    const int b0 = i0 < 0 ? (int)-i0 : 0;
    int y = (int)((i0 + b0) / W), x = (int)(i0 + b0 - (int64_t)y * W);
#pragma unroll
    for (int b = 0; b < 16; ++b) {
      if (b < b0) continue;
      if (i0 + b >= n) break;
      if ((w[b >> 2] >> (8 * (b & 3))) & 0xffu) {
        m[0] = max(m[0], (uint32_t)(W - x));
        m[1] = max(m[1], (uint32_t)(H - y));
        m[2] = max(m[2], (uint32_t)(x + 1));
        m[3] = max(m[3], (uint32_t)(y + 1));
      }
      if (++x == W) x = 0, ++y;
    }
  }
  __shared__ uint32_t s_m[kThreads / 32][4];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint32_t r = warp_max(m[q]);
    if (lane == 0) s_m[warp][q] = r;
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    uint32_t r = 0;
    for (int i = 0; i < kThreads / 32; ++i) r = max(r, s_m[i][threadIdx.x]);
    if (r) atomicMax(box + threadIdx.x, r);
  }
}

// S of one window from its integer sums (X, Y the two images' 49 samples of one channel):
//   S = (2 ux uy + C1)(2 vxy + C2) / ((ux^2 + uy^2 + C1)(vx + vy + C2)),  ux = Sx / 49, vx = (49 Sxx - Sx^2) / (48 * 49),
// with every 49 and 48 * 49 cancelled: the four factors are exact int32 values plus one rounded constant each.
__device__ __forceinline__ double window_ssim(uint32_t sxy_packed, int sxx, int syy, int sxy) {
  const int sx = (int)(sxy_packed & 0xffffu), sy = (int)(sxy_packed >> 16);
  const int nvx = 49 * sxx - sx * sx, nvy = 49 * syy - sy * sy, nvxy = 49 * sxy - sx * sy;
  const double a1 = (double)(2 * sx * sy) + kK1, b1 = (double)(sx * sx + sy * sy) + kK1;
  const double a2 = (double)(2 * nvxy) + kK2, b2 = (double)(nvx + nvy) + kK2;
  return (a1 * a2) / (b1 * b2);
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(kThreads) tile_kernel(const uint8_t* __restrict__ pred, const uint8_t* __restrict__ gt,
                                                        const uint8_t* __restrict__ mask, int W, int H,
                                                        const uint32_t* __restrict__ box, Slot* __restrict__ slots) {
  __shared__ __align__(16) uint32_t s_stage[2][kSH][kRowWords];   // raw row bytes of pred (0) and gt (1)
  __shared__ int s_shift[2][kSH];                                 // byte of staged column 0, channel 0 in its row
  __shared__ uint32_t s_sum[4][kSH][kTX + 1];                     // horizontal 7-sums: Sx | Sy << 16, Sxx, Syy, Sxy
  __shared__ double s_red[kThreads / 32][3];
  __shared__ long long s_red_i[kThreads / 32][3];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gx0 = blockIdx.x * kTX, gy0 = blockIdx.y * kTY;
  Slot* slot = slots + blockIdx.y * gridDim.x + blockIdx.x;
  const Roi roi = read_roi(box, W, H);
  // the tile's pixels [gx0, gx0 + kTX) x [gy0, gy0 + kTY) miss the ROI (or the mask is empty): nothing to add
  if (roi.x1 < roi.x0 || gx0 > roi.x1 || gx0 + kTX <= roi.x0 || gy0 > roi.y1 || gy0 + kTY <= roi.y0) {
    if (tid == 0) *slot = Slot{{0.0, 0.0, 0.0}, 0, 0, 0};
    return;
  }

  // ---- stage the ROI part of rows gy0-3 .. gy0+18, columns gx0-3 .. gx0+66, as aligned 32-bit words
  const int cl = max(gx0 - kR, roi.x0), ch = min(gx0 + kTX + kR, roi.x1 + 1);   // ROI columns of the staged span
  const int64_t row_bytes = 3 * (int64_t)W;
  for (int i = tid; i < 2 * kSH * kRowWords; i += kThreads) {
    const int m = i / (kSH * kRowWords), r = (i / kRowWords) % kSH, j = i % kRowWords;
    const int gy = gy0 - kR + r;
    const uintptr_t row = reinterpret_cast<uintptr_t>(m ? gt : pred) + (uintptr_t)(gy * row_bytes);
    const uintptr_t s = row + (uintptr_t)(3 * (int64_t)(gx0 - kR)), sbase = s & ~uintptr_t(3);
    if (j == 0) s_shift[m][r] = (int)(s - sbase);
    if (gy < roi.y0 || gy > roi.y1 || cl >= ch) continue;
    const uintptr_t a = (row + 3 * (uintptr_t)cl) & ~uintptr_t(3), b = (row + 3 * (uintptr_t)ch + 3) & ~uintptr_t(3);
    const int first = (int)((a - sbase) >> 2), count = (int)((b - a) >> 2);
    if (j >= first && j < first + count) s_stage[m][r][j] = __ldg(reinterpret_cast<const uint32_t*>(a) + (j - first));
  }

  // ---- squared error over the tile's masked pixels (every masked pixel is inside the ROI)
  uint32_t sse = 0, masked = 0;
  __syncthreads();
  for (int i = tid; i < kTX * kTY; i += kThreads) {
    const int xl = i % kTX, yl = i / kTX, gx = gx0 + xl, gy = gy0 + yl;
    if (gx < roi.x0 || gx > roi.x1 || gy < roi.y0 || gy > roi.y1) continue;
    if (__ldg(mask + (int64_t)gy * W + gx) == 0) continue;
    const uint8_t* p = reinterpret_cast<const uint8_t*>(s_stage[0][yl + kR]) + s_shift[0][yl + kR] + 3 * (xl + kR);
    const uint8_t* g = reinterpret_cast<const uint8_t*>(s_stage[1][yl + kR]) + s_shift[1][yl + kR] + 3 * (xl + kR);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int d = (int)p[c] - (int)g[c];
      sse += (uint32_t)(d * d);
    }
    ++masked;
  }

  // ---- SSIM windows: centres in [x0+3, x1-3] x [y0+3, y1-3]
  const int wx0 = max(gx0, roi.x0 + kR), wx1 = min(gx0 + kTX - 1, roi.x1 - kR);
  const int wy0 = max(gy0, roi.y0 + kR), wy1 = min(gy0 + kTY - 1, roi.y1 - kR);
  double ssim[3] = {0.0, 0.0, 0.0};
  uint32_t windows = 0;
  if (wx0 <= wx1 && wy0 <= wy1) {             // CTA-uniform
    const int xl = tid % kTX, yb = (tid / kTX) * kRowsPerThread;
#pragma unroll
    for (int c = 0; c < 3; ++c) {     // unrolled: ssim[c] stays in registers
      // horizontal pass: staged row r, window columns [8 seg, 8 seg + 8), sliding over the 7 taps
      for (int i = tid; i < kSH * kSegs; i += kThreads) {
        const int r = i / kSegs, x0 = (i % kSegs) * (kTX / kSegs), gy = gy0 - kR + r;
        if (gy < roi.y0 || gy > roi.y1) continue;       // rows outside the ROI feed no valid window
        // columns outside the ROI hold stale bytes: they only enter sums of invalid windows, and the unsigned sliding
        // sums take them out again exactly
        const uint8_t* p = reinterpret_cast<const uint8_t*>(s_stage[0][r]) + s_shift[0][r] + c;
        const uint8_t* g = reinterpret_cast<const uint8_t*>(s_stage[1][r]) + s_shift[1][r] + c;
        uint32_t pk = 0, sxx = 0, syy = 0, sxy = 0;
#pragma unroll
        for (int k = 0; k < 2 * kR; ++k) {
          const uint32_t a = p[3 * (x0 + k)], b = g[3 * (x0 + k)];
          pk += a | (b << 16), sxx += a * a, syy += b * b, sxy += a * b;
        }
#pragma unroll
        for (int o = 0; o < kTX / kSegs; ++o) {
          const uint32_t a = p[3 * (x0 + o + 2 * kR)], b = g[3 * (x0 + o + 2 * kR)];
          pk += a | (b << 16), sxx += a * a, syy += b * b, sxy += a * b;
          s_sum[0][r][x0 + o] = pk, s_sum[1][r][x0 + o] = sxx, s_sum[2][r][x0 + o] = syy, s_sum[3][r][x0 + o] = sxy;
          const uint32_t a0 = p[3 * (x0 + o)], b0 = g[3 * (x0 + o)];
          pk -= a0 | (b0 << 16), sxx -= a0 * a0, syy -= b0 * b0, sxy -= a0 * b0;
        }
      }
      __syncthreads();
      // vertical pass: window column xl, window rows [yb, yb + 4), sliding over staged rows
      const int gx = gx0 + xl;
      if (gx >= wx0 && gx <= wx1) {
        uint32_t pk = 0, sxx = 0, syy = 0, sxy = 0;
#pragma unroll
        for (int k = 0; k < 2 * kR; ++k) {
          const int r = yb + k;
          pk += s_sum[0][r][xl], sxx += s_sum[1][r][xl], syy += s_sum[2][r][xl], sxy += s_sum[3][r][xl];
        }
#pragma unroll
        for (int o = 0; o < kRowsPerThread; ++o) {
          const int r = yb + o + 2 * kR, r0 = yb + o, gy = gy0 + yb + o;
          pk += s_sum[0][r][xl], sxx += s_sum[1][r][xl], syy += s_sum[2][r][xl], sxy += s_sum[3][r][xl];
          if (gy >= wy0 && gy <= wy1) {
            ssim[c] += window_ssim(pk, (int)sxx, (int)syy, (int)sxy);
            windows += c == 0;
          }
          pk -= s_sum[0][r0][xl], sxx -= s_sum[1][r0][xl], syy -= s_sum[2][r0][xl], sxy -= s_sum[3][r0][xl];
        }
      }
      __syncthreads();
    }
  }

  // ---- fixed-order CTA reduction into the tile's slot
  double v[3] = {ssim[0], ssim[1], ssim[2]};
  long long u[3] = {(long long)sse, (long long)masked, (long long)windows};
#pragma unroll
  for (int q = 0; q < 3; ++q) v[q] = warp_sum(v[q]);
#pragma unroll
  for (int q = 0; q < 3; ++q) u[q] = warp_sum(u[q]);
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < 3; ++q) s_red[warp][q] = v[q], s_red_i[warp][q] = u[q];
  }
  __syncthreads();
  if (tid == 0) {
    Slot o{{0.0, 0.0, 0.0}, 0, 0, 0};
    for (int i = 0; i < kThreads / 32; ++i) {
      for (int q = 0; q < 3; ++q) o.ssim[q] += s_red[i][q];
      o.sse += s_red_i[i][0];
      o.masked += (int32_t)s_red_i[i][1];
      o.windows += (int32_t)s_red_i[i][2];
    }
    *slot = o;
  }
}

__global__ void __launch_bounds__(kFinishThreads) finish_kernel(const uint32_t* __restrict__ box,
                                                                const Slot* __restrict__ slots, int num_slots, int W,
                                                                int H, double* __restrict__ out, int32_t* __restrict__ roi_out) {
  __shared__ double s_d[kFinishThreads / 32][3];
  __shared__ long long s_i[kFinishThreads / 32][3];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double d[3] = {0.0, 0.0, 0.0};
  long long u[3] = {0, 0, 0};
  for (int i = tid; i < num_slots; i += kFinishThreads) {
    const Slot s = slots[i];
#pragma unroll
    for (int q = 0; q < 3; ++q) d[q] += s.ssim[q];
    u[0] += s.sse, u[1] += s.masked, u[2] += s.windows;
  }
#pragma unroll
  for (int q = 0; q < 3; ++q) d[q] = warp_sum(d[q]), u[q] = warp_sum(u[q]);
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < 3; ++q) s_d[warp][q] = d[q], s_i[warp][q] = u[q];
  }
  __syncthreads();
  if (tid != 0) return;
  double t[3] = {0.0, 0.0, 0.0};
  long long sse = 0, masked = 0, windows = 0;
  for (int i = 0; i < kFinishThreads / 32; ++i) {
    for (int q = 0; q < 3; ++q) t[q] += s_d[i][q];
    sse += s_i[i][0], masked += s_i[i][1], windows += s_i[i][2];
  }
  const Roi r = read_roi(box, W, H);
  const bool empty = r.x1 < r.x0;
  roi_out[0] = empty ? 0 : r.x0;
  roi_out[1] = empty ? 0 : r.y0;
  roi_out[2] = empty ? 0 : r.x1 - r.x0 + 1;
  roi_out[3] = empty ? 0 : r.y1 - r.y0 + 1;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  // MSE = sse / (3 * 255^2 * masked); sse == 0 gives -10 log10(0) = +inf
  out[0] = masked == 0 ? nan : -10.0 * log10((double)sse / (195075.0 * (double)masked));
  const double w = (double)windows;
  out[1] = windows == 0 ? nan : (t[0] / w + t[1] / w + t[2] / w) / 3.0;
}

int64_t num_tiles(int width, int height) {
  return (int64_t)((width + kTX - 1) / kTX) * ((height + kTY - 1) / kTY);
}

}  // namespace
}  // namespace hrf

using namespace hrf;

extern "C" int64_t hrf_image_metrics_workspace_bytes(int width, int height) {
  if (width <= 0 || height <= 0) return 0;
  return kSlotOffset + num_tiles(width, height) * (int64_t)sizeof(Slot);
}

extern "C" int hrf_image_metrics(const uint8_t* pred, const uint8_t* gt, const uint8_t* mask, int width, int height,
                                 double* out, int32_t* roi, void* workspace, void* stream) {
  HRF_REQUIRE(pred && gt && mask && out && roi && workspace, "null argument");
  HRF_REQUIRE(width > 0 && height > 0 && (int64_t)width * height * 3 < (int64_t)1 << 31, "bad image size");
  HRF_REQUIRE(reinterpret_cast<uintptr_t>(workspace) % 16 == 0, "workspace must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint32_t* box = reinterpret_cast<uint32_t*>(workspace);
  Slot* slots = reinterpret_cast<Slot*>(reinterpret_cast<char*>(workspace) + kSlotOffset);
  HRF_CUDA(cudaMemsetAsync(box, 0, 4 * sizeof(uint32_t), st));
  const int64_t chunks = ((int64_t)width * height + 30) / 16 + 1;
  const int64_t roi_blocks = std::min<int64_t>((chunks + kThreads - 1) / kThreads, (int64_t)sm_count() * 8);
  roi_kernel<<<(unsigned)roi_blocks, kThreads, 0, st>>>(mask, width, height, box);
  HRF_CHECK_LAUNCH();
  const dim3 tiles((width + kTX - 1) / kTX, (height + kTY - 1) / kTY);
  tile_kernel<<<tiles, kThreads, 0, st>>>(pred, gt, mask, width, height, box, slots);
  HRF_CHECK_LAUNCH();
  finish_kernel<<<1, kFinishThreads, 0, st>>>(box, slots, (int)num_tiles(width, height), width, height, out, roi);
  HRF_CHECK_LAUNCH();
  return 0;
}
