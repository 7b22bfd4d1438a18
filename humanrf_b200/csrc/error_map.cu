// Per-tile error map of the training pool (toolbox/error_map.py ErrorMap, DESIGN.md §3.20): the fused train step adds
// each ray's colour Huber error into its pixel's tile (hrf_error_map_accumulate), one update per step folds the step's
// tile means into a running average and rebuilds the integer CDF of the tile weights (hrf_error_map_update), and the
// loader draws the next batch's pool indices from that CDF (hrf_error_map_draw).
//
// Pool geometry: pool pixel slot * P + p, P = W * H.  The pixel's (x, y) is the sampler's (ray_minmax_kernel): a
// landscape slot is w = W wide and h = H high, a portrait slot (landscape_modes[slot] == 0) h = W wide and W = H high,
// x = p % w, y = p / w.  Tiles are T x T pixels in the slot's own orientation, ceil(w/T) per row, row-major; a slot has
// ceil(W/T) * ceil(H/T) tiles either way, and tile t = slot * tiles_per_slot + (y / T) * ceil(w/T) + x / T.  A border
// tile holds min(T, w - i T) * min(T, h - j T) pixels (npix).
//
// Everything summed is an integer, so every output is independent of scheduling:
//   accumulate : q_r = min(rint(e_r 2^32), 2^32 - 1) added with 64-bit atomics into the ray's tile, and count += 1; the
//                lanes of a warp that share a tile add their q and count first (__match_any_sync, reduce_peers).
//   update     : ema_kernel (tile means into the EMA, sums cleared, per-block weight totals), scan_blocks_kernel (one CTA:
//                exclusive scan of the block totals), cdf_kernel (each block rescans its tiles' weights from the new EMA
//                and adds its block's offset): three launches, about 20 bytes of traffic per tile.
//   draw       : counter-based SplitMix64 hashes mapped onto a range with __umul64hi, a binary search (upper_bound).
#include <algorithm>
#include <cmath>

#include "camera_common.cuh"

namespace hrf {

constexpr int kMapThreads = 256;
constexpr int kMapItems = 8;
constexpr int64_t kMapBlockTiles = (int64_t)kMapThreads * kMapItems;   // tiles per update block
constexpr int kMapMaxTile = 4096;                                       // npix <= 2^24: w = fmax(ema, floor) npix 2^24 is exact in double

struct MapGeo {
  const uint8_t* landscape;
  int64_t slots, pixels_per_slot, tiles_per_slot;
  int W, H, T, tiles_w, tiles_h;       // tiles_w = ceil(W/T), tiles_h = ceil(H/T)
};

__device__ __forceinline__ void slot_shape(const MapGeo& g, int64_t slot, int& w, int& h, int& row_tiles) {
  const bool ls = __ldg(g.landscape + slot) != 0;
  w = ls ? g.W : g.H;
  h = ls ? g.H : g.W;
  row_tiles = ls ? g.tiles_w : g.tiles_h;
}

__device__ __forceinline__ int64_t tile_of_pixel(const MapGeo& g, int64_t idx) {
  const int64_t slot = idx / g.pixels_per_slot, p = idx - slot * g.pixels_per_slot;
  int w, h, rt;
  slot_shape(g, slot, w, h, rt);
  const int x = (int)(p % w), y = (int)(p / w);
  return slot * g.tiles_per_slot + (int64_t)(y / g.T) * rt + x / g.T;
}

// The tile's first pixel (x0, y0), its extent (cw, ch) and its slot's width w.
__device__ __forceinline__ void tile_extent(const MapGeo& g, int64_t t, int64_t& slot, int& x0, int& y0, int& cw, int& ch,
                                            int& w) {
  slot = t / g.tiles_per_slot;
  const int l = (int)(t - slot * g.tiles_per_slot);
  int h, rt;
  slot_shape(g, slot, w, h, rt);
  x0 = (l % rt) * g.T, y0 = (l / rt) * g.T;
  cw = min(g.T, w - x0), ch = min(g.T, h - y0);
}

__device__ __forceinline__ uint64_t tile_weight(const MapGeo& g, int64_t t, float ema, float floor_) {
  int64_t slot;
  int x0, y0, cw, ch, w;
  tile_extent(g, t, slot, x0, y0, cw, ch, w);
  return __double2ull_rn((double)fmaxf(ema, floor_) * (double)(cw * ch) * 0x1p24);
}

// The colour Huber term of ray r as the loss kernels compute it, summed over the three channels in order, without the
// kernels' 1 / (3R) and loss_scale.  The kernels round gt = rgb m + bg (1 - m) differently as compiled: train_loss_kernel
// as fma(m, rgb, (1 - m) bg), response_loss_kernel as fma(1 - m, bg, m rgb), and x = respond(...) - gt there.  Both take
// h = (x / 2) x or (|x| - delta / 2) delta (test_error_map_gpu.py pins this against both kernels).
__device__ __forceinline__ float ray_error(const float* color, const float* wsum, const float* rgba, const float* bg,
                                           const float* table, const int32_t* cams, int num_cameras, float delta,
                                           int64_t r) {
  const float m = rgba[4 * r + 3], om = __fsub_rn(1.f, m);
  const float* row = nullptr;
  float w = 0.f;
  if (table != nullptr) {
    const int c = __ldg(cams + r);
    if (c >= 0 && c < num_cameras) row = table + 6 * c;
    w = wsum[r];
  }
  float e = 0.f;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float c = color[3 * r + k];
    const float b = bg[3 * r + k];
    if (row != nullptr) {
      float fg;
      c = respond(c, w, b, __ldg(row + k), __ldg(row + 3 + k), fg);
    }
    const float gt = table != nullptr ? __fmaf_rn(om, b, __fmul_rn(m, rgba[4 * r + k]))
                                      : __fmaf_rn(m, rgba[4 * r + k], __fmul_rn(om, b));
    const float x = __fsub_rn(c, gt), ax = fabsf(x);
    const float h = ax < delta ? __fmul_rn(__fmul_rn(x, 0.5f), x) : __fmul_rn(__fmaf_rn(delta, -0.5f, ax), delta);
    e = k == 0 ? h : __fadd_rn(e, h);
  }
  return e;
}

__global__ void __launch_bounds__(kMapThreads) error_map_accumulate_kernel(
    const float* __restrict__ color, const float* __restrict__ wsum, const float* __restrict__ rgba,
    const float* __restrict__ bg, const int64_t* __restrict__ pixels, int64_t num_rays, const float* __restrict__ table,
    const int32_t* __restrict__ cams, int num_cameras, float delta, const MapGeo g, unsigned long long* __restrict__ sum,
    unsigned* __restrict__ count, int32_t* __restrict__ error) {
  const int64_t r = (int64_t)blockIdx.x * kMapThreads + threadIdx.x;
  long long tile = -1;
  uint64_t q = 0;
  bool bad = false;
  if (r < num_rays) {
    const int64_t idx = __ldg(pixels + r);
    if (idx < 0 || idx >= g.slots * g.pixels_per_slot) {
      bad = true;
    } else {
      tile = tile_of_pixel(g, idx);
      const float s = __fmul_rn(ray_error(color, wsum, rgba, bg, table, cams, num_cameras, delta, r), 0x1p32f);
      q = s < 0x1p32f ? __float2ull_rn(s) : 0xffffffffull;        // NaN and e >= 1 take the cap
    }
  }
  const unsigned peers = __match_any_sync(0xffffffffu, tile);
  unsigned long long qs[1] = {q};
  reduce_peers<1>(peers, qs);                    // an integer sum: the same whatever the lanes' order
  if (tile >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) {
    atomicAdd(sum + tile, qs[0]);
    atomicAdd(count + tile, (unsigned)__popc(peers));
  }
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(error, 1);
}

// Block-wide sum / exclusive scan of one uint64 per thread (kMapThreads threads).
__device__ __forceinline__ uint64_t block_exclusive_scan(uint64_t v, uint64_t& total) {
  __shared__ uint64_t warp_tot[kMapThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint64_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint64_t t = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += t;
  }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  uint64_t off = 0;
  total = 0;
#pragma unroll
  for (int k = 0; k < kMapThreads / 32; ++k) {
    if (k < warp) off += warp_tot[k];
    total += warp_tot[k];
  }
  __syncthreads();
  return off + inc - v;
}

__global__ void __launch_bounds__(kMapThreads) error_map_ema_kernel(const MapGeo g, int64_t num_tiles,
                                                                    float* __restrict__ ema,
                                                                    unsigned long long* __restrict__ sum,
                                                                    unsigned* __restrict__ count, float beta,
                                                                    float floor_, uint64_t* __restrict__ block_sums) {
  const int64_t base = (int64_t)blockIdx.x * kMapBlockTiles;
  uint64_t local = 0;
#pragma unroll
  for (int k = 0; k < kMapItems; ++k) {
    const int64_t t = base + (int64_t)k * kMapThreads + threadIdx.x;
    if (t >= num_tiles) break;
    float e = ema[t];
    const unsigned c = count[t];
    if (c != 0) {
      const float m = (float)((double)sum[t] / (double)c * 0x1p-32);
      e = __fmaf_rn(beta, __fsub_rn(m, e), e);
      ema[t] = e;
      sum[t] = 0;
      count[t] = 0;
    }
    local += tile_weight(g, t, e, floor_);
  }
  uint64_t total;
  block_exclusive_scan(local, total);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// One CTA: block_sums becomes its exclusive scan.
__global__ void __launch_bounds__(kMapThreads) error_map_scan_blocks_kernel(uint64_t* __restrict__ block_sums,
                                                                            int64_t num_blocks) {
  uint64_t carry = 0;
  for (int64_t b0 = 0; b0 < num_blocks; b0 += kMapThreads) {
    const int64_t b = b0 + threadIdx.x;
    const uint64_t v = b < num_blocks ? block_sums[b] : 0;
    uint64_t total;
    const uint64_t ex = block_exclusive_scan(v, total);
    if (b < num_blocks) block_sums[b] = carry + ex;
    carry += total;
  }
}

// Inclusive CDF of the weights: thread j of block b holds tiles b * kMapBlockTiles + j * kMapItems + [0, kMapItems).
__global__ void __launch_bounds__(kMapThreads) error_map_cdf_kernel(const MapGeo g, int64_t num_tiles,
                                                                    const float* __restrict__ ema, float floor_,
                                                                    const uint64_t* __restrict__ block_offsets,
                                                                    uint64_t* __restrict__ cdf) {
  const int64_t t0 = (int64_t)blockIdx.x * kMapBlockTiles + (int64_t)threadIdx.x * kMapItems;
  uint64_t w[kMapItems], local = 0;
#pragma unroll
  for (int k = 0; k < kMapItems; ++k) {
    w[k] = t0 + k < num_tiles ? tile_weight(g, t0 + k, ema[t0 + k], floor_) : 0;
    local += w[k];
  }
  uint64_t total;
  uint64_t run = block_offsets[blockIdx.x] + block_exclusive_scan(local, total);
#pragma unroll
  for (int k = 0; k < kMapItems; ++k) {
    run += w[k];
    if (t0 + k < num_tiles) cdf[t0 + k] = run;
  }
}

__global__ void __launch_bounds__(kMapThreads) error_map_draw_kernel(const uint64_t* __restrict__ cdf, const MapGeo g,
                                                                     int64_t num_tiles, uint64_t key, int64_t num_rays,
                                                                     int64_t num_uniform, int64_t* __restrict__ out) {
  const int64_t r = (int64_t)blockIdx.x * kMapThreads + threadIdx.x;
  if (r >= num_rays) return;
  const uint64_t h0 = splitmix64(key ^ (uint64_t)(4 * r));
  if (r < num_uniform) {
    out[r] = (int64_t)__umul64hi(h0, (uint64_t)(g.slots * g.pixels_per_slot));
    return;
  }
  const uint64_t target = __umul64hi(h0, __ldg(cdf + num_tiles - 1));
  int64_t lo = 0, hi = num_tiles;                    // upper_bound: the first tile whose inclusive CDF exceeds target
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(cdf + mid) <= target) lo = mid + 1;
    else hi = mid;
  }
  int64_t slot;
  int x0, y0, cw, ch, w;
  tile_extent(g, lo, slot, x0, y0, cw, ch, w);
  const int k = (int)__umul64hi(splitmix64(key ^ (uint64_t)(4 * r + 1)), (uint64_t)(cw * ch));
  out[r] = slot * g.pixels_per_slot + (int64_t)(y0 + k / cw) * w + x0 + k % cw;
}

__global__ void error_map_reset_kernel(float* __restrict__ ema, int64_t first, int64_t n, float prior) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ema[first + i] = prior;
}

// Validated geometry; false when a field is out of range.
bool map_geo(const hrf_error_map_geometry* in, MapGeo& g) {
  if (in == nullptr || in->landscape_modes == nullptr || in->num_slots < 1 || in->image_width < 1 ||
      in->image_height < 1 || in->tile < 1 || in->tile > kMapMaxTile)
    return false;
  g.landscape = in->landscape_modes;
  g.slots = in->num_slots;
  g.W = in->image_width, g.H = in->image_height, g.T = in->tile;
  g.pixels_per_slot = (int64_t)g.W * g.H;
  g.tiles_w = (g.W + g.T - 1) / g.T, g.tiles_h = (g.H + g.T - 1) / g.T;
  g.tiles_per_slot = (int64_t)g.tiles_w * g.tiles_h;
  return true;
}

}  // namespace hrf

using namespace hrf;

// Every weight is at most max(ema, floor) npix 2^24 + 1/2, and the tiles' npix sum to B P: with every EMA and the floor
// at most `top`, the total stays below 2^63 when this holds.
static bool weights_fit(const MapGeo& g, float top) {
  const long double bound = (long double)g.slots * g.pixels_per_slot * std::max(top, 1.f) * 0x1p24L +
                            (long double)g.slots * g.tiles_per_slot;
  return bound < 0x1p63L;
}

extern "C" int64_t hrf_error_map_num_tiles(const hrf_error_map_geometry* geometry, float max_ema) {
  MapGeo g;
  if (!map_geo(geometry, g) || !(max_ema > 0.f) || !std::isfinite(max_ema) || !weights_fit(g, max_ema)) return -1;
  return g.slots * g.tiles_per_slot;
}

extern "C" int64_t hrf_error_map_workspace_bytes(int64_t num_tiles) {
  if (num_tiles < 1) return -1;
  return (num_tiles + kMapBlockTiles - 1) / kMapBlockTiles * 8;
}

extern "C" int hrf_error_map_accumulate(const float* color, const float* weights_sum, const float* rgba,
                                        const float* background, const int64_t* pixels, int64_t num_rays,
                                        const float* response_table, const int32_t* camera_numbers, int num_cameras,
                                        float huber_delta, const hrf_error_map_geometry* geometry, uint64_t* tile_sum,
                                        uint32_t* tile_count, int32_t* error, void* stream) {
  MapGeo g;
  HRF_REQUIRE(map_geo(geometry, g), "bad error-map geometry");
  HRF_REQUIRE(num_rays >= 0 && num_rays < ((int64_t)1 << 40), "ray count outside [0, 2^40)");
  HRF_REQUIRE(huber_delta > 0.f, "huber_delta must be positive");
  HRF_REQUIRE(tile_sum != nullptr && tile_count != nullptr && error != nullptr, "null argument");
  HRF_REQUIRE(response_table == nullptr || (camera_numbers != nullptr && weights_sum != nullptr && num_cameras >= 1),
              "a response table needs camera_numbers, weights_sum and num_cameras >= 1");
  if (num_rays == 0) return 0;
  HRF_REQUIRE(color && rgba && background && pixels, "null input");
  error_map_accumulate_kernel<<<(unsigned)((num_rays + kMapThreads - 1) / kMapThreads), kMapThreads, 0,
                                reinterpret_cast<cudaStream_t>(stream)>>>(
      color, weights_sum, rgba, background, pixels, num_rays, response_table, camera_numbers, num_cameras, huber_delta,
      g, reinterpret_cast<unsigned long long*>(tile_sum), tile_count, error);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_error_map_update(const hrf_error_map_geometry* geometry, float* ema, uint64_t* tile_sum,
                                    uint32_t* tile_count, float beta, float floor_weight, uint64_t* cdf,
                                    void* workspace, void* stream) {
  MapGeo g;
  HRF_REQUIRE(map_geo(geometry, g), "bad error-map geometry");
  HRF_REQUIRE(ema && tile_sum && tile_count && cdf && workspace, "null argument");
  HRF_REQUIRE(beta > 0.f && beta <= 1.f, "beta outside (0, 1]");
  HRF_REQUIRE(floor_weight >= 0x1p-24f && std::isfinite(floor_weight), "floor outside [2^-24, inf)");
  HRF_REQUIRE(weights_fit(g, floor_weight), "floor too large: the tile weights could overflow 64 bits");
  const int64_t n = g.slots * g.tiles_per_slot;
  const int64_t blocks = (n + kMapBlockTiles - 1) / kMapBlockTiles;
  HRF_REQUIRE(blocks < ((int64_t)1 << 31), "too many tiles");
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint64_t* block_sums = reinterpret_cast<uint64_t*>(workspace);
  error_map_ema_kernel<<<(unsigned)blocks, kMapThreads, 0, st>>>(g, n, ema, reinterpret_cast<unsigned long long*>(tile_sum),
                                                                 tile_count, beta, floor_weight, block_sums);
  HRF_CHECK_LAUNCH();
  error_map_scan_blocks_kernel<<<1, kMapThreads, 0, st>>>(block_sums, blocks);
  HRF_CHECK_LAUNCH();
  error_map_cdf_kernel<<<(unsigned)blocks, kMapThreads, 0, st>>>(g, n, ema, floor_weight, block_sums, cdf);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_error_map_draw(const uint64_t* cdf, const hrf_error_map_geometry* geometry, uint64_t seed,
                                  uint64_t counter, int64_t num_rays, double uniform_fraction, int64_t* out,
                                  void* stream) {
  MapGeo g;
  HRF_REQUIRE(map_geo(geometry, g), "bad error-map geometry");
  HRF_REQUIRE(num_rays >= 0 && num_rays < ((int64_t)1 << 40), "ray count outside [0, 2^40)");
  HRF_REQUIRE(uniform_fraction >= 0.0 && uniform_fraction <= 1.0, "uniform_fraction outside [0, 1]");
  if (num_rays == 0) return 0;
  HRF_REQUIRE(cdf != nullptr && out != nullptr, "null argument");
  const int64_t num_uniform = (int64_t)std::floor(uniform_fraction * (double)num_rays);
  const uint64_t key = splitmix64(splitmix64(seed) ^ counter);
  error_map_draw_kernel<<<(unsigned)((num_rays + kMapThreads - 1) / kMapThreads), kMapThreads, 0,
                          reinterpret_cast<cudaStream_t>(stream)>>>(cdf, g, g.slots * g.tiles_per_slot, key, num_rays,
                                                                    num_uniform, out);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_error_map_reset_slots(const hrf_error_map_geometry* geometry, int64_t first_slot, int64_t num_slots,
                                         float prior, float* ema, void* stream) {
  MapGeo g;
  HRF_REQUIRE(map_geo(geometry, g), "bad error-map geometry");
  HRF_REQUIRE(first_slot >= 0 && num_slots >= 0 && first_slot + num_slots <= g.slots, "slots outside the pool");
  HRF_REQUIRE(ema != nullptr && prior >= 0.f && std::isfinite(prior), "bad argument");
  const int64_t n = num_slots * g.tiles_per_slot;
  if (n == 0) return 0;
  error_map_reset_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      ema, first_slot * g.tiles_per_slot, n, prior);
  HRF_CHECK_LAUNCH();
  return 0;
}
