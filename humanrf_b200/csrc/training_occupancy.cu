// Occupancy grids of the training sampler learned from the density field while it trains (toolbox/training_occupancy.py
// TrainingOccupancy, include/humanrf_b200.h, DESIGN.md §3.21).  Per frame: the hull's voxel ids (compact, once), a
// density bound per listed voxel refreshed from one hashed point per voxel (update), and the grid hull AND dilate(live)
// written in place into the frame's occupancy ring slot (pack).
//
//   compact : occ_count_kernel (occupied voxels per 8192-voxel block) -> occ_block_scan_kernel (one CTA: exclusive scan
//             of the block counts, the total) -> occ_write_kernel (ids in ascending order): no atomics, so the list
//             does not depend on scheduling.
//   update  : the bake's persistent tile loop (density_tile.cuh), one row per listed voxel.
//   pack    : a memset of a G^3 byte map, occ_mark_kernel (bit 0 = hull, bit 1 = live, per listed voxel) and
//             occ_dilate_pack_kernel (hull AND 26-neighbourhood dilation of live, straight into the slot's bits).
#include <cmath>

#include "density_tile.cuh"

namespace hrf {

constexpr int kOccThreads = 256;
constexpr int kOccIters = 32;
constexpr int64_t kOccBlockVoxels = (int64_t)kOccThreads * kOccIters;   // voxels per compaction block
constexpr int64_t kOccHeaderBytes = 256;

__device__ __forceinline__ bool occ_hull_at(const uint8_t* __restrict__ hull, int64_t v, int64_t n) {
  return v < n && __ldg(hull + v) != 0;
}

__global__ void __launch_bounds__(kOccThreads) occ_count_kernel(const uint8_t* __restrict__ hull, int64_t n,
                                                                int32_t* __restrict__ block_counts) {
  __shared__ int warp_c[kOccThreads / 32];
  const int64_t base = (int64_t)blockIdx.x * kOccBlockVoxels;
  int c = 0;
  for (int j = 0; j < kOccIters; ++j)
    c += __popc(__ballot_sync(0xffffffffu, occ_hull_at(hull, base + j * kOccThreads + threadIdx.x, n)));
  if ((threadIdx.x & 31) == 0) warp_c[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < kOccThreads / 32; ++w) s += warp_c[w];
    block_counts[blockIdx.x] = s;
  }
}

// One CTA: block_counts -> exclusive offsets in place, total -> *count.
__global__ void __launch_bounds__(1024) occ_block_scan_kernel(int32_t* __restrict__ block_counts, int64_t nb,
                                                              int32_t* __restrict__ count) {
  __shared__ int warp_s[32];
  __shared__ int carry;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int64_t base = 0; base < nb; base += 1024) {
    const int64_t i = base + tid;
    const int c = i < nb ? block_counts[i] : 0;
    int s = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += t;
    }
    if (lane == 31) warp_s[wid] = s;
    __syncthreads();
    if (wid == 0) {
      const int t0 = warp_s[lane];
      int a = t0;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, a, d);
        if (lane >= d) a += t;
      }
      warp_s[lane] = a - t0;
    }
    __syncthreads();
    const int o = carry + warp_s[wid] + s - c;
    if (i < nb) block_counts[i] = o;
    __syncthreads();
    if (tid == 1023) carry = o + c;
    __syncthreads();
  }
  if (tid == 0) *count = carry;
}

__global__ void __launch_bounds__(kOccThreads) occ_write_kernel(const uint8_t* __restrict__ hull, int64_t n,
                                                                const int32_t* __restrict__ block_offsets,
                                                                int32_t* __restrict__ ids) {
  __shared__ int warp_c[kOccThreads / 32];
  const int64_t base = (int64_t)blockIdx.x * kOccBlockVoxels;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int carry = block_offsets[blockIdx.x];
  for (int j = 0; j < kOccIters; ++j) {
    const int64_t v = base + j * kOccThreads + threadIdx.x;
    const bool occ = occ_hull_at(hull, v, n);
    const uint32_t b = __ballot_sync(0xffffffffu, occ);
    if (lane == 0) warp_c[wid] = __popc(b);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < kOccThreads / 32; ++w) {
      before += w < wid ? warp_c[w] : 0;
      total += warp_c[w];
    }
    if (occ) ids[carry + before + __popc(b & ((1u << lane) - 1u))] = (int32_t)v;
    carry += total;
    __syncthreads();
  }
}

// The point of voxel vid: u_x = (h >> 40) 2^-24, u_y = ((h >> 16) & (2^24 - 1)) 2^-24, u_z = (s(h) >> 40) 2^-24 with
// h = s(key ^ vid), and p = __fsub_rn(__fdiv_rn(__fadd_rn((float)x, u_x), (float)G), 0.5f) per axis.
__device__ __forceinline__ void training_point(int32_t vid, int G, uint64_t key, float& px, float& py, float& pz) {
  const int x = vid % G, yz = vid / G, y = yz % G, z = yz / G;
  const uint64_t h = splitmix64(key ^ (uint64_t)(uint32_t)vid), g = splitmix64(h);
  const float ux = __fmul_rn((float)(uint32_t)(h >> 40), 5.9604644775390625e-8f);
  const float uy = __fmul_rn((float)(uint32_t)((h >> 16) & 0xFFFFFFull), 5.9604644775390625e-8f);
  const float uz = __fmul_rn((float)(uint32_t)(g >> 40), 5.9604644775390625e-8f);
  const float Gf = (float)G;
  px = __fsub_rn(__fdiv_rn(__fadd_rn((float)x, ux), Gf), 0.5f);
  py = __fsub_rn(__fdiv_rn(__fadd_rn((float)y, uy), Gf), 0.5f);
  pz = __fsub_rn(__fdiv_rn(__fadd_rn((float)z, uz), Gf), 0.5f);
}

// Update item: one listed voxel = one row, at its hashed point.
struct TrainingArgs : DensityTileArgs {
  static constexpr int kItemsPerTile = kTile;
  uint64_t key;
  float decay;
  float* bound;
  float* points;

  __device__ __forceinline__ void position(int32_t vid, int, Sample& s) const {
    float px, py, pz;
    training_point(vid, G, key, px, py, pz);
    // humanrf.py:175 (positions + 0.5), as load_sample does for a query-form position
    s.x = __fadd_rn(px, 0.5f);
    s.y = __fadd_rn(py, 0.5f);
    s.z = __fadd_rn(pz, 0.5f);
  }
  __device__ __forceinline__ void store(bool valid, int64_t k, int32_t vid, int, float m, const hrf_segment* seg) const {
    if (!valid) return;
    if (seg == nullptr) m = 0.f;
    const float b = bound[k];
    bound[k] = !isfinite(m) ? INFINITY : (isinf(b) ? m : fmaxf(__fmul_rn(decay, b), m));
    if (points != nullptr) {
      float px, py, pz;
      training_point(vid, G, key, px, py, pz);
      points[3 * k] = px, points[3 * k + 1] = py, points[3 * k + 2] = pz;
    }
  }
};

__global__ void __launch_bounds__(kTile, kBakeCtasPerSm) training_occupancy_kernel(const __grid_constant__ TrainingArgs args) {
  density_tile_loop(args);
}

// map[ids[k]] = 1 (hull) | 2 (live), live = the bake's alpha test on the bound; counts[0] += live voxels.
__global__ void __launch_bounds__(kOccThreads) occ_mark_kernel(const int32_t* __restrict__ ids,
                                                               const float* __restrict__ bound, int64_t num_ids,
                                                               float step, float alpha_thre, uint8_t* __restrict__ map,
                                                               unsigned long long* __restrict__ counts) {
  const int64_t k = (int64_t)blockIdx.x * kOccThreads + threadIdx.x;
  bool live = false;
  if (k < num_ids) {
    const float m = __ldg(bound + k);
    // composite.cu visibility_kernel: alpha = 1 - exp(-sigma * step), kept when alpha >= alpha_thre
    live = 1.f - expf(-m * step) >= alpha_thre;
    map[__ldg(ids + k)] = live ? 3 : 1;
  }
  const uint32_t b = __ballot_sync(0xffffffffu, live);
  if (counts != nullptr && (threadIdx.x & 31) == 0 && b != 0u) atomicAdd(counts, (unsigned long long)__popc(b));
}

// slot bit v = (map[v] & 1) AND some voxel of v's 3x3x3 neighbourhood has (map & 2); counts[1] += set bits.
__global__ void __launch_bounds__(kOccThreads) occ_dilate_pack_kernel(const uint8_t* __restrict__ map, int G, int64_t n,
                                                                      uint32_t* __restrict__ bits,
                                                                      unsigned long long* __restrict__ counts) {
  const int64_t v = (int64_t)blockIdx.x * kOccThreads + threadIdx.x;
  bool any = false;
  if (v < n && (__ldg(map + v) & 1)) {
    const int x = (int)(v % G), yz = (int)(v / G), y = yz % G, z = yz / G;
    for (int dz = -1; dz <= 1 && !any; ++dz) {
      const int zz = z + dz;
      if (zz < 0 || zz >= G) continue;
      for (int dy = -1; dy <= 1 && !any; ++dy) {
        const int yy = y + dy;
        if (yy < 0 || yy >= G) continue;
        const uint8_t* row = map + ((int64_t)zz * G + yy) * G;
        for (int dx = -1; dx <= 1; ++dx) {
          const int xx = x + dx;
          if (xx >= 0 && xx < G && (__ldg(row + xx) & 2)) any = true;
        }
      }
    }
  }
  store_occupancy_bits(bits, v, n, any);
  const uint32_t b = __ballot_sync(0xffffffffu, any);
  if (counts != nullptr && (threadIdx.x & 31) == 0 && b != 0u) atomicAdd(counts + 1, (unsigned long long)__popc(b));
}

static int64_t occ_blocks(int G) {
  const int64_t n = (int64_t)G * G * G;
  return (n + kOccBlockVoxels - 1) / kOccBlockVoxels;
}

}  // namespace hrf

using namespace hrf;

extern "C" uint64_t hrf_training_occupancy_key(uint64_t seed, int32_t frame_number, uint64_t counter) {
  return splitmix64(splitmix64(splitmix64(seed) ^ (uint64_t)(uint32_t)frame_number) ^ counter);
}

extern "C" int64_t hrf_training_occupancy_workspace_bytes(int grid_resolution) {
  if (grid_resolution < 1 || grid_resolution > 1024) return 0;
  const int64_t n = (int64_t)grid_resolution * grid_resolution * grid_resolution;
  return kOccHeaderBytes + ((4 * occ_blocks(grid_resolution) + 255) / 256) * 256 + n;
}

extern "C" int hrf_training_occupancy_compact(const uint8_t* hull_u8, int grid_resolution, int32_t* ids,
                                              int32_t* count, void* workspace, void* stream) {
  HRF_REQUIRE(hull_u8 != nullptr && count != nullptr && workspace != nullptr, "null argument");
  HRF_REQUIRE(grid_resolution >= 1 && grid_resolution <= 1024, "grid resolution must be in [1, 1024] (int32 voxel ids)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t n = (int64_t)grid_resolution * grid_resolution * grid_resolution;
  const int64_t nb = occ_blocks(grid_resolution);
  int32_t* block_counts = reinterpret_cast<int32_t*>(reinterpret_cast<char*>(workspace) + kOccHeaderBytes);
  occ_count_kernel<<<(unsigned)nb, kOccThreads, 0, st>>>(hull_u8, n, block_counts);
  HRF_CHECK_LAUNCH();
  occ_block_scan_kernel<<<1, 1024, 0, st>>>(block_counts, nb, count);
  HRF_CHECK_LAUNCH();
  if (ids != nullptr) {
    occ_write_kernel<<<(unsigned)nb, kOccThreads, 0, st>>>(hull_u8, n, block_counts, ids);
    HRF_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int hrf_training_occupancy_update(const hrf_field* f, int32_t frame_number, int grid_resolution,
                                             const int32_t* ids, const int32_t* count, int64_t num_ids, uint64_t seed,
                                             uint64_t counter, float decay, float* bound, float* points,
                                             void* stream) {
  HRF_REQUIRE(f != nullptr && count != nullptr && (num_ids == 0 || (ids != nullptr && bound != nullptr)),
              "null argument");
  HRF_REQUIRE(f->mlp_blob != nullptr && f->segments != nullptr && f->frame_to_segment != nullptr, "field not initialised");
  HRF_REQUIRE(f->table_format == HRF_TABLE_BF16X2, "training occupancy needs a trainable (bf16 table) field");
  HRF_REQUIRE(grid_resolution >= 1 && grid_resolution <= 1024, "grid resolution must be in [1, 1024] (int32 voxel ids)");
  HRF_REQUIRE(num_ids >= 0 && num_ids <= (int64_t)grid_resolution * grid_resolution * grid_resolution,
              "more ids than voxels");
  HRF_REQUIRE(frame_number >= 0 && frame_number < f->lut_size, "frame number outside the model's frame table");
  HRF_REQUIRE(decay > 0.f && decay <= 1.f, "decay must be in (0, 1]");
  if (num_ids == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  TrainingArgs a;
  a.f = *f;
  a.count = count, a.ids = ids;
  a.frame = frame_number, a.G = grid_resolution;
  a.key = hrf_training_occupancy_key(seed, frame_number, counter);
  a.decay = decay;
  a.bound = bound, a.points = points;
  const int smem = density_tile_smem();
  HRF_CUDA(cudaFuncSetAttribute(training_occupancy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  training_occupancy_kernel<<<density_tile_grid(num_ids, TrainingArgs::kItemsPerTile), kTile, smem, st>>>(a);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_training_occupancy_pack(const int32_t* ids, const float* bound, int64_t num_ids, int grid_resolution,
                                           float step, float alpha_thre, uint32_t* slot_bits, int64_t* counts,
                                           void* workspace, void* stream) {
  HRF_REQUIRE(slot_bits != nullptr && workspace != nullptr && (num_ids == 0 || (ids != nullptr && bound != nullptr)),
              "null argument");
  HRF_REQUIRE(grid_resolution >= 1 && grid_resolution <= 1024, "grid resolution must be in [1, 1024] (int32 voxel ids)");
  const int64_t n = (int64_t)grid_resolution * grid_resolution * grid_resolution;
  HRF_REQUIRE(num_ids >= 0 && num_ids <= n, "more ids than voxels");
  HRF_REQUIRE(step > 0.f && alpha_thre > 0.f && alpha_thre < 1.f, "step must be positive and alpha_thre in (0, 1)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* map = reinterpret_cast<uint8_t*>(workspace) + kOccHeaderBytes +
                 ((4 * occ_blocks(grid_resolution) + 255) / 256) * 256;
  auto* cnt = reinterpret_cast<unsigned long long*>(counts);
  if (cnt != nullptr) HRF_CUDA(cudaMemsetAsync(cnt, 0, 2 * sizeof(int64_t), st));
  HRF_CUDA(cudaMemsetAsync(map, 0, (size_t)n, st));
  if (num_ids > 0) {
    occ_mark_kernel<<<(unsigned)((num_ids + kOccThreads - 1) / kOccThreads), kOccThreads, 0, st>>>(
        ids, bound, num_ids, step, alpha_thre, map, cnt);
    HRF_CHECK_LAUNCH();
  }
  occ_dilate_pack_kernel<<<(unsigned)((n + kOccThreads - 1) / kOccThreads), kOccThreads, 0, st>>>(map, grid_resolution, n,
                                                                                                  slot_bits, cnt);
  HRF_CHECK_LAUNCH();
  return 0;
}
