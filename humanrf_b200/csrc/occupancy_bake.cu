// The trained density field evaluated on grids, for inference.  Two entry points share one persistent tile loop
// (density_tile_loop: one warpgroup per CTA, 128-row tiles, positions generated in the kernel -> encode -> sigma MLP
// (wgmma) -> density), each with its own item shape:
//
// Learned occupancy grid (include/humanrf_b200.h, hrf_bake_occupancy).  Three launches, no host read:
//   hull_compact_kernel   : ids of the hull's occupied voxels -> device list + device count; zeroes `live` / max_sigma
//                           outside the hull
//   occupancy_bake_kernel : tiles of 16 voxels x 8 sub-samples; per-voxel max (3 xor shuffles over the voxel's 8
//                           consecutive lanes) -> max_sigma, live byte
//   dilate_and_kernel     : out = hull AND (26-neighbourhood dilation of live by one voxel), {0,255}
//
// Density lattice (hrf_density_lattice), the input of marching cubes.  Two launches, no host read:
//   lattice_compact_kernel: ids of the (G+1)^3 lattice vertices that are a corner of an occupied mask voxel (every
//                           vertex without a mask) -> device list + device count; zeroes sigma at the other vertices
//   density_lattice_kernel: tiles of 128 vertices, one sample each -> sigma
//
// The density of every sample is bit for bit what hrf_field_forward (mode 0, query form) returns for its position
// (density_tile.cuh).
#include "density_tile.cuh"

namespace hrf {

constexpr int64_t kBakeHeaderBytes = 256;       // device count, then the id list

__global__ void __launch_bounds__(256) hull_compact_kernel(const uint8_t* __restrict__ hull, uint32_t n,
                                                           int32_t* __restrict__ count, int32_t* __restrict__ ids,
                                                           uint8_t* __restrict__ live, float* __restrict__ max_sigma) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = v < n;
  const bool occ = in && hull[v] != 0;
  const uint32_t b = __ballot_sync(0xffffffffu, occ);
  const int lane = threadIdx.x & 31;
  int base = 0;
  if (lane == 0 && b != 0u) base = atomicAdd(count, __popc(b));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (occ) {
    ids[base + __popc(b & ((1u << lane) - 1u))] = (int32_t)v;
  } else if (in) {   // hull voxels are written by the bake kernel
    live[v] = 0;
    if (max_sigma != nullptr) max_sigma[v] = 0.f;
  }
}

// Sub-sample position along one axis: the cell-centred convention of the texture lookup the sampler emulates (voxel i
// covers [i/G, (i+1)/G) of p + 0.5), sub-samples at 1/4 and 3/4 of the cell.
__device__ __forceinline__ float bake_coord(int i, int half, float G) {
  return __fsub_rn(__fdiv_rn((float)i + 0.25f + 0.5f * (float)half, G), 0.5f);
}

// Bake item: one hull voxel = 8 consecutive rows (sub-samples).
struct BakeArgs : DensityTileArgs {
  static constexpr int kItemsPerTile = kTile / 8;
  float step, alpha_thre;
  uint8_t* live;
  float* max_sigma;

  __device__ __forceinline__ void position(int32_t vid, int sub, Sample& s) const {
    const int x = vid % G, yz = vid / G, y = yz % G, z = yz / G;
    const float Gf = (float)G;
    // humanrf.py:175 (positions + 0.5), as load_sample does for a query-form position
    s.x = __fadd_rn(bake_coord(x, sub & 1, Gf), 0.5f);
    s.y = __fadd_rn(bake_coord(y, (sub >> 1) & 1, Gf), 0.5f);
    s.z = __fadd_rn(bake_coord(z, sub >> 2, Gf), 0.5f);
  }
  __device__ __forceinline__ void store(bool valid, int64_t, int32_t vid, int sub, float m, const hrf_segment* seg) const {
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
    if (valid && sub == 0) {
      if (seg == nullptr) m = 0.f;
      if (max_sigma != nullptr) max_sigma[vid] = m;
      // composite.cu visibility_kernel: alpha = 1 - exp(-sigma * step), kept when alpha >= alpha_thre
      live[vid] = (1.f - expf(-m * step) >= alpha_thre) ? 1 : 0;
    }
  }
};

// Lattice item: one vertex of the (G+1)^3 lattice = one row, at the corner (i/G - 0.5) of the grid's voxels.
struct LatticeArgs : DensityTileArgs {
  static constexpr int kItemsPerTile = kTile;
  float* sigma;

  __device__ __forceinline__ void position(int32_t vid, int, Sample& s) const {
    const int Gp = G + 1;
    const int x = vid % Gp, yz = vid / Gp, y = yz % Gp, z = yz / Gp;
    const float Gf = (float)G;
    s.x = __fadd_rn(__fsub_rn(__fdiv_rn((float)x, Gf), 0.5f), 0.5f);
    s.y = __fadd_rn(__fsub_rn(__fdiv_rn((float)y, Gf), 0.5f), 0.5f);
    s.z = __fadd_rn(__fsub_rn(__fdiv_rn((float)z, Gf), 0.5f), 0.5f);
  }
  __device__ __forceinline__ void store(bool valid, int64_t, int32_t vid, int, float m, const hrf_segment*) const {
    if (valid) sigma[vid] = m;
  }
};

__global__ void __launch_bounds__(kTile, kBakeCtasPerSm) occupancy_bake_kernel(const __grid_constant__ BakeArgs args) {
  density_tile_loop(args);
}

__global__ void __launch_bounds__(kTile, kBakeCtasPerSm) density_lattice_kernel(const __grid_constant__ LatticeArgs args) {
  density_tile_loop(args);
}

// The same two for a field with HRF_TABLE_INT8X2 tables.
__global__ void __launch_bounds__(kTile, kBakeCtasPerSm) occupancy_bake_i8_kernel(const __grid_constant__ BakeArgs args) {
  density_tile_loop<BakeArgs, TabInt8x2>(args);
}

__global__ void __launch_bounds__(kTile, kBakeCtasPerSm) density_lattice_i8_kernel(const __grid_constant__ LatticeArgs args) {
  density_tile_loop<LatticeArgs, TabInt8x2>(args);
}

// out = hull AND (any live voxel in the 3x3x3 neighbourhood), one thread per voxel; `live` is 0 outside the hull.
__global__ void __launch_bounds__(256) dilate_and_kernel(const uint8_t* __restrict__ hull, const uint8_t* __restrict__ live,
                                                         int G, uint8_t* __restrict__ out) {
  const uint32_t n = (uint32_t)G * (uint32_t)G * (uint32_t)G;
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  bool any = false;
  if (hull[v] != 0) {
    const int x = (int)(v % (uint32_t)G), yz = (int)(v / (uint32_t)G), y = yz % G, z = yz / G;
    for (int dz = -1; dz <= 1 && !any; ++dz) {
      const int zz = z + dz;
      if (zz < 0 || zz >= G) continue;
      for (int dy = -1; dy <= 1 && !any; ++dy) {
        const int yy = y + dy;
        if (yy < 0 || yy >= G) continue;
        const uint8_t* row = live + ((uint32_t)zz * (uint32_t)G + (uint32_t)yy) * (uint32_t)G;
        for (int dx = -1; dx <= 1; ++dx) {
          const int xx = x + dx;
          if (xx >= 0 && xx < G && __ldg(row + xx) != 0) any = true;
        }
      }
    }
  }
  out[v] = any ? 255 : 0;
}

// Lattice vertex v = (x, y, z) of the (G+1)^3 lattice is evaluated when it is a corner of an occupied voxel of the
// G^3 mask (voxels x-1..x, y-1..y, z-1..z inside the grid), or always when there is no mask.
__global__ void __launch_bounds__(256) lattice_compact_kernel(const uint8_t* __restrict__ mask, int G, uint32_t n,
                                                              int32_t* __restrict__ count, int32_t* __restrict__ ids,
                                                              float* __restrict__ sigma) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = v < n;
  bool occ = in && mask == nullptr;
  if (in && mask != nullptr) {
    const uint32_t Gp = (uint32_t)G + 1u, Gu = (uint32_t)G;
    const int x = (int)(v % Gp), yz = (int)(v / Gp), y = yz % (int)Gp, z = yz / (int)Gp;
    for (int zz = z - 1; zz <= z && !occ; ++zz) {
      if (zz < 0 || zz >= G) continue;
      for (int yy = y - 1; yy <= y && !occ; ++yy) {
        if (yy < 0 || yy >= G) continue;
        const uint8_t* row = mask + ((uint32_t)zz * Gu + (uint32_t)yy) * Gu;
        for (int xx = x - 1; xx <= x; ++xx)
          if (xx >= 0 && xx < G && __ldg(row + xx) != 0) occ = true;
      }
    }
  }
  const uint32_t b = __ballot_sync(0xffffffffu, occ);
  const int lane = threadIdx.x & 31;
  int base = 0;
  if (lane == 0 && b != 0u) base = atomicAdd(count, __popc(b));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (occ) ids[base + __popc(b & ((1u << lane) - 1u))] = (int32_t)v;
  else if (in) sigma[v] = 0.f;
}

}  // namespace hrf

using namespace hrf;

extern "C" int64_t hrf_bake_occupancy_workspace_bytes(int grid_resolution) {
  if (grid_resolution < 1 || grid_resolution > 1024) return 0;
  const int64_t n = (int64_t)grid_resolution * grid_resolution * grid_resolution;
  return kBakeHeaderBytes + ((4 * n + 255) / 256) * 256 + n;
}

extern "C" int hrf_bake_occupancy(const hrf_field* f, int32_t frame_number, const uint8_t* hull_u8, int grid_resolution,
                                  float step, float alpha_thre, uint8_t* out_u8, float* max_sigma, void* workspace,
                                  void* stream) {
  HRF_REQUIRE(f != nullptr && hull_u8 != nullptr && out_u8 != nullptr && workspace != nullptr, "null argument");
  HRF_REQUIRE(f->mlp_blob != nullptr && f->segments != nullptr && f->frame_to_segment != nullptr, "field not initialised");
  HRF_REQUIRE(f->table_format == HRF_TABLE_BF16X2 || f->table_format == HRF_TABLE_INT8X2, "unknown table format");
  HRF_REQUIRE(grid_resolution >= 1 && grid_resolution <= 1024, "grid resolution must be in [1, 1024] (int32 voxel ids)");
  HRF_REQUIRE(frame_number >= 0 && frame_number < f->lut_size, "frame number outside the model's frame table");
  HRF_REQUIRE(step > 0.f && alpha_thre > 0.f && alpha_thre < 1.f, "step must be positive and alpha_thre in (0, 1)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t n = (int64_t)grid_resolution * grid_resolution * grid_resolution;
  char* ws = reinterpret_cast<char*>(workspace);
  int32_t* count = reinterpret_cast<int32_t*>(ws);
  int32_t* ids = reinterpret_cast<int32_t*>(ws + kBakeHeaderBytes);
  uint8_t* live = reinterpret_cast<uint8_t*>(ws + kBakeHeaderBytes + ((4 * n + 255) / 256) * 256);
  HRF_CUDA(cudaMemsetAsync(count, 0, sizeof(int32_t), st));
  const unsigned blocks = (unsigned)((n + 255) / 256);
  hull_compact_kernel<<<blocks, 256, 0, st>>>(hull_u8, (uint32_t)n, count, ids, live, max_sigma);
  HRF_CHECK_LAUNCH();

  BakeArgs a;
  a.f = *f;
  a.count = count, a.ids = ids;
  a.frame = frame_number, a.G = grid_resolution;
  a.step = step, a.alpha_thre = alpha_thre;
  a.live = live, a.max_sigma = max_sigma;
  const int smem = density_tile_smem();
  auto* kernel = f->table_format == HRF_TABLE_INT8X2 ? occupancy_bake_i8_kernel : occupancy_bake_kernel;
  HRF_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  kernel<<<density_tile_grid(n, BakeArgs::kItemsPerTile), kTile, smem, st>>>(a);
  HRF_CHECK_LAUNCH();

  dilate_and_kernel<<<blocks, 256, 0, st>>>(hull_u8, live, grid_resolution, out_u8);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int64_t hrf_density_lattice_workspace_bytes(int grid_resolution) {
  if (grid_resolution < 1 || grid_resolution > 1024) return 0;
  const int64_t gp = (int64_t)grid_resolution + 1;
  return kBakeHeaderBytes + 4 * gp * gp * gp;
}

extern "C" int hrf_density_lattice(const hrf_field* f, int32_t frame_number, const uint8_t* mask_u8, int grid_resolution,
                                   float* sigma, void* workspace, void* stream) {
  HRF_REQUIRE(f != nullptr && sigma != nullptr && workspace != nullptr, "null argument");
  HRF_REQUIRE(f->mlp_blob != nullptr && f->segments != nullptr && f->frame_to_segment != nullptr, "field not initialised");
  HRF_REQUIRE(f->table_format == HRF_TABLE_BF16X2 || f->table_format == HRF_TABLE_INT8X2, "unknown table format");
  HRF_REQUIRE(grid_resolution >= 1 && grid_resolution <= 1024,
              "grid resolution must be in [1, 1024] ((G+1)^3 int32 vertex ids)");
  HRF_REQUIRE(frame_number >= 0 && frame_number < f->lut_size, "frame number outside the model's frame table");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t gp = (int64_t)grid_resolution + 1;
  const int64_t n = gp * gp * gp;
  char* ws = reinterpret_cast<char*>(workspace);
  int32_t* count = reinterpret_cast<int32_t*>(ws);
  int32_t* ids = reinterpret_cast<int32_t*>(ws + kBakeHeaderBytes);
  HRF_CUDA(cudaMemsetAsync(count, 0, sizeof(int32_t), st));
  lattice_compact_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(mask_u8, grid_resolution, (uint32_t)n, count, ids,
                                                                     sigma);
  HRF_CHECK_LAUNCH();

  LatticeArgs a;
  a.f = *f;
  a.count = count, a.ids = ids;
  a.frame = frame_number, a.G = grid_resolution;
  a.sigma = sigma;
  const int smem = density_tile_smem();
  auto* kernel = f->table_format == HRF_TABLE_INT8X2 ? density_lattice_i8_kernel : density_lattice_kernel;
  HRF_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  kernel<<<density_tile_grid(n, LatticeArgs::kItemsPerTile), kTile, smem, st>>>(a);
  HRF_CHECK_LAUNCH();
  return 0;
}
