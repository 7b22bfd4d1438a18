// Offline-preprocessing kernels of the reference that feed the hot path (SURVEY 8f-4):
//   * visual-hull occupancy carving  (actorshq/toolbox/native/occupancy_grid_generation.cu:16-81)
//   * union + population count of occupancy grids for adaptive temporal partitioning
//     (humanrf/adaptive_temporal_partitioning.py:11-26, equations (2)-(4))
#include <cstdlib>

#include "common.cuh"

namespace hrf {

struct CarveArgs {
  const uint8_t* masks;      // [C, H*W]
  const float* proj;         // [C, 16], stored transposed as the reference stores it for GLM (column i = floats 4i..4i+3)
  const uint8_t* landscape;  // [C]
  int threshold, num_cameras, G, width, height;
  uint8_t* grid;             // [G,G,G] (z,y,x)
};

constexpr int kMaxCarveCameras = 160;   // the reference's constant-memory capacity (occupancy_grid_generation.cu:10)

// trunc(a / b) of the correctly rounded quotient: the approximate divide (2 ulp) truncates to the same integer unless the
// quotient sits within ~1e-5 relative of an integer, and only then is the IEEE divide evaluated.
__device__ __forceinline__ int trunc_div(float a, float b) {
  float q = __fdividef(a, b);
  if (!(fabsf(q - rintf(q)) > 1e-5f * fabsf(q))) q = __fdiv_rn(a, b);
  return (int)q;
}

// One thread per voxel, cameras visited in order with the reference's two early exits; the 3 used rows of every
// projection matrix are staged in shared memory once per CTA.  Arithmetic is the canonical IEEE sequence of
// oracle/occupancy_tools.py (glm::mat4 * vec4 with GLM's association, correctly rounded divisions).
__global__ void __launch_bounds__(256) carve_kernel(const __grid_constant__ CarveArgs a) {
  __shared__ float4 s_m[kMaxCarveCameras][3];   // per camera: (m0k, m1k, m2k, m3k) for k = x, y, z
  __shared__ uint8_t s_ls[kMaxCarveCameras];
  for (int i = threadIdx.x; i < a.num_cameras * 3; i += blockDim.x) {
    const int c = i / 3, k = i % 3;
    const float* m = a.proj + 16 * c;
    s_m[c][k] = make_float4(m[k], m[4 + k], m[8 + k], m[12 + k]);
  }
  for (int i = threadIdx.x; i < a.num_cameras; i += blockDim.x) s_ls[i] = a.landscape[i];
  __syncthreads();
  const uint32_t G = (uint32_t)a.G, n = G * G * G;   // G <= 1024 (host check): 32-bit index arithmetic
  const uint8_t* __restrict__ masks = a.masks;
  // grid-stride: the staging above is paid once per CTA, not once per 256 voxels
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
  const uint32_t gx = v % G, gyz = v / G, gy = gyz % G, gz = gyz / G;
  const float inv = (float)(G - 1);
  const float x = __fsub_rn(__fdiv_rn((float)gx, inv), 0.5f), y = __fsub_rn(__fdiv_rn((float)gy, inv), 0.5f),
              z = __fsub_rn(__fdiv_rn((float)gz, inv), 0.5f);
  int covered = 0;
  bool in_hull = false;
  for (int c = 0; c < a.num_cameras; ++c) {
    const bool ls = s_ls[c] != 0;
    const int cw = ls ? a.width : a.height, ch = ls ? a.height : a.width;
    // glm::mat4 * vec4(x,y,z,1), GLM's association: (m0*x + m1*y) + (m2*z + m3*1), contracted as fma(m1,y,m0*x) + fma(m2,z,m3)
    auto comp = [&](int k) {
      const float4 m = s_m[c][k];
      return __fadd_rn(__fmaf_rn(m.y, y, __fmul_rn(m.x, x)), __fmaf_rn(m.z, z, m.w));
    };
    const float px = comp(0), py = comp(1), pz = comp(2);
    const int ix = trunc_div(px, pz), iy = trunc_div(py, pz);   // C truncation, as the reference
    if (ix >= 0 && ix < cw && iy >= 0 && iy < ch) {
      const int ix1 = min(ix + 1, cw - 1), iy1 = min(iy + 1, ch - 1);
      const uint8_t* mk = masks + (size_t)c * a.width * a.height;
      if (__ldg(mk + ix + iy * cw) == 0 && __ldg(mk + ix1 + iy * cw) == 0 && __ldg(mk + ix + iy1 * cw) == 0 &&
          __ldg(mk + ix1 + iy1 * cw) == 0) {
        if (covered + (a.num_cameras - c - 1) < a.threshold) break;
      } else {
        ++covered;
        in_hull = covered >= a.threshold;
        if (in_hull) break;
      }
    }
  }
  a.grid[v] = in_hull ? 255 : 0;
  }
}

// cluster |= (grid == 255), count = popcount(cluster): the cluster is a bit-packed union of occupancy grids.
__global__ void __launch_bounds__(256) union_count_kernel(uint32_t* __restrict__ cluster, const uint8_t* __restrict__ grid,
                                                          int64_t n, unsigned long long* __restrict__ count) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool occ = (i < n) && grid != nullptr && grid[i] == 255;
  const uint32_t b = __ballot_sync(0xffffffffu, occ);
  if ((threadIdx.x & 31) == 0 && i < n) {
    const uint32_t u = cluster[i >> 5] | b;
    cluster[i >> 5] = u;
    if (u) atomicAdd(count, (unsigned long long)__popc(u));
  }
}

}  // namespace hrf

using namespace hrf;

extern "C" int hrf_occupancy_from_masks(const uint8_t* masks, const float* projection_matrices, const uint8_t* landscape_modes,
                                        int num_cameras, int camera_coverage_threshold, int grid_resolution, int width,
                                        int height, uint8_t* occupancy_grid, void* stream) {
  HRF_REQUIRE(masks && projection_matrices && landscape_modes && occupancy_grid, "null argument");
  HRF_REQUIRE(num_cameras > 0 && grid_resolution > 1 && grid_resolution <= 1024 && width > 0 && height > 0, "bad sizes");
  HRF_REQUIRE(num_cameras <= kMaxCarveCameras, "at most 160 cameras (the reference's kMaxNumCameras)");
  CarveArgs a{masks, projection_matrices, landscape_modes, camera_coverage_threshold, num_cameras, grid_resolution, width,
              height, occupancy_grid};
  const int64_t n = (int64_t)grid_resolution * grid_resolution * grid_resolution;
  // 4 strided chunks of 256 voxels per CTA (HRF_CARVE_CHUNKS overrides, scripts/carve_probe.py compares settings):
  // voxels differ a lot in cost (early exits), so many short CTAs balance better than a one-wave persistent grid
  const int64_t want = (n + 255) / 256, floor_ = (int64_t)sm_count() * 8;
  static const int chunks = [] { const char* e = getenv("HRF_CARVE_CHUNKS"); const int v = e ? atoi(e) : 0; return v > 0 ? v : 4; }();
  const int64_t blocks = want <= floor_ ? want : (want / chunks > floor_ ? want / chunks : floor_);
  carve_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_occupancy_union_count(void* cluster_bits, const uint8_t* grid_u8, int64_t num_voxels, int64_t* count_dev,
                                         void* stream) {
  HRF_REQUIRE(cluster_bits && count_dev && num_voxels > 0, "null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  HRF_CUDA(cudaMemsetAsync(count_dev, 0, sizeof(int64_t), st));
  union_count_kernel<<<(unsigned)((num_voxels + 255) / 256), 256, 0, st>>>(reinterpret_cast<uint32_t*>(cluster_bits), grid_u8,
                                                                          num_voxels,
                                                                          reinterpret_cast<unsigned long long*>(count_dev));
  HRF_CHECK_LAUNCH();
  return 0;
}
