// Ray generation, AABB slab test, occupancy march and sample generation for sm_90a.
// Replaces actorshq/dataset/native/{occupancy_grid.cu, ray_sampler.cu}.  Design choices:
//   * occupancy volumes are bit-packed (G^3/8 bytes: 2 MB at G=256, L2-resident) and the
//     texture unit's 1.8 fixed-point trilinear ">0" test is emulated exactly in integer math;
//   * one WARP per ray marches 32 steps at a time (ballot + ffs) instead of one divergent
//     thread per ray; sample counts are produced in the same pass, compaction is a device-side
//     scan, so the whole call needs a single host read of two counters (the reference needs
//     >= 5 implicit syncs and a D2H->CPU->H2D bounce, ray_sampler.cu:254-266).
// Arithmetic is the canonical IEEE sequence documented in oracle/sampler.py (bit-exact with it).
#include <vector>

#include "common.cuh"

struct hrf_occgrid {
  uint64_t res;
  int buffer_size;
  int next;
  std::vector<uint32_t*> slots;  // device, res^3/32 words each
};

namespace hrf {

__global__ void pack_bits_kernel(const uint8_t* __restrict__ g, uint32_t* __restrict__ bits, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  store_occupancy_bits(bits, i, n, (i < n) && (g[i] != 0));
}

// Emulates tex3D<float>(clamp, linear, normalised coords, normalised-float uint8) > 0.
__device__ __forceinline__ int fix8(float p, float G) {
  const float xb = __fsub_rn(__fmul_rn(p, G), 0.5f);
  return (int)floorf(__fadd_rn(__fmul_rn(xb, 256.f), 0.5f));
}
// Per-corner weight of the hardware filter (fitted on a texture unit, see oracle/sampler.py; tests/test_texture_probe_gpu.py
// checks it against the texture unit of the GPU it runs on):
// W = (((wx*wz + 128) >> 8) * wy + 128) >> 8 in 1/256 units; the sample is "> 0" iff an occupied
// corner has W >= 1.
__device__ __forceinline__ bool occ_lookup(const uint32_t* __restrict__ bits, int G, float x, float y, float z) {
  const float Gf = (float)G;
  const int qx = fix8(x, Gf), qy = fix8(y, Gf), qz = fix8(z, Gf);
  const int ix = qx >> 8, iy = qy >> 8, iz = qz >> 8;
  const int ax = qx & 255, ay = qy & 255, az = qz & 255;
  const int x0 = min(max(ix, 0), G - 1), x1 = min(max(ix + 1, 0), G - 1);
  const int y0 = min(max(iy, 0), G - 1), y1 = min(max(iy + 1, 0), G - 1);
  const int z0 = min(max(iz, 0), G - 1), z1 = min(max(iz + 1, 0), G - 1);
  bool occ = false;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int wx = (c & 1) ? ax : 256 - ax, wy = (c & 2) ? ay : 256 - ay, wz = (c & 4) ? az : 256 - az;
    const int w = ((((wx * wz + 128) >> 8) * wy) + 128) >> 8;
    if (w > 0) {
      const uint32_t bit = ((uint32_t)((c & 4) ? z1 : z0) * (uint32_t)G + (uint32_t)((c & 2) ? y1 : y0)) * (uint32_t)G +
                           (uint32_t)((c & 1) ? x1 : x0);
      occ |= (__ldg(bits + (bit >> 5)) >> (bit & 31u)) & 1u;
    }
  }
  return occ;
}
__global__ void occ_lookup_kernel(const uint32_t* bits, int G, const float* p, int64_t n, uint8_t* out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = occ_lookup(bits, G, p[3 * i], p[3 * i + 1], p[3 * i + 2]) ? 1 : 0;
}

struct Ray {
  float ox, oy, oz, dx, dy, dz;
};
__device__ __forceinline__ bool occ_at(const uint32_t* bits, int G, const Ray& r, float t) {
  // ray_sampler.cu:39 : origin + direction * t + 0.5f
  return occ_lookup(bits, G, __fadd_rn(__fmaf_rn(r.dx, t, r.ox), 0.5f), __fadd_rn(__fmaf_rn(r.dy, t, r.oy), 0.5f),
                    __fadd_rn(__fmaf_rn(r.dz, t, r.oz), 0.5f));
}
__device__ __forceinline__ float gmin(float a, float b) { return (b < a) ? b : a; }  // glm::min
__device__ __forceinline__ float gmax(float a, float b) { return (a < b) ? b : a; }  // glm::max

// number of candidate samples of a ray: int((tmax - tmin) / step) with torch's reciprocal-multiply
__device__ __forceinline__ int candidate_count(float tmin, float tmax, float inv_step) {
  const int c = (int)__fmul_rn(__fsub_rn(tmax, tmin), inv_step);
  return c > 0 ? c : 0;
}

struct RaysArgs {
  hrf_sampler_params p;
  const int64_t* ray_indices;
  int64_t num_rays;
  float inv_step;
  uint8_t* ray_mask;
  float* dirs_full;     // [R,3]
  float* minmax_full;   // [R,2]
  int32_t* counts_full; // [R]
};

// compute_minmax_kernel (ray_sampler.cu:80-147) + per-ray kept-sample count; one warp per ray.
__global__ void __launch_bounds__(256) ray_minmax_kernel(const __grid_constant__ RaysArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (ray >= a.num_rays) return;
  const hrf_sampler_params& p = a.p;
  const int64_t idx = __ldg(a.ray_indices + ray);
  const int64_t npix = (int64_t)p.image_width * p.image_height;
  const int img = (int)(idx / npix);
  int w = p.image_width, h = p.image_height;
  if (!__ldg(p.landscape_modes + img)) {
    const int t = w;
    w = h;
    h = t;
  }
  const float px = (float)(idx % w) + 0.5f;
  const float py = (float)((idx / w) % h) + 0.5f;
  const float* T = p.inverse_krs + 9 * img;  // T[i*3+k] = GLM column i, component k
  float v[3];
#pragma unroll
  for (int k = 0; k < 3; ++k)
    v[k] = __fmaf_rn(__ldg(T + 6 + k), 1.0f, __fmaf_rn(__ldg(T + 3 + k), py, __fmul_rn(__ldg(T + k), px)));
  const float dot = __fmaf_rn(v[2], v[2], __fmaf_rn(v[1], v[1], __fmul_rn(v[0], v[0])));
  const float inv = __fdiv_rn(1.0f, __fsqrt_rn(dot));
  Ray r;
  r.dx = __fmul_rn(v[0], inv), r.dy = __fmul_rn(v[1], inv), r.dz = __fmul_rn(v[2], inv);
  r.ox = __ldg(p.camera_origins + 3 * img), r.oy = __ldg(p.camera_origins + 3 * img + 1),
  r.oz = __ldg(p.camera_origins + 3 * img + 2);
  // compute_aabb_minmax (ray_sampler.cu:11-26)
  float bb[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) bb[k] = __ldg(p.aabb + k);
  const float ix = __fdiv_rn(1.0f, r.dx), iy = __fdiv_rn(1.0f, r.dy), iz = __fdiv_rn(1.0f, r.dz);
  const float t0x = __fmul_rn(__fsub_rn(bb[0], r.ox), ix), t1x = __fmul_rn(__fsub_rn(bb[3], r.ox), ix);
  const float t0y = __fmul_rn(__fsub_rn(bb[1], r.oy), iy), t1y = __fmul_rn(__fsub_rn(bb[4], r.oy), iy);
  const float t0z = __fmul_rn(__fsub_rn(bb[2], r.oz), iz), t1z = __fmul_rn(__fsub_rn(bb[5], r.oz), iz);
  float tmin = gmax(gmin(t0x, t1x), gmax(gmin(t0y, t1y), gmin(t0z, t1z)));
  float tmax = gmin(gmax(t0x, t1x), gmin(gmax(t0y, t1y), gmax(t0z, t1z)));

  const uint32_t* bits = nullptr;
  const int G = p.grid_resolution;
  if (p.occupancy) {
    bits = reinterpret_cast<const uint32_t*>(__ldg(p.grid_handles + img));
    // compute_occupancy_minmax (ray_sampler.cu:28-78), 32 march steps per warp iteration
    const float step = __fdiv_rn(0.5f, (float)G);
    const float tend = tmax;
    {  // forward march: first t_k with (t_k >= tend) or occupied
      float t = tmin;
      while (true) {
        float mine = t;
        float cur = t;
#pragma unroll 1
        for (int k = 0; k < 32; ++k) {
          if (k == lane) mine = cur;
          cur = __fadd_rn(cur, step);
        }
        const bool stop = !(mine < tend) || occ_at(bits, G, r, mine);
        const uint32_t m = __ballot_sync(0xffffffffu, stop);
        if (m) {
          tmin = __shfl_sync(0xffffffffu, mine, __ffs(m) - 1);
          break;
        }
        t = cur;
      }
    }
    if (tmin < tend) {  // 5-step bisection refine (ray_sampler.cu:47-64); all lanes redundantly
      float ref = __fmul_rn(-step, 0.5f);
      for (int i = 0; i < 5; ++i) {
        tmin = __fadd_rn(tmin, ref);
        const float mag = __fmul_rn(fabsf(ref), 0.5f);
        ref = occ_at(bits, G, r, tmin) ? -mag : mag;
      }
    }
    {  // backward march: first t_k with (t_k <= tmin) or occupied
      float t = tend;
      while (true) {
        float mine = t;
        float cur = t;
#pragma unroll 1
        for (int k = 0; k < 32; ++k) {
          if (k == lane) mine = cur;
          cur = __fsub_rn(cur, step);
        }
        const bool stop = !(mine > tmin) || occ_at(bits, G, r, mine);
        const uint32_t m = __ballot_sync(0xffffffffu, stop);
        if (m) {
          tmax = __shfl_sync(0xffffffffu, mine, __ffs(m) - 1);
          break;
        }
        t = cur;
      }
    }
  }
  bool keep = tmin < tmax;
  if (keep && p.filter_light_bloom) {  // ray_sampler.cu:254-257
    if (p.light_mask_rays != nullptr) keep = !__ldg(p.light_mask_rays + ray);
    else if (p.light_mask != nullptr) keep = !__ldg(p.light_mask + idx);
  }

  // kept-sample count: candidates t_k = fma(k, step, tmin), occupancy filtered (ray_sampler.cu:175-189)
  int count = 0;
  if (keep && p.want_samples) {
    const int cand = candidate_count(tmin, tmax, a.inv_step);
    if (p.occupancy) {
      for (int k0 = 0; k0 < cand; k0 += 32) {
        const int k = k0 + lane;
        const bool o = (k < cand) && occ_at(bits, G, r, __fmaf_rn((float)k, p.step, tmin));
        count += __popc(__ballot_sync(0xffffffffu, o));
      }
    } else {
      count = cand;
    }
  }
  if (lane == 0) {
    a.dirs_full[3 * ray] = r.dx, a.dirs_full[3 * ray + 1] = r.dy, a.dirs_full[3 * ray + 2] = r.dz;
    a.minmax_full[2 * ray] = tmin, a.minmax_full[2 * ray + 1] = tmax;
    a.ray_mask[ray] = keep ? 1 : 0;
    a.counts_full[ray] = count;
  }
}

// Single-CTA dual exclusive scan over the R candidate rays: kept-ray positions and sample offsets.  The sample sums
// run in 64 bits, so counters[1] is the exact total even past 2^31 - 1; the per-ray offsets stay int32 (the caller
// refuses totals they cannot hold before any sample is written).
__global__ void __launch_bounds__(1024) ray_scan_kernel(const uint8_t* __restrict__ mask,
                                                        const int32_t* __restrict__ counts, int64_t n,
                                                        int32_t* __restrict__ ray_pos, int32_t* __restrict__ sample_pos,
                                                        int64_t* __restrict__ counters) {
  __shared__ int warp_m[32];
  __shared__ long long warp_c[32];
  __shared__ long long carry_m, carry_c;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) carry_m = 0, carry_c = 0;
  __syncthreads();
  for (int64_t base = 0; base < n; base += 1024) {
    const int64_t i = base + tid;
    const int m = (i < n) ? (int)mask[i] : 0;
    const long long c = (i < n && m) ? counts[i] : 0;
    int sm = m;
    long long sc = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int tm = __shfl_up_sync(0xffffffffu, sm, d);
      const long long tc = __shfl_up_sync(0xffffffffu, sc, d);
      if (lane >= d) sm += tm, sc += tc;
    }
    if (lane == 31) warp_m[wid] = sm, warp_c[wid] = sc;
    __syncthreads();
    if (wid == 0) {
      const int tm0 = warp_m[lane];
      const long long tc0 = warp_c[lane];
      int am = tm0;
      long long ac = tc0;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int tm = __shfl_up_sync(0xffffffffu, am, d);
        const long long tc = __shfl_up_sync(0xffffffffu, ac, d);
        if (lane >= d) am += tm, ac += tc;
      }
      warp_m[lane] = am - tm0;  // exclusive warp offsets
      warp_c[lane] = ac - tc0;
    }
    __syncthreads();
    const long long om = carry_m + warp_m[wid], oc = carry_c + warp_c[wid];
    if (i < n) {
      ray_pos[i] = (int32_t)(om + sm - m);
      sample_pos[i] = (int32_t)(oc + sc - c);
    }
    __syncthreads();
    if (tid == 1023) carry_m = om + sm, carry_c = oc + sc;
    __syncthreads();
  }
  if (tid == 0) {
    counters[0] = carry_m;
    counters[1] = carry_c;
  }
}

struct ScatterArgs {
  hrf_sampler_params p;
  const int64_t* ray_indices;
  int64_t num_rays;
  const uint8_t* ray_mask;
  const float* dirs_full;
  const float* minmax_full;
  const int32_t* ray_pos;
  const int32_t* sample_pos;
  const int64_t* counters;
  float *ray_origins, *ray_directions, *rgba, *minmaxes;
  int32_t *frame_numbers, *camera_numbers, *sample_offsets;
  int64_t* kept_ray_indices;
};

// Compaction + per-ray gathers (ray_sampler.cu:258-266).
__global__ void ray_scatter_kernel(const __grid_constant__ ScatterArgs a) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r == 0) a.sample_offsets[a.counters[0]] = (int32_t)a.counters[1];
  if (r >= a.num_rays || !a.ray_mask[r]) return;
  const int j = a.ray_pos[r];
  const int64_t idx = a.ray_indices[r];
  const int img = (int)(idx / ((int64_t)a.p.image_width * a.p.image_height));
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    a.ray_origins[3 * j + k] = a.p.camera_origins[3 * img + k];
    a.ray_directions[3 * j + k] = a.dirs_full[3 * r + k];
  }
  a.minmaxes[2 * j] = a.minmax_full[2 * r], a.minmaxes[2 * j + 1] = a.minmax_full[2 * r + 1];
  a.frame_numbers[j] = a.p.frame_numbers[img];
  a.camera_numbers[j] = a.p.camera_numbers[img];
  a.kept_ray_indices[j] = idx;
  a.sample_offsets[j] = a.sample_pos[r];
  if (a.rgba != nullptr && a.p.rgba_pool != nullptr) {
    const uchar4 c = *reinterpret_cast<const uchar4*>(a.p.rgba_pool + 4 * idx);
    // (rgba / 255.0f): true division in float32 (ray_sampler.cu:262)
    *reinterpret_cast<float4*>(a.rgba + 4 * j) = make_float4(__fdiv_rn((float)c.x, 255.f), __fdiv_rn((float)c.y, 255.f),
                                                              __fdiv_rn((float)c.z, 255.f), __fdiv_rn((float)c.w, 255.f));
  }
}

struct SamplesArgs {
  hrf_sampler_params p;
  int64_t num_kept;
  float inv_step;
  const int64_t* kept_ray_indices;
  const float *ray_origins, *ray_directions, *minmaxes;
  const int32_t* sample_offsets;
  float* distances;
  int32_t* rel;
};

// compute_sample_distances_kernel (ray_sampler.cu:149-194) + final compaction (:322-323); warp per ray.
__global__ void __launch_bounds__(256) ray_samples_kernel(const __grid_constant__ SamplesArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t j = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (j >= a.num_kept) return;
  const float tmin = a.minmaxes[2 * j], tmax = a.minmaxes[2 * j + 1];
  const int cand = candidate_count(tmin, tmax, a.inv_step);
  int base = a.sample_offsets[j];
  Ray r;
  r.ox = a.ray_origins[3 * j], r.oy = a.ray_origins[3 * j + 1], r.oz = a.ray_origins[3 * j + 2];
  r.dx = a.ray_directions[3 * j], r.dy = a.ray_directions[3 * j + 1], r.dz = a.ray_directions[3 * j + 2];
  const uint32_t* bits = nullptr;
  if (a.p.occupancy) {
    const int img = (int)(a.kept_ray_indices[j] / ((int64_t)a.p.image_width * a.p.image_height));
    bits = reinterpret_cast<const uint32_t*>(__ldg(a.p.grid_handles + img));
  }
  for (int k0 = 0; k0 < cand; k0 += 32) {
    const int k = k0 + lane;
    const float t = __fmaf_rn((float)k, a.p.step, tmin);
    const bool o = (k < cand) && (!a.p.occupancy || occ_at(bits, a.p.grid_resolution, r, t));
    const uint32_t m = __ballot_sync(0xffffffffu, o);
    if (o) {
      const int pos = base + __popc(m & ((1u << lane) - 1u));
      a.distances[pos] = t;
      a.rel[pos] = (int32_t)j;
    }
    base += __popc(m);
  }
}

}  // namespace hrf

using namespace hrf;

extern "C" int hrf_occgrid_create(uint64_t grid_resolution, int buffer_size, hrf_occgrid** out) {
  HRF_REQUIRE(out != nullptr && grid_resolution > 0 && buffer_size > 0, "bad occupancy grid arguments");
  HRF_REQUIRE(grid_resolution <= 1024, "grid resolution above 1024 not supported (32-bit voxel index)");
  auto* g = new hrf_occgrid();
  g->res = grid_resolution;
  g->buffer_size = buffer_size;
  g->next = 0;
  const size_t words = (size_t)((grid_resolution * grid_resolution * grid_resolution + 31) / 32);
  for (int i = 0; i < buffer_size; ++i) {
    uint32_t* d = nullptr;
    cudaError_t e = cudaMalloc(&d, words * sizeof(uint32_t));
    if (e == cudaSuccess) e = cudaMemset(d, 0, words * sizeof(uint32_t));
    if (e != cudaSuccess) {
      for (auto* q : g->slots) cudaFree(q);
      delete g;
      return cuda_fail(e, "cudaMalloc(occupancy slot)", __FILE__, __LINE__);
    }
    g->slots.push_back(d);
  }
  *out = g;
  return 0;
}

extern "C" int hrf_occgrid_destroy(hrf_occgrid* g) {
  if (g == nullptr) return 0;
  for (auto* q : g->slots) cudaFree(q);
  delete g;
  return 0;
}

extern "C" int hrf_occgrid_add(hrf_occgrid* g, const uint8_t* grid_u8, uint64_t r0, uint64_t r1, uint64_t r2,
                               void* stream, int64_t* handle_out) {
  HRF_REQUIRE(g != nullptr && grid_u8 != nullptr && handle_out != nullptr, "null argument");
  // occupancy_grid.cu:60-63
  HRF_REQUIRE(r0 == g->res && r1 == g->res && r2 == g->res, "Provided grid doesn't have the correct resolution!");
  const int used = g->next;
  g->next = (g->next + 1) % g->buffer_size;  // occupancy_grid.cu:65-66 ring policy
  const int64_t n = (int64_t)(g->res * g->res * g->res);
  pack_bits_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(grid_u8,
                                                                                                      g->slots[used], n);
  HRF_CHECK_LAUNCH();
  *handle_out = (int64_t)reinterpret_cast<uintptr_t>(g->slots[used]);
  return 0;
}

extern "C" int hrf_occgrid_lookup(int64_t handle, int grid_resolution, const float* points_xyz, int64_t n, uint8_t* out,
                                  void* stream) {
  if (n == 0) return 0;
  occ_lookup_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint32_t*>((uintptr_t)handle), grid_resolution, points_xyz, n, out);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int64_t hrf_sampler_workspace_bytes(int64_t num_rays) { return 32 * (num_rays + 64) + 1024; }

extern "C" int hrf_sampler_rays(const hrf_sampler_params* p, const int64_t* all_ray_indices, int64_t num_rays,
                                uint8_t* ray_mask, float* ray_origins, float* ray_directions, float* rgba,
                                int32_t* frame_numbers, int32_t* camera_numbers, float* minmaxes,
                                int64_t* kept_ray_indices, int32_t* sample_offsets, int64_t* counters, void* workspace,
                                int64_t workspace_bytes, void* stream) {
  HRF_REQUIRE(p != nullptr && counters != nullptr, "null argument");
  HRF_REQUIRE(workspace_bytes >= hrf_sampler_workspace_bytes(num_rays), "sampler workspace too small");
  HRF_REQUIRE(p->step > 0.f, "raymarching step must be positive");
  HRF_REQUIRE(!p->occupancy || p->grid_resolution > 0, "occupancy mode needs a grid resolution");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (num_rays == 0) {
    HRF_CUDA(cudaMemsetAsync(counters, 0, 2 * sizeof(int64_t), st));
    HRF_CUDA(cudaMemsetAsync(sample_offsets, 0, sizeof(int32_t), st));
    return 0;
  }
  char* ws = reinterpret_cast<char*>(workspace);
  const int64_t R = num_rays;
  RaysArgs a;
  a.p = *p;
  a.ray_indices = all_ray_indices;
  a.num_rays = R;
  a.inv_step = 1.0f / p->step;
  a.ray_mask = ray_mask;
  a.dirs_full = reinterpret_cast<float*>(ws);
  a.minmax_full = reinterpret_cast<float*>(ws + 12 * R);
  a.counts_full = reinterpret_cast<int32_t*>(ws + 20 * R);
  int32_t* ray_pos = reinterpret_cast<int32_t*>(ws + 24 * R);
  int32_t* sample_pos = reinterpret_cast<int32_t*>(ws + 28 * R);
  ray_minmax_kernel<<<(unsigned)((R * 32 + 255) / 256), 256, 0, st>>>(a);
  HRF_CHECK_LAUNCH();
  ray_scan_kernel<<<1, 1024, 0, st>>>(ray_mask, a.counts_full, R, ray_pos, sample_pos, counters);
  HRF_CHECK_LAUNCH();
  ScatterArgs s;
  s.p = *p;
  s.ray_indices = all_ray_indices;
  s.num_rays = R;
  s.ray_mask = ray_mask;
  s.dirs_full = a.dirs_full;
  s.minmax_full = a.minmax_full;
  s.ray_pos = ray_pos;
  s.sample_pos = sample_pos;
  s.counters = counters;
  s.ray_origins = ray_origins, s.ray_directions = ray_directions, s.rgba = rgba, s.minmaxes = minmaxes;
  s.frame_numbers = frame_numbers, s.camera_numbers = camera_numbers, s.sample_offsets = sample_offsets;
  s.kept_ray_indices = kept_ray_indices;
  ray_scatter_kernel<<<(unsigned)((R + 255) / 256), 256, 0, st>>>(s);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_sampler_samples(const hrf_sampler_params* p, int64_t num_kept_rays, const int64_t* kept_ray_indices,
                                   const float* ray_origins, const float* ray_directions, const float* minmaxes,
                                   const int32_t* sample_offsets, float* distances, int32_t* relative_ray_indices,
                                   void* stream) {
  HRF_REQUIRE(p != nullptr, "null argument");
  if (num_kept_rays == 0) return 0;
  SamplesArgs a;
  a.p = *p;
  a.num_kept = num_kept_rays;
  a.inv_step = 1.0f / p->step;
  a.kept_ray_indices = kept_ray_indices;
  a.ray_origins = ray_origins, a.ray_directions = ray_directions, a.minmaxes = minmaxes;
  a.sample_offsets = sample_offsets;
  a.distances = distances;
  a.rel = relative_ray_indices;
  ray_samples_kernel<<<(unsigned)((num_kept_rays * 32 + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  HRF_CHECK_LAUNCH();
  return 0;
}
