// Data-parallel exchange step of training (SURVEY 8e) as ONE kernel over NVLink peer memory:
//     reduce-scatter of the gradient buckets  +  rank-sharded fused Adam  +  all-gather of the bf16 shadow tables.
// Every rank owns a contiguous 1/world slice of each hash-table tensor.  For its slice it reads the gradient from all
// peers' buckets (P2P loads over NVLink/NVSwitch, summed in rank order), runs Adam on its local fp32 master / moments,
// and stores the refreshed bf16 shadow entry into every peer's shadow table (P2P stores): the forward kernels of all
// ranks read shadows only, so nobody needs the other ranks' fp32 masters during training.  NVLink traffic per step and
// GPU: (world-1)/world x 4 B/param in + (world-1)/world x 2 B/param out -- against 2 x (world-1)/world x 4 B/param each
// way for an fp32 ring all-reduce -- and the optimiser's HBM traffic drops by the factor `world`.  Small tensors
// (vectors, MLPs, camera embeddings) are reduced redundantly on every rank in the same fixed order, so the replicas stay
// bit-identical without a broadcast.
// The reference has no multi-GPU path (SURVEY 2.4); the step this wraps is humanrf/trainer.py:250-253 + run.py:101-104.
#include <algorithm>
#include <cstring>

#include "common.cuh"

namespace hrf {

struct DpPeers {
  const float* grad[HRF_DP_MAX_WORLD];
  __nv_bfloat16* shadow[HRF_DP_MAX_WORLD];
  int world, rank;
};

template <int kWorld>
__global__ void __launch_bounds__(256) dp_reduce_adam_kernel(const DpPeers P, const hrf_dp_tensor* __restrict__ T, int num,
                                                             int64_t block_first, float lr, float b1, float b2, float eps,
                                                             float gscale) {
  int lo = 0, hi = num - 1;
  const int64_t b = block_first + blockIdx.x;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (T[mid].first_block <= b) lo = mid;
    else hi = mid - 1;
  }
  const hrf_dp_tensor t = T[lo];
  if (t.active != nullptr && *t.active == 0) return;
  const int step = *t.step;   // advanced by dp_steps_kernel
  const float bc1 = 1.f - powf(b1, (float)step);
  const float bc2s = sqrtf(1.f - powf(b2, (float)step));
  const float lr1 = lr / bc1;
  const int64_t start = t.shard_begin + (b - t.first_block) * HRF_ADAM_BLOCK_ELEMS;
  const int64_t end = start + HRF_ADAM_BLOCK_ELEMS < t.shard_end ? start + HRF_ADAM_BLOCK_ELEMS : t.shard_end;
  const float omb1 = 1.f - b1, omb2 = 1.f - b2;
  auto upd = [&](float& p, float& m, float& v, float g) { adam_update(p, m, v, g, gscale, b1, b2, omb1, omb2, eps, lr1, bc2s); };
  const bool vec = t.blob_perm == nullptr && ((t.grad_offset | start | (t.shadow_offset < 0 ? 0 : t.shadow_offset)) & 3) == 0 &&
                   ((end - start) & 3) == 0 &&
                   ((reinterpret_cast<uintptr_t>(t.param) | reinterpret_cast<uintptr_t>(t.exp_avg) |
                     reinterpret_cast<uintptr_t>(t.exp_avg_sq)) & 15u) == 0;
  if (vec) {
    for (int64_t i = start + 4 * (int64_t)threadIdx.x; i < end; i += 4 * 256) {
      float4 g[kWorld];
#pragma unroll
      for (int r = 0; r < kWorld; ++r)   // all peers' loads in flight before the first add
        g[r] = __ldcg(reinterpret_cast<const float4*>(P.grad[r] + t.grad_offset + i));
      float4 s = g[0];
#pragma unroll
      for (int r = 1; r < kWorld; ++r) s.x += g[r].x, s.y += g[r].y, s.z += g[r].z, s.w += g[r].w;
      float4 p = *reinterpret_cast<float4*>(t.param + i), m = *reinterpret_cast<float4*>(t.exp_avg + i),
             v = *reinterpret_cast<float4*>(t.exp_avg_sq + i);
      upd(p.x, m.x, v.x, s.x), upd(p.y, m.y, v.y, s.y), upd(p.z, m.z, v.z, s.z), upd(p.w, m.w, v.w, s.w);
      *reinterpret_cast<float4*>(t.param + i) = p;
      *reinterpret_cast<float4*>(t.exp_avg + i) = m;
      *reinterpret_cast<float4*>(t.exp_avg_sq + i) = v;
      const uint2 q = make_uint2(pack_bf16x2(p.x, p.y), pack_bf16x2(p.z, p.w));
      if (t.sharded) {
#pragma unroll
        for (int r = 0; r < kWorld; ++r) *reinterpret_cast<uint2*>(P.shadow[r] + t.shadow_offset + i) = q;
      } else if (t.local_shadow_bf16 != nullptr) {
        *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(t.local_shadow_bf16) + i) = q;
      }
      if (t.vectors_t != nullptr) {
        *reinterpret_cast<float2*>(t.vectors_t + vectors_t_index(i, t.vec_res)) = make_float2(p.x, p.y);
        *reinterpret_cast<float2*>(t.vectors_t + vectors_t_index(i + 2, t.vec_res)) = make_float2(p.z, p.w);
      }
    }
  } else {
    for (int64_t i = start + threadIdx.x; i < end; i += 256) {
      float s = __ldcg(P.grad[0] + t.grad_offset + i);   // rank order, as the float4 path
#pragma unroll
      for (int r = 1; r < kWorld; ++r) s += __ldcg(P.grad[r] + t.grad_offset + i);
      float p = t.param[i], m = t.exp_avg[i], v = t.exp_avg_sq[i];
      upd(p, m, v, s);
      t.param[i] = p, t.exp_avg[i] = m, t.exp_avg_sq[i] = v;
      const __nv_bfloat16 q = __float2bfloat16_rn(p);
      if (t.sharded) {
#pragma unroll
        for (int r = 0; r < kWorld; ++r) P.shadow[r][t.shadow_offset + i] = q;
      } else if (t.local_shadow_bf16 != nullptr) {
        reinterpret_cast<__nv_bfloat16*>(t.local_shadow_bf16)[t.blob_perm != nullptr ? (int64_t)t.blob_perm[i] : i] = q;
      }
      if (t.vectors_t != nullptr) t.vectors_t[vectors_t_index(i, t.vec_res)] = p;
    }
  }
}

__global__ void dp_steps_kernel(const hrf_dp_tensor* __restrict__ T, int num) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= num) return;
  if (T[t].active != nullptr && *T[t].active == 0) return;
  *T[t].step += 1;
}

}  // namespace hrf

using namespace hrf;

extern "C" int hrf_peer_alloc(int64_t bytes, void** ptr_out) {
  HRF_REQUIRE(ptr_out != nullptr && bytes > 0, "bad argument");
  HRF_CUDA(cudaMalloc(ptr_out, (size_t)bytes));
  HRF_CUDA(cudaMemset(*ptr_out, 0, (size_t)bytes));
  return 0;
}
extern "C" int hrf_peer_free(void* ptr) {
  if (ptr != nullptr) HRF_CUDA(cudaFree(ptr));
  return 0;
}
extern "C" int hrf_peer_export(void* ptr, void* handle_out64) {
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  HRF_REQUIRE(ptr != nullptr && handle_out64 != nullptr, "null argument");
  HRF_CUDA(cudaIpcGetMemHandle(reinterpret_cast<cudaIpcMemHandle_t*>(handle_out64), ptr));
  return 0;
}
extern "C" int hrf_peer_open(const void* handle64, void** ptr_out) {
  HRF_REQUIRE(handle64 != nullptr && ptr_out != nullptr, "null argument");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, sizeof(h));
  HRF_CUDA(cudaIpcOpenMemHandle(ptr_out, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}
extern "C" int hrf_peer_close(void* ptr) {
  if (ptr != nullptr) HRF_CUDA(cudaIpcCloseMemHandle(ptr));
  return 0;
}

extern "C" int hrf_dp_reduce_adam(const hrf_dp_peers* peers, const hrf_dp_tensor* tensors, int num_tensors,
                                  int64_t block_first, int64_t block_count, int advance_steps, float lr, float beta1,
                                  float beta2, float eps, float grad_scale, void* stream) {
  const int64_t total_blocks = block_count;
  HRF_REQUIRE(peers != nullptr && tensors != nullptr && num_tensors >= 1, "null argument");
  HRF_REQUIRE(peers->world >= 1 && peers->world <= HRF_DP_MAX_WORLD && peers->rank >= 0 && peers->rank < peers->world,
              "world size must be 1..8 (one NVSwitch domain)");
  HRF_REQUIRE(block_first >= 0 && total_blocks >= 0 && total_blocks < (1ll << 31), "bad block range");
  if (total_blocks == 0 && !advance_steps) return 0;
  DpPeers P;
  for (int r = 0; r < HRF_DP_MAX_WORLD; ++r) {
    P.grad[r] = r < peers->world ? peers->grad[r] : nullptr;
    P.shadow[r] = r < peers->world ? reinterpret_cast<__nv_bfloat16*>(peers->shadow[r]) : nullptr;
    HRF_REQUIRE(r >= peers->world || (P.grad[r] != nullptr && P.shadow[r] != nullptr), "missing peer pointer");
  }
  P.world = peers->world, P.rank = peers->rank;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (advance_steps) {
    dp_steps_kernel<<<(num_tensors + 127) / 128, 128, 0, st>>>(tensors, num_tensors);
    HRF_CHECK_LAUNCH();
  }
  const unsigned grid = (unsigned)total_blocks;
  if (grid == 0) return 0;
  switch (peers->world) {
    case 1: dp_reduce_adam_kernel<1><<<grid, 256, 0, st>>>(P, tensors, num_tensors, block_first, lr, beta1, beta2, eps, grad_scale); break;
    case 2: dp_reduce_adam_kernel<2><<<grid, 256, 0, st>>>(P, tensors, num_tensors, block_first, lr, beta1, beta2, eps, grad_scale); break;
    case 3: dp_reduce_adam_kernel<3><<<grid, 256, 0, st>>>(P, tensors, num_tensors, block_first, lr, beta1, beta2, eps, grad_scale); break;
    case 4: dp_reduce_adam_kernel<4><<<grid, 256, 0, st>>>(P, tensors, num_tensors, block_first, lr, beta1, beta2, eps, grad_scale); break;
    case 5: dp_reduce_adam_kernel<5><<<grid, 256, 0, st>>>(P, tensors, num_tensors, block_first, lr, beta1, beta2, eps, grad_scale); break;
    case 6: dp_reduce_adam_kernel<6><<<grid, 256, 0, st>>>(P, tensors, num_tensors, block_first, lr, beta1, beta2, eps, grad_scale); break;
    case 7: dp_reduce_adam_kernel<7><<<grid, 256, 0, st>>>(P, tensors, num_tensors, block_first, lr, beta1, beta2, eps, grad_scale); break;
    default: dp_reduce_adam_kernel<8><<<grid, 256, 0, st>>>(P, tensors, num_tensors, block_first, lr, beta1, beta2, eps, grad_scale); break;
  }
  HRF_CHECK_LAUNCH();
  return 0;
}
