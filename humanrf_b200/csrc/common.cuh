// Shared device helpers for the sm_90a kernels: PTX wrappers for mbarrier, TMA bulk copies,
// wgmma (warpgroup MMA from shared-memory descriptors) and small math utilities.  No CUTLASS dependency.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "../../include/humanrf_b200.h"

namespace hrf {

// ---------------------------------------------------------------------------------------
// host-side error plumbing
// ---------------------------------------------------------------------------------------
void set_error(const std::string& msg);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);
#define HRF_CUDA(expr)                                                           \
  do {                                                                           \
    cudaError_t _e = (expr);                                                     \
    if (_e != cudaSuccess) return hrf::cuda_fail(_e, #expr, __FILE__, __LINE__); \
  } while (0)
#define HRF_CHECK_LAUNCH() HRF_CUDA(cudaGetLastError())
#define HRF_REQUIRE(cond, msg)                                                      \
  do {                                                                              \
    if (!(cond)) {                                                                  \
      hrf::set_error(std::string(msg) + " [" #cond "] at " __FILE__ ":" + std::to_string(__LINE__)); \
      return -1;                                                                    \
    }                                                                               \
  } while (0)

int sm_count();

// ---------------------------------------------------------------------------------------
// small device utilities
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// SplitMix64: the finaliser of x + golden gamma (the counter-based hash of the error map's draws, the mesh sampler and
// the training occupancy's points).
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// The bit layout of an occupancy ring slot (hrf_occgrid_add): voxel i is bit i & 31 of word i >> 5, and the bits past
// the last voxel of the last word are 0.  Called by every lane of a full warp whose lane l holds voxel i0 + l, i0 a
// multiple of 32; occ is the voxel's occupancy (false for i >= n).
__device__ __forceinline__ void store_occupancy_bits(uint32_t* __restrict__ bits, int64_t i, int64_t n, bool occ) {
  const uint32_t b = __ballot_sync(0xffffffffu, occ);
  if ((threadIdx.x & 31) == 0 && i < n) bits[i >> 5] = b;
}

// One Adam update of one element (torch.optim.Adam, no weight decay), with every rounding spelled out so that all
// optimiser kernels and both of their paths (float4 and scalar) produce the same bits: ptxas may otherwise contract
// the plain multiplies and adds into FMAs differently at each call site.  Replicated tensors rely on this -- every
// data-parallel rank updates them itself, with no broadcast.
//   g' = g * gscale ; m' = fma(b1, m, (1-b1) g') ; v' = fma(b2, v, ((1-b2) g') g')
//   p' = fma(-lr1, m' / (sqrt(v') / bc2s + eps), p)        lr1 = lr / (1 - b1^k), bc2s = sqrt(1 - b2^k)
// (torch: denom = sqrt(v)/sqrt(bias_correction2) + eps ; p -= lr/bias_correction1 * m/denom.)  tests/adam_oracle.py
// bounds each of these roundings.
__device__ __forceinline__ void adam_update(float& p, float& m, float& v, float g, float gscale, float b1, float b2,
                                            float one_minus_b1, float one_minus_b2, float eps, float lr1, float bc2s) {
  g = __fmul_rn(g, gscale);
  m = __fmaf_rn(b1, m, __fmul_rn(one_minus_b1, g));
  v = __fmaf_rn(b2, v, __fmul_rn(__fmul_rn(one_minus_b2, g), g));
  p = __fmaf_rn(-lr1, __fdiv_rn(m, __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2s), eps)), p);
}

// element i of a `vectors` tensor [4, VR, 32] inside its transposed copy [4, 16, VR, 2] (hrf_segment.vectors_t)
__device__ __forceinline__ int64_t vectors_t_index(int64_t i, int vr) {
  const int c = (int)(i & 31);
  const int64_t row = (i >> 5) % vr, axis = (i >> 5) / vr;
  return ((axis * 16 + (c >> 1)) * vr + row) * 2 + (c & 1);
}

// ---------------------------------------------------------------------------------------
// mbarrier + proxies
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  // make generic-proxy st.shared visible to the async proxy (wgmma / TMA reads)
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
// TMA 1-D bulk copy global -> shared (UBLKCP), completion on an mbarrier.
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ---------------------------------------------------------------------------------------
// wgmma: warpgroup MMA with both operands in shared memory and fp32 accumulators in registers.
// Every thread of the warpgroup (the 128 threads of a CTA here) issues every call.
// ---------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, no swizzle: start>>4 | LBO>>4 <<16 | SBO>>4 <<32.  LBO is the byte stride between
// core matrices (8 rows x 16 bytes) along K, SBO the stride along M/N, for K-major and MN-major operands alike.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;
}

template <int N>
struct Wgmma;
template <>
struct Wgmma<16> {
  template <int kTransA, int kTransB>
  static __device__ __forceinline__ void run(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(kTransA), "n"(kTransB)
        : "memory");
  }
};
template <>
struct Wgmma<32> {
  template <int kTransA, int kTransB>
  static __device__ __forceinline__ void run(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(kTransA), "n"(kTransB)
        : "memory");
  }
};
template <>
struct Wgmma<48> {
  template <int kTransA, int kTransB>
  static __device__ __forceinline__ void run(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1, %27, %28;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(kTransA), "n"(kTransB)
        : "memory");
  }
};
template <>
struct Wgmma<64> {
  template <int kTransA, int kTransB>
  static __device__ __forceinline__ void run(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(kTransA), "n"(kTransB)
        : "memory");
  }
};

// D[64,N] (+)= A[64,16] * B[N,16]^T, bf16 x bf16 -> f32.  kTransA / kTransB: that operand is MN-major.  d holds this
// thread's N/2 accumulators: register 4j + 2h + e is row 16*warp + lane/4 + 8h, column 8j + 2*(lane%4) + e.
template <int N, int kTransA = 0, int kTransB = 0>
__device__ __forceinline__ void wgmma_bf16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  Wgmma<N>::template run<kTransA, kTransB>(d, adesc, bdesc, accumulate);
}

// TF32 wgmma, k8: both operands K-major (tf32 has no transposed form), a core matrix is 8 rows x 4 tf32, so one call
// spans two core matrices along K.  The MMA reads only the tf32 bits of each operand: operands rounded beforehand with
// tf32_rna lose nothing more.
template <int N>
struct WgmmaTf32;
template <>
struct WgmmaTf32<64> {
  static __device__ __forceinline__ void run(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
  }
};
template <>
struct WgmmaTf32<128> {
  static __device__ __forceinline__ void run(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
  }
};

// D[64,N] (+)= A[64,8] * B[N,8]^T, tf32 x tf32 -> f32; accumulator register layout as wgmma_bf16's.
template <int N>
__device__ __forceinline__ void wgmma_tf32(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  WgmmaTf32<N>::run(d, adesc, bdesc, accumulate);
}
// fp32 -> tf32 (10 mantissa bits), round to nearest with ties away from zero; the 13 low bits of the result are zero.
__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Keeps every access to accumulator registers on its side of a wgmma fence / wait: the asynchronous MMA writes them
// after the issuing asm statement has returned.
template <int kRegs>
__device__ __forceinline__ void wgmma_fence_regs(float* d) {
#pragma unroll
  for (int i = 0; i < kRegs; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

}  // namespace hrf
