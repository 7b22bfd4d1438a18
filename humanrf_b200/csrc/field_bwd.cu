// Fused backward of the HumanRF radiance field for sm_90a (autograd of humanrf.py:158-208).
// Per 128-sample tile (thread r = sample r = operand row r; the CTA is one warpgroup):
//   1. forward recompute of both MLPs from the saved composed features (or a re-encode),
//      keeping every activation tile in shared memory (bf16, K-major core-matrix layout);
//   2. MLP backward on the tensor cores (wgmma).  The SAME shared-memory tiles serve three roles by
//      switching descriptors only:  K-major A operand of the forward / dgrad GEMMs, and
//      MN-major A / B operands of the wgrad GEMMs (contraction over the 128 samples).  The
//      packed forward weight blob is re-used as the MN-major B operand of the dgrad GEMMs.
//      Weight-gradient accumulators (M=64 each, 88 registers a thread) live in registers for the whole
//      persistent CTA and are flushed once with fp32 atomics;
//   3. d(composed features) goes to a level-major [16][N] workspace, next to each sample's position and segment id;
//      a second, high-occupancy kernel (scatter_v6.cu, walking each cell's corners in lane pairs, scatter_pairs.cuh)
//      issues red.global.add.v2.f32 into the fp32 table and vector-row gradients.  scatter_v5.cu, the same walk over
//      a different CTA shape, is its reference in the tests.  (One fused kernel was latency-bound at its low occupancy.)
// The kDirs instantiation also writes d(view directions): dCin columns 0..15 contracted with the SH Jacobian (sh4_vjp).
#include <cstddef>
#include <cstdlib>

#include "field_common.cuh"

namespace hrf {

struct __align__(1024) BwdSmem {
  unsigned char w[kWBlobBytesMax];
  unsigned char feat[kTile * 32 * 2];  // composed features            (A32)
  unsigned char cin[kTile * 48 * 2];   // colour-net input              (A32 / A48)
  unsigned char hs[kTile * 64 * 2];    // sigma hidden, then d(hidden)  (A64)
  unsigned char h1[kTile * 64 * 2];    // colour hidden 1, then its gradient, then dFeat staging
  unsigned char h2[kTile * 64 * 2];    // colour hidden 2, then its gradient, then d(colour input) staging
  unsigned char g3[kTile * 16 * 2];    // d(colour pre-activation)  [128,16]
  unsigned char gs[kTile * 16 * 2];    // colour-net output staging, then d(sigma-net output) [128,16]
  uint64_t bar_w;
};

struct BwdArgs {
  hrf_field f;
  hrf_samples s;
  const hrf_segment_grads* seg_grads;
  const float* d_sigma;
  const float* d_rgb;
  const float* d_geo;    // [N,15] gradient of the geometry features, or NULL
  const uint4* feat_in;  // bf16 [M,32] saved by a forward pass, or NULL (re-encode)
  const int32_t* feat_index;  // row of feat_in per sample, or NULL (identity)
  float* d_mlp;
  float* d_emb;   // camera-embedding gradient [num_cameras, E] or NULL
  float2* dfeat;  // [16][N] float2 workspace: d(composed features)
  float4* pos4;   // [N] normalised (x,y,z,t) of every sample, for the scatter
  uint8_t* seg8;  // [N] segment index (255 = no segment)
  // [N,3] d(view directions), written by the kDirs instantiation only.  Kept last: the offsets of the members above
  // are the kernel-parameter offsets field_backward_kernel was compiled against.
  float* d_dirs;
};

// D[128,Nin] = G[128,Kout] * W[Kout,Nin]  : A = gradient tile (K-major), B = forward blob read MN-major
template <int Nin, int Kout>
__device__ __forceinline__ void issue_dgrad(float* d, uint32_t g_addr, uint32_t w_addr) {
  constexpr uint32_t b_sbo = (uint32_t)(Kout >> 3) * 128u;
#pragma unroll
  for (int k = 0; k < Kout / 16; ++k) {
    const uint64_t bd = make_smem_desc(w_addr + (uint32_t)k * 256u, 128u, b_sbo);
#pragma unroll
    for (int h = 0; h < 2; ++h)
      wgmma_bf16<Nin, 0, 1>(d + h * (Nin / 2), make_smem_desc(g_addr + h * kAHalf + (uint32_t)k * 2u * kAChunk, kAChunk, 128u),
                            bd, k > 0 ? 1u : 0u);
  }
}
// D[64,N] += X^T[64,128] * Y[128,N] : both tiles read MN-major, contraction over the 128 samples
template <int N>
__device__ __forceinline__ void issue_wgrad(float* d, uint32_t x_addr, uint32_t y_addr) {
#pragma unroll
  for (int k = 0; k < kTile / 16; ++k) {
    const uint64_t ad = make_smem_desc(x_addr + (uint32_t)k * 256u, 128u, kAChunk);
    const uint64_t bd = make_smem_desc(y_addr + (uint32_t)k * 256u, 128u, kAChunk);
    wgmma_bf16<N, 1, 1>(d, ad, bd, 1u);
  }
}

// in place: the tile holds relu(h) (bf16, K = 64); replace it by D * (h > 0) (bf16), D[128,64] in fragments
__device__ __forceinline__ void frag_relu_backward64(unsigned char* buf, const float* d) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int q = 0; q < 32; q += 2) {
      const int r = frag_row(h, q), c = frag_col(q);
      uint32_t* p = reinterpret_cast<uint32_t*>(buf + (c >> 3) * kAChunk + a_row_off(r) + (c & 7) * 2);
      const uint32_t a = *p;
      const float lo = (a & 0x7fffu) != 0u && !(a & 0x8000u) ? d[h * 32 + q] : 0.f;
      const float hi = (a & 0x7fff0000u) != 0u && !(a & 0x80000000u) ? d[h * 32 + q + 1] : 0.f;
      *p = pack_bf16x2(lo, hi);
    }
}

__device__ __forceinline__ void red_add2(float* addr, float a, float b) {
  // no return value wanted: the vector RED, not the ATOM the float2 atomicAdd intrinsic compiles to
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// Flush of an M = 64 weight-gradient fragment D (kRegs registers): dst[m * ld + c] += D[m][c] for c < n, the two
// adjacent columns a thread holds as one 8-byte RED when dst is 8-byte aligned.
template <int kRegs>
__device__ __forceinline__ void flush_rows(float* dst, int ld, const float* acc, int n, bool v2ok) {
#pragma unroll
  for (int q = 0; q < kRegs; q += 2) {
    const int m = frag_row(0, q), c = frag_col(q);
    if (c < n) {
      if (v2ok) red_add2(dst + m * ld + c, acc[q], acc[q + 1]);
      else atomicAdd(dst + m * ld + c, acc[q]), atomicAdd(dst + m * ld + c + 1, acc[q + 1]);
    }
  }
}
// Transposed flush of an M = 64, N = 16 fragment: dst[c * 64 + m] += D[m][c].
__device__ __forceinline__ void flush_cols(float* dst, const float* acc) {
#pragma unroll
  for (int q = 0; q < 8; ++q) atomicAdd(dst + frag_col(q) * 64 + frag_row(0, q), acc[q]);
}

// Vector-Jacobian product of sh4 (field_common.cuh): g = sum_j dsh[j] * dSH_j/d(x, y, z), at the fp32 x, y, z sh4 evaluates.
// The map d -> ((d + 1) * 0.5) * 2 - 1 in front of it and the bf16 rounding of the SH values behind it count as the
// identity, as autograd treats them (tcnn's SH input gradient, x2, composed with the reference's (d + 1) * 0.5, x0.5).
__device__ __forceinline__ void sh4_vjp(float dx, float dy, float dz, const float* dsh, float* g) {
  const float x = ((dx + 1.f) * 0.5f) * 2.f - 1.f, y = ((dy + 1.f) * 0.5f) * 2.f - 1.f,
              z = ((dz + 1.f) * 0.5f) * 2.f - 1.f;
  const float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
  constexpr float a = 0.48860251190291987f, b = 1.0925484305920792f, c = 0.94617469575755997f,
                  e = 0.54627421529603959f, f = 0.59004358992664352f, gg = 2.8906114426405538f,
                  h = 0.45704579946446572f, k = 0.3731763325901154f, m = 1.4453057213202769f;
  // SH 1..15 of sh4 and their partial derivatives (SH 0 is a constant)
  g[0] = -a * dsh[3] + b * y * dsh[4] - b * z * dsh[7] + 2.f * e * x * dsh[8] - 6.f * f * xy * dsh[9] +
         gg * yz * dsh[10] + h * (1.f - 5.f * z2) * dsh[13] + 2.f * m * xz * dsh[14] + 3.f * f * (y2 - x2) * dsh[15];
  g[1] = -a * dsh[1] + b * x * dsh[4] - b * z * dsh[5] - 2.f * e * y * dsh[8] + 3.f * f * (y2 - x2) * dsh[9] +
         gg * xz * dsh[10] + h * (1.f - 5.f * z2) * dsh[11] - 2.f * m * yz * dsh[14] + 6.f * f * xy * dsh[15];
  g[2] = a * dsh[2] - b * y * dsh[5] + 2.f * c * z * dsh[6] - b * x * dsh[7] + gg * xy * dsh[10] -
         10.f * h * yz * dsh[11] + k * (15.f * z2 - 3.f) * dsh[12] - 10.f * h * xz * dsh[13] + m * (x2 - y2) * dsh[14];
}

// kLevelUnroll: levels unrolled in the re-encode loop (only taken when the forward's features were not saved).
// kDirs: also write d(view directions) [N,3] to args.d_dirs (hrf_field_backward_mlp_dirs).  The kDirs = false
// instantiations compile to the instruction stream they had before kDirs existed.
template <int kLevelUnroll = 4, bool kDirs = false>
__global__ void __launch_bounds__(kTile, 2) field_backward_kernel(const __grid_constant__ BwdArgs args) {
  extern __shared__ unsigned char smem_raw[];
  BwdSmem& sm = *reinterpret_cast<BwdSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x;
  const hrf_field& f = args.f;
  const uint32_t roff = a_row_off(tid);

  if (tid == 0) {
    mbar_init(&sm.bar_w, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(&sm.bar_w, w_blob_bytes(f.color_in_width));
    tma_load_1d(sm.w, f.mlp_blob, w_blob_bytes(f.color_in_width), &sm.bar_w);
  }
  const uint32_t wbase = smem_u32(sm.w);
  const uint32_t a_feat = smem_u32(sm.feat), a_cin = smem_u32(sm.cin), a_hs = smem_u32(sm.hs),
                 a_h1 = smem_u32(sm.h1), a_h2 = smem_u32(sm.h2), a_g3 = smem_u32(sm.g3), a_gs = smem_u32(sm.gs);
  bool weights_ready = false, have_acc = false;
  // weight-gradient accumulators, M = 64 wgmma fragments (see wgmma_bf16), summed over every tile of the CTA
  float gw1s[16], gw2s[8], gw1c[24], gw2c[32], gw3c[8];   // dW1s [64 out,32 in], dW2s^T [64 in,16 out],
#pragma unroll                                             // dW1c [64 out,K1 in], dW2c [64,64], dW3c^T [64 in,16 out]
  for (int q = 0; q < 32; ++q) {
    if (q < 16) gw1s[q] = 0.f;
    if (q < 8) gw2s[q] = 0.f, gw3c[q] = 0.f;
    if (q < 24) gw1c[q] = 0.f;
    gw2c[q] = 0.f;
  }
  const int K1 = f.color_in_width;

  const int64_t n = live_samples(args.s);
  const int64_t ns = args.s.num_samples;   // row length of the level-major workspace
  const int64_t num_tiles = (n + kTile - 1) / kTile;
  for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int64_t i = tile * kTile + tid;
    const bool valid = i < n;
    const Sample s = load_sample(f, args.s, i, n);
    if (valid) {
      args.pos4[i] = make_float4(s.x, s.y, s.z, s.t);
      args.seg8[i] = s.seg != nullptr ? (uint8_t)(s.seg - f.segments) : (uint8_t)255;
    }
    if (args.feat_in != nullptr) {
      const int64_t row = !(valid && s.seg != nullptr) ? -1 : (args.feat_index != nullptr ? (int64_t)__ldg(args.feat_index + i) : i);
#pragma unroll
      for (int kg = 0; kg < 4; ++kg)
        *reinterpret_cast<uint4*>(sm.feat + kg * kAChunk + roff) =
            row >= 0 ? __ldg(args.feat_in + row * 4 + kg) : make_uint4(0, 0, 0, 0);
    } else {
      encode_to_smem<false, kLevelUnroll>(f, s, sm.feat, tid);
    }
    // Everything else this tile will read from global memory is requested here, before the ten MMA rounds: each round
    // ends in asm statements that clobber memory, so the compiler cannot move a later load above them, and at 8 warps
    // per SM a load issued where its value is needed is a fully exposed round trip.
    const View vw = load_view(f, args.s, i, n);
    float up_sigma = 0.f, up_rgb[3] = {0.f, 0.f, 0.f};
    if (valid) {
      if (args.d_sigma != nullptr) up_sigma = __ldg(args.d_sigma + i);
      if (args.d_rgb != nullptr) up_rgb[0] = __ldg(args.d_rgb + 3 * i), up_rgb[1] = __ldg(args.d_rgb + 3 * i + 1), up_rgb[2] = __ldg(args.d_rgb + 3 * i + 2);
    }
    if (!weights_ready) {
      mbar_wait(&sm.bar_w, 0);
      weights_ready = true;
    }
    float d[64], o[16];
    // ---------------- forward recompute ----------------
    mma_begin();
    mma_layer<64, 32>(d, a_feat, wbase + kWSig1);
    mma_end();
    wgmma_fence_regs<64>(d);
    frag_store_relu64(sm.hs, d);
    mma_begin();
    mma_layer<16, 64>(d, a_hs, wbase + kWSig2);
    mma_end();
    wgmma_fence_regs<16>(d);
    frag_stage<16, 16>(reinterpret_cast<float*>(sm.h1), d);   // h1 is written by the next round only
    __syncthreads();
    stage_read_row<16>(reinterpret_cast<const float*>(sm.h1), o);
    const float h0 = o[0];
    write_color_input(f, sm.cin, roff, vw, o);
    mma_begin();
    if (K1 == 48) mma_layer<64, 48>(d, a_cin, wbase + kWCol1);
    else mma_layer<64, 32>(d, a_cin, wbase + kWCol1);
    mma_end();
    wgmma_fence_regs<64>(d);
    frag_store_relu64(sm.h1, d);
    mma_begin();
    mma_layer<64, 64>(d, a_h1, wbase + w_col2(K1));
    mma_end();
    wgmma_fence_regs<64>(d);
    frag_store_relu64(sm.h2, d);
    mma_begin();
    mma_layer<16, 64>(d, a_h2, wbase + w_col3(K1));
    mma_end();
    wgmma_fence_regs<16>(d);
    frag_stage<16, 4>(reinterpret_cast<float*>(sm.gs), d);    // colour pre-activation 0..2; gs is written much later
    __syncthreads();
    stage_read_row<4>(reinterpret_cast<const float*>(sm.gs), o);

    // ---------------- backward ----------------
    {  // d(colour pre-activation) = d_rgb * rgb * (1 - rgb), cols 3..15 = 0
      float d3[3] = {0.f, 0.f, 0.f};
      if (valid && args.d_rgb != nullptr) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float r = 1.f / (1.f + __expf(-o[c]));
          d3[c] = up_rgb[c] * r * (1.f - r);
        }
      }
      *reinterpret_cast<uint4*>(sm.g3 + 0 * kAChunk + roff) =
          make_uint4(pack_bf16x2(d3[0], d3[1]), pack_bf16x2(d3[2], 0.f), 0u, 0u);
      *reinterpret_cast<uint4*>(sm.g3 + 1 * kAChunk + roff) = make_uint4(0u, 0u, 0u, 0u);
    }
    wgmma_fence_regs<8>(gw3c);
    mma_begin();
    issue_wgrad<16>(gw3c, a_h2, a_g3);                          // dW3c^T += H2^T dO3
    issue_dgrad<64, 16>(d, a_g3, wbase + w_col3(K1));           // dH2 = dO3 W3c
    mma_end();
    wgmma_fence_regs<8>(gw3c);
    wgmma_fence_regs<64>(d);
    frag_relu_backward64(sm.h2, d);
    wgmma_fence_regs<32>(gw2c);
    mma_begin();
    issue_wgrad<64>(gw2c, a_h2, a_h1);                          // dW2c += dH2^T H1
    issue_dgrad<64, 64>(d, a_h2, wbase + w_col2(K1));           // dH1 = dH2 W2c
    mma_end();
    wgmma_fence_regs<32>(gw2c);
    wgmma_fence_regs<64>(d);
    frag_relu_backward64(sm.h1, d);
    wgmma_fence_regs<24>(gw1c);
    mma_begin();
    if (K1 == 48) {
      issue_wgrad<48>(gw1c, a_h1, a_cin);                       // dW1c += dH1^T Cin
      issue_dgrad<48, 64>(d, a_h1, wbase + kWCol1);             // dCin = dH1 W1c
    } else {
      issue_wgrad<32>(gw1c, a_h1, a_cin);
      issue_dgrad<32, 64>(d, a_h1, wbase + kWCol1);
    }
    mma_end();
    wgmma_fence_regs<24>(gw1c);
    wgmma_fence_regs<48>(d);
    {
      // colour-input columns 16..47 (geometry features, camera embedding) staged in h2, free since the last round
      float dc[48];
      if (K1 == 48) frag_stage<48, 32, 16>(reinterpret_cast<float*>(sm.h2), d);
      else frag_stage<32, 32, 16>(reinterpret_cast<float*>(sm.h2), d);
      if constexpr (kDirs) {  // columns 0..15 (SH of the view direction) in h1, whose last reader was the round just ended
        if (K1 == 48) frag_stage<48, 16, 0>(reinterpret_cast<float*>(sm.h1), d);
        else frag_stage<32, 16, 0>(reinterpret_cast<float*>(sm.h1), d);
      }
      __syncthreads();
      if constexpr (kDirs) {
        // d(direction) = dSH^T . dCin[0..15], finished before columns 16..47 are read so that the two sets of 16 and 32
        // values are never live together; 0 for samples without a segment and without a colour gradient
        stage_read_row<16>(reinterpret_cast<const float*>(sm.h1), dc);
        if (valid) {
          float g[3] = {0.f, 0.f, 0.f};
          if (s.seg != nullptr && args.d_rgb != nullptr) sh4_vjp(vw.dx, vw.dy, vw.dz, dc, g);
          args.d_dirs[3 * i] = g[0], args.d_dirs[3 * i + 1] = g[1], args.d_dirs[3 * i + 2] = g[2];
        }
      }
      stage_read_row<32>(reinterpret_cast<const float*>(sm.h2), dc + 16);
      if (args.d_emb != nullptr && vw.cam >= 0) {  // d(camera embedding): colour-input features 31..30+E
        const int E = f.camera_embedding_dim;
#pragma unroll
        for (int e = 0; e < HRF_MAX_CAMERA_EMBEDDING_DIM; ++e)
          if (e < E) atomicAdd(args.d_emb + (size_t)vw.cam * E + e, dc[31 + e]);
      }
      // d(sigma-net output): col 0 from the density (truncated_exp backward, activation.py:21), 1..15 = d geo: what the
      // colour net sends back plus the caller's own gradient of QueryOutput.geometry_features (humanrf.py:185-186)
      if (args.d_geo != nullptr && valid) {
#pragma unroll
        for (int j = 0; j < HRF_GEO_DIM; ++j) dc[16 + j] += __ldg(args.d_geo + i * HRF_GEO_DIM + j);
      }
      float dh0 = 0.f;
      if (valid && args.d_sigma != nullptr)
        dh0 = up_sigma * f.density_scale * __expf(fminf(fmaxf(h0, -15.f), 15.f));
      *reinterpret_cast<uint4*>(sm.gs + 0 * kAChunk + roff) = make_uint4(
          pack_bf16x2(dh0, dc[16]), pack_bf16x2(dc[17], dc[18]), pack_bf16x2(dc[19], dc[20]), pack_bf16x2(dc[21], dc[22]));
      *reinterpret_cast<uint4*>(sm.gs + 1 * kAChunk + roff) = make_uint4(
          pack_bf16x2(dc[23], dc[24]), pack_bf16x2(dc[25], dc[26]), pack_bf16x2(dc[27], dc[28]), pack_bf16x2(dc[29], dc[30]));
    }
    wgmma_fence_regs<8>(gw2s);
    mma_begin();
    issue_wgrad<16>(gw2s, a_hs, a_gs);                          // dW2s^T += Hs^T dOs
    issue_dgrad<64, 16>(d, a_gs, wbase + kWSig2);               // dHs = dOs W2s
    mma_end();
    wgmma_fence_regs<8>(gw2s);
    wgmma_fence_regs<64>(d);
    frag_relu_backward64(sm.hs, d);
    wgmma_fence_regs<16>(gw1s);
    mma_begin();
    issue_wgrad<32>(gw1s, a_hs, a_feat);                        // dW1s += dHs^T feat
    issue_dgrad<32, 64>(d, a_hs, wbase + kWSig1);               // dFeat = dHs W1s
    mma_end();
    wgmma_fence_regs<16>(gw1s);
    wgmma_fence_regs<32>(d);
    have_acc = true;
    {
      // d(composed features) -> global, level-major [16][N] float2 (coalesced here and in the scatter)
      float df[32];
      frag_stage<32, 32>(reinterpret_cast<float*>(sm.h1), d);   // h1 is free until the next tile's recompute
      __syncthreads();
      stage_read_row<32>(reinterpret_cast<const float*>(sm.h1), df);
      if (valid) {
#pragma unroll
        for (int l = 0; l < 16; ++l) args.dfeat[(size_t)l * ns + i] = make_float2(df[2 * l], df[2 * l + 1]);
      }
    }
  }

  if (!weights_ready) mbar_wait(&sm.bar_w, 0);
  // ---------------- flush the weight-gradient accumulators ----------------
  if (have_acc && args.d_mlp != nullptr) {
    // Every CTA adds its 11 264 partial sums into the same 44 KB at the same moment (persistent CTAs finish together):
    // the two adjacent columns a thread holds go out as one 8-byte RED where the destination row is contiguous.
    const bool v2ok = (reinterpret_cast<uintptr_t>(args.d_mlp) & 7u) == 0;
    const int gcol2 = kGCol1 + 64 * K1, gcol3 = gcol2 + 4096;
    flush_rows<16>(args.d_mlp + kGSig1, 32, gw1s, 32, v2ok);
    flush_cols(args.d_mlp + kGSig2, gw2s);
    flush_rows<24>(args.d_mlp + kGCol1, K1, gw1c, K1, v2ok);
    flush_rows<32>(args.d_mlp + gcol2, 64, gw2c, 64, v2ok);
    flush_cols(args.d_mlp + gcol3, gw3c);
  }
}

}  // namespace hrf

using namespace hrf;

static int field_backward_mlp(const hrf_field* f, const hrf_samples* s, const float* d_sigma, const float* d_rgb,
                              const float* d_geo, const void* feat_bf16, const int32_t* feat_index, float* d_mlp,
                              float* d_camera_embeddings, float* d_directions, void* workspace, void* stream) {
  HRF_REQUIRE(f != nullptr && s != nullptr, "null argument");
  HRF_REQUIRE(f->table_format == HRF_TABLE_BF16X2, "an int8 field (compact model) serves inference only: it has no gradients");
  HRF_REQUIRE(f->num_segments < 255, "at most 254 temporal segments");
  if (s->num_samples == 0) return 0;
  HRF_REQUIRE(workspace != nullptr, "hrf_field_backward needs a workspace of 160 bytes per sample");
  HRF_REQUIRE(d_sigma != nullptr || d_rgb != nullptr || d_geo != nullptr, "no upstream gradient given");
  if (s->ray_origins == nullptr) {
    HRF_REQUIRE(s->positions && s->frame_numbers, "query form needs positions and frame numbers");
    HRF_REQUIRE(d_rgb == nullptr || s->directions, "radiance gradients need directions");
  }
  BwdArgs a;
  a.f = *f;
  a.s = *s;
  a.seg_grads = nullptr;
  a.d_sigma = d_sigma;
  a.d_rgb = d_rgb;
  a.d_geo = d_geo;
  a.feat_in = reinterpret_cast<const uint4*>(feat_bf16);
  a.feat_index = feat_bf16 != nullptr ? feat_index : nullptr;
  a.d_mlp = d_mlp;
  a.d_emb = d_camera_embeddings;
  a.dfeat = reinterpret_cast<float2*>(workspace);
  a.pos4 = reinterpret_cast<float4*>(reinterpret_cast<char*>(workspace) + 128 * (size_t)s->num_samples);
  a.seg8 = reinterpret_cast<uint8_t*>(reinterpret_cast<char*>(workspace) + 144 * (size_t)s->num_samples);
  a.d_dirs = d_directions;
  const int64_t tiles = (s->num_samples + kTile - 1) / kTile;
  const int smem = (int)sizeof(BwdSmem) + 1024;
  const int64_t max_ctas = (int64_t)sm_count() * 2;
  const int grid = (int)(tiles < max_ctas ? tiles : max_ctas);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (d_directions != nullptr) {
    HRF_CUDA(cudaFuncSetAttribute(field_backward_kernel<4, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    field_backward_kernel<4, true><<<grid, kTile, smem, st>>>(a);
    HRF_CHECK_LAUNCH();
    return 0;
  }
  // HRF_BWD_UNROLL=1: experiment for round 2 (the forward gained 19 % from the smaller loop; this kernel is 155 KB of SASS)
  static const bool compact = [] { const char* e = getenv("HRF_BWD_UNROLL"); return e && e[0] == '1'; }();
  if (compact) {
    HRF_CUDA(cudaFuncSetAttribute(field_backward_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    field_backward_kernel<1><<<grid, kTile, smem, st>>>(a);
  } else {
    HRF_CUDA(cudaFuncSetAttribute(field_backward_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    field_backward_kernel<4><<<grid, kTile, smem, st>>>(a);
  }
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_field_backward_mlp(const hrf_field* f, const hrf_samples* s, const float* d_sigma, const float* d_rgb,
                                      const float* d_geo, const void* feat_bf16, const int32_t* feat_index, float* d_mlp,
                                      float* d_camera_embeddings, void* workspace, void* stream) {
  return field_backward_mlp(f, s, d_sigma, d_rgb, d_geo, feat_bf16, feat_index, d_mlp, d_camera_embeddings, nullptr,
                            workspace, stream);
}

extern "C" int hrf_field_backward_mlp_dirs(const hrf_field* f, const hrf_samples* s, const float* d_sigma, const float* d_rgb,
                                           const float* d_geo, const void* feat_bf16, const int32_t* feat_index, float* d_mlp,
                                           float* d_camera_embeddings, float* d_directions, void* workspace, void* stream) {
  HRF_REQUIRE(s != nullptr, "null argument");
  HRF_REQUIRE(s->num_samples == 0 || d_directions != nullptr, "null d_directions");
  return field_backward_mlp(f, s, d_sigma, d_rgb, d_geo, feat_bf16, feat_index, d_mlp, d_camera_embeddings, d_directions,
                            workspace, stream);
}

int hrf_launch_scatter_v5(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads, const void* grid_feat_bf16,
                          const int32_t* feat_index, int64_t grid_feat_stride, const void* workspace, int grid_first, int grid_count,
                          cudaStream_t st);   // scatter_v5.cu
int hrf_launch_scatter_v6(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads, const void* grid_feat_bf16,
                          const int32_t* feat_index, int64_t grid_feat_stride, const void* workspace, int grid_first, int grid_count,
                          cudaStream_t st);   // scatter_v6.cu
constexpr int kScatterDefault = 6;   // the faster generation on the train bench on an H100 (DESIGN.md section 3.3)

extern "C" int hrf_field_backward_tables(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads,
                                         const void* grid_feat_bf16, const int32_t* feat_index, int64_t grid_feat_stride,
                                         const void* workspace, int grid_first, int grid_count, void* stream) {
  HRF_REQUIRE(f != nullptr && s != nullptr && seg_grads != nullptr, "null argument");
  HRF_REQUIRE(f->table_format == HRF_TABLE_BF16X2, "an int8 field (compact model) serves inference only: it has no gradients");
  HRF_REQUIRE(grid_first >= 0 && grid_count >= 1 && grid_first + grid_count <= 4, "grids are 0..3 (xyz, xyt, yzt, xzt)");
  // HRF_SCATTER = 6 (the default) | 5, read per call so that the tests can switch it: scatter_v6.cu, or scatter_v5.cu, v6's
  // reference in tests/test_scatter_gpu.py.  Any other value is an error: a stale setting must not time one generation
  // under another's name.
  const char* gen_env = getenv("HRF_SCATTER");
  const int gen = gen_env != nullptr ? atoi(gen_env) : kScatterDefault;
  HRF_REQUIRE(gen == 6 || gen == 5, "HRF_SCATTER must be 6 (the default) or 5");
  if (s->num_samples == 0) return 0;
  HRF_REQUIRE(workspace != nullptr, "needs the workspace hrf_field_backward_mlp filled");
  if (gen == 5)
    return hrf_launch_scatter_v5(f, s, seg_grads, grid_feat_bf16, feat_index, grid_feat_stride, workspace, grid_first, grid_count,
                                 reinterpret_cast<cudaStream_t>(stream));
  return hrf_launch_scatter_v6(f, s, seg_grads, grid_feat_bf16, feat_index, grid_feat_stride, workspace, grid_first, grid_count,
                               reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int hrf_field_backward(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads,
                                  const float* d_sigma, const float* d_rgb, const float* d_geo, const void* feat_bf16,
                                  const void* grid_feat_bf16, const int32_t* feat_index, int64_t grid_feat_stride,
                                  float* d_mlp, float* d_camera_embeddings, void* workspace, void* stream) {
  HRF_REQUIRE(f != nullptr && seg_grads != nullptr, "null argument");
  HRF_REQUIRE(f->table_format == HRF_TABLE_BF16X2, "an int8 field (compact model) serves inference only: it has no gradients");
  if (int rc = hrf_field_backward_mlp(f, s, d_sigma, d_rgb, d_geo, feat_bf16, feat_index, d_mlp, d_camera_embeddings, workspace,
                                      stream))
    return rc;
  return hrf_field_backward_tables(f, s, seg_grads, grid_feat_bf16, feat_index, grid_feat_stride, workspace, 0, 4, stream);
}
