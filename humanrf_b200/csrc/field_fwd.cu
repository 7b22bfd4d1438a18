// Fused forward of the HumanRF radiance field for sm_90a:
//   sample load -> 4 hash grids x 16 levels gather -> vector composition -> sigma MLP (wgmma)
//   -> truncated_exp density -> SH + colour MLP (wgmma) -> sigmoid radiance.
// One persistent CTA of 128 threads (one warpgroup) owns one 128-sample tile at a time; thread r owns sample r
// (= row r of every MMA operand), so the whole encode -> MLP chain stays in registers / shared memory.
// Reference semantics: humanrf/scene_representation/humanrf.py:158-208,
// decomposition4d.py:124-135, native/tensor_composition.cu:9-55.
#include <stddef.h>
#include <stdlib.h>

#include "field_mlp.cuh"

namespace hrf {


__device__ __forceinline__ float warp_sum_fwd(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

// kFromFeat: the composed features come from an earlier pass (args.feat_in, optionally through args.feat_index) and the
// encode is skipped: the MLP half of the kernel alone (render pass of the survivors of prune_samples).
// kComposite: the per-ray compositing of humanrf/volume_rendering.py:123-145 (nerfacc render_weight_from_density +
// accumulate_along_rays + background blend) runs as the epilogue of the tile: sigma / rgb never go to HBM.  Samples are
// sorted by ray, so a tile holds a run of whole rays plus at most one ray cut by its first border and one cut by its
// last: whole rays are finished here; the (at most two) cut segments leave a 5-float partial
// (optical depth, transmittance-weighted colour and weight relative to the segment start) that composite_fixup_kernel
// chains in tile order.  Segmented warp-shuffle scans keyed by the ray index; warps are joined through 3 words of smem.
// kDepth (kComposite only): one more scan, of w * t_mid with t_mid = (t + (t + step)) / 2, gives each ray the unnormalised
// expected distance sum w * t_mid (args.depth; slot 5 of a cut segment's partial).  The other scans are unchanged, so
// colour and weights sum are bit-identical to those of the kernel without it.
// Fmt: the table entry format (field_common.cuh); the bf16 kernels are field_forward_kernel, the int8 ones
// field_forward_i8_kernel.
template <bool kSimt, bool kSaveGrid, int kLevelUnroll, bool kFromFeat, bool kComposite, bool kDepth, class Fmt>
__device__ __forceinline__ void field_forward_body(const FieldArgs& args) {
  static_assert(kComposite || !kDepth, "the depth scan is part of the compositing epilogue");
  extern __shared__ unsigned char smem_raw[];
  FwdSmem& sm = *reinterpret_cast<FwdSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  const int tid = threadIdx.x;
  const hrf_field& f = args.f;

  // ---- one-time CTA setup: barrier, weights via TMA bulk copy -------------------
  if (tid == 0) {
    mbar_init(&sm.bar_w, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(&sm.bar_w, w_blob_bytes(f.color_in_width));
    tma_load_1d(sm.w, f.mlp_blob, w_blob_bytes(f.color_in_width), &sm.bar_w);
  }
  bool weights_ready = false;

  const int64_t n = live_samples(args.s);
  const int64_t n_stride = args.s.num_samples;   // row length of the level-major [64][N] output
  const int64_t num_tiles = (n + kTile - 1) / kTile;
  // Early-stop schedule (density-only pass of prune_samples, volume_rendering.py:66-84).  Work items are
  // (chunk k, ray r) = samples [off[r]+128k, off[r]+128(k+1)) of ray r, pulled from a global counter in the order
  // c = k*R + r, i.e. all rays' first chunks, then all second chunks, ...  Every finished item adds its optical depth
  // sum(sigma*step) to ray_depth[r].  render_visibility drops every sample whose transmittance
  // T = exp(-depth before it) is below 1e-4 whatever its own density, so an item whose ray has already
  // accumulated depth >= stop_depth (exp(-9.4) = 8.3e-5 < 1e-4, a margin over float rounding) is provably dead:
  // its densities are never evaluated and are reported as 0.  The depth seen at pull time only contains earlier
  // chunks of the same ray, so the kept set is exactly the reference's.
  const bool es = args.es.ray_offsets != nullptr;
  int64_t tile = blockIdx.x;
  while (true) {
    int64_t i;
    bool valid;
    int ray = -1;
    if (!es) {
      if (tile >= num_tiles) break;
      i = tile * kTile + tid;
      valid = i < n;
      tile += gridDim.x;
    } else {
      __syncthreads();  // everybody is done with the previous item's shared fields
      if (tid == 0) {
        const unsigned long long R = (unsigned long long)args.es.num_rays;
        const unsigned long long total = (unsigned long long)__ldg(args.es.max_chunks) * R;
        sm.item_start = -1;
        while (true) {
          const unsigned long long c = atomicAdd(args.es.counter, 1ull);
          if (c >= total) break;
          const int r = (int)(c % R);
          const int64_t k = (int64_t)(c / R);
          const int64_t b = __ldg(args.es.ray_offsets + r), e = __ldg(args.es.ray_offsets + r + 1);
          if (b + k * kTile >= e) continue;  // this ray has no chunk k
          sm.item_start = b + k * kTile;
          sm.item_end = e;
          sm.item_ray = r;
          sm.item_skip = __ldcg(args.es.ray_depth + r) >= args.es.stop_depth;
          break;
        }
      }
      __syncthreads();
      if (sm.item_start < 0) break;
      i = sm.item_start + tid;
      valid = i < sm.item_end;
      ray = sm.item_ray;
      if (sm.item_skip) {
        if (valid && args.sigma != nullptr) args.sigma[i] = 0.f;
        continue;
      }
    }
    if constexpr (kFromFeat) {
      const uint32_t ro = a_row_off(tid);
      const int64_t row = !valid ? -1 : (args.feat_index != nullptr ? (int64_t)__ldg(args.feat_index + i) : i);
#pragma unroll
      for (int kg = 0; kg < 4; ++kg)
        *reinterpret_cast<uint4*>(sm.a + kg * kAChunk + ro) = row >= 0 ? __ldg(args.feat_in + row * 4 + kg) : make_uint4(0, 0, 0, 0);
    } else {
      const Sample s = load_sample(f, args.s, valid ? i : n, n);
      encode_to_smem<kSaveGrid, kLevelUnroll, Fmt>(f, s, sm.a, tid, (kSaveGrid && valid && s.seg != nullptr) ? args.egrid : nullptr, i, n_stride);
    }
    if (!kFromFeat && args.feat != nullptr && valid) {
      const uint32_t ro = a_row_off(tid);
#pragma unroll
      for (int kg = 0; kg < 4; ++kg) args.feat[i * 4 + kg] = *reinterpret_cast<const uint4*>(sm.a + kg * kAChunk + ro);
    }
    if (!weights_ready) {
      mbar_wait(&sm.bar_w, 0);
      weights_ready = true;
    }

    // ---- sigma net: 32 -> 64 (ReLU) -> 16 ------------------------------------------------
    run_hidden<kSimt, 32>(sm, kWSig1);
    float o[16];
    run_layer16<kSimt, 64>(sm, kWSig2, o);
    // humanrf.py:184 : density = truncated_exp(h[...,0]) * density_scale  (exp in fp32)
    const float sigma = __expf(o[0]) * f.density_scale;
    if (es) {  // publish this item's optical depth
      const float part = warp_sum_fwd(valid ? sigma * args.es.step : 0.f);
      if ((tid & 31) == 0 && part > 0.f) atomicAdd(args.es.ray_depth + ray, part);
    }
    if (valid) {
      if (args.sigma != nullptr) args.sigma[i] = sigma;
      if (args.geo != nullptr) {
        uint4* gp = reinterpret_cast<uint4*>(args.geo + i * 8);
        gp[0] = make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]),
                           pack_bf16x2(o[6], o[7]));
        gp[1] = make_uint4(pack_bf16x2(o[8], o[9]), pack_bf16x2(o[10], o[11]), pack_bf16x2(o[12], o[13]),
                           pack_bf16x2(o[14], o[15]));
      }
    }
    if (args.mode == 0) continue;

    // ---- colour net: [SH16 | geo15 | 1.0] -> 64 (ReLU) -> 64 (ReLU) -> 16 -> sigmoid[:3] ----
    write_color_input(f, sm.a, a_row_off(tid), load_view(f, args.s, valid ? i : n, n), o);
    if (f.color_in_width == 48) run_hidden<kSimt, 48>(sm, kWCol1);
    else run_hidden<kSimt, 32>(sm, kWCol1);
    run_hidden<kSimt, 64>(sm, w_col2(f.color_in_width));
    run_layer16<kSimt, 64>(sm, w_col3(f.color_in_width), o);
    const float c0 = 1.f / (1.f + __expf(-o[0])), c1 = 1.f / (1.f + __expf(-o[1])), c2 = 1.f / (1.f + __expf(-o[2]));
    if (valid && args.rgb != nullptr) {
      float* rp = args.rgb + 3 * i;
      rp[0] = c0, rp[1] = c1, rp[2] = c2;
    }
    if constexpr (kComposite) {
      // The activation tile is free (the last MMA that read it has committed): its first bytes join the four warps.
      constexpr int kTail = kDepth ? 6 : 5;                 // scanned quantities per warp
      int* x_first = reinterpret_cast<int*>(sm.a);          // [4] ray of lane 0
      int* x_last = x_first + 4;                            // [4] ray of lane 31
      float* x_tail = reinterpret_cast<float*>(x_first + 8);  // [4][kTail] inclusive sums of the warp's last ray at lane 31
      const int lane = tid & 31, warp = tid >> 5;
      const int ray = valid ? (int)__ldg(args.s.ray_indices + i) : -1;
      float sdt = 0.f;
      float tmid = 0.f;
      if (valid) {
        const float t = __ldg(args.s.sample_distances + i);
        sdt = sigma * __fsub_rn(__fadd_rn(t, args.comp.step), t);   // sigmas * (t_ends - t_starts), volume_rendering.py:124-129
        if constexpr (kDepth) tmid = __fmul_rn(0.5f, __fadd_rn(t, __fadd_rn(t, args.comp.step)));   // (t_starts + t_ends) / 2
      }
      auto seg_scan = [&](float v) {   // inclusive sum over the lanes of this warp that carry the same ray
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const float u = __shfl_up_sync(0xffffffffu, v, d);
          const int ru = __shfl_up_sync(0xffffffffu, ray, d);
          if (lane >= d && ru == ray) v += u;
        }
        return v;
      };
      auto carry_in = [&](int k) {   // what the earlier warps of the tile hold for this thread's ray
        float c = 0.f;
        for (int w = warp - 1; w >= 0; --w) {
          if (x_last[w] != ray) break;
          c += x_tail[w * kTail + k];
          if (x_first[w] != ray) break;
        }
        return c;
      };
      float depth = seg_scan(sdt);
      __syncthreads();   // every thread is done with the tile's operands
      if (lane == 0) x_first[warp] = ray;
      if (lane == 31) x_last[warp] = ray, x_tail[warp * kTail] = depth;
      __syncthreads();
      // exclusive depth = the lane before's inclusive one if it holds the same ray (not depth - sdt: inf - inf = NaN)
      const float c_in = carry_in(0);
      const float prev = __shfl_up_sync(0xffffffffu, depth, 1);
      const int ray_prev = __shfl_up_sync(0xffffffffu, ray, 1);
      const float excl = (lane > 0 && ray_prev == ray) ? prev + c_in : c_in;
      depth += c_in;
      const float wgt = valid ? __expf(-excl) * (1.f - __expf(-sdt)) : 0.f;
      float a0 = seg_scan(wgt * c0), a1 = seg_scan(wgt * c1), a2 = seg_scan(wgt * c2), a3 = seg_scan(wgt);
      float a4 = 0.f;
      if constexpr (kDepth) a4 = seg_scan(wgt * tmid);
      if (lane == 31) x_tail[warp * kTail + 1] = a0, x_tail[warp * kTail + 2] = a1, x_tail[warp * kTail + 3] = a2, x_tail[warp * kTail + 4] = a3;
      if constexpr (kDepth) if (lane == 31) x_tail[warp * kTail + 5] = a4;
      __syncthreads();
      a0 += carry_in(1), a1 += carry_in(2), a2 += carry_in(3), a3 += carry_in(4);
      if constexpr (kDepth) a4 += carry_in(5);
      int ray_next = __shfl_down_sync(0xffffffffu, ray, 1);
      if (lane == 31) ray_next = warp < 3 ? x_first[warp + 1] : -2;
      if (valid && ray_next != ray) {   // last sample of this ray inside the tile
        const int64_t tile_start = i - tid;
        const int b = __ldg(args.comp.ray_offsets + ray), e = __ldg(args.comp.ray_offsets + ray + 1);
        if (b >= tile_start && e <= tile_start + kTile) {   // the whole ray lives in this tile
          const float k = 1.f - a3;
          const float* bg = args.comp.background;
          float* cp = args.comp.color + 3 * (int64_t)ray;
          cp[0] = a0 + (bg != nullptr ? bg[3 * ray] * k : 0.f);
          cp[1] = a1 + (bg != nullptr ? bg[3 * ray + 1] * k : 0.f);
          cp[2] = a2 + (bg != nullptr ? bg[3 * ray + 2] * k : 0.f);
          args.comp.wsum[ray] = a3;
          if constexpr (kDepth) args.depth[ray] = a4;
        } else {
          float* pp = args.comp.partial + ((tile_start / kTile) * 2 + (b < tile_start ? 0 : 1)) * 8;
          pp[0] = depth, pp[1] = a0, pp[2] = a1, pp[3] = a2, pp[4] = a3;
          if constexpr (kDepth) pp[5] = a4;
        }
      }
      __syncthreads();   // the scratch words are overwritten by the next tile's operands
    }
  }

  // ---- teardown ---------------------------------------------------------------------------
  if (!weights_ready) mbar_wait(&sm.bar_w, 0);  // never leave a bulk copy in flight
}

template <bool kSimt, int kCtasPerSm, bool kSaveGrid = false, int kLevelUnroll = 4, bool kFromFeat = false, bool kComposite = false,
          bool kDepth = false>
__global__ void __launch_bounds__(kTile, kCtasPerSm) field_forward_kernel(const __grid_constant__ FieldArgs args) {
  field_forward_body<kSimt, kSaveGrid, kLevelUnroll, kFromFeat, kComposite, kDepth, TabBf16x2>(args);
}

// HRF_TABLE_INT8X2 fields: inference only (no per-grid features, no SIMT path), one level per encode step.
template <int kCtasPerSm, bool kComposite = false, bool kDepth = false>
__global__ void __launch_bounds__(kTile, kCtasPerSm) field_forward_i8_kernel(const __grid_constant__ FieldArgs args) {
  field_forward_body<false, false, 1, false, kComposite, kDepth, TabInt8x2>(args);
}

}  // namespace hrf

using namespace hrf;

static int launch_field_forward(const FieldArgs& a, int mlp_impl, cudaStream_t st, bool persistent_full) {
  const int64_t tiles = (a.s.num_samples + kTile - 1) / kTile;
  const int smem = (int)(offsetof(FwdSmem, w) + w_blob_bytes(a.f.color_in_width)) + 128;
  // CTAs per SM, measured on an H100 (400 W) on the render bench (scripts/tuning_ab.sh): 5 (96 regs) 1.38 ms per step,
  // 4 (4-level unroll) 1.61 ms, 6 (80 regs, spills) 1.99 ms.  HRF_FWD_CTAS overrides for experiments (4 keeps the 4-level
  // unroll).
  static const int ctas_per_sm = [] {
    const char* e = getenv("HRF_FWD_CTAS");
    const int v = e ? atoi(e) : 5;
    return (v == 4 || v == 6) ? v : 5;
  }();
  static const bool ctas_forced = getenv("HRF_FWD_CTAS") != nullptr;
  // with camera embeddings the blob is 2 KB larger: 5 CTAs would need the 228 KB carve-out (almost no L1) -> use 4.
  // An int8 field takes the defaults whatever HRF_FWD_CTAS / HRF_FWD_UNROLL say: only those are instantiated for it.
  const bool i8 = a.f.table_format == HRF_TABLE_INT8X2;
  const int ctas = ((!ctas_forced || i8) && a.f.color_in_width == 48) ? 4 : i8 ? 5 : ctas_per_sm;
  const int64_t max_ctas = (int64_t)sm_count() * ctas;
  const int grid = (int)((tiles < max_ctas && !persistent_full) ? tiles : max_ctas);
  auto launch = [&](auto kernel) -> int {
    HRF_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kernel<<<grid, kTile, smem, st>>>(a);
    return 0;
  };
  // Levels unrolled in the encode loop (HRF_FWD_UNROLL = 1 | 2 | 4).  The 4-level loop is over twice the code of the
  // 1-level one, and the instruction cache, not gather ILP, limits it; on an H100 (400 W, render bench) 1 level takes
  // 1.38 ms per step, 2 and 4 levels 1.40 ms.  Default 1.
  static const int unroll = [] { const char* e = getenv("HRF_FWD_UNROLL"); const int v = e ? atoi(e) : 1; return (v == 2 || v == 4) ? v : 1; }();
  int rc;
  if (i8 && a.feat_in == nullptr) {   // (the kFromFeat kernels read composed features, not tables)
    if (a.comp.ray_offsets != nullptr && a.depth != nullptr) rc = launch(field_forward_i8_kernel<5, true, true>);
    else if (a.comp.ray_offsets != nullptr) rc = launch(field_forward_i8_kernel<5, true>);
    else if (ctas == 4) rc = launch(field_forward_i8_kernel<4>);
    else rc = launch(field_forward_i8_kernel<5>);
  } else if (a.comp.ray_offsets != nullptr && a.depth != nullptr && a.feat_in != nullptr)
    rc = launch(field_forward_kernel<false, 5, false, 1, true, true, true>);
  else if (a.comp.ray_offsets != nullptr && a.depth != nullptr) rc = launch(field_forward_kernel<false, 5, false, 1, false, true, true>);
  else if (a.comp.ray_offsets != nullptr && a.feat_in != nullptr) rc = launch(field_forward_kernel<false, 5, false, 1, true, true>);
  else if (a.comp.ray_offsets != nullptr) rc = launch(field_forward_kernel<false, 5, false, 1, false, true>);
  else if (a.feat_in != nullptr) rc = launch(field_forward_kernel<false, 5, false, 1, true>);
  else if (mlp_impl != 0 && a.egrid != nullptr) rc = launch(field_forward_kernel<true, 4, true>);   // simt debug path, e_k too
  else if (mlp_impl != 0) rc = launch(field_forward_kernel<true, 4>);
  else if (a.egrid != nullptr && unroll == 2) rc = launch(field_forward_kernel<false, 5, true, 2>);
  else if (a.egrid != nullptr && unroll == 1) rc = launch(field_forward_kernel<false, 5, true, 1>);
  else if (a.egrid != nullptr) rc = launch(field_forward_kernel<false, 5, true>);   // training forward: also saves e_k
  else if (ctas == 5 && unroll == 2) rc = launch(field_forward_kernel<false, 5, false, 2>);
  else if (ctas == 5 && unroll == 1) rc = launch(field_forward_kernel<false, 5, false, 1>);
  else if (ctas == 6 && unroll == 1 && ctas_forced) rc = launch(field_forward_kernel<false, 6, false, 1>);   // round-2 experiment
  else if (ctas == 6) rc = launch(field_forward_kernel<false, 6>);
  else if (ctas == 4) rc = launch(field_forward_kernel<false, 4>);
  else rc = launch(field_forward_kernel<false, 5>);
  if (rc) return rc;
  HRF_CHECK_LAUNCH();
  return 0;
}

static int check_field_args(const hrf_field* f, const hrf_samples* s, int mode) {
  HRF_REQUIRE(f != nullptr && s != nullptr, "null field/samples");
  HRF_REQUIRE(mode == 0 || mode == 1, "mode must be 0 (density) or 1 (density+radiance)");
  HRF_REQUIRE(s->num_samples >= 0, "negative sample count");
  HRF_REQUIRE(f->mlp_blob != nullptr && f->segments != nullptr, "field not initialised");
  HRF_REQUIRE(f->color_in_width == 32 || f->color_in_width == 48, "color_in_width must be 32 or 48");
  HRF_REQUIRE(f->camera_embedding_dim >= 0 && 31 + f->camera_embedding_dim <= f->color_in_width,
              "camera embedding does not fit the colour-net input width");
  HRF_REQUIRE(f->table_format == HRF_TABLE_BF16X2 || f->table_format == HRF_TABLE_INT8X2, "unknown table format");
  if (s->num_samples == 0) return 0;
  if (s->ray_origins != nullptr) {
    HRF_REQUIRE(s->ray_directions && s->ray_frame_numbers && s->sample_distances && s->ray_indices,
                "ray-batch form needs origins, directions, frame numbers, distances and ray indices");
  } else {
    HRF_REQUIRE(s->positions && s->frame_numbers, "query form needs positions and frame numbers");
    HRF_REQUIRE(mode == 0 || s->directions, "radiance queries need directions");
  }
  return 0;
}

extern "C" int hrf_field_forward(const hrf_field* f, const hrf_samples* s, int mode, int mlp_impl, float* sigma,
                                 void* geo_bf16, float* rgb, void* feat_bf16, void* grid_feat_bf16, void* stream) {
  if (int rc = check_field_args(f, s, mode)) return rc;
  HRF_REQUIRE(f->table_format != HRF_TABLE_INT8X2 || (grid_feat_bf16 == nullptr && mlp_impl == 0),
              "an int8 field (compact model) has no per-grid features and no SIMT path: it serves inference only");
  if (s->num_samples == 0) return 0;
  FieldArgs a;
  a.f = *f;
  a.s = *s;
  a.es = EarlyStop{};
  a.comp = Composite{};
  a.sigma = sigma;
  a.geo = reinterpret_cast<uint32_t*>(geo_bf16);
  a.rgb = rgb;
  a.feat = reinterpret_cast<uint4*>(feat_bf16);
  a.egrid = reinterpret_cast<uint32_t*>(grid_feat_bf16);
  a.feat_in = nullptr;
  a.feat_index = nullptr;
  a.mode = mode;
  a.depth = nullptr;
  return launch_field_forward(a, mlp_impl, reinterpret_cast<cudaStream_t>(stream), false);
}

extern "C" int hrf_field_forward_from_features(const hrf_field* f, const hrf_samples* s, const void* feat_in_bf16,
                                               const int32_t* feat_index, float* sigma, float* rgb, void* stream) {
  if (int rc = check_field_args(f, s, 1)) return rc;
  HRF_REQUIRE(feat_in_bf16 != nullptr, "null feature buffer");
  HRF_REQUIRE(s->ray_origins != nullptr, "hrf_field_forward_from_features needs the ray-batch form");
  if (s->num_samples == 0) return 0;
  FieldArgs a;
  a.f = *f;
  a.s = *s;
  a.es = EarlyStop{};
  a.comp = Composite{};
  a.sigma = sigma;
  a.geo = nullptr;
  a.rgb = rgb;
  a.feat = nullptr;
  a.egrid = nullptr;
  a.feat_in = reinterpret_cast<const uint4*>(feat_in_bf16);
  a.feat_index = feat_index;
  a.mode = 1;
  a.depth = nullptr;
  return launch_field_forward(a, 0, reinterpret_cast<cudaStream_t>(stream), s->num_samples_dev != nullptr);
}

namespace hrf {
__global__ void ray_max_chunks_kernel(const int32_t* __restrict__ off, int64_t num_rays, int32_t* __restrict__ out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int c = 0;
  if (r < num_rays) c = (off[r + 1] - off[r] + kTile - 1) / kTile;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) c = max(c, __shfl_xor_sync(0xffffffffu, c, d));
  if ((threadIdx.x & 31) == 0 && c > 0) atomicMax(out, c);
}
}  // namespace hrf

namespace hrf {
// Rays whose samples straddle tile borders: chain the per-tile partials front to back.  Rays without samples are pure
// background (volume_rendering.py:144-145 with weights_sum = 0).  One thread per ray.  ray_depth (or NULL): sum w*t_mid,
// chained from slot 5 of the partials with the same transmittance factor as the colour; 0 for rays without samples.
__global__ void __launch_bounds__(256) composite_fixup_kernel(const Composite c, int64_t num_rays, float* ray_depth) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= num_rays) return;
  const int b = c.ray_offsets[r], e = c.ray_offsets[r + 1];
  float col0 = 0.f, col1 = 0.f, col2 = 0.f, w = 0.f, wm = 0.f;
  if (e > b) {
    const int tf = b / kTile, tl = (e - 1) / kTile;
    if (tf == tl) return;   // finished by the forward kernel
    float depth = 0.f;
    for (int t = tf; t <= tl; ++t) {
      const float* pp = c.partial + ((int64_t)t * 2 + (t == tf ? 1 : 0)) * 8;
      const float T = __expf(-depth);
      col0 += T * pp[1], col1 += T * pp[2], col2 += T * pp[3], w += T * pp[4];
      if (ray_depth != nullptr) wm += T * pp[5];
      depth += pp[0];
    }
  }
  const float k = 1.f - w;
  if (c.background != nullptr) col0 += c.background[3 * r] * k, col1 += c.background[3 * r + 1] * k, col2 += c.background[3 * r + 2] * k;
  c.color[3 * r] = col0, c.color[3 * r + 1] = col1, c.color[3 * r + 2] = col2;
  c.wsum[r] = w;
  if (ray_depth != nullptr) ray_depth[r] = wm;
}
}  // namespace hrf

extern "C" int64_t hrf_render_fused_workspace_bytes(int64_t num_samples_capacity) {
  return ((num_samples_capacity + kTile - 1) / kTile) * 2 * 8 * (int64_t)sizeof(float) + 64;
}

// hrf_render_fused (depth = NULL) and hrf_render_fused_depth.
static int render_fused(const hrf_field* f, const hrf_samples* s, const int32_t* ray_offsets, int64_t num_rays, float step,
                        const float* background, const void* feat_in_bf16, const int32_t* feat_index, float* color,
                        float* weights_sum, float* depth, void* workspace, void* stream) {
  if (int rc = check_field_args(f, s, 1)) return rc;
  HRF_REQUIRE(ray_offsets != nullptr && color != nullptr && weights_sum != nullptr, "null argument");
  HRF_REQUIRE(s->ray_origins != nullptr, "hrf_render_fused needs the ray-batch form (samples sorted by ray)");
  HRF_REQUIRE(s->num_samples < (1ll << 31) && num_rays < (1ll << 31), "more than 2^31 samples / rays per call is not supported");
  if (num_rays == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  Composite c;
  c.ray_offsets = ray_offsets, c.background = background, c.color = color, c.wsum = weights_sum;
  c.partial = reinterpret_cast<float*>(workspace), c.step = step;
  if (s->num_samples > 0) {
    HRF_REQUIRE(workspace != nullptr, "null workspace");
    FieldArgs a;
    a.f = *f;
    a.s = *s;
    a.es = EarlyStop{};
  a.comp = Composite{};
    a.comp = c;
    a.sigma = nullptr, a.geo = nullptr, a.rgb = nullptr, a.feat = nullptr, a.egrid = nullptr;
    a.feat_in = reinterpret_cast<const uint4*>(feat_in_bf16);
    a.feat_index = feat_in_bf16 != nullptr ? feat_index : nullptr;
    a.mode = 1;
    a.depth = depth;
    if (int rc = launch_field_forward(a, 0, st, s->num_samples_dev != nullptr)) return rc;
  }
  composite_fixup_kernel<<<(unsigned)((num_rays + 255) / 256), 256, 0, st>>>(c, num_rays, depth);
  HRF_CHECK_LAUNCH();
  return 0;
}

extern "C" int hrf_render_fused(const hrf_field* f, const hrf_samples* s, const int32_t* ray_offsets, int64_t num_rays, float step,
                                const float* background, const void* feat_in_bf16, const int32_t* feat_index, float* color,
                                float* weights_sum, void* workspace, void* stream) {
  return render_fused(f, s, ray_offsets, num_rays, step, background, feat_in_bf16, feat_index, color, weights_sum, nullptr,
                      workspace, stream);
}

extern "C" int hrf_render_fused_depth(const hrf_field* f, const hrf_samples* s, const int32_t* ray_offsets, int64_t num_rays,
                                      float step, const float* background, const void* feat_in_bf16, const int32_t* feat_index,
                                      float* color, float* weights_sum, float* depth, void* workspace, void* stream) {
  HRF_REQUIRE(depth != nullptr, "null depth");
  return render_fused(f, s, ray_offsets, num_rays, step, background, feat_in_bf16, feat_index, color, weights_sum, depth,
                      workspace, stream);
}

extern "C" int64_t hrf_density_early_stop_workspace_bytes(int64_t num_rays) { return 4 * num_rays + 64; }

extern "C" int hrf_field_density_early_stop(const hrf_field* f, const hrf_samples* s, const int32_t* ray_offsets,
                                            int64_t num_rays, float step, float stop_depth, float* sigma,
                                            void* feat_bf16, void* grid_feat_bf16, void* workspace, void* stream) {
  if (int rc = check_field_args(f, s, 0)) return rc;
  HRF_REQUIRE(s->ray_origins != nullptr, "the early-stop density pass needs the ray-batch form");
  HRF_REQUIRE(ray_offsets != nullptr && sigma != nullptr && workspace != nullptr, "null argument");
  HRF_REQUIRE(step > 0.f && stop_depth > 9.2104f, "stop_depth must stay above -ln(1e-4) so the kept set is exact");
  HRF_REQUIRE(f->table_format != HRF_TABLE_INT8X2 || grid_feat_bf16 == nullptr,
              "an int8 field (compact model) has no per-grid features: it serves inference only");
  if (s->num_samples == 0 || num_rays == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  char* ws = reinterpret_cast<char*>(workspace);
  HRF_CUDA(cudaMemsetAsync(ws, 0, (size_t)hrf_density_early_stop_workspace_bytes(num_rays), st));
  FieldArgs a;
  a.f = *f;
  a.s = *s;
  a.comp = Composite{};
  a.es.ray_offsets = ray_offsets;
  a.es.num_rays = num_rays;
  a.es.ray_depth = reinterpret_cast<float*>(ws + 64);
  a.es.counter = reinterpret_cast<unsigned long long*>(ws);
  a.es.max_chunks = reinterpret_cast<const int32_t*>(ws + 16);
  a.es.step = step;
  a.es.stop_depth = stop_depth;
  a.sigma = sigma;
  a.geo = nullptr;
  a.rgb = nullptr;
  a.feat = reinterpret_cast<uint4*>(feat_bf16);
  a.egrid = reinterpret_cast<uint32_t*>(grid_feat_bf16);
  a.feat_in = nullptr;
  a.feat_index = nullptr;
  a.mode = 0;
  a.depth = nullptr;
  ray_max_chunks_kernel<<<(unsigned)((num_rays + 255) / 256), 256, 0, st>>>(ray_offsets, num_rays,
                                                                           reinterpret_cast<int32_t*>(ws + 16));
  HRF_CHECK_LAUNCH();
  return launch_field_forward(a, 0, st, true);
}
