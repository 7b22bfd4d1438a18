// Derivative of the composed features with respect to the sample positions, contracted with d(composed features):
// d_positions[i] = sum over levels l and grids k of J_{k,l}(p_i)^T . dF_l(i)  (hrf_field_position_grad).
//
// The read-only twin of the table-gradient scatter: it reads the workspace hrf_field_backward_mlp filled (dF level-major,
// normalised positions, segment ids) and gathers the same 4 grids x 16 levels x 8 corners the forward encode reads,
// through the forward's own index, weight and tap helpers (field_common.cuh).  One thread per sample, three fp32
// accumulators, levels in order: no atomics, two runs write identical bytes.
//
// Per level, with u = p + 0.5, pos_d = scale * u_d + 0.5 and frac_d = pos_d - floor(pos_d):
//   e_k  = sum_c w_c(frac) T[c]                      w_c = prod_d (bit_d(c) ? frac_d : 1 - frac_d)
//   de_k/du_d = scale * sum_c dw_c/dfrac_d T[c]      for the spatial dimensions of grid k only
//   F    = e_xyz V_t + e_xyt V_z + e_yzt V_x + e_xzt V_y,   V_a = lerp(vectors[a], u_a)   (make_row_tap2)
//   dV_a/du_a = vec_res (v[i1] - v[i0]), 0 where the tap clamps (i0 == i1)
// The bf16 rounding of F before the MLP is treated as the identity (as autograd treats it).
#include "field_common.cuh"

namespace hrf {

// One level of one grid: the interpolated feature pair and its derivatives along the grid's three dimensions (per unit
// of frac, i.e. before the level scale).  Same corners, weights and fp32 blend order as gather_level.
struct GridJet {
  float2 e, d0, d1, d2;
};

__device__ __forceinline__ GridJet gather_level_jet(const uint32_t* __restrict__ tab, bool hashed, uint32_t res,
                                                    uint32_t size, Cell a, Cell b, Cell c) {
  uint32_t idx[8], raw[8];
  float w[8];
  corner_indices(hashed, res, size, a, b, c, idx);
#pragma unroll
  for (int k = 0; k < 8; ++k) raw[k] = __ldg(tab + idx[k]);
  corner_weights(a, b, c, w);
  GridJet j;
  j.e = j.d0 = j.d1 = j.d2 = make_float2(0.f, 0.f);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float lo = bf16_lo(raw[k]), hi = bf16_hi(raw[k]);
    j.e.x = __fmaf_rn(w[k], lo, j.e.x);
    j.e.y = __fmaf_rn(w[k], hi, j.e.y);
    const float fa = (k & 1) ? a.f : 1.f - a.f, fb = (k & 2) ? b.f : 1.f - b.f, fc = (k & 4) ? c.f : 1.f - c.f;
    const float wa = (k & 1) ? fb * fc : -(fb * fc);   // dw/dfrac_a
    const float wb = (k & 2) ? fa * fc : -(fa * fc);   // dw/dfrac_b
    const float wc = (k & 4) ? fa * fb : -(fa * fb);   // dw/dfrac_c
    j.d0.x = __fmaf_rn(wa, lo, j.d0.x), j.d0.y = __fmaf_rn(wa, hi, j.d0.y);
    j.d1.x = __fmaf_rn(wb, lo, j.d1.x), j.d1.y = __fmaf_rn(wb, hi, j.d1.y);
    j.d2.x = __fmaf_rn(wc, lo, j.d2.x), j.d2.y = __fmaf_rn(wc, hi, j.d2.y);
  }
  return j;
}

// V = lerp of one level's feature pair along one axis (lerp_row_tap's arithmetic) and dV/dcoord.
struct VecJet {
  float2 v, dv;
};
__device__ __forceinline__ VecJet lerp_row_jet(const float* __restrict__ base, uint32_t stride, const RowTap2& t,
                                               float vec_res) {
  const float2 v0 = __ldg(reinterpret_cast<const float2*>(base + t.i0 * stride));
  const float2 v1 = __ldg(reinterpret_cast<const float2*>(base + t.i1 * stride));
  VecJet j;
  j.v = make_float2(v0.x + t.frac * (v1.x - v0.x), v0.y + t.frac * (v1.y - v0.y));
  j.dv = make_float2(vec_res * (v1.x - v0.x), vec_res * (v1.y - v0.y));   // exactly 0 where i0 == i1
  return j;
}

struct PosGradArgs {
  hrf_field f;
  hrf_samples s;
  const float2* dfeat;  // [16][num_samples] d(composed features)
  const float4* pos4;   // [num_samples] normalised (x, y, z, t)
  const uint8_t* seg8;  // [num_samples] segment index, 255 = none
  float* d_positions;   // [N,3]
};

__global__ void __launch_bounds__(256) field_position_grad_kernel(const __grid_constant__ PosGradArgs a) {
  const hrf_field& f = a.f;
  const int64_t n = live_samples(a.s);
  const int64_t ns = a.s.num_samples;   // row length of the level-major workspace
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float* out = a.d_positions + 3 * i;
  const uint32_t sgi = a.seg8[i];
  if (sgi == 255u) {
    out[0] = out[1] = out[2] = 0.f;
    return;
  }
  const float4 p4 = __ldg(a.pos4 + i);
  const float ux = p4.x, uy = p4.y, uz = p4.z, ut = p4.w;
  const hrf_segment* sg = f.segments + sgi;
  const uint32_t* g0 = sg->grid[0];
  const uint32_t* g1 = sg->grid[1];
  const uint32_t* g2 = sg->grid[2];
  const uint32_t* g3 = sg->grid[3];
  const uint32_t hmask = sg->hashed_mask;
  // the vector taps and their layout exactly as encode_to_smem reads them
  const RowTap2 tx = make_row_tap2(ux, f.vec_res), ty = make_row_tap2(uy, f.vec_res), tz = make_row_tap2(uz, f.vec_res),
                tt = make_row_tap2(ut, f.vec_res);
  const bool vt = sg->vectors_t != nullptr;
  const float* vbase = vt ? sg->vectors_t : sg->vectors;
  const uint32_t vstride = vt ? 2u : (uint32_t)HRF_N_FEATURES;
  const uint32_t vaxis = (uint32_t)f.vec_res * (vt ? 2u * HRF_N_LEVELS : (uint32_t)HRF_N_FEATURES);
  const uint32_t vlevel = vt ? 2u * (uint32_t)f.vec_res : 2u;
  const float vres = (float)f.vec_res;

  float gx = 0.f, gy = 0.f, gz = 0.f;
#pragma unroll 1
  for (int l = 0; l < HRF_N_LEVELS; ++l) {
    const float2 dO = __ldg(a.dfeat + (size_t)l * ns + i);
    const float scale = f.level_scale[l];
    const uint32_t res = f.level_res[l];
    const uint32_t off = sg->level_offset[l];
    const uint32_t size = sg->level_size[l];
    const bool hashed = (hmask >> l) & 1u;
    const Cell cx = to_cell(scale, ux), cy = to_cell(scale, uy), cz = to_cell(scale, uz), ct = to_cell(scale, ut);
    // decomposition4d.py:126-129 : xyz, xyt, yzt, xzt -- dimension j of each grid is the axis named at position j
    const GridJet e0 = gather_level_jet(g0 + off, hashed, res, size, cx, cy, cz);   // d0 = x, d1 = y, d2 = z
    const GridJet e1 = gather_level_jet(g1 + off, hashed, res, size, cx, cy, ct);   // d0 = x, d1 = y, (d2 = t)
    const GridJet e2 = gather_level_jet(g2 + off, hashed, res, size, cy, cz, ct);   // d0 = y, d1 = z, (d2 = t)
    const GridJet e3 = gather_level_jet(g3 + off, hashed, res, size, cx, cz, ct);   // d0 = x, d1 = z, (d2 = t)
    const float* vl = vbase + (uint32_t)l * vlevel;
    const VecJet vx = lerp_row_jet(vl, vstride, tx, vres), vy = lerp_row_jet(vl + vaxis, vstride, ty, vres),
                 vz = lerp_row_jet(vl + 2u * vaxis, vstride, tz, vres), vtt = lerp_row_jet(vl + 3u * vaxis, vstride, tt, vres);
    // F = e0 V_t + e1 V_z + e2 V_x + e3 V_y; the vector terms: e2 dV_x/dx, e3 dV_y/dy, e1 dV_z/dz
    const float jx0 = scale * (e0.d0.x * vtt.v.x + e1.d0.x * vz.v.x + e3.d0.x * vy.v.x) + e2.e.x * vx.dv.x;
    const float jx1 = scale * (e0.d0.y * vtt.v.y + e1.d0.y * vz.v.y + e3.d0.y * vy.v.y) + e2.e.y * vx.dv.y;
    const float jy0 = scale * (e0.d1.x * vtt.v.x + e1.d1.x * vz.v.x + e2.d0.x * vx.v.x) + e3.e.x * vy.dv.x;
    const float jy1 = scale * (e0.d1.y * vtt.v.y + e1.d1.y * vz.v.y + e2.d0.y * vx.v.y) + e3.e.y * vy.dv.y;
    const float jz0 = scale * (e0.d2.x * vtt.v.x + e2.d1.x * vx.v.x + e3.d1.x * vy.v.x) + e1.e.x * vz.dv.x;
    const float jz1 = scale * (e0.d2.y * vtt.v.y + e2.d1.y * vx.v.y + e3.d1.y * vy.v.y) + e1.e.y * vz.dv.y;
    gx += dO.x * jx0 + dO.y * jx1;
    gy += dO.x * jy0 + dO.y * jy1;
    gz += dO.x * jz0 + dO.y * jz1;
  }
  out[0] = gx, out[1] = gy, out[2] = gz;
}

}  // namespace hrf

using namespace hrf;

extern "C" int hrf_field_position_grad(const hrf_field* f, const hrf_samples* s, const void* workspace, float* d_positions,
                                       void* stream) {
  HRF_REQUIRE(f != nullptr && s != nullptr, "null argument");
  HRF_REQUIRE(f->table_format == HRF_TABLE_BF16X2, "an int8 field (compact model) serves inference only: it has no gradients");
  HRF_REQUIRE(s->num_samples >= 0, "negative sample count");
  if (s->num_samples == 0) return 0;
  HRF_REQUIRE(workspace != nullptr, "needs the workspace hrf_field_backward_mlp filled");
  HRF_REQUIRE(d_positions != nullptr, "null d_positions");
  HRF_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 15u) == 0, "the workspace must be 16-byte aligned");
  PosGradArgs a;
  a.f = *f;
  a.s = *s;
  a.dfeat = reinterpret_cast<const float2*>(workspace);
  a.pos4 = reinterpret_cast<const float4*>(reinterpret_cast<const char*>(workspace) + 128 * (size_t)s->num_samples);
  a.seg8 = reinterpret_cast<const uint8_t*>(reinterpret_cast<const char*>(workspace) + 144 * (size_t)s->num_samples);
  a.d_positions = d_positions;
  const int64_t blocks = (s->num_samples + 255) / 256;
  field_position_grad_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  HRF_CHECK_LAUNCH();
  return 0;
}
