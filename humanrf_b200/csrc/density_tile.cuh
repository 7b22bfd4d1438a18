// The persistent density tile loop of the grid evaluators (occupancy_bake.cu, training_occupancy.cu): one warpgroup per
// CTA, 128-row tiles, positions generated in the kernel -> encode -> sigma MLP (wgmma) -> density.  Every item shape
// supplies position() and store(); the density of every row is bit for bit what hrf_field_forward (mode 0, query form)
// returns for its position: the same encode_to_smem, the same two wgmma layers and the same epilogue.
#pragma once
#include "field_mlp.cuh"

namespace hrf {

constexpr int kBakeCtasPerSm = 5;

// What every item shape of the tile loop reads: the field, the frame, the grid resolution and the compacted id list
// with its device count.
struct DensityTileArgs {
  hrf_field f;
  const int32_t* count;
  const int32_t* ids;
  int32_t frame, G;
};

// The persistent tile loop: the item count stays on the device, every CTA walks tiles of Item::kItemsPerTile items of
// kTile / kItemsPerTile rows each.  Only the sigma net is evaluated: its two layers are the first kWCol1 bytes of the
// blob, whatever the colour net's width.  Fmt: the table entry format (field_common.cuh).  store() also gets the item's
// index k in the id list.
template <class Item, class Fmt = TabBf16x2>
__device__ __forceinline__ void density_tile_loop(const Item& args) {
  extern __shared__ unsigned char smem_raw[];
  FwdSmem& sm = *reinterpret_cast<FwdSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  const int tid = threadIdx.x;
  const hrf_field& f = args.f;

  if (tid == 0) {
    mbar_init(&sm.bar_w, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(&sm.bar_w, kWCol1);
    tma_load_1d(sm.w, f.mlp_blob, kWCol1, &sm.bar_w);
  }
  bool weights_ready = false;

  // frame -> segment and normalised local time, once (the host checked that the frame lies inside the LUT)
  const int sg = __ldg(f.frame_to_segment + args.frame);
  const float t_local = __ldg(f.frame_to_tlocal + args.frame);
  const hrf_segment* seg = (sg >= 0 && sg < f.num_segments) ? f.segments + sg : nullptr;

  constexpr int kRows = kTile / Item::kItemsPerTile;
  const int64_t n = *reinterpret_cast<const volatile int32_t*>(args.count);
  const int64_t num_tiles = (n + Item::kItemsPerTile - 1) / Item::kItemsPerTile;
  const int slot = (int)((unsigned)tid / kRows), sub = (int)((unsigned)tid % kRows);
  for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int64_t k = tile * Item::kItemsPerTile + slot;
    const bool valid = k < n;
    const int32_t id = valid ? __ldg(args.ids + k) : 0;
    Sample s;
    s.seg = valid ? seg : nullptr;
    s.t = t_local;
    args.position(id, sub, s);
    encode_to_smem<false, 1, Fmt>(f, s, sm.a, tid);
    if (!weights_ready) {
      mbar_wait(&sm.bar_w, 0);
      weights_ready = true;
    }
    run_hidden<false, 32>(sm, kWSig1);
    float o[16];
    run_layer16<false, 64>(sm, kWSig2, o);
    // humanrf.py:184 : density = truncated_exp(h[...,0]) * density_scale, exactly the forward's epilogue
    args.store(valid, k, id, sub, __expf(o[0]) * f.density_scale, seg);
  }
  if (!weights_ready) mbar_wait(&sm.bar_w, 0);  // never leave a bulk copy in flight
}

// Dynamic shared memory of the tile loop, and its persistent grid: one full wave, capped by the tiles of a full list.
inline int density_tile_smem() { return (int)(offsetof(FwdSmem, w) + kWCol1) + 128; }
inline int density_tile_grid(int64_t max_items, int items_per_tile) {
  const int64_t max_tiles = (max_items + items_per_tile - 1) / items_per_tile;
  const int64_t wave = (int64_t)sm_count() * kBakeCtasPerSm;
  return (int)(max_tiles < wave ? max_tiles : wave);
}

}  // namespace hrf
