/*
 * humanrf_b200 -- C ABI of the H100-native (sm_90a) HumanRF per-ray hot path.
 *
 * Drop-in boundary for the reference's three pybind11 torch extensions and the two
 * third-party CUDA packages its hot path calls (SURVEY.md section 8b).  Every entry point
 * takes plain DEVICE pointers (unless the name says host) + sizes + a CUDA stream handle
 * (cudaStream_t passed as void*, NULL = legacy default stream); no torch types.  All
 * functions return 0 on success and a non-zero code on failure; hrf_last_error() gives the
 * message (the reference throws std::runtime_error from CHECK_CONTIGUITY_AND_DEVICE,
 * actorshq/toolbox/native/utils.cuh:5-19; the Python host mirror raises RuntimeError).
 * Launches are asynchronous on the given stream; nothing here synchronises except the
 * functions documented as doing so.
 */
#ifndef HUMANRF_B200_H_
#define HUMANRF_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HRF_N_LEVELS 16        /* humanrf/args/model_args.py:26 n_levels            */
#define HRF_N_FEATURES 32      /* n_levels * n_features_per_level (2)               */
#define HRF_MLP_WIDTH 64       /* model_args.py:12 n_neurons                        */
#define HRF_GEO_DIM 15         /* model_args.py:10 geometry_feature_dim             */
#define HRF_MLP_BLOB_BYTES 22528 /* packed bf16 weights: sigma 64x32,16x64; colour 64x(32|48),64x64,16x64 */
#define HRF_MAX_CAMERA_EMBEDDING_DIM 17 /* 16 SH + 15 geo + E <= 48 */

const char* hrf_last_error(void);
int hrf_version(void);
/* device properties the host mirror needs: out[0]=SM count, out[1]=cc major, out[2]=cc minor */
int hrf_device_info(int* out3);

/* ------------------------------------------------------------------------------------------
 * Occupancy grid ring.  Replaces occupancy_grid_native.OccupanyGrid
 * (actorshq/dataset/native/occupancy_grid.cu:8-95): a ring of `buffer_size` G^3 occupancy
 * volumes; add_grid copies a uint8 [G][G][G] (z,y,x) device tensor into the next slot and
 * returns an int64 handle the sampler understands (the reference returns a
 * cudaTextureObject_t; here it is the device address of a bit-packed G^3 volume).
 * ---------------------------------------------------------------------------------------- */
typedef struct hrf_occgrid hrf_occgrid;
int hrf_occgrid_create(uint64_t grid_resolution, int buffer_size, hrf_occgrid** out);
int hrf_occgrid_destroy(hrf_occgrid* g);
int hrf_occgrid_add(hrf_occgrid* g, const uint8_t* grid_u8, uint64_t res0, uint64_t res1, uint64_t res2,
                    void* stream, int64_t* handle_out);
/* test hook: evaluates the emulated `tex3D(handle, p) > 0` for n points (xyz normalised) */
int hrf_occgrid_lookup(int64_t handle, int grid_resolution, const float* points_xyz, int64_t n,
                       uint8_t* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * Ray sampler.  Replaces ray_sampler_native.get_{rays,samples}_{aabb,occupancy}_minmax
 * (actorshq/dataset/native/ray_sampler.cu:196-325).  Three phases, no host round trip inside:
 *   hrf_sampler_rays   : compute_minmax_kernel (:80-147) for all R candidate rays, ray mask
 *                        (optionally AND NOT light_mask, :254-257), device-side compaction,
 *                        per-ray gathers (:258-266) and per-ray sample counts/offsets
 *                        (:283-290, occupancy filter of :183-189 already applied).
 *                        counters[0]=R' (kept rays), counters[1]=N' (kept samples).  N' is summed
 *                        in 64 bits and exact, but sample_offsets are int32: a caller must not
 *                        call hrf_sampler_samples when N' > 2^31 - 1 (the offsets have wrapped).
 *   hrf_sampler_samples: compute_sample_distances_kernel (:149-194) + final compaction
 *                        (:322-323) written directly at the scanned offsets.
 * rgba_pool / light_mask are DEVICE-resident pools here (the reference indexes a CPU pool and
 * bounces through the host, :262); the Python mirror keeps the CPU-pool call signature.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  const int32_t* frame_numbers;      /* [B] */
  const int32_t* camera_numbers;     /* [B] */
  const int64_t* grid_handles;       /* [B] from hrf_occgrid_add (unused for aabb mode) */
  const uint8_t* landscape_modes;    /* [B] bool */
  const float*   inverse_krs;        /* [B,3,3], stored transposed as the reference does (data_loader.py:194-207) */
  const float*   camera_origins;     /* [B,3] */
  const float*   aabb;               /* [2,3] */
  const uint8_t* rgba_pool;          /* [P,4] uint8 or NULL */
  const uint8_t* light_mask;         /* [P] bool, indexed by pool pixel, or NULL */
  const uint8_t* light_mask_rays;    /* [R] bool, indexed by candidate ray (host-pool callers), or NULL */
  int32_t grid_resolution, image_width, image_height;
  float step;
  int32_t occupancy;                 /* 1: occupancy minmax + filter, 0: aabb only */
  int32_t filter_light_bloom;
  int32_t want_samples;              /* 0: get_rays_* variants (counts are all zero) */
} hrf_sampler_params;

int hrf_sampler_rays(const hrf_sampler_params* p, const int64_t* all_ray_indices, int64_t num_rays,
                     /* full-size outputs [R] */
                     uint8_t* ray_mask,
                     /* compacted outputs, capacity R */
                     float* ray_origins, float* ray_directions, float* rgba, int32_t* frame_numbers,
                     int32_t* camera_numbers, float* minmaxes, int64_t* kept_ray_indices,
                     int32_t* sample_offsets /* [R+1] exclusive scan of kept-sample counts */,
                     int64_t* counters /* [2] device */, void* workspace, int64_t workspace_bytes, void* stream);
int64_t hrf_sampler_workspace_bytes(int64_t num_rays);
int hrf_sampler_samples(const hrf_sampler_params* p, int64_t num_kept_rays, const int64_t* kept_ray_indices,
                        const float* ray_origins, const float* ray_directions, const float* minmaxes,
                        const int32_t* sample_offsets, float* distances /* [N'] */,
                        int32_t* relative_ray_indices /* [N'] */, void* stream);

/* ------------------------------------------------------------------------------------------
 * Radiance field.  Replaces HumanRF.density / HumanRF.forward
 * (humanrf/scene_representation/humanrf.py:158-208): 4 tcnn HashGrids per segment
 * (decomposition4d.py:79-129), compose_tensors (tensor_composition.cu:9-55), sigma MLP +
 * truncated_exp (humanrf.py:181-186), SH/identity colour MLP (:188-206) in ONE kernel.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  const uint32_t* grid[4];           /* bf16x2 entries: xyz, xyt, yzt, xzt encodings     */
  const float*    vectors;           /* [4, vec_res, 32] fp32 (decomposition4d.py:76-78) */
  uint32_t level_offset[HRF_N_LEVELS]; /* entry offset of each level                      */
  uint32_t level_size[HRF_N_LEVELS];   /* hashmap_size of each level (entries)            */
  uint32_t hashed_mask;              /* bit l: level l uses the spatial hash             */
  uint32_t n_entries;                /* entries per grid                                 */
  /* Optional transposed fp32 copy of `vectors`, [4 axes][16 levels][vec_res][2] (hrf_transpose_vectors; kept current by
   * hrf_adam_multi / hrf_dp_reduce_adam through hrf_adam_tensor.vectors_t): the gradient scatter reads one level's
   * feature pair of consecutive rows from consecutive addresses.  NULL: the scatter reads `vectors` itself. */
  const float*    vectors_t;
} hrf_segment;

typedef struct {
  const hrf_segment* segments;       /* device array [num_segments]                      */
  const int32_t* frame_to_segment;   /* device [lut_size]   (humanrf.py:99)              */
  const float*   frame_to_tlocal;    /* device [lut_size]   (humanrf.py:100-103)         */
  const void*    mlp_blob;           /* device, HRF_MLP_BLOB_BYTES, see hrf_pack_layout   */
  float    level_scale[HRF_N_LEVELS];
  uint32_t level_res[HRF_N_LEVELS];
  int32_t  num_segments, lut_size, vec_res;
  float    density_scale;
  /* camera embeddings (humanrf.py:75-76,194-204): fp32 [num_cameras, camera_embedding_dim], or NULL / 0 */
  const float* camera_embeddings;
  int32_t  camera_embedding_dim, num_cameras;
  int32_t  color_in_width;           /* 32 (no embedding) or 48: width of the padded colour-net input */
  /* HRF_TABLE_BF16X2: hrf_segment.grid[k] holds bf16x2 entries (uint32_t each).
   * HRF_TABLE_INT8X2: it holds int8x2 entries (uint16_t each: feature 0 in the low byte) with the same entry indexing,
   * and `vectors` / `vectors_t` carry each slice's scale folded in (hrf_quantize_tables_write).  Only inference reads
   * such a field: every backward entry, hrf_field_position_grad, a forward asking for the per-grid features and the
   * SIMT debug path (mlp_impl != 0) refuse it, because the per-grid features are no longer the model's. */
  int32_t  table_format;
} hrf_field;
#define HRF_TABLE_BF16X2 0
#define HRF_TABLE_INT8X2 1

/* Sample source: either explicit per-sample queries (QueryInput, query_io.py:6-13) or the
 * ray-batch form used by prune_samples/render (volume_rendering.py:66-72,110-119). */
typedef struct {
  /* query form (ray_origins == NULL) */
  const float* positions;            /* [N,3] in [-0.5,0.5] */
  const float* directions;           /* [N,3] or NULL for density-only */
  const int32_t* frame_numbers;      /* [N] */
  /* ray-batch form */
  const float* ray_origins;          /* [R,3] */
  const float* ray_directions;       /* [R,3] */
  const int32_t* ray_frame_numbers;  /* [R] */
  const float* sample_distances;     /* [N] */
  const int64_t* ray_indices;        /* [N] sorted ascending */
  int64_t num_samples;
  /* camera numbers, only read when the field has camera embeddings and use_camera_embeddings != 0
   * (is_training; at evaluation the embedding is all zeros, humanrf.py:196-204) */
  const int32_t* camera_numbers;     /* query form: [N] */
  const int32_t* ray_camera_numbers; /* ray-batch form: [R] */
  int32_t use_camera_embeddings;
  /* Sync-free pipelines: when non-NULL the kernels read the LIVE number of samples from this device scalar and
   * num_samples is the capacity of the per-sample arrays (grid sizing, strides of the [..][N] buffers).  This is what
   * lets a training step prune on the device and keep going without reading the survivor count back
   * (the reference reads it implicitly through boolean-mask indexing, volume_rendering.py:83-84). */
  const int64_t* num_samples_dev;
} hrf_samples;

/* mode: 0 = density only (sigma, geo), 1 = density + radiance.  Any output may be NULL.
 * mlp_impl: 0 = wgmma tensor-core path (the product); 1 = SIMT fp32 debug path used only by
 * tests to localise tensor-core descriptor faults. */
int hrf_field_forward(const hrf_field* f, const hrf_samples* s, int mode, int mlp_impl,
                      float* sigma /* [N] */, void* geo_bf16 /* [N,16] (col 0 = raw h0) */,
                      float* rgb /* [N,3] */, void* feat_bf16 /* [N,32] composed features saved for backward, or NULL */,
                      void* grid_feat_bf16 /* [64,N] bf16x2 per-(level,grid) interpolated features for backward, or NULL */,
                      void* stream);

/* The MLP half of hrf_field_forward for samples whose composed features already exist (the density-only pass of
 * prune_samples encodes every candidate; the render pass of the survivors does not have to encode them again):
 * feat_in_bf16 [M,32] as written by a previous pass, feat_index[i] = its row for sample i (NULL = identity).
 * `s` must be in ray-batch form (view directions / camera numbers are read through ray_indices). */
int hrf_field_forward_from_features(const hrf_field* f, const hrf_samples* s, const void* feat_in_bf16,
                                    const int32_t* feat_index, float* sigma /* [N] */, float* rgb /* [N,3] */,
                                    void* stream);

/* Inference render in ONE field kernel (humanrf/volume_rendering.py:87-150 without gradients): encode -> sigma MLP ->
 * colour MLP -> per-ray compositing, w_i = exp(-sum_{j<i} sigma_j dt_j) (1 - exp(-sigma_i dt_i)), colour = sum w rgb +
 * background (1 - sum w).  Per-sample sigma / rgb never leave the SM; a small second kernel chains the rays that
 * straddle 128-sample tile borders and writes the background for rays without samples.  Samples must be sorted by
 * ray (ray_offsets[r] = first sample of ray r).  feat_in / feat_index: optional composed features of an earlier
 * pass (hrf_field_forward_from_features semantics; then nothing is encoded here).  s->num_samples_dev is honoured.
 * workspace: hrf_render_fused_workspace_bytes(s->num_samples) bytes of device scratch. */
int64_t hrf_render_fused_workspace_bytes(int64_t num_samples_capacity);
int hrf_render_fused(const hrf_field* f, const hrf_samples* s /* ray-batch form */, const int32_t* ray_offsets /* [R+1] */,
                     int64_t num_rays, float step, const float* background /* [R,3] or NULL */, const void* feat_in_bf16,
                     const int32_t* feat_index, float* color /* [R,3] */, float* weights_sum /* [R] */, void* workspace,
                     void* stream);
/* hrf_render_fused plus a depth map, with the same inputs, workspace and rules.  For each ray r, over exactly the samples
 * its colour is composited from, in order: depth[r] = sum_i w_i * m_i with m_i = __fmul_rn(0.5f, __fadd_rn(t_i,
 * __fadd_rn(t_i, step))), nerfacc's (t_starts + t_ends) / 2, i.e. accumulate_along_rays(weights, values=t_mid).  It is
 * unnormalised (depth / weights_sum is the expected distance along the ray direction), has no background term, and is 0
 * for rays without samples.  color and weights_sum are bit-identical to what hrf_render_fused writes. */
int hrf_render_fused_depth(const hrf_field* f, const hrf_samples* s /* ray-batch form */, const int32_t* ray_offsets /* [R+1] */,
                           int64_t num_rays, float step, const float* background /* [R,3] or NULL */, const void* feat_in_bf16,
                           const int32_t* feat_index, float* color /* [R,3] */, float* weights_sum /* [R] */,
                           float* depth /* [R], non-NULL */, void* workspace, void* stream);

/* Density-only pass of prune_samples (volume_rendering.py:66-84) with an exact early stop: ray chunks are
 * evaluated front to back; once a ray's accumulated optical depth makes every later sample fail nerfacc's
 * transmittance test (T < 1e-4) those samples are reported with sigma = 0 without being evaluated.  The kept
 * set of hrf_prune on this sigma equals the one on the fully evaluated sigma.  workspace: device scratch of
 * hrf_density_early_stop_workspace_bytes(num_rays) bytes. */
int64_t hrf_density_early_stop_workspace_bytes(int64_t num_rays);
int hrf_field_density_early_stop(const hrf_field* f, const hrf_samples* s /* ray-batch form */,
                                 const int32_t* ray_offsets /* [R+1] */, int64_t num_rays, float step,
                                 float stop_depth /* > -ln(1e-4); 9.4 recommended */, float* sigma /* [N] */,
                                 void* feat_bf16 /* [N,32] composed features of every evaluated sample, or NULL */,
                                 void* grid_feat_bf16 /* [64,N] per-(level,grid) features, or NULL */,
                                 void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------
 * Compositing.  Replaces nerfacc.render_visibility / render_weight_from_density /
 * accumulate_along_rays as called from humanrf/volume_rendering.py:75-84,123-145.
 * ---------------------------------------------------------------------------------------- */
/* ray_offsets[r] = first sample of ray r in the sorted ray_indices; ray_offsets[R] = N */
int hrf_ray_offsets(const int64_t* ray_indices, int64_t num_samples, int64_t num_rays,
                    int32_t* ray_offsets /* [R+1] */, void* stream);
/* prune: keep_i = (T_i >= 1e-4) & (alpha_i >= 1e-4), alpha = 1-exp(-sigma*step); writes the
 * kept samples compacted; counters[0] = kept count.  kept_offsets [R+1] workspace. */
int hrf_prune(const float* sigma, const float* sample_distances, const int64_t* ray_indices,
              const int32_t* ray_offsets, int64_t num_rays, float step, float early_stop_eps, float alpha_thre,
              uint8_t* keep_mask /* [N] or NULL */, int32_t* kept_offsets /* [R+1] */,
              float* out_distances, int64_t* out_ray_indices, int32_t* out_source_index /* [N] index of each kept sample
              in the input arrays, or NULL */, int64_t* counters, void* stream);
/* render: w_i = exp(-sum_{j<i} sigma_j*dt_j) * (1-exp(-sigma_i*dt_i)), dt=(t+step)-t;
 * color = sum w*rgb (+ background*(1-sum w)), weights_sum = sum w. background: [R,3] or NULL. */
int hrf_composite_forward(const float* sigma, const float* rgb, const float* sample_distances,
                          const int32_t* ray_offsets, int64_t num_rays, float step, const float* background,
                          float* color /* [R,3] */, float* weights_sum /* [R] */,
                          float* weights /* [N] or NULL */, void* stream);
/* backward of the above w.r.t. sigma and rgb given d_color [R,3], d_weights_sum [R] */
int hrf_composite_backward(const float* sigma, const float* rgb, const float* sample_distances,
                           const int32_t* ray_offsets, int64_t num_rays, float step, const float* background,
                           const float* d_color, const float* d_weights_sum,
                           float* d_sigma /* [N] */, float* d_rgb /* [N,3] */, void* stream);

/* ------------------------------------------------------------------------------------------
 * Backward of the radiance field (autograd of humanrf.py:158-208): recomputes the forward per
 * 128-sample tile, runs MLP dgrad/wgrad on the tensor cores, scatters table / vector gradients.
 * Gradients are ACCUMULATED (+=) into the fp32 buffers; the caller zeroes them.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  float* grid[4];                    /* [n_entries,2] fp32, same order as hrf_segment.grid */
  float* vectors;                    /* [4, vec_res, 32] fp32 */
} hrf_segment_grads;

int hrf_field_backward(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads /* device array */,
                       const float* d_sigma /* [N] */, const float* d_rgb /* [N,3] or NULL */,
                       const float* d_geo /* [N,15] gradient of the geometry features, or NULL */,
                       const void* feat_bf16 /* composed features from a forward pass, or NULL to re-encode */,
                       const void* grid_feat_bf16 /* [64,stride] from a forward pass, or NULL to re-gather the tables */,
                       const int32_t* feat_index /* row of sample i in feat / grid_feat (NULL = identity) */,
                       int64_t grid_feat_stride /* row length of grid_feat (0 = num_samples) */,
                       float* d_mlp /* fp32 [3072 + 64*color_in_width + 5120]: sigma W1,W2, colour W1,W2,W3 row-major [out,in] */,
                       float* d_camera_embeddings /* fp32 [num_cameras, dim] accumulated into, or NULL */,
                       void* workspace /* 160 bytes per sample (16-byte aligned): d(features) level-major, positions, segment ids */, void* stream);
/* The same backward in two phases, so that a data-parallel trainer can start reducing one table's gradient while the
 * next table's scatter still runs: hrf_field_backward == hrf_field_backward_mlp + hrf_field_backward_tables(0, 4).
 * Table k's gradient is complete after the launch covering grid k; the vector gradients after the last launch. */
int hrf_field_backward_mlp(const hrf_field* f, const hrf_samples* s, const float* d_sigma, const float* d_rgb,
                           const float* d_geo, const void* feat_bf16, const int32_t* feat_index, float* d_mlp,
                           float* d_camera_embeddings, void* workspace, void* stream);
int hrf_field_backward_tables(const hrf_field* f, const hrf_samples* s, const hrf_segment_grads* seg_grads,
                              const void* grid_feat_bf16, const int32_t* feat_index, int64_t grid_feat_stride,
                              const void* workspace, int grid_first, int grid_count, void* stream);
/* hrf_field_backward_mlp that also writes the view-direction gradient d_directions [N,3] (row i: sample i's direction,
 * in the ray-batch form its ray's direction): d_dir = sum_j dCin[j] * dSH_j/d(x, y, z) over the 16 SH inputs of the colour
 * net, at the fp32 x, y, z the forward's SH evaluates.  The map d -> ((d + 1) / 2) * 2 - 1 and the bf16 rounding of the
 * SH values count as the identity (tcnn's SH input gradient composed with the reference's (d + 1) / 2).  Written, not
 * accumulated, for i < live count; rows past it are untouched; rows of samples without a segment, and every row when
 * d_rgb is NULL, are 0.  Everything else (d_mlp, d_camera_embeddings, the workspace) is as hrf_field_backward_mlp's. */
int hrf_field_backward_mlp_dirs(const hrf_field* f, const hrf_samples* s, const float* d_sigma, const float* d_rgb,
                                const float* d_geo, const void* feat_bf16, const int32_t* feat_index, float* d_mlp,
                                float* d_camera_embeddings, float* d_directions /* [N,3] */, void* workspace, void* stream);
/* Position gradient: d_positions[i] = sum over levels l and grids k of J_{k,l}(p_i)^T . dF_l(i), the derivative of the
 * composed features hrf_field_forward computes, contracted with d(composed features).  `workspace` is what
 * hrf_field_backward_mlp filled for the same `s`: dF as float2 [16][N] at 0, normalised positions at 128 N, segment ids
 * at 144 N (N = s->num_samples).  J includes both the grid term (the corner weights' derivative, scaled by the level
 * scale; a grid's time dimension feeds no position component) and the vector term e_k * vec_res * (v[i1] - v[i0]) of
 * the one grid whose vector runs along the axis (0 where the tap clamps).  The bf16 rounding of the features before the
 * MLP counts as the identity.  Written, not accumulated, for i < live count (s->num_samples_dev honoured); rows past
 * the live count are untouched; rows of samples whose frame has no segment are 0.  Query and ray-batch form.  No
 * atomics: two runs write identical bytes.  Nothing here synchronises. */
int hrf_field_position_grad(const hrf_field* f, const hrf_samples* s, const void* workspace,
                            float* d_positions /* [N,3] */, void* stream);
/* Ray-form reduction of the per-sample gradients, for positions p_i = o_r + t_i d_r and view direction d_r of the
 * samples i of ray r (ray_offsets [R+1] as hrf_ray_offsets writes it):
 *   d_origins[r] = sum_i dpos_i;   d_ray_directions[r] = sum_i (t_i dpos_i + ddir_i);   d_sample_distances[i] = dpos_i . d_r
 * d_directions (per-sample view-direction gradient) and d_sample_distances may be NULL.  All outputs are written, not
 * accumulated; a ray without samples gets zeros.  A batch without samples passes d_positions = sample_distances = NULL
 * (ray_offsets and ray_directions may then be NULL too): every ray gets zeros.  One warp per ray, a fixed summation
 * order and no atomics: two runs write identical bytes. */
int hrf_ray_gradients(const float* d_positions /* [N,3] */, const float* d_directions /* [N,3] or NULL */,
                      const float* sample_distances /* [N] */, const float* ray_directions /* [R,3] */,
                      const int32_t* ray_offsets /* [R+1] */, int64_t num_rays, float* d_origins /* [R,3] */,
                      float* d_ray_directions /* [R,3] */, float* d_sample_distances /* [N] or NULL */, void* stream);

/* ------------------------------------------------------------------------------------------
 * Per-camera pose refinement in the fused train step (toolbox/camera_refinement.py CameraPoses, DESIGN.md §3.14).
 * Camera c carries an increment (omega_c, tau_c) in normalised scene units: R' = exp([omega_c]x) R, c' = c + tau_c.  Its
 * sampler table is (exp([omega_c]x) M_c)^T with M_c = base_inverse_krs[c]^T, its origin base_camera_origins[c] + tau_c.
 * ---------------------------------------------------------------------------------------- */
/* Workspace of hrf_camera_pose_grad for `num_cameras` cameras (any ray count), or -1 outside [1, 1024]. */
int64_t hrf_camera_pose_grad_workspace_bytes(int num_cameras);
/* Pose gradients of a ray batch sampled from the current tables (o_r = c_c + tau_c, d_r = exp([omega_c]x) d0_r):
 *   pose_grad[c] = (J_l(omega_c)^T sum_{r in c} d_r x d_ray_directions[r],  sum_{r in c} d_origins[r])
 *   J_l(w) = I + (1 - cos t)/t^2 [w]x + (t - sin t)/t^3 [w]x^2, t = |w|
 * and ray_count[c] = the rays of camera c.  Written for every camera (0 for a camera without rays).  The sums are fp32
 * in an order fixed by the batch (no float atomics): two runs write identical bytes; J_l^T is applied in float64.  A
 * camera number outside [0, num_cameras) sets bit 0 of error[0] (or'ed, the caller zeroes it) and the ray is left out.
 * num_cameras <= 1024.  Nothing here synchronises. */
int hrf_camera_pose_grad(const float* d_origins /* [R,3] */, const float* d_ray_directions /* [R,3] */,
                         const float* ray_directions /* [R,3] */, const int32_t* camera_numbers /* [R] */,
                         int64_t num_rays, const double* omega /* [C,3] */, int num_cameras,
                         float* pose_grad /* [C,6] */, int32_t* ray_count /* [C] */, int32_t* error /* [1] */,
                         void* workspace, void* stream);
typedef struct {
  double* omega;                      /* [C,3] rotation increments */
  double* tau;                        /* [C,3] centre increments */
  double* exp_avg;                    /* [C,6] Adam moments, (omega, tau) order */
  double* exp_avg_sq;                 /* [C,6] */
  int32_t* step;                      /* [C] Adam step counters */
  const uint8_t* fixed;               /* [C] non-zero: the camera is never moved */
  const float* base_inverse_krs;      /* [C,3,3] tables at omega = 0 (the loader's, transposed inverse KR) */
  const float* base_camera_origins;   /* [C,3] origins at tau = 0 */
  float* inverse_krs;                 /* [C,3,3] rewritten: the loader's all_inverse_krs */
  float* camera_origins;              /* [C,3] rewritten: the loader's all_camera_origins */
  float* slot_inverse_krs;            /* [B,3,3] rewritten: the pool slots' tables */
  float* slot_camera_origins;         /* [B,3] */
  const int32_t* slot_camera_numbers; /* [B] camera of each slot; -1 = empty slot, left untouched */
  int num_cameras;                    /* C, 1..1024 */
  int num_slots;                      /* B */
} hrf_camera_poses;
/* One launch: Adam (torch.optim.Adam's update, float64) on (omega_c, tau_c) of every camera with ray_count[c] > 0 that
 * is not fixed, each with its own step counter and bias correction; its tables are rebuilt in float64 from the base
 * tables and rounded once (omega = 0 gives the base table bit for bit).  Cameras without rays, and fixed cameras, keep
 * parameters, moments, step counter and tables.  Then every slot with a camera copies that camera's tables.  When
 * error is non-NULL and error[0] != 0 (a bad camera number in hrf_camera_pose_grad), nothing is written.  No host read. */
int hrf_camera_pose_step(const hrf_camera_poses* poses, const float* pose_grad /* [C,6] */,
                         const int32_t* ray_count /* [C] */, const int32_t* error /* [1] or NULL */, double lr,
                         double beta1, double beta2, double eps, void* stream);

/* ------------------------------------------------------------------------------------------
 * Per-camera intrinsics refined with the pose (CameraPoses(intrinsics=True), DESIGN.md §3.15).  Camera c also carries
 * alpha_c = (alpha_x, alpha_y), log focal scales, and beta_c = (beta_x, beta_y), principal-point offsets in units of the
 * base focal length.  For a pixel (px, py) with base camera coordinates u0 = K0^-1 (px, py, 1) = (x0, y0, 1):
 *   u' = ((x0 - beta_x) e^-alpha_x, (y0 - beta_y) e^-alpha_y, 1),  v = exp([omega_c]x) R u',  d = v / |v|
 * i.e. fx = fx0 e^alpha_x, cx = cx0 + fx0 beta_x (same for y).  The sampler table is (exp([omega_c]x) (M0 B))^T with
 * M0 = base_inverse_krs[c]^T and B = K0 A K0^-1 =
 *   [[e^-ax, 0, -cx0 expm1(-ax) - fx0 bx e^-ax], [0, e^-ay, -cy0 expm1(-ay) - fy0 by e^-ay], [0, 0, 1]]
 * in float64, rounded once; alpha = beta = 0 gives hrf_camera_pose_step's table bit for bit.
 * ---------------------------------------------------------------------------------------- */
/* Workspace of hrf_camera_calib_grad for `num_cameras` cameras (any ray count), or -1 outside [1, 1024]. */
int64_t hrf_camera_calib_grad_workspace_bytes(int num_cameras);
/* hrf_camera_pose_grad's outputs (the pose columns bit-identical to it on the same inputs) and, with R'_c = rotations[c]
 * (row-major, the camera's current camera-to-world rotation), q = R'^T d_r, h = R'^T (g_d - d_r (d_r . g_d)):
 *   intrinsics_grad[c] = (-sum q_x h_x, -sum q_y h_y, -e^-alpha_x sum q_z h_x, -e^-alpha_y sum q_z h_y)
 * = d(loss)/d(alpha_x, alpha_y, beta_x, beta_y).  Same sums' order, determinism, error word and camera limit as
 * hrf_camera_pose_grad.  Nothing here synchronises. */
int hrf_camera_calib_grad(const float* d_origins /* [R,3] */, const float* d_ray_directions /* [R,3] */,
                          const float* ray_directions /* [R,3] */, const int32_t* camera_numbers /* [R] */,
                          int64_t num_rays, const double* omega /* [C,3] */, const double* alpha /* [C,2] */,
                          const float* rotations /* [C,3,3] */, int num_cameras, float* pose_grad /* [C,6] */,
                          float* intrinsics_grad /* [C,4] */, int32_t* ray_count /* [C] */, int32_t* error /* [1] */,
                          void* workspace, void* stream);
typedef struct {
  double* alpha;                      /* [C,2] log focal scales */
  double* beta;                       /* [C,2] principal-point offsets / base focal length */
  double* exp_avg;                    /* [C,4] Adam moments, (alpha_x, alpha_y, beta_x, beta_y) order */
  double* exp_avg_sq;                 /* [C,4] */
  const double* base_intrinsics;      /* [C,4] fx0, fy0, cx0, cy0 in pixels */
  const double* base_rotations;       /* [C,3,3] R, camera-to-world, row-major */
  float* rotations;                   /* [C,3,3] rewritten: exp([omega_c]x) R rounded once, hrf_camera_calib_grad's input */
} hrf_camera_intrinsics;
/* hrf_camera_pose_step with the intrinsics: the same cameras take one Adam step on (omega, tau) at lr and on
 * (alpha, beta) at lr_intrinsics, sharing the camera's step counter; tables as above, origin and pool slots as
 * hrf_camera_pose_step, and rotations[c] rewritten.  Nothing is written when error[0] != 0.  No host read. */
int hrf_camera_calib_step(const hrf_camera_poses* poses, const hrf_camera_intrinsics* intrinsics,
                          const float* pose_grad /* [C,6] */, const float* intrinsics_grad /* [C,4] */,
                          const int32_t* ray_count /* [C] */, const int32_t* error /* [1] or NULL */, double lr,
                          double lr_intrinsics, double beta1, double beta2, double eps, void* stream);

/* ------------------------------------------------------------------------------------------
 * Training loss on the per-ray outputs, forward and backward in one launch (trainer.py:205-215,229-238,
 * utils/loss.py:4-10): gt = rgb*mask + background*(1-mask); HuberLoss(delta, mean) over [R,3] +
 * bce_weight * mean(BCE(clamp(weights_sum,0,1), mask)) with eps 1e-10.  loss_out[0] += loss (caller zeroes);
 * d_color / d_weights_sum are d(loss * *loss_scale_dev) (loss_scale_dev NULL = 1: data-parallel ranks weight their
 * share of the union batch with it).
 * ---------------------------------------------------------------------------------------- */
int hrf_train_loss(const float* color /* [R,3] */, const float* weights_sum /* [R] */, const float* rgba /* [R,4] */,
                   const float* background /* [R,3] */, int64_t num_rays, float huber_delta, float bce_weight,
                   const float* loss_scale_dev, float* d_color /* [R,3] */, float* d_weights_sum /* [R] */,
                   float* loss_out /* [1], accumulated */, void* stream);

/* ------------------------------------------------------------------------------------------
 * tensor_composition_native parity (tensor_composition.cu:120-219): stand-alone fwd/bwd of
 * sum_k feat3D_k * lerp(vector_k, coord_k) on fp16 features, as the reference's extension.
 * ---------------------------------------------------------------------------------------- */
int hrf_compose_tensors_forward(const void* xyz, const void* xyt, const void* yzt, const void* xzt /* half [N,F] */,
                                const float* vectors /* [4,VR,F] */, const float* coords /* [N,4] */,
                                int64_t n, int feature_dim, int vec_res, void* out /* half [N,F] */, void* stream);
int hrf_compose_tensors_backward(const void* xyz, const void* xyt, const void* yzt, const void* xzt,
                                 const float* vectors, const float* coords, const void* d_out, int64_t n,
                                 int feature_dim, int vec_res, void* d_xyz, void* d_xyt, void* d_yzt, void* d_xzt,
                                 float* d_vectors /* zero-initialised by the callee */, void* stream);

/* ------------------------------------------------------------------------------------------
 * Optimiser: fused Adam (run.py:101-104: betas (0.9,0.99), eps 1e-15) over a flat fp32 buffer,
 * optionally refreshing the bf16 shadow copy the forward reads.  grad_scale multiplies the
 * gradient first (1/global_ray_count for data-parallel means).
 * ---------------------------------------------------------------------------------------- */
int hrf_adam_step(float* param, float* exp_avg, float* exp_avg_sq, const float* grad, void* shadow_bf16 /* or NULL */,
                  int64_t n, float lr, float beta1, float beta2, float eps, int step, float grad_scale,
                  void* stream);
int hrf_cast_bf16(const float* src, void* dst_bf16, int64_t n, void* stream);
/* vectors [4, vec_res, 32] -> vectors_t [4, 16, vec_res, 2] (hrf_segment.vectors_t) */
int hrf_transpose_vectors(const float* vectors, float* vectors_t, int vec_res, void* stream);

/* 8-bit tables for inference (HRF_TABLE_INT8X2, DESIGN.md §3.19), from the fp32 masters of one segment.  masters: host
 * array of the 4 grids' device tables [n_entries, 2] (tcnn layout), level_offset / level_size: host [16].  A slice is one
 * (grid, level, feature); its scale s and codes q follow, with every rounding pinned:
 *   s = (c * absmax) / 127 (two fp32 roundings), q = s == 0 ? 0 : clamp(rint(x / s), -127, 127)
 * with the clip ratio c taken from the fixed list {1, 0.9, ..., 0.3} that minimises sum (x - s q)^2 over the slice
 * (float64; ties go to the larger c).
 * Pass one: scale / clip (index into the list) [4][16][2] and sq_err [4][16][2][8] (float64, per candidate), all device;
 * status is device scratch [4][16].  It reads the stream's result back: a non-finite master value fails, naming the
 * segment (`segment`, for the message), grid and level, and nothing else is to be used then. */
#define HRF_QUANT_CLIPS 8
int hrf_quantize_tables_select(const float* const* masters, const uint32_t* level_offset, const uint32_t* level_size,
                               int segment, float* scale, int32_t* clip, double* sq_err, int32_t* status, void* stream);
/* Pass two: the codes of the 4 grids, int8x2 [n_entries] each (codes: host array of 4 device pointers). */
int hrf_quantize_tables_write(const float* const* masters, const uint32_t* level_offset, const uint32_t* level_size,
                              const float* scale /* device [4][16][2] */, void* const* codes, void* stream);
/* The scales folded into the vectors: folded[a][row][2l+f] = s(grid(a), l, f) * vectors[a][row][2l+f], the grid composed
 * with axis a being yzt, xzt, xyt, xyz for a = x, y, z, t.  Then hrf_transpose_vectors(folded) gives vectors_t. */
int hrf_quantize_fold_vectors(const float* vectors, const float* scale /* device [4][16][2] */, int vec_res, float* folded,
                              void* stream);

/* All parameter tensors of a model in ONE launch (the per-tensor entry point above costs one launch per tensor: 23
 * for a single segment).  tensors: device array of descriptors; a tensor whose *active flag is 0 is skipped entirely
 * -- parameters, moments AND its step counter -- which is what torch.optim.Adam does with a parameter whose .grad is
 * None (the reference gives untouched temporal segments no gradient, humanrf.py:162-179, trainer.py:174).  Step
 * counters live on the device (int32 per tensor, incremented here), so a step needs no host decision.  After reading
 * a gradient element the kernel writes 0 back when zero_grad != 0 (the bucket is then clean for the next backward).
 * blob_perm: for the MLP tensors, element i of the tensor is also written as bf16 to shadow[blob_perm[i]] (the packed
 * wgmma weight blob) instead of shadow[i]. */
typedef struct {
  float* param; float* exp_avg; float* exp_avg_sq; float* grad;
  void* shadow_bf16;                 /* or NULL */
  const int32_t* blob_perm;          /* or NULL */
  const int32_t* active;             /* device flag (segment used by this step) or NULL = always active */
  int32_t* step;                     /* device step counter of this tensor */
  int64_t n;
  int64_t first_block;               /* exclusive prefix of ceil(n / HRF_ADAM_BLOCK_ELEMS) over the tensors */
  float* vectors_t;                  /* `vectors` tensors only: the transposed copy to refresh (hrf_segment.vectors_t), or NULL */
  int32_t vec_res;
} hrf_adam_tensor;
#define HRF_ADAM_BLOCK_ELEMS 4096
int hrf_adam_multi(const hrf_adam_tensor* tensors /* device */, int num_tensors, int64_t total_blocks, float lr, float beta1,
                   float beta2, float eps, float grad_scale, int zero_grad, void* stream);

/* ------------------------------------------------------------------------------------------
 * Data-parallel training (SURVEY 8e; the reference is single-GPU, the step wrapped is trainer.py:250-253).
 * One process per GPU.  Gradient buckets and bf16 shadow tables live in peer-visible device memory
 * (hrf_peer_alloc + CUDA IPC handles exchanged by the host side); hrf_dp_reduce_adam is the whole exchange step in one
 * kernel over NVLink peer memory: for this rank's 1/world slice of every sharded tensor it sums the gradient slices of
 * all ranks (P2P loads, rank order), runs Adam on the local fp32 master / moments and stores the refreshed bf16 shadow
 * entries into every rank's shadow buffer (P2P stores); replicated (small) tensors are reduced on every rank.  The
 * caller brackets it with two cross-rank barriers (all gradients complete before; all shadows written / all buckets
 * read after) and clears its own bucket afterwards.
 * ---------------------------------------------------------------------------------------- */
#define HRF_DP_MAX_WORLD 8
int hrf_peer_alloc(int64_t bytes, void** ptr_out);        /* zero-filled, exportable (not from a pooled allocator) */
int hrf_peer_free(void* ptr);
int hrf_peer_export(void* ptr, void* handle_out64 /* 64 bytes, host */);
int hrf_peer_open(const void* handle64, void** ptr_out);  /* a handle exported by ANOTHER process */
int hrf_peer_close(void* ptr);
typedef struct {
  float* grad[HRF_DP_MAX_WORLD];     /* every rank's gradient bucket (own entry = local pointer) */
  void*  shadow[HRF_DP_MAX_WORLD];   /* every rank's flat bf16 shadow buffer */
  int32_t world, rank;
} hrf_dp_peers;
typedef struct {
  float* param; float* exp_avg; float* exp_avg_sq;   /* local tensors, full size (a sharded tensor only touches its slice) */
  int64_t grad_offset;               /* element offset of the tensor inside every gradient bucket */
  int64_t shadow_offset;             /* element offset inside every shadow buffer (sharded tensors), or -1 */
  void* local_shadow_bf16;           /* replicated tensors: local bf16 copy / packed MLP blob, or NULL */
  const int32_t* blob_perm;          /* as hrf_adam_tensor */
  const int32_t* active;
  int32_t* step;
  int64_t n;
  int64_t shard_begin, shard_end;    /* this rank's element range; [0, n) for replicated tensors */
  int64_t first_block;               /* exclusive prefix of ceil((shard_end - shard_begin) / HRF_ADAM_BLOCK_ELEMS) */
  int32_t sharded;
  int32_t vec_res;
  float* vectors_t;                  /* as hrf_adam_tensor */
} hrf_dp_tensor;
/* block_first / block_count: the range of blocks (in the first_block numbering of the descriptor table) this launch
 * covers -- the whole table, or the tensors of one hash grid so that its exchange runs while the next grid's gradient is
 * still being scattered.  advance_steps != 0 on the first launch of a step (it advances the step counters of the active
 * tensors, once). */
int hrf_dp_reduce_adam(const hrf_dp_peers* peers /* host */, const hrf_dp_tensor* tensors /* device */, int num_tensors,
                       int64_t block_first, int64_t block_count, int advance_steps, float lr, float beta1, float beta2,
                       float eps, float grad_scale, void* stream);

/* ------------------------------------------------------------------------------------------
 * Camera poses (and intrinsics) in data-parallel training (DESIGN.md §3.16).  Each rank's hrf_camera_pose_grad /
 * hrf_camera_calib_grad writes one contiguous gradient record of C cameras, 4-byte words:
 *   [pose_grad C x 6 float | intrinsics_grad C x 4 float | ray_count C int32 | error 1 int32]
 * (the intrinsics part is unused without intrinsics).  Every rank then takes the same step from all W records, either
 * read from the peers' memory or gathered into one [W, record] tensor: the two give the same bits.
 *   gradient g_c = (sum over r = 0..W-1, in rank order, of (double)grad_r[c]) / W, in float64 (W = 1: the single-rank
 *                  step's input exactly, so hrf_camera_pose_step / hrf_camera_calib_step's bits);
 *   a camera moves iff some rank's ray_count[c] > 0 and it is not fixed (the union of the ranks' batches);
 *   if any rank's error word is non-zero, nothing is written, and a rank that sees bit 0 (a bad camera number) in
 *   another rank's word sets bit 1 of its own `error` word (sticky, like bit 0).
 * Adam, tables, origins, rotations and this rank's pool slots as hrf_camera_pose_step / hrf_camera_calib_step.
 * ---------------------------------------------------------------------------------------- */
/* Bytes of one gradient record for `num_cameras` cameras (11 C + 1 words), or -1 outside [1, 1024]. */
int64_t hrf_camera_grad_record_bytes(int num_cameras);
typedef struct {
  const void* record[HRF_DP_MAX_WORLD];   /* every rank's record, rank order (device addresses this device can read) */
  int32_t world, rank;                    /* W in [1, 8]; this rank */
} hrf_camera_grad_records;
/* One single-CTA launch; `error` is this rank's own sticky error word (in p2p, the error word of its own record). */
int hrf_camera_pose_step_ranks(const hrf_camera_poses* poses, const hrf_camera_grad_records* records /* host */,
                               int32_t* error /* [1] */, double lr, double beta1, double beta2, double eps,
                               void* stream);
int hrf_camera_calib_step_ranks(const hrf_camera_poses* poses, const hrf_camera_intrinsics* intrinsics,
                                const hrf_camera_grad_records* records /* host */, int32_t* error /* [1] */, double lr,
                                double lr_intrinsics, double beta1, double beta2, double eps, void* stream);

/* ------------------------------------------------------------------------------------------
 * Per-camera colour response refined with the field (toolbox/camera_response.py CameraResponses, DESIGN.md §3.17).
 * Camera c carries a per-channel log gain gamma_c and offset b_c.  With w = weights_sum and fg = color - (1 - w) bg:
 *   pred = color + expm1(gamma) fg + w b   (= e^gamma fg + w b + (1 - w) bg; the background was never seen by a camera)
 * The loss kernel reads the response table [C,6] = ((float)expm1(gamma) x 3, (float)b x 3), written by the step kernels
 * (and by the caller for the initial state).  A channel with em = b = 0 is the identity bit for bit.
 * Gradient record of C cameras, 4-byte words: [response_grad C x 6 float | ray_count C int32 | error 1 int32]. */
int64_t hrf_train_loss_response_workspace_bytes(int num_cameras);    /* -1 outside [1, 1024] */
int64_t hrf_camera_response_record_bytes(int num_cameras);           /* (7 C + 1) * 4, -1 outside [1, 1024] */
/* Two launches.  hrf_train_loss's loss, d_color and d_weights_sum with pred in place of color for the Huber term (the BCE
 * term unchanged), at the response of each ray's camera and the same loss_scale_dev: d_color = g dpred with g = 1 + em,
 * d_weights_sum = the BCE term + sum_k dpred_k (em_k bg_k + b_k).  At identity the outputs are hrf_train_loss's bytes,
 * and the loss takes hrf_train_loss's addends (one atomicAdd per 256 rays, summed by the same tree).  response_grad[c] =
 * (g_k sum_r dpred_k fg_k, sum_r dpred_k w) per channel, summed in a fixed order (the lane tree of hrf_camera_pose_grad,
 * blocks in order, float64 across blocks), and ray_count[c]; written for every camera.  Two runs write identical bytes
 * (loss_out aside: atomics).  A camera number outside [0, num_cameras) sets bit 0 of error[0]; that ray takes the
 * identity and stays out of the sums.  No host synchronisation. */
int hrf_train_loss_response(const float* color /* [R,3] */, const float* weights_sum /* [R] */,
                            const float* rgba /* [R,4] */, const float* background /* [R,3] */,
                            const int32_t* camera_numbers /* [R] */, int64_t num_rays,
                            const float* response_table /* [C,6] */, int num_cameras, float huber_delta,
                            float bce_weight, const float* loss_scale_dev, float* d_color /* [R,3] */,
                            float* d_weights_sum /* [R] */, float* loss_out /* [1] accumulated into, or NULL */,
                            float* response_grad /* [C,6] */, int32_t* ray_count /* [C] */, int32_t* error /* [1] */,
                            void* workspace, void* stream);
typedef struct {
  double* params;                     /* [C,6] (gamma rgb, b rgb) */
  double* exp_avg;                    /* [C,6] */
  double* exp_avg_sq;                 /* [C,6] */
  int32_t* step;                      /* [C] Adam step per camera */
  const uint8_t* fixed;               /* [C] non-zero: the camera is never moved */
  float* table;                       /* [C,6] rewritten for every camera that moves: (expm1(gamma), b) rounded once */
  int num_cameras;                    /* C, 1..1024 */
} hrf_camera_responses;
/* One single-CTA launch: torch.optim.Adam (float64, roundings spelled out as hrf_camera_pose_step's) on (gamma_c, b_c)
 * of every camera with ray_count[c] > 0 that is not fixed, then its table row.  Other cameras keep parameters, moments,
 * step counter and table.  When error is non-NULL and error[0] != 0, nothing is written.  No host read. */
int hrf_camera_response_step(const hrf_camera_responses* responses, const float* response_grad /* [C,6] */,
                             const int32_t* ray_count /* [C] */, const int32_t* error /* [1] or NULL */, double lr,
                             double beta1, double beta2, double eps, void* stream);
/* Data parallel: the step on (sum over r = 0..W-1, in rank order, of (double)response_grad_r) / W, a camera moving iff
 * some rank's ray_count > 0 and it is not fixed; the error rule of hrf_camera_pose_step_ranks (records in the response
 * record's layout, `error` this rank's own sticky word).  W = 1 gives hrf_camera_response_step's bits. */
int hrf_camera_response_step_ranks(const hrf_camera_responses* responses, const hrf_camera_grad_records* records /* host */,
                                   int32_t* error /* [1] */, double lr, double beta1, double beta2, double eps,
                                   void* stream);
/* Rewrites the table row of every camera from its params, with the step kernels' expression (expm1 in float64, rounded
 * once): after parameters are loaded, the table is the one the step would have written.  No host read. */
int hrf_camera_response_write_table(const hrf_camera_responses* responses, void* stream);
/* Applies camera `camera`'s response (its row of response_table) to a rendered image in place: color = color +
 * em (color - (1 - alpha) background) + alpha b per channel.  Identity leaves the bytes unchanged. */
int hrf_camera_response_apply(float* color /* [P,3] */, const float* alpha /* [P] */, int64_t num_pixels,
                              const float* response_table /* [C,6] */, int camera, int num_cameras,
                              const float* background /* [3] device */, void* stream);

/* Held-out response fit (CameraResponses.fit_held_out, DESIGN.md §3.18).  Per camera and channel, the gain g and offset
 * b minimising  sum over the fit pixels of (g f + a b - y / 255)^2 + lambda n ((g - 1)^2 + b^2)  with f the rendered
 * colour, a its alpha (background 0) and y the dataset's 8-bit colour.  Moments row of a camera, float64 [17]:
 *   [n, S_aa, then per channel r, g, b: S_ff, S_fa, S_fy, S_ay, S_yy]   (y the integer 0..255)
 * Every addend is exact in float64, so the only rounding is the summation; n and S_yy are exact integers. */
#define HRF_FIT_OK 0
#define HRF_FIT_TOO_FEW_PIXELS 1      /* n < min_pixels */
#define HRF_FIT_NOT_FINITE 2          /* a gain or offset is inf or NaN (a singular system) */
#define HRF_FIT_GAIN_NOT_POSITIVE 3   /* g <= 0: log g cannot represent it */
#define HRF_FIT_BAD_CAMERA 4          /* the listed camera is outside [0, C) */
int64_t hrf_response_fit_workspace_bytes(int64_t num_pixels);       /* -1 for a negative count */
/* Adds the sums of one view (the pixels with mask != 0) to row `camera` of moments [C,17].  Two launches: block
 * partials from a grid that depends on P alone, then one block adding them in block order into the row.  No float
 * atomics: a rerun writes the same bytes.  A camera outside [0, num_cameras) sets error[0] |= 1 and writes nothing;
 * P = 0 writes nothing.  No host synchronisation. */
int hrf_response_fit_accumulate(const float* color /* [P,3] */, const float* alpha /* [P] */,
                                const uint8_t* gt /* [P,3] */, const uint8_t* mask /* [P] */, int64_t num_pixels,
                                int camera, int num_cameras, double* moments /* [C,17] */, int32_t* error /* [1] */,
                                void* workspace, void* stream);
/* One CTA.  For each listed camera, the three 2x2 systems in float64 by Cramer's rule; report [K,8] = (n, SSE at the
 * identity r g b, SSE at the fit r g b, status), the data SSEs from the moments, and status [K] (HRF_FIT_*).  When every
 * listed camera succeeds, its params (gamma = log g, b) and table row are written and nothing else; otherwise no params
 * or table row at all.  Moments, moments of Adam and step counters are never written.  No host read. */
int hrf_response_fit_solve(const hrf_camera_responses* responses, const double* moments /* [C,17] */,
                           const int32_t* cameras /* [K] */, int num_listed, double lambda, double min_pixels,
                           double* report /* [K,8] */, int32_t* status /* [K] */, void* stream);

/* ------------------------------------------------------------------------------------------
 * Pre-processing that feeds the hot path (SURVEY 8f-4).
 * hrf_occupancy_from_masks: visual-hull carving, replaces occupancy_grid_generation_native.generate_from_masks
 * (actorshq/toolbox/native/occupancy_grid_generation.cu:16-123).  projection_matrices [C,4,4] are stored transposed
 * exactly as the reference passes them (GLM is column-major).
 * hrf_occupancy_union_count: cluster |= (grid == 255); *count_dev = popcount(cluster) -- equations (2)-(4) of
 * humanrf/adaptive_temporal_partitioning.py:11-26 on a bit-packed union (grid_u8 may be NULL to only count).
 * ---------------------------------------------------------------------------------------- */
int hrf_occupancy_from_masks(const uint8_t* masks /* [C, H*W] */, const float* projection_matrices /* [C,4,4] */,
                             const uint8_t* landscape_modes /* [C] bool */, int num_cameras, int camera_coverage_threshold,
                             int grid_resolution, int width, int height, uint8_t* occupancy_grid /* [G,G,G] */, void* stream);
int hrf_occupancy_union_count(void* cluster_bits /* ceil(n/32) u32, caller-zeroed per cluster */, const uint8_t* grid_u8 /* [n] */,
                              int64_t num_voxels, int64_t* count_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * Learned occupancy grid for inference: the trained density field evaluated over the occupied voxels of a hull grid
 * (uint8 [G][G][G] indexed [z][y][x], non-zero = occupied, 255 as hrf_occupancy_from_masks writes it).  The result is a
 * tighter grid in the format hrf_occgrid_add takes.  For every hull voxel (x, y, z):
 *   1. eight sub-sample positions, a, b, c in {0,1}:
 *        px = __fsub_rn(__fdiv_rn((float)x + 0.25f + 0.5f*a, (float)G), 0.5f), and the same for py (b) and pz (c)
 *      (the texture lookup's cell-centred convention: voxel i covers [i/G, (i+1)/G) of p + 0.5);
 *   2. sigma = exactly what hrf_field_forward (mode 0, query form) returns for that position and frame; m = max of the 8;
 *   3. live = (1.f - expf(-m * step) >= alpha_thre), the alpha test of hrf_prune: a voxel is dead only if pruning would
 *      drop every one of its sub-samples;
 *   4. out = hull AND dilate(live), a one-voxel 26-neighbourhood dilation that never leaves the hull, values {0,255};
 *   5. max_sigma (optional, float32 [G^3]) = m on hull voxels, 0 elsewhere.
 * Meant for rendering (step = render_step_size 4e-4, alpha_thre = 1e-4 as hrf_prune is called); training keeps its
 * hull grids.  Reads the sigma part of the MLP blob only, so models with camera embeddings are handled.  The hull's
 * voxel count stays on the device: nothing here synchronises.  G must be in [1, 1024] and the frame inside the
 * model's frame table; a frame of the table that belongs to no segment gives an all-zero grid (the Python entry
 * point rejects it).  workspace: hrf_bake_occupancy_workspace_bytes(G) bytes of device scratch.
 * ---------------------------------------------------------------------------------------- */
int64_t hrf_bake_occupancy_workspace_bytes(int grid_resolution);
int hrf_bake_occupancy(const hrf_field* f, int32_t frame_number, const uint8_t* hull_u8 /* [G^3] */, int grid_resolution,
                       float step, float alpha_thre, uint8_t* out_u8 /* [G^3] */, float* max_sigma /* [G^3] or NULL */,
                       void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------
 * Mesh extraction: a density lattice at the corners of a G^3 grid's voxels, then marching cubes over it.
 *
 * hrf_density_lattice: sigma [(G+1)^3] fp32 indexed [k][j][i] (z, y, x).  Vertex (i, j, k), i, j, k in [0, G], sits at
 *   p = __fsub_rn(__fdiv_rn((float)i, (float)G), 0.5f) per axis: the corners of the voxels of hrf_bake_occupancy's
 *   cell-centred convention, so the cubes of marching cubes are exactly the grid's voxels.  sigma at a vertex that is a
 *   corner of at least one occupied mask voxel (uint8 [G^3], non-zero = occupied; mask NULL = every vertex) is exactly
 *   what hrf_field_forward (mode 0, query form) returns at that position and frame; every other vertex gets 0.  The
 *   vertex count stays on the device: nothing here synchronises.  G in [1, 1024], the frame inside the model's frame
 *   table.  workspace: hrf_density_lattice_workspace_bytes(G) bytes of device scratch.
 *
 * hrf_marching_cubes_count / _emit: the surface {sigma >= level} of any fp32 lattice [(G+1)^3] indexed [k][j][i].
 *   - inside <=> sigma >= level; a lattice edge crosses <=> exactly one endpoint is inside.
 *   - one mesh vertex per crossing lattice edge, owned by its lower endpoint; vertices are numbered in the order
 *     (owner's linear index i + (G+1)(j + (G+1)k), axis x < y < z).  With s0 at the lower endpoint,
 *     t = __fdiv_rn(__fsub_rn(level, s0), __fsub_rn(s1, s0)); the coordinate along the edge's axis is
 *     __fsub_rn(__fdiv_rn(__fadd_rn((float)i, t), (float)G), 0.5f), the other two are the owner's lattice coordinates.
 *     Neighbouring cubes share vertex ids: the mesh is indexed.
 *   - faces (int32 [F,3]) in the order of the cube's linear index, then of the case table; they wind counter-clockwise
 *     seen from the outside (lower sigma): the geometric normal points toward decreasing sigma.
 *   - case table, generated from a face rule: on a cube face with two crossing edges they are joined; with four, the
 *     two edges at each inside corner are joined (inside corners are not connected across a face).  The segments chain
 *     into loops, taken from the smallest unused crossing edge (cube edge e = 4 axis + idx, idx = the other two corner
 *     bits in axis order) and fan-triangulated from their first vertex whose diagonals join no two edges of a common
 *     cube face.  Both cubes sharing a face draw the same segments there, so the mesh is closed wherever the lattice
 *     border is outside.
 *   - normals (optional, fp32 [V,3]): -grad sigma from central differences on the lattice (one-sided at its border),
 *     interpolated along the edge by t, then normalised (0 where the gradient vanishes).
 *   Deterministic: places come from prefix sums, two runs write identical bytes.
 *   _count writes counts[2] = {V, F} (device int64).  The caller reads them back -- the only host synchronisation of an
 *   extraction -- sizes the outputs and calls _emit with the same lattice, level and workspace.  V must fit int32.
 *   workspace: hrf_marching_cubes_workspace_bytes(G) bytes, kept between the two calls.
 * ---------------------------------------------------------------------------------------- */
int64_t hrf_density_lattice_workspace_bytes(int grid_resolution);
int hrf_density_lattice(const hrf_field* f, int32_t frame_number, const uint8_t* mask_u8 /* [G^3] or NULL */,
                        int grid_resolution, float* sigma /* [(G+1)^3] */, void* workspace, void* stream);
int64_t hrf_marching_cubes_workspace_bytes(int grid_resolution);
int hrf_marching_cubes_count(const float* lattice /* [(G+1)^3] */, int grid_resolution, float level,
                             int64_t* counts /* [2] device */, void* workspace, void* stream);
int hrf_marching_cubes_emit(const float* lattice, int grid_resolution, float level, int64_t num_vertices,
                            int64_t num_faces, float* vertices /* [V,3] */, float* normals /* [V,3] or NULL */,
                            int32_t* faces /* [F,3] */, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------
 * Image scores of the ActorsHQ evaluation (actorshq/evaluation/evaluate.py:76-85,117-125) on one pair of 8-bit images.
 * pred, gt: uint8 [H*W*3] RGB, row-major pixels; mask: uint8 [H*W], non-zero = foreground.
 *   ROI : cv2.boundingRect of the pixels with mask != 0, written as roi = {x, y, w, h}; {0, 0, 0, 0} for an empty mask.
 *   PSNR: out[0] = -10 log10(MSE), MSE = sum over masked pixels of sum_c (p_c - g_c)^2 / (3 * 255^2 * masked count);
 *         the sum is exact (int64), the log fp64.  MSE = 0 gives +inf.
 *   SSIM: out[1] = scikit-image's structural_similarity(gt_roi, pred_roi, channel_axis=2) with its defaults for uint8
 *         (data_range 255, 7x7 uniform window, K1 0.01, K2 0.03, sample covariance vx = 49/48 (E[x^2] - E[x]^2)):
 *         S = (2 ux uy + C1)(2 vxy + C2) / ((ux^2 + uy^2 + C1)(vx + vy + C2)), C1 = (0.01*255)^2, C2 = (0.03*255)^2,
 *         averaged over the windows lying wholly inside the ROI (skimage's crop of 3 pixels on every side; its
 *         reflect-mode border never reaches them), then over the 3 channels.  Window sums are exact int32, S is fp64.
 *   NaN : SSIM when the ROI is narrower or shorter than 7 pixels (scikit-image raises there); both for an empty mask.
 * Image bytes are read as the aligned 32-bit words containing them.  Nothing here synchronises: out / roi may be rows
 * of larger device arrays that are read back once after many calls.  Partial sums are folded in a fixed order, so two
 * calls write identical bytes.  width * height * 3 < 2^31.  workspace: hrf_image_metrics_workspace_bytes(width, height)
 * bytes of device scratch, 16-byte aligned.
 * ---------------------------------------------------------------------------------------- */
int64_t hrf_image_metrics_workspace_bytes(int width, int height);
int hrf_image_metrics(const uint8_t* pred /* [H*W*3] RGB */, const uint8_t* gt /* [H*W*3] RGB */,
                      const uint8_t* mask /* [H*W], non-zero = foreground */, int width, int height,
                      double* out /* [2] device: PSNR (dB), SSIM */, int32_t* roi /* [4] device: x, y, w, h */,
                      void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------
 * LPIPS of the ActorsHQ evaluation and the reference trainer's checkpoint choice (evaluate.py:66-73,
 * trainer.py:408-412): lpips.LPIPS(net="alex", version="0.1") called with normalize=True on the ROI crop of both images.
 *   Input: pred, gt [H*W*3] RGB, row-major pixels, dtype 0 = uint8 (v = u / 255.0f, correctly rounded), 1 = float32
 *          (v as given).  roi = device int32 {x, y, w, h} (e.g. what hrf_image_metrics writes), or NULL for the whole
 *          image.  Then x = 2v - 1 and x = (x - shift) / scale in fp32 with IEEE division, shift = (-.030, -.088, -.188),
 *          scale = (.458, .448, .450) as fp32 values of those literals, channels in RGB order.
 *   Trunk: torchvision's alexnet().features[0:12]: conv1 3->64 11x11/4 pad 2, ReLU, maxpool 3/2, conv2 64->192 5x5
 *          pad 2, ReLU, maxpool 3/2, conv3 192->384 3x3 pad 1, ReLU, conv4 384->256, ReLU, conv5 256->256, ReLU (3x3
 *          pad 1).  The five ReLU outputs are the LPIPS layers.  The convolutions are implicit GEMMs on TF32 wgmma:
 *          every operand is rounded to tf32 explicitly (cvt.rna: nearest, ties away from zero), the activations in the
 *          epilogue that writes them (after bias and ReLU) and the input after the scaling above, the weights once when
 *          packed, so the MMA's own truncation changes nothing.  Accumulation, bias and ReLU are fp32.
 *   Tail : per layer k and pixel, f = y / (sqrt(sum_c y^2) + 1e-10) for each image, d = sum_c lin_k[c] (f0 - f1)^2, all
 *          fp32; d is averaged over the layer's H x W (spatial sums folded in fp64) and out[0] = the sum of the five
 *          means (fp64).  This is torch's own precision class: cuDNN convolutions use TF32 by default on Ampere and
 *          later GPUs.
 *   NaN  : out[0] when the ROI is narrower or shorter than 31 pixels (torch raises there: pool2 would be empty), which
 *          includes the empty-mask ROI {0, 0, 0, 0}, and when it does not lie inside the image.
 * No floating-point atomics, every fold in a fixed order: two calls (and a CUDA-graph replay) write identical bytes,
 * swapping pred and gt gives identical bytes and identical images give exactly 0.  Nothing here synchronises: grids
 * are sized from width x height and CTAs outside the ROI exit.  width * height * 3 < 2^31.
 *
 * Weights: hrf_lpips_pack_weights packs torchvision's five OIHW fp32 conv weights (features.{0,3,6,8,10}.weight) into
 * hrf_lpips_packed_bytes() bytes of device memory (16-byte aligned); the layout is private to the library.  bias[k]
 * (features.*.bias) and lin[k] (lpips' lin{k}.model.1.weight, flattened) are fp32 device arrays of 64, 192, 384, 256 and
 * 256 values.
 *
 * workspace: hrf_lpips_workspace_bytes(width, height) bytes of device scratch, 256-byte aligned; about 1.6 GB at
 * 4112x3008 (sized for ROI = whole image).  It holds eight fp32 NHWC tensors, each [2][h][w][C] with image 0 = pred and
 * image 1 = gt and (h, w) the tensor's size for the ROI: input (C = 4, the 4th channel zero), conv1 (64), pool1 (64),
 * conv2 (192), pool2 (192), conv3 (384), conv4 (256), conv5 (256).  Tensor i starts at byte offset
 * sum_{j<i} roundup(2 * H_j * W_j * C_j * 4, 256), with H_j x W_j its size for the whole image; the tail's fp64 per-CTA
 * sums follow.  Sizes: conv1 (n - 7) / 4 + 1, each pool (n - 3) / 2 + 1, every other layer keeps its input's size.
 * ---------------------------------------------------------------------------------------- */
typedef struct hrf_lpips_weights {
  const void* packed;    /* hrf_lpips_packed_bytes() bytes written by hrf_lpips_pack_weights */
  const float* bias[5];  /* conv biases, device fp32 */
  const float* lin[5];   /* lin weights, device fp32 */
} hrf_lpips_weights;
int64_t hrf_lpips_packed_bytes(void);
int hrf_lpips_pack_weights(const float* const* conv_w /* [5] device pointers, OIHW fp32 */, void* packed, void* stream);
int64_t hrf_lpips_workspace_bytes(int width, int height);
int hrf_lpips(const hrf_lpips_weights* weights, const void* pred, const void* gt, int dtype /* 0 uint8, 1 float32 */,
              int width, int height, const int32_t* roi /* device x, y, w, h, or NULL */,
              double* out /* [1] device */, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------
 * Surface distance of one direction between two triangle meshes (DESIGN.md §3.11; restated in numpy in
 * tests/geometry_oracle.py): N points sampled on the source S by area, each queried against the target T.  Vertices
 * fp32 [V*3], faces int32 [F*3], both meshes in the same units.  u = round-to-nearest fp32 operations, each rounded on
 * its own (no FMA contraction).
 *   Eligible face: indices in [0, V) and 0 < |n|^2 < inf for n = e1 x e2, e1 = v1 - v0, e2 = v2 - v0,
 *          n = (e1.y e2.z - e1.z e2.y, e1.z e2.x - e1.x e2.z, e1.x e2.y - e1.y e2.x), |n|^2 = (n.x^2 + n.y^2) + n.z^2.
 *          Ineligible faces are never sampled and never a target.  area = 0.5 sqrt(|n|^2), n^ = n / sqrt(|n|^2).
 *   Sampling: q_f = floor(area_f / area_max * 2^32) (uint64; division in fp64; area_max = largest eligible area;
 *          q_f = 0 when ineligible), P = exclusive prefix sum of q, Q = sum of q.  Sample k (0 <= k < N) draws
 *          x_j = splitmix64(seed * 2^40 + 3k + j), j = 0, 1, 2 (uint64 arithmetic; splitmix64(x): z = x +
 *          0x9E3779B97F4A7C15, z = (z ^ z >> 30) * 0xBF58476D1CE4E5B9, z = (z ^ z >> 27) * 0x94D049BB133111EB,
 *          z ^ z >> 31).  Its face is the f with P_f <= mulhi64(x_0, Q) < P_f + q_f; u1 = (x_1 >> 40) 2^-24,
 *          u2 = (x_2 >> 40) 2^-24, r = sqrt(u1), w0 = 1 - r, w1 = r (1 - u2), w2 = r u2 and per component
 *          p = (w0 v0 + w1 v1) + w2 v2.
 *   Distance: d2(p, t) = Ericson's closest point on a triangle (Real-Time Collision Detection §5.1.5) in fp32, its
 *          point clamped per component into the triangle's bounding box, then |p - q|^2 = (e.x^2 + e.y^2) + e.z^2.
 *          closest = the eligible target face of least d2, the lowest face id on ties; d = sqrt(d2).  Both equal a
 *          brute-force scan bit for bit (the tree prunes a node only when a lower bound, rounded down, is strictly
 *          greater than the best d2 so far).  Normal term: |n^_S(face_k) . n^_T(closest)|.
 *   Scores: out = {sum d, sum d^2, sum normal term} / N in fp64 (d^2 of the fp32 d, exact in fp64), partial sums per
 *          CTA folded in a fixed order; counts[i] = #{k : d_k <= taus[i]} (fp32 comparison), num_taus <= 8.
 *          out = NaN and counts = -1 when *error != 0, when S or T has no eligible face (Q = 0), or F = 0.
 *   error: device int32, bit 0 = a source face index outside [0, V), bit 1 = a target one; such faces are ineligible
 *          and their vertices are never read.
 * Optional per-sample outputs (device, nullable): points [N*3], sample_faces [N], distances [N] (+inf when T has no
 * eligible face, NaN when S has none) and closest_faces [N] (-1 when none).  No floating-point atomics, no host
 * synchronisation: two calls (and a CUDA-graph replay) write identical bytes.  F < 2^31, 1 <= N < 2^31.  taus is a host
 * array.  workspace: hrf_mesh_distance_workspace_bytes(F_src, F_tgt, N, num_taus) bytes of device scratch (0 = bad
 * sizes), 256-byte aligned.
 * ---------------------------------------------------------------------------------------- */
int64_t hrf_mesh_distance_workspace_bytes(int64_t num_src_faces, int64_t num_tgt_faces, int64_t num_samples,
                                          int num_taus);
int hrf_mesh_distance(const float* src_vertices, int64_t num_src_vertices, const int32_t* src_faces,
                      int64_t num_src_faces, const float* tgt_vertices, int64_t num_tgt_vertices,
                      const int32_t* tgt_faces, int64_t num_tgt_faces, int64_t num_samples, uint64_t seed,
                      const float* taus /* host [num_taus] */, int num_taus, double* out /* [3] device */,
                      int64_t* counts /* [num_taus] device */, int32_t* error /* [1] device */, float* points,
                      int32_t* sample_faces, float* distances, int32_t* closest_faces, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------
 * Mesh rasterisation into a depth map and a mask: the outputs of the ActorsHQ toolbox's mesh renderer
 * (mesh_tools/renderer: camera-space z of an RDF camera, GL_LESS, no culling, 0 on background), deterministic and
 * exact (DESIGN.md §3.12; restated in numpy in tests/raster_oracle.py).  Vertices fp32 [V*3], faces int32 [F*3].
 * world2cam = host fp64 [12], row-major 3x4 (the host takes (inv(cam2world) diag(s, s, s, 1))[:3] in fp64); fxW, fyH,
 * cxW, cyH = focal length and principal point in pixels, the principal point measured from the image's corner.  Every
 * fp64 operation below is rounded to nearest on its own (no contraction).
 *   1 Vertex: p in fp64; X = ((m00 p.x + m01 p.y) + m02 p.z) + m03, Y and Z likewise with rows 1 and 2;
 *          u = (fxW X) / Z + cxW, v = (fyH Y) / Z + cyH; U = rint(256 u), V = rint(256 v) (ties to even) as integers.
 *          A vertex is out when !(near <= Z <= DBL_MAX) or !(|256 u| <= 2^29 and |256 v| <= 2^29) (NaN included).
 *   2 Faces that draw nothing (their vertices are never read, or read only for the check): a face with an index
 *          outside [0, V) (sets error bit 0); a face with a vertex out (a documented divergence from GL, which clips;
 *          counted in *skipped); a face with A = (U1 - U0)(V2 - V0) - (V1 - V0)(U2 - U0) = 0; a face whose clipped box
 *          is empty: pixel columns ceil((min U - 128) / 256) .. floor((max U - 128) / 256) within [0, width), rows
 *          likewise within [0, height).
 *   3 Coverage: pixel (x, y) (column x, row y, row 0 at the top) samples S = (256 x + 128, 256 y + 128), the pixel
 *          centre.  Edge k runs from vertex k+1 to vertex k+2 (indices mod 3), d_k = v_{k+2} - v_{k+1},
 *          E_k = sgn(A) (d_k.x (S.y - v_{k+1}.y) - d_k.y (S.x - v_{k+1}.x)), exact in int64 (every product < 2^60), so
 *          E_0 + E_1 + E_2 = |A| and both windings draw.  S is covered when for every k: E_k > 0, or E_k = 0 and
 *          P(sgn(A) d_k) with P(d) = d.y > 0 or (d.y = 0 and d.x < 0).  P(d) != P(-d): of two faces on opposite sides
 *          of a shared edge exactly one covers a sample on it, and a closed fan covers its centre once.
 *   4 Depth: b_k = (double)E_k / (double)|A|, z = (float)(1 / ((b_0 / Z_0 + b_1 / Z_1) + b_2 / Z_2)): the
 *          perspective-correct camera z of the face's plane along the pixel's ray.  A covered sample is a fragment
 *          when near <= z <= far (z as fp64).
 *   5 Visibility: each pixel keeps the least key (float bits of z) << 32 | face over its fragments: the nearest
 *          face, on equal z the lowest face id (GL_LESS in draw order).  Integer atomics only: two calls (and a
 *          CUDA-graph replay) write identical bytes.
 * Outputs [height*width], row-major: z fp32 (0 without a fragment), mask uint8 (255 / 0), face int32 (-1; nullable),
 * hits int32 (the number of faces of step 3 that cover the pixel centre, before the near / far test; nullable).
 * error: device int32, bit 0 as above.  skipped: device int64.  No host synchronisation.  F < 2^31,
 * width * height < 2^31, 0 < near <= far < inf.  workspace: hrf_rasterize_mesh_workspace_bytes(V, F, width, height)
 * bytes of device scratch (0 = bad sizes), 256-byte aligned; O(V + F + width * height).
 * ---------------------------------------------------------------------------------------- */
int64_t hrf_rasterize_mesh_workspace_bytes(int64_t num_vertices, int64_t num_faces, int width, int height);
int hrf_rasterize_mesh(const float* vertices, int64_t num_vertices, const int32_t* faces, int64_t num_faces,
                       const double* world2cam /* host [12] */, double fxW, double fyH, double cxW, double cyH,
                       int width, int height, double near, double far, float* z, uint8_t* mask, int32_t* face,
                       int32_t* hits, int32_t* error /* [1] device */, int64_t* skipped /* [1] device */,
                       void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------
 * Depth and mask scores of a depth map against a reference (DESIGN.md §3.12).  pred_z, ref_z fp32 [N]; pred_mask,
 * ref_mask uint8 [N], non-zero = foreground.  B = pixels where both masks are set; for a pixel of B,
 * d = (double)pred - (double)ref (rounded to nearest).  Per CTA in fp64, folded by one CTA in a fixed order:
 *   out[0] = sum d / n (bias), out[1] = sum |d| / n (MAE), out[2] = sqrt(sum d^2 / n) (RMSE),
 *   out[3] = sum (|d| / ref) / n (AbsRel), n = |B|;
 *   counts (int64) = {n, |P|, |R|, |P and R|, |P or R|, #{|d| <= taus[i]} for i < num_taus (fp64 comparison)}.
 * A pixel of B with a z on either side that is not finite and > 0 sets error bit 0 and is left out of the sums.
 * out = NaN when *error != 0 or n = 0; counts are always written.  No floating-point atomics, no host synchronisation
 * (out and counts may be rows of larger arrays): two calls write identical bytes.  1 <= N < 2^31, num_taus <= 8, taus
 * a host array.  workspace: hrf_depth_metrics_workspace_bytes(N) bytes of device scratch (0 = bad size), 16-byte
 * aligned.
 * ---------------------------------------------------------------------------------------- */
int64_t hrf_depth_metrics_workspace_bytes(int64_t num_pixels);
int hrf_depth_metrics(const float* pred_z, const uint8_t* pred_mask, const float* ref_z, const uint8_t* ref_mask,
                      int64_t num_pixels, const double* taus /* host [num_taus] */, int num_taus,
                      double* out /* [4] device */, int64_t* counts /* [5 + num_taus] device */,
                      int32_t* error /* [1] device */, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------
 * Error map of the training pool (toolbox/error_map.py ErrorMap, DESIGN.md §3.20): a running per-tile colour error of
 * every pooled image, fed by the fused train step, from which the loader draws the next batch's pool indices.
 * Pool pixel slot * P + p (P = W H).  Its (x, y) is the sampler's: a slot with landscape_modes[slot] != 0 is W wide and
 * H high, any other slot H wide and W high; x = p % width, y = p / width.  Tiles are T x T pixels in the slot's own
 * orientation, row-major, ceil(width / T) per row: every slot has ceil(W/T) ceil(H/T) tiles, tile t of slot s is global
 * tile s * tiles_per_slot + t, and a border tile holds npix = min(T, width - x0) min(T, height - y0) pixels.
 * Every entry is asynchronous on `stream` and reads nothing back to the host.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  const uint8_t* landscape_modes;     /* [B] device: the loader's landscape_mode_cuda */
  int64_t num_slots;                  /* B */
  int32_t image_width;                /* W, as the sampler takes it */
  int32_t image_height;               /* H */
  int32_t tile;                       /* T, 1..4096 */
} hrf_error_map_geometry;
/* B ceil(W/T) ceil(H/T), or -1 for a bad geometry or one where the total weight could reach 2^63 with every EMA and the
 * floor at most max(max_ema, 1) (pass max(prior, floor): the EMA of values below 1 started at the prior never exceeds
 * max(prior, 1)). */
int64_t hrf_error_map_num_tiles(const hrf_error_map_geometry* geometry, float max_ema);
int64_t hrf_error_map_workspace_bytes(int64_t num_tiles);          /* 8 ceil(tiles / 2048), -1 for tiles < 1 */
/* One launch.  Per ray, e_r = h_0 + h_1 + h_2 (fp32, in channel order) with h_k hrf_train_loss's Huber value of
 * channel k before its 1 / (3R) and loss_scale, rounded as that kernel is compiled: gt = fma(m, rgb_k, (1 - m) bg_k),
 * x = color_k - gt, h = (x / 2) x when |x| < delta, else (|x| - delta / 2) delta.  With response_table (then
 * camera_numbers and weights_sum too) it is hrf_train_loss_response's value as that kernel is compiled: color_k is first
 * taken through the ray's camera response (a camera outside [0, num_cameras) takes the identity), and
 * gt = fma(1 - m, bg_k, m rgb_k).  q_r = min(rint(e_r 2^32),
 * 2^32 - 1) (NaN: the cap) is added into tile_sum of the ray's tile and tile_count += 1 (integer atomics: the result
 * does not depend on scheduling).  A pixel outside [0, B P) sets bit 0 of error[0] and the ray is skipped. */
int hrf_error_map_accumulate(const float* color /* [R,3] */, const float* weights_sum /* [R] or NULL */,
                             const float* rgba /* [R,4] */, const float* background /* [R,3] */,
                             const int64_t* pixels /* [R] pool indices */, int64_t num_rays,
                             const float* response_table /* [C,6] or NULL */, const int32_t* camera_numbers /* [R] */,
                             int num_cameras, float huber_delta, const hrf_error_map_geometry* geometry,
                             uint64_t* tile_sum /* [tiles] */, uint32_t* tile_count /* [tiles] */,
                             int32_t* error /* [1] */, void* stream);
/* Three launches.  Every tile with count > 0: m = (float)((double)sum / count 2^-32), ema = fma(beta, m - ema, ema),
 * sum = count = 0; other tiles keep their ema.  Then w_t = rint(max(ema_t, floor) npix_t 2^24) (exact in double) and
 * cdf = the inclusive scan of w over all tiles (integer, exact).  beta in (0, 1], floor >= 2^-24 (every w_t >= 1), and a
 * floor for which hrf_error_map_num_tiles(geometry, floor) >= 0.
 * workspace: hrf_error_map_workspace_bytes(tiles) bytes. */
int hrf_error_map_update(const hrf_error_map_geometry* geometry, float* ema /* [tiles] */,
                         uint64_t* tile_sum /* [tiles] */, uint32_t* tile_count /* [tiles] */, float beta,
                         float floor_weight, uint64_t* cdf /* [tiles] */, void* workspace, void* stream);
/* One launch.  With key = s(s(seed) ^ counter), s(x) the SplitMix64 finaliser of x + 0x9E3779B97F4A7C15, and
 * h(r, k) = s(key ^ (4 r + k)): rays r < floor(uniform_fraction R) take out[r] = umulhi(h(r, 0), B P); every other ray
 * takes tile t = upper_bound(cdf, umulhi(h(r, 0), cdf[tiles - 1])) (the first tile whose CDF exceeds it) and pixel
 * k = umulhi(h(r, 1), npix_t) of that tile, row-major inside it. */
int hrf_error_map_draw(const uint64_t* cdf /* [tiles] */, const hrf_error_map_geometry* geometry, uint64_t seed,
                       uint64_t counter, int64_t num_rays, double uniform_fraction, int64_t* out /* [R] */,
                       void* stream);
/* ema = prior on every tile of slots [first_slot, first_slot + num_slots), one launch over those tiles only.  The CDF
 * (and so the draw) changes at the next update. */
int hrf_error_map_reset_slots(const hrf_error_map_geometry* geometry, int64_t first_slot, int64_t num_slots,
                              float prior, float* ema /* [tiles] */, void* stream);

/* ------------------------------------------------------------------------------------------
 * Occupancy grids of the training sampler learned while training (toolbox/training_occupancy.py TrainingOccupancy,
 * DESIGN.md §3.21).  Per frame f, from its hull (uint8 [G][G][G] indexed [z][y][x], non-zero = occupied):
 *   1. ids: the hull's voxel indices z G^2 + y G + x, int32, ascending (hrf_training_occupancy_compact).  The caller
 *      reads the device count back once per newly seen frame to size ids and bound.
 *   2. bound: float32 per listed voxel, starting at +inf (a voxel never evaluated is live).
 *   3. evaluate (refresh counter c, seed s; hrf_training_occupancy_update):
 *        key = S(S(S(s) ^ f) ^ c) (hrf_training_occupancy_key), S the SplitMix64 finaliser of x + 0x9E3779B97F4A7C15,
 *        h = S(key ^ id), g = S(h); u_x = (h >> 40) 2^-24, u_y = ((h >> 16) & (2^24 - 1)) 2^-24, u_z = (g >> 40) 2^-24;
 *        px = __fsub_rn(__fdiv_rn(__fadd_rn((float)x, u_x), (float)G), 0.5f), the same for y and z (the bake's
 *        cell-centred convention with a hashed offset; the rounding of x + u_x can put the point on the voxel's upper
 *        face);
 *        sigma = exactly what hrf_field_forward (mode 0, query form) returns at p and frame f;
 *        bound = !isfinite(sigma) ? +inf : isinf(bound) ? sigma : fmaxf(__fmul_rn(decay, bound), sigma).
 *   4. pack (hrf_training_occupancy_pack): live <=> 1.f - expf(-bound * step) >= alpha_thre (the bake's alpha test);
 *      grid = hull AND dilate(live), a 26-neighbourhood dilation by one voxel that never leaves the hull, the hull
 *      rebuilt from ids; written in place into an occupancy ring slot (the handle of hrf_occgrid_add, ceil(G^3 / 32)
 *      words) in hrf_occgrid_add's bit layout: voxel i is bit i & 31 of word i >> 5.  The ring does not advance.
 * G in [1, 1024].  Every entry is asynchronous on `stream` and reads nothing back.  workspace:
 * hrf_training_occupancy_workspace_bytes(G) bytes of device scratch, shared by compact and pack.
 * ---------------------------------------------------------------------------------------- */
uint64_t hrf_training_occupancy_key(uint64_t seed, int32_t frame_number, uint64_t counter);
int64_t hrf_training_occupancy_workspace_bytes(int grid_resolution);
/* Writes *count (device int32) and, when ids is not NULL, the ids (capacity: the count). */
int hrf_training_occupancy_compact(const uint8_t* hull_u8 /* [G^3] */, int grid_resolution, int32_t* ids /* or NULL */,
                                   int32_t* count /* [1] device */, void* workspace, void* stream);
/* One launch over the num_ids listed voxels (num_ids: the count compact wrote, which `count` holds on the device).
 * points (optional, float32 [num_ids, 3]) receives p.  Needs a bf16-table field and the frame inside its frame table;
 * decay in (0, 1]. */
int hrf_training_occupancy_update(const hrf_field* f, int32_t frame_number, int grid_resolution,
                                  const int32_t* ids /* [num_ids] */, const int32_t* count /* [1] device */,
                                  int64_t num_ids, uint64_t seed, uint64_t counter, float decay,
                                  float* bound /* [num_ids] */, float* points /* [num_ids, 3] or NULL */, void* stream);
/* counts (optional, int64 [2] device): {live voxels, set bits of the grid}. */
int hrf_training_occupancy_pack(const int32_t* ids /* [num_ids] */, const float* bound /* [num_ids] */,
                                int64_t num_ids, int grid_resolution, float step, float alpha_thre,
                                uint32_t* slot_bits /* [ceil(G^3 / 32)] */, int64_t* counts /* [2] or NULL */,
                                void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------
 * Self tests (used by tests/ only): one 128xN x K (or 64xNxK) wgmma with caller-chosen descriptor
 * fields, to pin the shared-memory descriptor encoding on real hardware.
 * ---------------------------------------------------------------------------------------- */
int hrf_selftest_umma(const void* a_bf16 /* [M,K] row-major */, const void* b_bf16 /* [N,K] row-major */,
                      float* d /* [M,N] */, int m /* 64 or 128 */, int n /* 16, 32, 48 or 64 */, int k,
                      /* physical placement of the 8x8 core matrices in shared memory (bytes) */
                      uint32_t a_kstride, uint32_t a_mstride, uint32_t b_kstride, uint32_t b_nstride,
                      /* descriptor fields (bytes) */
                      uint32_t a_lbo, uint32_t a_sbo, uint32_t b_lbo, uint32_t b_sbo,
                      int mn_major /* bit 0: A is MN-major, bit 1: B is MN-major */, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* HUMANRF_B200_H_ */
