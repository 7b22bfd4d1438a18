"""HumanRF scene representation backed by the fused sm_90a kernels.

Drop-in for humanrf/scene_representation/humanrf.py:14-220 (+ decomposition4d.py:41-135): same
constructor kwargs, ``density`` / ``forward`` / ``get_params``, same state-dict keys

    feature_grids.{s}.vectors                              [4, 2048, 32] fp32
    feature_grids.{s}.{xyz,xyt,yzt,xzt}_encoding.params    flat fp32 (tcnn layout: level-major, 2 features/entry)
    sigma_net.params / color_net.params                    flat fp32 (tcnn FullyFusedMLP row-major [out,in] per layer)
    frame_numbers_to_segment_numbers / frame_numbers_to_normalized_local_frame_numbers (buffers)

so checkpoints written by the reference trainer load unchanged (trainer.py:528-620).  What is
different by design: tables are read by the kernels from bf16 shadow copies of the fp32 master
parameters (refreshed whenever a parameter's version changes); all segments stay resident in
HBM (the reference off-loads idle segments to the host, humanrf.py:169-179; a 50-frame segment with its
optimiser state takes about 0.5 GB of the GPU's 80 GB); encode -> MLP runs in one kernel instead of 4 tcnn encodings + compose + 2 tcnn nets.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Tuple

import numpy as np
import torch

from .. import _lib as L
from .grid_layout import (MLP_BLOB_ELEMS, MLP_SIGMA_PARAMS, GridLayout, color_in_width, mlp_blob_permutation,
                          mlp_color_params, mlp_layers, segment_log2_hashmap_size)
from .query_io import QueryInput, QueryOutput

GRID_NAMES = ("xyz_encoding", "xyt_encoding", "yzt_encoding", "xzt_encoding")  # decomposition4d.py:126-129


class _FlatParams(torch.nn.Module):
    """Stands in for a tcnn module: a single flat fp32 ``params`` (tcnn bindings/torch/modules.py)."""

    def __init__(self, init: torch.Tensor):
        super().__init__()
        self.params = torch.nn.Parameter(init)


class Decomposition4D(torch.nn.Module):
    """Parameter container mirroring decomposition4d.py:41-122 (4 hash grids + 4 dense 1-D vector tables)."""

    def __init__(self, ngp_n_levels=16, ngp_n_features_per_level=2, ngp_log2_hashmap_size=19, ngp_base_resolution=32,
                 ngp_finest_resolution=2048, vectors_finest_resolution=2048):
        super().__init__()
        if ngp_n_levels != 16 or ngp_n_features_per_level != 2:
            raise NotImplementedError("the sm_90a kernels are specialised for n_levels=16, n_features_per_level=2")
        self.layout = GridLayout(ngp_log2_hashmap_size, ngp_n_levels, ngp_base_resolution, ngp_finest_resolution)
        feature_size = ngp_n_levels * ngp_n_features_per_level
        self.vectors = torch.nn.Parameter(torch.randn((4, vectors_finest_resolution, feature_size)) * 0.1)  # :76-78
        for name in GRID_NAMES:
            # tcnn GridEncoding initialises U(-1e-4, 1e-4)
            init = (torch.rand(self.layout.n_params) * 2 - 1) * 1e-4
            setattr(self, name, _FlatParams(init))

    def grids(self) -> List[torch.nn.Parameter]:
        return [getattr(self, n).params for n in GRID_NAMES]


def _xavier_flat(shapes, gen=None) -> torch.Tensor:
    out = []
    for o, i in shapes:
        a = float(np.sqrt(6.0 / (i + o)))
        out.append(((torch.rand((o, i), generator=gen) * 2 - 1) * a).reshape(-1))
    return torch.cat(out)


class HumanRF(torch.nn.Module):
    def __init__(self, density_scale: float, sorted_frame_numbers: Tuple[int, ...], n_features_per_level: int,
                 log2_hashmap_size: int, n_levels: int, coarsest_resolution: int, finest_resolution: int,
                 geometry_feature_dim: int, n_neurons: int, n_hidden_layers_density: int, n_hidden_layers_color: int,
                 sh_degree: int, segment_sizes: Tuple[int, ...], camera_embedding_dim: int, **kwargs):
        super().__init__()
        if (n_neurons, geometry_feature_dim, n_hidden_layers_density, n_hidden_layers_color, sh_degree) != (64, 15, 1, 2, 4):
            raise NotImplementedError(
                "the fused sm_90a kernel is specialised for the reference defaults (model_args.py:10-19): "
                "n_neurons=64, geometry_feature_dim=15, 1/2 hidden layers, sh_degree=4")
        if not 0 <= camera_embedding_dim <= 17:
            raise NotImplementedError("camera_embedding_dim must be in [0, 17] (16 SH + 15 geometry + E <= 48 inputs)")
        self.density_scale = float(density_scale)
        self.num_frames = len(sorted_frame_numbers)
        self.sorted_frame_numbers = tuple(int(f) for f in sorted_frame_numbers)
        self.num_segments = len(segment_sizes)
        self.segment_sizes = tuple(int(s) for s in segment_sizes)
        self.log2_hashmap_size = int(log2_hashmap_size)
        self.coarsest_resolution, self.finest_resolution = int(coarsest_resolution), int(finest_resolution)
        self.camera_embedding_dim = camera_embedding_dim
        if camera_embedding_dim > 0:
            self.camera_embeddings = torch.nn.Embedding(160, camera_embedding_dim)  # humanrf.py:75-76

        # humanrf.py:79-103
        end = np.cumsum(segment_sizes, dtype=np.int32)
        end[-1] = min(end[-1], self.num_frames)
        start = np.concatenate((np.zeros(1, dtype=np.int32), end[:-1]))
        f2s = np.full((sorted_frame_numbers[-1] + 1), fill_value=-1, dtype=np.int32)
        f2t = np.full((sorted_frame_numbers[-1] + 1), fill_value=-1, dtype=np.float32)
        for s in range(self.num_segments):
            frames = [sorted_frame_numbers[j] for j in range(start[s], end[s])]
            for local, frame in enumerate(frames):
                f2s[frame] = s
                f2t[frame] = local / len(frames)
        self.register_buffer("frame_numbers_to_segment_numbers", torch.from_numpy(f2s))
        self.register_buffer("frame_numbers_to_normalized_local_frame_numbers", torch.from_numpy(f2t))

        self.feature_grids = torch.nn.ModuleList()
        for segment_size in segment_sizes:
            self.feature_grids.append(Decomposition4D(
                ngp_n_levels=n_levels, ngp_n_features_per_level=n_features_per_level,
                ngp_log2_hashmap_size=segment_log2_hashmap_size(segment_size, log2_hashmap_size),
                ngp_base_resolution=coarsest_resolution, ngp_finest_resolution=finest_resolution,
                vectors_finest_resolution=finest_resolution))
        self.total_feature_dim = n_levels * n_features_per_level
        layers = mlp_layers(camera_embedding_dim)
        self.sigma_net = _FlatParams(_xavier_flat(layers[:2]))
        self.color_net = _FlatParams(_xavier_flat(layers[2:]))
        assert self.sigma_net.params.numel() == MLP_SIGMA_PARAMS
        assert self.color_net.params.numel() == mlp_color_params(camera_embedding_dim)
        self._native: Optional[_NativeField] = None

    # ------------------------------------------------------------------ reference API
    def density(self, query_input: QueryInput) -> QueryOutput:
        """sigma and the geometry features.  When ``query_input.positions`` requires grad, the backward also returns
        d(positions) [N,3] (hrf_field_position_grad): the exact derivative of what the kernels compute, grid and vector
        terms both, with the bf16 rounding of the composed features treated as the identity.  First-order only
        (``create_graph=True`` is not supported)."""
        needs_grad = self._needs_grad(query_input.positions)
        active = (self.active_segment_list(query_input.frame_numbers, query_input.unique_frame_numbers)
                  if self._needs_grad() else None)
        sigma, geo, _ = _FieldFunction.apply(self, 0, query_input.positions, None, query_input.frame_numbers, None,
                                             needs_grad, active, *self.hot_parameters())
        return QueryOutput(density=sigma, geometry_features=geo)

    def forward(self, query_input: QueryInput) -> QueryOutput:
        # humanrf.py:194-204: the camera embedding is looked up while training and is all zeros otherwise
        cams = query_input.camera_numbers if (self.camera_embedding_dim > 0 and query_input.is_training) else None
        # d(positions) as in density(); the radiance reaches the positions through the geometry features.  d(directions)
        # when they require grad: the SH encoding's input gradient (hrf_field_backward_mlp_dirs)
        needs_grad = self._needs_grad(query_input.positions, query_input.directions)
        active = (self.active_segment_list(query_input.frame_numbers, query_input.unique_frame_numbers)
                  if self._needs_grad() else None)
        sigma, geo, rgb = _FieldFunction.apply(self, 1, query_input.positions, query_input.directions,
                                               query_input.frame_numbers, cams, needs_grad, active, *self.hot_parameters())
        return QueryOutput(density=sigma, geometry_features=geo, radiance=rgb)

    def active_segment_list(self, frame_numbers, unique_frame_numbers=None) -> Optional[List[bool]]:
        """Which temporal segments a batch touches (humanrf.py:162-163), as a host list; None for a single-segment
        model (nothing to decide, no host sync).  The reference only runs -- and so only gives a gradient to -- these
        segments; `unique_frame_numbers` is the per-ray set the DataLoader provides (data_loader.py:648)."""
        if self.num_segments == 1:
            return None
        from ..parallel import active_segments

        src = unique_frame_numbers if unique_frame_numbers is not None else frame_numbers
        return active_segments(self.frame_numbers_to_segment_numbers, src, self.num_segments).cpu().tolist()

    def _needs_grad(self, *inputs: Optional[torch.Tensor]) -> bool:
        # ctx.needs_input_grad ignores torch.no_grad(); decide outside whether to save the backward buffers.  Inputs
        # (positions, directions, rays) that require grad count too: their gradients need the same saved features.
        if not torch.is_grad_enabled():
            return False
        return any(t is not None and t.requires_grad for t in inputs) or any(p.requires_grad for p in self.hot_parameters())

    def get_params(self, lr):
        params = [
            {'params': self.feature_grids.parameters(), 'lr': lr},
            {'params': self.sigma_net.parameters(), 'lr': lr},
            {'params': self.color_net.parameters(), 'lr': lr},
        ]
        if self.camera_embedding_dim > 0:
            params.append({'params': self.camera_embeddings.parameters(), 'lr': lr})
        return params

    @property
    def device(self) -> torch.device:
        return self.sigma_net.params.device

    # ------------------------------------------------------------------ native plumbing
    def hot_parameters(self) -> List[torch.nn.Parameter]:
        """Per segment: 4 grids + vectors; then sigma and colour MLP parameters; then the camera embedding table
        if there is one (gradient order)."""
        ps: List[torch.nn.Parameter] = []
        for fg in self.feature_grids:
            ps += fg.grids() + [fg.vectors]
        ps += [self.sigma_net.params, self.color_net.params]
        if self.camera_embedding_dim > 0:
            ps.append(self.camera_embeddings.weight)
        return ps

    @property
    def mlp_grad_elems(self) -> int:
        return MLP_SIGMA_PARAMS + mlp_color_params(self.camera_embedding_dim)

    def native(self) -> "_NativeField":
        if self._native is None:
            self._native = _NativeField(self)
        self._native.refresh()
        return self._native

    def invalidate_native(self) -> None:
        """Forces the next native() to re-cast every bf16 shadow table and repack the MLP blob.  refresh() follows the
        parameters' autograd version counters; a write through `p.data` or a raw pointer does not move them."""
        if self._native is not None:
            self._native.versions = None


class _NativeField:
    """Device-side view of a HumanRF module: bf16 shadow tables, packed MLP blob, descriptors."""

    def __init__(self, model: HumanRF):
        self.model = model
        self.keys = None
        self.versions = None
        self.shadows: List[torch.Tensor] = []
        self.blob: Optional[torch.Tensor] = None
        self.perm: Optional[torch.Tensor] = None
        self.seg_dev: Optional[torch.Tensor] = None
        self.field = L.Field()

    def _device(self) -> torch.device:
        dev = self.model.sigma_net.params.device
        if dev.type != "cuda":
            raise RuntimeError("humanrf_b200: the scene representation must live on a CUDA device "
                               "(there is no CPU path); call .to('cuda') first")
        return dev

    def refresh(self) -> None:
        m = self.model
        dev = self._device()
        params = m.hot_parameters()
        keys = tuple(p.data_ptr() for p in params) + (m.frame_numbers_to_segment_numbers.data_ptr(),)
        rebuild = keys != self.keys
        lib = L.lib()
        if rebuild:
            for p in params:
                if p.device != dev or p.dtype != torch.float32 or not p.is_contiguous():
                    raise RuntimeError("humanrf_b200: parameters must be contiguous fp32 CUDA tensors on one device")
            self.shadows = []
            self.vec_t = []     # transposed fp32 copies of `vectors`, [4][16][VR][2]: what the gradient scatter reads
            for fg in m.feature_grids:
                self.shadows.append([torch.empty(g.numel(), dtype=torch.bfloat16, device=dev) for g in fg.grids()])
                self.vec_t.append(torch.empty(fg.vectors.numel(), dtype=torch.float32, device=dev))
            self.blob = torch.zeros(MLP_BLOB_ELEMS, dtype=torch.bfloat16, device=dev)
            dst, src = mlp_blob_permutation(m.camera_embedding_dim)
            self.perm = (torch.from_numpy(dst).to(dev), torch.from_numpy(src).to(dev))
            segs = (L.Segment * m.num_segments)()
            for s, fg in enumerate(m.feature_grids):
                lay = fg.layout
                for k in range(4):
                    segs[s].grid[k] = self.shadows[s][k].data_ptr()
                segs[s].vectors = fg.vectors.data_ptr()
                segs[s].vectors_t = self.vec_t[s].data_ptr()
                for l in range(16):
                    segs[s].level_offset[l] = int(lay.offset[l])
                    segs[s].level_size[l] = int(lay.size[l])
                segs[s].hashed_mask = lay.hashed_mask
                segs[s].n_entries = lay.n_entries
            raw = np.frombuffer(bytes(segs), dtype=np.uint8).copy()
            self.seg_dev = torch.from_numpy(raw).to(dev)
            lay0 = m.feature_grids[0].layout
            f = self.field
            f.segments = self.seg_dev.data_ptr()
            f.frame_to_segment = m.frame_numbers_to_segment_numbers.data_ptr()
            f.frame_to_tlocal = m.frame_numbers_to_normalized_local_frame_numbers.data_ptr()
            f.mlp_blob = self.blob.data_ptr()
            for l in range(16):
                f.level_scale[l] = float(lay0.scale[l])
                f.level_res[l] = int(lay0.res[l])
            f.num_segments = m.num_segments
            f.lut_size = m.frame_numbers_to_segment_numbers.numel()
            f.vec_res = m.feature_grids[0].vectors.shape[1]
            f.density_scale = m.density_scale
            f.camera_embedding_dim = m.camera_embedding_dim
            f.color_in_width = color_in_width(m.camera_embedding_dim)
            if m.camera_embedding_dim > 0:
                f.camera_embeddings = m.camera_embeddings.weight.data_ptr()
                f.num_cameras = m.camera_embeddings.weight.shape[0]
            else:
                f.camera_embeddings, f.num_cameras = None, 0
            self.keys = keys
            self.versions = None
        versions = tuple(p._version for p in params)
        if versions != self.versions:
            old = self.versions
            with torch.no_grad():
                i = 0
                for s, fg in enumerate(m.feature_grids):
                    for k, g in enumerate(fg.grids()):
                        if old is None or old[i] != versions[i]:
                            L.check(lib.hrf_cast_bf16(g.data_ptr(), self.shadows[s][k].data_ptr(), g.numel(), L.stream()))
                        i += 1
                    if old is None or old[i] != versions[i]:   # vectors: read as fp32 directly; refresh the transposed copy
                        L.check(lib.hrf_transpose_vectors(fg.vectors.data_ptr(), self.vec_t[s].data_ptr(), fg.vectors.shape[1],
                                                          L.stream()))
                    i += 1
                if old is None or old[self.n_table_params:] != versions[self.n_table_params:]:
                    self.repack_mlp()
            self.versions = versions

    def adopt_shadows(self, views: List[List[torch.Tensor]]) -> None:
        """Re-point the bf16 shadow tables at caller-provided storage (views[s][k], already holding the current values):
        the data-parallel trainer keeps them in one peer-visible buffer that the owners of the slices write remotely."""
        m = self.model
        segs = (L.Segment * m.num_segments)()
        raw = self.seg_dev.cpu().numpy().tobytes()
        C.memmove(segs, raw, len(raw))
        for s in range(m.num_segments):
            for k in range(4):
                assert views[s][k].numel() == self.shadows[s][k].numel() and views[s][k].dtype == torch.bfloat16
                segs[s].grid[k] = views[s][k].data_ptr()
        self.shadows = views
        self.seg_dev.copy_(torch.from_numpy(np.frombuffer(bytes(segs), dtype=np.uint8).copy()))

    @property
    def n_table_params(self) -> int:
        return 5 * self.model.num_segments

    def repack_mlp(self) -> None:
        m = self.model
        flat = torch.cat((m.sigma_net.params.detach(), m.color_net.params.detach()))
        self.blob[self.perm[0]] = flat[self.perm[1]].to(torch.bfloat16)

    def mark_shadows_current(self) -> None:
        """Called by the fused optimiser, which writes the shadows itself."""
        self.versions = tuple(p._version for p in self.model.hot_parameters())

    # -------------------------------------------------------------------------------------
    def samples_query(self, positions, directions, frame_numbers, camera_numbers=None) -> L.Samples:
        s = L.Samples()
        s.positions = positions.data_ptr()
        s.directions = None if directions is None else directions.data_ptr()
        s.frame_numbers = frame_numbers.data_ptr()
        s.num_samples = positions.shape[0]
        if camera_numbers is not None:
            s.camera_numbers = camera_numbers.data_ptr()
            s.use_camera_embeddings = 1
        s._keep = (positions, directions, frame_numbers, camera_numbers)   # raw pointers inside: keep the tensors alive
        return s

    def samples_rays(self, ray_origins, ray_directions, ray_frames, distances, ray_indices,
                     ray_cameras=None, count_dev: Optional[torch.Tensor] = None) -> L.Samples:
        """`count_dev` (int64 device scalar): the live number of samples; distances / ray_indices are then capacity-sized
        buffers and nothing has to be read back to launch the kernels (hrf_samples.num_samples_dev)."""
        s = L.Samples()
        s.ray_origins = ray_origins.data_ptr()
        s.ray_directions = ray_directions.data_ptr()
        s.ray_frame_numbers = ray_frames.data_ptr()
        s.sample_distances = distances.data_ptr()
        s.ray_indices = ray_indices.data_ptr()
        s.num_samples = distances.shape[0]
        if ray_cameras is not None:
            s.ray_camera_numbers = ray_cameras.data_ptr()
            s.use_camera_embeddings = 1
        if count_dev is not None:
            s.num_samples_dev = count_dev.data_ptr()
        s._keep = (ray_origins, ray_directions, ray_frames, distances, ray_indices, ray_cameras, count_dev)
        return s

    def forward(self, samples: L.Samples, mode: int, want_geo: bool, want_feat: bool, mlp_impl: int = 0):
        """Returns (sigma, geo, rgb, saved).  `saved` (when want_feat) is ONE flat bf16 buffer of 160 elements per
        sample: the composed features [N,32] (64 B/sample, `saved_features(saved, n)`), followed by the per-(level,grid)
        interpolated features [64][N] bf16x2 (256 B/sample) -- everything the backward needs instead of re-gathering."""
        dev = self._device()
        n = int(samples.num_samples)
        sigma = torch.empty(n, dtype=torch.float32, device=dev)
        geo = torch.empty((n, 16), dtype=torch.bfloat16, device=dev) if want_geo else None
        rgb = torch.empty((n, 3), dtype=torch.float32, device=dev) if mode == 1 else None
        saved = torch.empty(n * 160, dtype=torch.bfloat16, device=dev) if want_feat else None
        egrid = saved.data_ptr() + 64 * n if (want_feat and n > 0) else None
        L.check(L.lib().hrf_field_forward(C.byref(self.field), C.byref(samples), mode, mlp_impl, sigma.data_ptr(),
                                          L.ptr(geo), L.ptr(rgb), L.ptr(saved), egrid, L.stream()))
        return sigma, geo, rgb, saved

    @staticmethod
    def saved_features(saved: torch.Tensor, n: int) -> torch.Tensor:
        return saved[: n * 32].view(n, 32)

    def forward_from_features(self, samples: L.Samples, feat_in: torch.Tensor, feat_index: Optional[torch.Tensor],
                              sigma: Optional[torch.Tensor] = None, rgb: Optional[torch.Tensor] = None):
        """Sigma / colour MLPs on composed features an earlier pass wrote (`feat_in` bf16 [M,32], row `feat_index[i]`
        for sample i): the render pass of the survivors of prune_samples without a second encode."""
        dev = self._device()
        n = int(samples.num_samples)
        sigma = torch.empty(n, dtype=torch.float32, device=dev) if sigma is None else sigma
        rgb = torch.empty((n, 3), dtype=torch.float32, device=dev) if rgb is None else rgb
        L.check(L.lib().hrf_field_forward_from_features(C.byref(self.field), C.byref(samples), feat_in.data_ptr(),
                                                        L.ptr(feat_index), sigma.data_ptr(), rgb.data_ptr(), L.stream()))
        return sigma, rgb

    def density_early_stop(self, samples: L.Samples, ray_offsets: torch.Tensor, num_rays: int, step: float,
                           stop_depth: float = 9.4, save: str = "none", sigma: Optional[torch.Tensor] = None,
                           saved: Optional[torch.Tensor] = None):
        """Density-only pass for prune_samples with the exact early stop (hrf_field_density_early_stop).
        save = "none" -> sigma; "feat" -> (sigma, saved) with the composed features [N,32] bf16 of every evaluated sample;
        "feat+grid" -> the same buffer followed by the per-(level, grid) features [64][N] (layout of forward())."""
        dev = self._device()
        n = int(samples.num_samples)
        sigma = torch.empty(n, dtype=torch.float32, device=dev) if sigma is None else sigma
        lib = L.lib()
        ws = torch.empty(int(lib.hrf_density_early_stop_workspace_bytes(num_rays)), dtype=torch.uint8, device=dev)
        if save != "none" and saved is None:
            saved = torch.empty(n * (160 if save == "feat+grid" else 32), dtype=torch.bfloat16, device=dev)
        egrid = saved.data_ptr() + 64 * n if (save == "feat+grid" and n > 0) else None
        L.check(lib.hrf_field_density_early_stop(C.byref(self.field), C.byref(samples), ray_offsets.data_ptr(), num_rays,
                                                 float(step), float(stop_depth), sigma.data_ptr(),
                                                 L.ptr(saved) if save != "none" else None, egrid, ws.data_ptr(), L.stream()))
        return sigma if save == "none" else (sigma, saved)

    def backward(self, samples: L.Samples, d_sigma, d_rgb, feat, grad_tensors: List[torch.Tensor], per_table: bool = False,
                 d_geo=None, feat_index=None, d_positions: Optional[torch.Tensor] = None,
                 d_directions: Optional[torch.Tensor] = None):
        """grad_tensors: fp32 buffers in hot_parameters() order (accumulated into).  per_table launches the scatter once
        per grid instead of once for all four.  d_geo: fp32 [N,15] gradient of the geometry features, or None.
        d_positions: fp32 [N,3] written with the position gradient (hrf_field_position_grad, after the scatter, on the
        same workspace: the parameter gradients are the launches without it), or None.  d_directions: fp32 [N,3] written
        with the view-direction gradient: the MLP backward is then hrf_field_backward_mlp_dirs, whose weight gradients and
        workspace are hrf_field_backward_mlp's, followed by the same scatter; or None."""
        m = self.model
        dev = self._device()
        sg = (L.SegmentGrads * m.num_segments)()
        i = 0
        for s in range(m.num_segments):
            for k in range(4):
                sg[s].grid[k] = grad_tensors[i].data_ptr()
                i += 1
            sg[s].vectors = grad_tensors[i].data_ptr()
            i += 1
        sg_dev = torch.from_numpy(np.frombuffer(bytes(sg), dtype=np.uint8).copy()).to(dev)
        d_mlp = torch.zeros(m.mlp_grad_elems, dtype=torch.float32, device=dev)
        d_emb = grad_tensors[i + 2] if m.camera_embedding_dim > 0 else None
        ws = torch.empty(int(samples.num_samples) * 40, dtype=torch.float32, device=dev)   # 160 B / sample
        n = int(samples.num_samples)
        # `feat` with a row index = composed features of a pruning pass (no per-grid features: the scatter re-gathers)
        egrid = feat.data_ptr() + 64 * n if (feat is not None and feat_index is None and feat.numel() >= n * 160 and n > 0) else None
        if d_directions is not None:
            L.check(L.lib().hrf_field_backward_mlp_dirs(C.byref(self.field), C.byref(samples), L.ptr(d_sigma), L.ptr(d_rgb),
                                                        L.ptr(d_geo), L.ptr(feat), L.ptr(feat_index), d_mlp.data_ptr(),
                                                        L.ptr(d_emb), d_directions.data_ptr(), ws.data_ptr(), L.stream()))
            for k in (range(4) if per_table else (None,)):
                L.check(L.lib().hrf_field_backward_tables(C.byref(self.field), C.byref(samples), sg_dev.data_ptr(), egrid,
                                                          L.ptr(feat_index), 0, ws.data_ptr(), 0 if k is None else k,
                                                          4 if k is None else 1, L.stream()))
        elif per_table:
            L.check(L.lib().hrf_field_backward_mlp(C.byref(self.field), C.byref(samples), L.ptr(d_sigma), L.ptr(d_rgb),
                                                   L.ptr(d_geo), L.ptr(feat), L.ptr(feat_index), d_mlp.data_ptr(), L.ptr(d_emb),
                                                   ws.data_ptr(), L.stream()))
            for k in range(4):
                L.check(L.lib().hrf_field_backward_tables(C.byref(self.field), C.byref(samples), sg_dev.data_ptr(), egrid,
                                                          None, 0, ws.data_ptr(), k, 1, L.stream()))
        else:
            L.check(L.lib().hrf_field_backward(C.byref(self.field), C.byref(samples), sg_dev.data_ptr(), L.ptr(d_sigma),
                                               L.ptr(d_rgb), L.ptr(d_geo), L.ptr(feat), egrid, L.ptr(feat_index), 0, d_mlp.data_ptr(),
                                               L.ptr(d_emb), ws.data_ptr(), L.stream()))
        if d_positions is not None:
            L.check(L.lib().hrf_field_position_grad(C.byref(self.field), C.byref(samples), ws.data_ptr(), d_positions.data_ptr(),
                                                    L.stream()))
        grad_tensors[i].add_(d_mlp[:MLP_SIGMA_PARAMS])
        grad_tensors[i + 1].add_(d_mlp[MLP_SIGMA_PARAMS:])
        return sg_dev  # keep alive until the kernel has run (stream-ordered free is safe, but be explicit)

    def position_backward(self, samples: L.Samples, d_sigma, d_rgb, feat, d_geo=None, feat_index=None,
                          d_positions: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The position gradient alone, for frozen parameters: the MLP backward (its weight gradients go to a scratch
        buffer that is dropped) and hrf_field_position_grad on its workspace; no table scatter.  Returns d_positions
        fp32 [N,3] (rows past a device-side live count are left as they were: zeros when allocated here)."""
        if d_positions is None:
            d_positions = torch.zeros((int(samples.num_samples), 3), dtype=torch.float32, device=self._device())
        self.input_backward(samples, d_sigma, d_rgb, feat, d_geo=d_geo, feat_index=feat_index, d_positions=d_positions)
        return d_positions

    def input_backward(self, samples: L.Samples, d_sigma, d_rgb, feat, d_geo=None, feat_index=None,
                       d_positions: Optional[torch.Tensor] = None, d_directions: Optional[torch.Tensor] = None) -> None:
        """Gradients of the inputs alone, for frozen parameters: the MLP backward (hrf_field_backward_mlp_dirs when
        `d_directions` is given; its weight gradients go to a scratch buffer that is dropped), then, when `d_positions`
        is given, hrf_field_position_grad on its workspace.  No table scatter.  Both outputs are fp32 [N,3], written."""
        dev = self._device()
        n = int(samples.num_samples)
        d_mlp = torch.empty(self.model.mlp_grad_elems, dtype=torch.float32, device=dev)
        ws = torch.empty(n * 40, dtype=torch.float32, device=dev)   # 160 B / sample
        lib = L.lib()
        if d_directions is not None:
            L.check(lib.hrf_field_backward_mlp_dirs(C.byref(self.field), C.byref(samples), L.ptr(d_sigma), L.ptr(d_rgb),
                                                    L.ptr(d_geo), L.ptr(feat), L.ptr(feat_index), d_mlp.data_ptr(), None,
                                                    d_directions.data_ptr(), ws.data_ptr(), L.stream()))
        else:
            L.check(lib.hrf_field_backward_mlp(C.byref(self.field), C.byref(samples), L.ptr(d_sigma), L.ptr(d_rgb),
                                               L.ptr(d_geo), L.ptr(feat), L.ptr(feat_index), d_mlp.data_ptr(), None,
                                               ws.data_ptr(), L.stream()))
        if d_positions is not None:
            L.check(lib.hrf_field_position_grad(C.byref(self.field), C.byref(samples), ws.data_ptr(), d_positions.data_ptr(),
                                                L.stream()))


def _as_f32c(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.float32).contiguous()


def _as_frames(t: torch.Tensor) -> torch.Tensor:
    return t.detach().reshape(-1).to(torch.int32).contiguous()


class _FieldFunction(torch.autograd.Function):
    """autograd wrapper of the fused kernels in QueryInput form (humanrf.py:158-208)."""

    @staticmethod
    def forward(ctx, model: HumanRF, mode: int, positions, directions, frame_numbers, camera_numbers, needs_grad, active,
                *params):
        nat = model.native()
        pos = L.require_cuda(_as_f32c(positions), "positions")
        dirs = None if directions is None else L.require_cuda(_as_f32c(directions), "directions")
        frames = L.require_cuda(_as_frames(frame_numbers), "frame_numbers")
        cams = None if camera_numbers is None else L.require_cuda(_as_frames(camera_numbers), "camera_numbers")
        samples = nat.samples_query(pos, dirs, frames, cams)
        sigma, geo, rgb, feat = nat.forward(samples, mode, want_geo=True, want_feat=needs_grad)
        ctx.model, ctx.mode, ctx.active = model, mode, active
        ctx.set_materialize_grads(False)    # outputs the caller does not use arrive as None in backward, not as zero tensors
        ctx.save_for_backward(pos, dirs if dirs is not None else pos, frames, feat if feat is not None else pos,
                              cams if cams is not None else frames)
        ctx.has_dirs, ctx.has_cams = dirs is not None, cams is not None
        ctx.pos_dtype, ctx.pos_shape = positions.dtype, positions.shape
        if directions is not None:
            ctx.dir_dtype, ctx.dir_shape = directions.dtype, directions.shape
        geo_out = geo[:, 1:]            # differentiable: humanrf.py:185-186 hands sigma_net's outputs 1..15 to the caller
        if rgb is None:
            rgb = sigma.new_zeros((0, 3))
            ctx.mark_non_differentiable(rgb)
        return sigma, geo_out, rgb

    @staticmethod
    def backward(ctx, d_sigma, d_geo, d_rgb):
        model = ctx.model
        pos, dirs, frames, feat, cams = ctx.saved_tensors
        nat = model.native()
        params = model.hot_parameters()
        samples = nat.samples_query(pos, dirs if ctx.has_dirs else None, frames, cams if ctx.has_cams else None)
        ds = None if d_sigma is None else _as_f32c(d_sigma)
        dr = None if (d_rgb is None or ctx.mode == 0) else _as_f32c(d_rgb)
        if ds is None:
            ds = torch.zeros(pos.shape[0], dtype=torch.float32, device=pos.device)
        dg = None if d_geo is None else _as_f32c(d_geo)
        want_pos = ctx.needs_input_grad[2]
        want_dir = ctx.needs_input_grad[3] and ctx.has_dirs and ctx.mode == 1
        d_pos = torch.empty((pos.shape[0], 3), dtype=torch.float32, device=pos.device) if want_pos else None
        # 0 without a colour gradient: the density does not depend on the direction
        d_dir = (torch.empty if dr is not None else torch.zeros)((pos.shape[0], 3), dtype=torch.float32,
                                                                  device=pos.device) if want_dir else None
        if not any(ctx.needs_input_grad[8:]):
            if not want_pos and not want_dir:
                return (None,) * (8 + len(params))
            # every parameter frozen: the MLP backward and the position kernel only, no table scatter
            if want_pos or dr is not None:
                nat.input_backward(samples, ds, dr, feat, d_geo=dg, d_positions=d_pos,
                                   d_directions=d_dir if dr is not None else None)
            d_pos_out = None if d_pos is None else d_pos.to(ctx.pos_dtype).reshape(ctx.pos_shape)
            d_dir_out = None if d_dir is None else d_dir.to(ctx.dir_dtype).reshape(ctx.dir_shape)
            return (None, None, d_pos_out, d_dir_out, None, None, None, None, *([None] * len(params)))
        grads = [torch.zeros_like(p) for p in params]
        keep = nat.backward(samples, ds, dr, feat, grads, d_geo=dg, d_positions=d_pos,
                            d_directions=d_dir if dr is not None else None)
        del keep
        if ctx.active is not None:      # segments the batch did not touch get no gradient at all (None), as in the reference
            from ..parallel import mask_inactive_segment_grads

            grads = mask_inactive_segment_grads(grads, ctx.active)
        d_pos_out = None if d_pos is None else d_pos.to(ctx.pos_dtype).reshape(ctx.pos_shape)
        d_dir_out = None if d_dir is None else d_dir.to(ctx.dir_dtype).reshape(ctx.dir_shape)
        return (None, None, d_pos_out, d_dir_out, None, None, None, None, *grads)
