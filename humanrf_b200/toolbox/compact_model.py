"""A compact, render-only HumanRF: the hash tables as 8-bit codes (DESIGN.md §3.19).

``quantize_model(model)`` turns a trained ``HumanRF`` into a ``CompactHumanRF`` on the GPU, from the fp32 masters.  Each
slice (segment, grid, level, feature) of a table gets one fp32 scale s = c * absmax / 127 and int8 codes
q = clamp(rint(x / s), -127, 127); the clip ratio c is chosen per slice from ``CLIP_RATIOS`` by the least squared
reconstruction error.  Each grid is composed with exactly one vector axis, so the scales are folded into the vectors
(v' = s * v) and the kernels' gathers read the codes with no scale at all.  MLP weights (the packed bf16 blob), vectors,
frame tables and camera embeddings are kept as they are.

A ``CompactHumanRF`` holds only that: no fp32 or bf16 copy of any table.  It renders through every inference path of
the package (``volume_rendering.prune_samples`` / ``render`` / ``render_with_depth`` without gradients,
``TileShardedRenderer``, ``evaluate_sequence``, the occupancy bake, the density lattice and meshes, depth maps and the
depth and geometry scores).  Anything that needs a gradient -- normal maps, camera refinement, held-out colour fits,
training -- refuses it.

After data-parallel training with ``exchange="p2p"`` each rank holds only its shard of the fp32 masters: call
``FusedTrainer.gather_master_parameters()`` before ``quantize_model``.
"""
from __future__ import annotations

from typing import List, Optional

import numpy as np
import torch

from .. import _lib as L
from ..scene_representation.grid_layout import (MLP_BLOB_ELEMS, GridLayout, color_in_width,
                                                segment_log2_hashmap_size)
from ..scene_representation.humanrf import GRID_NAMES, _NativeField, _as_f32c, _as_frames
from ..scene_representation.query_io import QueryInput, QueryOutput

CLIP_RATIOS = (1.0, 0.9, 0.8, 0.7, 0.6, 0.5, 0.4, 0.3)   # fixed in csrc/quantize.cu (kClip)
FORMAT_TAG = "humanrf_b200.compact"
FORMAT_VERSION = 1
_CONFIG_KEYS = ("density_scale", "sorted_frame_numbers", "segment_sizes", "log2_hashmap_size", "coarsest_resolution",
                "finest_resolution", "camera_embedding_dim")


def require_trainable(model, what: str) -> None:
    """Raises when `model` is a CompactHumanRF: `what` needs gradients of the model, which 8-bit tables do not have."""
    if isinstance(model, CompactHumanRF):
        raise RuntimeError(f"{what} needs the trained HumanRF: a CompactHumanRF holds 8-bit tables for rendering only "
                           "and has no gradients")


class CompactHumanRF:
    """Render-only model with int8 hash tables.  Build it with ``quantize_model`` or ``CompactHumanRF.load``."""

    def __init__(self, config: dict, codes: List[List[torch.Tensor]], scales: torch.Tensor, vectors: List[torch.Tensor],
                 mlp_blob: torch.Tensor, frame_to_segment: torch.Tensor, frame_to_tlocal: torch.Tensor,
                 camera_embeddings: Optional[torch.Tensor], clip: torch.Tensor, rms: torch.Tensor):
        self.config = dict(config)
        self.density_scale = float(config["density_scale"])
        self.sorted_frame_numbers = tuple(int(f) for f in config["sorted_frame_numbers"])
        self.segment_sizes = tuple(int(s) for s in config["segment_sizes"])
        self.num_segments = len(self.segment_sizes)
        self.camera_embedding_dim = int(config["camera_embedding_dim"])
        self.layouts = [GridLayout(segment_log2_hashmap_size(s, int(config["log2_hashmap_size"])),
                                   base_resolution=int(config["coarsest_resolution"]),
                                   finest_resolution=int(config["finest_resolution"])) for s in self.segment_sizes]
        self.codes = codes                  # [S][4] int8 [n_entries, 2]
        self.scales = scales                # f32 [S, 4, 16, 2]
        self.vectors = vectors              # [S] f32 [4, vec_res, 32], scales folded in
        self.mlp_blob = mlp_blob            # bf16 [MLP_BLOB_ELEMS], packed as HumanRF's native view packs it
        self.frame_numbers_to_segment_numbers = frame_to_segment
        self.frame_numbers_to_normalized_local_frame_numbers = frame_to_tlocal
        self.camera_embeddings = camera_embeddings
        self.clip = clip                    # int32 [S, 4, 16, 2]: index into CLIP_RATIOS
        self.rms = rms                      # f32 [S, 4, 16, 2]: RMS reconstruction error of the chosen ratio
        self._native: Optional[_CompactNative] = None

    # ------------------------------------------------------------------ what the render paths read
    @property
    def device(self) -> torch.device:
        return self.mlp_blob.device

    def native(self) -> "_CompactNative":
        if self._native is None:
            self._native = _CompactNative(self)
        return self._native

    def invalidate_native(self) -> None:
        """Nothing to refresh: the compact model is immutable."""

    def hot_parameters(self) -> list:
        return []

    def active_segment_list(self, frame_numbers, unique_frame_numbers=None) -> None:
        return None

    def _needs_grad(self, *inputs: Optional[torch.Tensor]) -> bool:
        if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in inputs):
            raise RuntimeError("a CompactHumanRF renders without gradients: its 8-bit tables have no derivative "
                               "(render or query from inputs that do not require grad)")
        return False

    def _query(self, q: QueryInput, mode: int) -> QueryOutput:
        self._needs_grad(q.positions, q.directions if mode == 1 else None)
        nat = self.native()
        pos = L.require_cuda(_as_f32c(q.positions), "positions")
        dirs = None if mode == 0 else L.require_cuda(_as_f32c(q.directions), "directions")
        frames = L.require_cuda(_as_frames(q.frame_numbers), "frame_numbers")
        cams = None
        if mode == 1 and self.camera_embedding_dim > 0 and q.is_training:
            cams = L.require_cuda(_as_frames(q.camera_numbers), "camera_numbers")
        sigma, geo, rgb, _ = nat.forward(nat.samples_query(pos, dirs, frames, cams), mode, want_geo=True, want_feat=False)
        return QueryOutput(density=sigma, geometry_features=geo[:, 1:], radiance=rgb)

    def density(self, query_input: QueryInput) -> QueryOutput:
        """sigma and the geometry features, as ``HumanRF.density`` without gradients."""
        return self._query(query_input, 0)

    def forward(self, query_input: QueryInput) -> QueryOutput:
        """sigma, geometry features and radiance, as ``HumanRF.forward`` without gradients."""
        return self._query(query_input, 1)

    __call__ = forward

    # ------------------------------------------------------------------ sizes
    def parts(self) -> dict:
        """Bytes of each part of the format."""
        emb = 0 if self.camera_embeddings is None else self.camera_embeddings.numel() * 4
        return dict(tables=sum(c.numel() for cs in self.codes for c in cs), scales=self.scales.numel() * 4,
                    vectors=sum(v.numel() * 4 for v in self.vectors), mlp_blob=self.mlp_blob.numel() * 2,
                    frame_luts=(self.frame_numbers_to_segment_numbers.numel()
                                + self.frame_numbers_to_normalized_local_frame_numbers.numel()) * 4,
                    camera_embeddings=emb)

    def device_bytes(self) -> int:
        """Device memory this model holds: the format's tensors, the report's two small arrays and, once rendered from,
        the native view (a transposed copy of the vectors and the segment descriptors)."""
        n = sum(self.parts().values()) + self.clip.numel() * 4 + self.rms.numel() * 4
        if self._native is not None:
            n += sum(v.numel() * 4 for v in self._native.vec_t) + self._native.seg_dev.numel()
        return n

    def report(self) -> dict:
        """Bytes per part, and per slice (segment, grid, level, feature) the chosen clip ratio and its RMS error."""
        clip = self.clip.cpu().numpy()
        rms = self.rms.cpu().numpy()
        slices = []
        for s in range(self.num_segments):
            for k, name in enumerate(GRID_NAMES):
                for l in range(16):
                    for f in range(2):
                        slices.append(dict(segment=s, grid=name, level=l, feature=f,
                                           clip=CLIP_RATIOS[int(clip[s, k, l, f])], scale=float(self.scales[s, k, l, f]),
                                           rms=float(rms[s, k, l, f])))
        parts = self.parts()
        return dict(bytes=parts, total_bytes=sum(parts.values()), slices=slices)

    # ------------------------------------------------------------------ file
    def _payload(self) -> dict:
        cpu = lambda t: None if t is None else t.detach().cpu().contiguous()    # noqa: E731
        return dict(format=FORMAT_TAG, version=FORMAT_VERSION, config=dict(self.config),
                    codes=[[cpu(c) for c in cs] for cs in self.codes], scales=cpu(self.scales),
                    vectors=[cpu(v) for v in self.vectors], mlp_blob=cpu(self.mlp_blob),
                    frame_to_segment=cpu(self.frame_numbers_to_segment_numbers),
                    frame_to_tlocal=cpu(self.frame_numbers_to_normalized_local_frame_numbers),
                    camera_embeddings=cpu(self.camera_embeddings), clip=cpu(self.clip), rms=cpu(self.rms))

    def save(self, path) -> None:
        """One file: ``torch.save`` of plain tensors, ints and floats with a format tag and version."""
        torch.save(self._payload(), path)

    @classmethod
    def load(cls, path, device) -> "CompactHumanRF":
        """Reads a file written by ``save``.  The file is outside input: every field is checked (version, dtypes, shapes,
        each table's length against the layout its configuration implies, the frame tables, finiteness of the scales,
        vectors and MLP weights, no code -128); a malformed file raises ``ValueError`` naming the field."""
        try:
            d = torch.load(path, map_location="cpu", weights_only=True)
        except Exception as e:  # noqa: BLE001  (truncated or not a torch file: every failure of the reader)
            raise ValueError(f"not a readable compact model file: {e}") from e
        p = _validate(d)
        dev = torch.device(device)
        to = lambda t: None if t is None else t.to(dev).contiguous()     # noqa: E731
        return cls(p["config"], [[to(c) for c in cs] for cs in p["codes"]], to(p["scales"]),
                   [to(v) for v in p["vectors"]], to(p["mlp_blob"]), to(p["frame_to_segment"]),
                   to(p["frame_to_tlocal"]), to(p["camera_embeddings"]), to(p["clip"]), to(p["rms"]))


def _validate(d) -> dict:
    def bad(field, why):
        raise ValueError(f"compact model file: {field}: {why}")

    def tensor(field, x, dtype, shape):
        if not isinstance(x, torch.Tensor):
            bad(field, "not a tensor")
        if x.dtype != dtype:
            bad(field, f"dtype {x.dtype}, expected {dtype}")
        if tuple(x.shape) != tuple(shape):
            bad(field, f"shape {tuple(x.shape)}, expected {tuple(shape)}")
        return x

    def finite(field, x):
        if not torch.isfinite(x.float()).all():
            bad(field, "holds non-finite values")

    if not isinstance(d, dict) or d.get("format") != FORMAT_TAG:
        bad("format", f"expected the tag {FORMAT_TAG!r}")
    if d.get("version") != FORMAT_VERSION:
        bad("version", f"{d.get('version')!r}, this reader reads version {FORMAT_VERSION}")
    cfg = d.get("config")
    if not isinstance(cfg, dict) or any(k not in cfg for k in _CONFIG_KEYS):
        bad("config", f"needs the keys {_CONFIG_KEYS}")
    try:
        frames = tuple(int(f) for f in cfg["sorted_frame_numbers"])
        segs = tuple(int(s) for s in cfg["segment_sizes"])
        log2 = int(cfg["log2_hashmap_size"])
        base, finest, emb_dim = int(cfg["coarsest_resolution"]), int(cfg["finest_resolution"]), int(cfg["camera_embedding_dim"])
        float(cfg["density_scale"])
    except (TypeError, ValueError) as e:
        bad("config", str(e))
    if not frames or list(frames) != sorted(set(frames)) or frames[0] < 0:
        bad("config.sorted_frame_numbers", "must be distinct non-negative frame numbers in ascending order")
    if not segs or min(segs) < 1 or not 0 <= emb_dim <= 17 or not 1 <= log2 <= 24 or base < 1 or finest < base:
        bad("config", "segment sizes, table size, resolutions or camera embedding out of range")
    S = len(segs)
    for key in ("codes", "vectors"):
        if not isinstance(d.get(key), list) or len(d[key]) != S:
            bad(key, f"expected a list of {S} segments")
    for s in range(S):
        lay = GridLayout(segment_log2_hashmap_size(segs[s], log2), base_resolution=base, finest_resolution=finest)
        if not isinstance(d["codes"][s], list) or len(d["codes"][s]) != 4:
            bad(f"codes[{s}]", "expected 4 grids")
        for k in range(4):
            c = tensor(f"codes[{s}][{k}]", d["codes"][s][k], torch.int8, (lay.n_entries, 2))
            if (c == -128).any():
                bad(f"codes[{s}][{k}]", "holds the code -128, which the format never produces")
        finite(f"vectors[{s}]", tensor(f"vectors[{s}]", d["vectors"][s], torch.float32, (4, finest, 32)))
    scales = tensor("scales", d.get("scales"), torch.float32, (S, 4, 16, 2))
    finite("scales", scales)
    if (scales < 0).any():
        bad("scales", "negative scale")
    tensor("clip", d.get("clip"), torch.int32, (S, 4, 16, 2))
    if ((d["clip"] < 0) | (d["clip"] >= len(CLIP_RATIOS))).any():
        bad("clip", "index outside the clip-ratio list")
    tensor("rms", d.get("rms"), torch.float32, (S, 4, 16, 2))
    finite("mlp_blob", tensor("mlp_blob", d.get("mlp_blob"), torch.bfloat16, (MLP_BLOB_ELEMS,)))
    lut = frames[-1] + 1
    f2s = tensor("frame_to_segment", d.get("frame_to_segment"), torch.int32, (lut,))
    if ((f2s < -1) | (f2s >= S)).any():
        bad("frame_to_segment", f"segment numbers must lie in [-1, {S})")
    finite("frame_to_tlocal", tensor("frame_to_tlocal", d.get("frame_to_tlocal"), torch.float32, (lut,)))
    emb = d.get("camera_embeddings")
    if emb_dim > 0:
        finite("camera_embeddings", tensor("camera_embeddings", emb, torch.float32, (160, emb_dim)))
    elif emb is not None:
        bad("camera_embeddings", "present although camera_embedding_dim is 0")
    return d


class _CompactNative(_NativeField):
    """The device view of a CompactHumanRF: the same hrf_field the kernels read, with table_format = int8x2.  The query,
    ray-batch, early-stop and fused-render launches are HumanRF's own (inherited); the backward ones are refused by the
    library."""

    def __init__(self, cm: CompactHumanRF):
        self.model = cm
        self.field = L.Field()
        dev = cm.device
        if dev.type != "cuda":
            raise RuntimeError("humanrf_b200: a CompactHumanRF renders on a CUDA device; load it with device='cuda'")
        lib = L.lib()
        vr = cm.vectors[0].shape[1]
        self.vec_t = []
        segs = (L.Segment * cm.num_segments)()
        for s in range(cm.num_segments):
            lay = cm.layouts[s]
            vt = torch.empty_like(cm.vectors[s])
            L.check(lib.hrf_transpose_vectors(cm.vectors[s].data_ptr(), vt.data_ptr(), vr, L.stream()))
            self.vec_t.append(vt)
            for k in range(4):
                segs[s].grid[k] = cm.codes[s][k].data_ptr()
            segs[s].vectors = cm.vectors[s].data_ptr()
            segs[s].vectors_t = vt.data_ptr()
            for l in range(16):
                segs[s].level_offset[l] = int(lay.offset[l])
                segs[s].level_size[l] = int(lay.size[l])
            segs[s].hashed_mask = lay.hashed_mask
            segs[s].n_entries = lay.n_entries
        self.seg_dev = torch.from_numpy(np.frombuffer(bytes(segs), dtype=np.uint8).copy()).to(dev)
        f = self.field
        f.segments = self.seg_dev.data_ptr()
        f.frame_to_segment = cm.frame_numbers_to_segment_numbers.data_ptr()
        f.frame_to_tlocal = cm.frame_numbers_to_normalized_local_frame_numbers.data_ptr()
        f.mlp_blob = cm.mlp_blob.data_ptr()
        lay0 = cm.layouts[0]
        for l in range(16):
            f.level_scale[l] = float(lay0.scale[l])
            f.level_res[l] = int(lay0.res[l])
        f.num_segments = cm.num_segments
        f.lut_size = cm.frame_numbers_to_segment_numbers.numel()
        f.vec_res = vr
        f.density_scale = cm.density_scale
        f.camera_embedding_dim = cm.camera_embedding_dim
        f.color_in_width = color_in_width(cm.camera_embedding_dim)
        if cm.camera_embedding_dim > 0:
            f.camera_embeddings = cm.camera_embeddings.data_ptr()
            f.num_cameras = cm.camera_embeddings.shape[0]
        f.table_format = L.TABLE_INT8X2

    def _device(self) -> torch.device:
        return self.model.device

    def refresh(self) -> None:
        pass


@torch.no_grad()
def quantize_model(model) -> CompactHumanRF:
    """The compact model of a trained ``HumanRF`` (on a CUDA device), computed on the GPU from its fp32 masters.  After
    data-parallel training with the p2p exchange, call ``FusedTrainer.gather_master_parameters()`` first: each rank
    otherwise holds only its own shard of the masters.  Raises, naming the segment, grid and level, if a master value is
    not finite."""
    from ..scene_representation.humanrf import HumanRF

    if not isinstance(model, HumanRF):
        raise TypeError(f"quantize_model takes a HumanRF, not {type(model).__name__}")
    nat = model.native()          # checks the device and dtypes, and packs the MLP blob from the current weights
    dev = nat._device()
    lib = L.lib()
    S = model.num_segments
    scales = torch.empty((S, 4, 16, 2), dtype=torch.float32, device=dev)
    clip = torch.empty((S, 4, 16, 2), dtype=torch.int32, device=dev)
    sq_err = torch.empty((S, 4, 16, 2, L.QUANT_CLIPS), dtype=torch.float64, device=dev)
    status = torch.zeros((4, 16), dtype=torch.int32, device=dev)
    codes, vectors = [], []
    for s, fg in enumerate(model.feature_grids):
        lay = fg.layout
        masters = (L.vp * 4)(*[g.data_ptr() for g in fg.grids()])
        off = (L.u32 * 16)(*[int(x) for x in lay.offset])
        size = (L.u32 * 16)(*[int(x) for x in lay.size])
        L.check(lib.hrf_quantize_tables_select(masters, off, size, s, scales[s].data_ptr(), clip[s].data_ptr(),
                                               sq_err[s].data_ptr(), status.data_ptr(), L.stream()))
        cs = [torch.empty((lay.n_entries, 2), dtype=torch.int8, device=dev) for _ in range(4)]
        L.check(lib.hrf_quantize_tables_write(masters, off, size, scales[s].data_ptr(),
                                              (L.vp * 4)(*[c.data_ptr() for c in cs]), L.stream()))
        folded = torch.empty_like(fg.vectors)
        L.check(lib.hrf_quantize_fold_vectors(fg.vectors.data_ptr(), scales[s].data_ptr(), fg.vectors.shape[1],
                                              folded.data_ptr(), L.stream()))
        codes.append(cs)
        vectors.append(folded.detach())
    n = torch.tensor([[int(x) for x in fg.layout.size] for fg in model.feature_grids], dtype=torch.float64, device=dev)
    best = torch.gather(sq_err, 4, clip.long().unsqueeze(-1)).squeeze(-1)
    rms = torch.sqrt(best / n[:, None, :, None]).float()
    cfg = dict(density_scale=float(model.density_scale), sorted_frame_numbers=tuple(model.sorted_frame_numbers),
               segment_sizes=tuple(model.segment_sizes), log2_hashmap_size=int(model.log2_hashmap_size),
               coarsest_resolution=int(model.coarsest_resolution), finest_resolution=int(model.finest_resolution),
               camera_embedding_dim=int(model.camera_embedding_dim))
    emb = model.camera_embeddings.weight.detach().clone() if model.camera_embedding_dim > 0 else None
    return CompactHumanRF(cfg, codes, scales, vectors, nat.blob.detach().clone(),
                          model.frame_numbers_to_segment_numbers.detach().clone(),
                          model.frame_numbers_to_normalized_local_frame_numbers.detach().clone(), emb, clip, rms)

