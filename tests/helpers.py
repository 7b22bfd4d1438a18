"""Shared builders for the parity tests: identical parameters in the oracle model and the
CUDA-backed HumanRF module, the seeded synthetic ray batch of SURVEY 8(d), and the pieces of the gradient-scatter
tests (the workspace, the gradient descriptors, float64 autograd of the scatter)."""
from __future__ import annotations

import numpy as np
import torch

from oracle import field as ofield
from oracle import hashgrid

from humanrf_b200.synthetic import MODEL_KW, input_batch_of, synthetic_rays  # noqa: F401,E402

GRID_AXES = ([0, 1, 2], [0, 1, 3], [1, 2, 3], [0, 2, 3])     # xyz, xyt, yzt, xzt (decomposition4d.py:126-129)
VECTOR_OF_GRID = (3, 2, 0, 1)                                 # xyz*v_t, xyt*v_z, yzt*v_x, xzt*v_y (tensor_composition.cu:49-52)


def make_pair(segment_sizes=(6,), seed=123, table_std=6.0, device="cuda", bf16=True, first_frame=15, cam_emb=0):
    """Returns (oracle_model, humanrf_module) holding the same parameter values."""
    from humanrf_b200.scene_representation.humanrf import HumanRF

    frames = tuple(range(first_frame, first_frame + sum(segment_sizes)))
    om = ofield.make_model(segment_sizes, frames, seed=seed, table_init="trained", bf16=bf16, table_std=table_std,
                           camera_embedding_dim=cam_emb)
    m = HumanRF(sorted_frame_numbers=frames, segment_sizes=tuple(segment_sizes), **{**MODEL_KW, "camera_embedding_dim": cam_emb})
    with torch.no_grad():
        for s, fg in enumerate(m.feature_grids):
            for k, g in enumerate(fg.grids()):
                g.copy_(om.segments[s].grids[k].reshape(-1))
            fg.vectors.copy_(om.segments[s].vectors)
        m.sigma_net.params.copy_(torch.cat([w.reshape(-1) for w in om.w_sigma]))
        m.color_net.params.copy_(torch.cat([w.reshape(-1) for w in om.w_color]))
        if cam_emb:
            m.camera_embeddings.weight.copy_(om.camera_embeddings)
    return om, m.to(device), frames


def positions_of(b):
    """volume_rendering.py:66-69 in fp32 (mul then add)."""
    return b["o"][b["ri"]] + b["t"].unsqueeze(1) * b["d"][b["ri"]]


def rel_err(a, b, floor=1e-6):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b) / np.maximum(np.abs(b), floor)


def scatter_workspace(d_out, xyzt, seg, cuda):
    """What hrf_field_backward_mlp leaves for the scatter: d(features) level-major [16][n] float2 | (x,y,z,t) [n] float4
    | segment [n] u8."""
    n = d_out.shape[0]
    ws = torch.zeros(n * 40, dtype=torch.float32, device=cuda)
    ws[: 32 * n] = d_out.reshape(n, 16, 2).permute(1, 0, 2).reshape(-1).to(cuda)
    ws[32 * n: 36 * n] = xyzt.reshape(-1).to(cuda)
    ws.view(torch.uint8)[144 * n: 145 * n] = torch.from_numpy(seg.astype(np.uint8)).to(cuda)
    return ws


def segment_grads(m):
    """Zeroed gradients of m.hot_parameters() and the device array of hrf_segment_grads that points into them."""
    from humanrf_b200 import _lib as L

    grads = [torch.zeros_like(p) for p in m.hot_parameters()]
    sg = (L.SegmentGrads * m.num_segments)()
    for s in range(m.num_segments):
        for k in range(4):
            sg[s].grid[k] = grads[5 * s + k].data_ptr()
        sg[s].vectors = grads[5 * s + 4].data_ptr()
    sg_dev = torch.from_numpy(np.frombuffer(bytes(sg), dtype=np.uint8).copy()).to(grads[0].device)
    return grads, sg_dev


def scatter_autograd_reference(om, seg, xyzt, d_out, lerp):
    """float64 autograd of sum_k encode_k * lerp(vector_k) against d_out, per segment.  Table gradients do not depend on
    the features; the vector gradients of the egrid path use the saved bf16 features, those of the re-gather path the
    exact blend of the (bf16) tables.  Also returns every sample's exact per-grid features [n, 4, 32]."""
    ref_tables, ref_vec_gather, ref_vec_egrid = [], [], []
    enc_all = torch.zeros(xyzt.shape[0], 4, 32, dtype=torch.float64)
    for s, sd in enumerate(om.segments):
        sel = torch.from_numpy(np.nonzero(seg == s)[0])
        tabs = [t.double().requires_grad_(True) for t in sd.grids]
        c = xyzt[sel]
        enc = [hashgrid.encode(tabs[k], c[:, GRID_AXES[k]], sd.log2T) for k in range(4)]
        for k in range(4):
            enc_all[sel, k] = enc[k].detach()
        saved = [e.detach().float().bfloat16().double() for e in enc]
        vg = sd.vectors.double().requires_grad_(True)
        ve = sd.vectors.double().requires_grad_(True)
        sv_g, sv_e = lerp(vg, c), lerp(ve, c)
        out_g = sum(enc[k] * sv_g[VECTOR_OF_GRID[k]] for k in range(4))
        out_e = sum(saved[k] * sv_e[VECTOR_OF_GRID[k]] for k in range(4))
        (((out_g + out_e) * d_out[sel].double()).sum()).backward()
        ref_tables.append([t.grad.reshape(-1) if t.grad is not None else torch.zeros(t.numel(), dtype=torch.float64) for t in tabs])
        ref_vec_gather.append(vg.grad if vg.grad is not None else torch.zeros_like(vg))
        ref_vec_egrid.append(ve.grad if ve.grad is not None else torch.zeros_like(ve))
    return ref_tables, {"gather": ref_vec_gather, "egrid": ref_vec_egrid}, enc_all


def field_without_vectors_t(nat):
    """A copy of the field whose segment descriptors have vectors_t = NULL: the encode then reads `vectors` itself."""
    import ctypes as C

    from humanrf_b200 import _lib as L

    seg = nat.seg_dev.clone()
    size, off = C.sizeof(L.Segment), L.Segment.vectors_t.offset
    for s in range(nat.model.num_segments):
        seg[s * size + off: s * size + off + 8] = 0
    f = L.Field.from_buffer_copy(nat.field)
    f.segments = seg.data_ptr()
    return f, seg
