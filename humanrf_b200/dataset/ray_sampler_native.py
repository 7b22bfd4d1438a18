"""ray_sampler_native, mirroring the four pybind functions of
actorshq/dataset/native/ray_sampler.cu:327-333 with the identical 15-argument signature
(:197-213) and the identical 9-tensor return list (:314-324).

As in the reference, ``rgba`` (uint8 [P,4]) and ``light_mask`` (bool [P]) may live on the CPU
(CHECK_CONTIGUITY_AND_DEVICE(..., kCPU), :215-216); then the per-ray gathers are done the
reference's way (index on the host, one H2D copy, :254-257,262).  Extension: when they
are CUDA tensors (a GPU-resident image pool, SURVEY 8f-1) the gathers happen inside the sampler
kernels and nothing touches the host.  The whole call performs ONE host read (two counters) to
size its outputs; the reference needs >= 5 implicit syncs.
"""
from __future__ import annotations

import ctypes as C
from typing import List

import torch

from .. import _lib as L

INT32_MAX = 2**31 - 1  # sample offsets and relative ray indices are int32, as in the reference's API


def _get_data(occupancy: bool, samples: bool, rgba, light_mask, frame_numbers, camera_numbers, grid_texture_objects,
              landscape_modes, all_ray_indices, inverse_krs, camera_origins, aabb, grid_resolution, image_width,
              image_height, raymarching_step_size, filter_light_bloom) -> List[torch.Tensor]:
    for name, t in (("rgba", rgba), ("light_mask", light_mask)):
        if not t.is_contiguous():
            raise RuntimeError(f"Tensor not contiguous: {name}")
    L.require_cuda(frame_numbers, "frame_numbers", torch.int32)
    L.require_cuda(camera_numbers, "camera_numbers", torch.int32)
    L.require_cuda(grid_texture_objects, "grid_texture_objects", torch.int64)
    L.require_cuda(landscape_modes, "landscape_modes", torch.bool)
    L.require_cuda(all_ray_indices, "all_ray_indices", torch.int64)
    L.require_cuda(inverse_krs, "inverse_krs", torch.float32)
    L.require_cuda(camera_origins, "camera_origins", torch.float32)
    L.require_cuda(aabb, "aabb", torch.float32)
    dev = aabb.device
    R = all_ray_indices.shape[0]
    pool_on_gpu = rgba.is_cuda
    host_idx = None

    p = L.SamplerParams()
    p.frame_numbers, p.camera_numbers = frame_numbers.data_ptr(), camera_numbers.data_ptr()
    p.grid_handles, p.landscape_modes = grid_texture_objects.data_ptr(), landscape_modes.data_ptr()
    p.inverse_krs, p.camera_origins, p.aabb = inverse_krs.data_ptr(), camera_origins.data_ptr(), aabb.data_ptr()
    keep_alive = []
    if filter_light_bloom:
        if light_mask.is_cuda:
            lm = light_mask.view(torch.uint8)
            p.light_mask = lm.data_ptr()
        else:
            host_idx = all_ray_indices.cpu()
            lm = light_mask[host_idx].to(dev).view(torch.uint8)  # ray_sampler.cu:256
            p.light_mask_rays = lm.data_ptr()
        keep_alive.append(lm)
    p.rgba_pool = rgba.data_ptr() if pool_on_gpu else None
    p.grid_resolution, p.image_width, p.image_height = int(grid_resolution), int(image_width), int(image_height)
    p.step = float(raymarching_step_size)
    p.occupancy, p.want_samples, p.filter_light_bloom = int(occupancy), int(samples), int(bool(filter_light_bloom))

    lib = L.lib()
    f32 = dict(dtype=torch.float32, device=dev)
    ray_mask = torch.empty(R, dtype=torch.bool, device=dev)
    o = torch.empty((R, 3), **f32)
    d = torch.empty((R, 3), **f32)
    rgba_out = torch.empty((R, 4), **f32) if pool_on_gpu else None
    fn = torch.empty(R, dtype=torch.int32, device=dev)
    cn = torch.empty(R, dtype=torch.int32, device=dev)
    mm = torch.empty((R, 2), **f32)
    kept_idx = torch.empty(R, dtype=torch.int64, device=dev)
    offs = torch.empty(R + 1, dtype=torch.int32, device=dev)
    counters = torch.zeros(2, dtype=torch.int64, device=dev)
    ws_bytes = int(lib.hrf_sampler_workspace_bytes(R))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    L.check(lib.hrf_sampler_rays(C.byref(p), all_ray_indices.data_ptr(), R, ray_mask.data_ptr(), o.data_ptr(),
                                 d.data_ptr(), L.ptr(rgba_out), fn.data_ptr(), cn.data_ptr(), mm.data_ptr(),
                                 kept_idx.data_ptr(), offs.data_ptr(), counters.data_ptr(), ws.data_ptr(), ws_bytes,
                                 L.stream()))
    n_rays, n_samples = (int(v) for v in counters.cpu())  # the one host sync of the call
    if n_samples > INT32_MAX:
        raise RuntimeError(f"ray sampler: {n_samples} samples in one call exceed the int32 sample offsets' cap of "
                           f"{INT32_MAX} (2^31 - 1); sample fewer rays per call or use a coarser raymarching step")
    o, d, mm = o[:n_rays], d[:n_rays], mm[:n_rays]
    fn, cn, kept_idx = fn[:n_rays], cn[:n_rays], kept_idx[:n_rays]
    if pool_on_gpu:
        rgba_out = rgba_out[:n_rays]
    else:
        rgba_out = (rgba[kept_idx.cpu()] / 255.0).to(dev)  # ray_sampler.cu:262
    if not samples:
        return [o, d, rgba_out, fn, cn, mm, ray_mask, torch.empty(0, **f32),
                torch.empty(0, dtype=torch.int32, device=dev)]
    dist = torch.empty(n_samples, **f32)
    rel = torch.empty(n_samples, dtype=torch.int32, device=dev)
    L.check(lib.hrf_sampler_samples(C.byref(p), n_rays, kept_idx.data_ptr(), o.data_ptr(), d.data_ptr(), mm.data_ptr(),
                                    offs.data_ptr(), dist.data_ptr(), rel.data_ptr(), L.stream()))
    del keep_alive
    return [o, d, rgba_out, fn, cn, mm, ray_mask, dist, rel]


def get_rays_aabb_minmax(*args):
    return _get_data(False, False, *args)


def get_rays_occupancy_minmax(*args):
    return _get_data(True, False, *args)


def get_samples_aabb_minmax(*args):
    return _get_data(False, True, *args)


def get_samples_occupancy_minmax(*args):
    return _get_data(True, True, *args)
