#!/usr/bin/env python
"""End-to-end integration on synthetic data: DataLoader (GPU pool) -> prune_samples -> merge_input_batches ->
FusedTrainer.step, following the reference's adaptive-batch training loop (humanrf/trainer.py:135-172), then
full-image validation through the tile renderer with PSNR (trainer.py:218-222).

The "dataset" is rendered from a smooth random TEACHER radiance field (there is no ActorsHQ data and no network),
so a held-out camera has a meaningful ground truth and PSNR must rise as the student trains.

    python examples/train_synthetic.py --steps 300
"""
from __future__ import annotations

import argparse
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))

from humanrf_b200.dataset.data_loader import DataLoader  # noqa: E402
from humanrf_b200.input import merge_input_batches  # noqa: E402
from humanrf_b200.parallel import TileShardedRenderer  # noqa: E402
from humanrf_b200.synthetic import make_model  # noqa: E402
from humanrf_b200.training import FusedTrainer  # noqa: E402
from humanrf_b200.volume_rendering import prune_samples  # noqa: E402
from humanrf_b200.synthetic_scene import SyntheticDataset  # noqa: E402


class TeacherDataset(SyntheticDataset):
    """SyntheticDataset whose images are renderings of a teacher HumanRF through the product's own renderer."""

    def __init__(self, teacher, device, **kw):
        super().__init__(**kw)
        self._images = {}
        self.teacher, self.device = teacher, device

    def bake(self, loader_tables, og):
        r = TileShardedRenderer(self.teacher, og, rays_per_batch=8192)
        for c in range(len(self.cameras)):
            for f in self.frames:
                cam = loader_tables(c, f)
                img = r.render_range(cam, 0, cam["width"] * cam["height"])
                self._images[(c, f)] = img.clamp(0, 1).cpu().numpy().reshape(cam["height"], cam["width"], 3)

    def get_rgb(self, camera_number, frame_number, normalize=True):
        return self._images[(camera_number, frame_number)][..., ::-1].copy()      # the reference reads BGR (cv2)

    def get_mask(self, camera_number, frame_number, normalize=True):
        return (self._images[(camera_number, frame_number)].sum(-1, keepdims=True) > 1e-3).astype(np.float32)


def smooth_teacher(device, frames):
    """Teacher with energy only in the 6 coarsest levels -> a smooth, learnable field."""
    model, _ = make_model((len(frames),), first_frame=frames[0], seed=7, table_std=1.5, device=device)
    with torch.no_grad():
        for fg in model.feature_grids:
            lay = fg.layout
            for p in fg.grids():
                p.view(-1, 2)[int(lay.offset[6]):] = 0
    model.density_scale = 60.0
    model._native = None
    return model


def camera_tables(dl: DataLoader, og, ds):
    def tables(camera_number, frame_number):
        dev = dl.aabb.device
        grid = torch.from_numpy(ds.get_occupancy_grid(frame_number)).to(dev).contiguous()
        cam = dl.cameras[camera_number]
        return dict(frame_numbers=torch.tensor([frame_number], dtype=torch.int32, device=dev),
                    camera_numbers=torch.tensor([camera_number], dtype=torch.int32, device=dev),
                    grid_handles=torch.tensor([og.add_grid(grid)], dtype=torch.int64, device=dev),
                    landscape=torch.tensor([cam.width > cam.height], device=dev),
                    inverse_krs=dl.all_inverse_krs[camera_number:camera_number + 1].contiguous(),
                    camera_origins=dl.all_camera_origins[camera_number:camera_number + 1].contiguous(), aabb=dl.aabb,
                    G=dl.occupancy_grid_resolution, width=cam.width, height=cam.height)
    return tables


def psnr(a, b):
    return float(-10 * torch.log10(torch.mean((a - b) ** 2)))      # trainer.py:218-222


def main(steps=300, samples_max=200_000, rays_initial=4096, log_every=100, quiet=False, return_state=False, seed=0,
         error_map=None, sample_budget=None, training_occupancy=None, loose_hull=False):
    """Returns the held-out PSNR history [(step, dB)]; with `return_state` also a dict of the trained student, the
    dataset, the occupancy grid, the camera-table builder, the frames, the held-out camera and the samples trained on.
    `seed` seeds the run (the student, the pair schedule, the trainer's jitter and backgrounds; the teacher and the scene
    stay).  `error_map`: keyword arguments of toolbox.error_map.ErrorMap, whose seed is `seed`: the rays are drawn from
    it.  `sample_budget`: stop once the steps have trained on that many samples (`steps` stays the limit).
    `training_occupancy`: keyword arguments of toolbox.training_occupancy.TrainingOccupancy, whose seed is `seed`: the
    training sampler's grids are learned while training.  `loose_hull`: the images are rendered through the dataset's
    hulls, then every hull is dilated by 6 voxels for training and validation, so the scene's density sits well inside
    hulls with slack around it (as around a body seen by few cameras)."""
    from humanrf_b200.dataset.occupancy_grid_native import OccupanyGrid

    dev = torch.device("cuda:0")
    torch.manual_seed(seed); np.random.seed(seed)
    frames = list(range(15, 21))
    teacher = smooth_teacher(dev, frames)
    ds = TeacherDataset(teacher, dev, num_cameras=6, frames=frames, width=96, height=72, G=64)
    # a loader on placeholder images first, only to get the normalised camera tables for baking
    ds._images = {(c, f): np.zeros((72, 96, 3), np.float32) for c in range(6) for f in frames}
    M = DataLoader.Mode
    boot = DataLoader(ds, "cuda", M.TEST, DataLoader.OutputMode.RAYS_AND_SAMPLES, DataLoader.SpacePruningMode.OCCUPANCY_GRID,
                      batch_size=8192, camera_numbers=tuple(range(6)), frame_numbers=tuple(frames), max_buffer_size=1,
                      render_sequence=[(0, frames[0])])
    og = OccupanyGrid(64, 2)
    tables = camera_tables(boot, og, ds)
    ds.bake(tables, og)
    if loose_hull:
        with torch.no_grad():
            for f in frames:
                g = torch.from_numpy(ds._grids[f]).to(dev).float()[None, None]
                ds._grids[f] = (torch.nn.functional.max_pool3d(g, 13, stride=1, padding=6)[0, 0] > 0).to(
                    torch.uint8).mul(255).cpu().numpy()
    train_cams, held_out = (0, 1, 2, 3, 4), 5
    dl = DataLoader(ds, "cuda", M.TRAINING, DataLoader.OutputMode.RAYS_AND_SAMPLES, DataLoader.SpacePruningMode.OCCUPANCY_GRID,
                    batch_size=rays_initial, camera_numbers=train_cams, frame_numbers=tuple(frames), max_buffer_size=64,
                    max_num_frames_per_batch=8, use_mask=True, filter_light_bloom=False)
    student, _ = make_model((len(frames),), first_frame=frames[0], seed=1 + seed, table_std=1e-4, device=dev)
    emap = None
    if error_map is not None:
        from humanrf_b200.toolbox.error_map import ErrorMap

        emap = ErrorMap(dl, seed=seed, **error_map)
    tocc = None
    if training_occupancy is not None:
        from humanrf_b200.toolbox.training_occupancy import TrainingOccupancy

        tocc = TrainingOccupancy(dl, student, seed=seed, **training_occupancy)
    trainer = FusedTrainer(student, lr=1e-2, max_steps=steps, prune=False, seed=123 + seed, error_map=emap,
                           training_occupancy=tocc)
    renderer = TileShardedRenderer(student, og, rays_per_batch=8192)

    def validate():
        out = []
        for f in (frames[0], frames[-1]):
            cam = tables(held_out, f)
            img = renderer.render_range(cam, 0, cam["width"] * cam["height"]).clamp(0, 1)
            gt = torch.from_numpy(ds._images[(held_out, f)].reshape(-1, 3).copy()).to(dev)
            out.append(psnr(img, gt))
        return float(np.mean(out))

    history = [(0, validate())]
    it = iter(dl)
    t0 = time.time()
    rays_done = samples_done = 0
    for step in range(1, steps + 1):
        dl.batch_size = rays_initial                                             # trainer.py:139
        total_rays = total_samples = 0
        batches, pixels = [], []
        while True:                                                              # trainer.py:143-163
            b = next(it)
            if emap is not None:                                                 # the pool index of each kept ray
                pixels.append(dl.last_ray_indices[b.ray_masks.view(-1)])
            prune_samples(b, student, is_training=True)
            batches.append(b)
            total_rays += dl.batch_size
            total_samples += b.num_samples
            if total_samples < 0.9 * samples_max:
                avg = max(total_samples / total_rays, 1e-3)
                dl.batch_size = max(256, min(int((samples_max - total_samples) / avg), 65536))
            else:
                break
        ib = merge_input_batches(batches, max_num_samples=int(samples_max * 1.1))   # trainer.py:170-172
        if ib.num_samples == 0:
            continue
        px = torch.cat(pixels)[:ib.num_rays] if emap is not None else None     # merging keeps a prefix of the rays
        trainer.step(ib.ray_origins.contiguous(), ib.ray_directions.contiguous(), ib.frame_numbers.view(-1).contiguous(),
                     ib.sample_distances.view(-1).contiguous(), ib.ray_indices.contiguous(), ib.rgba.contiguous(), ib.num_rays,
                     pixels=px)
        rays_done += ib.num_rays
        samples_done += ib.num_samples
        last = step == steps or (sample_budget is not None and samples_done >= sample_budget)
        if step % log_every == 0 or last:
            history.append((step, validate()))
            if not quiet:
                print(f"step {step:5d}  loss {float(trainer.last['loss']):.5f}  samples {ib.num_samples}  rays {ib.num_rays}  "
                      f"held-out PSNR {history[-1][1]:.2f} dB  ({rays_done / (time.time() - t0):.0f} rays/s incl. validation)")
        if last:
            break
    if return_state:
        return history, dict(student=student, dataset=ds, occupancy_grid=og, tables=tables, frames=frames,
                             held_out=held_out, samples=samples_done, steps=step, loader=dl, training_occupancy=tocc)
    return history


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    a = ap.parse_args()
    h = main(a.steps)
    print("PSNR history:", h)
