"""DataLoader with a GPU-resident image pool (SURVEY 8f-1), mirroring the call contract of
actorshq/dataset/data_loader.py: same constructor arguments / enums, iterator protocol
``__iter__`` / ``__next__ -> InputBatch`` (:519-660), mutable ``batch_size`` (trainer.py:139,161),
``pause_replacing`` / ``continue_replacing`` (:525-529), ``num_batches_per_full_image``,
``num_camera_frame_pairs``, ``render_sequence``, ``cameras``, ``dataset``, ``resolution``, ``aabb``.

What is different by design (the reference's default pool of 200 images, RGBA + light mask, takes 12 GB of the GPU's
80 GB at full resolution and 0.8 GB at 4x downscale: no reason to bounce pixels through the host):
* the uint8 RGBA pool and the light-bloom mask live ON THE GPU; the sampler gathers ground-truth colours inside
  its kernels (the reference keeps the pool on the CPU and does ``rgba.index({ray_indices.cpu()}) -> .cuda()`` per
  call, ray_sampler.cu:262);
* no replacer thread, no locks, no semaphores: if the pool cannot hold every (camera, frame) pair, slots are
  replaced synchronously on the calling thread (``replace_per_next`` slots per ``__next__`` in TRAINING; the next
  image on demand in VALIDATION / TEST).  The (camera, frame) schedule is the reference's
  (``_camera_frame_pair_generator``, :356-394), so ``max_num_frames_per_batch`` bounds the distinct frames in the
  pool exactly as there.
The ``dataset`` argument is duck-typed on the VolumetricDataset methods the reference calls (volumetric_dataset.py:
``get_aabb``, ``get_scaled_cameras``, ``get_rgb``, ``get_mask``, ``get_occupancy_grid``, ``get_light_annotations``).
"""
from __future__ import annotations

import itertools
from enum import Enum
from typing import Any, List, Optional, Tuple

import numpy as np
import torch

from . import occupancy_grid_native, ray_sampler_native
from .input_batch import InputBatch


class DataLoader:
    class Mode(Enum):
        TRAINING = 0
        VALIDATION = 1
        TEST = 2

    class OutputMode(Enum):
        RAYS = 0
        RAYS_AND_SAMPLES = 1

    class SpacePruningMode(Enum):
        AABB = 0
        OCCUPANCY_GRID = 1

    def __init__(self, dataset, device: str, mode: "DataLoader.Mode", dataloader_output_mode: "DataLoader.OutputMode",
                 space_pruning_mode: "DataLoader.SpacePruningMode", batch_size: int, camera_numbers: Tuple[int],
                 frame_numbers: Tuple[int], max_buffer_size: int, max_num_frames_per_batch: Optional[int] = None,
                 use_mask: Optional[bool] = None, filter_light_bloom: Optional[bool] = None,
                 render_sequence: Optional[List[Tuple[int, int]]] = None, replace_per_next: int = 1) -> None:
        self.device, self.mode, self.batch_size = device, mode, batch_size
        self.camera_numbers, self.frame_numbers = tuple(camera_numbers), tuple(frame_numbers)
        if len(set(self.camera_numbers)) != len(self.camera_numbers):
            raise RuntimeError("Provided camera numbers cannot have duplicates.")
        if len(set(self.frame_numbers)) != len(self.frame_numbers):
            raise RuntimeError("Provided frame numbers cannot have duplicates.")

        def _check_and_get_arg(arg: Any, arg_name: str, valid_modes, non_valid_default: Any):
            if self.mode in valid_modes:
                if arg is None:
                    raise RuntimeError(f"'{arg_name}' has to be given for {str(self.mode)}")
                return arg
            if arg is not None:
                raise RuntimeError(f"'{arg_name}' cannot be used for {str(self.mode)}")
            return non_valid_default

        M = DataLoader.Mode
        self.max_num_frames_per_batch = _check_and_get_arg(max_num_frames_per_batch, "max_num_frames_per_batch", [M.TRAINING], None)
        if self.mode == M.TRAINING:
            if len(self.frame_numbers) > 1 and self.max_num_frames_per_batch < 2:
                raise RuntimeError("'max_num_frames_per_batch >= 2' has to be met.")
            self.max_num_frames_per_batch = min(self.max_num_frames_per_batch, len(self.frame_numbers))
        self.use_mask = _check_and_get_arg(use_mask, "use_mask", [M.TRAINING, M.VALIDATION], False)
        self.filter_light_bloom = _check_and_get_arg(filter_light_bloom, "filter_light_bloom", [M.TRAINING, M.VALIDATION], False)
        self.render_sequence = _check_and_get_arg(render_sequence, "render_sequence", [M.VALIDATION, M.TEST], None)
        self.num_camera_frame_pairs = (len(self.camera_numbers) * len(self.frame_numbers) if self.mode == M.TRAINING
                                       else len(self.render_sequence))
        self.space_pruning_mode = space_pruning_mode
        om = "rays" if dataloader_output_mode == DataLoader.OutputMode.RAYS else "samples"
        sp = "aabb" if space_pruning_mode == DataLoader.SpacePruningMode.AABB else "occupancy"
        self.ray_sampler_func = getattr(ray_sampler_native, f"get_{om}_{sp}_minmax")
        self.dataset = dataset
        self.replace_per_next = replace_per_next

        # scene normalisation (data_loader.py:182-215)
        aabb = np.asarray(self.dataset.get_aabb(), np.float64)
        self.scene_offset = -aabb.mean(0)
        self.scene_scale = 1 / np.max(aabb[1] - aabb[0])
        self.cameras = self.dataset.get_scaled_cameras(scene_offset=self.scene_offset, scene_scale=self.scene_scale)
        self.all_inverse_krs = torch.from_numpy(np.stack(
            [np.linalg.inv(cam.projection_matrix_world2pixel()) for cam in self.cameras], axis=0))[..., :3, :3] \
            .transpose(-1, -2).float().to(device).contiguous()
        self.all_camera_origins = torch.from_numpy(np.stack([cam.translation for cam in self.cameras], 0)).float().to(device).contiguous()
        self.aabb = torch.from_numpy((aabb + self.scene_offset) * self.scene_scale).to(device).float().contiguous()

        pix = list(set(self.cameras[cn].width * self.cameras[cn].height for cn in self.camera_numbers))
        if len(pix) != 1:
            raise RuntimeError("Each camera should have the same number of pixels!")
        self.num_pixels_per_camera = pix[0]
        res = list(set((self.cameras[cn].width, self.cameras[cn].height) for cn in self.camera_numbers))
        if len(res) > 2 or (len(res) == 2 and not (res[0][0] == res[1][1] and res[0][1] == res[1][0])):
            raise RuntimeError("Currently, we only support one image resolution with landspace or portrait mode!"
                               " (effectively two different resolutions)")
        self.resolution = max(res[0]), min(res[0])

        self.light_annotations = None
        if self.filter_light_bloom:
            self.light_annotations = self.dataset.get_light_annotations()

        # pool sizing (data_loader.py:249-258)
        self.buffer_size = min(max_buffer_size, self.num_camera_frame_pairs)
        if self.mode == M.TRAINING:
            if self.max_num_frames_per_batch > 1:
                self.buffer_size = min(self.buffer_size, len(self.camera_numbers) * (self.max_num_frames_per_batch - 1))
            self.occupancy_grids_buffer_size = min(self.buffer_size, self.max_num_frames_per_batch)
        else:
            self.occupancy_grids_buffer_size = min(self.buffer_size, len(self.frame_numbers))

        B, P = self.buffer_size, self.num_pixels_per_camera
        self.pixel_colors = torch.zeros((B, P, 4), device=device, dtype=torch.uint8)       # GPU-resident pool
        self.light_mask = torch.zeros((B, P), device=device, dtype=torch.bool)
        self.frame_numbers_cuda = torch.full((B,), -1, device=device, dtype=torch.int32)
        self.camera_numbers_cuda = torch.full((B,), -1, device=device, dtype=torch.int32)
        self.landscape_mode_cuda = torch.ones((B,), device=device, dtype=torch.bool)
        self.inverse_krs_cuda = torch.zeros((B, 3, 3), device=device, dtype=torch.float)
        self.camera_origins_cuda = torch.zeros((B, 3), device=device, dtype=torch.float)
        self.grid_texture_objects_cuda = torch.zeros((B,), device=device, dtype=torch.int64)

        self.occupancy_grid_resolution = 0
        self.frame_to_grid_texture = {}
        if space_pruning_mode == DataLoader.SpacePruningMode.OCCUPANCY_GRID:
            self.occupancy_grid_resolution = self.dataset.get_occupancy_grid(frame_number=self.frame_numbers[0]).shape[0]
            self.cuda_grid_texture = occupancy_grid_native.OccupanyGrid(self.occupancy_grid_resolution,
                                                                        self.occupancy_grids_buffer_size)
        self.replacing = False
        self.slot_pairs = [None] * self.buffer_size           # the (camera, frame) pair every pool slot currently holds
        self.camera_frame_pairs = self._camera_frame_pair_generator()
        for slot in range(self.buffer_size):
            self._load_and_copy_camera_frame_data(next(self.camera_frame_pairs), slot)
        self.pair_load_index = self.buffer_size
        self.iternum = 0
        self.last_ray_indices = None

    # ------------------------------------------------------------------------------------------------
    def _camera_frame_pair_generator(self):
        """data_loader.py:356-394."""
        if self.mode != DataLoader.Mode.TRAINING:
            for pair in itertools.cycle(self.render_sequence):
                yield pair
        else:
            if self.max_num_frames_per_batch > 1:
                per_frame = int(np.ceil(self.buffer_size / (self.max_num_frames_per_batch - 1)))
            else:
                assert len(self.frame_numbers) == 1
                per_frame = len(self.camera_numbers)
            assert per_frame <= len(self.camera_numbers)
            info = {f: {"next": 0, "cams": list(self.camera_numbers)} for f in self.frame_numbers}
            frames = list(self.frame_numbers)
            while True:
                np.random.shuffle(frames)
                for f in frames:
                    it = info[f]
                    for _ in range(per_frame):
                        if it["next"] == 0:
                            np.random.shuffle(it["cams"])
                        yield it["cams"][it["next"]], f
                        it["next"] = (it["next"] + 1) % len(it["cams"])

    def _load_and_copy_camera_frame_data(self, camera_frame_pair: Tuple[int, int], buffer_index: int) -> None:
        """data_loader.py:424-506, writing straight into the device pool."""
        camera_number, frame_number = camera_frame_pair
        camera = self.cameras[camera_number]
        M = DataLoader.Mode
        if self.mode != M.TEST:
            rgb = np.ascontiguousarray(self.dataset.get_rgb(camera_number, frame_number)[..., [2, 1, 0]])  # BGR -> RGB
            if self.use_mask:
                mask = self.dataset.get_mask(camera_number, frame_number)
                rgb = rgb * mask
            else:
                mask = np.ones_like(rgb[..., 0:1])
            rgba = (np.concatenate((rgb, mask), axis=-1) * np.float32(255)).astype(np.uint8).reshape(-1, 4)
            self.pixel_colors[buffer_index].copy_(torch.from_numpy(rgba), non_blocking=False)
            if self.light_annotations is not None:
                import cv2  # only needed for the light-bloom border filter, as in the reference

                w = self.resolution[0]
                k = round((80 / 4088) * w)
                border = mask - cv2.erode(mask, np.ones((k, k), np.uint8))[..., np.newaxis]
                lm = np.zeros_like(rgb[..., 0:1], dtype=np.uint8)
                for c in self.light_annotations[camera_number]:
                    lm = cv2.circle(lm, (c[0], c[1]), c[2], (255), -1)
                self.light_mask[buffer_index].copy_(torch.from_numpy(((border > 0) & (lm > 0)).reshape(-1)))
        if self.space_pruning_mode == DataLoader.SpacePruningMode.OCCUPANCY_GRID:
            if self.mode == M.TRAINING:   # drop cache entries of frames that left the pool (data_loader.py:406-415)
                live = set(self.frame_numbers_cuda.tolist()) - {int(self.frame_numbers_cuda[buffer_index])}
                for f in [f for f in self.frame_to_grid_texture if f not in live and f != frame_number]:
                    self.frame_to_grid_texture.pop(f)
            if frame_number in self.frame_to_grid_texture:
                handle = self.frame_to_grid_texture[frame_number]
            else:
                grid = torch.from_numpy(self.dataset.get_occupancy_grid(frame_number)).to(self.device).contiguous()
                handle = self.cuda_grid_texture.add_grid(grid)
                if self.mode == M.TRAINING:
                    self.frame_to_grid_texture[frame_number] = handle
            self.grid_texture_objects_cuda[buffer_index] = handle
        self.slot_pairs[buffer_index] = (int(camera_number), int(frame_number))
        self.frame_numbers_cuda[buffer_index] = frame_number
        self.camera_numbers_cuda[buffer_index] = camera_number
        self.landscape_mode_cuda[buffer_index] = camera.width > camera.height
        self.inverse_krs_cuda[buffer_index].copy_(self.all_inverse_krs[camera_number])
        self.camera_origins_cuda[buffer_index].copy_(self.all_camera_origins[camera_number])

    # ------------------------------------------------------------------------------------------------
    @property
    def num_batches_per_full_image(self) -> int:
        return int(np.ceil(self.num_pixels_per_camera / self.batch_size))

    def __len__(self):
        if self.mode == DataLoader.Mode.TRAINING:
            raise NotImplementedError("Size of the training data loader is not defined.")
        return self.num_camera_frame_pairs * self.num_pixels_per_camera

    def __iter__(self):
        self.iternum = 0
        self.continue_replacing()
        return self

    def pause_replacing(self):
        self.replacing = False

    def continue_replacing(self):
        self.replacing = True

    def __next__(self) -> InputBatch:
        M = DataLoader.Mode
        width, height = self.resolution
        if self.mode == M.TRAINING:
            if self.replacing and self.buffer_size < self.num_camera_frame_pairs:
                for _ in range(self.replace_per_next):        # what the reference's replacer thread does in the background
                    self._load_and_copy_camera_frame_data(next(self.camera_frame_pairs), self.pair_load_index % self.buffer_size)
                    self.pair_load_index += 1
            ray_indices = torch.randint(0, self.buffer_size * self.num_pixels_per_camera, size=(self.batch_size,),
                                        dtype=torch.int64, device=self.device)
            out = self.ray_sampler_func(self.pixel_colors.view(-1, 4), self.light_mask.view(-1), self.frame_numbers_cuda,
                                        self.camera_numbers_cuda, self.grid_texture_objects_cuda, self.landscape_mode_cuda,
                                        ray_indices, self.inverse_krs_cuda, self.camera_origins_cuda, self.aabb,
                                        self.occupancy_grid_resolution, width, height, 4e-4, self.filter_light_bloom)
        else:
            if self.iternum >= len(self):
                self.pause_replacing()
                raise StopIteration
            start = self.iternum % self.num_pixels_per_camera
            end = min(start + self.batch_size, self.num_pixels_per_camera)
            ray_indices = torch.arange(start, end, dtype=torch.int64, device=self.device)
            image_num = self.iternum // self.num_pixels_per_camera
            slot = image_num % self.buffer_size
            camera_number, frame_number = self.render_sequence[image_num]
            # Load the image on demand into its ring slot whenever the slot holds another pair: the first pass beyond the
            # pool size, and EVERY later pass (the reference's replacer thread keeps cycling through render_sequence,
            # data_loader.py:471-506; the trainer re-iterates the validation loader every N steps).
            if self.slot_pairs[slot] != (int(camera_number), int(frame_number)):
                self._load_and_copy_camera_frame_data((camera_number, frame_number), slot)
            if not bool(self.landscape_mode_cuda[slot]):
                height, width = self.resolution
            one = lambda t: t[slot:slot + 1]
            out = self.ray_sampler_func(self.pixel_colors[slot], self.light_mask[slot],
                                        torch.tensor([frame_number], dtype=torch.int32, device=self.device),
                                        torch.tensor([camera_number], dtype=torch.int32, device=self.device),
                                        one(self.grid_texture_objects_cuda), torch.tensor([True], device=self.device),
                                        ray_indices, one(self.inverse_krs_cuda), one(self.camera_origins_cuda), self.aabb,
                                        self.occupancy_grid_resolution, width, height, 4e-4, self.filter_light_bloom)
        (ray_origins, ray_directions, rgba, frame_numbers, camera_numbers, minmaxes, ray_masks, dist, rel) = out
        self.iternum += ray_indices.numel()
        self.last_ray_indices = ray_indices
        return InputBatch(
            ray_origins=ray_origins.view(-1, 3), ray_directions=ray_directions.view(-1, 3), minmaxes=minmaxes.view(-1, 2),
            rgba=None if self.mode == M.TEST else rgba.view(-1, 4), ray_masks=ray_masks.view(-1, 1),
            frame_numbers=frame_numbers.view(-1, 1), camera_numbers=camera_numbers.view(-1, 1),
            unique_frame_numbers=torch.unique(frame_numbers, sorted=False, return_inverse=False).view(-1, 1),
            sample_distances=dist.view(-1, 1), ray_indices=rel.view(-1).long(), width=width, height=height)
