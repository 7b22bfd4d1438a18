"""Makes the reference's own import paths resolve to this implementation, so `humanrf/run.py` and
`humanrf/trainer.py` run unchanged (SURVEY 8b):

    import humanrf_b200.dropin; humanrf_b200.dropin.install()      # before importing humanrf.run / humanrf.trainer

Only the hot-path modules are replaced; everything else (args, configs, Trainer, DataLoader, dataset IO,
evaluation) keeps coming from the reference checkout on PYTHONPATH."""
from __future__ import annotations

import importlib
import sys

_MAP = {
    "humanrf.scene_representation.humanrf": "humanrf_b200.scene_representation.humanrf",
    "humanrf.scene_representation.query_io": "humanrf_b200.scene_representation.query_io",
    "humanrf.scene_representation.tensor_composition_native": "humanrf_b200.scene_representation.tensor_composition_native",
    "humanrf.volume_rendering": "humanrf_b200.volume_rendering",
    "humanrf.input": "humanrf_b200.input",
    "actorshq.dataset.input_batch": "humanrf_b200.dataset.input_batch",
    "actorshq.dataset.ray_sampler_native": "humanrf_b200.dataset.ray_sampler_native",
    "actorshq.dataset.occupancy_grid_native": "humanrf_b200.dataset.occupancy_grid_native",
    "actorshq.toolbox.occupancy_grid_generation_native": "humanrf_b200.toolbox.occupancy_grid_generation_native",
    "humanrf.adaptive_temporal_partitioning": "humanrf_b200.adaptive_temporal_partitioning",
}


def install() -> None:
    for ref_name, our_name in _MAP.items():
        mod = importlib.import_module(our_name)
        sys.modules[ref_name] = mod
        parent_name, leaf = ref_name.rsplit(".", 1)
        try:  # bind the attribute on the (reference's) parent package so `import a.b.c as x` resolves too
            setattr(importlib.import_module(parent_name), leaf, mod)
        except ImportError:
            pass  # reference checkout not on sys.path yet; the sys.modules entry still serves `from a.b.c import x`
