"""Writes tests/golden/reference_live.npz: what the reference's own first-party Python computes on the randomized inputs of
tests/test_reference_live_cpu.py (every `reference_*` function there).  Needs a checkout of the reference:

    python tests/golden/make_reference_live_golden.py <path to the reference checkout>
"""
import sys
import types
from pathlib import Path

import numpy as np

TESTS = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(TESTS.parent), str(TESTS)]


def main(ref_root):
    sys.path.insert(0, str(ref_root))
    import actorshq.dataset.input_batch as ib
    import humanrf.input as inp
    import humanrf.scene_representation.query_io as qio
    import humanrf.utils.activation as act
    import humanrf.utils.loss as loss
    # adaptive_temporal_partitioning imports VolumetricDataset only for an annotation (needs cv2 etc.): stub it
    if "actorshq.dataset.volumetric_dataset" not in sys.modules:
        stub = types.ModuleType("actorshq.dataset.volumetric_dataset")
        stub.VolumetricDataset = object
        sys.modules["actorshq.dataset.volumetric_dataset"] = stub
    import humanrf.adaptive_temporal_partitioning as atp
    import test_reference_live_cpu as T

    ref = types.SimpleNamespace(ib=ib, inp=inp, qio=qio, act=act, loss=loss, atp=atp)
    out = {}
    for name in sorted(n for n in dir(T) if n.startswith("reference_")):
        out.update(getattr(T, name)(ref))
    np.savez_compressed(T.GOLD, **out)
    print("wrote", T.GOLD, len(out), "arrays")


if __name__ == "__main__":
    main(sys.argv[1])
