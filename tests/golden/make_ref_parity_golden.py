"""Writes tests/golden/ref_parity.npz: what the reference's own CUDA extensions (oracle/_ref, built by oracle/build_ref.py
from a checkout of the reference) compute on the seeded inputs of tests/test_ref_parity_gpu.py and
tests/test_occupancy_tools_gpu.py (every `reference_*` function there).  Needs a GPU:

    python tests/golden/make_ref_parity_golden.py [output .npz, default tests/golden/ref_parity.npz]
"""
import importlib
import sys
from pathlib import Path

import numpy as np
import torch

TESTS = Path(__file__).resolve().parent.parent
REF = TESTS.parent / "oracle" / "_ref"
sys.path[:0] = [str(TESTS.parent), str(TESTS), str(REF)]


def ref(name):
    if not (REF / f"{name}.so").exists():
        raise SystemExit(f"oracle/_ref/{name}.so not built (python oracle/build_ref.py)")
    return importlib.import_module(name)


def main(out_path):
    import test_occupancy_tools_gpu
    import test_ref_parity_gpu

    cuda = torch.device("cuda:0")
    out = {}
    for mod in (test_ref_parity_gpu, test_occupancy_tools_gpu):
        for name in sorted(n for n in dir(mod) if n.startswith("reference_")):
            out.update(getattr(mod, name)(ref, cuda))
    np.savez_compressed(out_path, **out)
    print("wrote", out_path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else str(TESTS / "golden" / "ref_parity.npz"))
