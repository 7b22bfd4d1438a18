"""CPU oracle for the HumanRF per-ray hot path.  TEST INFRASTRUCTURE ONLY.

This package restates, on the CPU (numpy / PyTorch-CPU), the algorithm of the
reference's per-ray hot path (SURVEY.md section 8a):

    sampler (ray_sampler.cu) -> 4D-decomposed hash-grid encoding (tcnn HashGrid x4 +
    tensor_composition.cu) -> sigma / colour MLPs (tcnn FullyFusedMLP) ->
    transmittance / compositing (nerfacc 0.3.1) -> loss (trainer.py).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this package.  The product package
``humanrf_b200`` never imports it and fails loudly when its CUDA library is missing.

PARITY PINNING STATUS (see DESIGN.md "Oracle"):
  * first-party reference code that runs on the CPU here (``humanrf/input.py``,
    ``humanrf/utils/activation.py``, ``humanrf/utils/loss.py``, ``InputBatch``,
    ``CameraData``) is pinned by golden vectors generated from the reference itself
    (``tests/golden/make_golden.py``).
  * first-party reference code that needs tcnn / nerfacc only as callees -- ``HumanRF.__init__`` /
    ``density`` / ``forward``, ``Decomposition4D.forward``, ``prune_samples``, ``render``,
    ``merge_render_outputs``, ``adaptive_temporal_partitioning`` -- is executed LIVE on the CPU
    with those callees stubbed (a recording stub, or this package's restatement of the callee)
    and compared with this package (``tests/test_reference_live_cpu.py``, where the
    reference is mounted).
  * first-party CUDA (``tensor_composition.cu``, ``ray_sampler.cu``, ``occupancy_grid.cu``,
    ``occupancy_grid_generation.cu``) is pinned on the GPU box against ``oracle/_ref`` builds
    of the reference sources (``oracle/build_ref.py``) when those built here.
  * tiny-cuda-nn (un-pinned git HEAD) and nerfacc==0.3.1 are NOT part of the reference checkout and
    cannot be installed here: their published algorithms are restated from memory of the
    public sources and are **parity unpinned**.
"""
