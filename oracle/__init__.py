"""CPU oracle for the IDE-3D volumetric-rendering hot path.

TEST INFRASTRUCTURE ONLY.  This package is a CPU restatement (torch-CPU / numpy, fp32) of the
reference algorithm so that the CUDA kernels in ``ide-3d_b200/csrc`` can be checked against it.
Only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference`` legs of
``bench.py`` may import it.  The product package (``ide3d_b200``) never imports it and has no CPU
compute path of its own.

Pinning status
--------------
The reference repository ships **no tests and no golden vectors** (SURVEY.md §4, §8c), so the oracle
is pinned the only way available: every function here was compared, in the build container, against
the reference's own Python functions imported from the reference tree (``tests/golden/make_golden.py``)
and the resulting input/output tensors are committed under ``tests/golden/*.npz``.
``tests/test_oracle_golden.py`` replays those fixtures on every run (no reference tree needed).

What is NOT pinned by the reference ("parity unpinned" — the generator class that composes the
free functions is absent from the reference tree, SURVEY.md §0): the decoder MLP widths, the
world->plane coordinate scale and the order of composition.  Those are restated in
``oracle.renderer.render_frames`` from the call-site contract and documented in DESIGN.md.
"""

from . import camera, ops, renderer  # noqa: F401
