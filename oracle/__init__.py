"""oracle/ — TEST INFRASTRUCTURE ONLY.

CPU restatement of the JoHof/lungmask hot path (`LMInferer.apply`: preprocess -> U-Net forward ->
postprocess -> reshape), used as the checker for the CUDA engine in `lungmask_b200/`.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s CPU-baseline / `--impl reference` legs may
import anything from here.  The product path (`lungmask_b200`) never imports `oracle` and has no
CPU fallback.

Pinning status (see DESIGN.md "Oracle"):
  * `oracle.restate` is checked in this container against the reference's own modules imported
    verbatim from a reference checkout (`oracle.ref_loader`) and against the reference's known-answer
    tests (tests/test_utils.py:58-63,73-107,124-159), and against fixtures in tests/golden/ that
    were generated from the verbatim reference by `oracle/make_golden.py`.
  * The reference's third-party natives skimage / fill_voids are NOT installed here; their
    behaviour is restated from documented semantics in `oracle.standins` and pinned only by the
    reference's six known-answer tests.  `skimage.morphology.area_closing` (single-slice volumes)
    has no reference test at all: PARITY UNPINNED for that branch.
  * Trained-weight goldens (tests/test_mask.py:30-60) need the released .pth files (no network):
    PARITY UNPINNED for trained weights; parity is established on synthetic state_dicts with the
    exact reference key layout.
"""
