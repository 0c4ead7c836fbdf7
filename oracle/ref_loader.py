"""Import the UNMODIFIED reference modules from a reference checkout (LUNGMASK_REFERENCE_ROOT).

TEST INFRASTRUCTURE ONLY.  Used by oracle/make_golden.py and by the `not gpu` tests that validate
`oracle.restate` against the reference itself.  Tests, smoke() and bench.py read the fixtures it
produced (tests/golden/) and never call this.
"""
import importlib
import os
import sys

from . import standins

REFERENCE_ROOT = os.environ.get("LUNGMASK_REFERENCE_ROOT", "")


def available() -> bool:
    """True when LUNGMASK_REFERENCE_ROOT names a directory holding the reference's lungmask/mask.py (no default: an
    unset or empty value never falls back to whatever the current directory holds)."""
    return bool(REFERENCE_ROOT) and os.path.isabs(REFERENCE_ROOT) and os.path.isfile(os.path.join(REFERENCE_ROOT, "lungmask", "mask.py"))


_cached = None


def load():
    """Returns a namespace with the reference's `mask`, `utils`, `resunet` modules (verbatim)."""
    global _cached
    if _cached is not None:
        return _cached
    if not available():
        raise RuntimeError("set LUNGMASK_REFERENCE_ROOT to the absolute path of a reference checkout (now %r)" % REFERENCE_ROOT)
    standins.install()
    # The reference imports itself as `lungmask`; this repo ships a same-named drop-in shim, so
    # park whatever is registered under that name while the reference is being imported.
    parked = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "lungmask" or k.startswith("lungmask.")}
    sys.path.insert(0, REFERENCE_ROOT)
    try:
        mask = importlib.import_module("lungmask.mask")
        utils = importlib.import_module("lungmask.utils")
        resunet = importlib.import_module("lungmask.resunet")
    finally:
        sys.path.remove(REFERENCE_ROOT)
        for k in [k for k in sys.modules if k == "lungmask" or k.startswith("lungmask.")]:
            del sys.modules[k]
        sys.modules.update(parked)

    class Ref:
        pass

    ref = Ref()
    ref.mask, ref.utils, ref.resunet = mask, utils, resunet
    _cached = ref
    return ref
