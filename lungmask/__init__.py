"""Drop-in alias: `import lungmask` resolves to the H100 engine's mirror of the reference package.

`from lungmask import LMInferer`, `from lungmask.mask import MODEL_URLS, get_model, apply, apply_fused`,
`from lungmask.utils import preprocess, postprocessing, ...` and `python -m lungmask IN OUT` all reach
`lungmask_b200` (see INTEGRATION.md).  Nothing is implemented here.
"""
import sys as _sys

import lungmask_b200 as _impl
from lungmask_b200 import mask as _mask, utils as _utils, logger as _logger

_sys.modules[__name__ + ".mask"] = _mask
_sys.modules[__name__ + ".utils"] = _utils
_sys.modules[__name__ + ".logger"] = _logger
mask, utils, logger = _mask, _utils, _logger
LMInferer = _impl.LMInferer
__all__ = ["LMInferer"]
