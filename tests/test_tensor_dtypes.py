"""The torch dtype -> LM_DTYPE_* map of LMInferer's tensor inputs (no GPU needed): the codes are the header's, and the
dtypes the engine does not read are refused with a TypeError before anything reaches the device."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_dtype_codes_match_header():
    from lungmask_b200 import _native
    header = open(os.path.join(ROOT, "include", "lungmask_b200.h")).read()
    defined = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define LM_DTYPE_(\w+)\s+(\d+)", header)}
    assert defined == {name: getattr(_native, "DTYPE_" + name) for name in defined}
    assert sorted(defined) == sorted(["I16", "F32", "F64", "U8", "I8", "I32", "I64", "F16", "BF16"])


def test_tensor_dtype_map():
    import torch
    from lungmask_b200 import _native
    from lungmask_b200.mask import _tensor_dtype_code
    want = {torch.bool: _native.DTYPE_U8, torch.uint8: _native.DTYPE_U8, torch.int8: _native.DTYPE_I8,
            torch.int16: _native.DTYPE_I16, torch.int32: _native.DTYPE_I32, torch.int64: _native.DTYPE_I64,
            torch.float16: _native.DTYPE_F16, torch.bfloat16: _native.DTYPE_BF16, torch.float32: _native.DTYPE_F32,
            torch.float64: _native.DTYPE_F64}
    for dt, code in want.items():
        assert _tensor_dtype_code(torch.zeros(1, dtype=dt)) == code, dt
    for dt in (torch.complex64, torch.complex128, torch.uint16, torch.uint32, torch.uint64):
        with pytest.raises(TypeError, match="not supported"):
            _tensor_dtype_code(torch.zeros(1, dtype=dt))
