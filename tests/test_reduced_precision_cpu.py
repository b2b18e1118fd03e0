"""CPU: what the 16-bit feature path still refuses, and the dtype -> CL3D_DTYPE_* map (no GPU needed)."""
import re

import pytest
import torch

from closerlook3d_b200 import ops
from closerlook3d_b200.local_aggregation_operators import _check_inputs

FLOATS = [torch.float32, torch.float16, torch.bfloat16]


def test_dtype_map_is_total_over_the_floating_types_and_matches_the_header():
    import os
    hdr = open(os.path.join(os.path.dirname(ops.__file__), "..", "include", "cl3d.h")).read()
    codes = {n: int(v) for n, v in re.findall(r"#define CL3D_DTYPE_(\w+) (\d+)", hdr)}
    assert codes == {"F32": 0, "F16": 1, "BF16": 2}
    assert ops.DTYPE_CODE == {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
    assert set(ops.DTYPE_CODE) == set(FLOATS)


class _FakeCuda:
    """stands in for a CUDA tensor of the given dtype (the checks look at is_cuda / dtype / contiguity only)"""

    def __init__(self, dtype):
        self.dtype, self.is_cuda = dtype, True

    def is_contiguous(self):
        return True


@pytest.mark.parametrize("dtype", [torch.float64, torch.int32, torch.int64, torch.uint8])
def test_non_float_features_still_raise(dtype):
    with pytest.raises(RuntimeError, match="float tensor"):
        ops.require_features(_FakeCuda(dtype), "features")
    xyz, m = _FakeCuda(torch.float32), _FakeCuda(torch.int32)
    with pytest.raises(RuntimeError, match="float tensor"):
        _check_inputs(xyz, xyz, m, m, _FakeCuda(dtype))


@pytest.mark.parametrize("dtype", FLOATS)
def test_accepted_feature_dtypes_map_to_their_code(dtype):
    assert ops.require_features(_FakeCuda(dtype), "features") == ops.DTYPE_CODE[dtype]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float64])
def test_cpu_features_still_raise_cuda(dtype):
    """xyz and masks pass the CUDA checks (fakes), so it is the CPU features that raise"""
    feats = torch.rand(1, 12, 32).to(dtype)
    xyz, m = _FakeCuda(torch.float32), _FakeCuda(torch.int32)
    with pytest.raises(RuntimeError, match="points must be a CUDA tensor"):
        _check_inputs(xyz, xyz, m, m, feats)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.require_features(feats, "features")
