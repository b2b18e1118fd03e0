"""CPU: what the fused multi-shape head refuses at its 16-bit boundary (no GPU needed)."""
import ctypes

import pytest
import torch

from closerlook3d_b200 import _lib, ops, partseg

CL3D_ERR_BAD_ARG = -1


class _FakeCuda:
    """stands in for a CUDA tensor of the given dtype (the checks look at is_cuda / dtype / contiguity only)"""

    def __init__(self, dtype):
        self.dtype, self.is_cuda = dtype, True

    def is_contiguous(self):
        return True


def _desc(grads=False):
    d = _lib.MHeadDesc()
    d.S, d.C = 1, 8
    d.num_parts[0] = 2
    if grads:
        d.grad_logits[0] = 16    # never dereferenced: the dtype is refused first
    return d


@pytest.mark.parametrize("code", [-1, 3, 7])
def test_unknown_dtype_codes_are_refused_by_both_entry_points(code):
    L = _lib.lib()
    d = _desc()
    dp = ctypes.addressof(d)
    rc = L.cl3d_mhead_fwd(dp, None, code, 2, 16, None, None, None, None, None, 1e-5, 0.1, 1, None, None, None, 0, None)
    assert rc == CL3D_ERR_BAD_ARG
    assert f"unknown dtype code {code}" in L.cl3d_last_error().decode()
    d = _desc(grads=True)
    dp = ctypes.addressof(d)
    rc = L.cl3d_mhead_bwd(dp, None, code, 2, 16, None, None, None, 1, None, None, None, None, None, None, None, 0,
                          None)
    assert rc == CL3D_ERR_BAD_ARG
    assert f"unknown dtype code {code}" in L.cl3d_last_error().decode()


def test_workspace_sizes_do_not_take_a_dtype():
    L = _lib.lib()
    d = _desc()
    dp = ctypes.addressof(d)
    assert L.cl3d_mhead_fwd_workspace_bytes(dp, 2, 16) > 0 and L.cl3d_mhead_bwd_workspace_bytes(dp, 2, 16) > 0


@pytest.mark.parametrize("x_dt,g_dt", [(torch.bfloat16, torch.float32), (torch.float16, torch.bfloat16),
                                       (torch.float32, torch.float16)])
def test_grad_logits_in_another_dtype_than_x_raise(x_dt, g_dt):
    with pytest.raises(RuntimeError, match="d/dlogits must have x's dtype"):
        ops.mhead_bwd(_FakeCuda(x_dt), None, None, None, [2, 3], [None, _FakeCuda(g_dt)], True)


@pytest.mark.parametrize("dtype", [torch.float64, torch.int32])
def test_non_float_x_is_refused(dtype):
    with pytest.raises(RuntimeError, match="float tensor"):
        ops.mhead_fwd(_FakeCuda(dtype), None, None, None, None, None, [2], None, None, None, 1e-5, 0.1, True)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_cpu_input_is_not_eligible(dtype):
    heads = torch.nn.ModuleList([torch.nn.Sequential(torch.nn.Conv1d(8, 8, 1, bias=False), torch.nn.BatchNorm1d(8),
                                                     torch.nn.ReLU(), torch.nn.Conv1d(8, 3, 1))])
    assert not partseg.fused_eligible(heads, torch.zeros(2, 8, 16, dtype=dtype))
