"""The check of caller-supplied point outputs (Engine.transform(out=), register(transform_out=)),
without a device: the library writes 24 n_mov bytes into such a buffer, so anything but an
(n_mov, 3) float64 C-contiguous array or tensor must be refused before it is called."""
import numpy as np
import pytest
import torch

from simpleicp_b200._capi import _xyz_out_ptr

N = 7


def test_valid_outputs_pass():
    a = np.empty((N, 3))
    assert _xyz_out_ptr(a, N) == a.ctypes.data
    # offset by one element: any alignment of float64 is accepted (the library stages it)
    b = np.empty(3 * N + 1)[1:].reshape(N, 3)
    assert _xyz_out_ptr(b, N) == b.ctypes.data
    t = torch.empty((N, 3), dtype=torch.float64)
    assert _xyz_out_ptr(t, N) == t.data_ptr()
    assert _xyz_out_ptr(torch.empty(N + 1, 3, dtype=torch.float64)[1:], N) != 0


@pytest.mark.parametrize("make", [
    lambda: np.empty((N, 3), dtype=np.float32),
    lambda: np.empty((N, 3), dtype=np.int64),
    lambda: torch.empty((N, 3), dtype=torch.float32),
], ids=["numpy_f32", "numpy_i64", "torch_f32"])
def test_wrong_dtype_raises(make):
    with pytest.raises(ValueError, match="float64"):
        _xyz_out_ptr(make(), N)


@pytest.mark.parametrize("shape", [(N - 1, 3), (N + 1, 3), (N, 4), (3 * N,), (3, N), (1, N, 3)])
def test_wrong_shape_raises(shape):
    with pytest.raises(ValueError, match="shape"):
        _xyz_out_ptr(np.empty(shape), N)
    with pytest.raises(ValueError, match="shape"):
        _xyz_out_ptr(torch.empty(shape, dtype=torch.float64), N)


def test_non_contiguous_raises():
    with pytest.raises(ValueError, match="not contiguous"):
        _xyz_out_ptr(np.empty((3, N)).T, N)
    with pytest.raises(ValueError, match="not contiguous"):
        _xyz_out_ptr(np.empty((N, 6))[:, ::2], N)
    with pytest.raises(ValueError, match="not contiguous"):
        _xyz_out_ptr(np.asfortranarray(np.empty((N, 3))), N)
    with pytest.raises(ValueError, match="not contiguous"):
        _xyz_out_ptr(torch.empty((3, N), dtype=torch.float64).T, N)
    with pytest.raises(ValueError, match="not contiguous"):
        _xyz_out_ptr(torch.empty((2 * N, 3), dtype=torch.float64)[::2], N)


def test_other_types_raise():
    with pytest.raises(ValueError):
        _xyz_out_ptr([[0.0, 0.0, 0.0]] * N, N)
    with pytest.raises(ValueError):
        _xyz_out_ptr(memoryview(np.empty((N, 3))), N)
