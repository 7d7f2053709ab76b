"""CPU-side checks of osb200_create_pairs64, the constructor of 64-bit-key handles with uint32 payloads: argument errors
come before any device access, a machine without a GPU gets OSB200_ERR_NO_DEVICE, and the workspace of the (8, 4) shape
covers its alternate keys and payloads.  No compute calls."""
import ctypes

import pytest

INVALID_ARG, UNSUPPORTED, NO_DEVICE = -1, -3, -4


def test_create_pairs64_rejects_bad_arguments_without_touching_a_device():
    import gpusorting_b200 as g

    h = ctypes.c_void_p()
    assert g.lib.osb200_create_pairs64(None, 1024) == INVALID_ARG
    assert g.lib.osb200_create_pairs64(ctypes.byref(h), 0) == INVALID_ARG
    assert g.lib.osb200_create_pairs64(ctypes.byref(h), (1 << 34) + 1) == INVALID_ARG
    assert h.value is None
    assert g.lib.osb200_create(ctypes.byref(h), 1024, 8, 4) == UNSUPPORTED  # the shape comes from the new constructor only


def test_create_pairs64_without_gpu():
    import torch

    import gpusorting_b200 as g

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    h = ctypes.c_void_p()
    assert g.lib.osb200_create_pairs64(ctypes.byref(h), 1024) == NO_DEVICE
    assert h.value is None
    with pytest.raises(RuntimeError):
        g.OneSweepSorter(1024, 8, 4)


def test_workspace_bytes_of_the_pairs64_shape():
    import gpusorting_b200 as g

    for n in (1, 1000, 1 << 20, 1 << 30):
        ws = g.lib.osb200_workspace_bytes(n, 8, 4)
        assert ws >= 12 * n
        # the same descriptors and reductions as a (8, 0) handle, plus the alternate payloads
        assert ws == g.lib.osb200_workspace_bytes(n, 8, 0) + 4 * n
