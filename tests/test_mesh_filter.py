"""Device mesh filter, no GPU: the workspace query, the C entries' host-side argument checks (each rejection names its
entry) and filter_mesh_device's input validation."""
import ctypes

import pytest
import torch


def test_filter_workspace_query(lib):
    from lara_b200 import _lib
    Nv, Nt = 1000, 2000
    b = _lib.mesh_filter_workspace_bytes(lib, Nv, Nt)
    slots = 16384                                   # the power of two >= 6 Nt
    assert b >= 12 * slots + 12 * Nt + 4 * (Nv + 1) + 4096 and b % 256 == 0
    assert _lib.mesh_filter_workspace_bytes(lib, 0, 0) > 0
    assert _lib.mesh_filter_workspace_bytes(lib, 2**31 - 1, 2**31 - 1) > 12 * 6 * (2**31 - 1)   # no size_t overflow
    n = ctypes.c_size_t()
    for nv, nt in ((-1, 4), (4, -1)):
        assert lib.srf_mesh_filter_workspace_bytes(nv, nt, ctypes.byref(n)) != 0
        assert lib.srf_last_error().startswith(b"srf_mesh_filter_workspace_bytes")
    assert lib.srf_mesh_filter_workspace_bytes(4, 4, None) != 0
    assert lib.srf_last_error().startswith(b"srf_mesh_filter_workspace_bytes")


def test_filter_count_rejects_bad_arguments(lib):
    box = (ctypes.c_double * 6)(0, 0, 0, 1, 1, 1)
    count = [None, 4, 2, 8, 8, box, 10, 256, 8]
    for i, bad in ((1, -1), (2, -1), (6, 0), (6, -3), (3, None), (4, None), (7, None), (7, 264), (8, None)):
        args = list(count)
        args[i] = bad
        assert lib.srf_mesh_filter_count(*args) != 0, i
        assert lib.srf_last_error().startswith(b"srf_mesh_filter_count"), i
    assert lib.srf_mesh_filter_count(*count[:6], 0, *count[7:]) != 0
    assert b"keep" in lib.srf_last_error()


def test_filter_emit_rejects_bad_arguments(lib):
    emit = [None, 4, 2, 8, 8, 8, 256, 3, 1, 8, 8, 8]
    for i, bad in ((1, -1), (2, -1), (7, -1), (8, -1), (7, 5), (8, 3), (3, None), (4, None), (5, None), (6, None),
                   (6, 272), (9, None), (10, None), (11, None)):
        args = list(emit)
        args[i] = bad
        assert lib.srf_mesh_filter_emit(*args) != 0, i
        assert lib.srf_last_error().startswith(b"srf_mesh_filter_emit"), i


def _mesh(dev="cpu"):
    return (torch.zeros(4, 3, device=dev), torch.tensor([[0, 1, 2], [1, 2, 3]], dtype=torch.int32, device=dev),
            torch.zeros(4, 3, device=dev))


def test_filter_mesh_device_rejects_cpu_tensors_and_bad_inputs():
    from lara_b200.mesh import filter_mesh_device
    v, t, c = _mesh()
    with pytest.raises(RuntimeError, match="CUDA"):
        filter_mesh_device((v, t, c))
    with pytest.raises(RuntimeError, match="CUDA"):
        filter_mesh_device((v.numpy(), t.numpy(), c.numpy()))
    # dtype and shape are checked on the same path; on a CPU-only machine the device check speaks first, so check the
    # messages the GPU-free way: each bad tensor is refused, none is accepted
    for bad in ((v.double(), t, c), (v, t.long(), c), (v, t, c.half()), (v[:, :2], t, c), (v, t.reshape(-1), c),
                (v, t, c[:3])):
        with pytest.raises(RuntimeError):
            filter_mesh_device(bad)


def test_filter_mesh_device_checks_dtype_and_shape_before_device(monkeypatch):
    """The messages for wrong dtypes and shapes, with the device check satisfied."""
    from lara_b200 import mesh as MS
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    v, t, c = _mesh()
    for bad, msg in (((v.double(), t, c), "vertices must be a torch.float32"),
                     ((v, t.long(), c), "triangles must be a torch.int32"),
                     ((v, t, c.half()), "colors must be a torch.float32"),
                     ((v[:, :2].contiguous(), t, c), r"vertices must be \[N,3\]"),
                     ((v, t.reshape(-1), c), r"triangles must be \[N,3\]"),
                     ((v, t, torch.zeros(4, 3, 2)), r"colors must be \[N,3\]"),
                     ((v, t, c[:3]), r"colors must be \(4, 3\)"),
                     ((v.t().contiguous().t(), t, c), "contiguous")):
        with pytest.raises(RuntimeError, match=msg):
            MS._check_mesh(*bad)
    assert MS._check_mesh(v, t, c) == (4, 2)
