"""CPU tests of the point-cloud marshaller (_cloud / _clouds in elevation_mapping.py) that input_pointcloud, input_sensors
and ShardedElevationMap.input_sensors share: NumPy and CPU torch inputs, no GPU and no libemap.so."""
import threading

import numpy as np
import pytest

from elevation_mapping_cupy_b200 import _lib
from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap, _cloud, _clouds


@pytest.fixture(autouse=True)
def no_library(monkeypatch):
    def load():
        raise AssertionError("the marshaller loaded libemap.so")
    monkeypatch.setattr(_lib, "load", load)


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError(f"the library was called: {name}")


def _bare_map():
    """an ElevationMap with no handle: any library call fails the test"""
    em = object.__new__(ElevationMap)
    em._L, em._h, em.map_lock = _NoLibrary(), None, threading.Lock()
    return em


def _rows(n=5, k=4, dtype=np.float32):
    return (np.arange(n * k).reshape(n, k) * 0.5).astype(dtype)


@pytest.mark.parametrize("dtype,code", [(np.float32, _lib.EMAP_F32), (np.float64, _lib.EMAP_F64)])
def test_float_arrays_are_read_in_place(dtype, code):
    a = _rows(dtype=dtype)
    ptr, n, row, dt, keep = _cloud(a, False)
    assert (ptr, n, row, dt) == (a.ctypes.data, 5, 4, code) and keep is a


@pytest.mark.parametrize("dtype", [np.int32, np.int64, np.float16])
def test_other_dtypes_become_float32(dtype):
    a = _rows(dtype=dtype)
    ptr, n, row, dt, keep = _cloud(a, False)
    assert (n, row, dt) == (5, 4, _lib.EMAP_F32)
    assert keep.dtype == np.float32 and keep.flags.c_contiguous and ptr == keep.ctypes.data
    assert np.array_equal(keep, a.astype(np.float32))


def test_cpu_torch_tensors_are_read_in_place():
    torch = pytest.importorskip("torch")
    t = torch.from_numpy(_rows(dtype=np.float64))
    ptr, n, row, dt, keep = _cloud(t, False)
    assert (ptr, n, row, dt) == (t.data_ptr(), 5, 4, _lib.EMAP_F64)
    ptr, n, row, dt, keep = _cloud(torch.arange(12, dtype=torch.int32).reshape(4, 3), False)
    assert (n, row, dt) == (4, 3, _lib.EMAP_F32) and np.array_equal(keep, np.arange(12, dtype=np.float32).reshape(4, 3))


@pytest.mark.parametrize("view", ["columns", "transposed", "every-other-row"])
def test_non_contiguous_input_is_copied_contiguous(view):
    a = _rows(n=6, k=6)
    v = {"columns": a[:, 1:4], "transposed": a.T, "every-other-row": a[::2]}[view]
    ptr, n, row, dt, keep = _cloud(v, False)
    assert keep.flags.c_contiguous and ptr == keep.ctypes.data and (n, row) == v.shape and np.array_equal(keep, v)


@pytest.mark.parametrize("shape", [(5, 2), (5, 0), (12,), (2, 3, 4)])
def test_fewer_than_three_columns_or_not_2d_is_rejected(shape):
    with pytest.raises(ValueError, match=r"\(N, >=3\)"):
        _cloud(np.zeros(shape, np.float32), False)


@pytest.mark.parametrize("other", [_rows(k=5), _rows(dtype=np.float64)], ids=["stride", "dtype"])
def test_clouds_of_one_frame_share_stride_and_dtype(other):
    with pytest.raises(ValueError, match="share row stride and dtype"):
        _clouds([_rows(), other], False)


def test_clouds_of_one_frame():
    a, b = _rows(n=5), _rows(n=7).astype(np.int16)
    ptrs, counts, stride, dt, keep = _clouds([a, b], False)
    assert list(counts) == [5, 7] and (stride, dt) == (4, _lib.EMAP_F32)
    assert list(ptrs) == [a.ctypes.data, keep[1][4].ctypes.data]


def test_device_ptrs_rejects_host_arrays():
    torch = pytest.importorskip("torch")
    for host in (_rows(), torch.from_numpy(_rows())):
        with pytest.raises(ValueError, match="device memory"):
            _cloud(host, True)
        with pytest.raises(ValueError, match="device memory"):
            _clouds([host], True)


def test_input_calls_reject_before_calling_the_library():
    em = _bare_map()
    R, t = np.eye(3, dtype=np.float32), np.zeros(3, np.float32)
    with pytest.raises(ValueError, match="device memory"):
        em.input_sensors([_rows()], [R], [t], 0.02, 0.02, device_ptrs=True)
    with pytest.raises(ValueError, match=r"\(N, >=3\)"):
        em.input_sensors([np.zeros((4, 2), np.float32)], [R], [t], 0.02, 0.02)
    with pytest.raises(ValueError, match=r"\(N, >=3\)"):
        em.input_pointcloud(np.zeros((4, 2), np.float32), None, R, t, 0.02, 0.02)
