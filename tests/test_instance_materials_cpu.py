"""
CPU checks of per-instance materials (rt_set_instance_materials, include/rt_b200.h): the null-context check of the entry point and
the arrays Context.set_instance_materials / HostRender.set_instance_materials pass to it.
"""
import numpy as np
import pytest

from raytracing_b200 import capi


def test_entry_point_rejects_a_null_context():
    L = capi.load_library()
    rows = np.zeros(8, np.uint32)
    of = np.zeros(1, np.uint32)
    assert L.rt_set_instance_materials(None, rows.ctypes.data, 1, of.ctypes.data, 1) == -1
    assert L.rt_set_instance_materials(None, None, 0, None, 0) == -1


def test_arrays_of_the_binding():
    rows, of = capi.instance_material_arrays([[1, 0, 2], [0, 1, 2]], [1, -1, None, 0, 0xFFFFFFFF])
    assert rows.dtype == np.dtype("<u4") and rows.shape == (2, 3) and rows.flags.c_contiguous
    assert of.dtype == np.dtype("<u4") and of.tolist() == [1, 0xFFFFFFFF, 0xFFFFFFFF, 0, 0xFFFFFFFF]
    rows, of = capi.instance_material_arrays([], [])
    assert rows.shape == (0, 0) and of.shape == (0,)
    rows, _ = capi.instance_material_arrays(np.arange(6, dtype=np.int64).reshape(2, 3)[:, ::-1], [0])
    assert rows.tolist() == [[2, 1, 0], [5, 4, 3]] and rows.flags.c_contiguous


@pytest.mark.parametrize("remaps, of", [([1, 0, 2], [0]), ([[0, 1]], [-2]), ([[0, 1]], [1 << 32])])
def test_arrays_of_the_binding_refuse(remaps, of):
    with pytest.raises(ValueError):
        capi.instance_material_arrays(remaps, of)
