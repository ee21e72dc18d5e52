"""bgs_entity_list without a GPU: the ctypes prototypes against the header, the C calls' refusal of a NULL context or list,
the Python mirror's ValueErrors before any call, and the matrix layouts set_transforms derives from host arrays and from
__cuda_array_interface__ objects."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import EntityList, matrices_arg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "bgs.h")
SRC = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def _params(name):
    return [p.strip() for p in re.search(rf"(?:bgs_status|void|uint32_t) {name}\((.*?)\);", SRC, flags=re.S).group(1).split(",")]


def test_prototypes():
    """Each call's parameter count matches abi.py's; the render calls take bgs_render_entities_many's frame arguments."""
    for name, _, args in abi.SYMBOLS:
        if "entity_list" in name:
            assert len(_params(name)) == len(args), name
    tail = _params("bgs_render_entities_many")[6:]
    assert _params("bgs_render_entity_list")[2:] == tail
    assert _params("bgs_render_entity_list_pick")[2:] == _params("bgs_render_entities_pick_many")[6:]
    assert "BGS_MATRIX_COLUMN_MAJOR = 0, BGS_MATRIX_ROW_MAJOR = 1" in SRC
    assert (abi.BGS_MATRIX_COLUMN_MAJOR, abi.BGS_MATRIX_ROW_MAJOR) == (0, 1)


def test_null_context_or_list():
    lib = abi.load()
    out = C.c_void_p()
    assert lib.bgs_entity_list_create(None, None, None, None, None, 0, C.byref(out)) == abi.BGS_EINVAL
    assert not out.value
    assert lib.bgs_entity_list_set(None, None, 0, None, None, None, None) == abi.BGS_EINVAL
    assert lib.bgs_entity_list_append(None, 0, None, None, None, None) == abi.BGS_EINVAL
    assert lib.bgs_entity_list_truncate(None, 0) == abi.BGS_EINVAL
    assert lib.bgs_entity_list_set_transforms(None, 0, 0, None, 0, 0) == abi.BGS_EINVAL
    assert lib.bgs_entity_list_size(None) == 0
    lib.bgs_entity_list_destroy(None)
    assert lib.bgs_render_entity_list(None, None, None, None, None, None, None, 0, 0) == abi.BGS_EINVAL
    assert lib.bgs_render_entity_list_pick(None, None, None, None, None, None, None, 0, 0, None) == abi.BGS_EINVAL


class _Handle:
    temporal = False
    precompute_covariance = False
    n = 4


class _Refused(Exception):
    pass


def _offline_list(entities):
    """An EntityList with no context whose C calls all raise: what it refuses, it refuses before any call."""
    lst = EntityList.__new__(EntityList)
    lst._h = C.c_void_p()
    lst._handles = [h for h, _, _ in entities]
    lst._settings = [st for _, st, _ in entities]

    class _Plugin:
        def __getattr__(self, name):
            raise _Refused(name)

    lst._plugin = _Plugin()
    lst._lib = _Plugin()
    return lst


def test_python_mirror_refuses_before_any_call():
    a = B.CloudSettings()
    lst = _offline_list([(_Handle(), a, None)] * 3)
    assert len(lst) == 3
    e = (_Handle(), a, None)
    with pytest.raises(ValueError, match="entity 4 has radix_sort_depth_bits = 16, entity 0"):
        lst.append([e, (_Handle(), B.CloudSettings(radix_sort_depth_bits=16), None)])
    with pytest.raises(ValueError, match="entity 2 has radix_sort_depth_bits"):
        lst.set([2], [(_Handle(), B.CloudSettings(radix_sort_depth_bits=24), None)])
    with pytest.raises(ValueError, match="indices"):
        lst.set([3], [e])
    with pytest.raises(ValueError, match="indices"):
        lst.set([1, 1], [e, e])
    with pytest.raises(ValueError, match="2 indices for 1"):
        lst.set([0, 1], [e])
    with pytest.raises(ValueError, match="truncate"):
        lst.truncate(4)
    with pytest.raises(ValueError, match="at most 65536"):
        lst.append([e] * (abi.BGS_ENTITIES_MANY_MAX - 2))
    with pytest.raises(ValueError, match="beyond 3"):
        lst.set_transforms(2, np.zeros((2, 4, 4), np.float32))
    with pytest.raises(ValueError, match="shape"):
        lst.set_transforms(0, np.zeros((2, 3, 4), np.float32))
    with pytest.raises(ValueError, match="no entities"):
        _offline_list([])._frame("render_entity_list")
    # accepted edits reach the library (here: the refusing stand-in)
    with pytest.raises(_Refused):
        lst.set([2], [e])


class _Cai:
    def __init__(self, shape, strides, typestr="<f4", stream=None):
        self.__cuda_array_interface__ = {"shape": shape, "strides": strides, "typestr": typestr, "data": (0x1000, False),
                                         "version": 3, "stream": stream}


def test_matrix_layouts():
    m = np.arange(2 * 16, dtype=np.float64).reshape(2, 4, 4)
    ptr, count, layout, device, stream, keep = matrices_arg(m)
    assert (count, layout, device, stream) == (2, abi.BGS_MATRIX_ROW_MAJOR, False, None)
    assert keep.dtype == np.float32 and keep.flags.c_contiguous and ptr == keep.ctypes.data
    # a transposed host array is made contiguous row-major (its values, not its memory)
    t = np.ascontiguousarray(m.astype(np.float32)).transpose(0, 2, 1)
    _, _, layout, _, _, keep = matrices_arg(t)
    assert layout == abi.BGS_MATRIX_ROW_MAJOR and np.array_equal(keep, t)
    assert matrices_arg(_Cai((3, 4, 4), None))[1:5] == (3, abi.BGS_MATRIX_ROW_MAJOR, True, None)
    assert matrices_arg(_Cai((3, 4, 4), (64, 16, 4), stream=7))[1:5] == (3, abi.BGS_MATRIX_ROW_MAJOR, True, 7)
    assert matrices_arg(_Cai((3, 4, 4), (64, 4, 16)))[2] == abi.BGS_MATRIX_COLUMN_MAJOR
    assert matrices_arg(_Cai((3, 4, 4), (64, 4, 16)))[0] == 0x1000
    with pytest.raises(ValueError, match="neither contiguous"):
        matrices_arg(_Cai((3, 4, 4), (128, 16, 4)))   # every other matrix of a larger array
    with pytest.raises(ValueError, match="shape"):
        matrices_arg(_Cai((3, 16), None))
    with pytest.raises(TypeError, match="float32"):
        matrices_arg(_Cai((3, 4, 4), None, "<f8"))
