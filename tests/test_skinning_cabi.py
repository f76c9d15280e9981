"""The skinning C-ABI: the ctypes prototypes, and every refusal returned before any launch (no GPU needed)."""
import ctypes as C

import pytest

from deodr_b200 import _cabi

P = 0x1000  # a fake, never dereferenced, device pointer
ARRAYS = ("parents", "centres", "level_offset", "level_index", "child_offset", "child_index", "skin_index",
          "skin_weight", "joint_offset", "joint_entry", "chunk_offset")


def _skeleton(J=4, V=10, K=2, levels=2, chunks=4, **null):
    s = _cabi.Skeleton()
    for name in ARRAYS:
        setattr(s, name, None if null.get(name) else P)
    s.nb_joints, s.nb_vertices, s.nb_influences, s.nb_levels, s.nb_chunks = J, V, K, levels, chunks
    return s


def _skin(lib, s=None, vertices=P, rotations=P, transforms=P, skinned=P):
    s = _skeleton() if s is None else s
    return lib.deodr_b200_skin(C.byref(s), vertices, rotations, transforms, skinned, None)


def _skin_b(lib, s=None, vertices=P, rotations=P, transforms=P, skinned_b=P, grad_in=None, vertices_b=P,
            weights_b=None, rotations_b=P, scratch=P):
    s = _skeleton() if s is None else s
    return lib.deodr_b200_skin_b(C.byref(s), vertices, rotations, transforms, skinned_b, grad_in, vertices_b,
                                 weights_b, rotations_b, scratch, None)


def test_the_prototypes_are_declared(build_native):
    lib = _cabi.load()
    declared = {name: (res, args) for name, res, args in _cabi.SYMBOLS}
    for name, n in (("deodr_b200_skin", 6), ("deodr_b200_skin_b", 11)):
        assert getattr(lib, name).restype is C.c_int
        assert len(declared[name][1]) == n


def test_the_struct_is_eleven_pointers_and_six_int32s():
    assert C.sizeof(_cabi.Skeleton) == 11 * 8 + 6 * 4


def test_a_null_skeleton_is_refused(build_native):
    lib = _cabi.load()
    assert lib.deodr_b200_skin(None, P, P, P, P, None) == _cabi.EINVAL
    assert lib.deodr_b200_skin_b(None, P, P, P, P, None, P, None, P, P, None) == _cabi.EINVAL


@pytest.mark.parametrize("name", ARRAYS)
def test_a_null_skeleton_array_is_refused(name, build_native):
    lib = _cabi.load()
    assert _skin(lib, _skeleton(**{name: True})) == _cabi.EINVAL
    assert _skin_b(lib, _skeleton(**{name: True})) == _cabi.EINVAL


@pytest.mark.parametrize("kw", [dict(vertices=None), dict(rotations=None), dict(transforms=None), dict(skinned=None)])
def test_a_null_forward_argument_is_refused(kw, build_native):
    lib = _cabi.load()
    assert _skin(lib, **kw) == _cabi.EINVAL
    assert b"bad argument" in lib.deodr_b200_last_error()


@pytest.mark.parametrize("kw", [dict(vertices=None), dict(rotations=None), dict(transforms=None),
                                dict(skinned_b=None), dict(vertices_b=None), dict(rotations_b=None),
                                dict(scratch=None)])
def test_a_null_adjoint_argument_is_refused(kw, build_native):
    lib = _cabi.load()
    assert _skin_b(lib, **kw) == _cabi.EINVAL
    assert b"bad argument" in lib.deodr_b200_last_error()


@pytest.mark.parametrize("sizes", [dict(J=0), dict(J=1025), dict(J=-1), dict(V=0), dict(V=-5), dict(K=0), dict(K=9),
                                   dict(levels=0), dict(levels=5), dict(chunks=-1)])
def test_sizes_out_of_range_are_refused(sizes, build_native):
    lib = _cabi.load()
    assert _skin(lib, _skeleton(**sizes)) == _cabi.EINVAL
    assert _skin_b(lib, _skeleton(**sizes)) == _cabi.EINVAL
    assert b"bad argument" in lib.deodr_b200_last_error()


def test_v_times_k_beyond_int32_is_unsupported(build_native):
    lib = _cabi.load()
    assert _skin(lib, _skeleton(V=2 ** 30, K=2)) == _cabi.EUNSUPPORTED
