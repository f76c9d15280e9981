"""The normal map's C-ABI: the ctypes prototypes, and every refusal returned before any launch (no GPU needed)."""
import ctypes as C

import pytest

from deodr_b200 import _cabi

P = 0x1000  # a fake, never dereferenced, device pointer
NAMES = ("deodr_b200_vertex_tangents", "deodr_b200_vertex_tangents_b", "deodr_b200_normal_map",
         "deodr_b200_normal_map_b")
ARGS = (8, 12, 6, 8)


def _mesh(T=4, V=5, **null):
    m = _cabi.MeshTopology()
    for name in ("faces", "faces_edges", "edge_face_offset", "edge_face_index", "vertex_face_offset",
                 "vertex_face_index"):
        setattr(m, name, None if null.get(name) else P)
    m.nb_faces, m.nb_edges, m.nb_vertices = T, 8, V
    return m


def _calls(lib, only, mesh=None, nb_uv=6, H=4, W=5, null=None):
    """The entry points of index in ``only``, each called with an argument it refuses (a call with valid arguments
    would launch on these fake pointers), ``null`` the index of a buffer argument set to NULL."""
    def q(i):
        return None if null == i else P
    m = mesh if mesh is not None else _mesh()
    calls = [
        lambda: lib.deodr_b200_vertex_tangents(C.byref(m), q(0), q(1), q(2), nb_uv, q(3), q(4), None),
        lambda: lib.deodr_b200_vertex_tangents_b(C.byref(m), q(0), q(1), q(2), nb_uv, q(3), q(4), q(5), q(6), q(7),
                                                 q(8), None),
        lambda: lib.deodr_b200_normal_map(q(0), q(1), H, W, q(2), None),
        lambda: lib.deodr_b200_normal_map_b(q(0), q(1), H, W, q(2), q(3), q(4), None),
    ]
    return [calls[i]() for i in only]


def test_the_prototypes_are_declared(build_native):
    lib = _cabi.load()
    declared = {name: (res, args) for name, res, args in _cabi.SYMBOLS}
    for name, n in zip(NAMES, ARGS):
        assert name in declared
        assert getattr(lib, name).restype is C.c_int
        assert len(declared[name][1]) == n


@pytest.mark.parametrize("null", range(9))
def test_a_null_buffer_is_refused(null, build_native):
    lib = _cabi.load()
    counts = (5, 9, 3, 5)  # buffer arguments of each entry point taken from the list
    only = [i for i in range(4) if null < counts[i]]
    assert _calls(lib, only, null=null) == [_cabi.EINVAL] * len(only)
    assert b"bad argument" in lib.deodr_b200_last_error()


@pytest.mark.parametrize("field", ["faces", "vertex_face_offset", "vertex_face_index"])
def test_a_topology_without_faces_or_its_vertex_csr_is_refused(field, build_native):
    lib = _cabi.load()
    assert _calls(lib, (0, 1), mesh=_mesh(**{field: True})) == [_cabi.EINVAL] * 2
    assert lib.deodr_b200_vertex_tangents(None, P, P, P, 6, P, P, None) == _cabi.EINVAL


@pytest.mark.parametrize("T,V,nb_uv", [(0, 5, 6), (4, 0, 6), (4, 5, 0), (-1, 5, 6), (4, 5, -3)])
def test_an_empty_mesh_or_uv_set_is_refused(T, V, nb_uv, build_native):
    assert _calls(_cabi.load(), (0, 1), mesh=_mesh(T, V), nb_uv=nb_uv) == [_cabi.EINVAL] * 2


@pytest.mark.parametrize("H,W", [(0, 5), (4, 0), (-1, 5), (4, -2)])
def test_an_empty_image_is_refused(H, W, build_native):
    assert _calls(_cabi.load(), (2, 3), H=H, W=W) == [_cabi.EINVAL] * 2
