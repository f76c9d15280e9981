"""The self-collision C-ABI: the ctypes prototypes, and every refusal returned before any launch (no GPU needed)."""
import ctypes as C
import math

import numpy as np
import pytest

from deodr_b200 import _cabi
from deodr_b200.mesh_fitter import collision_mesh_arrays

P = 0x1000  # a fake, never dereferenced, device pointer
ARRAYS = ("faces", "edges", "neighbour_offset", "neighbour_index", "corner_offset", "corner_index", "end_offset",
          "end_index")


def _mesh(F=4, E=6, V=4, **null):
    m = _cabi.CollisionMesh()
    for name in ARRAYS:
        setattr(m, name, None if null.get(name) else P)
    m.nb_faces, m.nb_edges, m.nb_vertices = F, E, V
    return m


def _collide(lib, mesh=None, ws=P, vertices=P, thickness=0.02, weight=1.0, cell=0.05, grad_in=None, grad=P, energy=P,
             dmin=P):
    mesh = _mesh() if mesh is None else mesh
    return lib.deodr_b200_self_collision(ws, C.byref(mesh), vertices, thickness, weight, cell, grad_in, grad, energy,
                                         dmin, None)


def _intersect(lib, mesh=None, ws=P, vertices=P, cell=0.05, pairs=P, capacity=16, count=True):
    mesh = _mesh() if mesh is None else mesh
    n = C.c_int64(-1)
    return lib.deodr_b200_self_intersections(ws, C.byref(mesh), vertices, cell, pairs, capacity,
                                             C.byref(n) if count else None, None)


def test_the_prototypes_are_declared(build_native):
    lib = _cabi.load()
    declared = {name: (res, args) for name, res, args in _cabi.SYMBOLS}
    for name, n in (("deodr_b200_self_collision", 11), ("deodr_b200_self_intersections", 8)):
        assert name in declared
        assert getattr(lib, name).restype is C.c_int
        assert len(declared[name][1]) == n


@pytest.mark.parametrize("kw", [dict(ws=None), dict(vertices=None), dict(grad=None), dict(energy=None),
                                dict(dmin=None)])
def test_a_null_pointer_is_refused(kw, build_native):
    lib = _cabi.load()
    assert _collide(lib, **kw) == _cabi.EINVAL
    assert b"bad argument" in lib.deodr_b200_last_error()
    assert lib.deodr_b200_self_collision(P, None, P, 0.02, 1.0, 0.05, None, P, P, P, None) == _cabi.EINVAL


@pytest.mark.parametrize("name", ARRAYS)
def test_a_null_mesh_array_is_refused(name, build_native):
    lib = _cabi.load()
    assert _collide(lib, _mesh(**{name: True})) == _cabi.EINVAL
    assert _intersect(lib, _mesh(**{name: True})) == _cabi.EINVAL


@pytest.mark.parametrize("F,E,V", [(0, 6, 4), (4, 0, 4), (4, 6, 0), (-1, 6, 4)])
def test_an_empty_mesh_is_refused(F, E, V, build_native):
    lib = _cabi.load()
    assert _collide(lib, _mesh(F, E, V)) == _cabi.EINVAL
    assert _intersect(lib, _mesh(F, E, V)) == _cabi.EINVAL


@pytest.mark.parametrize("kw", [dict(thickness=0.0), dict(thickness=-0.1), dict(thickness=math.nan),
                                dict(thickness=math.inf), dict(weight=-1.0), dict(weight=math.nan),
                                dict(weight=math.inf), dict(cell=math.nan), dict(cell=math.inf)])
def test_bad_parameters_are_refused(kw, build_native):
    lib = _cabi.load()
    assert _collide(lib, **kw) == _cabi.EINVAL
    assert b"bad argument" in lib.deodr_b200_last_error()


@pytest.mark.parametrize("kw", [dict(count=False), dict(pairs=None), dict(capacity=-1), dict(cell=0.0),
                                dict(cell=-1.0), dict(cell=math.nan), dict(ws=None), dict(vertices=None)])
def test_the_intersection_query_refuses_bad_arguments(kw, build_native):
    lib = _cabi.load()
    assert _intersect(lib, **kw) == _cabi.EINVAL
    assert b"bad argument" in lib.deodr_b200_last_error()


def test_face_indices_out_of_range_are_refused_where_the_topology_is_built():
    with pytest.raises(ValueError):
        collision_mesh_arrays(np.array([[0, 1, 2], [1, 2, 4]]), 4)
    with pytest.raises(ValueError):
        collision_mesh_arrays(np.array([[0, 1, -1]]), 3)
