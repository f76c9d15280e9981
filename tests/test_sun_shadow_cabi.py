"""The directional light's shadow C-ABI: the ctypes prototypes, and every refusal returned before any launch (no GPU
needed)."""
import ctypes as C
import math

import pytest

from deodr_b200 import _cabi

P = 0x1000  # a fake, never dereferenced, device pointer
NAMES = ("deodr_b200_sun_project", "deodr_b200_sun_project_b", "deodr_b200_sun_visibility",
         "deodr_b200_sun_visibility_b", "deodr_b200_phong_shade_sun_shadowed", "deodr_b200_phong_shade_sun_shadowed_b")
ARGS = (9, 12, 9, 12, 10, 16)


def _io(nc=3, split=False):
    io = _cabi.PhongIO()
    for name in ("channels", "params", "camera_center", "background", "image", "image_b", "channels_b", "params_b"):
        setattr(io, name, P)
    io.H, io.W, io.C = 4, 5, nc
    if split:
        io.off_albedo, io.off_normal, io.off_position, io.off_coverage = -1, 0, 3, 6
    else:
        io.off_albedo, io.off_normal, io.off_position, io.off_coverage = 0, nc, nc + 3, nc + 6
    return io


def _center(c=(0.0, 0.0, 0.0)):
    return (C.c_double * 3)(*c)


def _calls(lib, only, io=None, center=None, radius=1.0, M=64, bias=0.01, soft=0.05, lights=P, L=2, LS=1, vis=None,
           sh=None, S=0, null=None):
    """The entry points of index in ``only`` (each called with an argument it refuses: a call with valid arguments
    would launch on these fake pointers) with ``null`` the index of a buffer argument set to NULL."""
    ptrs = [P] * 8

    def q(i):
        return None if null == i else ptrs[i]
    io = io if io is not None else _io()
    center = center if center is not None else _center()
    calls = [
        lambda: lib.deodr_b200_sun_project(q(0), 10, q(1), center, radius, M, q(2), q(3), None),
        lambda: lib.deodr_b200_sun_project_b(q(0), 10, q(1), center, radius, M, q(2), q(3), q(4), q(5), q(6), None),
        lambda: lib.deodr_b200_sun_visibility(C.byref(io), center, radius, q(0), M, bias, soft, q(1), None),
        lambda: lib.deodr_b200_sun_visibility_b(C.byref(io), center, radius, q(0), M, bias, soft, q(1), q(2), q(3),
                                                q(4), None),
        lambda: lib.deodr_b200_phong_shade_sun_shadowed(C.byref(io), None, sh, S, lights, L, LS, vis, q(0), None),
        lambda: lib.deodr_b200_phong_shade_sun_shadowed_b(C.byref(io), None, None, sh, S, sh, lights, L, LS, q(1),
                                                          vis, vis, q(0), q(2), q(3), None),
    ]
    return [calls[i]() for i in only]


ALL = range(6)


def test_the_prototypes_are_declared(build_native):
    lib = _cabi.load()
    declared = {name: (res, args) for name, res, args in _cabi.SYMBOLS}
    for name, n in zip(NAMES, ARGS):
        assert name in declared
        assert getattr(lib, name).restype is C.c_int
        assert len(declared[name][1]) == n


@pytest.mark.parametrize("null", range(7))
def test_a_null_buffer_is_refused(null, build_native):
    lib = _cabi.load()
    counts = (4, 7, 2, 5, 1, 4)  # buffer arguments of each entry point taken from the list
    only = [i for i in ALL if null < counts[i]]
    assert _calls(lib, only, null=null, L=9) == [_cabi.EINVAL] * len(only)


def test_a_null_center_or_light_is_refused(build_native):
    lib = _cabi.load()
    center = C.cast(None, C.POINTER(C.c_double))
    assert _calls(lib, range(4), center=center) == [_cabi.EINVAL] * 4
    io = _io()
    io.params = None  # the light l = params[0..2]
    assert _calls(lib, (2, 3, 4, 5), io=io, L=9) == [_cabi.EINVAL] * 4


@pytest.mark.parametrize("M", [0, 7, 4097, -1])
def test_a_map_size_outside_8_to_4096_is_refused(M, build_native):
    assert _calls(_cabi.load(), range(4), M=M) == [_cabi.EINVAL] * 4


@pytest.mark.parametrize("radius", [0.0, -1.0, math.inf, math.nan])
def test_a_bad_radius_is_refused(radius, build_native):
    lib = _cabi.load()
    assert _calls(lib, range(4), radius=radius) == [_cabi.EINVAL] * 4
    assert b"radius" in lib.deodr_b200_last_error()


@pytest.mark.parametrize("c", [(math.nan, 0, 0), (0, math.inf, 0), (0, 0, -math.inf)])
def test_a_non_finite_center_is_refused(c, build_native):
    assert _calls(_cabi.load(), range(4), center=_center(c)) == [_cabi.EINVAL] * 4


@pytest.mark.parametrize("bias,soft", [(0.0, 0.1), (-1e-3, 0.1), (0.01, 0.0), (0.01, -1.0), (math.inf, 0.1),
                                       (0.01, math.nan), (math.nan, 0.1), (0.01, math.inf)])
def test_a_bad_bias_or_softness_is_refused(bias, soft, build_native):
    lib = _cabi.load()
    assert _calls(lib, (2, 3), bias=bias, soft=soft) == [_cabi.EINVAL] * 2
    assert b"bias, softness" in lib.deodr_b200_last_error()


def test_bad_gbuffer_offsets_are_refused(build_native):
    lib = _cabi.load()
    io = _io()
    io.off_coverage = io.off_position + 1  # inside the position slice
    assert _calls(lib, (2, 3, 4, 5), io=io, L=9) == [_cabi.EINVAL] * 4
    io = _io(split=True)
    io.off_position = 5  # the split G-buffer has 7 channels
    assert _calls(lib, (2, 3), io=io) == [_cabi.EINVAL] * 2


@pytest.mark.parametrize("L", [0, -1, 9])
def test_a_light_count_outside_1_to_8_is_unsupported(L, build_native):
    assert _calls(_cabi.load(), (4, 5), L=L) == [_cabi.EUNSUPPORTED] * 2


def test_lights_are_needed_for_a_light_count_or_a_visibility(build_native):
    lib = _cabi.load()
    assert _calls(lib, (4, 5), lights=None, L=2) == [_cabi.EINVAL] * 2
    assert _calls(lib, (4, 5), lights=None, L=0, vis=P) == [_cabi.EINVAL] * 2


@pytest.mark.parametrize("nc,LS", [(3, 0), (3, 2), (3, 5), (5, 5), (2, 3)])
def test_a_bad_light_channel_count_is_unsupported(nc, LS, build_native):
    assert _calls(_cabi.load(), (4, 5), io=_io(nc), LS=LS) == [_cabi.EUNSUPPORTED] * 2


@pytest.mark.parametrize("nc,S", [(3, 2), (3, 5), (5, 5)])
def test_a_bad_environment_channel_count_is_unsupported(nc, S, build_native):
    assert _calls(_cabi.load(), (4, 5), io=_io(nc), sh=P, S=S, lights=None, L=0) == [_cabi.EUNSUPPORTED] * 2
