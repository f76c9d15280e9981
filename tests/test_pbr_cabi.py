"""The metallic-roughness C-ABI: the ctypes prototypes, and every refusal returned before any launch (no GPU needed)."""
import ctypes as C

import pytest

from deodr_b200 import _cabi

P = 0x1000  # a fake, never dereferenced, device pointer
NAMES = ("deodr_b200_pbr_shade", "deodr_b200_pbr_shade_b")
ARGS = (11, 18)


def _io(H=4, W=5, Cn=3, **null):
    io = _cabi.PhongIO()
    for name in ("channels", "params", "camera_center", "background", "image", "image_b", "channels_b", "params_b"):
        setattr(io, name, None if null.get(name) else P)
    io.H, io.W, io.C = H, W, Cn
    io.off_albedo, io.off_normal, io.off_position, io.off_coverage = -1, 0, 3, 6
    return io


def _fwd(lib, io, albedo=P, mr=P, sh=None, S=0, lights=None, L=0, Pc=0, vis=None, sun=None):
    return lib.deodr_b200_pbr_shade(C.byref(io), albedo, mr, sh, S, lights, L, Pc, vis, sun, None)


def _bwd(lib, io, albedo=P, mr=P, sh=None, S=0, lights=None, L=0, Pc=0, vis=None, sun=None, albedo_b=P, mr_b=P,
         sh_b=None, lights_b=None, vis_b=None, sun_b=None, scratch=P):
    return lib.deodr_b200_pbr_shade_b(C.byref(io), albedo, mr, sh, S, lights, L, Pc, vis, sun, albedo_b, mr_b, sh_b,
                                      lights_b, vis_b, sun_b, scratch, None)


def test_the_prototypes_are_declared(build_native):
    lib = _cabi.load()
    declared = {name: (res, args) for name, res, args in _cabi.SYMBOLS}
    for name, n in zip(NAMES, ARGS):
        assert name in declared
        assert getattr(lib, name).restype is C.c_int
        assert len(declared[name][1]) == n


@pytest.mark.parametrize("kw", [dict(albedo=None), dict(S=1), dict(L=1), dict(vis=P)])
def test_the_forward_refuses_a_missing_input(kw, build_native):
    lib = _cabi.load()
    assert _fwd(lib, _io(), **kw) == _cabi.EINVAL
    assert b"bad argument" in lib.deodr_b200_last_error()


@pytest.mark.parametrize("kw", [dict(albedo=None), dict(albedo_b=None), dict(mr_b=None), dict(mr=None),
                                dict(scratch=None), dict(sh=P, S=1), dict(lights=P, L=1, Pc=1),
                                dict(lights=P, L=1, Pc=1, lights_b=P, vis=P), dict(sun=P), dict(S=1),
                                dict(vis=P, vis_b=P)])
def test_the_adjoint_refuses_a_missing_input_or_gradient(kw, build_native):
    """mr_b must be given exactly when mr is."""
    lib = _cabi.load()
    assert _bwd(lib, _io(), **kw) == _cabi.EINVAL
    assert b"bad argument" in lib.deodr_b200_last_error()


@pytest.mark.parametrize("field", ["channels", "params", "camera_center", "background", "image"])
def test_a_null_io_buffer_is_refused(field, build_native):
    lib = _cabi.load()
    assert _fwd(lib, _io(**{field: True})) == _cabi.EINVAL
    assert lib.deodr_b200_pbr_shade(None, P, P, None, 0, None, 0, 0, None, None, None) == _cabi.EINVAL


@pytest.mark.parametrize("field", ["image_b", "channels_b", "params_b", "channels"])
def test_a_null_adjoint_io_buffer_is_refused(field, build_native):
    assert _bwd(_cabi.load(), _io(**{field: True})) == _cabi.EINVAL


@pytest.mark.parametrize("H,W,Cn", [(0, 5, 3), (4, 0, 3), (4, 5, 0), (4, 5, 40000)])
def test_bad_sizes_are_refused(H, W, Cn, build_native):
    lib = _cabi.load()
    assert _fwd(lib, _io(H, W, Cn)) == _cabi.EINVAL
    assert _bwd(lib, _io(H, W, Cn)) == _cabi.EINVAL


def test_a_g_buffer_with_the_albedo_inside_is_refused(build_native):
    """The form reads a separate albedo: off_albedo must be -1."""
    io = _io()
    io.off_albedo, io.off_normal, io.off_position, io.off_coverage = 0, 3, 6, 9
    lib = _cabi.load()
    assert _fwd(lib, io) == _cabi.EINVAL
    assert _bwd(lib, io) == _cabi.EINVAL


@pytest.mark.parametrize("kw", [dict(sh=P, S=2), dict(sh=P, S=5), dict(lights=P, L=9, Pc=1),
                                dict(lights=P, L=0, Pc=1), dict(lights=P, L=1, Pc=2)])
def test_bad_channel_or_light_counts_are_unsupported(kw, build_native):
    lib = _cabi.load()
    assert _fwd(lib, _io(), **kw) == _cabi.EUNSUPPORTED
    grads = dict(sh_b=P if "sh" in kw else None, lights_b=P if "lights" in kw else None)
    assert _bwd(lib, _io(), **kw, **grads) == _cabi.EUNSUPPORTED
