"""The steps either side of the raster, on the device (SURVEY.md 8f1 / 8f2): thin wrappers over
``deodr_b200_project_points*``, ``deodr_b200_vertex_luminosity*``, ``deodr_b200_edge_on_silhouette`` and
``deodr_b200_vertex_normals*`` (include/deodr_b200.h, kernels in csrc/scene_ops.cu), plus ``DeviceMeshView``: one view
of a mesh rendered and back-propagated without a host round trip - vertices in, image out, ``vertices_b`` back.

Reference code these replace:
  Camera.project_points / project_points_backward        deodr/differentiable_renderer.py:341-438
  Scene3D.compute_vertices_luminosity (+ backward)        deodr/differentiable_renderer.py:814-850
  TriMeshAdjacencies (adjacency, normals, silhouette)     deodr/triangulated_mesh.py:21-166
PyTorch is used for device memory and streams only.
"""

from __future__ import annotations

import copy
import ctypes as C
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _cabi


def _stream(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _f64(t: torch.Tensor, device) -> torch.Tensor:
    return t.to(device=device, dtype=torch.float64).contiguous()


class CameraParams:
    """Pinhole camera + OpenCV-style distortion, the fields of ``deodr.differentiable_renderer.Camera`` (:248-279)."""

    def __init__(self, extrinsic, intrinsic, distortion=None):
        self.extrinsic = np.ascontiguousarray(extrinsic, dtype=np.float64).reshape(3, 4)
        self.intrinsic = np.ascontiguousarray(intrinsic, dtype=np.float64).reshape(3, 3)
        self.distortion = None if distortion is None else np.ascontiguousarray(distortion, dtype=np.float64).reshape(5)

    @classmethod
    def from_reference(cls, camera) -> "CameraParams":
        """From any object with ``extrinsic`` / ``intrinsic`` / ``distortion`` (e.g. the reference's ``Camera``)."""
        return cls(camera.extrinsic, camera.intrinsic, camera.distortion)

    def c_struct(self) -> _cabi.Camera:
        c = _cabi.Camera()
        c.extrinsic[:] = self.extrinsic.reshape(-1).tolist()
        c.intrinsic[:] = self.intrinsic.reshape(-1).tolist()
        if self.distortion is not None:
            c.distortion[:] = self.distortion.tolist()
            c.has_distortion = 1
        return c

    @property
    def has_distortion(self) -> bool:
        return self.distortion is not None

    def vector(self) -> np.ndarray:
        """The camera vector [26] fp64 of the device-camera entry points: extrinsic (12), intrinsic (9), distortion (5,
        zeros without distortion)."""
        dist = self.distortion if self.distortion is not None else np.zeros(5)
        return np.concatenate((self.extrinsic.reshape(-1), self.intrinsic.reshape(-1), dist))

    def device_vector(self, device) -> torch.Tensor:
        """:meth:`vector` on ``device``, uploaded again only when the camera's values have changed."""
        vec = self.vector()
        key = (torch.device(device), vec.tobytes())
        if getattr(self, "_device_key", None) != key:
            self._device_vector = torch.from_numpy(vec).to(device, non_blocking=True)
            self._device_key = key
        return self._device_vector


CAMERA_VECTOR_SIZE = 26  # extrinsic [3,4] (12), intrinsic [3,3] (9), distortion k1 k2 p1 p2 k3 (5)


def split_camera_vector(vec: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(extrinsic [3,4], intrinsic [3,3], distortion [5]) views of a camera vector [26]."""
    return vec[:12].reshape(3, 4), vec[12:21].reshape(3, 3), vec[21:26]


def camera_center_of(vec: torch.Tensor) -> torch.Tensor:
    """The camera centre -R^T t [3] of a camera vector [26], computed on its device (differentiable)."""
    extrinsic = vec[:12].reshape(3, 4)
    return -(extrinsic[:, :3].T @ extrinsic[:, 3])


def _check_camera_vector(vec: torch.Tensor, device) -> torch.Tensor:
    if not isinstance(vec, torch.Tensor) or vec.dtype != torch.float64 or tuple(vec.shape) != (CAMERA_VECTOR_SIZE,) \
            or vec.device != torch.device(device) or not vec.is_contiguous():
        raise ValueError(f"the camera vector must be a contiguous [26] fp64 tensor on {device}; got "
                         f"{getattr(vec, 'dtype', type(vec))} {tuple(getattr(vec, 'shape', ()))}")
    return vec


def project_points(points: torch.Tensor, camera: CameraParams) -> Tuple[torch.Tensor, torch.Tensor]:
    """``Camera.project_points``: points [N,3] (CUDA fp64) -> (ij [N,2] fp64 with column 0 = x, depths [N] fp64)."""
    points = _f64(points, points.device)
    n = points.shape[0]
    ij = torch.empty((n, 2), dtype=torch.float64, device=points.device)
    depths = torch.empty((n,), dtype=torch.float64, device=points.device)
    cam = camera.c_struct()
    _cabi.check(_cabi.load().deodr_b200_project_points(points.data_ptr(), n, C.byref(cam), ij.data_ptr(),
                                                       depths.data_ptr(), _stream(points.device)))
    return ij, depths


def project_points_backward(points: torch.Tensor, camera: CameraParams, ij_b: torch.Tensor,
                            depths_b: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                            reference_transpose: bool = False) -> torch.Tensor:
    """``Camera.project_points_backward``: accumulates into ``out`` ([N,3] fp64, created zeroed if None).

    ``reference_transpose=True`` reproduces the reference's ``ij_b.dot(intrinsic[:2,:2].T)`` (:399, :412) and final
    ``p_camera_b.dot(extrinsic[:3,:3].T)`` (:438), which are the adjoint only for zero skew with ``K[1,0] == 0`` and a
    symmetric rotation (INTEGRATION.md, defect #3); the default is the true adjoint."""
    points = _f64(points, points.device)
    n = points.shape[0]
    ij_b = ij_b.to(device=points.device, dtype=torch.float32).contiguous()
    if depths_b is not None:
        depths_b = _f64(depths_b, points.device)
    if out is None:
        out = torch.zeros((n, 3), dtype=torch.float64, device=points.device)
    cam = camera.c_struct()
    _cabi.check(_cabi.load().deodr_b200_project_points_b(
        points.data_ptr(), n, C.byref(cam), ij_b.data_ptr(), depths_b.data_ptr() if depths_b is not None else None,
        out.data_ptr(), int(bool(reference_transpose)), _stream(points.device)))
    return out


def project_points_backward_f64(points: torch.Tensor, camera: CameraParams, ij_b: Optional[torch.Tensor],
                                depths_b: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The true adjoint of :func:`project_points` from an fp64 ``ij_b`` [N,2] (not rounded to fp32) and ``depths_b``
    [N], either of them None for zero -> points_b [N,3] fp64, a new tensor (deodr_b200_project_points_b64)."""
    points = _f64(points, points.device)
    n = points.shape[0]
    ij_b = _f64(ij_b, points.device) if ij_b is not None else None
    depths_b = _f64(depths_b, points.device) if depths_b is not None else None
    out = torch.empty((n, 3), dtype=torch.float64, device=points.device)
    cam = camera.c_struct()
    _cabi.check(_cabi.load().deodr_b200_project_points_b64(
        points.data_ptr(), n, C.byref(cam), ij_b.data_ptr() if ij_b is not None else None,
        depths_b.data_ptr() if depths_b is not None else None, out.data_ptr(), _stream(points.device)))
    return out


def project_points_dev(points: torch.Tensor, camera: torch.Tensor,
                       has_distortion: bool) -> Tuple[torch.Tensor, torch.Tensor]:
    """:func:`project_points` with the camera vector ``camera`` [26] fp64 read from device memory (so it may change on
    the device between calls): for the same values, bit-identical ij and depths (deodr_b200_project_points_dev)."""
    points = _f64(points, points.device)
    camera = _check_camera_vector(camera, points.device)
    n = points.shape[0]
    ij = torch.empty((n, 2), dtype=torch.float64, device=points.device)
    depths = torch.empty((n,), dtype=torch.float64, device=points.device)
    _cabi.check(_cabi.load().deodr_b200_project_points_dev(points.data_ptr(), n, camera.data_ptr(),
                                                           int(bool(has_distortion)), ij.data_ptr(), depths.data_ptr(),
                                                           _stream(points.device)))
    return ij, depths


def project_points_camera_backward(points: torch.Tensor, camera: torch.Tensor, has_distortion: bool,
                                   ij_b: Optional[torch.Tensor], depths_b: Optional[torch.Tensor],
                                   scratch: torch.Tensor, points_b: Optional[torch.Tensor] = None,
                                   accumulate: bool = True) -> torch.Tensor:
    """The true adjoint of :func:`project_points_dev` in the camera and the points, in one pass
    (deodr_b200_project_points_camera_b) -> camera_b [26] fp64, summed in a fixed order.  ``ij_b`` [N,2] is fp32 (the
    rasteriser's) or fp64; ``ij_b`` and ``depths_b`` may be None (zero).  ``points_b`` [N,3] fp64, when given, receives
    the points' adjoint: accumulated, or overwritten with ``accumulate=False``.  ``scratch``: a buffer of
    ``mesh_fitter.new_scratch``."""
    points = _f64(points, points.device)
    dev = points.device
    camera = _check_camera_vector(camera, dev)
    n = points.shape[0]
    ij32 = ij64 = None
    if ij_b is not None:
        if ij_b.dtype == torch.float32:
            ij32 = ij_b.to(dev).contiguous()
        else:
            ij64 = _f64(ij_b, dev)
    if depths_b is not None:
        depths_b = _f64(depths_b, dev)
    if points_b is not None and (points_b.dtype != torch.float64 or not points_b.is_contiguous()
                                 or tuple(points_b.shape) != (n, 3)):
        raise ValueError(f"points_b must be a contiguous [{n},3] fp64 tensor")
    camera_b = torch.empty((CAMERA_VECTOR_SIZE,), dtype=torch.float64, device=dev)
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    _cabi.check(_cabi.load().deodr_b200_project_points_camera_b(
        points.data_ptr(), n, camera.data_ptr(), int(bool(has_distortion)), ptr(ij32), ptr(ij64), ptr(depths_b),
        ptr(points_b), int(bool(accumulate)), camera_b.data_ptr(), scratch.data_ptr(), _stream(dev)))
    return camera_b


def camera_gradients(camera: torch.Tensor, camera_b: torch.Tensor, has_distortion: bool,
                     center_b: Optional[torch.Tensor] = None) -> Dict[str, Optional[torch.Tensor]]:
    """Splits camera_b [26] into dict(extrinsic_b [3,4], intrinsic_b [3,3], distortion_b [5] or None), adding the
    share of a camera-centre gradient ``center_b`` [3] through c = -R^T t (R_b -= t c_b^T, t_b -= R c_b), on the
    device."""
    extrinsic_b, intrinsic_b, distortion_b = (x.clone() for x in split_camera_vector(camera_b))
    if center_b is not None:
        extrinsic = camera[:12].reshape(3, 4)
        extrinsic_b[:, :3] -= torch.outer(extrinsic[:, 3], center_b)
        extrinsic_b[:, 3] -= extrinsic[:, :3] @ center_b
    return {"extrinsic_b": extrinsic_b, "intrinsic_b": intrinsic_b,
            "distortion_b": distortion_b if has_distortion else None}


def lit_vertex_colors(normals: torch.Tensor, vertex_colors: torch.Tensor, light: torch.Tensor,
                      directional: bool = True) -> torch.Tensor:
    """colours [V,C] fp64 = vertex_colors * (max(0, -<normals, light[:3]>) + light[3]) with ``light`` [4] fp64 on the
    device (deodr_b200_lit_vertex_colors); without ``directional`` only the ambient light[3]."""
    dev = normals.device
    normals, vertex_colors, light = _f64(normals, dev), _f64(vertex_colors, dev), _f64(light, dev)
    n, nc = vertex_colors.shape
    colors = torch.empty((n, nc), dtype=torch.float64, device=dev)
    _cabi.check(_cabi.load().deodr_b200_lit_vertex_colors(normals.data_ptr(), vertex_colors.data_ptr(), n, nc,
                                                          light.data_ptr(), int(bool(directional)), colors.data_ptr(),
                                                          _stream(dev)))
    return colors


def lit_vertex_colors_backward(normals: torch.Tensor, vertex_colors: torch.Tensor, light: torch.Tensor,
                               colors_b: torch.Tensor, scratch: torch.Tensor,
                               directional: bool = True) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """-> (normals_b [V,3], vertex_colors_b [V,C], light_b [4]) fp64, the adjoint of :func:`lit_vertex_colors` from
    ``colors_b`` [V,C] fp32 or fp64; ``light_b`` summed in a fixed order (bit-reproducible).  ``scratch``: a buffer
    of ``mesh_fitter.new_scratch``."""
    dev = normals.device
    normals, vertex_colors, light = _f64(normals, dev), _f64(vertex_colors, dev), _f64(light, dev)
    if colors_b.dtype not in (torch.float32, torch.float64):
        colors_b = colors_b.to(torch.float64)
    colors_b = colors_b.to(dev).contiguous()
    n, nc = vertex_colors.shape
    normals_b = torch.empty((n, 3), dtype=torch.float64, device=dev)
    vcol_b = torch.empty((n, nc), dtype=torch.float64, device=dev)
    light_b = torch.empty((4,), dtype=torch.float64, device=dev)
    _cabi.check(_cabi.load().deodr_b200_lit_vertex_colors_b(
        normals.data_ptr(), vertex_colors.data_ptr(), n, nc, light.data_ptr(), int(bool(directional)),
        colors_b.data_ptr(), int(colors_b.dtype == torch.float64), normals_b.data_ptr(), vcol_b.data_ptr(),
        light_b.data_ptr(), scratch.data_ptr(), _stream(dev)))
    return normals_b, vcol_b, light_b


def _check_sh(sh: torch.Tensor, device) -> Tuple[torch.Tensor, int]:
    """-> (sh, S) for an environment [9] (S = 1) or [9, S] fp64, contiguous, on ``device``."""
    dev = torch.device(device)
    if not isinstance(sh, torch.Tensor) or sh.dtype != torch.float64 or sh.device.type != dev.type \
            or (dev.index is not None and sh.device.index != dev.index) or not sh.is_contiguous() \
            or sh.dim() not in (1, 2) or sh.shape[0] != 9:
        raise ValueError(f"sh must be a contiguous [9] or [9,S] fp64 tensor on {device}; got "
                         f"{getattr(sh, 'dtype', type(sh))} {tuple(getattr(sh, 'shape', ()))} "
                         f"on {getattr(sh, 'device', None)}")
    return sh, (1 if sh.dim() == 1 else sh.shape[1])


def sh_lit_vertex_colors(normals: torch.Tensor, vertex_colors: Optional[torch.Tensor], light: torch.Tensor,
                         sh: torch.Tensor, directional: bool = True) -> torch.Tensor:
    """:func:`lit_vertex_colors` with a spherical-harmonics environment ``sh`` [9] or [9,S] fp64 on the device (the
    model in include/deodr_b200.h; deodr_b200_sh_lit_vertex_colors): colours [V,C] fp64 = vertex_colors * ((relu(-<n,
    l>) + ambient) + sh_c(n)), or, with ``vertex_colors`` None, the luminosity [V] of a grey environment."""
    dev = normals.device
    normals, light = _f64(normals, dev), _f64(light, dev)
    sh, S = _check_sh(sh, dev)
    n = normals.shape[0]
    if vertex_colors is not None:
        vertex_colors = _f64(vertex_colors, dev)
        nc = vertex_colors.shape[1]
        colors = torch.empty((n, nc), dtype=torch.float64, device=dev)
    else:
        nc = 1
        colors = torch.empty((n,), dtype=torch.float64, device=dev)
    _cabi.check(_cabi.load().deodr_b200_sh_lit_vertex_colors(
        normals.data_ptr(), vertex_colors.data_ptr() if vertex_colors is not None else None, n, nc, light.data_ptr(),
        int(bool(directional)), sh.data_ptr(), S, colors.data_ptr(), _stream(dev)))
    return colors


def sh_lit_vertex_colors_backward(normals: torch.Tensor, vertex_colors: Optional[torch.Tensor], light: torch.Tensor,
                                  sh: torch.Tensor, colors_b: torch.Tensor, scratch: torch.Tensor,
                                  directional: bool = True) -> Tuple[Optional[torch.Tensor], ...]:
    """-> (normals_b [V,3], vertex_colors_b [V,C] or None, light_b [4], sh_b shaped like ``sh``) fp64, the adjoint of
    :func:`sh_lit_vertex_colors` from ``colors_b`` ([V,C], or [V] without vertex colours; fp32 or fp64); light_b and
    sh_b summed in a fixed order (bit-reproducible).  ``scratch``: a buffer of ``mesh_fitter.new_scratch``."""
    dev = normals.device
    normals, light = _f64(normals, dev), _f64(light, dev)
    sh, S = _check_sh(sh, dev)
    if colors_b.dtype not in (torch.float32, torch.float64):
        colors_b = colors_b.to(torch.float64)
    colors_b = colors_b.to(dev).contiguous()
    n = normals.shape[0]
    vcol_b = None
    nc = 1
    if vertex_colors is not None:
        vertex_colors = _f64(vertex_colors, dev)
        nc = vertex_colors.shape[1]
        vcol_b = torch.empty((n, nc), dtype=torch.float64, device=dev)
    normals_b = torch.empty((n, 3), dtype=torch.float64, device=dev)
    light_b = torch.empty((4,), dtype=torch.float64, device=dev)
    sh_b = torch.empty_like(sh)
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    _cabi.check(_cabi.load().deodr_b200_sh_lit_vertex_colors_b(
        normals.data_ptr(), ptr(vertex_colors), n, nc, light.data_ptr(), int(bool(directional)), sh.data_ptr(), S,
        colors_b.data_ptr(), int(colors_b.dtype == torch.float64), normals_b.data_ptr(), ptr(vcol_b),
        light_b.data_ptr(), sh_b.data_ptr(), scratch.data_ptr(), _stream(dev)))
    return normals_b, vcol_b, light_b, sh_b


MAX_POINT_LIGHTS = 8


def _check_point_lights(lights: torch.Tensor, device) -> Tuple[torch.Tensor, int, int]:
    """-> (lights, L, S) for a point-light table [L, 3 + S] fp64, contiguous, on ``device`` (rows: position, then the
    intensity, grey (S = 1) or one per channel).  L and S are checked against the channel count by the kernels."""
    dev = torch.device(device)
    if not isinstance(lights, torch.Tensor) or lights.dtype != torch.float64 or lights.device.type != dev.type \
            or (dev.index is not None and lights.device.index != dev.index) or not lights.is_contiguous() \
            or lights.dim() != 2 or lights.shape[1] < 4 or not 1 <= lights.shape[0] <= MAX_POINT_LIGHTS:
        raise ValueError(f"point lights must be a contiguous [L, 3 + S] fp64 tensor on {device} with L from 1 to "
                         f"{MAX_POINT_LIGHTS}; got {getattr(lights, 'dtype', type(lights))} "
                         f"{tuple(getattr(lights, 'shape', ()))} on {getattr(lights, 'device', None)}")
    return lights, lights.shape[0], lights.shape[1] - 3


def point_lit_vertex_colors(normals: torch.Tensor, positions: torch.Tensor, vertex_colors: Optional[torch.Tensor],
                            light: torch.Tensor, lights: torch.Tensor, sh: Optional[torch.Tensor] = None,
                            directional: bool = True) -> torch.Tensor:
    """:func:`sh_lit_vertex_colors` with point lights ``lights`` [L, 3 + S] fp64 on the device at the vertex
    ``positions`` [V,3] (the model in include/deodr_b200.h; deodr_b200_point_lit_vertex_colors): colours [V,C] fp64 =
    vertex_colors * (((relu(-<n, l>) + ambient) + sh_c(n)) + P_c(n, x)), the environment ``sh`` optional, or, with
    ``vertex_colors`` None, the luminosity [V] under grey lights."""
    dev = normals.device
    normals, positions, light = _f64(normals, dev), _f64(positions, dev), _f64(light, dev)
    lights, L, P = _check_point_lights(lights, dev)
    sh, S = _check_sh(sh, dev) if sh is not None else (None, 0)
    n = normals.shape[0]
    if vertex_colors is not None:
        vertex_colors = _f64(vertex_colors, dev)
        nc = vertex_colors.shape[1]
        colors = torch.empty((n, nc), dtype=torch.float64, device=dev)
    else:
        nc = 1
        colors = torch.empty((n,), dtype=torch.float64, device=dev)
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    _cabi.check(_cabi.load().deodr_b200_point_lit_vertex_colors(
        normals.data_ptr(), positions.data_ptr(), ptr(vertex_colors), n, nc, light.data_ptr(), int(bool(directional)),
        ptr(sh), S, lights.data_ptr(), L, P, colors.data_ptr(), _stream(dev)))
    return colors


def point_lit_vertex_colors_backward(normals: torch.Tensor, positions: torch.Tensor,
                                     vertex_colors: Optional[torch.Tensor], light: torch.Tensor, lights: torch.Tensor,
                                     colors_b: torch.Tensor, scratch: torch.Tensor, sh: Optional[torch.Tensor] = None,
                                     directional: bool = True) -> Tuple[Optional[torch.Tensor], ...]:
    """-> (normals_b [V,3], positions_b [V,3], vertex_colors_b [V,C] or None, light_b [4], sh_b shaped like ``sh`` or
    None, lights_b [L, 3 + S]) fp64, the adjoint of :func:`point_lit_vertex_colors` from ``colors_b`` ([V,C], or [V]
    without vertex colours; fp32 or fp64); light_b, sh_b and lights_b summed in a fixed order (bit-reproducible).
    ``scratch``: a buffer of ``mesh_fitter.new_scratch``."""
    dev = normals.device
    normals, positions, light = _f64(normals, dev), _f64(positions, dev), _f64(light, dev)
    lights, L, P = _check_point_lights(lights, dev)
    sh, S = _check_sh(sh, dev) if sh is not None else (None, 0)
    if colors_b.dtype not in (torch.float32, torch.float64):
        colors_b = colors_b.to(torch.float64)
    colors_b = colors_b.to(dev).contiguous()
    n = normals.shape[0]
    vcol_b = None
    nc = 1
    if vertex_colors is not None:
        vertex_colors = _f64(vertex_colors, dev)
        nc = vertex_colors.shape[1]
        vcol_b = torch.empty((n, nc), dtype=torch.float64, device=dev)
    normals_b = torch.empty((n, 3), dtype=torch.float64, device=dev)
    positions_b = torch.empty((n, 3), dtype=torch.float64, device=dev)
    light_b = torch.empty((4,), dtype=torch.float64, device=dev)
    sh_b = torch.empty_like(sh) if sh is not None else None
    lights_b = torch.empty_like(lights)
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    _cabi.check(_cabi.load().deodr_b200_point_lit_vertex_colors_b(
        normals.data_ptr(), positions.data_ptr(), ptr(vertex_colors), n, nc, light.data_ptr(), int(bool(directional)),
        ptr(sh), S, lights.data_ptr(), L, P, colors_b.data_ptr(), int(colors_b.dtype == torch.float64),
        normals_b.data_ptr(), positions_b.data_ptr(), ptr(vcol_b), light_b.data_ptr(), ptr(sh_b), lights_b.data_ptr(),
        scratch.data_ptr(), _stream(dev)))
    return normals_b, positions_b, vcol_b, light_b, sh_b, lights_b


PHONG_EXTRA_CHANNELS = 7  # the unit normal (3), the world position (3) and the coverage (1) after the C albedo channels


def camera_center(camera: CameraParams) -> np.ndarray:
    """The camera centre -R^T t [3] fp64 of a camera's extrinsic [R | t]."""
    return -camera.extrinsic[:, :3].T @ camera.extrinsic[:, 3]


def _phong_io(channels: torch.Tensor, params: torch.Tensor, center: torch.Tensor, background: torch.Tensor,
              albedo: Optional[torch.Tensor] = None) -> Tuple[_cabi.PhongIO, Tuple[torch.Tensor, ...]]:
    """-> (io, kept tensors: channels, params, center, background, albedo or None).  With ``albedo`` [H,W,C] the
    G-buffer ``channels`` is [H,W,7] (normal, position, coverage); without, [H,W,C+7] with the albedo first."""
    if albedo is None and (channels.dim() != 3 or channels.shape[2] <= PHONG_EXTRA_CHANNELS):
        raise ValueError(f"channels must be [H,W,C+7] with C >= 1; got {tuple(channels.shape)}")
    if albedo is not None and (channels.dim() != 3 or channels.shape[2] != PHONG_EXTRA_CHANNELS or albedo.dim() != 3
                               or tuple(albedo.shape[:2]) != tuple(channels.shape[:2]) or albedo.shape[2] < 1):
        raise ValueError(f"with an albedo [H,W,C], channels must be [H,W,7]; got albedo "
                         f"{tuple(albedo.shape)} and channels {tuple(channels.shape)}")
    dev = channels.device
    H, W, K = channels.shape
    nc = K - PHONG_EXTRA_CHANNELS if albedo is None else albedo.shape[2]
    channels = channels.to(dtype=torch.float32).contiguous()
    if albedo is not None:
        albedo = albedo.to(device=dev, dtype=torch.float32).contiguous()
    params, center = _f64(params, dev).reshape(-1), _f64(center, dev).reshape(-1)
    background = background.to(device=dev, dtype=torch.float32).contiguous().reshape(-1)
    if params.numel() != 6 or center.numel() != 3 or background.numel() != nc:
        raise ValueError(f"params must have 6 entries, camera_center 3 and background C = {nc}; got "
                         f"{params.numel()}, {center.numel()} and {background.numel()}")
    io = _cabi.PhongIO()
    io.channels, io.params, io.camera_center, io.background = (channels.data_ptr(), params.data_ptr(),
                                                              center.data_ptr(), background.data_ptr())
    io.H, io.W, io.C = H, W, nc
    if albedo is None:
        io.off_albedo, io.off_normal, io.off_position, io.off_coverage = 0, nc, nc + 3, nc + 6
    else:
        io.off_albedo, io.off_normal, io.off_position, io.off_coverage = -1, 0, 3, 6
    return io, (channels, params, center, background, albedo)


def _check_specular(spec: torch.Tensor, albedo: Optional[torch.Tensor], H: int, W: int, device) -> torch.Tensor:
    """The specular map's raster [H,W,2] as a contiguous f32 tensor on ``device``; it needs the separate albedo."""
    if albedo is None:
        raise ValueError("a specular map's raster is read beside a separate albedo (a textured Phong view's)")
    if not isinstance(spec, torch.Tensor) or tuple(spec.shape) != (H, W, 2):
        raise ValueError(f"specular must be an [{H},{W},2] tensor; got {tuple(getattr(spec, 'shape', ()))}")
    return spec.to(device=device, dtype=torch.float32).contiguous()


def phong_shade(channels: torch.Tensor, params: torch.Tensor, camera_center: torch.Tensor,
                background: torch.Tensor, sh: Optional[torch.Tensor] = None,
                albedo: Optional[torch.Tensor] = None, point_lights: Optional[torch.Tensor] = None,
                visibility: Optional[torch.Tensor] = None,
                sun_visibility: Optional[torch.Tensor] = None,
                specular: Optional[torch.Tensor] = None, brdf: str = "phong") -> torch.Tensor:
    """The per-pixel shading of a G-buffer (deodr_b200_phong_shade, or deodr_b200_sh_phong_shade with ``sh``; model in
    include/deodr_b200.h): ``channels``
    [H,W,C+7] f32 laid out (albedo C, normal 3, position 3, coverage 1), ``params`` [6] fp64 on the device = (light
    direction times intensity (3), ambient, specular strength ks, shininess e), ``camera_center`` [3] fp64 and
    ``background`` [C] -> image [H,W,C] f32.  ``sh``: an optional spherical-harmonics environment [9] or [9,C] fp64
    on the device.  ``albedo``: the albedo [H,W,C] f32 as a raster of its own (a textured mesh's), with ``channels``
    then [H,W,7] = (normal, position, coverage) (deodr_b200_phong_shade_albedo).  ``point_lights``: a point-light
    table [L, 3 + S] fp64 on the device, in either form (deodr_b200_point_phong_shade).  ``visibility``: with point
    lights, the lights' visibility [H,W,L] f32 (:func:`shadow_visibility`), which multiplies each light's diffuse and
    specular terms (deodr_b200_point_phong_shade_shadowed).  ``sun_visibility``: the directional light's visibility
    [H,W] f32 (:func:`sun_visibility`), which multiplies its diffuse and specular terms, with or without an
    environment, point lights and their ``visibility`` (deodr_b200_phong_shade_sun_shadowed).  ``specular``: with an
    albedo, the specular map's raster [H,W,2] = (K, E) (the model in include/deodr_b200.h), which gives every specular
    term aks = ks K and e(p) = e E / a, with any of the inputs above (deodr_b200_phong_shade_specular_map).
    ``brdf="ggx"`` is the metallic-roughness form instead (deodr_b200_pbr_shade; the model in include/deodr_b200.h):
    it needs an albedo, ``params`` [6] = (light, ambient, metallic mf, roughness rf), and ``specular`` is then the
    metallic-roughness map's raster [H,W,2] = (R, M) or None (the factors alone)."""
    io, keep = _phong_io(channels, params, camera_center, background, albedo)
    H, W = keep[0].shape[:2]
    image = torch.empty((H, W, io.C), dtype=torch.float32, device=keep[0].device)
    io.image = image.data_ptr()
    if brdf not in ("phong", "ggx"):
        raise ValueError(f"brdf must be 'phong' or 'ggx'; got {brdf!r}")
    if brdf == "ggx":
        if albedo is None:
            raise ValueError("the metallic-roughness form reads a separate albedo (a textured view's)")
        mr = _check_specular(specular, albedo, H, W, image.device) if specular is not None else None
        sun = _check_sun_visibility(sun_visibility, H, W, image.device) if sun_visibility is not None else None
        lights, L, P = _check_point_lights(point_lights, image.device) if point_lights is not None else (None, 0, 0)
        vis = _check_visibility(visibility, H, W, L, image.device) if visibility is not None else None
        if vis is not None and lights is None:
            raise ValueError("visibility multiplies the point lights' terms: it needs point_lights")
        sh, S = _check_sh(sh, image.device) if sh is not None else (None, 0)
        ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        _cabi.check(_cabi.load().deodr_b200_pbr_shade(
            C.byref(io), keep[4].data_ptr(), ptr(mr), ptr(sh), S, ptr(lights), L, P, ptr(vis), ptr(sun),
            _stream(image.device)))
    elif specular is not None:
        spec = _check_specular(specular, albedo, H, W, image.device)
        sun = _check_sun_visibility(sun_visibility, H, W, image.device) if sun_visibility is not None else None
        lights, L, P = _check_point_lights(point_lights, image.device) if point_lights is not None else (None, 0, 0)
        vis = _check_visibility(visibility, H, W, L, image.device) if visibility is not None else None
        if vis is not None and lights is None:
            raise ValueError("visibility multiplies the point lights' terms: it needs point_lights")
        sh, S = _check_sh(sh, image.device) if sh is not None else (None, 0)
        ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        _cabi.check(_cabi.load().deodr_b200_phong_shade_specular_map(
            C.byref(io), keep[4].data_ptr(), spec.data_ptr(), ptr(sh), S, ptr(lights), L, P, ptr(vis), ptr(sun),
            _stream(image.device)))
    elif sun_visibility is not None:
        sun = _check_sun_visibility(sun_visibility, H, W, image.device)
        lights, L, P = _check_point_lights(point_lights, image.device) if point_lights is not None else (None, 0, 0)
        vis = _check_visibility(visibility, H, W, L, image.device) if visibility is not None else None
        if vis is not None and lights is None:
            raise ValueError("visibility multiplies the point lights' terms: it needs point_lights")
        sh, S = _check_sh(sh, image.device) if sh is not None else (None, 0)
        ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        _cabi.check(_cabi.load().deodr_b200_phong_shade_sun_shadowed(
            C.byref(io), ptr(keep[4]), ptr(sh), S, ptr(lights), L, P, ptr(vis), sun.data_ptr(),
            _stream(image.device)))
    elif visibility is not None:
        if point_lights is None:
            raise ValueError("visibility multiplies the point lights' terms: it needs point_lights")
        lights, L, P = _check_point_lights(point_lights, image.device)
        vis = _check_visibility(visibility, H, W, L, image.device)
        sh, S = _check_sh(sh, image.device) if sh is not None else (None, 0)
        ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        _cabi.check(_cabi.load().deodr_b200_point_phong_shade_shadowed(
            C.byref(io), ptr(keep[4]), ptr(sh), S, lights.data_ptr(), L, P, vis.data_ptr(), _stream(image.device)))
    elif point_lights is not None:
        lights, L, P = _check_point_lights(point_lights, image.device)
        sh, S = _check_sh(sh, image.device) if sh is not None else (None, 0)
        ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        _cabi.check(_cabi.load().deodr_b200_point_phong_shade(C.byref(io), ptr(keep[4]), ptr(sh), S,
                                                               lights.data_ptr(), L, P, _stream(image.device)))
    elif albedo is not None:
        sh, S = _check_sh(sh, image.device) if sh is not None else (None, 0)
        _cabi.check(_cabi.load().deodr_b200_phong_shade_albedo(C.byref(io), keep[4].data_ptr(),
                                                               sh.data_ptr() if sh is not None else None, S,
                                                               _stream(image.device)))
    elif sh is None:
        _cabi.check(_cabi.load().deodr_b200_phong_shade(C.byref(io), _stream(image.device)))
    else:
        sh, S = _check_sh(sh, image.device)
        _cabi.check(_cabi.load().deodr_b200_sh_phong_shade(C.byref(io), sh.data_ptr(), S, _stream(image.device)))
    del keep
    return image


def phong_shade_backward(channels: torch.Tensor, params: torch.Tensor, camera_center: torch.Tensor,
                         background: torch.Tensor, image_b: torch.Tensor, scratch: torch.Tensor,
                         center_grad: bool = False, sh: Optional[torch.Tensor] = None,
                         albedo: Optional[torch.Tensor] = None,
                         point_lights: Optional[torch.Tensor] = None,
                         visibility: Optional[torch.Tensor] = None,
                         sun_visibility: Optional[torch.Tensor] = None,
                         specular: Optional[torch.Tensor] = None, brdf: str = "phong") -> Tuple[torch.Tensor, ...]:
    """-> (channels_b [H,W,C+7] f32, params_b [6] fp64), the adjoint of :func:`phong_shade` from ``image_b`` [H,W,C]
    (deodr_b200_phong_shade_b, or deodr_b200_sh_phong_shade_b with ``sh``).  channels_b includes the coverage channel's gradient; ``params_b`` is summed over the
    pixels in a fixed order (bit-reproducible).  ``scratch``: a buffer of ``mesh_fitter.new_scratch``.  With
    ``center_grad`` the result also holds camera_center_b [3] fp64, summed with params_b; with an environment ``sh``
    it then holds sh_b, shaped like ``sh``, also summed in a fixed order.  With a separate ``albedo`` (see
    :func:`phong_shade`; channels_b is then [H,W,7]) the result ends with albedo_b [H,W,C] f32
    (deodr_b200_phong_shade_albedo_b).  With ``point_lights`` the result ends with lights_b [L, 3 + S] fp64, summed
    in a fixed order (deodr_b200_point_phong_shade_b); with ``visibility`` too it then ends with vis_b [H,W,L] f32
    (deodr_b200_point_phong_shade_shadowed_b).  With ``sun_visibility`` the result ends with sun_vis_b [H,W] f32
    (deodr_b200_phong_shade_sun_shadowed_b).  With ``specular`` (the map raster of :func:`phong_shade`) it ends with
    spec_b [H,W,2] f32 (deodr_b200_phong_shade_specular_map_b).  With ``brdf="ggx"`` it is the adjoint of the
    metallic-roughness form (deodr_b200_pbr_shade_b): params_b[4:6] are the metallic and roughness factors' gradients,
    and with a map raster ``specular`` the result ends with its gradient mr_b [H,W,2] f32."""
    io, keep = _phong_io(channels, params, camera_center, background, albedo)
    dev = keep[0].device
    S = _check_sh(sh, dev)[1] if sh is not None else 0
    sh_b = torch.empty_like(sh) if sh is not None else None
    H, W, K = keep[0].shape
    image_b = image_b.to(device=dev, dtype=torch.float32).contiguous()
    if tuple(image_b.shape) != (H, W, io.C):
        raise ValueError(f"image_b must be {(H, W, io.C)}; got {tuple(image_b.shape)}")
    channels_b = torch.empty((H, W, K), dtype=torch.float32, device=dev)
    params_b = torch.empty((6,), dtype=torch.float64, device=dev)
    io.image_b, io.channels_b, io.params_b = image_b.data_ptr(), channels_b.data_ptr(), params_b.data_ptr()
    center_b = torch.empty((3,), dtype=torch.float64, device=dev) if center_grad else None
    if center_b is not None:
        io.camera_center_b = center_b.data_ptr()
    albedo_b = None
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    if albedo is not None:
        albedo_b = torch.empty((H, W, io.C), dtype=torch.float32, device=dev)
    lights_b = vis_b = sun_b = spec_b = None
    if brdf not in ("phong", "ggx"):
        raise ValueError(f"brdf must be 'phong' or 'ggx'; got {brdf!r}")
    if brdf == "ggx":
        if albedo is None:
            raise ValueError("the metallic-roughness form reads a separate albedo (a textured view's)")
        mr = _check_specular(specular, albedo, H, W, dev) if specular is not None else None
        sun = _check_sun_visibility(sun_visibility, H, W, dev) if sun_visibility is not None else None
        lights, L, P = _check_point_lights(point_lights, dev) if point_lights is not None else (None, 0, 0)
        vis = _check_visibility(visibility, H, W, L, dev) if visibility is not None else None
        if vis is not None and lights is None:
            raise ValueError("visibility multiplies the point lights' terms: it needs point_lights")
        lights_b = torch.empty_like(lights) if lights is not None else None
        vis_b = torch.empty((H, W, L), dtype=torch.float32, device=dev) if vis is not None else None
        sun_b = torch.empty((H, W), dtype=torch.float32, device=dev) if sun is not None else None
        spec_b = torch.empty((H, W, 2), dtype=torch.float32, device=dev) if mr is not None else None
        _cabi.check(_cabi.load().deodr_b200_pbr_shade_b(
            C.byref(io), keep[4].data_ptr(), ptr(mr), ptr(sh), S, ptr(lights), L, P, ptr(vis), ptr(sun),
            albedo_b.data_ptr(), ptr(spec_b), ptr(sh_b), ptr(lights_b), ptr(vis_b), ptr(sun_b),
            scratch.data_ptr(), _stream(dev)))
    elif specular is not None:
        spec = _check_specular(specular, albedo, H, W, dev)
        sun = _check_sun_visibility(sun_visibility, H, W, dev) if sun_visibility is not None else None
        lights, L, P = _check_point_lights(point_lights, dev) if point_lights is not None else (None, 0, 0)
        vis = _check_visibility(visibility, H, W, L, dev) if visibility is not None else None
        if vis is not None and lights is None:
            raise ValueError("visibility multiplies the point lights' terms: it needs point_lights")
        lights_b = torch.empty_like(lights) if lights is not None else None
        vis_b = torch.empty((H, W, L), dtype=torch.float32, device=dev) if vis is not None else None
        sun_b = torch.empty((H, W), dtype=torch.float32, device=dev) if sun is not None else None
        spec_b = torch.empty((H, W, 2), dtype=torch.float32, device=dev)
        _cabi.check(_cabi.load().deodr_b200_phong_shade_specular_map_b(
            C.byref(io), keep[4].data_ptr(), spec.data_ptr(), ptr(sh), S, ptr(lights), L, P, ptr(vis), ptr(sun),
            albedo_b.data_ptr(), spec_b.data_ptr(), ptr(sh_b), ptr(lights_b), ptr(vis_b), ptr(sun_b),
            scratch.data_ptr(), _stream(dev)))
    elif sun_visibility is not None:
        sun = _check_sun_visibility(sun_visibility, H, W, dev)
        lights, L, P = _check_point_lights(point_lights, dev) if point_lights is not None else (None, 0, 0)
        vis = _check_visibility(visibility, H, W, L, dev) if visibility is not None else None
        if vis is not None and lights is None:
            raise ValueError("visibility multiplies the point lights' terms: it needs point_lights")
        lights_b = torch.empty_like(lights) if lights is not None else None
        vis_b = torch.empty((H, W, L), dtype=torch.float32, device=dev) if vis is not None else None
        sun_b = torch.empty((H, W), dtype=torch.float32, device=dev)
        _cabi.check(_cabi.load().deodr_b200_phong_shade_sun_shadowed_b(
            C.byref(io), ptr(keep[4]), ptr(albedo_b), ptr(sh), S, ptr(sh_b), ptr(lights), L, P, ptr(lights_b),
            ptr(vis), ptr(vis_b), sun.data_ptr(), sun_b.data_ptr(), scratch.data_ptr(), _stream(dev)))
    elif visibility is not None:
        if point_lights is None:
            raise ValueError("visibility multiplies the point lights' terms: it needs point_lights")
        lights, L, P = _check_point_lights(point_lights, dev)
        vis = _check_visibility(visibility, H, W, L, dev)
        lights_b = torch.empty_like(lights)
        vis_b = torch.empty((H, W, L), dtype=torch.float32, device=dev)
        _cabi.check(_cabi.load().deodr_b200_point_phong_shade_shadowed_b(
            C.byref(io), ptr(keep[4]), ptr(albedo_b), ptr(sh), S, ptr(sh_b), lights.data_ptr(), L, P,
            lights_b.data_ptr(), vis.data_ptr(), vis_b.data_ptr(), scratch.data_ptr(), _stream(dev)))
    elif point_lights is not None:
        lights, L, P = _check_point_lights(point_lights, dev)
        lights_b = torch.empty_like(lights)
        _cabi.check(_cabi.load().deodr_b200_point_phong_shade_b(
            C.byref(io), ptr(keep[4]), ptr(albedo_b), ptr(sh), S, ptr(sh_b), lights.data_ptr(), L, P,
            lights_b.data_ptr(), scratch.data_ptr(), _stream(dev)))
    elif albedo is not None:
        _cabi.check(_cabi.load().deodr_b200_phong_shade_albedo_b(
            C.byref(io), keep[4].data_ptr(), albedo_b.data_ptr(), ptr(sh), S, ptr(sh_b), scratch.data_ptr(),
            _stream(dev)))
    elif sh is None:
        _cabi.check(_cabi.load().deodr_b200_phong_shade_b(C.byref(io), scratch.data_ptr(), _stream(dev)))
    else:
        _cabi.check(_cabi.load().deodr_b200_sh_phong_shade_b(C.byref(io), sh.data_ptr(), S, sh_b.data_ptr(),
                                                             scratch.data_ptr(), _stream(dev)))
    del keep
    out = (channels_b, params_b) if center_b is None else (channels_b, params_b, center_b)
    out = out if sh_b is None else out + (sh_b,)
    out = out if albedo_b is None else out + (albedo_b,)
    out = out if lights_b is None else out + (lights_b,)
    out = out if vis_b is None else out + (vis_b,)
    out = out if sun_b is None else out + (sun_b,)
    return out if spec_b is None else out + (spec_b,)


# ---- shadows from point lights (the model in include/deodr_b200.h) ---------------------------------------------------

SHADOW_FAR = 1e30  # DEODR_B200_SHADOW_FAR: the background depth of the cube shadow maps


def _check_visibility(vis: torch.Tensor, H: int, W: int, L: int, device) -> torch.Tensor:
    if not isinstance(vis, torch.Tensor) or vis.dtype != torch.float32 or tuple(vis.shape) != (H, W, L) \
            or not vis.is_contiguous() or vis.device != torch.device(device):
        raise ValueError(f"visibility must be a contiguous [{H},{W},{L}] f32 tensor on {device}; got "
                         f"{getattr(vis, 'dtype', type(vis))} {tuple(getattr(vis, 'shape', ()))}")
    return vis


def _check_maps(maps: torch.Tensor, L: int, device) -> Tuple[torch.Tensor, int]:
    """-> (maps, M) for cube maps [6L, M, M] f32, contiguous, on ``device``."""
    if not isinstance(maps, torch.Tensor) or maps.dtype != torch.float32 or maps.dim() != 3 \
            or maps.shape[0] != 6 * L or maps.shape[1] != maps.shape[2] or not maps.is_contiguous() \
            or maps.device != torch.device(device):
        raise ValueError(f"maps must be a contiguous [6L, M, M] f32 tensor on {device} with L = {L}; got "
                         f"{getattr(maps, 'dtype', type(maps))} {tuple(getattr(maps, 'shape', ()))}")
    return maps, maps.shape[1]


def _shadow_io(channels: torch.Tensor, albedo: Optional[torch.Tensor]) -> Tuple[_cabi.PhongIO, torch.Tensor]:
    """The G-buffer part of a ``DeodrPhongIO`` the visibility reads: [H,W,C+7] (albedo first), or [H,W,7] with a
    separate ``albedo`` [H,W,C] (only its channel count is used)."""
    channels = channels.to(dtype=torch.float32).contiguous()
    if channels.dim() != 3 or channels.shape[2] < PHONG_EXTRA_CHANNELS + (0 if albedo is not None else 1) \
            or (albedo is not None and channels.shape[2] != PHONG_EXTRA_CHANNELS):
        raise ValueError(f"channels must be [H,W,C+7], or [H,W,7] with an albedo; got {tuple(channels.shape)}")
    H, W, K = channels.shape
    nc = K - PHONG_EXTRA_CHANNELS if albedo is None else albedo.shape[-1]
    io = _cabi.PhongIO()
    io.channels, io.H, io.W, io.C = channels.data_ptr(), H, W, nc
    if albedo is None:
        io.off_albedo, io.off_normal, io.off_position, io.off_coverage = 0, nc, nc + 3, nc + 6
    else:
        io.off_albedo, io.off_normal, io.off_position, io.off_coverage = -1, 0, 3, 6
    return io, channels


def cube_project(vertices: torch.Tensor, lights: torch.Tensor,
                 map_size: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """The cube cameras of the point lights ``lights`` [L, 3 + S] and the vertices [V,3] projected through them
    (deodr_b200_cube_project) -> (cameras [6L, 26], ij [6L, V, 2], depths [6L, V]) fp64; face 6 j + k is light j's
    +x, -x, +y, -y, +z or -z face.  Each face's ij and depths are bit-identical to :func:`project_points_dev` with its
    camera vector."""
    dev = vertices.device
    vertices = _f64(vertices, dev)
    lights, L, S = _check_point_lights(lights, dev)
    n = vertices.shape[0]
    cameras = torch.empty((6 * L, CAMERA_VECTOR_SIZE), dtype=torch.float64, device=dev)
    ij = torch.empty((6 * L, n, 2), dtype=torch.float64, device=dev)
    depths = torch.empty((6 * L, n), dtype=torch.float64, device=dev)
    _cabi.check(_cabi.load().deodr_b200_cube_project(vertices.data_ptr(), n, lights.data_ptr(), L, S, int(map_size),
                                                     cameras.data_ptr(), ij.data_ptr(), depths.data_ptr(),
                                                     _stream(dev)))
    return cameras, ij, depths


def cube_project_backward(vertices: torch.Tensor, lights: torch.Tensor, map_size: int, cameras: torch.Tensor,
                          ij_b: torch.Tensor, depths_b: torch.Tensor, scratch: torch.Tensor,
                          vertices_b: Optional[torch.Tensor] = None,
                          lights_b: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """The adjoint of :func:`cube_project` from ``ij_b`` [6L, V, 2] and ``depths_b`` [6L, V] (fp32, the rasteriser's)
    -> (vertices_b [V,3], lights_b [L, 3 + S]) fp64, accumulated into the given tensors (created zeroed if None):
    every vertex adds its 6L faces in a fixed order, and the lights' positions their faces' share, summed in a fixed
    order (deodr_b200_cube_project_b).  ``scratch``: a buffer of ``mesh_fitter.new_scratch``."""
    dev = vertices.device
    vertices = _f64(vertices, dev)
    lights, L, S = _check_point_lights(lights, dev)
    n = vertices.shape[0]
    ij_b = ij_b.to(device=dev, dtype=torch.float32).contiguous()
    depths_b = depths_b.to(device=dev, dtype=torch.float32).contiguous()
    if tuple(ij_b.shape) != (6 * L, n, 2) or depths_b.numel() != 6 * L * n:
        raise ValueError(f"ij_b must be [{6 * L},{n},2] and depths_b [{6 * L},{n}]; got {tuple(ij_b.shape)} and "
                         f"{tuple(depths_b.shape)}")
    if vertices_b is None:
        vertices_b = torch.zeros((n, 3), dtype=torch.float64, device=dev)
    if lights_b is None:
        lights_b = torch.zeros_like(lights)
    _cabi.check(_cabi.load().deodr_b200_cube_project_b(
        vertices.data_ptr(), n, lights.data_ptr(), L, S, int(map_size), cameras.data_ptr(), ij_b.data_ptr(),
        depths_b.data_ptr(), vertices_b.data_ptr(), lights_b.data_ptr(), scratch.data_ptr(), _stream(dev)))
    return vertices_b, lights_b


def shadow_visibility(channels: torch.Tensor, lights: torch.Tensor, maps: torch.Tensor, bias: float,
                      softness: float, albedo: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The visibility [H,W,L] f32 of a Phong G-buffer's pixels (``channels`` [H,W,C+7], or [H,W,7] beside a separate
    ``albedo``) under the point lights' cube shadow maps ``maps`` [6L, M, M] f32 (deodr_b200_shadow_visibility; the
    model in include/deodr_b200.h): a 2x2 bilinear filter of smoothstep depth tests, ``bias`` and ``softness`` in
    world units.  1 where the coverage is 0."""
    dev = channels.device
    io, channels = _shadow_io(channels, albedo)
    lights, L, S = _check_point_lights(lights, dev)
    maps, M = _check_maps(maps, L, dev)
    vis = torch.empty((io.H, io.W, L), dtype=torch.float32, device=dev)
    _cabi.check(_cabi.load().deodr_b200_shadow_visibility(C.byref(io), lights.data_ptr(), L, S, maps.data_ptr(), M,
                                                          float(bias), float(softness), vis.data_ptr(),
                                                          _stream(dev)))
    return vis


def shadow_visibility_backward(channels: torch.Tensor, lights: torch.Tensor, maps: torch.Tensor, bias: float,
                               softness: float, vis_b: torch.Tensor, scratch: torch.Tensor,
                               albedo: Optional[torch.Tensor] = None, channels_b: Optional[torch.Tensor] = None,
                               maps_b: Optional[torch.Tensor] = None,
                               lights_b: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, ...]:
    """The adjoint of :func:`shadow_visibility` from ``vis_b`` [H,W,L] -> (channels_b, maps_b [6L, M, M] f32,
    lights_b [L, 3 + S] fp64), each accumulated into the given tensor (created zeroed if None): the position and
    coverage slices of channels_b, the texels (fp32 atomics) and the lights' positions, summed in a fixed order
    (deodr_b200_shadow_visibility_b).  ``scratch``: a buffer of ``mesh_fitter.new_scratch``."""
    dev = channels.device
    io, channels = _shadow_io(channels, albedo)
    lights, L, S = _check_point_lights(lights, dev)
    maps, M = _check_maps(maps, L, dev)
    vis_b = _check_visibility(vis_b.to(dev, torch.float32).contiguous(), io.H, io.W, L, dev)
    if channels_b is None:
        channels_b = torch.zeros_like(channels)
    if tuple(channels_b.shape) != tuple(channels.shape) or channels_b.dtype != torch.float32 \
            or not channels_b.is_contiguous():
        raise ValueError(f"channels_b must be a contiguous f32 tensor shaped like channels {tuple(channels.shape)}")
    maps_b = torch.zeros_like(maps) if maps_b is None else maps_b
    lights_b = torch.zeros_like(lights) if lights_b is None else lights_b
    io.channels_b = channels_b.data_ptr()
    _cabi.check(_cabi.load().deodr_b200_shadow_visibility_b(
        C.byref(io), lights.data_ptr(), L, S, maps.data_ptr(), M, float(bias), float(softness), vis_b.data_ptr(),
        maps_b.data_ptr(), lights_b.data_ptr(), scratch.data_ptr(), _stream(dev)))
    return channels_b, maps_b, lights_b


# ---- shadows from the directional light (the model in include/deodr_b200.h) ------------------------------------------


def _check_sun_visibility(vis: torch.Tensor, H: int, W: int, device) -> torch.Tensor:
    if not isinstance(vis, torch.Tensor) or vis.dtype != torch.float32 or tuple(vis.shape) != (H, W) \
            or not vis.is_contiguous() or vis.device != torch.device(device):
        raise ValueError(f"sun_visibility must be a contiguous [{H},{W}] f32 tensor on {device}; got "
                         f"{getattr(vis, 'dtype', type(vis))} {tuple(getattr(vis, 'shape', ()))}")
    return vis


def _check_sun_map(sun_map: torch.Tensor, device) -> Tuple[torch.Tensor, int]:
    if not isinstance(sun_map, torch.Tensor) or sun_map.dtype != torch.float32 or sun_map.dim() != 2 \
            or sun_map.shape[0] != sun_map.shape[1] or not sun_map.is_contiguous() \
            or sun_map.device != torch.device(device):
        raise ValueError(f"the sun map must be a contiguous [M, M] f32 tensor on {device}; got "
                         f"{getattr(sun_map, 'dtype', type(sun_map))} {tuple(getattr(sun_map, 'shape', ()))}")
    return sun_map, sun_map.shape[0]


def _sun_bounds(bounds) -> Tuple[C.Array, float]:
    """(centre as a C double[3], radius) of bounds (cx, cy, cz, r); the C entry points refuse bad values."""
    b = [float(x) for x in bounds]
    if len(b) != 4:
        raise ValueError(f"bounds must be (cx, cy, cz, r); got {bounds!r}")
    return (C.c_double * 3)(*b[:3]), b[3]


def _light_vector(light: torch.Tensor, device) -> torch.Tensor:
    """The directional light l [3] fp64 on ``device``: a [3] tensor, or the Phong params [6] whose first three it is."""
    if not isinstance(light, torch.Tensor) or light.dtype != torch.float64 or light.dim() != 1 \
            or light.shape[0] not in (3, 6) or not light.is_contiguous() or light.device != torch.device(device):
        raise ValueError(f"light must be a contiguous [3] (or Phong params [6]) fp64 tensor on {device}; got "
                         f"{getattr(light, 'dtype', type(light))} {tuple(getattr(light, 'shape', ()))}")
    return light


def sun_project(vertices: torch.Tensor, light: torch.Tensor, bounds, map_size: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The vertices [V,3] projected into the directional light's shadow map (deodr_b200_sun_project; the model in
    include/deodr_b200.h) -> (ij [V,2], depths [V]) fp64.  ``light``: l [3] fp64 on the device (or the Phong params
    [6]), read there; ``bounds``: the window (cx, cy, cz, r), host values."""
    dev = vertices.device
    vertices = _f64(vertices, dev)
    light = _light_vector(light, dev)
    center, radius = _sun_bounds(bounds)
    n = vertices.shape[0]
    ij = torch.empty((n, 2), dtype=torch.float64, device=dev)
    depths = torch.empty((n,), dtype=torch.float64, device=dev)
    _cabi.check(_cabi.load().deodr_b200_sun_project(vertices.data_ptr(), n, light.data_ptr(), center, radius,
                                                    int(map_size), ij.data_ptr(), depths.data_ptr(), _stream(dev)))
    return ij, depths


def sun_project_backward(vertices: torch.Tensor, light: torch.Tensor, bounds, map_size: int, ij_b: torch.Tensor,
                         depths_b: torch.Tensor, scratch: torch.Tensor, vertices_b: Optional[torch.Tensor] = None,
                         light_b: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """The adjoint of :func:`sun_project` from ``ij_b`` [V,2] and ``depths_b`` [V] (fp32, the rasteriser's) ->
    (vertices_b [V,3], light_b [3] or [6]) fp64, accumulated into the given tensors (created zeroed if None; a
    ``light_b`` of [6] takes the gradient in its first three entries), summed in a fixed order
    (deodr_b200_sun_project_b).  ``scratch``: a buffer of ``mesh_fitter.new_scratch``."""
    dev = vertices.device
    vertices = _f64(vertices, dev)
    light = _light_vector(light, dev)
    center, radius = _sun_bounds(bounds)
    n = vertices.shape[0]
    ij_b = ij_b.to(device=dev, dtype=torch.float32).contiguous()
    depths_b = depths_b.to(device=dev, dtype=torch.float32).contiguous()
    if tuple(ij_b.shape) != (n, 2) or depths_b.numel() != n:
        raise ValueError(f"ij_b must be [{n},2] and depths_b [{n}]; got {tuple(ij_b.shape)} and {tuple(depths_b.shape)}")
    vertices_b = torch.zeros((n, 3), dtype=torch.float64, device=dev) if vertices_b is None else vertices_b
    light_b = torch.zeros((3,), dtype=torch.float64, device=dev) if light_b is None else _light_vector(light_b, dev)
    _cabi.check(_cabi.load().deodr_b200_sun_project_b(
        vertices.data_ptr(), n, light.data_ptr(), center, radius, int(map_size), ij_b.data_ptr(), depths_b.data_ptr(),
        vertices_b.data_ptr(), light_b.data_ptr(), scratch.data_ptr(), _stream(dev)))
    return vertices_b, light_b


def _sun_io(channels: torch.Tensor, light: torch.Tensor, albedo: Optional[torch.Tensor]):
    io, channels = _shadow_io(channels, albedo)
    io.params = _light_vector(light, channels.device).data_ptr()
    return io, channels


def sun_visibility(channels: torch.Tensor, light: torch.Tensor, sun_map: torch.Tensor, bounds, bias: float,
                   softness: float, albedo: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The directional light's visibility [H,W] f32 of a Phong G-buffer's pixels (``channels`` [H,W,C+7], or [H,W,7]
    beside a separate ``albedo``) under its shadow map ``sun_map`` [M,M] f32 (deodr_b200_sun_visibility; the model in
    include/deodr_b200.h): ``light`` l [3] (or the Phong params [6]) fp64 on the device, ``bounds`` (cx, cy, cz, r),
    ``bias`` and ``softness`` in world units.  1 where the coverage is 0, outside the bounds' sphere, or where l = 0."""
    dev = channels.device
    io, channels = _sun_io(channels, light, albedo)
    sun_map, M = _check_sun_map(sun_map, dev)
    center, radius = _sun_bounds(bounds)
    vis = torch.empty((io.H, io.W), dtype=torch.float32, device=dev)
    _cabi.check(_cabi.load().deodr_b200_sun_visibility(C.byref(io), center, radius, sun_map.data_ptr(), M, float(bias),
                                                       float(softness), vis.data_ptr(), _stream(dev)))
    return vis


def sun_visibility_backward(channels: torch.Tensor, light: torch.Tensor, sun_map: torch.Tensor, bounds, bias: float,
                            softness: float, vis_b: torch.Tensor, scratch: torch.Tensor,
                            albedo: Optional[torch.Tensor] = None, channels_b: Optional[torch.Tensor] = None,
                            map_b: Optional[torch.Tensor] = None,
                            light_b: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, ...]:
    """The adjoint of :func:`sun_visibility` from ``vis_b`` [H,W] -> (channels_b, map_b [M,M] f32, light_b [3] or [6]
    fp64), each accumulated into the given tensor (created zeroed if None; a ``light_b`` of [6], such as the shading's
    params_b, takes the gradient in its first three entries): the position and coverage slices of channels_b, the
    texels (fp32 atomics) and l, summed in a fixed order (deodr_b200_sun_visibility_b)."""
    dev = channels.device
    io, channels = _sun_io(channels, light, albedo)
    sun_map, M = _check_sun_map(sun_map, dev)
    center, radius = _sun_bounds(bounds)
    vis_b = _check_sun_visibility(vis_b.to(dev, torch.float32).contiguous(), io.H, io.W, dev)
    if channels_b is None:
        channels_b = torch.zeros_like(channels)
    if tuple(channels_b.shape) != tuple(channels.shape) or channels_b.dtype != torch.float32 \
            or not channels_b.is_contiguous():
        raise ValueError(f"channels_b must be a contiguous f32 tensor shaped like channels {tuple(channels.shape)}")
    map_b = torch.zeros_like(sun_map) if map_b is None else map_b
    light_b = torch.zeros((3,), dtype=torch.float64, device=dev) if light_b is None else _light_vector(light_b, dev)
    io.channels_b = channels_b.data_ptr()
    _cabi.check(_cabi.load().deodr_b200_sun_visibility_b(
        C.byref(io), center, radius, sun_map.data_ptr(), M, float(bias), float(softness), vis_b.data_ptr(),
        map_b.data_ptr(), light_b.data_ptr(), scratch.data_ptr(), _stream(dev)))
    return channels_b, map_b, light_b


# ---- tangent-space normal maps (the model in include/deodr_b200.h) ---------------------------------------------------

NORMAL_MAP_CHANNELS = 13  # the normal-mapped G-buffer: normal (3), position (3), coverage (1), tangent (3), bitangent (3)


def uv_face_csr(faces_uv, nb_uv: int) -> Tuple[np.ndarray, np.ndarray]:
    """The faces of every uv vertex as a CSR (offset [nb_uv+1], index [3T], int32): ascending inside a uv vertex, with
    multiplicity, as the topology's vertex-face CSR."""
    flat = np.ascontiguousarray(np.asarray(faces_uv), dtype=np.int64).reshape(-1)
    if flat.size and (flat.min() < 0 or flat.max() >= nb_uv):
        raise ValueError(f"faces_uv indices must lie in [0, {nb_uv}); got [{flat.min()}, {flat.max()}]")
    offset = np.zeros(nb_uv + 1, dtype=np.int32)
    np.cumsum(np.bincount(flat, minlength=nb_uv), out=offset[1:])
    return offset, np.ascontiguousarray((np.argsort(flat, kind="stable") // 3).astype(np.int32))


class VertexTangents:
    """The per-vertex tangent frames (T, B) of a textured mesh (deodr_b200_vertex_tangents / _b): the faces_uv and the
    uv-vertex-face CSR are uploaded once, beside the mesh's :class:`MeshTopology`.  Neither call synchronises with the
    host; the adjoint is a fixed-order gather (bit-reproducible)."""

    def __init__(self, topology: MeshTopology, faces_uv, nb_uv: int):
        self.topology, self.nb_uv, self.device = topology, int(nb_uv), topology.device
        faces_uv = np.ascontiguousarray(np.asarray(faces_uv), dtype=np.int64)
        if faces_uv.shape != (topology.nb_faces, 3):
            raise ValueError(f"faces_uv must be [{topology.nb_faces},3]; got {faces_uv.shape}")
        offset, index = uv_face_csr(faces_uv, self.nb_uv)
        self.faces_uv = torch.from_numpy(faces_uv.astype(np.uint32).view(np.int32)).to(self.device)
        self.uv_face_offset = torch.from_numpy(offset).to(self.device)
        self.uv_face_index = torch.from_numpy(index).to(self.device)

    def _uv(self, uv: torch.Tensor) -> torch.Tensor:
        uv = _f64(uv, self.device)
        if tuple(uv.shape) != (self.nb_uv, 2):
            raise ValueError(f"uv must be [{self.nb_uv},2]; got {tuple(uv.shape)}")
        return uv

    def frames(self, vertices: torch.Tensor, uv: torch.Tensor) -> torch.Tensor:
        """-> frames [V,6] fp64 = (T_v, B_v) of ``vertices`` [V,3] and ``uv`` [Nuv,2]."""
        vertices, uv = _f64(vertices, self.device), self._uv(uv)
        T, V = self.topology.nb_faces, self.topology.nb_vertices
        face_frames = torch.empty((T, 6), dtype=torch.float64, device=self.device)
        frames = torch.empty((V, 6), dtype=torch.float64, device=self.device)
        m = self.topology.c_struct()
        _cabi.check(_cabi.load().deodr_b200_vertex_tangents(
            C.byref(m), vertices.data_ptr(), self.faces_uv.data_ptr(), uv.data_ptr(), self.nb_uv,
            face_frames.data_ptr(), frames.data_ptr(), _stream(self.device)))
        return frames

    def backward(self, vertices: torch.Tensor, uv: torch.Tensor, frames_b: torch.Tensor,
                 vertices_b: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """The adjoint of :meth:`frames` from ``frames_b`` [V,6] -> (vertices_b [V,3], accumulated into the given
        tensor or a new zeroed one, uv_b [Nuv,2] a new tensor), fp64."""
        vertices, uv = _f64(vertices, self.device), self._uv(uv)
        T, V = self.topology.nb_faces, self.topology.nb_vertices
        frames_b = _f64(frames_b, self.device)
        if tuple(frames_b.shape) != (V, 6):
            raise ValueError(f"frames_b must be [{V},6]; got {tuple(frames_b.shape)}")
        if vertices_b is None:
            vertices_b = torch.zeros((V, 3), dtype=torch.float64, device=self.device)
        uv_b = torch.empty((self.nb_uv, 2), dtype=torch.float64, device=self.device)
        scratch = torch.empty((6 * V + 10 * T,), dtype=torch.float64, device=self.device)
        m = self.topology.c_struct()
        _cabi.check(_cabi.load().deodr_b200_vertex_tangents_b(
            C.byref(m), vertices.data_ptr(), self.faces_uv.data_ptr(), uv.data_ptr(), self.nb_uv,
            self.uv_face_offset.data_ptr(), self.uv_face_index.data_ptr(), frames_b.data_ptr(), scratch.data_ptr(),
            vertices_b.data_ptr(), uv_b.data_ptr(), _stream(self.device)))
        return vertices_b, uv_b


def _check_normal_map_io(gbuffer: torch.Tensor, nmap: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    gbuffer = gbuffer.to(dtype=torch.float32).contiguous()
    nmap = nmap.to(device=gbuffer.device, dtype=torch.float32).contiguous()
    if gbuffer.dim() != 3 or gbuffer.shape[2] != NORMAL_MAP_CHANNELS or tuple(nmap.shape) != tuple(gbuffer.shape[:2]) + (3,):
        raise ValueError(f"the normal-mapped G-buffer must be [H,W,13] and the map raster [H,W,3]; got "
                         f"{tuple(gbuffer.shape)} and {tuple(nmap.shape)}")
    return gbuffer, nmap


def normal_map(gbuffer: torch.Tensor, nmap: torch.Tensor) -> torch.Tensor:
    """The perturbed G-buffer [H,W,7] = (N', X, a) f32 of a normal-mapped G-buffer ``gbuffer`` [H,W,13] = (N, X, a, T,
    B) and the normal map's raster ``nmap`` [H,W,3] (deodr_b200_normal_map; the model in include/deodr_b200.h)."""
    gbuffer, nmap = _check_normal_map_io(gbuffer, nmap)
    H, W = gbuffer.shape[:2]
    out = torch.empty((H, W, PHONG_EXTRA_CHANNELS), dtype=torch.float32, device=gbuffer.device)
    _cabi.check(_cabi.load().deodr_b200_normal_map(gbuffer.data_ptr(), nmap.data_ptr(), H, W, out.data_ptr(),
                                                   _stream(gbuffer.device)))
    return out


def normal_map_backward(gbuffer: torch.Tensor, nmap: torch.Tensor,
                        out_b: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The adjoint of :func:`normal_map` from ``out_b`` [H,W,7] -> (gbuffer_b [H,W,13], nmap_b [H,W,3]) f32
    (deodr_b200_normal_map_b)."""
    gbuffer, nmap = _check_normal_map_io(gbuffer, nmap)
    H, W = gbuffer.shape[:2]
    out_b = out_b.to(device=gbuffer.device, dtype=torch.float32).contiguous()
    if tuple(out_b.shape) != (H, W, PHONG_EXTRA_CHANNELS):
        raise ValueError(f"out_b must be [{H},{W},7]; got {tuple(out_b.shape)}")
    gbuffer_b = torch.empty_like(gbuffer)
    nmap_b = torch.empty_like(nmap)
    _cabi.check(_cabi.load().deodr_b200_normal_map_b(gbuffer.data_ptr(), nmap.data_ptr(), H, W, out_b.data_ptr(),
                                                     gbuffer_b.data_ptr(), nmap_b.data_ptr(), _stream(gbuffer.device)))
    return gbuffer_b, nmap_b


def _light(light_directional):
    if light_directional is None:
        return None, None
    arr = np.ascontiguousarray(light_directional, dtype=np.float64).reshape(3)
    return arr, arr.ctypes.data


def vertex_luminosity(normals: torch.Tensor, vertex_colors: Optional[torch.Tensor], light_directional,
                      ambient: float) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """-> (luminosity [V] f32, colors [V,C] f32 = vertex_colors * luminosity, or None without vertex_colors)."""
    dev = normals.device
    normals = _f64(normals, dev)
    n = normals.shape[0]
    lum = torch.empty((n,), dtype=torch.float32, device=dev)
    colors = None
    C_ = 0
    if vertex_colors is not None:
        vertex_colors = _f64(vertex_colors, dev)
        C_ = vertex_colors.shape[1]
        colors = torch.empty((n, C_), dtype=torch.float32, device=dev)
    keep, lptr = _light(light_directional)
    _cabi.check(_cabi.load().deodr_b200_vertex_luminosity(
        normals.data_ptr(), vertex_colors.data_ptr() if vertex_colors is not None else None, n, C_, lptr, float(ambient),
        lum.data_ptr(), colors.data_ptr() if colors is not None else None, _stream(dev)))
    del keep
    return lum, colors


def vertex_luminosity_backward(normals: torch.Tensor, vertex_colors: Optional[torch.Tensor], light_directional,
                               ambient: float, colors_b: Optional[torch.Tensor] = None,
                               luminosity_b: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """-> dict(normals_b [V,3] f64, vertex_colors_b [V,C] f64 | None, light_b [4] f64 = (directional_b, ambient_b))."""
    dev = normals.device
    normals = _f64(normals, dev)
    n = normals.shape[0]
    C_ = 0
    vcol_b = None
    if vertex_colors is not None:
        vertex_colors = _f64(vertex_colors, dev)
        C_ = vertex_colors.shape[1]
        vcol_b = torch.zeros((n, C_), dtype=torch.float64, device=dev)
    if colors_b is not None:
        colors_b = colors_b.to(device=dev, dtype=torch.float32).contiguous()
    if luminosity_b is not None:
        luminosity_b = luminosity_b.to(device=dev, dtype=torch.float32).contiguous()
    normals_b = torch.zeros((n, 3), dtype=torch.float64, device=dev)
    light_b = torch.zeros((4,), dtype=torch.float64, device=dev)
    keep, lptr = _light(light_directional)
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    _cabi.check(_cabi.load().deodr_b200_vertex_luminosity_b(
        normals.data_ptr(), ptr(vertex_colors), n, C_, lptr, float(ambient), ptr(colors_b), ptr(luminosity_b),
        normals_b.data_ptr(), ptr(vcol_b), light_b.data_ptr(), _stream(dev)))
    del keep
    return {"normals_b": normals_b, "vertex_colors_b": vcol_b, "light_b": light_b}


def topology_arrays(faces, nb_vertices: Optional[int] = None) -> dict:
    """Host-side adjacency arrays of ``DeodrMeshTopology`` (numpy, int32): unique undirected edges, faces per edge and
    faces per vertex as CSR.  Edge n of a face joins its vertices n and (n + 1) % 3 (TriMeshAdjacencies, :42-44)."""
    faces = np.ascontiguousarray(np.asarray(faces), dtype=np.int64)
    assert faces.ndim == 2 and faces.shape[1] == 3
    T = faces.shape[0]
    V = int(faces.max()) + 1 if nb_vertices is None else int(nb_vertices)
    # the kernels index vertices through these arrays unchecked: an index outside [0, V) would read and scatter
    # (vertices_b) out of bounds on the device
    if faces.size and (faces.min() < 0 or faces.max() >= V):
        raise ValueError(f"face vertex indices must lie in [0, {V}); got [{faces.min()}, {faces.max()}]")
    # unique undirected edges: any injective key works, only equality matters
    a = np.concatenate((faces[:, 0], faces[:, 1], faces[:, 2]))
    b = np.concatenate((faces[:, 1], faces[:, 2], faces[:, 0]))
    key = np.maximum(a, b) + np.minimum(a, b) * V
    _, edge_of = np.unique(key, return_inverse=True)
    edge_of = edge_of.reshape(-1)
    nb_edges = int(edge_of.max()) + 1 if T else 0
    face_of = np.tile(np.arange(T), 3)
    faces_edges = np.empty((T, 3), dtype=np.int32)
    faces_edges[face_of, np.repeat(np.arange(3), T)] = edge_of
    order = np.argsort(edge_of, kind="stable")
    edge_face_offset = np.zeros(nb_edges + 1, dtype=np.int32)
    np.cumsum(np.bincount(edge_of, minlength=nb_edges), out=edge_face_offset[1:])
    flat = faces.reshape(-1)
    vorder = np.argsort(flat, kind="stable")  # faces ascending inside a vertex, with multiplicity
    vertex_face_offset = np.zeros(V + 1, dtype=np.int32)
    np.cumsum(np.bincount(flat, minlength=V), out=vertex_face_offset[1:])
    return {
        "faces": np.ascontiguousarray(faces.astype(np.uint32).view(np.int32)),
        "faces_edges": faces_edges,
        "edge_face_offset": edge_face_offset,
        "edge_face_index": np.ascontiguousarray(face_of[order].astype(np.int32)),
        "vertex_face_offset": vertex_face_offset,
        "vertex_face_index": np.ascontiguousarray((vorder // 3).astype(np.int32)),
        "nb_faces": T, "nb_vertices": V, "nb_edges": nb_edges,
    }


class MeshTopology:
    """Static adjacency of a triangulated mesh on the device (``DeodrMeshTopology``), built once on the host from the
    same arrays as the reference's ``TriMeshAdjacencies`` (deodr/triangulated_mesh.py:21-98): unique undirected edges,
    the faces incident to every edge and to every vertex (CSR).  Edge n of a face joins vertices n and (n + 1) % 3, the
    order of ``faces_edges`` in the reference - which is also the order of the rasteriser's ``edgeflags`` columns."""

    def __init__(self, faces, nb_vertices: Optional[int] = None, clockwise: bool = False, device="cuda"):
        arrays = topology_arrays(faces, nb_vertices)
        self.nb_faces, self.nb_vertices, self.nb_edges = arrays["nb_faces"], arrays["nb_vertices"], arrays["nb_edges"]
        self.clockwise = bool(clockwise)
        dev = torch.device(device)
        self.device = dev
        self.t = {k: torch.from_numpy(v).to(dev) for k, v in arrays.items() if isinstance(v, np.ndarray)}

    def c_struct(self) -> _cabi.MeshTopology:
        m = _cabi.MeshTopology()
        for name, t in self.t.items():
            setattr(m, name, t.data_ptr())
        m.nb_faces, m.nb_edges, m.nb_vertices, m.clockwise = self.nb_faces, self.nb_edges, self.nb_vertices, int(self.clockwise)
        return m

    def edge_on_silhouette(self, ij: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``TriMeshAdjacencies.edge_on_silhouette`` (:153-166): edgeflags [T,3] uint8 for the projection ``ij`` [V,2]."""
        ij = _f64(ij, self.device)
        if out is None:
            out = torch.empty((self.nb_faces, 3), dtype=torch.uint8, device=self.device)
        visible = torch.empty((self.nb_faces,), dtype=torch.uint8, device=self.device)
        m = self.c_struct()
        _cabi.check(_cabi.load().deodr_b200_edge_on_silhouette(C.byref(m), ij.data_ptr(), visible.data_ptr(),
                                                               out.data_ptr(), _stream(self.device)))
        return out

    def vertex_normals(self, vertices: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """-> (face_normals [T,3], vertex_normals [V,3]) fp64 (compute_face_normals + compute_vertex_normals)."""
        vertices = _f64(vertices, self.device)
        fn = torch.empty((self.nb_faces, 3), dtype=torch.float64, device=self.device)
        vn = torch.empty((self.nb_vertices, 3), dtype=torch.float64, device=self.device)
        m = self.c_struct()
        _cabi.check(_cabi.load().deodr_b200_vertex_normals(C.byref(m), vertices.data_ptr(), fn.data_ptr(), vn.data_ptr(),
                                                           _stream(self.device)))
        return fn, vn

    def vertex_normals_backward(self, vertices: torch.Tensor, vertex_normals_b: torch.Tensor,
                                out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Accumulates the adjoint of :meth:`vertex_normals` into ``out`` ([V,3] fp64, created zeroed if None)."""
        vertices = _f64(vertices, self.device)
        vertex_normals_b = _f64(vertex_normals_b, self.device)
        if out is None:
            out = torch.zeros((self.nb_vertices, 3), dtype=torch.float64, device=self.device)
        scratch = torch.empty((self.nb_vertices, 3), dtype=torch.float64, device=self.device)
        m = self.c_struct()
        _cabi.check(_cabi.load().deodr_b200_vertex_normals_b(C.byref(m), vertices.data_ptr(), vertex_normals_b.data_ptr(),
                                                             scratch.data_ptr(), out.data_ptr(), _stream(self.device)))
        return out


def subdivision_level_arrays(faces, nb_vertices: int) -> dict:
    """Host-side arrays of one ``DeodrLoopLevel`` (numpy): :func:`topology_arrays` of the coarse mesh plus the
    "shares a face" neighbour CSR (itself excluded, neighbours ascending, as ``mesh_fitter.laplacian_neighbours``) with
    the id of the edge joining every neighbour, the edge of every vertex to itself (-1 if none), the edge endpoints, and
    ``fine_faces`` [4T,3] int64 in the reference's order (faces1; faces2; faces3; faces4, triangulated_mesh.py:521-549)."""
    arrays = topology_arrays(faces, nb_vertices)
    V, E = arrays["nb_vertices"], arrays["nb_edges"]
    faces = np.asarray(arrays["faces"]).view(np.uint32).astype(np.int64).reshape(-1, 3)
    a = np.concatenate((faces[:, 0], faces[:, 1], faces[:, 2]))
    b = np.concatenate((faces[:, 1], faces[:, 2], faces[:, 0]))
    first = np.zeros(E, dtype=np.int64)
    first[arrays["faces_edges"].T.reshape(-1)] = np.arange(a.size)  # one occurrence of every unique edge
    ea, eb = a[first], b[first]
    edge_ids = np.arange(E)
    loop = ea == eb  # the edge from a vertex to itself of a degenerate face
    self_edge = np.full(V, -1, dtype=np.int32)
    self_edge[ea[loop]] = edge_ids[loop]
    keep = ~loop
    rows = np.concatenate((ea[keep], eb[keep]))
    cols = np.concatenate((eb[keep], ea[keep]))
    eids = np.concatenate((edge_ids[keep], edge_ids[keep]))
    order = np.lexsort((cols, rows))
    offset = np.zeros(V + 1, dtype=np.int32)
    np.cumsum(np.bincount(rows, minlength=V), out=offset[1:])
    fe = arrays["faces_edges"].astype(np.int64) + V
    fine_faces = np.vstack((np.column_stack((faces[:, 0], fe[:, 0], fe[:, 2])),
                            np.column_stack((faces[:, 1], fe[:, 1], fe[:, 0])),
                            np.column_stack((faces[:, 2], fe[:, 2], fe[:, 1])),
                            fe))
    arrays.update(neighbour_offset=offset, neighbour_index=np.ascontiguousarray(cols[order].astype(np.int32)),
                  neighbour_edge=np.ascontiguousarray(eids[order].astype(np.int32)), self_edge=self_edge,
                  edge_vertices=np.ascontiguousarray(np.stack((ea, eb), axis=1).astype(np.int32)),
                  fine_faces=np.ascontiguousarray(fine_faces))
    return arrays


class LoopSubdivision:
    """``n_iter`` levels of the reference's Loop subdivision (``ColoredTriMesh.subdivise``, deodr/triangulated_mesh.py:
    499-562) of a fixed topology, on the device: every level's adjacency is built once on the host and uploaded, then
    :meth:`apply` maps coarse vertices [V,3] (and colours [V,C]) to fine ones with one launch per level
    (deodr_b200_loop_subdivide), and :meth:`backward` maps fine gradients back with the transpose, one launch per level
    in reverse (deodr_b200_loop_subdivide_b, bit-reproducible).  Neither synchronises with the host.

    ``faces`` [4^n T, 3] int64 are the fine faces, equal to the reference's; ``nb_vertices`` the fine vertex count.
    The reference's quirks are kept (include/deodr_b200.h, INTEGRATION.md section 5): boundary edge points get weights
    that sum to 5/8, a vertex in no face stays where it is.  ``clockwise`` is the winding of the coarse faces, which the
    fine faces keep (the reference's returned mesh drops it)."""

    def __init__(self, faces, nb_vertices: int, n_iter: int, clockwise: bool = False, device="cuda"):
        if int(n_iter) < 0:
            raise ValueError(f"n_iter must be >= 0; got {n_iter}")
        self.device = torch.device(device)
        self.n_iter, self.clockwise = int(n_iter), bool(clockwise)
        self.coarse_nb_vertices = int(nb_vertices)
        faces = np.ascontiguousarray(np.asarray(faces), dtype=np.int64)
        V = self.coarse_nb_vertices
        self.levels = []  # per level: (device tensors, nb_faces, nb_edges, nb_vertices)
        for _ in range(self.n_iter):
            arrays = subdivision_level_arrays(faces, V)
            t = {k: torch.from_numpy(v).to(self.device) for k, v in arrays.items()
                 if isinstance(v, np.ndarray) and k != "fine_faces"}
            self.levels.append((t, arrays["nb_faces"], arrays["nb_edges"], V))
            faces, V = arrays["fine_faces"], V + arrays["nb_edges"]
        self.faces, self.nb_vertices = faces, V

    @staticmethod
    def _struct(level) -> _cabi.LoopLevel:
        t, T, E, V = level
        s = _cabi.LoopLevel()
        for name in ("faces", "faces_edges", "edge_face_offset", "edge_face_index", "vertex_face_offset",
                     "vertex_face_index"):
            setattr(s.topology, name, t[name].data_ptr())
        s.topology.nb_faces, s.topology.nb_edges, s.topology.nb_vertices = T, E, V
        for name in ("neighbour_offset", "neighbour_index", "neighbour_edge", "self_edge", "edge_vertices"):
            setattr(s, name, t[name].data_ptr())
        return s

    def _check(self, x: Optional[torch.Tensor], rows: int, name: str, cols: Optional[int] = None):
        if x is None:
            return None
        if x.dim() != 2 or x.shape[0] != rows or (cols is not None and x.shape[1] != cols):
            raise ValueError(f"{name} must be [{rows},{cols if cols is not None else 'C'}]; got {tuple(x.shape)}")
        return _f64(x, self.device)

    def apply(self, vertices: torch.Tensor,
              colors: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """coarse vertices [V,3] (and colours [V,C] or None) -> (fine vertices [V',3], fine colours [V',C] or None),
        new fp64 tensors."""
        v = self._check(vertices, self.coarse_nb_vertices, "vertices", 3)
        c = self._check(colors, self.coarse_nb_vertices, "colors")
        if self.n_iter == 0:
            return v.clone(), (c.clone() if c is not None else None)
        lib, stream = _cabi.load(), _stream(self.device)
        for level in self.levels:
            rows = level[3] + level[2]
            fv = torch.empty((rows, 3), dtype=torch.float64, device=self.device)
            fc = torch.empty((rows, c.shape[1]), dtype=torch.float64, device=self.device) if c is not None else None
            s = self._struct(level)
            _cabi.check(lib.deodr_b200_loop_subdivide(C.byref(s), v.data_ptr(), c.data_ptr() if c is not None else None,
                                                      c.shape[1] if c is not None else 0, fv.data_ptr(),
                                                      fc.data_ptr() if fc is not None else None, stream))
            v, c = fv, fc
        return v, c

    def backward(self, vertices_b: Optional[torch.Tensor],
                 colors_b: Optional[torch.Tensor] = None) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """The transpose of :meth:`apply`: fine gradients [V',3] (and [V',C]; either may be None) -> coarse gradients
        [V,3] (and [V,C]), new fp64 tensors (None where the fine gradient is None)."""
        g = self._check(vertices_b, self.nb_vertices, "vertices_b", 3)
        gc = self._check(colors_b, self.nb_vertices, "colors_b")
        if self.n_iter == 0:
            return (g.clone() if g is not None else None), (gc.clone() if gc is not None else None)
        lib, stream = _cabi.load(), _stream(self.device)
        for level in reversed(self.levels):
            V = level[3]
            vb = torch.empty((V, 3), dtype=torch.float64, device=self.device) if g is not None else None
            cb = torch.empty((V, gc.shape[1]), dtype=torch.float64, device=self.device) if gc is not None else None
            s = self._struct(level)
            ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
            _cabi.check(lib.deodr_b200_loop_subdivide_b(C.byref(s), ptr(g), ptr(gc), gc.shape[1] if gc is not None else 0,
                                                        ptr(vb), ptr(cb), stream))
            g, gc = vb, cb
        return g, gc


def loop_subdivision(faces, vertices, colors=None, n_iter: int = 1):
    """The reference's ``loop_subdivision(mesh, n_iter)`` as a function of arrays: -> (fine faces [4^n T,3] int64,
    fine vertices [V',3], fine colours [V',C] or None), computed on the device.  Arrays in, arrays out (numpy);
    tensors in, fp64 tensors on their device out."""
    as_tensor = isinstance(vertices, torch.Tensor)
    device = vertices.device if as_tensor else torch.device("cuda")
    v = vertices if as_tensor else torch.from_numpy(np.ascontiguousarray(vertices, dtype=np.float64))
    c = None
    if colors is not None:
        c = colors if isinstance(colors, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(colors, np.float64))
    sub = LoopSubdivision(faces, v.shape[0], n_iter, device=device)
    fv, fc = sub.apply(v.to(device), c.to(device) if c is not None else None)
    if as_tensor:
        return sub.faces, fv, fc
    return sub.faces, fv.cpu().numpy(), (fc.cpu().numpy() if fc is not None else None)


def skeleton_arrays(parents, joints, skin_index, skin_weight) -> dict:
    """Host arrays of ``DeodrSkeleton`` (include/deodr_b200.h, "Linear blend skinning"), built and checked here:
    ``parents`` [J] (parents[j] < j, -1 for a root), ``joints`` [J,3] rest centres, ``skin_index`` [V,K] joints in
    [0, J) and ``skin_weight`` [V,K] (not renormalised), 1 <= J <= 1024 and 1 <= K <= 8.  Adds the depth levels (the
    roots first), the children CSR and the joint CSR of the entries i*K+k (ascending in every row), cut in chunks of
    ``SKIN_CHUNK`` entries.  Raises ValueError for a parent that is not lower than its joint, an index outside
    [0, J), a non-finite centre or weight, or a J, V or K out of range."""
    parents = np.asarray(parents)
    joints = np.asarray(joints, dtype=np.float64)
    skin_index = np.asarray(skin_index)
    skin_weight = np.asarray(skin_weight, dtype=np.float64)
    if parents.ndim != 1 or not 1 <= parents.size <= _cabi.SKIN_MAX_JOINTS:
        raise ValueError(f"parents must be [J] with 1 <= J <= {_cabi.SKIN_MAX_JOINTS}; got shape {parents.shape}")
    J = parents.size
    if not np.issubdtype(parents.dtype, np.integer) or not np.issubdtype(skin_index.dtype, np.integer):
        raise ValueError("parents and skin_index must be integer arrays")
    parents = parents.astype(np.int64)
    if np.any(parents >= np.arange(J)):
        raise ValueError("every parent must be lower than its joint (parents[j] < j)")
    if np.any(parents < -1):
        raise ValueError("a parent must be a joint index in [0, J) or -1 for a root")
    if joints.shape != (J, 3):
        raise ValueError(f"joints must be [{J},3]; got {joints.shape}")
    if skin_index.ndim != 2 or skin_index.shape[0] < 1 or not 1 <= skin_index.shape[1] <= _cabi.SKIN_MAX_INFLUENCES:
        raise ValueError(f"skin_index must be [V,K] with V >= 1 and 1 <= K <= {_cabi.SKIN_MAX_INFLUENCES}; "
                         f"got shape {skin_index.shape}")
    if skin_weight.shape != skin_index.shape:
        raise ValueError(f"skin_weight must be {skin_index.shape} like skin_index; got {skin_weight.shape}")
    V, K = skin_index.shape
    if V * K > 0x7FFFFFFF:
        raise ValueError("V * K must fit in int32")
    if np.any(skin_index < 0) or np.any(skin_index >= J):
        raise ValueError(f"skin_index must lie in [0, {J})")
    if not np.all(np.isfinite(joints)) or not np.all(np.isfinite(skin_weight)):
        raise ValueError("joint centres and skinning weights must be finite")
    depth = np.zeros(J, dtype=np.int64)
    for j in range(J):
        if parents[j] >= 0:
            depth[j] = depth[parents[j]] + 1
    nb_levels = int(depth.max()) + 1

    def csr(rows, n):
        offset = np.zeros(n + 1, dtype=np.int32)
        np.cumsum(np.bincount(rows, minlength=n), out=offset[1:])
        return offset, np.argsort(rows, kind="stable").astype(np.int32)

    level_offset, level_index = csr(depth, nb_levels)
    non_roots = np.flatnonzero(parents >= 0)
    child_offset = np.zeros(J + 1, dtype=np.int32)
    np.cumsum(np.bincount(parents[non_roots], minlength=J), out=child_offset[1:])
    child_index = non_roots[np.argsort(parents[non_roots], kind="stable")].astype(np.int32)
    joint_offset, joint_entry = csr(skin_index.reshape(-1).astype(np.int64), J)
    chunks = (np.diff(joint_offset) + _cabi.SKIN_CHUNK - 1) // _cabi.SKIN_CHUNK
    chunk_offset = np.zeros(J + 1, dtype=np.int32)
    np.cumsum(chunks, out=chunk_offset[1:])
    return {"parents": parents.astype(np.int32), "centres": np.ascontiguousarray(joints),
            "level_offset": level_offset, "level_index": level_index, "child_offset": child_offset,
            "child_index": child_index if child_index.size else np.zeros(1, np.int32),
            "skin_index": np.ascontiguousarray(skin_index, dtype=np.int32),
            "skin_weight": np.ascontiguousarray(skin_weight), "joint_offset": joint_offset, "joint_entry": joint_entry,
            "chunk_offset": chunk_offset, "nb_joints": J, "nb_vertices": V, "nb_influences": K,
            "nb_levels": nb_levels, "nb_chunks": int(chunk_offset[-1])}


class LinearBlendSkinning:
    """A mesh articulated by a skeleton (include/deodr_b200.h, "Linear blend skinning"), on the device: the host
    arrays of :func:`skeleton_arrays` are built and uploaded once, then :meth:`apply` maps rest vertices [V,3] and
    axis-angle joint rotations [J,3] to skinned vertices, and :meth:`backward` maps their gradient back to the rest
    vertices, the rotations and, on request, the weights.  Neither synchronises with the host; the adjoint uses no
    atomics, so it gives the same bits from call to call.  The joint centres are constants.

    ``transforms`` [J,24] is the forward kinematics table (Rg, tg, M, b per joint) that :meth:`apply` writes and
    :meth:`backward` re-reads: both use the binding's own table unless given one, so a backward belongs to the last
    apply unless the two share a table.  ``skin_weight`` [V,K] replaces the bound weights in a call (the joint CSR
    depends on the indices only)."""

    def __init__(self, parents, joints, skin_index, skin_weight, device="cuda"):
        self.device = torch.device(device)
        arrays = skeleton_arrays(parents, joints, skin_index, skin_weight)
        self.parents = arrays["parents"]
        self.nb_joints, self.nb_vertices, self.nb_influences = (arrays["nb_joints"], arrays["nb_vertices"],
                                                                arrays["nb_influences"])
        self.nb_chunks = arrays["nb_chunks"]
        self.t = {k: torch.from_numpy(v).to(self.device) for k, v in arrays.items() if isinstance(v, np.ndarray)}
        self.device = self.t["parents"].device  # "cuda" -> "cuda:N", as the tensors of the calls report it
        self.skin_weight = self.t["skin_weight"]
        self._struct = _cabi.Skeleton()
        for name, t in self.t.items():
            setattr(self._struct, name, t.data_ptr())
        for name in ("nb_joints", "nb_vertices", "nb_influences", "nb_levels", "nb_chunks"):
            setattr(self._struct, name, arrays[name])
        self.transforms = torch.zeros((self.nb_joints, 24), dtype=torch.float64, device=self.device)
        self._scratch = torch.empty(((self.nb_chunks + self.nb_joints) * 12,), dtype=torch.float64, device=self.device)

    def _check(self, x: torch.Tensor, shape: Tuple[int, int], name: str) -> torch.Tensor:
        if tuple(x.shape) != shape:
            raise ValueError(f"{name} must be {list(shape)}; got {tuple(x.shape)}")
        return _f64(x, self.device)

    def _skeleton(self, skin_weight: Optional[torch.Tensor]) -> Tuple[_cabi.Skeleton, Optional[torch.Tensor]]:
        if skin_weight is None:
            return self._struct, None
        w = self._check(skin_weight, (self.nb_vertices, self.nb_influences), "skin_weight")
        s = _cabi.Skeleton.from_buffer_copy(self._struct)
        s.skin_weight = w.data_ptr()
        return s, w

    def _table(self, transforms: Optional[torch.Tensor]) -> torch.Tensor:
        if transforms is None:
            return self.transforms
        if tuple(transforms.shape) != (self.nb_joints, 24) or transforms.dtype != torch.float64 or \
                transforms.device != self.device or not transforms.is_contiguous():
            raise ValueError(f"transforms must be a contiguous [{self.nb_joints},24] fp64 tensor on {self.device}")
        return transforms

    def apply(self, vertices: torch.Tensor, rotations: torch.Tensor, skin_weight: Optional[torch.Tensor] = None,
              transforms: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """rest vertices [V,3] and rotations [J,3] -> skinned vertices [V,3] fp64 (into ``out`` when given)."""
        v = self._check(vertices, (self.nb_vertices, 3), "vertices")
        r = self._check(rotations, (self.nb_joints, 3), "rotations")
        s, w = self._skeleton(skin_weight)
        table = self._table(transforms)
        if out is None:
            out = torch.empty((self.nb_vertices, 3), dtype=torch.float64, device=self.device)
        _cabi.check(_cabi.load().deodr_b200_skin(C.byref(s), v.data_ptr(), r.data_ptr(), table.data_ptr(),
                                                 out.data_ptr(), _stream(self.device)))
        return out

    def backward(self, vertices: torch.Tensor, rotations: torch.Tensor, skinned_b: torch.Tensor,
                 weights_grad: bool = False, skin_weight: Optional[torch.Tensor] = None,
                 transforms: Optional[torch.Tensor] = None, add_to: Optional[torch.Tensor] = None, out=None):
        """-> (vertices_b [V,3], rotations_b [J,3]) or, with ``weights_grad``, (vertices_b, rotations_b, weights_b
        [V,K]), fp64, from skinned_b [V,3].  vertices_b = add_to + the adjoint (``add_to`` may be ``vertices_b``
        itself).  ``out`` = (vertices_b, rotations_b) buffers to write into."""
        v = self._check(vertices, (self.nb_vertices, 3), "vertices")
        r = self._check(rotations, (self.nb_joints, 3), "rotations")
        g = self._check(skinned_b, (self.nb_vertices, 3), "skinned_b")
        s, w = self._skeleton(skin_weight)
        table = self._table(transforms)
        if out is None:
            out = (torch.empty((self.nb_vertices, 3), dtype=torch.float64, device=self.device),
                   torch.empty((self.nb_joints, 3), dtype=torch.float64, device=self.device))
        v_b, r_b = out
        w_b = (torch.empty((self.nb_vertices, self.nb_influences), dtype=torch.float64, device=self.device)
               if weights_grad else None)
        _cabi.check(_cabi.load().deodr_b200_skin_b(
            C.byref(s), v.data_ptr(), r.data_ptr(), table.data_ptr(), g.data_ptr(),
            add_to.data_ptr() if add_to is not None else None, v_b.data_ptr(),
            w_b.data_ptr() if w_b is not None else None, r_b.data_ptr(), self._scratch.data_ptr(),
            _stream(self.device)))
        return (v_b, r_b, w_b) if weights_grad else (v_b, r_b)


SHADOW_MAP_SIZES = (8, 4096)


def check_shadow_arguments(shading: str, point_lights, size: int, bias, softness) -> int:
    """The refusals of a view's (or a scene's) shadow arguments -> the map size M (0: no shadows)."""
    size = int(size)
    if size == 0:
        return 0
    if shading not in ("phong", "phong_textured", "pbr_textured"):
        raise ValueError("shadows need per-pixel shading (shading='phong', 'phong_textured' or 'pbr_textured'): a "
                         "shadow edge crosses triangles, and per-vertex visibility would smear it over each one")
    if point_lights is None:
        raise ValueError("shadows are cast from point lights: this view has none")
    if not SHADOW_MAP_SIZES[0] <= size <= SHADOW_MAP_SIZES[1]:
        raise ValueError(f"shadow_map_size must be 0 or lie in [{SHADOW_MAP_SIZES[0]}, {SHADOW_MAP_SIZES[1]}]; got {size}")
    if bias is None or softness is None:
        raise ValueError("shadows need both shadow_bias and shadow_softness (world units: no default is free of scale)")
    if not (np.isfinite(bias) and np.isfinite(softness) and bias > 0 and softness > 0):
        raise ValueError(f"shadow_bias and shadow_softness must be finite and > 0; got {bias} and {softness}")
    return size


def check_sun_shadow_arguments(shading: str, light_directional, size: int, bias, softness, bounds) -> int:
    """The refusals of a view's (or a scene's) directional-light shadow arguments -> the map size M (0: none)."""
    size = int(size)
    if size == 0:
        return 0
    if shading not in ("phong", "phong_textured", "pbr_textured"):
        raise ValueError("light shadows need per-pixel shading (shading='phong', 'phong_textured' or 'pbr_textured'): "
                         "a shadow edge crosses triangles, and per-vertex visibility would smear it over each one")
    if light_directional is None:
        raise ValueError("light shadows are cast from the directional light: this view has none")
    if not SHADOW_MAP_SIZES[0] <= size <= SHADOW_MAP_SIZES[1]:
        raise ValueError(f"light_shadow_map_size must be 0 or lie in [{SHADOW_MAP_SIZES[0]}, {SHADOW_MAP_SIZES[1]}]; "
                         f"got {size}")
    if bias is None or softness is None or bounds is None:
        raise ValueError("light shadows need light_shadow_bias, light_shadow_softness and light_shadow_bounds (world "
                         "units: the light has no position, so no default is free of scale)")
    if not (np.isfinite(bias) and np.isfinite(softness) and bias > 0 and softness > 0):
        raise ValueError(f"light_shadow_bias and light_shadow_softness must be finite and > 0; got {bias} and "
                         f"{softness}")
    b = np.asarray(bounds, dtype=np.float64).reshape(-1)
    if b.shape != (4,) or not np.all(np.isfinite(b)) or not b[3] > 0:
        raise ValueError(f"light_shadow_bounds must be (cx, cy, cz, r), finite, with r > 0; got {bounds!r}")
    return size


class DepthMaps:
    """NF one-channel M x M depth scenes of a mesh (the shadow maps), whose ij, depths, colours (the depth) and
    silhouette flags are slices of one buffer each, filled by one projection launch and one silhouette launch over a
    topology of NF disjoint copies of the faces.  The caller renders :attr:`scenes` beside its own in one renderer
    call, with :meth:`outputs` as their results, and back-propagates them in one call with :meth:`image_bs` and
    :meth:`grads`, then calls the subclass's ``backward``."""

    def __init__(self, faces_u32: np.ndarray, V: int, NF: int, M: int, clockwise: bool, device):
        from .renderer import DeviceScene
        from .scenes import SceneArrays

        T = faces_u32.shape[0]
        self.NF, self.M, self.V, self.device = NF, M, V, device
        tiled = (faces_u32[None].astype(np.int64) + (np.arange(NF) * V)[:, None, None]).reshape(-1, 3)
        self.topology = MeshTopology(tiled, NF * V, clockwise=clockwise, device=device)
        self.edgeflags = torch.zeros((NF * T, 3), dtype=torch.uint8, device=device)
        self.colors = torch.zeros((NF, V, 1), dtype=torch.float32, device=device)
        self.ij_b = torch.zeros((NF, V, 2), dtype=torch.float32, device=device)
        self.colors_b = torch.zeros((NF, V, 1), dtype=torch.float32, device=device)
        self.maps4 = torch.empty((NF, M, M, 1), dtype=torch.float32, device=device)
        self.maps = self.maps4.view(NF, M, M)
        self.maps_b = torch.zeros((NF, M, M), dtype=torch.float32, device=device)
        self.cameras = self.ij = self.depths = None
        self.fwds = None
        # a depth render (DeviceMeshView.render_depth) with culling on over the background depth SHADOW_FAR
        base = DeviceScene(SceneArrays(
            faces=faces_u32, faces_uv=np.zeros((T, 3), np.uint32), ij=np.zeros((V, 2)), depths=np.ones(V),
            textured=np.zeros(T, bool), uv=np.zeros((1, 2)), shade=np.zeros(V), colors=np.zeros((V, 1)),
            shaded=np.zeros(T, bool), edgeflags=np.zeros((T, 3), bool), height=M, width=M, nb_colors=1,
            texture=np.zeros((2, 2, 1)), background_image=None, background_color=np.array([SHADOW_FAR]),
            clockwise=clockwise, backface_culling=True, strict_edge=True, perspective_correct=False,
            integer_pixel_centers=True), device)
        self._base = base
        self.scenes = []
        for f in range(NF):
            sc = copy.copy(base)
            sc.t = dict(base.t)
            sc.t.update(colors=self.colors[f], edgeflags=self.edgeflags[f * T:(f + 1) * T])
            self.scenes.append(sc)
        # the outputs of every face (the image a slice of the maps), and the shared gradient slots a depth scene
        # never writes (no texture, no shade)
        self._outputs = [{"image": self.maps4[f], "z_buffer": torch.empty((M, M), dtype=torch.float64, device=device),
                          "owner": torch.empty((M, M), dtype=torch.int32, device=device), "face_id": None,
                          "barycentric": None, "err_buffer": None} for f in range(NF)]
        self._unused_b = base.zero_grads()

    def _set_projection(self, ij: torch.Tensor, depths: torch.Tensor) -> None:
        """Sets the scenes' ij [NF, V, 2], depths [NF, V], colours and silhouette flags."""
        self.ij, self.depths = ij, depths
        self.colors.copy_(self.depths[:, :, None])
        self.topology.edge_on_silhouette(self.ij.view(-1, 2), out=self.edgeflags)
        for f, sc in enumerate(self.scenes):
            sc.t["ij"], sc.t["depths"] = self.ij[f], self.depths[f]

    def outputs(self):
        return self._outputs

    def zero_maps_b(self) -> torch.Tensor:
        self.maps_b.zero_()
        return self.maps_b

    def image_bs(self, maps_b: torch.Tensor):
        return [maps_b[f].view(self.M, self.M, 1) for f in range(self.NF)]

    def grads(self):
        """The faces' gradient slots: ij_b and colors_b slices of one buffer each, zeroed."""
        self.ij_b.zero_()
        self.colors_b.zero_()
        u = self._unused_b
        return [{"ij_b": self.ij_b[f], "colors_b": self.colors_b[f], "uv_b": u["uv_b"], "shade_b": u["shade_b"],
                 "texture_b": u["texture_b"]} for f in range(self.NF)]


class ShadowCubes(DepthMaps):
    """The cube shadow maps of L point lights: 6L depth scenes (face 6 j + k) projected by :func:`cube_project`."""

    def __init__(self, faces_u32: np.ndarray, V: int, L: int, M: int, clockwise: bool, device):
        super().__init__(faces_u32, V, 6 * L, M, clockwise, device)
        self.L = L

    def prepare(self, vertices: torch.Tensor, lights: torch.Tensor) -> None:
        """Projects the vertices through the cube cameras of ``lights`` (read on the device) and sets the scenes'
        ij, depths, colours and silhouette flags."""
        if lights.shape[0] != self.L:
            raise ValueError(f"the view's shadow maps were made for {self.L} lights; the table has {lights.shape[0]}")
        self.cameras, ij, depths = cube_project(vertices, lights, self.M)
        self._set_projection(ij, depths)

    def backward(self, vertices: torch.Tensor, lights: torch.Tensor, vertices_b: torch.Tensor,
                 lights_b: torch.Tensor, scratch: torch.Tensor) -> None:
        """The cube projection's adjoint after the faces' raster adjoint: depths_b = colors_b (the colour is the
        depth), accumulated into vertices_b and the positions of lights_b."""
        cube_project_backward(vertices, lights, self.M, self.cameras, self.ij_b, self.colors_b.view(6 * self.L, -1),
                              scratch, vertices_b=vertices_b, lights_b=lights_b)


class SunShadowMap(DepthMaps):
    """The directional light's shadow map: one depth scene projected by :func:`sun_project` over the window
    ``bounds`` (cx, cy, cz, r)."""

    def __init__(self, faces_u32: np.ndarray, V: int, M: int, bounds, clockwise: bool, device):
        super().__init__(faces_u32, V, 1, M, clockwise, device)
        self.bounds = tuple(float(b) for b in bounds)

    @property
    def map(self) -> torch.Tensor:
        return self.maps[0]

    def prepare(self, vertices: torch.Tensor, light: torch.Tensor) -> None:
        """Projects the vertices into the map of ``light`` (l [3] or the Phong params [6], read on the device) and
        sets the scene's ij, depths, colour and silhouette flags."""
        ij, depths = sun_project(vertices, light, self.bounds, self.M)
        self._set_projection(ij[None], depths[None])

    def backward(self, vertices: torch.Tensor, light: torch.Tensor, vertices_b: torch.Tensor, light_b: torch.Tensor,
                 scratch: torch.Tensor) -> None:
        """The projection's adjoint after the map's raster adjoint, accumulated into vertices_b and light_b (l's
        gradient: [3], or the Phong params_b [6])."""
        sun_project_backward(vertices, light, self.bounds, self.M, self.ij_b[0], self.colors_b.view(-1), scratch,
                             vertices_b=vertices_b, light_b=light_b)


class DeviceMeshView:
    """One view of a lit mesh (Gouraud by default), device-resident end to end: the chain of ``Scene3D.render`` /
    ``render_backward`` (deodr/differentiable_renderer.py:871-1052) with every step on the GPU -

        vertices -> normals -> luminosity -> colours        project_points -> ij, depths -> silhouette flags
        -> rasteriser (deodr_b200_render) -> image          image_b -> rasteriser adjoint -> ij_b, colors_b
        -> luminosity / normals / projection adjoints -> vertices_b (+ vertex_colors_b, light_b)

    No tensor crosses PCIe inside :meth:`render` / :meth:`backward`; the shared gradients of several views are plain
    CUDA tensors that a caller sums over views and all-reduces over ranks (deodr_b200.distributed).

    A TEXTURED view (``uv`` [Nuv,2], ``faces_uv`` [T,3] and ``texture`` [Ht,Wt,C] given, in the conventions of the
    reference's ``ColoredTriMesh``: uv in texel units, shifted by -0.5) renders the texture shaded by the vertex
    luminosity, as ``Scene3D.render`` does for a mesh with ``uv`` (:921-930); its :meth:`backward` also returns
    ``texture_b`` and ``uv_b`` - an adjoint the reference does not have (INTEGRATION.md section 5).

    ``shading="phong"`` lights an untextured view per pixel instead (the model of ``DeodrPhongIO``,
    include/deodr_b200.h): a second scene of K = C + 7 channels per vertex - the vertex colours, the unit normals, the
    world positions and a coverage of 1 - is rasterised over a zero background with the view's sigma, and
    :func:`phong_shade` turns that G-buffer into the image, adding a specular highlight of strength ``specular`` (ks)
    and exponent ``shininess`` (e).  Its :meth:`backward` also returns ``specular_b`` [2] = (ks_b, e_b).  A Phong view
    refuses textures and ``perspective_correct``; :meth:`render_depth` and :meth:`render_deferred` do not shade and are
    those of a Gouraud view.

    ``shading="phong_textured"`` lights a TEXTURED view per pixel (the albedo form of ``deodr_b200_phong_shade_albedo``,
    include/deodr_b200.h): two rasters of the same geometry, rendered in one call - the textured scene with a shade of
    1 over a zero background (the albedo A, the texture sample times the coverage) and a G-buffer of 7 channels (unit
    normals, world positions, 1) - shaded as a Phong view's, coloured environments [9,C] included.  Its
    :meth:`backward` returns vertices_b, texture_b, uv_b, light_b and specular_b (and sh_b, and with ``camera_grad`` the
    camera's gradient with the centre's share), from one adjoint call over both rasters.  It refuses untextured views
    and ``perspective_correct``; :meth:`render_depth` and :meth:`render_deferred` are those of a textured view.

    ``normal_map`` [Ht,Wt,3] (the texture's Ht and Wt; raw tangent-space vectors, x along +u, y along +v, z along the
    outward normal) perturbs a textured Phong view's per-pixel normal (the model in include/deodr_b200.h): the G-buffer
    gets 13 channels, the per-vertex tangent frames (T, B) after the coverage, a third raster samples the map through
    the view's uv, and :func:`normal_map` turns the two into the 7-channel G-buffer that every shading and shadow reads.
    The three rasters (and any shadow maps) are rendered by one renderer call and back-propagated by one;
    :meth:`backward` adds ``normal_map_b`` [Ht,Wt,3] f32 and folds the tangent frames' share into ``vertices_b`` and
    ``uv_b``.  ``render(..., normal_map=)`` copies a new map in.  Every other shading refuses a normal map.

    ``specular_map`` [Ht,Wt,2] (the texture's Ht and Wt) varies a textured Phong view's highlight per texel (the model
    in include/deodr_b200.h): texel (ks_t, e_t) multiplies ``specular`` and ``shininess``, so a map of ones is the view
    without a map.  One more raster samples the map through the view's uv, rendered and back-propagated in the same
    renderer calls as the others (and any shadow maps), and the shading reads it per pixel.  :meth:`backward` adds
    ``specular_map_b`` [Ht,Wt,2] f32 and the map raster's share of ``uv_b`` and of the vertices' gradient.
    ``render(..., specular_map=)`` copies a new map in.  Every other shading refuses a specular map.

    ``shading="pbr_textured"`` shades a textured view per pixel with a metallic-roughness material (a GGX highlight
    coloured by the metal, the model in include/deodr_b200.h): the factors ``metallic`` (default 0) and ``roughness``
    (default 0.5), and an optional ``metallic_roughness_map`` [Ht,Wt,2] = (roughness_t, metallic_t) per texel that
    multiplies them (glTF's factor x texture; its G and B channels).  Every other layer is the textured Phong view's:
    the map's raster takes the specular map's place, and normal maps, environments, point lights and both kinds of
    shadows compose with it.  :meth:`backward` returns ``material_b`` [2] = (metallic_b, roughness_b) in place of
    ``specular_b``, and ``metallic_roughness_map_b`` [Ht,Wt,2] f32 with a map.  ``render(..., metallic_roughness_map=)``
    copies a new map in.  The view refuses ``specular``, ``shininess`` and ``specular_map``; every other shading
    refuses ``metallic``, ``roughness`` and a metallic-roughness map.

    ``camera`` is a :class:`CameraParams`, or a camera vector [26] fp64 tensor on the view's device (extrinsic,
    intrinsic, distortion; ``has_distortion`` says whether its distortion is applied).  A tensor is read at every
    render, so a fit can update it in place between steps without a host read.  ``backward(..., camera_grad=True)``
    and ``render_depth_backward(..., camera_grad=True)`` also return the camera's gradient, ``extrinsic_b`` [3,4],
    ``intrinsic_b`` [3,3] and ``distortion_b`` [5] (None without distortion), fp64 on the device; a Phong view includes
    the share of the camera centre in its specular term.

    ``sh`` adds a second-order spherical-harmonics environment to the light (the model in include/deodr_b200.h): a
    [9] (grey) or [9,C] (coloured, C from 1 to 4) fp64 tensor on the view's device, read at every render, so that a
    fit can update it in place.  Gouraud, Phong and textured Phong views use it, textured Gouraud views a grey one
    only; :meth:`backward` then also
    returns ``sh_b``, shaped like ``sh`` and summed in a fixed order.  Depth and deferred renders ignore it.

    ``point_lights`` adds point lights near the mesh (the model in include/deodr_b200.h): an [L, 3 + S] fp64 tensor on
    the view's device, row j the light's world position then its intensity, grey (S = 1) or one per channel (S = C up
    to 4), L from 1 to 8.  It is read at every render, so a fit can update it in place.  Every shading uses it,
    textured Gouraud views grey lights only; :meth:`backward` then also returns ``point_lights_b``, shaped like the
    table and summed in a fixed order, and a Gouraud view adds the lights' share of the vertex positions into
    ``vertices_b``.  Depth and deferred renders ignore it.

    ``shadow_map_size`` M > 0 makes the point lights cast shadows in a Phong or textured Phong view (the model in
    include/deodr_b200.h): every light gets a cube of six M x M depth maps of the mesh, rendered with the view's sigma
    in map pixels, and each pixel's light terms are multiplied by a soft 2x2 depth test against them,
    ``shadow_bias`` and ``shadow_softness`` (world units, both required) setting where it starts and how wide it is.
    The view's raster(s) and the 6L cube faces are rendered by one renderer call and back-propagated by one, and
    :meth:`backward` adds the shadows' share to ``vertices_b`` (occluders and receivers) and to the lights' positions
    in ``point_lights_b``; the camera's gradient has none (the lookup does not read the camera).  Gouraud views refuse
    shadows: a shadow edge crosses triangles, and per-vertex visibility would smear it over each one.
    :meth:`shadow_maps` returns the last maps.

    ``light_shadow_map_size`` M > 0 makes the directional light cast shadows in a Phong or textured Phong view (the
    model in include/deodr_b200.h): one orthographic M x M depth map of the mesh, seen along the light's direction
    over the window ``light_shadow_bounds`` = (cx, cy, cz, r), with the soft 2x2 test of the cube maps set by
    ``light_shadow_bias`` and ``light_shadow_softness`` (bias, softness and bounds in world units, all required: the
    light has no position, so no default is free of scale).  The directional diffuse and specular terms are
    multiplied by it; receivers outside the bounds' sphere are lit.  The map is rendered and back-propagated in the
    same renderer calls as the view's raster(s) and any cube faces, and :meth:`backward` adds the shadow's share to
    ``vertices_b`` and to the light's direction in ``light_b[0:3]``.  The view needs a directional light, and Gouraud
    views refuse it.  :meth:`light_shadow_map` and :meth:`light_shadow_visibility` return the last map and
    visibility."""

    def __init__(self, faces, nb_vertices: int, camera, height: int, width: int, renderer=None,
                 light_directional=None, ambient: float = 1.0, background_color=(0.0, 0.0, 0.0), sigma: float = 1.0,
                 clockwise: bool = False, device="cuda", slot: int = 0, uv=None, faces_uv=None, texture=None,
                 backface_culling: bool = True, perspective_correct: bool = False, shading: str = "gouraud",
                 specular: Optional[float] = None, shininess: Optional[float] = None, has_distortion: bool = True,
                 sh: Optional[torch.Tensor] = None, point_lights: Optional[torch.Tensor] = None,
                 shadow_map_size: int = 0, shadow_bias: Optional[float] = None,
                 shadow_softness: Optional[float] = None, light_shadow_map_size: int = 0,
                 light_shadow_bias: Optional[float] = None, light_shadow_softness: Optional[float] = None,
                 light_shadow_bounds=None, normal_map=None, specular_map=None, metallic: Optional[float] = None,
                 roughness: Optional[float] = None, metallic_roughness_map=None):
        from .renderer import DeviceScene, default_renderer
        from .scenes import SceneArrays

        nb_colors = len(background_color)
        textured = uv is not None or faces_uv is not None or texture is not None
        if shading not in ("gouraud", "phong", "phong_textured", "pbr_textured"):
            raise ValueError(f"shading must be 'gouraud', 'phong', 'phong_textured' or 'pbr_textured'; got {shading!r}")
        self.pbr = shading == "pbr_textured"
        if self.pbr:
            if not textured:
                raise ValueError("shading='pbr_textured' needs a textured view (uv, faces_uv and texture)")
            if specular is not None or shininess is not None or specular_map is not None:
                raise ValueError("a 'pbr_textured' view takes metallic, roughness and metallic_roughness_map, not the "
                                 "Phong form's specular, shininess or specular_map")
        elif metallic is not None or roughness is not None or metallic_roughness_map is not None:
            raise ValueError("metallic, roughness and metallic_roughness_map need shading='pbr_textured'")
        # the textured per-pixel forms share every layer but the shading kernel
        per_pixel_textured = shading in ("phong_textured", "pbr_textured")
        if shading == "phong" and textured:
            raise ValueError("phong shading of a textured mesh is shading='phong_textured' (its albedo is a raster of "
                             "its own)")
        if shading == "phong_textured" and not textured:
            raise ValueError("shading='phong_textured' needs a textured view (uv, faces_uv and texture); an untextured "
                             "view takes shading='phong'")
        if shading != "gouraud" and perspective_correct:
            raise ValueError("phong shading interpolates linearly in screen space; perspective_correct is refused")
        self.shading = shading
        self.specular = 0.0 if specular is None else float(specular)
        self.shininess = 16.0 if shininess is None else float(shininess)
        self.metallic = 0.0 if metallic is None else float(metallic)
        self.roughness = 0.5 if roughness is None else float(roughness)
        if sh is not None:
            S = _check_sh(sh, torch.device(device))[1]
            if S != 1 and (S != nb_colors or S > 4):
                raise ValueError(f"sh must be [9], or [9,C] with C = {nb_colors} from 1 to 4; got {tuple(sh.shape)}")
            if textured and S != 1 and not per_pixel_textured:
                raise ValueError("a textured view takes a grey environment [9] only: its shade has one channel (or "
                                 "shading='phong_textured')")
        self.sh = sh
        if point_lights is not None:
            S = _check_point_lights(point_lights, torch.device(device))[2]
            if S != 1 and (S != nb_colors or S > 4):
                raise ValueError(f"point lights must be [L, 4], or [L, 3 + C] with C = {nb_colors} from 1 to 4; got "
                                 f"{tuple(point_lights.shape)}")
            if textured and S != 1 and not per_pixel_textured:
                raise ValueError("a textured view takes grey point lights [L, 4] only: its shade has one channel (or "
                                 "shading='phong_textured')")
        self.point_lights = point_lights
        self.shadow_map_size = check_shadow_arguments(shading, point_lights, shadow_map_size, shadow_bias,
                                                      shadow_softness)
        self.shadow_bias = float(shadow_bias) if self.shadow_map_size else None
        self.shadow_softness = float(shadow_softness) if self.shadow_map_size else None
        self.light_shadow_map_size = check_sun_shadow_arguments(shading, light_directional, light_shadow_map_size,
                                                                light_shadow_bias, light_shadow_softness,
                                                                light_shadow_bounds)
        sun = self.light_shadow_map_size
        self.light_shadow_bias = float(light_shadow_bias) if sun else None
        self.light_shadow_softness = float(light_shadow_softness) if sun else None
        self.light_shadow_bounds = tuple(float(b) for b in light_shadow_bounds) if sun else None
        self._sh_scratch, self._sh_key = None, None
        if textured:
            if uv is None or faces_uv is None or texture is None:
                raise ValueError("a textured view needs uv, faces_uv and texture together")
            uv = np.ascontiguousarray(uv, dtype=np.float64)
            faces_uv = np.ascontiguousarray(faces_uv, dtype=np.uint32)
            texture = np.asarray(texture, dtype=np.float64)
            if texture.ndim != 3 or texture.shape[2] != nb_colors:
                raise ValueError(f"texture must be [Ht,Wt,C] with C = len(background_color) = {nb_colors}; "
                                 f"got shape {texture.shape}")
            if uv.ndim != 2 or uv.shape[1] != 2 or faces_uv.shape != np.shape(faces):
                raise ValueError("uv must be [Nuv,2] and faces_uv [T,3] like faces")
        if normal_map is not None:
            if not per_pixel_textured:
                raise ValueError("a normal map perturbs the per-pixel normal of a textured view: it needs "
                                 "shading='phong_textured' or 'pbr_textured'")
            normal_map = np.asarray(normal_map.detach().cpu() if isinstance(normal_map, torch.Tensor) else normal_map,
                                    dtype=np.float64)
            if normal_map.shape != texture.shape[:2] + (3,):
                raise ValueError(f"normal_map must be [Ht,Wt,3] with the texture's Ht and Wt = {texture.shape[:2]}; "
                                 f"got shape {normal_map.shape}")
        self.normal_mapped = normal_map is not None
        if specular_map is not None:
            if shading != "phong_textured":
                raise ValueError("a specular map varies the per-pixel highlight of a textured view: it needs "
                                 "shading='phong_textured'")
            specular_map = np.asarray(specular_map.detach().cpu() if isinstance(specular_map, torch.Tensor)
                                      else specular_map, dtype=np.float64)
            if specular_map.shape != texture.shape[:2] + (2,):
                raise ValueError(f"specular_map must be [Ht,Wt,2] with the texture's Ht and Wt = {texture.shape[:2]}; "
                                 f"got shape {specular_map.shape}")
        self.specular_mapped = specular_map is not None
        if metallic_roughness_map is not None:
            metallic_roughness_map = np.asarray(
                metallic_roughness_map.detach().cpu() if isinstance(metallic_roughness_map, torch.Tensor)
                else metallic_roughness_map, dtype=np.float64)
            if metallic_roughness_map.shape != texture.shape[:2] + (2,):
                raise ValueError(f"metallic_roughness_map must be [Ht,Wt,2] with the texture's Ht and Wt = "
                                 f"{texture.shape[:2]}; got shape {metallic_roughness_map.shape}")
        self.metallic_roughness_mapped = metallic_roughness_map is not None
        # a specular map or a metallic-roughness map: one 2-channel raster beside the albedo (a view has at most one)
        material_map = specular_map if specular_map is not None else metallic_roughness_map
        self._material_mapped = material_map is not None
        self.device = torch.device(device)
        self.topology = MeshTopology(faces, nb_vertices, clockwise=clockwise, device=self.device)
        self.camera, self.sigma = camera, float(sigma)
        if isinstance(camera, torch.Tensor):
            _check_camera_vector(camera, self.device)
            self._camera_distorted = bool(has_distortion)
        else:
            self._camera_distorted = camera.distortion is not None
        self._camera_scratch = None
        self.light_directional, self.ambient = light_directional, float(ambient)
        self.textured, self.perspective_correct = textured, bool(perspective_correct)
        faces_u32 = np.ascontiguousarray(faces, dtype=np.uint32)
        T, V = faces_u32.shape[0], int(nb_vertices)
        flags = np.ones(T, bool) if textured else np.zeros(T, bool)
        # a textured Phong view's scene is its albedo raster: a shade of 1, set here once, over a zero background
        albedo_raster = per_pixel_textured
        background = np.asarray(background_color, dtype=np.float64)
        arrays = SceneArrays(
            faces=faces_u32, faces_uv=faces_uv if textured else np.zeros((T, 3), np.uint32), ij=np.zeros((V, 2)),
            depths=np.ones(V), textured=flags, uv=uv if textured else np.zeros((1, 2)),
            shade=np.ones(V) if albedo_raster else np.zeros(V),
            colors=np.zeros((V, nb_colors)), shaded=flags, edgeflags=np.zeros((T, 3), bool), height=height, width=width,
            nb_colors=nb_colors, texture=texture if textured else np.zeros((2, 2, nb_colors)), background_image=None,
            background_color=np.zeros(nb_colors) if albedo_raster else background, clockwise=clockwise,
            backface_culling=bool(backface_culling), strict_edge=True, perspective_correct=self.perspective_correct,
            integer_pixel_centers=True)
        self.scene = DeviceScene(arrays, self.device)
        # render_deferred's forward pass: the reference's soup scene (:1148-1167) - sigma 0, no silhouette edges,
        # untextured, counter-clockwise, no perspective correction - with one zero colour channel (only its face ids and
        # z-buffer are used).  Its ij / depths are its own, so that a deferred render leaves the view's scene untouched.
        self._deferred_scene = DeviceScene(SceneArrays(
            faces=faces_u32, faces_uv=np.zeros((T, 3), np.uint32), ij=np.zeros((V, 2)), depths=np.ones(V),
            textured=np.zeros(T, bool), uv=np.zeros((1, 2)), shade=np.zeros(V), colors=np.zeros((V, 1)),
            shaded=np.zeros(T, bool), edgeflags=np.zeros((T, 3), bool), height=height, width=width, nb_colors=1,
            texture=np.zeros((2, 2, 1)), background_image=None, background_color=np.zeros(1), clockwise=False,
            backface_culling=bool(backface_culling), strict_edge=True, perspective_correct=False,
            integer_pixel_centers=True), self.device)
        self.renderer = renderer if renderer is not None else default_renderer(self.device.index)
        self._saved = None
        self._saved_depth = None
        if shading != "gouraud":
            from .mesh_fitter import new_scratch

            # the G-buffer scene: [vertex colours | normals | positions | 1] per vertex over a zero background (without
            # the vertex colours for a textured view, whose albedo is its own raster); the coverage column is set here
            # once and never rewritten
            K = (0 if textured else nb_colors) + PHONG_EXTRA_CHANNELS
            colors = np.concatenate((np.zeros((V, K - 1)), np.ones((V, 1))), axis=1)
            if self.normal_mapped:
                # (normals, positions, 1, tangents, bitangents): the coverage stays at column 6
                K = NORMAL_MAP_CHANNELS
                colors = np.concatenate((colors, np.zeros((V, 6))), axis=1)
            self._phong_scene = DeviceScene(SceneArrays(
                faces=faces_u32, faces_uv=np.zeros((T, 3), np.uint32), ij=np.zeros((V, 2)), depths=np.ones(V),
                textured=np.zeros(T, bool), uv=np.zeros((1, 2)), shade=np.zeros(V),
                colors=colors, shaded=np.zeros(T, bool),
                edgeflags=np.zeros((T, 3), bool), height=height, width=width, nb_colors=K,
                texture=np.zeros((2, 2, K)), background_image=None, background_color=np.zeros(K), clockwise=clockwise,
                backface_culling=bool(backface_culling), strict_edge=True, perspective_correct=False,
                integer_pixel_centers=True), self.device)
            self._phong_scratch = new_scratch(self.device)
            self._phong_key = None
            self._phong_background = torch.from_numpy(background.astype(np.float32)).to(self.device)
        if self.normal_mapped:
            # the normal map's raster: the albedo raster's arrays with the map as a 3-channel texture
            self._map_scene = DeviceScene(SceneArrays(
                faces=faces_u32, faces_uv=faces_uv, ij=np.zeros((V, 2)), depths=np.ones(V), textured=flags, uv=uv,
                shade=np.ones(V), colors=np.zeros((V, 3)), shaded=flags, edgeflags=np.zeros((T, 3), bool),
                height=height, width=width, nb_colors=3, texture=normal_map, background_image=None,
                background_color=np.zeros(3), clockwise=clockwise, backface_culling=bool(backface_culling),
                strict_edge=True, perspective_correct=False, integer_pixel_centers=True), self.device)
            self._tangents = VertexTangents(self.topology, faces_uv, uv.shape[0])
        if self._material_mapped:
            # the material map's raster: the albedo raster's arrays with the map as a 2-channel texture
            self._spec_scene = DeviceScene(SceneArrays(
                faces=faces_u32, faces_uv=faces_uv, ij=np.zeros((V, 2)), depths=np.ones(V), textured=flags, uv=uv,
                shade=np.ones(V), colors=np.zeros((V, 2)), shaded=flags, edgeflags=np.zeros((T, 3), bool),
                height=height, width=width, nb_colors=2, texture=material_map, background_image=None,
                background_color=np.zeros(2), clockwise=clockwise, backface_culling=bool(backface_culling),
                strict_edge=True, perspective_correct=False, integer_pixel_centers=True), self.device)
        self._maps = []  # the shadow maps rendered beside the view's raster(s): the cube maps, then the sun map
        if self.shadow_map_size:
            self._cube = ShadowCubes(faces_u32, V, point_lights.shape[0], self.shadow_map_size, clockwise, self.device)
            self._maps.append(self._cube)
        if self.light_shadow_map_size:
            self._sun = SunShadowMap(faces_u32, V, self.light_shadow_map_size, self.light_shadow_bounds, clockwise,
                                     self.device)
            self._maps.append(self._sun)

    def _new_outputs(self, scene) -> dict:
        return self.renderer._new_outputs(scene, False, False, False)

    def shadow_maps(self) -> torch.Tensor:
        """The cube shadow maps [6L, M, M] f32 of the last render (face 6 j + k: light j's +x, -x, +y, -y, +z, -z;
        overwritten by the next render)."""
        if not self.shadow_map_size:
            raise ValueError("this view casts no shadows (shadow_map_size 0)")
        return self._cube.maps

    def shadow_visibility(self) -> torch.Tensor:
        """The lights' visibility [H,W,L] f32 of the last render's pixels (1 where the coverage is 0)."""
        if not self.shadow_map_size:
            raise ValueError("this view casts no shadows (shadow_map_size 0)")
        return self._saved[-2]

    def light_shadow_map(self) -> torch.Tensor:
        """The directional light's shadow map [M, M] f32 of the last render (overwritten by the next render)."""
        if not self.light_shadow_map_size:
            raise ValueError("the directional light casts no shadows in this view (light_shadow_map_size 0)")
        return self._sun.map

    def light_shadow_visibility(self) -> torch.Tensor:
        """The directional light's visibility [H,W] f32 of the last render's pixels (1 where the coverage is 0)."""
        if not self.light_shadow_map_size:
            raise ValueError("the directional light casts no shadows in this view (light_shadow_map_size 0)")
        return self._saved[-1]

    def _render_with_maps(self, scenes: list, vertices: torch.Tensor, params: torch.Tensor) -> list:
        """The view's scenes and every shadow map in one renderer call (one live forward per slot) -> the scenes'
        forward results; the maps keep theirs."""
        if not self._maps:
            return self.renderer.render_views(scenes, self.sigma) if len(scenes) > 1 else \
                [self.renderer.render(scenes[0], self.sigma)]
        if self.shadow_map_size:
            self._cube.prepare(vertices, self.point_lights)
        if self.light_shadow_map_size:
            self._sun.prepare(vertices, params)
        fwds = self.renderer.render_views(scenes + [sc for m in self._maps for sc in m.scenes], self.sigma,
                                          out=[self._new_outputs(sc) for sc in scenes]
                                          + [o for m in self._maps for o in m.outputs()])
        k = len(scenes)
        for m in self._maps:
            m.fwds, k = fwds[k:k + m.NF], k + m.NF
        return fwds[:len(scenes)]

    def _render_b_with_maps(self, scenes: list, fwds: list, image_bs: list, maps_bs: list) -> list:
        """The adjoint of :meth:`_render_with_maps` in one renderer call -> the scenes' gradients."""
        if not self._maps:
            if len(scenes) == 1:
                return [self.renderer.render_b(scenes[0], self.sigma, fwds[0], image_bs[0])]
            return self.renderer.render_b_views(scenes, self.sigma, fwds, image_bs)
        grads = self.renderer.render_b_views(
            scenes + [sc for m in self._maps for sc in m.scenes], self.sigma,
            list(fwds) + [f for m in self._maps for f in m.fwds],
            list(image_bs) + [b for m, mb in zip(self._maps, maps_bs) for b in m.image_bs(mb)],
            [sc.zero_grads() for sc in scenes] + [g for m in self._maps for g in m.grads()])
        return grads[:len(scenes)]

    def _maps_backward(self, vertices: torch.Tensor, params: torch.Tensor, vertices_b: torch.Tensor,
                       params_b: torch.Tensor, lights_b: Optional[torch.Tensor]) -> None:
        """The shadow maps' projection adjoints into vertices_b, the point lights' positions and l = params_b[0:3]."""
        if self.shadow_map_size:
            self._cube.backward(vertices, self.point_lights, vertices_b, lights_b, self._phong_scratch)
        if self.light_shadow_map_size:
            self._sun.backward(vertices, params, vertices_b, params_b, self._phong_scratch)

    def _shade(self, gbuffer: torch.Tensor, params: torch.Tensor, center: torch.Tensor, background: torch.Tensor,
               albedo: Optional[torch.Tensor] = None,
               spec: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """phong_shade of a G-buffer (with the specular map's raster ``spec`` in a view with a map), under the point
        lights' and the directional light's visibility in a view with shadows -> (image, vis or None, sun_vis or
        None)."""
        vis = sun_vis = None
        if self.shadow_map_size:
            vis = shadow_visibility(gbuffer, self.point_lights, self._cube.maps, self.shadow_bias,
                                    self.shadow_softness, albedo=albedo)
        if self.light_shadow_map_size:
            sun_vis = sun_visibility(gbuffer, params, self._sun.map, self.light_shadow_bounds, self.light_shadow_bias,
                                     self.light_shadow_softness, albedo=albedo)
        return phong_shade(gbuffer, params, center, background, sh=self.sh, albedo=albedo,
                           point_lights=self.point_lights, visibility=vis, sun_visibility=sun_vis,
                           specular=spec, brdf="ggx" if self.pbr else "phong"), vis, sun_vis

    def _shade_backward(self, gbuffer, params, center, background, image_b, camera_grad, albedo, vis, sun_vis,
                        spec=None):
        """phong_shade_backward, and in a view with shadows the visibilities' adjoints added into channels_b, lights_b
        and params_b -> (the result of phong_shade_backward without vis_b, sun_vis_b and spec_b, the maps' gradients in
        the order of self._maps, spec_b or None)."""
        shaded = phong_shade_backward(gbuffer, params, center, background, image_b, self._phong_scratch,
                                      center_grad=camera_grad, sh=self.sh, albedo=albedo,
                                      point_lights=self.point_lights, visibility=vis, sun_visibility=sun_vis,
                                      specular=spec, brdf="ggx" if self.pbr else "phong")
        spec_b = None
        if spec is not None:
            shaded, spec_b = shaded[:-1], shaded[-1]
        maps_b = []
        sun_b = None
        if sun_vis is not None:
            shaded, sun_b = shaded[:-1], shaded[-1]
        if vis is not None:
            shaded, vis_b = shaded[:-1], shaded[-1]
            maps_b.append(shadow_visibility_backward(gbuffer, self.point_lights, self._cube.maps, self.shadow_bias,
                                                     self.shadow_softness, vis_b, self._phong_scratch, albedo=albedo,
                                                     channels_b=shaded[0], maps_b=self._cube.zero_maps_b(),
                                                     lights_b=shaded[-1])[1])
        if sun_b is not None:
            maps_b.append(sun_visibility_backward(gbuffer, params, self._sun.map, self.light_shadow_bounds,
                                                  self.light_shadow_bias, self.light_shadow_softness, sun_b,
                                                  self._phong_scratch, albedo=albedo, channels_b=shaded[0],
                                                  map_b=self._sun.zero_maps_b()[0], light_b=shaded[1])[1][None])
        return shaded, maps_b, spec_b

    def _phong_params(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """(params [6], camera_center [3]) fp64 on the device, uploaded again only when the light, the specular (or
        metallic-roughness) parameters or the camera have changed since the last render (so that a render normally
        copies nothing)."""
        l = (0.0, 0.0, 0.0) if self.light_directional is None else \
            tuple(np.asarray(self.light_directional, dtype=np.float64).reshape(3).tolist())
        material = (self.metallic, self.roughness) if self.pbr else (self.specular, self.shininess)
        params = l + (float(self.ambient), float(material[0]), float(material[1]))
        if isinstance(self.camera, torch.Tensor):
            if self._phong_key != params:
                self._phong_key = params
                self._phong_params_t = torch.tensor(params, dtype=torch.float64).to(self.device, non_blocking=True)
            return self._phong_params_t, camera_center_of(self.camera)
        center = tuple(camera_center(self.camera).tolist())
        if self._phong_key != params + center:
            self._phong_key = params + center
            self._phong_params_t = torch.tensor(params, dtype=torch.float64).to(self.device, non_blocking=True)
            self._phong_center_t = torch.tensor(center, dtype=torch.float64).to(self.device, non_blocking=True)
        return self._phong_params_t, self._phong_center_t

    def _sh_light(self) -> torch.Tensor:
        """The light [4] fp64 on the device = (directional (0 without one), ambient), uploaded again only when it has
        changed since the last render."""
        l = (0.0, 0.0, 0.0) if self.light_directional is None else \
            tuple(np.asarray(self.light_directional, dtype=np.float64).reshape(3).tolist())
        key = l + (float(self.ambient),)
        if self._sh_key != key:
            self._sh_key = key
            self._sh_light_t = torch.tensor(key, dtype=torch.float64).to(self.device, non_blocking=True)
        return self._sh_light_t

    def _sh_backward(self, normals: torch.Tensor, vertex_colors: Optional[torch.Tensor], colors_b: torch.Tensor):
        if self._sh_scratch is None:
            from .mesh_fitter import new_scratch

            self._sh_scratch = new_scratch(self.device)
        return sh_lit_vertex_colors_backward(normals, vertex_colors, self._sh_light(), self.sh, colors_b,
                                             self._sh_scratch, self.light_directional is not None)

    def _project(self, vertices: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        if isinstance(self.camera, torch.Tensor):
            return project_points_dev(vertices, self.camera, self._camera_distorted)
        return project_points(vertices, self.camera)

    def _project_backward(self, vertices: torch.Tensor, ij_b: torch.Tensor, depths_b: Optional[torch.Tensor],
                          out: Optional[torch.Tensor], reference_transpose: bool,
                          camera_grad: bool) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """The projection's adjoint accumulated into ``out`` (created zeroed if None) -> (out, camera_b [26] or None).
        A tensor camera, or ``camera_grad``, takes the fused adjoint of the device camera."""
        if camera_grad and (reference_transpose or self.perspective_correct):
            raise ValueError("camera_grad is the true adjoint: it refuses reference_transpose and perspective_correct")
        if not camera_grad and not isinstance(self.camera, torch.Tensor):
            return project_points_backward(vertices, self.camera, ij_b, depths_b=depths_b, out=out,
                                           reference_transpose=reference_transpose), None
        if reference_transpose:
            raise ValueError("reference_transpose needs a CameraParams camera (a camera vector takes the true adjoint)")
        if out is None:
            out = torch.zeros((vertices.shape[0], 3), dtype=torch.float64, device=self.device)
        if self._camera_scratch is None:
            from .mesh_fitter import new_scratch

            self._camera_scratch = new_scratch(self.device)
        camera = self.camera if isinstance(self.camera, torch.Tensor) else self.camera.device_vector(self.device)
        camera_b = project_points_camera_backward(vertices, camera, self._camera_distorted,
                                                  ij_b.to(self.device, torch.float32), depths_b, self._camera_scratch,
                                                  points_b=out, accumulate=True)
        return out, camera_b

    def _camera_result(self, camera_b: torch.Tensor,
                       center_b: Optional[torch.Tensor] = None) -> Dict[str, Optional[torch.Tensor]]:
        camera = self.camera if isinstance(self.camera, torch.Tensor) else self.camera.device_vector(self.device)
        return camera_gradients(camera, camera_b, self._camera_distorted, center_b)

    def render(self, vertices: torch.Tensor, vertex_colors: Optional[torch.Tensor] = None,
               texture: Optional[torch.Tensor] = None, normal_map: Optional[torch.Tensor] = None,
               specular_map: Optional[torch.Tensor] = None,
               metallic_roughness_map: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The image [H,W,C] f32 of the mesh at ``vertices`` [V,3]: Gouraud-lit ``vertex_colors`` [V,C] for an untextured
        view; for a textured one the texture shaded by the vertex luminosity, with ``texture`` [Ht,Wt,C] (if given)
        copied into the view's texture first, so that a fit can vary it.  ``normal_map`` [Ht,Wt,3], in a view made with
        one, is copied into the view's normal map in the same way, ``specular_map`` [Ht,Wt,2] into its specular
        map and ``metallic_roughness_map`` [Ht,Wt,2] into its metallic-roughness map."""
        if normal_map is not None:
            if not self.normal_mapped:
                raise ValueError("this view has no normal map (DeviceMeshView(..., normal_map=) makes one)")
            if tuple(normal_map.shape) != tuple(self._map_scene.t["texture"].shape):
                raise ValueError(f"normal_map has shape {tuple(normal_map.shape)}, expected "
                                 f"{tuple(self._map_scene.t['texture'].shape)}")
            self._map_scene.t["texture"].copy_(normal_map)
        if specular_map is not None:
            if not self.specular_mapped:
                raise ValueError("this view has no specular map (DeviceMeshView(..., specular_map=) makes one)")
            if tuple(specular_map.shape) != tuple(self._spec_scene.t["texture"].shape):
                raise ValueError(f"specular_map has shape {tuple(specular_map.shape)}, expected "
                                 f"{tuple(self._spec_scene.t['texture'].shape)}")
            self._spec_scene.t["texture"].copy_(specular_map)
        if metallic_roughness_map is not None:
            if not self.metallic_roughness_mapped:
                raise ValueError("this view has no metallic-roughness map (DeviceMeshView(..., "
                                 "metallic_roughness_map=) makes one)")
            if tuple(metallic_roughness_map.shape) != tuple(self._spec_scene.t["texture"].shape):
                raise ValueError(f"metallic_roughness_map has shape {tuple(metallic_roughness_map.shape)}, expected "
                                 f"{tuple(self._spec_scene.t['texture'].shape)}")
            self._spec_scene.t["texture"].copy_(metallic_roughness_map)
        if self.textured:
            if vertex_colors is not None:
                raise ValueError("a textured view takes no vertex_colors (its colour is the shaded texture)")
            if self.shading in ("phong_textured", "pbr_textured"):
                return self._render_phong_textured(vertices, texture)
            return self._render_textured(vertices, texture)
        if vertex_colors is None:
            raise ValueError("an untextured view needs vertex_colors")
        if texture is not None:
            raise ValueError("an untextured view takes no texture")
        if self.shading == "phong":
            return self._render_phong(vertices, vertex_colors)
        vertices = _f64(vertices, self.device)
        _, normals = self.topology.vertex_normals(vertices)
        if self.point_lights is not None:
            colors = point_lit_vertex_colors(normals, vertices, vertex_colors, self._sh_light(), self.point_lights,
                                             sh=self.sh, directional=self.light_directional is not None)
        elif self.sh is None:
            _, colors = vertex_luminosity(normals, vertex_colors, self.light_directional, self.ambient)
        else:
            colors = sh_lit_vertex_colors(normals, vertex_colors, self._sh_light(), self.sh,
                                          self.light_directional is not None)
        ij, depths = self._project(vertices)
        t = self.scene.t
        t["ij"].copy_(ij)
        t["depths"].copy_(depths)
        t["colors"].copy_(colors)
        self.topology.edge_on_silhouette(ij, out=t["edgeflags"])
        fwd = self.renderer.render(self.scene, self.sigma)
        self._saved = (vertices, _f64(vertex_colors, self.device), normals, fwd)
        return fwd["image"]

    def _render_phong(self, vertices: torch.Tensor, vertex_colors: torch.Tensor) -> torch.Tensor:
        nc = self.scene.nb_colors
        vertices, vertex_colors = _f64(vertices, self.device), _f64(vertex_colors, self.device)
        if tuple(vertex_colors.shape) != (self.topology.nb_vertices, nc):
            raise ValueError(f"vertex_colors has shape {tuple(vertex_colors.shape)}, "
                             f"expected {(self.topology.nb_vertices, nc)}")
        _, normals = self.topology.vertex_normals(vertices)
        ij, depths = self._project(vertices)
        t = self._phong_scene.t
        t["ij"].copy_(ij)
        t["depths"].copy_(depths)
        t["colors"][:, :nc].copy_(vertex_colors)
        t["colors"][:, nc:nc + 3].copy_(normals)
        t["colors"][:, nc + 3:nc + 6].copy_(vertices)
        self.topology.edge_on_silhouette(ij, out=t["edgeflags"])
        params, center = self._phong_params()
        fwd = self._render_with_maps([self._phong_scene], vertices, params)[0]
        image, vis, sun_vis = self._shade(fwd["image"], params, center, self.scene.t["background_color"])
        self._saved = (vertices, vertex_colors, normals, fwd, params, center, vis, sun_vis)
        return image

    def _backward_phong(self, image_b: torch.Tensor, reference_transpose: bool,
                        camera_grad: bool) -> Dict[str, torch.Tensor]:
        # phong_shade_b -> channels_b; raster adjoint -> colors_b [V,K], ij_b; the albedo slice is vertex_colors_b, the
        # normal slice goes through the normal adjoint, the position slice adds to vertices_b, ij_b through the
        # projection's adjoint
        vertices, _, _, fwd, params, center, vis, sun_vis = self._saved
        nc = self.scene.nb_colors
        shaded, maps_b, _ = self._shade_backward(fwd["image"], params, center, self.scene.t["background_color"],
                                                 image_b, camera_grad, None, vis, sun_vis)
        lights_b = None
        if self.point_lights is not None:
            shaded, lights_b = shaded[:-1], shaded[-1]
        channels_b, params_b = shaded[:2]
        grads = self._render_b_with_maps([self._phong_scene], [fwd], [channels_b], maps_b)[0]
        colors_b = grads["colors_b"]
        vertices_b = self.topology.vertex_normals_backward(vertices, colors_b[:, nc:nc + 3])
        vertices_b += colors_b[:, nc + 3:nc + 6]
        self._maps_backward(vertices, params, vertices_b, params_b, lights_b)
        _, camera_b = self._project_backward(vertices, grads["ij_b"], None, vertices_b, reference_transpose,
                                             camera_grad)
        out = {"vertices_b": vertices_b, "vertex_colors_b": colors_b[:, :nc].to(torch.float64),
               "light_b": params_b[:4], "specular_b": params_b[4:]}
        if camera_grad:
            out.update(self._camera_result(camera_b, shaded[2]))
        if self.sh is not None:
            out["sh_b"] = shaded[-1]
        if lights_b is not None:
            out["point_lights_b"] = lights_b
        return out

    def _set_texture(self, texture: Optional[torch.Tensor]) -> None:
        t = self.scene.t
        if texture is not None:
            if tuple(texture.shape) != tuple(t["texture"].shape):
                raise ValueError(f"texture has shape {tuple(texture.shape)}, expected {tuple(t['texture'].shape)}")
            t["texture"].copy_(texture)

    def _render_phong_textured(self, vertices: torch.Tensor, texture: Optional[torch.Tensor]) -> torch.Tensor:
        # the albedo raster (self.scene, shade 1) and the 7-channel G-buffer share ij, depths and edge flags; both are
        # rendered by one library call, so the second overlaps the first and the verdict is read once
        self._set_texture(texture)
        vertices = _f64(vertices, self.device)
        _, normals = self.topology.vertex_normals(vertices)
        ij, depths = self._project(vertices)
        a, g = self.scene.t, self._phong_scene.t
        for t in (a, g):
            t["ij"].copy_(ij)
            t["depths"].copy_(depths)
        g["colors"][:, 0:3].copy_(normals)
        g["colors"][:, 3:6].copy_(vertices)
        self.topology.edge_on_silhouette(ij, out=a["edgeflags"])
        g["edgeflags"].copy_(a["edgeflags"])
        scenes = [self.scene, self._phong_scene]
        if self.normal_mapped:
            # the G-buffer's tangent and bitangent columns, and the map's raster, which shares the geometry
            g["colors"][:, 7:13].copy_(self._tangents.frames(vertices, a["uv"]))
            m = self._map_scene.t
            m["ij"].copy_(ij)
            m["depths"].copy_(depths)
            m["edgeflags"].copy_(a["edgeflags"])
            scenes.append(self._map_scene)
        if self._material_mapped:
            # the material map's raster (specular or metallic-roughness), last, which shares the geometry too
            s = self._spec_scene.t
            s["ij"].copy_(ij)
            s["depths"].copy_(depths)
            s["edgeflags"].copy_(a["edgeflags"])
            scenes.append(self._spec_scene)
        params, center = self._phong_params()
        fwds = self._render_with_maps(scenes, vertices, params)
        gbuffer = normal_map(fwds[1]["image"], fwds[2]["image"]) if self.normal_mapped else fwds[1]["image"]
        spec = fwds[-1]["image"] if self._material_mapped else None
        image, vis, sun_vis = self._shade(gbuffer, params, center, self._phong_background, albedo=fwds[0]["image"],
                                          spec=spec)
        self._gbuffer = gbuffer
        self._saved = (vertices, None, normals, fwds, params, center, vis, sun_vis)
        return image

    def _backward_phong_textured(self, image_b: torch.Tensor, reference_transpose: bool,
                                 camera_grad: bool) -> Dict[str, torch.Tensor]:
        # the shading's adjoint -> albedo_b, channels_b; one adjoint call over both rasters -> texture_b, uv_b and the
        # G-buffer's colors_b (normal slice through the normal adjoint, position slice into vertices_b); the two ij_b
        # are summed before the projection's adjoint.  The albedo raster's shade_b is not used: its shade is constant
        # with a normal map, the perturbation's adjoint first takes the 7-channel channels_b to the 13-channel
        # G-buffer's and the map raster's image gradients; the three rasters' adjoint is one call, the tangent slices
        # of colors_b go through the tangent frame's adjoint into vertices_b and uv_b, and the ij_b and uv_b summed.
        # A material map's raster (specular or metallic-roughness), last, takes the shading's spec_b in the same
        # adjoint call; its ij_b and uv_b are summed in too
        vertices, _, _, fwds, params, center, vis, sun_vis = self._saved
        spec = fwds[-1]["image"] if self._material_mapped else None
        shaded, maps_b, spec_b = self._shade_backward(self._gbuffer, params, center, self._phong_background, image_b,
                                                      camera_grad, fwds[0]["image"], vis, sun_vis, spec)
        lights_b = None
        if self.point_lights is not None:
            shaded, lights_b = shaded[:-1], shaded[-1]
        channels_b, params_b, albedo_b = shaded[0], shaded[1], shaded[-1]
        scenes, image_bs = [self.scene, self._phong_scene], [albedo_b, channels_b]
        if self.normal_mapped:
            image_bs[1], map_image_b = normal_map_backward(fwds[1]["image"], fwds[2]["image"], channels_b)
            scenes.append(self._map_scene)
            image_bs.append(map_image_b)
        if self._material_mapped:
            scenes.append(self._spec_scene)
            image_bs.append(spec_b)
        grads = self._render_b_with_maps(scenes, fwds, image_bs, maps_b)
        ga, gg = grads[:2]
        colors_b = gg["colors_b"]
        vertices_b = self.topology.vertex_normals_backward(vertices, colors_b[:, 0:3])
        vertices_b += colors_b[:, 3:6]
        uv_b = ga["uv_b"]
        if self.normal_mapped:
            _, tangent_uv_b = self._tangents.backward(vertices, self.scene.t["uv"], colors_b[:, 7:13], vertices_b)
            uv_b = (uv_b + grads[2]["uv_b"]) + tangent_uv_b.to(uv_b.dtype)
        ij_b = ga["ij_b"] + gg["ij_b"]
        if self.normal_mapped:
            ij_b = ij_b + grads[2]["ij_b"]
        if self._material_mapped:
            ij_b = ij_b + grads[-1]["ij_b"]
            uv_b = uv_b + grads[-1]["uv_b"]
        self._maps_backward(vertices, params, vertices_b, params_b, lights_b)
        _, camera_b = self._project_backward(vertices, ij_b, None, vertices_b, reference_transpose, camera_grad)
        out = {"vertices_b": vertices_b, "texture_b": ga["texture_b"], "uv_b": uv_b, "light_b": params_b[:4],
               "material_b" if self.pbr else "specular_b": params_b[4:]}
        if self.normal_mapped:
            out["normal_map_b"] = grads[2]["texture_b"]
        if self._material_mapped:
            out["metallic_roughness_map_b" if self.pbr else "specular_map_b"] = grads[-1]["texture_b"]
        if camera_grad:
            out.update(self._camera_result(camera_b, shaded[2]))
        if self.sh is not None:
            out["sh_b"] = shaded[-2]
        if lights_b is not None:
            out["point_lights_b"] = lights_b
        return out

    def _render_textured(self, vertices: torch.Tensor, texture: Optional[torch.Tensor]) -> torch.Tensor:
        # Scene3D.render with mesh.uv (:921-930): textured = shaded = 1, shade = the vertex luminosity, colours zero
        t = self.scene.t
        self._set_texture(texture)
        vertices = _f64(vertices, self.device)
        _, normals = self.topology.vertex_normals(vertices)
        if self.point_lights is not None:
            lum = point_lit_vertex_colors(normals, vertices, None, self._sh_light(), self.point_lights, sh=self.sh,
                                          directional=self.light_directional is not None)
        elif self.sh is None:
            lum, _ = vertex_luminosity(normals, None, self.light_directional, self.ambient)
        else:
            lum = sh_lit_vertex_colors(normals, None, self._sh_light(), self.sh, self.light_directional is not None)
        ij, depths = self._project(vertices)
        t["ij"].copy_(ij)
        t["depths"].copy_(depths)
        t["shade"].copy_(lum)
        self.topology.edge_on_silhouette(ij, out=t["edgeflags"])
        fwd = self.renderer.render(self.scene, self.sigma)
        self._saved = (vertices, None, normals, fwd)
        return fwd["image"]

    def backward(self, image_b: torch.Tensor, reference_transpose: bool = False,
                 camera_grad: bool = False) -> Dict[str, torch.Tensor]:
        """-> dict(vertices_b [V,3] f64, vertex_colors_b [V,C] f64, light_b [4] f64), plus specular_b [2] f64 = (ks_b,
        e_b) for a Phong view, sh_b for a view with an environment and point_lights_b for a view with point lights;
        for a textured view
        dict(vertices_b, texture_b [Ht,Wt,C] f32, uv_b [Nuv,2] f32, light_b), plus specular_b for a textured Phong
        view (and normal_map_b [Ht,Wt,3] f32 for a normal-mapped one, specular_map_b [Ht,Wt,2] f32 for one with a
        specular map): the luminosity's adjoint ``shade_b`` goes
        through the luminosity and normal adjoints, ``ij_b`` through the projection's.  With ``camera_grad`` the dict
        also holds extrinsic_b, intrinsic_b and distortion_b (see the class); it refuses ``reference_transpose``."""
        if camera_grad and reference_transpose:
            raise ValueError("camera_grad is the true adjoint: it refuses reference_transpose and perspective_correct")
        if self.perspective_correct:
            raise ValueError("perspective_correct has no adjoint (as in the reference, Scene3D.render_backward)")
        if self.shading == "phong":
            return self._backward_phong(image_b, reference_transpose, camera_grad)
        if self.shading in ("phong_textured", "pbr_textured"):
            return self._backward_phong_textured(image_b, reference_transpose, camera_grad)
        vertices, vertex_colors, normals, fwd = self._saved
        grads = self.renderer.render_b(self.scene, self.sigma, fwd, image_b)
        positions_b = None
        if self.point_lights is not None:
            if self._sh_scratch is None:
                from .mesh_fitter import new_scratch

                self._sh_scratch = new_scratch(self.device)
            nb, positions_b, vcb, lb, sh_b, lights_b = point_lit_vertex_colors_backward(
                normals, vertices, None if self.textured else vertex_colors, self._sh_light(), self.point_lights,
                grads["shade_b"] if self.textured else grads["colors_b"], self._sh_scratch, sh=self.sh,
                directional=self.light_directional is not None)
            lum = {"normals_b": nb, "vertex_colors_b": vcb, "light_b": lb}
        elif self.sh is not None:
            nb, vcb, lb, sh_b = self._sh_backward(normals, None if self.textured else vertex_colors,
                                                  grads["shade_b"] if self.textured else grads["colors_b"])
            lum = {"normals_b": nb, "vertex_colors_b": vcb, "light_b": lb}
        elif self.textured:
            lum = vertex_luminosity_backward(normals, None, self.light_directional, self.ambient,
                                             luminosity_b=grads["shade_b"])
        else:
            lum = vertex_luminosity_backward(normals, vertex_colors, self.light_directional, self.ambient,
                                             colors_b=grads["colors_b"])
        vertices_b = self.topology.vertex_normals_backward(vertices, lum["normals_b"])
        if positions_b is not None:
            vertices_b += positions_b
        _, camera_b = self._project_backward(vertices, grads["ij_b"], None, vertices_b, reference_transpose,
                                             camera_grad)
        if self.textured:
            out = {"vertices_b": vertices_b, "texture_b": grads["texture_b"], "uv_b": grads["uv_b"],
                   "light_b": lum["light_b"]}
        else:
            out = {"vertices_b": vertices_b, "vertex_colors_b": lum["vertex_colors_b"], "light_b": lum["light_b"]}
        if camera_grad:
            out.update(self._camera_result(camera_b))
        if self.sh is not None:
            out["sh_b"] = sh_b
        if self.point_lights is not None:
            out["point_lights_b"] = lights_b
        return out

    def render_deferred(self, vertices: torch.Tensor, vertex_colors: Optional[torch.Tensor] = None,
                        depth_scale: float = 1.0, color: bool = True, depth: bool = True, face_id: bool = True,
                        barycentric: bool = True, normal: bool = True, luminosity: bool = True, uv: bool = True,
                        xyz: bool = True) -> Dict[str, torch.Tensor]:
        """``Scene3D.render_deferred`` (deodr/differentiable_renderer.py:1053-1174): per-pixel channels of the mesh at
        ``vertices``, as fp32 [H,W,k] CUDA tensors that are views into one [H,W,K] buffer, under the reference's keys in
        its order: depth (x ``depth_scale``), face_id, barycentric, normal, luminosity, xyz, then color (unlit
        ``vertex_colors``, all C channels; untextured views) or uv (textured views).  The background is 0 in every
        channel but depth, where it is the largest vertex depth, unscaled; face_id is 0 there too, as is face 0, so the
        result also holds ``"face_index"``: the int32 face-id map with -1 at the background.

        One forward pass of the mesh at sigma 0 gives the face ids, then one gather kernel interpolates the attributes
        of each pixel's face (csrc/deferred.cu).  The view's sigma must be 0, as the reference requires.  The call
        reuses the renderer's slot: a :meth:`render` before it must be rendered again before :meth:`backward`."""
        if self.sigma != 0:
            raise ValueError("render_deferred needs a view with sigma == 0 (no antialiasing), as the reference")
        if self.textured and vertex_colors is not None:
            raise ValueError("a textured view takes no vertex_colors")
        want_color = color and not self.textured
        if want_color and vertex_colors is None:
            raise ValueError("color=True on an untextured view needs vertex_colors")
        want_uv = uv and self.textured
        C_ = self.scene.nb_colors
        if want_color and tuple(vertex_colors.shape) != (self.topology.nb_vertices, C_):
            raise ValueError(f"vertex_colors has shape {tuple(vertex_colors.shape)}, "
                             f"expected {(self.topology.nb_vertices, C_)}")
        layout = [(name, n) for name, n, on in (
            ("depth", 1, depth), ("face_id", 1, face_id), ("barycentric", 3, barycentric), ("normal", 3, normal),
            ("luminosity", 1, luminosity), ("xyz", 3, xyz), ("color", C_, want_color), ("uv", 2, want_uv)) if on]
        vertices = _f64(vertices, self.device)
        ij, depths = self._project(vertices)
        ds = self._deferred_scene
        ds.t["ij"].copy_(ij)
        ds.t["depths"].copy_(depths)
        fwd = self.renderer.render(ds, 0.0, face_id=True)
        H, W = ds.height, ds.width
        K = sum(n for _, n in layout)
        out = torch.empty((H, W, max(K, 1)), dtype=torch.float32, device=self.device)
        io = _cabi.DeferredIO()
        io.face_index = fwd["face_id"].data_ptr()
        io.out, io.K, io.depth_scale, io.background, io.nb_color = out.data_ptr(), max(K, 1), float(depth_scale), 0.0, C_
        keep = [vertices, depths]
        offsets, off = {}, 0
        for name, n in layout:
            offsets[name] = off
            off += n
        for name in ("depth", "face_id", "barycentric", "normal", "luminosity", "xyz", "uv", "color"):
            setattr(io, "off_" + name, offsets.get(name, -1))
        if depth:
            depth_background = depths.max()
            keep.append(depth_background)
            io.depth, io.depth_background = depths.data_ptr(), depth_background.data_ptr()
        if normal or luminosity:
            _, normals = self.topology.vertex_normals(vertices)
            keep.append(normals)
            if normal:
                io.normal = normals.data_ptr()
            if luminosity:
                lum, _ = vertex_luminosity(normals, None, self.light_directional, self.ambient)
                keep.append(lum)
                io.luminosity = lum.data_ptr()
        if xyz:
            io.xyz = vertices.data_ptr()
        if want_color:
            vc = _f64(vertex_colors, self.device)
            keep.append(vc)
            io.color = vc.data_ptr()
        view = ds.view()
        if want_uv:
            view.faces_uv = self.scene.t["faces_uv"].data_ptr()
            view.nb_uv = self.scene.t["uv"].shape[0]
            io.uv = self.scene.t["uv"].data_ptr()
        if K > 0:
            _cabi.check(_cabi.load().deodr_b200_render_deferred_channels(C.byref(view), C.byref(io),
                                                                         _stream(self.device)))
        del keep
        result = {name: out[:, :, offsets[name]:offsets[name] + n] for name, n in layout}
        result["face_index"] = fwd["face_id"]
        return result

    def render_depth(self, vertices: torch.Tensor, depth_scale: float = 1.0) -> torch.Tensor:
        """``Scene3D.render_depth`` (deodr/differentiable_renderer.py:1001-1037): a one-channel render [H,W,1] f32 whose
        colour is the vertex depth times ``depth_scale``, over the view's background colour (which must have exactly
        one entry)."""
        if self.scene.nb_colors != 1:
            raise ValueError(f"render_depth needs a one-entry background colour; this view has {self.scene.nb_colors}")
        if self.textured:
            raise ValueError("render_depth renders the colour scene of an untextured view; this view is textured")
        vertices = _f64(vertices, self.device)
        ij, depths = self._project(vertices)
        t = self.scene.t
        t["ij"].copy_(ij)
        t["depths"].copy_(depths)
        t["colors"].copy_((depths * float(depth_scale))[:, None])
        self.topology.edge_on_silhouette(ij, out=t["edgeflags"])
        fwd = self.renderer.render(self.scene, self.sigma)
        self._saved_depth = (vertices, float(depth_scale), fwd)
        return fwd["image"]

    def render_depth_backward(self, depth_b: torch.Tensor, reference_transpose: bool = False,
                              camera_grad: bool = False):
        """``Scene3D.render_depth_backward`` (:1039-1051) from ``depth_b`` [H,W,1] -> vertices_b [V,3] f64: the raster
        adjoint gives ij_b and colors_b, and depths_b = colors_b * depth_scale.  With ``camera_grad``: dict(vertices_b,
        extrinsic_b, intrinsic_b, distortion_b)."""
        if camera_grad and reference_transpose:
            raise ValueError("camera_grad is the true adjoint: it refuses reference_transpose and perspective_correct")
        if self.perspective_correct:
            raise ValueError("perspective_correct has no adjoint (as in the reference, Scene3D.render_depth_backward)")
        vertices, depth_scale, fwd = self._saved_depth
        grads = self.renderer.render_b(self.scene, self.sigma, fwd, depth_b)
        depths_b = grads["colors_b"][:, 0].to(torch.float64) * depth_scale
        vertices_b, camera_b = self._project_backward(vertices, grads["ij_b"], depths_b, None, reference_transpose,
                                                      camera_grad)
        if not camera_grad:
            return vertices_b
        return {"vertices_b": vertices_b, **self._camera_result(camera_b)}
