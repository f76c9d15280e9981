"""Mesh fitting on the device: ``MeshDepthFitter``, ``MeshRGBFitterWithPose`` and
``MeshRGBFitterWithPoseMultiFrame`` of the reference (deodr/mesh_fitter.py) with their state in CUDA tensors, and
``DeviceLaplacianRigidEnergy`` (deodr/laplacian_rigid_energy.py).

A step centres the vertices, applies the rigid pose, renders (depth or colour), compares with the observation,
back-propagates through the render and the pose, adds the gradient of the Laplacian rigidity energy and takes clamped
heavy-ball steps - every part on the GPU: the renderer and the scene ops (mesh_ops.py), and for the fitter's own maths
the kernels of csrc/fitter.cu (include/deodr_b200.h, "mesh fitting").  Nothing is read back to the host inside
``step()`` apart from the renderer's own verdict (and, with ``cself > 0``, the self-collision's); its energy is a 0-d
fp64 CUDA tensor.  With ``cself > 0`` the step adds ``DeviceSelfCollisionEnergy`` of the un-posed vertices to the
rigidity's gradient and energy; ``energy_self_collision`` holds its energy.

``MeshDepthFitter`` and ``MeshRGBFitterWithPose`` also take ``skeleton``: a ``LinearBlendSkinning`` (or its four
arrays), whose joint rotations [J,3] are fitted with the rest.  The step then skins the vertices before the rigid pose,
evaluates the self-collision at the skinned vertices (where joints bend, distances change), back-propagates through the
skinning to the rest vertices and the rotations, and keeps the Laplacian rigidity on the rest vertices.
"""

from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Tuple

import numpy as np
import torch

from . import _cabi
from .mesh_ops import (CameraParams, DeviceMeshView, LinearBlendSkinning, MeshTopology, _f64, _stream,
                       project_points, project_points_backward, topology_arrays)


def _ptr(t: Optional[torch.Tensor]):
    return t.data_ptr() if t is not None else None


def new_scratch(device) -> torch.Tensor:
    """A zeroed scratch buffer of the fitting entry points (``deodr_b200_fitter_scratch_bytes`` bytes)."""
    n = (int(_cabi.load().deodr_b200_fitter_scratch_bytes()) + 7) // 8
    return torch.zeros((n,), dtype=torch.float64, device=device)


def euler_to_quaternion(euler) -> np.ndarray:
    """(x, y, z, w) of ``scipy.spatial.transform.Rotation.from_euler("zyx", euler)``, as the reference's fitters."""
    from scipy.spatial.transform import Rotation

    return Rotation.from_euler("zyx", np.asarray(euler, dtype=np.float64)).as_quat()


def edge_neighbours(faces, nb_vertices: int) -> Tuple[np.ndarray, np.ndarray]:
    """Neighbour CSR (offset [V+1], index) int32 of the "shares a face" adjacency, itself excluded, neighbours
    ascending: the matrix A of the Laplacian L = D - A, and the one-ring of the self-collision exclusion."""
    arr = topology_arrays(faces, nb_vertices)
    V = arr["nb_vertices"]
    faces = np.asarray(arr["faces"]).view(np.uint32).astype(np.int64)
    a = np.concatenate((faces[:, 0], faces[:, 1], faces[:, 2]))
    b = np.concatenate((faces[:, 1], faces[:, 2], faces[:, 0]))
    first = np.zeros(arr["nb_edges"], dtype=np.int64)
    first[arr["faces_edges"].T.reshape(-1)] = np.arange(a.size)  # one occurrence of every unique edge
    ea, eb = a[first], b[first]
    keep = ea != eb  # a degenerate face's edge from a vertex to itself is no adjacency
    rows = np.concatenate((ea[keep], eb[keep]))
    cols = np.concatenate((eb[keep], ea[keep]))
    order = np.lexsort((cols, rows))
    rows, cols = rows[order], cols[order]
    offset = np.zeros(V + 1, dtype=np.int32)
    np.cumsum(np.bincount(rows, minlength=V), out=offset[1:])
    return offset, cols.astype(np.int32)


def laplacian_neighbours(faces, nb_vertices: int) -> Tuple[np.ndarray, np.ndarray]:
    """:func:`edge_neighbours`, for a mesh of one connected component: raises ValueError for more (a vertex in no face
    is a component of its own), where the rigidity energy leaves a component free to drift."""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import connected_components

    offset, index = edge_neighbours(faces, nb_vertices)
    V = offset.size - 1
    adjacency = csr_matrix((np.ones(index.size), index, offset), shape=(V, V))
    n_components, _ = connected_components(adjacency, directed=False)
    if n_components > 1:
        raise ValueError(f"the mesh has {n_components} connected components; the Laplacian rigidity energy needs one")
    return offset, index


# ---- thin wrappers over the C-ABI (device tensors in, device tensors out; no host read) ------------------------------


def pose(vertices: torch.Tensor, quaternion: torch.Tensor, translation: torch.Tensor, scratch: torch.Tensor,
         out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Centres ``vertices`` [V,3] f64 in place and returns qrot(q / |q|, vertices) + translation (deodr_b200_pose)."""
    if out is None:
        out = torch.empty_like(vertices)
    _cabi.check(_cabi.load().deodr_b200_pose(vertices.data_ptr(), vertices.shape[0], quaternion.data_ptr(),
                                             translation.data_ptr(), out.data_ptr(), scratch.data_ptr(),
                                             _stream(vertices.device)))
    return out


def pose_backward(vertices: torch.Tensor, quaternion: torch.Tensor, transformed_b: torch.Tensor, scratch: torch.Tensor,
                  out: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None):
    """-> (vertices_b [V,3] centred, quaternion_b [4], translation_b [3]), f64 (deodr_b200_pose_b)."""
    dev = vertices.device
    if out is None:
        out = (torch.empty_like(vertices), torch.empty((4,), dtype=torch.float64, device=dev),
               torch.empty((3,), dtype=torch.float64, device=dev))
    v_b, q_b, t_b = out
    _cabi.check(_cabi.load().deodr_b200_pose_b(vertices.data_ptr(), vertices.shape[0], quaternion.data_ptr(),
                                               transformed_b.data_ptr(), v_b.data_ptr(), q_b.data_ptr(), t_b.data_ptr(),
                                               scratch.data_ptr(), _stream(dev)))
    return v_b, q_b, t_b


def pose_frames(vertices: torch.Tensor, quaternions: torch.Tensor, translations: torch.Tensor, scratch: torch.Tensor,
                out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Centres ``vertices`` [V,3] f64 in place and returns transformed [F,V,3] with transformed[f] =
    qrot(q_f / |q_f|, vertices) + t_f, for ``quaternions`` [F,4] and ``translations`` [F,3] (deodr_b200_pose_frames)."""
    F, V = quaternions.shape[0], vertices.shape[0]
    if out is None:
        out = torch.empty((F, V, 3), dtype=torch.float64, device=vertices.device)
    _cabi.check(_cabi.load().deodr_b200_pose_frames(vertices.data_ptr(), V, quaternions.data_ptr(),
                                                    translations.data_ptr(), F, out.data_ptr(), scratch.data_ptr(),
                                                    _stream(vertices.device)))
    return out


def pose_frames_backward(vertices: torch.Tensor, quaternions: torch.Tensor, transformed_b: torch.Tensor,
                         scratch: torch.Tensor, center: bool = True, scale: float = 1.0,
                         losses: Optional[torch.Tensor] = None, energy_data: Optional[torch.Tensor] = None, out=None):
    """-> (vertices_b [V,3], quaternions_b [F,4], translations_b [F,3]), f64, the adjoint of :func:`pose_frames` from
    ``transformed_b`` [F,V,3] times ``scale``; ``vertices_b`` summed over the frames and centred when ``center``.
    With ``losses`` [F] f64, also writes ``energy_data`` (0-d f64) = scale * sum(losses) (deodr_b200_pose_frames_b)."""
    dev = vertices.device
    F, V = quaternions.shape[0], vertices.shape[0]
    if out is None:
        out = (torch.empty_like(vertices), torch.empty((F, 4), dtype=torch.float64, device=dev),
               torch.empty((F, 3), dtype=torch.float64, device=dev))
    v_b, q_b, t_b = out
    _cabi.check(_cabi.load().deodr_b200_pose_frames_b(
        vertices.data_ptr(), V, quaternions.data_ptr(), transformed_b.data_ptr(), F, int(bool(center)), float(scale),
        _ptr(losses), _ptr(energy_data), v_b.data_ptr(), q_b.data_ptr(), t_b.data_ptr(), scratch.data_ptr(),
        _stream(dev)))
    return v_b, q_b, t_b


def depth_compare(render: torch.Tensor, obs: torch.Tensor, max_depth: float, scratch: torch.Tensor) -> dict:
    """The comparison of MeshDepthFitter.step (deodr_b200_depth_compare): ``render`` [H,W,1] f32, ``obs`` [H,W] f64 ->
    dict(depth [H,W] f64 = clip(render, 0, max_depth), diff [H,W] f64, depth_b [H,W,1] f32, energy 0-d f64)."""
    dev = render.device
    H, W = obs.shape
    out = {"depth": torch.empty((H, W), dtype=torch.float64, device=dev),
           "diff": torch.empty((H, W), dtype=torch.float64, device=dev),
           "depth_b": torch.empty((H, W, 1), dtype=torch.float32, device=dev),
           "energy": torch.empty((), dtype=torch.float64, device=dev)}
    _cabi.check(_cabi.load().deodr_b200_depth_compare(
        render.data_ptr(), obs.data_ptr(), H * W, float(max_depth), out["depth"].data_ptr(), out["diff"].data_ptr(),
        out["depth_b"].data_ptr(), out["energy"].data_ptr(), scratch.data_ptr(), _stream(dev)))
    return out


def uniform_color_luminosity(normals: torch.Tensor, color: torch.Tensor, light: torch.Tensor,
                             out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """colours [V,C] f32 = color [C] * (max(0, -<normals, light[:3]>) + light[3]); color and light on the device.
    Written into ``out`` when given."""
    n, nc = normals.shape[0], color.shape[0]
    colors = torch.empty((n, nc), dtype=torch.float32, device=normals.device) if out is None else out
    _cabi.check(_cabi.load().deodr_b200_uniform_color_luminosity(normals.data_ptr(), n, color.data_ptr(), nc,
                                                                 light.data_ptr(), colors.data_ptr(),
                                                                 _stream(normals.device)))
    return colors


def uniform_color_luminosity_backward(normals: torch.Tensor, color: torch.Tensor, light: torch.Tensor,
                                      colors_b: torch.Tensor, scratch: torch.Tensor, out=None):
    """-> (normals_b [V,3], color_b [C], light_b [4] = (directional_b, ambient_b)), f64."""
    dev = normals.device
    n, nc = normals.shape[0], color.shape[0]
    if out is None:
        out = (torch.empty((n, 3), dtype=torch.float64, device=dev), torch.empty((nc,), dtype=torch.float64, device=dev),
               torch.empty((4,), dtype=torch.float64, device=dev))
    normals_b, color_b, light_b = out
    _cabi.check(_cabi.load().deodr_b200_uniform_color_luminosity_b(
        normals.data_ptr(), n, color.data_ptr(), nc, light.data_ptr(), colors_b.data_ptr(), normals_b.data_ptr(),
        color_b.data_ptr(), light_b.data_ptr(), scratch.data_ptr(), _stream(dev)))
    return normals_b, color_b, light_b


def heavy_ball(value: torch.Tensor, speed: torch.Tensor, grad: torch.Tensor, factor: float,
               max_step: float = math.inf, normalize: bool = False) -> _cabi.HeavyBall:
    """One parameter of :func:`fitter_update` (``DeodrHeavyBall``); the tensors must stay alive until it has run."""
    return _cabi.HeavyBall(value.data_ptr(), speed.data_ptr(), grad.data_ptr(), float(factor), float(max_step),
                           value.numel(), int(bool(normalize)))


def fitter_update(vertices: _cabi.HeavyBall, grad_rigid: Optional[torch.Tensor], params, inertia: float,
                  damping: float, energy_data=None, energy_rigid=None, energy=None, device=None) -> None:
    """The heavy-ball update of a fitting step in one kernel (deodr_b200_fitter_update)."""
    arr = (_cabi.HeavyBall * max(1, len(params)))(*params)
    _cabi.check(_cabi.load().deodr_b200_fitter_update(C.byref(vertices), _ptr(grad_rigid), arr, len(params),
                                                      float(inertia), float(damping), _ptr(energy_data),
                                                      _ptr(energy_rigid), _ptr(energy), _stream(device)))


class DeviceLaplacianRigidEnergy:
    """``LaplacianRigidEnergy`` on the device: ``evaluate(vertices)`` -> (energy 0-d f64, grad [V,3] f64) with
    grad = cregu L (L (v - v_ref)) and energy = 1/2 <v - v_ref, grad>.  The reference's third result, its constant
    approximate Hessian ``cregu * kron(L^T L, I3)``, is not returned."""

    def __init__(self, faces, vertices_ref, cregu: float, device="cuda"):
        self.device = torch.device(device)
        vertices_ref = np.asarray(vertices_ref, dtype=np.float64)
        offset, index = laplacian_neighbours(faces, vertices_ref.shape[0])
        self.nb_vertices = vertices_ref.shape[0]
        self.offset = torch.from_numpy(offset).to(self.device)
        self.index = torch.from_numpy(index if index.size else np.zeros(1, np.int32)).to(self.device)
        self.vertices_ref = torch.from_numpy(vertices_ref.copy()).to(self.device)
        self.cregu = float(cregu)
        self._lap = torch.empty_like(self.vertices_ref)
        self._scratch = new_scratch(self.device)

    def evaluate(self, vertices: torch.Tensor, grad: Optional[torch.Tensor] = None,
                 energy: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        vertices = _f64(vertices, self.device)
        if grad is None:
            grad = torch.empty_like(self.vertices_ref)
        if energy is None:
            energy = torch.empty((), dtype=torch.float64, device=self.device)
        _cabi.check(_cabi.load().deodr_b200_laplacian_rigid(
            self.offset.data_ptr(), self.index.data_ptr(), self.nb_vertices, vertices.data_ptr(),
            self.vertices_ref.data_ptr(), self.cregu, grad.data_ptr(), energy.data_ptr(), self._lap.data_ptr(),
            self._scratch.data_ptr(), _stream(self.device)))
        return energy, grad


def collision_mesh_arrays(faces, nb_vertices: int) -> dict:
    """Host arrays of ``DeodrCollisionMesh`` (numpy int32): the faces, the unique undirected edges (lo, hi) ordered by
    (lo, hi) - the edge order of :func:`topology_arrays` -, the one-ring CSR of :func:`edge_neighbours`, and the
    corners 3f + k and edge ends 2e + j of every vertex as CSR, ascending.  Face indices are checked here."""
    arr = topology_arrays(faces, nb_vertices)
    V = arr["nb_vertices"]
    f = np.asarray(arr["faces"]).view(np.uint32).astype(np.int64)
    a = f.reshape(-1)
    b = f[:, [1, 2, 0]].reshape(-1)
    key = np.unique(np.minimum(a, b) * V + np.maximum(a, b))
    edges = np.stack((key // V, key % V), axis=1)
    offset, index = edge_neighbours(faces, V)

    def csr(flat):
        off = np.zeros(V + 1, dtype=np.int32)
        np.cumsum(np.bincount(flat, minlength=V), out=off[1:])
        return off, np.argsort(flat, kind="stable").astype(np.int32)

    corner_offset, corner_index = csr(a)
    end_offset, end_index = csr(edges.reshape(-1))
    return {"faces": arr["faces"], "edges": np.ascontiguousarray(edges, dtype=np.int32), "neighbour_offset": offset,
            "neighbour_index": index if index.size else np.zeros(1, np.int32), "corner_offset": corner_offset,
            "corner_index": corner_index, "end_offset": end_offset, "end_index": end_index,
            "nb_faces": arr["nb_faces"], "nb_edges": int(edges.shape[0]), "nb_vertices": V}


class DeviceSelfCollisionEnergy:
    """A self-collision penalty on the device (include/deodr_b200.h, "Self-collision"): for thickness delta and weight
    w, E = w sum phi(d) over the vertex-triangle and edge-edge pairs outside each other's one-ring, with
    phi(d) = (delta - d)^2 below delta.  ``evaluate(vertices)`` -> (energy 0-d f64, grad [V,3] f64); ``min_distance``
    (0-d) is the smallest such distance of the last evaluation, or delta when there is none; ``intersections`` lists the
    face pairs that cross.  ``vertices_ref`` only sizes the grid's cells (their median edge length, at least delta).
    Meshes of several connected components are accepted.  Each call reads one word back from the device."""

    def __init__(self, faces, vertices_ref, thickness: float, weight: float, device="cuda"):
        from .renderer import default_renderer

        self.device = torch.device(device)
        vertices_ref = np.asarray(vertices_ref, dtype=np.float64)
        self.thickness, self.weight = float(thickness), float(weight)
        arrays = collision_mesh_arrays(faces, vertices_ref.shape[0])
        self.nb_vertices, self.nb_faces = arrays["nb_vertices"], arrays["nb_faces"]
        self.t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(self.device) for k, v in arrays.items()
                  if isinstance(v, np.ndarray)}
        self._mesh = _cabi.CollisionMesh()
        for name, t in self.t.items():
            setattr(self._mesh, name, t.data_ptr())
        self._mesh.nb_faces, self._mesh.nb_edges, self._mesh.nb_vertices = (arrays["nb_faces"], arrays["nb_edges"],
                                                                            arrays["nb_vertices"])
        e = arrays["edges"]
        lengths = np.linalg.norm(vertices_ref[e[:, 0]] - vertices_ref[e[:, 1]], axis=1)
        self.cell_size = max(float(np.median(lengths)) if lengths.size else 0.0, self.thickness)
        self.min_distance = torch.empty((), dtype=torch.float64, device=self.device)
        self._renderer = default_renderer(self.device.index if self.device.index is not None else None)
        self._pairs = torch.empty((max(16, self.nb_faces // 8), 2), dtype=torch.int32, device=self.device)

    def _vertices(self, vertices: torch.Tensor) -> torch.Tensor:
        if tuple(vertices.shape) != (self.nb_vertices, 3):
            raise ValueError(f"vertices must be [{self.nb_vertices},3]; got {tuple(vertices.shape)}")
        return _f64(vertices, self.device)

    def evaluate(self, vertices: torch.Tensor, grad: Optional[torch.Tensor] = None,
                 energy: Optional[torch.Tensor] = None,
                 add_to: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """-> (energy, grad): grad = add_to + dE/dvertices (``add_to`` may be ``grad`` itself, to add in place)."""
        vertices = self._vertices(vertices)
        if grad is None:
            grad = torch.empty((self.nb_vertices, 3), dtype=torch.float64, device=self.device)
        if energy is None:
            energy = torch.empty((), dtype=torch.float64, device=self.device)
        r = self._renderer
        with r._lock:
            _cabi.check(r.lib.deodr_b200_self_collision(
                r._ws, C.byref(self._mesh), vertices.data_ptr(), self.thickness, self.weight, self.cell_size,
                _ptr(add_to), grad.data_ptr(), energy.data_ptr(), self.min_distance.data_ptr(), _stream(self.device)))
        return energy, grad

    def intersections(self, vertices: torch.Tensor) -> torch.Tensor:
        """The face pairs (i < j) that share no vertex and where an edge of one properly crosses the other: [P,2]
        int64, sorted.  Coplanar and touching contacts are not reported."""
        vertices = self._vertices(vertices)
        r = self._renderer
        count = C.c_int64(0)
        for _ in range(2):
            with r._lock:
                _cabi.check(r.lib.deodr_b200_self_intersections(
                    r._ws, C.byref(self._mesh), vertices.data_ptr(), self.cell_size, self._pairs.data_ptr(),
                    self._pairs.shape[0], C.byref(count), _stream(self.device)))
            if count.value <= self._pairs.shape[0]:
                break
            self._pairs = torch.empty((count.value + count.value // 4, 2), dtype=torch.int32, device=self.device)
        pairs = self._pairs[:count.value].to(torch.int64)
        order = torch.argsort(pairs[:, 0] * self.nb_faces + pairs[:, 1])
        return pairs[order]


def fitter_camera(camera_center, width: int, height: int, focal=None, distortion=None) -> CameraParams:
    """The camera of the reference fitters' ``set_image``: rotation diag(1, -1, -1), centre ``camera_center``, focal
    ``2 * width`` by default, principal point at the image centre."""
    if focal is None:
        focal = 2 * width
    rot = np.array([[1, 0, 0], [0, -1, 0], [0, 0, -1]], dtype=np.float64)
    trans = -rot.T.dot(np.asarray(camera_center, dtype=np.float64))
    intrinsic = np.array([[focal, 0, width / 2], [0, focal, height / 2], [0, 0, 1]], dtype=np.float64)
    return CameraParams(np.column_stack((rot, trans)), intrinsic, distortion)


# The heavy-ball step of the joint rotations (radians).  On the articulated-fit tube of tests/test_gpu_skinning.py
# (128 x 128 colour image, bends of 0.3 - 0.4 rad) the joint gradients start near 3e3, so the step runs at its clamp
# at first; 0.05 rad (about 3 degrees) per step bounds it.  Measured on an H100 over 800 steps: with the per-vertex
# deformation held still, 0.002 recovers the bends within 0.046 rad in 16 runs out of 16 (0.0005 within 0.015); with
# it free, 0.0005 leaves the joints nearly where they start, since the vertices take the bend, and of 0.002, 0.005,
# 0.02 and 0.05, 0.002 ends closest.  The free deformation then absorbs part of the bend whatever the factor.
STEP_FACTOR_JOINTS = 0.002
STEP_MAX_JOINTS = 0.05


class _PoseFitter:
    """State and update rule shared by the two fitters: vertices, quaternion and translation with their speeds."""

    def _init_pose(self, vertices, faces, euler_init, translation_init, cregu, inertia, damping, device, cself=0.0,
                   self_collision_thickness=None, skeleton=None):
        self.device = torch.device(device)
        self.cregu, self.inertia, self.damping = cregu, inertia, damping
        self.faces = np.ascontiguousarray(np.asarray(faces), dtype=np.int64)
        self.vertices_init = np.array(vertices, dtype=np.float64)
        self.nb_vertices = self.vertices_init.shape[0]
        self.rigid_energy = DeviceLaplacianRigidEnergy(self.faces, self.vertices_init, cregu, self.device)
        self.skinning = self._skinning(skeleton)
        # the self-collision term, evaluated at the vertices the rigid pose moves (the pose is rigid: distances do not
        # change under it), i.e. the skinned vertices with a skeleton
        self.cself = float(cself)
        self.self_collision = None
        self.energy_self_collision = torch.zeros((), dtype=torch.float64, device=self.device)
        if self.cself < 0:
            raise ValueError(f"cself must be >= 0; got {cself}")
        if self.cself > 0:
            if self_collision_thickness is None:
                raise ValueError("cself > 0 needs self_collision_thickness")
            self.self_collision = DeviceSelfCollisionEnergy(self.faces, self.vertices_init, self_collision_thickness,
                                                            self.cself, self.device)
        self._scratch = new_scratch(self.device)
        self.view: Optional[DeviceMeshView] = None
        self.set_mesh_transform_init(euler=euler_init, translation=translation_init)

    def _skinning(self, skeleton) -> Optional[LinearBlendSkinning]:
        """The skeleton of the articulated fit, or None.  A single root at joint 0 is required: its rotation would
        duplicate the rigid quaternion, so it stays fixed and rows 1..J-1 of ``joint_rotations`` are fitted."""
        if skeleton is None:
            return None
        if not isinstance(skeleton, LinearBlendSkinning):
            skeleton = LinearBlendSkinning(*skeleton, device=self.device)
        device = self.rigid_energy.vertices_ref.device
        if skeleton.device != device or skeleton.nb_vertices != self.nb_vertices:
            raise ValueError(f"the skeleton binds {skeleton.nb_vertices} vertices on {skeleton.device}; the mesh has "
                             f"{self.nb_vertices} on {device}")
        roots = np.flatnonzero(skeleton.parents < 0)
        if roots.tolist() != [0]:
            raise ValueError("the fitters need a skeleton with a single root at joint 0; "
                             f"its roots are {roots.tolist()}")
        self.joint_rotations_init = np.zeros((skeleton.nb_joints, 3))
        return skeleton

    def set_joint_rotations_init(self, rotations) -> None:
        """The joint rotations [J,3] (axis-angle) that :meth:`reset` starts from; row 0, the root's, stays fixed."""
        if self.skinning is None:
            raise ValueError("set_joint_rotations_init needs a fitter built with a skeleton")
        rotations = np.array(rotations, dtype=np.float64)
        if rotations.shape != (self.skinning.nb_joints, 3) or not np.all(np.isfinite(rotations)):
            raise ValueError(f"rotations must be finite [{self.skinning.nb_joints},3]; got shape {rotations.shape}")
        self.joint_rotations_init = rotations

    def _tensor(self, a) -> torch.Tensor:
        return torch.tensor(np.array(a, dtype=np.float64), device=self.device)

    def set_mesh_transform_init(self, euler, translation) -> None:
        self.transform_quaternion_init = euler_to_quaternion(euler)
        self.transform_translation_init = np.array(translation, dtype=np.float64)

    def _reset_pose(self) -> None:
        V = self.nb_vertices
        dev = self.device
        self.vertices = self._tensor(self.vertices_init)
        self.speed_vertices = torch.zeros((V, 3), dtype=torch.float64, device=dev)
        self.transform_quaternion = self._tensor(self.transform_quaternion_init)
        self.transform_translation = self._tensor(self.transform_translation_init)
        self.speed_quaternion = torch.zeros(4, dtype=torch.float64, device=dev)
        self.speed_translation = torch.zeros(3, dtype=torch.float64, device=dev)
        self._transformed = torch.empty((V, 3), dtype=torch.float64, device=dev)
        self._vertices_b = torch.empty((V, 3), dtype=torch.float64, device=dev)
        self.transform_quaternion_b = torch.empty(4, dtype=torch.float64, device=dev)
        self.transform_translation_b = torch.empty(3, dtype=torch.float64, device=dev)
        self._grad_rigid = torch.empty((V, 3), dtype=torch.float64, device=dev)
        self._energy_rigid = torch.empty((), dtype=torch.float64, device=dev)
        if self.skinning is not None:
            self.joint_rotations = self._tensor(self.joint_rotations_init)
            self.speed_joint_rotations = torch.zeros_like(self.joint_rotations)
            self.joint_rotations_b = torch.empty_like(self.joint_rotations)
            self._skinned = torch.empty((V, 3), dtype=torch.float64, device=dev)
            self._skinned_b = torch.empty((V, 3), dtype=torch.float64, device=dev)
        self.iter = 0

    def _camera(self, mesh_image, focal, distortion) -> CameraParams:
        self.width, self.height = mesh_image.shape[1], mesh_image.shape[0]
        self.iter = 0
        return fitter_camera(self.camera_center, self.width, self.height, focal, distortion)

    def _regularisers(self) -> None:
        """The rigidity's gradient and energy into ``_grad_rigid`` and ``_energy_rigid``, plus the self-collision's
        when ``cself > 0`` (then also in ``energy_self_collision``)."""
        self.rigid_energy.evaluate(self.vertices, grad=self._grad_rigid, energy=self._energy_rigid)
        if self.self_collision is not None:
            self.self_collision.evaluate(self.vertices, grad=self._grad_rigid, energy=self.energy_self_collision,
                                         add_to=self._grad_rigid)
            self._energy_rigid += self.energy_self_collision

    def _render_pose(self) -> torch.Tensor:
        vertices = self.vertices
        if self.skinning is not None:
            vertices = self.skinning.apply(self.vertices, self.joint_rotations, out=self._skinned)
        return pose(vertices, self.transform_quaternion, self.transform_translation, self._scratch,
                    out=self._transformed)

    def _skinning_backward(self, transformed_b: torch.Tensor) -> None:
        """The articulated step's adjoint: the pose's to the (centred) skinned vertices, plus the self-collision's
        there, then the skinning's to the rest vertices and the joint rotations; the rigidity on the rest vertices."""
        pose_backward(self._skinned, self.transform_quaternion, transformed_b, self._scratch,
                      out=(self._skinned_b, self.transform_quaternion_b, self.transform_translation_b))
        if self.self_collision is not None:
            self.self_collision.evaluate(self._skinned, grad=self._skinned_b, energy=self.energy_self_collision,
                                         add_to=self._skinned_b)
        self.skinning.backward(self.vertices, self.joint_rotations, self._skinned_b,
                               out=(self._vertices_b, self.joint_rotations_b))
        self.rigid_energy.evaluate(self.vertices, grad=self._grad_rigid, energy=self._energy_rigid)
        if self.self_collision is not None:
            self._energy_rigid += self.energy_self_collision

    def _pose_backward_rigid_update(self, transformed_b: torch.Tensor, energy_data: torch.Tensor,
                                    extra_params=()) -> torch.Tensor:
        if self.skinning is None:
            pose_backward(self.vertices, self.transform_quaternion, transformed_b, self._scratch,
                          out=(self._vertices_b, self.transform_quaternion_b, self.transform_translation_b))
            self._regularisers()
        else:
            self._skinning_backward(transformed_b)
        energy = torch.empty((), dtype=torch.float64, device=self.device)
        params = [heavy_ball(self.transform_quaternion, self.speed_quaternion, self.transform_quaternion_b,
                             self.step_factor_quaternion, self.step_max_quaternion, normalize=True),
                  heavy_ball(self.transform_translation, self.speed_translation, self.transform_translation_b,
                             self.step_factor_translation, self.step_max_translation)] + list(extra_params)
        if self.skinning is not None and self.skinning.nb_joints > 1:  # rows 1..J-1: the root stays fixed
            params.append(heavy_ball(self.joint_rotations[1:], self.speed_joint_rotations[1:],
                                     self.joint_rotations_b[1:], self.step_factor_joints, self.step_max_joints))
        fitter_update(heavy_ball(self.vertices, self.speed_vertices, self._vertices_b, self.step_factor_vertices,
                                 self.step_max_vertices), self._grad_rigid, params, self.inertia, self.damping,
                      energy_data, self._energy_rigid, energy, self.device)
        self.iter += 1
        return energy


class MeshDepthFitter(_PoseFitter):
    """``deodr.mesh_fitter.MeshDepthFitter`` on the device: fits a deformable mesh and its rigid pose to a depth image.
    ``step()`` -> (energy 0-d f64, depth [H,W] f64 clipped to [0, max_depth], diff_image [H,W] f64), CUDA tensors."""

    def __init__(self, vertices, faces, euler_init, translation_init, cregu: float = 2000, inertia: float = 0.96,
                 damping: float = 0.05, device="cuda", cself: float = 0.0,
                 self_collision_thickness: Optional[float] = None, skeleton=None):
        self.step_factor_vertices = 0.0005
        self.step_max_vertices = 1
        self.step_factor_quaternion = 0.00006
        self.step_max_quaternion = 0.1
        self.step_factor_translation = 0.00005
        self.step_max_translation = 0.1
        self.step_factor_joints, self.step_max_joints = STEP_FACTOR_JOINTS, STEP_MAX_JOINTS
        vertices = np.asarray(vertices, dtype=np.float64)
        object_center = vertices.mean(axis=0)
        object_radius = np.max(np.std(vertices, axis=0))
        self.camera_center = object_center + np.array([-0.5, 0, 5]) * object_radius
        self.max_depth = None
        self.depth_scale = 1.0
        self._init_pose(vertices, faces, euler_init, translation_init, cregu, inertia, damping, device, cself,
                        self_collision_thickness, skeleton)
        self.reset()

    def reset(self) -> None:
        self._reset_pose()

    def set_max_depth(self, max_depth: float) -> None:
        """The far plane: depths are clipped to [0, max_depth], and the background is at max_depth."""
        self.max_depth = float(max_depth)
        if self.view is not None:
            self.view.scene.t["background_color"].fill_(self.max_depth)

    def set_depth_scale(self, depth_scale: float) -> None:
        self.depth_scale = float(depth_scale)

    def set_image(self, mesh_image, focal: Optional[float] = None, distortion=None) -> None:
        mesh_image = np.asarray(mesh_image, dtype=np.float64)
        if mesh_image.ndim != 2:
            raise ValueError(f"MeshDepthFitter.set_image: expected a [H,W] depth image, got shape {mesh_image.shape}")
        camera = self._camera(mesh_image, focal, distortion)
        self.mesh_image = torch.from_numpy(np.ascontiguousarray(mesh_image)).to(self.device)
        background = 0.0 if self.max_depth is None else self.max_depth
        self.view = DeviceMeshView(self.faces, self.nb_vertices, camera, self.height, self.width,
                                   background_color=(background,), device=self.device)
        self.camera = camera

    def step(self):
        if self.view is None or self.max_depth is None:
            raise RuntimeError("MeshDepthFitter.step: call set_image and set_max_depth first")
        transformed = self._render_pose()
        render = self.view.render_depth(transformed, self.depth_scale)
        cmp = depth_compare(render, self.mesh_image, self.max_depth, self._scratch)
        transformed_b = self.view.render_depth_backward(cmp["depth_b"])
        energy = self._pose_backward_rigid_update(transformed_b, cmp["energy"])
        return energy, cmp["depth"], cmp["diff"]


class MeshRGBFitterWithPose(_PoseFitter):
    """``deodr.mesh_fitter.MeshRGBFitterWithPose`` on the device: fits a deformable mesh, its rigid pose, a uniform
    colour and a directional + ambient light to a colour image.  ``step()`` -> (energy 0-d f64, image [H,W,C] f32,
    diff_image [H,W] f32), CUDA tensors.  The lights and the colour are device tensors: ``light_directional`` [3],
    ``light_ambient`` (0-d) and ``mesh_color`` [C]."""

    def __init__(self, vertices, faces, euler_init, translation_init, default_color, default_light_directional,
                 default_light_ambient: float, cregu: float = 2000, inertia: float = 0.96, damping: float = 0.05,
                 update_lights: bool = True, update_color: bool = True, device="cuda",
                 cself: float = 0.0, self_collision_thickness: Optional[float] = None, skeleton=None):
        self.step_factor_vertices = 0.0005
        self.step_max_vertices = 0.5
        self.step_factor_quaternion = 0.00006
        self.step_max_quaternion = 0.05
        self.step_factor_translation = 0.00005
        self.step_max_translation = 0.1
        self.step_factor_joints, self.step_max_joints = STEP_FACTOR_JOINTS, STEP_MAX_JOINTS
        self.default_color = np.array(default_color, dtype=np.float64)
        self.default_light_directional = np.array(default_light_directional, dtype=np.float64)
        self.default_light_ambient = float(default_light_ambient)
        self.update_lights = update_lights  # stored, as in the reference, whose step updates both regardless
        self.update_color = update_color
        vertices = np.asarray(vertices, dtype=np.float64)
        object_center = vertices.mean(axis=0) + np.asarray(translation_init, dtype=np.float64)
        object_radius = np.max(np.std(vertices, axis=0))
        self.camera_center = object_center + np.array([0, 0, 9]) * object_radius
        self.background_color = None
        self.sigma = 1.0
        self._init_pose(vertices, faces, euler_init, translation_init, cregu, inertia, damping, device, cself,
                        self_collision_thickness, skeleton)
        self.reset()

    def reset(self) -> None:
        self._reset_pose()
        dev = self.device
        # light = (directional x, y, z, ambient): the layout of the light kernels and of their adjoint light_b
        self._light = self._tensor(np.concatenate((self.default_light_directional, [self.default_light_ambient])))
        self.mesh_color = self._tensor(self.default_color)
        self._speed_light = torch.zeros(4, dtype=torch.float64, device=dev)
        self.speed_mesh_color = torch.zeros_like(self.mesh_color)
        self._light_b = torch.empty(4, dtype=torch.float64, device=dev)
        self.mesh_color_b = torch.empty_like(self.mesh_color)
        self._normals_b = torch.empty((self.nb_vertices, 3), dtype=torch.float64, device=dev)

    @property
    def light_directional(self) -> torch.Tensor:
        return self._light[:3]

    @property
    def light_ambient(self) -> torch.Tensor:
        return self._light[3]

    def set_background_color(self, background_color) -> None:
        self.background_color = np.array(background_color, dtype=np.float64)
        if self.view is not None:
            self.view.scene.t["background_color"].copy_(torch.from_numpy(self.background_color))

    def set_image(self, mesh_image, focal: Optional[float] = None, distortion=None) -> None:
        mesh_image = np.asarray(mesh_image, dtype=np.float64)
        if mesh_image.ndim != 3:
            raise ValueError(f"MeshRGBFitterWithPose.set_image: expected a [H,W,C] image, got shape {mesh_image.shape}")
        camera = self._camera(mesh_image, focal, distortion)
        self.mesh_image = torch.from_numpy(np.ascontiguousarray(mesh_image, dtype=np.float32)).to(self.device)
        nc = mesh_image.shape[2]
        if nc != self.default_color.shape[0]:
            raise ValueError(f"the image has {nc} channels and the mesh colour {self.default_color.shape[0]}")
        background = self.background_color if self.background_color is not None else np.zeros(nc)
        self.view = DeviceMeshView(self.faces, self.nb_vertices, camera, self.height, self.width,
                                   background_color=tuple(background), sigma=self.sigma, device=self.device)
        self.camera = camera

    def step(self):
        if self.view is None:
            raise RuntimeError("MeshRGBFitterWithPose.step: call set_image first")
        view = self.view
        transformed = self._render_pose()
        _, normals = view.topology.vertex_normals(transformed)
        colors = uniform_color_luminosity(normals, self.mesh_color, self._light)
        ij, depths = project_points_and_flags(view, transformed, colors)
        res = view.renderer.render_compare_and_backward(view.scene, view.sigma, self.mesh_image)
        grads = res["grads"]
        uniform_color_luminosity_backward(normals, self.mesh_color, self._light, grads["colors_b"], self._scratch,
                                          out=(self._normals_b, self.mesh_color_b, self._light_b))
        transformed_b = view.topology.vertex_normals_backward(transformed, self._normals_b)
        project_points_backward(transformed, view.camera, grads["ij_b"], out=transformed_b)
        energy = self._pose_backward_rigid_update(
            transformed_b, res["loss"],
            (heavy_ball(self._light, self._speed_light, self._light_b, 0.0001),
             heavy_ball(self.mesh_color, self.speed_mesh_color, self.mesh_color_b, 0.00001)))
        return energy, res["image"], res["err_pixel"]


class MeshRGBFitterWithPoseMultiFrame(_PoseFitter):
    """``deodr.mesh_fitter.MeshRGBFitterWithPoseMultiFrame`` on the device: fits one deformable mesh to F colour images,
    with one rigid pose per image and a uniform colour and a directional + ambient light shared by all of them, seen
    by one camera (that of the reference's ``set_images``).  The F frames are rendered, compared and back-propagated
    in one ``render_compare_views`` / ``render_b_views`` call each; the mesh-side steps run once over the F * V
    posed vertices (one topology over F disjoint copies of the faces).

    ``step()`` -> (energy 0-d f64, images: F tensors [H,W,C] f32, diff_images: F tensors [H,W] f32 holding the
    unweighted sum_c d_f^2), CUDA tensors, with d_f = image_f - obs_f and
    ``energy = cdata / F * sum_f sum d_f^2 + rigidity``.  The reference compares ``image[idframe]``, a row of the
    render, instead of frame ``idframe``'s image (deodr/mesh_fitter.py:539, :543), and does not converge; this class
    compares the frame's image and back-propagates the exact gradient of that energy (INTEGRATION.md section 5).
    As in the reference, the vertex gradient loses its mean only while ``iter < 500``, and the quaternions [F,4] are
    divided by their joint Frobenius norm after each update.

    State (CUDA tensors): ``vertices`` [V,3], ``transform_quaternion`` [F,4], ``transform_translation`` [F,3],
    ``light_directional`` [3], ``light_ambient`` (0-d), ``mesh_color`` [C] and their speeds.  The data weight
    cdata / F scales the pose and vertex adjoints inside ``deodr_b200_pose_frames_b``; ``mesh_color_b`` and
    ``light_b`` hold the unweighted frame sums, and the weight is in their step factors."""

    def __init__(self, vertices, faces, euler_init, translation_init, default_color, default_light_directional,
                 default_light_ambient: float, cregu: float = 2000, cdata: float = 1, inertia: float = 0.97,
                 damping: float = 0.15, update_lights: bool = True, update_color: bool = True, device="cuda",
                 cself: float = 0.0, self_collision_thickness: Optional[float] = None):
        self.step_factor_vertices = 0.0005
        self.step_max_vertices = 0.5
        self.step_factor_quaternion = 0.00005
        self.step_max_quaternion = 0.05
        self.step_factor_translation = 0.00004
        self.step_max_translation = 0.1
        self.step_factor_light = 0.0001
        self.step_factor_color = 0.00001
        self.cdata = float(cdata)
        self.default_color = np.array(default_color, dtype=np.float64)
        self.default_light_directional = np.array(default_light_directional, dtype=np.float64)
        self.default_light_ambient = float(default_light_ambient)
        self.update_lights = update_lights  # stored, as in the reference, whose step updates both regardless
        self.update_color = update_color
        vertices = np.asarray(vertices, dtype=np.float64)
        self.camera_center = vertices.mean(axis=0) + np.array([0, 0, 6]) * np.max(np.std(vertices, axis=0))
        self.background_color = None
        self.sigma = 1.0
        self.scenes = None
        self._init_pose(vertices, faces, euler_init, translation_init, cregu, inertia, damping, device, cself,
                        self_collision_thickness)
        self.reset()

    def set_mesh_transform_init(self, euler, translation) -> None:
        """euler [F,3] ("zyx", as the reference) and translation [F,3]: one pose per frame, applied by :meth:`reset`."""
        euler = np.atleast_2d(np.asarray(euler, dtype=np.float64))
        translation = np.atleast_2d(np.asarray(translation, dtype=np.float64))
        if euler.shape[1] != 3 or translation.shape != euler.shape:
            raise ValueError(f"euler and translation must both be [F,3]; got {euler.shape} and {translation.shape}")
        super().set_mesh_transform_init(euler, translation)

    @property
    def nb_frames(self) -> int:
        return self.transform_quaternion_init.shape[0]

    def reset(self) -> None:
        F, V, nc = self.nb_frames, self.nb_vertices, self.default_color.shape[0]
        T = self.faces.shape[0]
        dev = self.device
        f64 = dict(dtype=torch.float64, device=dev)
        self.vertices = self._tensor(self.vertices_init)
        self.speed_vertices = torch.zeros((V, 3), **f64)
        self.transform_quaternion = self._tensor(self.transform_quaternion_init)
        self.transform_translation = self._tensor(self.transform_translation_init)
        self.speed_quaternion = torch.zeros((F, 4), **f64)
        self.speed_translation = torch.zeros((F, 3), **f64)
        # light = (directional x, y, z, ambient): the layout of the light kernels and of their adjoint light_b
        self._light = self._tensor(np.concatenate((self.default_light_directional, [self.default_light_ambient])))
        self.mesh_color = self._tensor(self.default_color)
        self._speed_light = torch.zeros(4, **f64)
        self.speed_mesh_color = torch.zeros_like(self.mesh_color)
        # gradients and the F * V batch buffers of a step
        self._vertices_b = torch.empty((V, 3), **f64)
        self.transform_quaternion_b = torch.empty((F, 4), **f64)
        self.transform_translation_b = torch.empty((F, 3), **f64)
        self._light_b = torch.empty(4, **f64)
        self.mesh_color_b = torch.empty_like(self.mesh_color)
        self._grad_rigid = torch.empty((V, 3), **f64)
        self._energy_rigid = torch.empty((), **f64)
        self._energy_data = torch.empty((), **f64)
        self._losses = torch.zeros(F, **f64)
        self._posed = torch.empty((V, 3), **f64)  # the vertices render() centres
        self._transformed = torch.empty((F, V, 3), **f64)
        self._ij = torch.empty((F * V, 2), **f64)
        self._depths = torch.empty((F * V,), **f64)
        self._colors = torch.empty((F * V, nc), dtype=torch.float32, device=dev)
        self._edgeflags = torch.empty((F * T, 3), dtype=torch.uint8, device=dev)
        # the renderer's gradient slots of every frame in one buffer, zeroed once per step: ij_b [F*V,2],
        # colors_b [F*V,C], and shade_b [F*V], uv_b [F,1,2], texture_b [F,2,2,C], which an untextured scene leaves zero
        sizes = (F * V * 2, F * V * nc, F * V, F * 2, F * 4 * nc)
        self._grad_buffer = torch.zeros(sum(sizes), dtype=torch.float32, device=dev)
        ij_b, colors_b, shade_b, uv_b, texture_b = torch.split(self._grad_buffer, sizes)
        self._ij_b, self._colors_b = ij_b.view(F * V, 2), colors_b.view(F * V, nc)
        self._shade_b, self._uv_b, self._texture_b = shade_b, uv_b.view(F, 1, 2), texture_b.view(F, 2, 2, nc)
        self._normals_b = torch.empty((F * V, 3), **f64)
        self.topology = MeshTopology(np.concatenate([self.faces + f * V for f in range(F)]), F * V, device=dev)
        self.iter = 0
        if self.scenes is not None and len(self.scenes) != F:
            self.scenes = None  # the number of poses changed: set_images again
        if self.scenes is not None:
            self._bind_scenes()

    @property
    def light_directional(self) -> torch.Tensor:
        return self._light[:3]

    @property
    def light_ambient(self) -> torch.Tensor:
        return self._light[3]

    def set_background_color(self, background_color) -> None:
        self.background_color = np.array(background_color, dtype=np.float64)
        for scene in self.scenes or ():
            scene.t["background_color"].copy_(torch.from_numpy(self.background_color))

    def set_images(self, mesh_images, focal: Optional[float] = None) -> None:
        """The F observed images [H,W,C], one per pose, in frame order.  All frames share the camera of the
        reference's ``set_images``: centre mean(vertices) + [0, 0, 6] * radius, focal ``2 * width`` by default."""
        from .renderer import DeviceScene, default_renderer
        from .scenes import SceneArrays

        images = [np.asarray(im, dtype=np.float64) for im in mesh_images]
        if len(images) != self.nb_frames:
            raise ValueError(f"{len(images)} images for {self.nb_frames} poses: give one image per pose")
        if any(im.ndim != 3 for im in images):
            raise ValueError("every image must be [H,W,C]")
        if any(im.shape != images[0].shape for im in images):
            raise ValueError(f"the images differ in shape: {sorted(set(im.shape for im in images))}")
        nc = images[0].shape[2]
        if nc != self.default_color.shape[0]:
            raise ValueError(f"the images have {nc} channels and the mesh colour {self.default_color.shape[0]}")
        self.height, self.width = images[0].shape[:2]
        self.camera = fitter_camera(self.camera_center, self.width, self.height, focal)
        self._camera_c = self.camera.c_struct()
        self.mesh_images = torch.from_numpy(np.ascontiguousarray(np.stack(images), dtype=np.float32)).to(self.device)
        background = self.background_color if self.background_color is not None else np.zeros(nc)
        T, V = self.faces.shape[0], self.nb_vertices
        faces_u32 = np.ascontiguousarray(self.faces, dtype=np.uint32)
        arrays = SceneArrays(
            faces=faces_u32, faces_uv=np.zeros((T, 3), np.uint32), ij=np.zeros((V, 2)), depths=np.ones(V),
            textured=np.zeros(T, bool), uv=np.zeros((1, 2)), shade=np.zeros(V), colors=np.zeros((V, nc)),
            shaded=np.zeros(T, bool), edgeflags=np.zeros((T, 3), bool), height=self.height, width=self.width,
            nb_colors=nc, texture=np.zeros((2, 2, nc)), background_image=None, background_color=background,
            clockwise=False, backface_culling=True, strict_edge=True, perspective_correct=False,
            integer_pixel_centers=True)
        self.renderer = default_renderer(self.device.index)
        self.scenes = [DeviceScene(arrays, self.device) for _ in range(self.nb_frames)]
        self._bind_scenes()
        self.iter = 0

    def _bind_scenes(self) -> None:
        """Points frame f's scene inputs and gradients at slice f of the batch buffers, and makes the comparison
        write frame f's loss into ``_losses[f]``."""
        from .renderer import Renderer

        V, T = self.nb_vertices, self.faces.shape[0]
        self._grads, self._outs = [], []
        for f, scene in enumerate(self.scenes):
            v, t = slice(f * V, (f + 1) * V), slice(f * T, (f + 1) * T)
            scene.t.update(ij=self._ij[v], depths=self._depths[v], colors=self._colors[v], edgeflags=self._edgeflags[t])
            self._grads.append({"ij_b": self._ij_b[v], "colors_b": self._colors_b[v], "shade_b": self._shade_b[v],
                                "uv_b": self._uv_b[f], "texture_b": self._texture_b[f]})
            out = Renderer._new_outputs(scene, False, False, False)
            out["loss"] = self._losses[f]
            self._outs.append(out)

    def set_image(self, mesh_image, focal: Optional[float] = None) -> None:
        """``set_images([mesh_image])``: only for a fitter with one frame."""
        if self.nb_frames != 1:
            raise ValueError(f"set_image sets one image; this fitter has {self.nb_frames} frames: use set_images")
        self.set_images([mesh_image], focal)

    def _pose_and_scenes(self, vertices: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """Centres ``vertices`` in place, poses them in every frame and fills the frames' scenes -> (the posed vertices
        [F*V,3], their normals)."""
        pose_frames(vertices, self.transform_quaternion, self.transform_translation, self._scratch,
                    out=self._transformed)
        flat = self._transformed.view(-1, 3)
        _, normals = self.topology.vertex_normals(flat)
        uniform_color_luminosity(normals, self.mesh_color, self._light, out=self._colors)
        _cabi.check(_cabi.load().deodr_b200_project_points(flat.data_ptr(), flat.shape[0], C.byref(self._camera_c),
                                                           self._ij.data_ptr(), self._depths.data_ptr(),
                                                           _stream(self.device)))
        self.topology.edge_on_silhouette(self._ij, out=self._edgeflags)
        return flat, normals

    def render(self, idframe: int) -> torch.Tensor:
        """The image [H,W,C] f32 of frame ``idframe`` that the next :meth:`step` renders: the current vertices centred
        (step centres them; the state is left as it is), under that frame's pose."""
        if self.scenes is None:
            raise RuntimeError("MeshRGBFitterWithPoseMultiFrame.render: call set_images first")
        if not 0 <= idframe < self.nb_frames:
            raise IndexError(f"frame {idframe} of {self.nb_frames}")
        self._posed.copy_(self.vertices)
        self._pose_and_scenes(self._posed)
        return self.renderer.render(self.scenes[idframe], self.sigma)["image"]

    def step(self, check_gradient: bool = False):
        if check_gradient:
            raise NotImplementedError("check_gradient: the reference's finite-difference check is not run on the device")
        if self.scenes is None:
            raise RuntimeError("MeshRGBFitterWithPoseMultiFrame.step: call set_images first")
        flat, normals = self._pose_and_scenes(self.vertices)
        self._grad_buffer.zero_()
        for out in self._outs:  # fresh images for the caller; the comparison's other buffers are reused
            out["image"] = torch.empty_like(out["image"])
            out["err_pixel"] = None
        obs = list(self.mesh_images)
        outs = self.renderer.render_compare_views(self.scenes, self.sigma, obs, err_pixel=True, out=self._outs)
        self.renderer.render_b_views(self.scenes, self.sigma, outs, [o["image_b"] for o in outs], self._grads)
        uniform_color_luminosity_backward(normals, self.mesh_color, self._light, self._colors_b, self._scratch,
                                          out=(self._normals_b, self.mesh_color_b, self._light_b))
        transformed_b = self.topology.vertex_normals_backward(flat, self._normals_b)
        project_points_backward(flat, self.camera, self._ij_b, out=transformed_b)
        coef = self.cdata / self.nb_frames
        pose_frames_backward(self.vertices, self.transform_quaternion, transformed_b, self._scratch,
                             center=self.iter < 500, scale=coef, losses=self._losses, energy_data=self._energy_data,
                             out=(self._vertices_b, self.transform_quaternion_b, self.transform_translation_b))
        self._regularisers()
        energy = torch.empty((), dtype=torch.float64, device=self.device)
        params = [heavy_ball(self.transform_quaternion, self.speed_quaternion, self.transform_quaternion_b,
                             self.step_factor_quaternion, self.step_max_quaternion, normalize=True),
                  heavy_ball(self.transform_translation, self.speed_translation, self.transform_translation_b,
                             self.step_factor_translation, self.step_max_translation),
                  heavy_ball(self._light, self._speed_light, self._light_b, self.step_factor_light * coef),
                  heavy_ball(self.mesh_color, self.speed_mesh_color, self.mesh_color_b, self.step_factor_color * coef)]
        fitter_update(heavy_ball(self.vertices, self.speed_vertices, self._vertices_b, self.step_factor_vertices,
                                 self.step_max_vertices), self._grad_rigid, params, self.inertia, self.damping,
                      self._energy_data, self._energy_rigid, energy, self.device)
        self.iter += 1
        return energy, [o["image"] for o in outs], [o["err_pixel"] for o in outs]


def project_points_and_flags(view: DeviceMeshView, vertices: torch.Tensor, colors: torch.Tensor):
    """Fills ``view``'s scene with the projection of ``vertices``, their depths, ``colors`` and the silhouette flags."""
    ij, depths = project_points(vertices, view.camera)
    t = view.scene.t
    t["ij"].copy_(ij)
    t["depths"].copy_(depths)
    t["colors"].copy_(colors)
    view.topology.edge_on_silhouette(ij, out=t["edgeflags"])
    return ij, depths
