"""autograd surface of the 3D render, mirroring deodr/pytorch/differentiable_renderer_pytorch.py (``CameraPytorch``,
``Scene3DPytorch``), triangulated_mesh_pytorch.py (``ColoredTriMeshPytorch``) and laplacian_rigid_energy_pytorch.py
(``LaplacianRigidEnergyPytorch``), on CUDA tensors.

Every step of a mesh render is a Function whose forward and backward are the project's kernels (csrc/scene_ops.cu,
csrc/fitter.cu, the rasteriser), so ``loss.backward()`` goes through a mesh render without leaving the device, and a
caller may add terms of its own to the loss or step the parameters with ``torch.optim``:

    ProjectPointsFunc      (points [N,3], camera) -> (ij [N,2], depths [N])            gradients for both outputs
    VertexNormalsFunc      (vertices [V,3], topology) -> vertex_normals [V,3]
    LitVertexColorsFunc    (vertex_normals, vertex_colors [V,C], light_directional [3] | None, light_ambient 0-d)
                           -> colours [V,C]
    RenderMesh2DFunc       (ij, colors, depths, edgeflags, DeviceScene, sigma) -> image [H,W,C] fp32
                           gradients to ij and colors (depths get none, as in the reference)
    RenderMesh2DTexturedFunc  (ij, uv, shade, texture, depths, edgeflags, DeviceScene, sigma) -> image [H,W,C] fp32
                           gradients to ij, uv, shade and texture (a textured mesh: Scene3D.render's uv branch)
    PoseFunc              (vertices, quaternion [4], translation [3]) -> qrot(q / |q|, v - mean v) + t
    RigidEnergyFunc        (vertices, DeviceLaplacianRigidEnergy) -> energy 0-d

All maths is fp64 but the rasteriser's (fp32 image and image gradients).  ``RenderMesh2DFunc`` and
``RenderMesh2DTexturedFunc`` follow the snapshot / replay rule of the 2D Functions (differentiable_renderer_pytorch.py):
the renderer keeps one forward state per slot, so if another forward has used the slot before ``backward`` runs, the
forward is replayed from the node's own copy of its inputs (depths and edge flags included).
"""

from __future__ import annotations

from typing import Any, Dict, Optional, Tuple

import numpy as np
import torch

from ..mesh_fitter import DeviceLaplacianRigidEnergy, new_scratch, pose, pose_backward
from ..mesh_ops import (CameraParams, MeshTopology, lit_vertex_colors, lit_vertex_colors_backward, project_points,
                        project_points_backward_f64)
from ..renderer import DeviceScene, default_renderer
from .differentiable_renderer_pytorch import check_scene_inputs, gradients_of, requested_grads

_scratch: Dict[torch.device, torch.Tensor] = {}


def _scratch_of(device: torch.device) -> torch.Tensor:
    """One zeroed reduction scratch per device, shared by the Functions: its users are ordered by the stream of the
    forward (autograd runs a node's backward on the stream its forward ran on)."""
    if device not in _scratch:
        _scratch[device] = new_scratch(device)
    return _scratch[device]


def _f64(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.float64).contiguous()


# ---- Functions ------------------------------------------------------------------------------------------------------


class ProjectPointsFunc(torch.autograd.Function):
    """``Camera.project_points``: (points [N,3], camera) -> (ij [N,2], depths [N]), fp64; backward is the true adjoint
    (deodr_b200_project_points_b64) of whichever outputs received a gradient."""

    @staticmethod
    def forward(ctx: Any, points: torch.Tensor, camera: CameraParams):  # type: ignore
        p = _f64(points)
        ij, depths = project_points(p, camera)
        ctx.save_for_backward(p)
        ctx.camera, ctx.dtype = camera, points.dtype
        ctx.set_materialize_grads(False)
        return ij, depths

    @staticmethod
    def backward(ctx: Any, ij_b: Optional[torch.Tensor], depths_b: Optional[torch.Tensor]):  # type: ignore
        (p,) = ctx.saved_tensors
        if ij_b is None and depths_b is None:
            return None, None
        return project_points_backward_f64(p, ctx.camera, ij_b, depths_b).to(ctx.dtype), None


class VertexNormalsFunc(torch.autograd.Function):
    """``compute_vertex_normals(compute_face_normals(vertices))``: (vertices [V,3], MeshTopology) -> vertex_normals
    [V,3] fp64 (deodr_b200_vertex_normals / _b)."""

    @staticmethod
    def forward(ctx: Any, vertices: torch.Tensor, topology: MeshTopology):  # type: ignore
        v = _f64(vertices)
        _, vn = topology.vertex_normals(v)
        ctx.save_for_backward(v)
        ctx.topology, ctx.dtype = topology, vertices.dtype
        return vn

    @staticmethod
    def backward(ctx: Any, vn_b: torch.Tensor):  # type: ignore
        (v,) = ctx.saved_tensors
        return ctx.topology.vertex_normals_backward(v, vn_b).to(ctx.dtype), None


class LitVertexColorsFunc(torch.autograd.Function):
    """``Scene3DPytorch._compute_vertices_colors_with_illumination``: (vertex_normals [V,3], vertex_colors [V,C],
    light_directional [3] or None, light_ambient 0-d) -> colours [V,C] fp64 = vertex_colors * (relu(-<n, l>) +
    ambient), with the light on the device (deodr_b200_lit_vertex_colors / _b: its gradient summed in a fixed
    order)."""

    @staticmethod
    def forward(ctx: Any, normals: torch.Tensor, vertex_colors: torch.Tensor,  # type: ignore
                light_directional: Optional[torch.Tensor], light_ambient: torch.Tensor):
        dev = vertex_colors.device
        amb = _f64(light_ambient).reshape(1)
        directional = light_directional is not None
        ld = _f64(light_directional).reshape(3) if directional else torch.zeros(3, dtype=torch.float64, device=dev)
        light = torch.cat((ld, amb))
        n, vc = _f64(normals), _f64(vertex_colors)
        ctx.save_for_backward(n, vc, light)
        ctx.directional = directional
        ctx.dtypes = (normals.dtype, vertex_colors.dtype, light_directional.dtype if directional else None,
                      light_ambient.dtype)
        ctx.ambient_shape = light_ambient.shape
        return lit_vertex_colors(n, vc, light, directional)

    @staticmethod
    def backward(ctx: Any, colors_b: torch.Tensor):  # type: ignore
        n, vc, light = ctx.saved_tensors
        normals_b, vcol_b, light_b = lit_vertex_colors_backward(n, vc, light, colors_b, _scratch_of(n.device),
                                                                ctx.directional)
        nd, cd, ld, ad = ctx.dtypes
        return (normals_b.to(nd), vcol_b.to(cd), light_b[:3].to(ld) if ctx.directional else None,
                light_b[3].reshape(ctx.ambient_shape).to(ad))


class RenderMesh2DFunc(torch.autograd.Function):
    """The rasteriser under a 3D render: (ij [V,2], colors [V,C], depths [V], edgeflags [T,3], DeviceScene, sigma)
    -> image [H,W,C] fp32.  Backward returns ``(ij_b, colors_b, None, ...)``: no gradient for the depths, as in the
    reference, whose 2D Function does not take them.  The node snapshots all four inputs and replays the forward
    when another forward has used the renderer's slot before its ``backward``."""

    @staticmethod
    def forward(ctx: Any, ij: torch.Tensor, colors: torch.Tensor, depths: torch.Tensor,  # type: ignore
                edgeflags: torch.Tensor, scene: DeviceScene, sigma: float = 1.0):
        inputs = {"ij": ij.detach(), "colors": colors.detach(), "depths": depths.detach(), "edgeflags": edgeflags}
        scene.update(**inputs)
        fwd = default_renderer(scene.device.index).render(scene, sigma)
        ctx.scene, ctx.sigma, ctx.fwd = scene, float(sigma), fwd
        ctx.in_dtypes = (ij.dtype, colors.dtype)
        ctx.save_for_backward(*(t.clone() for t in inputs.values()))
        # the caller gets its own tensor: the framebuffers of ctx.fwd may be re-rendered into by backward
        return fwd["image"].clone()

    @staticmethod
    def backward(ctx: Any, image_b: torch.Tensor):  # type: ignore
        renderer = default_renderer(ctx.scene.device.index)
        ij, colors, depths, edgeflags = ctx.saved_tensors
        # the shared scene may hold another node's inputs by now
        ctx.scene.update(ij=ij, colors=colors, depths=depths, edgeflags=edgeflags)
        if ctx.fwd["generation"] != renderer.generation(ctx.fwd["slot"]):
            ctx.fwd = renderer.render(ctx.scene, ctx.sigma, out=ctx.fwd)
        grads = renderer.render_b(ctx.scene, ctx.sigma, ctx.fwd, image_b.contiguous())
        return grads["ij_b"].to(ctx.in_dtypes[0]), grads["colors_b"].to(ctx.in_dtypes[1]), None, None, None, None


class RenderMesh2DTexturedFunc(torch.autograd.Function):
    """The rasteriser under a textured 3D render: (ij [V,2], uv [Nuv,2], shade [V], texture [Ht,Wt,C], depths [V],
    edgeflags [T,3], DeviceScene, sigma) -> image [H,W,C] fp32, on a scene whose triangles are all textured and shaded
    and whose colours are zero.  Backward returns the gradients of ij, uv, shade and texture that autograd asks for
    (the texture's adjoint slot stays NULL when its gradient is not asked for), none for the depths and edge flags.  Same snapshot / replay rule as
    ``RenderMesh2DFunc``, over all six inputs."""

    NAMES = ("ij", "uv", "shade", "texture")

    @staticmethod
    def forward(ctx: Any, ij: torch.Tensor, uv: torch.Tensor, shade: torch.Tensor, texture: torch.Tensor,  # type: ignore
                depths: torch.Tensor, edgeflags: torch.Tensor, scene: DeviceScene, sigma: float = 1.0):
        check_scene_inputs(scene, uv=uv, texture=texture)
        inputs = {"ij": ij.detach(), "uv": uv.detach(), "shade": shade.detach(), "texture": texture.detach(),
                  "depths": depths.detach(), "edgeflags": edgeflags}
        scene.update(**inputs)
        fwd = default_renderer(scene.device.index).render(scene, sigma)
        ctx.scene, ctx.sigma, ctx.fwd = scene, float(sigma), fwd
        ctx.in_dtypes = (ij.dtype, uv.dtype, shade.dtype, texture.dtype)
        ctx.save_for_backward(*(t.clone() for t in inputs.values()))
        # the caller gets its own tensor: the framebuffers of ctx.fwd may be re-rendered into by backward
        return fwd["image"].clone()

    @staticmethod
    def backward(ctx: Any, image_b: torch.Tensor):  # type: ignore
        names = RenderMesh2DTexturedFunc.NAMES
        needs = ctx.needs_input_grad[:4]
        if not any(needs):
            return (None,) * 8
        renderer = default_renderer(ctx.scene.device.index)
        # the shared scene may hold another node's inputs by now
        ctx.scene.update(**dict(zip(names + ("depths", "edgeflags"), ctx.saved_tensors)))
        if ctx.fwd["generation"] != renderer.generation(ctx.fwd["slot"]):
            ctx.fwd = renderer.render(ctx.scene, ctx.sigma, out=ctx.fwd)
        grads = requested_grads(ctx.scene, names, needs)
        renderer.render_b(ctx.scene, ctx.sigma, ctx.fwd, image_b.contiguous(), grads=grads)
        return gradients_of(grads, names, ctx.in_dtypes, needs) + (None,) * 4


class PoseFunc(torch.autograd.Function):
    """(vertices [V,3], quaternion [4], translation [3]) -> qrot(q / |q|, v - mean v) + t, fp64 (deodr_b200_pose /
    _pose_b; quaternion stored x, y, z, w).  The input is not modified: the kernel centres a copy."""

    @staticmethod
    def forward(ctx: Any, vertices: torch.Tensor, quaternion: torch.Tensor, translation: torch.Tensor):  # type: ignore
        centred = vertices.detach().to(torch.float64).clone(memory_format=torch.contiguous_format)
        q, t = _f64(quaternion), _f64(translation)
        out = pose(centred, q, t, _scratch_of(centred.device))
        ctx.save_for_backward(centred, q)
        ctx.dtypes = (vertices.dtype, quaternion.dtype, translation.dtype)
        return out

    @staticmethod
    def backward(ctx: Any, out_b: torch.Tensor):  # type: ignore
        centred, q = ctx.saved_tensors
        v_b, q_b, t_b = pose_backward(centred, q, out_b.to(torch.float64).contiguous(), _scratch_of(centred.device))
        vd, qd, td = ctx.dtypes
        return v_b.to(vd), q_b.to(qd), t_b.to(td)


class RigidEnergyFunc(torch.autograd.Function):
    """(vertices [V,3], DeviceLaplacianRigidEnergy) -> (energy 0-d fp64 = 1/2 <v - v_ref, grad>, grad [V,3] =
    cregu L^T L (v - v_ref)); the energy's backward is ``grad_out * grad``, ``grad`` is not differentiable."""

    @staticmethod
    def forward(ctx: Any, vertices: torch.Tensor, energy_model: DeviceLaplacianRigidEnergy):  # type: ignore
        energy, grad = energy_model.evaluate(_f64(vertices))
        ctx.save_for_backward(grad)
        ctx.dtype = vertices.dtype
        ctx.mark_non_differentiable(grad)
        ctx.set_materialize_grads(False)
        return energy, grad

    @staticmethod
    def backward(ctx: Any, energy_b: Optional[torch.Tensor], grad_b: Optional[torch.Tensor]):  # type: ignore
        if energy_b is None:
            return None, None
        (grad,) = ctx.saved_tensors
        return (energy_b * grad).to(ctx.dtype), None


project_points_autograd = ProjectPointsFunc.apply
vertex_normals_autograd = VertexNormalsFunc.apply
lit_vertex_colors_autograd = LitVertexColorsFunc.apply
render_mesh_2d = RenderMesh2DFunc.apply
render_mesh_2d_textured = RenderMesh2DTexturedFunc.apply
pose_autograd = PoseFunc.apply
rigid_energy_autograd = RigidEnergyFunc.apply


def vertex_luminosity_autograd(normals: torch.Tensor, light_directional: Optional[torch.Tensor],
                               light_ambient: torch.Tensor) -> torch.Tensor:
    """``Scene3D.compute_vertices_luminosity``: [V] fp64 = relu(-<n, l>) + ambient, :class:`LitVertexColorsFunc` on a
    column of ones (the same arithmetic as ``mesh_ops.vertex_luminosity``, rounded to fp32 only by the rasteriser)."""
    ones = torch.ones((normals.shape[0], 1), dtype=torch.float64, device=normals.device)
    return lit_vertex_colors_autograd(normals, ones, light_directional, light_ambient)[:, 0]


# ---- the reference's classes ------------------------------------------------------------------------------------------


def _device(device) -> torch.device:
    dev = torch.device(device if device is not None else "cuda")
    if dev.type == "cuda" and dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


class CameraPytorch(CameraParams):
    """``deodr.pytorch.CameraPytorch(extrinsic, intrinsic, height, width, distortion=None)``: the pinhole camera with
    OpenCV distortion, projecting CUDA tensors through :class:`ProjectPointsFunc`."""

    def __init__(self, extrinsic, intrinsic, height: int, width: int, distortion=None):
        super().__init__(extrinsic, intrinsic, distortion)
        self.height, self.width = int(height), int(width)

    def project_points(self, points_3d: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """-> (ij [N,2], depths [N]), differentiable in ``points_3d``."""
        return project_points_autograd(points_3d, self)


class ColoredTriMeshPytorch:
    """``deodr.pytorch.ColoredTriMeshPytorch(faces, vertices, clockwise=False, colors=None)`` on the device: the
    vertices [V,3] and vertex colours [V,C] are CUDA tensors (either may require grad), the adjacency a
    :class:`MeshTopology` built once.

    ``faces_uv`` [T,3], ``uv`` [Nuv,2] and ``texture`` [Ht,Wt,C], given together, make the mesh textured, in the
    conventions of the reference's ``ColoredTriMesh`` (uv in texel units).  ``uv`` and ``texture`` are tensors (fp32 or
    fp64, either may require grad) or arrays, uploaded once; the attributes ``uv`` and ``texture`` may be reassigned
    between renders."""

    def __init__(self, faces, vertices, clockwise: bool = False, colors=None, device=None, faces_uv=None, uv=None,
                 texture=None):
        self.device = _device(device if device is not None else
                              (vertices.device if isinstance(vertices, torch.Tensor) else None))
        self.faces = np.ascontiguousarray(np.asarray(faces), dtype=np.int64)
        self.nb_faces = self.faces.shape[0]
        self.clockwise = bool(clockwise)
        self.set_vertices(vertices)
        self.nb_vertices = self.vertices.shape[0]
        self.topology = MeshTopology(self.faces, self.nb_vertices, clockwise=self.clockwise, device=self.device)
        self.vertices_colors = None
        if colors is not None:
            self.set_vertices_colors(colors)
        self.faces_uv = self.uv = self.texture = None
        if faces_uv is not None or uv is not None or texture is not None:
            if faces_uv is None or uv is None or texture is None:
                raise ValueError("a textured mesh needs faces_uv, uv and texture together")
            self.uv, self.texture = self._tensor(uv), self._tensor(texture)
            self.faces_uv = np.ascontiguousarray(np.asarray(faces_uv), dtype=np.int64)
            if self.texture.dim() != 3:
                raise ValueError(f"texture must be [Ht,Wt,C]; got shape {tuple(self.texture.shape)}")
            if self.uv.dim() != 2 or self.uv.shape[1] != 2 or self.faces_uv.shape != self.faces.shape:
                raise ValueError(f"uv must be [Nuv,2] and faces_uv [T,3] like faces = {self.faces.shape}; got "
                                 f"{tuple(self.uv.shape)} and {self.faces_uv.shape}")
            # the rasteriser reads uv through faces_uv unchecked
            if self.faces_uv.size and (self.faces_uv.min() < 0 or self.faces_uv.max() >= self.uv.shape[0]):
                raise ValueError(f"faces_uv indices must lie in [0, {self.uv.shape[0]})")

    @property
    def textured(self) -> bool:
        return self.faces_uv is not None

    def _tensor(self, a) -> torch.Tensor:
        if isinstance(a, torch.Tensor):
            return a if a.device == self.device else a.to(self.device)
        return torch.as_tensor(np.asarray(a, dtype=np.float64), device=self.device)

    def set_vertices(self, vertices) -> None:
        self.vertices = self._tensor(vertices)

    def set_vertices_colors(self, colors) -> None:
        self.vertices_colors = self._tensor(colors)

    @property
    def vertex_normals(self) -> torch.Tensor:
        """Unit vertex normals [V,3] fp64 of the current vertices, differentiable."""
        return vertex_normals_autograd(self.vertices, self.topology)


class Scene3DPytorch:
    """``deodr.pytorch.Scene3DPytorch`` on the device: ``set_mesh``, ``set_light(light_directional, light_ambient)``,
    ``set_background_color``, ``render(camera)`` -> image [H,W,C] and ``render_depth(camera, depth_scale)`` -> [H,W,1],
    fp32 CUDA tensors differentiable in the mesh's vertices and colours (or uv and texture, for a textured mesh) and in
    the light.

    A render is the chain of Functions of this module; ``sigma`` is the antialiasing width of the reference's Scene3D
    (1 by default; at 0 no silhouette edge is drawn).  The backgrounds are set on the device by
    ``set_background_color``, so a render copies nothing from the host."""

    def __init__(self, sigma: float = 1.0, backface_culling: bool = True):
        self.sigma = float(sigma)
        self.backface_culling = bool(backface_culling)
        self.mesh: Optional[ColoredTriMeshPytorch] = None
        self.light_directional: Optional[torch.Tensor] = None
        self.light_ambient: Optional[torch.Tensor] = None
        self.background_color: Optional[np.ndarray] = None
        self._scenes: Dict[tuple, DeviceScene] = {}

    def set_mesh(self, mesh: ColoredTriMeshPytorch) -> None:
        self.mesh = mesh
        self._scenes = {}

    def set_light(self, light_directional, light_ambient) -> None:
        """``light_directional`` [3] (None: ambient light only) and ``light_ambient`` (a number or 0-d tensor); tensors
        are used as given, so a light that requires grad receives its gradient."""
        dev = self.mesh.device if self.mesh is not None else _device(None)
        if light_directional is not None and not isinstance(light_directional, torch.Tensor):
            light_directional = torch.as_tensor(np.asarray(light_directional, dtype=np.float64), device=dev)
        if not isinstance(light_ambient, torch.Tensor):
            light_ambient = torch.tensor(float(light_ambient), dtype=torch.float64, device=dev)
        self.light_directional, self.light_ambient = light_directional, light_ambient

    def set_background_color(self, background_color) -> None:
        self.background_color = np.array(background_color, dtype=np.float64).reshape(-1)
        for scene in self._scenes.values():
            if scene.nb_colors == self.background_color.shape[0]:
                scene.t["background_color"].copy_(torch.from_numpy(self.background_color))

    def _scene(self, camera: CameraPytorch, nb_colors: int, uv: Optional[torch.Tensor] = None,
               texture: Optional[torch.Tensor] = None) -> DeviceScene:
        """The cached 2D scene of the mesh for ``camera``: untextured, or with ``uv`` / ``texture`` given, textured
        (all triangles textured and shaded, colours zero; the mesh's faces_uv uploaded with it)."""
        from ..scenes import SceneArrays

        if self.background_color is None:
            raise ValueError("set_background_color first")
        if self.background_color.shape[0] != nb_colors:
            raise ValueError(f"the background colour has {self.background_color.shape[0]} entries and the render "
                             f"{nb_colors} channels")
        textured = texture is not None
        key = (camera.height, camera.width, nb_colors) + ((tuple(texture.shape), uv.shape[0]) if textured else ())
        if key not in self._scenes:
            m = self.mesh
            T, V = m.nb_faces, m.nb_vertices
            faces = np.ascontiguousarray(m.faces, dtype=np.uint32)
            flags = np.full(T, textured)
            self._scenes[key] = DeviceScene(SceneArrays(
                faces=faces, faces_uv=np.ascontiguousarray(m.faces_uv, dtype=np.uint32) if textured else faces,
                ij=np.zeros((V, 2)), depths=np.ones(V), textured=flags,
                uv=np.zeros((uv.shape[0] if textured else V, 2)), shade=np.zeros(V), colors=np.zeros((V, nb_colors)),
                shaded=flags, edgeflags=np.zeros((T, 3), bool), height=camera.height, width=camera.width,
                nb_colors=nb_colors, texture=np.zeros(tuple(texture.shape) if textured else (2, 2, nb_colors)),
                background_image=None, background_color=self.background_color, clockwise=m.clockwise,
                backface_culling=self.backface_culling, strict_edge=True, perspective_correct=False,
                integer_pixel_centers=True), m.device)
        return self._scenes[key]

    def _edgeflags(self, ij: torch.Tensor) -> torch.Tensor:
        if self.sigma > 0:
            return self.mesh.topology.edge_on_silhouette(ij.detach())
        return torch.zeros((self.mesh.nb_faces, 3), dtype=torch.uint8, device=self.mesh.device)

    def _compute_vertices_colors_with_illumination(self) -> torch.Tensor:
        m = self.mesh
        if self.light_ambient is None:
            raise ValueError("set_light first")
        normals = m.vertex_normals if self.light_directional is not None else torch.zeros(
            (m.nb_vertices, 3), dtype=torch.float64, device=m.device)
        return lit_vertex_colors_autograd(normals, m.vertices_colors, self.light_directional, self.light_ambient)

    def _compute_vertices_luminosity(self) -> torch.Tensor:
        m = self.mesh
        if self.light_ambient is None:
            raise ValueError("set_light first")
        normals = m.vertex_normals if self.light_directional is not None else torch.zeros(
            (m.nb_vertices, 3), dtype=torch.float64, device=m.device)
        return vertex_luminosity_autograd(normals, self.light_directional, self.light_ambient)

    def render(self, camera: CameraPytorch) -> torch.Tensor:
        """The mesh's vertex colours, Gouraud-lit, rendered by ``camera`` -> image [H,W,C] fp32.  For a textured mesh,
        ``Scene3D.render``'s uv branch: the texture, sampled at the interpolated uv, times the interpolated vertex
        luminosity (differentiable in the vertices, uv, texture and light)."""
        if self.mesh is not None and self.mesh.textured:
            return self._render_textured(camera)
        if self.mesh is None or self.mesh.vertices_colors is None:
            raise ValueError("render needs a mesh with vertex colours (set_mesh, set_vertices_colors)")
        ij, depths = camera.project_points(self.mesh.vertices)
        colors = self._compute_vertices_colors_with_illumination()
        scene = self._scene(camera, colors.shape[1])
        return render_mesh_2d(ij, colors, depths, self._edgeflags(ij), scene, self.sigma)

    def _render_textured(self, camera: CameraPytorch) -> torch.Tensor:
        m = self.mesh
        uv, texture = m._tensor(m.uv), m._tensor(m.texture)
        if texture.dim() != 3 or uv.dim() != 2 or uv.shape[1] != 2:
            raise ValueError(f"a textured mesh needs texture [Ht,Wt,C] and uv [Nuv,2]; got {tuple(texture.shape)} and "
                             f"{tuple(uv.shape)}")
        if m.faces_uv.size and int(m.faces_uv.max()) >= uv.shape[0]:
            raise ValueError(f"uv has {uv.shape[0]} rows; faces_uv indexes row {int(m.faces_uv.max())}")
        ij, depths = camera.project_points(m.vertices)
        shade = self._compute_vertices_luminosity()
        scene = self._scene(camera, texture.shape[2], uv=uv, texture=texture)
        return render_mesh_2d_textured(ij, uv, shade, texture, depths, self._edgeflags(ij), scene, self.sigma)

    def render_depth(self, camera: CameraPytorch, depth_scale: float = 1.0) -> torch.Tensor:
        """``Scene3D.render_depth``: a one-channel image [H,W,1] fp32 whose colour is the vertex depth times
        ``depth_scale``, over the background colour (which must have one entry); differentiable through the depths."""
        if self.mesh is None:
            raise ValueError("set_mesh first")
        ij, depths = camera.project_points(self.mesh.vertices)
        scene = self._scene(camera, 1)
        return render_mesh_2d(ij, (depths * depth_scale)[:, None], depths, self._edgeflags(ij), scene, self.sigma)


class LaplacianRigidEnergyPytorch:
    """``deodr.pytorch.LaplacianRigidEnergyPytorch(mesh, vertices, cregu)`` on the device.  ``evaluate(v)`` ->
    ``(energy 0-d, grad [V,3], None)`` with grad = cregu L^T L (v - v_ref) and energy = 1/2 <v - v_ref, grad>.
    The energy is differentiable when ``v`` requires grad (the reference's own path for that case fails, INTEGRATION.md
    section 5); the approximate Hessian, the reference's third result, is not formed (None)."""

    def __init__(self, mesh, vertices, cregu: float, device=None):
        faces = mesh.faces if hasattr(mesh, "faces") else mesh
        dev = device if device is not None else getattr(mesh, "device", None)
        self.model = DeviceLaplacianRigidEnergy(np.asarray(faces), np.asarray(vertices, dtype=np.float64), cregu,
                                                _device(dev))
        self.cregu = float(cregu)

    def evaluate(self, vertices: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, None]:
        if vertices.requires_grad:
            energy, grad = rigid_energy_autograd(vertices, self.model)
            return energy, grad, None
        energy, grad = self.model.evaluate(vertices)
        return energy, grad, None
