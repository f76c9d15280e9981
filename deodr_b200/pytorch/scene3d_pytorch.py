"""autograd surface of the 3D render, mirroring deodr/pytorch/differentiable_renderer_pytorch.py (``CameraPytorch``,
``Scene3DPytorch``), triangulated_mesh_pytorch.py (``ColoredTriMeshPytorch``) and laplacian_rigid_energy_pytorch.py
(``LaplacianRigidEnergyPytorch``), on CUDA tensors.

Every step of a mesh render is a Function whose forward and backward are the project's kernels (csrc/scene_ops.cu,
csrc/fitter.cu, the rasteriser), so ``loss.backward()`` goes through a mesh render without leaving the device, and a
caller may add terms of its own to the loss or step the parameters with ``torch.optim``:

    ProjectPointsFunc      (points [N,3], camera) -> (ij [N,2], depths [N])            gradients for both outputs;
                           a camera vector [26] as camera receives its gradient too
    VertexNormalsFunc      (vertices [V,3], topology) -> vertex_normals [V,3]
    LitVertexColorsFunc    (vertex_normals, vertex_colors [V,C], light_directional [3] | None, light_ambient 0-d)
                           -> colours [V,C]
    ShLitVertexColorsFunc  (vertex_normals, vertex_colors [V,C] | None, light_directional, light_ambient, sh [9] |
                           [9,C]) -> colours [V,C] (luminosity [V] without vertex colours) under a spherical-harmonics
                           environment too; sh receives its gradient
    PointLitVertexColorsFunc  (vertex_normals, vertices [V,3], vertex_colors [V,C] | None, light_directional,
                           light_ambient, sh | None, point_lights [L, 3 + S]) -> colours [V,C] (luminosity [V] without
                           vertex colours) under point lights too; the vertices and the lights receive their gradients
    RenderMesh2DFunc       (ij, colors, depths, edgeflags, DeviceScene, sigma) -> image [H,W,C] fp32
                           gradients to ij and colors (depths get none, as in the reference)
    RenderMesh2DTexturedFunc  (ij, uv, shade, texture, depths, edgeflags, DeviceScene, sigma) -> image [H,W,C] fp32
                           gradients to ij, uv, shade and texture (a textured mesh: Scene3D.render's uv branch)
    PoseFunc              (vertices, quaternion [4], translation [3]) -> qrot(q / |q|, v - mean v) + t
    RigidEnergyFunc        (vertices, DeviceLaplacianRigidEnergy) -> energy 0-d
    SelfCollisionEnergyFunc (vertices, DeviceSelfCollisionEnergy) -> energy 0-d
    LoopSubdivisionFunc    (vertices [V,3], colors [V,C] | None, LoopSubdivision) -> (fine vertices, fine colours)
                           the reference's Loop subdivision (ColoredTriMeshPytorch.subdivise), its transpose backward
    PhongShadeFunc         (channels [H,W,C+7], light_directional [3] | None, light_ambient, specular, shininess,
                           camera or its centre [3], background [C], sh [9] | [9,C] | None, albedo [H,W,C] | None)
                           -> image [H,W,C] fp32, the per-pixel shading of a G-buffer; a centre tensor and sh receive
                           their gradients.  With a separate albedo the G-buffer is [H,W,7] and the albedo gets one;
                           point_lights [L, 3 + S] | None get theirs; the specular map's raster [H,W,2] | None (with
                           the albedo) gives the per-pixel ks and e, and receives its gradient.  brdf="ggx" is the
                           metallic-roughness form: specular and shininess are the metallic and roughness factors,
                           and the 2-channel raster is the metallic-roughness map's
    RenderMeshPhongTexturedFunc  (ij, uv, texture, channels [V,7], depths, edgeflags, albedo scene, G-buffer scene,
                           sigma) -> (albedo [H,W,C], G-buffer [H,W,7]): the two rasters of a textured Phong render
                           in one forward call and one adjoint call; gradients to ij, uv, texture and channels.  With
                           a normal map [Ht,Wt,3] and its scene, channels are [V,13] and a third raster, the map's
                           [H,W,3], is rendered in the same calls; the map receives its gradient.  With a specular map
                           [Ht,Wt,2] (or a metallic-roughness map) and its scene, one more raster, the map's [H,W,2],
                           is rendered last in the same calls; the map receives its gradient
    RenderShadowedPhongFunc  (ij, uv | None, texture | None, channels, depths, edgeflags, vertices, point_lights,
                           albedo scene | None, G-buffer scene, ShadowCubes, sigma) -> ([albedo,] G-buffer, cube maps
                           [6L,M,M]): a Phong render's raster(s) and the lights' cube shadow maps in one forward call
                           and one adjoint call; the maps' share reaches the vertices and the lights' positions.  A
                           textured render's normal map and specular map add their rasters as above
    ShadowVisibilityFunc   (G-buffer, point_lights, maps, bias, softness, albedo | None) -> visibility [H,W,L]; the
                           G-buffer, the maps and the lights' positions receive their gradients
    SunVisibilityFunc      (G-buffer, light_directional [3], map [M,M], bounds, bias, softness, albedo | None) ->
                           visibility [H,W] of the directional light; the G-buffer, the map and the light receive
                           their gradients
    VertexTangentsFunc     (vertices [V,3], uv [Nuv,2], VertexTangents) -> frames [V,6] = (T, B), the per-vertex
                           tangent frames of a normal-mapped mesh; the vertices and the uv receive their gradients
    NormalMapFunc          (G-buffer [H,W,13], map raster [H,W,3]) -> G-buffer [H,W,7], the normal map's per-pixel
                           perturbation; both inputs receive their gradients

All maths is fp64 but the rasteriser's (fp32 image and image gradients).  ``RenderMesh2DFunc``,
``RenderMesh2DTexturedFunc`` and ``RenderMeshPhongTexturedFunc`` follow the snapshot / replay rule of the 2D Functions (differentiable_renderer_pytorch.py):
the renderer keeps one forward state per slot, so if another forward has used the slot before ``backward`` runs, the
forward is replayed from the node's own copy of its inputs (depths and edge flags included).
"""

from __future__ import annotations

from typing import Any, Dict, Optional, Tuple

import numpy as np
import torch

from ..mesh_fitter import DeviceLaplacianRigidEnergy, DeviceSelfCollisionEnergy, new_scratch, pose, pose_backward
from ..mesh_ops import (CameraParams, LinearBlendSkinning, LoopSubdivision, MeshTopology, camera_center,
                        lit_vertex_colors,
                        ShadowCubes, SunShadowMap, check_shadow_arguments, check_sun_shadow_arguments,
                        cube_project_backward, lit_vertex_colors_backward, sun_project_backward, sun_visibility,
                        sun_visibility_backward,
                        phong_shade, phong_shade_backward, project_points, shadow_visibility,
                        shadow_visibility_backward,
                        point_lit_vertex_colors, point_lit_vertex_colors_backward, sh_lit_vertex_colors,
                        sh_lit_vertex_colors_backward,
                        project_points_backward_f64, project_points_camera_backward, project_points_dev,
                        VertexTangents, normal_map, normal_map_backward)
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
    (deodr_b200_project_points_b64) of whichever outputs received a gradient.

    ``camera`` is a :class:`CameraParams` (a constant), or a camera vector [26] fp64 tensor on the points' device
    (``mesh_ops.CameraParams.vector``'s layout) with ``has_distortion`` saying whether its distortion is applied: it is
    read on the device (deodr_b200_project_points_dev) and gets its gradient from the fused adjoint
    (deodr_b200_project_points_camera_b)."""

    @staticmethod
    def forward(ctx: Any, points: torch.Tensor, camera, has_distortion: bool = False):  # type: ignore
        p = _f64(points)
        ctx.dtype = points.dtype
        ctx.set_materialize_grads(False)
        if isinstance(camera, torch.Tensor):
            cam = _f64(camera)
            ij, depths = project_points_dev(p, cam, has_distortion)
            ctx.save_for_backward(p, cam)
            ctx.camera, ctx.has_distortion, ctx.camera_dtype = None, bool(has_distortion), camera.dtype
            return ij, depths
        ij, depths = project_points(p, camera)
        ctx.save_for_backward(p)
        ctx.camera = camera
        return ij, depths

    @staticmethod
    def backward(ctx: Any, ij_b: Optional[torch.Tensor], depths_b: Optional[torch.Tensor]):  # type: ignore
        if ij_b is None and depths_b is None:
            return None, None, None
        if ctx.camera is not None:
            (p,) = ctx.saved_tensors
            return project_points_backward_f64(p, ctx.camera, ij_b, depths_b).to(ctx.dtype), None, None
        p, cam = ctx.saved_tensors
        need_p = ctx.needs_input_grad[0]
        points_b = torch.empty_like(p) if need_p else None
        camera_b = project_points_camera_backward(p, cam, ctx.has_distortion, ij_b, depths_b, _scratch_of(p.device),
                                                  points_b=points_b, accumulate=False)
        return (points_b.to(ctx.dtype) if need_p else None,
                camera_b.to(ctx.camera_dtype) if ctx.needs_input_grad[1] else None, None)


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


class ShLitVertexColorsFunc(torch.autograd.Function):
    """:class:`LitVertexColorsFunc` with a spherical-harmonics environment (the model in include/deodr_b200.h):
    (vertex_normals [V,3], vertex_colors [V,C] or None, light_directional [3] or None, light_ambient 0-d, sh [9] or
    [9,S]) -> colours [V,C] fp64 = vertex_colors * ((relu(-<n, l>) + ambient) + sh_c(n)), or the luminosity [V] of
    a grey environment without vertex colours (deodr_b200_sh_lit_vertex_colors / _b: light and sh gradients summed in
    a fixed order)."""

    @staticmethod
    def forward(ctx: Any, normals: torch.Tensor, vertex_colors: Optional[torch.Tensor],  # type: ignore
                light_directional: Optional[torch.Tensor], light_ambient: torch.Tensor, sh: torch.Tensor):
        dev = normals.device
        amb = _f64(light_ambient).reshape(1)
        directional = light_directional is not None
        ld = _f64(light_directional).reshape(3) if directional else torch.zeros(3, dtype=torch.float64, device=dev)
        light = torch.cat((ld, amb))
        n, shd = _f64(normals), _f64(sh)
        vc = _f64(vertex_colors) if vertex_colors is not None else None
        ctx.save_for_backward(n, vc, light, shd)
        ctx.directional = directional
        ctx.dtypes = (normals.dtype, vertex_colors.dtype if vc is not None else None,
                      light_directional.dtype if directional else None, light_ambient.dtype, sh.dtype)
        ctx.ambient_shape = light_ambient.shape
        return sh_lit_vertex_colors(n, vc, light, shd, directional)

    @staticmethod
    def backward(ctx: Any, colors_b: torch.Tensor):  # type: ignore
        n, vc, light, shd = ctx.saved_tensors
        normals_b, vcol_b, light_b, sh_b = sh_lit_vertex_colors_backward(n, vc, light, shd, colors_b,
                                                                         _scratch_of(n.device), ctx.directional)
        nd, cd, ld, ad, sd = ctx.dtypes
        return (normals_b.to(nd), vcol_b.to(cd) if vcol_b is not None else None,
                light_b[:3].to(ld) if ctx.directional else None, light_b[3].reshape(ctx.ambient_shape).to(ad),
                sh_b.to(sd))


class PointLitVertexColorsFunc(torch.autograd.Function):
    """:class:`ShLitVertexColorsFunc` with point lights (the model in include/deodr_b200.h): (vertex_normals [V,3],
    vertices [V,3], vertex_colors [V,C] or None, light_directional [3] or None, light_ambient 0-d, sh [9] | [9,S] | None,
    point_lights [L, 3 + S]) -> colours [V,C] fp64 = vertex_colors * (((relu(-<n, l>) + ambient) + sh_c(n)) + P_c(n,
    x)), or the luminosity [V] under grey lights without vertex colours (deodr_b200_point_lit_vertex_colors / _b: the
    light, sh and point-light gradients summed in a fixed order)."""

    @staticmethod
    def forward(ctx: Any, normals: torch.Tensor, vertices: torch.Tensor,  # type: ignore
                vertex_colors: Optional[torch.Tensor], light_directional: Optional[torch.Tensor],
                light_ambient: torch.Tensor, sh: Optional[torch.Tensor], point_lights: torch.Tensor):
        dev = normals.device
        amb = _f64(light_ambient).reshape(1)
        directional = light_directional is not None
        ld = _f64(light_directional).reshape(3) if directional else torch.zeros(3, dtype=torch.float64, device=dev)
        light = torch.cat((ld, amb))
        n, x, pl = _f64(normals), _f64(vertices), _f64(point_lights)
        vc = _f64(vertex_colors) if vertex_colors is not None else None
        shd = _f64(sh) if sh is not None else None
        ctx.save_for_backward(n, x, vc, light, shd, pl)
        ctx.directional = directional
        ctx.dtypes = (normals.dtype, vertices.dtype, vertex_colors.dtype if vc is not None else None,
                      light_directional.dtype if directional else None, light_ambient.dtype,
                      sh.dtype if sh is not None else None, point_lights.dtype)
        ctx.ambient_shape = light_ambient.shape
        return point_lit_vertex_colors(n, x, vc, light, pl, sh=shd, directional=directional)

    @staticmethod
    def backward(ctx: Any, colors_b: torch.Tensor):  # type: ignore
        n, x, vc, light, shd, pl = ctx.saved_tensors
        normals_b, positions_b, vcol_b, light_b, sh_b, lights_b = point_lit_vertex_colors_backward(
            n, x, vc, light, pl, colors_b, _scratch_of(n.device), sh=shd, directional=ctx.directional)
        nd, xd, cd, ld, ad, sd, pd = ctx.dtypes
        return (normals_b.to(nd), positions_b.to(xd), vcol_b.to(cd) if vcol_b is not None else None,
                light_b[:3].to(ld) if ctx.directional else None, light_b[3].reshape(ctx.ambient_shape).to(ad),
                sh_b.to(sd) if sh_b is not None else None, lights_b.to(pd))


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


class RenderMeshPhongTexturedFunc(torch.autograd.Function):
    """The two rasters of a textured Phong render (``DeviceMeshView(shading="phong_textured")``'s model), as one node:
    (ij [V,2], uv [Nuv,2], texture [Ht,Wt,C], channels [V,7] = (unit normals, vertices, 1), depths [V], edgeflags
    [T,3], albedo scene, G-buffer scene, sigma) -> (albedo [H,W,C], G-buffer [H,W,7]) fp32.  The albedo scene is
    textured with a shade of 1 over a zero background, the G-buffer scene untextured with 7 channels over a zero
    background; both share ij, depths and edge flags.  The forward is one ``render_views`` call and the adjoint one
    ``render_b_views`` call; the two ij gradients are summed.  Same snapshot / replay rule as ``RenderMesh2DFunc``,
    over both slots: a backward right after its forward replays nothing.  The rasters are [albedo, G-buffer, normal
    map's (with one), specular map's (with one)]."""

    NAMES = ("ij", "uv", "shade", "texture")

    @staticmethod
    def forward(ctx: Any, ij: torch.Tensor, uv: torch.Tensor, texture: torch.Tensor,  # type: ignore
                channels: torch.Tensor, depths: torch.Tensor, edgeflags: torch.Tensor, albedo_scene: DeviceScene,
                gbuffer_scene: DeviceScene, sigma: float = 1.0, normal_map: Optional[torch.Tensor] = None,
                map_scene: Optional[DeviceScene] = None, specular_map: Optional[torch.Tensor] = None,
                spec_scene: Optional[DeviceScene] = None):
        if (normal_map is None) != (map_scene is None) or (specular_map is None) != (spec_scene is None):
            raise ValueError("a normal map or a specular map comes with its scene")
        check_scene_inputs(albedo_scene, uv=uv, texture=texture)
        check_scene_inputs(gbuffer_scene, colors=channels)
        scenes = [albedo_scene, gbuffer_scene]
        for m, sc in ((normal_map, map_scene), (specular_map, spec_scene)):
            if sc is not None:
                check_scene_inputs(sc, uv=uv, texture=m)
                scenes.append(sc)
        inputs = (ij.detach(), uv.detach(), texture.detach(), channels.detach(), depths.detach(), edgeflags,
                  normal_map.detach() if normal_map is not None else None,
                  specular_map.detach() if specular_map is not None else None)
        RenderMeshPhongTexturedFunc._update(scenes, *inputs)
        fwds = default_renderer(albedo_scene.device.index).render_views(scenes, sigma)
        ctx.scenes, ctx.sigma, ctx.fwds = scenes, float(sigma), fwds
        ctx.in_dtypes = (ij.dtype, uv.dtype, texture.dtype, channels.dtype,
                         normal_map.dtype if normal_map is not None else None,
                         specular_map.dtype if specular_map is not None else None)
        ctx.save_for_backward(*(t.clone() if t is not None else None for t in inputs))
        # the caller gets its own tensors: the framebuffers of ctx.fwds may be re-rendered into by backward
        return tuple(f["image"].clone() for f in fwds)

    @staticmethod
    def _update(scenes, ij, uv, texture, channels, depths, edgeflags, normal_map, specular_map) -> None:
        scenes[0].update(ij=ij, uv=uv, texture=texture, depths=depths, edgeflags=edgeflags)
        scenes[1].update(ij=ij, colors=channels, depths=depths, edgeflags=edgeflags)
        for sc, m in zip(scenes[2:], [t for t in (normal_map, specular_map) if t is not None]):
            sc.update(ij=ij, uv=uv, texture=m, depths=depths, edgeflags=edgeflags)

    @staticmethod
    def backward(ctx: Any, *image_bs):  # type: ignore
        ng = ctx.needs_input_grad
        needs = ng[:4] + ng[9:10] + ng[11:12]
        if not any(needs):
            return (None,) * 13
        scenes = ctx.scenes
        renderer = default_renderer(scenes[0].device.index)
        # the shared scenes may hold another node's inputs by now
        RenderMeshPhongTexturedFunc._update(scenes, *ctx.saved_tensors)
        if any(f["generation"] != renderer.generation(f["slot"]) for f in ctx.fwds):
            ctx.fwds = renderer.render_views(scenes, ctx.sigma, out=ctx.fwds)
        names = RenderMeshPhongTexturedFunc.NAMES
        ij_d, uv_d, tex_d, ch_d, nm_d, sm_d = ctx.in_dtypes
        # the map rasters and which of normal_map (4) and specular_map (5) each one's texture_b goes to
        maps = [k for k, d in ((4, nm_d), (5, sm_d)) if d is not None]
        grads = [requested_grads(scenes[0], names, (needs[0], needs[1], False, needs[2])), scenes[1].zero_grads()]
        grads += [requested_grads(sc, names, (needs[0], needs[1], False, needs[k])) for sc, k in zip(scenes[2:], maps)]
        renderer.render_b_views(scenes, ctx.sigma, ctx.fwds, [b.contiguous() for b in image_bs], grads=grads)
        ga, gg = grads[:2]
        ij_b, uv_b = ga["ij_b"] + gg["ij_b"], ga["uv_b"]
        map_b = {}
        for g, k in zip(grads[2:], maps):
            ij_b, uv_b = ij_b + g["ij_b"], uv_b + g["uv_b"]
            map_b[k] = g["texture_b"].to(nm_d if k == 4 else sm_d) if needs[k] else None
        return (ij_b.to(ij_d) if needs[0] else None, uv_b.to(uv_d) if needs[1] else None,
                ga["texture_b"].to(tex_d) if needs[2] else None, gg["colors_b"].to(ch_d) if needs[3] else None,
                None, None, None, None, None, map_b.get(4), None, map_b.get(5), None)


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


class SelfCollisionEnergyFunc(torch.autograd.Function):
    """(vertices [V,3], DeviceSelfCollisionEnergy) -> energy 0-d fp64; the backward is ``energy_b * grad`` with the
    gradient of the same evaluation."""

    @staticmethod
    def forward(ctx: Any, vertices: torch.Tensor, model: DeviceSelfCollisionEnergy):  # type: ignore
        energy, grad = model.evaluate(_f64(vertices))
        ctx.save_for_backward(grad)
        ctx.dtype = vertices.dtype
        return energy

    @staticmethod
    def backward(ctx: Any, energy_b: torch.Tensor):  # type: ignore
        (grad,) = ctx.saved_tensors
        return (energy_b * grad).to(ctx.dtype), None


class LoopSubdivisionFunc(torch.autograd.Function):
    """``ColoredTriMesh.subdivise``'s geometry: (vertices [V,3], colors [V,C] or None, LoopSubdivision) -> (fine
    vertices [V',3], fine colours [V',C] or None), fp64 (deodr_b200_loop_subdivide, one launch per level).  Subdivision
    is linear, so backward is the transpose (deodr_b200_loop_subdivide_b, levels in reverse, bit-reproducible) of
    whichever outputs received a gradient; nothing is saved but the levels."""

    @staticmethod
    def forward(ctx: Any, vertices: torch.Tensor, colors: Optional[torch.Tensor], sub: LoopSubdivision):  # type: ignore
        fv, fc = sub.apply(_f64(vertices), _f64(colors) if colors is not None else None)
        ctx.sub = sub
        ctx.dtypes = (vertices.dtype, colors.dtype if colors is not None else None)
        ctx.set_materialize_grads(False)
        return fv, fc

    @staticmethod
    def backward(ctx: Any, vertices_b: Optional[torch.Tensor], colors_b: Optional[torch.Tensor]):  # type: ignore
        need_v, need_c = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        vb = vertices_b if need_v else None
        cb = colors_b if need_c else None
        if vb is None and cb is None:
            return None, None, None
        gv, gc = ctx.sub.backward(vb, cb)
        vd, cd = ctx.dtypes
        return (gv.to(vd) if gv is not None else None), (gc.to(cd) if gc is not None else None), None


class LinearBlendSkinningFunc(torch.autograd.Function):
    """Linear blend skinning: (vertices [V,3], rotations [J,3] axis-angle, skin_weight [V,K], LinearBlendSkinning) ->
    skinned vertices [V,3], fp64 (deodr_b200_skin).  The forward kinematics table is the node's own, so forwards may
    run in any order before their backwards; backward (deodr_b200_skin_b, bit-reproducible) returns the gradients of
    the vertices and the rotations, and of the weights when they require it.  The joint centres are constants."""

    @staticmethod
    def forward(ctx: Any, vertices: torch.Tensor, rotations: torch.Tensor, skin_weight: torch.Tensor,  # type: ignore
                skinning: LinearBlendSkinning):
        v, r, w = _f64(vertices), _f64(rotations), _f64(skin_weight)
        table = torch.empty((skinning.nb_joints, 24), dtype=torch.float64, device=skinning.device)
        out = skinning.apply(v, r, skin_weight=w, transforms=table)
        ctx.save_for_backward(v, r, w, table)
        ctx.skinning = skinning
        ctx.dtypes = (vertices.dtype, rotations.dtype, skin_weight.dtype)
        return out

    @staticmethod
    def backward(ctx: Any, skinned_b: torch.Tensor):  # type: ignore
        v, r, w, table = ctx.saved_tensors
        need_w = ctx.needs_input_grad[2]
        res = ctx.skinning.backward(v, r, skinned_b.to(torch.float64).contiguous(), weights_grad=need_w,
                                    skin_weight=w, transforms=table)
        vd, rd, wd = ctx.dtypes
        return res[0].to(vd), res[1].to(rd), (res[2].to(wd) if need_w else None), None


class PhongShadeFunc(torch.autograd.Function):
    """The per-pixel shading of a G-buffer (deodr_b200_phong_shade / _b, model in include/deodr_b200.h): (channels
    [H,W,C+7] = (albedo C, normal 3, position 3, coverage 1) as rasterised over a zero background, light_directional
    [3] or None, light_ambient, specular (ks), shininess (e), camera (a CameraParams, whose centre -R^T t is used, or
    the centre [3] as a tensor), background [C], sh, albedo) -> image [H,W,C] fp32.  Backward returns the gradients of
    the channels, of each light and specular parameter and of a centre tensor that needs one, in its dtype; the
    parameter and centre gradients are summed over the pixels in a fixed order.  With ``albedo`` [H,W,C] (a textured
    mesh's albedo raster) the channels are [H,W,7] = (normal, position, coverage) and the albedo gets its gradient.
    ``specular_raster`` [H,W,2] (with the albedo) is the specular map's raster (K, E), which gives every specular term
    aks = ks K and e(p) = e E / a (the model in include/deodr_b200.h), and gets its gradient.  ``brdf="ggx"`` (with the
    albedo) is the metallic-roughness form instead: ``specular`` and ``shininess`` are then the metallic and roughness
    factors, and ``specular_raster`` the metallic-roughness map's raster (R, M) or None."""

    @staticmethod
    def forward(ctx: Any, channels: torch.Tensor, light_directional: Optional[torch.Tensor],  # type: ignore
                light_ambient, specular, shininess, camera: CameraParams, background,
                sh: Optional[torch.Tensor] = None, albedo: Optional[torch.Tensor] = None,
                point_lights: Optional[torch.Tensor] = None, visibility: Optional[torch.Tensor] = None,
                sun_visibility: Optional[torch.Tensor] = None, specular_raster: Optional[torch.Tensor] = None,
                brdf: str = "phong"):
        dev = channels.device
        scalars = [x if isinstance(x, torch.Tensor) else torch.tensor(float(x), dtype=torch.float64, device=dev)
                   for x in (light_ambient, specular, shininess)]
        directional = light_directional is not None
        ld = _f64(light_directional).reshape(3) if directional else torch.zeros(3, dtype=torch.float64, device=dev)
        params = torch.cat([ld] + [_f64(x).reshape(1).to(dev) for x in scalars])
        ctx.center_is_input = isinstance(camera, torch.Tensor)
        if ctx.center_is_input:
            center = _f64(camera).reshape(3).to(dev)
            ctx.center_dtype = camera.dtype
        else:
            center = torch.from_numpy(camera_center(camera)).to(dev, non_blocking=True)
        bg = background if isinstance(background, torch.Tensor) else torch.from_numpy(
            np.ascontiguousarray(background, dtype=np.float32)).to(dev, non_blocking=True)
        ch = channels.detach().to(torch.float32).contiguous()
        shd = _f64(sh) if sh is not None else None
        alb = albedo.detach().to(torch.float32).contiguous() if albedo is not None else None
        pl = _f64(point_lights) if point_lights is not None else None
        vis = visibility.detach().to(torch.float32).contiguous() if visibility is not None else None
        sun = sun_visibility.detach().to(torch.float32).contiguous() if sun_visibility is not None else None
        spec = specular_raster.detach().to(torch.float32).contiguous() if specular_raster is not None else None
        image = phong_shade(ch, params, center, bg, sh=shd, albedo=alb, point_lights=pl, visibility=vis,
                            sun_visibility=sun, specular=spec, brdf=brdf)
        ctx.brdf = brdf
        ctx.save_for_backward(ch, params, center, bg.to(dev, torch.float32), shd, alb, pl, vis, sun, spec)
        ctx.spec_dtype = specular_raster.dtype if specular_raster is not None else None
        ctx.vis_dtype = visibility.dtype if visibility is not None else None
        ctx.sun_dtype = sun_visibility.dtype if sun_visibility is not None else None
        ctx.lights_dtype = point_lights.dtype if point_lights is not None else None
        ctx.albedo_dtype = albedo.dtype if albedo is not None else None
        ctx.sh_dtype = sh.dtype if sh is not None else None
        ctx.directional = directional
        ctx.dtypes = (channels.dtype, light_directional.dtype if directional else None) + tuple(x.dtype for x in scalars)
        ctx.shapes = tuple(x.shape for x in scalars)
        return image

    @staticmethod
    def backward(ctx: Any, image_b: torch.Tensor):  # type: ignore
        ch, params, center, bg, shd, alb, pl, vis, sun, spec = ctx.saved_tensors
        needs = ctx.needs_input_grad
        center_grad = ctx.center_is_input and needs[5]
        shaded = phong_shade_backward(ch, params, center, bg, image_b, _scratch_of(ch.device), center_grad=center_grad,
                                      sh=shd, albedo=alb, point_lights=pl, visibility=vis, sun_visibility=sun,
                                      specular=spec, brdf=ctx.brdf)
        spec_b = None
        if spec is not None:
            shaded, spec_b = shaded[:-1], shaded[-1]
        sun_b = None
        if sun is not None:
            shaded, sun_b = shaded[:-1], shaded[-1]
        vis_b = None
        if vis is not None:
            shaded, vis_b = shaded[:-1], shaded[-1]
        lights_b = None
        if pl is not None:
            shaded, lights_b = shaded[:-1], shaded[-1]
        albedo_b = None
        if alb is not None:
            shaded, albedo_b = shaded[:-1], shaded[-1]
        channels_b, params_b = shaded[:2]
        cd, ld = ctx.dtypes[:2]
        out = [channels_b.to(cd) if needs[0] else None,
               params_b[:3].to(ld) if ctx.directional and needs[1] else None]
        for k in range(3):
            out.append(params_b[3 + k].reshape(ctx.shapes[k]).to(ctx.dtypes[2 + k]) if needs[2 + k] else None)
        out.append(shaded[2].to(ctx.center_dtype) if center_grad else None)
        out.append(None)  # background
        out.append(shaded[-1].to(ctx.sh_dtype) if shd is not None and needs[7] else None)
        out.append(albedo_b.to(ctx.albedo_dtype) if albedo_b is not None and needs[8] else None)
        out.append(lights_b.to(ctx.lights_dtype) if lights_b is not None and needs[9] else None)
        out.append(vis_b.to(ctx.vis_dtype) if vis_b is not None and needs[10] else None)
        out.append(sun_b.to(ctx.sun_dtype) if sun_b is not None and needs[11] else None)
        out.append(spec_b.to(ctx.spec_dtype) if spec_b is not None and needs[12] else None)
        out.append(None)  # brdf
        return tuple(out)


class RenderShadowedPhongFunc(torch.autograd.Function):
    """The rasters of a Phong render with shadows, as one node: the G-buffer (beside the albedo raster of a textured
    mesh, as ``RenderMeshPhongTexturedFunc``), the 6L cube shadow maps of the point lights (``ShadowCubes``) and the
    directional light's map (``SunShadowMap``; the models in include/deodr_b200.h), rendered by one ``render_views``
    call and back-propagated by one ``render_b_views`` call, the renderer keeping one live forward per slot.  (ij,
    uv | None, texture | None, channels, depths, edgeflags, vertices [V,3], point_lights [L, 3 + S] | None, albedo
    scene | None, G-buffer scene, cubes | None, sigma, light_directional [3] | None, sun | None) -> ([albedo [H,W,C],]
    G-buffer[, maps [6L,M,M]][, sun map [M,M]]) fp32.  The maps' projections happen inside the node, so their gradient
    reaches the vertices, the lights' positions and the directional light through their adjoints.  Same snapshot /
    replay rule as ``RenderMesh2DFunc``."""

    NAMES = ("ij", "uv", "shade", "texture")

    @staticmethod
    def forward(ctx: Any, ij: torch.Tensor, uv: Optional[torch.Tensor], texture: Optional[torch.Tensor],  # type: ignore
                channels: torch.Tensor, depths: torch.Tensor, edgeflags: torch.Tensor, vertices: torch.Tensor,
                point_lights: Optional[torch.Tensor], albedo_scene: Optional[DeviceScene], gbuffer_scene: DeviceScene,
                cubes: Optional[ShadowCubes], sigma: float = 1.0, light_directional: Optional[torch.Tensor] = None,
                sun: Optional[SunShadowMap] = None, normal_map: Optional[torch.Tensor] = None,
                map_scene: Optional[DeviceScene] = None, specular_map: Optional[torch.Tensor] = None,
                spec_scene: Optional[DeviceScene] = None):
        textured = albedo_scene is not None
        if textured:
            check_scene_inputs(albedo_scene, uv=uv, texture=texture)
        check_scene_inputs(gbuffer_scene, colors=channels)
        if (cubes is None) != (point_lights is None) or (sun is None) != (light_directional is None):
            raise ValueError("the cube maps come with point_lights, and the sun map with light_directional")
        mapped = map_scene is not None
        if (normal_map is None) != (not mapped) or (mapped and not textured):
            raise ValueError("a normal map comes with its scene, in a textured render")
        if mapped:
            check_scene_inputs(map_scene, uv=uv, texture=normal_map)
        spec_mapped = spec_scene is not None
        if (specular_map is None) != (not spec_mapped) or (spec_mapped and not textured):
            raise ValueError("a specular map comes with its scene, in a textured render")
        if spec_mapped:
            check_scene_inputs(spec_scene, uv=uv, texture=specular_map)
        inputs = (ij.detach(), uv.detach() if textured else None, texture.detach() if textured else None,
                  channels.detach(), depths.detach(), edgeflags, _f64(vertices.detach()),
                  _f64(point_lights.detach()) if cubes is not None else None,
                  _f64(light_directional.detach()).reshape(3).contiguous() if sun is not None else None,
                  normal_map.detach() if mapped else None, specular_map.detach() if spec_mapped else None)
        # the rasters: [albedo,] G-buffer[, normal map][, specular map]; mi and si index the map rasters
        ctx.scenes = ([albedo_scene] if textured else []) + [gbuffer_scene] + ([map_scene] if mapped else []) + \
            ([spec_scene] if spec_mapped else [])
        ctx.gi = 1 if textured else 0
        ctx.mi = 2 if mapped else None
        ctx.si = len(ctx.scenes) - 1 if spec_mapped else None
        ctx.maps = [m for m in (cubes, sun) if m is not None]
        ctx.cubes, ctx.sun, ctx.sigma, ctx.textured, ctx.mapped = cubes, sun, float(sigma), textured, mapped
        renderer = default_renderer(gbuffer_scene.device.index)
        ctx.fwds = RenderShadowedPhongFunc._render(renderer, ctx, inputs, None)
        ctx.in_dtypes = (ij.dtype, uv.dtype if textured else None, texture.dtype if textured else None, channels.dtype,
                         vertices.dtype, point_lights.dtype if cubes is not None else None,
                         light_directional.dtype if sun is not None else None,
                         normal_map.dtype if mapped else None, specular_map.dtype if spec_mapped else None)
        ctx.save_for_backward(*(t.clone() if t is not None else None for t in inputs))
        rasters = tuple(f["image"].clone() for f in ctx.fwds[:len(ctx.scenes)])
        return rasters + ((cubes.maps.clone(),) if cubes is not None else ()) + \
            ((sun.map.clone(),) if sun is not None else ())

    @staticmethod
    def _prepare(ctx, inputs):
        if ctx.cubes is not None:
            ctx.cubes.prepare(inputs[6], inputs[7])
        if ctx.sun is not None:
            ctx.sun.prepare(inputs[6], inputs[8])

    @staticmethod
    def _update(ctx, inputs):
        ij, uv, texture, channels, depths, edgeflags = inputs[:6]
        if ctx.textured:
            ctx.scenes[0].update(ij=ij, uv=uv, texture=texture, depths=depths, edgeflags=edgeflags)
        ctx.scenes[ctx.gi].update(ij=ij, colors=channels, depths=depths, edgeflags=edgeflags)
        if ctx.mi is not None:
            ctx.scenes[ctx.mi].update(ij=ij, uv=uv, texture=inputs[9], depths=depths, edgeflags=edgeflags)
        if ctx.si is not None:
            ctx.scenes[ctx.si].update(ij=ij, uv=uv, texture=inputs[10], depths=depths, edgeflags=edgeflags)
        RenderShadowedPhongFunc._prepare(ctx, inputs)

    @staticmethod
    def _render(renderer, ctx, inputs, out):
        RenderShadowedPhongFunc._update(ctx, inputs)
        if out is None:
            out = [renderer._new_outputs(sc, False, False, False) for sc in ctx.scenes] + \
                [o for m in ctx.maps for o in m.outputs()]
        return renderer.render_views(ctx.scenes + [sc for m in ctx.maps for sc in m.scenes], ctx.sigma, out=out)

    @staticmethod
    def backward(ctx: Any, *grads):  # type: ignore
        needs = ctx.needs_input_grad
        if not any(needs[:8]) and not needs[12] and not needs[14] and not needs[16]:
            return (None,) * 18
        inputs = ctx.saved_tensors
        renderer = default_renderer(ctx.scenes[ctx.gi].device.index)
        n = len(ctx.scenes)
        # the shared scenes and maps may hold another node's inputs by now
        if any(f["generation"] != renderer.generation(f["slot"]) for f in ctx.fwds):
            ctx.fwds = RenderShadowedPhongFunc._render(renderer, ctx, inputs, ctx.fwds)
        else:
            RenderShadowedPhongFunc._update(ctx, inputs)
        if ctx.textured:
            gs = [requested_grads(ctx.scenes[0], RenderShadowedPhongFunc.NAMES, (True, needs[1], False, needs[2])),
                  ctx.scenes[1].zero_grads()]
            if ctx.mi is not None:
                gs.append(requested_grads(ctx.scenes[ctx.mi], RenderShadowedPhongFunc.NAMES,
                                          (True, needs[1], False, needs[14])))
            if ctx.si is not None:
                gs.append(requested_grads(ctx.scenes[ctx.si], RenderShadowedPhongFunc.NAMES,
                                          (True, needs[1], False, needs[16])))
        else:
            gs = [ctx.scenes[0].zero_grads()]
        image_bs = [g.to(torch.float32).contiguous() for g in grads[:n]]
        maps_bs = [g.to(torch.float32).contiguous() for g in grads[n:]]
        if ctx.sun is not None:
            maps_bs[-1] = maps_bs[-1][None]
        renderer.render_b_views(ctx.scenes + [sc for m in ctx.maps for sc in m.scenes], ctx.sigma, ctx.fwds,
                                image_bs + [b for m, mb in zip(ctx.maps, maps_bs) for b in m.image_bs(mb)],
                                grads=gs + [g for m in ctx.maps for g in m.grads()])
        scratch = _scratch_of(inputs[6].device)
        vertices_b = torch.zeros_like(inputs[6])
        lights_b = light_b = None
        if ctx.cubes is not None:
            _, lights_b = cube_project_backward(inputs[6], inputs[7], ctx.cubes.M, ctx.cubes.cameras, ctx.cubes.ij_b,
                                                ctx.cubes.colors_b.view(6 * ctx.cubes.L, -1), scratch,
                                                vertices_b=vertices_b)
        if ctx.sun is not None:
            _, light_b = sun_project_backward(inputs[6], inputs[8], ctx.sun.bounds, ctx.sun.M, ctx.sun.ij_b[0],
                                              ctx.sun.colors_b.view(-1), scratch, vertices_b=vertices_b)
        ij_d, uv_d, tex_d, ch_d, v_d, l_d, d_d, nm_d, sm_d = ctx.in_dtypes
        ij_b = sum(g["ij_b"] for g in gs)
        uv_b = gs[0]["uv_b"] if ctx.textured else None
        for i in (ctx.mi, ctx.si):
            if i is not None:
                uv_b = uv_b + gs[i]["uv_b"]
        return (ij_b.to(ij_d) if needs[0] else None,
                uv_b.to(uv_d) if ctx.textured and needs[1] else None,
                gs[0]["texture_b"].to(tex_d) if ctx.textured and needs[2] else None,
                gs[ctx.gi]["colors_b"].to(ch_d) if needs[3] else None, None, None,
                vertices_b.to(v_d) if needs[6] else None,
                lights_b.to(l_d) if lights_b is not None and needs[7] else None,
                None, None, None, None, light_b.to(d_d) if light_b is not None and needs[12] else None, None,
                gs[ctx.mi]["texture_b"].to(nm_d) if ctx.mi is not None and needs[14] else None, None,
                gs[ctx.si]["texture_b"].to(sm_d) if ctx.si is not None and needs[16] else None, None)


class ShadowVisibilityFunc(torch.autograd.Function):
    """The point lights' visibility of a G-buffer's pixels (deodr_b200_shadow_visibility / _b, the model in
    include/deodr_b200.h): (channels [H,W,C+7], or [H,W,7] beside an albedo, point_lights [L, 3 + S], maps [6L,M,M],
    bias, softness, albedo | None) -> visibility [H,W,L] fp32.  Backward returns the gradients of the G-buffer's
    position and coverage slices, of the maps and of the lights' positions; the albedo, only read for its channel
    count, gets none."""

    @staticmethod
    def forward(ctx: Any, channels: torch.Tensor, point_lights: torch.Tensor, maps: torch.Tensor,  # type: ignore
                bias: float, softness: float, albedo: Optional[torch.Tensor] = None):
        ch = channels.detach().to(torch.float32).contiguous()
        pl, mp = _f64(point_lights.detach()), maps.detach().to(torch.float32).contiguous()
        alb = albedo.detach() if albedo is not None else None
        vis = shadow_visibility(ch, pl, mp, bias, softness, albedo=alb)
        ctx.save_for_backward(ch, pl, mp, alb)
        ctx.band = (float(bias), float(softness))
        ctx.dtypes = (channels.dtype, point_lights.dtype, maps.dtype)
        return vis

    @staticmethod
    def backward(ctx: Any, vis_b: torch.Tensor):  # type: ignore
        ch, pl, mp, alb = ctx.saved_tensors
        channels_b, maps_b, lights_b = shadow_visibility_backward(ch, pl, mp, *ctx.band, vis_b, _scratch_of(ch.device),
                                                                  albedo=alb)
        needs = ctx.needs_input_grad
        cd, ld, md = ctx.dtypes
        return (channels_b.to(cd) if needs[0] else None, lights_b.to(ld) if needs[1] else None,
                maps_b.to(md) if needs[2] else None, None, None, None)


class SunVisibilityFunc(torch.autograd.Function):
    """The directional light's visibility of a G-buffer's pixels (deodr_b200_sun_visibility / _b, the model in
    include/deodr_b200.h): (channels [H,W,C+7], or [H,W,7] beside an albedo, light_directional [3], map [M,M],
    bounds (cx, cy, cz, r), bias, softness, albedo | None) -> visibility [H,W] fp32.  Backward returns the gradients
    of the G-buffer's position and coverage slices, of the map and of the light; the albedo, only read for its channel
    count, gets none."""

    @staticmethod
    def forward(ctx: Any, channels: torch.Tensor, light_directional: torch.Tensor, sun_map: torch.Tensor,  # type: ignore
                bounds, bias: float, softness: float, albedo: Optional[torch.Tensor] = None):
        ch = channels.detach().to(torch.float32).contiguous()
        ld = _f64(light_directional.detach()).reshape(3).contiguous()
        mp = sun_map.detach().to(torch.float32).contiguous()
        alb = albedo.detach() if albedo is not None else None
        vis = sun_visibility(ch, ld, mp, bounds, bias, softness, albedo=alb)
        ctx.save_for_backward(ch, ld, mp, alb)
        ctx.args = (tuple(bounds), float(bias), float(softness))
        ctx.dtypes = (channels.dtype, light_directional.dtype, sun_map.dtype)
        return vis

    @staticmethod
    def backward(ctx: Any, vis_b: torch.Tensor):  # type: ignore
        ch, ld, mp, alb = ctx.saved_tensors
        channels_b, map_b, light_b = sun_visibility_backward(ch, ld, mp, *ctx.args, vis_b, _scratch_of(ch.device),
                                                             albedo=alb)
        needs = ctx.needs_input_grad
        cd, ld_d, md = ctx.dtypes
        return (channels_b.to(cd) if needs[0] else None, light_b.to(ld_d) if needs[1] else None,
                map_b.to(md) if needs[2] else None, None, None, None, None)


class VertexTangentsFunc(torch.autograd.Function):
    """The per-vertex tangent frames of a normal-mapped mesh (deodr_b200_vertex_tangents / _b, the model in
    include/deodr_b200.h): (vertices [V,3], uv [Nuv,2], VertexTangents) -> frames [V,6] = (T, B) fp64.  Backward
    returns the gradients of the vertices and the uv, each a fixed-order gather."""

    @staticmethod
    def forward(ctx: Any, vertices: torch.Tensor, uv: torch.Tensor, tangents: VertexTangents):  # type: ignore
        v, w = _f64(vertices), _f64(uv)
        ctx.save_for_backward(v, w)
        ctx.tangents, ctx.dtypes = tangents, (vertices.dtype, uv.dtype)
        return tangents.frames(v, w)

    @staticmethod
    def backward(ctx: Any, frames_b: torch.Tensor):  # type: ignore
        v, w = ctx.saved_tensors
        vertices_b, uv_b = ctx.tangents.backward(v, w, frames_b)
        needs = ctx.needs_input_grad
        return (vertices_b.to(ctx.dtypes[0]) if needs[0] else None, uv_b.to(ctx.dtypes[1]) if needs[1] else None,
                None)


class NormalMapFunc(torch.autograd.Function):
    """The normal map's per-pixel perturbation (deodr_b200_normal_map / _b, the model in include/deodr_b200.h):
    (G-buffer [H,W,13] = (N, X, a, T, B), map raster [H,W,3]) -> G-buffer [H,W,7] = (N', X, a) fp32."""

    @staticmethod
    def forward(ctx: Any, gbuffer: torch.Tensor, nmap: torch.Tensor):  # type: ignore
        g, m = gbuffer.detach().to(torch.float32).contiguous(), nmap.detach().to(torch.float32).contiguous()
        ctx.save_for_backward(g, m)
        ctx.dtypes = (gbuffer.dtype, nmap.dtype)
        return normal_map(g, m)

    @staticmethod
    def backward(ctx: Any, out_b: torch.Tensor):  # type: ignore
        g, m = ctx.saved_tensors
        g_b, m_b = normal_map_backward(g, m, out_b)
        needs = ctx.needs_input_grad
        return g_b.to(ctx.dtypes[0]) if needs[0] else None, m_b.to(ctx.dtypes[1]) if needs[1] else None


project_points_autograd = ProjectPointsFunc.apply
vertex_normals_autograd = VertexNormalsFunc.apply
lit_vertex_colors_autograd = LitVertexColorsFunc.apply
sh_lit_vertex_colors_autograd = ShLitVertexColorsFunc.apply
point_lit_vertex_colors_autograd = PointLitVertexColorsFunc.apply
render_mesh_2d = RenderMesh2DFunc.apply
render_mesh_2d_textured = RenderMesh2DTexturedFunc.apply
render_mesh_phong_textured = RenderMeshPhongTexturedFunc.apply
pose_autograd = PoseFunc.apply
rigid_energy_autograd = RigidEnergyFunc.apply
loop_subdivision_autograd = LoopSubdivisionFunc.apply
phong_shade_autograd = PhongShadeFunc.apply
render_shadowed_phong = RenderShadowedPhongFunc.apply
shadow_visibility_autograd = ShadowVisibilityFunc.apply
sun_visibility_autograd = SunVisibilityFunc.apply
vertex_tangents_autograd = VertexTangentsFunc.apply
normal_map_autograd = NormalMapFunc.apply


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
    OpenCV distortion, projecting CUDA tensors through :class:`ProjectPointsFunc`.

    Each of ``extrinsic`` [3,4], ``intrinsic`` [3,3] and ``distortion`` [5] is an array (a constant, uploaded once) or
    a CUDA tensor, which may require grad and may be any torch expression (a rotation built from a quaternion, say).
    With no tensor among them the camera is the constant of the reference's class.  With one, every render builds the
    camera vector [26] from them on the device and back-propagates into those that require grad; the reference's
    ``CameraPytorch`` holds detached copies and has no camera gradient."""

    def __init__(self, extrinsic, intrinsic, height: int, width: int, distortion=None):
        self.height, self.width = int(height), int(width)
        given = [x for x in (extrinsic, intrinsic, distortion) if isinstance(x, torch.Tensor)]
        if not given:
            super().__init__(extrinsic, intrinsic, distortion)
            return
        dev = _device(given[0].device)

        def tensor(x, shape):
            t = x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x, dtype=np.float64), device=dev)
            if t.device != dev or t.numel() != int(np.prod(shape)):
                raise ValueError(f"camera tensors must be on {dev} with {int(np.prod(shape))} entries; got "
                                 f"{tuple(t.shape)} on {t.device}")
            return t.reshape(shape)

        self.extrinsic, self.intrinsic = tensor(extrinsic, (3, 4)), tensor(intrinsic, (3, 3))
        self.distortion = tensor(distortion, (5,)) if distortion is not None else None

    @property
    def is_tensor(self) -> bool:
        """True for a camera given as tensors (see the class)."""
        return isinstance(self.extrinsic, torch.Tensor)

    def vector(self):
        """The camera vector [26]: a differentiable fp64 tensor for a tensor camera, else ``CameraParams.vector``."""
        if not self.is_tensor:
            return super().vector()
        dist = self.distortion if self.distortion is not None else torch.zeros(5, dtype=torch.float64,
                                                                               device=self.extrinsic.device)
        return torch.cat([x.reshape(-1).to(torch.float64) for x in (self.extrinsic, self.intrinsic, dist)])

    def center(self):
        """The camera centre -R^T t [3]: a differentiable fp64 tensor for a tensor camera, else an array."""
        if not self.is_tensor:
            return camera_center(self)
        e = self.extrinsic.to(torch.float64)
        return -(e[:, :3].T @ e[:, 3])

    def project_points(self, points_3d: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """-> (ij [N,2], depths [N]), differentiable in ``points_3d`` and, for a tensor camera, in its tensors."""
        if self.is_tensor:
            return project_points_autograd(points_3d, self.vector(), self.distortion is not None)
        return project_points_autograd(points_3d, self)


class ColoredTriMeshPytorch:
    """``deodr.pytorch.ColoredTriMeshPytorch(faces, vertices, clockwise=False, colors=None)`` on the device: the
    vertices [V,3] and vertex colours [V,C] are CUDA tensors (either may require grad), the adjacency a
    :class:`MeshTopology` built once.

    ``faces_uv`` [T,3], ``uv`` [Nuv,2] and ``texture`` [Ht,Wt,C], given together, make the mesh textured, in the
    conventions of the reference's ``ColoredTriMesh`` (uv in texel units).  ``uv`` and ``texture`` are tensors (fp32 or
    fp64, either may require grad) or arrays, uploaded once; the attributes ``uv`` and ``texture`` may be reassigned
    between renders.

    ``normal_map`` [Ht,Wt,3] (a textured mesh's, with the texture's Ht and Wt; a tensor that may require grad, or an
    array) is a tangent-space normal map, read by ``Scene3DPytorch(shading="phong_textured")`` (the model in
    include/deodr_b200.h); the attribute may be reassigned between renders.

    ``metallic_roughness_map`` [Ht,Wt,2] = (roughness_t, metallic_t) (a textured mesh's, likewise; not with a specular
    map) multiplies the scene's metallic and roughness factors in a ``pbr_textured`` render.
    ``specular_map`` [Ht,Wt,2] (a textured mesh's, likewise) is a specular map whose texel (ks_t, e_t) multiplies the
    scene's specular strength and shininess in a ``phong_textured`` render (the model in include/deodr_b200.h); a tensor
    that may require grad, or an array, and the attribute may be reassigned between renders."""

    def __init__(self, faces, vertices, clockwise: bool = False, colors=None, device=None, faces_uv=None, uv=None,
                 texture=None, normal_map=None, specular_map=None, metallic_roughness_map=None):
        self.device = _device(device if device is not None else
                              (vertices.device if isinstance(vertices, torch.Tensor) else None))
        self.faces = np.ascontiguousarray(np.asarray(faces), dtype=np.int64)
        self.nb_faces = self.faces.shape[0]
        self.clockwise = bool(clockwise)
        self.set_vertices(vertices)
        self.nb_vertices = self.vertices.shape[0]
        self.topology = MeshTopology(self.faces, self.nb_vertices, clockwise=self.clockwise, device=self.device)
        self._subdivisions: Dict[int, LoopSubdivision] = {}
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
        self.normal_map = None
        self._tangents: Optional[VertexTangents] = None
        if normal_map is not None:
            if not self.textured:
                raise ValueError("a normal map is addressed by the uv: it needs a textured mesh")
            self.normal_map = self._tensor(normal_map)
            if tuple(self.normal_map.shape) != tuple(self.texture.shape[:2]) + (3,):
                raise ValueError(f"normal_map must be [Ht,Wt,3] with the texture's Ht and Wt = "
                                 f"{tuple(self.texture.shape[:2])}; got {tuple(self.normal_map.shape)}")
        self.specular_map = None
        if specular_map is not None:
            if not self.textured:
                raise ValueError("a specular map is addressed by the uv: it needs a textured mesh")
            self.specular_map = self._tensor(specular_map)
            if tuple(self.specular_map.shape) != tuple(self.texture.shape[:2]) + (2,):
                raise ValueError(f"specular_map must be [Ht,Wt,2] with the texture's Ht and Wt = "
                                 f"{tuple(self.texture.shape[:2])}; got {tuple(self.specular_map.shape)}")
        self.metallic_roughness_map = None
        if metallic_roughness_map is not None:
            if not self.textured:
                raise ValueError("a metallic-roughness map is addressed by the uv: it needs a textured mesh")
            if specular_map is not None:
                raise ValueError("a mesh takes a specular map (Phong) or a metallic-roughness map (PBR), not both")
            self.metallic_roughness_map = self._tensor(metallic_roughness_map)
            if tuple(self.metallic_roughness_map.shape) != tuple(self.texture.shape[:2]) + (2,):
                raise ValueError(f"metallic_roughness_map must be [Ht,Wt,2] with the texture's Ht and Wt = "
                                 f"{tuple(self.texture.shape[:2])}; got {tuple(self.metallic_roughness_map.shape)}")

    @property
    def tangents(self) -> VertexTangents:
        """The mesh's :class:`~deodr_b200.mesh_ops.VertexTangents` (faces_uv and the uv-vertex-face CSR on the device),
        built on first use."""
        if self._tangents is None:
            self._tangents = VertexTangents(self.topology, self.faces_uv, self.uv.shape[0])
        return self._tangents

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

    def subdivise(self, n_iter: int) -> "ColoredTriMeshPytorch":
        """``ColoredTriMesh.subdivise(n_iter)``: ``n_iter`` levels of the reference's Loop subdivision
        (:class:`~deodr_b200.mesh_ops.LoopSubdivision`) -> a new mesh whose faces are the reference's fine faces and
        whose vertices and colours are computed on the device through :class:`LoopSubdivisionFunc`, so they are
        differentiable in this mesh's when those require grad: rendering the fine mesh and calling ``backward`` gives
        gradients to the coarse vertices.  Unlike the reference, the fine mesh keeps ``clockwise`` (its faces keep the
        coarse winding).  ``n_iter = 0`` returns this mesh.  Textured meshes raise ValueError, as in the reference.

        The levels' adjacency is built on the host on the first call for a given ``n_iter`` and kept for later calls."""
        if self.textured:
            raise ValueError("Textured mesh not supported yet in subdivision")
        if n_iter == 0:
            return self
        if n_iter not in self._subdivisions:
            self._subdivisions[n_iter] = LoopSubdivision(self.faces, self.nb_vertices, n_iter, clockwise=self.clockwise,
                                                         device=self.device)
        sub = self._subdivisions[n_iter]
        vertices, colors = loop_subdivision_autograd(self.vertices, self.vertices_colors, sub)
        return ColoredTriMeshPytorch(sub.faces, vertices, clockwise=self.clockwise, colors=colors, device=self.device)


class Scene3DPytorch:
    """``deodr.pytorch.Scene3DPytorch`` on the device: ``set_mesh``, ``set_light(light_directional, light_ambient)``,
    ``set_background_color``, ``render(camera)`` -> image [H,W,C] and ``render_depth(camera, depth_scale)`` -> [H,W,1],
    fp32 CUDA tensors differentiable in the mesh's vertices and colours (or uv and texture, for a textured mesh) and in
    the light.

    A render is the chain of Functions of this module; ``sigma`` is the antialiasing width of the reference's Scene3D
    (1 by default; at 0 no silhouette edge is drawn).  The backgrounds are set on the device by
    ``set_background_color``, so a render copies nothing from the host.

    ``shading="phong"`` lights an untextured mesh per pixel (the model of ``DeodrPhongIO``, include/deodr_b200.h):
    ``render`` rasterises ``[colours | normals | vertices | 1]`` over a zero background and shades the result with
    :class:`PhongShadeFunc`, with the specular strength and shininess of ``set_specular``.

    ``shading="phong_textured"`` lights a textured mesh per pixel: the albedo raster (the texture with a shade of 1
    over a zero background) and a G-buffer ``[normals | vertices | 1]`` are rendered by one
    :class:`RenderMeshPhongTexturedFunc` node and shaded by :class:`PhongShadeFunc` with the albedo apart; grey and
    coloured environments apply.  A mesh with a ``normal_map`` adds its tangent frames (:class:`VertexTangentsFunc`)
    to the G-buffer and the map's raster to the same node, and :class:`NormalMapFunc` perturbs the G-buffer's normal
    before the shading and the shadows read it; the map, the uv and the vertices receive their gradients.  A mesh with
    a ``specular_map`` adds the map's raster to the same node, and :class:`PhongShadeFunc` reads it per pixel; the map
    receives its gradient.

    ``shading="pbr_textured"`` is the same chain with the metallic-roughness form of :class:`PhongShadeFunc`
    (``brdf="ggx"``; the model in include/deodr_b200.h): the factors of ``set_material(metallic, roughness)``, which
    may be tensors that require grad, and a mesh's ``metallic_roughness_map`` rasterised in the specular map's slot.

    ``set_point_lights`` adds point lights near the mesh in every shading; a table that requires grad receives its
    gradient, and the vertices receive the lights' share through their normals and their positions.  A flash is a
    light whose position the caller computes from the camera's tensors: its gradient then reaches the camera.  In a
    Phong or textured Phong render, ``set_point_lights(..., shadow_map_size=M)`` makes them cast shadows (the model in
    include/deodr_b200.h): the rasters and the lights' cube maps are one :class:`RenderShadowedPhongFunc` node, the
    visibility a :class:`ShadowVisibilityFunc`, and the shadows' gradient reaches the vertices and the lights.
    ``set_light(..., shadow_map_size=M, shadow_bias=, shadow_softness=, shadow_bounds=(cx, cy, cz, r))`` makes the
    directional light cast shadows too: its map is rendered in the same :class:`RenderShadowedPhongFunc` node, its
    visibility is a :class:`SunVisibilityFunc`, and a light that requires grad receives the shadow's share."""

    def __init__(self, sigma: float = 1.0, backface_culling: bool = True, shading: str = "gouraud"):
        if shading not in ("gouraud", "phong", "phong_textured", "pbr_textured"):
            raise ValueError(f"shading must be 'gouraud', 'phong', 'phong_textured' or 'pbr_textured'; got {shading!r}")
        self.sigma = float(sigma)
        self.backface_culling = bool(backface_culling)
        self.shading = shading
        self.mesh: Optional[ColoredTriMeshPytorch] = None
        self.light_directional: Optional[torch.Tensor] = None
        self.light_ambient: Optional[torch.Tensor] = None
        self.light_sh: Optional[torch.Tensor] = None
        self.point_lights: Optional[torch.Tensor] = None
        self.shadow_map_size, self.shadow_bias, self.shadow_softness = 0, None, None
        self._cubes: Dict[tuple, ShadowCubes] = {}
        self.light_shadow_map_size, self.light_shadow_bias, self.light_shadow_softness = 0, None, None
        self.light_shadow_bounds: Optional[tuple] = None
        self._suns: Dict[tuple, SunShadowMap] = {}
        self.specular: Any = 0.0
        self.shininess: Any = 16.0
        self.metallic: Any = 0.0
        self.roughness: Any = 0.5
        self.background_color: Optional[np.ndarray] = None
        self._scenes: Dict[tuple, DeviceScene] = {}
        self._phong_scenes: Dict[tuple, DeviceScene] = {}
        self._albedo_scenes: Dict[tuple, DeviceScene] = {}

    def set_mesh(self, mesh: ColoredTriMeshPytorch) -> None:
        self.mesh = mesh
        self._cubes = {}
        self._suns = {}
        self._scenes = {}
        self._phong_scenes = {}
        self._albedo_scenes = {}

    def set_specular(self, specular, shininess) -> None:
        """The specular strength ks >= 0 and the shininess e of a Phong render (numbers or 0-d tensors); tensors are
        used as given, so a ``specular`` or ``shininess`` that requires grad receives its gradient."""
        if self.shading == "pbr_textured":
            raise ValueError("a 'pbr_textured' render takes set_material(metallic, roughness), not set_specular")
        dev = self.mesh.device if self.mesh is not None else _device(None)
        self.specular, self.shininess = [x if isinstance(x, torch.Tensor) else
                                         torch.tensor(float(x), dtype=torch.float64, device=dev)
                                         for x in (specular, shininess)]

    def set_material(self, metallic, roughness) -> None:
        """The metallic and roughness factors of a ``pbr_textured`` render (numbers or 0-d tensors); tensors are used
        as given, so a factor that requires grad receives its gradient."""
        if self.shading != "pbr_textured":
            raise ValueError("set_material sets the factors of shading='pbr_textured'; a Phong render takes "
                             "set_specular")
        dev = self.mesh.device if self.mesh is not None else _device(None)
        self.metallic, self.roughness = [x if isinstance(x, torch.Tensor) else
                                         torch.tensor(float(x), dtype=torch.float64, device=dev)
                                         for x in (metallic, roughness)]

    def set_light(self, light_directional, light_ambient, shadow_map_size: int = 0, shadow_bias: Optional[float] = None,
                  shadow_softness: Optional[float] = None, shadow_bounds=None) -> None:
        """``light_directional`` [3] (None: ambient light only) and ``light_ambient`` (a number or 0-d tensor); tensors
        are used as given, so a light that requires grad receives its gradient.  A ``shadow_map_size`` M > 0 makes
        the directional light cast shadows in a Phong render (the model in include/deodr_b200.h), with
        ``shadow_bias``, ``shadow_softness`` and ``shadow_bounds`` = (cx, cy, cz, r) (world units, all required) and
        the refusals of ``DeviceMeshView``'s ``light_shadow_*`` arguments."""
        size = check_sun_shadow_arguments(self.shading, light_directional, shadow_map_size, shadow_bias,
                                          shadow_softness, shadow_bounds)
        self.light_shadow_map_size = size
        self.light_shadow_bias = float(shadow_bias) if size else None
        self.light_shadow_softness = float(shadow_softness) if size else None
        self.light_shadow_bounds = tuple(float(b) for b in shadow_bounds) if size else None
        dev = self.mesh.device if self.mesh is not None else _device(None)
        if light_directional is not None and not isinstance(light_directional, torch.Tensor):
            light_directional = torch.as_tensor(np.asarray(light_directional, dtype=np.float64), device=dev)
        if not isinstance(light_ambient, torch.Tensor):
            light_ambient = torch.tensor(float(light_ambient), dtype=torch.float64, device=dev)
        self.light_directional, self.light_ambient = light_directional, light_ambient

    def set_light_sh(self, sh) -> None:
        """A second-order spherical-harmonics environment added to the light (the model in include/deodr_b200.h):
        [9] (grey) or [9,C] (coloured, C from 1 to 4) coefficients, a tensor used as given (so one that requires
        grad receives its gradient) or an array; None goes back to the directional and ambient light alone.  A
        textured mesh takes a grey environment only, unless it is shaded per pixel (``shading="phong_textured"``)."""
        if sh is not None:
            dev = self.mesh.device if self.mesh is not None else _device(None)
            if not isinstance(sh, torch.Tensor):
                sh = torch.as_tensor(np.asarray(sh, dtype=np.float64), device=dev)
            if sh.dim() not in (1, 2) or sh.shape[0] != 9 or (sh.dim() == 2 and not 1 <= sh.shape[1] <= 4):
                raise ValueError(f"sh must be [9] or [9,C] with C from 1 to 4; got {tuple(sh.shape)}")
        self.light_sh = sh

    def set_point_lights(self, lights, shadow_map_size: int = 0, shadow_bias: Optional[float] = None,
                         shadow_softness: Optional[float] = None) -> None:
        """Point lights added to the light (the model in include/deodr_b200.h): [L, 3 + S], row j the light's world
        position then its intensity, grey (S = 1) or one per channel (S = C up to 4), L from 1 to 8; a tensor used as
        given (so one that requires grad, or one computed from other tensors, receives its gradient) or an array.
        None removes them.  A textured mesh takes grey lights only, unless it is shaded per pixel.  A
        ``shadow_map_size`` M > 0 makes them cast shadows in a Phong render, with ``shadow_bias`` and
        ``shadow_softness`` (world units, both required) and the refusals of ``DeviceMeshView``."""
        size = check_shadow_arguments(self.shading, lights, shadow_map_size, shadow_bias, shadow_softness)
        self.shadow_map_size = size
        self.shadow_bias = float(shadow_bias) if size else None
        self.shadow_softness = float(shadow_softness) if size else None
        if lights is not None:
            dev = self.mesh.device if self.mesh is not None else _device(None)
            if not isinstance(lights, torch.Tensor):
                lights = torch.as_tensor(np.asarray(lights, dtype=np.float64), device=dev)
            if lights.dim() != 2 or not 1 <= lights.shape[0] <= 8 or not 4 <= lights.shape[1] <= 7:
                raise ValueError(f"point lights must be [L, 3 + S] with L from 1 to 8 and S from 1 to 4; got "
                                 f"{tuple(lights.shape)}")
        self.point_lights = lights

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

    def _phong_scene(self, camera: CameraPytorch, nb_colors: int, normal_mapped: bool = False) -> DeviceScene:
        """The cached G-buffer scene of the mesh for ``camera``: C + 7 channels (13 for a normal-mapped textured mesh),
        zero background."""
        from ..scenes import SceneArrays

        key = (camera.height, camera.width, nb_colors + (6 if normal_mapped else 0))
        if key not in self._phong_scenes:
            m = self.mesh
            T, V, K = m.nb_faces, m.nb_vertices, key[2] + 7
            faces = np.ascontiguousarray(m.faces, dtype=np.uint32)
            self._phong_scenes[key] = DeviceScene(SceneArrays(
                faces=faces, faces_uv=faces, ij=np.zeros((V, 2)), depths=np.ones(V), textured=np.zeros(T, bool),
                uv=np.zeros((V, 2)), shade=np.zeros(V), colors=np.zeros((V, K)), shaded=np.zeros(T, bool),
                edgeflags=np.zeros((T, 3), bool), height=camera.height, width=camera.width, nb_colors=K,
                texture=np.zeros((2, 2, K)), background_image=None, background_color=np.zeros(K),
                clockwise=m.clockwise, backface_culling=self.backface_culling, strict_edge=True,
                perspective_correct=False, integer_pixel_centers=True), m.device)
        return self._phong_scenes[key]

    def _albedo_scene(self, camera: CameraPytorch, uv: torch.Tensor, texture: torch.Tensor,
                      kind: str = "albedo") -> DeviceScene:
        """The cached albedo raster of a textured mesh for ``camera`` (with ``kind`` "normal_map" or "specular_map", that
        map's raster, its texture the map): all triangles textured and shaded, a shade of 1 at every vertex (set here
        once), colours zero, zero background."""
        from ..scenes import SceneArrays

        key = (camera.height, camera.width, tuple(texture.shape), uv.shape[0], kind)
        if key not in self._albedo_scenes:
            m = self.mesh
            T, V, nc = m.nb_faces, m.nb_vertices, texture.shape[2]
            self._albedo_scenes[key] = DeviceScene(SceneArrays(
                faces=np.ascontiguousarray(m.faces, dtype=np.uint32),
                faces_uv=np.ascontiguousarray(m.faces_uv, dtype=np.uint32), ij=np.zeros((V, 2)), depths=np.ones(V),
                textured=np.ones(T, bool), uv=np.zeros((uv.shape[0], 2)), shade=np.ones(V), colors=np.zeros((V, nc)),
                shaded=np.ones(T, bool), edgeflags=np.zeros((T, 3), bool), height=camera.height, width=camera.width,
                nb_colors=nc, texture=np.zeros(tuple(texture.shape)), background_image=None,
                background_color=np.zeros(nc), clockwise=m.clockwise, backface_culling=self.backface_culling,
                strict_edge=True, perspective_correct=False, integer_pixel_centers=True), m.device)
        return self._albedo_scenes[key]

    def _render_phong_textured(self, camera: CameraPytorch) -> torch.Tensor:
        m = self.mesh
        if self.light_ambient is None:
            raise ValueError("set_light first")
        if self.background_color is None:
            raise ValueError("set_background_color first")
        uv, texture = self._textured_inputs()
        if self.background_color.shape[0] != texture.shape[2]:
            raise ValueError(f"the background colour has {self.background_color.shape[0]} entries and the texture "
                             f"{texture.shape[2]} channels")
        ij, depths = camera.project_points(m.vertices)
        ones = torch.ones((m.nb_vertices, 1), dtype=torch.float64, device=m.device)
        channels = torch.cat((m.vertex_normals, m.vertices.to(torch.float64), ones), dim=1)
        nmap = map_scene = None
        if m.normal_map is not None:
            # (normals, positions, 1, tangents, bitangents), and the map's raster beside the albedo's
            nmap = m._tensor(m.normal_map)
            if tuple(nmap.shape) != tuple(texture.shape[:2]) + (3,):
                raise ValueError(f"normal_map must be [Ht,Wt,3] with the texture's Ht and Wt = "
                                 f"{tuple(texture.shape[:2])}; got {tuple(nmap.shape)}")
            channels = torch.cat((channels, vertex_tangents_autograd(m.vertices, uv, m.tangents)), dim=1)
            map_scene = self._albedo_scene(camera, uv, nmap, kind="normal_map")
        smap = spec_scene = None
        pbr = self.shading == "pbr_textured"
        if pbr and m.specular_map is not None:
            raise ValueError("shading='pbr_textured' reads a metallic-roughness map, not a specular map")
        if not pbr and m.metallic_roughness_map is not None:
            raise ValueError("a metallic-roughness map needs shading='pbr_textured'")
        material_map = m.metallic_roughness_map if pbr else m.specular_map
        if material_map is not None:
            # the material map's raster (specular or metallic-roughness), after the others
            kind = "metallic_roughness_map" if pbr else "specular_map"
            smap = m._tensor(material_map)
            if tuple(smap.shape) != tuple(texture.shape[:2]) + (2,):
                raise ValueError(f"{kind} must be [Ht,Wt,2] with the texture's Ht and Wt = "
                                 f"{tuple(texture.shape[:2])}; got {tuple(smap.shape)}")
            spec_scene = self._albedo_scene(camera, uv, smap, kind=kind)
        rasters = 2 + (nmap is not None) + (smap is not None)
        vis = sun = None
        if self.shadow_map_size or self.light_shadow_map_size:
            out = self._render_shadowed(ij, uv, texture, channels, depths, self._albedo_scene(camera, uv, texture),
                                        self._phong_scene(camera, 0, nmap is not None), nmap, map_scene, smap,
                                        spec_scene)
            albedo, gbuffer = out[:2]
            if nmap is not None:
                gbuffer = normal_map_autograd(gbuffer, out[2])
            vis, sun = self._visibilities(gbuffer, out[rasters:], albedo)
        else:
            out = render_mesh_phong_textured(ij, uv, texture, channels, depths, self._edgeflags(ij),
                                             self._albedo_scene(camera, uv, texture),
                                             self._phong_scene(camera, 0, nmap is not None), self.sigma, nmap,
                                             map_scene, smap, spec_scene)
            albedo, gbuffer = out[:2]
            if nmap is not None:
                gbuffer = normal_map_autograd(gbuffer, out[2])
        spec = out[rasters - 1] if smap is not None else None
        material = (self.metallic, self.roughness) if pbr else (self.specular, self.shininess)
        return phong_shade_autograd(gbuffer, self.light_directional, self.light_ambient, material[0], material[1],
                                    camera.center() if camera.is_tensor else camera, self.background_color,
                                    self.light_sh, albedo, self.point_lights, vis, sun, spec,
                                    "ggx" if pbr else "phong")

    def _render_phong(self, camera: CameraPytorch) -> torch.Tensor:
        m = self.mesh
        if self.light_ambient is None:
            raise ValueError("set_light first")
        if self.background_color is None:
            raise ValueError("set_background_color first")
        nc = m.vertices_colors.shape[1]
        if self.background_color.shape[0] != nc:
            raise ValueError(f"the background colour has {self.background_color.shape[0]} entries and the mesh "
                             f"{nc} colour channels")
        ij, depths = camera.project_points(m.vertices)
        ones = torch.ones((m.nb_vertices, 1), dtype=torch.float64, device=m.device)
        channels = torch.cat((m.vertices_colors.to(torch.float64), m.vertex_normals, m.vertices.to(torch.float64),
                              ones), dim=1)
        vis = sun = None
        if self.shadow_map_size or self.light_shadow_map_size:
            out = self._render_shadowed(ij, None, None, channels, depths, None, self._phong_scene(camera, nc))
            raster = out[0]
            vis, sun = self._visibilities(raster, out[1:], None)
        else:
            raster = render_mesh_2d(ij, channels, depths, self._edgeflags(ij), self._phong_scene(camera, nc),
                                    self.sigma)
        return phong_shade_autograd(raster, self.light_directional, self.light_ambient, self.specular, self.shininess,
                                    camera.center() if camera.is_tensor else camera, self.background_color,
                                    self.light_sh, None, self.point_lights, vis, sun)

    def _render_shadowed(self, ij, uv, texture, channels, depths, albedo_scene, gbuffer_scene, normal_map=None,
                         map_scene=None, specular_map=None, spec_scene=None) -> tuple:
        """The rasters and the shadow maps in one :class:`RenderShadowedPhongFunc` node."""
        m = self.mesh
        cubes = self._shadow_cubes() if self.shadow_map_size else None
        sun = self._sun_map() if self.light_shadow_map_size else None
        return render_shadowed_phong(ij, uv, texture, channels, depths, self._edgeflags(ij), m.vertices,
                                     self.point_lights if cubes is not None else None, albedo_scene, gbuffer_scene,
                                     cubes, self.sigma, self.light_directional if sun is not None else None, sun,
                                     normal_map, map_scene, specular_map, spec_scene)

    def _visibilities(self, gbuffer, maps, albedo) -> tuple:
        """(the point lights' visibility or None, the directional light's or None) from the node's maps."""
        vis = sun = None
        if self.shadow_map_size:
            vis = shadow_visibility_autograd(gbuffer, self.point_lights, maps[0], self.shadow_bias,
                                             self.shadow_softness, albedo)
        if self.light_shadow_map_size:
            sun = sun_visibility_autograd(gbuffer, self.light_directional, maps[-1], self.light_shadow_bounds,
                                          self.light_shadow_bias, self.light_shadow_softness, albedo)
        return vis, sun

    def _sun_map(self) -> SunShadowMap:
        """The cached directional-light shadow map of the mesh for the map size and the window."""
        m = self.mesh
        key = (self.light_shadow_map_size, self.light_shadow_bounds)
        if key not in self._suns:
            self._suns[key] = SunShadowMap(np.ascontiguousarray(m.faces, dtype=np.uint32), m.nb_vertices, key[0],
                                           key[1], m.clockwise, m.device)
        return self._suns[key]

    def _shadow_cubes(self) -> ShadowCubes:
        """The cached cube shadow maps of the mesh for the lights' count and the map size."""
        m = self.mesh
        key = (self.point_lights.shape[0], self.shadow_map_size)
        if key not in self._cubes:
            self._cubes[key] = ShadowCubes(np.ascontiguousarray(m.faces, dtype=np.uint32), m.nb_vertices, key[0],
                                           key[1], m.clockwise, m.device)
        return self._cubes[key]

    def _edgeflags(self, ij: torch.Tensor) -> torch.Tensor:
        if self.sigma > 0:
            return self.mesh.topology.edge_on_silhouette(ij.detach())
        return torch.zeros((self.mesh.nb_faces, 3), dtype=torch.uint8, device=self.mesh.device)

    def _compute_vertices_colors_with_illumination(self) -> torch.Tensor:
        m = self.mesh
        if self.light_ambient is None:
            raise ValueError("set_light first")
        if self.point_lights is not None:
            return point_lit_vertex_colors_autograd(m.vertex_normals, m.vertices, m.vertices_colors,
                                                    self.light_directional, self.light_ambient, self.light_sh,
                                                    self.point_lights)
        if self.light_sh is not None:  # the environment reads the normals, with or without a directional light
            return sh_lit_vertex_colors_autograd(m.vertex_normals, m.vertices_colors, self.light_directional,
                                                 self.light_ambient, self.light_sh)
        normals = m.vertex_normals if self.light_directional is not None else torch.zeros(
            (m.nb_vertices, 3), dtype=torch.float64, device=m.device)
        return lit_vertex_colors_autograd(normals, m.vertices_colors, self.light_directional, self.light_ambient)

    def _compute_vertices_luminosity(self) -> torch.Tensor:
        m = self.mesh
        if self.light_ambient is None:
            raise ValueError("set_light first")
        if self.point_lights is not None:
            if self.point_lights.shape[1] != 4:
                raise ValueError("a textured mesh takes grey point lights [L, 4] only: its shade has one channel")
            sh = self.light_sh
            if sh is not None and sh.dim() == 2 and sh.shape[1] != 1:
                raise ValueError("a textured mesh takes a grey environment [9] only: its shade has one channel")
            return point_lit_vertex_colors_autograd(m.vertex_normals, m.vertices, None, self.light_directional,
                                                    self.light_ambient, sh.reshape(9) if sh is not None else None,
                                                    self.point_lights)
        if self.light_sh is not None:
            if self.light_sh.dim() == 2 and self.light_sh.shape[1] != 1:
                raise ValueError("a textured mesh takes a grey environment [9] only: its shade has one channel")
            return sh_lit_vertex_colors_autograd(m.vertex_normals, None, self.light_directional, self.light_ambient,
                                                 self.light_sh.reshape(9))
        normals = m.vertex_normals if self.light_directional is not None else torch.zeros(
            (m.nb_vertices, 3), dtype=torch.float64, device=m.device)
        return vertex_luminosity_autograd(normals, self.light_directional, self.light_ambient)

    def render(self, camera: CameraPytorch) -> torch.Tensor:
        """The mesh's vertex colours, Gouraud-lit (per pixel with ``shading="phong"``), rendered by ``camera`` -> image
        [H,W,C] fp32.  For a textured mesh,
        ``Scene3D.render``'s uv branch: the texture, sampled at the interpolated uv, times the interpolated vertex
        luminosity (differentiable in the vertices, uv, texture and light); with ``shading="phong_textured"`` the
        sampled texture lit per pixel, and with ``shading="pbr_textured"`` the metallic-roughness form."""
        if self.mesh is not None and self.mesh.textured:
            if self.shading == "phong":
                raise ValueError("phong shading of a textured mesh is shading='phong_textured'")
            if self.shading in ("phong_textured", "pbr_textured"):
                return self._render_phong_textured(camera)
            return self._render_textured(camera)
        if self.shading in ("phong_textured", "pbr_textured"):
            raise ValueError(f"shading={self.shading!r} needs a textured mesh; an untextured one takes "
                             f"shading='phong'")
        if self.mesh is None or self.mesh.vertices_colors is None:
            raise ValueError("render needs a mesh with vertex colours (set_mesh, set_vertices_colors)")
        if self.shading == "phong":
            return self._render_phong(camera)
        ij, depths = camera.project_points(self.mesh.vertices)
        colors = self._compute_vertices_colors_with_illumination()
        scene = self._scene(camera, colors.shape[1])
        return render_mesh_2d(ij, colors, depths, self._edgeflags(ij), scene, self.sigma)

    def _textured_inputs(self) -> Tuple[torch.Tensor, torch.Tensor]:
        m = self.mesh
        uv, texture = m._tensor(m.uv), m._tensor(m.texture)
        if texture.dim() != 3 or uv.dim() != 2 or uv.shape[1] != 2:
            raise ValueError(f"a textured mesh needs texture [Ht,Wt,C] and uv [Nuv,2]; got {tuple(texture.shape)} and "
                             f"{tuple(uv.shape)}")
        if m.faces_uv.size and int(m.faces_uv.max()) >= uv.shape[0]:
            raise ValueError(f"uv has {uv.shape[0]} rows; faces_uv indexes row {int(m.faces_uv.max())}")
        return uv, texture

    def _render_textured(self, camera: CameraPytorch) -> torch.Tensor:
        m = self.mesh
        uv, texture = self._textured_inputs()
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


class SelfCollisionEnergyPytorch:
    """A self-collision penalty under autograd (``DeviceSelfCollisionEnergy``): ``evaluate(v)`` -> energy 0-d fp64,
    differentiable when ``v`` requires grad.  ``min_distance`` and ``intersections(v)`` are the device model's."""

    def __init__(self, faces, vertices_ref, thickness: float, weight: float, device=None):
        faces = faces.faces if hasattr(faces, "faces") else faces
        if isinstance(faces, torch.Tensor):
            faces = faces.cpu().numpy()
        if isinstance(vertices_ref, torch.Tensor):
            device = vertices_ref.device if device is None else device
            vertices_ref = vertices_ref.detach().cpu().numpy()
        self.model = DeviceSelfCollisionEnergy(np.asarray(faces), np.asarray(vertices_ref, dtype=np.float64), thickness,
                                               weight, _device(device))

    @property
    def min_distance(self) -> torch.Tensor:
        return self.model.min_distance

    def intersections(self, vertices: torch.Tensor) -> torch.Tensor:
        return self.model.intersections(vertices.detach())

    def evaluate(self, vertices: torch.Tensor) -> torch.Tensor:
        if vertices.requires_grad:
            return SelfCollisionEnergyFunc.apply(vertices, self.model)
        return self.model.evaluate(vertices)[0]
