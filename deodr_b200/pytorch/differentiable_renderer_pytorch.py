"""autograd surface of the 2D render, mirroring deodr/pytorch/differentiable_renderer_pytorch.py:41-81.

Two Functions with the reference contract ``(ij, colors, scene) -> image[H,W,C]``, backward ``(ij_b, colors_b, None)``:

* ``TorchDifferentiableRenderer2DFunc`` - signature-compatible with the reference class of the same name: ``scene`` is
  an object with a ``scene_2d`` attribute (``Scene3DPytorch`` in the reference), tensors are CPU float64, sigma is 1;
  data crosses to the GPU through the reference-shaped host entry points.
* ``CudaDifferentiableRenderer2DFunc`` - the zero-copy variant: ``scene`` is a ``deodr_b200.renderer.DeviceScene``,
  ``ij`` / ``colors`` are CUDA tensors, the image stays on the device.

and one without a reference counterpart (its scene has no background gradient):

* ``CudaDifferentiableRender2DWithBackground`` - ``(ij, colors, background, scene, sigma) -> image``, with the
  background ([C] colour or [H,W,C] image, the kind the ``DeviceScene`` holds) as a differentiable input too.

and the fitting step of the reference's ``Scene2D.render_compare_and_backward`` as a Function:

* ``CudaRenderCompare2D`` - ``(ij, colors, obs, mask, scene, sigma, antialiase_error) -> loss``, the render compared
  with an observed image on the device.

and their textured counterparts, differentiable in all five per-scene inputs of the rasteriser's adjoint (the
reference's 2D Function returns ``(ij_b, colors_b)`` only; its ``Scene2D`` computes ``uv_b``, ``shade_b`` and
``texture_b`` but no Function exposes them):

* ``CudaDifferentiableRender2DTextured`` - ``(ij, colors, uv, shade, texture, scene, sigma) -> image``;
* ``CudaRenderCompare2DTextured`` - ``(ij, colors, uv, shade, texture, obs, mask, scene, sigma, antialiase_error)
  -> loss``.

Their texture gradient is the summed adjoint of the bilinear sample (the reference's overwrites, INTEGRATION.md
section 5).  Backward returns only the gradients autograd asks for, and leaves the texture's adjoint slot NULL (not
computed) when its gradient is not asked for.
"""

from __future__ import annotations

from typing import Any, Dict, Optional

import numpy as np
import torch

from .. import differentiable_renderer_cython
from ..renderer import DeviceScene, default_renderer


class TorchDifferentiableRenderer2DFunc(torch.autograd.Function):
    """CPU-tensor in / CPU-tensor out, same contract as the reference Function."""

    @staticmethod
    def forward(ctx: Any, ij: torch.Tensor, colors: torch.Tensor, scene: Any) -> torch.Tensor:  # type: ignore
        scene_2d = scene.scene_2d
        image = np.empty((scene_2d.height, scene_2d.width, colors.shape[1]))
        z_buffer = np.empty((scene_2d.height, scene_2d.width))
        ctx.scene = scene
        scene_2d.ij = ij.detach().numpy()
        scene.colors = colors.detach().numpy()
        differentiable_renderer_cython.renderSceneCpp(scene_2d, 1, image, z_buffer)
        ctx.save_for_backward(ij, colors)
        ctx.image = image.copy()
        ctx.z_buffer = z_buffer
        return torch.as_tensor(image)

    @staticmethod
    def backward(ctx: Any, *grad_outputs: Any) -> Any:
        assert len(grad_outputs) == 1
        image_b = np.ascontiguousarray(grad_outputs[0].detach().numpy(), dtype=np.float64)
        scene_2d = ctx.scene.scene_2d
        scene_2d.uv_b = np.zeros(scene_2d.uv.shape)
        scene_2d.ij_b = np.zeros(scene_2d.ij.shape)
        scene_2d.shade_b = np.zeros(scene_2d.shade.shape)
        scene_2d.colors_b = np.zeros(scene_2d.colors.shape)
        scene_2d.texture_b = np.zeros(scene_2d.texture.shape)
        differentiable_renderer_cython.renderSceneBCpp(scene_2d, 1, ctx.image, ctx.z_buffer, image_b)
        return torch.as_tensor(scene_2d.ij_b), torch.as_tensor(scene_2d.colors_b), None


TorchDifferentiableRender2D = TorchDifferentiableRenderer2DFunc.apply


class CudaDifferentiableRenderer2DFunc(torch.autograd.Function):
    """Device-resident variant: ``image = f(ij[V,2] f64 cuda, colors[V,C] cuda, DeviceScene, sigma)``.

    The renderer keeps ONE live forward state per slot, and the ``DeviceScene`` is shared and mutable, so the node
    snapshots its inputs; if another forward has used the slot by the time ``backward`` runs (two renders before
    ``loss.backward()``), the forward is replayed from the snapshot first."""

    @staticmethod
    def forward(ctx: Any, ij: torch.Tensor, colors: torch.Tensor, scene: DeviceScene, sigma: float = 1.0):  # type: ignore
        scene.update(ij=ij.detach(), colors=colors.detach())
        fwd = default_renderer(scene.device.index).render(scene, sigma)
        ctx.scene, ctx.sigma, ctx.fwd = scene, float(sigma), fwd
        ctx.in_dtypes = (ij.dtype, colors.dtype)
        ctx.save_for_backward(ij.detach().clone(), colors.detach().clone())
        # the caller gets its own tensor: the framebuffers of ctx.fwd may be re-rendered into by backward
        return fwd["image"].clone()

    @staticmethod
    def backward(ctx: Any, *grad_outputs: Any) -> Any:
        (image_b,) = grad_outputs
        renderer = default_renderer(ctx.scene.device.index)
        ij, colors = ctx.saved_tensors
        if ctx.fwd["generation"] != renderer.generation(ctx.fwd["slot"]):
            ctx.scene.update(ij=ij, colors=colors)
            ctx.fwd = renderer.render(ctx.scene, ctx.sigma, out=ctx.fwd)
        else:
            ctx.scene.update(ij=ij, colors=colors)  # the shared scene may hold another node's inputs by now
        grads = renderer.render_b(ctx.scene, ctx.sigma, ctx.fwd, image_b)
        return grads["ij_b"].to(ctx.in_dtypes[0]), grads["colors_b"].to(ctx.in_dtypes[1]), None, None


CudaDifferentiableRender2D = CudaDifferentiableRenderer2DFunc.apply


class CudaDifferentiableRenderer2DWithBackgroundFunc(torch.autograd.Function):
    """``image = f(ij[V,2], colors[V,C], background, DeviceScene, sigma)`` on the device, differentiable in the
    background as well: ``background`` is a [C] CUDA tensor for a scene rendered over a background colour, [H,W,C] for
    one rendered over a background image.  Backward returns ``(ij_b, colors_b, background_b, None, None)``.  Same
    snapshot / re-render logic as ``CudaDifferentiableRenderer2DFunc``."""

    @staticmethod
    def forward(ctx: Any, ij: torch.Tensor, colors: torch.Tensor, background: torch.Tensor, scene: DeviceScene,  # type: ignore
                sigma: float = 1.0):
        kind = scene.background_kind
        if tuple(background.shape) != tuple(scene.t[kind].shape):
            raise ValueError(f"background has shape {tuple(background.shape)}; the scene is rendered with {kind} of "
                             f"shape {tuple(scene.t[kind].shape)}")
        scene.update(ij=ij.detach(), colors=colors.detach(), **{kind: background.detach()})
        fwd = default_renderer(scene.device.index).render(scene, sigma)
        ctx.scene, ctx.sigma, ctx.fwd, ctx.kind = scene, float(sigma), fwd, kind
        ctx.in_dtypes = (ij.dtype, colors.dtype, background.dtype)
        ctx.save_for_backward(ij.detach().clone(), colors.detach().clone(), background.detach().clone())
        return fwd["image"].clone()

    @staticmethod
    def backward(ctx: Any, *grad_outputs: Any) -> Any:
        (image_b,) = grad_outputs
        renderer = default_renderer(ctx.scene.device.index)
        ij, colors, background = ctx.saved_tensors
        # the shared scene may hold another node's inputs by now
        ctx.scene.update(ij=ij, colors=colors, **{ctx.kind: background})
        if ctx.fwd["generation"] != renderer.generation(ctx.fwd["slot"]):
            ctx.fwd = renderer.render(ctx.scene, ctx.sigma, out=ctx.fwd)
        bg = ctx.scene.zero_background_grads()
        grads = renderer.render_b(ctx.scene, ctx.sigma, ctx.fwd, image_b, background_grads=bg)
        return (grads["ij_b"].to(ctx.in_dtypes[0]), grads["colors_b"].to(ctx.in_dtypes[1]),
                bg[ctx.kind + "_b"].to(ctx.in_dtypes[2]), None, None)


CudaDifferentiableRender2DWithBackground = CudaDifferentiableRenderer2DWithBackgroundFunc.apply


class CudaRenderCompare2DFunc(torch.autograd.Function):
    """``loss = f(ij[V,2], colors[V,C], obs[H,W,C], mask[H,W] | None, DeviceScene, sigma, antialiase_error)``: the render
    compared with ``obs`` on the device (``Renderer.render_compare``), a 0-d fp64 CUDA tensor differentiable in ``ij``
    and ``colors``.  The comparison computes the adjoint input of the loss with the loss (``image_b = 2 * m * d``, or
    ``err_buffer_b = m`` in antialiase_error mode), so no image is returned and autograd builds no elementwise graph.
    The adjoint is linear in its input: ``backward`` scales the fresh gradients by ``grad_loss`` on the device, without
    a host synchronisation.  Same snapshot / re-render logic as ``CudaDifferentiableRenderer2DFunc``; a re-render
    recomputes ``image_b`` too.  ``obs`` and ``mask`` must not be modified in place before ``backward`` (autograd
    checks)."""

    @staticmethod
    def forward(ctx: Any, ij: torch.Tensor, colors: torch.Tensor, obs: torch.Tensor, mask: Any,  # type: ignore
                scene: DeviceScene, sigma: float = 1.0, antialiase_error: bool = False):
        scene.update(ij=ij.detach(), colors=colors.detach())
        res = default_renderer(scene.device.index).render_compare(scene, sigma, obs, mask,
                                                                  antialiase_error=antialiase_error)
        ctx.scene, ctx.sigma, ctx.res, ctx.err_mode = scene, float(sigma), res, bool(antialiase_error)
        ctx.in_dtypes = (ij.dtype, colors.dtype)
        ctx.save_for_backward(ij.detach().clone(), colors.detach().clone(), obs, mask)
        # the caller gets its own scalar: ctx.res may be re-rendered into by backward
        return res["loss"].clone()

    @staticmethod
    def backward(ctx: Any, *grad_outputs: Any) -> Any:
        (grad_loss,) = grad_outputs
        renderer = default_renderer(ctx.scene.device.index)
        ij, colors, obs, mask = ctx.saved_tensors
        ctx.scene.update(ij=ij, colors=colors)  # the shared scene may hold another node's inputs by now
        if ctx.res["generation"] != renderer.generation(ctx.res["slot"]):
            ctx.res = renderer.render_compare(ctx.scene, ctx.sigma, obs, mask, antialiase_error=ctx.err_mode,
                                              out=ctx.res)
        if ctx.err_mode:
            grads = renderer.render_b(ctx.scene, ctx.sigma, ctx.res, err_buffer_b=renderer.compare_adjoint_input(ctx.res))
        else:
            grads = renderer.render_b(ctx.scene, ctx.sigma, ctx.res, ctx.res["image_b"])
        scale = grad_loss.to(torch.float32)
        return ((grads["ij_b"] * scale).to(ctx.in_dtypes[0]), (grads["colors_b"] * scale).to(ctx.in_dtypes[1]),
                None, None, None, None, None)


CudaRenderCompare2D = CudaRenderCompare2DFunc.apply


TEXTURED_INPUTS = ("ij", "colors", "uv", "shade", "texture")


def check_scene_inputs(scene: DeviceScene, **inputs: torch.Tensor) -> None:
    """``ValueError`` unless every tensor is a CUDA tensor of the shape the ``DeviceScene`` holds under its name."""
    for name, t in inputs.items():
        want = tuple(scene.t[name].shape)
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise ValueError(f"{name} must be a CUDA tensor of shape {want}")
        if tuple(t.shape) != want:
            raise ValueError(f"{name} has shape {tuple(t.shape)}; the scene expects {want}")


def requested_grads(scene: DeviceScene, names, needs) -> Dict[str, torch.Tensor]:
    """Zeroed fp32 gradient slots ``{name + "_b": ...}`` for the adjoint of a textured scene.  The library needs the
    ij, colour, uv and shade slots; the texture slot, the only one it may leave NULL (and the largest), is allocated
    only when ``needs`` asks for the texture gradient (``names`` and ``needs`` as the Function's inputs)."""
    want_texture = dict(zip(names, needs)).get("texture", False)
    return {n + "_b": torch.zeros(scene.t[n].shape, dtype=torch.float32, device=scene.device)
            for n in TEXTURED_INPUTS if n != "texture" or want_texture}


def gradients_of(grads: Dict[str, torch.Tensor], names, dtypes, needs,
                 scale: Optional[torch.Tensor] = None) -> tuple:
    """The gradients of ``names`` in their inputs' dtypes (times ``scale``), None where ``needs`` asks for none."""
    out = []
    for n, dtype, need in zip(names, dtypes, needs):
        g = grads[n + "_b"] if need else None
        if g is not None and scale is not None:
            g = g * scale
        out.append(g.to(dtype) if g is not None else None)
    return tuple(out)


class CudaDifferentiableRenderer2DTexturedFunc(torch.autograd.Function):
    """``image = f(ij [V,2], colors [V,C], uv [Nuv,2], shade [V], texture [Ht,Wt,C], DeviceScene, sigma)`` on the
    device, CUDA tensors shaped like the scene's.  Backward returns the gradient of each of the five inputs that needs
    one, in its own dtype (None for the others), then ``None, None``.  Same snapshot / re-render logic as
    ``CudaDifferentiableRenderer2DFunc``, over all five inputs."""

    @staticmethod
    def forward(ctx: Any, ij: torch.Tensor, colors: torch.Tensor, uv: torch.Tensor, shade: torch.Tensor,  # type: ignore
                texture: torch.Tensor, scene: DeviceScene, sigma: float = 1.0):
        inputs = dict(zip(TEXTURED_INPUTS, (ij, colors, uv, shade, texture)))
        check_scene_inputs(scene, **inputs)
        scene.update(**{k: t.detach() for k, t in inputs.items()})
        fwd = default_renderer(scene.device.index).render(scene, sigma)
        ctx.scene, ctx.sigma, ctx.fwd = scene, float(sigma), fwd
        ctx.in_dtypes = tuple(t.dtype for t in inputs.values())
        ctx.save_for_backward(*(t.detach().clone() for t in inputs.values()))
        # the caller gets its own tensor: the framebuffers of ctx.fwd may be re-rendered into by backward
        return fwd["image"].clone()

    @staticmethod
    def backward(ctx: Any, image_b: torch.Tensor):  # type: ignore
        needs = ctx.needs_input_grad[:5]
        if not any(needs):
            return (None,) * 7
        renderer = default_renderer(ctx.scene.device.index)
        # the shared scene may hold another node's inputs by now
        ctx.scene.update(**dict(zip(TEXTURED_INPUTS, ctx.saved_tensors)))
        if ctx.fwd["generation"] != renderer.generation(ctx.fwd["slot"]):
            ctx.fwd = renderer.render(ctx.scene, ctx.sigma, out=ctx.fwd)
        grads = requested_grads(ctx.scene, TEXTURED_INPUTS, needs)
        renderer.render_b(ctx.scene, ctx.sigma, ctx.fwd, image_b.contiguous(), grads=grads)
        return gradients_of(grads, TEXTURED_INPUTS, ctx.in_dtypes, needs) + (None, None)


CudaDifferentiableRender2DTextured = CudaDifferentiableRenderer2DTexturedFunc.apply


class CudaRenderCompare2DTexturedFunc(torch.autograd.Function):
    """``loss = f(ij, colors, uv, shade, texture, obs [H,W,C], mask [H,W] | None, DeviceScene, sigma,
    antialiase_error)``: ``CudaRenderCompare2DFunc`` (same loss, both modes, the gradients scaled by ``grad_loss`` on
    the device) differentiable in the five inputs of ``CudaDifferentiableRenderer2DTexturedFunc``."""

    @staticmethod
    def forward(ctx: Any, ij: torch.Tensor, colors: torch.Tensor, uv: torch.Tensor, shade: torch.Tensor,  # type: ignore
                texture: torch.Tensor, obs: torch.Tensor, mask: Any, scene: DeviceScene, sigma: float = 1.0,
                antialiase_error: bool = False):
        inputs = dict(zip(TEXTURED_INPUTS, (ij, colors, uv, shade, texture)))
        check_scene_inputs(scene, **inputs)
        scene.update(**{k: t.detach() for k, t in inputs.items()})
        res = default_renderer(scene.device.index).render_compare(scene, sigma, obs, mask,
                                                                  antialiase_error=antialiase_error)
        ctx.scene, ctx.sigma, ctx.res, ctx.err_mode = scene, float(sigma), res, bool(antialiase_error)
        ctx.in_dtypes = tuple(t.dtype for t in inputs.values())
        ctx.save_for_backward(*(t.detach().clone() for t in inputs.values()), obs, mask)
        # the caller gets its own scalar: ctx.res may be re-rendered into by backward
        return res["loss"].clone()

    @staticmethod
    def backward(ctx: Any, grad_loss: torch.Tensor):  # type: ignore
        needs = ctx.needs_input_grad[:5]
        if not any(needs):
            return (None,) * 10
        renderer = default_renderer(ctx.scene.device.index)
        *inputs, obs, mask = ctx.saved_tensors
        ctx.scene.update(**dict(zip(TEXTURED_INPUTS, inputs)))  # the shared scene may hold another node's inputs
        if ctx.res["generation"] != renderer.generation(ctx.res["slot"]):
            ctx.res = renderer.render_compare(ctx.scene, ctx.sigma, obs, mask, antialiase_error=ctx.err_mode,
                                              out=ctx.res)
        grads = requested_grads(ctx.scene, TEXTURED_INPUTS, needs)
        if ctx.err_mode:
            renderer.render_b(ctx.scene, ctx.sigma, ctx.res, grads=grads,
                              err_buffer_b=renderer.compare_adjoint_input(ctx.res))
        else:
            renderer.render_b(ctx.scene, ctx.sigma, ctx.res, ctx.res["image_b"], grads=grads)
        return gradients_of(grads, TEXTURED_INPUTS, ctx.in_dtypes, needs, grad_loss.to(torch.float32)) + (None,) * 5


CudaRenderCompare2DTextured = CudaRenderCompare2DTexturedFunc.apply
