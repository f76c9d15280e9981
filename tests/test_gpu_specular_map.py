"""GPU: specular maps in textured Phong views - the shading kernels against the fp64 restatement
(tests/specular_map_ref.py) with and without shadows, a map of ones against the view without a map on the duck under
an environment, a shadowed point light and the sun's shadow, gradients against central differences, the PyTorch path
against the device view, the refusals, no host synchronisation, and a fit of a glossy / matte map."""
import json
import os

import numpy as np
import pytest
import specular_map_ref as ref

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from deodr_b200 import mesh_ops  # noqa: E402
from deodr_b200.mesh_fitter import new_scratch  # noqa: E402
from deodr_b200.mesh_ops import CameraParams, DeviceMeshView  # noqa: E402
from deodr_b200.pytorch import scene3d_pytorch as P  # noqa: E402

DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def host(t):
    return t.detach().cpu().numpy().astype(np.float64)


def cuda(a, dtype=torch.float64):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def f32(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def record(name, value):
    print(json.dumps({"measured": name, "value": value}))


def rel(got, want):
    return float(np.abs(np.asarray(got) - np.asarray(want)).max() / max(np.abs(np.asarray(want)).max(), 1e-300))


SIZE, FOCAL = 128, 120.0


def camera(size=SIZE, focal=FOCAL):
    return CameraParams(np.eye(3, 4), np.array([[focal, 0, (size - 1) / 2], [0, focal, (size - 1) / 2], [0, 0, 1]]))


def duck():
    """The duck, centred at (0, 0, 4) with a radius of about 1.3, in front of :func:`camera`."""
    d = np.load(f"{GOLDEN}/duck_textured.npz")
    v = d["vertices"]
    v = (v - (v.min(0) + v.max(0)) / 2) + np.array([0.0, 0.0, 4.0])
    return v, d["faces"].astype(np.int64), d["uv"], d["faces_uv"].astype(np.int64), d["texture_u8"] / 255.0


def grid_plane(z=4.0, half=1.0, n=16, texels=32):
    """The square |x|, |y| <= half at depth z, facing -z (the camera), uv covering the texture: u along +x."""
    g = np.linspace(-half, half, n + 1)
    x, y = np.meshgrid(g, g, indexing="ij")
    v = np.stack((x, y, np.full_like(x, z)), axis=-1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    q = (i * (n + 1) + j).ravel()
    f = np.concatenate((np.stack((q, q + n + 1, q + n + 2), 1), np.stack((q, q + n + 2, q + 1), 1)))
    tri = v[f]
    flip = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])[:, 2] > 0
    f[flip] = f[flip][:, ::-1]
    uv = (v[:, :2] + half) / (2 * half) * (texels - 1)
    return v, f.astype(np.int64), uv, f.copy()


# ------------------------------------------------------------------------------------- 1. the shading kernels

KERNEL_CASES = {
    "plain": dict(),
    "sh_grey_point": dict(sh="grey", lights="grey"),
    "sh_colour_points_colour": dict(sh="colour", lights="colour"),
    "points_vis": dict(lights="grey", vis=True),
    "sun": dict(sun=True),
    "sh_points_vis_sun": dict(sh="colour", lights="colour", vis=True, sun=True),
}


def _pixels(rng, H=17, W=23, C=3, L=2, sh=None, lights=None, vis=False, sun=False):
    P_ = H * W
    G, A, spec = ref.random_pixels(rng, C, P_, (0.0, 0.1, -5.0))
    G[0::13] = 0.0  # a = 0 (the albedo raster is 0 there too)
    A[0::13] = 0.0
    spec[2::13, 0] = 0.0  # K = 0
    G[3::13, 0:3] = np.array([0.0, 0.0, 5.0]) * G[3::13, 6:7]  # facing away from every light: s = 0
    G, A, spec = f32(G), f32(A), f32(spec)
    shv = {None: None, "grey": rng.normal(size=9) * 0.2, "colour": rng.normal(size=(9, C)) * 0.2}[sh]
    S = {None: 0, "grey": 1, "colour": C}[lights]
    table = None
    if lights:
        table = np.concatenate((np.array([0.0, 0.1, -5.0]) + rng.uniform(-2, 2, (L, 3)),
                                rng.uniform(0.5, 2.0, (L, S))), axis=1)
    V = f32(rng.uniform(0, 1, (P_, L))) if vis else None
    sv = f32(rng.uniform(0, 1, P_)) if sun else None
    return dict(G=G, A=A, spec=spec, sh=shv, lights=table, vis=V, sun_vis=sv), (H, W, C, L)


@pytest.mark.parametrize("case", list(KERNEL_CASES))
def test_the_kernels_match_the_restatement(case):
    rng = np.random.default_rng(11)
    kw, (H, W, C, L) = _pixels(rng, **KERNEL_CASES[case])
    params = np.array([0.3, 0.5, 0.8, 0.4, 0.7, 12.0])
    cam = np.array([0.0, 0.1, -5.0])
    bg = f32([0.2, 0.3, 0.4])
    g = f32(rng.normal(size=(H * W, C)))
    want = ref.shade(kw["G"], kw["A"], kw["spec"], params, cam, bg, kw["sh"], kw["lights"], kw["vis"], kw["sun_vis"])
    grads = ref.shade_b(g, kw["G"], kw["A"], kw["spec"], params, cam, bg, kw["sh"], kw["lights"], kw["vis"],
                        kw["sun_vis"])
    dev = dict(albedo=cuda(kw["A"].reshape(H, W, C), torch.float32),
               specular=cuda(kw["spec"].reshape(H, W, 2), torch.float32),
               sh=cuda(kw["sh"]) if kw["sh"] is not None else None,
               point_lights=cuda(kw["lights"]) if kw["lights"] is not None else None,
               visibility=cuda(kw["vis"].reshape(H, W, L), torch.float32) if kw["vis"] is not None else None,
               sun_visibility=cuda(kw["sun_vis"].reshape(H, W), torch.float32) if kw["sun_vis"] is not None else None)
    ch, pd, cd, bd = cuda(kw["G"].reshape(H, W, 7), torch.float32), cuda(params), cuda(cam), cuda(bg, torch.float32)
    image = host(mesh_ops.phong_shade(ch, pd, cd, bd, **dev))
    out = mesh_ops.phong_shade_backward(ch, pd, cd, bd, cuda(g.reshape(H, W, C), torch.float32), new_scratch(DEV),
                                        center_grad=True, **dev)
    out = list(out)
    spec_b = host(out.pop())
    sun_b = host(out.pop()) if kw["sun_vis"] is not None else None
    vis_b = host(out.pop()) if kw["vis"] is not None else None
    lights_b = host(out.pop()) if kw["lights"] is not None else None
    albedo_b = host(out.pop())
    sh_b = host(out.pop()) if kw["sh"] is not None else None
    channels_b, params_b, center_b = (host(t) for t in out)
    errs = {"image": float(np.abs(image.reshape(-1, C) - want).max()),
            "spec_b": rel(spec_b.reshape(-1, 2), grads["spec_b"]), "albedo_b": rel(albedo_b.reshape(-1, C),
                                                                                  grads["A_b"]),
            "channels_b": rel(channels_b.reshape(-1, 7), grads["G_b"]),
            "params_b": rel(params_b, grads["params_b"]), "camera_center_b": rel(center_b, grads["cam_b"])}
    if lights_b is not None:
        errs["lights_b"] = rel(lights_b, grads["lights_b"])
    if sh_b is not None:
        errs["sh_b"] = rel(sh_b, grads["sh_b"])
    if vis_b is not None:
        errs["vis_b"] = rel(vis_b.reshape(-1, L), grads["vis_b"])
    if sun_b is not None:
        errs["sun_vis_b"] = rel(sun_b.reshape(-1), grads["sun_vis_b"])
    record(f"specular_map_kernels_{case}", errs)
    assert errs["image"] <= 2e-6
    for k in ("spec_b", "albedo_b", "channels_b", "vis_b", "sun_vis_b"):
        assert errs.get(k, 0.0) <= 1e-5, k
    for k in ("params_b", "camera_center_b", "lights_b", "sh_b"):
        assert errs.get(k, 0.0) <= 1e-9, k
    assert not np.any(spec_b.reshape(-1, 2)[0::13])  # 0 where a = 0


# ----------------------------------------------------------------------------------------- 2. a map of ones

LIGHT = np.array([0.3, -0.4, 0.8])
POINT = np.array([[1.5, -1.0, 2.0, 4.0]])
SH = np.array([0.5, 0.1, -0.2, 0.05, 0.02, -0.03, 0.04, 0.01, -0.02])
SHADOWS = dict(point_lights="POINT", shadow_map_size=128, shadow_bias=0.02, shadow_softness=0.05,
               light_shadow_map_size=256, light_shadow_bias=0.02, light_shadow_softness=0.05,
               light_shadow_bounds=(0.0, 0.0, 4.0, 1.6))
KS, E = 0.6, 10.0


def textured_view(V, F, uv, fuv, texture, smap=None, light=LIGHT, ambient=0.2, specular=KS, shininess=E, size=SIZE,
                  **kw):
    if kw.get("point_lights") == "POINT":
        kw["point_lights"] = cuda(POINT)
    if kw.get("sh") == "SH":
        kw["sh"] = cuda(SH)
    return DeviceMeshView(F, V.shape[0], camera(size), size, size, light_directional=light, ambient=ambient,
                          background_color=(0.1, 0.2, 0.3), sigma=1.0, device=DEV, uv=uv, faces_uv=fuv,
                          texture=texture, shading="phong_textured", specular=specular, shininess=shininess,
                          specular_map=smap, **kw)


def test_a_map_of_ones_gives_the_view_without_a_map():
    V, F, uv, fuv, texture = duck()
    ones = np.ones(texture.shape[:2] + (2,))
    kw = dict(SHADOWS, sh="SH")
    plain = textured_view(V, F, uv, fuv, texture, **kw)
    mapped = textured_view(V, F, uv, fuv, texture, ones, **kw)
    # the views share the renderer's slot: each is back-propagated before the other renders
    a = plain.render(cuda(V)).clone()
    g = cuda(np.random.default_rng(1).normal(size=tuple(a.shape)), torch.float32)
    ga = plain.backward(g)
    b = mapped.render(cuda(V))
    gb = mapped.backward(g)
    errs = {"image": float((a - b).abs().max())}
    for k in ("vertices_b", "texture_b", "uv_b", "light_b", "specular_b", "sh_b", "point_lights_b"):
        errs[k] = rel(host(gb[k]), host(ga[k]))
    sb = host(gb["specular_map_b"]).sum(axis=(0, 1))
    spb = host(ga["specular_b"])
    errs["sum_ks_t_b"] = float(abs(sb[0] - KS * spb[0]) / abs(KS * spb[0]))
    errs["sum_e_t_b"] = float(abs(sb[1] - E * spb[1]) / abs(E * spb[1]))
    record("specular_map_ones_duck", errs)
    assert np.abs(host(a) - np.array([0.1, 0.2, 0.3])).max() > 0.1  # the duck is in view
    assert errs["image"] <= 1e-6
    for k in ("vertices_b", "texture_b", "uv_b", "light_b", "specular_b", "sh_b", "point_lights_b"):
        assert errs[k] <= 1e-4, k
    assert errs["sum_ks_t_b"] <= 1e-4 and errs["sum_e_t_b"] <= 1e-4


# ------------------------------------------------------------------------------------ 3. central differences

def _glossy_setup(texels=16):
    V, F, uv, fuv = grid_plane(n=12, texels=texels)
    rng = np.random.default_rng(9)
    texture = rng.uniform(0.4, 1.0, (texels, texels, 3))
    smap = np.stack((rng.uniform(0.5, 1.5, (texels, texels)), rng.uniform(0.6, 1.4, (texels, texels))), axis=2)
    w = rng.uniform(0, 1, (SIZE, SIZE, 3))
    return V, F, uv, fuv, texture, smap, w


def test_gradients_agree_with_central_differences():
    """<image, w> is linear in ks_t, so a large step is exact up to the image's fp32 rounding (h = 0.25); it is smooth
    in e_t (h = 0.02, relative error bound 1e-2 for both, recorded)."""
    V, F, uv, fuv, texture, smap, w = _glossy_setup()
    light = np.array([0.1, 0.05, 1.0])  # from behind the camera: a highlight near the plane's centre
    view = textured_view(V, F, uv, fuv, texture, smap, light=light, specular=0.8, shininess=8.0)
    loss = lambda m: float(np.sum(host(view.render(cuda(V), specular_map=cuda(m, torch.float32))) * w))  # noqa
    loss(smap)
    sb = host(view.backward(cuda(w, torch.float32))["specular_map_b"])
    res = {}
    for k, h in ((0, 0.25), (1, 0.02)):
        an, fd = [], []
        for (i, j) in [(5, 7), (8, 4), (10, 10), (6, 11), (7, 7)]:
            p, m = smap.copy(), smap.copy()
            p[i, j, k] += h
            m[i, j, k] -= h
            fd.append((loss(p) - loss(m)) / (2 * h))
            an.append(sb[i, j, k])
        res["ks_t" if k == 0 else "e_t"] = {"h": h, "analytic": an, "fd": fd, "rel_err": rel(an, fd)}
    record("specular_map_fd", res)
    for k, r in res.items():
        assert np.linalg.norm(r["fd"]) > 0, k
        assert r["rel_err"] <= 1e-2, k


# --------------------------------------------------------------------------------------------------- 4. PyTorch

@pytest.mark.parametrize("case", ["plain", "shadows"])
def test_pytorch_gradients_equal_the_device_view(case):
    V, F, uv, fuv, texture = duck()
    rng = np.random.default_rng(2)
    smap = rng.uniform(0.5, 1.5, texture.shape[:2] + (2,))
    kw = dict(SHADOWS) if case == "shadows" else {}
    view = textured_view(V, F, uv, fuv, texture, smap, **kw)
    dimage = view.render(cuda(V))
    image_b = cuda(rng.normal(size=tuple(dimage.shape)), torch.float32)
    out = view.backward(image_b)
    vertices, uv_t = cuda(V).requires_grad_(True), cuda(uv).requires_grad_(True)
    tex_t, smap_t = cuda(texture).requires_grad_(True), cuda(smap).requires_grad_(True)
    scene = P.Scene3DPytorch(shading="phong_textured")
    scene.set_mesh(P.ColoredTriMeshPytorch(F, vertices, faces_uv=fuv, uv=uv_t, texture=tex_t, specular_map=smap_t,
                                           device=DEV))
    if case == "shadows":
        scene.set_light(cuda(LIGHT), 0.2, shadow_map_size=kw["light_shadow_map_size"],
                        shadow_bias=kw["light_shadow_bias"], shadow_softness=kw["light_shadow_softness"],
                        shadow_bounds=kw["light_shadow_bounds"])
        scene.set_point_lights(cuda(POINT), shadow_map_size=kw["shadow_map_size"], shadow_bias=kw["shadow_bias"],
                               shadow_softness=kw["shadow_softness"])
    else:
        scene.set_light(cuda(LIGHT), 0.2)
    scene.set_specular(KS, E)
    scene.set_background_color((0.1, 0.2, 0.3))
    cam = camera()
    image = scene.render(P.CameraPytorch(cam.extrinsic, cam.intrinsic, SIZE, SIZE, cam.distortion))
    img_err = float((image.detach() - dimage).abs().max())
    (image.double() * image_b.double()).sum().backward()
    errs = {k: rel(host(t.grad), host(out[o])) for k, t, o in (
        ("specular_map", smap_t, "specular_map_b"), ("texture", tex_t, "texture_b"), ("uv", uv_t, "uv_b"),
        ("vertices", vertices, "vertices_b"))}
    errs["image"] = img_err
    record(f"specular_map_pytorch_vs_view_{case}", errs)
    assert img_err <= 1e-6
    for k in ("specular_map", "texture", "uv", "vertices"):
        assert errs[k] <= 1e-6, k


def test_views_refuse_a_map_they_cannot_use():
    V, F, uv, fuv = grid_plane()
    tex, smap = np.ones((32, 32, 3)), np.ones((32, 32, 2))
    with pytest.raises(ValueError, match="phong_textured"):
        DeviceMeshView(F, V.shape[0], camera(), 32, 32, device=DEV, uv=uv, faces_uv=fuv, texture=tex,
                       specular_map=smap)
    with pytest.raises(ValueError, match="phong_textured"):
        DeviceMeshView(F, V.shape[0], camera(), 32, 32, device=DEV, shading="phong", specular_map=smap)
    with pytest.raises(ValueError, match="Ht and Wt"):
        textured_view(V, F, uv, fuv, tex, np.ones((32, 32, 3)))
    with pytest.raises(ValueError, match="Ht and Wt"):
        textured_view(V, F, uv, fuv, tex, np.ones((16, 32, 2)))
    view = textured_view(V, F, uv, fuv, tex)
    with pytest.raises(ValueError, match="no specular map"):
        view.render(cuda(V), specular_map=cuda(smap, torch.float32))
    mapped = textured_view(V, F, uv, fuv, tex, smap)
    with pytest.raises(ValueError, match="expected"):
        mapped.render(cuda(V), specular_map=cuda(np.ones((16, 16, 2)), torch.float32))
    with pytest.raises(ValueError, match="textured mesh"):
        P.ColoredTriMeshPytorch(F, cuda(V), device=DEV, specular_map=smap)
    with pytest.raises(ValueError, match="Ht and Wt"):
        P.ColoredTriMeshPytorch(F, cuda(V), device=DEV, faces_uv=fuv, uv=uv, texture=tex, specular_map=np.ones((4, 4, 2)))
    with pytest.raises(ValueError, match="separate albedo"):
        g = cuda(np.zeros((4, 4, 10)), torch.float32)
        mesh_ops.phong_shade(g, cuda(np.zeros(6)), cuda(np.zeros(3)), cuda(np.zeros(3)),
                             specular=cuda(np.zeros((4, 4, 2)), torch.float32))


def test_render_and_backward_make_no_host_sync():
    V, F, uv, fuv, texture, smap, w = _glossy_setup()
    view = textured_view(V, F, uv, fuv, texture, smap, **dict(SHADOWS, sh="SH"))
    Vd, sd, wd = cuda(V), cuda(smap, torch.float32), cuda(w, torch.float32)
    view.render(Vd, specular_map=sd)
    view.backward(wd)
    smap_t = cuda(smap).requires_grad_(True)
    scene = P.Scene3DPytorch(shading="phong_textured")
    scene.set_mesh(P.ColoredTriMeshPytorch(F, cuda(V).requires_grad_(True), faces_uv=fuv, uv=cuda(uv),
                                           texture=cuda(texture), specular_map=smap_t, device=DEV))
    scene.set_light(cuda(LIGHT), 0.2)
    scene.set_point_lights(cuda(POINT))
    scene.set_specular(KS, E)  # on the device: a host number would be uploaded at every render
    scene.set_background_color((0.1, 0.2, 0.3))
    cam = camera()
    cam = P.CameraPytorch(cam.extrinsic, cam.intrinsic, SIZE, SIZE, cam.distortion)
    scene.render(cam).sum().backward()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        view.render(Vd, specular_map=sd)
        view.backward(wd)
        scene.render(cam).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert smap_t.grad is not None and float(smap_t.grad.abs().max()) > 0


# ------------------------------------------------------------------------------------------------------ 5. a fit

FIT_STEPS = 1000


def test_adam_recovers_a_glossy_and_a_matte_region():
    """A plane whose map is glossy (ks_t, e_t) = (1, 1) for u < half the texture and matte (0.15, 0.4) beyond, the
    albedo known, rendered under four directional lights from near the camera (each puts its highlight elsewhere on
    the plane); the fit starts from the uniform map (0.5, 0.6) and steps the map's logarithm, so that the glossy and
    the matte texels move by the same relative steps.  A texel carries a highlight when its ks_t moves the image by a
    quarter of the most any texel does, in at least one render."""
    texels = 32
    V, F, uv, fuv = grid_plane(n=16, texels=texels)
    cols = np.arange(texels)[None, :].repeat(texels, 0)  # texture columns: u
    glossy = cols < texels // 2
    target = np.stack((np.where(glossy, 1.0, 0.15), np.where(glossy, 1.0, 0.4)), axis=-1)
    albedo = np.tile([0.5, 0.45, 0.4], (texels, texels, 1))
    lights = [np.array([sx * 0.2, sy * 0.2, 1.0]) for sx in (-1, 1) for sy in (-1, 1)]
    views = [textured_view(V, F, uv, fuv, albedo, target, light=l, ambient=0.1, specular=0.8, shininess=20.0)
             for l in lights]
    Vd = cuda(V)
    targets = [v.render(Vd, specular_map=cuda(target, torch.float32)).clone() for v in views]
    # the texels that carry a highlight in at least one render: those whose ks_t moves the image
    reach = np.zeros((texels, texels))
    for v in views:
        v.render(Vd, specular_map=cuda(target, torch.float32))
        reach = np.maximum(reach, host(v.backward(torch.ones_like(targets[0]))["specular_map_b"])[..., 0])
    lit = reach > 0.25 * reach.max()
    param = cuda(np.log(np.tile([0.5, 0.6], (texels, texels, 1))), torch.float32).requires_grad_(True)
    opt = torch.optim.Adam([param], lr=0.05)
    # the step decays to 1/30 of its start, so that Adam's last steps stay well inside the error bounds
    decay = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=(1 / 30) ** (1 / FIT_STEPS))

    def errors():
        m = np.exp(host(param))
        ks_err = np.abs(m[..., 0] - target[..., 0]) / target[..., 0]
        e_err = np.abs(m[..., 1] - target[..., 1]) / target[..., 1]
        return float(np.median(ks_err[lit])), float(np.median(e_err[lit & glossy]))

    start = errors()
    for _ in range(FIT_STEPS):
        opt.zero_grad()
        grad = torch.zeros_like(param)
        smap = param.detach().exp()
        for v, t in zip(views, targets):
            image = v.render(Vd, specular_map=smap)
            grad += v.backward(2 * (image - t))["specular_map_b"]
        param.grad = grad * smap
        opt.step()
        decay.step()
    end = errors()
    record("specular_map_fit", {"steps": FIT_STEPS, "lit_texels": int(lit.sum()),
                                "glossy_lit_texels": int((lit & glossy).sum()),
                                "median_ks_rel_err_start": start[0], "median_ks_rel_err_end": end[0],
                                "median_e_rel_err_glossy_start": start[1], "median_e_rel_err_glossy_end": end[1]})
    assert (lit & glossy).sum() >= 20 and (lit & ~glossy).sum() >= 20
    assert end[0] <= 0.05 and end[1] <= 0.10
