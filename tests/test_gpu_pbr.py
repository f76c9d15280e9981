"""GPU: metallic-roughness (GGX) materials in textured views - the shading kernels against the fp64 restatement
(tests/pbr_ref.py), a closed form on a camera-facing plane, a map of ones against the factors alone on the duck under an
environment, shadows and a normal map, gradients against central differences, the refusals, no host synchronisation,
the PyTorch path against the device view, and a fit of a two-material map."""
import json
import os

import numpy as np
import pytest
import pbr_ref as ref

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
    "plain_map": dict(mapped=True),
    "sh1_grey_point": dict(sh="grey", lights="grey"),
    "sh1_grey_point_map": dict(sh="grey", lights="grey", mapped=True),
    "sh3_colour_points": dict(sh="colour", lights="colour", mapped=True),
    "grey_points_vis": dict(lights="grey", vis=True),
    "colour_points_vis_map": dict(lights="colour", vis=True, mapped=True),
    "sun": dict(sun=True),
    "sun_map": dict(sun=True, mapped=True),
    "sh3_colour_points_vis_sun_map": dict(sh="colour", lights="colour", vis=True, sun=True, mapped=True),
    "sh1_grey_points_vis_sun": dict(sh="grey", lights="grey", vis=True, sun=True),
    "c4_colour_points_map": dict(C=4, sh="colour", lights="colour", mapped=True),
    "c2_sh_grey_points": dict(C=2, sh="colour", lights="grey", mapped=True),
    "c5_grey": dict(C=5, sh="grey", lights="grey", mapped=True),
}
CAM = np.array([0.0, 0.1, -5.0])


def _pixels(rng, H=17, W=23, C=3, L=2, sh=None, lights=None, vis=False, sun=False, mapped=False):
    P_ = H * W
    G, A, mr = ref.random_pixels(rng, C, P_, CAM)
    G[0::13] = 0.0  # a = 0 (the albedo and map rasters are 0 there too)
    A[0::13] = 0.0
    mr[0::13] = 0.0
    G[3::13, 0:3] = np.array([0.0, 0.0, 5.0]) * G[3::13, 6:7]  # facing away from every light: nl <= 0
    G[5::13, 0:3] = np.array([1.0, 0.0, 0.0]) * G[5::13, 6:7]  # nv = 0: x on the camera's y-z plane
    G[5::13, 3] = 0.0
    G, A, mr = f32(G), f32(A), f32(mr)
    shv = {None: None, "grey": rng.normal(size=9) * 0.2, "colour": rng.normal(size=(9, C)) * 0.2}[sh]
    S = {None: 0, "grey": 1, "colour": C}[lights]
    table = None
    if lights:
        table = np.concatenate((CAM + rng.uniform(-2, 2, (L, 3)), rng.uniform(0.5, 2.0, (L, S))), axis=1)
    V = f32(rng.uniform(0, 1, (P_, L))) if vis else None
    sv = f32(rng.uniform(0, 1, P_)) if sun else None
    return dict(G=G, A=A, mr=mr if mapped else None, sh=shv, lights=table, vis=V, sun_vis=sv), (H, W, C, L)


def _device_run(kw, params, cam, bg, g, H, W, C, L):
    dev = dict(albedo=cuda(kw["A"].reshape(H, W, C), torch.float32),
               specular=cuda(kw["mr"].reshape(H, W, 2), torch.float32) if kw["mr"] is not None else None,
               sh=cuda(kw["sh"]) if kw["sh"] is not None else None,
               point_lights=cuda(kw["lights"]) if kw["lights"] is not None else None,
               visibility=cuda(kw["vis"].reshape(H, W, L), torch.float32) if kw["vis"] is not None else None,
               sun_visibility=cuda(kw["sun_vis"].reshape(H, W), torch.float32) if kw["sun_vis"] is not None else None,
               brdf="ggx")
    ch, pd, cd, bd = cuda(kw["G"].reshape(H, W, 7), torch.float32), cuda(params), cuda(cam), cuda(bg, torch.float32)
    image = host(mesh_ops.phong_shade(ch, pd, cd, bd, **dev))
    out = list(mesh_ops.phong_shade_backward(ch, pd, cd, bd, cuda(g.reshape(H, W, C), torch.float32),
                                             new_scratch(DEV), center_grad=True, **dev))
    res = {"image": image.reshape(-1, C)}
    res["mr_b"] = host(out.pop()).reshape(-1, 2) if kw["mr"] is not None else None
    res["sun_vis_b"] = host(out.pop()).reshape(-1) if kw["sun_vis"] is not None else None
    res["vis_b"] = host(out.pop()).reshape(-1, L) if kw["vis"] is not None else None
    res["lights_b"] = host(out.pop()) if kw["lights"] is not None else None
    res["A_b"] = host(out.pop()).reshape(-1, C)
    res["sh_b"] = host(out.pop()) if kw["sh"] is not None else None
    channels_b, params_b, center_b = (host(t) for t in out)
    res.update(G_b=channels_b.reshape(-1, 7), params_b=params_b, cam_b=center_b)
    return res


@pytest.mark.parametrize("case", list(KERNEL_CASES))
def test_the_kernels_match_the_restatement(case):
    rng = np.random.default_rng(11)
    kw, (H, W, C, L) = _pixels(rng, **KERNEL_CASES[case])
    params = np.array([0.3, 0.5, 0.8, 0.4, 0.7, 0.6])  # l, ambient, mf, rf
    bg = f32([0.2, 0.3, 0.4, 0.5, 0.6][:C])
    g = f32(rng.normal(size=(H * W, C)))
    want = ref.shade(kw["G"], kw["A"], kw["mr"], params, CAM, bg, kw["sh"], kw["lights"], kw["vis"], kw["sun_vis"])
    grads = ref.shade_b(g, kw["G"], kw["A"], kw["mr"], params, CAM, bg, kw["sh"], kw["lights"], kw["vis"],
                        kw["sun_vis"])
    got = _device_run(kw, params, CAM, bg, g, H, W, C, L)
    again = _device_run(kw, params, CAM, bg, g, H, W, C, L)
    for k, v in got.items():
        assert v is None or np.array_equal(v, again[k]), f"two runs differ in {k}"
    # the image is fp32: held to 1e-6 of its largest entry, like the per-pixel gradients
    errs = {"image": rel(got["image"], want), "image_abs": float(np.abs(got["image"] - want).max())}
    for k in ("A_b", "G_b", "mr_b", "vis_b", "sun_vis_b", "params_b", "cam_b", "lights_b", "sh_b"):
        if got[k] is not None:
            errs[k] = rel(got[k], grads[k])
    record(f"pbr_kernels_{case}", errs)
    assert errs["image"] <= 1e-6
    for k in ("A_b", "G_b", "mr_b", "vis_b", "sun_vis_b"):
        assert errs.get(k, 0.0) <= 1e-6, k
    for k in ("params_b", "cam_b", "lights_b", "sh_b"):
        assert errs.get(k, 0.0) <= 1e-12, k
    if got["mr_b"] is not None:
        assert not np.any(got["mr_b"][0::13])  # 0 where a = 0


# ------------------------------------------------------------------------------------------- 2. a closed form

def _plane_view(texture, mr=None, light=(0.0, 0.0, 2.0), size=SIZE, metallic=0.3, roughness=0.5, ambient=0.25,
                n=16, **kw):
    texels = texture.shape[0]
    V, F, uv, fuv = grid_plane(n=n, texels=texels)
    view = DeviceMeshView(F, V.shape[0], camera(size), size, size, light_directional=np.asarray(light),
                          ambient=ambient, background_color=(0.1, 0.2, 0.3), sigma=1.0, device=DEV, uv=uv,
                          faces_uv=fuv, texture=texture, shading="pbr_textured", metallic=metallic,
                          roughness=roughness, metallic_roughness_map=mr, **kw)
    return view, V


def test_a_camera_facing_plane_lit_along_the_axis_matches_the_closed_form():
    """At the on-axis pixel n = v = w, so nl = nv = nh = vh = 1: F = F0, S = 1 / (4 alpha^2)."""
    size = 65  # an odd size: pixel (32, 32) is on the optical axis
    b = np.array([0.6, 0.4, 0.2])
    m, r, ll, amb = 0.3, 0.5, 2.0, 0.25
    view, V = _plane_view(np.tile(b, (8, 8, 1)), size=size, metallic=m, roughness=r, light=(0.0, 0.0, ll),
                          ambient=amb)
    got = host(view.render(cuda(V)))[32, 32]
    F0 = 0.04 * (1 - m) + m * b
    alpha2 = r ** 4
    want = ll * ((1 - F0) * (1 - m) * b + F0 / (4 * alpha2)) + (1 - m) * b * amb
    record("pbr_closed_form", {"got": got.tolist(), "want": want.tolist(), "err": float(np.abs(got - want).max())})
    assert np.abs(got - want).max() <= 1e-6


# ----------------------------------------------------------------------------------------- 3. a map of ones

LIGHT = np.array([0.3, -0.4, 0.8])
POINT = np.array([[1.5, -1.0, 2.0, 4.0]])
SH = np.array([0.5, 0.1, -0.2, 0.05, 0.02, -0.03, 0.04, 0.01, -0.02])
SHADOWS = dict(shadow_map_size=128, shadow_bias=0.02, shadow_softness=0.05, light_shadow_map_size=256,
               light_shadow_bias=0.02, light_shadow_softness=0.05, light_shadow_bounds=(0.0, 0.0, 4.0, 1.6))
MF, RF = 0.4, 0.45


def duck_view(mr=None, **kw):
    V, F, uv, fuv, texture = duck()
    nmap = np.random.default_rng(5).normal(size=texture.shape[:2] + (3,)) * 0.1 + np.array([0.0, 0.0, 1.0])
    view = DeviceMeshView(F, V.shape[0], camera(), SIZE, SIZE, light_directional=LIGHT, ambient=0.2,
                          background_color=(0.1, 0.2, 0.3), sigma=1.0, device=DEV, uv=uv, faces_uv=fuv,
                          texture=texture, shading="pbr_textured", metallic=MF, roughness=RF,
                          metallic_roughness_map=mr, sh=cuda(SH), point_lights=cuda(POINT), normal_map=nmap,
                          **dict(SHADOWS, **kw))
    return view, V, texture


def test_a_map_of_ones_gives_the_factors_alone():
    texture = duck()[4]
    plain, V, _ = duck_view()
    mapped, _, _ = duck_view(np.ones(texture.shape[:2] + (2,)))
    # the views share the renderer's slot: each is back-propagated before the other renders
    a = plain.render(cuda(V)).clone()
    g = cuda(np.random.default_rng(1).normal(size=tuple(a.shape)), torch.float32)
    ga = plain.backward(g)
    b = mapped.render(cuda(V))
    gb = mapped.backward(g)
    errs = {"image": float((a - b).abs().max()), "image_bitwise": bool(torch.equal(a, b))}
    keys = ("vertices_b", "texture_b", "uv_b", "light_b", "material_b", "sh_b", "point_lights_b", "normal_map_b")
    for k in keys:
        errs[k] = rel(host(gb[k]), host(ga[k]))
    sb = host(gb["metallic_roughness_map_b"]).sum(axis=(0, 1))
    mb = host(ga["material_b"])  # (metallic_b, roughness_b)
    errs["sum_roughness_t_b"] = float(abs(sb[0] - RF * mb[1]) / abs(RF * mb[1]))
    errs["sum_metallic_t_b"] = float(abs(sb[1] - MF * mb[0]) / abs(MF * mb[0]))
    record("pbr_ones_duck", errs)
    assert np.abs(host(a) - np.array([0.1, 0.2, 0.3])).max() > 0.1  # the duck is in view
    assert errs["image_bitwise"]
    # vertices_b and uv_b are fp32 sums that the rasteriser's adjoint forms with atomics, in an order that varies from
    # run to run, and the mapped view adds a fourth raster's terms to them: they agree to about one fp32 ulp
    for k in keys:
        assert errs[k] <= 1e-6, k
    assert errs["sum_roughness_t_b"] <= 1e-7 and errs["sum_metallic_t_b"] <= 1e-7


# ------------------------------------------------------------------------------------ 4. central differences

def test_gradients_agree_with_central_differences():
    texels = 16
    rng = np.random.default_rng(9)
    texture = rng.uniform(0.4, 1.0, (texels, texels, 3))
    mr = np.stack((rng.uniform(0.4, 0.8, (texels, texels)), rng.uniform(0.2, 0.8, (texels, texels))), axis=2)
    view, V = _plane_view(texture, mr, light=np.array([0.1, 0.05, 1.0]), n=12, point_lights=cuda(POINT))
    w = rng.uniform(0, 1, (SIZE, SIZE, 3))

    def loss(m=mr, tex=texture, verts=V):
        return float(np.sum(host(view.render(cuda(verts), texture=cuda(tex, torch.float32),
                                             metallic_roughness_map=cuda(m, torch.float32))) * w))

    loss()
    grads = view.backward(cuda(w, torch.float32))
    mb, tb = host(grads["metallic_roughness_map_b"]), host(grads["texture_b"])
    matb, vb = host(grads["material_b"]), host(grads["vertices_b"])
    res = {}
    for k, name, h in ((0, "roughness_t", 0.01), (1, "metallic_t", 0.05)):
        an, fd = [], []
        for (i, j) in [(5, 7), (8, 4), (10, 10), (6, 11), (7, 7)]:
            p, m = mr.copy(), mr.copy()
            p[i, j, k] += h
            m[i, j, k] -= h
            fd.append((loss(m=p) - loss(m=m)) / (2 * h))
            an.append(mb[i, j, k])
        res[name] = {"h": h, "analytic": an, "fd": fd, "rel_err": rel(an, fd)}
    for k, name, attr, h in ((0, "mf", "metallic", 0.01), (1, "rf", "roughness", 0.005)):
        x0 = getattr(view, attr)
        setattr(view, attr, x0 + h)
        lp = loss()
        setattr(view, attr, x0 - h)
        lm = loss()
        setattr(view, attr, x0)
        fd = (lp - lm) / (2 * h)
        res[name] = {"h": h, "analytic": float(matb[k]), "fd": fd, "rel_err": rel([matb[k]], [fd])}
    an, fd = [], []
    for (i, j, c) in [(5, 7, 0), (8, 4, 1), (10, 10, 2)]:
        p, m = texture.copy(), texture.copy()
        p[i, j, c] += 0.05
        m[i, j, c] -= 0.05
        fd.append((loss(tex=p) - loss(tex=m)) / 0.1)
        an.append(tb[i, j, c])
    res["texture"] = {"h": 0.05, "analytic": an, "fd": fd, "rel_err": rel(an, fd)}
    an, fd = [], []
    for axis in range(3):
        step = np.zeros(3)
        step[axis] = 1e-3
        fd.append((loss(verts=V + step) - loss(verts=V - step)) / 2e-3)
        an.append(float(vb[:, axis].sum()))
    res["vertices_translation"] = {"h": 1e-3, "analytic": an, "fd": fd, "rel_err": rel(an, fd)}
    record("pbr_fd", res)
    for k, r in res.items():
        assert np.linalg.norm(r["fd"]) > 0, k
        assert r["rel_err"] <= 1e-3, k


# --------------------------------------------------------------------------------------------------- 5. PyTorch

def _pytorch_scene(F, vertices, uv, fuv, texture, mr, shadows, metallic, roughness):
    scene = P.Scene3DPytorch(shading="pbr_textured")
    scene.set_mesh(P.ColoredTriMeshPytorch(F, vertices, faces_uv=fuv, uv=uv, texture=texture,
                                           metallic_roughness_map=mr, device=DEV))
    if shadows:
        scene.set_light(cuda(LIGHT), 0.2, shadow_map_size=SHADOWS["light_shadow_map_size"],
                        shadow_bias=SHADOWS["light_shadow_bias"], shadow_softness=SHADOWS["light_shadow_softness"],
                        shadow_bounds=SHADOWS["light_shadow_bounds"])
        scene.set_point_lights(cuda(POINT), shadow_map_size=SHADOWS["shadow_map_size"],
                               shadow_bias=SHADOWS["shadow_bias"], shadow_softness=SHADOWS["shadow_softness"])
    else:
        scene.set_light(cuda(LIGHT), 0.2)
        scene.set_point_lights(cuda(POINT))
    scene.set_material(metallic, roughness)
    scene.set_background_color((0.1, 0.2, 0.3))
    return scene


@pytest.mark.parametrize("case", ["plain", "shadows"])
def test_pytorch_gradients_equal_the_device_view(case):
    V, F, uv, fuv, texture = duck()
    rng = np.random.default_rng(2)
    mr = np.stack((rng.uniform(0.4, 1.0, texture.shape[:2]), rng.uniform(0.2, 1.0, texture.shape[:2])), axis=2)
    kw = dict(SHADOWS) if case == "shadows" else {}
    view = DeviceMeshView(F, V.shape[0], camera(), SIZE, SIZE, light_directional=LIGHT, ambient=0.2,
                          background_color=(0.1, 0.2, 0.3), sigma=1.0, device=DEV, uv=uv, faces_uv=fuv,
                          texture=texture, shading="pbr_textured", metallic=MF, roughness=RF,
                          metallic_roughness_map=mr, point_lights=cuda(POINT), **kw)
    dimage = view.render(cuda(V))
    image_b = cuda(rng.normal(size=tuple(dimage.shape)), torch.float32)
    out = view.backward(image_b)
    vertices, uv_t = cuda(V).requires_grad_(True), cuda(uv).requires_grad_(True)
    tex_t, mr_t = cuda(texture).requires_grad_(True), cuda(mr).requires_grad_(True)
    mf_t, rf_t = cuda(np.array(MF)).requires_grad_(True), cuda(np.array(RF)).requires_grad_(True)
    scene = _pytorch_scene(F, vertices, uv_t, fuv, tex_t, mr_t, case == "shadows", mf_t, rf_t)
    cam = camera()
    image = scene.render(P.CameraPytorch(cam.extrinsic, cam.intrinsic, SIZE, SIZE, cam.distortion))
    img_err = float((image.detach() - dimage).abs().max())
    (image.double() * image_b.double()).sum().backward()
    errs = {k: rel(host(t.grad), host(out[o])) for k, t, o in (
        ("metallic_roughness_map", mr_t, "metallic_roughness_map_b"), ("texture", tex_t, "texture_b"),
        ("uv", uv_t, "uv_b"), ("vertices", vertices, "vertices_b"))}
    errs["factors"] = rel([float(mf_t.grad), float(rf_t.grad)], host(out["material_b"]))
    errs["image"] = img_err
    record(f"pbr_pytorch_vs_view_{case}", errs)
    assert img_err <= 1e-6
    for k in ("metallic_roughness_map", "factors", "texture", "uv", "vertices"):
        assert errs[k] <= 1e-6, k


def test_pytorch_refuses_what_it_cannot_use():
    V, F, uv, fuv = grid_plane()
    tex, mr = np.ones((32, 32, 3)), np.ones((32, 32, 2))
    with pytest.raises(ValueError, match="textured mesh"):
        P.ColoredTriMeshPytorch(F, cuda(V), device=DEV, metallic_roughness_map=mr)
    with pytest.raises(ValueError, match="Ht and Wt"):
        P.ColoredTriMeshPytorch(F, cuda(V), device=DEV, faces_uv=fuv, uv=uv, texture=tex,
                                metallic_roughness_map=np.ones((4, 4, 2)))
    with pytest.raises(ValueError, match="not both"):
        P.ColoredTriMeshPytorch(F, cuda(V), device=DEV, faces_uv=fuv, uv=uv, texture=tex, specular_map=mr,
                                metallic_roughness_map=mr)
    with pytest.raises(ValueError, match="set_specular"):
        P.Scene3DPytorch(shading="phong_textured").set_material(0.5, 0.5)
    with pytest.raises(ValueError, match="set_material"):
        P.Scene3DPytorch(shading="pbr_textured").set_specular(0.5, 8.0)
    cam = camera(32)
    cam = P.CameraPytorch(cam.extrinsic, cam.intrinsic, 32, 32, cam.distortion)
    for shading, mesh_kw in (("phong_textured", dict(metallic_roughness_map=mr)),
                             ("pbr_textured", dict(specular_map=mr))):
        scene = P.Scene3DPytorch(shading=shading)
        scene.set_mesh(P.ColoredTriMeshPytorch(F, cuda(V), device=DEV, faces_uv=fuv, uv=uv, texture=tex, **mesh_kw))
        scene.set_light(cuda(LIGHT), 0.2)
        scene.set_background_color((0.1, 0.2, 0.3))
        with pytest.raises(ValueError, match="pbr_textured"):
            scene.render(cam)


# --------------------------------------------------------------------------------------------- 6. refusals

def test_views_refuse_what_they_cannot_use():
    V, F, uv, fuv = grid_plane()
    tex, mr = np.ones((32, 32, 3)), np.ones((32, 32, 2))
    base = dict(device=DEV, uv=uv, faces_uv=fuv, texture=tex)
    for bad in (dict(specular_map=mr), dict(specular=0.5), dict(shininess=8.0)):
        with pytest.raises(ValueError, match="pbr_textured"):
            DeviceMeshView(F, V.shape[0], camera(), 32, 32, shading="pbr_textured", **base, **bad)
    for shading in ("gouraud", "phong_textured"):
        with pytest.raises(ValueError, match="pbr_textured"):
            DeviceMeshView(F, V.shape[0], camera(), 32, 32, shading=shading, metallic_roughness_map=mr, **base)
    with pytest.raises(ValueError, match="Ht and Wt"):
        DeviceMeshView(F, V.shape[0], camera(), 32, 32, shading="pbr_textured", metallic_roughness_map=np.ones(
            (16, 32, 2)), **base)
    with pytest.raises(ValueError, match="perspective_correct"):
        DeviceMeshView(F, V.shape[0], camera(), 32, 32, shading="pbr_textured", perspective_correct=True, **base)
    with pytest.raises(ValueError, match="textured view"):
        DeviceMeshView(F, V.shape[0], camera(), 32, 32, shading="pbr_textured", device=DEV)
    view, _ = _plane_view(tex)
    with pytest.raises(ValueError, match="no metallic-roughness map"):
        view.render(cuda(V), metallic_roughness_map=cuda(mr, torch.float32))
    mapped, _ = _plane_view(tex, mr)
    with pytest.raises(ValueError, match="expected"):
        mapped.render(cuda(V), metallic_roughness_map=cuda(np.ones((16, 16, 2)), torch.float32))
    with pytest.raises(ValueError, match="separate albedo"):
        g = cuda(np.zeros((4, 4, 10)), torch.float32)
        mesh_ops.phong_shade(g, cuda(np.zeros(6)), cuda(np.zeros(3)), cuda(np.zeros(3)), brdf="ggx")


def test_render_and_backward_make_no_host_sync():
    view, V, texture = duck_view(np.full(duck()[4].shape[:2] + (2,), 0.7))
    Vd = cuda(V)
    md = cuda(np.full(texture.shape[:2] + (2,), 0.6), torch.float32)
    w = cuda(np.random.default_rng(3).normal(size=(SIZE, SIZE, 3)), torch.float32)
    view.render(Vd, metallic_roughness_map=md)
    view.backward(w)
    V_, F, uv, fuv, _ = duck()
    scene = _pytorch_scene(F, cuda(V_).requires_grad_(True), cuda(uv), fuv, cuda(texture),
                           cuda(np.full(texture.shape[:2] + (2,), 0.6)).requires_grad_(True), True,
                           cuda(np.array(MF)), cuda(np.array(RF)))  # on the device: no upload at every render
    cam = camera()
    cam = P.CameraPytorch(cam.extrinsic, cam.intrinsic, SIZE, SIZE, cam.distortion)
    scene.render(cam).sum().backward()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        view.render(Vd, metallic_roughness_map=md)
        view.backward(w)
        scene.render(cam).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")


# -------------------------------------------------------------------------------------------------- 7. a fit

def test_a_fit_recovers_a_two_material_map():
    """A 32x32 map on a plane of known albedo: a rough dielectric half (0.8, 0) and a polished metal half (0.3, 1),
    rendered under four directional lights and one point light.  Adam on the map through a sigmoid from (0.5, 0.5);
    the error is taken over the texels that carry a highlight in at least one render."""
    texels = 32
    albedo = np.tile(np.array([0.7, 0.5, 0.3]), (texels, texels, 1))
    truth = np.zeros((texels, texels, 2))
    truth[:, : texels // 2] = (0.8, 0.0)
    truth[:, texels // 2:] = (0.3, 1.0)
    lights = [np.array(d) for d in ([0.2, 0.2, 1.0], [-0.3, 0.1, 1.0], [0.1, -0.35, 1.0], [-0.15, -0.2, 1.0])]
    views = []
    for d in lights:
        views.append(_plane_view(albedo, truth, light=2.0 * d / np.linalg.norm(d), metallic=1.0, roughness=1.0,
                                 ambient=0.3)[0])
    V = _plane_view(albedo, truth, light=(0.0, 0.0, 0.0), metallic=1.0, roughness=1.0, ambient=0.3,
                    point_lights=cuda(np.array([[0.3, -0.2, 2.5, 8.0]])))[1]
    views.append(_plane_view(albedo, truth, light=(0.0, 0.0, 0.0), metallic=1.0, roughness=1.0, ambient=0.3,
                             point_lights=cuda(np.array([[0.3, -0.2, 2.5, 8.0]])))[0])
    Vd = cuda(V)
    truth_d = cuda(truth, torch.float32)
    targets, highlight = [], np.zeros((texels, texels), bool)
    for view in views:
        targets.append(view.render(Vd, metallic_roughness_map=truth_d).clone())
        # a texel carries a highlight where the image's roughness gradient is not negligible
        rb = np.abs(host(view.backward(torch.ones_like(targets[-1]))["metallic_roughness_map_b"])[..., 0])
        highlight |= rb > 0.02 * rb.max()
    theta = torch.zeros((texels, texels, 2), dtype=torch.float64, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([theta], lr=0.05)
    for _ in range(400):
        opt.zero_grad()
        m = torch.sigmoid(theta)
        grad = torch.zeros_like(theta)
        for view, target in zip(views, targets):
            image = view.render(Vd, metallic_roughness_map=m.detach().float())
            grad += view.backward(2.0 * (image - target))["metallic_roughness_map_b"].double()
        theta.grad = grad * m.detach() * (1 - m.detach())
        opt.step()
    fitted = host(torch.sigmoid(theta))
    err = np.abs(fitted - truth)[highlight]
    res = {"texels": int(highlight.sum()), "median_abs_err_roughness": float(np.median(err[:, 0])),
           "median_abs_err_metallic": float(np.median(err[:, 1]))}
    record("pbr_fit", res)
    assert res["texels"] > 0.25 * texels * texels
    assert res["median_abs_err_roughness"] < 0.02
    assert res["median_abs_err_metallic"] < 0.05
