"""GPU: tangent-space normal maps in textured Phong views - the tangent kernels and the per-pixel perturbation against
the fp64 restatement (tests/normal_map_ref.py), a flat map against the view without a map under every lighting, an
analytic plane pinning the u / v convention, gradients against central differences, the PyTorch path against the
device view, the refusals, no host synchronisation, and a fit of a bump map."""
import json

import normal_map_ref as ref
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from deodr_b200 import mesh_ops  # noqa: E402
from deodr_b200.mesh_ops import CameraParams, DeviceMeshView, MeshTopology, VertexTangents  # noqa: E402
from deodr_b200.pytorch import scene3d_pytorch as P  # noqa: E402

DEV = "cuda:0"
GOLDEN = __import__("os").path.join(__import__("os").path.dirname(__file__), "golden")


def host(t):
    return t.detach().cpu().numpy().astype(np.float64)


def cuda(a, dtype=torch.float64):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def record(name, value):
    print(json.dumps({"measured": name, "value": value}))


def rel(got, want):
    return float(np.abs(np.asarray(got) - np.asarray(want)).max() / max(np.abs(np.asarray(want)).max(), 1e-300))


# ------------------------------------------------------------------------------------------------------ meshes

def torus(nu=48, nv=24, R=1.0, r=0.4, center=(0.0, 0.0, 4.0), tilt=1.0, texels=64):
    """A torus whose position vertices are shared across the uv seam and whose uv vertices are split there: uv
    [(nu+1)(nv+1), 2] in texel units, faces outward (faces_uv turned with them)."""
    a = 2 * np.pi * np.arange(nu) / nu
    b = 2 * np.pi * np.arange(nv) / nv
    aa, bb = np.meshgrid(a, b, indexing="ij")
    p = np.stack(((R + r * np.cos(bb)) * np.cos(aa), (R + r * np.cos(bb)) * np.sin(aa), r * np.sin(bb)), -1)
    c, s = np.cos(tilt), np.sin(tilt)
    p = p.reshape(-1, 3) @ np.array([[1, 0, 0], [0, c, -s], [0, s, c]]).T + np.asarray(center)
    i, j = np.meshgrid(np.arange(nu), np.arange(nv), indexing="ij")
    i, j = i.ravel(), j.ravel()
    pid = lambda i, j: (i % nu) * nv + (j % nv)  # noqa: E731
    uid = lambda i, j: i * (nv + 1) + j  # noqa: E731
    faces = np.concatenate((np.stack((pid(i, j), pid(i + 1, j), pid(i + 1, j + 1)), 1),
                            np.stack((pid(i, j), pid(i + 1, j + 1), pid(i, j + 1)), 1)))
    faces_uv = np.concatenate((np.stack((uid(i, j), uid(i + 1, j), uid(i + 1, j + 1)), 1),
                               np.stack((uid(i, j), uid(i + 1, j + 1), uid(i, j + 1)), 1)))
    ui, vj = np.meshgrid(np.arange(nu + 1), np.arange(nv + 1), indexing="ij")
    uv = np.stack((ui.ravel() / nu, vj.ravel() / nv), 1) * (texels - 1)
    # outward: the face normal against the direction from the tube's centre line
    tri = p[faces]
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    ring_a = 2 * np.pi * (i + 0.5) / nu
    ring = np.stack((R * np.cos(ring_a), R * np.sin(ring_a), np.zeros_like(ring_a)), 1)
    ring = np.concatenate((ring, ring)) @ np.array([[1, 0, 0], [0, c, -s], [0, s, c]]).T + np.asarray(center)
    flip = np.sum(n * (tri.mean(axis=1) - ring), axis=1) < 0
    faces[flip], faces_uv[flip] = faces[flip][:, ::-1], faces_uv[flip][:, ::-1]
    return p, faces.astype(np.int64), uv, faces_uv.astype(np.int64)


def duck():
    d = np.load(f"{GOLDEN}/duck_textured.npz")
    return d["vertices"], d["faces"].astype(np.int64), d["uv"], d["faces_uv"].astype(np.int64)


def grid_plane(z=4.0, half=1.0, n=16, texels=32):
    """The square |x|, |y| <= half at depth z, facing -z (the camera), with uv = ((x, y) + half) scaled to cover the
    texture: u along +x, v along +y."""
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


SIZE, FOCAL = 128, 120.0


def camera(size=SIZE, focal=FOCAL):
    return CameraParams(np.eye(3, 4), np.array([[focal, 0, (size - 1) / 2], [0, focal, (size - 1) / 2], [0, 0, 1]]))


# ------------------------------------------------------------------------------------- 1. tangent kernels

@pytest.mark.parametrize("mesh", ["duck", "torus"])
def test_tangent_kernels_match_the_restatement(mesh):
    V, F, uv, fuv = duck() if mesh == "duck" else torus()
    topo = MeshTopology(F, V.shape[0], device=DEV)
    tangents = VertexTangents(topo, fuv, uv.shape[0])
    frames = host(tangents.frames(cuda(V), cuda(uv)))
    want = ref.vertex_frames(V, F, uv, fuv)
    err_f = rel(frames, want)
    w = np.random.default_rng(3).normal(size=(V.shape[0], 6))
    vb0, uvb0 = tangents.backward(cuda(V), cuda(uv), cuda(w))
    vb1, uvb1 = tangents.backward(cuda(V), cuda(uv), cuda(w))
    want_vb, want_uvb = ref.vertex_frames_b(V, F, uv, fuv, w)
    err_v, err_uv = rel(host(vb0), want_vb), rel(host(uvb0), want_uvb)
    record(f"normal_map_tangents_{mesh}", {"frames_rel": err_f, "vertices_b_rel": err_v, "uv_b_rel": err_uv})
    assert err_f <= 1e-12 and err_v <= 1e-12 and err_uv <= 1e-12
    assert torch.equal(vb0, vb1) and torch.equal(uvb0, uvb1)


def test_the_torus_seam_keeps_its_tangents_continuous():
    # the position vertices are shared across the seam, the uv split: the seam's frames are those of its neighbours
    V, F, uv, fuv = torus()
    frames = ref.vertex_frames(V, F, uv, fuv)
    topo = MeshTopology(F, V.shape[0], device=DEV)
    got = host(VertexTangents(topo, fuv, uv.shape[0]).frames(cuda(V), cuda(uv)))
    assert np.allclose(got, frames, atol=1e-13)
    nv = 24
    seam, next_ring = got[:nv], got[nv:2 * nv]
    assert np.min(np.sum(seam[:, :3] * next_ring[:, :3], axis=1)) > 0.9


# ------------------------------------------------------------------------------------- 2. per-pixel kernels

def _gbuffer(rng, H=37, W=53):
    g = rng.normal(size=(H * W, 13))
    g[:, 6] = rng.uniform(0.2, 1.0, H * W)
    M = rng.normal(size=(H * W, 3)) * 0.3 + [0, 0, 1]
    g[0::11, 6] = 0.0                                  # a = 0
    M[1::11] = 0.0                                     # |p| = 0
    g[2::11, 0:3], g[2::11, 7:10] = [0, 0, 1.5], [0, 0, -3.0]  # T parallel to N (exact in fp32): t = 0
    g[3::11, 0:3] = 0.0                                # |N| = 0
    g = g.astype(np.float32).astype(np.float64)
    M = M.astype(np.float32).astype(np.float64)
    return g.reshape(H, W, 13), M.reshape(H, W, 3)


def test_normal_map_kernels_match_the_restatement():
    rng = np.random.default_rng(5)
    g, M = _gbuffer(rng)
    H, W = g.shape[:2]
    out = host(mesh_ops.normal_map(cuda(g, torch.float32), cuda(M, torch.float32)))
    want = ref.normal_map(g.reshape(-1, 13), M.reshape(-1, 3)).reshape(H, W, 7)
    ob = rng.normal(size=(H, W, 7)).astype(np.float32).astype(np.float64)
    gb, Mb = mesh_ops.normal_map_backward(cuda(g, torch.float32), cuda(M, torch.float32), cuda(ob, torch.float32))
    want_gb, want_Mb = ref.normal_map_b(g.reshape(-1, 13), M.reshape(-1, 3), ob.reshape(-1, 7))
    # fp64 maths, fp32 results: one rounding per entry
    errs = {"out": float(np.abs(out - want).max()), "gbuffer_b": float(np.abs(host(gb) - want_gb.reshape(H, W, 13)).max()
                                                                       / np.abs(want_gb).max()),
            "map_b": float(np.abs(host(Mb) - want_Mb.reshape(H, W, 3)).max() / np.abs(want_Mb).max())}
    record("normal_map_pixel_kernels", errs)
    assert np.allclose(out, want, rtol=1e-6, atol=1e-7)
    assert np.allclose(host(gb), want_gb.reshape(H, W, 13), rtol=1e-6, atol=1e-6 * np.abs(want_gb).max())
    assert np.allclose(host(Mb), want_Mb.reshape(H, W, 3), rtol=1e-6, atol=1e-6 * np.abs(want_Mb).max())
    assert not np.any(out[0, 0, :3]) and not np.any(host(gb).reshape(-1, 13)[0::11, 7:13])


# ------------------------------------------------------------------------------------------ views

LIGHT = np.array([0.3, -0.4, 0.8])
POINT = np.array([[1.5, -1.0, 2.0, 4.0]])
SH = np.array([0.5, 0.1, -0.2, 0.05, 0.02, -0.03, 0.04, 0.01, -0.02])


def textured_view(V, F, uv, fuv, texture, nmap=None, light=LIGHT, ambient=0.2, specular=0.3, **kw):
    return DeviceMeshView(F, V.shape[0], camera(), SIZE, SIZE, light_directional=light, ambient=ambient,
                          background_color=(0.1, 0.2, 0.3), sigma=1.0, device=DEV, uv=uv, faces_uv=fuv,
                          texture=texture, shading="phong_textured", specular=specular, shininess=10.0,
                          normal_map=nmap, **kw)


CASES = {
    "plain": {},
    "sh": dict(sh="SH"),
    "point": dict(point_lights="POINT"),
    "cube": dict(point_lights="POINT", shadow_map_size=128, shadow_bias=0.02, shadow_softness=0.05),
    "sun": dict(light_shadow_map_size=256, light_shadow_bias=0.02, light_shadow_softness=0.05,
                light_shadow_bounds=(0.0, 0.0, 4.0, 1.6)),
}


def _case(name):
    kw = dict(CASES[name])
    if "sh" in kw:
        kw["sh"] = cuda(SH)
    if "point_lights" in kw:
        kw["point_lights"] = cuda(POINT)
    return kw


@pytest.mark.parametrize("case", list(CASES))
def test_a_flat_map_gives_the_image_without_a_map(case):
    V, F, uv, fuv = torus()
    texture = np.random.default_rng(0).uniform(0.3, 1.0, (64, 64, 3))
    flat = np.tile([0.0, 0.0, 1.0], (64, 64, 1))
    plain = textured_view(V, F, uv, fuv, texture, **_case(case))
    mapped = textured_view(V, F, uv, fuv, texture, flat, **_case(case))
    a = host(plain.render(cuda(V)))
    b = host(mapped.render(cuda(V)))
    err = float(np.abs(a - b).max())
    record(f"normal_map_flat_{case}", {"max_abs_diff": err})
    assert err <= 1e-5
    assert np.abs(a - 0.1 * np.array([1, 2, 3])).max() > 0.1  # the torus is in view


@pytest.mark.parametrize("axis", [0, 1])
def test_a_tilted_constant_map_shades_a_plane_as_lambert(axis):
    """A camera-facing plane with u along +x and v along +y: the map (sin t, 0, cos t) tilts the normal toward +x,
    (0, sin t, cos t) toward +y, so the interior is albedo (ambient + max(0, -<n', l>)) with n' = sin t e + cos t n."""
    V, F, uv, fuv = grid_plane()
    theta = np.radians(35.0)
    m = np.zeros(3)
    m[axis], m[2] = np.sin(theta), np.cos(theta)
    albedo = np.array([0.8, 0.6, 0.4])
    light = np.array([-0.5, 0.3, 0.7])
    view = textured_view(V, F, uv, fuv, np.tile(albedo, (32, 32, 1)), np.tile(m, (32, 32, 1)), light=light,
                         ambient=0.1, specular=0.0)
    image = host(view.render(cuda(V)))
    e = np.zeros(3)
    e[axis] = 1.0
    n = np.array([0.0, 0.0, -1.0])
    n_tilted = np.sin(theta) * e + np.cos(theta) * n
    want = albedo * (0.1 + max(0.0, -n_tilted @ light))
    # pixels well inside the plane's projection (it spans about +-30 pixels around the centre)
    c = (SIZE - 1) // 2
    interior = image[c - 20:c + 20, c - 20:c + 20]
    err = float(np.abs(interior - want).max())
    other = albedo * (0.1 + max(0.0, -(-np.sin(theta) * e + np.cos(theta) * n) @ light))
    record(f"normal_map_plane_axis{axis}", {"max_abs_err": err, "mirrored_tilt_would_give": other.tolist()})
    assert err <= 1e-5
    assert np.abs(other - want).max() > 0.05  # the test tells the two signs apart


# ------------------------------------------------------------------------------------ 4. central differences

FD_TOL = 5e-3


def _bumpy_setup():
    V, F, uv, fuv = grid_plane(n=12, texels=16)
    rng = np.random.default_rng(9)
    texture = rng.uniform(0.4, 1.0, (16, 16, 3))
    nmap = np.concatenate((rng.normal(size=(16, 16, 2)) * 0.3, np.ones((16, 16, 1))), axis=2)
    w = rng.uniform(0, 1, (SIZE, SIZE, 3))
    return V, F, uv, fuv, texture, nmap, w


def _loss(view, V, nmap, w):
    return float(np.sum(host(view.render(cuda(V), normal_map=cuda(nmap, torch.float32))) * w))


def test_gradients_agree_with_central_differences():
    V, F, uv, fuv, texture, nmap, w = _bumpy_setup()
    view = textured_view(V, F, uv, fuv, texture, nmap, specular=0.2)
    view.render(cuda(V))
    out = view.backward(cuda(w, torch.float32))
    nb, uvb, vb = host(out["normal_map_b"]), host(out["uv_b"]), host(out["vertices_b"])
    h = 1e-2
    res = {}
    # interior texels, each channel
    texels = [(5, 7, 0), (8, 4, 1), (10, 10, 2), (6, 11, 0)]
    an, fd = [], []
    for (i, j, k) in texels:
        p, m = nmap.copy(), nmap.copy()
        p[i, j, k] += h
        m[i, j, k] -= h
        fd.append((_loss(view, V, p, w) - _loss(view, V, m, w)) / (2 * h))
        an.append(nb[i, j, k])
    res["normal_map_b"] = {"analytic": an, "fd": fd, "rel_err": rel(an, fd)}
    # a rigid translation of the uv (a view per offset: the view's uv is fixed) and of the vertices
    an, fd = [], []
    for k in range(2):
        e = np.zeros(2)
        e[k] = 5e-3  # texels: a small step crosses few of the bilinear sampling's kinks
        lp = _loss(textured_view(V, F, uv + e, fuv, texture, nmap, specular=0.2), V, nmap, w)
        lm = _loss(textured_view(V, F, uv - e, fuv, texture, nmap, specular=0.2), V, nmap, w)
        fd.append((lp - lm) / 1e-2)
        an.append(uvb[:, k].sum())
    res["uv_b_translation"] = {"analytic": an, "fd": fd, "rel_err": rel(an, fd)}
    an, fd = [], []
    for k in range(3):
        e = np.zeros(3)
        e[k] = 2e-3
        fd.append((_loss(view, V + e, nmap, w) - _loss(view, V - e, nmap, w)) / 4e-3)
        an.append(vb[:, k].sum())
    res["vertices_b_translation"] = {"analytic": an, "fd": fd, "rel_err": rel(an, fd)}
    record("normal_map_fd", res)
    for k, r in res.items():
        assert np.linalg.norm(r["fd"]) > 0, k
        assert r["rel_err"] <= FD_TOL, k


# --------------------------------------------------------------------------------------------------- 5. PyTorch

@pytest.mark.parametrize("case", ["plain", "sun"])
def test_pytorch_gradients_equal_the_device_view(case):
    V, F, uv, fuv = torus()
    rng = np.random.default_rng(2)
    texture = rng.uniform(0.3, 1.0, (64, 64, 3))
    nmap = np.concatenate((rng.normal(size=(64, 64, 2)) * 0.2, np.ones((64, 64, 1))), axis=2)
    kw = _case(case)
    view = textured_view(V, F, uv, fuv, texture, nmap, **kw)
    dimage = view.render(cuda(V))
    image_b = cuda(rng.normal(size=tuple(dimage.shape)), torch.float32)
    out = view.backward(image_b)
    vertices, uv_t = cuda(V).requires_grad_(True), cuda(uv).requires_grad_(True)
    tex_t, nmap_t = cuda(texture).requires_grad_(True), cuda(nmap).requires_grad_(True)
    scene = P.Scene3DPytorch(shading="phong_textured")
    scene.set_mesh(P.ColoredTriMeshPytorch(F, vertices, faces_uv=fuv, uv=uv_t, texture=tex_t, normal_map=nmap_t,
                                           device=DEV))
    if case == "sun":
        scene.set_light(cuda(LIGHT), 0.2, shadow_map_size=kw["light_shadow_map_size"],
                        shadow_bias=kw["light_shadow_bias"], shadow_softness=kw["light_shadow_softness"],
                        shadow_bounds=kw["light_shadow_bounds"])
    else:
        scene.set_light(cuda(LIGHT), 0.2)
    scene.set_specular(0.3, 10.0)
    scene.set_background_color((0.1, 0.2, 0.3))
    cam = camera()
    image = scene.render(P.CameraPytorch(cam.extrinsic, cam.intrinsic, SIZE, SIZE, cam.distortion))
    assert torch.allclose(image, dimage, rtol=0, atol=1e-6)
    (image.double() * image_b.double()).sum().backward()
    errs = {k: rel(host(t.grad), host(out[o])) for k, t, o in (
        ("normal_map", nmap_t, "normal_map_b"), ("texture", tex_t, "texture_b"), ("uv", uv_t, "uv_b"),
        ("vertices", vertices, "vertices_b"))}
    record(f"normal_map_pytorch_vs_view_{case}", errs)
    # the raster adjoints add with fp32 atomics whose order varies between the two runs
    for k, e in errs.items():
        assert e <= 1e-3, k


def test_views_refuse_a_normal_map_they_cannot_use():
    V, F, uv, fuv = grid_plane()
    tex, nmap = np.ones((32, 32, 3)), np.tile([0.0, 0.0, 1.0], (32, 32, 1))
    with pytest.raises(ValueError, match="phong_textured"):
        DeviceMeshView(F, V.shape[0], camera(), 32, 32, device=DEV, uv=uv, faces_uv=fuv, texture=tex, normal_map=nmap)
    with pytest.raises(ValueError, match="phong_textured"):
        DeviceMeshView(F, V.shape[0], camera(), 32, 32, device=DEV, shading="phong", normal_map=nmap)
    with pytest.raises(ValueError, match="Ht and Wt"):
        textured_view(V, F, uv, fuv, tex, np.zeros((16, 32, 3)))
    view = textured_view(V, F, uv, fuv, tex)
    with pytest.raises(ValueError, match="no normal map"):
        view.render(cuda(V), normal_map=cuda(nmap, torch.float32))
    with pytest.raises(ValueError, match="textured mesh"):
        P.ColoredTriMeshPytorch(F, cuda(V), device=DEV, normal_map=nmap)


# -------------------------------------------------------------------------------------------- 6. no host sync

def test_render_and_backward_make_no_host_sync():
    V, F, uv, fuv, texture, nmap, w = _bumpy_setup()
    kw = _case("sun")
    kw.update(point_lights=cuda(POINT), shadow_map_size=128, shadow_bias=0.02, shadow_softness=0.05)
    view = textured_view(V, F, uv, fuv, texture, nmap, **kw)
    Vd, nd, wd = cuda(V), cuda(nmap, torch.float32), cuda(w, torch.float32)
    view.render(Vd, normal_map=nd)
    view.backward(wd)
    nmap_t = cuda(nmap).requires_grad_(True)
    scene = P.Scene3DPytorch(shading="phong_textured")
    scene.set_mesh(P.ColoredTriMeshPytorch(F, cuda(V).requires_grad_(True), faces_uv=fuv, uv=cuda(uv),
                                           texture=cuda(texture), normal_map=nmap_t, device=DEV))
    scene.set_light(cuda(LIGHT), 0.2)
    scene.set_specular(0.3, 10.0)  # on the device: a host number would be uploaded at every render
    scene.set_background_color((0.1, 0.2, 0.3))
    cam = camera()
    cam = P.CameraPytorch(cam.extrinsic, cam.intrinsic, SIZE, SIZE, cam.distortion)
    scene.render(cam).sum().backward()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        view.render(Vd, normal_map=nd)
        view.backward(wd)
        scene.render(cam).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------ 7. a fit

FIT_STEPS = 150


def _unit(x):
    return x / np.linalg.norm(x, axis=-1, keepdims=True)


def test_adam_recovers_a_bump_map_from_three_lights():
    """A plane with a bump normal map, rendered under three directional lights (one light leaves the normal's
    rotation about it undetermined); the fit starts from the flat map (0, 0, 1)."""
    texels = 32
    V, F, uv, fuv = grid_plane(n=16, texels=texels)
    g = (np.arange(texels) - (texels - 1) / 2) / (texels / 4)
    x, y = np.meshgrid(g, g, indexing="xy")  # rows along v (+y), columns along u (+x)
    height = 0.8 * np.exp(-(x ** 2 + y ** 2) / 2)
    target = _unit(np.stack((-np.gradient(height, axis=1) * 4, -np.gradient(height, axis=0) * 4,
                             np.ones_like(height)), axis=-1))
    albedo = np.tile([0.8, 0.7, 0.6], (texels, texels, 1))
    lights = [np.array([0.6, 0.0, 0.8]), np.array([-0.3, 0.5, 0.8]), np.array([-0.3, -0.5, 0.8])]
    views = [textured_view(V, F, uv, fuv, albedo, target, light=l, ambient=0.1, specular=0.0) for l in lights]
    Vd = cuda(V)
    targets = [v.render(Vd, normal_map=cuda(target, torch.float32)).clone() for v in views]
    param = cuda(np.tile([0.0, 0.0, 1.0], (texels, texels, 1)), torch.float32).requires_grad_(True)
    opt = torch.optim.Adam([param], lr=0.02)
    inner = (slice(2, -2), slice(2, -2))

    def median_angle():
        cos = np.sum(_unit(host(param))[inner] * target[inner], axis=-1)
        return float(np.median(np.degrees(np.arccos(np.clip(cos, -1, 1)))))

    start = median_angle()
    for _ in range(FIT_STEPS):
        opt.zero_grad()
        grad = torch.zeros_like(param)
        for v, t in zip(views, targets):
            image = v.render(Vd, normal_map=param.detach())
            grad += v.backward(2 * (image - t))["normal_map_b"]
        param.grad = grad
        opt.step()
    end = median_angle()
    record("normal_map_fit", {"steps": FIT_STEPS, "median_error_start_deg": start, "median_error_end_deg": end})
    assert end <= 0.5 * start
