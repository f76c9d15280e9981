"""GPU: shadows from the directional light - the sun projection against the fp64 restatement and its map against a
plain depth render, the visibility kernels against the restatement (tests/sun_shadow_ref.py), the sun-shadowed Phong
kernels at V = 1 against the unshadowed ones, a known shadow against an analytic ray cast, no acne on a lit sphere,
gradients against central differences, the PyTorch path against the device view, sun and point-light shadows in one
view, the refusals, no host synchronisation, and a fit of the light's direction."""
import json

import numpy as np
import phong_ref
import point_light_ref
import pytest
import sun_shadow_ref as ref

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from deodr_b200 import mesh_ops  # noqa: E402
from deodr_b200.mesh_fitter import new_scratch  # noqa: E402
from deodr_b200.mesh_ops import CameraParams, DeviceMeshView, MeshTopology  # noqa: E402
from deodr_b200.pytorch import scene3d_pytorch as P  # noqa: E402

DEV = "cuda:0"


def host(t):
    return t.detach().cpu().numpy().astype(np.float64)


def cuda(a, dtype=torch.float64):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def record(name, value):
    print(json.dumps({"measured": name, "value": value}))


def rel(got, want):
    return float(np.abs(np.asarray(got) - np.asarray(want)).max() / max(np.abs(np.asarray(want)).max(), 1e-300))


# ------------------------------------------------------------------------------------------------------ the scene

def _turned(vertices, faces, toward):
    tri = vertices[faces]
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    flip = np.sum(n * toward, axis=1) < 0
    faces = faces.copy()
    faces[flip] = faces[flip][:, ::-1]
    return faces


def sphere(center, radius, n=24):
    """A cube sphere: six n x n grids projected on the sphere, shared vertices merged, faces outward."""
    g = np.linspace(-1, 1, n + 1)
    verts, faces = [], []
    for axis in range(3):
        for sign in (-1, 1):
            a, b = np.meshgrid(g, g, indexing="ij")
            p = np.zeros((n + 1, n + 1, 3))
            p[..., axis] = sign
            p[..., (axis + 1) % 3], p[..., (axis + 2) % 3] = a, b
            base = sum(len(v) for v in verts)
            verts.append(p.reshape(-1, 3))
            i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
            q = (i * (n + 1) + j).ravel() + base
            faces += [np.stack((q, q + n + 1, q + n + 2), 1), np.stack((q, q + n + 2, q + 1), 1)]
    v = np.concatenate(verts)
    v, inv = np.unique(np.round(v, 12), axis=0, return_inverse=True)
    f = inv.reshape(-1)[np.concatenate(faces)]
    v = v / np.linalg.norm(v, axis=1, keepdims=True) * radius + center
    return v, _turned(v, f, v[f].mean(axis=1) - center)


def plane(z, half, n=40):
    """The square |x|, |y| <= half at depth z, facing -z (the camera and the light)."""
    g = np.linspace(-half, half, n + 1)
    x, y = np.meshgrid(g, g, indexing="ij")
    v = np.stack((x, y, np.full_like(x, z)), axis=-1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    q = (i * (n + 1) + j).ravel()
    f = np.concatenate((np.stack((q, q + n + 1, q + n + 2), 1), np.stack((q, q + n + 2, q + 1), 1)))
    return v, _turned(v, f, np.array([[0.0, 0.0, -1.0]]))


SPHERE_C, SPHERE_R, PLANE_Z = np.array([0.0, 0.0, 3.0]), 0.5, 4.0
# the direction the light travels, from beside the camera and obliquely onto the plane (far from the pole d = -z)
LIGHT = 0.9 * np.array([0.5, -0.4, 1.0]) / np.linalg.norm([0.5, -0.4, 1.0])
BOUNDS = (0.0, 0.0, 3.5, 3.6)  # the window: the sphere and the plane's corners
SIZE, FOCAL = 256, 240.0


def scene_mesh():
    sv, sf = sphere(SPHERE_C, SPHERE_R)
    pv, pf = plane(PLANE_Z, 2.5)
    V = np.concatenate((sv, pv))
    F = np.concatenate((sf, pf + len(sv)))
    return F.astype(np.int64), V, len(sv)


def camera():
    K = np.array([[FOCAL, 0, (SIZE - 1) / 2], [0, FOCAL, (SIZE - 1) / 2], [0, 0, 1]])
    return CameraParams(np.eye(3, 4), K)


def make_view(light=LIGHT, M=1024, bias=0.02, softness=0.05, sigma=1.0, kind="phong", shadows=True, faces=None,
              V=None, bounds=BOUNDS, specular=0.3, **kw):
    F, Vx, _ = scene_mesh() if faces is None else (faces, V, None)
    if shadows:
        kw.update(light_shadow_map_size=M, light_shadow_bias=bias, light_shadow_softness=softness,
                  light_shadow_bounds=bounds)
    view = DeviceMeshView(F, Vx.shape[0], camera(), SIZE, SIZE, light_directional=light, ambient=0.1,
                          background_color=(0.1, 0.2, 0.3), sigma=sigma, device=DEV, shading=kind, specular=specular,
                          shininess=10.0, **kw)
    colors = np.random.default_rng(0).uniform(0.5, 1.0, (Vx.shape[0], 3))
    return view, Vx, colors


# -------------------------------------------------------------------------------------------- 1. projection, map

@pytest.mark.parametrize("l", [LIGHT, [0.0, 0.0, -2.0], [1e-5, 0.0, -1.0], [0.0, 0.0, 0.0], [-1.0, 2.0, 0.5]])
def test_sun_projection_matches_the_restatement(l):
    F, V, _ = scene_mesh()
    l = np.asarray(l, dtype=np.float64)
    for M in (8, 1024, 4096):
        ij, depths = mesh_ops.sun_project(cuda(V), cuda(l), BOUNDS, M)
        u, v, z = ref.project(V, l, np.array(BOUNDS[:3]), BOUNDS[3], M)
        assert rel(host(ij)[:, 0], u) <= 1e-12 and rel(host(ij)[:, 1], v) <= 1e-12 and rel(host(depths), z) <= 1e-12
        # the Phong params [6] serve as the light too
        ij6, d6 = mesh_ops.sun_project(cuda(V), cuda(np.concatenate((l, [0.1, 0.3, 10.0]))), BOUNDS, M)
        assert torch.equal(ij6, ij) and torch.equal(d6, depths)


def test_the_map_is_a_plain_depth_render_of_the_projection():
    from deodr_b200.renderer import DeviceScene, default_renderer
    from deodr_b200.scenes import SceneArrays

    F, V, _ = scene_mesh()
    M = 256
    view, _, colors = make_view(M=M)
    view.render(cuda(V), cuda(colors))
    sun_map = view.light_shadow_map().clone()
    ij, depths = mesh_ops.sun_project(cuda(V), cuda(LIGHT), BOUNDS, M)
    flags = MeshTopology(F, V.shape[0], device=DEV).edge_on_silhouette(ij)
    T = F.shape[0]
    scene = DeviceScene(SceneArrays(
        faces=F.astype(np.uint32), faces_uv=np.zeros((T, 3), np.uint32), ij=host(ij), depths=host(depths),
        textured=np.zeros(T, bool), uv=np.zeros((1, 2)), shade=np.zeros(V.shape[0]), colors=host(depths)[:, None],
        shaded=np.zeros(T, bool), edgeflags=host(flags).astype(bool), height=M, width=M, nb_colors=1,
        texture=np.zeros((2, 2, 1)), background_image=None, background_color=np.array([mesh_ops.SHADOW_FAR]),
        clockwise=False, backface_culling=True, strict_edge=True, perspective_correct=False,
        integer_pixel_centers=True), torch.device(DEV))
    plain = default_renderer(0).render(scene, 1.0)["image"][..., 0]
    assert torch.equal(plain, sun_map)
    assert float(sun_map.min()) > 0 and float((sun_map < 1e29).float().mean()) > 0.2


# ---------------------------------------------------------------------------------- 2. kernels vs the restatement

@pytest.mark.parametrize("l", [LIGHT, [0.0, 0.0, -2.0], [0.0, 0.0, 0.0]])
def test_sun_projection_adjoint_matches_the_restatement(l):
    F, V, _ = scene_mesh()
    rng = np.random.default_rng(7)
    l, M = np.asarray(l, dtype=np.float64), 512
    g = rng.normal(size=(V.shape[0], 3)).astype(np.float32)
    g[rng.random(V.shape[0]) < 0.3] = 0  # vertices the rasteriser gives no gradient
    vb0, lb0 = rng.normal(size=(V.shape[0], 3)), rng.normal(size=6)
    vertices_b, light_b = mesh_ops.sun_project_backward(
        cuda(V), cuda(l), BOUNDS, M, cuda(g[:, :2], torch.float32), cuda(g[:, 2], torch.float32), new_scratch(DEV),
        vertices_b=cuda(vb0), light_b=cuda(lb0))
    x_b, l_b = ref.project_b(V, l, np.array(BOUNDS[:3]), BOUNDS[3], M, *(g.astype(np.float64).T))
    assert rel(host(vertices_b) - vb0, x_b) <= 1e-12
    if np.any(l):
        assert rel(host(light_b)[:3] - lb0[:3], l_b) <= 1e-9
    else:
        assert np.array_equal(host(light_b)[:3], lb0[:3])
    assert np.array_equal(host(light_b)[3:], lb0[3:])


def _random_gbuffer(rng, C, c, r, H=37, W=53):
    x = c + rng.normal(size=(H * W, 3)) * r * 0.6
    x[rng.random(H * W) < 0.1] *= 3  # some outside the window
    a = np.where(rng.random(H * W) < 0.15, 0.0, rng.uniform(0.3, 1.0, H * W))
    n = rng.normal(size=(H * W, 3))
    ch = np.concatenate((rng.uniform(0.2, 1, (H * W, C)), n, x * a[:, None], a[:, None]), axis=1)
    return ch.astype(np.float32).astype(np.float64), H, W


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("l", [[0.6, -0.3, 0.7], [0.0, 0.0, -1.5]])
def test_visibility_kernels_match_the_restatement(split, l):
    rng = np.random.default_rng(10 + split)
    C, M, bias, soft = 3, 32, 0.05, 0.8
    c, r = np.array([0.2, -0.1, 1.0]), 2.0
    bounds = tuple(c) + (r,)
    l = np.asarray(l)
    params = np.concatenate((l, [0.2, 0.5, 12.0]))
    ch, H, W = _random_gbuffer(rng, C, c, r)
    D = rng.uniform(r, 3 * r, (M, M)).astype(np.float32)
    D[rng.random(D.shape) < 0.2] = ref.FAR
    if split:
        chd, kw = cuda(ch[:, C:].reshape(H, W, 7), torch.float32), dict(albedo=cuda(ch[:, :C].reshape(H, W, C),
                                                                                     torch.float32))
    else:
        chd, kw = cuda(ch.reshape(H, W, -1), torch.float32), {}
    pos, cov = ch[:, C + 3:C + 6], ch[:, C + 6]
    vis = mesh_ops.sun_visibility(chd, cuda(params), cuda(D, torch.float32), bounds, bias, soft, **kw)
    want = ref.gbuffer_visibility(pos, cov, l, D.astype(np.float64), c, r, M, bias, soft)
    assert np.abs(host(vis).reshape(-1) - want).max() <= 1e-6
    assert np.all(host(vis).reshape(-1)[cov == 0] == 1.0)
    assert np.any(want < 1) and np.any((want > 0) & (want < 1))
    g = rng.normal(size=(H * W,)).astype(np.float32)
    params_b = cuda(rng.normal(size=6))
    before = host(params_b)
    out = mesh_ops.sun_visibility_backward(chd, cuda(params), cuda(D, torch.float32), bounds, bias, soft,
                                           cuda(g.reshape(H, W), torch.float32), new_scratch(DEV), light_b=params_b,
                                           **kw)
    pos_b, cov_b, D_b, l_b = ref.gbuffer_visibility_b(pos, cov, l, D.astype(np.float64), c, r, M, bias, soft,
                                                      g.astype(np.float64))
    got = host(out[0]).reshape(H * W, -1)
    off = 3 if split else C + 3
    assert np.all(np.abs(got[:, off:off + 3] - pos_b) <= 1e-5 * np.abs(pos_b).max() + 1e-6)
    assert np.all(np.abs(got[:, off + 3] - cov_b) <= 1e-5 * np.abs(cov_b).max() + 1e-6)
    assert np.all(got[:, :off] == 0)  # nothing but the position and coverage slices
    assert np.abs(host(out[1]) - D_b).max() <= 1e-5 * np.abs(D_b).max()
    # accumulated into params_b[0:3] (the shading's l_b), the rest untouched
    assert rel(host(out[2])[:3] - before[:3], l_b) <= 1e-9
    assert np.array_equal(host(out[2])[3:], before[3:])


def _phong_inputs(C, split, seed=3, H=41, W=59):
    rng = np.random.default_rng(seed)
    cam = np.array([0.2, -0.1, -5.0])
    ch = phong_ref.random_pixels(rng, C, P=H * W, cam=cam).astype(np.float32).astype(np.float64)
    bg = cuda(rng.uniform(0, 1, C), torch.float32)
    params = cuda([0.3, -0.3, 0.6, 0.4, 0.7, 12.0])
    if split:
        kw = dict(albedo=cuda(ch[:, :C].reshape(H, W, C), torch.float32))
        chd = cuda(ch[:, C:].reshape(H, W, 7), torch.float32)
    else:
        kw, chd = {}, cuda(ch.reshape(H, W, -1), torch.float32)
    g = cuda(rng.normal(size=(H, W, C)), torch.float32)
    return chd, params, cuda(cam), bg, g, kw, rng, ch


CASES = [dict(), dict(S=1), dict(S=3), dict(L=2), dict(S=3, L=1, P=3), dict(L=2, vis=True), dict(S=1, L=3, vis=True)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(f"{k}{v}" for k, v in c.items()) or "plain")
@pytest.mark.parametrize("split", [False, True])
def test_sun_shadowed_phong_at_full_visibility_is_the_unshadowed_one(case, split):
    C = 3
    chd, params, cam, bg, g, kw, rng, _ = _phong_inputs(C, split)
    H, W = chd.shape[:2]
    S, L, Pc = case.get("S"), case.get("L"), case.get("P", 1)
    if S:
        kw["sh"] = cuda(rng.normal(size=(9, S)) * 0.2 if S > 1 else rng.normal(size=9) * 0.2)
    if L:
        kw["point_lights"] = cuda(point_light_ref.random_lights(rng, L, Pc, center=np.array([0.2, -0.1, -0.5]),
                                                                spread=2.0))
        if case.get("vis"):
            kw["visibility"] = cuda(rng.uniform(0, 1, (H, W, L)), torch.float32)
    ones = torch.ones((H, W), dtype=torch.float32, device=DEV)
    want = mesh_ops.phong_shade(chd, params, cam, bg, **kw)
    assert torch.equal(mesh_ops.phong_shade(chd, params, cam, bg, sun_visibility=ones, **kw), want)
    scratch = new_scratch(DEV)
    want_b = mesh_ops.phong_shade_backward(chd, params, cam, bg, g, scratch, center_grad=True, **kw)
    got_b = mesh_ops.phong_shade_backward(chd, params, cam, bg, g, scratch, center_grad=True, sun_visibility=ones,
                                          **kw)
    assert len(got_b) == len(want_b) + 1
    for a, b in zip(got_b, want_b):
        assert torch.equal(a, b)


@pytest.mark.parametrize("split", [False, True])
def test_sun_shadowed_phong_matches_the_restatement(split):
    C = 3
    chd, params, cam, bg, g, kw, rng, ch = _phong_inputs(C, split, seed=5)
    H, W = chd.shape[:2]
    V = rng.uniform(0, 1, (H, W)).astype(np.float32)
    image = mesh_ops.phong_shade(chd, params, cam, bg, sun_visibility=cuda(V, torch.float32), **kw)
    args = (ch, host(params), host(cam), host(bg))
    want = ref.shade(*args, V.reshape(-1).astype(np.float64))
    assert np.abs(host(image).reshape(-1, C) - want).max() <= 1e-5
    out = mesh_ops.phong_shade_backward(chd, params, cam, bg, g, new_scratch(DEV), sun_visibility=cuda(V, torch.float32),
                                        **kw)
    ch_b, params_b, V_b = ref.shade_b(*args, V.reshape(-1).astype(np.float64), host(g).reshape(-1, C))
    assert np.abs(host(out[-1]).reshape(-1) - V_b).max() <= 1e-5 * max(1.0, np.abs(V_b).max())
    assert rel(host(out[1]), params_b) <= 1e-6
    got = host(out[0]).reshape(H * W, -1)
    want_ch = ch_b[:, C:] if split else ch_b
    assert np.abs(got - want_ch).max() <= 1e-4 * max(1.0, np.abs(want_ch).max())


# --------------------------------------------------------------------------------------------- 3. a known shadow

def _rays():
    r, c = np.meshgrid(np.arange(SIZE), np.arange(SIZE), indexing="ij")
    d = np.stack(((c - (SIZE - 1) / 2) / FOCAL, (r - (SIZE - 1) / 2) / FOCAL, np.ones_like(r, dtype=float)), -1)
    return d / np.linalg.norm(d, axis=-1, keepdims=True)


def _ray_sphere_distance(x, d):
    """The distance from the sphere's centre to the rays from x [N,3] towards the light (along -d)."""
    u = d / np.linalg.norm(d)
    w = SPHERE_C - x
    t = np.maximum(w @ -u, 0)
    return np.linalg.norm(x - t[:, None] * u[None] - SPHERE_C, axis=1)


def test_a_sphere_casts_its_analytic_shadow_on_a_plane():
    M, band_texels = 1024, 4
    view, V, colors = make_view(M=M)
    view.render(cuda(V), cuda(colors))
    vis = host(view.light_shadow_visibility()).reshape(-1)
    d = _rays().reshape(-1, 3)
    # plane pixels whose view ray passes well clear of the sphere (no mixed G-buffer positions at its silhouette)
    clear = np.linalg.norm(np.cross(d, SPHERE_C[None]), axis=1) > SPHERE_R + 4 * PLANE_Z / FOCAL
    x = d * (PLANE_Z / d[:, 2:3])
    keep = clear & (np.abs(x[:, 0]) < 2.4) & (np.abs(x[:, 1]) < 2.4)
    texel = 2 * BOUNDS[3] / (M - 4)  # a map texel's width in world units
    dist = _ray_sphere_distance(x, LIGHT)
    shadowed, lit = keep & (dist < SPHERE_R - band_texels * texel), keep & (dist > SPHERE_R + band_texels * texel)
    bad_in = int(np.count_nonzero(vis[shadowed] != 0.0))
    bad_out = int(np.count_nonzero(vis[lit] != 1.0))
    record("sun_shadow_known", {"band_texels": band_texels, "shadowed_pixels": int(shadowed.sum()),
                                "lit_pixels": int(lit.sum()), "disagree_in": bad_in, "disagree_out": bad_out})
    assert shadowed.sum() > 500 and lit.sum() > 10_000
    assert bad_in == 0 and bad_out == 0


# ------------------------------------------------------------------------------------------------------ 4. no acne

def test_a_lit_sphere_has_no_acne_and_renders_as_without_shadows():
    F, V = sphere(SPHERE_C, SPHERE_R, n=32)
    F = F.astype(np.int64)
    # from just behind the camera: every pixel the camera sees is lit
    light = np.array([0.05, -0.03, 1.0])
    bounds = tuple(SPHERE_C) + (SPHERE_R * 1.05,)
    view, _, colors = make_view(light=light, M=1024, bias=0.02, softness=0.02, faces=F, V=V, bounds=bounds)
    plain = make_view(light=light, shadows=False, faces=F, V=V)[0]
    image = view.render(cuda(V), cuda(colors))
    vis = host(view.light_shadow_visibility()).reshape(-1)
    record("sun_shadow_acne", {"covered_pixels": int(np.count_nonzero(vis < 2)),
                               "below_one": int(np.count_nonzero(vis != 1))})
    assert np.all(vis == 1.0)
    assert torch.equal(image, plain.render(cuda(V), cuda(colors)))


# -------------------------------------------------------------------------------- 5. gradients vs differences

def _loss(view, V, colors, w):
    return float((view.render(V, colors).double() * w).sum())


# The shadow edge moves with the light and with the occluder.  The lookup's own motion is exact (the bilinear taps),
# but the map's motion reaches the loss only through the map's silhouette antialiasing (DEODR's approximation of a
# moving edge), resampled by the 2x2 taps, as for the cube maps (DESIGN.md section 14).  Angle steps of 1e-3 rad and a
# translation step of 1e-3 of the sphere's distance to the plane (a seventh of a map texel at M = 1024).  Measured on
# an H100: 1.1e-2 in the light's two angles and 1.5e-1 in the occluder's translation (the map's share alone).
FD_STEP = 1e-3
FD_TOL_LIGHT = 0.05
FD_TOL_OCCLUDER = 0.2


def _light_of(theta, phi, norm=0.9):
    return norm * np.array([np.sin(theta) * np.cos(phi), np.sin(theta) * np.sin(phi), np.cos(theta)])


def test_light_direction_gradient_agrees_with_central_differences():
    d = LIGHT / np.linalg.norm(LIGHT)
    theta, phi = np.arccos(d[2]), np.arctan2(d[1], d[0])
    view, V, colors = make_view(light=_light_of(theta, phi), M=1024, softness=0.2, sigma=2.0)
    Vd, cd = cuda(V), cuda(colors)
    image = view.render(Vd, cd)
    w = cuda(np.random.default_rng(4).uniform(0, 1, tuple(image.shape)))
    lb = host(view.backward(w.float())["light_b"])[:3]
    h = FD_STEP
    analytic, fd = [], []
    for k in range(2):
        e = np.zeros(2)
        e[k] = h
        lp, lm = _light_of(theta + e[0], phi + e[1]), _light_of(theta - e[0], phi - e[1])
        analytic.append(float(lb @ (lp - lm) / (2 * h)))
        view.light_directional = lp
        fp = _loss(view, Vd, cd, w)
        view.light_directional = lm
        fm = _loss(view, Vd, cd, w)
        fd.append((fp - fm) / (2 * h))
    view.light_directional = _light_of(theta, phi)
    err = rel(analytic, fd)
    # the shadow's share alone: the same view without shadows
    plain = make_view(light=_light_of(theta, phi), shadows=False, sigma=2.0)[0]
    plain.render(Vd, cd)
    lb_plain = host(plain.backward(w.float())["light_b"])[:3]
    record("sun_shadow_fd_light_direction", {"analytic": analytic, "fd": fd, "rel_err": err,
                                             "shadow_share": (lb - lb_plain).tolist()})
    assert np.linalg.norm(lb - lb_plain) > 0
    assert err <= FD_TOL_LIGHT


def test_occluder_translation_gradient_agrees_with_central_differences():
    view, V, colors = make_view(M=1024, softness=0.2, sigma=2.0)
    _, _, ns = scene_mesh()
    cd = cuda(colors)
    image = view.render(cuda(V), cd)
    # weights on the plane's pixels only: the loss then sees the sphere through its shadow alone
    d = _rays().reshape(SIZE, SIZE, 3)
    off_sphere = np.linalg.norm(np.cross(d, SPHERE_C), axis=-1) > SPHERE_R + 4 * PLANE_Z / FOCAL
    w = cuda(np.random.default_rng(5).uniform(0, 1, tuple(image.shape)) * off_sphere[..., None])
    vb = host(view.backward(w.float())["vertices_b"])[:ns].sum(axis=0)
    h = FD_STEP * (PLANE_Z - SPHERE_C[2])
    fd = []
    for k in range(3):
        e = np.zeros(3)
        e[k] = h
        Vp, Vm = V.copy(), V.copy()
        Vp[:ns] += e
        Vm[:ns] -= e
        fd.append((_loss(view, cuda(Vp), cd, w) - _loss(view, cuda(Vm), cd, w)) / (2 * h))
    err = rel(vb, fd)
    record("sun_shadow_fd_occluder_translation", {"analytic": vb.tolist(), "fd": fd, "rel_err": err})
    assert np.linalg.norm(fd) > 0
    assert err <= FD_TOL_OCCLUDER


# --------------------------------------------------------------------------------------------------- 6. PyTorch

def _scene(light, M=1024, point=None, kind="phong"):
    F, V, _ = scene_mesh()
    colors = np.random.default_rng(0).uniform(0.5, 1.0, (V.shape[0], 3))
    scene = P.Scene3DPytorch(shading=kind)
    vertices = cuda(V).requires_grad_(True)
    scene.set_mesh(P.ColoredTriMeshPytorch(F, vertices, colors=cuda(colors), device=DEV))
    if M:
        scene.set_light(light, 0.1, shadow_map_size=M, shadow_bias=0.02, shadow_softness=0.05, shadow_bounds=BOUNDS)
    else:
        scene.set_light(light, 0.1)
    scene.set_specular(0.3, 10.0)
    if point is not None:
        scene.set_point_lights(point, shadow_map_size=256, shadow_bias=0.02, shadow_softness=0.05)
    scene.set_background_color((0.1, 0.2, 0.3))
    cam = camera()
    return scene, P.CameraPytorch(cam.extrinsic, cam.intrinsic, SIZE, SIZE, cam.distortion), vertices


POINT = np.array([[1.2, -1.2, 1.0, 3.0]])


@pytest.mark.parametrize("with_point", [False, True])
def test_pytorch_gradients_equal_the_device_view(with_point):
    kw = dict(point_lights=cuda(POINT), shadow_map_size=256, shadow_bias=0.02, shadow_softness=0.05) \
        if with_point else {}
    view, V, colors = make_view(**kw)
    dimage = view.render(cuda(V), cuda(colors))
    image_b = cuda(np.random.default_rng(1).normal(size=tuple(dimage.shape)), torch.float32)
    out = view.backward(image_b)
    light = cuda(LIGHT).requires_grad_(True)
    point = cuda(POINT).requires_grad_(True) if with_point else None
    scene, cam, vertices = _scene(light, point=point)
    image = scene.render(cam)
    assert torch.allclose(image, dimage, rtol=0, atol=1e-6)
    (image.double() * image_b.double()).sum().backward()
    assert rel(host(light.grad), host(out["light_b"])[:3]) <= 1e-4
    if with_point:
        assert rel(host(point.grad), host(out["point_lights_b"])) <= 1e-4
    # the raster adjoints add with fp32 atomics whose order varies between the two runs
    assert rel(host(vertices.grad), host(out["vertices_b"])) <= 1e-3


def test_sun_and_point_light_shadows_in_one_view():
    point = cuda(POINT)
    both, V, colors = make_view(point_lights=point, shadow_map_size=256, shadow_bias=0.02, shadow_softness=0.05)
    sun_only = make_view(point_lights=point)[0]
    cube_only = make_view(shadows=False, point_lights=point, shadow_map_size=256, shadow_bias=0.02,
                          shadow_softness=0.05)[0]
    Vd, cd = cuda(V), cuda(colors)
    image = both.render(Vd, cd)
    sun_vis, vis = both.light_shadow_visibility().clone(), both.shadow_visibility().clone()
    sun_map, maps = both.light_shadow_map().clone(), both.shadow_maps().clone()
    sun_only.render(Vd, cd)
    cube_only.render(Vd, cd)
    assert torch.equal(sun_map, sun_only.light_shadow_map()) and torch.equal(maps, cube_only.shadow_maps())
    assert torch.equal(sun_vis, sun_only.light_shadow_visibility())
    assert torch.equal(vis, cube_only.shadow_visibility())
    assert float((sun_vis < 1).float().sum()) > 500 and float((vis < 1).float().sum()) > 500
    # the same two lights, each view shadowing one of them: shadowing both darkens the image the most
    images = [host(v.render(Vd, cd)).sum() for v in (sun_only, cube_only)]
    assert host(image).sum() < min(images)
    # render again before the backward: the renderer keeps one live forward per slot
    assert torch.equal(both.render(Vd, cd), image)
    out = both.backward(torch.ones_like(image))
    for k in ("vertices_b", "light_b", "point_lights_b"):
        assert torch.isfinite(out[k]).all(), k


def test_views_refuse_bad_sun_shadow_arguments():
    F, V, _ = scene_mesh()
    ok = dict(light_shadow_map_size=64, light_shadow_bias=0.1, light_shadow_softness=0.1, light_shadow_bounds=BOUNDS)
    with pytest.raises(ValueError, match="smear"):
        DeviceMeshView(F, V.shape[0], camera(), 32, 32, device=DEV, light_directional=LIGHT, **ok)
    with pytest.raises(ValueError, match="smear"):
        DeviceMeshView(F, V.shape[0], camera(), 32, 32, device=DEV, light_directional=LIGHT, uv=np.zeros((V.shape[0], 2)),
                       faces_uv=F, texture=np.zeros((4, 4, 3)), **ok)
    with pytest.raises(ValueError, match="directional light"):
        DeviceMeshView(F, V.shape[0], camera(), 32, 32, device=DEV, shading="phong", **ok)
    for k in ("light_shadow_bias", "light_shadow_softness", "light_shadow_bounds"):
        kw = dict(ok)
        del kw[k]
        with pytest.raises(ValueError, match="no default is free of scale"):
            DeviceMeshView(F, V.shape[0], camera(), 32, 32, device=DEV, shading="phong", light_directional=LIGHT, **kw)
    for k, bad in (("light_shadow_map_size", 4), ("light_shadow_map_size", 8192), ("light_shadow_bias", -1.0),
                   ("light_shadow_softness", float("nan")), ("light_shadow_bounds", (0, 0, 0, 0.0)),
                   ("light_shadow_bounds", (0, float("inf"), 0, 1.0)), ("light_shadow_bounds", (0, 0, 1.0))):
        with pytest.raises(ValueError):
            DeviceMeshView(F, V.shape[0], camera(), 32, 32, device=DEV, shading="phong", light_directional=LIGHT,
                           **{**ok, k: bad})
    view = DeviceMeshView(F, V.shape[0], camera(), 32, 32, device=DEV, shading="phong", light_directional=LIGHT)
    with pytest.raises(ValueError, match="light_shadow_map_size 0"):
        view.light_shadow_map()
    scene = P.Scene3DPytorch(shading="gouraud")
    with pytest.raises(ValueError, match="smear"):
        scene.set_light(LIGHT, 0.1, shadow_map_size=64, shadow_bias=0.1, shadow_softness=0.1, shadow_bounds=BOUNDS)
    with pytest.raises(ValueError, match="directional light"):
        P.Scene3DPytorch(shading="phong").set_light(None, 0.1, shadow_map_size=64, shadow_bias=0.1,
                                                    shadow_softness=0.1, shadow_bounds=BOUNDS)


# -------------------------------------------------------------------------------------------- 7. no host sync

def test_render_and_backward_make_no_host_sync():
    view, V, colors = make_view(M=512, point_lights=cuda(POINT), shadow_map_size=256, shadow_bias=0.02,
                                shadow_softness=0.05)
    Vd, cd = cuda(V), cuda(colors)
    ones = torch.ones_like(view.render(Vd, cd))
    view.backward(ones)
    scene, cam, _ = _scene(cuda(LIGHT).requires_grad_(True), M=512)
    scene.render(cam).sum().backward()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        view.render(Vd, cd)
        view.backward(ones)
        scene.render(cam).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------ 8. a fit

FIT_STEPS = 200


def _angle(a, b):
    return float(np.degrees(np.arccos(np.clip(a @ b / (np.linalg.norm(a) * np.linalg.norm(b)), -1, 1))))


def _fit(shadows, target, start):
    x = cuda(start).requires_grad_(True)
    scene, cam, _ = _scene(x, M=1024 if shadows else 0)
    scene.set_specular(0.0, 10.0)
    opt = torch.optim.Adam([x], lr=0.01)
    decay = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=1e-2 ** (1 / FIT_STEPS))
    for _ in range(FIT_STEPS):
        opt.zero_grad()
        loss = ((scene.render(cam) - target).double() ** 2).sum()
        loss.backward()
        opt.step()
        decay.step()
    return host(x)


def test_adam_recovers_the_light_direction_from_a_shadow():
    """The fit starts 10 degrees off the light's direction.  The same fit without shadows explains the target with
    the shading alone."""
    scene, cam, _ = _scene(cuda(LIGHT), M=1024)
    scene.set_specular(0.0, 10.0)
    with torch.no_grad():
        target = scene.render(cam).clone()
    axis = np.cross(LIGHT, [0.0, 0.0, 1.0])
    axis /= np.linalg.norm(axis)
    t = np.radians(10.0)
    u = LIGHT / np.linalg.norm(LIGHT)
    start = np.linalg.norm(LIGHT) * (u * np.cos(t) + np.cross(axis, u) * np.sin(t) + axis * (axis @ u) * (1 - np.cos(t)))
    got = _fit(True, target, start)
    plain = _fit(False, target, start)
    err, err_plain = _angle(got, LIGHT), _angle(plain, LIGHT)
    record("sun_shadow_fit", {"steps": FIT_STEPS, "start_deg": _angle(start, LIGHT), "error_deg": err,
                              "error_without_shadows_deg": err_plain})
    assert err < err_plain
    assert err <= 1.0
