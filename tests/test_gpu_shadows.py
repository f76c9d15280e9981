"""GPU: shadows from point lights - the cube projection and maps against project_points_dev and render_depth, the
visibility kernels against the fp64 restatement (tests/shadow_ref.py), the shadowed Phong kernels at V = 1 against the
unshadowed ones, a known shadow against an analytic ray cast, no acne on a lit sphere, gradients against central
differences, the PyTorch path against the device view, no host synchronisation, and a fit of a light's position."""
import json

import numpy as np
import phong_ref
import point_light_ref
import pytest
import shadow_ref as ref

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from deodr_b200 import mesh_ops  # noqa: E402
from deodr_b200.mesh_fitter import new_scratch  # noqa: E402
from deodr_b200.mesh_ops import CameraParams, DeviceMeshView  # noqa: E402
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
    """faces turned so that cross(v1 - v0, v2 - v0) points along ``toward`` [T,3] (the front-facing winding)."""
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
    """The square |x|, |y| <= half at depth z, facing -z (the camera and the lights)."""
    g = np.linspace(-half, half, n + 1)
    x, y = np.meshgrid(g, g, indexing="ij")
    v = np.stack((x, y, np.full_like(x, z)), axis=-1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    q = (i * (n + 1) + j).ravel()
    f = np.concatenate((np.stack((q, q + n + 1, q + n + 2), 1), np.stack((q, q + n + 2, q + 1), 1)))
    return v, _turned(v, f, np.array([[0.0, 0.0, -1.0]]))


SPHERE_C, SPHERE_R, PLANE_Z = np.array([0.0, 0.0, 3.0]), 0.5, 4.0
LIGHT_P = np.array([1.2, -1.2, 1.0])
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


def lights_of(p=LIGHT_P, intensity=None, S=1):
    dist2 = float(np.sum((np.asarray(p) - SPHERE_C) ** 2))
    I = np.full(S, 0.8 * dist2 if intensity is None else intensity)
    return np.concatenate((p, I))[None]


def make_view(lights, M=512, bias=0.02, softness=0.05, sigma=1.0, kind="phong", shadows=True, faces=None, V=None):
    F, Vx, _ = scene_mesh() if faces is None else (faces, V, None)
    kw = dict(shadow_map_size=M, shadow_bias=bias, shadow_softness=softness) if shadows else {}
    view = DeviceMeshView(F, Vx.shape[0], camera(), SIZE, SIZE, light_directional=None, ambient=0.05,
                          background_color=(0.1, 0.2, 0.3), sigma=sigma, device=DEV, shading=kind, specular=0.3,
                          shininess=10.0, point_lights=lights, **kw)
    colors = np.random.default_rng(0).uniform(0.5, 1.0, (Vx.shape[0], 3))
    return view, Vx, colors


# -------------------------------------------------------------------------------------------- 1. projection, maps

def test_cube_projection_is_project_points_dev_of_each_face():
    F, V, _ = scene_mesh()
    lights = cuda(np.concatenate((lights_of(), lights_of(p=[-0.5, 0.7, 2.0]))))
    cams, ij, depths = mesh_ops.cube_project(cuda(V), lights, 512)
    assert np.array_equal(host(cams), ref.cameras(host(lights), 512))
    for f in range(12):
        ij_f, d_f = mesh_ops.project_points_dev(cuda(V), cams[f].contiguous(), False)
        # bit for bit; a vertex in a face's camera plane projects to the same NaN or inf in both
        torch.testing.assert_close(ij[f], ij_f, rtol=0, atol=0, equal_nan=True)
        torch.testing.assert_close(depths[f], d_f, rtol=0, atol=0, equal_nan=True)


def test_each_face_map_is_the_depth_render_of_its_camera():
    F, V, _ = scene_mesh()
    lights = cuda(lights_of())
    M = 128
    view, _, colors = make_view(lights, M=M)
    view.render(cuda(V), cuda(colors))
    maps = view.shadow_maps().clone()
    cams = mesh_ops.cube_project(cuda(V), lights, M)[0]
    for f in range(6):
        depth = DeviceMeshView(F, V.shape[0], cams[f].contiguous(), M, M, background_color=(mesh_ops.SHADOW_FAR,),
                               sigma=1.0, device=DEV, backface_culling=True, has_distortion=False)
        assert torch.equal(depth.render_depth(cuda(V))[..., 0], maps[f]), f
    assert float(maps.min()) > 0 and float((maps < 1e29).float().mean()) > 0.05


# ---------------------------------------------------------------------------------- 2. kernels vs the restatement

def _random_gbuffer(rng, lights, C, H=37, W=53):
    x = lights[rng.integers(0, len(lights), H * W), :3] + rng.normal(size=(H * W, 3)) * rng.uniform(0.5, 2.5, (H * W, 1))
    a = np.where(rng.random(H * W) < 0.15, 0.0, rng.uniform(0.3, 1.0, H * W))
    n = rng.normal(size=(H * W, 3))
    ch = np.concatenate((rng.uniform(0.2, 1, (H * W, C)), n, x * a[:, None], a[:, None]), axis=1)
    return ch.astype(np.float32).astype(np.float64), H, W


@pytest.mark.parametrize("L", [1, 2, 8])
@pytest.mark.parametrize("split", [False, True])
def test_visibility_kernels_match_the_restatement(L, split):
    rng = np.random.default_rng(L + 10 * split)
    C, M, bias, soft = 3, 32, 0.05, 0.8
    lights = np.concatenate((rng.uniform(-2, 2, (L, 3)), rng.uniform(0.5, 1, (L, 1))), axis=1)
    ch, H, W = _random_gbuffer(rng, lights, C)
    maps = rng.uniform(0.0, 3.0, (6 * L, M, M)).astype(np.float32)
    maps[rng.random(maps.shape) < 0.2] = ref.FAR
    if split:
        chd, kw = cuda(ch[:, C:].reshape(H, W, 7), torch.float32), dict(albedo=cuda(ch[:, :C].reshape(H, W, C),
                                                                                     torch.float32))
    else:
        chd, kw = cuda(ch.reshape(H, W, -1), torch.float32), {}
    pos, cov = ch[:, C + 3:C + 6], ch[:, C + 6]
    vis = mesh_ops.shadow_visibility(chd, cuda(lights), cuda(maps, torch.float32), bias, soft, **kw)
    want = ref.gbuffer_visibility(pos, cov, lights, maps.astype(np.float64), M, bias, soft)
    assert np.abs(host(vis).reshape(-1, L) - want).max() <= 1e-6
    assert np.all(host(vis).reshape(-1, L)[cov == 0] == 1.0)
    g = rng.normal(size=(H * W, L)).astype(np.float32)
    out = mesh_ops.shadow_visibility_backward(chd, cuda(lights), cuda(maps, torch.float32), bias, soft,
                                              cuda(g.reshape(H, W, L), torch.float32), new_scratch(DEV), **kw)
    pos_b, cov_b, maps_b, lights_b = ref.gbuffer_visibility_b(pos, cov, lights, maps.astype(np.float64), M, bias,
                                                              soft, g.astype(np.float64))
    got = host(out[0]).reshape(H * W, -1)
    off = 3 if split else C + 3
    assert np.all(np.abs(got[:, off:off + 3] - pos_b) <= 1e-5 * np.abs(pos_b).max() + 1e-6)
    assert np.all(np.abs(got[:, off + 3] - cov_b) <= 1e-5 * np.abs(cov_b).max() + 1e-6)
    assert np.all(got[:, :off] == 0)  # nothing but the position and coverage slices
    assert np.abs(host(out[1]) - maps_b).max() <= 1e-5 * np.abs(maps_b).max()
    assert rel(host(out[2])[:, :3], lights_b) <= 1e-9
    assert np.all(host(out[2])[:, 3:] == 0)


def _phong_inputs(C, L, split, seed=3, H=41, W=59):
    rng = np.random.default_rng(seed)
    cam = np.array([0.2, -0.1, -5.0])
    ch = phong_ref.random_pixels(rng, C, P=H * W, cam=cam).astype(np.float32).astype(np.float64)
    bg = cuda(rng.uniform(0, 1, C), torch.float32)
    lights = cuda(point_light_ref.random_lights(rng, L, 1, center=cam + [0, 0, 4.5], spread=2.0))
    params = cuda([0.3, -0.3, 0.6, 0.4, 0.7, 12.0])
    if split:
        kw = dict(albedo=cuda(ch[:, :C].reshape(H, W, C), torch.float32))
        chd = cuda(ch[:, C:].reshape(H, W, 7), torch.float32)
    else:
        kw, chd = {}, cuda(ch.reshape(H, W, -1), torch.float32)
    g = cuda(rng.normal(size=(H, W, C)), torch.float32)
    return chd, params, cuda(cam), bg, lights, g, kw, rng


@pytest.mark.parametrize("L", [1, 3])
@pytest.mark.parametrize("split", [False, True])
def test_shadowed_phong_kernels_at_full_visibility_are_the_unshadowed_ones(L, split):
    chd, params, cam, bg, lights, g, kw, _ = _phong_inputs(3, L, split)
    H, W = chd.shape[:2]
    ones = torch.ones((H, W, L), dtype=torch.float32, device=DEV)
    want = mesh_ops.phong_shade(chd, params, cam, bg, point_lights=lights, **kw)
    assert torch.equal(mesh_ops.phong_shade(chd, params, cam, bg, point_lights=lights, visibility=ones, **kw), want)
    scratch = new_scratch(DEV)
    want_b = mesh_ops.phong_shade_backward(chd, params, cam, bg, g, scratch, center_grad=True, point_lights=lights,
                                           **kw)
    got_b = mesh_ops.phong_shade_backward(chd, params, cam, bg, g, scratch, center_grad=True, point_lights=lights,
                                          visibility=ones, **kw)
    assert len(got_b) == len(want_b) + 1
    for a, b in zip(got_b, want_b):
        assert torch.equal(a, b)


@pytest.mark.parametrize("split", [False, True])
def test_shadowed_phong_is_affine_in_the_visibility_and_vis_b_is_its_slope(split):
    L = 2
    chd, params, cam, bg, lights, g, kw, rng = _phong_inputs(3, L, split, seed=5)
    H, W = chd.shape[:2]
    vis = cuda(rng.uniform(0, 1, (H, W, L)), torch.float32)
    out = mesh_ops.phong_shade_backward(chd, params, cam, bg, g, new_scratch(DEV), point_lights=lights,
                                        visibility=vis, **kw)
    vis_b = host(out[-1])
    for j in range(L):
        lo, hi = vis.clone(), vis.clone()
        lo[..., j], hi[..., j] = 0, 1
        i_lo = host(mesh_ops.phong_shade(chd, params, cam, bg, point_lights=lights, visibility=lo, **kw))
        i_hi = host(mesh_ops.phong_shade(chd, params, cam, bg, point_lights=lights, visibility=hi, **kw))
        i_v = host(mesh_ops.phong_shade(chd, params, cam, bg, point_lights=lights, visibility=vis, **kw))
        v = host(vis)[..., j:j + 1]
        assert np.abs(i_v - (i_lo + v * (i_hi - i_lo))).max() <= 1e-5 * max(1.0, np.abs(i_hi).max())
        slope = np.sum(host(g) * (i_hi - i_lo), axis=-1)
        assert np.abs(vis_b[..., j] - slope).max() <= 1e-4 * max(1.0, np.abs(slope).max())


# --------------------------------------------------------------------------------------------- 3. a known shadow

def _rays():
    r, c = np.meshgrid(np.arange(SIZE), np.arange(SIZE), indexing="ij")
    d = np.stack(((c - (SIZE - 1) / 2) / FOCAL, (r - (SIZE - 1) / 2) / FOCAL, np.ones_like(r, dtype=float)), -1)
    return d / np.linalg.norm(d, axis=-1, keepdims=True)


def _segment_sphere_distance(x, p):
    """The distance from the sphere's centre to the segments x [N,3] -> p."""
    seg = p[None] - x
    t = np.clip(np.sum((SPHERE_C - x) * seg, axis=1) / np.sum(seg * seg, axis=1), 0, 1)
    return np.linalg.norm(x + t[:, None] * seg - SPHERE_C, axis=1)


def test_a_sphere_casts_its_analytic_shadow_on_a_plane():
    M, band_texels = 512, 4
    lights = cuda(lights_of())
    view, V, colors = make_view(lights, M=M)
    view.render(cuda(V), cuda(colors))
    vis = host(view.shadow_visibility())[..., 0].reshape(-1)
    d = _rays().reshape(-1, 3)
    # plane pixels whose view ray passes well clear of the sphere (no mixed G-buffer positions at its silhouette)
    clear = np.linalg.norm(np.cross(d, SPHERE_C[None]), axis=1) > SPHERE_R + 4 * PLANE_Z / FOCAL
    x = d * (PLANE_Z / d[:, 2:3])
    inside = (np.abs(x[:, 0]) < 2.4) & (np.abs(x[:, 1]) < 2.4)
    keep = clear & inside
    texel = np.linalg.norm(SPHERE_C - LIGHT_P) * 2 / (M - 4)  # a map texel's width at the sphere
    dist = _segment_sphere_distance(x, LIGHT_P)
    shadowed, lit = keep & (dist < SPHERE_R - band_texels * texel), keep & (dist > SPHERE_R + band_texels * texel)
    bad_in = int(np.count_nonzero(vis[shadowed] != 0.0))
    bad_out = int(np.count_nonzero(vis[lit] != 1.0))
    record("shadow_known", {"band_texels": band_texels, "shadowed_pixels": int(shadowed.sum()),
                            "lit_pixels": int(lit.sum()), "disagree_in": bad_in, "disagree_out": bad_out})
    assert shadowed.sum() > 500 and lit.sum() > 10_000
    assert bad_in == 0 and bad_out == 0


# ------------------------------------------------------------------------------------------------------ 4. no acne

def test_a_lit_sphere_has_no_acne_and_renders_as_without_shadows():
    F, V = sphere(SPHERE_C, SPHERE_R, n=32)
    F = F.astype(np.int64)
    p = SPHERE_C + np.array([1.5, -1.0, -1.2])
    lights = cuda(np.concatenate((p, [2.0]))[None])
    view, _, colors = make_view(lights, M=512, bias=0.15, softness=0.1, faces=F, V=V)
    plain = make_view(lights, shadows=False, faces=F, V=V)[0]
    image = view.render(cuda(V), cuda(colors))
    vis = host(view.shadow_visibility())[..., 0].reshape(-1)
    d = _rays().reshape(-1, 3)
    # the first hit of each view ray on the ideal sphere, and its normal
    b = d @ SPHERE_C
    disc = b * b - (SPHERE_C @ SPHERE_C - SPHERE_R ** 2)
    hit = disc > (4 * np.linalg.norm(SPHERE_C) / FOCAL) ** 2  # clear of the silhouette
    x = d * (b - np.sqrt(np.maximum(disc, 0)))[:, None]
    n = (x - SPHERE_C) / SPHERE_R
    w = p[None] - x
    cos = np.sum(n * w, axis=1) / np.linalg.norm(w, axis=1)
    facing = hit & (cos > 0.1)
    record("shadow_acne", {"facing_pixels": int(facing.sum()), "below_one": int(np.count_nonzero(vis[facing] != 1))})
    assert facing.sum() > 2000 and np.all(vis[facing] == 1.0)
    assert np.all(host(view.shadow_visibility()) == 1.0)  # the sphere has no other occluder
    assert torch.equal(image, plain.render(cuda(V), cuda(colors)))


# -------------------------------------------------------------------------------- 5. gradients vs differences

def _loss(view, V, colors, w):
    return float((view.render(V, colors).double() * w).sum())


# A shadow edge moves with the light and with the occluder.  The lookup's own motion is exact (the bilinear taps), but
# the map's motion reaches the loss only through the maps' silhouette antialiasing, DEODR's approximation of a moving
# edge (the one the camera gradient also rests on), resampled by the 2x2 taps: the analytic gradient then holds to a
# few per cent of the central difference, not to rounding.  The step is 1e-3 of the light's distance to the sphere
# (about a fifth of a map texel at M = 512).  Measured on an H100: 3.4e-2 in the light's position (where the lookup's
# share dominates) and 9.9e-2 in the occluder's translation (the maps' share alone).
FD_STEP = 1e-3
FD_TOL_LIGHT = 0.05
FD_TOL_OCCLUDER = 0.15


def test_light_position_gradient_agrees_with_central_differences():
    ln = lights_of()
    lights = cuda(ln)
    view, V, colors = make_view(lights, M=512, bias=0.02, softness=0.2, sigma=2.0)
    Vd, cd = cuda(V), cuda(colors)
    image = view.render(Vd, cd)
    w = cuda(np.random.default_rng(4).uniform(0, 1, tuple(image.shape)))
    lb = host(view.backward(w.float())["point_lights_b"])[0, :3]
    h = FD_STEP * np.linalg.norm(LIGHT_P - SPHERE_C)
    flat = lights.view(-1)
    fd = []
    for k in range(3):
        base = float(flat[k])
        flat[k] = base + h
        lp = _loss(view, Vd, cd, w)
        flat[k] = base - h
        lm = _loss(view, Vd, cd, w)
        flat[k] = base
        fd.append((lp - lm) / (2 * h))
    err = rel(lb, fd)
    record("shadow_fd_light_position", {"analytic": lb.tolist(), "fd": fd, "rel_err": err})
    assert err <= FD_TOL_LIGHT


def test_occluder_translation_gradient_agrees_with_central_differences():
    lights = cuda(lights_of())
    view, V, colors = make_view(lights, M=512, bias=0.02, softness=0.2, sigma=2.0)
    _, _, ns = scene_mesh()
    cd = cuda(colors)
    image = view.render(cuda(V), cd)
    # weights on the plane's pixels only: the loss then sees the sphere through its shadow alone
    d = _rays().reshape(SIZE, SIZE, 3)
    off_sphere = np.linalg.norm(np.cross(d, SPHERE_C), axis=-1) > SPHERE_R + 4 * PLANE_Z / FOCAL
    wn = np.random.default_rng(5).uniform(0, 1, tuple(image.shape)) * off_sphere[..., None]
    w = cuda(wn)
    vb = host(view.backward(w.float())["vertices_b"])[:ns].sum(axis=0)
    h = FD_STEP * np.linalg.norm(LIGHT_P - SPHERE_C)
    fd = []
    for k in range(3):
        e = np.zeros(3)
        e[k] = h
        Vp, Vm = V.copy(), V.copy()
        Vp[:ns] += e
        Vm[:ns] -= e
        fd.append((_loss(view, cuda(Vp), cd, w) - _loss(view, cuda(Vm), cd, w)) / (2 * h))
    err = rel(vb, fd)
    record("shadow_fd_occluder_translation", {"analytic": vb.tolist(), "fd": fd, "rel_err": err})
    assert np.linalg.norm(fd) > 0
    assert err <= FD_TOL_OCCLUDER


# --------------------------------------------------------------------------------------------------- 6. PyTorch

def _scene(lights, M=256, camera_tensors=False):
    F, V, _ = scene_mesh()
    colors = np.random.default_rng(0).uniform(0.5, 1.0, (V.shape[0], 3))
    scene = P.Scene3DPytorch(shading="phong")
    vertices = cuda(V).requires_grad_(True)
    scene.set_mesh(P.ColoredTriMeshPytorch(F, vertices, colors=cuda(colors), device=DEV))
    scene.set_light(None, 0.05)
    scene.set_specular(0.3, 10.0)
    if lights is not None:
        scene.set_point_lights(lights, shadow_map_size=M, shadow_bias=0.02, shadow_softness=0.05)
    scene.set_background_color((0.1, 0.2, 0.3))
    cam = camera()
    extrinsic = None
    if camera_tensors:
        extrinsic = cuda(cam.extrinsic).requires_grad_(True)
        pc = P.CameraPytorch(extrinsic, cuda(cam.intrinsic), SIZE, SIZE)
    else:
        pc = P.CameraPytorch(cam.extrinsic, cam.intrinsic, SIZE, SIZE, cam.distortion)
    return scene, pc, vertices, extrinsic


def test_pytorch_gradients_equal_the_device_view():
    ln = lights_of()
    view, V, colors = make_view(cuda(ln), M=256)
    dimage = view.render(cuda(V), cuda(colors))
    image_b = cuda(np.random.default_rng(1).normal(size=tuple(dimage.shape)), torch.float32)
    out = view.backward(image_b)
    lights = cuda(ln).requires_grad_(True)
    scene, cam, vertices, _ = _scene(lights)
    image = scene.render(cam)
    assert torch.allclose(image, dimage, rtol=0, atol=1e-6)
    (image.double() * image_b.double()).sum().backward()
    assert rel(host(lights.grad), host(out["point_lights_b"])) <= 1e-4
    # the raster adjoints add with fp32 atomics whose order varies between the two runs
    assert rel(host(vertices.grad), host(out["vertices_b"])) <= 1e-3


def test_gouraud_views_and_views_without_point_lights_refuse_shadows():
    F, V, _ = scene_mesh()
    with pytest.raises(ValueError, match="smear"):
        DeviceMeshView(F, V.shape[0], camera(), 32, 32, device=DEV, point_lights=cuda(lights_of()),
                       shadow_map_size=64, shadow_bias=0.1, shadow_softness=0.1)
    with pytest.raises(ValueError, match="point lights"):
        DeviceMeshView(F, V.shape[0], camera(), 32, 32, device=DEV, shading="phong", shadow_map_size=64,
                       shadow_bias=0.1, shadow_softness=0.1)
    with pytest.raises(ValueError, match="both"):
        DeviceMeshView(F, V.shape[0], camera(), 32, 32, device=DEV, shading="phong", point_lights=cuda(lights_of()),
                       shadow_map_size=64, shadow_bias=0.1)
    scene = P.Scene3DPytorch(shading="gouraud")
    with pytest.raises(ValueError, match="smear"):
        scene.set_point_lights(cuda(lights_of()), shadow_map_size=64, shadow_bias=0.1, shadow_softness=0.1)


def test_a_flash_back_propagates_to_the_camera():
    intensity = cuda(np.array([[0.3]]))

    def run(detached):
        scene, cam, _, extrinsic = _scene(None, camera_tensors=True)
        center = cam.center()
        pos = center.detach().requires_grad_(True) if detached else center
        scene.set_point_lights(torch.cat((pos.reshape(1, 3) + cuda([0.3, -0.3, 0.0]), intensity), dim=1),
                               shadow_map_size=256, shadow_bias=0.02, shadow_softness=0.05)
        image = scene.render(cam)
        w = cuda(np.random.default_rng(6).uniform(0, 1, tuple(image.shape)), torch.float32)
        (image.double() * w.double()).sum().backward()
        return extrinsic, pos

    ext_a, _ = run(False)
    ext_b, pos_b = run(True)
    assert float(pos_b.grad.abs().max()) > 0
    e = ext_b.detach().requires_grad_(True)
    share = torch.autograd.grad(-(e[:, :3].T @ e[:, 3]), e, pos_b.grad)[0]
    assert rel(host(ext_a.grad), host(ext_b.grad + share)) <= 1e-3


# -------------------------------------------------------------------------------------------- 7. no host sync

def test_render_and_backward_make_no_host_sync():
    lights = cuda(lights_of())
    view, V, colors = make_view(lights, M=256)
    Vd, cd = cuda(V), cuda(colors)
    ones = torch.ones_like(view.render(Vd, cd))
    view.backward(ones)
    scene, cam, _, _ = _scene(lights)
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

FIT_STEPS = 300


def _fit(shadows, target, start):
    scene, cam, _, _ = _scene(None)
    x = cuda(start).requires_grad_(True)
    opt = torch.optim.Adam([x], lr=0.02)
    decay = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=1e-2 ** (1 / FIT_STEPS))
    I = cuda(lights_of()[:, 3:])
    for _ in range(FIT_STEPS):
        opt.zero_grad()
        lights = torch.cat((x[None], I), dim=1)
        if shadows:
            scene.set_point_lights(lights, shadow_map_size=256, shadow_bias=0.02, shadow_softness=0.1)
        else:
            scene.set_point_lights(lights)
        loss = ((scene.render(cam) - target).double() ** 2).sum()
        loss.backward()
        opt.step()
        decay.step()
    return host(x)


def test_adam_recovers_a_light_from_its_shadow():
    """The light 2.7 above the plane; the fit starts 20 % of that height sideways.  The same fit without shadows
    explains the target with the falloff alone."""
    scene, cam, _, _ = _scene(cuda(lights_of()))
    scene.set_point_lights(cuda(lights_of()), shadow_map_size=256, shadow_bias=0.02, shadow_softness=0.1)
    with torch.no_grad():
        target = scene.render(cam).clone()
    height = PLANE_Z - LIGHT_P[2]
    start = LIGHT_P + np.array([0.2 * height, 0.0, 0.0])
    got = _fit(True, target, start)
    plain = _fit(False, target, start)
    err, err_plain = (float(np.linalg.norm(g - LIGHT_P) / height) for g in (got, plain))
    record("shadow_fit", {"steps": FIT_STEPS, "start_error": 0.2, "error": err, "error_without_shadows": err_plain})
    assert err <= 0.02
