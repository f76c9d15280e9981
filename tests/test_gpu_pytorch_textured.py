"""GPU: textured renders under torch autograd.

2D Functions (``CudaDifferentiableRender2DTextured``, ``CudaRenderCompare2DTextured``) on the small textured torus and
the duck's 2D scene:
* the image is bit-identical to ``Renderer.render`` on the same ``DeviceScene``;
* the five gradients meet the project's gradient criterion (tests/test_gpu_parity.py) against ``Renderer.render_b`` and
  against the checker oracle (summed texture adjoint), in both compare modes;
* central differences: texture and shade everywhere (the image is linear in them), ij and uv on pixels at least two
  pixels away from any change of face;
* the texture gradient asked for alone is that of the five asked for together; fp64 leaves get fp64 gradients; two
  forwards then two backwards give the gradients of isolated calls; no torch synchronisation; shape refusals.

Textured ``Scene3DPytorch`` on the duck: the image is ``DeviceMeshView``'s bit for bit and the reference's duck.png;
``loss.backward()`` gives ``DeviceMeshView.backward``'s gradients; the luminosity passes gradcheck; Adam on texture and
light lowers a loss; replay; partial meshes and mismatched backgrounds are refused.
"""
import numpy as np
import pytest
from conftest import load_small
from test_gpu_parity import assert_gradient_close
from textured_ref import duck, textured_scene

from deodr_b200.scenes import dense_image_b

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

DEV = "cuda:0"
NAMES = ("ij", "colors", "uv", "shade", "texture")


@pytest.fixture(scope="module")
def P(build_native):
    import deodr_b200.pytorch as P

    return P


def torus():
    scene, _ = load_small("torus_tex")
    scene.uv = scene.uv * 0.9973 + 0.0131  # off the texel grid (the bilinear adjoint is discontinuous on it)
    return scene


def duck2d():
    d = duck()
    return textured_scene(d["faces"], d["faces_uv"], d["uv"], d["texture"], d["s2_ij"], d["s2_depths"],
                          d["luminosity"], d["s2_edgeflags"], 240, 320, d["background_color"])


SCENES = {"torus": torus, "duck": duck2d}


def leaves(scene, dtype=None, grad=True, only=None):
    """The five inputs as CUDA leaves: ij / uv fp64, colors / shade / texture fp32 (or all ``dtype``)."""
    out = []
    for name in NAMES:
        dt = dtype or (torch.float64 if name in ("ij", "uv") else torch.float32)
        t = torch.tensor(np.asarray(getattr(scene, name), dtype=np.float64), dtype=dt, device=DEV)
        out.append(t.requires_grad_(grad and (only is None or name in only)))
    return out


def host(t):
    return t.detach().cpu().numpy().astype(np.float64)


def device_scene(scene):
    from deodr_b200.renderer import DeviceScene

    return DeviceScene(scene, DEV)


# ---- 2D Functions -------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("which", SCENES)
def test_image_and_gradients_match_the_renderer(which, P):
    from deodr_b200.renderer import default_renderer

    scene = SCENES[which]()
    ds = device_scene(scene)
    x = leaves(scene)
    image = P.CudaDifferentiableRender2DTextured(*x, ds, 1.0)
    image_b = torch.from_numpy(dense_image_b(host(image)).astype(np.float32)).to(DEV)
    (image * image_b).sum().backward()
    renderer = default_renderer(0)
    fwd = renderer.render(ds, 1.0)
    assert torch.equal(image, fwd["image"])
    ref = renderer.render_b(ds, 1.0, fwd, image_b)
    for name, t in zip(NAMES, x):
        assert t.grad.dtype == t.dtype
        assert_gradient_close(host(t.grad), host(ref[name + "_b"]), name)
    assert np.abs(host(x[3].grad)).max() > 0 and np.abs(host(x[4].grad)).max() > 0


@pytest.mark.parametrize("which", SCENES)
@pytest.mark.parametrize("antialiase_error", [False, True])
def test_compare_gradients_match_the_checker(which, antialiase_error, P, checker):
    scene = SCENES[which]()
    ds = device_scene(scene)
    rng = np.random.default_rng(7)
    obs = rng.random((scene.height, scene.width, scene.nb_colors))
    mask = rng.random((scene.height, scene.width))
    x = leaves(scene)
    loss = P.CudaRenderCompare2DTextured(*x, torch.tensor(obs, dtype=torch.float32, device=DEV),
                                         torch.tensor(mask, dtype=torch.float32, device=DEV), ds, 1.0, antialiase_error)
    assert loss.dtype == torch.float64 and loss.dim() == 0
    (2.5 * loss).backward()
    if antialiase_error:
        image, z, err = checker.render(scene, 1.0, antialiase_error=True, obs=obs)
        ref_loss = float((mask * err).sum())
        ref = checker.render_b(scene, 1.0, image, z, None, antialiase_error=True, obs=obs, err_buffer=err,
                               err_buffer_b=mask)
    else:
        image, z = checker.render(scene, 1.0)
        d = (image - obs) * mask[:, :, None]
        ref_loss = float((d * (image - obs)).sum())
        ref = checker.render_b(scene, 1.0, image, z, 2 * d)
    assert abs(loss.item() - ref_loss) <= 1e-5 * ref_loss
    for name, t in zip(NAMES, x):
        assert_gradient_close(host(t.grad), 2.5 * ref[name + "_b"], name)


def _weighted_loss(P, ds, x, w):
    return float((P.CudaDifferentiableRender2DTextured(*x, ds, 1.0).double() * w).sum())


def _interior_weights(scene, rng):
    """Random weights on the pixels whose 3 x 3 neighbourhood lies in one face (their centre is at least a pixel inside
    it, so a small move of a vertex changes no coverage), zero elsewhere."""
    from deodr_b200.renderer import default_renderer

    fid = default_renderer(0).render(device_scene(scene), 1.0, face_id=True)["face_id"].cpu().numpy()
    H, W = fid.shape
    pad = np.pad(fid, 1, constant_values=-2)
    interior = fid >= 0
    for dy in range(3):
        for dx in range(3):
            interior &= pad[dy:dy + H, dx:dx + W] == fid
    assert interior.sum() > 500
    return torch.tensor(rng.normal(size=(H, W, scene.nb_colors)) * interior[:, :, None], device=DEV)


@pytest.mark.parametrize("names", [("texture", "shade"), ("ij", "uv")])
def test_central_differences(names, P):
    """texture and shade on the torus: the image is linear in them, so central differences are exact up to the fp32
    image.  ij and uv on the eigen-faces grid (large triangles, a smooth texture), with a loss on pixels away from any
    change of face: there the image is smooth in them but at the kinks of the bilinear sample."""
    import eigen_faces_ref as ef

    rng = np.random.default_rng(8)
    if names == ("texture", "shade"):
        scene = torus()
        w = torch.tensor(rng.normal(size=(scene.height, scene.width, 3)), device=DEV)
        h, rtol = 0.25, 1e-4
    else:
        d = ef.load_inputs()
        scene = ef.scene_of(d, d["points_deformed"], d["texture_gt"])
        w = _interior_weights(scene, rng)
        h, rtol = 1e-3, 1e-2
    ds = device_scene(scene)
    x = leaves(scene, dtype=torch.float64)
    (P.CudaDifferentiableRender2DTextured(*x, ds, 1.0).double() * w).sum().backward()
    for name in names:
        i = NAMES.index(name)
        g = host(x[i].grad)
        assert np.abs(g).max() > 0, name
        for flat in np.argsort(-np.abs(g).ravel())[:5]:
            idx = np.unravel_index(flat, g.shape)
            xp = [t.detach().clone() for t in x]
            xm = [t.detach().clone() for t in x]
            xp[i][idx] += h
            xm[i][idx] -= h
            fd = (_weighted_loss(P, ds, xp, w) - _weighted_loss(P, ds, xm, w)) / (2 * h)
            assert abs(fd - g[idx]) <= rtol * abs(g[idx]) + 1e-4 * np.abs(g).max(), (name, idx, fd, g[idx])


@pytest.mark.parametrize("which", SCENES)
def test_texture_gradient_alone_is_that_of_all_five(which, P):
    scene = SCENES[which]()
    ds = device_scene(scene)
    image_b = torch.tensor(dense_image_b(np.zeros((scene.height, scene.width, scene.nb_colors))), device=DEV)
    x = leaves(scene)
    (P.CudaDifferentiableRender2DTextured(*x, ds, 1.0) * image_b).sum().backward()
    y = leaves(scene, only=("texture",))
    (P.CudaDifferentiableRender2DTextured(*y, ds, 1.0) * image_b).sum().backward()
    assert all(t.grad is None for t in y[:4])
    assert_gradient_close(host(y[4].grad), host(x[4].grad), "texture alone")


def test_two_forwards_then_two_backwards(P):
    scene = duck2d()
    ds = device_scene(scene)
    rng = np.random.default_rng(9)
    weights = [torch.tensor(rng.normal(size=(240, 320, 3)), device=DEV) for _ in range(2)]
    shifts = [0.0, 1.5]

    def inputs(shift):
        x = leaves(scene)
        with torch.no_grad():
            x[0] += shift
        return x

    isolated = []
    for s, w in zip(shifts, weights):
        x = inputs(s)
        (P.CudaDifferentiableRender2DTextured(*x, ds, 1.0) * w).sum().backward()
        isolated.append([host(t.grad) for t in x])
    xs = [inputs(s) for s in shifts]
    losses = [(P.CudaDifferentiableRender2DTextured(*x, ds, 1.0) * w).sum() for x, w in zip(xs, weights)]
    losses[0].backward()  # replays the first render, on its own inputs
    losses[1].backward()
    for x, ref in zip(xs, isolated):
        for name, t, r in zip(NAMES, x, ref):
            assert_gradient_close(host(t.grad), r, name)
    # the same for the comparison
    obs = torch.rand((240, 320, 3), device=DEV)
    ref = []
    for s in shifts:
        x = inputs(s)
        P.CudaRenderCompare2DTextured(*x, obs, None, ds, 1.0).backward()
        ref.append([host(t.grad) for t in x])
    xs = [inputs(s) for s in shifts]
    losses = [P.CudaRenderCompare2DTextured(*x, obs, None, ds, 1.0) for x in xs]
    losses[0].backward()
    losses[1].backward()
    for x, r in zip(xs, ref):
        for name, t, g in zip(NAMES, x, r):
            assert_gradient_close(host(t.grad), g, "compare " + name)


def test_fp64_leaves_get_fp64_gradients(P):
    scene = torus()
    ds = device_scene(scene)
    x = leaves(scene, dtype=torch.float64)
    P.CudaDifferentiableRender2DTextured(*x, ds, 1.0).sum().backward()
    assert all(t.grad.dtype == torch.float64 for t in x)
    y = leaves(scene, dtype=torch.float64)
    P.CudaRenderCompare2DTextured(*y, torch.rand((40, 48, 3), device=DEV), None, ds, 1.0).backward()
    assert all(t.grad.dtype == torch.float64 for t in y)


def test_no_torch_synchronisation(P):
    scene = duck2d()
    ds = device_scene(scene)
    obs = torch.rand((240, 320, 3), device=DEV)
    mask = torch.rand((240, 320), device=DEV)
    w = torch.ones((240, 320, 3), device=DEV)
    base = leaves(scene, grad=False)  # uploaded here: a host-to-device copy synchronises

    def fresh():
        return [t.clone().requires_grad_(True) for t in base]

    def once():
        x = fresh()
        (P.CudaDifferentiableRender2DTextured(*x, ds, 1.0) * w).sum().backward()
        y = fresh()
        P.CudaRenderCompare2DTextured(*y, obs, mask, ds, 1.0).backward()
        z = fresh()
        P.CudaRenderCompare2DTextured(*z, obs, mask, ds, 1.0, True).backward()

    once()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(2):
            once()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_shapes_are_checked_before_any_launch(P):
    scene = torus()
    ds = device_scene(scene)
    obs = torch.rand((40, 48, 3), device=DEV)
    for i, name in enumerate(NAMES):
        x = leaves(scene, grad=False)
        x[i] = x[i][:-1]
        with pytest.raises(ValueError, match=name):
            P.CudaDifferentiableRender2DTextured(*x, ds, 1.0)
        with pytest.raises(ValueError, match=name):
            P.CudaRenderCompare2DTextured(*x, obs, None, ds, 1.0)
    x = leaves(scene, grad=False)
    x[4] = x[4].cpu()
    with pytest.raises(ValueError, match="CUDA"):
        P.CudaDifferentiableRender2DTextured(*x, ds, 1.0)


# ---- textured Scene3DPytorch ----------------------------------------------------------------------------------------


def duck_setup(P, W=320, H=240, texture=None, light=None, grad=True):
    from deodr_b200.mesh_ops import CameraParams, DeviceMeshView

    d = duck()
    cam = CameraParams(d[f"extrinsic_{W}"], d[f"intrinsic_{W}"], d["distortion"])
    view = DeviceMeshView(d["faces"], d["vertices"].shape[0], cam, H, W, light_directional=d["light_directional"],
                          ambient=float(d["light_ambient"]), background_color=d["background_color"], uv=d["uv"],
                          faces_uv=d["faces_uv"], texture=d["texture"], device=DEV)
    camera = P.CameraPytorch(d[f"extrinsic_{W}"], d[f"intrinsic_{W}"], H, W, d["distortion"])
    t = lambda a: torch.tensor(np.asarray(a, dtype=np.float64), device=DEV).requires_grad_(grad)  # noqa: E731
    mesh = P.ColoredTriMeshPytorch(d["faces"], t(d["vertices"]), faces_uv=d["faces_uv"], uv=t(d["uv"]),
                                   texture=t(d["texture"] if texture is None else texture))
    scene = P.Scene3DPytorch()
    scene.set_mesh(mesh)
    ld = t(d["light_directional"] if light is None else light[:3])
    amb = t(d["light_ambient"] if light is None else light[3])
    scene.set_light(ld, amb)
    scene.set_background_color(d["background_color"])
    return d, view, camera, mesh, scene, ld, amb


def test_duck_image_is_the_device_views_and_duck_png(P):
    d, view, camera, mesh, scene, ld, amb = duck_setup(P)
    image = scene.render(camera)
    ref = view.render(torch.tensor(d["vertices"], device=DEV))
    assert image.dtype == torch.float32 and torch.equal(image, ref)
    got = (image.detach().cpu().numpy() * 255).astype(np.uint8)
    assert not np.any(got != d["duck_png"])


def test_duck_gradients_match_the_device_view(P):
    d, view, camera, mesh, scene, ld, amb = duck_setup(P)
    image = scene.render(camera)
    image_b = torch.tensor(dense_image_b(host(image)), dtype=torch.float32, device=DEV)
    (image * image_b).sum().backward()
    view.render(torch.tensor(d["vertices"], device=DEV))
    ref = view.backward(image_b)
    assert_gradient_close(host(mesh.vertices.grad), host(ref["vertices_b"]), "vertices")
    assert_gradient_close(host(mesh.texture.grad), host(ref["texture_b"]), "texture")
    assert_gradient_close(host(mesh.uv.grad), host(ref["uv_b"]), "uv")
    light_b = np.concatenate((host(ld.grad), host(amb.grad).reshape(1)))
    want = host(ref["light_b"])
    assert np.abs(light_b - want).max() <= 1e-5 * np.abs(want).max(), (light_b, want)


def test_gradcheck_luminosity(P):
    from deodr_b200.pytorch.scene3d_pytorch import vertex_luminosity_autograd

    rng = np.random.default_rng(10)
    n = rng.normal(size=(9, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    t = lambda a: torch.tensor(a, dtype=torch.float64, device=DEV, requires_grad=True)  # noqa: E731
    args = (t(n), t(rng.normal(size=3)), t(np.array(0.3)))
    assert torch.autograd.gradcheck(vertex_luminosity_autograd, args, eps=1e-6, atol=1e-6)
    assert torch.autograd.gradcheck(lambda a, b: vertex_luminosity_autograd(a, None, b), (args[0], args[2]),
                                    eps=1e-6, atol=1e-6)


def test_adam_on_texture_and_light_lowers_the_loss(P):
    d, view, camera, mesh, scene, ld, amb = duck_setup(P, grad=False)
    with torch.no_grad():
        target = scene.render(camera)
    texture = torch.full(d["texture"].shape, 0.5, dtype=torch.float64, device=DEV, requires_grad=True)
    light = torch.tensor([0.2, -0.1, 0.1, 0.3], dtype=torch.float64, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([texture, light], lr=2e-2)
    losses = []
    for _ in range(10):
        opt.zero_grad()
        mesh.texture = texture
        scene.set_light(light[:3], light[3])
        loss = ((scene.render(camera) - target) ** 2).sum()
        loss.backward()
        assert texture.grad is not None and light.grad is not None
        losses.append(float(loss))
        opt.step()
    assert losses[-1] < 0.8 * losses[0], losses


def test_two_textured_renders_then_two_backwards(P):
    d, view, camera, mesh, scene, ld, amb = duck_setup(P, grad=False)
    rng = np.random.default_rng(11)
    weights = [torch.tensor(rng.normal(size=(240, 320, 3)), device=DEV) for _ in range(2)]
    poses = [d["vertices"], d["vertices"] + 0.01 * rng.normal(size=d["vertices"].shape)]

    def loss_of(v, w):
        mesh.set_vertices(v)
        return (scene.render(camera) * w).sum()

    isolated = []
    for p, w in zip(poses, weights):
        v = torch.tensor(p, device=DEV, requires_grad=True)
        loss_of(v, w).backward()
        isolated.append(host(v.grad))
    vs = [torch.tensor(p, device=DEV, requires_grad=True) for p in poses]
    losses = [loss_of(v, w) for v, w in zip(vs, weights)]
    losses[0].backward()
    losses[1].backward()
    for v, ref in zip(vs, isolated):
        assert_gradient_close(host(v.grad), ref, "vertices")


def test_render_depth_of_a_textured_mesh_is_the_untextured_one(P):
    d, view, camera, mesh, scene, ld, amb = duck_setup(P, grad=False)
    plain = P.ColoredTriMeshPytorch(d["faces"], torch.tensor(d["vertices"], device=DEV))
    other = P.Scene3DPytorch()
    other.set_mesh(plain)
    scene.set_background_color([1.0])
    other.set_background_color([1.0])
    assert torch.equal(scene.render_depth(camera, 0.3), other.render_depth(camera, 0.3))


def test_refusals(P):
    d = duck()
    v = torch.tensor(d["vertices"], device=DEV)
    for kw in ({"uv": d["uv"]}, {"texture": d["texture"]}, {"faces_uv": d["faces_uv"], "uv": d["uv"]},
               {"faces_uv": d["faces_uv"], "texture": d["texture"]}):
        with pytest.raises(ValueError, match="together"):
            P.ColoredTriMeshPytorch(d["faces"], v, **kw)
    d, view, camera, mesh, scene, ld, amb = duck_setup(P, grad=False)
    scene.set_background_color([0.0, 0.0])
    with pytest.raises(ValueError, match="background colour"):
        scene.render(camera)
    untextured = P.ColoredTriMeshPytorch(d["faces"], v)
    scene.set_mesh(untextured)
    with pytest.raises(ValueError, match="vertex colours"):
        scene.render(camera)
