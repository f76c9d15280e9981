"""GPU (-m gpu): every kernel instance the device rasteriser can dispatch, on each of its size-chosen paths, against the
checker (the compiled reference, tests/conftest.py) - the matrix of tests/path_matrix.py: regime (few / records /
small-textured triangle counts) x C (1, 2, 3, 4, 7, 16, 17) x variant (flags, sigma, background gradient, error mode).

Criteria (those of tests/test_gpu_parity.py): z-buffer bit-exact, face id >= 0 exactly where z is finite, image within
1e-6, err_buffer within 2e-6 * max(1, max err), the five gradients within the three-part criterion of
assert_gradient_close, background gradients against the exact oracle of tests/test_background_grad.py.  The complete
error adjoint (no reference to compare with) is held to the CPU emulation of the kernel phases, and on one small scene
per channel instance to central differences of the checker's error-mode forward.

Proof of the path: owner codes equal those of the emulation set to the device's choices for the scene's triangle count;
textured pixels carry SMALL_FLAG at the small-textured triangle count and never below it.  (The record path of the
medium triangles leaves their owner codes as they are: that regime is set by the triangle count alone.)

Measured on an H100 SXM: the whole file in under 3 minutes, most of it in the CPU checker.
"""
import copy

import numpy as np
import pytest
from canon import Emulator
from path_matrix import (CHANNELS, COLOR_SLAB, REGIMES, SMALL_FLAG, VARIANTS, build_case_scene, case_scenes,
                         matrix_scene, record_rows_for, small_textured_for, with_ballast)
from test_background_grad import expected_background_grads, weight_map
from test_gpu_parity import IMAGE_TOL, assert_gradient_close
from test_gpu_tilez_warp_test import same_owners

from deodr_b200.scenes import dense_image_b

pytestmark = pytest.mark.gpu

GRADS = ("ij_b", "colors_b", "uv_b", "shade_b", "texture_b")


@pytest.fixture(scope="module")
def gpu(build_native):
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from deodr_b200.renderer import Renderer

    return Renderer(0)


@pytest.fixture(scope="module")
def emul():
    return Emulator()


def cuda(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def host(d):
    return {k: v.cpu().numpy() for k, v in d.items() if hasattr(v, "cpu")}


def emulate(emul, scene, sigma, obs=None):
    """The emulated forward with the device's size-chosen paths (owner codes depend on the geometry alone: a scene
    wider than the emulation's 16 channels is emulated on its first channel)."""
    T = scene.faces.shape[0]
    emul.set_record_rows(record_rows_for(T))
    emul.set_small_textured(small_textured_for(T))
    if scene.nb_colors > COLOR_SLAB:
        scene = copy.copy(scene)
        scene.nb_colors, scene.colors = 1, np.ascontiguousarray(scene.colors[:, :1])
        scene.texture = np.ascontiguousarray(scene.texture[:, :, :1])
        if scene.background_image is not None:
            scene.background_image = np.ascontiguousarray(scene.background_image[:, :, :1])
        else:
            scene.background_color = scene.background_color[:1]
    return emul.render(scene, sigma) if obs is None else emul.render_error(scene, sigma, obs)


def assert_path(got, ref, scene):
    """Owner codes of the emulation; SMALL_FLAG on textured pixels exactly at the small-textured triangle count."""
    same_owners(got, ref)
    owner = got["owner"]
    drawn = owner >= 0
    tri = np.where(drawn, owner & ~SMALL_FLAG, 0)
    tex_px = drawn & scene.textured[tri] & scene.shaded[tri]
    flagged = tex_px & ((owner & SMALL_FLAG) != 0)
    if small_textured_for(scene.faces.shape[0]):
        assert flagged.any() or not tex_px.any(), "no textured small triangle took the triangle-parallel adjoint"
    else:
        assert not flagged.any(), "a textured triangle took the triangle-parallel adjoint below the threshold"


def check_forward(gpu, checker, emul, scene, sigma, obs=None):
    from deodr_b200.renderer import DeviceScene

    ds = DeviceScene(scene, "cuda:0")
    if obs is None:
        image, z = checker.render(scene, sigma)
        err = None
    else:
        image, z, err = checker.render(scene, sigma, antialiase_error=True, obs=obs)
    fwd = gpu.render(ds, sigma, face_id=True, obs=cuda(obs) if obs is not None else None)
    got = host(fwd)
    assert np.array_equal(got["z_buffer"], z), "z-buffer not bit-exact"
    assert np.abs(got["image"] - image).max() <= IMAGE_TOL
    assert np.array_equal(got["face_id"] >= 0, np.isfinite(z))
    if obs is not None:
        assert np.abs(got["err_buffer"] - err).max() <= 2e-6 * max(1.0, err.max())
    ref = emulate(emul, scene, sigma, obs)
    assert np.array_equal(ref["z"], z)
    assert_path(got, ref, scene)
    return ds, fwd, image, z, err, ref


def run_scene(gpu, checker, emul, scene, sigma, call):
    from deodr_b200 import _cabi
    from deodr_b200.renderer import DeviceScene

    C = scene.nb_colors
    rng = np.random.default_rng(C)
    obs = rng.random((scene.height, scene.width, C)).astype(np.float32).astype(np.float64)
    if call in ("error", "error_complete") and C > COLOR_SLAB:
        with pytest.raises(_cabi.DeodrB200Error, match="at most 16 colour channels"):
            gpu.render(DeviceScene(scene, "cuda:0"), sigma, obs=cuda(obs))
        return
    if call in ("fwd", "fwd+error", "bwd", "bg"):
        ds, fwd, image, z, _, _ = check_forward(gpu, checker, emul, scene, sigma)
        if call == "fwd+error" and C <= COLOR_SLAB:
            check_forward(gpu, checker, emul, scene, sigma, obs)
        if call in ("fwd", "fwd+error"):
            return
        image_b = dense_image_b(image).astype(np.float32).astype(np.float64)
        bg = ds.zero_background_grads() if call == "bg" else None
        grads = host(gpu.render_b(ds, sigma, fwd, cuda(image_b), background_grads=bg))
        ref = checker.render_b(scene, sigma, image, z, image_b)
        for name in GRADS:
            if ref[name].size:
                assert_gradient_close(grads[name], ref[name], name)
        if bg is not None:
            expected = expected_background_grads(weight_map(checker, scene, sigma), image_b)
            assert_gradient_close(bg["background_image_b"].cpu().numpy(), expected[0], "background_image_b")
        return
    complete = call == "error_complete"
    ds, fwd, image, z, err, emu_fwd = check_forward(gpu, checker, emul, scene, sigma, obs)
    err_b = (rng.random((scene.height, scene.width)) * 2 - 1).astype(np.float32).astype(np.float64)
    bg = ds.zero_background_grads() if complete else None
    grads = host(gpu.render_b(ds, sigma, fwd, err_buffer_b=cuda(err_b), error_adjoint_complete=complete,
                              background_grads=bg))
    if complete:  # the reference has no complete adjoint: the emulated phases are the yardstick
        ref = emul.render_error_b(scene, sigma, emu_fwd, err_b, compat=False)
    else:
        ref = checker.render_b(scene, sigma, image, z, None, antialiase_error=True, obs=obs, err_buffer=err,
                               err_buffer_b=err_b)
    for name in GRADS:
        if ref[name].size:
            assert_gradient_close(grads[name], ref[name].astype(np.float64), name)
    if bg is not None:
        expected = expected_background_grads(weight_map(checker, scene, sigma), err_b=err_b, image=image, obs=obs)
        assert_gradient_close(bg["background_color_b"].cpu().numpy(), expected[1], "error-mode background_color_b")


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("C", CHANNELS)
@pytest.mark.parametrize("regime", list(REGIMES))
def test_path_matrix(regime, C, variant, gpu, checker, emul):
    for width, height, textured in case_scenes(regime, C, variant):
        scene, sigma, call = build_case_scene(regime, C, variant, width, height, textured)
        run_scene(gpu, checker, emul, scene, sigma, call)


@pytest.mark.parametrize("C", [1, 2, 3, 7])
def test_complete_error_adjoint_matches_finite_differences(C, gpu, checker):
    """One small scene per channel instance (MAXC 1, 4, 3, 16): the complete error adjoint's colour gradient against
    central differences of the checker's error-mode forward (sum of err_buffer * weights as the scalar), at 40
    vertex channels drawn among those with the largest gradients and at random."""
    from deodr_b200.renderer import DeviceScene

    scene = matrix_scene(64, 48, C, seed=40 + C)
    rng = np.random.default_rng(C)
    obs = rng.random((48, 64, C)).astype(np.float32).astype(np.float64)
    weights = rng.random((48, 64)).astype(np.float32).astype(np.float64)
    ds = DeviceScene(scene, "cuda:0")
    fwd = gpu.render(ds, 1.0, obs=cuda(obs))
    colors_b = gpu.render_b(ds, 1.0, fwd, err_buffer_b=cuda(weights), error_adjoint_complete=True)["colors_b"]
    colors_b = colors_b.cpu().numpy()
    flat = np.argsort(-np.abs(colors_b).ravel())
    picks = np.concatenate((flat[:25], rng.choice(flat.size, 15, replace=False)))
    base = scene.colors.copy()

    def loss(colors):
        scene.colors = colors
        return float(np.sum(checker.render(scene, 1.0, antialiase_error=True, obs=obs)[2] * weights))

    eps, worst = 1e-5, 0.0
    for p in picks:
        v, c = divmod(int(p), C)
        hi, lo = base.copy(), base.copy()
        hi[v, c] += eps
        lo[v, c] -= eps
        worst = max(worst, abs((loss(hi) - loss(lo)) / (2 * eps) - colors_b[v, c]))
    scene.colors = base
    assert worst <= 2e-3 * np.abs(colors_b).max() + 1e-4, worst


def test_mixed_regime_batch(gpu, checker):
    """One render_views / render_b_views batch of a view per regime and C in {1, 3, 7}: z-buffer and image identical
    to the single-view calls, gradients within the criterion against the checker."""
    from deodr_b200.renderer import DeviceScene

    scenes = []
    for i, regime in enumerate(REGIMES):
        for j, C in enumerate((1, 3, 7)):
            base = matrix_scene(*((157, 93) if (i + j) % 2 else (160, 96)), C, seed=70 + 3 * i + j,
                                textured=(i + j) % 2 == 0)
            scenes.append(base if REGIMES[regime] is None else with_ballast(base, REGIMES[regime], seed=i))
    dss = [DeviceScene(s, "cuda:0") for s in scenes]
    alone = [host(gpu.render(ds, 1.0)) for ds in dss]
    fwds = gpu.render_views(dss, 1.0)
    refs = [checker.render(s, 1.0) for s in scenes]
    image_bs = [dense_image_b(image, seed=k).astype(np.float32).astype(np.float64) for k, (image, _) in enumerate(refs)]
    grads = gpu.render_b_views(dss, 1.0, fwds, [cuda(b) for b in image_bs])
    for k, (s, fwd, a, g, (image, z)) in enumerate(zip(scenes, fwds, alone, grads, refs)):
        f = host(fwd)
        assert np.array_equal(f["z_buffer"], a["z_buffer"]) and np.array_equal(f["image"], a["image"]), k
        assert np.array_equal(f["z_buffer"], z), k
        ref = checker.render_b(s, 1.0, image, z, image_bs[k])
        g = host(g)
        for name in GRADS:
            if ref[name].size:
                assert_gradient_close(g[name], ref[name], f"view {k} {name}")
