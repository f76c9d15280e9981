"""CPU: the kernel-path matrix of tests/path_matrix.py without a GPU.

  * the scene builder: every class of triangle is there, the scenes are in generic position, and the ballast that puts
    a picture on the path of a larger triangle count is invisible (checker outputs bit-identical, gradients equal);
  * coverage: the cases of tests/test_gpu_path_matrix.py reach every kernel instance the dispatch can select;
  * the matrix (C <= 16) through the CPU emulation of the kernel phases, set to the paths the device picks for each
    triangle count, against the checker with the GPU file's criteria: a phase bug fails here, a device-kernel bug only
    on the GPU.
"""
import numpy as np
import pytest
from canon import Emulator
from path_matrix import (ALL_INSTANCES, CHANNELS, COLOR_SLAB, REGIMES, SIZES, SMALL_FLAG, UNREACHABLE, VARIANTS,
                         all_cases, assert_generic, build_case_scene, case_instances, case_scenes, matrix_scene,
                         record_rows_for, small_textured_for, triangle_classes, with_ballast)
from test_gpu_parity import IMAGE_TOL, assert_gradient_close

from deodr_b200.scenes import dense_image_b

GRADS = ("ij_b", "colors_b", "uv_b", "shade_b", "texture_b")


@pytest.fixture(scope="module")
def emul():
    return Emulator()


@pytest.mark.parametrize("width,height", SIZES)
@pytest.mark.parametrize("textured", [False, True])
def test_scene_has_every_class_in_generic_position(width, height, textured, emul):
    for C, seed in ((1, 3), (3, 4), (16, 5)):
        scene = matrix_scene(width, height, C, seed, textured=textured)
        kinds = scene.extra["kinds"]
        cls = triangle_classes(scene)
        assert (cls[kinds == "small"] == "small").all() and (kinds == "small").sum() >= 400
        assert (cls[kinds == "medium"] == "medium").all() and (kinds == "medium").sum() >= 150
        assert (cls[kinds == "large"] == "large").all() and (kinds == "large").sum() >= 20
        assert sorted(cls[kinds == "clipped"]) == ["medium"] * 4 + ["small"] * 4
        # few triangles: medium ones go to the tile kernel by reference; textured ones stay off the small path
        few = triangle_classes(scene, record_rows=0, small_textured=False)
        assert (few[kinds == "medium"] == "large").all()
        assert not ((few == "small") & scene.textured).any()
        if textured:
            assert 0.3 < scene.textured.mean() < 0.5 and (scene.textured & (cls == "small")).sum() >= 100
        assert_generic(scene, emul)


@pytest.mark.parametrize("total", [REGIMES["records"], REGIMES["small-textured"]])
def test_ballast_is_invisible(total, checker):
    scene = matrix_scene(157, 93, 3, 9, textured=True)
    padded = with_ballast(scene, total, seed=1)
    assert padded.faces.shape[0] == total and not padded.edgeflags[scene.faces.shape[0]:].any()
    assert (triangle_classes(padded)[scene.faces.shape[0]:] == "off").all()
    image, z = checker.render(scene, 1.0)
    image_p, z_p = checker.render(padded, 1.0)
    assert np.array_equal(z, z_p) and np.array_equal(image, image_p)
    image_b = dense_image_b(image)
    ref = checker.render_b(scene, 1.0, image, z, image_b)
    got = checker.render_b(padded, 1.0, image_p, z_p, image_b)
    V = scene.ij.shape[0]
    for name in ("ij_b", "colors_b", "shade_b"):
        assert np.array_equal(got[name][:V], ref[name]), name
        assert not got[name][V:].any(), name
    for name in ("uv_b", "texture_b"):
        assert np.array_equal(got[name], ref[name]), name


def test_gpu_cases_reach_every_instance():
    """The union over the GPU file's cases of the instances they select is everything the dispatch can select: a new
    template instance or dispatch rule fails here until a case reaches it."""
    reached = set()
    for case in all_cases():
        got = case_instances(*case)
        assert got <= ALL_INSTANCES, (case, got - ALL_INSTANCES)
        reached |= got
    assert reached == set(ALL_INSTANCES), sorted(ALL_INSTANCES - reached, key=str)
    assert len(all_cases()) == len(REGIMES) * len(CHANNELS) * len(VARIANTS)
    assert UNREACHABLE  # the combinations left out say why


def emulated_case(emul, checker, scene, sigma, call):
    T = scene.faces.shape[0]
    emul.set_record_rows(record_rows_for(T))
    emul.set_small_textured(small_textured_for(T))
    try:
        rng = np.random.default_rng(scene.nb_colors)
        obs = rng.random((scene.height, scene.width, scene.nb_colors)).astype(np.float32).astype(np.float64)
        if call in ("error", "error_complete"):
            image, z, err = checker.render(scene, sigma, antialiase_error=True, obs=obs)
            fwd = emul.render_error(scene, sigma, obs)
            assert np.abs(fwd["err"] - err).max() <= 2e-6 * max(1.0, err.max())
        else:
            image, z = checker.render(scene, sigma)
            fwd = emul.render(scene, sigma)
        assert np.array_equal(fwd["z"], z), "z-buffer not bit-exact"
        assert np.abs(fwd["image"] - image).max() <= IMAGE_TOL
        assert np.array_equal(fwd["face_id"] >= 0, np.isfinite(z))
        owner = fwd["owner"]
        tri = np.where(owner >= 0, owner & ~SMALL_FLAG, 0)
        flagged = (owner >= 0) & scene.textured[tri] & ((owner & SMALL_FLAG) != 0)
        assert flagged.any() == (small_textured_for(T) and bool(scene.textured.any()))
        if call == "fwd+error":
            image, z, err = checker.render(scene, sigma, antialiase_error=True, obs=obs)
            e = emul.render_error(scene, sigma, obs)
            assert np.array_equal(e["z"], z) and np.abs(e["err"] - err).max() <= 2e-6 * max(1.0, err.max())
        if call in ("fwd", "fwd+error"):
            return
        if call in ("error", "error_complete"):
            err_b = (rng.random((scene.height, scene.width)) * 2 - 1).astype(np.float32).astype(np.float64)
            ref = checker.render_b(scene, sigma, image, z, None, antialiase_error=True, obs=obs, err_buffer=err,
                                   err_buffer_b=err_b)
            got = emul.render_error_b(scene, sigma, fwd, err_b, compat=True)
        else:
            image_b = dense_image_b(image).astype(np.float32).astype(np.float64)
            ref = checker.render_b(scene, sigma, image, z, image_b)
            got = emul.render_b(scene, sigma, fwd, image_b)
        for name in GRADS:
            if ref[name].size:
                assert_gradient_close(got[name].astype(np.float64), ref[name], name)
    finally:
        emul.set_record_rows(16)
        emul.set_small_textured(True)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("C", [c for c in CHANNELS if c <= COLOR_SLAB])
@pytest.mark.parametrize("regime", list(REGIMES))
def test_path_matrix_through_the_emulation(regime, C, variant, emul, checker):
    for width, height, textured in case_scenes(regime, C, variant):
        scene, sigma, call = build_case_scene(regime, C, variant, width, height, textured)
        emulated_case(emul, checker, scene, sigma, call)
