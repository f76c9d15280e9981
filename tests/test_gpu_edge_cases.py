"""GPU (-m gpu): the rasteriser on the device at the edges of its input domain, where the CPU emulation of the kernel
phases (tests/test_emul.py, scripts/probe_edge_cases.py) cannot stand in for it: the launch geometry of thin and
huge images, partial tiles through the TMA tile store / loads and through the plain-load fall-back, edge bands from
a thousandth of a pixel to wider than the scene, non-finite and degenerate inputs (the device's double -> int
conversions are not the host's), vertices far beyond the reference's `short` range, tiny textures.

Criteria (those of tests/test_gpu_parity.py, with NaN counted as equal to NaN):
  z-buffer   bit-exact                 face id   >= 0 exactly where z is finite
  image      |err| <= 1e-6 on the non-NaN pixels, the same NaN pattern
  gradients  the three-part criterion on the finite entries, the same finite / non-finite pattern as the checker
The checker is the reference (or its C restatement) with the summed texture adjoint.  Where the documented behaviour
IS a deviation from the reference (vertices beyond +-32767 px in the default build, INTEGRATION.md section 5), the
device is held to the CPU emulation of the same build instead, face ids included."""
import copy

import numpy as np
import pytest
from canon import Emulator
from test_emul import far_vertex_scene
from test_gpu_parity import IMAGE_TOL, assert_gradient_close, run_device

from deodr_b200.scenes import confetti_scene, dense_image_b, soup_scene, torus_scene

pytestmark = pytest.mark.gpu

GRADS = ("ij_b", "colors_b", "uv_b", "shade_b", "texture_b")


@pytest.fixture(scope="module")
def gpu(build_native):
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from deodr_b200.renderer import Renderer

    return Renderer(0)


def exact_wrap_build():
    """Is the loaded library the DEODR_EXACT_SHORT_WRAP=1 build (rmath.h)?  Its version string names it."""
    from deodr_b200 import _cabi

    return b"exact short wrap" in _cabi.load().deodr_b200_version()


def assert_image_close(got, ref):
    assert np.array_equal(np.isnan(got), np.isnan(ref)), "NaN pattern of the image"
    ok = ~np.isnan(ref)
    if ok.any():
        with np.errstate(invalid="ignore"):
            assert np.array_equal(np.isinf(got[ok]), np.isinf(ref[ok])) and np.all(got[ok][np.isinf(ref[ok])] ==
                                                                                     ref[ok][np.isinf(ref[ok])])
            fin = np.isfinite(ref[ok])
            assert np.abs(got[ok][fin] - ref[ok][fin]).max(initial=0.0) <= IMAGE_TOL


def assert_gradients_close(got, ref, fewer_non_finite=False):
    """fewer_non_finite: the device's non-finite entries need only be a subset of the checker's (INTEGRATION.md
    section 5, row "non-finite inputs"); the three-part criterion then holds on the entries finite in both."""
    for name in GRADS:
        if ref[name].size == 0:
            continue
        fin, fin_got = np.isfinite(ref[name]), np.isfinite(got[name])
        if fewer_non_finite:
            assert not (fin & ~fin_got).any(), (name, "non-finite where the checker's is finite")
        else:
            assert np.array_equal(fin_got, fin), (name, "finite pattern", int((~fin).sum()), int((~fin_got).sum()))
        if fin.any():
            assert_gradient_close(got[name][fin & fin_got], ref[name][fin & fin_got], name)


def check_edge(gpu, checker, scene, sigma, image=True, gradients=True, emul=None):
    """check() of tests/test_gpu_parity.py for inputs with non-finite values.  image=False: z-buffer and face ids only;
    gradients=False: forward only.  emul: the CPU emulation of the kernel phases, whose non-finite gradient entries
    the device must reproduce exactly; the checker's may then be more (see assert_gradients_close)."""
    with np.errstate(all="ignore"):
        ref_image, z = checker.render(scene, sigma)
    differentiable = gradients and image and scene.backface_culling and not scene.perspective_correct
    image_b = dense_image_b(np.nan_to_num(ref_image)) if differentiable else None
    got = run_device(gpu, scene, sigma, image_b)
    assert np.array_equal(got["z_buffer"], z, equal_nan=True), "z-buffer not bit-exact"
    assert np.array_equal(got["face_id"] >= 0, np.isfinite(z))
    if image:
        assert_image_close(got["image"], ref_image)
    if differentiable:
        with np.errstate(all="ignore"):
            ref = checker.render_b(scene, sigma, ref_image, z, image_b)
        assert_gradients_close(got, ref, fewer_non_finite=emul is not None)
        if emul is not None:
            with np.errstate(all="ignore"):
                own = emul.render_b(scene, sigma, emul.render(scene, sigma), image_b)
            for name in GRADS:
                assert np.array_equal(np.isfinite(got[name]), np.isfinite(own[name])), (name, "finite pattern")
    return got


def check_against_emulation(gpu, emul, scene, sigma, colours=True):
    """The device against the CPU emulation of the kernel phases of the same build: z-buffer, face ids, image and
    gradients (fp32 on both sides, different summation orders).  colours=False: z-buffer, face ids and the NaN pattern
    of the image only."""
    with np.errstate(all="ignore"):
        fwd = emul.render(scene, sigma)
        image_b = dense_image_b(np.nan_to_num(fwd["image"].astype(np.float64)))
        ref = emul.render_b(scene, sigma, fwd, image_b)
    got = run_device(gpu, scene, sigma, image_b)
    assert np.array_equal(got["z_buffer"], fwd["z"], equal_nan=True), "z-buffer differs from the emulation"
    assert np.array_equal(got["face_id"], fwd["face_id"])
    assert np.array_equal(np.isnan(got["image"]), np.isnan(fwd["image"]))
    if colours:
        assert_image_close(got["image"], fwd["image"])
        assert_gradients_close(got, ref)


def base_scene():
    """The scene of scripts/probe_edge_cases.py: 300 overlapping triangles, 40 % of the edges silhouettes, 64 x 48."""
    return confetti_scene(300, 64, 48, size=6.0, seed=3, edge_ratio=0.4)


# ---------------------------------------------------------------------------------------------- a. image sides

def scene_of_side(width, height, nb_colors=3, seed=0):
    """The base scene stretched to width x height (vertices kept inside the `short` range), with nb_colors channels."""
    rng = np.random.default_rng(seed)
    s = confetti_scene(300, 64, 48, size=6.0, seed=3, edge_ratio=0.4, nb_colors=nb_colors)
    s.width, s.height = width, height
    s.ij = s.ij * np.array([width / 64.0, height / 48.0])
    s.ij += rng.normal(size=s.ij.shape) * 3
    s.ij = np.clip(s.ij, -32000, 32766.5)
    return s


@pytest.mark.parametrize("width,height", [(1, 1), (1, 97), (130, 1), (32767, 3), (3, 32767), (20000, 17), (32767, 40),
                                          (15, 17), (16, 16), (17, 15)])
def test_image_sides(gpu, checker, width, height):
    """One-pixel and 32767-pixel sides, and one partial 16 x 16 tile on either side of a full one."""
    got = check_edge(gpu, checker, scene_of_side(width, height), 1.0)
    assert np.isfinite(got["z_buffer"]).any()


@pytest.mark.parametrize("width", [20, 18])
@pytest.mark.parametrize("nb_colors", [1, 3, 4])
def test_tile_store_and_plain_loads_at_one_side(gpu, checker, width, nb_colors):
    """Width 20: the image (W*C floats), owner (W int32) and z-buffer (W doubles) rows are 16-byte multiples, so the
    forward stores tiles and the adjoint loads them by TMA for every C <= 4.  Width 18: only C = 4 keeps the forward's
    tile store, and the adjoint's owner rows never qualify: its plain loads.  13 rows: a partial row of tiles."""
    check_edge(gpu, checker, scene_of_side(width, 13, nb_colors, seed=width + nb_colors), 1.0)


def test_seventeen_channels_at_a_thin_side(gpu, checker):
    """More than 16 channels (the slab path of DESIGN.md section 4) on a 3-pixel-wide image."""
    check_edge(gpu, checker, scene_of_side(3, 130, 17, seed=17), 1.0)


@pytest.mark.parametrize("width,height", [(0, 5), (5, 0), (32768, 2), (2, 32768)])
def test_image_sides_outside_the_short_range_are_refused(gpu, width, height):
    """Sides must lie in [1, 32767] (the reference's `short` loop counters): render and render_b refuse the others
    with EINVAL before touching the device."""
    import torch

    from deodr_b200 import _cabi
    from deodr_b200.renderer import DeviceScene

    s = copy.copy(base_scene())
    s.width, s.height = width, height
    ds = DeviceScene(s, "cuda:0")
    with pytest.raises(_cabi.DeodrB200Error, match="image sides") as err:
        gpu.render(ds, 1.0)
    assert err.value.code == _cabi.EINVAL
    fwd = {k: torch.zeros((height, width) + (() if k != "image" else (3,)), dtype=dt, device="cuda:0")
           for k, dt in (("image", torch.float32), ("z_buffer", torch.float64), ("owner", torch.int32))}
    with pytest.raises(_cabi.DeodrB200Error, match="image sides") as err:
        gpu.render_b(ds, 1.0, fwd, torch.zeros((height, width, 3), dtype=torch.float32, device="cuda:0"))
    assert err.value.code == _cabi.EINVAL


# ---------------------------------------------------------------------------------------------- b. band widths

@pytest.mark.parametrize("sigma", [1e-3, 0.05, 9.0, 45.0])
def test_band_widths(gpu, checker, texture, sigma):
    """GPU twin of tests/test_emul.py::test_emulated_kernels_extreme_sigma.  At 45 px every tile holds every
    silhouette edge: the heavy-tile order, several 64-edge chunks per pixel mask, the span cache the adjoint reads."""
    np.random.seed(2)
    check_edge(gpu, checker, soup_scene(clockwise=False, texture=texture), sigma)
    check_edge(gpu, checker, torus_scene(24, 160, 120), sigma)
    check_edge(gpu, checker, confetti_scene(800, 96, 80, size=3.0, seed=3, edge_ratio=0.5), sigma)


# ------------------------------------------------------------------------------ c. non-finite and degenerate inputs

def _pick(n, seed):
    return np.random.default_rng(seed).choice(900, n, replace=False)


def _set(name, n, value, seed, column=None):
    def edit(s):
        a = getattr(s, name)
        if column is None:
            a[_pick(n, seed)] = value
        else:
            a[_pick(n, seed), column] = value
    return edit


def _scale_depths(f):
    def edit(s):
        s.depths = s.depths * f
    return edit


def _negate_depths(s):
    s.depths[_pick(30, 4)] *= -1


def _repeated_vertex(s):
    s.faces[::7, 1] = s.faces[::7, 0]


def _coincident_vertices(s):
    s.ij[s.faces[::5, 2]] = s.ij[s.faces[::5, 1]]


def _all_edges(s):
    s.edgeflags[:] = True


def _no_culling(s):
    s.backface_culling = False


def _perspective_tiny_depths(s):
    s.perspective_correct = True
    s.depths[::9] = 1e-12


NON_FINITE = {
    "nan_positions": _set("ij", 10, np.nan, 1),
    "pos_inf_positions": _set("ij", 10, np.inf, 2),
    "neg_inf_positions": _set("ij", 10, -np.inf, 3),
    "pos_inf_rows": _set("ij", 10, np.inf, 5, column=1),
    "pos_inf_columns": _set("ij", 10, np.inf, 6, column=0),
    "negative_depths": _negate_depths,
    "zero_depths": _set("depths", 30, 0.0, 7),
    "depths_1e-300": _scale_depths(1e-300),
    "depths_1e300": _scale_depths(1e300),
    "nan_colours": _set("colors", 10, np.nan, 8),
    "repeated_vertex": _repeated_vertex,
    "coincident_vertices": _coincident_vertices,
    "every_edge_flagged": _all_edges,
    "no_culling": _no_culling,
    "perspective_depths_1e-12": _perspective_tiny_depths,
}


# INTEGRATION.md section 5, row "non-finite inputs": the reference runs the adjoint of every front-facing triangle's
# matrix inverse even when none of its pixels passed a gradient back (DR.h:838-858), so a triangle with an infinite
# coordinate or a NaN colour that owns no pixel gets 0 * inf or 0 * NaN = NaN on all three vertices; here a zero
# adjoint is never propagated.  The reference's non-finite entries are then a superset of ours, and the device must
# have exactly the non-finite entries of its emulation.
SPREADS_NON_FINITE = {"pos_inf_positions", "pos_inf_rows", "pos_inf_columns", "nan_colours"}


@pytest.fixture(scope="module")
def emul(gpu):
    """The CPU emulation of the build that is loaded."""
    return Emulator(exact_short_wrap=exact_wrap_build())


@pytest.mark.parametrize("case", list(NON_FINITE))
def test_non_finite_and_degenerate_inputs(gpu, checker, emul, case):
    s = base_scene()
    NON_FINITE[case](s)
    check_edge(gpu, checker, s, 1.0, emul=emul if case in SPREADS_NON_FINITE else None)


def test_nan_depths(gpu, checker):
    """INTEGRATION.md section 5, row "non-finite inputs": with a NaN depth the reference's std::sort of the depth sums
    has no defined order, so the edge overdraw (the antialiased pixels) may differ: z-buffer and face ids only."""
    s = base_scene()
    s.depths[_pick(10, 9)] = np.nan
    check_edge(gpu, checker, s, 1.0, image=False)


def test_integer_vertex_positions(gpu, checker):
    """INTEGRATION.md section 5, last row: pixel centres ON silhouette edges (T = 0) make the edge gradients a
    division by a tiny T in fp32: forward only."""
    s = base_scene()
    s.ij = np.round(s.ij)
    check_edge(gpu, checker, s, 1.0, gradients=False)


# ---------------------------------------------------------------------------------------------- d. far vertices

@pytest.mark.parametrize("far", [1e3, 3.2e4])
def test_far_vertices_within_the_short_range(gpu, checker, far):
    """Long triangles crossing the image from up to 32000 px outside: the reference's results, gradients included."""
    for seed in range(4):
        check_edge(gpu, checker, far_vertex_scene(seed, far), 1.0)


def inf_vertex_scene(seed):
    """A far-vertex scene with three of its vertices at +inf (both coordinates, the row, the column)."""
    s = far_vertex_scene(seed, 1e3)
    idx = np.random.default_rng(100 + seed).choice(s.ij.shape[0], 3, replace=False)
    s.ij[idx[0]] = np.inf
    s.ij[idx[1], 1] = np.inf
    s.ij[idx[2], 0] = np.inf
    return s


@pytest.mark.parametrize("far", [4e4, 7e4, 1e6, 3e9, 1e15, np.inf])
def test_far_vertices_beyond_the_short_range(gpu, checker, emul, far):
    """Beyond +-32767 px the default build culls what the reference draws at wrapped coordinates (INTEGRATION.md
    section 5, row "vertex coordinates beyond +-32767 px"): the device must do exactly what the CPU emulation of that
    build does.  The DEODR_EXACT_SHORT_WRAP=1 build must give the reference's z-buffer and, up to 3e9 px, its image,
    and the emulation of that build in every other respect.  Beyond 3e9 px colours and gradients are not compared: the
    interpolation of a triangle with a vertex 1e12 px away is ill-conditioned in any arithmetic (1.5e-5 between the
    device's fp32 and the host's at 1e15 px).  far = inf: scenes with a few +inf vertices."""
    exact = exact_wrap_build()
    for seed in range(4):
        scene = inf_vertex_scene(seed) if np.isinf(far) else far_vertex_scene(seed, far)
        check_against_emulation(gpu, emul, scene, 1.0, colours=np.isinf(far) or far <= 3e9)
        if exact:
            with np.errstate(all="ignore"):
                image, z = checker.render(scene, 1.0)
            got = run_device(gpu, scene, 1.0)
            assert np.array_equal(got["z_buffer"], z, equal_nan=True), (far, seed)
            if far <= 3e9:
                assert_image_close(got["image"], image)


# ---------------------------------------------------------------------------------------------- e. textures

@pytest.mark.parametrize("shape", [(2, 2), (3, 5)])
def test_tiny_textures(gpu, checker, shape):
    th, tw = shape
    rng = np.random.default_rng(th * 10 + tw)
    np.random.seed(2)
    s = soup_scene(clockwise=False, texture=rng.random((th, tw, 3)))
    s.uv = rng.random(s.uv.shape) * np.array([tw - 1, th - 1]) * 1.2 - 0.1
    check_edge(gpu, checker, s, 1.0)


def test_uv_far_outside_the_texture(gpu, checker, texture):
    np.random.seed(2)
    s = soup_scene(clockwise=False, texture=texture[::4, ::4].copy())
    s.uv = s.uv * 50 - 500
    check_edge(gpu, checker, s, 1.0)


@pytest.mark.parametrize("textured,shaded", [(1, 0), (0, 1), (1, 1), (0, 0)])
def test_every_textured_shaded_combination(gpu, checker, texture, textured, shaded):
    np.random.seed(2)
    s = soup_scene(clockwise=False, texture=texture[::4, ::4].copy())
    s.textured[:] = textured
    s.shaded[:] = shaded
    s.uv = s.uv * 0.9973 + 0.0131  # off the texel grid (see test_uv_on_the_texel_grid)
    check_edge(gpu, checker, s, 1.0)


def test_uv_on_the_texel_grid(gpu, checker, texture):
    """INTEGRATION.md section 5, last row: on a texel boundary the bilinear adjoint is discontinuous and fp32 attributes
    may pick the other side: forward only."""
    np.random.seed(2)
    s = soup_scene(clockwise=False, texture=texture[::4, ::4].copy())
    s.uv = np.round(s.uv)
    check_edge(gpu, checker, s, 1.0, gradients=False)
