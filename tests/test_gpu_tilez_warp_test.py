"""GPU (-m gpu): the z pass's two record paths - the warp-local test of small chunks and the candidate scatter of the
others - give the exact results on the device: z-buffer bit-exact and image / gradients within the
parity tolerances against the CPU oracle, owner codes and face ids equal to the CPU emulation of the kernel phases.

Covers tiles holding exactly 1, 31, 32, 33, 127, 128, 129 and 300 records (one partial chunk on either side of the
warp-test threshold, one full chunk, a full chunk plus a one-record tail, three chunks), pixels with more than
PIX_SLOTS candidates, exact z ties between distinct triangles, perspective-correct instances, the 1M-triangle 2048^2
scene and the eight 512^2 views of the 200k-triangle mesh rendered as one batch."""
import numpy as np
import pytest
from canon import Emulator
from test_gpu_parity import IMAGE_TOL, check, run_device

from deodr_b200.scenes import SceneArrays, torus_scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu(build_native):
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from deodr_b200.renderer import Renderer

    return Renderer(0)


@pytest.fixture(scope="module")
def emul():
    return Emulator()


def one_tile_scene(k: int, seed: int, ties: bool = True, crowd: bool = False) -> SceneArrays:
    """k front-facing micro-triangles inside tile (1, 1) of a 48 x 48 image, each covering at least its centre pixel:
    exactly k records in that tile.  ties: every fourth triangle repeats an earlier one (same vertices and depths,
    another index): exact z ties.  crowd: all centres within 2 px, so that pixels collect more than PIX_SLOTS
    candidates."""
    rng = np.random.default_rng(seed)
    lo, hi = (22, 25) if crowd else (20, 28)
    centre = rng.integers(lo, hi, size=(k, 2)).astype(np.float64)
    tri = np.empty((k, 3, 2))
    tri[:, 0] = centre + [-1.6, -1.6]  # a fixed triangle around the centre pixel, jittered a little
    tri[:, 1] = centre + [1.7, -0.9] + rng.uniform(0, 0.2, size=(k, 2))
    tri[:, 2] = centre + [-0.4, 1.8] + rng.uniform(0, 0.2, size=(k, 2))
    depth = rng.uniform(1.0, 5.0, size=k)
    if ties:
        for t in range(3, k, 4):
            src = int(rng.integers(0, t))
            tri[t] = tri[src]
            depth[t] = depth[src]
        if k >= 4:  # one tied pair in front of everything: its pixels certainly tie
            tri[3] = tri[0]
            depth[0] = depth[3] = 0.5
    det = (tri[:, 1, 0] - tri[:, 0, 0]) * (tri[:, 2, 1] - tri[:, 0, 1]) - (tri[:, 2, 0] - tri[:, 0, 0]) * (
        tri[:, 1, 1] - tri[:, 0, 1])
    flip = det > 0
    tri[flip] = tri[flip][:, ::-1]
    faces = np.arange(3 * k, dtype=np.uint32).reshape(-1, 3)
    return SceneArrays(
        faces=faces, faces_uv=faces.copy(), ij=np.ascontiguousarray(tri.reshape(-1, 2)),
        depths=np.repeat(depth, 3), textured=np.zeros(k, dtype=bool), uv=np.zeros((3 * k, 2)),
        shade=np.zeros(3 * k), colors=rng.random((3 * k, 3)), shaded=np.zeros(k, dtype=bool),
        edgeflags=rng.random((k, 3)) < 0.2, height=48, width=48, nb_colors=3, texture=np.zeros((2, 2, 3)),
        background_image=None, background_color=np.array([0.2, 0.4, 0.6]), clockwise=False, backface_culling=True,
        perspective_correct=False,
    )


def same_owners(got, ref):
    """Owner codes equal except the tie-table index; the same pixels tie; face ids (the forward owner) equal."""
    tie_g, tie_r = got["owner"] <= -2, ref["owner"] <= -2
    assert np.array_equal(tie_g, tie_r)
    assert np.array_equal(got["owner"][~tie_g], ref["owner"][~tie_r])
    assert np.array_equal(got["face_id"], ref["face_id"])


@pytest.mark.parametrize("k", [1, 31, 32, 33, 127, 128, 129, 300])
@pytest.mark.parametrize("persp", [False, True])
def test_records_per_tile(gpu, checker, emul, k, persp):
    scene = one_tile_scene(k, seed=k, crowd=k >= 127)
    scene.perspective_correct = persp
    got = check(gpu, checker, scene, 1.0)
    ref = emul.render(scene, 1.0)
    assert np.array_equal(got["z_buffer"], ref["z"])
    same_owners(got, ref)
    if k > 3:
        assert (got["owner"] <= -2).any(), "exact ties should reach the side table"


def test_crowded_pixels(gpu, checker, emul):
    """Dozens of candidates per pixel within one chunk: the pixel test's scan fall-back, and the warp test's
    candidate masks with many bits set."""
    scene = one_tile_scene(96, seed=5, ties=False, crowd=True)
    got = check(gpu, checker, scene, 1.0)
    same_owners(got, emul.render(scene, 1.0))


def test_config5_full_size(gpu, checker):
    check(gpu, checker, torus_scene(708, 2048, 2048), 1.0)


def test_config4_eight_views_one_batch(gpu, checker):
    """The eight 512^2 views of the 200k-triangle mesh in one render_views call: every view's z-buffer bit-exact."""
    from deodr_b200.renderer import DeviceScene

    scenes = [torus_scene(316, 512, 512, view=v, n_views=8) for v in range(8)]
    outs = gpu.render_views([DeviceScene(s, "cuda:0") for s in scenes], 1.0, face_id=True)
    for v, (s, out) in enumerate(zip(scenes, outs)):
        image, z = checker.render(s, 1.0)
        assert np.array_equal(out["z_buffer"].cpu().numpy(), z), f"view {v}: z-buffer not bit-exact"
        assert np.abs(out["image"].cpu().numpy() - image).max() <= IMAGE_TOL, f"view {v}"
        alone = run_device(gpu, s, 1.0)
        assert np.array_equal(out["face_id"].cpu().numpy(), alone["face_id"])
