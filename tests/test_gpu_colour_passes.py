"""GPU (-m gpu): the two colour passes of the forward - the epilogue fused into the z pass (k_tile_z) and the separate
colour pass (k_shade) a forward uses when the colours arrive late - and the pixel-parallel adjoints, on scenes where
the lanes of one warp shade very different owners.

The scenes hold a warp whose 32 lanes have 32 distinct owners (one micro-triangle per pixel, textured and untextured
ones alternating), warps that one triangle covers whole, exact z ties between two differently coloured copies of one
triangle (owner codes <= -2: the colour is the lower index's, the adjoint the higher's), medium triangles, background
lanes, and image sides that are not a multiple of 16.  (The tied copies are both untextured: at a tie that involves a
textured triangle the reference gives the gradient to more than one triangle, INTEGRATION.md section 5.)  For each,
with 1, 3, 4 and 16 channels and perspective-correct or not:
  - z-buffer bit-exact, image and gradients within the parity tolerances against the CPU checker;
  - the fused epilogue's image and G-buffer weights equal the unfused colour pass's bit for bit.  The unfused pass runs
    in a child process: it is reached through a colours-ready event with DEODR_B200_LATE_COLORS=shade, a switch read
    once per process."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if __name__ == "__main__":  # the child process of fused_vs_unfused (no conftest to set the path up)
    sys.path[:0] = [ROOT, HERE]

from test_gpu_parity import check  # noqa: E402

from deodr_b200.scenes import SceneArrays  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = [(C, persp, True) for C in (1, 3, 4, 16) for persp in (False, True)] + [(3, False, False)]
CASE_IDS = [f"C{C}-{'persp' if p else 'affine'}-{'mixed' if t else 'plain'}" for C, p, t in CASES]


def warp_scene(C: int, persp: bool, textured: bool, seed: int = 0) -> SceneArrays:
    """45 x 37 image (3 x 3 tiles, the last column and row partial), integer pixel centres:
    - one micro-triangle around each pixel of rows 0-1, columns 0-15 (warp 0 of tile (0, 0)): 32 distinct owners;
    - a large triangle over most of tile (1, 0): warps with a single owner;
    - a triangle over tiles (1..2, 1..2) and an exact copy of it with another index and other colours, in front of the
      large one: every pixel they cover is an exact tie;
    - a few medium triangles (about 12 x 8 px) in tiles (0, 1) and (0, 2);
    the rest is background."""
    rng = np.random.default_rng(seed)
    tris, depths = [], []
    for y in range(2):
        for x in range(16):
            c = np.array([x, y], dtype=np.float64)
            tris.append([c + [-0.3, -0.3], c + [0.35, -0.1] + rng.uniform(0, 0.05, 2), c + [-0.05, 0.35]])
            depths.append(rng.uniform(1.0, 1.5, 3))
    n_micro = len(tris)
    tris.append([[17.0, -3.0], [40.0, -2.0], [30.0, 14.5]])
    depths.append(np.array([4.0, 4.5, 5.0]))
    tie = len(tris)
    tris.append([[14.2, 12.3], [44.6, 15.1], [21.7, 36.4]])
    depths.append(np.array([2.0, 2.5, 3.0]))
    tris.append(list(tris[tie]))
    depths.append(depths[tie].copy())
    for _ in range(4):
        c = np.array([rng.uniform(2, 12), rng.uniform(18, 32)])
        tris.append([c + [-6, -4], c + [6, rng.uniform(-4, 0)], c + [rng.uniform(-3, 3), 4]])
        depths.append(rng.uniform(2.0, 6.0, 3))
    tri = np.array(tris, dtype=np.float64)
    k = len(tri)
    det = (tri[:, 1, 0] - tri[:, 0, 0]) * (tri[:, 2, 1] - tri[:, 0, 1]) - (tri[:, 2, 0] - tri[:, 0, 0]) * (
        tri[:, 1, 1] - tri[:, 0, 1])
    flip = det > 0
    tri[flip] = tri[flip][:, ::-1]
    dep = np.array(depths)
    dep[flip] = dep[flip][:, ::-1]
    tex = np.zeros(k, dtype=bool)
    if textured:
        tex[0:n_micro:2] = True  # every other micro-triangle: both kinds in warp 0 of tile (0, 0)
        tex[tie + 2] = True      # the first medium triangle
    faces = np.arange(3 * k, dtype=np.uint32).reshape(-1, 3)
    t_side = 8
    return SceneArrays(
        faces=faces, faces_uv=faces.copy(), ij=np.ascontiguousarray(tri.reshape(-1, 2)), depths=dep.reshape(-1),
        textured=tex, uv=rng.uniform(0.5, t_side - 1.5, size=(3 * k, 2)), shade=rng.uniform(0.5, 1.0, 3 * k),
        colors=rng.random((3 * k, C)), shaded=tex.copy(), edgeflags=rng.random((k, 3)) < 0.3, height=37, width=45,
        nb_colors=C, texture=rng.random((t_side, t_side, C)), background_image=None,
        background_color=rng.random(C), clockwise=False, backface_culling=True, perspective_correct=persp,
    )


@pytest.fixture(scope="module")
def gpu(build_native):
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from deodr_b200.renderer import Renderer

    return Renderer(0)


@pytest.fixture(scope="module")
def fused_vs_unfused(build_native):
    """{case id: {output: equal?}} from a child process that renders every case fused and unfused."""
    with tempfile.TemporaryDirectory() as out:
        env = dict(os.environ, DEODR_B200_LATE_COLORS="shade")
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), out]
        subprocess.run(cmd, check=True, env=env, cwd=ROOT)
        with open(os.path.join(out, "result.json")) as f:
            return json.load(f)


@pytest.mark.parametrize("sigma", [0.0, 1.0])  # 0: no silhouette edge, every medium / large owner in k_interior_bwd
@pytest.mark.parametrize("C, persp, textured", CASES, ids=CASE_IDS)
def test_against_checker(gpu, checker, C, persp, textured, sigma):
    got = check(gpu, checker, warp_scene(C, persp, textured), sigma)
    assert (got["owner"] <= -2).any(), "the scene should hold exact ties"
    assert (got["owner"] == -1).any(), "the scene should hold background pixels"


@pytest.mark.parametrize("C, persp, textured", CASES, ids=CASE_IDS)
def test_fused_epilogue_equals_colour_pass(fused_vs_unfused, C, persp, textured):
    res = fused_vs_unfused[CASE_IDS[CASES.index((C, persp, textured))]]
    assert res == {"image": True, "barycentric": True}, res


def _render_fused_and_unfused(out_dir):
    import torch

    from deodr_b200.renderer import DeviceScene, Renderer

    assert os.environ.get("DEODR_B200_LATE_COLORS") == "shade"
    renderer = Renderer(0)
    result = {}
    for case, case_id in zip(CASES, CASE_IDS):
        ds = DeviceScene(warp_scene(*case), "cuda:0")
        sigma = 1.0
        fused = renderer.render(ds, sigma, face_id=True, barycentric=True)
        fused = {k: fused[k].clone() for k in ("image", "barycentric")}
        ready = torch.cuda.Event()
        ready.record()
        renderer.set_colors_ready(ready)  # colours late: z pass unfused, then the colour pass
        unfused = renderer.render(ds, sigma, face_id=True, barycentric=True)
        torch.cuda.synchronize()
        result[case_id] = {k: bool(torch.equal(fused[k], unfused[k])) for k in ("image", "barycentric")}
    with open(os.path.join(out_dir, "result.json"), "w") as f:
        json.dump(result, f)


if __name__ == "__main__":
    _render_fused_and_unfused(sys.argv[1])
