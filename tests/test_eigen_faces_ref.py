"""CPU: the fp64 restatement of the eigen-faces fit (tests/eigen_faces_ref.py) over the C restatement of the rasteriser
follows the reference's trajectories of tests/golden/eigen_faces_reference.json over all 100 steps: the reference's
own Scene2D run with its overwriting texture adjoint ("as_written", port with texfix=False) and the reference core
with the summed adjoint ("texfix").  This pins the restatement the GPU fit is checked against to the reference."""
import json
import os

import numpy as np
import pytest
from conftest import GOLDEN

import eigen_faces_ref as ef


@pytest.fixture(scope="module")
def reference():
    with open(os.path.join(GOLDEN, "eigen_faces_reference.json")) as f:
        return json.load(f)


def test_inputs_are_the_examples_grid_and_displacement():
    d = ef.load_inputs()
    n = 5
    points = np.column_stack([t.flatten() for t in np.meshgrid(np.arange(n + 1) / n, np.arange(n + 1) / n)])
    assert np.array_equal(d["points"], points)
    assert d["triangles"].shape == (50, 3) and set(np.unique(d["triangles"])) == set(range(36))
    rng = np.random.RandomState(0)
    deformed = points + (rng.rand(*points.shape) - 0.5) * 0.5 / n
    border = ef.on_border(points)
    deformed[border] = points[border]
    assert np.array_equal(d["points_deformed"], deformed)
    K = d["components"].shape[0]
    assert 10 <= K <= 16 and d["components"].shape[1] == 64 * 64
    np.testing.assert_allclose(d["components"] @ d["components"].T, np.eye(K), atol=1e-12)
    assert d["image_obs"].shape == (64, 64, 1) and d["texture_gt"].shape == (64, 64, 1)


@pytest.mark.parametrize("run,texfix", [("as_written", False), ("texfix", True)])
def test_restatement_follows_the_reference(run, texfix, reference, build_native):
    from oracle.oracle import Oracle

    got = np.array(ef.fit(Oracle("port", texfix=texfix), ef.load_inputs()))
    want = np.array(reference[run]["energies"])
    assert got.shape == want.shape == (ef.NB_ITER,)
    rel = np.abs(got / want - 1)
    assert rel.max() <= 1e-9, (rel.argmax(), rel.max())
