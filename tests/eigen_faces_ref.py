"""Plain fp64 restatement of the reference's eigen-faces fit (deodr/examples/eigen_faces.py) on the synthetic faces of
tests/golden/eigen_faces_inputs.npz (make_eigen_faces_golden.py):

    scene       64 x 64, one channel, every triangle textured and shaded, shade 1, no silhouette edge, clockwise,
                backface culling; ij = 64 p - 0.5, uv = 64 p0 + 0.5 (p0 the regular grid)
    texture     mean + coefs @ components, reshaped to [64, 64, 1]
    energy      E = sum (image - obs)^2, image_b = 2 (image - obs)    (Scene2D.render_compare_and_backward, no mask)
    gradients   points_grad = 64 ij_b,  coefs_grad = components @ texture_b
    step        p -= 1e-4 points_grad,  coefs -= 0.5 coefs_grad, then the border points reset to the grid

The render and its adjoint come from a CPU oracle (oracle/oracle.py): ``Oracle("port", texfix=...)`` is the C
restatement of the rasteriser; ``texfix=False`` keeps the reference's overwriting texture adjoint (``=``), ``True``
sums it (``+=``), as the device does.
"""
import os

import numpy as np

from deodr_b200.scenes import SceneArrays

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SIZE = 64
STEP_POINTS, STEP_COEFS = 1e-4, 0.5
NB_ITER = 100


def load_inputs() -> dict:
    return dict(np.load(os.path.join(GOLDEN, "eigen_faces_inputs.npz")))


def on_border(points: np.ndarray) -> np.ndarray:
    return np.any((points == 0) | (points == 1), axis=1)


def texture_of(d: dict, coefs: np.ndarray) -> np.ndarray:
    return (d["mean"] + coefs @ d["components"]).reshape(SIZE, SIZE, 1)


def scene_of(d: dict, points: np.ndarray, texture: np.ndarray) -> SceneArrays:
    P, T = d["points"].shape[0], d["triangles"].shape[0]
    return SceneArrays(
        faces=d["triangles"], faces_uv=d["triangles"], ij=points * SIZE - 0.5, depths=np.ones(P),
        textured=np.ones(T, bool), uv=d["points"] * SIZE + 0.5, shade=np.ones(P), colors=np.ones((P, 1)),
        shaded=np.ones(T, bool), edgeflags=np.zeros((T, 3), bool), height=SIZE, width=SIZE, nb_colors=1,
        texture=texture, background_image=None, background_color=np.zeros(1), clockwise=True, backface_culling=True,
        strict_edge=True, perspective_correct=False, integer_pixel_centers=True)


def energy_and_gradients(oracle, d: dict, points: np.ndarray, coefs: np.ndarray):
    """-> (E, points_grad [P,2], coefs_grad [K]) at (points, coefs)."""
    scene = scene_of(d, points, texture_of(d, coefs))
    image, z_buffer = oracle.render(scene, 1.0)
    diff = image - d["image_obs"]
    grads = oracle.render_b(scene, 1.0, image, z_buffer, 2 * diff)
    return float(np.sum(diff ** 2)), grads["ij_b"] * SIZE, d["components"] @ grads["texture_b"].ravel()


def fit(oracle, d: dict, nb_iter: int = NB_ITER):
    """The example's loop -> energies [nb_iter] (the energy before each step)."""
    border = on_border(d["points"])
    points, coefs = d["points"].copy(), np.zeros(d["components"].shape[0])
    energies = []
    for _ in range(nb_iter):
        energy, points_grad, coefs_grad = energy_and_gradients(oracle, d, points, coefs)
        energies.append(energy)
        points = points - STEP_POINTS * points_grad
        coefs = coefs - STEP_COEFS * coefs_grad
        points[border] = d["points"][border]
    return energies
