"""Generates the fixtures of the eigen-faces fit (deodr/examples/eigen_faces.py) from a DEODR checkout whose Cython
extension is built (``python setup.py build_ext --inplace``), with oracle/_ref built from the same checkout
(``make -C oracle DEODR_REFERENCE=...``):

    DEODR_REFERENCE=<built DEODR checkout> python tests/golden/make_eigen_faces_golden.py

The example fits the Olivetti faces, downloaded through scikit-learn.  Here the faces are synthetic, made only from
fixtures of this directory: 18 grey 64 x 64 crops (the RGB mean / 255, Gaussian-blurred with sigma 2 px) at fixed
offsets, 9 of trefle_texture_u8.npy and 9 of the textured part of duck_textured.npz's texture_u8, and their PCA by
numpy SVD, K = 12 unit components.  The ground-truth texture
is crop 10, as the example uses face 10.  The grid, displacement, scene and step are the example's.

eigen_faces_inputs.npz
  points [36,2]          the regular 6 x 6 grid on [0,1]^2 (n = 5)
  triangles [50,3] u32   its Delaunay triangulation by scipy (stored: on a regular grid it is not unique across
                         qhull versions)
  points_deformed [36,2] np.random.seed(0), displacement (rand - 0.5) * 0.5 / n, border points pinned
  mean [4096], components [12,4096]   the PCA
  texture_gt [64,64,1]   crop 10
  image_obs [64,64,1]    the reference's Scene2D render of texture_gt at points_deformed, sigma 1

eigen_faces_reference.json: the energies of the example's 100 steps from zero coefficients and the regular grid
  "as_written"  the reference's own Scene2D.render_compare_and_backward (its texture adjoint overwrites, ``=``)
  "texfix"      the same loop (tests/eigen_faces_ref.py) on oracle/_ref's texfix build of the reference core (``+=``)
"""
import json
import os
import sys

import numpy as np
from scipy.ndimage import gaussian_filter
from scipy.spatial import Delaunay

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
# tests/dropin/stubs stands in for the modules the reference imports at module level but this fit does not use
sys.path[:0] = [ROOT, os.path.dirname(HERE), os.path.join(os.path.dirname(HERE), "dropin", "stubs"),
                os.environ["DEODR_REFERENCE"]]

from deodr.differentiable_renderer import Scene2D  # noqa: E402

import eigen_faces_ref as ef  # noqa: E402
from oracle.oracle import Oracle  # noqa: E402

K = 12
# grey, and blurred to the smoothness of a face photograph: the sharp edges of the raw images make the example's
# point step (1e-4) overshoot, and the fit oscillate instead of descending
grey = lambda a: gaussian_filter(a.astype(np.float64).mean(axis=2) / 255, 2.0)  # noqa: E731
trefle = grey(np.load(os.path.join(HERE, "trefle_texture_u8.npy")))
duck = grey(np.load(os.path.join(HERE, "duck_textured.npz"))["texture_u8"])
# offsets where both images vary (much of the duck's texture is one flat colour, which would make a degenerate fit)
crops = [trefle[r:r + 64, c:c + 64] for r in (0, 40, 80) for c in (0, 61, 123)]
crops += [duck[r:r + 64, c:c + 64] for r in (16, 96, 176) for c in (320, 384, 448)]
data = np.stack([c.ravel() for c in crops])
mean = data.mean(axis=0)
_, _, vt = np.linalg.svd(data - mean, full_matrices=False)
components = vt[:K]

n = 5
points = np.column_stack([t.flatten() for t in np.meshgrid(np.arange(n + 1) / n, np.arange(n + 1) / n)])
triangles = Delaunay(points).simplices.astype(np.uint32)
border = ef.on_border(points)
np.random.seed(0)
points_deformed = points + (np.random.rand(*points.shape) - 0.5) * 0.5 / n
points_deformed[border] = points[border]
texture_gt = crops[10][:, :, None]

P, T = points.shape[0], triangles.shape[0]


def scene2d(ij, texture):
    return Scene2D(triangles, triangles, ij, np.ones(P), np.ones(T, dtype=bool), points * 64 + 0.5, np.ones(P),
                   np.ones((P, 1)), np.ones(T, dtype=bool), np.zeros((T, 3), dtype=bool), 64, 64, 1, texture,
                   background_image=None, background_color=np.array([0]), clockwise=True, backface_culling=True)


image_obs, _ = scene2d(points_deformed * 64 - 0.5, texture_gt).render(sigma=1)
np.savez_compressed(os.path.join(HERE, "eigen_faces_inputs.npz"), points=points, triangles=triangles,
                    points_deformed=points_deformed, mean=mean, components=components, texture_gt=texture_gt,
                    image_obs=image_obs)
d = ef.load_inputs()

# the example's loop, verbatim but for the display
scene = scene2d(points * 64 - 0.5, texture_gt)
variables = {"points_deformed": points.copy(), "pca_coefs": np.zeros(K)}
as_written = []
for _ in range(ef.NB_ITER):
    scene.ij = variables["points_deformed"] * 64 - 0.5
    scene.texture = (mean + variables["pca_coefs"].dot(components)).reshape((64, 64))[:, :, None]
    _, _, _, err = scene.render_compare_and_backward(obs=image_obs, sigma=1)
    grads = {"points_deformed": scene.ij_b * 64, "pca_coefs": components.dot(scene.texture_b.flatten())}
    as_written.append(float(err))
    for name, lam in (("points_deformed", ef.STEP_POINTS), ("pca_coefs", ef.STEP_COEFS)):
        variables[name] = variables[name] - lam * grads[name]
    variables["points_deformed"][border] = points[border]

# the restated loop on the unpatched reference core follows the example's own run
check = ef.fit(Oracle("reference", texfix=False), d)
assert np.allclose(check, as_written, rtol=1e-12, atol=0), np.abs(np.array(check) / as_written - 1).max()
out = {"as_written": {"energies": as_written}, "texfix": {"energies": ef.fit(Oracle("reference", texfix=True), d)}}
with open(os.path.join(HERE, "eigen_faces_reference.json"), "w") as f:
    json.dump(out, f, indent=1)
    f.write("\n")
print({k: (v["energies"][0], v["energies"][10], v["energies"][-1]) for k, v in out.items()})
