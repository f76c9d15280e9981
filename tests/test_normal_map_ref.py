"""CPU: the fp64 restatement of the tangent-space normal map (tests/normal_map_ref.py) - the tangent frame's and the
perturbation's adjoints against complex-step derivatives, on the degenerate cases the model names, and a flat map
leaving the normal unchanged."""
import numpy as np
import pytest

import normal_map_ref as ref

H = 1e-30  # the complex step


def _complex_step_grad(f, x, w):
    """d <w, f(x)> / dx by complex steps, entry by entry."""
    g = np.zeros(x.shape)
    for idx in np.ndindex(x.shape):
        xc = x.astype(complex)
        xc[idx] += 1j * H
        g[idx] = np.sum(w * f(xc)).imag / H
    return g


def _mesh(kind):
    """(vertices, faces, uv, faces_uv) of a small test mesh."""
    rng = np.random.default_rng(3)
    if kind == "grid":  # a bumpy 3x3 grid with a uv chart rotated and scaled
        ii, jj = np.meshgrid(np.arange(4), np.arange(4), indexing="ij")
        v = np.stack((jj.ravel(), ii.ravel(), 0.2 * rng.normal(size=16)), axis=1).astype(float)
        f = []
        for i in range(3):
            for j in range(3):
                a, b, c, d = 4 * i + j, 4 * i + j + 1, 4 * i + j + 4, 4 * i + j + 5
                f += [(a, b, d), (a, d, c)]
        f = np.array(f)
        uv = v[:, :2] @ np.array([[1.3, 0.4], [-0.2, 1.1]]) + 0.1 * rng.normal(size=(16, 2))
        return v, f, uv, f.copy()
    if kind == "mirrored":  # two charts sharing the middle position vertices, the second mirrored in u
        v = np.array([[0, 0, 0], [1, 0, 0.1], [2, 0, 0.3], [0, 1, 0.2], [1, 1, -0.1], [2, 1, 0.4]], float)
        f = np.array([[0, 1, 4], [0, 4, 3], [1, 2, 5], [1, 5, 4]])
        uv = np.array([[0, 0], [1, 0], [0, 1], [1, 1], [1.7, 0], [1.6, 1.2]], float)
        fuv = np.array([[0, 1, 3], [0, 3, 2], [4, 1, 3], [4, 3, 5]])
        return v, f, uv, fuv
    if kind == "degenerate_uv":  # a face whose uv triangle has det = 0 (collinear uv)
        v, f, uv, fuv = _mesh("grid")
        uv[5] = 0.5 * (uv[4] + uv[6])
        uv[1] = uv[0] + (uv[5] - uv[4])  # rows of the same collinear shape
        f = np.concatenate((f, [[4, 5, 6]]))
        fuv = np.concatenate((fuv, [[4, 5, 6]]))
        return v, f, uv, fuv
    if kind == "clockwise":  # the grid with every face reversed
        v, f, uv, fuv = _mesh("grid")
        return v, f[:, ::-1].copy(), uv, fuv[:, ::-1].copy()
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["grid", "mirrored", "degenerate_uv", "clockwise"])
def test_the_tangent_adjoint_matches_complex_steps(kind):
    v, f, uv, fuv = _mesh(kind)
    rng = np.random.default_rng(7)
    w = rng.normal(size=(v.shape[0], 6))
    vb, uvb = ref.vertex_frames_b(v, f, uv, fuv, w)
    gv = _complex_step_grad(lambda x: ref.vertex_frames(x, f, uv, fuv), v, w)
    guv = _complex_step_grad(lambda x: ref.vertex_frames(v, f, x, fuv), uv, w)
    assert np.allclose(vb, gv, rtol=1e-10, atol=1e-12)
    assert np.allclose(uvb, guv, rtol=1e-10, atol=1e-12)


def test_a_zero_area_uv_face_adds_nothing():
    v, f, uv, fuv = _mesh("degenerate_uv")
    _, _, _, sigma, t, b = ref.face_terms(v, f, uv, fuv)
    assert sigma[-1] == 0 and not np.any(t[-1]) and not np.any(b[-1])


def test_the_frame_follows_u_and_v_on_a_plane():
    # a plane z = 0 with uv = (x, y): T = +x, B = +y, whatever the winding
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0]], float)
    f = np.array([[0, 1, 3], [0, 3, 2]])
    for faces in (f, f[:, ::-1].copy()):
        frames = ref.vertex_frames(v, faces, v[:, :2] * 7.0, faces)
        assert np.allclose(frames[:, :3], [1, 0, 0]) and np.allclose(frames[:, 3:], [0, 1, 0])


def _pixels(rng, n=40):
    g = rng.normal(size=(n, 13))
    g[:, 6] = rng.uniform(0.2, 1.0, n)
    M = rng.normal(size=(n, 3)) * 0.3 + [0, 0, 1]
    g[0, 6] = 0.0                         # a = 0
    M[1] = 0.0                            # |p| = 0
    g[2, 0:3], g[2, 7:10] = [0, 0, 1.7], [0, 0, -3.0]  # T parallel to N (exactly, along an axis): t = 0
    g[3, 0:3] = 0.0                       # |N| = 0
    g[4, 10:13] = -np.cross(g[4, 0:3], g[4, 7:10])  # B against n x t: s = -1
    return g, M


def test_the_degenerate_pixels_give_what_the_model_says():
    g, M = _pixels(np.random.default_rng(1))
    out = ref.normal_map(g, M)
    assert np.array_equal(out[:, 3:7], g[:, 3:7])
    assert not np.any(out[0, :3]) and not np.any(out[1, :3])
    assert np.array_equal(out[2, :3], [0, 0, g[2, 6] * np.sign(M[2, 2])])  # t = b = 0: p = M_z n
    assert np.allclose(np.linalg.norm(out[4:, :3], axis=1), g[4:, 6])


def test_the_perturbation_adjoint_matches_complex_steps():
    rng = np.random.default_rng(2)
    g, M = _pixels(rng)
    w = rng.normal(size=(g.shape[0], 7))
    gb, Mb = ref.normal_map_b(g, M, w)
    assert np.allclose(gb, _complex_step_grad(lambda x: ref.normal_map(x, M), g, w), rtol=1e-10, atol=1e-12)
    assert np.allclose(Mb, _complex_step_grad(lambda x: ref.normal_map(g, x), M, w), rtol=1e-10, atol=1e-12)
    assert not np.any(gb[0, [0, 1, 2, 7, 8, 9, 10, 11, 12]]) and not np.any(Mb[0])  # a = 0: only the pass-through
    assert not np.any(gb[:, 10:13])


def test_a_flat_map_leaves_the_normal_unchanged():
    g, _ = _pixels(np.random.default_rng(4))
    g = g[4:]
    a = g[:, 6:7]
    for scale in (1.0, 0.37):  # M carries the coverage as a factor
        out = ref.normal_map(g, np.tile([0, 0, scale], (g.shape[0], 1)))
        assert np.allclose(out[:, :3], a * g[:, :3] / np.linalg.norm(g[:, :3], axis=1, keepdims=True), atol=1e-15)
