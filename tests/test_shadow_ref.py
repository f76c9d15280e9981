"""CPU: the fp64 restatement of the cube shadow maps (tests/shadow_ref.py) - its adjoint against complex-step
derivatives, exact visibility in front of the map, and the cube's six face cameras."""
import numpy as np
import pytest

import shadow_ref as ref

M = 64
BIAS, SOFT = 0.01, 0.05


def _banded_point(rng, p):
    """A point x around p away from face and tap boundaries, with a map whose four taps put each tap's smoothstep
    inside its band (0.2 < y < 0.8); every other texel at FAR."""
    while True:
        x = p + rng.normal(size=3) * rng.uniform(0.5, 3.0)
        d = np.abs(x - p)
        top = np.sort(d)
        if top[2] < 1.05 * top[1]:
            continue  # near a face boundary
        k = ref.face_of((x - p)[None])
        u, v, z = ref.project(x[None], p, k, M)
        idx, fu, fv = ref.taps(u, v, M)
        if not (0.1 < fu[0] < 0.9 and 0.1 < fv[0] < 0.9):
            continue  # near a tap boundary
        maps = np.full((6, M * M), ref.FAR)
        y = rng.uniform(0.2, 0.8, 4)
        maps[k[0], idx[0]] = z[0] - BIAS + SOFT * (y - 1)
        return x, maps.reshape(6, M, M), k[0], idx[0]


def test_the_adjoint_matches_complex_steps():
    rng = np.random.default_rng(0)
    h = 1e-30
    for _ in range(40):
        p = rng.uniform(-1, 1, 3)
        x, maps, k, idx = _banded_point(rng, p)
        g = rng.normal()
        x_b, p_b, maps_b = ref.visibility_b(x[None], p, maps, M, BIAS, SOFT, np.array([g]))
        for i in range(3):
            e = np.zeros(3, complex)
            e[i] = 1j * h
            want_x = g * np.imag(ref.visibility((x + e)[None], p, maps, M, BIAS, SOFT))[0] / h
            want_p = g * np.imag(ref.visibility(x[None], p + e, maps, M, BIAS, SOFT))[0] / h
            assert abs(x_b[0, i] - want_x) <= 1e-9 * max(1.0, abs(want_x))
            assert abs(p_b[i] - want_p) <= 1e-9 * max(1.0, abs(want_p))
        for q in range(4):
            m = maps.astype(complex).reshape(6, M * M)
            m[k, idx[q]] += 1j * h
            want = g * np.imag(ref.visibility(x[None], p, m.reshape(6, M, M), M, BIAS, SOFT))[0] / h
            got = maps_b.reshape(6, M * M)[k, idx[q]]
            assert abs(got - want) <= 1e-9 * max(1.0, abs(want))
        assert np.count_nonzero(maps_b) <= 4


def test_points_in_front_of_their_map_are_fully_visible():
    rng = np.random.default_rng(1)
    p = np.zeros(3)
    x = rng.normal(size=(5000, 3))
    x *= rng.uniform(0.5, 5, (5000, 1)) / np.linalg.norm(x, axis=1, keepdims=True)
    # every texel exactly at each point's depth, or behind it: D + bias >= z with any bias > 0
    for scale in (1.0, 1.5):
        k = ref.face_of(x - p)
        _, _, z = ref.project(x, p, k, M)
        maps = np.full((6, M * M), 0.0)
        for f in range(6):
            maps[f] = scale * z[k == f].max() if np.any(k == f) else 0.0
        V = ref.visibility(x, p, maps.reshape(6, M, M), M, BIAS, SOFT)
        assert np.all(V == 1.0)
    # and over FAR
    V = ref.visibility(x, p, np.full((6, M, M), ref.FAR), M, BIAS, SOFT)
    assert np.all(V == 1.0)


def test_points_far_behind_the_map_are_fully_shadowed():
    rng = np.random.default_rng(2)
    x = rng.normal(size=(1000, 3)) * 3
    V = ref.visibility(x, np.zeros(3), np.full((6, M, M), 1e-3), M, BIAS, SOFT)
    z = ref.project(x, np.zeros(3), ref.face_of(x), M)[2]
    assert np.all(V[z > 1e-3 + BIAS + SOFT] == 0.0)


def test_the_six_rotations_are_proper_and_axis_aligned():
    R = ref.ROTATIONS
    for k in range(6):
        assert np.array_equal(R[k] @ R[k].T, np.eye(3))
        assert np.linalg.det(R[k]) == pytest.approx(1.0, abs=0)
        axis, sign = k // 2, 1 - 2 * (k % 2)
        assert np.array_equal(R[k][2], sign * np.eye(3)[axis])  # the face looks along its axis


def test_the_frusta_cover_every_direction_with_the_taps_inside_the_map():
    rng = np.random.default_rng(3)
    d = rng.normal(size=(200_000, 3))
    d[:1000] = np.sign(rng.normal(size=(1000, 3)))  # cube corners and edges
    d[1000:2000, 0] = d[1000:2000, 1]               # ties between axes
    k = ref.face_of(d)
    for Msz in (8, 64, 512, 4096):
        u, v, z = ref.project(d, np.zeros(3), k, Msz)
        assert np.all(z > 0)
        idx, fu, fv = ref.taps(u, v, Msz)
        # the 2x2 taps never need clamping: 1 <= floor(u) and floor(u) + 1 <= M - 2
        assert np.all(np.floor(u) >= 1) and np.all(np.floor(u) + 1 <= Msz - 2)
        assert np.all(np.floor(v) >= 1) and np.all(np.floor(v) + 1 <= Msz - 2)


def test_the_camera_vector_projects_like_the_restatement():
    rng = np.random.default_rng(4)
    p = rng.normal(size=3)
    x = p + rng.normal(size=(100, 3))
    k = ref.face_of(x - p)
    u, v, z = ref.project(x, p, k, M)
    for i in range(100):
        cam = ref.camera(p, k[i], M)
        ext, K = cam[:12].reshape(3, 4), cam[12:21].reshape(3, 3)
        pc = ext[:, :3] @ x[i] + ext[:, 3]
        assert np.allclose([pc[0] / pc[2] * K[0, 0] + K[0, 2], pc[1] / pc[2] * K[1, 1] + K[1, 2], pc[2]],
                           [u[i], v[i], z[i]], rtol=1e-13, atol=1e-12)
