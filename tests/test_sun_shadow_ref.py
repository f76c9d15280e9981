"""CPU: the fp64 restatement of the directional light's shadow map (tests/sun_shadow_ref.py) - its frame, its window,
its adjoints against complex-step derivatives, exact visibility in front of the map, and its reduction to the
unshadowed Phong restatement at V = 1."""
import numpy as np
import pytest

import phong_ref
import sun_shadow_ref as ref

M = 64
BIAS, SOFT = 0.01, 0.05
C0, R0 = np.array([0.1, -0.2, 0.3]), 2.0


def _directions(rng, n):
    d = rng.normal(size=(n, 3))
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def test_the_frame_is_orthonormal_and_right_handed():
    rng = np.random.default_rng(0)
    ls = np.concatenate((_directions(rng, 2000) * rng.uniform(0.1, 10, (2000, 1)),
                         [[0, 0, -1.0], [1e-9, 0, -1], [0, 0, 1], [1, 0, 0], [0, 0, 0]]))
    for l in ls:
        e1, e2, d = ref.frame(l)
        F = np.stack((e1, e2, d))
        # inside the pole's band d_z < -0.9999999 the fixed (e1, e2) are orthogonal to d only to |d_xy| < 4.5e-4
        tol = 5e-4 if d[2] < ref.POLE else 1e-12
        assert np.allclose(F @ F.T, np.eye(3), atol=tol)
        assert np.allclose(np.cross(e1, e2), d, atol=tol)
        if np.linalg.norm(l) > 0:
            assert np.allclose(d, l / np.linalg.norm(l), atol=1e-15)
        else:
            assert np.array_equal(d, [0, 0, 1.0])


def test_the_frame_is_continuous_away_from_the_pole():
    rng = np.random.default_rng(1)
    d = _directions(rng, 5000)
    d = d[d[:, 2] > -0.99]
    for l in d:
        step = rng.normal(size=3) * 1e-7
        a, b = np.stack(ref.frame(l)), np.stack(ref.frame(l + step))
        assert np.max(np.abs(a - b)) < 1e-5
    # at the pole only the rotation about d jumps, never d
    e1a, e2a, da = ref.frame([1e-4, 0, -1])
    e1b, e2b, db = ref.frame([0, 0, -1])
    assert np.allclose(da, db, atol=1e-4)


def test_every_point_of_the_bounds_has_its_taps_inside_the_map():
    rng = np.random.default_rng(2)
    x = _directions(rng, 100_000) * rng.uniform(0, 1, (100_000, 1)) ** (1 / 3)
    x[:20_000] = _directions(rng, 20_000)          # the sphere itself
    for l in _directions(rng, 6).tolist() + [[0, 0, -1.0], [0, 0, 1.0], [0.0, 0.0, 0.0]]:
        for Msz in (8, 9, 64, 513, 4096):
            c, r = rng.normal(size=3), rng.uniform(0.01, 100)
            u, v, z = ref.project(c + r * x, l, c, r, Msz)
            # the 2x2 taps never need clamping: 0 <= floor(u) and floor(u) + 1 <= M - 1
            for q in (u, v):
                assert np.all(np.floor(q) >= 0) and np.all(np.floor(q) + 1 <= Msz - 1)
            assert np.all(z >= r * (1 - 1e-12)) and np.all(z <= 3 * r * (1 + 1e-12))


def _banded_point(rng, l, c, r):
    """A point x in the window away from tap boundaries, with a map whose four taps put each smoothstep inside its
    band (0.2 < y < 0.8); every other texel at FAR."""
    while True:
        x = c + _directions(rng, 1)[0] * r * rng.uniform(0, 0.9)
        u, v, z = ref.project(x[None], l, c, r, M)
        idx, fu, fv = ref.taps(u, v, M)
        if not (0.1 < fu[0] < 0.9 and 0.1 < fv[0] < 0.9):
            continue
        D = np.full(M * M, ref.FAR)
        D[idx[0]] = z[0] - BIAS + SOFT * (rng.uniform(0.2, 0.8, 4) - 1)
        return x, D.reshape(M, M), idx[0]


def test_the_visibility_adjoint_matches_complex_steps():
    rng = np.random.default_rng(3)
    h = 1e-30
    for trial in range(60):
        l = _directions(rng, 1)[0] * rng.uniform(0.2, 3)
        if trial == 0:
            l = np.array([0.0, 0.0, -2.0])     # the pole: only d's own derivative
        x, D, idx = _banded_point(rng, l, C0, R0)
        g = rng.normal()
        x_b, l_b, D_b = ref.visibility_b(x[None], l, D, C0, R0, M, BIAS, SOFT, np.array([g]))
        for i in range(3):
            e = np.zeros(3, complex)
            e[i] = 1j * h
            want_x = g * np.imag(ref.visibility((x + e)[None], l, D, C0, R0, M, BIAS, SOFT))[0] / h
            want_l = g * np.imag(ref.visibility(x[None], l + e, D, C0, R0, M, BIAS, SOFT))[0] / h
            assert abs(x_b[0, i] - want_x) <= 1e-9 * max(1.0, abs(want_x))
            assert abs(l_b[i] - want_l) <= 1e-9 * max(1.0, abs(want_l))
        for q in range(4):
            m = D.astype(complex).reshape(-1)
            m[idx[q]] += 1j * h
            want = g * np.imag(ref.visibility(x[None], l, m.reshape(M, M), C0, R0, M, BIAS, SOFT))[0] / h
            assert abs(D_b.reshape(-1)[idx[q]] - want) <= 1e-9 * max(1.0, abs(want))
        assert np.count_nonzero(D_b) <= 4
        # the intensity |l| gets nothing from the shadow
        assert abs(l_b @ l) <= 1e-12 * np.linalg.norm(l_b) * np.linalg.norm(l) + 1e-300


def test_the_projection_adjoint_matches_complex_steps():
    rng = np.random.default_rng(4)
    h = 1e-30
    for _ in range(30):
        l = _directions(rng, 1)[0] * rng.uniform(0.2, 3)
        x = C0 + rng.normal(size=(5, 3))
        gu, gv, gz = rng.normal(size=(3, 5))
        x_b, l_b = ref.project_b(x, l, C0, R0, M, gu, gv, gz)

        def f(xx, ll):
            u, v, z = ref.project(xx, ll, C0, R0, M)
            return gu @ u + gv @ v + gz @ z

        for i in range(3):
            e = np.zeros(3, complex)
            e[i] = 1j * h
            want = np.imag(f(x, l + e)) / h
            assert abs(l_b[i] - want) <= 1e-9 * max(1.0, abs(want))
            for p in range(5):
                xe = x.astype(complex)
                xe[p, i] += 1j * h
                want = np.imag(f(xe, l)) / h
                assert abs(x_b[p, i] - want) <= 1e-9 * max(1.0, abs(want))


def test_points_in_front_of_the_map_are_fully_visible():
    rng = np.random.default_rng(5)
    x = C0 + _directions(rng, 5000) * R0 * rng.uniform(0, 1, (5000, 1))
    for l in _directions(rng, 4):
        z = ref.project(x, l, C0, R0, M)[2]
        for D in (np.full((M, M), z.max()), np.full((M, M), 1.5 * z.max()), np.full((M, M), ref.FAR)):
            assert np.all(ref.visibility(x, l, D, C0, R0, M, BIAS, SOFT) == 1.0)
        V = ref.visibility(x, l, np.full((M, M), 1e-6), C0, R0, M, BIAS, SOFT)
        assert np.all(V[z > 1e-6 + BIAS + SOFT] == 0.0)


def test_the_map_does_not_decide_outside_the_window_nor_without_light():
    rng = np.random.default_rng(6)
    l = _directions(rng, 1)[0]
    D = np.full((M, M), 1e-6)  # everything inside would be shadowed
    outside = C0 + _directions(rng, 100) * R0 * rng.uniform(1.001, 3, (100, 1))
    bad = np.array([[np.nan, 0, 0], [np.inf, 0, 0]])
    for x in (outside, bad):
        assert np.all(ref.visibility(x, l, D, C0, R0, M, BIAS, SOFT) == 1.0)
        x_b, l_b, D_b = ref.visibility_b(x, l, D, C0, R0, M, BIAS, SOFT, np.ones(len(x)))
        assert not np.any(x_b) and not np.any(l_b) and not np.any(D_b)
    inside = C0 + _directions(rng, 100) * R0 * 0.5
    assert np.all(ref.visibility(inside, np.zeros(3), D, C0, R0, M, BIAS, SOFT) == 1.0)
    assert np.all(ref.visibility(inside, l, D, C0, R0, M, BIAS, SOFT) == 0.0)


@pytest.mark.parametrize("C", [1, 3])
def test_the_shaded_product_reduces_to_phong_at_full_visibility(C):
    rng = np.random.default_rng(7 + C)
    ch = phong_ref.random_pixels(rng, C)
    params = np.array([0.3, -0.5, 0.8, 0.4, 0.6, 12.0])
    cam, bg = np.array([0.0, 0.0, -5.0]), rng.uniform(0, 1, C)
    g = rng.normal(size=(ch.shape[0], C))
    ones = np.ones(ch.shape[0])
    assert np.array_equal(ref.shade(ch, params, cam, bg, ones), phong_ref.shade(ch, params, cam, bg))
    ch_b, params_b, _ = ref.shade_b(ch, params, cam, bg, ones, g)
    want_ch, want_params = phong_ref.shade_b(ch, params, cam, bg, g)
    assert np.array_equal(ch_b, want_ch) and np.array_equal(params_b, want_params)


def test_the_shaded_products_visibility_gradient():
    rng = np.random.default_rng(9)
    C = 3
    ch = phong_ref.random_pixels(rng, C, P=512)
    params = np.array([0.3, -0.5, 0.8, 0.4, 0.6, 12.0])
    cam, bg = np.array([0.0, 0.0, -5.0]), rng.uniform(0, 1, C)
    V = rng.uniform(0, 1, ch.shape[0])
    g = rng.normal(size=(ch.shape[0], C))
    _, _, V_b = ref.shade_b(ch, params, cam, bg, V, g)
    h = 1e-30
    want = np.sum(g * np.imag(ref.shade(ch, params, cam, bg, V + 1j * h)) / h, axis=1)
    assert np.allclose(V_b, want, rtol=1e-12, atol=1e-12)
    # and the rest against central differences of the product in the G-buffer and the light
    ch_b, params_b, _ = ref.shade_b(ch, params, cam, bg, V, g)
    on = ch[:, C + 6] == 1
    for k in (0, 1, 2, 3):
        e = np.zeros(6)
        e[k] = 1e-6
        fd = (np.sum(g * ref.shade(ch, params + e, cam, bg, V)) - np.sum(g * ref.shade(ch, params - e, cam, bg, V)))
        assert params_b[k] == pytest.approx(fd / 2e-6, rel=1e-5, abs=1e-6)
    assert np.any(on)
