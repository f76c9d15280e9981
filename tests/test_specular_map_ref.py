"""The specular-map restatement (tests/specular_map_ref.py): a map of ones is the view without a map, its adjoint
agrees with central differences and ties to the unmapped model's, and the degenerate pixels stay finite."""
import itertools

import numpy as np
import pytest

import specular_map_ref as ref

C = 3
CAM = np.array([0.0, 0.1, -5.0])
BG = np.array([0.2, 0.3, 0.4])
PARAMS = np.array([0.3, 0.5, 0.8, 0.4, 0.7, 12.0])


def _case(rng, env, lights, vis, sun, P=48):
    G, A, spec = ref.random_pixels(rng, C, P, CAM)
    sh = {None: None, "grey": rng.normal(size=9) * 0.2, "colour": rng.normal(size=(9, C)) * 0.2}[env]
    S = {None: 0, "grey": 1, "colour": C}[lights]
    L = 2
    table = None
    if lights:
        table = np.concatenate((CAM + rng.uniform(-2, 2, (L, 3)), rng.uniform(0.5, 2.0, (L, S))), axis=1)
    V = rng.uniform(0.0, 1.0, (P, L)) if vis and lights else None
    sv = rng.uniform(0.0, 1.0, P) if sun else None
    return dict(G=G, A=A, spec=spec, params=PARAMS, cam=CAM, bg=BG, sh=sh, lights=table, vis=V, sun_vis=sv)


COMBOS = [c for c in itertools.product((None, "grey", "colour"), (None, "grey", "colour"), (False, True),
                                       (False, True)) if c[1] or not c[2]]


def _ones(kw):
    """The case with a map of ones: K = E = a."""
    a = kw["G"][:, 6]
    return dict(kw, spec=np.stack((a, a), axis=1))


@pytest.mark.parametrize("env,lights,vis,sun", COMBOS)
def test_a_map_of_ones_is_the_view_without_a_map(env, lights, vis, sun):
    kw = _ones(_case(np.random.default_rng(1), env, lights, vis, sun))
    assert np.array_equal(ref.shade(**kw), ref.shade(**kw, mapped=False))


@pytest.mark.parametrize("env,lights,vis,sun", COMBOS)
def test_the_adjoint_agrees_with_central_differences(env, lights, vis, sun):
    rng = np.random.default_rng(2)
    kw = _case(rng, env, lights, vis, sun, P=16)
    g = rng.normal(size=(16, C))
    grads = ref.shade_b(g, **kw)
    f = lambda k: np.sum(ref.shade(**k) * g)  # noqa: E731
    for name in ("spec", "G", "params"):
        x = kw[name]
        for idx in [(0, 0), (3, 1), (7, 1)] if name == "spec" else [(2, 6), (5, 3), (9, 0)] if name == "G" else \
                [(4,), (5,), (0,)]:
            h = 1e-6 * max(1.0, abs(x[idx]))
            xp, xm = x.copy(), x.copy()
            xp[idx] += h
            xm[idx] -= h
            fd = (f(dict(kw, **{name: xp})) - f(dict(kw, **{name: xm}))) / (2 * h)
            assert abs(grads[name + "_b"][idx] - fd) <= 1e-6 * max(1.0, abs(fd)), (name, idx)


@pytest.mark.parametrize("env,lights,vis,sun", COMBOS)
def test_with_a_map_of_ones_the_adjoint_ties_to_the_unmapped_model(env, lights, vis, sun):
    """K = E = a: the coverage's total gradient is a_b + K_b + E_b, and a-weighted sums of (K_b, E_b) are ks ks_b and
    e e_b of the view without a map (the texel sums of a map raster of coverage a)."""
    rng = np.random.default_rng(3)
    kw = _ones(_case(rng, env, lights, vis, sun, P=24))
    g = rng.normal(size=(24, C))
    m = ref.shade_b(g, **kw)
    u = ref.shade_b(g, **kw, mapped=False)
    a = kw["G"][:, 6]
    ks, e = PARAMS[4], PARAMS[5]
    tol = 1e-9 * max(1.0, np.abs(u["G_b"]).max())
    assert np.allclose(m["G_b"][:, :6], u["G_b"][:, :6], rtol=0, atol=tol)
    assert np.allclose(m["G_b"][:, 6] + m["spec_b"].sum(axis=1), u["G_b"][:, 6], rtol=0, atol=tol)
    assert np.allclose(m["A_b"], u["A_b"], rtol=0, atol=tol)
    assert np.allclose(m["params_b"][:4], u["params_b"][:4], rtol=1e-9, atol=tol)
    assert np.isclose(np.sum(m["spec_b"][:, 0] * a), ks * u["params_b"][4], rtol=1e-9, atol=tol)
    assert np.isclose(np.sum(m["spec_b"][:, 1] * a), e * u["params_b"][5], rtol=1e-9, atol=tol)
    # the map's chain rule of the issue, with q = K_b / ks and e_b(p) = E_b a / e
    q, eb = m["spec_b"][:, 0] / ks, m["spec_b"][:, 1] * a / e
    spec_b, ks_b, e_b, a_b = ref.map_adjoint(q, eb, kw["G"], kw["spec"], PARAMS)
    assert np.allclose(spec_b, m["spec_b"], rtol=1e-12, atol=0)
    assert np.isclose(ks_b, m["params_b"][4], rtol=1e-9, atol=tol)
    assert np.isclose(e_b, m["params_b"][5], rtol=1e-9, atol=tol)
    if lights:
        assert np.allclose(m["lights_b"], u["lights_b"], rtol=1e-9, atol=tol)


def test_degenerate_pixels():
    """a = 0 shows the background with a zero map gradient; s = 0 (a normal facing away from every half vector), K = 0
    and |l| = 0 give no specular term and finite gradients."""
    rng = np.random.default_rng(4)
    kw = _case(rng, "grey", "grey", True, True, P=8)
    G, spec = kw["G"].copy(), kw["spec"].copy()
    G[0] = 0.0  # a = 0, where the albedo raster is 0 too
    A = kw["A"].copy()
    A[0] = 0.0
    spec[0] = rng.uniform(0.5, 1.0, 2)  # a map sample where nothing is covered is not read
    G[1, 0:3] = np.array([0.0, 0.0, 5.0]) * G[1, 6]  # facing away from the camera and the lights: s = 0
    spec[2, 0] = 0.0  # K = 0
    kw.update(G=G, A=A, spec=spec)
    image = ref.shade(**kw)
    g = np.ones((8, C))
    grads = ref.shade_b(g, **kw)
    assert np.array_equal(image[0], BG)
    assert np.array_equal(grads["spec_b"][0], [0.0, 0.0])
    assert all(np.isfinite(v).all() for v in grads.values())
    no_k = dict(kw, spec=np.stack((np.zeros(8), spec[:, 1]), axis=1))
    no_ks = dict(kw, params=np.concatenate((PARAMS[:4], [0.0, PARAMS[5]])))
    assert np.allclose(ref.shade(**no_k), ref.shade(**no_ks), rtol=0, atol=1e-15)
    dark = dict(kw, params=np.concatenate(([0.0, 0.0, 0.0], PARAMS[3:])), lights=None, vis=None)
    plain = dict(dark, spec=np.zeros_like(spec))
    assert np.array_equal(ref.shade(**dark), ref.shade(**plain))
    assert all(np.isfinite(v).all() for v in ref.shade_b(g, **dark).values())
