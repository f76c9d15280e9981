"""The metallic-roughness restatement (tests/pbr_ref.py): its adjoint agrees with central differences, its pi-cancelled
highlight is glTF's literal product, its D is normalised, it reduces as the model says, and the degenerate pixels
stay finite."""
import itertools

import numpy as np
import pytest
from scipy.integrate import quad

import pbr_ref as ref

C = 3
CAM = np.array([0.0, 0.1, -5.0])
BG = np.array([0.2, 0.3, 0.4])
PARAMS = np.array([0.3, 0.5, 0.8, 0.4, 0.6, 0.5])  # l, ambient, mf, rf


def _case(rng, env, lights, vis, sun, mapped, P=48):
    G, A, mr = ref.random_pixels(rng, C, P, CAM)
    sh = {None: None, "grey": rng.normal(size=9) * 0.2, "colour": rng.normal(size=(9, C)) * 0.2}[env]
    S = {None: 0, "grey": 1, "colour": C}[lights]
    L = 2
    table = None
    if lights:
        table = np.concatenate((CAM + rng.uniform(-2, 2, (L, 3)), rng.uniform(0.5, 2.0, (L, S))), axis=1)
    V = rng.uniform(0.0, 1.0, (P, L)) if vis and lights else None
    sv = rng.uniform(0.0, 1.0, P) if sun else None
    return dict(G=G, A=A, mr=mr if mapped else None, params=PARAMS, cam=CAM, bg=BG, sh=sh, lights=table, vis=V,
                sun_vis=sv)


COMBOS = [c for c in itertools.product((None, "grey", "colour"), (None, "grey", "colour"), (False, True),
                                       (False, True), (False, True)) if c[1] or not c[2]]


@pytest.mark.parametrize("env,lights,vis,sun,mapped", COMBOS)
def test_the_adjoint_agrees_with_central_differences(env, lights, vis, sun, mapped):
    rng = np.random.default_rng(2)
    kw = _case(rng, env, lights, vis, sun, mapped, P=16)
    g = rng.normal(size=(16, C))
    grads = ref.shade_b(g, **kw)
    f = lambda k: np.sum(ref.shade(**k) * g)  # noqa: E731
    names = ["G", "A", "params", "cam"] + (["mr"] if mapped else []) + (["lights"] if lights else []) + \
        (["vis"] if vis and lights else []) + (["sun_vis"] if sun else []) + (["sh"] if env else [])
    for name in names:
        x = kw[name]
        for n in range(3):
            idx = tuple(int(i) for i in np.unravel_index((7 * n + 3) % x.size, x.shape))
            h = 1e-6 * max(1.0, abs(x[idx]))
            xp, xm = x.copy(), x.copy()
            xp[idx] += h
            xm[idx] -= h
            fd = (f(dict(kw, **{name: xp})) - f(dict(kw, **{name: xm}))) / (2 * h)
            got = grads[name + "_b"][idx]
            assert abs(got - fd) <= 1e-6 * max(1.0, abs(fd)), (name, idx, got, fd)


def test_the_pi_cancelled_highlight_is_gltf_literal_product():
    """S F = pi F D G / (4 nl nv), with glTF 2.0 Appendix B's D and G = G1(l) G1(v) written out independently."""
    rng = np.random.default_rng(3)
    nl, nv, nh = rng.uniform(0.05, 1.0, (3, 1000))
    alpha = rng.uniform(0.05, 1.0, 1000)
    F = rng.uniform(0.04, 1.0, 1000)
    a2 = alpha ** 2
    D = a2 / (np.pi * (nh ** 2 * (a2 - 1) + 1) ** 2)

    def G1(c):
        return 2 * c / (c + np.sqrt(a2 + (1 - a2) * c ** 2))

    literal = np.pi * F * D * G1(nl) * G1(nv) / (4 * nl * nv)
    ours = ref.ggx_s(nl, nv, nh, a2) * F  # k = alpha^2
    assert np.max(np.abs(ours - literal) / np.abs(literal)) < 1e-12


@pytest.mark.parametrize("alpha", [0.1, 0.5, 1.0])
def test_the_restated_d_is_normalised(alpha):
    """integral of D(h) <n, h> over the hemisphere = 1, with the restatement's pi D (ggx_pi_d, the D of ggx_s)."""
    k = alpha ** 2

    def integrand(mu):  # 2 pi D mu over d(mu), mu = <n, h>
        return 2.0 * float(ref.ggx_pi_d(np.array(mu), np.array(k))) * mu

    total, _ = quad(integrand, 0.0, 1.0, points=[1.0 - alpha], limit=200, epsabs=1e-13, epsrel=1e-13)
    assert abs(total - 1.0) < 1e-6


def test_fresnel_is_f0_at_normal_incidence_and_diffuse_vanishes_for_metal():
    """vh = 1 (light and view along the normal) gives F = F0; m = 1 leaves no diffuse or ambient."""
    G = np.array([[0.0, 0.0, -1.0, 0.0, 0.0, 0.0, 1.0]])
    A = np.array([[0.6, 0.3, 0.2]])
    params = np.array([0.0, 0.0, 2.0, 0.3, 0.0, 0.5])  # light along +z (toward the camera side: w = -z), m = 0
    b = A[0]
    F0 = 0.04
    alpha2 = 0.5 ** 4
    expected = 2.0 * ((1 - F0) * b + F0 / (4 * alpha2)) + b * 0.3
    got = ref.shade(G, A, None, params, np.array([0.0, 0.0, -5.0]), BG)[0]
    assert np.allclose(got, expected, rtol=1e-12)
    metal = params.copy()
    metal[4] = 1.0
    got = ref.shade(G, A, None, metal, np.array([0.0, 0.0, -5.0]), BG)[0]
    assert np.allclose(got, 2.0 * b / (4 * alpha2), rtol=1e-12)  # F0 = b, no diffuse, no ambient


@pytest.mark.parametrize("env,lights,vis,sun,mapped", [c for c in COMBOS if c[4]])
def test_a_map_of_ones_is_the_factors_alone(env, lights, vis, sun, mapped):
    kw = _case(np.random.default_rng(1), env, lights, vis, sun, mapped)
    a = kw["G"][:, 6]
    ones = dict(kw, mr=np.stack((a, a), axis=1))
    assert np.array_equal(ref.shade(**ones), ref.shade(**dict(kw, mr=None)))


def _finite(kw, g):
    image = ref.shade(**kw)
    grads = ref.shade_b(g, **kw)
    assert np.all(np.isfinite(image))
    for v in grads.values():
        assert np.all(np.isfinite(v))
    return image, grads


def test_degenerate_pixels():
    rng = np.random.default_rng(4)
    G, A, mr = ref.random_pixels(rng, C, 8, CAM)
    lights = np.array([[0.0, 0.0, -4.0, 1.0], [0.3, 0.2, -3.0, 0.5]])
    kw = dict(G=G, A=A, mr=mr, params=PARAMS, cam=CAM, bg=BG, sh=rng.normal(size=9) * 0.2, lights=lights,
              vis=rng.uniform(0, 1, (8, 2)), sun_vis=rng.uniform(0, 1, 8))
    G[0, 6] = 0.0  # a = 0
    G[0, :6] = rng.normal(size=6)
    A[0] = 0.0
    mr[0] = 0.0
    G[1, 0:3] = 0.0  # |N| = 0
    G[2, 0:3] = np.array([0.0, 0.0, 1.0]) * G[2, 6]  # facing away: nl <= 0 for every light
    G[3, 0:3] = np.array([1.0, 0.0, 0.0]) * G[3, 6]  # grazing: nv = 0 (the camera is on the z axis, x near 0)
    G[3, 3:6] = np.array([0.0, 0.1, 0.0]) * G[3, 6]
    g = rng.normal(size=(8, C))
    image, grads = _finite(kw, g)
    assert np.array_equal(image[0], BG)
    for name in ("A_b", "mr_b", "vis_b", "sun_vis_b"):
        assert np.all(grads[name][0] == 0), name
    assert np.all(grads["G_b"][0, :6] == 0)
    # |l| = 0 and no other light: the environment's diffuse and the background alone
    off = dict(kw, params=np.array([0.0, 0.0, 0.0] + list(PARAMS[3:])), lights=None, vis=None)
    image, _ = _finite(off, g)
    n = G[:, 0:3] / np.maximum(np.linalg.norm(G[:, 0:3], axis=1), 1e-300)[:, None]
    r, m = ref.material(G, mr, PARAMS)
    env = PARAMS[3] + ref.sh_ref.basis(n) @ kw["sh"].reshape(9, 1)
    want = np.where(G[:, 6:7] != 0, (1 - m)[:, None] * A * env, 0) + (1 - G[:, 6:7]) * BG[None, :]
    assert np.allclose(image, want, rtol=1e-12, atol=1e-15)
    # alpha = 0: no highlight, so a pure metal without an environment shows the background's share only
    metal = dict(kw, mr=None, sh=None, params=np.array(list(PARAMS[:3]) + [0.4, 1.0, 0.0]), lights=None, vis=None)
    image, _ = _finite(metal, g)
    assert np.array_equal(image, (1 - G[:, 6])[:, None] * BG[None, :])
    # w + v = 0: the directional light's w exactly opposite the view, on a surface facing the light
    G2 = G.copy()
    G2[5, 0:3] = np.array([0.0, 0.0, 1.0]) * G2[5, 6]
    G2[5, 3:6] = 0.0
    opposite = dict(kw, G=G2, cam=np.array([0.0, 0.0, -5.0]), params=np.array([0.0, 0.0, -1.0] + list(PARAMS[3:])),
                    lights=None, vis=None, sh=None)
    image, _ = _finite(opposite, g)
    # h = 0, so nh = vh = 0 and F = 1; nl = 1 and nv = 0: the term is E a S = E a k / (2 sqrt(k)) (Dd = 1, Vl = 2,
    # Vv = sqrt(k)), with E = |l| V = V
    a5 = G2[5, 6]
    k = r[5] ** 4
    want = kw["sun_vis"][5] * a5 * k / (2 * np.sqrt(k)) + (1 - m[5]) * A[5] * PARAMS[3] + (1 - a5) * BG
    assert np.allclose(image[5], want, rtol=1e-12)
