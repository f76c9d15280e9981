"""An fp64 restatement of the metallic-roughness (GGX) shading of textured views (the model in include/deodr_b200.h):
per pixel of a G-buffer (N, X, a) with a separate albedo A and an optional map raster (R, M), a GGX highlight and a
Lambert diffuse from the directional light and any point lights, each under its optional visibility, and an
environment that lights the diffuse lobe only.

The forward takes complex inputs (branches are taken on real parts), so its derivatives are exact complex steps.
:func:`shade_b` is the adjoint as the Jacobian's transpose applied to the image gradient, each column formed by one
complex step: the pixels are independent, so one step of a per-pixel input perturbs that input in every pixel at once.
It is an exact-derivative oracle for the kernels' hand-written adjoint."""
import numpy as np

import sh_ref

H_STEP = 1e-30


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _unit(w):
    norm = np.sqrt(_dot(w, w))
    ok = norm.real > 0
    return np.where(ok[..., None], w / np.where(ok, norm, 1)[..., None], 0), norm


def _pos(s):
    """max(0, s), gated on the real part."""
    return np.where(s.real > 0, s, 0)


def ggx_pi_d(nh, k):
    """pi D = k / Dd^2, Dd = nh^2 (k - 1) + 1: GGX's normal distribution times pi, with k = alpha^2 > 0."""
    Dd = nh * nh * (k - 1) + 1
    return k / (Dd * Dd)


def ggx_s(nl, nv, nh, k):
    """S = pi D V = pi D / (Vl Vv), Vl = nl + sqrt(k + (1 - k) nl^2) (Vv alike), with k = alpha^2; 0 where k = 0."""
    on = k.real > 0
    ks = np.where(on, k, 1)
    Vl = nl + np.sqrt(ks + (1 - ks) * nl * nl)
    Vv = nv + np.sqrt(ks + (1 - ks) * nv * nv)
    with np.errstate(divide="ignore", invalid="ignore"):  # Vl = 0 only where nl <= 0, a term that is masked
        return np.where(on, ggx_pi_d(nh, ks) / (Vl * Vv), 0)


def material(G, mr, params):
    """(r, m) per pixel: rf (R / a) and mf (M / a), or the factors alone without a map (mr None)."""
    a = G[:, 6]
    sa = np.where(a.real != 0, a, 1)
    if mr is None:
        R = M = np.ones(len(a))
    else:
        R, M = mr[:, 0] / sa, mr[:, 1] / sa
    return params[5] * R, params[4] * M


def shade(G, A, mr, params, cam, bg, sh=None, lights=None, vis=None, sun_vis=None):
    """image [P, C] of G-buffer pixels G [P,7] = (N, X, a), albedo A [P,C] and the map raster mr [P,2] = (R, M) or
    None.  ``params`` [6] = (l, ambient, mf, rf), ``cam`` [3], ``bg`` [C], ``sh`` [9,S] or None, ``lights`` [L, 3 +
    S] or None, ``vis`` [P,L] (the lights' V_j) or None, ``sun_vis`` [P] or None."""
    C = A.shape[1]
    N, X, a = G[:, 0:3], G[:, 3:6], G[:, 6]
    on = a.real != 0
    sa = np.where(on, a, 1)
    n, _ = _unit(N)
    x = X / sa[:, None]
    v, _ = _unit(cam[None, :] - x)
    b = A / sa[:, None]
    r, m = material(G, mr, params)
    alpha = r * r
    k = alpha * alpha
    F0 = 0.04 * (1 - m)[:, None] + m[:, None] * b
    kd = (1 - m)[:, None]
    terms = []  # (w [P,3], E [P,1 or C])
    l = params[0:3]
    ll = np.sqrt(_dot(l, l))
    if ll.real > 0:
        E = ll * np.ones(len(a), dtype=np.result_type(ll, G))
        if sun_vis is not None:
            E = E * sun_vis
        terms.append((np.broadcast_to(-l / ll, x.shape), E[:, None]))
    if lights is not None:
        for j in range(lights.shape[0]):
            w, rr = _unit(lights[j, None, 0:3] - x)
            ron = rr.real > 0
            E = np.where(ron[:, None], lights[j, None, 3:] / np.where(ron, rr * rr, 1)[:, None], 0)
            if vis is not None:
                E = E * vis[:, j, None]
            terms.append((w, E))
    out = kd * A * (params[3] + (0 if sh is None else sh_ref.basis(n) @ sh.reshape(9, -1)))
    for w, E in terms:
        nl = _dot(n, w)
        lit = nl.real > 0
        nv = _pos(_dot(n, v))
        h, _ = _unit(w + v)
        nh, vh = _pos(_dot(n, h)), _pos(_dot(v, h))
        F = F0 + (1 - F0) * ((1 - vh) ** 5)[:, None]
        S = ggx_s(nl, nv, nh, k)
        with np.errstate(invalid="ignore"):
            t = E * nl[:, None] * ((1 - F) * kd * A + (a * S)[:, None] * F)
        out = out + np.where(lit[:, None], t, 0)
    return np.where(on[:, None], out, 0) + (1 - a)[:, None] * bg[None, :C]


INPUTS = ("G", "A", "mr", "vis", "sun_vis")  # per pixel
SHARED = ("params", "cam", "sh", "lights")


def shade_b(image_b, G, A, mr, params, cam, bg, sh=None, lights=None, vis=None, sun_vis=None):
    """The adjoint of :func:`shade` from image_b [P, C] -> dict of the gradients of every given input (G, A, mr, vis,
    sun_vis per pixel; params, cam, sh, lights summed over the pixels), from exact complex steps."""
    args = dict(G=G, A=A, mr=mr, params=params, cam=cam, sh=sh, lights=lights, vis=vis, sun_vis=sun_vis)
    args = {k: (None if v is None else np.asarray(v, dtype=np.float64)) for k, v in args.items()}
    g = np.asarray(image_b, dtype=np.float64)
    bg = np.asarray(bg, dtype=np.float64)

    def run(name, step):
        kw = {k: (None if v is None else v.astype(np.complex128)) for k, v in args.items()}
        kw[name] = kw[name] + 1j * H_STEP * step
        return shade(kw["G"], kw["A"], kw["mr"], kw["params"], kw["cam"], bg, kw["sh"], kw["lights"], kw["vis"],
                     kw["sun_vis"]).imag / H_STEP

    out = {}
    for name, x in args.items():
        if x is None:
            continue
        grad = np.zeros_like(x)
        if name in INPUTS:
            P = x.shape[0]
            for k in np.ndindex(x.shape[1:]):
                step = np.zeros_like(x)
                step[(slice(None),) + k] = 1
                jac = run(name, step)  # [P, C]: d image[p] / d x[p, k]
                grad[(slice(None),) + k] = np.sum(jac * g, axis=1).reshape(P)
        else:
            for k in np.ndindex(x.shape):
                step = np.zeros_like(x)
                step[k] = 1
                grad[k] = np.sum(run(name, step) * g)
        out[name + "_b"] = grad
    return out


def random_pixels(rng, C, P=64, cam=(0.0, 0.0, -5.0)):
    """G [P,7], A [P,C] and mr [P,2] of covered pixels (a in (0.2, 1]) facing the camera at ``cam``, with (R, M) = a x
    a map sample: roughness in (0.3, 1), metallic in (0, 1)."""
    a = rng.uniform(0.2, 1.0, P)
    N = rng.normal(size=(P, 3)) * 0.3 + np.array([0.0, 0.0, -1.0])
    X = rng.normal(size=(P, 3)) * 0.5
    G = np.concatenate((N * a[:, None], X * a[:, None], a[:, None]), axis=1)
    A = rng.uniform(0.1, 1.0, (P, C)) * a[:, None]
    mr = np.stack((rng.uniform(0.3, 1.0, P), rng.uniform(0.0, 1.0, P)), axis=1) * a[:, None]
    return G, A, mr
