"""An fp64 restatement of textured Phong shading with a specular map (the model in include/deodr_b200.h): per pixel,
the map raster's (K, E) give aks = ks K and e(p) = e (E / a) in place of a ks and e, in the directional specular term
and in every point light's, with an optional environment, point lights, their visibilities V_j and the sun's V.

The forward takes complex inputs (branches are taken on real parts), so its derivatives are exact complex steps.
:func:`shade_b` is the adjoint as the Jacobian's transpose applied to the image gradient, each column formed by one
complex step: the pixels are independent, so one step of a per-pixel input perturbs that input in every pixel at once.
It is an exact-derivative oracle for the kernels' hand-written adjoint; :func:`map_adjoint` states the issue's chain
rule for the map on top of it (K_b = q ks, E_b = e_b(p) e / a)."""
import numpy as np

import sh_ref

H_STEP = 1e-30


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _unit(w):
    norm = np.sqrt(_dot(w, w))
    ok = norm.real > 0
    return np.where(ok[..., None], w / np.where(ok, norm, 1)[..., None], 0), norm


def _pow(s, e):
    """s^e where s > 0, 0 elsewhere (with its derivatives)."""
    on = s.real > 0
    return np.where(on, np.where(on, s, 1) ** e, 0)


def shade(G, A, spec, params, cam, bg, sh=None, lights=None, vis=None, sun_vis=None, mapped=True):
    """image [P, C] of G-buffer pixels G [P,7] = (N, X, a), albedo A [P,C] and the map raster spec [P,2] = (K, E).
    ``params`` [6] = (l, ambient, ks, e), ``cam`` [3], ``bg`` [C], ``sh`` [9,S] or None, ``lights`` [L, 3 + S] or
    None, ``vis`` [P,L] (the lights' V_j) or None, ``sun_vis`` [P] or None.  ``mapped=False`` is the view without a
    map (aks = a ks, e(p) = e; ``spec`` is not read)."""
    C = A.shape[1]
    N, X, a = G[:, 0:3], G[:, 3:6], G[:, 6]
    n, _ = _unit(N)
    l = params[0:3]
    ll = np.sqrt(_dot(l, l))
    lit = ll.real > 0
    dot_nl = _dot(n, l[None, :]) if lit else np.zeros(len(a), dtype=n.dtype)
    diff = np.where(dot_nl.real >= 0, 0, -dot_nl)
    V = 1.0 if sun_vis is None else sun_vis
    lum = params[3] + V * diff
    on = a.real != 0
    sa = np.where(on, a, 1)
    if mapped:
        aks, e = params[4] * spec[:, 0], params[5] * (spec[:, 1] / sa)
    else:
        aks, e = a * params[4], params[5] + 0 * a
    x = X / sa[:, None]
    v, _ = _unit(cam[None, :] - x)
    spec_d = np.zeros(len(a), dtype=np.result_type(G, spec, params, cam))
    if lit:
        h, _ = _unit(v - (l / ll)[None, :])
        s = _dot(n, h)
        spec_d = np.where(on, (aks * ll) * _pow(s, e), 0)
    base = lum[:, None] + (0 if sh is None else sh_ref.basis(n) @ sh.reshape(9, -1))
    Pc = Qc = 0
    if lights is not None:
        for j in range(lights.shape[0]):
            d = lights[j, None, 0:3] - x
            w, r = _unit(d)
            r2 = np.where(r.real > 0, r * r, 1)
            cos = _dot(n, w)
            dj = np.where((cos.real > 0) & (r.real > 0), cos / r2, 0)
            hj, _ = _unit(w + v)
            sj = np.where(r.real > 0, _dot(n, hj), 0)
            qj = aks * _pow(sj, e) / r2
            if vis is not None:
                dj, qj = dj * vis[:, j], qj * vis[:, j]
            I = lights[j, 3:]
            Pc = Pc + np.where(on, dj, 0)[:, None] * I[None, :]
            Qc = Qc + np.where(on, qj, 0)[:, None] * I[None, :]
    return A * (base + Pc) + ((V * spec_d)[:, None] + Qc) + (1 - a)[:, None] * bg[None, :C]


INPUTS = ("G", "A", "spec", "vis", "sun_vis")  # per pixel
SHARED = ("params", "cam", "sh", "lights")


def shade_b(image_b, G, A, spec, params, cam, bg, sh=None, lights=None, vis=None, sun_vis=None, mapped=True):
    """The adjoint of :func:`shade` from image_b [P, C] -> dict of the gradients of every given input (G, A, spec,
    vis, sun_vis per pixel; params, cam, sh, lights summed over the pixels), from exact complex steps."""
    args = dict(G=G, A=A, spec=spec, params=params, cam=cam, sh=sh, lights=lights, vis=vis, sun_vis=sun_vis)
    args = {k: (None if v is None else np.asarray(v, dtype=np.float64)) for k, v in args.items()}
    g = np.asarray(image_b, dtype=np.float64)
    bg = np.asarray(bg, dtype=np.float64)

    def run(name, step):
        kw = {k: (None if v is None else v.astype(np.complex128)) for k, v in args.items()}
        kw[name] = kw[name] + 1j * H_STEP * step
        return shade(kw["G"], kw["A"], kw["spec"], kw["params"], kw["cam"], bg, kw["sh"], kw["lights"], kw["vis"],
                     kw["sun_vis"], mapped).imag / H_STEP

    out = {}
    for name, x in args.items():
        if x is None or (name == "spec" and not mapped):
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


def map_adjoint(q, e_b, G, spec, params):
    """The issue's chain rule for the map from q and e_b(p) [P], the gradients of aks(p) and e(p): -> (spec_b [P,2],
    ks_b, e_b (the view's), a_b [P]), 0 where a = 0."""
    a = G[:, 6]
    on = a != 0
    sa = np.where(on, a, 1)
    K, E = spec[:, 0], spec[:, 1]
    ks, e = params[4], params[5]
    spec_b = np.where(on[:, None], np.stack((q * ks, e_b * e / sa), axis=1), 0)
    return spec_b, np.sum(np.where(on, q * K, 0)), np.sum(np.where(on, e_b * E / sa, 0)), \
        np.where(on, -e_b * (e * (E / sa)) / sa, 0)


def random_pixels(rng, C, P=64, cam=(0.0, 0.0, -5.0)):
    """G [P,7], A [P,C] and spec [P,2] of covered pixels (a in (0.2, 1]) facing the camera at ``cam``, with K and E
    = a x a map sample in (0.2, 2)."""
    a = rng.uniform(0.2, 1.0, P)
    N = rng.normal(size=(P, 3)) * 0.3 + np.array([0.0, 0.0, -1.0])
    X = rng.normal(size=(P, 3)) * 0.5
    G = np.concatenate((N * a[:, None], X * a[:, None], a[:, None]), axis=1)
    A = rng.uniform(0.1, 1.0, (P, C)) * a[:, None]
    spec = rng.uniform(0.2, 2.0, (P, 2)) * a[:, None]
    return G, A, spec
