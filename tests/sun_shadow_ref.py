"""fp64 numpy restatement of the directional light's shadow map of include/deodr_b200.h, written out independently of
the kernels of csrc/scene_ops.cu and csrc/fitter.cu: Frisvad's frame around the light's direction, the orthographic
projection over the caller's window, the soft 2x2 visibility (the taps and smoothstep of tests/shadow_ref.py) and
the shaded product, with the adjoints of the projection and of the visibility in the point, the light and the texels,
and of the product in the visibility.

The forward functions accept complex points, lights and maps (complex-step derivatives); the pole test, the window
test, the tap indices and the smoothstep's clamp read the real parts.
"""

import numpy as np

import phong_ref
from shadow_ref import FAR, smoothstep, taps  # noqa: F401  (FAR: the maps' background depth)

POLE = -0.9999999


def focal(M):
    return M / 2.0 - 2.0


def frame(l):
    """(e1, e2, d) [3] each of the light l [3]: d = l / |l| (+z where |l| = 0) and Frisvad's basis around it."""
    l = np.asarray(l)
    ll = np.sqrt(np.sum(l * l))
    d = l / ll if np.real(ll) > 0 else np.array([0.0, 0.0, 1.0])
    if np.real(d[2]) < POLE:
        return np.array([0.0, -1.0, 0.0]), np.array([-1.0, 0.0, 0.0]), d
    a = 1.0 / (1.0 + d[2])
    b = -d[0] * d[1] * a
    return np.array([1 - d[0] ** 2 * a, b, -d[0]]), np.array([b, 1 - d[1] ** 2 * a, -d[1]]), d


def frame_b(l, e1_b, e2_b, d_b):
    """The adjoint of :func:`frame`: l_b [3] from the gradients of e1, e2 and d (0 where |l| = 0)."""
    l = np.asarray(l, dtype=np.float64)
    ll = np.sqrt(l @ l)
    if not ll > 0:
        return np.zeros(3)
    d = l / ll
    d_b = np.array(d_b, dtype=np.float64)
    if d[2] >= POLE:
        a = 1.0 / (1.0 + d[2])
        x, y = d[0], d[1]
        # e1 = (1 - x^2 a, -x y a, -x), e2 = (-x y a, 1 - y^2 a, -y), da/dz = -a^2
        B = e1_b[1] + e2_b[0]
        d_b[0] += -2 * x * a * e1_b[0] - y * a * B - e1_b[2]
        d_b[1] += -x * a * B - 2 * y * a * e2_b[1] - e2_b[2]
        d_b[2] += a * a * (x * x * e1_b[0] + x * y * B + y * y * e2_b[1])
    return (d_b - d * (d @ d_b)) / ll


def project(x, l, c, r, M):
    """(u, v, z) [P] of points x [P,3] in the map of light l over the window (c, r)."""
    e1, e2, d = frame(l)
    w = np.asarray(x) - np.asarray(c)[None]
    h = (M - 1) / 2.0
    return h + focal(M) * (w @ e1) / r, h + focal(M) * (w @ e2) / r, w @ d + 2 * r


def project_b(x, l, c, r, M, u_b, v_b, z_b):
    """The adjoint of :func:`project` from (u_b, v_b, z_b) [P] -> (x_b [P,3], l_b [3])."""
    e1, e2, d = frame(l)
    w = np.asarray(x, dtype=np.float64) - np.asarray(c)[None]
    k = focal(M) / r
    x_b = k * u_b[:, None] * e1[None] + k * v_b[:, None] * e2[None] + z_b[:, None] * d[None]
    return x_b, frame_b(l, k * (u_b @ w), k * (v_b @ w), z_b @ w)


def _lookup(x, l, D, c, r, M, bias, softness):
    """The test of points x [P,3]; `on` marks those the map decides (finite, inside the sphere, light on)."""
    x = np.asarray(x)
    l = np.asarray(l)
    P = x.shape[0]
    w = np.real(x) - np.asarray(c, dtype=np.float64)[None]
    on = np.all(np.isfinite(np.real(x)), axis=1) & (np.sum(w * w, axis=1) <= r * r) & \
        (np.real(np.sqrt(np.sum(l * l))) > 0)
    V = np.ones(P, dtype=np.result_type(x, l, D, np.float64))
    t = {"on": on, "V": V}
    if not np.any(on):
        return t
    u, v, z = project(x[on], l, c, r, M)
    idx, fu, fv = taps(u, v, M)
    Dt = np.asarray(D).reshape(M * M)[idx]
    s, ds = smoothstep(((Dt + bias) - z[:, None]) / softness + 1.0)
    top = s[:, 0] + fu * (s[:, 1] - s[:, 0])
    bottom = s[:, 2] + fu * (s[:, 3] - s[:, 2])
    V[on] = top + fv * (bottom - top)
    t.update(idx=idx, fu=fu, fv=fv, s=s, ds=ds, top=top, bottom=bottom)
    return t


def visibility(x, l, D, c, r, M, bias, softness):
    """V [P] of points x [P,3] under the map D [M,M] of light l over the window (c, r); 1 where the map does not
    decide."""
    return _lookup(x, l, D, c, r, M, bias, softness)["V"]


def visibility_b(x, l, D, c, r, M, bias, softness, g):
    """The adjoint of :func:`visibility` from g [P] -> (x_b [P,3], l_b [3], D_b [M,M])."""
    x = np.asarray(x, dtype=np.float64)
    t = _lookup(x, l, D, c, r, M, bias, softness)
    on = t["on"]
    x_b, D_b = np.zeros_like(x), np.zeros(M * M)
    if not np.any(on):
        return x_b, np.zeros(3), D_b.reshape(M, M)
    g = np.asarray(g, dtype=np.float64)[on]
    s, fu, fv = t["s"], t["fu"], t["fv"]
    top_b, bottom_b = g * (1 - fv), g * fv
    fv_b = g * (t["bottom"] - t["top"])
    fu_b = top_b * (s[:, 1] - s[:, 0]) + bottom_b * (s[:, 3] - s[:, 2])
    s_b = np.stack((top_b * (1 - fu), top_b * fu, bottom_b * (1 - fu), bottom_b * fu), axis=1)
    tap_b = s_b * t["ds"] / softness
    np.add.at(D_b, t["idx"].reshape(-1), tap_b.reshape(-1))
    xb, l_b = project_b(x[on], l, c, r, M, fu_b, fv_b, -tap_b.sum(axis=1))
    x_b[on] = xb
    return x_b, l_b, D_b.reshape(M, M)


def gbuffer_visibility(positions, coverage, l, D, c, r, M, bias, softness):
    """sun_vis [P] of G-buffer pixels (positions X [P,3], coverage a [P]; x = X / a, 1 where a = 0)."""
    a = np.asarray(coverage, dtype=np.float64)
    on = a != 0
    vis = np.ones(a.shape[0])
    vis[on] = visibility(positions[on] / a[on, None], l, D, c, r, M, bias, softness)
    return vis


def gbuffer_visibility_b(positions, coverage, l, D, c, r, M, bias, softness, vis_b):
    """The adjoint of :func:`gbuffer_visibility` -> (positions_b [P,3], coverage_b [P], D_b [M,M], l_b [3])."""
    a = np.asarray(coverage, dtype=np.float64)
    on = a != 0
    x = positions[on] / a[on, None]
    x_b, l_b, D_b = visibility_b(x, l, D, c, r, M, bias, softness, np.asarray(vis_b)[on])
    pos_b, cov_b = np.zeros((a.shape[0], 3)), np.zeros(a.shape[0])
    pos_b[on] = x_b / a[on, None]
    cov_b[on] = -np.sum(x_b * x, axis=1) / a[on]
    return pos_b, cov_b, D_b, l_b


def _directional(channels, params, cam):
    """(A, diff, spec, ambient, a) of the Phong restatement's pixels."""
    t = phong_ref._terms(channels, params, np.asarray(cam, dtype=np.float64))
    A = np.asarray(channels, dtype=np.float64)[:, :t["C"]]
    with np.errstate(invalid="ignore"):
        diff = np.where(t["dot_nl"] >= 0, 0.0, -t["dot_nl"])  # NaN propagates, as in the luminosity
    return A, diff, t["spec"], float(params[3]), t["a"]


def shade(channels, params, cam, bg, V):
    """image [P, C] = A (ambient + V diff) + V spec + (1 - a) bg (tests/phong_ref.py's model with the directional
    terms scaled by V [P])."""
    A, diff, spec, ambient, a = _directional(channels, params, cam)
    V = np.asarray(V)
    return A * (ambient + V * diff)[:, None] + (V * spec)[:, None] + (1 - a)[:, None] * np.asarray(bg)[None, :]


def shade_b(channels, params, cam, bg, V, image_b):
    """-> (channels_b [P, C + 7], params_b [6], V_b [P]), the adjoint of :func:`shade` from image_b [P, C].  The
    model is linear in the image's gradient: the directional terms take V g, the ambient and background terms g."""
    A, diff, spec, ambient, a = _directional(channels, params, cam)
    g = np.asarray(image_b, dtype=np.float64)
    V = np.asarray(V, dtype=np.float64)
    ch_b, params_b = phong_ref.shade_b(channels, params, cam, bg, V[:, None] * g)
    # the ambient and background terms' share of (1 - V) g
    h = (1 - V)[:, None] * g
    C = A.shape[1]
    ch_b[:, :C] += h * ambient
    params_b[3] += np.sum(h * A)
    ch_b[:, C + 6] -= h @ np.asarray(bg, dtype=np.float64)
    V_b = np.sum(g * (A * diff[:, None] + spec[:, None]), axis=1)
    return ch_b, params_b, V_b
