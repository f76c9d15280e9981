"""fp64 numpy restatement of the point lights' cube shadow maps of include/deodr_b200.h, written out independently of
the kernels of csrc/scene_ops.cu: the six face cameras, the face a point looks up, its projection, the 2x2 taps, the
clamped smoothstep and the visibility, with the adjoint of the visibility in the point, the light's position and the
map texels.

The forward functions accept complex points, positions and maps (complex-step derivatives); the face choice, the tap
indices and the smoothstep's clamp read the real parts.
"""

import numpy as np

FAR = 1e30

# rows of R_k (the face camera's x, y and z axes in world coordinates) for the faces +x, -x, +y, -y, +z, -z
ROTATIONS = np.array([
    [[0, 1, 0], [0, 0, 1], [1, 0, 0]],
    [[0, 0, 1], [0, 1, 0], [-1, 0, 0]],
    [[0, 0, 1], [1, 0, 0], [0, 1, 0]],
    [[1, 0, 0], [0, 0, 1], [0, -1, 0]],
    [[1, 0, 0], [0, 1, 0], [0, 0, 1]],
    [[0, 1, 0], [1, 0, 0], [0, 0, -1]],
], dtype=np.float64)


def focal(M):
    return M / 2.0 - 2.0


def camera(p, k, M):
    """The camera vector [26] of face k of the cube around p (extrinsic [R_k | -R_k p], intrinsic, no distortion)."""
    R = ROTATIONS[k]
    ext = np.concatenate((R, -(R @ np.asarray(p, dtype=np.float64))[:, None]), axis=1)
    c = (M - 1) / 2.0
    K = np.array([[focal(M), 0, c], [0, focal(M), c], [0, 0, 1.0]])
    return np.concatenate((ext.reshape(-1), K.reshape(-1), np.zeros(5)))


def cameras(lights, M):
    """[6L, 26]: face 6 j + k of light j."""
    return np.stack([camera(l[:3], k, M) for l in np.asarray(lights) for k in range(6)])


def face_of(d):
    """The face k [P] of directions d [P,3] from the light: the dominant axis with its sign, ties to x, then y, then z."""
    a = np.abs(np.real(d))
    axis = np.where((a[:, 0] >= a[:, 1]) & (a[:, 0] >= a[:, 2]), 0, np.where(a[:, 1] >= a[:, 2], 1, 2))
    da = np.real(d)[np.arange(d.shape[0]), axis]
    return 2 * axis + np.where(da > 0, 0, 1)


def project(x, p, k, M):
    """(u, v, z) [P] of points x [P,3] through face k [P] of the cube around p."""
    R = ROTATIONS[k]                                           # [P,3,3]
    pc = np.einsum("pij,pj->pi", R, x - np.asarray(p)[None])  # R (x - p) = R x + t
    c = (M - 1) / 2.0
    return focal(M) * pc[:, 0] / pc[:, 2] + c, focal(M) * pc[:, 1] / pc[:, 2] + c, pc[:, 2]


def smoothstep(y):
    """s(y) = 3 y^2 - 2 y^3 on y clamped to [0, 1], and s'(y) (0 outside (0, 1))."""
    inside = (np.real(y) > 0) & (np.real(y) < 1)
    s = np.where(inside, y * y * (3 - 2 * y), np.where(np.real(y) >= 1, 1.0, 0.0))
    return s, np.where(inside, 6 * y * (1 - y), 0.0)


def taps(u, v, M):
    """(flat indices [P,4] into an M x M map of the taps 00, 10, 01, 11, fu, fv)."""
    u0, v0 = np.floor(np.real(u)), np.floor(np.real(v))
    c0, c1 = np.clip(u0, 0, M - 1).astype(np.int64), np.clip(u0 + 1, 0, M - 1).astype(np.int64)
    r0, r1 = np.clip(v0, 0, M - 1).astype(np.int64), np.clip(v0 + 1, 0, M - 1).astype(np.int64)
    return np.stack((r0 * M + c0, r0 * M + c1, r1 * M + c0, r1 * M + c1), axis=1), u - u0, v - v0


def _lookup(x, p, maps, M, bias, softness):
    x = np.asarray(x)
    k = face_of(x - np.asarray(p)[None])
    u, v, z = project(x, p, k, M)
    idx, fu, fv = taps(u, v, M)
    D = np.asarray(maps).reshape(6, M * M)[k[:, None], idx]    # [P,4]
    y = ((D + bias) - z[:, None]) / softness + 1.0
    s, ds = smoothstep(y)
    top = s[:, 0] + fu * (s[:, 1] - s[:, 0])
    bottom = s[:, 2] + fu * (s[:, 3] - s[:, 2])
    return dict(k=k, u=u, v=v, z=z, idx=idx, fu=fu, fv=fv, s=s, ds=ds, top=top, bottom=bottom,
                V=top + fv * (bottom - top))


def visibility(x, p, maps, M, bias, softness):
    """V [P] of points x [P,3] under the six maps [6,M,M] of a light at p (every point in front of its face)."""
    return _lookup(x, p, maps, M, bias, softness)["V"]


def visibility_b(x, p, maps, M, bias, softness, g):
    """The adjoint of :func:`visibility` from g [P] -> (x_b [P,3], p_b [3], maps_b [6,M,M])."""
    t = _lookup(x, p, maps, M, bias, softness)
    g = np.asarray(g, dtype=np.float64)
    top_b, bottom_b = g * (1 - t["fv"]), g * t["fv"]
    fv_b = g * (t["bottom"] - t["top"])
    s = t["s"]
    fu_b = top_b * (s[:, 1] - s[:, 0]) + bottom_b * (s[:, 3] - s[:, 2])
    s_b = np.stack((top_b * (1 - t["fu"]), top_b * t["fu"], bottom_b * (1 - t["fu"]), bottom_b * t["fu"]), axis=1)
    D_b = s_b * t["ds"] / softness                              # [P,4]
    z_b = -D_b.sum(axis=1)
    maps_b = np.zeros(6 * M * M)
    np.add.at(maps_b, (t["k"][:, None] * M * M + t["idx"]).reshape(-1), D_b.reshape(-1))
    # (u, v, z) = (phi pc0 / pc2 + c, phi pc1 / pc2 + c, pc2), pc = R (x - p)
    R = ROTATIONS[t["k"]]
    pc = np.einsum("pij,pj->pi", R, np.asarray(x) - np.asarray(p)[None])
    phi = focal(M)
    pc_b = np.stack((fu_b * phi / pc[:, 2], fv_b * phi / pc[:, 2],
                     z_b - (fu_b * phi * pc[:, 0] + fv_b * phi * pc[:, 1]) / pc[:, 2] ** 2), axis=1)
    x_b = np.einsum("pij,pi->pj", R, pc_b)
    return x_b, -x_b.sum(axis=0), maps_b.reshape(6, M, M)


def gbuffer_visibility(positions, coverage, lights, maps, M, bias, softness):
    """vis [P, L] of G-buffer pixels (positions X [P,3], coverage a [P]; x = X / a, 1 where a = 0) under the maps
    [6L, M, M] of the lights [L, 3 + S]."""
    a = np.asarray(coverage, dtype=np.float64)
    on = a != 0
    x = positions[on] / a[on, None]
    vis = np.ones((a.shape[0], len(lights)))
    for j, l in enumerate(np.asarray(lights)):
        vis[on, j] = visibility(x, l[:3], maps[6 * j:6 * j + 6], M, bias, softness)
    return vis


def gbuffer_visibility_b(positions, coverage, lights, maps, M, bias, softness, vis_b):
    """The adjoint of :func:`gbuffer_visibility` -> (positions_b [P,3], coverage_b [P], maps_b [6L,M,M], lights_b
    [L,3]): x = X / a gives X_b = x_b / a and a_b = -<x_b, x> / a."""
    a = np.asarray(coverage, dtype=np.float64)
    on = a != 0
    x = positions[on] / a[on, None]
    x_b = np.zeros_like(x)
    maps_b = np.zeros_like(np.asarray(maps, dtype=np.float64))
    lights_b = np.zeros((len(lights), 3))
    for j, l in enumerate(np.asarray(lights)):
        xb, pb, mb = visibility_b(x, l[:3], maps[6 * j:6 * j + 6], M, bias, softness, vis_b[on, j])
        x_b += xb
        lights_b[j] = pb
        maps_b[6 * j:6 * j + 6] = mb
    pos_b = np.zeros((a.shape[0], 3))
    cov_b = np.zeros(a.shape[0])
    pos_b[on] = x_b / a[on, None]
    cov_b[on] = -np.sum(x_b * x, axis=1) / a[on]
    return pos_b, cov_b, maps_b, lights_b
