"""An fp64 restatement of the tangent-space normal map (the model in include/deodr_b200.h): the per-vertex tangent
frames, the per-pixel perturbation, and both adjoints.  Every forward takes complex inputs too, so that its adjoint can
be checked against complex steps; branches are taken on real parts."""
import numpy as np


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack((a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]), axis=-1)


def unit_or_zero(x):
    """x / |x| along the last axis, 0 where |x| = 0 (|x| = sqrt(<x, x>), analytic for complex steps)."""
    norm = np.sqrt(_dot(x, x))
    ok = norm.real > 0
    return np.where(ok[..., None], x / np.where(ok, norm, 1)[..., None], 0)


def unit_or_zero_b(x, u_b):
    norm = np.sqrt(_dot(x, x).real)
    ok = norm > 0
    safe = np.where(ok, norm, 1)[..., None]
    u = x / safe
    return np.where(ok[..., None], (u_b - u * _dot(u, u_b)[..., None]) / safe, 0)


def face_terms(vertices, faces, uv, faces_uv):
    """-> (e1, e2 [T,3], duv [T,4] = (du1, dv1, du2, dv2), sigma [T], t_f, b_f [T,3])."""
    x = vertices[faces]
    w = uv[faces_uv]
    e1, e2 = x[:, 1] - x[:, 0], x[:, 2] - x[:, 0]
    du1, dv1 = w[:, 1, 0] - w[:, 0, 0], w[:, 1, 1] - w[:, 0, 1]
    du2, dv2 = w[:, 2, 0] - w[:, 0, 0], w[:, 2, 1] - w[:, 0, 1]
    sigma = np.sign((du1 * dv2 - du2 * dv1).real)
    t = sigma[:, None] * (dv2[:, None] * e1 - dv1[:, None] * e2)
    b = sigma[:, None] * (du1[:, None] * e2 - du2[:, None] * e1)
    return e1, e2, np.stack((du1, dv1, du2, dv2), axis=1), sigma, t, b


def _vertex_sums(faces, nb_vertices, t, b):
    """The face terms summed per vertex over its faces in ascending order, with multiplicity (the CSR's order)."""
    dtype = np.result_type(t, b)
    st = np.zeros((nb_vertices, 3), dtype)
    sb = np.zeros((nb_vertices, 3), dtype)
    flat = faces.reshape(-1)
    np.add.at(st, flat, np.repeat(t, 3, axis=0))
    np.add.at(sb, flat, np.repeat(b, 3, axis=0))
    return st, sb


def vertex_frames(vertices, faces, uv, faces_uv):
    """-> frames [V,6] = (T_v, B_v)."""
    _, _, _, _, t, b = face_terms(vertices, faces, uv, faces_uv)
    st, sb = _vertex_sums(faces, vertices.shape[0], t, b)
    return np.concatenate((unit_or_zero(st), unit_or_zero(sb)), axis=1)


def vertex_frames_b(vertices, faces, uv, faces_uv, frames_b):
    """The adjoint of :func:`vertex_frames` -> (vertices_b [V,3], uv_b [Nuv,2])."""
    e1, e2, duv, sigma, t, b = face_terms(vertices, faces, uv, faces_uv)
    st, sb = _vertex_sums(faces, vertices.shape[0], t, b)
    st_b, sb_b = unit_or_zero_b(st, frames_b[:, :3]), unit_or_zero_b(sb, frames_b[:, 3:])
    tb, bb = st_b[faces].sum(axis=1), sb_b[faces].sum(axis=1)
    du1, dv1, du2, dv2 = duv.T
    s = sigma[:, None]
    e1_b = s * (dv2[:, None] * tb - du2[:, None] * bb)
    e2_b = s * (du1[:, None] * bb - dv1[:, None] * tb)
    du1_b, dv1_b = sigma * _dot(e2, bb), -sigma * _dot(e2, tb)
    du2_b, dv2_b = -sigma * _dot(e1, bb), sigma * _dot(e1, tb)
    vertices_b = np.zeros_like(vertices)
    np.add.at(vertices_b, faces[:, 0], -e1_b - e2_b)
    np.add.at(vertices_b, faces[:, 1], e1_b)
    np.add.at(vertices_b, faces[:, 2], e2_b)
    uv_b = np.zeros_like(uv)
    np.add.at(uv_b, faces_uv[:, 0], -np.stack((du1_b + du2_b, dv1_b + dv2_b), axis=1))
    np.add.at(uv_b, faces_uv[:, 1], np.stack((du1_b, dv1_b), axis=1))
    np.add.at(uv_b, faces_uv[:, 2], np.stack((du2_b, dv2_b), axis=1))
    return vertices_b, uv_b


def _frame(g, M):
    N, T, B = g[:, 0:3], g[:, 7:10], g[:, 10:13]
    n = unit_or_zero(N)
    tt = T - _dot(T, n)[:, None] * n
    t = unit_or_zero(tt)
    bt = _cross(n, t)
    s = np.where(_dot(bt, B).real >= 0, 1.0, -1.0)
    p = (M[:, 0:1] * t + M[:, 1:2] * (s[:, None] * bt)) + M[:, 2:3] * n
    return n, tt, t, bt, s, p


def normal_map(g, M):
    """Pixels g [P,13] = (N, X, a, T, B) and the map raster M [P,3] -> [P,7] = (N', X, a)."""
    a = g[:, 6]
    p = _frame(g, M)[-1]
    Np = np.where((a.real != 0)[:, None], a[:, None] * unit_or_zero(p), 0)
    return np.concatenate((Np, g[:, 3:7]), axis=1)


def normal_map_b(g, M, out_b):
    """The adjoint of :func:`normal_map` -> (g_b [P,13], M_b [P,3])."""
    a = g[:, 6]
    n, tt, t, bt, s, p = _frame(g, M)
    Np_b = np.where((a != 0)[:, None], out_b[:, 0:3], 0)
    u = unit_or_zero(p)
    a_b = out_b[:, 6] + _dot(Np_b, u)
    p_b = unit_or_zero_b(p, a[:, None] * Np_b)
    b = s[:, None] * bt
    M_b = np.stack((_dot(p_b, t), _dot(p_b, b), _dot(p_b, n)), axis=1)
    t_b = M[:, 0:1] * p_b
    bt_b = s[:, None] * (M[:, 1:2] * p_b)
    n_b = M[:, 2:3] * p_b + _cross(t, bt_b)
    t_b = t_b + _cross(bt_b, n)
    tt_b = unit_or_zero_b(tt, t_b)
    T = g[:, 7:10]
    ntt_b = _dot(n, tt_b)
    T_b = tt_b - ntt_b[:, None] * n
    n_b = n_b - (_dot(T, n)[:, None] * tt_b + ntt_b[:, None] * T)
    N_b = unit_or_zero_b(g[:, 0:3], n_b)
    g_b = np.concatenate((N_b, out_b[:, 3:6], a_b[:, None], T_b, np.zeros_like(T_b)), axis=1)
    return g_b, M_b
