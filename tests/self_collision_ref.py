"""fp64 numpy restatement of the self-collision energy and of self-intersection detection (include/deodr_b200.h,
"Self-collision"), by brute force over every pair, with a conservative bounding-box prefilter.

Every distance is formed with the kernels' products and sums in the same order (numpy rounds each elementwise
operation on its own, with no fused multiply-add), so d, the orientation signs and the minimum distance equal the
device's bit for bit; only the order of the sums of the energy and the gradient differs."""
from typing import Tuple

import numpy as np


def edges_of(faces: np.ndarray, nb_vertices: int) -> np.ndarray:
    """The unique undirected edges [E,2] (lo, hi), ordered by (lo, hi)."""
    f = np.asarray(faces, dtype=np.int64)
    a, b = f.reshape(-1), f[:, [1, 2, 0]].reshape(-1)
    key = np.unique(np.minimum(a, b) * nb_vertices + np.maximum(a, b))
    return np.stack((key // nb_vertices, key % nb_vertices), axis=1)


def neighbour_keys(faces: np.ndarray, nb_vertices: int) -> np.ndarray:
    """Sorted keys x V + y of the ordered pairs of edge neighbours (x != y)."""
    e = edges_of(faces, nb_vertices)
    e = e[e[:, 0] != e[:, 1]]
    return np.unique(np.concatenate((e[:, 0] * nb_vertices + e[:, 1], e[:, 1] * nb_vertices + e[:, 0])))


def near(keys: np.ndarray, V: int, x: np.ndarray, y: np.ndarray) -> np.ndarray:
    """x == y or x, y edge neighbours, elementwise."""
    k = x * V + y
    i = np.searchsorted(keys, k)
    hit = np.zeros(k.shape, bool)
    ok = i < keys.size
    hit[ok] = keys[i[ok]] == k[ok]
    return (x == y) | hit


def dot(a, b):
    return a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2]


def cross(a, b):
    return np.stack((a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]), axis=-1)


def clamp01(x):
    return np.where(x < 0.0, 0.0, np.where(x > 1.0, 1.0, x))


def closest_point_triangle(p, a, b, c) -> Tuple[np.ndarray, np.ndarray]:
    """Ericson's ClosestPtPointTriangle over arrays [n,3] -> (diff = p - q [n,3], barycentric weights [n,3])."""
    with np.errstate(divide="ignore", invalid="ignore"):
        ab, ac, ap = b - a, c - a, p - a
        d1, d2 = dot(ab, ap), dot(ac, ap)
        bp = p - b
        d3, d4 = dot(ab, bp), dot(ac, bp)
        vc = d1 * d4 - d3 * d2
        cp = p - c
        d5, d6 = dot(ab, cp), dot(ac, cp)
        vb = d5 * d2 - d1 * d6
        va = d3 * d6 - d5 * d4
        e43, e56 = d4 - d3, d5 - d6
        n = p.shape[0]
        one, zero = np.ones(n), np.zeros(n)
        v3 = d1 / (d1 - d3)
        t5 = d2 / (d2 - d6)
        t6 = e43 / (e43 + e56)
        den = 1.0 / ((va + vb) + vc)
        v7, t7 = vb * den, vc * den
        regions = [
            ((d1 <= 0) & (d2 <= 0), ap, (one, zero, zero)),
            ((d3 >= 0) & (d4 <= d3), bp, (zero, one, zero)),
            ((vc <= 0) & (d1 >= 0) & (d3 <= 0), p - (a + ab * v3[:, None]), (1.0 - v3, v3, zero)),
            ((d6 >= 0) & (d5 <= d6), cp, (zero, zero, one)),
            ((vb <= 0) & (d2 >= 0) & (d6 <= 0), p - (a + ac * t5[:, None]), (1.0 - t5, zero, t5)),
            ((va <= 0) & (e43 >= 0) & (e56 >= 0), p - (b + (c - b) * t6[:, None]), (zero, 1.0 - t6, t6)),
            (np.ones(n, bool), p - ((a + ab * v7[:, None]) + ac * t7[:, None]), ((1.0 - v7) - t7, v7, t7)),
        ]
        diff = np.empty_like(p)
        w = np.empty((n, 3))
        todo = np.ones(n, bool)
        for cond, dv, ws in regions:
            m = todo & cond
            diff[m] = dv[m]
            w[m] = np.stack(ws, axis=1)[m]
            todo &= ~m
    return diff, w


def closest_segment_segment(p1, q1, p2, q2) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Ericson's ClosestPtSegmentSegment with EPSILON = 0 over arrays [n,3] -> (diff = c1 - c2, s, t)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        d1, d2, r = q1 - p1, q2 - p2, p1 - p2
        a, e, f = dot(d1, d1), dot(d2, d2), dot(d2, r)
        c = dot(d1, r)
        b = dot(d1, d2)
        denom = a * e - b * b
        s0 = np.where(denom != 0.0, clamp01((b * f - c * e) / denom), 0.0)
        t0 = (b * s0 + f) / e
        lt, gt = t0 < 0.0, t0 > 1.0
        s_gen = np.where(lt, clamp01(-c / a), np.where(gt, clamp01((b - c) / a), s0))
        t_gen = np.where(lt, 0.0, np.where(gt, 1.0, t0))
        A, E = a <= 0.0, e <= 0.0
        s = np.where(A, 0.0, np.where(E, clamp01(-c / a), s_gen))
        t = np.where(A & E, 0.0, np.where(A, clamp01(f / e), np.where(E, 0.0, t_gen)))
    diff = (p1 + d1 * s[:, None]) - (p2 + d2 * t[:, None])
    return diff, s, t


def _box_pairs(lo_a, hi_a, lo_b, hi_b, chunk=256):
    """Index pairs (i, j) whose boxes [lo, hi] overlap (closed), by chunks of rows."""
    out_i, out_j = [], []
    for s in range(0, lo_a.shape[0], chunk):
        la, ha = lo_a[s:s + chunk, None, :], hi_a[s:s + chunk, None, :]
        m = np.all((la <= hi_b[None]) & (lo_b[None] <= ha), axis=2)
        i, j = np.nonzero(m)
        out_i.append(i + s)
        out_j.append(j)
    return np.concatenate(out_i), np.concatenate(out_j)


def vt_pairs(faces, vertices, delta):
    """Candidate vertex-triangle pairs (v, f) after the exclusion: vertices in a face, faces of non-zero area."""
    V = vertices.shape[0]
    f = np.asarray(faces, dtype=np.int64)
    tri = vertices[f]
    area = np.any(cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]) != 0.0, axis=1)
    used = np.zeros(V, bool)
    used[f.reshape(-1)] = True
    r = delta * (1 + 1e-6) + 1e-12
    verts = np.nonzero(used)[0]
    fs = np.nonzero(area)[0]
    i, j = _box_pairs(vertices[verts], vertices[verts], tri[fs].min(axis=1) - r, tri[fs].max(axis=1) + r)
    v, t = verts[i], fs[j]
    keys = neighbour_keys(f, V)
    excl = near(keys, V, f[t, 0], v) | near(keys, V, f[t, 1], v) | near(keys, V, f[t, 2], v)
    return v[~excl], t[~excl]


def ee_pairs(faces, vertices, delta):
    """Candidate edge-edge pairs (e, e') with e < e' after the exclusion."""
    V = vertices.shape[0]
    e = edges_of(faces, V)
    seg = vertices[e]
    r = 0.5 * delta * (1 + 1e-6) + 1e-12
    i, j = _box_pairs(seg.min(axis=1) - r, seg.max(axis=1) + r, seg.min(axis=1) - r, seg.max(axis=1) + r)
    keep = i < j
    i, j = i[keep], j[keep]
    keys = neighbour_keys(faces, V)
    a, b, c, d = e[i, 0], e[i, 1], e[j, 0], e[j, 1]
    excl = near(keys, V, a, c) | near(keys, V, a, d) | near(keys, V, b, c) | near(keys, V, b, d)
    return e, i[~excl], j[~excl]


def candidates(faces, vertices, delta: float):
    """The candidate pairs of :func:`self_collision` (a superset of the pairs closer than delta)."""
    return vt_pairs(faces, vertices, delta), ee_pairs(faces, vertices, delta)


def self_collision(faces, vertices, delta: float, weight: float, cand=None):
    """-> (energy, grad [V,3], min_distance, pairs: dict of the vertex-triangle and edge-edge distances below delta).
    ``cand`` (from :func:`candidates`) fixes the candidate pairs, for finite differences."""
    vertices = np.asarray(vertices, dtype=np.float64)
    f = np.asarray(faces, dtype=np.int64)
    grad = np.zeros_like(vertices)
    energy_terms = []
    dmin = delta
    (v, t), (e, i, j) = cand if cand is not None else candidates(f, vertices, delta)
    diff, w = closest_point_triangle(vertices[v], vertices[f[t, 0]], vertices[f[t, 1]], vertices[f[t, 2]])
    d = np.sqrt(dot(diff, diff))
    m = d < delta
    v, t, diff, w, d = v[m], t[m], diff[m], w[m], d[m]
    energy_terms.append((delta - d) ** 2)
    if d.size:
        dmin = min(dmin, float(d.min()))
    pos = d > 0
    c = 2.0 * weight * (delta - d[pos])
    n = diff[pos] / d[pos, None]
    np.add.at(grad, v[pos], -c[:, None] * n)
    for k in range(3):
        np.add.at(grad, f[t[pos], k], (c * w[pos, k])[:, None] * n)
    vt = {"v": v, "t": t, "d": d}

    diff, s, tt = closest_segment_segment(vertices[e[i, 0]], vertices[e[i, 1]], vertices[e[j, 0]], vertices[e[j, 1]])
    d = np.sqrt(dot(diff, diff))
    m = d < delta
    i, j, diff, s, tt, d = i[m], j[m], diff[m], s[m], tt[m], d[m]
    energy_terms.append((delta - d) ** 2)
    if d.size:
        dmin = min(dmin, float(d.min()))
    pos = d > 0
    c = 2.0 * weight * (delta - d[pos])
    n = diff[pos] / d[pos, None]
    ip, jp, sp, tp = i[pos], j[pos], s[pos], tt[pos]
    np.add.at(grad, e[ip, 0], -(c * (1.0 - sp))[:, None] * n)
    np.add.at(grad, e[ip, 1], -(c * sp)[:, None] * n)
    np.add.at(grad, e[jp, 0], (c * (1.0 - tp))[:, None] * n)
    np.add.at(grad, e[jp, 1], (c * tp)[:, None] * n)
    ee = {"e": i, "f": j, "d": d}
    energy = weight * float(np.sum(np.concatenate(energy_terms)))
    return energy, grad, dmin, {"vt": vt, "ee": ee}


def orient(a, b, c, d):
    return dot(cross(b - a, c - a), d - a)


def _edge_crosses(p, q, a, b, c):
    sp, sq = np.sign(orient(a, b, c, p)), np.sign(orient(a, b, c, q))
    s1, s2, s3 = np.sign(orient(p, q, a, b)), np.sign(orient(p, q, b, c)), np.sign(orient(p, q, c, a))
    return (sp != 0) & (sq != 0) & (sp != sq) & (s1 != 0) & (s1 == s2) & (s2 == s3)


def self_intersections(faces, vertices) -> np.ndarray:
    """Face pairs (i < j) [P,2] int64, sorted, that share no vertex and where an edge of one properly crosses the
    other."""
    vertices = np.asarray(vertices, dtype=np.float64)
    f = np.asarray(faces, dtype=np.int64)
    tri = vertices[f]
    finite = np.all(np.isfinite(tri), axis=(1, 2))
    ids = np.nonzero(finite)[0]
    lo, hi = tri[ids].min(axis=1), tri[ids].max(axis=1)
    i, j = _box_pairs(lo, hi, lo, hi)
    i, j = ids[i], ids[j]
    keep = i < j
    i, j = i[keep], j[keep]
    shared = np.zeros(i.size, bool)
    for a in range(3):
        for b in range(3):
            shared |= f[i, a] == f[j, b]
    i, j = i[~shared], j[~shared]
    x, y = tri[i], tri[j]
    hit = np.zeros(i.size, bool)
    for k in range(3):
        hit |= _edge_crosses(x[:, k], x[:, (k + 1) % 3], y[:, 0], y[:, 1], y[:, 2])
        hit |= _edge_crosses(y[:, k], y[:, (k + 1) % 3], x[:, 0], x[:, 1], x[:, 2])
    pairs = np.stack((i[hit], j[hit]), axis=1)
    return pairs[np.lexsort((pairs[:, 1], pairs[:, 0]))] if pairs.size else pairs.reshape(0, 2)


# ---- meshes -----------------------------------------------------------------------------------------------------------


def icosphere(subdivisions: int = 2):
    """A unit icosphere: (faces [F,3] int64, vertices [V,3])."""
    t = (1.0 + 5 ** 0.5) / 2
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
         [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
         [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10],
         [8, 6, 7], [9, 8, 1]]
    verts = [np.array(p, dtype=np.float64) / np.linalg.norm(p) for p in v]
    faces = [tuple(x) for x in f]
    for _ in range(subdivisions):
        mid = {}

        def midpoint(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                m = verts[a] + verts[b]
                verts.append(m / np.linalg.norm(m))
                mid[k] = len(verts) - 1
            return mid[k]

        nf = []
        for a, b, c in faces:
            ab, bc, ca = midpoint(a, b), midpoint(b, c), midpoint(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        faces = nf
    return np.array(faces, dtype=np.int64), np.array(verts)


def two_spheres(gap: float, subdivisions: int = 2, radius: float = 0.3):
    """Two icospheres of `radius` whose centres are 2 radius + gap apart along x, the second one turned so that no
    vertex faces a vertex: one mesh of two components."""
    from scipy.spatial.transform import Rotation

    f, v = icosphere(subdivisions)
    v = v * radius
    v1 = v - [radius + gap / 2, 0, 0]
    v2 = Rotation.from_euler("xyz", [0.3, 0.2, 0.1]).apply(v) + [radius + gap / 2, 0, 0]
    return np.vstack((f, f + v.shape[0])), np.vstack((v1, v2))


def vertex_normals(faces, vertices):
    f = np.asarray(faces, dtype=np.int64)
    tri = vertices[f]
    fn = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    vn = np.zeros_like(vertices)
    for k in range(3):
        np.add.at(vn, f[:, k], fn)
    return vn / np.maximum(np.linalg.norm(vn, axis=1, keepdims=True), 1e-300)


def hand():
    """The reference's hand (tests/golden/scene_ops.npz): (faces [F,3] int64, vertices [V,3])."""
    import os

    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "scene_ops.npz"))
    return np.asarray(d["hand_faces"], dtype=np.int64), np.asarray(d["hand_vertices"], dtype=np.float64)


def pushed_finger(faces, vertices, gap: float, radius: float = 0.08):
    """The hand with one finger pushed toward its neighbour: the closest vertex-triangle pair outside the one-ring at
    rest (v, closest point q) is found, and the vertices within `radius` of v move along q - v, by d(v, q) - gap at v
    and less farther out, so that v ends about `gap` from the other surface (behind it when gap < 0)."""
    _, _, _, pairs = self_collision(faces, vertices, 0.1, 1.0)
    vt = pairs["vt"]
    k = int(np.argmin(vt["d"]))
    v, t, d0 = int(vt["v"][k]), int(vt["t"][k]), float(vt["d"][k])
    f = np.asarray(faces, dtype=np.int64)
    diff, _ = closest_point_triangle(vertices[[v]], vertices[[f[t, 0]]], vertices[[f[t, 1]]], vertices[[f[t, 2]]])
    u = -diff[0] / np.linalg.norm(diff[0])
    r = np.linalg.norm(vertices - vertices[v], axis=1)
    sel = r < radius
    out = vertices.copy()
    out[sel] += ((d0 - gap) * (1.0 - r[sel] / radius))[:, None] * u
    return out
