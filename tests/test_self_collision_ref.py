"""The fp64 restatement of the self-collision energy and of self-intersection detection (tests/self_collision_ref.py):
its gradient against central differences, the rest hand, the one-ring exclusion, and detection on a spindle torus."""
import numpy as np
import pytest

import self_collision_ref as R
from deodr_b200.mesh_fitter import collision_mesh_arrays, edge_neighbours
from deodr_b200.scenes import torus_mesh

DELTA = 0.02


def _central_differences(faces, vertices, delta, rows, h=1e-7):
    cand = R.candidates(faces, vertices, delta)
    out = np.zeros((len(rows), 3))
    for n, v in enumerate(rows):
        for k in range(3):
            x = vertices.copy()
            x[v, k] += h
            ep = R.self_collision(faces, x, delta, 1.0, cand)[0]
            x[v, k] -= 2 * h
            em = R.self_collision(faces, x, delta, 1.0, cand)[0]
            out[n, k] = (ep - em) / (2 * h)
    return out


def _away_from_kinks(pairs, delta, margin=1e-4):
    d = np.concatenate((pairs["vt"]["d"], pairs["ee"]["d"]))
    return d.size > 0 and d.min() > margin and np.all(np.abs(d - delta) > margin)


@pytest.mark.parametrize("case", ["pushed_finger", "two_spheres"])
def test_the_gradient_matches_central_differences(case):
    if case == "pushed_finger":
        faces, rest = R.hand()
        vertices = R.pushed_finger(faces, rest, -0.01)
    else:
        faces, vertices = R.two_spheres(0.005, subdivisions=2)
    energy, grad, dmin, pairs = R.self_collision(faces, vertices, DELTA, 1.0)
    assert energy > 0 and dmin < DELTA
    assert _away_from_kinks(pairs, DELTA)
    rows = np.nonzero(np.any(grad != 0, axis=1))[0]
    assert rows.size >= 3
    fd = _central_differences(faces, vertices, DELTA, rows)
    assert np.abs(fd - grad[rows]).max() < 1e-6 * np.abs(grad).max()


def test_the_rest_hand_has_no_energy_at_the_thickness():
    faces, vertices = R.hand()
    energy, grad, dmin, _ = R.self_collision(faces, vertices, DELTA, 1.0)
    assert energy == 0.0 and not grad.any() and dmin == DELTA
    # the closest pairs outside the one-ring, at rest
    _, _, dmin, pairs = R.self_collision(faces, vertices, 0.03, 1.0)
    assert 0.0225 < pairs["vt"]["d"].min() < 0.0227 and 0.0225 < pairs["ee"]["d"].min() < 0.0227


def _bfs_rings(faces, V):
    adj = [set() for _ in range(V)]
    for a, b, c in np.asarray(faces):
        for x, y in ((a, b), (b, c), (c, a)):
            if x != y:
                adj[x].add(int(y))
                adj[y].add(int(x))
    return [adj[v] | {v} for v in range(V)]


@pytest.mark.parametrize("mesh", ["icosphere", "hand"])
def test_the_excluded_pairs_are_the_breadth_first_one_ring(mesh):
    faces, vertices = R.icosphere(1) if mesh == "icosphere" else R.hand()
    V = vertices.shape[0]
    ring = _bfs_rings(faces, V)
    offset, index = edge_neighbours(faces, V)
    for v in range(V):
        assert sorted(ring[v] - {v}) == index[offset[v]:offset[v + 1]].tolist()
    keys = R.neighbour_keys(faces, V)
    rng = np.random.default_rng(0)
    f = np.asarray(faces)
    vv = rng.integers(0, V, 20000)
    tt = rng.integers(0, f.shape[0], 20000)
    got = R.near(keys, V, f[tt, 0], vv) | R.near(keys, V, f[tt, 1], vv) | R.near(keys, V, f[tt, 2], vv)
    want = np.array([any(v in ring[c] for c in f[t]) for v, t in zip(vv, tt)])
    assert np.array_equal(got, want) and want.any() and not want.all()
    e = R.edges_of(faces, V)
    assert np.array_equal(e, collision_mesh_arrays(faces, V)["edges"])
    i, j = rng.integers(0, e.shape[0], 20000), rng.integers(0, e.shape[0], 20000)
    got = (R.near(keys, V, e[i, 0], e[j, 0]) | R.near(keys, V, e[i, 0], e[j, 1]) | R.near(keys, V, e[i, 1], e[j, 0])
           | R.near(keys, V, e[i, 1], e[j, 1]))
    want = np.array([any(y in ring[x] for x in e[a] for y in e[b]) for a, b in zip(i, j)])
    assert np.array_equal(got, want) and want.any() and not want.all()


def test_the_collision_mesh_csrs():
    faces, vertices = R.two_spheres(0.01, subdivisions=1)
    arr = collision_mesh_arrays(faces, vertices.shape[0])
    V = vertices.shape[0]
    flat = np.asarray(faces).reshape(-1)
    for v in range(V):
        corners = arr["corner_index"][arr["corner_offset"][v]:arr["corner_offset"][v + 1]]
        assert np.all(flat[corners] == v) and np.all(np.diff(corners) > 0)
        ends = arr["end_index"][arr["end_offset"][v]:arr["end_offset"][v + 1]]
        assert np.all(arr["edges"].reshape(-1)[ends] == v) and np.all(np.diff(ends) > 0)
    assert arr["corner_offset"][-1] == flat.size and arr["end_offset"][-1] == 2 * arr["nb_edges"]


def _moller_trumbore(p, q, a, b, c, eps):
    """Segment p-q against triangle a, b, c by Moller-Trumbore: -> (clearly crossing, possibly crossing)."""
    d = q - p
    e1, e2 = b - a, c - a
    h = np.cross(d, e2)
    det = np.einsum("ij,ij->i", e1, h)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / det
        s = p - a
        u = inv * np.einsum("ij,ij->i", s, h)
        qv = np.cross(s, e1)
        v = inv * np.einsum("ij,ij->i", d, qv)
        t = inv * np.einsum("ij,ij->i", e2, qv)
        ok = np.abs(det) > 1e-14
        clear = ok & (u > eps) & (v > eps) & (u + v < 1 - eps) & (t > eps) & (t < 1 - eps)
        maybe = ok & (u > -eps) & (v > -eps) & (u + v < 1 + eps) & (t > -eps) & (t < 1 + eps)
    return clear, maybe


def test_detection_on_a_spindle_torus_and_the_rest_hand():
    vertices, faces, _ = torus_mesh(40, 1.0, 1.2)
    faces = faces.astype(np.int64)
    pairs = R.self_intersections(faces, vertices)
    assert pairs.shape[0] > 0
    # every candidate pair by an independent segment-triangle test: clear crossings are reported, reported ones cross
    tri = vertices[faces]
    i, j = np.triu_indices(faces.shape[0], 1)
    lo, hi = tri.min(axis=1), tri.max(axis=1)
    keep = np.all((lo[i] <= hi[j]) & (lo[j] <= hi[i]), axis=1)
    i, j = i[keep], j[keep]
    shared = np.zeros(i.size, bool)
    for x in range(3):
        for y in range(3):
            shared |= faces[i, x] == faces[j, y]
    i, j = i[~shared], j[~shared]
    clear = np.zeros(i.size, bool)
    maybe = np.zeros(i.size, bool)
    for k in range(3):
        for s, o in ((i, j), (j, i)):
            c, m = _moller_trumbore(tri[s, k], tri[s, (k + 1) % 3], tri[o, 0], tri[o, 1], tri[o, 2], 1e-9)
            clear |= c
            maybe |= m
    reported = {tuple(p) for p in pairs.tolist()}
    assert {(a, b) for a, b in zip(i[clear].tolist(), j[clear].tolist())} <= reported
    assert reported <= {(a, b) for a, b in zip(i[maybe].tolist(), j[maybe].tolist())}
    # near the two spindle points on the axis, z = +-sqrt(1.2^2 - 1)
    centres = tri[pairs.reshape(-1)].mean(axis=1)
    assert np.all(np.hypot(centres[:, 0], centres[:, 1]) < 0.4)
    hf, hv = R.hand()
    assert R.self_intersections(hf, hv).shape == (0, 2)
