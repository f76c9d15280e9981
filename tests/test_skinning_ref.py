"""CPU: the fp64 skinning restatement (tests/skinning_ref.py) against scipy's rotations and central differences, and
the host arrays of ``skeleton_arrays`` (levels, children CSR, joint CSR and chunks) with their refusals."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import skinning_ref as ref
from deodr_b200 import _cabi
from deodr_b200.mesh_ops import skeleton_arrays


def _unit(rng):
    u = rng.normal(size=3)
    return u / np.linalg.norm(u)


ANGLES = [0.0, 1e-10, 1e-3, 0.0999999, 0.1, 0.1000001, 0.7, 2.0, np.pi - 1e-3]


@pytest.mark.parametrize("angle", ANGLES)
def test_rotation_is_scipys_rotvec(angle):
    rng = np.random.default_rng(1)
    for _ in range(5):
        theta = angle * _unit(rng)
        np.testing.assert_allclose(ref.rotation(theta), Rotation.from_rotvec(theta).as_matrix(), rtol=0, atol=2e-16 * 8)


def test_rotation_and_its_gradient_are_exact_at_zero():
    assert np.array_equal(ref.rotation(np.zeros(3)), np.eye(3))
    G = np.random.default_rng(2).normal(size=(3, 3))
    got = ref.rotation_b(np.zeros(3), G)
    want = np.array([np.sum(G * ref.skew(e)) for e in np.eye(3)])  # dR/dtheta_k = [e_k]x
    assert np.array_equal(got, want)


@pytest.mark.parametrize("angle", ANGLES)
def test_rotation_b_is_the_derivative(angle):
    rng = np.random.default_rng(3)
    h = 1e-6
    for _ in range(4):
        theta = angle * _unit(rng)
        G = rng.normal(size=(3, 3))
        got = ref.rotation_b(theta, G)
        fd = np.zeros(3)
        for k in range(3):
            e = np.zeros(3)
            e[k] = h
            fd[k] = (np.sum(G * ref.rotation(theta + e)) - np.sum(G * ref.rotation(theta - e))) / (2 * h)
        np.testing.assert_allclose(got, fd, rtol=0, atol=1e-8 * max(1.0, np.abs(fd).max()))


def _tree_case(seed=5, J=24, V=40, K=3):
    """A random branching tree of J joints with two roots (0 and 9) and depth >= 4; joints at theta = 0, at
    |theta| = 1e-10 and near pi among random rotations."""
    rng = np.random.default_rng(seed)
    parents = ref.random_tree(rng, J, roots=(0, 9), min_depth=4)
    centres = rng.normal(size=(J, 3))
    rotations = rng.normal(size=(J, 3)) * 0.8
    rotations[1] = 0.0
    rotations[4] = 1e-10 * _unit(rng)
    rotations[7] = (np.pi - 1e-3) * _unit(rng)
    rotations[9] = 0.0  # a root at rest
    skin_index, skin_weight = ref.random_binding(rng, V, J, K)
    vertices = rng.normal(size=(V, 3))
    g = rng.normal(size=(V, 3))
    return parents, centres, skin_index, skin_weight, vertices, rotations, g


def test_the_tree_has_the_shape_the_checks_need():
    parents = _tree_case()[0]
    assert np.sum(parents < 0) == 2
    arr = skeleton_arrays(parents, np.zeros((24, 3)), np.zeros((1, 1), np.int32), np.ones((1, 1)))
    assert arr["nb_levels"] >= 5
    assert np.max(np.diff(arr["child_offset"])) >= 2  # branching


def test_every_adjoint_output_matches_central_differences():
    parents, centres, idx, w, v, rot, g = _tree_case()
    vb, wb, rb = ref.skin_b(parents, centres, idx, w, v, rot, g)

    def loss(v=v, w=w, rot=rot):
        return float(np.sum(g * ref.skin(parents, centres, idx, w, v, rot)))

    h = 1e-6

    def fd(x, f):
        out = np.zeros_like(x)
        for n in np.ndindex(x.shape):
            xp, xm = x.copy(), x.copy()
            xp[n] += h
            xm[n] -= h
            out[n] = (f(xp) - f(xm)) / (2 * h)
        return out

    for got, want in ((vb, fd(v, lambda x: loss(v=x))), (wb, fd(w, lambda x: loss(w=x))),
                      (rb, fd(rot, lambda x: loss(rot=x)))):
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-7 * np.abs(want).max())
    assert np.abs(rb[[1, 4, 7]]).min() > 0  # the special joints take part


def test_identity_rotations_leave_a_partition_of_unity_at_rest():
    parents, centres, idx, w, v, _, _ = _tree_case()
    out = ref.skin(parents, centres, idx, w, v, np.zeros((len(parents), 3)))
    np.testing.assert_allclose(out, v, rtol=0, atol=1e-14)


def test_skeleton_arrays_builds_the_csrs():
    parents = np.array([-1, 0, 0, 1, -1, 4, 1])
    centres = np.arange(21, dtype=np.float64).reshape(7, 3)
    V, K = 300, 2
    skin_index = np.stack([np.arange(V) % 7, (np.arange(V) + 3) % 7], axis=1)
    skin_index[:, 1][skin_index[:, 0] == 6] = 3
    skin_index[:290, 0] = 1  # joint 1 gets more than one chunk
    w = np.full((V, K), 0.5)
    a = skeleton_arrays(parents, centres, skin_index, w)
    assert a["nb_joints"] == 7 and a["nb_vertices"] == V and a["nb_influences"] == K and a["nb_levels"] == 3
    assert a["level_offset"].tolist() == [0, 2, 5, 7]
    assert a["level_index"].tolist() == [0, 4, 1, 2, 5, 3, 6]
    assert a["child_offset"].tolist() == [0, 2, 4, 4, 4, 5, 5, 5]
    assert a["child_index"].tolist() == [1, 2, 3, 6, 5]
    flat = skin_index.reshape(-1)
    for j in range(7):
        row = a["joint_entry"][a["joint_offset"][j]:a["joint_offset"][j + 1]]
        assert row.tolist() == np.flatnonzero(flat == j).tolist()  # entries i*K+k, ascending
        n_chunks = a["chunk_offset"][j + 1] - a["chunk_offset"][j]
        assert n_chunks == -(-row.size // _cabi.SKIN_CHUNK)
    assert a["chunk_offset"][2] - a["chunk_offset"][1] == 2
    assert a["nb_chunks"] == a["chunk_offset"][-1]
    for name in ("parents", "level_offset", "level_index", "child_offset", "child_index", "skin_index",
                 "joint_offset", "joint_entry", "chunk_offset"):
        assert a[name].dtype == np.int32, name


def test_the_header_constants_are_mirrored():
    import os
    import re

    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                               "deodr_b200.h")).read()
    values = {n: int(v) for n, v in re.findall(r"\b(DEODR_B200_SKIN_[A-Z_]+)\s*=\s*(\d+)", header)}
    assert values == {"DEODR_B200_SKIN_MAX_JOINTS": _cabi.SKIN_MAX_JOINTS,
                      "DEODR_B200_SKIN_MAX_INFLUENCES": _cabi.SKIN_MAX_INFLUENCES,
                      "DEODR_B200_SKIN_CHUNK": _cabi.SKIN_CHUNK}


GOOD = dict(parents=np.array([-1, 0, 1]), joints=np.zeros((3, 3)), skin_index=np.array([[0, 1], [2, 1]]),
            skin_weight=np.full((2, 2), 0.5))


@pytest.mark.parametrize("bad", [
    dict(parents=np.array([-1, 1, 1])),                      # a parent not lower than its joint
    dict(parents=np.array([-1, 0, 3])),
    dict(parents=np.array([0, 0, 1])),                       # joint 0 cannot have a parent
    dict(parents=np.array([-1, -2, 1])),
    dict(skin_index=np.array([[0, 3], [2, 1]])),             # an index outside [0, J)
    dict(skin_index=np.array([[0, -1], [2, 1]])),
    dict(joints=np.array([[0, 0, 0], [np.nan, 0, 0], [0, 0, 0]])),  # a non-finite centre
    dict(skin_weight=np.array([[0.5, np.inf], [0.5, 0.5]])),        # a non-finite weight
    dict(skin_index=np.zeros((2, 9), np.int64), skin_weight=np.zeros((2, 9))),  # K out of range
    dict(skin_index=np.zeros((2, 0), np.int64), skin_weight=np.zeros((2, 0))),
    dict(skin_weight=np.full((2, 3), 0.5)),                  # shapes differ
    dict(joints=np.zeros((2, 3))),
    dict(parents=np.full(1025, -1)),                         # J out of range
    dict(skin_index=np.array([[0.0, 1.0], [2.0, 1.0]])),     # not integers
])
def test_skeleton_arrays_refusals(bad):
    kw = dict(GOOD, **bad)
    with pytest.raises(ValueError):
        skeleton_arrays(**kw)


def test_skeleton_arrays_accepts_the_good_case():
    a = skeleton_arrays(**GOOD)
    assert a["nb_levels"] == 3 and a["nb_chunks"] == 3
