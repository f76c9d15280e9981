"""Self-collision on the device (csrc/collision.cu) against the fp64 restatement (tests/self_collision_ref.py): energy,
gradient, minimum distance and intersections; determinism, re-planning, non-finite input, autograd, and the depth
fitter with the term."""
import os

import numpy as np
import pytest

import self_collision_ref as R
from deodr_b200.scenes import torus_mesh

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
DELTA = 0.02


@pytest.fixture(scope="module")
def torch():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch


@pytest.fixture(scope="module")
def mf(build_native, torch):
    import deodr_b200.mesh_fitter as mf

    return mf


def _torus(n, noise, seed=0, big_r=1.0, small_r=0.4):
    vertices, faces, _ = torus_mesh(n, big_r, small_r)
    faces = faces.astype(np.int64)
    e = R.edges_of(faces, vertices.shape[0])
    h = float(np.median(np.linalg.norm(vertices[e[:, 0]] - vertices[e[:, 1]], axis=1)))
    rng = np.random.default_rng(seed)
    return faces, vertices + noise * h * rng.normal(size=vertices.shape), vertices, 0.5 * h


def _case(name):
    """-> (faces, vertices, vertices_ref, delta)"""
    faces, rest = R.hand()
    if name == "hand_rest":
        return faces, rest, rest, 0.03
    if name == "hand_finger":
        return faces, R.pushed_finger(faces, rest, -0.01), rest, DELTA
    if name == "hand_noise":
        return faces, rest + 0.006 * np.random.default_rng(1).normal(size=rest.shape), rest, DELTA
    if name == "two_spheres":
        f, v = R.two_spheres(0.005)
        return f, v, v, DELTA
    if name == "torus_5k":
        return _torus(50, 0.3)
    raise KeyError(name)


CASES = ["hand_rest", "hand_finger", "hand_noise", "two_spheres", "torus_5k"]


def _run(torch, model, vertices):
    energy, grad = model.evaluate(torch.from_numpy(vertices).cuda())
    torch.cuda.synchronize()
    return float(energy), grad.cpu().numpy(), float(model.min_distance)


@pytest.mark.parametrize("case", CASES)
def test_the_energy_gradient_and_minimum_match_the_restatement(case, torch, mf):
    faces, vertices, ref, delta = _case(case)
    w = 3.0
    e_ref, g_ref, m_ref, pairs = R.self_collision(faces, vertices, delta, w)
    assert e_ref > 0, "the case must have pairs closer than the thickness"
    model = mf.DeviceSelfCollisionEnergy(faces, ref, delta, w)
    e, g, m = _run(torch, model, vertices)
    print(case, "pairs", pairs["vt"]["d"].size, pairs["ee"]["d"].size, "energy", e, "rel", abs(e - e_ref) / e_ref,
          "grad", np.abs(g - g_ref).max() / np.abs(g_ref).max(), "min", m)
    assert abs(e - e_ref) <= 1e-12 * e_ref
    assert np.abs(g - g_ref).max() <= 1e-12 * np.abs(g_ref).max()
    assert m == m_ref
    # added into a given gradient, in place
    base = np.random.default_rng(2).normal(size=g.shape)
    acc = torch.from_numpy(base).cuda()
    model.evaluate(torch.from_numpy(vertices).cuda(), grad=acc, add_to=acc)
    assert np.abs(acc.cpu().numpy() - (base + g_ref)).max() <= 1e-12 * (np.abs(g_ref).max() + np.abs(base).max())


def test_the_rest_hand_at_the_thickness_has_no_energy(torch, mf):
    faces, rest = R.hand()
    model = mf.DeviceSelfCollisionEnergy(faces, rest, DELTA, 1.0)
    e, g, m = _run(torch, model, rest)
    assert e == 0.0 and not g.any() and m == DELTA


@pytest.mark.parametrize("case", ["hand_rest", "hand_noise", "two_spheres_crossed", "spindle_torus"])
def test_the_intersections_match_the_restatement(case, torch, mf):
    if case == "two_spheres_crossed":
        faces, vertices = R.two_spheres(-0.01)
    elif case == "spindle_torus":
        vertices, faces, _ = torus_mesh(40, 1.0, 1.2)
        faces = faces.astype(np.int64)
    else:
        faces, vertices, _, _ = _case(case)
    want = R.self_intersections(faces, vertices)
    model = mf.DeviceSelfCollisionEnergy(faces, vertices, DELTA, 1.0)
    got = model.intersections(torch.from_numpy(vertices).cuda()).cpu().numpy()
    print(case, "pairs", want.shape[0])
    assert got.dtype == np.int64 and np.array_equal(got, want)
    if case in ("two_spheres_crossed", "spindle_torus"):
        assert want.shape[0] > 0


@pytest.mark.parametrize("case", ["hand_noise", "torus_200k"])
def test_repeated_calls_are_bit_identical(case, torch, mf):
    if case == "torus_200k":
        faces, vertices, ref, delta = _torus(316, 0.3)
    else:
        faces, vertices, ref, delta = _case(case)
    model = mf.DeviceSelfCollisionEnergy(faces, ref, delta, 1.0)
    x = torch.from_numpy(vertices).cuda()
    runs = []
    for _ in range(3):
        e, g = model.evaluate(x)
        runs.append((e.clone(), g.clone(), model.min_distance.clone()))
    for e, g, m in runs[1:]:
        assert torch.equal(e, runs[0][0]) and torch.equal(g, runs[0][1]) and torch.equal(m, runs[0][2])
    print(case, "energy", float(runs[0][0]), "min", float(runs[0][2]))
    if case == "torus_200k":
        pairs = model.intersections(x)
        assert torch.equal(pairs, model.intersections(x))


def test_a_grown_plan_gives_the_result_of_a_fresh_object(torch, mf):
    faces, rest = R.hand()
    c = rest.mean(axis=0)
    model = mf.DeviceSelfCollisionEnergy(faces, rest, DELTA, 1.0)
    _run(torch, model, rest)
    for scale in (0.5, 3.0):  # fewer and then more grid entries than the rest mesh's
        v = c + scale * (rest - c)
        got = _run(torch, model, v)
        fresh = _run(torch, mf.DeviceSelfCollisionEnergy(faces, rest, DELTA, 1.0), v)
        e_ref, g_ref, m_ref, _ = R.self_collision(faces, v, DELTA, 1.0)
        assert got[0] == fresh[0] and np.array_equal(got[1], fresh[1]) and got[2] == fresh[2]
        assert abs(got[0] - e_ref) <= 1e-12 * max(e_ref, 1e-300) and got[2] == m_ref


def test_a_non_finite_vertex_gives_a_nan_energy_then_recovers(torch, mf):
    faces, vertices, ref, delta = _case("hand_finger")
    model = mf.DeviceSelfCollisionEnergy(faces, ref, delta, 1.0)
    want = _run(torch, model, vertices)
    for bad in (np.nan, np.inf, 1e300):
        v = vertices.copy()
        v[17, 1] = bad
        e, _, m = _run(torch, model, v)
        if np.isfinite(bad):
            assert np.isfinite(e)  # a huge but finite coordinate: the grid's cells grow to hold it
        else:
            assert np.isnan(e) and np.isnan(m)
        got = _run(torch, model, vertices)
        assert got[0] == want[0] and np.array_equal(got[1], want[1]) and got[2] == want[2]
    assert model.intersections(torch.from_numpy(v).cuda()).shape[1] == 2


def _outside_one_ring(faces, nb_vertices, pairs):
    """The crossing face pairs none of whose vertices are edge neighbours: those the energy's pairs cover.  Faces in
    each other's one-ring are excluded from the energy, so it does not keep them from folding over each other."""
    f = np.asarray(faces)
    p = pairs.cpu().numpy()
    keys = R.neighbour_keys(f, nb_vertices)
    ring = np.zeros(len(p), bool)
    for a in range(3):
        for b in range(3):
            ring |= R.near(keys, nb_vertices, f[p[:, 0], a], f[p[:, 1], b])
    return int((~ring).sum())


def test_autograd_matches_evaluate_and_keeps_a_fit_from_passing_through_itself(torch, mf):
    from deodr_b200.pytorch import SelfCollisionEnergyFunc, SelfCollisionEnergyPytorch

    faces, rest = R.hand()
    energy_model = SelfCollisionEnergyPytorch(faces, rest, DELTA, 1e4)
    v0 = R.pushed_finger(faces, rest, -0.01)
    x = torch.from_numpy(v0).cuda().requires_grad_(True)
    SelfCollisionEnergyFunc.apply(x, energy_model.model).backward()
    _, g = energy_model.model.evaluate(x.detach())
    assert torch.equal(x.grad, g)

    k = 0.08  # the inward offset: past half the fingers' thickness, the target passes through itself
    target = torch.from_numpy(rest - k * R.vertex_normals(faces, rest)).cuda()
    assert R.self_intersections(faces, target.cpu().numpy()).shape[0] > 0

    def fit(with_term, steps=300):
        v = torch.from_numpy(rest.copy()).cuda().requires_grad_(True)
        opt = torch.optim.Adam([v], lr=1e-3)
        crossed, dmins = [], []
        for _ in range(steps):
            opt.zero_grad()
            loss = ((v - target) ** 2).sum()
            if with_term:
                loss = loss + energy_model.evaluate(v)
                dmins.append(float(energy_model.min_distance))
                crossed.append(_outside_one_ring(faces, rest.shape[0], energy_model.intersections(v)))
            loss.backward()
            opt.step()
        return v.detach(), crossed, dmins

    v_free, _, _ = fit(False)
    free_all = energy_model.intersections(v_free)
    free_pairs = _outside_one_ring(faces, rest.shape[0], free_all)
    v_held, crossed, dmins = fit(True)
    held_all = energy_model.intersections(v_held)
    held_pairs = _outside_one_ring(faces, rest.shape[0], held_all)
    print("k", k, "crossing pairs outside the one-ring without the term", free_pairs, "of", free_all.shape[0],
          "; with it, at worst", max(crossed + [held_pairs]), "(one-ring folds at the end:", held_all.shape[0],
          ") smallest min_distance", min(dmins))
    assert free_pairs > 0
    assert max(crossed) == 0 and held_pairs == 0
    assert min(dmins) > 0


def _depth_fitter(mf, inputs, faces, vertices, **kw):
    f = mf.MeshDepthFitter(vertices, faces, np.array([0.1, 0.1, 0.1]), np.zeros(3), cregu=1000, **kw)
    f.set_image(inputs["depth"], focal=241, distortion=np.array([1, 0, 0, 0, 0]))
    f.set_max_depth(1)
    f.set_depth_scale(110 / 450)
    return f


def test_the_depth_fitter_with_the_term(torch, mf):
    inputs = np.load(os.path.join(GOLDEN, "hand_fitting_inputs.npz"))
    faces, vertices = R.hand()
    plain = _depth_fitter(mf, inputs, faces, vertices)
    again = _depth_fitter(mf, inputs, faces, vertices)
    held = _depth_fitter(mf, inputs, faces, vertices, cself=1000.0, self_collision_thickness=DELTA)
    with pytest.raises(ValueError):
        mf.MeshDepthFitter(vertices, faces, np.zeros(3), np.zeros(3), cself=1.0)
    e_plain, e_again, e_held, e_coll = [], [], [], []
    for _ in range(50):
        e_plain.append(float(plain.step()[0]))
        e_again.append(float(again.step()[0]))
        e_held.append(float(held.step()[0]))
        e_coll.append(float(held.energy_self_collision))
    spread = max(abs(a - b) / a for a, b in zip(e_plain, e_again))
    print("collision energy per step:", e_coll)
    print("two runs without the term differ by up to", spread, "relative")
    # step 0 renders the same vertices: bit for bit.  After it, the rasteriser's adjoint sums the fp32 vertex gradients
    # with atomics, whose order varies from run to run, so two runs without the term already differ in the last bits
    assert e_coll[0] == 0.0 and e_held[0] == e_plain[0]
    for s in range(50):
        if any(e_coll[:s + 1]):
            break
        assert abs(e_held[s] - e_plain[s]) <= 1e-6 * e_plain[s], s
    assert all(np.isfinite(e_held))
