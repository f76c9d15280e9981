"""Linear blend skinning on the device (csrc/skinning.cu) against the fp64 restatement (tests/skinning_ref.py):
forward, every adjoint output, determinism and autograd; and articulated fits of a procedural tube with the device
fitter and with Adam through ``LinearBlendSkinningFunc``, with and without the self-collision term."""
import numpy as np
import pytest

import skinning_ref as ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch


@pytest.fixture(scope="module")
def ops(build_native, torch):
    import deodr_b200.mesh_ops as ops

    return ops


def _case(V, J, K, seed=0):
    rng = np.random.default_rng(seed)
    roots = (0, J // 2) if J > 3 else (0,)
    parents = ref.random_tree(rng, J, roots=roots, min_depth=min(4, J - len(roots)))
    centres = rng.normal(size=(J, 3))
    rotations = rng.normal(size=(J, 3)) * 0.8
    if J > 8:
        rotations[1] = 0.0
        rotations[4] = 1e-10 * rng.normal(size=3) / np.sqrt(3)
        rotations[7] = (np.pi - 1e-3) * np.array([0.6, 0.0, 0.8])
    if K <= J:
        skin_index, skin_weight = ref.random_binding(rng, V, J, K)
    else:
        skin_index = rng.integers(0, J, size=(V, K)).astype(np.int32)
        skin_weight = rng.uniform(0.1, 1.0, size=(V, K))
    if J > 8:
        skin_index[skin_index == 5] = 6  # a joint without influences
    vertices = rng.normal(size=(V, 3))
    g = rng.normal(size=(V, 3))
    return parents, centres, skin_index, skin_weight, vertices, rotations, g


def _device(torch, ops, case):
    parents, centres, skin_index, skin_weight, vertices, rotations, g = case
    lbs = ops.LinearBlendSkinning(parents, centres, skin_index, skin_weight, device="cuda")
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()  # noqa: E731
    return lbs, cuda(vertices), cuda(rotations), cuda(g)


def _close(got, want, name):
    err = np.abs(got - want).max()
    scale = np.abs(want).max()
    print(f"{name}: max |err| {err:.3e} of max |value| {scale:.3e} ({err / scale:.2e})")
    assert err <= 1e-12 * scale, name


@pytest.mark.parametrize("V,J,K", [(20000, 24, 4), (3000, 1024, 8), (5, 1, 1), (700, 3, 5)])
def test_the_device_matches_the_restatement(V, J, K, torch, ops):
    case = _case(V, J, K)
    parents, centres, skin_index, skin_weight, vertices, rotations, g = case
    lbs, v, r, gb = _device(torch, ops, case)
    skinned = lbs.apply(v, r)
    vb, rb, wb = lbs.backward(v, r, gb, weights_grad=True)
    torch.cuda.synchronize()
    want = ref.skin(parents, centres, skin_index, skin_weight, vertices, rotations)
    want_vb, want_wb, want_rb = ref.skin_b(parents, centres, skin_index, skin_weight, vertices, rotations, g)
    _close(skinned.cpu().numpy(), want, "skinned")
    _close(vb.cpu().numpy(), want_vb, "vertices_b")
    _close(wb.cpu().numpy(), want_wb, "weights_b")
    _close(rb.cpu().numpy(), want_rb, "rotations_b")
    # the table: (Rg, tg, M, b) of the restatement's forward kinematics
    Rg, tg, M, b = ref.forward_kinematics(parents, centres, rotations)
    table = np.concatenate([Rg.reshape(J, 9), tg, M.reshape(J, 9), b], axis=1)
    _close(lbs.transforms.cpu().numpy(), table, "transforms")
    # add_to in place
    acc = torch.ones_like(v)
    lbs.backward(v, r, gb, add_to=acc, out=(acc, torch.empty_like(r)))
    _close(acc.cpu().numpy(), want_vb + 1.0, "vertices_b + add_to")


def test_identity_rotations_leave_the_mesh_at_rest(torch, ops):
    case = _case(20000, 24, 4, seed=3)
    lbs, v, r, _ = _device(torch, ops, case)
    skinned = lbs.apply(v, torch.zeros_like(r))
    assert np.abs(skinned.cpu().numpy() - case[4]).max() <= 1e-14 * np.abs(case[4]).max()


def test_repeated_calls_are_bit_identical(torch, ops):
    lbs, v, r, gb = _device(torch, ops, _case(200000, 64, 4, seed=1))
    first = [lbs.apply(v, r).clone(), *[t.clone() for t in lbs.backward(v, r, gb, weights_grad=True)]]
    second = [lbs.apply(v, r), *lbs.backward(v, r, gb, weights_grad=True)]
    for a, b in zip(first, second):
        assert torch.equal(a, b)


def test_gradcheck_of_the_autograd_function(torch, ops):
    from deodr_b200.pytorch import LinearBlendSkinningFunc

    parents, centres, skin_index, skin_weight, vertices, rotations, _ = _case(60, 5, 2, seed=2)
    lbs = ops.LinearBlendSkinning(parents, centres, skin_index, skin_weight, device="cuda")
    cuda = lambda a: torch.from_numpy(np.array(a, dtype=np.float64)).cuda().requires_grad_(True)  # noqa: E731
    inputs = (cuda(vertices), cuda(rotations), cuda(skin_weight), lbs)
    assert torch.autograd.gradcheck(LinearBlendSkinningFunc.apply, inputs, eps=1e-6, atol=1e-7, rtol=1e-6)
    # the weights are optional: without requires_grad they get none
    v = cuda(vertices)
    LinearBlendSkinningFunc.apply(v, cuda(rotations), torch.from_numpy(skin_weight).cuda(), lbs).sum().backward()
    assert v.grad is not None


# ---- articulated fits of a procedural tube ---------------------------------------------------------------------------

BENDS = np.array([0.0, 0.35, -0.3, 0.4])  # about z: in the image plane of the fitters' camera
tube = ref.tube


def _bends(angles):
    r = np.zeros((4, 3))
    r[:, 2] = angles
    return r


COLOR, LIGHT, AMBIENT = np.array([0.9, 0.6, 0.3]), np.array([0.2, -0.3, -0.7]), 0.3


def _rgb_fitter(mf, lbs, vertices, faces, **kw):
    return mf.MeshRGBFitterWithPose(vertices, faces, np.zeros(3), np.zeros(3), COLOR, LIGHT, AMBIENT, skeleton=lbs,
                                    **kw)


def _target_image(torch, mf, lbs, vertices, faces, bends, H=128, W=128):
    """The image the RGB fitter renders at the given joint rotations: one step of a fitter started there."""
    f = _rgb_fitter(mf, lbs, vertices, faces)
    f.set_joint_rotations_init(bends)
    f.reset()
    f.set_image(np.zeros((H, W, 3)))
    _, image, _ = f.step()
    return image.cpu().numpy().astype(np.float64)


@pytest.fixture(scope="module")
def tube_setup(torch, ops):
    import deodr_b200.mesh_fitter as mf

    vertices, faces, parents, centres, skin_index, skin_weight = tube()
    lbs = ops.LinearBlendSkinning(parents, centres, skin_index, skin_weight, device="cuda")
    return mf, lbs, vertices, faces


def test_the_fitter_refuses_a_skeleton_without_a_single_root_at_zero(tube_setup, ops):
    mf, _, vertices, faces = tube_setup
    _, _, parents, centres, skin_index, skin_weight = tube()
    with pytest.raises(ValueError):
        _rgb_fitter(mf, (np.array([-1, 0, -1, 2]), centres, skin_index, skin_weight), vertices, faces)
    with pytest.raises(ValueError):
        _rgb_fitter(mf, (parents, centres, skin_index[:-1], skin_weight[:-1]), vertices, faces)
    f = _rgb_fitter(mf, (parents, centres, skin_index, skin_weight), vertices, faces)  # the four arrays
    assert f.skinning.nb_joints == 4


def test_the_rgb_fitter_recovers_the_bends(tube_setup, torch):
    """The articulated fit alone: the free per-vertex deformation is held still (``step_factor_vertices = 0``), so the
    bends are not shared with it; the joints, the rigid pose, the light and the colour are fitted from rest."""
    mf, lbs, vertices, faces = tube_setup
    target = _target_image(torch, mf, lbs, vertices, faces, _bends(BENDS))
    f = _rgb_fitter(mf, lbs, vertices, faces)
    f.step_factor_vertices = 0.0
    f.set_image(target)
    energies = [float(f.step()[0]) for _ in range(800)]
    got = f.joint_rotations.cpu().numpy()
    print("device fitter: energy", energies[0], "->", energies[-1], "; bends", got[:, 2], "want", BENDS,
          "; out of plane", got[:, 1], "; twist (not asserted)", got[:, 0])
    assert np.all(got[0] == 0)  # the root stays fixed
    # H100, 16 runs (the rasteriser's atomics make every fit differ): bend error median 0.016, max 0.046 rad; final
    # energy 0.20 % to 0.81 % of the first
    assert np.abs(got[1:, 2] - BENDS[1:]).max() < 0.1
    assert energies[-1] < 0.05 * energies[0]


def test_the_depth_fitter_takes_a_skeleton(tube_setup, torch):
    mf, lbs, vertices, faces = tube_setup
    f = mf.MeshDepthFitter(vertices, faces, np.zeros(3), np.zeros(3), skeleton=lbs)
    f.set_image(np.full((64, 64), 20.0))
    f.set_max_depth(20.0)
    e = [float(f.step()[0]) for _ in range(3)]
    assert np.all(np.isfinite(e)) and np.all(np.isfinite(f.joint_rotations.cpu().numpy()))


def test_adam_through_the_autograd_function_recovers_the_bends(tube_setup, torch):
    import deodr_b200.pytorch as P

    mf, lbs, vertices, faces = tube_setup
    H = W = 128
    skin_weight = lbs.skin_weight
    v = torch.from_numpy(vertices).cuda()
    probe = _rgb_fitter(mf, lbs, vertices, faces)
    probe.set_image(np.zeros((H, W, 3)))
    cam = probe.camera
    camera = P.CameraPytorch(cam.extrinsic, cam.intrinsic, H, W)

    def render(rotations):
        skinned = P.LinearBlendSkinningFunc.apply(v, rotations, skin_weight, lbs)
        mesh = P.ColoredTriMeshPytorch(faces, skinned, colors=torch.from_numpy(np.tile(COLOR, (len(vertices), 1)))
                                       .cuda())
        scene = P.Scene3DPytorch()
        scene.set_mesh(mesh)
        scene.set_light(LIGHT, AMBIENT)
        scene.set_background_color((0.0, 0.0, 0.0))
        return scene.render(camera)

    with torch.no_grad():
        target = render(torch.from_numpy(_bends(BENDS)).cuda())
    free = torch.zeros((3, 3), dtype=torch.float64, device="cuda", requires_grad=True)
    opt = torch.optim.Adam([free], lr=0.01)
    losses = []
    for _ in range(300):
        opt.zero_grad()
        rotations = torch.cat([torch.zeros((1, 3), dtype=torch.float64, device="cuda"), free])
        loss = ((render(rotations) - target) ** 2).sum()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    got = free.detach().cpu().numpy()
    print("adam: loss", losses[0], "->", losses[-1], "; bends", got[:, 2], "want", BENDS[1:], "; out of plane",
          got[:, 1], "; twist (not asserted)", got[:, 0])
    assert np.abs(got[:, 2] - BENDS[1:]).max() < 0.05  # H100: within 0.024 rad, loss 1382 -> 0.43


OVER_BEND = np.array([0.0, 1.5, 1.5, 1.5])  # folds the tube's end back across its start


def test_self_collision_holds_an_over_bent_fit_apart(tube_setup, torch):
    mf, lbs, vertices, faces = tube_setup
    target = _target_image(torch, mf, lbs, vertices, faces, _bends(OVER_BEND))
    probe = mf.DeviceSelfCollisionEnergy(faces, vertices, 0.05, 1.0, "cuda")

    def fit(**kw):
        f = _rgb_fitter(mf, lbs, vertices, faces, **kw)
        f.set_image(target)
        worst = 0
        for s in range(400):
            f.step()
            if s % 20 == 19:
                worst = max(worst, int(probe.intersections(f.skinning.apply(f.vertices, f.joint_rotations)).shape[0]))
        skinned = f.skinning.apply(f.vertices, f.joint_rotations)
        return f, int(probe.intersections(skinned).shape[0]), worst

    free, free_pairs, _ = fit()
    held, held_pairs, held_worst = fit(cself=1000.0, self_collision_thickness=0.05)
    print("over-bend: crossing face pairs without the term", free_pairs, "bends", free.joint_rotations[:, 2].tolist(),
          "; with it", held_pairs, "(at worst", held_worst, ") bends", held.joint_rotations[:, 2].tolist(),
          "; collision energy", float(held.energy_self_collision))
    assert free_pairs > 0  # H100: 73 to 82 crossing pairs in five runs
    assert held_pairs == 0 and held_worst == 0
