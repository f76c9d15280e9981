"""fp64 numpy restatement of linear blend skinning and its adjoint (include/deodr_b200.h, "Linear blend skinning"),
written from the model's formulas, joint by joint and vertex by vertex, to check the device kernels against."""
import numpy as np

TAYLOR_S = 1e-2  # phi^2 below which the series of a, b and their derivatives are used


def coefficients(s):
    """a = sin(phi)/phi, b = (1 - cos(phi))/phi^2 and their derivatives with respect to s = phi^2."""
    if s < TAYLOR_S:
        a = 1 - s / 6 + s ** 2 / 120 - s ** 3 / 5040 + s ** 4 / 362880
        b = 0.5 - s / 24 + s ** 2 / 720 - s ** 3 / 40320 + s ** 4 / 3628800
        da = -1 / 6 + s / 60 - s ** 2 / 1680 + s ** 3 / 90720 - s ** 4 / 7983360
        db = -1 / 24 + s / 360 - s ** 2 / 13440 + s ** 3 / 907200 - s ** 4 / 95800320
        return a, b, da, db
    phi = np.sqrt(s)
    a = np.sin(phi) / phi
    b = 2 * np.sin(phi / 2) ** 2 / s
    return a, b, (np.cos(phi) - a) / (2 * s), (a / 2 - b) / s


def skew(t):
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]], dtype=np.float64)


def rotation(theta):
    t = np.asarray(theta, dtype=np.float64)
    a, b, _, _ = coefficients(float(t @ t))
    K = skew(t)
    return np.eye(3) + a * K + b * K @ K


def rotation_b(theta, G):
    """d<G, R(theta)>/dtheta, term by term from R = I + a K + b K^2 with a, b functions of s = theta.theta."""
    t = np.asarray(theta, dtype=np.float64)
    s = float(t @ t)
    a, b, da, db = coefficients(s)
    K = skew(t)
    out = np.zeros(3)
    for k in range(3):
        e = np.zeros(3)
        e[k] = 1
        Ek = skew(e)
        dR = 2 * t[k] * da * K + a * Ek + 2 * t[k] * db * K @ K + b * (Ek @ K + K @ Ek)
        out[k] = np.sum(G * dR)
    return out


def forward_kinematics(parents, centres, rotations):
    """-> (Rg [J,3,3], tg [J,3], M [J,3,3], b [J,3]), in index order."""
    J = len(parents)
    Rg, tg = np.zeros((J, 3, 3)), np.zeros((J, 3))
    for j in range(J):
        R = rotation(rotations[j])
        p = parents[j]
        if p < 0:
            Rg[j], tg[j] = R, centres[j]
        else:
            Rg[j] = Rg[p] @ R
            tg[j] = tg[p] + Rg[p] @ (centres[j] - centres[p])
    b = tg - np.einsum("jmn,jn->jm", Rg, centres)
    return Rg, tg, Rg.copy(), b


def skin(parents, centres, skin_index, skin_weight, vertices, rotations):
    _, _, M, b = forward_kinematics(parents, centres, rotations)
    out = np.zeros_like(vertices, dtype=np.float64)
    for k in range(skin_index.shape[1]):
        j = skin_index[:, k]
        out += skin_weight[:, k, None] * (np.einsum("vmn,vn->vm", M[j], vertices) + b[j])
    return out


def skin_b(parents, centres, skin_index, skin_weight, vertices, rotations, g):
    """-> (vertices_b [V,3], weights_b [V,K], rotations_b [J,3]) for the gradient g [V,3] of the skinned vertices."""
    J = len(parents)
    Rg, tg, M, b = forward_kinematics(parents, centres, rotations)
    vertices_b = np.zeros_like(vertices)
    weights_b = np.zeros_like(skin_weight)
    M_b, b_b = np.zeros((J, 3, 3)), np.zeros((J, 3))
    for k in range(skin_index.shape[1]):
        j = skin_index[:, k]
        w = skin_weight[:, k, None]
        vertices_b += w * np.einsum("vnm,vn->vm", M[j], g)
        weights_b[:, k] = np.sum(g * (np.einsum("vmn,vn->vm", M[j], vertices) + b[j]), axis=1)
        np.add.at(M_b, j, (w * g)[:, :, None] * vertices[:, None, :])
        np.add.at(b_b, j, w * g)
    # b_j = tg_j - Rg_j c_j, M_j = Rg_j
    Rg_b = M_b - b_b[:, :, None] * centres[:, None, :]
    tg_b = b_b.copy()
    rotations_b = np.zeros((J, 3))
    for j in reversed(range(J)):
        p = parents[j]
        R = rotation(rotations[j])
        if p < 0:
            rotations_b[j] = rotation_b(rotations[j], Rg_b[j])
            continue
        rotations_b[j] = rotation_b(rotations[j], Rg[p].T @ Rg_b[j])
        Rg_b[p] += Rg_b[j] @ R.T + np.outer(tg_b[j], centres[j] - centres[p])
        tg_b[p] += tg_b[j]
    return vertices_b, weights_b, rotations_b


def random_tree(rng, J, roots=(0,), min_depth=1):
    """parents [J] of a random tree in index order with the given roots, deepened until its depth is >= min_depth."""
    while True:
        parents = np.full(J, -1, dtype=np.int64)
        for j in range(J):
            if j not in roots:
                lo = max(0, j - 4)
                choices = [q for q in range(lo, j)]
                parents[j] = rng.choice(choices)
        depth = np.zeros(J, dtype=np.int64)
        for j in range(J):
            depth[j] = 0 if parents[j] < 0 else depth[parents[j]] + 1
        if depth.max() >= min_depth:
            return parents


def random_binding(rng, V, J, K):
    """skin_index [V,K] (distinct joints per vertex) and skin_weight [V,K] summing to 1."""
    skin_index = np.stack([rng.choice(J, size=K, replace=False) for _ in range(V)]).astype(np.int32)
    w = rng.uniform(0.1, 1.0, size=(V, K))
    return skin_index, w / w.sum(axis=1, keepdims=True)


RADIUS, N_ALONG, N_AROUND = 0.35, 41, 16
JOINT_X = np.array([-2.0, -1.0, 0.0, 1.0])  # four chained joints along the axis; joint 0 is the root
BAND = 0.25  # the weights ramp between neighbouring joints over x in [c - BAND, c + BAND]


def tube(n_along=N_ALONG):
    """A closed tube along x from -2 to 2 (``n_along`` rings of N_AROUND and two cap centres, one component, outward
    winding) and its skeleton: (vertices, faces, parents, centres, skin_index [V,2], skin_weight [V,2])."""
    x = np.linspace(-2, 2, n_along)
    phi = 2 * np.pi * np.arange(N_AROUND) / N_AROUND
    rings = np.stack([np.repeat(x, N_AROUND), RADIUS * np.tile(np.cos(phi), n_along),
                      RADIUS * np.tile(np.sin(phi), n_along)], axis=1)
    vertices = np.vstack([rings, [[-2, 0, 0], [2, 0, 0]]])
    faces = []
    for i in range(n_along - 1):
        for j in range(N_AROUND):
            a, b = i * N_AROUND + j, i * N_AROUND + (j + 1) % N_AROUND
            c, d = a + N_AROUND, b + N_AROUND
            faces += [[a, b, d], [a, d, c]]
    s, e = n_along * N_AROUND, n_along * N_AROUND + 1
    last = (n_along - 1) * N_AROUND
    for j in range(N_AROUND):
        faces += [[s, (j + 1) % N_AROUND, j], [e, last + j, last + (j + 1) % N_AROUND]]
    faces = np.array(faces, dtype=np.int64)
    a, b, c = vertices[faces[:, 0]], vertices[faces[:, 1]], vertices[faces[:, 2]]
    if np.einsum("ij,ij->i", a, np.cross(b, c)).sum() < 0:
        faces = faces[:, [0, 2, 1]]
    parents = np.array([-1, 0, 1, 2])
    centres = np.stack([JOINT_X, np.zeros(4), np.zeros(4)], axis=1)
    V = vertices.shape[0]
    skin_index = np.zeros((V, 2), np.int32)
    skin_weight = np.zeros((V, 2))
    for i, px in enumerate(vertices[:, 0]):
        seg = int(np.clip(np.searchsorted(JOINT_X, px, side="right") - 1, 0, 3))
        skin_index[i] = (seg, seg)
        skin_weight[i] = (1.0, 0.0)
        for j in (1, 2, 3):
            if abs(px - JOINT_X[j]) < BAND:
                t = (px - JOINT_X[j] + BAND) / (2 * BAND)
                skin_index[i] = (j - 1, j)
                skin_weight[i] = (1 - t, t)
    return vertices, faces, parents, centres, skin_index, skin_weight
