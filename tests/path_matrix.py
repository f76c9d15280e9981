"""Test helper (no tests here): the scenes and the dispatch mirror of the kernel-path matrix.

The device rasteriser picks, for every scene, a template instance of each of its kernels and a binning path:

  * the channel instance MAXC: 1 for C = 1, 3 for C = 3, 4 for C = 2 or 4, 16 for C = 5..16; above 16 channels the
    slab path (kernels.cu: enqueue_forward / launch_raster_fwd_wide, kernels_bwd.cu: deodr_launch_backward);
  * from the scene and the call: perspective_correct (P), textured triangles in the plan (X), antialiase_error mode (R),
    background gradients requested (B), and TMA tile stores / loads or their cooperative fall-back (row pitch rule);
  * from the total triangle count T alone (kernels.cu:778-796): the record path of the "medium" triangles and the
    triangle-parallel adjoint of the textured small ones.

`matrix_scene` builds a 600-triangle picture with triangles of every size class in generic position, `with_ballast`
pads it with triangles that never reach a pixel, so that the same picture runs on each size-chosen path at the cost of
600 triangles, and `instances` mirrors the dispatch: the (kernel, template arguments, tile transfer) tuples a case of
tests/test_gpu_path_matrix.py selects.  ALL_INSTANCES is everything the dispatch can select; tests/test_path_matrix.py
checks that the GPU cases reach all of it.  Which cases reach which kernel (regime x C x variant, `textured` alternating
and both image sizes in every case, see `case_scenes`):

  kernel                               template arguments                    reached by
  k_tile_z<MAXC, P, X, true>           MAXC 1|3|4|16, P, X; TMA store         C <= 16, every variant (P: "perspective");
                                       when C <= 4 and W * C % 4 == 0         TMA at 160 px wide (C = 4: both widths)
  k_tile_z<1, P, false, false>         P                                     C = 17 (slab path: the z pass unfused)
  k_shade<16, P, X>                    P, X                                  C = 17
  k_edge_fwd<MAXC, P, X, R>            MAXC 1|3|4|16, P, X, R                sigma > 0; R: "error*", and "perspective"
                                                                             (its forward also runs in error mode)
  k_error_image_b                      -                                     "error", "error_complete"
  k_raster_bwd<MAXC, X, R, B>          MAXC 1|3|4|16, X, R, B; TMA loads      differentiable variants with sigma > 0;
                                       when C <= 4 and W % 4 == 0             B: "background_image", "error_complete";
                                                                             C = 17: MAXC 16 per slab, R false
  k_interior_bwd<MAXC, X>              MAXC 1|3|4|16, X                      every differentiable case (large triangles)
  k_small_tri_bwd<MAXC, X>             MAXC 1|3|4|16, X                      every differentiable case
  k_background_bwd<MAXC>               MAXC 1|3|4|16                         "background_image", "error_complete"

UNREACHABLE lists the combinations the dispatch cannot select, with the reason.
"""
import copy
from itertools import product

import numpy as np

from deodr_b200.scenes import SceneArrays

TS = 16                 # tile side (phases.h)
RECORD_ROWS = 16        # phases.h: RECORD_ROWS, the height limit of the record path of medium triangles
COLOR_SLAB = 16         # shade.h: widest channel instance
SMALL_FLAG = 0x40000000  # phases.h: owner code bit of a triangle owned by the triangle-parallel adjoint
# kernels.cu:778-796: record_rows_for (medium triangles take the record path from this many triangles on) and
# small_textured_for (textured small triangles get SMALL_FLAG and the triangle-parallel adjoint from this many on)
RECORD_MIN_TRIANGLES = 32768
SMALL_TEXTURED_MIN_TRIANGLES = 262144

# total triangle count of each regime (None: the picture alone)
REGIMES = {"few": None, "records": 40000, "small-textured": 270000}
SIZES = ((157, 93), (160, 96))  # (width, height): partial tiles; 157 px rows are not 16-byte multiples for C <= 3
CHANNELS = (1, 2, 3, 4, 7, 16, 17)
VARIANTS = ("default", "cw_nonstrict_halfpix", "sigma0", "no_culling", "perspective", "background_image", "error",
            "error_complete")
CLASS_COUNTS = {"small": 400, "medium": 150, "large": 20}
TEXTURE_SIDE = 32


def record_rows_for(T):
    return RECORD_ROWS if T >= RECORD_MIN_TRIANGLES else 0


def small_textured_for(T):
    return T >= SMALL_TEXTURED_MIN_TRIANGLES


def maxc(C):
    """The channel instance of the kernels for C channels (C > COLOR_SLAB: the slabs run in the 16-channel one)."""
    return 1 if C == 1 else 3 if C == 3 else 4 if C <= 4 else 16


# ---------------------------------------------------------------------------------------------------- classes

def _small_shift(box_w):
    sh = np.zeros_like(box_w)
    while True:
        more = (1 << sh) < box_w
        if not more.any():
            return sh
        sh = sh + more


def triangle_classes(scene, record_rows=RECORD_ROWS, small_textured=True):
    """Per triangle: "off" (not drawn, or its box misses the image), "small" (owned with SMALL_FLAG: triangle-parallel
    adjoint), "medium" (record path without SMALL_FLAG) or "large" (binned by reference into the tile kernel).
    A restatement of tri_bounds (rmath.h), tri_tile_box / is_small / takes_record_path (phases.h:131-144, 250-276) and
    the drawn test of TriClass (shade.h)."""
    faces = np.asarray(scene.faces, dtype=np.int64)
    ij = np.asarray(scene.ij, dtype=np.float64)
    V = ij[faces]                                   # [T, 3, 2] (x, y)
    d = np.asarray(scene.depths, dtype=np.float64)[faces]
    u, w = V[:, 1] - V[:, 0], V[:, 2] - V[:, 0]
    det = u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]
    front = det > 0 if scene.clockwise else det < 0
    area_positive = (d > 0).all(axis=1) & front
    textured = np.asarray(scene.textured, bool) & np.asarray(scene.shaded, bool)
    drawn = (area_positive | (not scene.backface_culling)) & (textured | ~np.asarray(scene.textured, bool))
    V = V - (0.0 if scene.integer_pixel_centers else 0.5)
    lo, hi = V.min(axis=1), V.max(axis=1)
    if scene.strict_edge:
        x0, y0 = np.floor(lo[:, 0]), np.floor(lo[:, 1]) + 1
    else:
        x0, y0 = np.ceil(lo[:, 0]), np.ceil(lo[:, 1])
    x1, y1 = np.floor(hi[:, 0]), np.floor(hi[:, 1])
    x0, y0 = np.maximum(x0, 0).astype(np.int64), np.maximum(y0, 0).astype(np.int64)
    x1 = np.minimum(x1, scene.width - 1).astype(np.int64)
    y1 = np.minimum(y1, scene.height - 1).astype(np.int64)
    on = drawn & (x0 <= x1) & (y0 <= y1)
    box_w, box_h = np.maximum(x1 - x0 + 1, 1), np.maximum(y1 - y0 + 1, 1)
    cols = x1 // TS - x0 // TS
    rows = y1 // TS - y0 // TS
    small = (cols <= 1) & (rows <= 1) & (box_w <= 32) & ((box_h << _small_shift(box_w)) <= 64)
    records = small | ((cols <= 1) & (box_w <= 32) & (box_h <= record_rows))
    small &= small_textured | ~textured
    out = np.full(faces.shape[0], "large", dtype=object)
    out[records & ~small] = "medium"
    out[small] = "small"
    out[~on] = "off"
    return out


def _stable_classes(scene):
    """Classes under every edge / pixel-centre convention and with the picture moved by half a pixel, or "unstable"."""
    ref = None
    for strict, integer, (dx, dy) in product((True, False), (True, False),
                                             ((0, 0), (0.5, 0), (-0.5, 0), (0, 0.5), (0, -0.5))):
        s = copy.copy(scene)
        s.strict_edge, s.integer_pixel_centers = strict, integer
        s.ij = scene.ij + np.array([dx, dy])
        c = triangle_classes(s)
        ref = c if ref is None else np.where(ref == c, ref, "unstable")
    return ref


# ---------------------------------------------------------------------------------------------------- scenes

def _off_half_pixels(xy):
    """Vertices off the integer and half-integer coordinates (where the rasterisation conventions differ)."""
    frac = np.mod(2 * xy, 1.0)
    return xy + np.where((frac < 0.03) | (frac > 0.97), 0.047, 0.0)


def _front(tri):
    """Front-facing for clockwise = False (the convention of scenes.confetti_scene)."""
    u, w = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
    flip = (u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]) > 0
    tri = tri.copy()
    tri[flip] = tri[flip][:, ::-1]
    return tri


def _aspect(tri):
    """longest side^2 / area (2.31 for an equilateral triangle), and the area."""
    u, w = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
    area = 0.5 * np.abs(u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0])
    sides = np.stack([np.sum((tri[:, (k + 1) % 3] - tri[:, k]) ** 2, axis=1) for k in range(3)], axis=1)
    return sides.max(axis=1) / np.maximum(area, 1e-300), area


def _in_box(rng, n, x0, y0, wx, wy):
    """Triangles spanning exactly [x0, x0 + wx] x [y0, y0 + wy]: one vertex on each of the left, right, top and bottom
    sides of the box (the third vertex takes two of them)."""
    t = np.empty((n, 3, 2))
    t[:, 0] = np.stack((x0, y0 + rng.random(n) * wy), axis=1)          # left side
    t[:, 1] = np.stack((x0 + wx, y0), axis=1)                          # top right corner
    t[:, 2] = np.stack((x0 + rng.random(n) * wx, y0 + wy), axis=1)     # bottom side
    return t


def _draw(rng, kind, n, width, height):
    if kind == "small":
        wx, wy = rng.uniform(1.6, 4.8, n), rng.uniform(1.6, 4.8, n)
        x0, y0 = rng.uniform(1.5, width - 7.0, n), rng.uniform(1.5, height - 7.0, n)
    elif kind == "medium":  # 18-27 px wide inside two tile columns, 5-13 rows
        wx, wy = rng.uniform(18.0, 27.0, n), rng.uniform(5.0, 13.0, n)
        col = rng.integers(0, (width - 32) // TS + 1, n)
        x0 = col * TS + 1.5 + rng.random(n) * (28.5 - wx)
        y0 = rng.uniform(1.5, height - 16.0, n)
    else:  # large: 36-110 px wide or 20-80 rows, most of it inside the image
        wx, wy = rng.uniform(36.0, 110.0, n), rng.uniform(20.0, 80.0, n)
        x0, y0 = rng.uniform(-0.3 * wx, width - 0.7 * wx), rng.uniform(-0.3 * wy, height - 0.7 * wy)
    return _in_box(rng, n, x0, y0, wx, wy)


def _clipped(width, height):
    """At each corner a huge triangle (sides of ~300 px) with one vertex just inside the image: the image clips its box
    to a small (5 x 5) or a medium (22 x 10 px) one.  Between them they touch every border."""
    out = []
    for apex in ((4.3, 4.6), (21.3, 9.6)):
        for sx, sy in ((1, 1), (-1, 1), (1, -1), (-1, -1)):
            ax = apex[0] if sx > 0 else width - 1 - apex[0]
            ay = apex[1] if sy > 0 else height - 1 - apex[1]
            far1 = (ax - sx * 310.0, ay - sy * 110.0)
            far2 = (ax - sx * 120.0, ay - sy * 290.0)
            out.append(np.array([(ax, ay), far1, far2]))
    return np.array(out)


def matrix_scene(width, height, nb_colors, seed, textured=False, edge_ratio=0.3, background_image=False):
    """~400 small, ~150 medium, ~20 large and 8 clipped triangles (class limits of phases.h:250-276, each triangle at
    least half a pixel inside them), overlapping in depth, in generic position (see `assert_generic`).  Front-facing
    for clockwise = False; with `textured`, about 40 % of them are textured and shaded."""
    rng = np.random.default_rng(seed)
    parts, kinds = [], []
    for kind, n in CLASS_COUNTS.items():
        got = 0
        while got < n:
            cand = _front(_off_half_pixels(_draw(rng, kind, 2 * (n - got) + 8, width, height)))
            aspect, area = _aspect(cand)
            cand = cand[(area >= 0.6) & (aspect <= 24.0)]
            probe = _soup(cand, np.ones(3 * len(cand)), width, height, 1)
            cand = cand[_stable_classes(probe) == kind][: n - got]
            parts.append(cand)
            kinds += [kind] * len(cand)
            got += len(cand)
    clipped = _front(_off_half_pixels(_clipped(width, height)))
    cls = _stable_classes(_soup(clipped, np.ones(3 * len(clipped)), width, height, 1))
    assert list(cls) == ["small"] * 4 + ["medium"] * 4, cls
    parts.append(clipped)
    kinds += ["clipped"] * len(clipped)
    tri = np.concatenate(parts)
    order = rng.permutation(len(tri))  # classes interleaved in index order (the reference's draw order)
    tri, kinds = tri[order], np.array(kinds, dtype=object)[order]
    T = len(tri)
    # a plane of its own per triangle: depth 1..5 with a per-vertex slope
    depths = np.repeat(rng.uniform(1.0, 5.0, T), 3) + rng.uniform(-0.3, 0.3, 3 * T)
    scene = _soup(tri, depths, width, height, nb_colors)
    scene.colors = rng.random((3 * T, nb_colors))
    scene.edgeflags = rng.random((T, 3)) < edge_ratio
    if textured:
        tex = rng.random(T) < 0.4
        scene.textured, scene.shaded = tex.copy(), tex.copy()
        scene.texture = rng.random((TEXTURE_SIDE, TEXTURE_SIDE, nb_colors))
        uv = rng.uniform(1.0, TEXTURE_SIDE - 2.0, (3 * T, 2)) * 0.9973 + 0.0131
        frac = np.mod(uv, 1.0)  # off the texel grid (the bilinear adjoint is discontinuous on it)
        scene.uv = uv + np.where((frac < 0.01) | (frac > 0.99), 0.037, 0.0)
        scene.shade = rng.uniform(0.3, 1.0, 3 * T)
    if background_image:
        scene.background_color, scene.background_image = None, rng.random((height, width, nb_colors))
    else:
        scene.background_color = rng.random(nb_colors)
    scene.extra["kinds"] = kinds
    return scene


def _soup(tri, depths, width, height, nb_colors):
    T = len(tri)
    faces = np.arange(3 * T, dtype=np.uint32).reshape(T, 3)
    return SceneArrays(
        faces=faces, faces_uv=faces.copy(), ij=np.ascontiguousarray(tri.reshape(-1, 2)),
        depths=np.ascontiguousarray(depths, dtype=np.float64), textured=np.zeros(T, bool), uv=np.zeros((3 * T, 2)),
        shade=np.zeros(3 * T), colors=np.zeros((3 * T, nb_colors)), shaded=np.zeros(T, bool),
        edgeflags=np.zeros((T, 3), bool), height=height, width=width, nb_colors=nb_colors,
        texture=np.zeros((2, 2, nb_colors)), background_image=None, background_color=np.zeros(nb_colors),
        clockwise=False, backface_culling=True, strict_edge=True, perspective_correct=False,
        integer_pixel_centers=True)


def assert_generic(scene, emulator, sigma=1.0):
    """Generic position: area >= 0.5 px^2 and a bounded aspect ratio, uv off the texel grid, vertices off half pixels,
    no two triangles sharing a depth plane, interpolation weights of every drawn pixel <= 64 in size."""
    tri = scene.ij[scene.faces.astype(np.int64)]
    kinds = scene.extra.get("kinds")
    real = np.ones(len(tri), bool) if kinds is None else np.array([k != "ballast" for k in kinds])
    aspect, area = _aspect(tri[real])
    assert area.min() >= 0.5 and aspect.max() <= 30.0, (area.min(), aspect.max())
    frac = np.mod(2 * scene.ij[scene.faces[real].ravel()], 1.0)
    assert ((frac > 0.02) & (frac < 0.98)).all(), "a vertex on a half pixel"
    if scene.textured.any():
        uv = scene.uv[scene.faces_uv[scene.textured & scene.shaded].ravel()]
        g = np.mod(uv, 1.0)
        assert ((g > 1e-3) & (g < 1 - 1e-3)).all(), "uv on the texel grid"
    planes = np.round(scene.depths[scene.faces[real]], 12)
    assert len(np.unique(planes, axis=0)) == real.sum(), "two triangles share a depth plane"
    ws = emulator.render(scene, sigma)["weight_scale"]
    assert ws.max() <= 64, ws.max()


# ---------------------------------------------------------------------------------------------------- ballast

def with_ballast(scene, total_T, seed=0):
    """`scene` padded to `total_T` triangles that never reach a pixel: off screen at x in [-400, -300] (inside the
    reference's `short` range), a few of them of zero area, no edge flags, neither textured nor shaded.  The size
    switches of the device read only the triangle count, so this runs the picture on the path of `total_T` triangles."""
    T = scene.faces.shape[0]
    n = total_T - T
    if n <= 0:
        return scene
    rng = np.random.default_rng(seed)
    pool = 3000  # ballast vertices, shared by the ballast triangles
    ij = np.stack((rng.uniform(-400.0, -300.0, pool), rng.uniform(0.0, scene.height, pool)), axis=1)
    V0 = scene.ij.shape[0]
    faces = V0 + rng.integers(0, pool, (n, 3))
    faces[:8] = V0 + np.array([[0, 0, 0], [1, 1, 2], [3, 4, 4], [5, 5, 5], [6, 7, 6], [8, 8, 8], [9, 9, 10],
                               [11, 12, 11]])  # zero area
    s = copy.copy(scene)
    s.faces = np.ascontiguousarray(np.concatenate((scene.faces, faces.astype(np.uint32))))
    s.faces_uv = np.ascontiguousarray(np.concatenate((scene.faces_uv, np.zeros((n, 3), np.uint32))))
    s.ij = np.ascontiguousarray(np.concatenate((scene.ij, ij)))
    s.depths = np.concatenate((scene.depths, rng.uniform(1.0, 5.0, pool)))
    s.colors = np.concatenate((scene.colors, rng.random((pool, scene.nb_colors))))
    s.shade = np.concatenate((scene.shade, np.zeros(pool)))
    s.textured = np.concatenate((scene.textured, np.zeros(n, bool)))
    s.shaded = np.concatenate((scene.shaded, np.zeros(n, bool)))
    s.edgeflags = np.concatenate((scene.edgeflags, np.zeros((n, 3), bool)))
    s.extra = dict(scene.extra, kinds=np.concatenate((scene.extra.get("kinds", np.full(T, "?", object)),
                                                      np.full(n, "ballast", object))),
                   ballast_vertices=slice(V0, V0 + pool))
    return s


# ---------------------------------------------------------------------------------------------------- cases

def case_scenes(regime, C, variant):
    """(width, height, textured) of the two scenes of a case: both image sizes, `textured` alternating over regimes,
    channel counts and variants (the two sizes of a case take opposite values)."""
    r, c, v = list(REGIMES).index(regime), CHANNELS.index(C), VARIANTS.index(variant)
    t = (r + c + v) % 2 == 1
    return [(SIZES[0][0], SIZES[0][1], t), (SIZES[1][0], SIZES[1][1], not t)]


def variant_setup(scene, variant):
    """The variant's scene flags and call -> (scene, sigma, call) with call one of "fwd" (forward only), "bwd"
    (forward + adjoint), "bg" (+ background gradient), "error" / "error_complete" (antialiase_error mode; the latter
    with the complete adjoint and the background gradient), "fwd+error" (forward in both modes)."""
    s = copy.copy(scene)
    if variant == "default":
        return s, 1.0, "bwd"
    if variant == "cw_nonstrict_halfpix":
        s.faces = np.ascontiguousarray(scene.faces[:, ::-1])
        s.faces_uv = np.ascontiguousarray(scene.faces_uv[:, ::-1])
        s.clockwise, s.strict_edge, s.integer_pixel_centers = True, False, False
        return s, 2.5, "bwd"
    if variant == "sigma0":
        return s, 0.0, "bwd"
    if variant == "no_culling":  # every fifth triangle turned away from the camera
        faces = scene.faces.copy()
        faces[::5] = faces[::5, ::-1]
        s.faces, s.backface_culling = faces, False
        s.faces_uv = np.ascontiguousarray(scene.faces_uv.copy())
        s.faces_uv[::5] = s.faces_uv[::5, ::-1]
        return s, 1.0, "fwd"
    if variant == "perspective":
        s.perspective_correct = True
        return s, 1.0, "fwd+error"
    if variant == "background_image":
        return s, 1.0, "bg"
    if variant == "error":
        return s, 1.0, "error"
    if variant == "error_complete":
        return s, 1.0, "error_complete"
    raise ValueError(variant)


def instances(regime, C, variant, width, textured):
    """The (kernel, template arguments, tile transfer) tuples the device selects for one scene of a case; tile
    transfer is "tma", "coop" (the cooperative fall-back) or None for kernels without tile-shaped transfers.
    A mirror of launch_raster_fwd / launch_raster_fwd_wide (kernels.cu) and launch_bwd / launch_bwd_wide
    (kernels_bwd.cu) with the default process settings."""
    sigma_pos = variant != "sigma0"
    P = variant == "perspective"
    X = bool(textured)
    out = set()
    # antialiase_error mode of the forward passes (the perspective variant runs its forward in both modes)
    modes = {"perspective": (False, True), "error": (True,), "error_complete": (True,)}.get(variant, (False,))
    if C > COLOR_SLAB:  # antialiase_error mode is refused there (kernels.cu: ERROR_MODE_CHANNELS)
        if not modes[0]:
            modes = (False,)
        else:
            return out
    M = maxc(C)
    for R in modes:
        if C <= COLOR_SLAB:
            store = "tma" if C <= 4 and (width * C) % 4 == 0 else "coop"
            out.add(("k_tile_z", (M, P, X, True), store))
        else:
            out.add(("k_tile_z", (1, P, False, False), None))
            out.add(("k_shade", (16, P, X), None))
        if sigma_pos:
            out.add(("k_edge_fwd", (M, P, X, R), None))
    differentiable = variant not in ("no_culling", "perspective")
    if not differentiable:
        return out
    R = variant in ("error", "error_complete")
    B = variant in ("background_image", "error_complete")
    if R:
        out.add(("k_error_image_b", (), None))
    if sigma_pos:
        load = "tma" if C <= 4 and width % 4 == 0 else "coop"
        out.add(("k_raster_bwd", (M, X, R, B), load))
    out.add(("k_interior_bwd", (M, X), None))
    out.add(("k_small_tri_bwd", (M, X), None))
    if B:
        out.add(("k_background_bwd", (M,), None))
    return out


def _all_instances():
    out = set()
    for M, P, X in product((1, 3, 4, 16), (False, True), (False, True)):
        for store in (("tma", "coop") if M <= 4 else ("coop",)):
            out.add(("k_tile_z", (M, P, X, True), store))
        for R in (False, True):
            out.add(("k_edge_fwd", (M, P, X, R), None))
    for P, X in product((False, True), (False, True)):
        out.add(("k_shade", (16, P, X), None))
    for P in (False, True):
        out.add(("k_tile_z", (1, P, False, False), None))
    out.add(("k_error_image_b", (), None))
    for M, X in product((1, 3, 4, 16), (False, True)):
        for R, B in product((False, True), (False, True)):
            for load in (("tma", "coop") if M <= 4 else ("coop",)):
                out.add(("k_raster_bwd", (M, X, R, B), load))
        out.add(("k_interior_bwd", (M, X), None))
        out.add(("k_small_tri_bwd", (M, X), None))
    for M in (1, 3, 4, 16):
        out.add(("k_background_bwd", (M,), None))
    return frozenset(out)


ALL_INSTANCES = _all_instances()

UNREACHABLE = {
    "k_edge_fwd / k_raster_bwd with R above 16 channels": "antialiase_error mode is refused above COLOR_SLAB channels "
                                                          "(kernels.cu: ERROR_MODE_CHANNELS)",
    "any adjoint instance with P": "the library refuses the adjoint of perspective_correct rendering",
    "k_tile_z<MAXC, P, X, false> for MAXC > 1, k_shade<MAXC < 16>": "the unfused z pass + colour pass only run with "
                                                                    "the process-wide DEODR_B200_FUSE_SHADE=0 / "
                                                                    "DEODR_B200_LATE_COLORS=shade switches",
    "k_tile_z<1, P, true, false>": "the unfused z pass reads no colour: it is never instantiated with X",
    "TMA tile transfers for MAXC = 16": "tile stores / loads need C <= 4 (kernels.cu, kernels_bwd.cu: encode_tile_map)",
    "k_small_rec_bwd": "the record-parallel small adjoint only runs with DEODR_B200_SMALL_ADJOINT=record",
}


def all_cases():
    return [(r, C, v) for r in REGIMES for C in CHANNELS for v in VARIANTS]


def case_instances(regime, C, variant):
    out = set()
    for width, _, textured in case_scenes(regime, C, variant):
        out |= instances(regime, C, variant, width, textured)
    return out


def build_case_scene(regime, C, variant, width, height, textured, seed=None):
    """The picture of a case with its variant's flags, padded to the regime's triangle count -> (scene, sigma, call)."""
    if seed is None:
        seed = 1000 * CHANNELS.index(C) + 10 * VARIANTS.index(variant) + list(REGIMES).index(regime)
    base = matrix_scene(width, height, C, seed, textured=textured, background_image=variant == "background_image")
    scene, sigma, call = variant_setup(base, variant)
    total = REGIMES[regime]
    if total is not None:
        scene = with_ballast(scene, total, seed=seed)
    return scene, sigma, call
