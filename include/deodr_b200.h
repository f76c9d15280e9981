/*
 * deodr_b200 - C-ABI of the H100 (sm_90a) differentiable rasteriser.
 *
 * This is the drop-in boundary for the reference's only native entry points,
 *     void renderScene  (Scene, double* image, double* z_buffer, double sigma, bool antialiaseError,
 *                        double* obs, double* err_buffer)                C++/DifferentiableRenderer.h:2717
 *     void renderScene_B(Scene, double* image, double* z_buffer, double* image_b, double sigma, bool,
 *                        double* obs, double* err_buffer, double* err_buffer_b)   C++/DifferentiableRenderer.h:2903
 * which the reference reaches through its Cython shim (deodr/differentiable_renderer_cython.pyx:50 renderSceneCpp,
 * :206 renderSceneBCpp; extern block :11-45).  Plain pointers and sizes only; no torch / numpy types.
 *
 * Two levels:
 *   - deodr_b200_render_host / deodr_b200_render_b_host take the reference's own `struct Scene`
 *     (DifferentiableRenderer.h:56-90: HOST pointers, fp64) and have the reference semantics (image / z_buffer
 *     fully overwritten; gradients ACCUMULATED into scene.*_b; image_b scaled in place is NOT reproduced - it is
 *     left untouched).  Host<->device copies happen inside the call.
 *   - deodr_b200_render / deodr_b200_render_b work on DEVICE-resident buffers in the canonical layout
 *     (fp64 ij / depths / uv / z_buffer, fp32 colours / shade / texture / image / gradients, int32 face ids) on a
 *     caller-supplied CUDA stream; this is what the PyTorch surface uses.
 *
 * All functions return 0 on success or a DEODR_B200_E* code; deodr_b200_last_error() gives the message of the last
 * failure on the calling thread (the reference throws `const char*` instead: DifferentiableRenderer.h:2664-2715,
 * 810, 2924).
 */
#ifndef DEODR_B200_H
#define DEODR_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
    DEODR_B200_OK = 0,
    DEODR_B200_EINVAL = 1,      /* null pointer / bad size / index out of range (checkSceneValid, DR.h:2664) */
    DEODR_B200_EUNSUPPORTED = 2,/* backward with perspective_correct or without backface_culling (DR.h:810, 2924) */
    DEODR_B200_ECUDA = 3,       /* CUDA runtime failure */
    DEODR_B200_ENOMEM = 4,
    DEODR_B200_EREPLAN = 5      /* deferred mode only: a forward overflowed the lists its plan had reserved; the
                                   results of that pass are void, the plan has been rebuilt: run the pass again */
};

/* flags of the *_views entry points */
enum {
    DEODR_B200_ANTIALIASE_ERROR = 1, /* renderScene(..., antialiaseError = true): the silhouette edges overdraw the
                                        squared residual err_buffer instead of the image (DR.h:2066-2618, 2824-2837) */
    DEODR_B200_ERROR_ADJOINT_COMPLETE = 2, /* adjoint of the mode above WITHOUT the reference's dropped row term
                                        (DR.h:2577-2583 never propagates A0y_B): the mathematically complete gradient.
                                        Default (flag clear) = bug-compatible with the reference. */
    /* A forward pass in two calls (deodr_b200_render_views only), for callers that overlap a collective with it:
     * GEOMETRY enqueues the head of the pass - list reset, index check, binning (with DEODR_B200_GEOMETRY_Z=1 in the
     * environment also the z pass, unfused): kernels that read only faces, ij, depths and the flags - and returns;
     * RESUME, with the same arguments, enqueues the rest (edge records, z pass + shading, edge overdraw: the readers of
     * colours / uv / shade / texture).  Between the two the caller makes `stream`
     * wait for whatever produces the colours (cudaStreamWaitEvent on its communication stream's event): unlike the
     * colours-ready event below, that wait is an ordinary stream dependency, so both halves can be captured in CUDA
     * graphs of their own and replayed with the wait in between.  The verdict of the pass belongs to the RESUME call. */
    DEODR_B200_FORWARD_GEOMETRY = 4,
    DEODR_B200_FORWARD_RESUME = 8
};

/* Device-resident scene ("SceneView"): the fields of struct Scene (DR.h:56-90) in the canonical device layout. */
typedef struct DeodrSceneView {
    const uint32_t *faces;            /* [T,3] */
    const uint32_t *faces_uv;         /* [T,3] */
    const double *ij;                 /* [V,2] col 0 = x (image column), col 1 = y (image row) */
    const double *depths;             /* [V] */
    const double *uv;                 /* [Nuv,2] texel coordinates, col 0 = texture column */
    const float *colors;              /* [V,C] */
    const float *shade;               /* [V] */
    const uint8_t *edgeflags;         /* [T,3] */
    const uint8_t *textured;          /* [T] */
    const uint8_t *shaded;            /* [T] */
    const float *texture;             /* [Ht,Wt,C] */
    const float *background_image;    /* [H,W,C] or NULL */
    const float *background_color;    /* [C] (device) or NULL; exactly one of the two backgrounds is set */
    int32_t nb_triangles, nb_vertices, nb_uv;
    int32_t height, width, nb_colors; /* nb_colors = C in [1, 32767]; antialiase_error mode: C <= 16 (more is
                                         DEODR_B200_EUNSUPPORTED).  Above 16 the colour passes run once per slab of
                                         16 channels, with workspace buffers of 16 channels per vertex, texel and pixel */
    int32_t texture_height, texture_width;
    int32_t clockwise, backface_culling, strict_edge, perspective_correct, integer_pixel_centers;
} DeodrSceneView;

/* Device-resident gradient slots (scene.*_b of DR.h:82-86), fp32, ACCUMULATED into.  Any pointer may be NULL. */
typedef struct DeodrGrads {
    float *ij_b;       /* [V,2] */
    float *colors_b;   /* [V,C] */
    float *uv_b;       /* [Nuv,2] */
    float *shade_b;    /* [V] */
    float *texture_b;  /* [Ht,Wt,C]  (summed: the reference's `=` defect DR.h:621-624 is not reproduced) */
} DeodrGrads;

/* The fields of the reference's scene struct (DR.h:56-90) in the SAME ORDER, with HOST pointers.  NOT layout-compatible
 * with `struct Scene`: the reference's five `bool` members are int32_t here (a C ABI has no C++ bool), so offsets and
 * size differ - a caller fills the fields one by one (as the pyx does, pyx:117-171), it cannot pass its Scene through. */
typedef struct DeodrHostScene {
    const uint32_t *faces;
    const uint32_t *faces_uv;
    const double *depths;
    const double *uv;
    const double *ij;
    const double *shade;
    const double *colors;
    const uint8_t *edgeflags;
    const uint8_t *textured;
    const uint8_t *shaded;
    int32_t nb_triangles;
    int32_t nb_vertices;
    int32_t clockwise;
    int32_t backface_culling;
    int32_t nb_uv;
    int32_t height;
    int32_t width;
    int32_t nb_colors;
    const double *texture;
    int32_t texture_height;
    int32_t texture_width;
    const double *background_image;
    const double *background_color;
    double *uv_b;
    double *ij_b;
    double *shade_b;
    double *colors_b;
    double *texture_b;
    int32_t strict_edge;
    int32_t perspective_correct;
    int32_t integer_pixel_centers;
} DeodrHostScene;

/* Opaque per-device workspace.  It holds VIEW SLOTS: the forward pass of view i leaves in slot i the state its adjoint
 * pass replays (tile edge lists, row-span cache, exact-tie table, compact triangle lists) together with the PLAN of the
 * pass - the capacities reserved for every per-tile list, learnt from an earlier pass over a scene of the same shape.
 * deodr_b200_render / _render_b use slot 0; the *_views entry points use slots 0 .. n_views-1.
 * Not thread-safe: one workspace per host thread (the Python layer serialises its calls with a lock). */
typedef struct DeodrWorkspace DeodrWorkspace;

int deodr_b200_workspace_create(DeodrWorkspace **ws, int device);
void deodr_b200_workspace_destroy(DeodrWorkspace *ws);
/* bytes of device memory currently held by the workspace */
int64_t deodr_b200_workspace_bytes(const DeodrWorkspace *ws);
/* number of kernels launched by the library on behalf of this workspace since creation */
int64_t deodr_b200_workspace_launches(const DeodrWorkspace *ws);

/* Forward pass on device buffers (replaces renderScene, DR.h:2717, antialiaseError = false).
 *   image   [H,W,C] fp32, fully overwritten
 *   z_buffer[H,W]   fp64, fully overwritten (bit-identical to the reference; +inf = background)
 *   owner   [H,W]   int32, adjoint-owner triangle per pixel (-1 = background); state consumed by the backward pass
 *   face_id [H,W]   int32 or NULL: forward owner (lowest index at the minimum z), i.e. rint() of the reference's
 *                   render_deferred face-id channel
 * `stream` is a cudaStream_t.  The pass is enqueued without waiting for the device; before returning the call reads
 * the verdict word the binning kernels publish in pinned memory (they are the first kernels of the pass, the rest of
 * it is already queued behind them) and, if a list outgrew its plan, re-plans and runs the pass again - the caller
 * always gets a valid result.  The first pass over a new shape builds the plan (one count pass + one read-back). */
int deodr_b200_render(DeodrWorkspace *ws, const DeodrSceneView *scene, double sigma, float *image, double *z_buffer,
                      int32_t *owner, int32_t *face_id, void *stream);

/* Adjoint pass on device buffers (replaces renderScene_B, DR.h:2903, antialiaseError = false).
 * Must follow deodr_b200_render on the same workspace, scene and sigma, with the z_buffer / owner arrays that pass
 * wrote (checked: DEODR_B200_EINVAL otherwise).  image_b [H,W,C] fp32 is read-only.  Gradients are accumulated (+=)
 * into `grads`.  No host synchronisation. */
int deodr_b200_render_b(DeodrWorkspace *ws, const DeodrSceneView *scene, double sigma, const double *z_buffer,
                        const int32_t *owner, const float *image_b, const DeodrGrads *grads, void *stream);

/* ---- batch of views (SURVEY 8b/8e; the frames loop of deodr/mesh_fitter.py:511-549) ---------------------------
 * Per-view device framebuffers.  Forward outputs: image, z_buffer, owner (required), face_id, barycentric (optional);
 * antialiase_error mode: obs [H,W,C] in, err_buffer [H,W] out.  Adjoint inputs: image_b [H,W,C] (normal mode) or
 * err_buffer_b [H,W] + obs + the forward's image (antialiase_error mode). */
typedef struct DeodrViewIO {
    float *image;              /* [H,W,C] */
    double *z_buffer;          /* [H,W] */
    int32_t *owner;            /* [H,W] */
    int32_t *face_id;          /* [H,W] or NULL */
    float *barycentric;        /* [H,W,3] or NULL: interpolation weights of the forward owner's three vertices (0 on the
                                  background): with face_id, the G-buffer of Scene3D.render_deferred
                                  (deodr/differentiable_renderer.py:1053-1174) without its C = 14 interpolated channels */
    const float *obs;          /* [H,W,C] or NULL */
    float *err_buffer;         /* [H,W] or NULL */
    const float *image_b;      /* [H,W,C] or NULL */
    const float *err_buffer_b; /* [H,W] or NULL */
} DeodrViewIO;

/* Forward passes of n_views views (views[i] -> slot i), interleaved on a few internal streams forked from / joined
 * to `stream`.  Same verdict handling as deodr_b200_render, after ALL the views have been enqueued. */
int deodr_b200_render_views(DeodrWorkspace *ws, int n_views, const DeodrSceneView *views, const DeodrViewIO *io,
                            double sigma, int flags, void *stream);

/* Adjoint passes of the same views.  grads[i] may alias each other: gradients of the parameters the views share
 * (colors_b, uv_b, shade_b, texture_b) accumulate in place - the `+=` of deodr/mesh_fitter.py:518-527 - while each view
 * gets its own ij_b. */
int deodr_b200_render_b_views(DeodrWorkspace *ws, int n_views, const DeodrSceneView *views, const DeodrViewIO *io,
                              const DeodrGrads *grads, double sigma, int flags, void *stream);

/* Gradient of a view's background, fp32 device buffers ACCUMULATED into (+=) like DeodrGrads.  Set the one that matches
 * the background the view is rendered with (the other stays NULL); either may be NULL.  Entries of different views may
 * alias: a background colour shared by the views sums their gradients, like colors_b.  The reference has no
 * counterpart (its struct Scene has no background gradient slot). */
typedef struct DeodrBackgroundGrads {
    float *background_image_b; /* [H,W,C] or NULL: only for a view rendered with background_image */
    float *background_color_b; /* [C] or NULL: only for a view rendered with background_color */
} DeodrBackgroundGrads;

/* deodr_b200_render_b_views plus the gradient of the background: bg_grads[i] (n_views entries) receives the colour
 * adjoint of the pixels view i shows its background at, times the transparency of the silhouette edges drawn over them
 * (antialiase_error mode: the residual's adjoint there).  bg_grads == NULL, or every pointer in it NULL, runs exactly
 * deodr_b200_render_b_views.  DEODR_B200_EINVAL when a gradient does not match the view's kind of background.  Same
 * flags, deferred mode and stream-capture behaviour as render_b_views; a pass that overflowed its plan accumulates
 * nothing here either. */
int deodr_b200_render_b_views_background(DeodrWorkspace *ws, int n_views, const DeodrSceneView *views,
                                         const DeodrViewIO *io, const DeodrGrads *grads,
                                         const DeodrBackgroundGrads *bg_grads, double sigma, int flags, void *stream);

/* Comparison of a view's render with an observed image (Scene2D.render_compare_and_backward,
 * deodr/differentiable_renderer.py:701-734), computed on the device right after the view's forward pass.  With m the
 * mask (1 everywhere when NULL) and d = image - obs:
 *   normal mode            loss = sum_p m_p * sum_c d_{p,c}^2   and   image_b = 2 * m * d, its exact gradient (the
 *                          reference's image_b; the reference's reported err squares the mask, sum (m*d)^2, which is the
 *                          same loss for a binary mask)
 *   antialiase_error mode  loss = sum_p m_p * err_buffer_p, whose adjoint input is err_buffer_b = m
 * The loss is summed in fp64 in a fixed order: the same inputs give the same loss bit for bit, alone or in a batch. */
typedef struct DeodrCompareIO {
    const float *obs;   /* [H,W,C], required */
    const float *mask;  /* [H,W] or NULL (all ones) */
    float *image_b;     /* [H,W,C] out or NULL (loss only); normal mode only (must be NULL with ANTIALIASE_ERROR) */
    float *err_pixel;   /* [H,W] out or NULL: m * sum_c d^2, or m * err_buffer in antialiase_error mode */
    double *loss;       /* device scalar, WRITTEN (not accumulated); must not alias another view's */
} DeodrCompareIO;

/* deodr_b200_render_views, then the comparison of every view (cmp[i], n_views entries) on the view's lane.  The caller
 * then runs deodr_b200_render_b_views (or _background) with io.image_b = cmp.image_b, or in antialiase_error mode with
 * io.err_buffer_b = the mask (all ones without one); in that mode io.obs must be cmp.obs.  DEODR_B200_EINVAL for a NULL
 * obs or loss, an image_b in antialiase_error mode, a different io.obs there, or two views sharing one loss.  Deferred
 * mode, stream capture and the overflow rule are those of render_views: a pass that overflowed its plan leaves its loss
 * void like its image.  With FORWARD_GEOMETRY nothing is compared; the FORWARD_RESUME call compares.  cmp == NULL
 * launches exactly what deodr_b200_render_views launches. */
int deodr_b200_render_compare_views(DeodrWorkspace *ws, int n_views, const DeodrSceneView *views, const DeodrViewIO *io,
                                    const DeodrCompareIO *cmp, double sigma, int flags, void *stream);

/* Deferred mode (on = 1): the entry points never read the verdict themselves - nothing in them touches the host side
 * of the device, so a forward + adjoint sequence can be captured in a CUDA graph (they also behave this way whenever
 * `stream` is being captured).  The caller then asks deodr_b200_workspace_status() after synchronising: OK, or
 * DEODR_B200_EREPLAN when a pass overflowed its plan (its outputs are void - gradients were not accumulated -, the plan
 * has been rebuilt; re-capture and run again). */
int deodr_b200_workspace_set_deferred(DeodrWorkspace *ws, int on);
int deodr_b200_workspace_status(DeodrWorkspace *ws);
/* Inspection of the binning pass (tests): what the last forward pass of view slot `view` appended, copied to host
 * memory after a device synchronisation.  sizes[3] <- (tiles, reserved records, small-id capacity); then, for every
 * pointer that is not NULL: scal[32] <- the pass's device scalars (the number of small ids at index 2),
 * small_offset[tiles + 1] <- the plan's record segments, small_cursor[tiles] <- records appended per tile (beyond the
 * segment's size on overflow), small_recs[reserved] <- the 64-byte records, small_ids[capacity] <- the list of small
 * triangles.  EINVAL when the slot holds no planned pass. */
int deodr_b200_view_bins(DeodrWorkspace *ws, int view, int32_t *sizes, int32_t *scal, int32_t *small_offset,
                         int32_t *small_cursor, void *small_recs, int32_t *small_ids);

/* "Colours ready" event (a cudaEvent_t, or NULL): the NEXT forward call makes only the kernels that read the vertex
 * colours (k_shade, the silhouette-edge records) wait for it; the geometry half of the pass - binning and the z pass,
 * more than half of its duration - starts at once.  This is how the all-reduce of the shared colour gradient and the
 * optimiser update that follows it (on the caller's communication stream, which records the event) overlap the next
 * step instead of sitting between two steps (DESIGN.md section 8).  One-shot: consumed by that call. */
int deodr_b200_workspace_set_colors_ready(DeodrWorkspace *ws, void *event);

/* Stamp of the last forward pass that ran in slot `view` (0 = none yet): lets a caller that keeps several forward
 * results alive (autograd) detect that the slot has been reused before it runs the adjoint. */
int64_t deodr_b200_view_generation(const DeodrWorkspace *ws, int view);

/* Reference-shaped host entry points (fp64 host buffers in, fp64 host buffers out). */
int deodr_b200_render_host(DeodrWorkspace *ws, const DeodrHostScene *scene, double *image, double *z_buffer,
                           double sigma, int antialiase_error, const double *obs, double *err_buffer);
int deodr_b200_render_b_host(DeodrWorkspace *ws, const DeodrHostScene *scene, double *image, double *z_buffer,
                             double *image_b, double sigma, int antialiase_error, const double *obs,
                             double *err_buffer, double *err_buffer_b);

/* Zero-fills `n` host buffers (ptrs[i], bytes[i]) with the host path's copy threads: what Scene2D.clear_gradients
 * (deodr/differentiable_renderer.py:599-610, five numpy `fill(0)` calls = 30+ MB on a 1M-triangle scene) does before
 * every adjoint call, at memory speed instead of one core's. */
int deodr_b200_host_zero(DeodrWorkspace *ws, void *const *ptrs, const int64_t *bytes, int n);

/* Index-range validation of a device scene (checkSceneValid, DR.h:2703-2714); synchronises the stream. */
int deodr_b200_check_scene(DeodrWorkspace *ws, const DeodrSceneView *scene, void *stream);

/* ---- the steps either side of the raster (SURVEY 8f1 / 8f2), on device buffers ------------------------------- */

/* Pinhole camera with the reference's OpenCV-style distortion (deodr/differentiable_renderer.py:341-438):
 * extrinsic [3,4] row-major, intrinsic [3,3] row-major, distortion k1 k2 p1 p2 k3 (has_distortion = 0: ignored). */
typedef struct DeodrCamera {
    double extrinsic[12];
    double intrinsic[9];
    double distortion[5];
    int32_t has_distortion;
    int32_t pad;
} DeodrCamera;

/* Camera.project_points (differentiable_renderer.py:391-418): points [N,3] fp64 -> ij [N,2] (col 0 = x), depths [N]. */
int deodr_b200_project_points(const double *points, int n, const DeodrCamera *camera, double *ij, double *depths,
                              void *stream);
/* Camera.project_points_backward (:420-438): points_b [N,3] fp64 += J^T (ij_b, depths_b); ij_b fp32 [N,2] is the
 * rasteriser's gradient, depths_b fp64 [N] or NULL.  The reference transposes twice where the adjoint must not: it
 * multiplies ij_b by K[:2,:2]^T (:399, :412) where the adjoint of `projected . K[:2,:2]^T` needs K[:2,:2] (the same
 * only for zero skew and K[1,0] == 0), and its last line multiplies by R^T, `p_camera_b.dot(extrinsic[:3,:3].T)`
 * (:438), where the adjoint of world_to_camera needs R (the same only for a symmetric rotation; INTEGRATION.md,
 * defect #3).  reference_transpose = 1 reproduces both of the reference's transposes; 0 is the true adjoint, J^T
 * (ij_b, depths_b), for any intrinsic matrix and rotation. */
int deodr_b200_project_points_b(const double *points, int n, const DeodrCamera *camera, const float *ij_b,
                                const double *depths_b, double *points_b, int reference_transpose, void *stream);
/* The true adjoint of deodr_b200_project_points from an fp64 ij_b [N,2] (an autograd gradient, which the fp32 ij_b of
 * deodr_b200_project_points_b would round): points_b [N,3] fp64 = J^T (ij_b, depths_b), OVERWRITTEN.  ij_b and
 * depths_b [N] may each be NULL (zero). */
int deodr_b200_project_points_b64(const double *points, int n, const DeodrCamera *camera, const double *ij_b,
                                  const double *depths_b, double *points_b, void *stream);

/* ---- the camera in device memory, and its gradient ----
 * The camera vector is [26] fp64 in DEVICE memory: extrinsic [R | t] (12, row-major: R row r at 4r, t_r at 4r + 3),
 * intrinsic (9, row-major, at 12) and distortion k1 k2 p1 p2 k3 (5, at 21).  has_distortion (host) selects the
 * distortion code; without it the distortion entries are not read.  A fit can update the vector on the device between
 * calls without a host read. */

/* deodr_b200_project_points with the camera vector read from device memory: for the same values, ij and depths are
 * bit-identical.  DEODR_B200_EINVAL for n < 0 or a NULL pointer (points, ij, depths only when n > 0). */
int deodr_b200_project_points_dev(const double *points, int n, const double *camera, int has_distortion, double *ij,
                                  double *depths, void *stream);
/* The true adjoint of deodr_b200_project_points_dev, in the points and in the camera, in one pass over the points.
 * Upstream: ij_b [N,2] fp32 (the rasteriser's) or ij_b64 fp64 (an autograd gradient), at most one of them (neither:
 * zero), and depths_b [N] fp64 or NULL (zero).
 *   points_b [N,3]: NULL (not written), or J^T (ij_b, depths_b) accumulated (accumulate != 0) or overwritten - bit-
 *            identical to deodr_b200_project_points_b (reference_transpose = 0) and _b64 respectively.
 *   camera_b [26]: overwritten, in the camera vector's layout.  With pc = R p + t per point and pc_b its gradient:
 *            R_b = sum pc_b p^T, t_b = sum pc_b; intrinsic rows 0 and 1 from ij_b and the distorted normalised
 *            coordinates; intrinsic row 2 is 0 (the projection never reads it); distortion_b from the partial
 *            derivatives of the distortion polynomial, 0 when has_distortion = 0.
 * A point whose upstream gradients (ij_b and depths_b) are all exactly 0 adds nothing to camera_b: a point on the
 * camera plane or culled behind the camera would otherwise make the sum NaN through 0 * inf.  Its points_b is written
 * all the same.  camera_b is summed in a fixed order without atomics (bit-reproducible; `scratch` as for the fitting
 * entry points below, whose size it keeps).  The reference's transposed adjoint has no camera gradient, so there is no
 * reference_transpose here.  DEODR_B200_EINVAL before any launch for n < 0, a NULL camera, camera_b or scratch, NULL
 * points with n > 0, or both ij_b and ij_b64.  No host synchronisation. */
int deodr_b200_project_points_camera_b(const double *points, int n, const double *camera, int has_distortion,
                                       const float *ij_b, const double *ij_b64, const double *depths_b,
                                       double *points_b, int accumulate, double *camera_b, double *scratch,
                                       void *stream);

/* Gouraud luminosity of Scene3D.compute_vertices_luminosity + _compute_vertices_colors_with_illumination (:814-833):
 *   luminosity[v] = max(0, -dot(normals[v], light_directional)) + ambient;  colors[v,c] = vertex_colors[v,c] * luminosity[v]
 * normals [V,3] fp64, vertex_colors [V,C] fp64 or NULL (then only the luminosity is written); outputs fp32 (the
 * rasteriser's attribute type), either may be NULL.  light_directional: three doubles in HOST memory, NULL = no
 * directional light. */
int deodr_b200_vertex_luminosity(const double *normals, const double *vertex_colors, int n_vertices, int nb_colors,
                                 const double *light_directional, double ambient, float *luminosity, float *colors,
                                 void *stream);
/* adjoint (:835-850) from colors_b [V,C] fp32 (and / or luminosity_b [V] fp32, added to it):
 * vertex_colors_b [V,C] = colors_b * luminosity (overwritten, as the reference assigns it), normals_b [V,3] overwritten,
 * light_b[4] (device, fp64) += (light_directional_b[3], light_ambient_b).  Any output may be NULL. */
int deodr_b200_vertex_luminosity_b(const double *normals, const double *vertex_colors, int n_vertices, int nb_colors,
                                   const double *light_directional, double ambient, const float *colors_b,
                                   const float *luminosity_b, double *normals_b, double *vertex_colors_b,
                                   double *light_b, void *stream);

/* Static adjacency of a triangulated mesh (device pointers; built once per mesh on the host, e.g. by
 * deodr_b200.mesh_ops.MeshTopology from the same arrays as TriMeshAdjacencies, deodr/triangulated_mesh.py:21-98). */
typedef struct DeodrMeshTopology {
    const uint32_t *faces;            /* [T,3] */
    const int32_t *faces_edges;       /* [T,3] unique-edge id of the face's edges (v0,v1), (v1,v2), (v2,v0) */
    const int32_t *edge_face_offset;  /* [E+1] CSR: faces incident to every unique edge ... */
    const int32_t *edge_face_index;   /* ... (length 3T) */
    const int32_t *vertex_face_offset;/* [V+1] CSR: faces incident to every vertex (ascending), with multiplicity ... */
    const int32_t *vertex_face_index; /* ... (length 3T) */
    int32_t nb_faces, nb_edges, nb_vertices, clockwise;
} DeodrMeshTopology;

/* TriMeshAdjacencies.edge_on_silhouette (triangulated_mesh.py:153-166): edgeflags[T,3] = "exactly one of the faces
 * that share the edge is visible", visibility from the 2D winding of ij [V,2] (exact: same products and difference as
 * np.cross).  face_visible [T] u8 is scratch / by-product. */
int deodr_b200_edge_on_silhouette(const DeodrMeshTopology *mesh, const double *ij, uint8_t *face_visible,
                                  uint8_t *edgeflags, void *stream);

/* compute_face_normals + compute_vertex_normals (triangulated_mesh.py:113-143): unit face normals [T,3] (sign by
 * `clockwise`), summed over the faces incident to each vertex and normalised -> vertex_normals [V,3]. */
int deodr_b200_vertex_normals(const DeodrMeshTopology *mesh, const double *vertices, double *face_normals,
                              double *vertex_normals, void *stream);
/* compute_vertex_normals_backward + compute_face_normals_backward (:145-151, :125-135): vertex_normals_b [V,3] ->
 * vertices_b [V,3] (accumulated, fp64 atomics).  vertex_scratch [V,3] fp64 is scratch. */
int deodr_b200_vertex_normals_b(const DeodrMeshTopology *mesh, const double *vertices, const double *vertex_normals_b,
                                double *vertex_scratch, double *vertices_b, void *stream);

/* ---- mesh fitting: the steps of MeshDepthFitter / MeshRGBFitterWithPose / MeshRGBFitterWithPoseMultiFrame.step
 * (deodr/mesh_fitter.py) around the
 * render, on fp64 device buffers.  Every sum these entry points report (energies, translation_b, quaternion_b,
 * color_b, light_b) is reproducible bit for bit: fixed-order fp64 partials per CTA, added in CTA order by the last
 * CTA, no atomics on them.  `scratch` is a device buffer of deodr_b200_fitter_scratch_bytes() bytes, zeroed once
 * before its first use (every call leaves it zeroed again); calls that share one must be ordered (one stream).
 * Quaternions are stored (x, y, z, w); qrot(q, v) = v + 2 (w (u x v) + u x (u x v)) with u = (x, y, z). */
int64_t deodr_b200_fitter_scratch_bytes(void);

/* Rigid pose: vertices [n,3] <- vertices - mean(vertices) (in place), then
 * transformed [n,3] = qrot(quaternion / |quaternion|, vertices) + translation.  quaternion [4], translation [3]: device. */
int deodr_b200_pose(double *vertices, int n, const double *quaternion, const double *translation, double *transformed,
                    double *scratch, void *stream);
/* Its adjoint from transformed_b [n,3], at the centred vertices: translation_b [3] = sum transformed_b;
 * quaternion_b [4] = the adjoint through qrot and the normalisation (q_b = (qh_b - qh (qh . qh_b)) / |q|);
 * vertices_b [n,3] = the adjoint of qrot in the vertices minus its mean over the vertices.  All outputs overwritten. */
int deodr_b200_pose_b(const double *vertices, int n, const double *quaternion, const double *transformed_b,
                      double *vertices_b, double *quaternion_b, double *translation_b, double *scratch, void *stream);

/* The rigid poses of MeshRGBFitterWithPoseMultiFrame: one mesh seen in nb_frames frames, each with its own pose.
 * vertices [n,3] <- vertices - mean(vertices) (in place, once), then for every frame f
 * transformed [nb_frames,n,3][f] = qrot(quaternions[f] / |quaternions[f]|, vertices) + translations[f], with
 * quaternions [nb_frames,4] and translations [nb_frames,3] on the device.  With nb_frames = 1 it computes what
 * deodr_b200_pose computes, with the same arithmetic. */
int deodr_b200_pose_frames(double *vertices, int n, const double *quaternions, const double *translations,
                           int nb_frames, double *transformed, double *scratch, void *stream);
/* Its adjoint from transformed_b [nb_frames,n,3], at the centred vertices, scaled by `scale`:
 *   translations_b [nb_frames,3]: translations_b[f] = scale * sum_v transformed_b[f];
 *   quaternions_b [nb_frames,4]:  the adjoint of frame f through qrot and its normalisation, times scale;
 *   vertices_b [n,3]:             scale * sum_f qrot_f^T(transformed_b[f]), minus its mean over the vertices when
 *                                 center_vertices_b is non-zero (the reference does so while iter < 500).
 * The frame sum of the data term is folded in here: `scale` is the data weight cdata / nb_frames, applied to the
 * adjoints in fp64 (the comparison runs unweighted, so its per-frame losses and image_b are those of weight 1), and
 * when losses [nb_frames] (the per-frame fp64 losses of the comparison) is given, *energy_data =
 * scale * sum_f losses[f], the frames added in order; losses and energy_data are both given or both NULL.  The colour
 * and light adjoints, which do not pass through here, carry the weight in their step factors instead.
 * All outputs overwritten and reproducible bit for bit.  nb_frames from 1 to 2340 (DEODR_B200_EUNSUPPORTED above);
 * with nb_frames = 1, scale = 1 and center_vertices_b = 1 the outputs are those of deodr_b200_pose_b. */
int deodr_b200_pose_frames_b(const double *vertices, int n, const double *quaternions, const double *transformed_b,
                             int nb_frames, int center_vertices_b, double scale, const double *losses,
                             double *energy_data, double *vertices_b, double *quaternions_b, double *translations_b,
                             double *scratch, void *stream);

/* Laplacian rigidity (LaplacianRigidEnergy.evaluate): grad [n,3] = cregu L (L (vertices - vertices_ref)) per
 * coordinate, *energy = 1/2 <vertices - vertices_ref, grad>, with L = D - A, A the "shares a face" adjacency and D its
 * degree, given as a neighbour CSR (neighbour_offset [n+1], neighbour_index: the neighbours of every vertex, itself
 * excluded).  vertex_scratch [n,3] fp64 holds L (vertices - vertices_ref). */
int deodr_b200_laplacian_rigid(const int32_t *neighbour_offset, const int32_t *neighbour_index, int n,
                               const double *vertices, const double *vertices_ref, double cregu, double *grad,
                               double *energy, double *vertex_scratch, double *scratch, void *stream);

/* Depth comparison of MeshDepthFitter.step, one pass over the pixels of a one-channel render (fp32) and an observation
 * obs (fp64): d = clip(render, 0, max_depth), depth = d, diff = (d - obs)^2, *energy = sum diff (fp64),
 * depth_b = 2 (d - obs), 0 where render < 0 or render > max_depth.  depth and diff may be NULL. */
int deodr_b200_depth_compare(const float *render, const double *obs, int64_t pixels, double max_depth, double *depth,
                             double *diff, float *depth_b, double *energy, double *scratch, void *stream);

/* The colours of MeshRGBFitterWithPose: every vertex has the colour color [C] (device), lit by light [4] (device:
 * directional x, y, z, ambient): colors [n,C] fp32 = color * (max(0, -<normals, light_xyz>) + ambient). */
int deodr_b200_uniform_color_luminosity(const double *normals, int n, const double *color, int nb_colors,
                                        const double *light, float *colors, void *stream);
/* Its adjoint from colors_b [n,C] fp32: color_b [C] = sum over the vertices of colors_b * luminosity, light_b [4]
 * (directional, ambient), normals_b [n,3] (or NULL); all overwritten.  nb_colors 1 to 4 (else DEODR_B200_EUNSUPPORTED). */
int deodr_b200_uniform_color_luminosity_b(const double *normals, int n, const double *color, int nb_colors,
                                          const double *light, const float *colors_b, double *normals_b,
                                          double *color_b, double *light_b, double *scratch, void *stream);

/* Per-vertex colours lit by a light in DEVICE memory, as Scene3DPytorch lights them: light [4] fp64 = (directional x,
 * y, z, ambient); colors [n,C] fp64 = vertex_colors [n,C] * (max(0, -<normals, light_xyz>) + ambient), the directional
 * term only when `directional` is non-zero (else light[0..2] are not read).  Any nb_colors >= 1.  fp64 output, so that
 * an fp64 caller differentiates exactly what it computes; the rasteriser's fp32 copy rounds it once, as the fp32
 * colours of deodr_b200_vertex_luminosity are rounded. */
int deodr_b200_lit_vertex_colors(const double *normals, const double *vertex_colors, int n, int nb_colors,
                                 const double *light, int directional, double *colors, void *stream);
/* Its adjoint from colors_b [n,C], fp32 (the rasteriser's, colors_b_fp64 = 0) or fp64 (colors_b_fp64 = 1):
 * vertex_colors_b [n,C] = colors_b * luminosity, normals_b [n,3], light_b [4] = (directional_b, ambient_b); all
 * overwritten.  light_b is summed like the other reductions of this section (fixed order, bit-reproducible; `scratch`
 * as above); its directional part is 0 without a directional light. */
int deodr_b200_lit_vertex_colors_b(const double *normals, const double *vertex_colors, int n, int nb_colors,
                                   const double *light, int directional, const void *colors_b, int colors_b_fp64,
                                   double *normals_b, double *vertex_colors_b, double *light_b, double *scratch,
                                   void *stream);

/* ---- per-pixel (Phong) shading of a rasterised G-buffer ------------------------------------------------------------
 * A mesh's untextured scene rendered with K = C + 7 colour channels per vertex - C albedo channels (the unlit vertex
 * colours), the unit vertex normal (3), the vertex's world position (3) and a coverage channel equal to 1 at every
 * vertex - over a background of 0 in every channel, with the view's own sigma, silhouette flags, culling and winding,
 * gives at each pixel (A[0..C), N, X, a).  With l the directional light (direction times intensity, 0 without one),
 * ambient, ks >= 0 (specular strength), e (shininess), cam the camera centre -R^T t and bg the view's background:
 *
 *   n    = N / |N|                                    (0 when |N| = 0)
 *   diff = max(0, -<n, l>)                            (0 when l = 0: the normals are then not read)
 *   spec = 0 when a = 0 or |l| = 0; otherwise
 *          x = X / a,  v = normalize(cam - x),  h = normalize(-l/|l| + v)  (h = 0 when -l/|l| + v = 0),
 *          s = max(0, <n, h>),  spec = a * ks * |l| * s^e   (s^e = 0, with its derivatives, at s = 0)
 *   image[c] = A[c] * (ambient + diff) + spec + (1 - a) * bg[c]
 *
 * Over the background the raster gives alpha * front in every channel, so n and x are the front surface's and the image
 * is alpha * phong(front) + (1 - alpha) * bg: DEODR's antialiased blend of the shaded surface.  At a self-occlusion
 * silhouette the front and back attributes are mixed before shading: the result is continuous but is not the blend of
 * the two shaded surfaces.  With ks = 0 and all vertex normals equal it is the Gouraud image.  The interpolation is the
 * rasteriser's (linear in screen space).  NaN normals (a zero-area face) propagate as in the Gouraud path. */
typedef struct DeodrPhongIO {
    const float *channels;        /* [H,W,K] the raster output, K = C + 7 */
    const double *params;         /* [6] device: l (3), ambient, ks, e */
    const double *camera_center;  /* [3] device: -R^T t */
    const float *background;      /* [C] device: the view's background colour */
    float *image;                 /* [H,W,C] forward output, overwritten */
    const float *image_b;         /* [H,W,C] adjoint input */
    float *channels_b;            /* [H,W,K] adjoint output, overwritten (the coverage channel's a_b included) */
    double *params_b;             /* [6] adjoint output, overwritten: (l_b (3), ambient_b, ks_b, e_b) */
    int32_t H, W, C;
    int32_t off_albedo, off_normal, off_position, off_coverage; /* channel offsets, tiling [0, C + 7) */
    double *camera_center_b;      /* [3] optional adjoint output, overwritten: the gradient of camera_center (NULL: not
                                     computed, and the adjoint is exactly that of a call without this field) */
} DeodrPhongIO;

/* image from channels (one thread per pixel, fp64 maths).  Reads io->channels, params, camera_center, background and
 * writes io->image; the adjoint fields are not read.  DEODR_B200_EINVAL before any launch for a NULL io or buffer,
 * H or W < 1, C outside [1, 32760], or offsets that do not tile [0, C + 7).  No host synchronisation. */
int deodr_b200_phong_shade(const DeodrPhongIO *io, void *stream);
/* Its adjoint from io->image_b: channels_b and params_b overwritten; params_b (and camera_center_b when it is given)
 * summed over the pixels without atomics in a fixed order (bit-reproducible; `scratch` as above).  io->image is not
 * read.  Same refusals; no host synchronisation. */
int deodr_b200_phong_shade_b(const DeodrPhongIO *io, double *scratch, void *stream);

/* ---- spherical-harmonics environments -------------------------------------------------------------------------------
 * A second-order spherical-harmonics (SH) environment adds coloured, low-frequency light from every direction to the
 * directional light and the ambient term (Ramamoorthi & Hanrahan, 2001).  With n = (x, y, z) the unit outward normal
 * (the normal the directional term uses, its sign set by the winding), the nine real basis functions of bands 0 to 2,
 * without the Condon-Shortley phase, are
 *
 *   Y0 = 1 / (2 sqrt(pi))           = 0.282094791773878
 *   Y1 = sqrt(3 / (4 pi)) y,  Y2 = sqrt(3 / (4 pi)) z,  Y3 = sqrt(3 / (4 pi)) x            (0.488602511902920)
 *   Y4 = sqrt(15 / (4 pi)) x y,  Y5 = sqrt(15 / (4 pi)) y z,  Y7 = sqrt(15 / (4 pi)) x z    (1.092548430592079)
 *   Y6 = sqrt(5 / (16 pi)) (3 z^2 - 1)                                                     (0.315391565252520)
 *   Y8 = sqrt(15 / (16 pi)) (x^2 - y^2)                                                    (0.546274215296040)
 *
 * The coefficients sh [9, S] fp64 live in device memory: S = 1 is a grey environment applied to every channel (any
 * channel count), S = C a coloured one (C from 1 to 4); anything else is DEODR_B200_EUNSUPPORTED before any launch.
 * sh_c(n) = sum_{k = 0..8} sh[k, c] Y_k(n), summed in that order, is added after the existing terms:
 *
 *   Gouraud (per vertex)  colors[v,c] = vertex_colors[v,c] * ((max(0, -<n_v, l>) + ambient) + sh_c(n_v))
 *   textured              shade[v]    = (max(0, -<n_v, l>) + ambient) + sh(n_v)                      (S = 1 only)
 *   Phong (per pixel)     image[c]    = A[c] * ((ambient + diff) + sh_c(n)) + spec + (1 - a) bg[c]
 *                         with n = N / |N| of DeodrPhongIO (the basis is evaluated at n = 0 when |N| = 0); the
 *                         specular term stays tied to the directional light
 *
 * so sh = 0 gives bit for bit the outputs of the calls without an environment.  A NaN normal (a zero-area face)
 * propagates into the SH term as into the directional one.  The normals are read whenever an environment is given,
 * with or without a directional light.
 *
 * Adjoint, with g_c = colors_b[v,c] * vertex_colors[v,c] (Gouraud), shade_b[v] (textured) or image_b[p,c] * A[p,c]
 * (Phong): sh_b[k, c] = sum over the vertices (pixels) of g_c Y_k(n) (S = 1: g summed over the channels), and the
 * normals receive sum_c g_c sum_k sh[k, c] grad Y_k(n) (Phong: through the adjoint of n = N / |N|).  Every sum is fp64,
 * in a fixed order, bit-reproducible (`scratch` as above). */

/* deodr_b200_lit_vertex_colors with an environment sh [9, sh_channels] (device): colors [n,C] fp64 as above, or,
 * with vertex_colors NULL, the luminosity [n] of a textured mesh (nb_colors 1, sh_channels 1).  DEODR_B200_EINVAL for
 * a NULL buffer when n > 0; DEODR_B200_EUNSUPPORTED for a bad sh_channels; both before any launch. */
int deodr_b200_sh_lit_vertex_colors(const double *normals, const double *vertex_colors, int n, int nb_colors,
                                    const double *light, int directional, const double *sh, int sh_channels,
                                    double *colors, void *stream);
/* Its adjoint from colors_b ([n,C], or [n] with vertex_colors NULL; fp32, or fp64 with colors_b_fp64 = 1):
 * normals_b [n,3], vertex_colors_b [n,C] (not written, and may be NULL, without vertex_colors), light_b [4] =
 * (directional_b, ambient_b) and sh_b [9, sh_channels], all overwritten.  Same refusals, n >= 1. */
int deodr_b200_sh_lit_vertex_colors_b(const double *normals, const double *vertex_colors, int n, int nb_colors,
                                      const double *light, int directional, const double *sh, int sh_channels,
                                      const void *colors_b, int colors_b_fp64, double *normals_b,
                                      double *vertex_colors_b, double *light_b, double *sh_b, double *scratch,
                                      void *stream);
/* deodr_b200_phong_shade with an environment sh [9, sh_channels] (device): the Phong form above.  DeodrPhongIO is
 * read as by deodr_b200_phong_shade; its layout is unchanged.  Same refusals, plus DEODR_B200_EINVAL for a NULL sh and
 * DEODR_B200_EUNSUPPORTED for a bad sh_channels, before any launch. */
int deodr_b200_sh_phong_shade(const DeodrPhongIO *io, const double *sh, int sh_channels, void *stream);
/* Its adjoint: deodr_b200_phong_shade_b's outputs with the environment's share, and sh_b [9, sh_channels] overwritten
 * (fixed-order sum, bit-reproducible).  Same refusals, plus DEODR_B200_EINVAL for a NULL sh_b. */
int deodr_b200_sh_phong_shade_b(const DeodrPhongIO *io, const double *sh, int sh_channels, double *sh_b,
                                double *scratch, void *stream);

/* ---- per-pixel shading of a textured mesh: the albedo from a raster of its own ----------------------------------------
 * A textured mesh's albedo is its texture, sampled per pixel, which a G-buffer of vertex attributes cannot carry.  The
 * two rasters below share the view's geometry (ij, depths, faces, silhouette flags, culling, winding and sigma):
 *
 *   albedo [H,W,C]    the textured scene with shade = 1 at every vertex over a zero background: A = alpha * texture
 *   channels [H,W,7]  an untextured scene of (unit vertex normal, world position, 1) over a zero background: (N, X, a)
 *
 * and the image is the Phong form above, environment included, with A read from `albedo`:
 *
 *   image[c] = A[c] * ((ambient + diff) + sh_c(n)) + spec + (1 - a) * bg[c]
 *
 * Over the background both rasters blend against 0 with the same coverage, so the image is still DEODR's antialiased
 * blend of the shaded surface; at self-occlusion silhouettes the approximation is that of the G-buffer form.
 *
 * DeodrPhongIO is read as by deodr_b200_phong_shade with io->channels [H,W,7]: off_albedo is -1 and off_normal,
 * off_position and off_coverage tile [0, 7).  sh [9, sh_channels] as above, or sh NULL with sh_channels 0 for no
 * environment.  DEODR_B200_EINVAL before any launch for a NULL io or buffer (albedo included), H or W < 1, C outside
 * [1, 32760], offsets that do not tile [0, 7) or an off_albedo other than -1, or a NULL sh with sh_channels != 0;
 * DEODR_B200_EUNSUPPORTED for a bad sh_channels.  No host synchronisation.  The kernels are those of
 * deodr_b200_phong_shade and deodr_b200_sh_phong_shade, with the albedo read from its own buffer. */
int deodr_b200_phong_shade_albedo(const DeodrPhongIO *io, const float *albedo, const double *sh, int sh_channels,
                                  void *stream);
/* Its adjoint from io->image_b: channels_b [H,W,7], albedo_b [H,W,C], params_b, camera_center_b (when given) and, with
 * an environment, sh_b [9, sh_channels] overwritten; params_b, camera_center_b and sh_b summed over the pixels without
 * atomics in a fixed order (bit-reproducible; `scratch` as above).  Same refusals, plus DEODR_B200_EINVAL for a NULL
 * image_b, channels_b, params_b, albedo_b or scratch, or a NULL sh_b with an environment. */
int deodr_b200_phong_shade_albedo_b(const DeodrPhongIO *io, const float *albedo, float *albedo_b, const double *sh,
                                    int sh_channels, double *sh_b, double *scratch, void *stream);

/* ---- point lights ---------------------------------------------------------------------------------------------------
 * L point lights near the object, lights [L, 3 + S] fp64 in device memory: row j is the world position p_j (3), then
 * the intensity I_j (S): S = 1 is a grey light applied to every channel, S = C a coloured one (C from 1 to 4, the rule
 * of sh_channels).  L from 1 to 8.  Any other S or L is DEODR_B200_EUNSUPPORTED before any launch.  For a surface point
 * x with unit normal n (the normal of the terms above, per vertex or n = N / |N| per pixel):
 *
 *   d_j = p_j - x,  r_j = |d_j|,  w_j = d_j / r_j             (term j is 0, with its derivatives, when r_j = 0)
 *   diff_j = max(0, <n, w_j>) / r_j^2
 *   spec_j = a * ks * max(0, <n, h_j>)^e / r_j^2,  h_j = normalize(w_j + v)   (h_j = 0 when w_j + v = 0)
 *   P_c(n, x) = sum_{j = 0..L-1} I_j[c] * diff_j,   Q_c(n, x) = sum_j I_j[c] * spec_j      (lights in index order)
 *
 * an inverse-square falloff with no other constant.  The terms are added after the existing ones:
 *
 *   Gouraud (per vertex)  colors[v,c] = vertex_colors[v,c] * (((max(0, -<n_v, l>) + ambient) + sh_c(n_v)) + P_c(n_v, x_v))
 *   textured              shade[v]    = ((max(0, -<n_v, l>) + ambient) + sh(n_v)) + P(n_v, x_v)        (S = 1 only)
 *   Phong (per pixel)     image[c]    = A[c] * (((ambient + diff) + sh_c(n)) + P_c(n, x)) + (spec + Q_c) + (1 - a) bg[c]
 *
 * with x_v the vertex's world position, no specular term per vertex, and per pixel x = X / a, v, a, ks and e those of
 * DeodrPhongIO; every point-light term is 0 where a = 0.  Without an environment its term is left out.  The
 * max(0, .) gates read `> 0`, so a NaN normal gives a zero point-light term, and a table of zero intensities gives bit
 * for bit the outputs of the calls without point lights.  No visibility here: per pixel, shadows are the
 * shadowed calls below.
 *
 * Adjoint: lights_b [L, 3 + S] is the gradient of every entry, summed in fp64 in a fixed order without atomics
 * (bit-reproducible; `scratch` as above).  The normals receive sum_j of the terms' normal gradients (Phong: through
 * the adjoint of n = N / |N|); x receives them through d_j - per vertex into positions_b, per pixel into the position
 * slice of channels_b and, through x = X / a, into the coverage slice; camera_center_b, when it is given, receives
 * the camera centre's share of Q through v. */

/* Per-vertex colours under point lights: deodr_b200_sh_lit_vertex_colors with positions [n,3] (the vertices), an
 * optional environment (sh NULL and sh_channels 0 for none) and the light table lights [nb_lights, 3 + light_channels].
 * vertex_colors NULL gives the luminosity [n] of a textured mesh (nb_colors 1, sh_channels 0 or 1, light_channels 1).
 * DEODR_B200_EINVAL for a NULL buffer when n > 0 or a NULL sh with sh_channels != 0; DEODR_B200_EUNSUPPORTED for a bad
 * sh_channels, light_channels or nb_lights; both before any launch. */
int deodr_b200_point_lit_vertex_colors(const double *normals, const double *positions, const double *vertex_colors,
                                       int n, int nb_colors, const double *light, int directional, const double *sh,
                                       int sh_channels, const double *lights, int nb_lights, int light_channels,
                                       double *colors, void *stream);
/* Its adjoint from colors_b ([n,C], or [n] without vertex colours; fp32, or fp64 with colors_b_fp64 = 1): normals_b
 * [n,3], positions_b [n,3], vertex_colors_b [n,C] (not written, and may be NULL, without vertex_colors), light_b [4],
 * sh_b [9, sh_channels] (with an environment; may be NULL without) and lights_b [nb_lights, 3 + light_channels], all
 * overwritten.  Same refusals, n >= 1. */
int deodr_b200_point_lit_vertex_colors_b(const double *normals, const double *positions, const double *vertex_colors,
                                         int n, int nb_colors, const double *light, int directional, const double *sh,
                                         int sh_channels, const double *lights, int nb_lights, int light_channels,
                                         const void *colors_b, int colors_b_fp64, double *normals_b,
                                         double *positions_b, double *vertex_colors_b, double *light_b, double *sh_b,
                                         double *lights_b, double *scratch, void *stream);
/* Per-pixel shading under point lights, both Phong forms: with albedo NULL the G-buffer of deodr_b200_phong_shade
 * (offsets tiling [0, C + 7)), else the separate albedo [H,W,C] of deodr_b200_phong_shade_albedo (off_albedo -1, the
 * other offsets tiling [0, 7)).  An optional environment (sh NULL and sh_channels 0 for none) and the light table
 * lights [nb_lights, 3 + light_channels].  DeodrPhongIO is read as by those calls; its layout is unchanged.  Their
 * refusals, plus DEODR_B200_EINVAL for a NULL lights and DEODR_B200_EUNSUPPORTED for a bad light_channels or
 * nb_lights, before any launch.  No host synchronisation. */
int deodr_b200_point_phong_shade(const DeodrPhongIO *io, const float *albedo, const double *sh, int sh_channels,
                                 const double *lights, int nb_lights, int light_channels, void *stream);
/* Its adjoint from io->image_b: the outputs of deodr_b200_phong_shade_b (deodr_b200_phong_shade_albedo_b with an
 * albedo, albedo_b [H,W,C] then overwritten), sh_b with an environment, and lights_b [nb_lights, 3 + light_channels]
 * overwritten.  Same refusals, plus DEODR_B200_EINVAL for a NULL lights_b, or a NULL albedo_b with an albedo. */
int deodr_b200_point_phong_shade_b(const DeodrPhongIO *io, const float *albedo, float *albedo_b, const double *sh,
                                   int sh_channels, double *sh_b, const double *lights, int nb_lights,
                                   int light_channels, double *lights_b, double *scratch, void *stream);

/* ---- shadows from point lights --------------------------------------------------------------------------------------
 * Every light j of a point-light table lights [L, 3 + S] gets a cube shadow map: six depth renders of the mesh, each
 * M x M (M from 8 to 4096), seen from p_j.  Face f = 6 j + k (k = 0..5: +x, -x, +y, -y, +z, -z) is the camera vector
 * [26] of the device-camera entry points with
 *
 *   extrinsic [R_k | -R_k p_j],  intrinsic [[phi, 0, (M-1)/2], [0, phi, (M-1)/2], [0, 0, 1]],  phi = M/2 - 2,
 *   no distortion, and the rows of R_k (the camera's x, y and z axes in world coordinates; each a proper rotation,
 *   so that every face keeps the mesh's winding):
 *     +x: (0,1,0) (0,0,1) (1,0,0)     -x: (0,0,1) (0,1,0) (-1,0,0)
 *     +y: (0,0,1) (1,0,0) (0,1,0)     -y: (1,0,0) (0,0,1) (0,-1,0)
 *     +z: (1,0,0) (0,1,0) (0,0,1)     -z: (0,1,0) (1,0,0) (0,0,-1)
 *
 * A face is slightly wider than 90 degrees, so that the 2x2 taps of a point on a face boundary stay inside its map.
 * The map D_f [M,M] (row v, column u) is the depth render of the mesh through that camera: the vertex depth as a
 * one-channel colour, antialiased with the caller's sigma in map pixels, with the mesh's winding and backface culling
 * on, over a background depth DEODR_B200_SHADOW_FAR (finite, so that the silhouette blend beta z + (1 - beta) FAR
 * stays finite).  The visibility of a surface point x (per pixel x = X / a, as for the point-light terms):
 *
 *   d = x - p_j;  k = the dominant axis of d with its sign (ties go to x, then y, then z);  f = 6 j + k
 *   (u, v, z) = the projection of x through face f (the arithmetic of deodr_b200_project_points_dev)
 *   taps: the 2x2 neighbourhood (u0, v0) = floor(u, v), (fu, fv) = (u - u0, v - v0), indices clamped into [0, M)
 *   s_k = s((D_f[tap k] + bias - z) / softness + 1),  s(y) = 3 y^2 - 2 y^3 on y clamped to [0, 1]
 *   V_j = lerp(lerp(s_00, s_10, fu), lerp(s_01, s_11, fu), fv),  lerp(a, b, t) = a + t (b - a)
 *
 * s is exactly 1 when D + bias >= z and exactly 0 when D + bias <= z - softness, and the lerps give V = 1 exactly when
 * every tap is 1.  bias > 0 and softness > 0 are world units.  V_j = 1 where a = 0, and where the projection is not in
 * front of the face or not finite (x at the light, or a NaN position).  Shading: per pixel, light j's diff_j and
 * spec_j (the point-light terms above) are multiplied by V_j, each product rounded on its own, so that where every V_j
 * is 1 the image is bit for bit the image of deodr_b200_point_phong_shade.  Every other term is unchanged.
 *
 * Adjoint: from vis_b [H,W,L], the gradient goes to x (through z and the bilinear weights; into the G-buffer's
 * position slice and, through x = X / a, its coverage slice), to the map texels (fp32 atomics) and to p_j through
 * t_f = -R_f p_j (the face choice is piecewise constant).  The maps' gradient then goes through the rasteriser's
 * adjoint of the 6L face renders, whose depths_b (= colors_b) and ij_b the cube projection's adjoint takes to the
 * vertices and to p_j.
 *
 * Limitations: a triangle with a vertex behind a face's camera plane is missing from that face's map (the rasteriser
 * drops it with culling on), which happens only for a triangle that subtends more than 45 degrees at the light; open
 * surfaces cast shadows from their front side only; at the view's self-occlusion silhouettes x is the G-buffer's
 * mixed position (the Phong approximation); D and the G-buffer's X are both interpolated linearly in screen space, so
 * a lit surface's own z and D differ by an amount that grows with triangle size, which bias must cover. */
#define DEODR_B200_SHADOW_FAR 1e30

/* The cube cameras and the projection of vertices [n,3] through them: cameras [6L, 26] (face f = 6 j + k), ij
 * [6L, n, 2] and depths [6L, n] fp64, all written; face f's are bit-identical to deodr_b200_project_points_dev with
 * camera vector cameras[f] and no distortion.  The lights stay in device memory (nothing is read back).
 * DEODR_B200_EINVAL for n < 1, a NULL buffer or map_size outside [8, 4096]; DEODR_B200_EUNSUPPORTED for nb_lights
 * outside [1, 8] or light_channels outside [1, 4]; both before any launch.  No host synchronisation. */
int deodr_b200_cube_project(const double *vertices, int n, const double *lights, int nb_lights, int light_channels,
                            int map_size, double *cameras, double *ij, double *depths, void *stream);
/* Its adjoint from ij_b [6L, n, 2] and depths_b [6L, n] (fp32, the rasteriser's): vertices_b [n,3] accumulated, one
 * thread per vertex adding its 6L faces in order (no atomics), and the position entries lights_b[j, 0:3] accumulated
 * with the faces' share -sum_k R_k^T t_b, summed in a fixed order (`scratch` of deodr_b200_fitter_scratch_bytes).
 * Same refusals, plus a NULL cameras (those of the forward), vertices_b, lights_b or scratch. */
int deodr_b200_cube_project_b(const double *vertices, int n, const double *lights, int nb_lights, int light_channels,
                              int map_size, const double *cameras, const float *ij_b, const float *depths_b,
                              double *vertices_b, double *lights_b, double *scratch, void *stream);
/* The visibility vis [H,W,L] fp32 of the G-buffer's pixels (io's channels, H, W, C, off_position and off_coverage,
 * with a stride of C + 7, or 7 with off_albedo -1; nothing else of io is read) under the lights' cube maps maps
 * [6L, M, M] fp32.  DEODR_B200_EINVAL for a NULL buffer, bad io sizes or offsets, map_size outside [8, 4096], or a
 * non-finite or non-positive bias or softness; DEODR_B200_EUNSUPPORTED for nb_lights or light_channels outside the
 * point-light rules; both before any launch.  No host synchronisation. */
int deodr_b200_shadow_visibility(const DeodrPhongIO *io, const double *lights, int nb_lights, int light_channels,
                                 const float *maps, int map_size, double bias, double softness, float *vis,
                                 void *stream);
/* Its adjoint from vis_b [H,W,L] fp32: io->channels_b's position and coverage slices accumulated, maps_b [6L,M,M]
 * accumulated with fp32 atomics, and lights_b[j, 0:3] accumulated, summed in a fixed order.  Same refusals, plus a
 * NULL channels_b, vis_b, maps_b, lights_b or scratch. */
int deodr_b200_shadow_visibility_b(const DeodrPhongIO *io, const double *lights, int nb_lights, int light_channels,
                                   const float *maps, int map_size, double bias, double softness, const float *vis_b,
                                   float *maps_b, double *lights_b, double *scratch, void *stream);
/* deodr_b200_point_phong_shade with light j's terms multiplied by vis [H,W,L] fp32 (its refusals, plus a NULL vis). */
int deodr_b200_point_phong_shade_shadowed(const DeodrPhongIO *io, const float *albedo, const double *sh,
                                          int sh_channels, const double *lights, int nb_lights, int light_channels,
                                          const float *vis, void *stream);
/* deodr_b200_point_phong_shade_b of the shadowed shading, which also writes vis_b [H,W,L] fp32 =
 * sum_c image_b[c] (A[c] I_j[c] diff_j + I_j[c] spec_j) (0 where a = 0).  Its refusals, plus a NULL vis or vis_b. */
int deodr_b200_point_phong_shade_shadowed_b(const DeodrPhongIO *io, const float *albedo, float *albedo_b,
                                            const double *sh, int sh_channels, double *sh_b, const double *lights,
                                            int nb_lights, int light_channels, double *lights_b, const float *vis,
                                            float *vis_b, double *scratch, void *stream);

/* ---- shadows from the directional light --------------------------------------------------------------------------
 * The directional light l = params[0..2] of DeodrPhongIO (in device memory) gets one orthographic shadow map of M x M
 * texels (M from 8 to 4096) over a window the caller fixes: a centre c (3) and a radius r > 0 in world units, host
 * values (the light has no position, so no default is free of scale).  With d = l / |l| the direction the light
 * travels (d = +z where |l| = 0, so that the map stays finite), the frame is Frisvad's orthonormal basis around d:
 *
 *   d_z < -0.9999999:  e1 = (0, -1, 0),  e2 = (-1, 0, 0)
 *   otherwise:         a = 1 / (1 + d_z),  b = -d_x d_y a,  e1 = (1 - d_x^2 a, b, -d_x),  e2 = (b, 1 - d_y^2 a, -d_y)
 *
 * (e1, e2, d) is a proper rotation, so the map keeps the mesh's winding.  The frame is smooth except at the pole
 * d = -z, where the map's rotation about d (never d itself) jumps: a camera looking along +z with the light beside it
 * puts the pole behind the scene.  Inside the pole's band the fixed e1 and e2 are orthogonal to d only to within
 * |d_xy| < 4.5e-4 (Frisvad's construction).  A point x projects to
 *
 *   u = (M-1)/2 + phi <e1, x - c> / r,   v = (M-1)/2 + phi <e2, x - c> / r,   z = <d, x - c> + 2 r,   phi = M/2 - 2
 *
 * so that a point of the sphere |x - c| <= r has its 2x2 taps inside the map and z in [r, 3r].  The map D [M,M] is
 * the depth render of (u, v, z) (the recipe of the cube faces above: the vertex depth as a one-channel colour, the
 * caller's sigma in map pixels, the mesh's winding, culling on, a background of DEODR_B200_SHADOW_FAR).  The
 * visibility of x (per pixel x = X / a) is the cube maps' soft test on (u, v, z) - the 2x2 lerp of
 * s((D + bias - z) / softness + 1) - and V = 1 exactly, with zero gradient, where a = 0, where x is not finite, where
 * |x - c| > r (receivers outside the window are lit: a limitation) or where |l| = 0.  Shading: per pixel the
 * directional diff and spec are each multiplied by V, each product rounded on its own, so that where V = 1 the image
 * is bit for bit the image without the sun's shadow; every other term (ambient, environment, point lights and their
 * own V_j) is unchanged.
 *
 * Adjoint: from sun_vis_b [H,W] = sum_c image_b[c] (A[c] diff + spec), the gradient goes to x (the G-buffer's
 * position slice and, through x = X / a, its coverage slice), to the map's texels (fp32 atomics) and to l through
 * (e1, e2, d); the map's gradient then goes through the rasteriser's adjoint of the one depth render, whose ij_b and
 * depths_b the projection's adjoint takes to the vertices and to l.  l receives (I - d d^T) / |l| applied to the
 * gradient of d: the intensity |l| gets nothing from the shadow.  Every fp64 sum is taken in a fixed order, without
 * fp64 atomics.  The limitations of the cube maps on triangle size and open surfaces apply too. */

/* The projection of vertices [n,3] into the sun map: ij [n,2] and depths [n] fp64, written; light [3] fp64 device
 * (read on the device, nothing read back), center [3] host.  DEODR_B200_EINVAL before any launch for n < 1, a NULL
 * buffer, map_size outside [8, 4096], a non-finite center or a non-finite or non-positive radius.  No host
 * synchronisation. */
int deodr_b200_sun_project(const double *vertices, int n, const double *light, const double *center, double radius,
                           int map_size, double *ij, double *depths, void *stream);
/* Its adjoint from ij_b [n,2] and depths_b [n] (fp32, the rasteriser's): vertices_b [n,3] accumulated, one thread per
 * vertex (no atomics), and light_b [3] accumulated, summed in a fixed order (`scratch` of
 * deodr_b200_fitter_scratch_bytes).  Same refusals, plus a NULL vertices_b, light_b or scratch. */
int deodr_b200_sun_project_b(const double *vertices, int n, const double *light, const double *center, double radius,
                             int map_size, const float *ij_b, const float *depths_b, double *vertices_b,
                             double *light_b, double *scratch, void *stream);
/* The visibility sun_vis [H,W] fp32 of the G-buffer's pixels (io's channels, params, H, W, C, off_position and
 * off_coverage as for deodr_b200_shadow_visibility) under the sun map map [M,M] fp32.  DEODR_B200_EINVAL before any
 * launch for a NULL buffer, bad io sizes or offsets, map_size outside [8, 4096], a non-finite or non-positive bias,
 * softness or radius, or a non-finite center.  No host synchronisation. */
int deodr_b200_sun_visibility(const DeodrPhongIO *io, const double *center, double radius, const float *map,
                              int map_size, double bias, double softness, float *vis, void *stream);
/* Its adjoint from vis_b [H,W] fp32: io->channels_b's position and coverage slices accumulated, map_b [M,M]
 * accumulated with fp32 atomics, and light_b [3] (l's gradient; params_b of the shading's adjoint may be passed)
 * accumulated, summed in a fixed order.  Same refusals, plus a NULL channels_b, vis_b, map_b, light_b or scratch. */
int deodr_b200_sun_visibility_b(const DeodrPhongIO *io, const double *center, double radius, const float *map,
                                int map_size, double bias, double softness, const float *vis_b, float *map_b,
                                double *light_b, double *scratch, void *stream);
/* The Phong shading (either form: albedo NULL reads it from the G-buffer) with the directional terms multiplied by
 * sun_vis [H,W] fp32, with an optional environment (sh NULL with sh_channels 0), and optional point lights (lights
 * NULL with nb_lights 0) with their optional visibility vis [H,W,L].  The refusals of the calls it extends, plus a
 * NULL sun_vis; DEODR_B200_EUNSUPPORTED for bad channel or light counts. */
int deodr_b200_phong_shade_sun_shadowed(const DeodrPhongIO *io, const float *albedo, const double *sh,
                                        int sh_channels, const double *lights, int nb_lights, int light_channels,
                                        const float *vis, const float *sun_vis, void *stream);
/* Its adjoint, which also writes sun_vis_b [H,W] fp32 = sum_c image_b[c] (A[c] diff + spec), and, with point lights,
 * lights_b (and, with vis, vis_b as deodr_b200_point_phong_shade_shadowed_b).  Its refusals, plus a NULL sun_vis or
 * sun_vis_b. */
int deodr_b200_phong_shade_sun_shadowed_b(const DeodrPhongIO *io, const float *albedo, float *albedo_b,
                                          const double *sh, int sh_channels, double *sh_b, const double *lights,
                                          int nb_lights, int light_channels, double *lights_b, const float *vis,
                                          float *vis_b, const float *sun_vis, float *sun_vis_b, double *scratch,
                                          void *stream);

/* ---- tangent-space normal maps (textured Phong) -------------------------------------------------------------------
 * A normal map [Ht, Wt, 3] fp32 has the albedo texture's Ht and Wt and is addressed by the same uv / faces_uv (texel
 * units, shifted by -0.5).  Its texels are raw tangent-space vectors (not [0, 1]-encoded: the caller decodes 8-bit
 * maps): x along +u (texture columns), y along +v (texture rows, downwards), z along the outward normal.  A map in the
 * OpenGL convention has its y negated by the caller.
 *
 * Per-vertex tangent frame.  Face f with position ids (i0, i1, i2) and uv ids (k0, k1, k2):
 *   e1 = x_i1 - x_i0,  e2 = x_i2 - x_i0,  (du1, dv1) = uv_k1 - uv_k0,  (du2, dv2) = uv_k2 - uv_k0
 *   det = du1 dv2 - du2 dv1,  sigma = sign(det) (0 when det = 0)
 *   t_f = sigma (dv2 e1 - dv1 e2),  b_f = sigma (du1 e2 - du2 e1)      (|det| dx/du and |det| dx/dv: uv-area weights)
 *   T_v = normalize(sum_{f ∋ v} t_f),  B_v = normalize(sum_{f ∋ v} b_f)  (0 for a zero sum)
 * The sums run over the topology's vertex-face CSR, in its order, as deodr_b200_vertex_normals's.
 *
 * G-buffer.  A normal-mapped view rasterises 13 channels per vertex, (N, X, 1, T, B), and a third raster, the normal
 * map sampled like the albedo (shade 1, zero background, 3 channels), M; all three share the view's geometry.  Per
 * pixel, with coverage a:
 *   a = 0:  N' = 0 (nothing else is read; every gradient is 0)
 *   n  = N / |N|                          (0 when |N| = 0)
 *   t~ = T - <T, n> n,  t = t~ / |t~|     (0 when |t~| = 0)
 *   b~ = n x t,  s = +1 if <b~, B> >= 0 else -1,  b = s b~
 *   p  = (M_x t + M_y b) + M_z n          (summed in that order)
 *   N' = a p / |p|                        (0 when |p| = 0)
 * M carries the coverage as a factor, which normalising p cancels.  The result is the 7-channel G-buffer (N', X, a)
 * of DeodrPhongIO's albedo form, which every shading and visibility entry point reads unchanged.
 *
 * Adjoint: N'_b goes to N_b, T_b, M_b and a_b (B_b = 0: s is piecewise constant, as sigma is); the X and a slices
 * pass through.  The rasteriser's adjoint of the three rasters then gives the G-buffer's colors_b, whose T and B slices
 * go to deodr_b200_vertex_tangents_b, and the map's texture_b.  Every sum is a gather in a fixed order (no atomics),
 * so the tangents' adjoint is bit-reproducible.
 *
 * Limitations: a vertex shared by mirrored uv charts gets cancelling tangents (the caller splits such vertices); the
 * frame is not MikkTSpace, so maps baked by other tools may shade slightly differently; sampling is the rasteriser's
 * bilinear sampling, without mip levels; at self-occlusion silhouettes the frame is the mixed frame of the Phong
 * G-buffer.
 *
 * Caller contract: faces_uv indexes [0, nb_uv) and the topology's faces [0, V); neither can be checked on the device
 * without a host synchronisation, so neither is.  None of these calls synchronises with the host. */

/* face_frames [T,6] = (t_f, b_f) and frames [V,6] = (T_v, B_v), fp64, overwritten, from vertices [V,3] fp64, faces_uv
 * [T,3] and uv [nb_uv,2] fp64.  DEODR_B200_EINVAL before any launch for a NULL buffer (the topology's faces and its
 * vertex-face CSR included) or T, V or nb_uv < 1. */
int deodr_b200_vertex_tangents(const DeodrMeshTopology *mesh, const double *vertices, const uint32_t *faces_uv,
                               const double *uv, int nb_uv, double *face_frames, double *frames, void *stream);
/* Its adjoint from frames_b [V,6] fp64: vertices_b [V,3] fp64 accumulated, one thread per position vertex; uv_b
 * [nb_uv,2] fp64 overwritten, one thread per uv vertex walking the uv-vertex-face CSR (uv_face_offset [nb_uv+1],
 * uv_face_index [3T]: the faces of every uv vertex, ascending, with multiplicity, as the topology's vertex-face CSR).
 * scratch: 6 V + 10 T doubles.  Same refusals, plus a NULL CSR, scratch or output. */
int deodr_b200_vertex_tangents_b(const DeodrMeshTopology *mesh, const double *vertices, const uint32_t *faces_uv,
                                 const double *uv, int nb_uv, const int32_t *uv_face_offset,
                                 const int32_t *uv_face_index, const double *frames_b, double *scratch,
                                 double *vertices_b, double *uv_b, void *stream);
/* out [H,W,7] = (N', X, a) from gbuffer [H,W,13] = (N, X, a, T, B) and the map raster map [H,W,3], fp32, one thread
 * per pixel, fp64 maths.  DEODR_B200_EINVAL before any launch for a NULL buffer or H or W < 1. */
int deodr_b200_normal_map(const float *gbuffer, const float *map, int H, int W, float *out, void *stream);
/* Its adjoint from out_b [H,W,7]: gbuffer_b [H,W,13] and map_b [H,W,3] fp32, overwritten.  Same refusals. */
int deodr_b200_normal_map_b(const float *gbuffer, const float *map, int H, int W, const float *out_b,
                            float *gbuffer_b, float *map_b, void *stream);

/* ---- specular maps (textured Phong) -------------------------------------------------------------------------------
 * A specular map S [Ht, Wt, 2] fp32 has the albedo texture's Ht and Wt and is addressed by the same uv / faces_uv.  It
 * follows the glTF convention, factor x texture: texel (ks_t, e_t) multiplies the view's ks = params[4] and e =
 * params[5], so a map of ones is the view without a map, and ks and e keep their meaning and their gradient.  The map
 * is rasterised like the albedo (shade 1, zero background, 2 channels, the view's geometry and sigma), which gives per
 * pixel (K, E) = a x (sample of S), a the G-buffer's coverage.  Per pixel, in the Phong form with a separate albedo:
 *
 *   aks(p) = ks * K          in place of a * ks, in spec and in every point light's spec_j
 *   e(p)   = e * (E / a)     in place of e (read only where a != 0: every specular term is 0 at a = 0)
 *
 * Nothing else changes: the diffuse, ambient and environment terms, the point lights' diffuse terms and the
 * visibilities V_j and V multiply as before.  E / a is rounded first, so that a map of ones (E = a) gives e exactly.
 * Over the background K / a and E / a are the front surface's values; at self-occlusion silhouettes front and back are
 * mixed, as for the normals.
 *
 * Adjoint, with q the gradient of aks(p) and e_b(p) that of e(p), each summed over the main term and the point lights:
 *
 *   K_b = q * ks,   ks_b += q * K
 *   E_b = e_b(p) * e / a,   e_b += e_b(p) * E / a,   a_b -= e_b(p) * e(p) / a
 *
 * The a * ks share of a_b of the view without a map is gone: ks reaches the image through K only.  spec_b = (K_b, E_b)
 * is 0 where a = 0.  params_b stays a fixed-order sum (bit-reproducible, no fp64 atomics); the map raster's gradient
 * then goes through the rasteriser's adjoint to the map's texels, the uv and ij.
 *
 * Limitations: grey specular only (one ks per texel); bilinear sampling without mip levels; e(p) <= 0 gives what pow
 * gives, so a fit that can drive e_t or e negative parametrises it itself. */

/* The Phong shading of deodr_b200_phong_shade_sun_shadowed with a separate albedo [H,W,C] and the specular map's
 * raster spec [H,W,2] = (K, E), both required, an optional environment (sh NULL with sh_channels 0), optional point
 * lights (lights NULL with nb_lights 0) with their optional visibility vis [H,W,L], and an optional sun visibility
 * sun_vis [H,W] (NULL: the directional light is unshadowed).  DeodrPhongIO is read as by
 * deodr_b200_phong_shade_albedo; its layout is unchanged.  The refusals of the calls it extends, before any launch:
 * DEODR_B200_EINVAL for a NULL io, buffer, albedo or spec, bad sizes or offsets (off_albedo must be -1), a NULL sh with
 * sh_channels != 0, or a NULL lights with nb_lights != 0 or a vis; DEODR_B200_EUNSUPPORTED for bad channel or light
 * counts.  No host synchronisation. */
int deodr_b200_phong_shade_specular_map(const DeodrPhongIO *io, const float *albedo, const float *spec,
                                        const double *sh, int sh_channels, const double *lights, int nb_lights,
                                        int light_channels, const float *vis, const float *sun_vis, void *stream);
/* Its adjoint from io->image_b: channels_b [H,W,7], albedo_b [H,W,C], spec_b [H,W,2], params_b and camera_center_b
 * (when given) overwritten, and with the optional inputs sh_b, lights_b, vis_b and sun_vis_b as the calls it extends
 * write them (each may be NULL without its input).  Same refusals, plus DEODR_B200_EINVAL for a NULL image_b,
 * channels_b, params_b, albedo_b, spec_b or scratch, or a NULL gradient of a given optional input. */
int deodr_b200_phong_shade_specular_map_b(const DeodrPhongIO *io, const float *albedo, const float *spec,
                                          const double *sh, int sh_channels, const double *lights, int nb_lights,
                                          int light_channels, const float *vis, const float *sun_vis,
                                          float *albedo_b, float *spec_b, double *sh_b, double *lights_b,
                                          float *vis_b, float *sun_vis_b, double *scratch, void *stream);

/* ---- metallic-roughness materials (textured, GGX) ------------------------------------------------------------------
 * A per-pixel form for textured views with a separate albedo A [H,W,C] beside the 7-channel G-buffer (N, X, a).  It
 * reads DeodrPhongIO with its layout unchanged, but params[4] is the metallic factor mf and params[5] the roughness
 * factor rf (params_b[4..5] their gradients).  An optional metallic-roughness map MR [Ht, Wt, 2] has the albedo
 * texture's Ht and Wt, is addressed by the same uv / faces_uv and holds (roughness_t, metallic_t) per texel (glTF keeps
 * them in the G and B channels: slicing them out is the caller's).  The map is rasterised like the albedo, which gives
 * (R, M) = a x (sample of MR) per pixel.  Per pixel where a != 0:
 *
 *   n = N / |N|,  x = X / a,  v = normalize(cam - x),  b_c = A_c / a
 *   r = rf (R / a),  m = mf (M / a)   (rf and mf without a map; R / a and M / a rounded first)
 *   alpha = r^2,  F0_c = 0.04 (1 - m) + m b_c
 *   for each light of unit direction w toward it and intensity E_c:
 *     directional: w = -l / |l|, E = |l| (grey), times the sun's visibility V when given
 *     point j:     w = w_j, E_c = I_j[c] / r_j^2, times V_j when given
 *     nl = <n, w> (the light's term is 0 unless nl > 0), nv = max(0, <n, v>), h = normalize(w + v) (0 when w + v =
 *     0), nh = max(0, <n, h>), vh = max(0, <v, h>)
 *     F_c = F0_c + (1 - F0_c) (1 - vh)^5
 *     S = alpha^2 / (nh^2 (alpha^2 - 1) + 1)^2 / ((nl + sqrt(alpha^2 + (1 - alpha^2) nl^2))
 *                                                 (nv + sqrt(alpha^2 + (1 - alpha^2) nv^2)))
 *       (= pi D Vis: GGX D and the separable Smith Vis of glTF 2.0 Appendix B, with pi cancelled)
 *     term_c = E_c nl [(1 - F_c)(1 - m) A_c + a S F_c]
 *   image_c = sum over the lights of term_c + (1 - m) A_c (ambient + sh_c(n)) + (1 - a) bg_c
 *
 * Conventions.  The clamps are max(0, .) gates that read `> 0`, as the Phong forms'; glTF's |.| differs only where
 * <n, v> < 0, at the silhouettes of interpolated normals.  Where a = 0 every surface term is 0, with its derivatives,
 * and the map raster's gradient is 0.  At alpha = 0 the highlight is 0; keeping r > 0 and m in [0, 1] is the caller's
 * job.  The environment (ambient and SH) lights the diffuse lobe only: there is no specular from the environment.  At
 * self-occlusion silhouettes front and back surfaces are mixed, as for the Phong form.  A map of ones (R = M = a)
 * gives the factors-only form bit for bit.
 *
 * The adjoint gives A_b (through b_c, F0 too), the G-buffer's (N, X, a) gradients, mr_b = (R_b, M_b), params_b (l,
 * ambient, mf, rf), lights_b, sh_b, vis_b, sun_vis_b and camera_center_b.  params_b stays a fixed-order sum
 * (bit-reproducible, no fp64 atomics).
 *
 * Limitations: no specular from the environment; bilinear sampling without mip levels; no emissive, occlusion,
 * clearcoat or anisotropy; textured views only (no per-vertex GGX). */

/* The metallic-roughness shading above with a separate albedo [H,W,C] (required), the map raster mr [H,W,2] = (R, M)
 * or NULL (the factors alone), an optional environment (sh NULL with sh_channels 0), optional point lights (lights
 * NULL with nb_lights 0) with their optional visibility vis [H,W,L], and an optional sun visibility sun_vis [H,W].
 * Refusals, before any launch: DEODR_B200_EINVAL for a NULL io, buffer or albedo, bad sizes or offsets (off_albedo
 * must be -1), a NULL sh with sh_channels != 0, or a NULL lights with nb_lights != 0 or a vis;
 * DEODR_B200_EUNSUPPORTED for bad channel or light counts.  No host synchronisation. */
int deodr_b200_pbr_shade(const DeodrPhongIO *io, const float *albedo, const float *mr, const double *sh,
                         int sh_channels, const double *lights, int nb_lights, int light_channels, const float *vis,
                         const float *sun_vis, void *stream);
/* Its adjoint from io->image_b: channels_b [H,W,7], albedo_b [H,W,C], mr_b [H,W,2] (with mr), params_b and
 * camera_center_b (when given) overwritten, and with the optional inputs sh_b, lights_b, vis_b and sun_vis_b.  Same
 * refusals, plus DEODR_B200_EINVAL for a NULL image_b, channels_b, params_b, albedo_b or scratch, an mr_b that is
 * non-NULL exactly when mr is not, or a NULL gradient of a given optional input. */
int deodr_b200_pbr_shade_b(const DeodrPhongIO *io, const float *albedo, const float *mr, const double *sh,
                           int sh_channels, const double *lights, int nb_lights, int light_channels, const float *vis,
                           const float *sun_vis, float *albedo_b, float *mr_b, double *sh_b, double *lights_b,
                           float *vis_b, float *sun_vis_b, double *scratch, void *stream);

/* One parameter vector of a heavy-ball update (device pointers, `size` entries each):
 *   step = clamp(-grad * factor, -max_step, max_step)   (max_step = INFINITY: unclamped)
 *   speed = (1 - damping) (speed * inertia + (1 - inertia) step);  value += speed
 * and, when `normalize`, value /= |value| afterwards (the quaternion). */
typedef struct DeodrHeavyBall {
    double *value;
    double *speed;
    const double *grad;
    double factor;
    double max_step;
    int32_t size;
    int32_t normalize;
} DeodrHeavyBall;

/* The update of a fitting step in one kernel: the vertices (value [n,3] with grad = vertices_b, plus grad_rigid [n,3]
 * when not NULL) and up to 8 small parameters; *energy = *energy_data + *energy_rigid when energy is not NULL. */
int deodr_b200_fitter_update(const DeodrHeavyBall *vertices, const double *grad_rigid, const DeodrHeavyBall *params,
                             int nb_params, double inertia, double damping, const double *energy_data,
                             const double *energy_rigid, double *energy, void *stream);

/* ---- deferred channels: the G-buffer of Scene3D.render_deferred (deodr/differentiable_renderer.py:1053-1174) -----
 * Per pixel of a forward pass's face-id map, the attributes of the owner face interpolated in fp64 with the weights of
 * the colour pass (no perspective correction, as the reference's sigma-0 soup), written as fp32 into `out` [H,W,K] at
 * each attribute's channel offset.  An offset of -1 skips the attribute (its pointer may then be NULL).  Channels:
 *   depth (1)       depth[V] * depth_scale; *depth_background (unscaled) at the background
 *   face_id (1)     the owner face as a float
 *   barycentric (3) the interpolation weights
 *   normal (3), luminosity (1), xyz (3), color (nb_color): per-vertex attributes, indexed through scene.faces
 *   uv (2)          per-uv attribute [Nuv,2], indexed through scene.faces_uv
 * Every channel but depth is `background` at the background (0 in the reference). */
typedef struct DeodrDeferredIO {
    const int32_t *face_index;        /* [H,W] forward owner of deodr_b200_render's face_id, -1 = background */
    const double *depth;              /* [V] or NULL */
    const double *xyz;                /* [V,3] or NULL */
    const double *normal;             /* [V,3] or NULL */
    const float *luminosity;          /* [V] or NULL */
    const double *uv;                 /* [Nuv,2] or NULL */
    const double *color;              /* [V,nb_color] or NULL */
    const double *depth_background;   /* device scalar, required with depth */
    float *out;                       /* [H,W,K] */
    double depth_scale;
    float background;
    int32_t K, nb_color;
    int32_t off_depth, off_face_id, off_barycentric, off_normal, off_luminosity, off_xyz, off_uv, off_color;
} DeodrDeferredIO;

/* k_deferred over the scene's H x W pixels on `stream`: reads scene.faces, faces_uv (uv only), ij, the sizes and
 * integer_pixel_centers.  DEODR_B200_EINVAL for a NULL scene, io, face_index or out, K < 1, an offset outside
 * [-1, K - channels], a requested attribute whose data is NULL, or a perspective_correct scene.  No host synchronisation. */
int deodr_b200_render_deferred_channels(const DeodrSceneView *scene, const DeodrDeferredIO *io, void *stream);

/* ---- Loop subdivision: one level of ColoredTriMesh.subdivise / loop_subdivision (deodr/triangulated_mesh.py:499-562)
 * and its adjoint, in fp64 on device buffers (csrc/subdivision.cu).  A level maps a coarse mesh with V vertices,
 * E unique edges and T faces to a fine one with V + E vertices and 4T faces; the fine faces depend on the topology
 * only and are built on the host (deodr_b200.mesh_ops.LoopSubdivision).  Fine rows:
 *   0..V-1 (vertex points)  5/8 v_i + (3/8) / deg_i * sum_{j in N(i)} v_j, N(i) the vertices that share a face with i
 *                           (itself excluded), deg_i = |N(i)|;  colour unchanged.
 *   V + e  (edge points)    1/8 (v_a + v_b) + 1/8 sum_{f in F(e)} (v_f0 + v_f1 + v_f2) for edge e = (a, b), F(e) its
 *                           faces with multiplicity (a face whose corners repeat lists the edge more than once);
 *                           colour (c_a + c_b) / 2.
 * The reference's quirks are kept: an edge with one face (a boundary edge) gets weights 2/8, 2/8, 1/8, which sum to
 * 5/8, so boundary edge points shrink towards the origin (this is not Loop's boundary rule); a vertex in no face
 * (deg = 0) stays where it is.  Edges are numbered as np.unique orders the key max(a,b) + min(a,b) V. */
typedef struct DeodrLoopLevel {
    DeodrMeshTopology topology;       /* the coarse level: faces, faces_edges, both face CSRs, V, E, T (clockwise unused) */
    const int32_t *neighbour_offset;  /* [V+1] CSR: N(i), ascending ... */
    const int32_t *neighbour_index;   /* ... (length 2 x the edges joining two distinct vertices) */
    const int32_t *neighbour_edge;    /* parallel to neighbour_index: the edge joining i and that neighbour */
    const int32_t *self_edge;         /* [V] the edge (i, i) of a degenerate face, -1 if none */
    const int32_t *edge_vertices;     /* [E,2] the endpoints of every edge */
} DeodrLoopLevel;

/* One level forward, one launch of one thread per fine row: fine_vertices [V+E,3] from vertices [V,3] and, when
 * colors [V,nb_colors] is not NULL, fine_colors [V+E,nb_colors].  Outputs are overwritten.  No host synchronisation. */
int deodr_b200_loop_subdivide(const DeodrLoopLevel *level, const double *vertices, const double *colors,
                              int nb_colors, double *fine_vertices, double *fine_colors, void *stream);
/* The adjoint of one level, one launch of one thread per coarse vertex, gathered in a fixed order without atomics
 * (bit-reproducible): vertices_b [V,3] from fine_vertices_b [V+E,3] and colors_b [V,nb_colors] from fine_colors_b
 * [V+E,nb_colors], each skipped when its fine gradient is NULL.  For coarse vertex i:
 *   vertices_b[i] = 5/8 g_i (g_i when deg_i = 0) + sum_{j in N(i)} (3/(8 deg_j) g_j + 1/8 g_{V+e(i,j)})
 *                   + 1/4 g_{V+self_edge[i]} + sum_{f incident to i, with multiplicity} sum_k 1/8 g_{V+faces_edges[f,k]}
 *   colors_b[i]   = gc_i + 1/2 sum_{edges e that end at i} gc_{V+e}   (the edge (i, i) counts twice)
 * Outputs are overwritten, so levels chain from the finest back to the coarsest.  No host synchronisation. */
int deodr_b200_loop_subdivide_b(const DeodrLoopLevel *level, const double *fine_vertices_b,
                                const double *fine_colors_b, int nb_colors, double *vertices_b, double *colors_b,
                                void *stream);

/* ---- Self-collision: a penalty that keeps a mesh from passing through itself, and a self-intersection query, in fp64
 * on device buffers (csrc/collision.cu).  For a mesh with faces [F,3], vertices [V,3], thickness delta > 0, weight w >= 0:
 *   E = w sum_{(v,t) in P_vt} phi(d(v,t)) + w sum_{{e,e'} in P_ee} phi(d(e,e')),  phi(d) = (delta - d)^2 if d < delta else 0
 * d(v,t) is the distance from a vertex to a closed triangle (Ericson, Real-Time Collision Detection 5.1.5,
 * ClosestPtPointTriangle), d(e,e') the distance between two closed segments, the mesh's unique undirected edges
 * (ClosestPtSegmentSegment, 5.1.9, with EPSILON = 0: its clamping order and its parallel case, s = 0 when
 * a e - b^2 = 0; the pair is evaluated with the lower edge id as the first segment).
 * Excluded pairs (the one-ring): (v,t) when v is a corner of t or an edge neighbour of a corner; {e,e'} when an
 * endpoint of one equals an endpoint of the other or is an edge neighbour of one.  A vertex in no face takes no part;
 * a face whose cross(b - a, c - a) is exactly zero takes part in no (v,t) pair, its edges still do.
 * Gradients from the closest points (envelope theorem), with c = 2 w (delta - d):
 *   (v,t): q = sum_i w_i a_i, n = (p - q) / d:   dE/dp = -c n,  dE/da_i = +c w_i n
 *   {e,e'}: c1 = p1 + s (q1 - p1), c2 = p2 + t (q2 - p2), n = (c1 - c2) / d:  p1, q1 get -c (1 - s) n, -c s n;
 *           p2, q2 get +c (1 - t) n, +c t n
 * A pair at d = 0 adds w delta^2 to E and nothing to the gradient.  *min_distance is the smallest d over the pairs
 * closer than delta, or delta when there is none.  A non-finite vertex coordinate (of a vertex in a face) makes
 * *energy and *min_distance NaN; the primitives that touch it are left out of the grid.
 * The distances use no fused multiply-add: each product and sum is rounded as the fp64 restatement
 * (tests/self_collision_ref.py) rounds it, so every d equals the restatement's bit for bit. */
typedef struct DeodrCollisionMesh {
    const uint32_t *faces;            /* [F,3] */
    const int32_t *edges;             /* [E,2] the unique undirected edges (lo, hi), lo <= hi, ordered by (lo, hi) */
    const int32_t *neighbour_offset;  /* [V+1] CSR: the edge neighbours of every vertex, itself excluded ... */
    const int32_t *neighbour_index;   /* ... ascending in every row (they are binary-searched) */
    const int32_t *corner_offset;     /* [V+1] CSR: the corners 3 f + k of every vertex, ascending ... */
    const int32_t *corner_index;      /* ... (length 3F) */
    const int32_t *end_offset;        /* [V+1] CSR: the edge ends 2 e + j of every vertex, ascending ... */
    const int32_t *end_index;         /* ... (length 2E) */
    int32_t nb_faces, nb_edges, nb_vertices;
} DeodrCollisionMesh;

/* E, its gradient and the minimum distance.  grad [V,3] = grad_in + dE/dvertices (grad_in may be NULL, or equal to
 * grad to add in place); *energy and *min_distance are device scalars.  Broad phase: a uniform grid of cells of
 * max(cell_size, thickness) (grown when the grid would exceed 2^21 cells or 1024 per axis), over the bounding box of
 * the finite vertices.  Every (cell, primitive) entry is sorted by a stable radix sort; the vertex-triangle pairs are
 * found from both sides and the edge-edge pairs once per edge at the first cell the two edges share.  The gradient is
 * gathered per vertex in CSR order and the sums are fixed-order grid reductions: no fp64 atomics, two calls on the same
 * input give the same bits.  The workspace keeps the entry capacity of the previous call: the call reads one word,
 * the entry count, from pinned memory after the grid is built and, when it exceeds the capacity, grows it and runs
 * again (the first call builds the plan this way).  Nothing else is read back.  Face indices are not checked here:
 * the host checks them where it builds the topology.  EINVAL for a NULL ws, mesh, array, vertices, grad, energy or
 * min_distance, an empty mesh, thickness <= 0 or non-finite, weight < 0 or non-finite, or a non-finite cell_size;
 * EUNSUPPORTED when the grid would need 2^31 entries or more. */
int deodr_b200_self_collision(DeodrWorkspace *ws, const DeodrCollisionMesh *mesh, const double *vertices,
                              double thickness, double weight, double cell_size, const double *grad_in, double *grad,
                              double *energy, double *min_distance, void *stream);

/* The face pairs (i < j) that share no vertex and where an edge of one properly crosses the other: the edge (p, q)
 * and the triangle (a, b, c) with O(x, y, z, w) = dot(cross(y - x, z - x), w - x) have O(a,b,c,p) and O(a,b,c,q) of
 * strictly opposite signs, and O(p,q,a,b), O(p,q,b,c), O(p,q,c,a) of the same non-zero sign.  Coplanar contacts and
 * touching contacts (a zero orientation) are not reported.  Faces that share a vertex are never paired.  Same
 * products and sums as the restatement, no fused multiply-add, so the signs are the restatement's bit for bit.
 * Writes up to `capacity` pairs to pairs [capacity,2] (int32, in an order fixed by the grid) and their number to
 * *count (host); when *count > capacity, call again with a buffer of *count pairs.  Grid as above with cells of
 * cell_size and the faces' bounding boxes; one read-back of the entry and pair counts.  Same refusals, with
 * cell_size > 0 and finite, and a NULL count (or a NULL pairs with capacity > 0). */
int deodr_b200_self_intersections(DeodrWorkspace *ws, const DeodrCollisionMesh *mesh, const double *vertices,
                                  double cell_size, int32_t *pairs, int64_t capacity, int64_t *count, void *stream);

/* ---- Linear blend skinning: a mesh articulated by a skeleton, and its adjoint, in fp64 on device buffers
 * (csrc/skinning.cu).  A skeleton has J joints; joint j has a parent parents[j] < j, or -1 for a root (several roots
 * are allowed), and a rest centre c_j [3].  Vertex i has K influences: joints skin_index[i,k] in [0, J) with weights
 * skin_weight[i,k].  Weights are not renormalised: identity rotations leave a vertex at rest only when its weights
 * sum to 1 (this is not checked).
 *   R(theta) = I + a [theta]x + b [theta]x^2,  phi = |theta|,  a = sin(phi) / phi,  b = (1 - cos(phi)) / phi^2
 *              (the axis-angle of MANO / SMPL; below phi = 0.1 the series of a, b and their derivatives, so R and
 *              dR/dtheta are exact and finite at theta = 0, where dR/dtheta_k = [e_k]x)
 *   forward kinematics, in index order:  root: Rg_j = R(theta_j), tg_j = c_j;
 *                                        else: Rg_j = Rg_p R(theta_j), tg_j = tg_p + Rg_p (c_j - c_p)
 *   skinning transforms:  M_j = Rg_j,  b_j = tg_j - Rg_j c_j      (identity rotations give (I, 0))
 *   skinned vertices:     v'_i = sum_k w_ik (M_j v_i + b_j),  j = skin_index[i,k]
 * Adjoint, from g = dL/dv' [V,3]:
 *   vertices_b_i  = sum_k w_ik M_j^T g_i
 *   weights_b_ik  = g_i . (M_j v_i + b_j)
 *   rotations_b   [J,3]: (M_b, b_b)_j = sum over the influences on j of (w g v^T, w g), back through the forward
 *                 kinematics.  The joint centres get no gradient.
 * The host builds the index arrays and checks their contents (deodr_b200.mesh_ops.skeleton_arrays); the calls check
 * sizes and pointers only. */
enum {
    DEODR_B200_SKIN_MAX_JOINTS = 1024,   /* the forward kinematics run in one CTA, one thread per joint of a level */
    DEODR_B200_SKIN_MAX_INFLUENCES = 8,  /* as glTF's JOINTS_n / WEIGHTS_n */
    DEODR_B200_SKIN_CHUNK = 256          /* entries of a joint's CSR row summed by one CTA of the adjoint */
};
typedef struct DeodrSkeleton {
    const int32_t *parents;       /* [J] */
    const double *centres;        /* [J,3] rest centres */
    const int32_t *level_offset;  /* [nb_levels+1] CSR: the joints of every depth (the roots are depth 0) ... */
    const int32_t *level_index;   /* ... [J], ascending in every level */
    const int32_t *child_offset;  /* [J+1] CSR: the children of every joint ... */
    const int32_t *child_index;   /* ... ascending (J minus the roots entries; required even when empty) */
    const int32_t *skin_index;    /* [V,K] */
    const double *skin_weight;    /* [V,K] */
    const int32_t *joint_offset;  /* [J+1] CSR: the influences i*K+k on every joint ... */
    const int32_t *joint_entry;   /* ... [V*K], ascending in every row */
    const int32_t *chunk_offset;  /* [J+1] the first chunk of every joint: row j has ceil(n_j / SKIN_CHUNK) chunks */
    int32_t nb_joints, nb_vertices, nb_influences, nb_levels, nb_chunks, pad;
} DeodrSkeleton;

/* skinned [V,3] from vertices [V,3] and rotations [J,3]: one single-CTA launch of the forward kinematics, a barrier per
 * depth level, which writes transforms [J,24] = (Rg [9], tg [3], M [9], b [3]) per joint, then one thread per vertex.
 * EINVAL before any launch for a NULL skeleton, skeleton array or argument, J outside [1, 1024], V < 1, K outside
 * [1, 8] or nb_levels outside [1, J]; EUNSUPPORTED when V * K does not fit in int32.  No host synchronisation. */
int deodr_b200_skin(const DeodrSkeleton *skeleton, const double *vertices, const double *rotations, double *transforms,
                    double *skinned, void *stream);
/* The adjoint of deodr_b200_skin from skinned_b [V,3], re-reading the transforms [J,24] the forward wrote for the same
 * rotations: vertices_b [V,3] = grad_in + sum_k w_ik M_j^T g_i (grad_in may be NULL, or equal to vertices_b to add in
 * place), weights_b [V,K] when not NULL, and rotations_b [J,3] (overwritten).  scratch holds (nb_chunks + J) * 12
 * doubles.  Three launches: one thread per vertex; one CTA per chunk of a joint's CSR row, summed in a fixed order;
 * one CTA that adds every joint's chunks in chunk order and walks the levels back, each parent gathering its children
 * in children-CSR order.  No fp64 atomics: two calls on the same input give the same bits.  Refusals as above, with
 * a NULL skinned_b, vertices_b, rotations_b or scratch.  No host synchronisation. */
int deodr_b200_skin_b(const DeodrSkeleton *skeleton, const double *vertices, const double *rotations,
                      const double *transforms, const double *skinned_b, const double *grad_in, double *vertices_b,
                      double *weights_b, double *rotations_b, double *scratch, void *stream);

/* Per-kernel device timing with CUDA events recorded on the launching stream (for bench.py's roofline).
 * enable: pre-creates `max_records` event pairs (0 disables and frees them).  Every instrumented launch group of the
 * following render / render_b calls then records one (phase, start, stop) triple until the pool is exhausted.
 * collect: synchronises the recorded events, writes up to `capacity` (phase, milliseconds) pairs in launch order,
 * resets the pool and returns the number of records written (negative on error). */
enum {
    DEODR_B200_PH_PLAN = 0,         /* plan building only: count-only binning pass + k_scan_tiles + read-back */
    DEODR_B200_PH_EDGE_BIN = 1,     /* k_bin_edges: stencil records of the silhouette edges + their tile lists */
    DEODR_B200_PH_BIN = 2,          /* memset + (index check) + k_bin: the single binning pass over the triangles */
    DEODR_B200_PH_EDGE_TILE_SORT = 3,/* k_sort_tile_edges: far-to-near order inside every tile */
    DEODR_B200_PH_TILE_Z = 4,       /* k_tile_z: z-buffer + owner ids */
    DEODR_B200_PH_SHADE = 5,        /* k_shade: colour of every pixel */
    DEODR_B200_PH_EDGE_FWD = 6,     /* k_edge_fwd: ordered silhouette-edge overdraw */
    DEODR_B200_PH_SMALL_BWD = 7,    /* k_small_tri_bwd: triangle-parallel interior adjoint */
    DEODR_B200_PH_INTERIOR_BWD = 8, /* k_interior_bwd: pixel-parallel interior adjoint (large triangles) */
    DEODR_B200_PH_EDGE_BWD = 9,     /* accumulator memset + k_raster_bwd: tiles with silhouette edges */
    DEODR_B200_PH_EDGE_FINALIZE = 10,/* k_finalize_edges */
    DEODR_B200_PH_BACKGROUND_BWD = 11,/* k_background_bwd: background gradient of the tiles without silhouette edges */
    DEODR_B200_PH_COUNT = 12
};
int deodr_b200_timing_enable(DeodrWorkspace *ws, int max_records);
int deodr_b200_timing_collect(DeodrWorkspace *ws, int32_t *phase, float *ms, int capacity);
const char *deodr_b200_phase_name(int phase);

const char *deodr_b200_last_error(void);
const char *deodr_b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* DEODR_B200_H */
