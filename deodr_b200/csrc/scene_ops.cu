// deodr_b200: the steps either side of the raster, on device buffers (SURVEY.md 8f1 / 8f2).
//
//   f1  Camera.project_points / project_points_backward   deodr/differentiable_renderer.py:341-438
//       Scene3D vertex luminosity + its adjoint             deodr/differentiable_renderer.py:814-850
//   f2  TriMeshAdjacencies.edge_on_silhouette               deodr/triangulated_mesh.py:153-166
//       compute_face_normals / compute_vertex_normals (+ adjoints)   deodr/triangulated_mesh.py:113-151
//
// They produce what the rasteriser consumes (ij, depths, colours, edge flags) and consume what it produces (ij_b,
// colors_b) without a round trip through the host: one thread per point / vertex / face, fp64 like the reference's
// numpy code (the flags are bit-exact: same products and differences as np.cross, never fused).
// All of them are elementwise or small gathers: HBM-bound, coalesced on the point index.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <type_traits>

#include "../../include/deodr_b200.h"
#include "reduce.cuh"
#include "rmath.h"
#include "workspace.h"

namespace {

constexpr int BLOCK = 256;
inline int grid_of(size_t n) { return (int)((n + BLOCK - 1) / BLOCK); }

struct Cam {
    double R[9], t[3], K00, K01, K02, K10, K11, K12, k1, k2, p1, p2, k3;
    int distorted;
};

Cam cam_of(const DeodrCamera *c) {
    Cam k;
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) k.R[3 * i + j] = c->extrinsic[4 * i + j];
        k.t[i] = c->extrinsic[4 * i + 3];
    }
    k.K00 = c->intrinsic[0]; k.K01 = c->intrinsic[1]; k.K02 = c->intrinsic[2];
    k.K10 = c->intrinsic[3]; k.K11 = c->intrinsic[4]; k.K12 = c->intrinsic[5];
    k.distorted = c->has_distortion;
    k.k1 = c->distortion[0]; k.k2 = c->distortion[1]; k.p1 = c->distortion[2]; k.p2 = c->distortion[3];
    k.k3 = c->distortion[4];
    return k;
}

// The camera vector of the device-camera entry points (include/deodr_b200.h): extrinsic [R | t] (12, row-major),
// intrinsic (9, row-major), distortion k1 k2 p1 p2 k3 (5).
__device__ __forceinline__ Cam load_cam(const double *v, int distorted) {
    Cam k;
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) k.R[3 * i + j] = v[4 * i + j];
        k.t[i] = v[4 * i + 3];
    }
    k.K00 = v[12]; k.K01 = v[13]; k.K02 = v[14];
    k.K10 = v[15]; k.K11 = v[16]; k.K12 = v[17];
    k.distorted = distorted;
    k.k1 = v[21]; k.k2 = v[22]; k.p1 = v[23]; k.p2 = v[24]; k.k3 = v[25];
    return k;
}

// world_to_camera (:290-292): p . R^T + t
__device__ __forceinline__ void to_camera(const Cam &c, const double *p, double out[3]) {
    for (int i = 0; i < 3; i++) out[i] = p[0] * c.R[3 * i] + p[1] * c.R[3 * i + 1] + p[2] * c.R[3 * i + 2] + c.t[i];
}

// one point of Camera.project_points
__device__ __forceinline__ void project_point(const Cam &c, const double *p, double *ij, double *depth) {
    double pc[3];
    to_camera(c, p, pc);
    const double d = pc[2];
    double x = pc[0] / d, y = pc[1] / d;  // projected (:352)
    if (c.distorted) {                   // (:358-375)
        const double x2 = x * x, y2 = y * y, r2 = x2 + y2, r4 = r2 * r2, r6 = r2 * r4;
        const double radial = 1 + c.k1 * r2 + c.k2 * r4 + c.k3 * r6;
        const double tx = 2 * c.p1 * x * y + c.p2 * (r2 + 2 * x2);
        const double ty = c.p1 * (r2 + 2 * y2) + 2 * c.p2 * x * y;
        const double dx = x * radial + tx, dy = y * radial + ty;
        x = dx;
        y = dy;
    }
    // left_mul_intrinsic (:303-306): projected . K[:2,:2]^T + K[:2,2]
    ij[0] = x * c.K00 + y * c.K01 + c.K02;
    ij[1] = x * c.K10 + y * c.K11 + c.K12;
    *depth = d;
}

__global__ void k_project(const double *points, int n, Cam c, double *ij, double *depths) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    project_point(c, points + 3 * (size_t)i, ij + 2 * (size_t)i, depths + i);
}

// k_project with the camera read from device memory
__global__ void k_project_dev(const double *points, int n, const double *camera, int distorted, double *ij,
                              double *depths) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    project_point(load_cam(camera, distorted), points + 3 * (size_t)i, ij + 2 * (size_t)i, depths + i);
}

// What the adjoint of one point's projection computes on the way, for the camera's adjoint: the camera-frame point pc,
// the undistorted (x, y) and the gradient (qx, qy) of the distorted coordinates, and pc_b.
struct PointAdjoint {
    double pc[3], x, y, qx, qy, pc_b[3];
};

// The adjoint of one point's projection from (gi, gj) and the depth gradient *gd (NULL = none): points_b -> v[3].
// Every product and sum is rounded on its own (DMUL / DADD, never contracted into an FMA), so that each kernel that
// inlines it computes the same bits whatever else the kernel does with the intermediate values.
__device__ __forceinline__ void project_point_b(const Cam &c, const double *p, double gi, double gj, const double *gd,
                                                int reference_transpose, PointAdjoint &a, double v[3]) {
    for (int i = 0; i < 3; i++)
        a.pc[i] = DADD(DADD(DADD(DMUL(p[0], c.R[3 * i]), DMUL(p[1], c.R[3 * i + 1])), DMUL(p[2], c.R[3 * i + 2])),
                       c.t[i]);
    const double d = a.pc[2];
    const double x = a.pc[0] / d, y = a.pc[1] / d;
    a.x = x;
    a.y = y;
    // adjoint of ij = projected . K[:2,:2]^T: projected_b = ij_b . K[:2,:2].  The reference writes ij_b . K[:2,:2]^T
    // (:399 / :412), which is the same only for zero skew and K[1,0] == 0.
    const double qx = reference_transpose ? DADD(DMUL(gi, c.K00), DMUL(gj, c.K01)) : DADD(DMUL(gi, c.K00), DMUL(gj, c.K10));
    const double qy = reference_transpose ? DADD(DMUL(gi, c.K10), DMUL(gj, c.K11)) : DADD(DMUL(gi, c.K01), DMUL(gj, c.K11));
    a.qx = qx;
    a.qy = qy;
    double x_b = qx, y_b = qy;
    if (c.distorted) {  // (:404-430)
        const double r2 = DADD(DMUL(x, x), DMUL(y, y));
        const double r4 = DMUL(r2, r2);
        const double radial = DADD(DADD(DADD(1.0, DMUL(c.k1, r2)), DMUL(c.k2, r4)), DMUL(c.k3, DMUL(r4, r2)));
        x_b = DMUL(qx, radial);
        y_b = DMUL(qy, radial);
        const double radial_b = DADD(DMUL(qx, x), DMUL(qy, y));
        x_b = DADD(x_b, DMUL(qx, DADD(DMUL(DMUL(2.0, c.p1), y), DMUL(DMUL(c.p2, 4.0), x))));
        y_b = DADD(y_b, DMUL(DMUL(DMUL(qx, 2.0), c.p1), x));
        x_b = DADD(x_b, DMUL(DMUL(DMUL(qy, 2.0), c.p2), y));
        y_b = DADD(y_b, DMUL(qy, DADD(DMUL(DMUL(2.0, c.p2), x), DMUL(DMUL(c.p1, 4.0), y))));
        double r2_b = DADD(DMUL(qx, c.p2), DMUL(qy, c.p1));
        r2_b = DADD(r2_b, DMUL(radial_b, DADD(DADD(c.k1, DMUL(DMUL(2.0, c.k2), r2)), DMUL(DMUL(3.0, c.k3), r4))));
        x_b = DADD(x_b, DMUL(DMUL(r2_b, 2.0), x));
        y_b = DADD(y_b, DMUL(DMUL(r2_b, 2.0), y));
    }
    // p_camera_b (:432-436)
    double *pb = a.pc_b;
    pb[0] = x_b / d;
    pb[1] = y_b / d;
    pb[2] = -DADD(DMUL(x_b, a.pc[0]), DMUL(y_b, a.pc[1])) / DMUL(d, d);
    if (gd) pb[2] = DADD(pb[2], *gd);
    for (int j = 0; j < 3; j++)
        // reference (:438): p_camera_b . R^T ; adjoint of world_to_camera: p_camera_b . R
        v[j] = reference_transpose
                   ? DADD(DADD(DMUL(pb[0], c.R[3 * j]), DMUL(pb[1], c.R[3 * j + 1])), DMUL(pb[2], c.R[3 * j + 2]))
                   : DADD(DADD(DMUL(pb[0], c.R[j]), DMUL(pb[1], c.R[3 + j])), DMUL(pb[2], c.R[6 + j]));
}

// ij_b fp32 (the rasteriser's) or fp64 (an autograd caller's, not rounded), NULL = zero; points_b accumulated, or
// overwritten when !ACCUMULATE
template <typename G, bool ACCUMULATE>
__global__ void k_project_b(const double *points, int n, Cam c, const G *ij_b, const double *depths_b,
                            double *points_b, int reference_transpose) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double gi = ij_b ? (double)ij_b[2 * (size_t)i] : 0.0, gj = ij_b ? (double)ij_b[2 * (size_t)i + 1] : 0.0;
    PointAdjoint a;
    double v[3];
    project_point_b(c, points + 3 * (size_t)i, gi, gj, depths_b ? depths_b + i : nullptr, reference_transpose, a, v);
    for (int j = 0; j < 3; j++) {
        if (ACCUMULATE)
            points_b[3 * (size_t)i + j] = DADD(points_b[3 * (size_t)i + j], v[j]);
        else
            points_b[3 * (size_t)i + j] = v[j];
    }
}

// ---- the camera's adjoint ----------------------------------------------------------------------------------------

constexpr int CAMERA_SUMS = 23;  // R_b (9), t_b (3), K_b rows 0-1 (6), distortion_b (5)
constexpr int CAMERA_MAX_CTAS = MAX_K * MAX_CTAS / CAMERA_SUMS;  // the partials of all sums fit the scratch
enum PointsB { POINTS_B_NONE = 0, POINTS_B_OVERWRITE = 1, POINTS_B_ACCUMULATE = 2 };

// The true adjoint of k_project_dev: per point the points_b of k_project_b, and the camera's gradient, summed over the
// points with grid_sum (grid-stride over at most CAMERA_MAX_CTAS CTAs).  Per point, with pc = R p + t, (x, y) the
// undistorted and (xd, yd) the distorted coordinates, q = (qx, qy) their gradient and pc_b the camera-frame gradient:
//   R_b += pc_b p^T,  t_b += pc_b,  K_b[0] += gi (xd, yd, 1),  K_b[1] += gj (xd, yd, 1),
//   (k1, k2, k3)_b += <q, (x, y)> (r2, r4, r6),  p1_b += 2 qx x y + qy (r2 + 2 y^2),  p2_b += qx (r2 + 2 x^2) + 2 qy x y.
// A point whose upstream gradients are all exactly 0 adds nothing (a point at depth 0 would add 0 * inf = NaN).
template <typename G, int MODE>
__global__ void __launch_bounds__(NT) k_project_camera_b(const double *points, int n, const double *camera,
                                                         int distorted, const G *ij_b, const double *depths_b,
                                                         double *points_b, double *camera_b, Scratch *s) {
    __shared__ double tot[CAMERA_SUMS];
    const Cam c = load_cam(camera, distorted);
    double acc[CAMERA_SUMS];
#pragma unroll
    for (int k = 0; k < CAMERA_SUMS; k++) acc[k] = 0;
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
        const double gi = ij_b ? (double)ij_b[2 * i] : 0.0, gj = ij_b ? (double)ij_b[2 * i + 1] : 0.0;
        const double *gd = depths_b ? depths_b + i : nullptr;
        const double p[3] = {points[3 * i], points[3 * i + 1], points[3 * i + 2]};
        PointAdjoint a;
        double v[3];
        project_point_b(c, p, gi, gj, gd, 0, a, v);
        if (MODE == POINTS_B_ACCUMULATE)
            for (int j = 0; j < 3; j++) points_b[3 * i + j] = DADD(points_b[3 * i + j], v[j]);
        else if (MODE == POINTS_B_OVERWRITE)
            for (int j = 0; j < 3; j++) points_b[3 * i + j] = v[j];
        if (gi == 0.0 && gj == 0.0 && (!gd || *gd == 0.0)) continue;
        for (int r = 0; r < 3; r++) {
            for (int j = 0; j < 3; j++) acc[3 * r + j] += a.pc_b[r] * p[j];
            acc[9 + r] += a.pc_b[r];
        }
        double xd = a.x, yd = a.y;
        if (distorted) {
            const double x = a.x, y = a.y, x2 = x * x, y2 = y * y, r2 = x2 + y2, r4 = r2 * r2, r6 = r2 * r4;
            const double radial = 1 + c.k1 * r2 + c.k2 * r4 + c.k3 * r6;
            xd = x * radial + (2 * c.p1 * x * y + c.p2 * (r2 + 2 * x2));
            yd = y * radial + (c.p1 * (r2 + 2 * y2) + 2 * c.p2 * x * y);
            const double radial_b = a.qx * x + a.qy * y;
            acc[18] += radial_b * r2;
            acc[19] += radial_b * r4;
            acc[20] += 2 * a.qx * x * y + a.qy * (r2 + 2 * y2);
            acc[21] += a.qx * (r2 + 2 * x2) + 2 * a.qy * x * y;
            acc[22] += radial_b * r6;
        }
        acc[12] += gi * xd;
        acc[13] += gi * yd;
        acc[14] += gi;
        acc[15] += gj * xd;
        acc[16] += gj * yd;
        acc[17] += gj;
    }
    if (grid_sum<CAMERA_SUMS>(acc, s, tot))
        for (int k = threadIdx.x; k < 26; k += NT) {
            // camera layout: R row r at 4r, t_r at 4r + 3; K at 12 (row 2 never read: 0); distortion at 21
            double x = 0;
            if (k < 12)
                x = (k & 3) == 3 ? tot[9 + k / 4] : tot[3 * (k / 4) + (k & 3)];
            else if (k < 18)
                x = tot[k];
            else if (k >= 21 && distorted)
                x = tot[k - 3];
            camera_b[k] = x;
        }
}

// ---- cube shadow maps (the model of the shadow entry points, include/deodr_b200.h) --------------------------------

constexpr int SHADOW_MAX_LIGHTS = 8;

// the rows of R_k for the faces +x, -x, +y, -y, +z, -z: each a proper rotation (x_c cross y_c = z_c)
__constant__ signed char CUBE_R[6][9] = {
    {0, 1, 0, 0, 0, 1, 1, 0, 0},  {0, 0, 1, 0, 1, 0, -1, 0, 0}, {0, 0, 1, 1, 0, 0, 0, 1, 0},
    {1, 0, 0, 0, 0, 1, 0, -1, 0}, {1, 0, 0, 0, 1, 0, 0, 0, 1},  {0, 1, 0, 1, 0, 0, 0, 0, -1}};

// The camera vector [26] of face k of the cube around p: t = -R_k p is exact (one non-zero product of +-1 per row).
__device__ __forceinline__ void cube_camera(const double *p, int k, int M, double v[26]) {
    for (int i = 0; i < 3; i++) {
        const double r0 = CUBE_R[k][3 * i], r1 = CUBE_R[k][3 * i + 1], r2 = CUBE_R[k][3 * i + 2];
        v[4 * i] = r0;
        v[4 * i + 1] = r1;
        v[4 * i + 2] = r2;
        v[4 * i + 3] = -(r0 * p[0] + r1 * p[1] + r2 * p[2]);
    }
    const double phi = 0.5 * M - 2.0, c = 0.5 * (M - 1);
    v[12] = phi; v[13] = 0; v[14] = c;
    v[15] = 0; v[16] = phi; v[17] = c;
    v[18] = 0; v[19] = 0; v[20] = 1;
    for (int i = 21; i < 26; i++) v[i] = 0;
}

__global__ void k_cube_cameras(const double *lights, int L, int stride, int M, double *cameras) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 6 * L) return;
    cube_camera(lights + (i / 6) * stride, i % 6, M, cameras + 26 * i);
}

// k_project_dev for every face: item i = f n + vertex; the same project_point of the same camera values
__global__ void k_cube_project(const double *points, int n, const double *cameras, long long items, int distorted,
                               double *ij, double *depths) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= items) return;
    const long long f = i / n, v = i - f * n;
    project_point(load_cam(cameras + 26 * f, distorted), points + 3 * v, ij + 2 * i, depths + i);
}

// The cube projection's adjoint: one thread per vertex adds its 6L faces in order into points_b (no atomics); light
// j's position receives -sum over its faces and vertices of R_k^T pc_b (t = -R_k p), summed with grid_sum.  A face
// whose upstream gradients are exactly 0 adds nothing (a vertex at depth 0 would add 0 * inf = NaN).
template <int L>
__global__ void __launch_bounds__(NT) k_cube_project_b(const double *points, int n, const double *cameras,
                                                       const float *ij_b, const float *depths_b, double *points_b,
                                                       double *lights_b, int stride, Scratch *s) {
    constexpr int K = 3 * L;
    __shared__ double tot[K];
    double acc[K];
#pragma unroll
    for (int k = 0; k < K; k++) acc[k] = 0;
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
        const double p[3] = {points[3 * i], points[3 * i + 1], points[3 * i + 2]};
        double sum[3] = {0, 0, 0};
#pragma unroll
        for (int j = 0; j < L; j++)
            for (int k = 0; k < 6; k++) {
                const long long f = 6 * j + k, e = f * n + i;
                const double gi = ij_b[2 * e], gj = ij_b[2 * e + 1], gd = depths_b[e];
                if (gi == 0.0 && gj == 0.0 && gd == 0.0) continue;
                PointAdjoint a;
                double v[3];
                project_point_b(load_cam(cameras + 26 * f, 0), p, gi, gj, &gd, 0, a, v);
                for (int c = 0; c < 3; c++) {
                    sum[c] = DADD(sum[c], v[c]);
                    acc[3 * j + c] -= v[c];
                }
            }
        for (int c = 0; c < 3; c++) points_b[3 * i + c] = DADD(points_b[3 * i + c], sum[c]);
    }
    if (grid_sum<K>(acc, s, tot))
        for (int k = threadIdx.x; k < K; k += NT) lights_b[(k / 3) * stride + k % 3] += tot[k];
}

// The soft 2x2 depth test of a point at map coordinates (u, v) and depth z, kept for the adjoint: the taps' texel
// indices, their smoothstep tests s and derivatives ds, and the two lerps in fu.  Shared by the cube and sun maps.
struct MapTaps {
    double u, v, z, fu, fv, s[4], ds[4], top, bottom;
    long long tap[4];  // texel indices, taps 00, 10, 01, 11
};

// The lookup of one surface point x in light p's cube map, kept for the adjoint.  valid: the projection is in front of
// the face and finite (else V = 1).
struct ShadowTap : MapTaps {
    double cam[26];
    bool valid;
};

// V = lerp(lerp(s_00, s_10, fu), lerp(s_01, s_11, fu), fv) at (t.u, t.v, t.z) in the M x M map starting at texel
// `base` of `maps`, s_k = s((D + bias - z) / softness + 1); indices clamped into [0, M)
__device__ __forceinline__ double map_taps(MapTaps &t, int M, long long base, const float *maps, double bias,
                                           double softness) {
    const double u0 = floor(t.u), v0 = floor(t.v), top = M - 1.0;
    t.fu = t.u - u0;
    t.fv = t.v - v0;
    const long long c0 = (long long)fmin(fmax(u0, 0.0), top), c1 = (long long)fmin(fmax(u0 + 1, 0.0), top);
    const long long r0 = (long long)fmin(fmax(v0, 0.0), top), r1 = (long long)fmin(fmax(v0 + 1, 0.0), top);
    t.tap[0] = base + r0 * M + c0;
    t.tap[1] = base + r0 * M + c1;
    t.tap[2] = base + r1 * M + c0;
    t.tap[3] = base + r1 * M + c1;
    for (int q = 0; q < 4; q++) {
        const double y = (((double)maps[t.tap[q]] + bias) - t.z) / softness + 1.0;
        const double yc = fmin(fmax(y, 0.0), 1.0);
        t.s[q] = yc * yc * (3.0 - 2.0 * yc);
        t.ds[q] = y > 0.0 && y < 1.0 ? 6.0 * yc * (1.0 - yc) : 0.0;
    }
    t.top = t.s[0] + t.fu * (t.s[1] - t.s[0]);
    t.bottom = t.s[2] + t.fu * (t.s[3] - t.s[2]);
    return t.top + t.fv * (t.bottom - t.top);
}

// The adjoint of map_taps from g = V_b: the texels' gradients into mb (fp32 atomics) and those of u, v and z
__device__ __forceinline__ void map_taps_b(const MapTaps &t, double g, double softness, float *mb, double &fu_b,
                                           double &fv_b, double &z_b) {
    // V = top + fv (bottom - top), top / bottom = lerps in fu of the taps 00, 10 / 01, 11
    const double top_b = g * (1.0 - t.fv), bottom_b = g * t.fv;
    fv_b = g * (t.bottom - t.top);
    fu_b = top_b * (t.s[1] - t.s[0]) + bottom_b * (t.s[3] - t.s[2]);
    const double s_b[4] = {top_b * (1.0 - t.fu), top_b * t.fu, bottom_b * (1.0 - t.fu), bottom_b * t.fu};
    z_b = 0;
    for (int q = 0; q < 4; q++) {
        const double D_b = s_b[q] * t.ds[q] / softness;
        if (D_b != 0.0) atomicAdd(mb + t.tap[q], (float)D_b);
        z_b -= D_b;
    }
}

__device__ __forceinline__ double shadow_lookup(const double x[3], const double *p, int M, const float *maps,
                                                double bias, double softness, ShadowTap &t) {
    const double d[3] = {x[0] - p[0], x[1] - p[1], x[2] - p[2]};
    const double ax = fabs(d[0]), ay = fabs(d[1]), az = fabs(d[2]);
    const int axis = ax >= ay && ax >= az ? 0 : (ay >= az ? 1 : 2);
    const double da = axis == 0 ? d[0] : (axis == 1 ? d[1] : d[2]);  // selects, not an indexed (local) array
    const int k = 2 * axis + (da > 0 ? 0 : 1);
    cube_camera(p, k, M, t.cam);
    double ij[2];
    project_point(load_cam(t.cam, 0), x, ij, &t.z);
    t.u = ij[0];
    t.v = ij[1];
    t.valid = t.z > 0 && isfinite(t.u) && isfinite(t.v);
    if (!t.valid) return 1.0;
    return map_taps(t, M, (long long)k * M * M, maps, bias, softness);
}

// vis [H,W,L] of the G-buffer's pixels, one thread per pixel (1 where a = 0)
__global__ void __launch_bounds__(NT) k_shadow_visibility(const float *ch, long long pixels, int stride, int off_pos,
                                                          int off_cov, const double *lights, int L, int lstride,
                                                          const float *maps, int M, double bias, double softness,
                                                          float *vis) {
    const long long p = (long long)blockIdx.x * NT + threadIdx.x;
    if (p >= pixels) return;
    const float *px = ch + p * stride;
    const double a = px[off_cov];
    float *out = vis + p * L;
    if (a == 0.0) {
        for (int j = 0; j < L; j++) out[j] = 1.0f;
        return;
    }
    const double x[3] = {px[off_pos] / a, px[off_pos + 1] / a, px[off_pos + 2] / a};
    for (int j = 0; j < L; j++) {
        ShadowTap t;
        out[j] = (float)shadow_lookup(x, lights + j * lstride, M, maps + (long long)6 * j * M * M, bias, softness, t);
    }
}

// The visibility's adjoint from vis_b: per pixel and light the taps' gradients (maps_b, fp32 atomics) and x's, which
// goes into the position and coverage slices of ch_b (accumulated) and, negated, into the light's position (summed
// with grid_sum in a fixed order and added to lights_b).
template <int L>
__global__ void __launch_bounds__(NT) k_shadow_visibility_b(const float *ch, float *ch_b, long long pixels, int stride,
                                                            int off_pos, int off_cov, const double *lights,
                                                            int lstride, const float *maps, int M, double bias,
                                                            double softness, const float *vis_b, float *maps_b,
                                                            double *lights_b, Scratch *s) {
    constexpr int K = 3 * L;
    __shared__ double tot[K];
    double acc[K];
#pragma unroll
    for (int k = 0; k < K; k++) acc[k] = 0;
    for (long long p = (long long)blockIdx.x * NT + threadIdx.x; p < pixels; p += (long long)gridDim.x * NT) {
        const float *px = ch + p * stride;
        const double a = px[off_cov];
        if (a == 0.0) continue;
        const double x[3] = {px[off_pos] / a, px[off_pos + 1] / a, px[off_pos + 2] / a};
        double x_b[3] = {0, 0, 0};
#pragma unroll
        for (int j = 0; j < L; j++) {
            const double g = vis_b[p * L + j];
            if (g == 0.0) continue;
            ShadowTap t;
            shadow_lookup(x, lights + j * lstride, M, maps + (long long)6 * j * M * M, bias, softness, t);
            if (!t.valid) continue;
            double fu_b, fv_b, z_b;
            map_taps_b(t, g, softness, maps_b + (long long)6 * j * M * M, fu_b, fv_b, z_b);
            PointAdjoint pa;
            double v[3];
            project_point_b(load_cam(t.cam, 0), x, fu_b, fv_b, &z_b, 0, pa, v);
            for (int c = 0; c < 3; c++) {
                x_b[c] += v[c];
                acc[3 * j + c] -= v[c];
            }
        }
        float *pb = ch_b + p * stride;
        for (int c = 0; c < 3; c++) pb[off_pos + c] = (float)((double)pb[off_pos + c] + x_b[c] / a);
        pb[off_cov] = (float)((double)pb[off_cov] - ((x_b[0] * x[0] + x_b[1] * x[1]) + x_b[2] * x[2]) / a);
    }
    if (grid_sum<K>(acc, s, tot))
        for (int k = threadIdx.x; k < K; k += NT) lights_b[(k / 3) * lstride + k % 3] += tot[k];
}

// ---- the directional light's shadow map (the model of the sun shadow entry points, include/deodr_b200.h) ---------

// Frisvad's orthonormal frame (e1, e2, d) around the direction d = l / |l| the light travels (d = +z where |l| = 0),
// with a = 1 / (1 + d_z) away from the pole d_z < -0.9999999
struct SunFrame {
    double e1[3], e2[3], d[3], ll, a;
    bool pole;
};

__device__ __forceinline__ void sun_frame(const double *l, SunFrame &f) {
    f.ll = sqrt((l[0] * l[0] + l[1] * l[1]) + l[2] * l[2]);
    for (int j = 0; j < 3; j++) f.d[j] = f.ll > 0 ? l[j] / f.ll : (j == 2 ? 1.0 : 0.0);
    f.pole = f.d[2] < -0.9999999;
    if (f.pole) {
        f.a = 0;
        f.e1[0] = 0; f.e1[1] = -1; f.e1[2] = 0;
        f.e2[0] = -1; f.e2[1] = 0; f.e2[2] = 0;
        return;
    }
    f.a = 1.0 / (1.0 + f.d[2]);
    const double b = -f.d[0] * f.d[1] * f.a;
    f.e1[0] = 1.0 - f.d[0] * f.d[0] * f.a; f.e1[1] = b; f.e1[2] = -f.d[0];
    f.e2[0] = b; f.e2[1] = 1.0 - f.d[1] * f.d[1] * f.a; f.e2[2] = -f.d[1];
}

// l_b [3] from the gradients of e1, e2 and d: the frame's derivative, then (I - d d^T) / |l| (0 where |l| = 0)
__device__ __forceinline__ void sun_frame_b(const SunFrame &f, const double *e1_b, const double *e2_b,
                                            const double *d_in_b, double *l_b) {
    double d_b[3] = {d_in_b[0], d_in_b[1], d_in_b[2]};
    if (!(f.ll > 0)) {
        l_b[0] = l_b[1] = l_b[2] = 0;
        return;
    }
    if (!f.pole) {
        const double a = f.a, x = f.d[0], y = f.d[1], B = e1_b[1] + e2_b[0];  // b = -x y a is e1_y and e2_x
        d_b[0] += (-2.0 * x * a * e1_b[0] - y * a * B) - e1_b[2];
        d_b[1] += (-x * a * B - 2.0 * y * a * e2_b[1]) - e2_b[2];
        d_b[2] += a * a * ((x * x * e1_b[0] + x * y * B) + y * y * e2_b[1]);
    }
    const double dd = (f.d[0] * d_b[0] + f.d[1] * d_b[1]) + f.d[2] * d_b[2];
    for (int j = 0; j < 3; j++) l_b[j] = (d_b[j] - f.d[j] * dd) / f.ll;
}

// The window of the map: its centre c, radius r and size M; k = phi / r, h = (M - 1) / 2
struct SunWindow {
    double c[3], r;
    int M;
};

// (u, v, z) of a world point x and w = x - c: u = h + k <e1, w>, v = h + k <e2, w>, z = <d, w> + 2 r
__device__ __forceinline__ void sun_point(const SunFrame &f, const SunWindow &win, const double *x, double w[3],
                                          double &u, double &v, double &z) {
    const double k = (0.5 * win.M - 2.0) / win.r, h = 0.5 * (win.M - 1);
    for (int j = 0; j < 3; j++) w[j] = x[j] - win.c[j];
    u = h + k * ((f.e1[0] * w[0] + f.e1[1] * w[1]) + f.e1[2] * w[2]);
    v = h + k * ((f.e2[0] * w[0] + f.e2[1] * w[1]) + f.e2[2] * w[2]);
    z = ((f.d[0] * w[0] + f.d[1] * w[1]) + f.d[2] * w[2]) + 2.0 * win.r;
}

// The adjoint of sun_point from (u_b, v_b, z_b): x_b, and the frame's gradients added into fb = (e1_b, e2_b, d_b)
__device__ __forceinline__ void sun_point_b(const SunFrame &f, const SunWindow &win, const double w[3], double u_b,
                                            double v_b, double z_b, double x_b[3], double fb[9]) {
    const double k = (0.5 * win.M - 2.0) / win.r, ku = k * u_b, kv = k * v_b;
    for (int j = 0; j < 3; j++) {
        x_b[j] = (ku * f.e1[j] + kv * f.e2[j]) + z_b * f.d[j];
        fb[j] += ku * w[j];
        fb[3 + j] += kv * w[j];
        fb[6 + j] += z_b * w[j];
    }
}

__global__ void __launch_bounds__(NT) k_sun_project(const double *points, int n, const double *light, SunWindow win,
                                                    double *ij, double *depths) {
    const long long i = (long long)blockIdx.x * NT + threadIdx.x;
    if (i >= n) return;
    SunFrame f;
    sun_frame(light, f);
    double w[3];
    sun_point(f, win, points + 3 * i, w, ij[2 * i], ij[2 * i + 1], depths[i]);
}

// grid_sum's 9 frame sums (e1_b, e2_b, d_b) taken through the frame's adjoint and added into light_b[0:3]
__device__ __forceinline__ void sun_light_b(const double *light, const double (&acc)[9], Scratch *s, double *light_b) {
    __shared__ double tot[9];
    if (grid_sum<9>(acc, s, tot) && threadIdx.x == 0) {
        SunFrame f;
        sun_frame(light, f);
        double l_b[3];
        sun_frame_b(f, tot, tot + 3, tot + 6, l_b);
        for (int j = 0; j < 3; j++) light_b[j] += l_b[j];
    }
}

// The sun projection's adjoint from the rasteriser's ij_b [n,2] and depths_b [n] (fp32): vertices_b accumulated, one
// thread per vertex (no atomics); light_b[0:3] through the frame, summed with grid_sum in a fixed order.  A vertex whose
// upstream gradients are exactly 0 adds nothing.
__global__ void __launch_bounds__(NT) k_sun_project_b(const double *points, int n, const double *light, SunWindow win,
                                                      const float *ij_b, const float *depths_b, double *points_b,
                                                      double *light_b, Scratch *s) {
    double acc[9];
#pragma unroll
    for (int k = 0; k < 9; k++) acc[k] = 0;
    SunFrame f;
    sun_frame(light, f);
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
        const double gi = ij_b[2 * i], gj = ij_b[2 * i + 1], gd = depths_b[i];
        if (gi == 0.0 && gj == 0.0 && gd == 0.0) continue;
        double w[3], u, v, z, x_b[3];
        sun_point(f, win, points + 3 * i, w, u, v, z);
        sun_point_b(f, win, w, gi, gj, gd, x_b, acc);
        for (int c = 0; c < 3; c++) points_b[3 * i + c] = DADD(points_b[3 * i + c], x_b[c]);
    }
    sun_light_b(light, acc, s, light_b);
}

// The lookup of one surface point x in the sun map: false (V = 1) where x is not finite, outside the window's sphere,
// or the light is off
__device__ __forceinline__ bool sun_lookup(const SunFrame &f, const SunWindow &win, const double x[3], double w[3],
                                           MapTaps &t) {
    if (!(f.ll > 0) || !isfinite(x[0]) || !isfinite(x[1]) || !isfinite(x[2])) return false;
    sun_point(f, win, x, w, t.u, t.v, t.z);
    return (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2] <= win.r * win.r;
}

// sun_vis [H,W] of the G-buffer's pixels, one thread per pixel (1 where a = 0)
__global__ void __launch_bounds__(NT) k_sun_visibility(const float *ch, long long pixels, int stride, int off_pos,
                                                       int off_cov, const double *light, SunWindow win,
                                                       const float *map, double bias, double softness, float *vis) {
    const long long p = (long long)blockIdx.x * NT + threadIdx.x;
    if (p >= pixels) return;
    const float *px = ch + p * stride;
    const double a = px[off_cov];
    double V = 1.0;
    if (a != 0.0) {
        SunFrame f;
        sun_frame(light, f);
        const double x[3] = {px[off_pos] / a, px[off_pos + 1] / a, px[off_pos + 2] / a};
        double w[3];
        MapTaps t;
        if (sun_lookup(f, win, x, w, t)) V = map_taps(t, win.M, 0, map, bias, softness);
    }
    vis[p] = (float)V;
}

// The sun visibility's adjoint from vis_b [H,W]: the taps' gradients (map_b, fp32 atomics) and x's, which goes into
// the position and coverage slices of ch_b (accumulated) and through the projection into light_b[0:3] (grid_sum)
__global__ void __launch_bounds__(NT) k_sun_visibility_b(const float *ch, float *ch_b, long long pixels, int stride,
                                                         int off_pos, int off_cov, const double *light, SunWindow win,
                                                         const float *map, double bias, double softness,
                                                         const float *vis_b, float *map_b, double *light_b,
                                                         Scratch *s) {
    double acc[9];
#pragma unroll
    for (int k = 0; k < 9; k++) acc[k] = 0;
    SunFrame f;
    sun_frame(light, f);
    for (long long p = (long long)blockIdx.x * NT + threadIdx.x; p < pixels; p += (long long)gridDim.x * NT) {
        const float *px = ch + p * stride;
        const double a = px[off_cov], g = vis_b[p];
        if (a == 0.0 || g == 0.0) continue;
        const double x[3] = {px[off_pos] / a, px[off_pos + 1] / a, px[off_pos + 2] / a};
        double w[3];
        MapTaps t;
        if (!sun_lookup(f, win, x, w, t)) continue;
        map_taps(t, win.M, 0, map, bias, softness);
        double fu_b, fv_b, z_b, x_b[3];
        map_taps_b(t, g, softness, map_b, fu_b, fv_b, z_b);
        sun_point_b(f, win, w, fu_b, fv_b, z_b, x_b, acc);
        float *pb = ch_b + p * stride;
        for (int c = 0; c < 3; c++) pb[off_pos + c] = (float)((double)pb[off_pos + c] + x_b[c] / a);
        pb[off_cov] = (float)((double)pb[off_cov] - ((x_b[0] * x[0] + x_b[1] * x[1]) + x_b[2] * x[2]) / a);
    }
    sun_light_b(light, acc, s, light_b);
}

// Calls f(L) with L from 1 to SHADOW_MAX_LIGHTS as a compile-time constant
template <typename F>
void with_lights(int L, F &&f) {
    switch (L) {
        case 1: return f(std::integral_constant<int, 1>{});
        case 2: return f(std::integral_constant<int, 2>{});
        case 3: return f(std::integral_constant<int, 3>{});
        case 4: return f(std::integral_constant<int, 4>{});
        case 5: return f(std::integral_constant<int, 5>{});
        case 6: return f(std::integral_constant<int, 6>{});
        case 7: return f(std::integral_constant<int, 7>{});
        default: return f(std::integral_constant<int, 8>{});
    }
}

// grid_sum of K sums: at most MAX_CTAS CTAs, and beyond MAX_K sums at most MAX_K * MAX_CTAS / K
int sum_grid(long long items, int K) {
    const long long g = std::max<long long>(1, (items + NT - 1) / NT);
    return (int)std::min<long long>(g, K <= MAX_K ? MAX_CTAS : MAX_K * MAX_CTAS / K);
}

bool shadow_map_ok(int M) { return M >= 8 && M <= 4096; }
bool shadow_band_ok(double bias, double softness) {
    return std::isfinite(bias) && std::isfinite(softness) && bias > 0 && softness > 0;
}
// the sun map's window: a finite centre and a finite radius > 0
bool sun_window_ok(const double *center, double radius) {
    return center && std::isfinite(center[0]) && std::isfinite(center[1]) && std::isfinite(center[2]) &&
           std::isfinite(radius) && radius > 0;
}
SunWindow sun_window(const double *center, double radius, int M) {
    SunWindow w;
    for (int j = 0; j < 3; j++) w.c[j] = center[j];
    w.r = radius;
    w.M = M;
    return w;
}
bool shadow_lights_ok(int L, int P) { return L >= 1 && L <= SHADOW_MAX_LIGHTS && P >= 1 && P <= 4; }

// the G-buffer sizes and the position and coverage offsets the lookup reads, in either Phong form
bool shadow_io_ok(const DeodrPhongIO *io) {
    if (!io || !io->channels || io->H < 1 || io->W < 1 || io->C < 1 || io->C > 32760) return false;
    const int K = io->off_albedo == -1 ? 7 : io->C + 7;
    return io->off_position >= 0 && io->off_position <= K - 3 && io->off_coverage >= 0 && io->off_coverage < K &&
           (io->off_coverage < io->off_position || io->off_coverage >= io->off_position + 3);
}

struct Light {
    double d[3], ambient;
    int directional;
};

// np.maximum(0, -s): NaN propagates (a zero-area face has a NaN normal), where fmax would return 0
__device__ __forceinline__ double directional_of(double s) { return s >= 0.0 ? 0.0 : -s; }

__global__ void k_luminosity(const double *normals, const double *vcol, int n, int C, Light L, float *lum, float *colors) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n) return;
    double dir = 0.0;
    if (L.directional) {
        const double *nv = normals + 3 * (size_t)v;
        const double s = (nv[0] * L.d[0] + nv[1] * L.d[1]) + nv[2] * L.d[2];  // np.sum(axis=1) of three terms
        dir = directional_of(s);
    }
    const double l = dir + L.ambient;
    if (lum) lum[v] = (float)l;
    if (colors && vcol)
        for (int c = 0; c < C; c++) colors[(size_t)v * C + c] = (float)(vcol[(size_t)v * C + c] * l);
}

// block-level sum of four doubles into out[0..3] (one fp64 atomic per block and component)
__device__ void block_add4(double v0, double v1, double v2, double v3, double *out) {
    __shared__ double part[4][BLOCK / 32];
    double v[4] = {v0, v1, v2, v3};
    for (int k = 0; k < 4; k++)
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], o);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0)
        for (int k = 0; k < 4; k++) part[k][warp] = v[k];
    __syncthreads();
    if (threadIdx.x < 4) {
        double s = 0;
        for (int w = 0; w < BLOCK / 32; w++) s += part[threadIdx.x][w];
        if (s != 0.0) atomicAdd(out + threadIdx.x, s);
    }
}

__global__ void k_luminosity_b(const double *normals, const double *vcol, int n, int C, Light L, const float *colors_b,
                               const float *lum_b_in, double *normals_b, double *vcol_b, double *light_b) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    double lb = 0.0, g[3] = {0, 0, 0};
    if (v < n) {
        double dir = 0.0;
        const double *nv = normals + 3 * (size_t)v;
        if (L.directional) dir = directional_of((nv[0] * L.d[0] + nv[1] * L.d[1]) + nv[2] * L.d[2]);
        const double l = dir + L.ambient;
        if (colors_b && vcol)
            for (int c = 0; c < C; c++) {
                const double cb = (double)colors_b[(size_t)v * C + c];
                lb += vcol[(size_t)v * C + c] * cb;                         // vertices_luminosity_b (:838)
                if (vcol_b) vcol_b[(size_t)v * C + c] = cb * l;             // vertices_colors_b (:839), assigned
            }
        if (lum_b_in) lb += (double)lum_b_in[v];
        const double gate = (L.directional && dir > 0) ? lb : 0.0;          // (:845-849)
        for (int j = 0; j < 3; j++) {
            g[j] = -gate * nv[j];
            if (normals_b) normals_b[3 * (size_t)v + j] = -gate * L.d[j];
        }
    }
    if (light_b) block_add4(g[0], g[1], g[2], lb, light_b);
}

// ---- f2 ------------------------------------------------------------------------------------------------------

// face_visible (:161-163): np.cross(u, v) of the 2-D edges, > 0 (clockwise) or < 0 - two products, one difference
__global__ void k_face_visible(DeodrMeshTopology m, const double *ij, uint8_t *visible) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= m.nb_faces) return;
    const uint32_t a = m.faces[3 * (size_t)f], b = m.faces[3 * (size_t)f + 1], c = m.faces[3 * (size_t)f + 2];
    const double ux = DSUB(ij[2 * (size_t)b], ij[2 * (size_t)a]), uy = DSUB(ij[2 * (size_t)b + 1], ij[2 * (size_t)a + 1]);
    const double vx = DSUB(ij[2 * (size_t)c], ij[2 * (size_t)a]), vy = DSUB(ij[2 * (size_t)c + 1], ij[2 * (size_t)a + 1]);
    const double cr = DSUB(DMUL(ux, vy), DMUL(uy, vx));
    visible[f] = (uint8_t)(m.clockwise ? cr > 0 : cr < 0);
}

// edge_bool = (edges_faces_ones * face_visible) == 1, gathered through faces_edges (:164-165)
__global__ void k_edge_flags(DeodrMeshTopology m, const uint8_t *visible, uint8_t *edgeflags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 3 * m.nb_faces) return;
    const int e = m.faces_edges[i];
    int count = 0;
    for (int k = m.edge_face_offset[e]; k < m.edge_face_offset[e + 1]; k++) count += visible[m.edge_face_index[k]];
    edgeflags[i] = (uint8_t)(count == 1);
}

__device__ __forceinline__ void face_cross(const DeodrMeshTopology &m, const double *vertices, int f, double u[3],
                                           double v[3], double n[3]) {
    const uint32_t a = m.faces[3 * (size_t)f], b = m.faces[3 * (size_t)f + 1], c = m.faces[3 * (size_t)f + 2];
    for (int j = 0; j < 3; j++) {
        u[j] = vertices[3 * (size_t)b + j] - vertices[3 * (size_t)a + j];
        v[j] = vertices[3 * (size_t)c + j] - vertices[3 * (size_t)a + j];
    }
    n[0] = u[1] * v[2] - u[2] * v[1];
    n[1] = u[2] * v[0] - u[0] * v[2];
    n[2] = u[0] * v[1] - u[1] * v[0];
    if (m.clockwise)
        for (int j = 0; j < 3; j++) n[j] = -n[j];
}

// compute_face_normals (:113-123): normalize(+-cross(u, v))
__global__ void k_face_normals(DeodrMeshTopology m, const double *vertices, double *face_normals) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= m.nb_faces) return;
    double u[3], v[3], n[3];
    face_cross(m, vertices, f, u, v, n);
    const double norm = sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]);
    for (int j = 0; j < 3; j++) face_normals[3 * (size_t)f + j] = n[j] / norm;
}

// compute_vertex_normals (:137-143): normalize(_vertices_faces * face_normals) - a gather over the incident faces
__global__ void k_vertex_normals(DeodrMeshTopology m, const double *face_normals, double *vertex_normals) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= m.nb_vertices) return;
    double n[3] = {0, 0, 0};
    for (int k = m.vertex_face_offset[v]; k < m.vertex_face_offset[v + 1]; k++) {
        const int f = m.vertex_face_index[k];
        for (int j = 0; j < 3; j++) n[j] += face_normals[3 * (size_t)f + j];
    }
    const double norm = sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]);
    for (int j = 0; j < 3; j++) vertex_normals[3 * (size_t)v + j] = n[j] / norm;
}

// normalize_backward (deodr/tools.py:42-47)
__device__ __forceinline__ void normalize_b(const double x[3], const double xn_b[3], double out[3]) {
    const double n2 = (x[0] * x[0] + x[1] * x[1]) + x[2] * x[2];
    const double inv_n = 1.0 / sqrt(n2);
    const double n_b = -((xn_b[0] * x[0] + xn_b[1] * x[1]) + xn_b[2] * x[2]) * (inv_n * inv_n);
    for (int j = 0; j < 3; j++) out[j] = (xn_b[j] + x[j] * n_b) * inv_n;
}

// compute_vertex_normals_backward (:145-151): face_normals_b = _vertices_faces^T * normalize_backward(n, normals_b);
// first per vertex (the un-normalised sum is recomputed from the unit face normals), then gathered per face
__global__ void k_vertex_normals_b1(DeodrMeshTopology m, const double *vertices, const double *vertex_normals_b,
                                    double *vertex_sum_b) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= m.nb_vertices) return;
    double n[3] = {0, 0, 0};
    for (int k = m.vertex_face_offset[v]; k < m.vertex_face_offset[v + 1]; k++) {
        const int f = m.vertex_face_index[k];
        double u[3], w[3], c[3];
        face_cross(m, vertices, f, u, w, c);
        const double norm = sqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]);
        for (int j = 0; j < 3; j++) n[j] += c[j] / norm;
    }
    double g[3] = {vertex_normals_b[3 * (size_t)v], vertex_normals_b[3 * (size_t)v + 1], vertex_normals_b[3 * (size_t)v + 2]};
    double out[3];
    normalize_b(n, g, out);
    for (int j = 0; j < 3; j++) vertex_sum_b[3 * (size_t)v + j] = out[j];
}

// compute_face_normals_backward (:125-135): per face, n_b = normalize_backward(n, normals_b); u_b, v_b =
// cross_backward(u, v, +-n_b); triangles_b = (-u_b - v_b, u_b, v_b) scattered with np.add.at
__global__ void k_face_normals_b(DeodrMeshTopology m, const double *vertices, const double *vertex_sum_b,
                                 double *face_normals_b, double *vertices_b) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= m.nb_faces) return;
    const uint32_t id[3] = {m.faces[3 * (size_t)f], m.faces[3 * (size_t)f + 1], m.faces[3 * (size_t)f + 2]};
    double fb[3] = {0, 0, 0};
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) fb[j] += vertex_sum_b[3 * (size_t)id[i] + j];
    if (face_normals_b)
        for (int j = 0; j < 3; j++) face_normals_b[3 * (size_t)f + j] = fb[j];
    double u[3], v[3], n[3], n_b[3];
    face_cross(m, vertices, f, u, v, n);
    normalize_b(n, fb, n_b);
    if (m.clockwise)
        for (int j = 0; j < 3; j++) n_b[j] = -n_b[j];
    // cross_backward (tools.py:50-53): v_b = cross(c_b, u), u_b = cross(v, c_b)
    const double v_b[3] = {n_b[1] * u[2] - n_b[2] * u[1], n_b[2] * u[0] - n_b[0] * u[2], n_b[0] * u[1] - n_b[1] * u[0]};
    const double u_b[3] = {v[1] * n_b[2] - v[2] * n_b[1], v[2] * n_b[0] - v[0] * n_b[2], v[0] * n_b[1] - v[1] * n_b[0]};
    for (int j = 0; j < 3; j++) {
        atomicAdd(vertices_b + 3 * (size_t)id[0] + j, -u_b[j] - v_b[j]);
        atomicAdd(vertices_b + 3 * (size_t)id[1] + j, u_b[j]);
        atomicAdd(vertices_b + 3 * (size_t)id[2] + j, v_b[j]);
    }
}

// ---- tangent frames and normal maps (the model in include/deodr_b200.h) --------------------------------------------

struct FaceTangent {
    double e1[3], e2[3], du1, dv1, du2, dv2, sigma;
};

// face f's edges, uv deltas and sigma = sign(det); t_f = sigma (dv2 e1 - dv1 e2), b_f = sigma (du1 e2 - du2 e1)
__device__ __forceinline__ FaceTangent face_tangent(const DeodrMeshTopology &m, const double *vertices,
                                                    const uint32_t *faces_uv, const double *uv, int f, double t[3],
                                                    double b[3]) {
    FaceTangent q;
    const uint32_t i0 = m.faces[3 * (size_t)f], i1 = m.faces[3 * (size_t)f + 1], i2 = m.faces[3 * (size_t)f + 2];
    const uint32_t k0 = faces_uv[3 * (size_t)f], k1 = faces_uv[3 * (size_t)f + 1], k2 = faces_uv[3 * (size_t)f + 2];
    for (int j = 0; j < 3; j++) {
        q.e1[j] = vertices[3 * (size_t)i1 + j] - vertices[3 * (size_t)i0 + j];
        q.e2[j] = vertices[3 * (size_t)i2 + j] - vertices[3 * (size_t)i0 + j];
    }
    q.du1 = uv[2 * (size_t)k1] - uv[2 * (size_t)k0];
    q.dv1 = uv[2 * (size_t)k1 + 1] - uv[2 * (size_t)k0 + 1];
    q.du2 = uv[2 * (size_t)k2] - uv[2 * (size_t)k0];
    q.dv2 = uv[2 * (size_t)k2 + 1] - uv[2 * (size_t)k0 + 1];
    const double det = q.du1 * q.dv2 - q.du2 * q.dv1;
    q.sigma = det > 0 ? 1.0 : (det < 0 ? -1.0 : 0.0);
    for (int j = 0; j < 3; j++) {
        t[j] = q.sigma * (q.dv2 * q.e1[j] - q.dv1 * q.e2[j]);
        b[j] = q.sigma * (q.du1 * q.e2[j] - q.du2 * q.e1[j]);
    }
    return q;
}

// x / |x|, or 0 when |x| = 0
__device__ __forceinline__ void unit_or_zero(const double x[3], double out[3]) {
    const double norm = sqrt((x[0] * x[0] + x[1] * x[1]) + x[2] * x[2]);
    for (int j = 0; j < 3; j++) out[j] = norm > 0 ? x[j] / norm : 0.0;
}

// the adjoint of unit_or_zero: 0 when |x| = 0
__device__ __forceinline__ void unit_or_zero_b(const double x[3], const double xn_b[3], double out[3]) {
    const double n2 = (x[0] * x[0] + x[1] * x[1]) + x[2] * x[2];
    if (!(n2 > 0)) {
        for (int j = 0; j < 3; j++) out[j] = 0.0;
        return;
    }
    normalize_b(x, xn_b, out);
}

__global__ void k_face_tangents(DeodrMeshTopology m, const double *vertices, const uint32_t *faces_uv,
                                const double *uv, double *face_frames) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= m.nb_faces) return;
    double t[3], b[3];
    face_tangent(m, vertices, faces_uv, uv, f, t, b);
    for (int j = 0; j < 3; j++) {
        face_frames[6 * (size_t)f + j] = t[j];
        face_frames[6 * (size_t)f + 3 + j] = b[j];
    }
}

// T_v, B_v: the face terms summed over the vertex-face CSR in its order (as k_vertex_normals), then normalised
__global__ void k_vertex_tangents(DeodrMeshTopology m, const double *face_frames, double *frames) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= m.nb_vertices) return;
    double s[6] = {0, 0, 0, 0, 0, 0};
    for (int k = m.vertex_face_offset[v]; k < m.vertex_face_offset[v + 1]; k++) {
        const int f = m.vertex_face_index[k];
        for (int j = 0; j < 6; j++) s[j] += face_frames[6 * (size_t)f + j];
    }
    double out[6];
    unit_or_zero(s, out);
    unit_or_zero(s + 3, out + 3);
    for (int j = 0; j < 6; j++) frames[6 * (size_t)v + j] = out[j];
}

// per vertex: the sums' adjoint (the sums recomputed from the faces in the forward's order)
__global__ void k_vertex_tangents_b1(DeodrMeshTopology m, const double *vertices, const uint32_t *faces_uv,
                                     const double *uv, const double *frames_b, double *sum_b) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= m.nb_vertices) return;
    double s[6] = {0, 0, 0, 0, 0, 0};
    for (int k = m.vertex_face_offset[v]; k < m.vertex_face_offset[v + 1]; k++) {
        double t[3], b[3];
        face_tangent(m, vertices, faces_uv, uv, m.vertex_face_index[k], t, b);
        for (int j = 0; j < 3; j++) {
            s[j] += t[j];
            s[3 + j] += b[j];
        }
    }
    double g[6], out[6];
    for (int j = 0; j < 6; j++) g[j] = frames_b[6 * (size_t)v + j];
    unit_or_zero_b(s, g, out);
    unit_or_zero_b(s + 3, g + 3, out + 3);
    for (int j = 0; j < 6; j++) sum_b[6 * (size_t)v + j] = out[j];
}

// per face: t_f_b and b_f_b gathered from its corners, taken to (e1_b, e2_b, du1_b, dv1_b, du2_b, dv2_b) [10]
__global__ void k_face_tangents_b(DeodrMeshTopology m, const double *vertices, const uint32_t *faces_uv,
                                  const double *uv, const double *sum_b, double *face_b) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= m.nb_faces) return;
    double t[3], b[3], tb[3] = {0, 0, 0}, bb[3] = {0, 0, 0};
    const FaceTangent q = face_tangent(m, vertices, faces_uv, uv, f, t, b);
    for (int c = 0; c < 3; c++) {
        const uint32_t id = m.faces[3 * (size_t)f + c];
        for (int j = 0; j < 3; j++) {
            tb[j] += sum_b[6 * (size_t)id + j];
            bb[j] += sum_b[6 * (size_t)id + 3 + j];
        }
    }
    double *o = face_b + 10 * (size_t)f;
    for (int j = 0; j < 3; j++) {
        o[j] = q.sigma * (q.dv2 * tb[j] - q.du2 * bb[j]);
        o[3 + j] = q.sigma * (q.du1 * bb[j] - q.dv1 * tb[j]);
    }
    o[6] = q.sigma * ((q.e2[0] * bb[0] + q.e2[1] * bb[1]) + q.e2[2] * bb[2]);
    o[7] = -q.sigma * ((q.e2[0] * tb[0] + q.e2[1] * tb[1]) + q.e2[2] * tb[2]);
    o[8] = -q.sigma * ((q.e1[0] * bb[0] + q.e1[1] * bb[1]) + q.e1[2] * bb[2]);
    o[9] = q.sigma * ((q.e1[0] * tb[0] + q.e1[1] * tb[1]) + q.e1[2] * tb[2]);
}

// per position vertex: the corners it holds in its faces (a face listed twice in the CSR, for a repeated corner, is
// visited once and adds every such corner), accumulated into vertices_b in the CSR's order
__global__ void k_tangents_vertices_b(DeodrMeshTopology m, const double *face_b, double *vertices_b) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= m.nb_vertices) return;
    double acc[3] = {0, 0, 0};
    const int k0 = m.vertex_face_offset[v];
    for (int k = k0; k < m.vertex_face_offset[v + 1]; k++) {
        const int f = m.vertex_face_index[k];
        if (k > k0 && m.vertex_face_index[k - 1] == f) continue;
        const double *o = face_b + 10 * (size_t)f;
        for (int c = 0; c < 3; c++) {
            if (m.faces[3 * (size_t)f + c] != (uint32_t)v) continue;
            for (int j = 0; j < 3; j++) acc[j] += c == 0 ? -o[j] - o[3 + j] : o[3 * (c - 1) + j];
        }
    }
    for (int j = 0; j < 3; j++) vertices_b[3 * (size_t)v + j] += acc[j];
}

// per uv vertex, the same gather over the uv-vertex-face CSR into uv_b (overwritten)
__global__ void k_tangents_uv_b(const uint32_t *faces_uv, const int32_t *uv_face_offset, const int32_t *uv_face_index,
                                int nb_uv, const double *face_b, double *uv_b) {
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= nb_uv) return;
    double acc[2] = {0, 0};
    const int k0 = uv_face_offset[u];
    for (int k = k0; k < uv_face_offset[u + 1]; k++) {
        const int f = uv_face_index[k];
        if (k > k0 && uv_face_index[k - 1] == f) continue;
        const double *o = face_b + 10 * (size_t)f;
        for (int c = 0; c < 3; c++) {
            if (faces_uv[3 * (size_t)f + c] != (uint32_t)u) continue;
            if (c == 0) {
                acc[0] += -(o[6] + o[8]);
                acc[1] += -(o[7] + o[9]);
            } else {
                acc[0] += o[6 + 2 * (c - 1)];
                acc[1] += o[7 + 2 * (c - 1)];
            }
        }
    }
    uv_b[2 * (size_t)u] = acc[0];
    uv_b[2 * (size_t)u + 1] = acc[1];
}

struct NormalMapFrame {
    double n[3], tt[3], t[3], bt[3], s, p[3];
};

// one pixel's frame and perturbed direction p = (M_x t + M_y b) + M_z n from the 13-channel G-buffer (N, X, a, T, B)
// and the map raster M
__device__ __forceinline__ NormalMapFrame normal_map_frame(const float *g, const double M[3]) {
    NormalMapFrame q;
    const double N[3] = {g[0], g[1], g[2]}, T[3] = {g[7], g[8], g[9]}, B[3] = {g[10], g[11], g[12]};
    unit_or_zero(N, q.n);
    const double tn = (T[0] * q.n[0] + T[1] * q.n[1]) + T[2] * q.n[2];
    for (int j = 0; j < 3; j++) q.tt[j] = T[j] - tn * q.n[j];
    unit_or_zero(q.tt, q.t);
    q.bt[0] = q.n[1] * q.t[2] - q.n[2] * q.t[1];
    q.bt[1] = q.n[2] * q.t[0] - q.n[0] * q.t[2];
    q.bt[2] = q.n[0] * q.t[1] - q.n[1] * q.t[0];
    q.s = ((q.bt[0] * B[0] + q.bt[1] * B[1]) + q.bt[2] * B[2]) >= 0 ? 1.0 : -1.0;
    for (int j = 0; j < 3; j++) q.p[j] = (M[0] * q.t[j] + M[1] * (q.s * q.bt[j])) + M[2] * q.n[j];
    return q;
}

__global__ void __launch_bounds__(BLOCK) k_normal_map(const float *gbuffer, const float *map, long long pixels,
                                                      float *out) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= pixels) return;
    const float *g = gbuffer + 13 * i;
    float *o = out + 7 * i;
    for (int j = 3; j < 7; j++) o[j] = g[j];
    const double a = g[6];
    double np[3] = {0, 0, 0};
    if (a != 0) {
        const double M[3] = {map[3 * i], map[3 * i + 1], map[3 * i + 2]};
        const NormalMapFrame q = normal_map_frame(g, M);
        double u[3];
        unit_or_zero(q.p, u);
        for (int j = 0; j < 3; j++) np[j] = a * u[j];
    }
    for (int j = 0; j < 3; j++) o[j] = (float)np[j];
}

__global__ void __launch_bounds__(BLOCK) k_normal_map_b(const float *gbuffer, const float *map, long long pixels,
                                                        const float *out_b, float *gbuffer_b, float *map_b) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= pixels) return;
    const float *g = gbuffer + 13 * i, *ob = out_b + 7 * i;
    float *gb = gbuffer_b + 13 * i;
    const double a = g[6];
    double N_b[3] = {0, 0, 0}, T_b[3] = {0, 0, 0}, M_b[3] = {0, 0, 0}, a_b = ob[6];
    const double np_b[3] = {ob[0], ob[1], ob[2]};
    if (a != 0) {
        const double M[3] = {map[3 * i], map[3 * i + 1], map[3 * i + 2]};
        const NormalMapFrame q = normal_map_frame(g, M);
        const double pn2 = (q.p[0] * q.p[0] + q.p[1] * q.p[1]) + q.p[2] * q.p[2];
        if (pn2 > 0) {
            double u[3], u_b[3], p_b[3];
            unit_or_zero(q.p, u);
            a_b += (np_b[0] * u[0] + np_b[1] * u[1]) + np_b[2] * u[2];
            for (int j = 0; j < 3; j++) u_b[j] = a * np_b[j];
            normalize_b(q.p, u_b, p_b);
            double b[3], t_b[3], bt_b[3], n_b[3];
            for (int j = 0; j < 3; j++) b[j] = q.s * q.bt[j];
            M_b[0] = (p_b[0] * q.t[0] + p_b[1] * q.t[1]) + p_b[2] * q.t[2];
            M_b[1] = (p_b[0] * b[0] + p_b[1] * b[1]) + p_b[2] * b[2];
            M_b[2] = (p_b[0] * q.n[0] + p_b[1] * q.n[1]) + p_b[2] * q.n[2];
            for (int j = 0; j < 3; j++) {
                t_b[j] = M[0] * p_b[j];
                bt_b[j] = q.s * (M[1] * p_b[j]);
                n_b[j] = M[2] * p_b[j];
            }
            // bt = n x t: n_b += t x bt_b, t_b += bt_b x n
            n_b[0] += q.t[1] * bt_b[2] - q.t[2] * bt_b[1];
            n_b[1] += q.t[2] * bt_b[0] - q.t[0] * bt_b[2];
            n_b[2] += q.t[0] * bt_b[1] - q.t[1] * bt_b[0];
            t_b[0] += bt_b[1] * q.n[2] - bt_b[2] * q.n[1];
            t_b[1] += bt_b[2] * q.n[0] - bt_b[0] * q.n[2];
            t_b[2] += bt_b[0] * q.n[1] - bt_b[1] * q.n[0];
            // t = tt / |tt|, tt = T - <T, n> n
            double tt_b[3];
            unit_or_zero_b(q.tt, t_b, tt_b);
            const double T[3] = {g[7], g[8], g[9]};
            const double tn = (T[0] * q.n[0] + T[1] * q.n[1]) + T[2] * q.n[2];
            const double ntt_b = (q.n[0] * tt_b[0] + q.n[1] * tt_b[1]) + q.n[2] * tt_b[2];
            for (int j = 0; j < 3; j++) {
                T_b[j] = tt_b[j] - ntt_b * q.n[j];
                n_b[j] -= tn * tt_b[j] + ntt_b * T[j];
            }
            const double N[3] = {g[0], g[1], g[2]};
            unit_or_zero_b(N, n_b, N_b);
        }
    }
    for (int j = 0; j < 3; j++) {
        gb[j] = (float)N_b[j];
        gb[3 + j] = ob[3 + j];
        gb[7 + j] = (float)T_b[j];
        gb[10 + j] = 0.0f;
        map_b[3 * i + j] = (float)M_b[j];
    }
    gb[6] = (float)a_b;
}

int check_launch() {
    CUDA_TRY(cudaGetLastError());
    return DEODR_B200_OK;
}

int check_mesh(const DeodrMeshTopology *m) {
    if (!m) return set_error(DEODR_B200_EINVAL, "mesh == NULL");
    if (m->nb_faces < 0 || m->nb_vertices < 0 || m->nb_edges < 0) return set_error(DEODR_B200_EINVAL, "negative size");
    if (m->nb_faces > 0 && !m->faces) return set_error(DEODR_B200_EINVAL, "mesh.faces == NULL");
    return DEODR_B200_OK;
}

}  // namespace

extern "C" {

int deodr_b200_project_points(const double *points, int n, const DeodrCamera *camera, double *ij, double *depths,
                              void *stream) {
    if (!camera || n < 0 || (n > 0 && (!points || !ij || !depths))) return set_error(DEODR_B200_EINVAL, "bad argument");
    if (n == 0) return DEODR_B200_OK;
    k_project<<<grid_of(n), BLOCK, 0, (cudaStream_t)stream>>>(points, n, cam_of(camera), ij, depths);
    return check_launch();
}

int deodr_b200_project_points_dev(const double *points, int n, const double *camera, int has_distortion, double *ij,
                                  double *depths, void *stream) {
    if (!camera || n < 0 || (n > 0 && (!points || !ij || !depths)))
        return set_error(DEODR_B200_EINVAL, "project_points_dev: bad argument (n >= 0 and every pointer non-NULL)");
    if (n == 0) return DEODR_B200_OK;
    k_project_dev<<<grid_of(n), BLOCK, 0, (cudaStream_t)stream>>>(points, n, camera, has_distortion != 0, ij, depths);
    return check_launch();
}

int deodr_b200_project_points_camera_b(const double *points, int n, const double *camera, int has_distortion,
                                       const float *ij_b, const double *ij_b64, const double *depths_b,
                                       double *points_b, int accumulate, double *camera_b, double *scratch,
                                       void *stream) {
    if (n < 0 || !camera || !camera_b || !scratch || (ij_b && ij_b64) || (n > 0 && !points))
        return set_error(DEODR_B200_EINVAL, "project_points_camera_b: bad argument (n >= 0; camera, camera_b, scratch "
                                            "and points non-NULL; at most one of ij_b and ij_b64)");
    cudaStream_t st = (cudaStream_t)stream;
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    const int g = (int)std::min<size_t>(CAMERA_MAX_CTAS, grid_of(n > 0 ? n : 1));
    const int distorted = has_distortion != 0;
    const int mode = !points_b ? POINTS_B_NONE : (accumulate ? POINTS_B_ACCUMULATE : POINTS_B_OVERWRITE);
#define DEODR_CAMERA_B(G, M, grad)                                                                                      \
    k_project_camera_b<G, M><<<g, NT, 0, st>>>(points, n, camera, distorted, grad, depths_b, points_b, camera_b, s)
    if (ij_b64) {
        if (mode == POINTS_B_NONE) DEODR_CAMERA_B(double, POINTS_B_NONE, ij_b64);
        else if (mode == POINTS_B_OVERWRITE) DEODR_CAMERA_B(double, POINTS_B_OVERWRITE, ij_b64);
        else DEODR_CAMERA_B(double, POINTS_B_ACCUMULATE, ij_b64);
    } else {
        if (mode == POINTS_B_NONE) DEODR_CAMERA_B(float, POINTS_B_NONE, ij_b);
        else if (mode == POINTS_B_OVERWRITE) DEODR_CAMERA_B(float, POINTS_B_OVERWRITE, ij_b);
        else DEODR_CAMERA_B(float, POINTS_B_ACCUMULATE, ij_b);
    }
#undef DEODR_CAMERA_B
    return check_launch();
}

int deodr_b200_project_points_b(const double *points, int n, const DeodrCamera *camera, const float *ij_b,
                                const double *depths_b, double *points_b, int reference_transpose, void *stream) {
    if (!camera || n < 0 || (n > 0 && (!points || !ij_b || !points_b))) return set_error(DEODR_B200_EINVAL, "bad argument");
    if (n == 0) return DEODR_B200_OK;
    k_project_b<float, true><<<grid_of(n), BLOCK, 0, (cudaStream_t)stream>>>(points, n, cam_of(camera), ij_b, depths_b,
                                                                            points_b, reference_transpose);
    return check_launch();
}

int deodr_b200_project_points_b64(const double *points, int n, const DeodrCamera *camera, const double *ij_b,
                                  const double *depths_b, double *points_b, void *stream) {
    if (!camera || n < 0 || (n > 0 && (!points || !points_b))) return set_error(DEODR_B200_EINVAL, "bad argument");
    if (n == 0) return DEODR_B200_OK;
    k_project_b<double, false><<<grid_of(n), BLOCK, 0, (cudaStream_t)stream>>>(points, n, cam_of(camera), ij_b,
                                                                              depths_b, points_b, 0);
    return check_launch();
}

static Light light_of(const double *directional, double ambient) {
    Light L;
    L.directional = directional != nullptr;
    for (int j = 0; j < 3; j++) L.d[j] = directional ? directional[j] : 0.0;
    L.ambient = ambient;
    return L;
}

int deodr_b200_vertex_luminosity(const double *normals, const double *vertex_colors, int n_vertices, int nb_colors,
                                 const double *light_directional, double ambient, float *luminosity, float *colors,
                                 void *stream) {
    if (n_vertices < 0 || nb_colors < 0 || (n_vertices > 0 && light_directional && !normals))
        return set_error(DEODR_B200_EINVAL, "bad argument");
    if (n_vertices == 0) return DEODR_B200_OK;
    k_luminosity<<<grid_of(n_vertices), BLOCK, 0, (cudaStream_t)stream>>>(normals, vertex_colors, n_vertices, nb_colors,
                                                                         light_of(light_directional, ambient),
                                                                         luminosity, colors);
    return check_launch();
}

int deodr_b200_vertex_luminosity_b(const double *normals, const double *vertex_colors, int n_vertices, int nb_colors,
                                   const double *light_directional, double ambient, const float *colors_b,
                                   const float *luminosity_b, double *normals_b, double *vertex_colors_b,
                                   double *light_b, void *stream) {
    if (n_vertices < 0 || nb_colors < 0 || (n_vertices > 0 && !normals))
        return set_error(DEODR_B200_EINVAL, "bad argument");
    if (n_vertices == 0) return DEODR_B200_OK;
    k_luminosity_b<<<grid_of(n_vertices), BLOCK, 0, (cudaStream_t)stream>>>(
        normals, vertex_colors, n_vertices, nb_colors, light_of(light_directional, ambient), colors_b, luminosity_b,
        normals_b, vertex_colors_b, light_b);
    return check_launch();
}

int deodr_b200_edge_on_silhouette(const DeodrMeshTopology *mesh, const double *ij, uint8_t *face_visible,
                                  uint8_t *edgeflags, void *stream) {
    if (int rc = check_mesh(mesh)) return rc;
    if (mesh->nb_faces == 0) return DEODR_B200_OK;
    if (!ij || !face_visible || !edgeflags || !mesh->faces_edges || !mesh->edge_face_offset || !mesh->edge_face_index)
        return set_error(DEODR_B200_EINVAL, "bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    k_face_visible<<<grid_of(mesh->nb_faces), BLOCK, 0, st>>>(*mesh, ij, face_visible);
    k_edge_flags<<<grid_of(3 * (size_t)mesh->nb_faces), BLOCK, 0, st>>>(*mesh, face_visible, edgeflags);
    return check_launch();
}

int deodr_b200_vertex_normals(const DeodrMeshTopology *mesh, const double *vertices, double *face_normals,
                              double *vertex_normals, void *stream) {
    if (int rc = check_mesh(mesh)) return rc;
    if (mesh->nb_faces == 0) return DEODR_B200_OK;
    if (!vertices || !face_normals) return set_error(DEODR_B200_EINVAL, "bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    k_face_normals<<<grid_of(mesh->nb_faces), BLOCK, 0, st>>>(*mesh, vertices, face_normals);
    if (vertex_normals) {
        if (!mesh->vertex_face_offset || !mesh->vertex_face_index) return set_error(DEODR_B200_EINVAL, "bad argument");
        k_vertex_normals<<<grid_of(mesh->nb_vertices), BLOCK, 0, st>>>(*mesh, face_normals, vertex_normals);
    }
    return check_launch();
}

int deodr_b200_vertex_normals_b(const DeodrMeshTopology *mesh, const double *vertices, const double *vertex_normals_b,
                                double *vertex_scratch, double *vertices_b, void *stream) {
    if (int rc = check_mesh(mesh)) return rc;
    if (mesh->nb_faces == 0) return DEODR_B200_OK;
    if (!vertices || !vertex_normals_b || !vertex_scratch || !vertices_b || !mesh->vertex_face_offset ||
        !mesh->vertex_face_index)
        return set_error(DEODR_B200_EINVAL, "bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    k_vertex_normals_b1<<<grid_of(mesh->nb_vertices), BLOCK, 0, st>>>(*mesh, vertices, vertex_normals_b, vertex_scratch);
    k_face_normals_b<<<grid_of(mesh->nb_faces), BLOCK, 0, st>>>(*mesh, vertices, vertex_scratch, nullptr, vertices_b);
    return check_launch();
}

int deodr_b200_cube_project(const double *vertices, int n, const double *lights, int nb_lights, int light_channels,
                            int map_size, double *cameras, double *ij, double *depths, void *stream) {
    if (n < 1 || !vertices || !lights || !cameras || !ij || !depths || !shadow_map_ok(map_size))
        return set_error(DEODR_B200_EINVAL, "cube_project: bad argument (n >= 1, every pointer non-NULL, map_size in "
                                            "[8, 4096])");
    if (!shadow_lights_ok(nb_lights, light_channels))
        return set_error(DEODR_B200_EUNSUPPORTED, "cube_project: nb_lights must be 1 to 8 and light_channels 1 to 4");
    cudaStream_t st = (cudaStream_t)stream;
    k_cube_cameras<<<1, 6 * SHADOW_MAX_LIGHTS, 0, st>>>(lights, nb_lights, 3 + light_channels, map_size, cameras);
    const long long items = 6LL * nb_lights * n;
    k_cube_project<<<(unsigned)((items + BLOCK - 1) / BLOCK), BLOCK, 0, st>>>(vertices, n, cameras, items, 0, ij,
                                                                            depths);
    return check_launch();
}

int deodr_b200_cube_project_b(const double *vertices, int n, const double *lights, int nb_lights, int light_channels,
                              int map_size, const double *cameras, const float *ij_b, const float *depths_b,
                              double *vertices_b, double *lights_b, double *scratch, void *stream) {
    if (n < 1 || !vertices || !lights || !cameras || !ij_b || !depths_b || !vertices_b || !lights_b || !scratch ||
        !shadow_map_ok(map_size))
        return set_error(DEODR_B200_EINVAL, "cube_project_b: bad argument (n >= 1, every pointer non-NULL, map_size "
                                            "in [8, 4096])");
    if (!shadow_lights_ok(nb_lights, light_channels))
        return set_error(DEODR_B200_EUNSUPPORTED, "cube_project_b: nb_lights must be 1 to 8 and light_channels 1 to 4");
    cudaStream_t st = (cudaStream_t)stream;
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    with_lights(nb_lights, [&](auto L) {
        k_cube_project_b<L><<<sum_grid(n, 3 * L), NT, 0, st>>>(vertices, n, cameras, ij_b, depths_b, vertices_b,
                                                               lights_b, 3 + light_channels, s);
    });
    return check_launch();
}

int deodr_b200_shadow_visibility(const DeodrPhongIO *io, const double *lights, int nb_lights, int light_channels,
                                 const float *maps, int map_size, double bias, double softness, float *vis,
                                 void *stream) {
    if (!shadow_io_ok(io) || !lights || !maps || !vis || !shadow_map_ok(map_size) || !shadow_band_ok(bias, softness))
        return set_error(DEODR_B200_EINVAL, "shadow_visibility: bad argument (H, W >= 1, C in [1, 32760], position and "
                                            "coverage offsets inside the G-buffer, every pointer non-NULL, map_size in "
                                            "[8, 4096], bias and softness finite and > 0)");
    if (nb_lights < 1 || nb_lights > SHADOW_MAX_LIGHTS || !(light_channels == 1 || (light_channels == io->C &&
                                                                                    io->C >= 2 && io->C <= 4)))
        return set_error(DEODR_B200_EUNSUPPORTED, "shadow_visibility: nb_lights must be 1 to 8, and light_channels 1, "
                                                  "or C from 1 to 4");
    const long long pixels = (long long)io->H * io->W;
    const int stride = io->off_albedo == -1 ? 7 : io->C + 7;
    k_shadow_visibility<<<(unsigned)((pixels + NT - 1) / NT), NT, 0, (cudaStream_t)stream>>>(
        io->channels, pixels, stride, io->off_position, io->off_coverage, lights, nb_lights, 3 + light_channels, maps,
        map_size, bias, softness, vis);
    return check_launch();
}

int deodr_b200_shadow_visibility_b(const DeodrPhongIO *io, const double *lights, int nb_lights, int light_channels,
                                   const float *maps, int map_size, double bias, double softness, const float *vis_b,
                                   float *maps_b, double *lights_b, double *scratch, void *stream) {
    if (!shadow_io_ok(io) || !io->channels_b || !lights || !maps || !vis_b || !maps_b || !lights_b || !scratch ||
        !shadow_map_ok(map_size) || !shadow_band_ok(bias, softness))
        return set_error(DEODR_B200_EINVAL, "shadow_visibility_b: bad argument (H, W >= 1, C in [1, 32760], position "
                                            "and coverage offsets inside the G-buffer, every pointer non-NULL, "
                                            "map_size in [8, 4096], bias and softness finite and > 0)");
    if (nb_lights < 1 || nb_lights > SHADOW_MAX_LIGHTS || !(light_channels == 1 || (light_channels == io->C &&
                                                                                    io->C >= 2 && io->C <= 4)))
        return set_error(DEODR_B200_EUNSUPPORTED, "shadow_visibility_b: nb_lights must be 1 to 8, and light_channels "
                                                  "1, or C from 1 to 4");
    const long long pixels = (long long)io->H * io->W;
    const int stride = io->off_albedo == -1 ? 7 : io->C + 7;
    cudaStream_t st = (cudaStream_t)stream;
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    with_lights(nb_lights, [&](auto L) {
        k_shadow_visibility_b<L><<<sum_grid(pixels, 3 * L), NT, 0, st>>>(
            io->channels, io->channels_b, pixels, stride, io->off_position, io->off_coverage, lights,
            3 + light_channels, maps, map_size, bias, softness, vis_b, maps_b, lights_b, s);
    });
    return check_launch();
}

int deodr_b200_sun_project(const double *vertices, int n, const double *light, const double *center, double radius,
                           int map_size, double *ij, double *depths, void *stream) {
    if (n < 1 || !vertices || !light || !ij || !depths || !shadow_map_ok(map_size) || !sun_window_ok(center, radius))
        return set_error(DEODR_B200_EINVAL, "sun_project: bad argument (n >= 1, every pointer non-NULL, map_size in "
                                            "[8, 4096], center finite, radius finite and > 0)");
    k_sun_project<<<(unsigned)((n + NT - 1) / NT), NT, 0, (cudaStream_t)stream>>>(
        vertices, n, light, sun_window(center, radius, map_size), ij, depths);
    return check_launch();
}

int deodr_b200_sun_project_b(const double *vertices, int n, const double *light, const double *center, double radius,
                             int map_size, const float *ij_b, const float *depths_b, double *vertices_b,
                             double *light_b, double *scratch, void *stream) {
    if (n < 1 || !vertices || !light || !ij_b || !depths_b || !vertices_b || !light_b || !scratch ||
        !shadow_map_ok(map_size) || !sun_window_ok(center, radius))
        return set_error(DEODR_B200_EINVAL, "sun_project_b: bad argument (n >= 1, every pointer non-NULL, map_size "
                                            "in [8, 4096], center finite, radius finite and > 0)");
    k_sun_project_b<<<sum_grid(n, 9), NT, 0, (cudaStream_t)stream>>>(
        vertices, n, light, sun_window(center, radius, map_size), ij_b, depths_b, vertices_b, light_b,
        reinterpret_cast<Scratch *>(scratch));
    return check_launch();
}

int deodr_b200_sun_visibility(const DeodrPhongIO *io, const double *center, double radius, const float *map,
                              int map_size, double bias, double softness, float *vis, void *stream) {
    if (!shadow_io_ok(io) || !io->params || !map || !vis || !shadow_map_ok(map_size) ||
        !shadow_band_ok(bias, softness) || !sun_window_ok(center, radius))
        return set_error(DEODR_B200_EINVAL, "sun_visibility: bad argument (H, W >= 1, C in [1, 32760], position and "
                                            "coverage offsets inside the G-buffer, every pointer non-NULL, map_size in "
                                            "[8, 4096], bias, softness and radius finite and > 0, center finite)");
    const long long pixels = (long long)io->H * io->W;
    const int stride = io->off_albedo == -1 ? 7 : io->C + 7;
    k_sun_visibility<<<(unsigned)((pixels + NT - 1) / NT), NT, 0, (cudaStream_t)stream>>>(
        io->channels, pixels, stride, io->off_position, io->off_coverage, io->params,
        sun_window(center, radius, map_size), map, bias, softness, vis);
    return check_launch();
}

int deodr_b200_sun_visibility_b(const DeodrPhongIO *io, const double *center, double radius, const float *map,
                                int map_size, double bias, double softness, const float *vis_b, float *map_b,
                                double *light_b, double *scratch, void *stream) {
    if (!shadow_io_ok(io) || !io->params || !io->channels_b || !map || !vis_b || !map_b || !light_b || !scratch ||
        !shadow_map_ok(map_size) || !shadow_band_ok(bias, softness) || !sun_window_ok(center, radius))
        return set_error(DEODR_B200_EINVAL, "sun_visibility_b: bad argument (H, W >= 1, C in [1, 32760], position "
                                            "and coverage offsets inside the G-buffer, every pointer non-NULL, "
                                            "map_size in [8, 4096], bias, softness and radius finite and > 0, center "
                                            "finite)");
    const long long pixels = (long long)io->H * io->W;
    const int stride = io->off_albedo == -1 ? 7 : io->C + 7;
    k_sun_visibility_b<<<sum_grid(pixels, 9), NT, 0, (cudaStream_t)stream>>>(
        io->channels, io->channels_b, pixels, stride, io->off_position, io->off_coverage, io->params,
        sun_window(center, radius, map_size), map, bias, softness, vis_b, map_b, light_b,
        reinterpret_cast<Scratch *>(scratch));
    return check_launch();
}

int deodr_b200_vertex_tangents(const DeodrMeshTopology *mesh, const double *vertices, const uint32_t *faces_uv,
                               const double *uv, int nb_uv, double *face_frames, double *frames, void *stream) {
    if (!mesh || !mesh->faces || !mesh->vertex_face_offset || !mesh->vertex_face_index || mesh->nb_faces < 1 ||
        mesh->nb_vertices < 1 || nb_uv < 1 || !vertices || !faces_uv || !uv || !face_frames || !frames)
        return set_error(DEODR_B200_EINVAL, "vertex_tangents: bad argument (T, V and nb_uv >= 1, every pointer "
                                            "non-NULL, the vertex-face CSR given)");
    cudaStream_t st = (cudaStream_t)stream;
    k_face_tangents<<<grid_of(mesh->nb_faces), BLOCK, 0, st>>>(*mesh, vertices, faces_uv, uv, face_frames);
    k_vertex_tangents<<<grid_of(mesh->nb_vertices), BLOCK, 0, st>>>(*mesh, face_frames, frames);
    return check_launch();
}

int deodr_b200_vertex_tangents_b(const DeodrMeshTopology *mesh, const double *vertices, const uint32_t *faces_uv,
                                 const double *uv, int nb_uv, const int32_t *uv_face_offset,
                                 const int32_t *uv_face_index, const double *frames_b, double *scratch,
                                 double *vertices_b, double *uv_b, void *stream) {
    if (!mesh || !mesh->faces || !mesh->vertex_face_offset || !mesh->vertex_face_index || mesh->nb_faces < 1 ||
        mesh->nb_vertices < 1 || nb_uv < 1 || !vertices || !faces_uv || !uv || !uv_face_offset || !uv_face_index ||
        !frames_b || !scratch || !vertices_b || !uv_b)
        return set_error(DEODR_B200_EINVAL, "vertex_tangents_b: bad argument (T, V and nb_uv >= 1, every pointer "
                                            "non-NULL, the vertex-face CSR given)");
    cudaStream_t st = (cudaStream_t)stream;
    double *sum_b = scratch, *face_b = scratch + 6 * (size_t)mesh->nb_vertices;
    k_vertex_tangents_b1<<<grid_of(mesh->nb_vertices), BLOCK, 0, st>>>(*mesh, vertices, faces_uv, uv, frames_b, sum_b);
    k_face_tangents_b<<<grid_of(mesh->nb_faces), BLOCK, 0, st>>>(*mesh, vertices, faces_uv, uv, sum_b, face_b);
    k_tangents_vertices_b<<<grid_of(mesh->nb_vertices), BLOCK, 0, st>>>(*mesh, face_b, vertices_b);
    k_tangents_uv_b<<<grid_of(nb_uv), BLOCK, 0, st>>>(faces_uv, uv_face_offset, uv_face_index, nb_uv, face_b, uv_b);
    return check_launch();
}

int deodr_b200_normal_map(const float *gbuffer, const float *map, int H, int W, float *out, void *stream) {
    if (!gbuffer || !map || !out || H < 1 || W < 1)
        return set_error(DEODR_B200_EINVAL, "normal_map: bad argument (H, W >= 1, every pointer non-NULL)");
    const long long pixels = (long long)H * W;
    k_normal_map<<<(unsigned)((pixels + BLOCK - 1) / BLOCK), BLOCK, 0, (cudaStream_t)stream>>>(gbuffer, map, pixels,
                                                                                               out);
    return check_launch();
}

int deodr_b200_normal_map_b(const float *gbuffer, const float *map, int H, int W, const float *out_b,
                            float *gbuffer_b, float *map_b, void *stream) {
    if (!gbuffer || !map || !out_b || !gbuffer_b || !map_b || H < 1 || W < 1)
        return set_error(DEODR_B200_EINVAL, "normal_map_b: bad argument (H, W >= 1, every pointer non-NULL)");
    const long long pixels = (long long)H * W;
    k_normal_map_b<<<(unsigned)((pixels + BLOCK - 1) / BLOCK), BLOCK, 0, (cudaStream_t)stream>>>(
        gbuffer, map, pixels, out_b, gbuffer_b, map_b);
    return check_launch();
}

}  // extern "C"
