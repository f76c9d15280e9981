// deodr_b200: the maths of a mesh-fitting step around the render (deodr/mesh_fitter.py: MeshDepthFitter,
// MeshRGBFitterWithPose), on fp64 device buffers:
//
//   rigid pose         v <- v - mean(v);  v' = qrot(q / |q|, v) + t                          (+ adjoint)
//   poses of F frames  v <- v - mean(v);  v'_f = qrot(q_f / |q_f|, v) + t_f                 (+ adjoint summed over f)
//   Laplacian rigidity grad = cregu L (L (v - v_ref)),  energy = 1/2 <v - v_ref, grad>,  L = D - A
//   depth comparison   d = clip(r, 0, max_depth),  energy = sum (d - o)^2,  depth_b = 2 (d - o) (0 outside the range)
//   uniform colour     colours = color * (max(0, -<n, light>) + ambient)                    (+ adjoint)
//   Phong shading      image = A (ambient + diff) + spec + (1 - a) bg per pixel of a G-buffer   (+ adjoint)
//   SH environment     + sh_c(n) beside ambient + diff, per vertex or per pixel                 (+ adjoint)
//   textured Phong     the same with A read from an albedo raster of its own                    (+ adjoint)
//   point lights       + P_c(n, x) (and + Q_c per pixel), per vertex or per pixel               (+ adjoint)
//   shadowed lights    per pixel, light j's terms times a visibility V_j (csrc/scene_ops.cu)    (+ adjoint)
//   update             heavy-ball steps on the vertices and the few-scalar parameters
//
// with qrot(q, v) = v + 2 (w (u x v) + u x (u x v)), u = q_xyz, w = q_w (quaternions stored x, y, z, w).
//
// Every reported sum is reproducible bit for bit: grid_sum (reduce.cuh) adds fixed-order per-CTA partials in CTA
// order.  No fp64 atomics.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <type_traits>

#include "../../include/deodr_b200.h"
#include "reduce.cuh"
#include "workspace.h"

namespace {

inline int grid_of(long long n) { return (int)std::max<long long>(1, (n + NT - 1) / NT); }
inline int reduce_grid(long long n) { return (int)std::min<long long>(MAX_CTAS, grid_of(n)); }

struct Quat {
    double x, y, z, w;
};

__device__ __forceinline__ Quat load_unit(const double *q) {
    const double n = sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]);
    return {q[0] / n, q[1] / n, q[2] / n, q[3] / n};
}

__device__ __forceinline__ void cross(const double a[3], const double b[3], double c[3]) {
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

__device__ __forceinline__ double dot(const double a[3], const double b[3]) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

// ---- rigid pose ------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(NT) k_mean(const double *v, int n, Scratch *s) {
    __shared__ double tot[3];
    double acc[3] = {0, 0, 0};
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT)
        for (int j = 0; j < 3; j++) acc[j] += v[3 * i + j];
    if (grid_sum<3>(acc, s, tot) && threadIdx.x < 3) s->result[threadIdx.x] = tot[threadIdx.x] / n;
}

// v <- v - mean (in place); v' = qrot(q / |q|, v) + t
__global__ void __launch_bounds__(NT) k_pose(double *v, int n, const double *q, const double *t, const Scratch *s,
                                             double *out) {
    const long long i = (long long)blockIdx.x * NT + threadIdx.x;
    if (i >= n) return;
    const Quat h = load_unit(q);
    const double u[3] = {h.x, h.y, h.z};
    double p[3];
    for (int j = 0; j < 3; j++) {
        p[j] = v[3 * i + j] - s->result[j];
        v[3 * i + j] = p[j];
    }
    double c[3], uc[3];
    cross(u, p, c);
    cross(u, c, uc);
    for (int j = 0; j < 3; j++) out[3 * i + j] = (p[j] + 2 * (h.w * c[j] + uc[j])) + t[j];
}

// From g = v'_b, per vertex: t_b += g;  w_b += 2 g.(u x v);  u_b += 2 (w (v x g) + g (u.v) + v (u.g) - 2 u (v.g)).
// The last CTA writes t_b and q_b = (qh_b - qh (qh . qh_b)) / |q|, the adjoint of qh = q / |q|.
__global__ void __launch_bounds__(NT) k_pose_b(const double *v, int n, const double *q, const double *g_all,
                                               double *q_b, double *t_b, Scratch *s) {
    __shared__ double tot[7];
    const Quat h = load_unit(q);
    const double u[3] = {h.x, h.y, h.z};
    double acc[7] = {0, 0, 0, 0, 0, 0, 0};  // t_b[3], u_b[3], w_b
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
        const double p[3] = {v[3 * i], v[3 * i + 1], v[3 * i + 2]};
        const double g[3] = {g_all[3 * i], g_all[3 * i + 1], g_all[3 * i + 2]};
        double c[3], pg[3];
        cross(u, p, c);
        cross(p, g, pg);
        const double up = dot(u, p), ug = dot(u, g), pgd = dot(p, g);
        for (int j = 0; j < 3; j++) {
            acc[j] += g[j];
            acc[3 + j] += 2 * (((h.w * pg[j] + g[j] * up) + p[j] * ug) - 2 * u[j] * pgd);
        }
        acc[6] += 2 * dot(g, c);
    }
    if (grid_sum<7>(acc, s, tot) && threadIdx.x == 0) {
        const double qh_b[4] = {tot[3], tot[4], tot[5], tot[6]};
        const double qh[4] = {h.x, h.y, h.z, h.w};
        const double norm = sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]);
        const double proj = ((qh[0] * qh_b[0] + qh[1] * qh_b[1]) + qh[2] * qh_b[2]) + qh[3] * qh_b[3];
        for (int j = 0; j < 4; j++) q_b[j] = (qh_b[j] - qh[j] * proj) / norm;
        for (int j = 0; j < 3; j++) t_b[j] = tot[j];
    }
}

// v_b = Q^T (g - t_b / n), with Q^T g = g + 2 w (g x u) + 2 (u (u.g) - g |u|^2) the adjoint of qrot in v: the centred
// adjoint v_b - mean(v_b), since the mean of Q^T g over the vertices is Q^T t_b / n.
__global__ void __launch_bounds__(NT) k_pose_b_vertices(int n, const double *q, const double *g_all, const double *t_b,
                                                        double *v_b) {
    const long long i = (long long)blockIdx.x * NT + threadIdx.x;
    if (i >= n) return;
    const Quat h = load_unit(q);
    const double u[3] = {h.x, h.y, h.z};
    double g[3];
    for (int j = 0; j < 3; j++) g[j] = g_all[3 * i + j] - t_b[j] / n;
    double gu[3];
    cross(g, u, gu);
    const double ug = dot(u, g), uu = dot(u, u);
    for (int j = 0; j < 3; j++) v_b[3 * i + j] = g[j] + 2 * (h.w * gu[j]) + 2 * (u[j] * ug - g[j] * uu);
}

// ---- rigid poses of several frames (MeshRGBFitterWithPoseMultiFrame) ----------------------------------------------

constexpr int POSE_SUMS = 7;                                      // t_b[3], u_b[3], w_b per frame
constexpr int MAX_FRAMES = MAX_K * MAX_CTAS / POSE_SUMS;          // one partial per (frame, sum) at least
static_assert(MAX_FRAMES == 2340, "the limit stated in deodr_b200.h and in the error message");

// v <- v - mean (in place); transformed[f] = qrot(q_f / |q_f|, v) + t_f for every frame.  One thread per vertex walks
// the frames: the centred vertex is then written by the only thread that reads it (a CTA per (vertex block, frame)
// would read vertices that the frame-0 CTAs are centring).  Per frame, the arithmetic of k_pose.
__global__ void __launch_bounds__(NT) k_pose_frames(double *v, int n, const double *q, const double *t, int F,
                                                    const Scratch *s, double *out) {
    const long long i = (long long)blockIdx.x * NT + threadIdx.x;
    if (i >= n) return;
    double p[3];
    for (int j = 0; j < 3; j++) {
        p[j] = v[3 * i + j] - s->result[j];
        v[3 * i + j] = p[j];
    }
    for (int f = 0; f < F; f++) {
        const Quat h = load_unit(q + 4 * f);
        const double u[3] = {h.x, h.y, h.z};
        double c[3], uc[3];
        cross(u, p, c);
        cross(u, c, uc);
        double *o = out + 3 * ((long long)f * n + i);
        for (int j = 0; j < 3; j++) o[j] = (p[j] + 2 * (h.w * c[j] + uc[j])) + t[3 * f + j];
    }
}

// The per-frame sums of k_pose_b over a grid of (CTAs per frame) x (frames): CTA (x, f) sums its vertices into the
// partials [f][k][x]; the last CTA to finish adds every (f, k) over x in CTA order (the order of grid_sum), writes
// t_b[f] and q_b[f] scaled by `scale`, and *energy = scale * sum_f losses[f] (frames in order) when energy is non-NULL.
__global__ void __launch_bounds__(NT) k_pose_frames_b(const double *v, int n, const double *q, const double *g_all,
                                                      double scale, const double *losses, double *energy, double *q_b,
                                                      double *t_b, Scratch *s) {
    __shared__ double warp_sums[POSE_SUMS][NT / 32];
    __shared__ bool last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int f = blockIdx.y, G = gridDim.x, F = gridDim.y;
    const Quat h = load_unit(q + 4 * f);
    const double u[3] = {h.x, h.y, h.z};
    const double *gf = g_all + 3 * (long long)f * n;
    double acc[POSE_SUMS] = {0, 0, 0, 0, 0, 0, 0};
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < n; i += (long long)G * NT) {
        const double p[3] = {v[3 * i], v[3 * i + 1], v[3 * i + 2]};
        const double g[3] = {gf[3 * i], gf[3 * i + 1], gf[3 * i + 2]};
        double c[3], pg[3];
        cross(u, p, c);
        cross(p, g, pg);
        const double up = dot(u, p), ug = dot(u, g), pgd = dot(p, g);
        for (int j = 0; j < 3; j++) {
            acc[j] += g[j];
            acc[3 + j] += 2 * (((h.w * pg[j] + g[j] * up) + p[j] * ug) - 2 * u[j] * pgd);
        }
        acc[6] += 2 * dot(g, c);
    }
#pragma unroll
    for (int k = 0; k < POSE_SUMS; k++) {
        double x = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
        if (lane == 0) warp_sums[k][warp] = x;
    }
    __syncthreads();
    if (threadIdx.x < POSE_SUMS) {
        double t = 0;
        for (int w = 0; w < NT / 32; w++) t += warp_sums[threadIdx.x][w];
        s->partials[((long long)f * POSE_SUMS + threadIdx.x) * G + blockIdx.x] = t;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        last = atomicAdd(&s->done, 1u) == (unsigned)(G * F) - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    // one warp per (frame, sum); the quaternion sums go to q_b first and are projected below
    for (int m = warp; m < F * POSE_SUMS; m += NT / 32) {
        double x = 0;
        for (int i = lane; i < G; i += 32) x += __ldcg(s->partials + (long long)m * G + i);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
        if (lane == 0) {
            const int fm = m / POSE_SUMS, k = m % POSE_SUMS;
            if (k < 3)
                t_b[3 * fm + k] = x * scale;
            else
                q_b[4 * fm + k - 3] = x * scale;
        }
    }
    __syncthreads();
    for (int fm = threadIdx.x; fm < F; fm += NT) {
        const double *qf = q + 4 * fm;
        const Quat hf = load_unit(qf);
        const double qh[4] = {hf.x, hf.y, hf.z, hf.w};
        double *qb = q_b + 4 * fm;
        const double qh_b[4] = {qb[0], qb[1], qb[2], qb[3]};
        const double norm = sqrt(((qf[0] * qf[0] + qf[1] * qf[1]) + qf[2] * qf[2]) + qf[3] * qf[3]);
        const double proj = ((qh[0] * qh_b[0] + qh[1] * qh_b[1]) + qh[2] * qh_b[2]) + qh[3] * qh_b[3];
        for (int j = 0; j < 4; j++) qb[j] = (qh_b[j] - qh[j] * proj) / norm;
    }
    if (threadIdx.x == 0) {
        if (energy) {
            double e = 0;
            for (int fm = 0; fm < F; fm++) e += losses[fm];
            *energy = scale * e;
        }
        s->done = 0;
    }
}

// v_b = sum_f Q_f^T (scale g_f - t_b_f / n) (frames in order): the centred adjoint, as k_pose_b_vertices, summed over
// the frames; without `center`, v_b = sum_f Q_f^T (scale g_f).
__global__ void __launch_bounds__(NT) k_pose_frames_b_vertices(int n, const double *q, const double *g_all, int F,
                                                               double scale, int center, const double *t_b,
                                                               double *v_b) {
    const long long i = (long long)blockIdx.x * NT + threadIdx.x;
    if (i >= n) return;
    double acc[3] = {0, 0, 0};
    for (int f = 0; f < F; f++) {
        const Quat h = load_unit(q + 4 * f);
        const double u[3] = {h.x, h.y, h.z};
        const double *gf = g_all + 3 * ((long long)f * n + i);
        double g[3];
        for (int j = 0; j < 3; j++) g[j] = center ? scale * gf[j] - t_b[3 * f + j] / n : scale * gf[j];
        double gu[3];
        cross(g, u, gu);
        const double ug = dot(u, g), uu = dot(u, u);
        for (int j = 0; j < 3; j++) acc[j] += g[j] + 2 * (h.w * gu[j]) + 2 * (u[j] * ug - g[j] * uu);
    }
    for (int j = 0; j < 3; j++) v_b[3 * i + j] = acc[j];
}

// ---- Laplacian rigidity -----------------------------------------------------------------------------------------

// y = L x for x = v - v_ref (first pass) or x = y (second): (L x)_i = deg_i x_i - sum_{j ~ i} x_j
__global__ void __launch_bounds__(NT) k_laplacian1(const int *off, const int *nbr, int n, const double *v,
                                                   const double *v_ref, double *y) {
    const long long i = (long long)blockIdx.x * NT + threadIdx.x;
    if (i >= n) return;
    const int b = off[i], e = off[i + 1];
    double s[3] = {0, 0, 0};
    for (int k = b; k < e; k++) {
        const long long j = nbr[k];
        for (int c = 0; c < 3; c++) s[c] += v[3 * j + c] - v_ref[3 * j + c];
    }
    for (int c = 0; c < 3; c++) y[3 * i + c] = (e - b) * (v[3 * i + c] - v_ref[3 * i + c]) - s[c];
}

__global__ void __launch_bounds__(NT) k_laplacian2(const int *off, const int *nbr, int n, const double *v,
                                                   const double *v_ref, const double *y, double cregu, double *grad,
                                                   double *energy, Scratch *s) {
    __shared__ double tot[1];
    double acc[1] = {0};
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
        const int b = off[i], e = off[i + 1];
        double t[3] = {0, 0, 0};
        for (int k = b; k < e; k++) {
            const long long j = nbr[k];
            for (int c = 0; c < 3; c++) t[c] += y[3 * j + c];
        }
        for (int c = 0; c < 3; c++) {
            const double g = cregu * ((e - b) * y[3 * i + c] - t[c]);
            grad[3 * i + c] = g;
            acc[0] += (v[3 * i + c] - v_ref[3 * i + c]) * g;
        }
    }
    if (grid_sum<1>(acc, s, tot) && threadIdx.x == 0) *energy = 0.5 * tot[0];
}

// ---- depth comparison -------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(NT) k_depth_compare(const float *r, const double *o, long long pixels, double max_depth,
                                                      double *depth, double *diff, float *depth_b, double *energy,
                                                      Scratch *s) {
    __shared__ double tot[1];
    double acc[1] = {0};
    for (long long p = (long long)blockIdx.x * NT + threadIdx.x; p < pixels; p += (long long)gridDim.x * NT) {
        const double x = r[p];
        const double d = x < 0 ? 0.0 : (x > max_depth ? max_depth : x);  // np.clip: NaN stays NaN
        const double e = d - o[p];
        const double sq = e * e;
        acc[0] += sq;
        if (depth) depth[p] = d;
        if (diff) diff[p] = sq;
        depth_b[p] = (x < 0 || x > max_depth) ? 0.0f : (float)(2 * e);
    }
    if (grid_sum<1>(acc, s, tot) && threadIdx.x == 0) *energy = tot[0];
}

// ---- uniform colour under a device-resident light ------------------------------------------------------------------

// max(0, -s) with NaN propagating like np.maximum
__device__ __forceinline__ double directional_of(double s) { return s >= 0.0 ? 0.0 : -s; }

__global__ void __launch_bounds__(NT) k_uniform_luminosity(const double *normals, int n, const double *color, int C,
                                                           const double *light, float *colors) {
    const long long v = (long long)blockIdx.x * NT + threadIdx.x;
    if (v >= n) return;
    const double *nv = normals + 3 * v;
    const double l = directional_of((nv[0] * light[0] + nv[1] * light[1]) + nv[2] * light[2]) + light[3];
    for (int c = 0; c < C; c++) colors[v * C + c] = (float)(color[c] * l);
}

// lum_b = <color, colors_b>;  color_b += colors_b * lum;  gate = lum_b where the directional term is > 0;
// normals_b = -gate * light;  light_b = (-sum gate * n, sum lum_b)
template <int C>
__global__ void __launch_bounds__(NT) k_uniform_luminosity_b(const double *normals, int n, const double *color,
                                                             const double *light, const float *colors_b,
                                                             double *normals_b, double *color_b, double *light_b,
                                                             Scratch *s) {
    __shared__ double tot[4 + C];
    double acc[4 + C];
#pragma unroll
    for (int k = 0; k < 4 + C; k++) acc[k] = 0;
    for (long long v = (long long)blockIdx.x * NT + threadIdx.x; v < n; v += (long long)gridDim.x * NT) {
        const double *nv = normals + 3 * v;
        const double dir = directional_of((nv[0] * light[0] + nv[1] * light[1]) + nv[2] * light[2]);
        const double l = dir + light[3];
        double lb = 0;
#pragma unroll
        for (int c = 0; c < C; c++) {
            const double cb = colors_b[v * C + c];
            lb += color[c] * cb;
            acc[4 + c] += cb * l;
        }
        const double gate = dir > 0 ? lb : 0.0;
        for (int j = 0; j < 3; j++) {
            acc[j] += -gate * nv[j];
            if (normals_b) normals_b[3 * v + j] = -gate * light[j];
        }
        acc[3] += lb;
    }
    if (grid_sum<4 + C>(acc, s, tot) && threadIdx.x == 0) {
        for (int k = 0; k < 4; k++) light_b[k] = tot[k];
        for (int c = 0; c < C; c++) color_b[c] = tot[4 + c];
    }
}

// ---- per-vertex colours under a device-resident light (the autograd path of Scene3D) ------------------------------

// colors [n,C] fp64 = vertex_colors * (max(0, -<n, light_xyz>) + ambient), the directional term only when `directional`
__global__ void __launch_bounds__(NT) k_lit_vertex_colors(const double *normals, const double *vcol, int n, int C,
                                                          const double *light, int directional, double *colors) {
    const long long v = (long long)blockIdx.x * NT + threadIdx.x;
    if (v >= n) return;
    const double *nv = normals + 3 * v;
    const double dir = directional ? directional_of((nv[0] * light[0] + nv[1] * light[1]) + nv[2] * light[2]) : 0.0;
    const double l = dir + light[3];
    for (int c = 0; c < C; c++) colors[v * C + c] = vcol[v * C + c] * l;
}

// lum_b = <vertex_colors, colors_b>;  vertex_colors_b = colors_b * lum;  gate = lum_b where the directional term is
// > 0;  normals_b = -gate * light;  light_b = (-sum gate * n, sum lum_b), summed with grid_sum (fixed order)
template <typename G>
__global__ void __launch_bounds__(NT) k_lit_vertex_colors_b(const double *normals, const double *vcol, int n, int C,
                                                            const double *light, int directional, const G *colors_b,
                                                            double *normals_b, double *vcol_b, double *light_b,
                                                            Scratch *s) {
    __shared__ double tot[4];
    double acc[4] = {0, 0, 0, 0};
    for (long long v = (long long)blockIdx.x * NT + threadIdx.x; v < n; v += (long long)gridDim.x * NT) {
        const double *nv = normals + 3 * v;
        const double dir = directional ? directional_of((nv[0] * light[0] + nv[1] * light[1]) + nv[2] * light[2]) : 0.0;
        const double l = dir + light[3];
        double lb = 0;
        for (int c = 0; c < C; c++) {
            const double cb = (double)colors_b[v * C + c];
            lb += vcol[v * C + c] * cb;
            vcol_b[v * C + c] = cb * l;
        }
        const double gate = (directional && dir > 0) ? lb : 0.0;
        for (int j = 0; j < 3; j++) {
            acc[j] += -gate * nv[j];
            normals_b[3 * v + j] = -gate * light[j];
        }
        acc[3] += lb;
    }
    if (grid_sum<4>(acc, s, tot) && threadIdx.x == 0)
        for (int k = 0; k < 4; k++) light_b[k] = tot[k];
}

// ---- second-order spherical-harmonics environments (the model of include/deodr_b200.h) ----------------------------

constexpr double SH_Y0 = 0.28209479177387814;  // 1 / (2 sqrt(pi))
constexpr double SH_Y1 = 0.48860251190291992;  // sqrt(3 / (4 pi))
constexpr double SH_Y4 = 1.0925484305920792;   // sqrt(15 / (4 pi))
constexpr double SH_Y6 = 0.31539156525252005;  // sqrt(5 / (16 pi))
constexpr double SH_Y8 = 0.54627421529603959;  // sqrt(15 / (16 pi))

// the nine real basis functions of bands 0 to 2 at n, without the Condon-Shortley phase
__device__ __forceinline__ void sh_basis(const double n[3], double Y[9]) {
    const double x = n[0], y = n[1], z = n[2];
    Y[0] = SH_Y0;
    Y[1] = SH_Y1 * y;
    Y[2] = SH_Y1 * z;
    Y[3] = SH_Y1 * x;
    Y[4] = SH_Y4 * (x * y);
    Y[5] = SH_Y4 * (y * z);
    Y[6] = SH_Y6 * (3 * (z * z) - 1);
    Y[7] = SH_Y4 * (x * z);
    Y[8] = SH_Y8 * (x * x - y * y);
}

// sh_s(n) = sum_k sh[k, s] Y_k, k = 0..8 in order; sh is [9, S]
template <int S>
__device__ __forceinline__ double sh_value(const double *sh, int s, const double Y[9]) {
    double e = 0;
#pragma unroll
    for (int k = 0; k < 9; k++) e += sh[k * S + s] * Y[k];
    return e;
}

// n_b += sum_k w_k grad Y_k(n): w_k = sum_c g_c sh[k, c] folds the channels into one set of coefficients
__device__ __forceinline__ void sh_grad_add(const double n[3], const double w[9], double n_b[3]) {
    const double x = n[0], y = n[1], z = n[2];
    n_b[0] += (SH_Y1 * w[3] + SH_Y4 * (y * w[4] + z * w[7])) + 2 * SH_Y8 * (x * w[8]);
    n_b[1] += (SH_Y1 * w[1] + SH_Y4 * (x * w[4] + z * w[5])) - 2 * SH_Y8 * (y * w[8]);
    n_b[2] += (SH_Y1 * w[2] + SH_Y4 * (y * w[5] + x * w[7])) + 6 * SH_Y6 * (z * w[6]);
}

// colors [n,C] fp64 = vertex_colors * ((max(0, -<n, light_xyz>) + ambient) + sh_c(n)), or, without vertex colours,
// the luminosity [n] (S = 1).  S = 1: one grey environment for every channel; S = C: one per channel.
template <int S>
__global__ void __launch_bounds__(NT) k_sh_lit_vertex_colors(const double *normals, const double *vcol, int n, int C,
                                                             const double *light, int directional, const double *sh,
                                                             double *colors) {
    const long long v = (long long)blockIdx.x * NT + threadIdx.x;
    if (v >= n) return;
    const double *nv = normals + 3 * v;
    const double dir = directional ? directional_of((nv[0] * light[0] + nv[1] * light[1]) + nv[2] * light[2]) : 0.0;
    const double l = dir + light[3];
    const double nn[3] = {nv[0], nv[1], nv[2]};
    double Y[9];
    sh_basis(nn, Y);
    if (!vcol) {
        colors[v] = l + sh_value<1>(sh, 0, Y);
        return;
    }
    if (S == 1) {
        const double lum = l + sh_value<1>(sh, 0, Y);
        for (int c = 0; c < C; c++) colors[v * C + c] = vcol[v * C + c] * lum;
    } else {
#pragma unroll
        for (int c = 0; c < S; c++) colors[v * S + c] = vcol[v * S + c] * (l + sh_value<S>(sh, c, Y));
    }
}

// The adjoint of k_sh_lit_vertex_colors from colors_b ([n,C], or the luminosity's [n] without vertex colours):
// g_c = colors_b * vertex_colors (colors_b alone for the luminosity);  vertex_colors_b = colors_b * (lum + sh_c);
// normals_b = -gate * light + sum_c g_c grad sh_c;  light_b = (-sum gate * n, sum_c g_c);  sh_b[k, s] = sum g_s Y_k
// (S = 1: g summed over the channels).  light_b and sh_b are summed with grid_sum (fixed order).
template <typename G, int S>
__global__ void __launch_bounds__(NT) k_sh_lit_vertex_colors_b(const double *normals, const double *vcol, int n, int C,
                                                               const double *light, int directional, const double *sh,
                                                               const G *colors_b, double *normals_b, double *vcol_b,
                                                               double *light_b, double *sh_b, Scratch *s) {
    constexpr int K = 4 + 9 * S;
    __shared__ double tot[K];
    double acc[K];
#pragma unroll
    for (int k = 0; k < K; k++) acc[k] = 0;
    for (long long v = (long long)blockIdx.x * NT + threadIdx.x; v < n; v += (long long)gridDim.x * NT) {
        const double *nv = normals + 3 * v;
        const double nn[3] = {nv[0], nv[1], nv[2]};
        const double dir = directional ? directional_of((nn[0] * light[0] + nn[1] * light[1]) + nn[2] * light[2]) : 0.0;
        const double l = dir + light[3];
        double Y[9], w[9], g[S];
        sh_basis(nn, Y);
        double lb = 0;
        if (!vcol) {
            lb = (double)colors_b[v];
            g[0] = lb;
        } else if (S == 1) {
            const double lum = l + sh_value<1>(sh, 0, Y);
            for (int c = 0; c < C; c++) {
                const double cb = (double)colors_b[v * C + c];
                lb += vcol[v * C + c] * cb;
                vcol_b[v * C + c] = cb * lum;
            }
            g[0] = lb;
        } else {
#pragma unroll
            for (int c = 0; c < S; c++) {
                const double cb = (double)colors_b[v * S + c];
                g[c] = vcol[v * S + c] * cb;
                lb += g[c];
                vcol_b[v * S + c] = cb * (l + sh_value<S>(sh, c, Y));
            }
        }
#pragma unroll
        for (int k = 0; k < 9; k++) {
            w[k] = 0;
#pragma unroll
            for (int c = 0; c < S; c++) {
                w[k] += g[c] * sh[k * S + c];
                acc[4 + k * S + c] += g[c] * Y[k];
            }
        }
        const double gate = (directional && dir > 0) ? lb : 0.0;
        double n_b[3];
        for (int j = 0; j < 3; j++) {
            acc[j] += -gate * nn[j];
            n_b[j] = -gate * light[j];
        }
        sh_grad_add(nn, w, n_b);
        for (int j = 0; j < 3; j++) normals_b[3 * v + j] = n_b[j];
        acc[3] += lb;
    }
    if (grid_sum<K>(acc, s, tot))
        for (int k = threadIdx.x; k < K; k += NT) (k < 4 ? light_b[k] : sh_b[k - 4]) = tot[k];
}

// (u_b - u <u, u_b>) / |w|, the adjoint of u = w / |w|, added to w_b
__device__ __forceinline__ void normalize_b(const double u[3], const double u_b[3], double norm, double w_b[3]) {
    const double proj = dot(u, u_b);
    for (int j = 0; j < 3; j++) w_b[j] += (u_b[j] - u[j] * proj) / norm;
}

// ---- point lights (the model of include/deodr_b200.h) -------------------------------------------------------------

constexpr int MAX_LIGHTS = 8;

// One point light at p seen from a surface point x with unit normal n: d = p - x, r = |d|, w = d / r,
// diff = max(0, <n, w>) / r^2 and, `specular`, spec = (a ks) max(0, <n, h>)^e / r^2 with h = normalize(w + v) (h = 0
// when w + v = 0).  Every field but r is 0 when r = 0 (or NaN): the term and its derivatives vanish there.  The gates
// read `> 0`, so a NaN normal gives a zero term rather than propagating.
struct PointTerm {
    double r, r2, w[3], cos, diff, hn, h[3], s, p, spec;
};

__device__ __forceinline__ void point_term(const double *pl, const double x[3], const double n[3], bool specular,
                                           const double v[3], double aks, double e, PointTerm &t) {
    double d[3];
    for (int j = 0; j < 3; j++) d[j] = pl[j] - x[j];
    t.r2 = dot(d, d);
    t.r = sqrt(t.r2);
    t.cos = t.diff = t.hn = t.s = t.p = t.spec = 0.0;
    if (!(t.r > 0)) return;
    for (int j = 0; j < 3; j++) t.w[j] = d[j] / t.r;
    t.cos = dot(n, t.w);
    if (t.cos > 0) t.diff = t.cos / t.r2;
    if (!specular) return;
    double hh[3];
    for (int j = 0; j < 3; j++) hh[j] = t.w[j] + v[j];
    t.hn = sqrt(dot(hh, hh));
    for (int j = 0; j < 3; j++) t.h[j] = t.hn == 0.0 ? 0.0 : hh[j] / t.hn;
    const double s = dot(n, t.h);
    if (s > 0) {
        t.s = s;
        t.p = pow(s, e);
        t.spec = (aks * t.p) / t.r2;
    }
}

// The adjoint of one term from alpha = the gradient of diff and beta = that of spec: adds to n_b, d_b (the light
// position's gradient; x receives -d_b) and v_b; q = beta p / r^2 (a_b += q ks, ks_b += q a) and e_b are added to.
__device__ __forceinline__ void point_term_b(const PointTerm &t, const double n[3], double alpha, double beta,
                                             double aks, double e, double n_b[3], double d_b[3], double v_b[3],
                                             double &q, double &e_b) {
    if (!(t.r > 0)) return;
    if (t.diff > 0) {  // diff = <n, d> / r^3
        const double r3 = t.r2 * t.r;
        for (int j = 0; j < 3; j++) {
            n_b[j] += alpha * t.w[j] / t.r2;
            d_b[j] += alpha * (n[j] - 3 * t.cos * t.w[j]) / r3;
        }
    }
    if (t.s > 0) {
        q += beta * t.p / t.r2;
        e_b += beta * (aks * t.p) * log(t.s) / t.r2;
        const double s_b = beta * aks * e * pow(t.s, e - 1) / t.r2;
        const double r_b = -2 * beta * t.spec / t.r;
        double h_b[3], hh_b[3] = {0, 0, 0};
        for (int j = 0; j < 3; j++) {
            d_b[j] += r_b * t.w[j];
            n_b[j] += s_b * t.h[j];
            h_b[j] = s_b * n[j];
        }
        if (t.hn != 0.0) {
            normalize_b(t.h, h_b, t.hn, hh_b);  // hh = w + v
            for (int j = 0; j < 3; j++) v_b[j] += hh_b[j];
            normalize_b(t.w, hh_b, t.r, d_b);   // w = d / r
        }
    }
}

// ---- metallic-roughness (GGX) shading (the model of include/deodr_b200.h) ----------------------------------------

// The scalars of one light of unit direction w for unit normal n and view v, with k = alpha^2: nl = <n, w>; where
// nl > 0, nv, nh and vh (clamped at 0), h = normalize(w + v) (0 when w + v = 0), Fs = (1 - vh)^5 and, where k > 0, S
// = pi D V = k / (Dd^2 Vl Vv), Dd = nh^2 (k - 1) + 1, Vl = nl + ql, ql = sqrt(k + (1 - k) nl^2) (Vv, qv alike).
// Every other field is 0.  The light's term is E nl [(1 - F)(1 - m) A + a S F] with F = F0 + (1 - F0) Fs.
struct GgxTerm {
    double nl, nv, nh, vh, hn, h[3], Dd, ql, qv, Vl, Vv, S, Fs;
};

__device__ __forceinline__ void ggx_term(const double n[3], const double v[3], const double w[3], double k,
                                         GgxTerm &t) {
    t.nl = dot(n, w);
    t.S = t.Fs = 0.0;
    if (!(t.nl > 0)) return;
    double hh[3];
    for (int j = 0; j < 3; j++) hh[j] = w[j] + v[j];
    t.hn = sqrt(dot(hh, hh));
    for (int j = 0; j < 3; j++) t.h[j] = t.hn == 0.0 ? 0.0 : hh[j] / t.hn;
    const double cv = dot(n, v), ch = dot(n, t.h), cvh = dot(v, t.h);
    t.nv = cv > 0 ? cv : 0.0;
    t.nh = ch > 0 ? ch : 0.0;
    t.vh = cvh > 0 ? cvh : 0.0;
    const double o = 1.0 - t.vh, o2 = o * o;
    t.Fs = (o2 * o2) * o;
    if (!(k > 0)) return;
    t.Dd = (t.nh * t.nh) * (k - 1.0) + 1.0;
    t.ql = sqrt(k + (1.0 - k) * (t.nl * t.nl));
    t.qv = sqrt(k + (1.0 - k) * (t.nv * t.nv));
    t.Vl = t.nl + t.ql;
    t.Vv = t.nv + t.qv;
    t.S = k / ((t.Dd * t.Dd) * (t.Vl * t.Vv));
}

// The adjoint of ggx_term from nl_b (nl's gradient through the term's factor nl), S_b and Fs_b: adds to n_b, v_b,
// w_b and k_b.
__device__ __forceinline__ void ggx_term_b(const GgxTerm &t, const double n[3], const double v[3], const double w[3],
                                           double k, double nl_b, double S_b, double Fs_b, double n_b[3],
                                           double v_b[3], double w_b[3], double &k_b) {
    if (!(t.nl > 0)) return;
    double nv_b = 0, nh_b = 0;
    if (k > 0) {
        const double Sl = t.S / t.Vl, Sv = t.S / t.Vv;
        k_b += S_b * (1.0 / ((t.Dd * t.Dd) * (t.Vl * t.Vv)) -
                      ((2.0 * t.S) * (t.nh * t.nh) / t.Dd + Sl * (1.0 - t.nl * t.nl) / (2.0 * t.ql) +
                       Sv * (1.0 - t.nv * t.nv) / (2.0 * t.qv)));
        nh_b = -S_b * (4.0 * t.S) * t.nh * (k - 1.0) / t.Dd;
        nl_b -= S_b * Sl * (1.0 + (1.0 - k) * t.nl / t.ql);
        nv_b = -S_b * Sv * (1.0 + (1.0 - k) * t.nv / t.qv);
    }
    const double o = 1.0 - t.vh, vh_b = -5.0 * Fs_b * ((o * o) * (o * o));
    double h_b[3] = {0, 0, 0};
    for (int j = 0; j < 3; j++) {
        n_b[j] += nl_b * w[j];
        w_b[j] += nl_b * n[j];
        if (t.nv > 0) {
            n_b[j] += nv_b * v[j];
            v_b[j] += nv_b * n[j];
        }
        if (t.nh > 0) {
            n_b[j] += nh_b * t.h[j];
            h_b[j] += nh_b * n[j];
        }
        if (t.vh > 0) {
            v_b[j] += vh_b * t.h[j];
            h_b[j] += vh_b * v[j];
        }
    }
    if (t.hn != 0.0) {
        double hh_b[3] = {0, 0, 0};
        normalize_b(t.h, h_b, t.hn, hh_b);  // hh = w + v
        for (int j = 0; j < 3; j++) {
            w_b[j] += hh_b[j];
            v_b[j] += hh_b[j];
        }
    }
}

// One light's shares of the three sums its term is formed from, for a grey factor E (the intensity and visibility
// with the falloff): t1 = E nl (1 - Fs), t2 = E nl S (1 - Fs) and t3 = E nl S Fs; a channel's term is then
// (1 - m) A (1 - F0) t1 + a F0 t2 + a t3.  Given u1..u3, the gradients of t1..t3, ggx_sums_b returns E's gradient
// and calls ggx_term_b with those of nl, S and Fs.
__device__ __forceinline__ void ggx_sums(const GgxTerm &t, double E, double out[3]) {
    const double e = t.nl > 0 ? E * t.nl : 0.0, es = e * t.S;
    out[0] = e * (1.0 - t.Fs);
    out[1] = es * (1.0 - t.Fs);
    out[2] = es * t.Fs;
}

__device__ __forceinline__ double ggx_sums_b(const GgxTerm &t, double E, const double u[3], const double n[3],
                                             const double v[3], const double w[3], double k, double n_b[3],
                                             double v_b[3], double w_b[3], double &k_b) {
    if (!(t.nl > 0)) return 0.0;
    const double f = (u[0] + u[1] * t.S) * (1.0 - t.Fs) + (u[2] * t.S) * t.Fs;
    const double e = E * t.nl;
    ggx_term_b(t, n, v, w, k, E * f, e * (u[1] * (1.0 - t.Fs) + u[2] * t.Fs), e * ((u[2] - u[1]) * t.S - u[0]),
               n_b, v_b, w_b, k_b);
    return t.nl * f;
}

// The material of a covered pixel (a != 0) from the factors mf = params[4] and rf = params[5], and the map raster mr
// [H,W,2] = (R, M) when given: r = rf (R / a), m = mf (M / a) (R / a and M / a rounded first), k = alpha^2 = r^4.
struct GgxMaterial {
    double R, M, r, m, k;  // R, M: R / a and M / a (1 without a map)
};

__device__ __forceinline__ void ggx_material(const double *prm, double a, const float *mr, long long p,
                                             GgxMaterial &mt) {
    mt.R = mr ? (double)mr[2 * p] / a : 1.0;
    mt.M = mr ? (double)mr[2 * p + 1] / a : 1.0;
    mt.r = prm[5] * mt.R;
    mt.m = prm[4] * mt.M;
    const double r2 = mt.r * mt.r;
    mt.k = r2 * r2;
}

// Sums v[0..K) over a grid of (rows) x (G CTAs per row) in a fixed order and writes the totals of row i to
// out[i K .. i K + K): CTA (i, y) sums its items into the partials [i][k][y]; the last CTA to finish adds them over y
// in CTA order (the pattern of k_pose_frames_b).  rows K G must not exceed MAX_K * MAX_CTAS.
template <int K>
__device__ void grid_sum_rows(const double (&v)[K], Scratch *s, double *out) {
    __shared__ double warp_sums[K][NT / 32];
    __shared__ bool last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int row = blockIdx.x, rows = gridDim.x, G = gridDim.y;
#pragma unroll
    for (int k = 0; k < K; k++) {
        double x = v[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
        if (lane == 0) warp_sums[k][warp] = x;
    }
    __syncthreads();
    if (threadIdx.x < K) {
        double t = 0;
        for (int w = 0; w < NT / 32; w++) t += warp_sums[threadIdx.x][w];
        s->partials[((long long)row * K + threadIdx.x) * G + blockIdx.y] = t;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        last = atomicAdd(&s->done, 1u) == (unsigned)(rows * G) - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    for (int m = warp; m < rows * K; m += NT / 32) {
        double x = 0;
        for (int i = lane; i < G; i += 32) x += __ldcg(s->partials + (long long)m * G + i);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
        if (lane == 0) out[m] = x;
    }
    __syncthreads();
    if (threadIdx.x == 0) s->done = 0;
}

// colors [n,C] fp64 = vertex_colors * (((max(0, -<n, light_xyz>) + ambient) + sh_c(n)) + P_c(n, x)) per vertex, with
// x the vertex position and P_c the diffuse point-light sum (no environment term at S = 0), or, without vertex
// colours, the luminosity [n] (S <= 1, P = 1).  lights [L, 3 + P]; P = 1 is grey, P = C one intensity per channel.
template <int S, int P>
__global__ void __launch_bounds__(NT) k_point_lit_vertex_colors(const double *normals, const double *positions,
                                                                const double *vcol, int n, int C, const double *light,
                                                                int directional, const double *sh,
                                                                const double *lights, int L, double *colors) {
    constexpr int NC = S > P ? S : P;
    const long long v = (long long)blockIdx.x * NT + threadIdx.x;
    if (v >= n) return;
    const double *nv = normals + 3 * v;
    const double nn[3] = {nv[0], nv[1], nv[2]};
    const double x[3] = {positions[3 * v], positions[3 * v + 1], positions[3 * v + 2]};
    const double dir = directional ? directional_of((nn[0] * light[0] + nn[1] * light[1]) + nn[2] * light[2]) : 0.0;
    const double l = dir + light[3];
    double Y[9], pd[P];
#pragma unroll
    for (int c = 0; c < P; c++) pd[c] = 0;
    if (S > 0) sh_basis(nn, Y);
    for (int j = 0; j < L; j++) {
        const double *lj = lights + j * (3 + P);
        PointTerm t;
        point_term(lj, x, nn, false, nullptr, 0.0, 0.0, t);
#pragma unroll
        for (int c = 0; c < P; c++) pd[c] += lj[3 + c] * t.diff;
    }
    auto lum = [&](int c) {
        const double b = S > 0 ? l + sh_value<(S > 0 ? S : 1)>(sh, S > 1 ? c : 0, Y) : l;
        return b + pd[P > 1 ? c : 0];
    };
    if (!vcol) {
        colors[v] = lum(0);
        return;
    }
    if (NC > 1) {
#pragma unroll
        for (int c = 0; c < NC; c++) colors[v * NC + c] = vcol[v * NC + c] * lum(c);
    } else {
        const double g = lum(0);
        for (int c = 0; c < C; c++) colors[v * C + c] = vcol[v * C + c] * g;
    }
}

// The adjoint of k_point_lit_vertex_colors but lights_b (k_point_lights_vertex_b): g_c = colors_b * vertex_colors
// (colors_b alone for the luminosity); vertex_colors_b = colors_b * lum_c; normals_b = -gate * light + sum_c g_c grad
// sh_c + sum_j alpha_j w_j / r_j^2 with alpha_j = sum_c g_c I_j[c]; positions_b = -sum_j (the gradient of d_j);
// light_b and sh_b as k_sh_lit_vertex_colors_b, summed with grid_sum (fixed order).
template <typename G, int S, int P>
__global__ void __launch_bounds__(NT) k_point_lit_vertex_colors_b(const double *normals, const double *positions,
                                                                  const double *vcol, int n, int C, const double *light,
                                                                  int directional, const double *sh,
                                                                  const double *lights, int L, const G *colors_b,
                                                                  double *normals_b, double *positions_b,
                                                                  double *vcol_b, double *light_b, double *sh_b,
                                                                  Scratch *s) {
    constexpr int NC = S > P ? S : P;
    constexpr int K = 4 + 9 * S;
    __shared__ double tot[K];
    double acc[K];
#pragma unroll
    for (int k = 0; k < K; k++) acc[k] = 0;
    for (long long v = (long long)blockIdx.x * NT + threadIdx.x; v < n; v += (long long)gridDim.x * NT) {
        const double *nv = normals + 3 * v;
        const double nn[3] = {nv[0], nv[1], nv[2]};
        const double x[3] = {positions[3 * v], positions[3 * v + 1], positions[3 * v + 2]};
        const double dir = directional ? directional_of((nn[0] * light[0] + nn[1] * light[1]) + nn[2] * light[2]) : 0.0;
        const double l = dir + light[3];
        double Y[9], g[NC], pd[P], n_b[3] = {0, 0, 0}, x_b[3] = {0, 0, 0}, unused[3] = {0, 0, 0}, q = 0, e_b = 0;
        if (S > 0) sh_basis(nn, Y);
        double lb = 0;
        if (!vcol) {
            lb = (double)colors_b[v];
            g[0] = lb;
        } else if (NC == 1) {
            for (int c = 0; c < C; c++) lb += vcol[v * C + c] * (double)colors_b[v * C + c];
            g[0] = lb;
        } else {
#pragma unroll
            for (int c = 0; c < NC; c++) {
                g[c] = vcol[v * NC + c] * (double)colors_b[v * NC + c];
                lb += g[c];
            }
        }
#pragma unroll
        for (int c = 0; c < P; c++) pd[c] = 0;
        for (int j = 0; j < L; j++) {
            const double *lj = lights + j * (3 + P);
            PointTerm t;
            point_term(lj, x, nn, false, nullptr, 0.0, 0.0, t);
            double alpha = 0, d_b[3] = {0, 0, 0};
            if (P > 1) {
#pragma unroll
                for (int c = 0; c < P; c++) alpha += g[c] * lj[3 + c];
            } else {
                alpha = lj[3] * lb;
            }
#pragma unroll
            for (int c = 0; c < P; c++) pd[c] += lj[3 + c] * t.diff;
            point_term_b(t, nn, alpha, 0.0, 0.0, 0.0, n_b, d_b, unused, q, e_b);
            for (int k = 0; k < 3; k++) x_b[k] -= d_b[k];
        }
        auto base = [&](int c) { return S > 0 ? l + sh_value<(S > 0 ? S : 1)>(sh, S > 1 ? c : 0, Y) : l; };
        if (vcol) {
            if (NC > 1) {
#pragma unroll
                for (int c = 0; c < NC; c++)
                    vcol_b[v * NC + c] = (double)colors_b[v * NC + c] * (base(c) + pd[P > 1 ? c : 0]);
            } else {
                const double lum = base(0) + pd[0];
                for (int c = 0; c < C; c++) vcol_b[v * C + c] = (double)colors_b[v * C + c] * lum;
            }
        }
        if (S > 0) {
            double w[9];
#pragma unroll
            for (int k = 0; k < 9; k++) {
                w[k] = 0;
#pragma unroll
                for (int c = 0; c < (S > 0 ? S : 1); c++) {
                    const double gs = S > 1 ? g[c] : lb;
                    w[k] += gs * sh[k * S + c];
                    acc[4 + k * S + c] += gs * Y[k];
                }
            }
            sh_grad_add(nn, w, n_b);
        }
        const double gate = (directional && dir > 0) ? lb : 0.0;
        for (int j = 0; j < 3; j++) {
            acc[j] += -gate * nn[j];
            normals_b[3 * v + j] = n_b[j] - gate * light[j];
            positions_b[3 * v + j] = x_b[j];
        }
        acc[3] += lb;
    }
    if (grid_sum<K>(acc, s, tot))
        for (int k = threadIdx.x; k < K; k += NT) (k < 4 ? light_b[k] : sh_b[k - 4]) = tot[k];
}

// lights_b [L, 3 + P] of k_point_lit_vertex_colors: CTA (j, y) sums light j over a fixed set of vertices, the
// position's gradient (the d_j share of k_point_lit_vertex_colors_b) and the intensity's, sum g_c diff_j (P = 1: g
// summed over the channels); grid_sum_rows adds the CTAs in a fixed order.  One CTA's registers: the default budget
// spills 12 bytes at P = 1 (DESIGN.md section 13)
template <typename G, int P>
__global__ void __launch_bounds__(NT, 1) k_point_lights_vertex_b(const double *normals, const double *positions,
                                                              const double *vcol, int n, int C, const double *lights,
                                                              const G *colors_b, double *lights_b, Scratch *s) {
    constexpr int K = 3 + P;
    const double *lj = lights + blockIdx.x * K;
    double acc[K];
#pragma unroll
    for (int k = 0; k < K; k++) acc[k] = 0;
    for (long long v = (long long)blockIdx.y * NT + threadIdx.x; v < n; v += (long long)gridDim.y * NT) {
        const double *nv = normals + 3 * v;
        const double nn[3] = {nv[0], nv[1], nv[2]};
        const double x[3] = {positions[3 * v], positions[3 * v + 1], positions[3 * v + 2]};
        double g[P], lb = 0;
        if (!vcol) {
            lb = (double)colors_b[v];
        } else if (P == 1) {
            for (int c = 0; c < C; c++) lb += vcol[v * C + c] * (double)colors_b[v * C + c];
        } else {
#pragma unroll
            for (int c = 0; c < P; c++) g[c] = vcol[v * P + c] * (double)colors_b[v * P + c];
        }
        if (P == 1) g[0] = lb;
        PointTerm t;
        point_term(lj, x, nn, false, nullptr, 0.0, 0.0, t);
        double alpha = 0, d_b[3] = {0, 0, 0}, n_b[3] = {0, 0, 0}, v_b[3] = {0, 0, 0}, q = 0, e_b = 0;
#pragma unroll
        for (int c = 0; c < P; c++) alpha += g[c] * lj[3 + c];
        point_term_b(t, nn, alpha, 0.0, 0.0, 0.0, n_b, d_b, v_b, q, e_b);
        for (int k = 0; k < 3; k++) acc[k] += d_b[k];
#pragma unroll
        for (int c = 0; c < P; c++) acc[3 + c] += g[c] * t.diff;
    }
    grid_sum_rows<K>(acc, s, lights_b);
}

// ---- per-pixel (Phong) shading of a rasterised G-buffer (the model of DeodrPhongIO, include/deodr_b200.h) ---------

constexpr int PHONG_SUMS = 6;  // l_b (3), ambient_b, ks_b, e_b; then camera_center_b (3) when it is asked for

// The shading terms of one pixel, kept for the adjoint.  `lit`: |l| > 0 (else the normals are not read); `spec_on`:
// lit and a != 0; `s` is max(0, <n, h>) and p = s^e (0 at s = 0).
// With a specular map (SPEC), `sp` is the pixel's (K, E) of the map raster and the term uses aks = ks K and
// e(p) = e E / a, kept in `aks` and `e` (set only where spec_on).
struct PhongTerms {
    double n[3], nn, dot_nl, lum;
    double a, ll, u[3], x[3], v[3], dn, h[3], hn, s, p, spec;
    double aks, e;
    bool lit, spec_on;
};

template <bool SPEC = false>
__device__ __forceinline__ void phong_terms(const float *px, const DeodrPhongIO &io, const double *prm,
                                            const double *cam, PhongTerms &t, const float *sp = nullptr) {
    const double N[3] = {px[io.off_normal], px[io.off_normal + 1], px[io.off_normal + 2]};
    const double l[3] = {prm[0], prm[1], prm[2]};
    t.nn = sqrt(dot(N, N));
    for (int j = 0; j < 3; j++) t.n[j] = t.nn == 0.0 ? 0.0 : N[j] / t.nn;  // NaN |N| stays NaN
    t.ll = sqrt(dot(l, l));
    t.lit = t.ll > 0;
    t.dot_nl = t.lit ? dot(t.n, l) : 0.0;
    t.lum = prm[3] + directional_of(t.dot_nl);
    t.a = px[io.off_coverage];
    t.spec_on = t.lit && t.a != 0.0;
    t.s = t.p = t.spec = 0.0;
    if (!t.spec_on) return;
    double hh[3];
    for (int j = 0; j < 3; j++) {
        t.u[j] = l[j] / t.ll;
        t.x[j] = px[io.off_position + j] / t.a;
        t.v[j] = cam[j] - t.x[j];
    }
    t.dn = sqrt(dot(t.v, t.v));
    for (int j = 0; j < 3; j++) {
        t.v[j] /= t.dn;
        hh[j] = t.v[j] - t.u[j];
    }
    t.hn = sqrt(dot(hh, hh));
    for (int j = 0; j < 3; j++) t.h[j] = t.hn == 0.0 ? 0.0 : hh[j] / t.hn;
    const double s = dot(t.n, t.h);
    t.s = s > 0 ? s : 0.0;
    if constexpr (SPEC) {
        t.aks = prm[4] * (double)sp[0];
        t.e = prm[5] * ((double)sp[1] / t.a);
        t.p = t.s > 0 ? pow(t.s, t.e) : 0.0;
        t.spec = (t.aks * t.ll) * t.p;
    } else {
        t.p = t.s > 0 ? pow(t.s, prm[5]) : 0.0;
        t.spec = ((t.a * prm[4]) * t.ll) * t.p;
    }
}

// Where the albedo A of pixel p is read and its adjoint written: the G-buffer's slice at off_albedo (a G-buffer of
// C + 7 channels), or, SPLIT, a buffer albedo [H,W,C] of its own beside a G-buffer of 7 channels (normal, position and
// coverage).  The albedo is the only input whose place differs: the shading and its adjoint are the same code.
template <bool SPLIT>
__device__ __forceinline__ int gbuffer_stride(int C) {
    return SPLIT ? 7 : C + 7;
}

template <bool SPLIT>
__device__ __forceinline__ float albedo_at(const float *px, const DeodrPhongIO &io, const float *albedo, long long p,
                                           int c) {
    return SPLIT ? albedo[p * io.C + c] : px[io.off_albedo + c];
}

template <bool SPLIT>
__device__ __forceinline__ float &albedo_b_at(float *pb, const DeodrPhongIO &io, float *albedo_b, long long p, int c) {
    return SPLIT ? albedo_b[p * io.C + c] : pb[io.off_albedo + c];
}

// The GGX form's image of pixel p (k_phong_shade with GGX; the model of include/deodr_b200.h).  Each light adds its
// ggx_sums into three grey sums (the directional light, grey point lights) or three per channel (coloured point
// lights, P > 1); the channels expand them where the image is formed.  0 surface terms where a = 0.
template <int S, int P, bool VIS, bool SUN>
__device__ __forceinline__ void ggx_shade(const DeodrPhongIO &io, const float *px, long long p, const double *sh,
                                          const float *albedo, const double *lights, int L, const float *vis,
                                          const float *sun_vis, const float *mr, float *out) {
    constexpr int NC = S > P ? S : P, PC = P > 1 ? P : 1;
    const int C = io.C;
    const double *prm = io.params;
    const double a = px[io.off_coverage];
    if (a == 0.0) {
        for (int c = 0; c < C; c++) out[c] = (float)((1.0 - a) * (double)io.background[c]);
        return;
    }
    const double N[3] = {px[io.off_normal], px[io.off_normal + 1], px[io.off_normal + 2]};
    const double nn = sqrt(dot(N, N));
    double n[3], x[3], v[3];
    for (int j = 0; j < 3; j++) {
        n[j] = nn == 0.0 ? 0.0 : N[j] / nn;
        x[j] = px[io.off_position + j] / a;
        v[j] = io.camera_center[j] - x[j];
    }
    const double dn = sqrt(dot(v, v));
    for (int j = 0; j < 3; j++) v[j] /= dn;
    GgxMaterial mt;
    ggx_material(prm, a, mr, p, mt);
    double sg[3] = {0, 0, 0}, sc[3][PC], tt[3];
#pragma unroll
    for (int c = 0; c < PC; c++) sc[0][c] = sc[1][c] = sc[2][c] = 0;
    const double l[3] = {prm[0], prm[1], prm[2]};
    const double ll = sqrt(dot(l, l));
    if (ll > 0) {
        const double w[3] = {-l[0] / ll, -l[1] / ll, -l[2] / ll};
        GgxTerm t;
        ggx_term(n, v, w, mt.k, t);
        ggx_sums(t, SUN ? ll * (double)sun_vis[p] : ll, tt);
        for (int k = 0; k < 3; k++) sg[k] += tt[k];
    }
    if constexpr (P > 0)
        for (int j = 0; j < L; j++) {
            const double *lj = lights + j * (3 + P);
            double d[3], w[3];
            for (int k = 0; k < 3; k++) d[k] = lj[k] - x[k];
            const double r2 = dot(d, d), r = sqrt(r2);
            if (!(r > 0)) continue;
            for (int k = 0; k < 3; k++) w[k] = d[k] / r;
            GgxTerm t;
            ggx_term(n, v, w, mt.k, t);
            double E = (P == 1 ? lj[3] : 1.0) / r2;
            if constexpr (VIS) E *= (double)vis[p * L + j];
            ggx_sums(t, E, tt);
            if (P == 1) {
                for (int k = 0; k < 3; k++) sg[k] += tt[k];
            } else {
#pragma unroll
                for (int c = 0; c < PC; c++)
                    for (int k = 0; k < 3; k++) sc[k][c] += lj[3 + c] * tt[k];
            }
        }
    double Y[9];
    if (S > 0) sh_basis(n, Y);
    const double kd = 1.0 - mt.m;
    auto shade = [&](int c) {
        const double A = albedo[p * C + c], F0 = 0.04 * kd + mt.m * (A / a);
        const int q = P > 1 ? c : 0;
        const double s1 = sg[0] + (P > 1 ? sc[0][q] : 0.0), s2 = sg[1] + (P > 1 ? sc[1][q] : 0.0),
                     s3 = sg[2] + (P > 1 ? sc[2][q] : 0.0);
        const double amb = S > 0 ? prm[3] + sh_value<(S > 0 ? S : 1)>(sh, S > 1 ? c : 0, Y) : prm[3];
        return (float)(((kd * A) * ((1.0 - F0) * s1 + amb) + a * (F0 * s2 + s3)) +
                       (1.0 - a) * (double)io.background[c]);
    };
    if (NC > 1) {
#pragma unroll
        for (int c = 0; c < NC; c++) out[c] = shade(c);
    } else {
        for (int c = 0; c < C; c++) out[c] = shade(c);
    }
}

// The adjoint of ggx_shade for pixel p (k_phong_shade_b with GGX): albedo_b, channels_b, mr_b (with mr), vis_b and
// sun_vis_b written; l_b, ambient_b, mf_b, rf_b (and, CENTER, camera_center_b) added to acc.  A first pass over the
// channels forms u = the gradients of the three sums (grey: U; per channel: uc), the environment's normal gradient
// and env_c; a forward pass over the lights forms the sums, a second pass over the channels takes the material's
// adjoint from them, and the lights' loop then takes each light's adjoint from u (ggx_sums_b).
template <bool CENTER, int S, int P, bool VIS, bool SUN, int K>
__device__ __forceinline__ void ggx_shade_b(const DeodrPhongIO &io, long long p, const double *sh,
                                            const float *albedo, float *albedo_b, const double *lights, int L,
                                            const float *vis, float *vis_b, const float *sun_vis, float *sun_vis_b,
                                            const float *mr, float *mr_b, double (&acc)[K]) {
    constexpr int NC = S > P ? S : P, PC = P > 1 ? P : 1;
    const int C = io.C;
    const double *prm = io.params;
    const float *px = io.channels + p * 7;
    const float *g = io.image_b + p * C;
    float *pb = io.channels_b + p * 7;
    const double a = px[io.off_coverage];
    if (a == 0.0) {
        double bg_b = 0;
        for (int c = 0; c < C; c++) {
            bg_b += (double)io.background[c] * (double)g[c];
            albedo_b[p * C + c] = 0.0f;
        }
        for (int j = 0; j < 3; j++) pb[io.off_normal + j] = pb[io.off_position + j] = 0.0f;
        pb[io.off_coverage] = (float)-bg_b;
        if (mr) mr_b[2 * p] = mr_b[2 * p + 1] = 0.0f;
        if constexpr (VIS)
            for (int j = 0; j < L; j++) vis_b[p * L + j] = 0.0f;
        if constexpr (SUN) sun_vis_b[p] = 0.0f;
        return;
    }
    const double N[3] = {px[io.off_normal], px[io.off_normal + 1], px[io.off_normal + 2]};
    const double nn = sqrt(dot(N, N));
    double n[3], x[3], v[3];
    for (int j = 0; j < 3; j++) {
        n[j] = nn == 0.0 ? 0.0 : N[j] / nn;
        x[j] = px[io.off_position + j] / a;
        v[j] = io.camera_center[j] - x[j];
    }
    const double dn = sqrt(dot(v, v));
    for (int j = 0; j < 3; j++) v[j] /= dn;
    GgxMaterial mt;
    ggx_material(prm, a, mr, p, mt);
    const double kd = 1.0 - mt.m;
    // u(c): channel c's gradients of the three sums; U = sum_c u(c), the grey lights'.  Coloured lights (P > 1)
    // form sum_c u(c) I_j[c] in their loop, from u(c) formed again there rather than kept
    auto u_of = [&](int c, double u[3]) {
        const double A = albedo[p * C + c], gc = g[c], F0 = 0.04 * kd + mt.m * (A / a);
        u[0] = gc * (kd * A) * (1.0 - F0);
        u[1] = gc * (a * F0);
        u[2] = gc * a;
    };
    double U[3] = {0, 0, 0}, env[S > 0 ? S : 1], n_b[3] = {0, 0, 0};
    {
        double Y[9], wsh[9];
        if (S > 0) {
            sh_basis(n, Y);
#pragma unroll
            for (int k = 0; k < 9; k++) wsh[k] = 0;
            if (S == 1) env[0] = sh_value<1>(sh, 0, Y);
        }
        auto pass1 = [&](int c) {
            double u[3];
            u_of(c, u);
            for (int k = 0; k < 3; k++) U[k] += u[k];
            if constexpr (S > 0) {
                const double gA = (double)g[c] * (kd * (double)albedo[p * C + c]);
#pragma unroll
                for (int k = 0; k < 9; k++) wsh[k] += gA * sh[k * S + (S > 1 ? c : 0)];
                if (S > 1) env[S > 1 ? c : 0] = sh_value<(S > 0 ? S : 1)>(sh, c, Y);
            }
        };
        if (NC > 1) {
#pragma unroll
            for (int c = 0; c < NC; c++) pass1(c);
        } else {
            for (int c = 0; c < C; c++) pass1(c);
        }
        if (S > 0) sh_grad_add(n, wsh, n_b);
    }
    // the sums, a forward pass over the lights: their per-channel values are not live in the adjoint's loop below
    double sg[3] = {0, 0, 0}, sc[3][PC], tt[3];
#pragma unroll
    for (int c = 0; c < PC; c++) sc[0][c] = sc[1][c] = sc[2][c] = 0;
    const double l[3] = {prm[0], prm[1], prm[2]};
    const double ll = sqrt(dot(l, l));
    const double sv = SUN ? (double)sun_vis[p] : 1.0;
    if (ll > 0) {
        const double w[3] = {-l[0] / ll, -l[1] / ll, -l[2] / ll};
        GgxTerm t;
        ggx_term(n, v, w, mt.k, t);
        ggx_sums(t, SUN ? ll * sv : ll, tt);
        for (int k = 0; k < 3; k++) sg[k] += tt[k];
    }
    if constexpr (P > 0)
        for (int j = 0; j < L; j++) {
            const double *lj = lights + j * (3 + P);
            double d[3], w[3];
            for (int k = 0; k < 3; k++) d[k] = lj[k] - x[k];
            const double r2 = dot(d, d), r = sqrt(r2);
            if (!(r > 0)) continue;
            for (int k = 0; k < 3; k++) w[k] = d[k] / r;
            GgxTerm t;
            ggx_term(n, v, w, mt.k, t);
            const double E0 = (P == 1 ? lj[3] : 1.0) / r2;
            ggx_sums(t, VIS ? E0 * (double)vis[p * L + j] : E0, tt);
            if (P == 1) {
                for (int k = 0; k < 3; k++) sg[k] += tt[k];
            } else {
#pragma unroll
                for (int c = 0; c < PC; c++)
                    for (int k = 0; k < 3; k++) sc[k][c] += lj[3 + c] * tt[k];
            }
        }
    // the material: F0_c = 0.04 kd + m b_c, b_c = A_c / a, kd = 1 - m
    double kd_b = 0, m_b = 0, a_b = 0;
    auto pass2 = [&](int c) {
        const double A = albedo[p * C + c], gc = g[c], b = A / a, F0 = 0.04 * kd + mt.m * b;
        const int q = P > 1 ? c : 0;
        const double s1 = sg[0] + (P > 1 ? sc[0][q] : 0.0), s2 = sg[1] + (P > 1 ? sc[1][q] : 0.0),
                     s3 = sg[2] + (P > 1 ? sc[2][q] : 0.0);
        const double lum = (1.0 - F0) * s1 + (S > 0 ? prm[3] + env[S > 1 ? c : 0] : prm[3]);
        const double F0_b = gc * (a * s2 - (kd * A) * s1), b_b = F0_b * mt.m;
        kd_b += gc * A * lum + 0.04 * F0_b;
        m_b += F0_b * b;
        a_b += gc * ((F0 * s2 + s3) - (double)io.background[c]) - b_b * b / a;
        acc[3] += gc * (kd * A);
        albedo_b[p * C + c] = (float)(gc * kd * lum + b_b / a);
    };
    if (NC > 1) {
#pragma unroll
        for (int c = 0; c < NC; c++) pass2(c);
    } else {
        for (int c = 0; c < C; c++) pass2(c);
    }
    m_b -= kd_b;
    // the lights' adjoint, each term formed again
    double v_b[3] = {0, 0, 0}, x_b[3] = {0, 0, 0}, k_b = 0;
    if (ll > 0) {
        // E = |l| V, w = -l / |l|
        const double w[3] = {-l[0] / ll, -l[1] / ll, -l[2] / ll};
        GgxTerm t;
        ggx_term(n, v, w, mt.k, t);
        double w_b[3] = {0, 0, 0};
        const double E_b = ggx_sums_b(t, SUN ? ll * sv : ll, U, n, v, w, mt.k, n_b, v_b, w_b, k_b);
        if constexpr (SUN) sun_vis_b[p] = (float)(E_b * ll);
        const double ll_b = SUN ? E_b * sv : E_b, pr = dot(w, w_b);
        for (int j = 0; j < 3; j++) acc[j] += -ll_b * w[j] - (w_b[j] - w[j] * pr) / ll;
    } else if constexpr (SUN) {
        sun_vis_b[p] = 0.0f;
    }
    if constexpr (P > 0)
        for (int j = 0; j < L; j++) {
            // E = I V / r^2 (I = 1 for coloured lights: their intensities are in uj), w = d / r, d = p_j - x
            const double *lj = lights + j * (3 + P);
            double d[3], w[3], w_b[3] = {0, 0, 0}, d_b[3] = {0, 0, 0};
            for (int k = 0; k < 3; k++) d[k] = lj[k] - x[k];
            const double r2 = dot(d, d), r = sqrt(r2);
            if (!(r > 0)) {
                if constexpr (VIS) vis_b[p * L + j] = 0.0f;
                continue;
            }
            for (int k = 0; k < 3; k++) w[k] = d[k] / r;
            GgxTerm t;
            ggx_term(n, v, w, mt.k, t);
            const double E0 = (P == 1 ? lj[3] : 1.0) / r2, E = VIS ? E0 * (double)vis[p * L + j] : E0;
            double uj[3];
            if (P == 1) {
                for (int k = 0; k < 3; k++) uj[k] = U[k];
            } else {
                for (int k = 0; k < 3; k++) uj[k] = 0;
#pragma unroll
                for (int c = 0; c < PC; c++) {
                    double u[3];
                    u_of(c, u);
                    for (int k = 0; k < 3; k++) uj[k] += u[k] * lj[3 + c];
                }
            }
            const double E_b = ggx_sums_b(t, E, uj, n, v, w, mt.k, n_b, v_b, w_b, k_b);
            if constexpr (VIS) vis_b[p * L + j] = (float)(E_b * E0);
            const double r_b = -2.0 * E_b * E / r;
            for (int k = 0; k < 3; k++) d_b[k] += r_b * w[k];
            normalize_b(w, w_b, r, d_b);
            for (int k = 0; k < 3; k++) x_b[k] -= d_b[k];
        }
    // m = mf (M / a), r = rf (R / a), k = r^4
    const double r_b = k_b * (4.0 * ((mt.r * mt.r) * mt.r));
    acc[4] += m_b * mt.M;
    acc[5] += r_b * mt.R;
    if (mr) {
        mr_b[2 * p] = (float)(r_b * prm[5] / a);
        mr_b[2 * p + 1] = (float)(m_b * prm[4] / a);
        a_b -= (r_b * mt.r + m_b * mt.m) / a;
    }
    double dv_b[3] = {0, 0, 0}, N_b[3] = {0, 0, 0};
    normalize_b(v, v_b, dn, dv_b);  // v = normalize(cam - x)
    for (int j = 0; j < 3; j++) {
        x_b[j] -= dv_b[j];
        if (CENTER) acc[PHONG_SUMS + j] += dv_b[j];
    }
    a_b -= dot(x_b, x) / a;  // x = X / a
    if (nn != 0.0) normalize_b(n, n_b, nn, N_b);
    for (int j = 0; j < 3; j++) {
        pb[io.off_normal + j] = (float)N_b[j];
        pb[io.off_position + j] = (float)(x_b[j] / a);
    }
    pb[io.off_coverage] = (float)a_b;
}

// image[c] = A[c] (ambient + diff) + spec + (1 - a) bg[c], one thread per pixel; with an environment of S > 0
// channels, A[c] ((ambient + diff) + sh_c(n)).  minBlocks 0 is no hint (the G-buffer instances are unchanged); with a
// separate albedo the default budget spills 8 bytes at S = 1 across the fp64 division calls, so those instances take
// the registers of one CTA per SM (ptxas -v, DESIGN.md section 12).  With P > 0, point lights [L, 3 + P] add P_c to
// the luminosity and Q_c to the specular term (P = 1: grey); at P = 3 the default budget spills 12 bytes across the
// pow calls, so the point-light instances take one CTA's registers too (DESIGN.md section 13).  With VIS (P > 0), light
// j's diffuse and specular terms are multiplied by its visibility vis [H,W,L] (DESIGN.md section 14); with SUN, the
// directional light's by sun_vis [H,W] (DESIGN.md section 15).  With SPEC (SPLIT only), the specular map's
// raster spec_map [H,W,2] = (K, E) gives every specular term, the point lights' included, aks = ks K and e(p) =
// e E / a in place of a ks and e (DESIGN.md section 17).  With GGX (SPLIT only), the metallic-roughness form
// (ggx_shade) replaces the Phong one, and spec_map is the metallic-roughness map's raster (R, M), or NULL for the
// factors alone (DESIGN.md section 18)
template <int S, bool SPLIT, int P = 0, bool VIS = false, bool SUN = false, bool SPEC = false, bool GGX = false>
__global__ void __launch_bounds__(NT, SPLIT || P > 0 ? 1 : 0) k_phong_shade(DeodrPhongIO io, const double *sh,
                                                                  const float *albedo, const double *lights, int L,
                                                                  const float *vis = nullptr,
                                                                  const float *sun_vis = nullptr,
                                                                  const float *spec_map = nullptr) {
    static_assert(SPLIT || !SPEC, "a specular map is read beside a separate albedo");
    static_assert(!GGX || (SPLIT && !SPEC), "the metallic-roughness form reads a separate albedo and no specular map");
    const long long p = (long long)blockIdx.x * NT + threadIdx.x;
    if (p >= (long long)io.H * io.W) return;
    const int C = io.C;
    const float *px = io.channels + p * gbuffer_stride<SPLIT>(C);
    if constexpr (GGX) {
        ggx_shade<S, P, VIS, SUN>(io, px, p, sh, albedo, lights, L, vis, sun_vis, spec_map, io.image + p * C);
        return;
    }
    PhongTerms t;
    phong_terms<SPEC>(px, io, io.params, io.camera_center, t, SPEC ? spec_map + 2 * p : nullptr);
    if constexpr (SUN) {
        // each product rounded on its own, so that V = 1 leaves the terms, and the image, bit for bit
        const double sv = sun_vis[p];
        t.lum = io.params[3] + __dmul_rn(directional_of(t.dot_nl), sv);
        t.spec = __dmul_rn(t.spec, sv);
    }
    float *out = io.image + p * C;
    if constexpr (P > 0) {
        // pd[c] = P_c and qs[c] = Q_c, the lights in index order; both 0 where a = 0
        constexpr int NC = S > P ? S : P;
        double pd[P], qs[P];
#pragma unroll
        for (int c = 0; c < P; c++) pd[c] = qs[c] = 0;
        if (t.a != 0.0) {
            double x[3], v[3];
            for (int j = 0; j < 3; j++) {
                x[j] = px[io.off_position + j] / t.a;
                v[j] = io.camera_center[j] - x[j];
            }
            const double dn = sqrt(dot(v, v));
            for (int j = 0; j < 3; j++) v[j] /= dn;
            const double aks = SPEC ? io.params[4] * (double)spec_map[2 * p] : t.a * io.params[4];
            const double e = SPEC ? io.params[5] * ((double)spec_map[2 * p + 1] / t.a) : io.params[5];
            for (int j = 0; j < L; j++) {
                const double *lj = lights + j * (3 + P);
                PointTerm pt;
                point_term(lj, x, t.n, true, v, aks, e, pt);
                if constexpr (VIS) {
                    // each product rounded on its own, so that V = 1 leaves the terms, and the image, bit for bit
                    const double vj = vis[p * L + j];
                    pt.diff = __dmul_rn(pt.diff, vj);
                    pt.spec = __dmul_rn(pt.spec, vj);
                }
#pragma unroll
                for (int c = 0; c < P; c++) {
                    pd[c] += lj[3 + c] * pt.diff;
                    qs[c] += lj[3 + c] * pt.spec;
                }
            }
        }
        double Y[9];
        if (S > 0) sh_basis(t.n, Y);
        auto shade = [&](int c) {
            const double b = S > 0 ? t.lum + sh_value<(S > 0 ? S : 1)>(sh, S > 1 ? c : 0, Y) : t.lum;
            const int k = P > 1 ? c : 0;
            return (float)(((double)albedo_at<SPLIT>(px, io, albedo, p, c) * (b + pd[k]) + (t.spec + qs[k])) +
                           (1.0 - t.a) * (double)io.background[c]);
        };
        if (NC > 1) {
#pragma unroll
            for (int c = 0; c < NC; c++) out[c] = shade(c);
        } else {
            for (int c = 0; c < C; c++) out[c] = shade(c);
        }
        return;
    }
    if (S == 0) {
        for (int c = 0; c < C; c++)
            out[c] = (float)(((double)albedo_at<SPLIT>(px, io, albedo, p, c) * t.lum + t.spec) +
                             (1.0 - t.a) * (double)io.background[c]);
        return;
    }
    double Y[9];
    sh_basis(t.n, Y);
    const double grey = S == 1 ? t.lum + sh_value<1>(sh, 0, Y) : 0.0;
    for (int c = 0; c < C; c++) {
        const double lum = S == 1 ? grey : t.lum + sh_value<S>(sh, c, Y);
        out[c] = (float)(((double)albedo_at<SPLIT>(px, io, albedo, p, c) * lum + t.spec) +
                         (1.0 - t.a) * (double)io.background[c]);
    }
}

// The adjoint of k_phong_shade: each thread a fixed set of pixels in order, params_b (and, with CENTER,
// camera_center_b) summed with grid_sum.  With an environment (S > 0) the albedo and normal adjoints take its share;
// sh_b is summed by k_phong_sh_b, a second pass, so that its 9 S sums do not hold registers here.
// minBlocks 0 is no hint (S = 0 compiles to the kernel without an environment); at S = 2 and 4 the default budget
// spills a few bytes, so those take the registers of one CTA per SM (ptxas -v, DESIGN.md section 11)
// With point lights (P > 0) the albedo, normal, position and coverage adjoints, params_b and camera_center_b take their
// share; lights_b is summed by k_point_lights_pixel_b, a pass of its own (up to 8 (3 + P) sums).
// With VIS, light j's terms are scaled by vis [H,W,L] and vis_b[p, j] = alpha_j diff_j + beta_j spec_j is written
// (0 where a = 0).  With SUN, the directional diff and spec are scaled by sun_vis [H,W] and sun_vis_b[p] =
// sum_c g_c (A_c diff + spec) is written; at S = 3 without point lights the default budget spills then too, so
// those take one CTA's registers (DESIGN.md section 15).
// With SPEC (SPLIT only), aks = ks K and e(p) = e E / a from spec_map [H,W,2] = (K, E): q and e_b(p), the
// gradients of aks and e(p) summed over the main term and the point lights, give spec_map_b [H,W,2] = (q ks,
// e_b(p) e / a) (0 where a = 0), ks_b += q K, e_b += e_b(p) E / a and a_b -= e_b(p) e(p) / a (DESIGN.md section 17).
// With GGX (SPLIT only), ggx_shade_b takes each pixel, spec_map is the metallic-roughness map's raster (R, M) or
// NULL, spec_map_b its gradient, and params_b[4..5] are mf_b and rf_b (DESIGN.md section 18).
template <bool CENTER, int S, bool SPLIT, int P = 0, bool VIS = false, bool SUN = false, bool SPEC = false,
          bool GGX = false>
__global__ void __launch_bounds__(NT, S == 2 || S == 4 || (SUN && S == 3 && P == 0) || SPEC || GGX ? 1 : 0)
    k_phong_shade_b(DeodrPhongIO io, Scratch *s, const double *sh, const float *albedo, float *albedo_b,
                    const double *lights, int L, const float *vis = nullptr, float *vis_b = nullptr,
                    const float *sun_vis = nullptr, float *sun_vis_b = nullptr, const float *spec_map = nullptr,
                    float *spec_map_b = nullptr) {
    static_assert(SPLIT || !SPEC, "a specular map is read beside a separate albedo");
    static_assert(!GGX || (SPLIT && !SPEC), "the metallic-roughness form reads a separate albedo and no specular map");
    constexpr int NC = S > P ? S : P;
    constexpr int K = PHONG_SUMS + (CENTER ? 3 : 0);
    __shared__ double tot[K];
    double acc[K];
#pragma unroll
    for (int k = 0; k < K; k++) acc[k] = 0;
    const int C = io.C;
    const double *prm = io.params;
    const double ks = prm[4], e = prm[5];
    const long long pixels = (long long)io.H * io.W;
    for (long long p = (long long)blockIdx.x * NT + threadIdx.x; p < pixels; p += (long long)gridDim.x * NT) {
        if constexpr (GGX) {
            ggx_shade_b<CENTER, S, P, VIS, SUN>(io, p, sh, albedo, albedo_b, lights, L, vis, vis_b, sun_vis,
                                                sun_vis_b, spec_map, spec_map_b, acc);
            continue;
        }
        const float *px = io.channels + p * gbuffer_stride<SPLIT>(C);
        const float *g = io.image_b + p * C;
        float *pb = io.channels_b + p * gbuffer_stride<SPLIT>(C);
        // the environment's share first, so that its basis and coefficients are not live beside PhongTerms: env[c] =
        // sh_c(n) and the normal's adjoint sum_c g_c grad sh_c, with n the normal phong_terms computes
        double env[S > 0 ? S : 1], n_b[3] = {0, 0, 0};
        if (S > 0) {
            const double N[3] = {px[io.off_normal], px[io.off_normal + 1], px[io.off_normal + 2]};
            const double nn = sqrt(dot(N, N));
            double n[3], Y[9], w[9];
            for (int j = 0; j < 3; j++) n[j] = nn == 0.0 ? 0.0 : N[j] / nn;
            sh_basis(n, Y);
            if (S == 1) {
                double gA = 0;
                for (int c = 0; c < C; c++) gA += (double)albedo_at<SPLIT>(px, io, albedo, p, c) * (double)g[c];
                env[0] = sh_value<1>(sh, 0, Y);
#pragma unroll
                for (int k = 0; k < 9; k++) w[k] = gA * sh[k];
            } else {
#pragma unroll
                for (int k = 0; k < 9; k++) w[k] = 0;
#pragma unroll
                for (int c = 0; c < (S > 1 ? S : 1); c++) {
                    const double gA = (double)albedo_at<SPLIT>(px, io, albedo, p, c) * (double)g[c];
                    env[c] = sh_value<S>(sh, c, Y);
#pragma unroll
                    for (int k = 0; k < 9; k++) w[k] += gA * sh[k * S + c];
                }
            }
            sh_grad_add(n, w, n_b);
        }
        // the point lights' share, before PhongTerms too: pd[c] = P_c for the albedo's adjoint, the normal's into n_b,
        // the position's and coverage's into pX_b and pa_b (x = X / a, v = normalize(cam - x)), ks_b, e_b and the
        // camera centre's into acc.  alpha_j = sum_c g_c A_c I_j[c] and beta_j = sum_c g_c I_j[c] are the gradients of
        // the light's diffuse and specular factors.
        double pd[P > 0 ? P : 1], pX_b[3] = {0, 0, 0}, pa_b = 0;
        double sq = 0, se_b = 0;  // with SPEC: the gradients of aks and e(p), summed over the terms
        if constexpr (P > 0) {
#pragma unroll
            for (int c = 0; c < P; c++) pd[c] = 0;
            const double a = px[io.off_coverage];
            if (a != 0.0) {
                const double N[3] = {px[io.off_normal], px[io.off_normal + 1], px[io.off_normal + 2]};
                const double nn = sqrt(dot(N, N));
                double n[3], x[3], v[3], gA[P], gs[P];
                for (int j = 0; j < 3; j++) {
                    n[j] = nn == 0.0 ? 0.0 : N[j] / nn;
                    x[j] = px[io.off_position + j] / a;
                    v[j] = io.camera_center[j] - x[j];
                }
                const double dn = sqrt(dot(v, v));
                for (int j = 0; j < 3; j++) v[j] /= dn;
                if (P > 1) {
#pragma unroll
                    for (int c = 0; c < P; c++) {
                        gs[c] = g[c];
                        gA[c] = (double)albedo_at<SPLIT>(px, io, albedo, p, c) * gs[c];
                    }
                } else {
                    gA[0] = gs[0] = 0;
                    for (int c = 0; c < C; c++) {
                        gA[0] += (double)albedo_at<SPLIT>(px, io, albedo, p, c) * (double)g[c];
                        gs[0] += g[c];
                    }
                }
                const double aks = SPEC ? ks * (double)spec_map[2 * p] : a * ks;
                const double ep = SPEC ? e * ((double)spec_map[2 * p + 1] / a) : e;
                double v_b[3] = {0, 0, 0}, x_b[3] = {0, 0, 0}, q = 0, e_b = 0;
                for (int j = 0; j < L; j++) {
                    const double *lj = lights + j * (3 + P);
                    PointTerm pt;
                    point_term(lj, x, n, true, v, aks, ep, pt);
                    double alpha = 0, beta = 0, d_b[3] = {0, 0, 0}, vj = 1.0;
                    if constexpr (VIS) vj = vis[p * L + j];
                    const double diff = VIS ? __dmul_rn(pt.diff, vj) : pt.diff;
#pragma unroll
                    for (int c = 0; c < P; c++) {
                        alpha += gA[c] * lj[3 + c];
                        beta += gs[c] * lj[3 + c];
                        pd[c] += lj[3 + c] * diff;
                    }
                    if constexpr (VIS) {
                        vis_b[p * L + j] = (float)(alpha * pt.diff + beta * pt.spec);
                        alpha = __dmul_rn(alpha, vj);
                        beta = __dmul_rn(beta, vj);
                    }
                    point_term_b(pt, n, alpha, beta, aks, ep, n_b, d_b, v_b, q, e_b);
                    for (int k = 0; k < 3; k++) x_b[k] -= d_b[k];
                }
                if constexpr (SPEC) {
                    sq = q;
                    se_b = e_b;
                } else {
                    acc[4] += q * a;
                    acc[5] += e_b;
                    pa_b = q * ks;
                }
                double dv_b[3] = {0, 0, 0};
                normalize_b(v, v_b, dn, dv_b);  // v = normalize(cam - x)
                for (int j = 0; j < 3; j++) {
                    x_b[j] -= dv_b[j];
                    if (CENTER) acc[PHONG_SUMS + j] += dv_b[j];
                    pX_b[j] = x_b[j] / a;
                }
                pa_b -= dot(x_b, x) / a;
            } else if constexpr (VIS) {
                for (int j = 0; j < L; j++) vis_b[p * L + j] = 0.0f;
            }
        }
        PhongTerms t;
        phong_terms<SPEC>(px, io, prm, io.camera_center, t, SPEC ? spec_map + 2 * p : nullptr);
        double sv = 1.0, diff0 = 0, spec0 = 0;  // with SUN: V and the unshadowed directional terms
        if constexpr (SUN) {
            sv = sun_vis[p];
            diff0 = directional_of(t.dot_nl);
            spec0 = t.spec;
            t.lum = prm[3] + __dmul_rn(diff0, sv);
        }
        double lum_b = 0, spec_b = 0, bg_b = 0;
        // the luminosity of channel c: (ambient + diff) (+ sh_c) (+ P_c)
        auto lum_of = [&](int c) {
            const double b = S == 0 ? t.lum : t.lum + env[S > 1 ? c : 0];
            if constexpr (P > 0)
                return b + pd[P > 1 ? c : 0];
            else
                return b;
        };
        if (NC > 1) {
#pragma unroll
            for (int c = 0; c < (NC > 1 ? NC : 1); c++) {
                const double gc = g[c];
                lum_b += (double)albedo_at<SPLIT>(px, io, albedo, p, c) * gc;
                spec_b += gc;
                bg_b += (double)io.background[c] * gc;
                albedo_b_at<SPLIT>(pb, io, albedo_b, p, c) = (float)(gc * lum_of(c));
            }
        } else {
            for (int c = 0; c < C; c++) {
                const double gc = g[c];
                lum_b += (double)albedo_at<SPLIT>(px, io, albedo, p, c) * gc;
                spec_b += gc;
                bg_b += (double)io.background[c] * gc;
                albedo_b_at<SPLIT>(pb, io, albedo_b, p, c) = (float)(gc * lum_of(0));
            }
        }
        acc[3] += lum_b;
        double diff_b = lum_b;
        if constexpr (SUN) {
            sun_vis_b[p] = (float)(lum_b * diff0 + spec_b * spec0);
            diff_b = __dmul_rn(lum_b, sv);
            spec_b = __dmul_rn(spec_b, sv);
        }
        double a_b = -bg_b, N_b[3] = {0, 0, 0}, X_b[3] = {0, 0, 0};
        if (t.lit && t.dot_nl < 0)
            for (int j = 0; j < 3; j++) {
                n_b[j] -= diff_b * prm[j];
                acc[j] -= diff_b * t.n[j];
            }
        if (t.spec_on) {
            double ll_b;
            if constexpr (SPEC) {
                sq += spec_b * (t.ll * t.p);
                ll_b = spec_b * (t.aks * t.p);
            } else {
                a_b += spec_b * ((ks * t.ll) * t.p);
                acc[4] += spec_b * ((t.a * t.ll) * t.p);
                ll_b = spec_b * ((t.a * ks) * t.p);
            }
            for (int j = 0; j < 3; j++) acc[j] += ll_b * t.u[j];
            if (t.s > 0) {
                const double p_b = spec_b * (SPEC ? t.aks * t.ll : (t.a * ks) * t.ll);
                const double ep = SPEC ? t.e : e;
                const double s_b = p_b * ep * pow(t.s, ep - 1);
                if constexpr (SPEC)
                    se_b += p_b * t.p * log(t.s);
                else
                    acc[5] += p_b * t.p * log(t.s);
                double h_b[3];
                for (int j = 0; j < 3; j++) {
                    n_b[j] += s_b * t.h[j];
                    h_b[j] = s_b * t.n[j];
                }
                if (t.hn != 0.0) {
                    double hh_b[3] = {0, 0, 0}, u_b[3], l_b[3] = {0, 0, 0}, d_b[3] = {0, 0, 0};
                    normalize_b(t.h, h_b, t.hn, hh_b);  // hh = v - u
                    for (int j = 0; j < 3; j++) u_b[j] = -hh_b[j];
                    normalize_b(t.u, u_b, t.ll, l_b);
                    normalize_b(t.v, hh_b, t.dn, d_b);  // d = cam - x, x = X / a
                    for (int j = 0; j < 3; j++) {
                        acc[j] += l_b[j];
                        X_b[j] = -d_b[j] / t.a;
                        if (CENTER) acc[PHONG_SUMS + j] += d_b[j];
                    }
                    a_b += dot(d_b, t.x) / t.a;
                }
            }
        }
        if constexpr (SPEC) {
            // aks = ks K and e(p) = e E / a: the map's gradient, ks_b and e_b, and e(p)'s share of a_b
            float *sb = spec_map_b + 2 * p;
            if (t.a != 0.0) {
                const double K = spec_map[2 * p], E = spec_map[2 * p + 1];
                sb[0] = (float)(sq * ks);
                sb[1] = (float)(se_b * e / t.a);
                acc[4] += sq * K;
                acc[5] += se_b * E / t.a;
                a_b -= se_b * (e * (E / t.a)) / t.a;
            } else {
                sb[0] = sb[1] = 0.0f;
            }
        }
        if ((t.lit || S > 0 || P > 0) && t.nn != 0.0) normalize_b(t.n, n_b, t.nn, N_b);
        for (int j = 0; j < 3; j++) {
            pb[io.off_normal + j] = (float)N_b[j];
            pb[io.off_position + j] = (float)(P > 0 ? X_b[j] + pX_b[j] : X_b[j]);
        }
        pb[io.off_coverage] = (float)(P > 0 ? a_b + pa_b : a_b);
    }
    if (grid_sum<K>(acc, s, tot) && threadIdx.x == 0) {
        for (int k = 0; k < PHONG_SUMS; k++) io.params_b[k] = tot[k];
        if (CENTER)
            for (int j = 0; j < 3; j++) io.camera_center_b[j] = tot[PHONG_SUMS + j];
    }
}

// sh_b[k, s] = sum over the pixels of g_s Y_k(n), g_c = image_b[c] A[c] (S = 1: summed over the channels, in the
// order of lum_b above), n = N / |N| (0 when |N| = 0).  A pass of its own over the G-buffer and image_b: 9 S
// accumulators beside k_phong_shade_b's would cost that kernel its occupancy (DESIGN.md section 11).  With GGX, the
// environment lights the diffuse lobe only: g_c is scaled by 1 - m, m = mf (M / a) from the map raster mr [H,W,2]
// (mf without one), and is 0 where a = 0.
template <int S, bool SPLIT, bool GGX = false>
__global__ void __launch_bounds__(NT) k_phong_sh_b(DeodrPhongIO io, Scratch *s, double *sh_b, const float *albedo,
                                                   const float *mr = nullptr) {
    constexpr int K = 9 * S;
    __shared__ double tot[K];
    double acc[K];
#pragma unroll
    for (int k = 0; k < K; k++) acc[k] = 0;
    const int C = io.C;
    const long long pixels = (long long)io.H * io.W;
    for (long long p = (long long)blockIdx.x * NT + threadIdx.x; p < pixels; p += (long long)gridDim.x * NT) {
        const float *px = io.channels + p * gbuffer_stride<SPLIT>(C);
        const float *gp = io.image_b + p * C;
        const double N[3] = {px[io.off_normal], px[io.off_normal + 1], px[io.off_normal + 2]};
        const double nn = sqrt(dot(N, N));
        double n[3], Y[9], g[S];
        for (int j = 0; j < 3; j++) n[j] = nn == 0.0 ? 0.0 : N[j] / nn;
        sh_basis(n, Y);
        if (S == 1) {
            g[0] = 0;
            for (int c = 0; c < C; c++) g[0] += (double)albedo_at<SPLIT>(px, io, albedo, p, c) * (double)gp[c];
        } else {
#pragma unroll
            for (int c = 0; c < S; c++) g[c] = (double)albedo_at<SPLIT>(px, io, albedo, p, c) * (double)gp[c];
        }
        if constexpr (GGX) {
            const double a = px[io.off_coverage];
            const double kd = a != 0.0 ? 1.0 - io.params[4] * (mr ? (double)mr[2 * p + 1] / a : 1.0) : 0.0;
#pragma unroll
            for (int c = 0; c < S; c++) g[c] *= kd;
        }
#pragma unroll
        for (int k = 0; k < 9; k++)
#pragma unroll
            for (int c = 0; c < S; c++) acc[k * S + c] += g[c] * Y[k];
    }
    if (grid_sum<K>(acc, s, tot))
        for (int k = threadIdx.x; k < K; k += NT) sh_b[k] = tot[k];
}

// lights_b [L, 3 + P] of the Phong forms: CTA (j, y) sums light j over a fixed set of pixels, the position's gradient
// (the d_j share of k_phong_shade_b) and the intensity's, g_c A_c diff_j + g_c spec_j (P = 1: summed over the
// channels); grid_sum_rows adds the CTAs in a fixed order.  The CTAs of one set of pixels are adjacent in the grid, so
// the G-buffer is read from DRAM about once.  With VIS, light j's terms are scaled by vis [H,W,L].  With SPEC, the
// terms use aks = ks K and e(p) = e E / a from spec_map [H,W,2]; the map's gradient is k_phong_shade_b's.  With GGX,
// the terms are the metallic-roughness form's (ggx_sums_b), with spec_map the map raster (R, M) or NULL.
template <int P, bool SPLIT, bool VIS = false, bool SPEC = false, bool GGX = false>
__global__ void __launch_bounds__(NT, GGX ? 1 : 0) k_point_lights_pixel_b(DeodrPhongIO io, const float *albedo,
                                                             const double *lights, double *lights_b, Scratch *s,
                                                             const float *vis = nullptr,
                                                             const float *spec_map = nullptr) {
    constexpr int K = 3 + P;
    const double *lj = lights + blockIdx.x * K;
    double acc[K];
#pragma unroll
    for (int k = 0; k < K; k++) acc[k] = 0;
    const int C = io.C;
    const double ks = io.params[4], e = io.params[5];
    const long long pixels = (long long)io.H * io.W;
    for (long long p = (long long)blockIdx.y * NT + threadIdx.x; p < pixels; p += (long long)gridDim.y * NT) {
        const float *px = io.channels + p * gbuffer_stride<SPLIT>(C);
        const float *g = io.image_b + p * C;
        const double a = px[io.off_coverage];
        if (a == 0.0) continue;
        const double N[3] = {px[io.off_normal], px[io.off_normal + 1], px[io.off_normal + 2]};
        const double nn = sqrt(dot(N, N));
        double n[3], x[3], v[3], gA[P], gs[P];
        for (int j = 0; j < 3; j++) {
            n[j] = nn == 0.0 ? 0.0 : N[j] / nn;
            x[j] = px[io.off_position + j] / a;
            v[j] = io.camera_center[j] - x[j];
        }
        const double dn = sqrt(dot(v, v));
        for (int j = 0; j < 3; j++) v[j] /= dn;
        if constexpr (GGX) {
            // u[k][c]: the gradients of light j's three sums, per channel (P > 1) or summed (P = 1), as ggx_shade_b
            GgxMaterial mt;
            ggx_material(io.params, a, spec_map, p, mt);
            const double kd = 1.0 - mt.m;
            auto u_of = [&](int c, double u[3]) {
                const double A = albedo[p * C + c], gc = g[c], F0 = 0.04 * kd + mt.m * (A / a);
                u[0] = gc * (kd * A) * (1.0 - F0);
                u[1] = gc * (a * F0);
                u[2] = gc * a;
            };
            double d[3], w[3], w_b[3] = {0, 0, 0}, d_b[3] = {0, 0, 0}, n_b[3] = {0, 0, 0}, v_b[3] = {0, 0, 0}, k_b = 0;
            double uj[3], tt[3];
            for (int k = 0; k < 3; k++) d[k] = lj[k] - x[k];
            const double r2 = dot(d, d), r = sqrt(r2);
            if (!(r > 0)) continue;
            for (int k = 0; k < 3; k++) w[k] = d[k] / r;
            GgxTerm t;
            ggx_term(n, v, w, mt.k, t);
            const double vj = VIS ? (double)vis[p * gridDim.x + blockIdx.x] : 1.0;
            const double E0 = (P == 1 ? lj[3] : 1.0) / r2, E = VIS ? E0 * vj : E0;
            for (int k = 0; k < 3; k++) uj[k] = 0;
            auto add_u = [&](int c) {
                double u[3];
                u_of(c, u);
                for (int k = 0; k < 3; k++) uj[k] += u[k] * (P == 1 ? 1.0 : lj[3 + c]);
            };
            if (P > 1) {
#pragma unroll
                for (int c = 0; c < P; c++) add_u(c);
            } else {
                for (int c = 0; c < C; c++) add_u(c);
            }
            const double E_b = ggx_sums_b(t, E, uj, n, v, w, mt.k, n_b, v_b, w_b, k_b);
            const double r_b = -2.0 * E_b * E / r;
            for (int k = 0; k < 3; k++) d_b[k] += r_b * w[k];
            normalize_b(w, w_b, r, d_b);
            for (int k = 0; k < 3; k++) acc[k] += d_b[k];
            // the intensity's: the sums at E = V / r^2
            ggx_sums(t, VIS ? vj / r2 : 1.0 / r2, tt);
            if (P > 1) {
#pragma unroll
                for (int c = 0; c < P; c++) {
                    double u[3];
                    u_of(c, u);
                    acc[3 + c] += (u[0] * tt[0] + u[1] * tt[1]) + u[2] * tt[2];
                }
            } else {
                acc[3] += (uj[0] * tt[0] + uj[1] * tt[1]) + uj[2] * tt[2];
            }
            continue;
        }
        if (P > 1) {
#pragma unroll
            for (int c = 0; c < P; c++) {
                gs[c] = g[c];
                gA[c] = (double)albedo_at<SPLIT>(px, io, albedo, p, c) * gs[c];
            }
        } else {
            gA[0] = gs[0] = 0;
            for (int c = 0; c < C; c++) {
                gA[0] += (double)albedo_at<SPLIT>(px, io, albedo, p, c) * (double)g[c];
                gs[0] += g[c];
            }
        }
        const double aks = SPEC ? ks * (double)spec_map[2 * p] : a * ks;
        const double ep = SPEC ? e * ((double)spec_map[2 * p + 1] / a) : e;
        PointTerm pt;
        point_term(lj, x, n, true, v, aks, ep, pt);
        double alpha = 0, beta = 0, d_b[3] = {0, 0, 0}, n_b[3] = {0, 0, 0}, v_b[3] = {0, 0, 0}, q = 0, e_b = 0;
#pragma unroll
        for (int c = 0; c < P; c++) {
            alpha += gA[c] * lj[3 + c];
            beta += gs[c] * lj[3 + c];
        }
        double vj = 1.0;
        if constexpr (VIS) {
            vj = vis[p * gridDim.x + blockIdx.x];
            alpha = __dmul_rn(alpha, vj);
            beta = __dmul_rn(beta, vj);
        }
        point_term_b(pt, n, alpha, beta, aks, ep, n_b, d_b, v_b, q, e_b);
        for (int k = 0; k < 3; k++) acc[k] += d_b[k];
        const double diff = VIS ? __dmul_rn(pt.diff, vj) : pt.diff, spec = VIS ? __dmul_rn(pt.spec, vj) : pt.spec;
#pragma unroll
        for (int c = 0; c < P; c++) acc[3 + c] += gA[c] * diff + gs[c] * spec;
    }
    grid_sum_rows<K>(acc, s, lights_b);
}

// ---- update -----------------------------------------------------------------------------------------------------

constexpr int MAX_PARAMS = 8;

struct Params {
    DeodrHeavyBall p[MAX_PARAMS];
    int count;
};

// step = clamp(-grad * factor, -max_step, max_step) (np.minimum(np.maximum(.)): NaN stays NaN);
// speed = (1 - damping) (speed inertia + (1 - inertia) step);  value += speed
__device__ __forceinline__ double heavy_ball(double value, double *speed, double grad, double factor, double max_step,
                                             double inertia, double damping) {
    double step = -grad * factor;
    step = step < -max_step ? -max_step : (step > max_step ? max_step : step);
    const double sp = (1 - damping) * (*speed * inertia + (1 - inertia) * step);
    *speed = sp;
    return value + sp;
}

__global__ void __launch_bounds__(NT) k_update(DeodrHeavyBall vert, const double *grad_rigid, Params ps, double inertia,
                                               double damping, const double *energy_data, const double *energy_rigid,
                                               double *energy) {
    const long long i = (long long)blockIdx.x * NT + threadIdx.x;
    if (i < vert.size) {
        const double g = vert.grad[i] + (grad_rigid ? grad_rigid[i] : 0.0);
        vert.value[i] = heavy_ball(vert.value[i], vert.speed + i, g, vert.factor, vert.max_step, inertia, damping);
    }
    if (i != 0) return;
    for (int k = 0; k < ps.count; k++) {
        const DeodrHeavyBall &p = ps.p[k];
        for (int j = 0; j < p.size; j++)
            p.value[j] = heavy_ball(p.value[j], p.speed + j, p.grad[j], p.factor, p.max_step, inertia, damping);
        if (p.normalize) {
            double n2 = 0;
            for (int j = 0; j < p.size; j++) n2 += p.value[j] * p.value[j];
            const double norm = sqrt(n2);
            for (int j = 0; j < p.size; j++) p.value[j] /= norm;
        }
    }
    if (energy) *energy = *energy_data + *energy_rigid;
}

int check_launch() {
    CUDA_TRY(cudaGetLastError());
    return DEODR_B200_OK;
}

int bad(const char *what) { return set_error(DEODR_B200_EINVAL, "%s", what); }

// the sizes, the channel offsets (the four segments tile [0, C + 7); with a separate albedo, off_albedo is -1 and the
// other three tile [0, 7)) and the buffers both directions read
bool phong_io_ok(const DeodrPhongIO *io, bool split = false) {
    if (!io || io->H < 1 || io->W < 1 || io->C < 1 || io->C > 32760) return false;
    if (!io->channels || !io->params || !io->camera_center || !io->background) return false;
    if (split && io->off_albedo != -1) return false;
    const int K = split ? 7 : io->C + 7;
    const int off[4] = {io->off_albedo, io->off_normal, io->off_position, io->off_coverage};
    const int len[4] = {io->C, 3, 3, 1};
    for (int i = split ? 1 : 0; i < 4; i++) {
        if (off[i] < 0 || off[i] > K - len[i]) return false;
        for (int j = split ? 1 : 0; j < i; j++)
            if (off[i] < off[j] + len[j] && off[j] < off[i] + len[i]) return false;
    }
    return true;
}

// an environment of S channels for C colour channels: grey (S = 1), or one per channel up to 4
bool sh_channels_ok(int S, int C) { return S == 1 || (S == C && S >= 2 && S <= 4); }

template <typename G, int S>
void launch_sh_lit_b(const double *normals, const double *vcol, int n, int C, const double *light, int directional,
                     const double *sh, const void *colors_b, double *normals_b, double *vcol_b, double *light_b,
                     double *sh_b, Scratch *s, cudaStream_t st) {
    // grid_sum beyond MAX_K sums stores gridDim.x partials per sum
    const int g = std::min(reduce_grid(n), MAX_K * MAX_CTAS / (4 + 9 * S));
    k_sh_lit_vertex_colors_b<G, S><<<g, NT, 0, st>>>(normals, vcol, n, C, light, directional, sh,
                                                     static_cast<const G *>(colors_b), normals_b, vcol_b, light_b,
                                                     sh_b, s);
}

template <int S, bool SPLIT = false, bool SUN = false, bool SPEC = false, bool GGX = false>
void launch_phong_b(const DeodrPhongIO &io, const double *sh, double *sh_b, Scratch *s, cudaStream_t st,
                    const float *albedo = nullptr, float *albedo_b = nullptr, const float *sun_vis = nullptr,
                    float *sun_vis_b = nullptr, const float *spec_map = nullptr, float *spec_map_b = nullptr) {
    const long long pixels = (long long)io.H * io.W;
    const int g = reduce_grid(pixels);
    if (io.camera_center_b)
        k_phong_shade_b<true, S, SPLIT, 0, false, SUN, SPEC, GGX><<<g, NT, 0, st>>>(
            io, s, sh, albedo, albedo_b, nullptr, 0, nullptr, nullptr, sun_vis, sun_vis_b, spec_map, spec_map_b);
    else
        k_phong_shade_b<false, S, SPLIT, 0, false, SUN, SPEC, GGX><<<g, NT, 0, st>>>(
            io, s, sh, albedo, albedo_b, nullptr, 0, nullptr, nullptr, sun_vis, sun_vis_b, spec_map, spec_map_b);
    if constexpr (S > 0)
        k_phong_sh_b<S, SPLIT, GGX><<<std::min(g, MAX_K * MAX_CTAS / (9 * S)), NT, 0, st>>>(io, s, sh_b, albedo,
                                                                                           GGX ? spec_map : nullptr);
}

// point lights of P channels for C colour channels: grey (P = 1), or one intensity per channel up to 4
bool light_channels_ok(int P, int C) { return P == 1 || (P == C && P >= 2 && P <= 4); }

// Calls f(S, P) as compile-time constants for the (environment, light) channel pairs that light_channels_ok and
// sh_channels_ok allow together (S = 0: no environment): two coloured ones have the same count.
template <typename F>
void with_point_channels(int S, int P, F &&f) {
#define POINT_CASE(s_, p_)                                                                                          \
    if (S == s_ && P == p_) return f(std::integral_constant<int, s_>{}, std::integral_constant<int, p_>{})
    POINT_CASE(0, 1); POINT_CASE(0, 2); POINT_CASE(0, 3); POINT_CASE(0, 4);
    POINT_CASE(1, 1); POINT_CASE(1, 2); POINT_CASE(1, 3); POINT_CASE(1, 4);
    POINT_CASE(2, 1); POINT_CASE(2, 2); POINT_CASE(3, 1); POINT_CASE(3, 3); POINT_CASE(4, 1); POINT_CASE(4, 4);
#undef POINT_CASE
}

// Calls f(S) with S from 0 to 4 as a compile-time constant (S = 0: no environment)
template <typename F>
void with_sh_channels(int S, F &&f) {
    switch (S) {
        case 0: return f(std::integral_constant<int, 0>{});
        case 1: return f(std::integral_constant<int, 1>{});
        case 2: return f(std::integral_constant<int, 2>{});
        case 3: return f(std::integral_constant<int, 3>{});
        default: return f(std::integral_constant<int, 4>{});
    }
}

// Calls f(b) with b as a compile-time constant
template <typename F>
void with_flag(bool b, F &&f) {
    if (b) return f(std::true_type{});
    return f(std::false_type{});
}

// the grid of a (L lights) x (CTAs per light) light sum over `items` items: at most MAX_K * MAX_CTAS partials
dim3 light_grid(long long items, int L, int P) {
    return dim3(L, std::max(1, std::min(reduce_grid(items), MAX_K * MAX_CTAS / (L * (3 + P)))));
}

template <int S, int P, bool SPLIT, bool VIS = false, bool SUN = false, bool SPEC = false, bool GGX = false>
void launch_point_phong_b(const DeodrPhongIO &io, const float *albedo, float *albedo_b, const double *sh,
                          double *sh_b, const double *lights, int L, double *lights_b, Scratch *s, cudaStream_t st,
                          const float *vis = nullptr, float *vis_b = nullptr, const float *sun_vis = nullptr,
                          float *sun_vis_b = nullptr, const float *spec_map = nullptr, float *spec_map_b = nullptr) {
    const long long pixels = (long long)io.H * io.W;
    const int g = reduce_grid(pixels);
    if (io.camera_center_b)
        k_phong_shade_b<true, S, SPLIT, P, VIS, SUN, SPEC, GGX><<<g, NT, 0, st>>>(io, s, sh, albedo, albedo_b, lights,
                                                                                  L, vis, vis_b, sun_vis, sun_vis_b,
                                                                                  spec_map, spec_map_b);
    else
        k_phong_shade_b<false, S, SPLIT, P, VIS, SUN, SPEC, GGX><<<g, NT, 0, st>>>(io, s, sh, albedo, albedo_b, lights,
                                                                                   L, vis, vis_b, sun_vis, sun_vis_b,
                                                                                   spec_map, spec_map_b);
    if constexpr (S > 0)
        k_phong_sh_b<S, SPLIT, GGX><<<std::min(g, MAX_K * MAX_CTAS / (9 * S)), NT, 0, st>>>(io, s, sh_b, albedo,
                                                                                           GGX ? spec_map : nullptr);
    k_point_lights_pixel_b<P, SPLIT, VIS, SPEC, GGX><<<light_grid(pixels, L, P), NT, 0, st>>>(
        io, albedo, lights, lights_b, s, vis, spec_map);
}

}  // namespace

extern "C" {

int64_t deodr_b200_fitter_scratch_bytes(void) { return (int64_t)sizeof(Scratch); }

int deodr_b200_pose(double *vertices, int n, const double *quaternion, const double *translation, double *transformed,
                    double *scratch, void *stream) {
    if (n < 1 || !vertices || !quaternion || !translation || !transformed || !scratch)
        return bad("pose: bad argument (n >= 1 and every pointer non-NULL)");
    cudaStream_t st = (cudaStream_t)stream;
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    k_mean<<<reduce_grid(n), NT, 0, st>>>(vertices, n, s);
    k_pose<<<grid_of(n), NT, 0, st>>>(vertices, n, quaternion, translation, s, transformed);
    return check_launch();
}

int deodr_b200_pose_b(const double *vertices, int n, const double *quaternion, const double *transformed_b,
                      double *vertices_b, double *quaternion_b, double *translation_b, double *scratch, void *stream) {
    if (n < 1 || !vertices || !quaternion || !transformed_b || !vertices_b || !quaternion_b || !translation_b || !scratch)
        return bad("pose_b: bad argument (n >= 1 and every pointer non-NULL)");
    cudaStream_t st = (cudaStream_t)stream;
    k_pose_b<<<reduce_grid(n), NT, 0, st>>>(vertices, n, quaternion, transformed_b, quaternion_b, translation_b,
                                            reinterpret_cast<Scratch *>(scratch));
    k_pose_b_vertices<<<grid_of(n), NT, 0, st>>>(n, quaternion, transformed_b, translation_b, vertices_b);
    return check_launch();
}

int deodr_b200_pose_frames(double *vertices, int n, const double *quaternions, const double *translations,
                           int nb_frames, double *transformed, double *scratch, void *stream) {
    if (n < 1 || nb_frames < 1 || !vertices || !quaternions || !translations || !transformed || !scratch)
        return bad("pose_frames: bad argument (n >= 1, nb_frames >= 1 and every pointer non-NULL)");
    cudaStream_t st = (cudaStream_t)stream;
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    k_mean<<<reduce_grid(n), NT, 0, st>>>(vertices, n, s);
    k_pose_frames<<<grid_of(n), NT, 0, st>>>(vertices, n, quaternions, translations, nb_frames, s, transformed);
    return check_launch();
}

int deodr_b200_pose_frames_b(const double *vertices, int n, const double *quaternions, const double *transformed_b,
                             int nb_frames, int center_vertices_b, double scale, const double *losses,
                             double *energy_data, double *vertices_b, double *quaternions_b, double *translations_b,
                             double *scratch, void *stream) {
    if (n < 1 || nb_frames < 1 || !vertices || !quaternions || !transformed_b || !vertices_b || !quaternions_b ||
        !translations_b || !scratch || (!losses != !energy_data))
        return bad("pose_frames_b: bad argument (n >= 1, nb_frames >= 1, every array non-NULL; losses and energy_data "
                   "both given or both NULL)");
    if (nb_frames > MAX_FRAMES)
        return set_error(DEODR_B200_EUNSUPPORTED, "pose_frames_b: at most 2340 frames (MAX_FRAMES)");
    cudaStream_t st = (cudaStream_t)stream;
    const int per_frame = std::max(1, std::min(reduce_grid(n), MAX_K * MAX_CTAS / (POSE_SUMS * nb_frames)));
    k_pose_frames_b<<<dim3(per_frame, nb_frames), NT, 0, st>>>(vertices, n, quaternions, transformed_b, scale, losses,
                                                               energy_data, quaternions_b, translations_b,
                                                               reinterpret_cast<Scratch *>(scratch));
    k_pose_frames_b_vertices<<<grid_of(n), NT, 0, st>>>(n, quaternions, transformed_b, nb_frames, scale,
                                                        center_vertices_b, translations_b, vertices_b);
    return check_launch();
}

int deodr_b200_laplacian_rigid(const int32_t *neighbour_offset,const int32_t *neighbour_index, int n,
                               const double *vertices, const double *vertices_ref, double cregu, double *grad,
                               double *energy, double *vertex_scratch, double *scratch, void *stream) {
    if (n < 1 || !neighbour_offset || !neighbour_index || !vertices || !vertices_ref || !grad || !energy ||
        !vertex_scratch || !scratch)
        return bad("laplacian_rigid: bad argument (n >= 1 and every pointer non-NULL)");
    cudaStream_t st = (cudaStream_t)stream;
    k_laplacian1<<<grid_of(n), NT, 0, st>>>(neighbour_offset, neighbour_index, n, vertices, vertices_ref, vertex_scratch);
    k_laplacian2<<<reduce_grid(n), NT, 0, st>>>(neighbour_offset, neighbour_index, n, vertices, vertices_ref,
                                                vertex_scratch, cregu, grad, energy, reinterpret_cast<Scratch *>(scratch));
    return check_launch();
}

int deodr_b200_depth_compare(const float *render, const double *obs, int64_t pixels, double max_depth, double *depth,
                             double *diff, float *depth_b, double *energy, double *scratch, void *stream) {
    if (pixels < 1 || !render || !obs || !depth_b || !energy || !scratch)
        return bad("depth_compare: bad argument (pixels >= 1; render, obs, depth_b, energy, scratch non-NULL)");
    k_depth_compare<<<reduce_grid(pixels), NT, 0, (cudaStream_t)stream>>>(
        render, obs, pixels, max_depth, depth, diff, depth_b, energy, reinterpret_cast<Scratch *>(scratch));
    return check_launch();
}

int deodr_b200_uniform_color_luminosity(const double *normals, int n, const double *color, int nb_colors,
                                        const double *light, float *colors, void *stream) {
    if (n < 1 || nb_colors < 1 || !normals || !color || !light || !colors)
        return bad("uniform_color_luminosity: bad argument");
    k_uniform_luminosity<<<grid_of(n), NT, 0, (cudaStream_t)stream>>>(normals, n, color, nb_colors, light, colors);
    return check_launch();
}

int deodr_b200_uniform_color_luminosity_b(const double *normals, int n, const double *color, int nb_colors,
                                          const double *light, const float *colors_b, double *normals_b,
                                          double *color_b, double *light_b, double *scratch, void *stream) {
    if (n < 1 || !normals || !color || !light || !colors_b || !color_b || !light_b || !scratch)
        return bad("uniform_color_luminosity_b: bad argument");
    if (nb_colors < 1 || nb_colors > 4)
        return set_error(DEODR_B200_EUNSUPPORTED, "uniform_color_luminosity_b: nb_colors must be 1 to 4");
    cudaStream_t st = (cudaStream_t)stream;
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    const int g = reduce_grid(n);
    switch (nb_colors) {
        case 1: k_uniform_luminosity_b<1><<<g, NT, 0, st>>>(normals, n, color, light, colors_b, normals_b, color_b, light_b, s); break;
        case 2: k_uniform_luminosity_b<2><<<g, NT, 0, st>>>(normals, n, color, light, colors_b, normals_b, color_b, light_b, s); break;
        case 3: k_uniform_luminosity_b<3><<<g, NT, 0, st>>>(normals, n, color, light, colors_b, normals_b, color_b, light_b, s); break;
        default: k_uniform_luminosity_b<4><<<g, NT, 0, st>>>(normals, n, color, light, colors_b, normals_b, color_b, light_b, s); break;
    }
    return check_launch();
}

int deodr_b200_lit_vertex_colors(const double *normals, const double *vertex_colors, int n, int nb_colors,
                                 const double *light, int directional, double *colors, void *stream) {
    if (n < 0 || nb_colors < 1 || (n > 0 && (!normals || !vertex_colors || !light || !colors)))
        return bad("lit_vertex_colors: bad argument (n >= 0, nb_colors >= 1, every pointer non-NULL)");
    if (n == 0) return DEODR_B200_OK;
    k_lit_vertex_colors<<<grid_of(n), NT, 0, (cudaStream_t)stream>>>(normals, vertex_colors, n, nb_colors, light,
                                                                     directional, colors);
    return check_launch();
}

int deodr_b200_lit_vertex_colors_b(const double *normals, const double *vertex_colors, int n, int nb_colors,
                                   const double *light, int directional, const void *colors_b, int colors_b_fp64,
                                   double *normals_b, double *vertex_colors_b, double *light_b, double *scratch,
                                   void *stream) {
    if (n < 1 || nb_colors < 1 || !normals || !vertex_colors || !light || !colors_b || !normals_b ||
        !vertex_colors_b || !light_b || !scratch)
        return bad("lit_vertex_colors_b: bad argument (n >= 1, nb_colors >= 1, every pointer non-NULL)");
    cudaStream_t st = (cudaStream_t)stream;
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    const int g = reduce_grid(n);
    if (colors_b_fp64)
        k_lit_vertex_colors_b<double><<<g, NT, 0, st>>>(normals, vertex_colors, n, nb_colors, light, directional,
                                                        static_cast<const double *>(colors_b), normals_b,
                                                        vertex_colors_b, light_b, s);
    else
        k_lit_vertex_colors_b<float><<<g, NT, 0, st>>>(normals, vertex_colors, n, nb_colors, light, directional,
                                                       static_cast<const float *>(colors_b), normals_b,
                                                       vertex_colors_b, light_b, s);
    return check_launch();
}

int deodr_b200_sh_lit_vertex_colors(const double *normals, const double *vertex_colors, int n, int nb_colors,
                                    const double *light, int directional, const double *sh, int sh_channels,
                                    double *colors, void *stream) {
    if (n < 0 || nb_colors < 1 || (!vertex_colors && nb_colors != 1) ||
        (n > 0 && (!normals || !light || !sh || !colors)))
        return bad("sh_lit_vertex_colors: bad argument (n >= 0, nb_colors >= 1 (1 without vertex_colors), normals, "
                   "light, sh and colors non-NULL)");
    if (!sh_channels_ok(sh_channels, vertex_colors ? nb_colors : 1))
        return set_error(DEODR_B200_EUNSUPPORTED, "sh_lit_vertex_colors: sh_channels must be 1, or nb_colors from 1 "
                                                  "to 4 with vertex_colors");
    if (n == 0) return DEODR_B200_OK;
    const int g = grid_of(n);
    cudaStream_t st = (cudaStream_t)stream;
    switch (sh_channels) {
        case 1: k_sh_lit_vertex_colors<1><<<g, NT, 0, st>>>(normals, vertex_colors, n, nb_colors, light, directional, sh, colors); break;
        case 2: k_sh_lit_vertex_colors<2><<<g, NT, 0, st>>>(normals, vertex_colors, n, nb_colors, light, directional, sh, colors); break;
        case 3: k_sh_lit_vertex_colors<3><<<g, NT, 0, st>>>(normals, vertex_colors, n, nb_colors, light, directional, sh, colors); break;
        default: k_sh_lit_vertex_colors<4><<<g, NT, 0, st>>>(normals, vertex_colors, n, nb_colors, light, directional, sh, colors); break;
    }
    return check_launch();
}

int deodr_b200_sh_lit_vertex_colors_b(const double *normals, const double *vertex_colors, int n, int nb_colors,
                                      const double *light, int directional, const double *sh, int sh_channels,
                                      const void *colors_b, int colors_b_fp64, double *normals_b,
                                      double *vertex_colors_b, double *light_b, double *sh_b, double *scratch,
                                      void *stream) {
    if (n < 1 || nb_colors < 1 || (!vertex_colors && nb_colors != 1) || !normals || !light || !sh || !colors_b ||
        !normals_b || (vertex_colors && !vertex_colors_b) || !light_b || !sh_b || !scratch)
        return bad("sh_lit_vertex_colors_b: bad argument (n >= 1, nb_colors >= 1 (1 without vertex_colors), every "
                   "pointer non-NULL but vertex_colors_b without vertex_colors)");
    if (!sh_channels_ok(sh_channels, vertex_colors ? nb_colors : 1))
        return set_error(DEODR_B200_EUNSUPPORTED, "sh_lit_vertex_colors_b: sh_channels must be 1, or nb_colors from "
                                                  "1 to 4 with vertex_colors");
    cudaStream_t st = (cudaStream_t)stream;
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
#define SH_LIT_B(G, S)                                                                                              \
    launch_sh_lit_b<G, S>(normals, vertex_colors, n, nb_colors, light, directional, sh, colors_b, normals_b,     \
                          vertex_colors_b, light_b, sh_b, s, st)
    if (colors_b_fp64) {
        switch (sh_channels) {
            case 1: SH_LIT_B(double, 1); break;
            case 2: SH_LIT_B(double, 2); break;
            case 3: SH_LIT_B(double, 3); break;
            default: SH_LIT_B(double, 4); break;
        }
    } else {
        switch (sh_channels) {
            case 1: SH_LIT_B(float, 1); break;
            case 2: SH_LIT_B(float, 2); break;
            case 3: SH_LIT_B(float, 3); break;
            default: SH_LIT_B(float, 4); break;
        }
    }
#undef SH_LIT_B
    return check_launch();
}

int deodr_b200_phong_shade(const DeodrPhongIO *io, void *stream) {
    if (!phong_io_ok(io) || !io->image)
        return bad("phong_shade: bad argument (H, W >= 1, C in [1, 32760], offsets tiling [0, C + 7), channels, "
                   "params, camera_center, background and image non-NULL)");
    k_phong_shade<0, false><<<grid_of((long long)io->H * io->W), NT, 0, (cudaStream_t)stream>>>(*io, nullptr,
                                                                                                 nullptr, nullptr, 0);
    return check_launch();
}

int deodr_b200_phong_shade_b(const DeodrPhongIO *io, double *scratch, void *stream) {
    if (!phong_io_ok(io) || !io->image_b || !io->channels_b || !io->params_b || !scratch)
        return bad("phong_shade_b: bad argument (H, W >= 1, C in [1, 32760], offsets tiling [0, C + 7), channels, "
                   "params, camera_center, background, image_b, channels_b, params_b and scratch non-NULL)");
    launch_phong_b<0>(*io, nullptr, nullptr, reinterpret_cast<Scratch *>(scratch), (cudaStream_t)stream);
    return check_launch();
}

int deodr_b200_sh_phong_shade(const DeodrPhongIO *io, const double *sh, int sh_channels, void *stream) {
    if (!phong_io_ok(io) || !io->image || !sh)
        return bad("sh_phong_shade: bad argument (H, W >= 1, C in [1, 32760], offsets tiling [0, C + 7), channels, "
                   "params, camera_center, background, image and sh non-NULL)");
    if (!sh_channels_ok(sh_channels, io->C))
        return set_error(DEODR_B200_EUNSUPPORTED, "sh_phong_shade: sh_channels must be 1, or C from 1 to 4");
    const int g = grid_of((long long)io->H * io->W);
    cudaStream_t st = (cudaStream_t)stream;
    switch (sh_channels) {
        case 1: k_phong_shade<1, false><<<g, NT, 0, st>>>(*io, sh, nullptr, nullptr, 0); break;
        case 2: k_phong_shade<2, false><<<g, NT, 0, st>>>(*io, sh, nullptr, nullptr, 0); break;
        case 3: k_phong_shade<3, false><<<g, NT, 0, st>>>(*io, sh, nullptr, nullptr, 0); break;
        default: k_phong_shade<4, false><<<g, NT, 0, st>>>(*io, sh, nullptr, nullptr, 0); break;
    }
    return check_launch();
}

int deodr_b200_sh_phong_shade_b(const DeodrPhongIO *io, const double *sh, int sh_channels, double *sh_b,
                                double *scratch, void *stream) {
    if (!phong_io_ok(io) || !io->image_b || !io->channels_b || !io->params_b || !sh || !sh_b || !scratch)
        return bad("sh_phong_shade_b: bad argument (H, W >= 1, C in [1, 32760], offsets tiling [0, C + 7), channels, "
                   "params, camera_center, background, image_b, channels_b, params_b, sh, sh_b and scratch non-NULL)");
    if (!sh_channels_ok(sh_channels, io->C))
        return set_error(DEODR_B200_EUNSUPPORTED, "sh_phong_shade_b: sh_channels must be 1, or C from 1 to 4");
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    cudaStream_t st = (cudaStream_t)stream;
    switch (sh_channels) {
        case 1: launch_phong_b<1>(*io, sh, sh_b, s, st); break;
        case 2: launch_phong_b<2>(*io, sh, sh_b, s, st); break;
        case 3: launch_phong_b<3>(*io, sh, sh_b, s, st); break;
        default: launch_phong_b<4>(*io, sh, sh_b, s, st); break;
    }
    return check_launch();
}

int deodr_b200_phong_shade_albedo(const DeodrPhongIO *io, const float *albedo, const double *sh, int sh_channels,
                                  void *stream) {
    if (!phong_io_ok(io, true) || !io->image || !albedo || (!sh && sh_channels != 0))
        return bad("phong_shade_albedo: bad argument (H, W >= 1, C in [1, 32760], off_albedo -1 and the other offsets "
                   "tiling [0, 7), channels, params, camera_center, background, image and albedo non-NULL, sh NULL "
                   "only with sh_channels 0)");
    if (sh && !sh_channels_ok(sh_channels, io->C))
        return set_error(DEODR_B200_EUNSUPPORTED, "phong_shade_albedo: sh_channels must be 1, or C from 1 to 4");
    const int g = grid_of((long long)io->H * io->W);
    cudaStream_t st = (cudaStream_t)stream;
    switch (sh ? sh_channels : 0) {
        case 0: k_phong_shade<0, true><<<g, NT, 0, st>>>(*io, nullptr, albedo, nullptr, 0); break;
        case 1: k_phong_shade<1, true><<<g, NT, 0, st>>>(*io, sh, albedo, nullptr, 0); break;
        case 2: k_phong_shade<2, true><<<g, NT, 0, st>>>(*io, sh, albedo, nullptr, 0); break;
        case 3: k_phong_shade<3, true><<<g, NT, 0, st>>>(*io, sh, albedo, nullptr, 0); break;
        default: k_phong_shade<4, true><<<g, NT, 0, st>>>(*io, sh, albedo, nullptr, 0); break;
    }
    return check_launch();
}

int deodr_b200_phong_shade_albedo_b(const DeodrPhongIO *io, const float *albedo, float *albedo_b, const double *sh,
                                    int sh_channels, double *sh_b, double *scratch, void *stream) {
    if (!phong_io_ok(io, true) || !io->image_b || !io->channels_b || !io->params_b || !albedo || !albedo_b ||
        !scratch || (!sh && sh_channels != 0) || (sh && !sh_b))
        return bad("phong_shade_albedo_b: bad argument (H, W >= 1, C in [1, 32760], off_albedo -1 and the other "
                   "offsets tiling [0, 7), channels, params, camera_center, background, image_b, channels_b, params_b, "
                   "albedo, albedo_b and scratch non-NULL, sh NULL only with sh_channels 0, sh_b non-NULL with sh)");
    if (sh && !sh_channels_ok(sh_channels, io->C))
        return set_error(DEODR_B200_EUNSUPPORTED, "phong_shade_albedo_b: sh_channels must be 1, or C from 1 to 4");
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    cudaStream_t st = (cudaStream_t)stream;
    switch (sh ? sh_channels : 0) {
        case 0: launch_phong_b<0, true>(*io, nullptr, nullptr, s, st, albedo, albedo_b); break;
        case 1: launch_phong_b<1, true>(*io, sh, sh_b, s, st, albedo, albedo_b); break;
        case 2: launch_phong_b<2, true>(*io, sh, sh_b, s, st, albedo, albedo_b); break;
        case 3: launch_phong_b<3, true>(*io, sh, sh_b, s, st, albedo, albedo_b); break;
        default: launch_phong_b<4, true>(*io, sh, sh_b, s, st, albedo, albedo_b); break;
    }
    return check_launch();
}

int deodr_b200_point_lit_vertex_colors(const double *normals, const double *positions, const double *vertex_colors,
                                       int n, int nb_colors, const double *light, int directional, const double *sh,
                                       int sh_channels, const double *lights, int nb_lights, int light_channels,
                                       double *colors, void *stream) {
    if (n < 0 || nb_colors < 1 || (!vertex_colors && nb_colors != 1) || (!sh && sh_channels != 0) ||
        (n > 0 && (!normals || !positions || !light || !lights || !colors)))
        return bad("point_lit_vertex_colors: bad argument (n >= 0, nb_colors >= 1 (1 without vertex_colors), "
                   "normals, positions, light, lights and colors non-NULL, sh NULL only with sh_channels 0)");
    const int C = vertex_colors ? nb_colors : 1;
    if ((sh && !sh_channels_ok(sh_channels, C)) || !light_channels_ok(light_channels, C) || nb_lights < 1 ||
        nb_lights > MAX_LIGHTS)
        return set_error(DEODR_B200_EUNSUPPORTED, "point_lit_vertex_colors: nb_lights must be 1 to 8, and "
                                                  "sh_channels and light_channels 1, or nb_colors from 1 to 4 with "
                                                  "vertex_colors");
    if (n == 0) return DEODR_B200_OK;
    const int g = grid_of(n);
    cudaStream_t st = (cudaStream_t)stream;
    with_point_channels(sh ? sh_channels : 0, light_channels, [&](auto S, auto P) {
        k_point_lit_vertex_colors<S, P><<<g, NT, 0, st>>>(normals, positions, vertex_colors, n, nb_colors, light,
                                                          directional, sh, lights, nb_lights, colors);
    });
    return check_launch();
}

int deodr_b200_point_lit_vertex_colors_b(const double *normals, const double *positions, const double *vertex_colors,
                                         int n, int nb_colors, const double *light, int directional, const double *sh,
                                         int sh_channels, const double *lights, int nb_lights, int light_channels,
                                         const void *colors_b, int colors_b_fp64, double *normals_b,
                                         double *positions_b, double *vertex_colors_b, double *light_b, double *sh_b,
                                         double *lights_b, double *scratch, void *stream) {
    if (n < 1 || nb_colors < 1 || (!vertex_colors && nb_colors != 1) || (!sh && sh_channels != 0) || !normals ||
        !positions || !light || !lights || !colors_b || !normals_b || !positions_b ||
        (vertex_colors && !vertex_colors_b) || !light_b || (sh && !sh_b) || !lights_b || !scratch)
        return bad("point_lit_vertex_colors_b: bad argument (n >= 1, nb_colors >= 1 (1 without vertex_colors), every "
                   "pointer non-NULL but vertex_colors_b without vertex_colors and sh, sh_b without an environment; "
                   "sh NULL only with sh_channels 0)");
    const int C = vertex_colors ? nb_colors : 1;
    if ((sh && !sh_channels_ok(sh_channels, C)) || !light_channels_ok(light_channels, C) || nb_lights < 1 ||
        nb_lights > MAX_LIGHTS)
        return set_error(DEODR_B200_EUNSUPPORTED, "point_lit_vertex_colors_b: nb_lights must be 1 to 8, and "
                                                  "sh_channels and light_channels 1, or nb_colors from 1 to 4 with "
                                                  "vertex_colors");
    cudaStream_t st = (cudaStream_t)stream;
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    const int S_ = sh ? sh_channels : 0;
    auto launch = [&](auto G_, auto S, auto P) {
        using G = decltype(G_);
        const G *cb = static_cast<const G *>(colors_b);
        // grid_sum beyond MAX_K sums stores gridDim.x partials per sum
        const int g = std::min(reduce_grid(n), MAX_K * MAX_CTAS / (4 + 9 * S));
        k_point_lit_vertex_colors_b<G, S, P><<<g, NT, 0, st>>>(normals, positions, vertex_colors, n, nb_colors, light,
                                                               directional, sh, lights, nb_lights, cb, normals_b,
                                                               positions_b, vertex_colors_b, light_b, sh_b, s);
        k_point_lights_vertex_b<G, P><<<light_grid(n, nb_lights, P), NT, 0, st>>>(
            normals, positions, vertex_colors, n, nb_colors, lights, cb, lights_b, s);
    };
    if (colors_b_fp64)
        with_point_channels(S_, light_channels, [&](auto S, auto P) { launch(double(), S, P); });
    else
        with_point_channels(S_, light_channels, [&](auto S, auto P) { launch(float(), S, P); });
    return check_launch();
}

int deodr_b200_point_phong_shade(const DeodrPhongIO *io, const float *albedo, const double *sh, int sh_channels,
                                 const double *lights, int nb_lights, int light_channels, void *stream) {
    if (!phong_io_ok(io, albedo != nullptr) || !io->image || (!sh && sh_channels != 0) || !lights)
        return bad("point_phong_shade: bad argument (H, W >= 1, C in [1, 32760], offsets tiling [0, C + 7), or [0, 7) "
                   "with off_albedo -1 and an albedo, channels, params, camera_center, background, image and lights "
                   "non-NULL, sh NULL only with sh_channels 0)");
    if ((sh && !sh_channels_ok(sh_channels, io->C)) || !light_channels_ok(light_channels, io->C) || nb_lights < 1 ||
        nb_lights > MAX_LIGHTS)
        return set_error(DEODR_B200_EUNSUPPORTED, "point_phong_shade: nb_lights must be 1 to 8, and sh_channels and "
                                                  "light_channels 1, or C from 1 to 4");
    const int g = grid_of((long long)io->H * io->W);
    cudaStream_t st = (cudaStream_t)stream;
    with_point_channels(sh ? sh_channels : 0, light_channels, [&](auto S, auto P) {
        if (albedo)
            k_phong_shade<S, true, P><<<g, NT, 0, st>>>(*io, sh, albedo, lights, nb_lights);
        else
            k_phong_shade<S, false, P><<<g, NT, 0, st>>>(*io, sh, nullptr, lights, nb_lights);
    });
    return check_launch();
}

int deodr_b200_point_phong_shade_b(const DeodrPhongIO *io, const float *albedo, float *albedo_b, const double *sh,
                                   int sh_channels, double *sh_b, const double *lights, int nb_lights,
                                   int light_channels, double *lights_b, double *scratch, void *stream) {
    if (!phong_io_ok(io, albedo != nullptr) || !io->image_b || !io->channels_b || !io->params_b ||
        (albedo && !albedo_b) || (!sh && sh_channels != 0) || (sh && !sh_b) || !lights || !lights_b || !scratch)
        return bad("point_phong_shade_b: bad argument (H, W >= 1, C in [1, 32760], offsets tiling [0, C + 7), or "
                   "[0, 7) with off_albedo -1 and an albedo, channels, params, camera_center, background, image_b, "
                   "channels_b, params_b, lights, lights_b and scratch non-NULL, albedo_b non-NULL with an albedo, sh "
                   "NULL only with sh_channels 0, sh_b non-NULL with sh)");
    if ((sh && !sh_channels_ok(sh_channels, io->C)) || !light_channels_ok(light_channels, io->C) || nb_lights < 1 ||
        nb_lights > MAX_LIGHTS)
        return set_error(DEODR_B200_EUNSUPPORTED, "point_phong_shade_b: nb_lights must be 1 to 8, and sh_channels and "
                                                  "light_channels 1, or C from 1 to 4");
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    cudaStream_t st = (cudaStream_t)stream;
    with_point_channels(sh ? sh_channels : 0, light_channels, [&](auto S, auto P) {
        if (albedo)
            launch_point_phong_b<S, P, true>(*io, albedo, albedo_b, sh, sh_b, lights, nb_lights, lights_b, s, st);
        else
            launch_point_phong_b<S, P, false>(*io, nullptr, nullptr, sh, sh_b, lights, nb_lights, lights_b, s, st);
    });
    return check_launch();
}

int deodr_b200_point_phong_shade_shadowed(const DeodrPhongIO *io, const float *albedo, const double *sh,
                                          int sh_channels, const double *lights, int nb_lights, int light_channels,
                                          const float *vis, void *stream) {
    if (!phong_io_ok(io, albedo != nullptr) || !io->image || (!sh && sh_channels != 0) || !lights || !vis)
        return bad("point_phong_shade_shadowed: bad argument (H, W >= 1, C in [1, 32760], offsets tiling [0, C + 7), "
                   "or [0, 7) with off_albedo -1 and an albedo, channels, params, camera_center, background, image, "
                   "lights and vis non-NULL, sh NULL only with sh_channels 0)");
    if ((sh && !sh_channels_ok(sh_channels, io->C)) || !light_channels_ok(light_channels, io->C) || nb_lights < 1 ||
        nb_lights > MAX_LIGHTS)
        return set_error(DEODR_B200_EUNSUPPORTED, "point_phong_shade_shadowed: nb_lights must be 1 to 8, and "
                                                  "sh_channels and light_channels 1, or C from 1 to 4");
    const int g = grid_of((long long)io->H * io->W);
    cudaStream_t st = (cudaStream_t)stream;
    with_point_channels(sh ? sh_channels : 0, light_channels, [&](auto S, auto P) {
        if (albedo)
            k_phong_shade<S, true, P, true><<<g, NT, 0, st>>>(*io, sh, albedo, lights, nb_lights, vis);
        else
            k_phong_shade<S, false, P, true><<<g, NT, 0, st>>>(*io, sh, nullptr, lights, nb_lights, vis);
    });
    return check_launch();
}

int deodr_b200_point_phong_shade_shadowed_b(const DeodrPhongIO *io, const float *albedo, float *albedo_b,
                                            const double *sh, int sh_channels, double *sh_b, const double *lights,
                                            int nb_lights, int light_channels, double *lights_b, const float *vis,
                                            float *vis_b, double *scratch, void *stream) {
    if (!phong_io_ok(io, albedo != nullptr) || !io->image_b || !io->channels_b || !io->params_b ||
        (albedo && !albedo_b) || (!sh && sh_channels != 0) || (sh && !sh_b) || !lights || !lights_b || !vis ||
        !vis_b || !scratch)
        return bad("point_phong_shade_shadowed_b: bad argument (H, W >= 1, C in [1, 32760], offsets tiling [0, C + 7), "
                   "or [0, 7) with off_albedo -1 and an albedo, channels, params, camera_center, background, image_b, "
                   "channels_b, params_b, lights, lights_b, vis, vis_b and scratch non-NULL, albedo_b non-NULL with an "
                   "albedo, sh NULL only with sh_channels 0, sh_b non-NULL with sh)");
    if ((sh && !sh_channels_ok(sh_channels, io->C)) || !light_channels_ok(light_channels, io->C) || nb_lights < 1 ||
        nb_lights > MAX_LIGHTS)
        return set_error(DEODR_B200_EUNSUPPORTED, "point_phong_shade_shadowed_b: nb_lights must be 1 to 8, and "
                                                  "sh_channels and light_channels 1, or C from 1 to 4");
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    cudaStream_t st = (cudaStream_t)stream;
    with_point_channels(sh ? sh_channels : 0, light_channels, [&](auto S, auto P) {
        if (albedo)
            launch_point_phong_b<S, P, true, true>(*io, albedo, albedo_b, sh, sh_b, lights, nb_lights, lights_b, s, st,
                                                   vis, vis_b);
        else
            launch_point_phong_b<S, P, false, true>(*io, nullptr, nullptr, sh, sh_b, lights, nb_lights, lights_b, s,
                                                    st, vis, vis_b);
    });
    return check_launch();
}

int deodr_b200_phong_shade_sun_shadowed(const DeodrPhongIO *io, const float *albedo, const double *sh,
                                        int sh_channels, const double *lights, int nb_lights, int light_channels,
                                        const float *vis, const float *sun_vis, void *stream) {
    if (!phong_io_ok(io, albedo != nullptr) || !io->image || (!sh && sh_channels != 0) ||
        (!lights && (nb_lights != 0 || vis)) || !sun_vis)
        return bad("phong_shade_sun_shadowed: bad argument (H, W >= 1, C in [1, 32760], offsets tiling [0, C + 7), "
                   "or [0, 7) with off_albedo -1 and an albedo, channels, params, camera_center, background, image "
                   "and sun_vis non-NULL, sh NULL only with sh_channels 0, lights NULL only with nb_lights 0 and no "
                   "vis)");
    if ((sh && !sh_channels_ok(sh_channels, io->C)) ||
        (lights && (!light_channels_ok(light_channels, io->C) || nb_lights < 1 || nb_lights > MAX_LIGHTS)))
        return set_error(DEODR_B200_EUNSUPPORTED, "phong_shade_sun_shadowed: nb_lights must be 1 to 8, and "
                                                  "sh_channels and light_channels 1, or C from 1 to 4");
    const int g = grid_of((long long)io->H * io->W);
    cudaStream_t st = (cudaStream_t)stream;
    const int S_ = sh ? sh_channels : 0;
    if (!lights) {
        with_sh_channels(S_, [&](auto S) {
            if (albedo)
                k_phong_shade<S, true, 0, false, true><<<g, NT, 0, st>>>(*io, sh, albedo, nullptr, 0, nullptr,
                                                                         sun_vis);
            else
                k_phong_shade<S, false, 0, false, true><<<g, NT, 0, st>>>(*io, sh, nullptr, nullptr, 0, nullptr,
                                                                          sun_vis);
        });
        return check_launch();
    }
    with_point_channels(S_, light_channels, [&](auto S, auto P) {
        with_flag(vis != nullptr, [&](auto VIS) {
            if (albedo)
                k_phong_shade<S, true, P, VIS, true><<<g, NT, 0, st>>>(*io, sh, albedo, lights, nb_lights, vis,
                                                                       sun_vis);
            else
                k_phong_shade<S, false, P, VIS, true><<<g, NT, 0, st>>>(*io, sh, nullptr, lights, nb_lights, vis,
                                                                        sun_vis);
        });
    });
    return check_launch();
}

int deodr_b200_phong_shade_sun_shadowed_b(const DeodrPhongIO *io, const float *albedo, float *albedo_b,
                                          const double *sh, int sh_channels, double *sh_b, const double *lights,
                                          int nb_lights, int light_channels, double *lights_b, const float *vis,
                                          float *vis_b, const float *sun_vis, float *sun_vis_b, double *scratch,
                                          void *stream) {
    if (!phong_io_ok(io, albedo != nullptr) || !io->image_b || !io->channels_b || !io->params_b ||
        (albedo && !albedo_b) || (!sh && sh_channels != 0) || (sh && !sh_b) || (!lights && (nb_lights != 0 || vis)) ||
        (lights && !lights_b) || (vis && !vis_b) || !sun_vis || !sun_vis_b || !scratch)
        return bad("phong_shade_sun_shadowed_b: bad argument (H, W >= 1, C in [1, 32760], offsets tiling [0, C + 7), "
                   "or [0, 7) with off_albedo -1 and an albedo, channels, params, camera_center, background, image_b, "
                   "channels_b, params_b, sun_vis, sun_vis_b and scratch non-NULL, albedo_b non-NULL with an albedo, "
                   "sh NULL only with sh_channels 0, sh_b non-NULL with sh, lights NULL only with nb_lights 0 and no "
                   "vis, lights_b non-NULL with lights, vis_b non-NULL with vis)");
    if ((sh && !sh_channels_ok(sh_channels, io->C)) ||
        (lights && (!light_channels_ok(light_channels, io->C) || nb_lights < 1 || nb_lights > MAX_LIGHTS)))
        return set_error(DEODR_B200_EUNSUPPORTED, "phong_shade_sun_shadowed_b: nb_lights must be 1 to 8, and "
                                                  "sh_channels and light_channels 1, or C from 1 to 4");
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    cudaStream_t st = (cudaStream_t)stream;
    const int S_ = sh ? sh_channels : 0;
    if (!lights) {
        with_sh_channels(S_, [&](auto S) {
            if (albedo)
                launch_phong_b<S, true, true>(*io, sh, sh_b, s, st, albedo, albedo_b, sun_vis, sun_vis_b);
            else
                launch_phong_b<S, false, true>(*io, sh, sh_b, s, st, nullptr, nullptr, sun_vis, sun_vis_b);
        });
        return check_launch();
    }
    with_point_channels(S_, light_channels, [&](auto S, auto P) {
        with_flag(vis != nullptr, [&](auto VIS) {
            if (albedo)
                launch_point_phong_b<S, P, true, VIS, true>(*io, albedo, albedo_b, sh, sh_b, lights, nb_lights,
                                                            lights_b, s, st, vis, vis_b, sun_vis, sun_vis_b);
            else
                launch_point_phong_b<S, P, false, VIS, true>(*io, nullptr, nullptr, sh, sh_b, lights, nb_lights,
                                                             lights_b, s, st, vis, vis_b, sun_vis, sun_vis_b);
        });
    });
    return check_launch();
}

int deodr_b200_phong_shade_specular_map(const DeodrPhongIO *io, const float *albedo, const float *spec,
                                        const double *sh, int sh_channels, const double *lights, int nb_lights,
                                        int light_channels, const float *vis, const float *sun_vis, void *stream) {
    if (!phong_io_ok(io, true) || !io->image || !albedo || !spec || (!sh && sh_channels != 0) ||
        (!lights && (nb_lights != 0 || vis)))
        return bad("phong_shade_specular_map: bad argument (H, W >= 1, C in [1, 32760], off_albedo -1 and the other "
                   "offsets tiling [0, 7), channels, params, camera_center, background, image, albedo and spec "
                   "non-NULL, sh NULL only with sh_channels 0, lights NULL only with nb_lights 0 and no vis)");
    if ((sh && !sh_channels_ok(sh_channels, io->C)) ||
        (lights && (!light_channels_ok(light_channels, io->C) || nb_lights < 1 || nb_lights > MAX_LIGHTS)))
        return set_error(DEODR_B200_EUNSUPPORTED, "phong_shade_specular_map: nb_lights must be 1 to 8, and "
                                                  "sh_channels and light_channels 1, or C from 1 to 4");
    const int g = grid_of((long long)io->H * io->W);
    cudaStream_t st = (cudaStream_t)stream;
    const int S_ = sh ? sh_channels : 0;
    if (!lights) {
        with_sh_channels(S_, [&](auto S) {
            with_flag(sun_vis != nullptr, [&](auto SUN) {
                k_phong_shade<S, true, 0, false, SUN, true><<<g, NT, 0, st>>>(*io, sh, albedo, nullptr, 0, nullptr,
                                                                              sun_vis, spec);
            });
        });
        return check_launch();
    }
    with_point_channels(S_, light_channels, [&](auto S, auto P) {
        with_flag(vis != nullptr, [&](auto VIS) {
            with_flag(sun_vis != nullptr, [&](auto SUN) {
                k_phong_shade<S, true, P, VIS, SUN, true><<<g, NT, 0, st>>>(*io, sh, albedo, lights, nb_lights, vis,
                                                                            sun_vis, spec);
            });
        });
    });
    return check_launch();
}

int deodr_b200_phong_shade_specular_map_b(const DeodrPhongIO *io, const float *albedo, const float *spec,
                                          const double *sh, int sh_channels, const double *lights, int nb_lights,
                                          int light_channels, const float *vis, const float *sun_vis,
                                          float *albedo_b, float *spec_b, double *sh_b, double *lights_b,
                                          float *vis_b, float *sun_vis_b, double *scratch, void *stream) {
    if (!phong_io_ok(io, true) || !io->image_b || !io->channels_b || !io->params_b || !albedo || !albedo_b ||
        !spec || !spec_b || (!sh && sh_channels != 0) || (sh && !sh_b) || (!lights && (nb_lights != 0 || vis)) ||
        (lights && !lights_b) || (vis && !vis_b) || (sun_vis && !sun_vis_b) || !scratch)
        return bad("phong_shade_specular_map_b: bad argument (H, W >= 1, C in [1, 32760], off_albedo -1 and the "
                   "other offsets tiling [0, 7), channels, params, camera_center, background, image_b, channels_b, "
                   "params_b, albedo, albedo_b, spec, spec_b and scratch non-NULL, sh NULL only with sh_channels 0, "
                   "sh_b non-NULL with sh, lights NULL only with nb_lights 0 and no vis, lights_b non-NULL with "
                   "lights, vis_b with vis, sun_vis_b with sun_vis)");
    if ((sh && !sh_channels_ok(sh_channels, io->C)) ||
        (lights && (!light_channels_ok(light_channels, io->C) || nb_lights < 1 || nb_lights > MAX_LIGHTS)))
        return set_error(DEODR_B200_EUNSUPPORTED, "phong_shade_specular_map_b: nb_lights must be 1 to 8, and "
                                                  "sh_channels and light_channels 1, or C from 1 to 4");
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    cudaStream_t st = (cudaStream_t)stream;
    const int S_ = sh ? sh_channels : 0;
    if (!lights) {
        with_sh_channels(S_, [&](auto S) {
            with_flag(sun_vis != nullptr, [&](auto SUN) {
                launch_phong_b<S, true, SUN, true>(*io, sh, sh_b, s, st, albedo, albedo_b, sun_vis, sun_vis_b, spec,
                                                   spec_b);
            });
        });
        return check_launch();
    }
    with_point_channels(S_, light_channels, [&](auto S, auto P) {
        with_flag(vis != nullptr, [&](auto VIS) {
            with_flag(sun_vis != nullptr, [&](auto SUN) {
                launch_point_phong_b<S, P, true, VIS, SUN, true>(*io, albedo, albedo_b, sh, sh_b, lights, nb_lights,
                                                                 lights_b, s, st, vis, vis_b, sun_vis, sun_vis_b,
                                                                 spec, spec_b);
            });
        });
    });
    return check_launch();
}

int deodr_b200_pbr_shade(const DeodrPhongIO *io, const float *albedo, const float *mr, const double *sh,
                         int sh_channels, const double *lights, int nb_lights, int light_channels, const float *vis,
                         const float *sun_vis, void *stream) {
    if (!phong_io_ok(io, true) || !io->image || !albedo || (!sh && sh_channels != 0) ||
        (!lights && (nb_lights != 0 || vis)))
        return bad("pbr_shade: bad argument (H, W >= 1, C in [1, 32760], off_albedo -1 and the other offsets tiling "
                   "[0, 7), channels, params, camera_center, background, image and albedo non-NULL, sh NULL only "
                   "with sh_channels 0, lights NULL only with nb_lights 0 and no vis)");
    if ((sh && !sh_channels_ok(sh_channels, io->C)) ||
        (lights && (!light_channels_ok(light_channels, io->C) || nb_lights < 1 || nb_lights > MAX_LIGHTS)))
        return set_error(DEODR_B200_EUNSUPPORTED, "pbr_shade: nb_lights must be 1 to 8, and sh_channels and "
                                                  "light_channels 1, or C from 1 to 4");
    const int g = grid_of((long long)io->H * io->W);
    cudaStream_t st = (cudaStream_t)stream;
    const int S_ = sh ? sh_channels : 0;
    if (!lights) {
        with_sh_channels(S_, [&](auto S) {
            with_flag(sun_vis != nullptr, [&](auto SUN) {
                k_phong_shade<S, true, 0, false, SUN, false, true><<<g, NT, 0, st>>>(*io, sh, albedo, nullptr, 0,
                                                                                     nullptr, sun_vis, mr);
            });
        });
        return check_launch();
    }
    with_point_channels(S_, light_channels, [&](auto S, auto P) {
        with_flag(vis != nullptr, [&](auto VIS) {
            with_flag(sun_vis != nullptr, [&](auto SUN) {
                k_phong_shade<S, true, P, VIS, SUN, false, true><<<g, NT, 0, st>>>(*io, sh, albedo, lights,
                                                                                   nb_lights, vis, sun_vis, mr);
            });
        });
    });
    return check_launch();
}

int deodr_b200_pbr_shade_b(const DeodrPhongIO *io, const float *albedo, const float *mr, const double *sh,
                           int sh_channels, const double *lights, int nb_lights, int light_channels, const float *vis,
                           const float *sun_vis, float *albedo_b, float *mr_b, double *sh_b, double *lights_b,
                           float *vis_b, float *sun_vis_b, double *scratch, void *stream) {
    if (!phong_io_ok(io, true) || !io->image_b || !io->channels_b || !io->params_b || !albedo || !albedo_b ||
        (!mr != !mr_b) || (!sh && sh_channels != 0) || (sh && !sh_b) || (!lights && (nb_lights != 0 || vis)) ||
        (lights && !lights_b) || (vis && !vis_b) || (sun_vis && !sun_vis_b) || !scratch)
        return bad("pbr_shade_b: bad argument (H, W >= 1, C in [1, 32760], off_albedo -1 and the other offsets "
                   "tiling [0, 7), channels, params, camera_center, background, image_b, channels_b, params_b, "
                   "albedo, albedo_b and scratch non-NULL, mr_b non-NULL exactly with mr, sh NULL only with "
                   "sh_channels 0, sh_b non-NULL with sh, lights NULL only with nb_lights 0 and no vis, lights_b "
                   "non-NULL with lights, vis_b with vis, sun_vis_b with sun_vis)");
    if ((sh && !sh_channels_ok(sh_channels, io->C)) ||
        (lights && (!light_channels_ok(light_channels, io->C) || nb_lights < 1 || nb_lights > MAX_LIGHTS)))
        return set_error(DEODR_B200_EUNSUPPORTED, "pbr_shade_b: nb_lights must be 1 to 8, and sh_channels and "
                                                  "light_channels 1, or C from 1 to 4");
    Scratch *s = reinterpret_cast<Scratch *>(scratch);
    cudaStream_t st = (cudaStream_t)stream;
    const int S_ = sh ? sh_channels : 0;
    if (!lights) {
        with_sh_channels(S_, [&](auto S) {
            with_flag(sun_vis != nullptr, [&](auto SUN) {
                launch_phong_b<S, true, SUN, false, true>(*io, sh, sh_b, s, st, albedo, albedo_b, sun_vis, sun_vis_b,
                                                          mr, mr_b);
            });
        });
        return check_launch();
    }
    with_point_channels(S_, light_channels, [&](auto S, auto P) {
        with_flag(vis != nullptr, [&](auto VIS) {
            with_flag(sun_vis != nullptr, [&](auto SUN) {
                launch_point_phong_b<S, P, true, VIS, SUN, false, true>(*io, albedo, albedo_b, sh, sh_b, lights,
                                                                        nb_lights, lights_b, s, st, vis, vis_b,
                                                                        sun_vis, sun_vis_b, mr, mr_b);
            });
        });
    });
    return check_launch();
}

int deodr_b200_fitter_update(const DeodrHeavyBall *vertices, const double *grad_rigid, const DeodrHeavyBall *params,
                             int nb_params, double inertia, double damping, const double *energy_data,
                             const double *energy_rigid, double *energy, void *stream) {
    if (!vertices || vertices->size < 0 || (vertices->size > 0 && (!vertices->value || !vertices->speed || !vertices->grad)))
        return bad("fitter_update: bad vertices");
    if (nb_params < 0 || nb_params > MAX_PARAMS || (nb_params > 0 && !params))
        return bad("fitter_update: nb_params must lie in [0, 8]");
    if (energy && (!energy_data || !energy_rigid)) return bad("fitter_update: energy needs energy_data and energy_rigid");
    Params ps;
    ps.count = nb_params;
    for (int k = 0; k < nb_params; k++) {
        const DeodrHeavyBall &p = params[k];
        if (p.size < 0 || (p.size > 0 && (!p.value || !p.speed || !p.grad))) return bad("fitter_update: bad parameter");
        ps.p[k] = p;
    }
    k_update<<<grid_of(vertices->size), NT, 0, (cudaStream_t)stream>>>(*vertices, grad_rigid, ps, inertia, damping,
                                                                       energy_data, energy_rigid, energy);
    return check_launch();
}

}  // extern "C"
