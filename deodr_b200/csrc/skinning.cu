// deodr_b200: linear blend skinning of a mesh by a skeleton, and its adjoint to the rest vertices, the skinning weights
// and the joint rotations, in fp64 on device buffers (include/deodr_b200.h, "Linear blend skinning").
//
// Forward: k_forward_kinematics (one CTA, one thread per joint of a depth level, a barrier per level) writes the
// [J,24] table (Rg, tg, M, b); k_skin (one thread per vertex) blends the K transforms of every vertex.
// Adjoint: k_skin_vertices_b (one thread per vertex) gives vertices_b and weights_b; k_skin_joint_partials (one CTA per
// chunk of a joint's influences) sums (M_b, b_b) over the chunk in a fixed order; k_forward_kinematics_b (one CTA) sums
// every joint's chunk partials in a fixed order (one warp per joint: lane-strided over the chunks, then a shuffle tree)
// and walks the levels back to the roots, each parent gathering its children in the order of the children CSR.  No fp64 atomics anywhere: two calls on the same input give the same bits.
// The vertex kernels are HBM-bound; the table is read through the read-only cache.
#include <cuda_runtime.h>

#include "../../include/deodr_b200.h"
#include "workspace.h"

namespace {

constexpr int BLOCK = 256;
constexpr int CHUNK = DEODR_B200_SKIN_CHUNK;
static_assert(CHUNK == BLOCK, "one thread per entry of a chunk");
constexpr int TABLE = 24;  // Rg [9], tg [3], M [9], b [3] per joint
constexpr int SUMS = 12;   // M_b [9], b_b [3] per joint
// the adjoint's single CTA: at most 512 threads, which leaves it 128 registers (at 1024 it would spill); its level
// loops stride over the joints of a level
constexpr int FK_B_THREADS = 512;
constexpr double TAYLOR_S = 1e-2;  // phi^2 below which a, b and their derivatives come from their series (phi < 0.1)

inline int grid_of(size_t n) { return (int)((n + BLOCK - 1) / BLOCK); }

// a = sin(phi) / phi, b = (1 - cos(phi)) / phi^2 and their derivatives with respect to s = phi^2.  Below TAYLOR_S the
// series up to s^4 (truncation below 1e-17); above, the closed forms, with b = 2 sin^2(phi / 2) / s (no cancellation).
__device__ __forceinline__ void rotation_coefficients(double s, double &a, double &b, double &da, double &db) {
    if (s < TAYLOR_S) {
        a = 1.0 + s * (-1.0 / 6 + s * (1.0 / 120 + s * (-1.0 / 5040 + s * (1.0 / 362880))));
        b = 0.5 + s * (-1.0 / 24 + s * (1.0 / 720 + s * (-1.0 / 40320 + s * (1.0 / 3628800))));
        da = -1.0 / 6 + s * (1.0 / 60 + s * (-1.0 / 1680 + s * (1.0 / 90720 + s * (-1.0 / 7983360))));
        db = -1.0 / 24 + s * (1.0 / 360 + s * (-1.0 / 13440 + s * (1.0 / 907200 + s * (-1.0 / 95800320))));
    } else {
        const double phi = sqrt(s);
        double sn, cs, sh, ch;
        sincos(phi, &sn, &cs);
        sincos(0.5 * phi, &sh, &ch);
        a = sn / phi;
        b = 2.0 * sh * sh / s;
        da = (cs - a) / (2.0 * s);
        db = (0.5 * a - b) / s;
    }
}

// R(theta) = I + a [theta]x + b [theta]x^2 = (1 - b s) I + a [theta]x + b theta theta^T, row-major
__device__ __forceinline__ void rotation(const double t[3], double R[9]) {
    const double s = t[0] * t[0] + t[1] * t[1] + t[2] * t[2];
    double a, b, da, db;
    rotation_coefficients(s, a, b, da, db);
    const double d = 1.0 - b * s;
    R[0] = d + b * t[0] * t[0];        R[1] = b * t[0] * t[1] - a * t[2]; R[2] = b * t[0] * t[2] + a * t[1];
    R[3] = b * t[1] * t[0] + a * t[2]; R[4] = d + b * t[1] * t[1];        R[5] = b * t[1] * t[2] - a * t[0];
    R[6] = b * t[2] * t[0] - a * t[1]; R[7] = b * t[2] * t[1] + a * t[0]; R[8] = d + b * t[2] * t[2];
}

// theta_b = d<G, R(theta)>/dtheta with w = vee(G) = (G21 - G12, G02 - G20, G10 - G01), <G, [theta]x> = w.theta,
// <G, [theta]x^2> = theta^T G theta - s tr G and d[theta]x^2/dtheta_k = e_k theta^T + theta e_k^T - 2 theta_k I:
//   theta_b = 2 da (w.theta) theta + a w + 2 db (theta^T G theta - s tr G) theta + b ((G + G^T) theta - 2 tr G theta)
// At theta = 0 this is w: dR/dtheta_k = [e_k]x.
__device__ __forceinline__ void rotation_b(const double t[3], const double G[9], double out[3]) {
    const double s = t[0] * t[0] + t[1] * t[1] + t[2] * t[2];
    double a, b, da, db;
    rotation_coefficients(s, a, b, da, db);
    const double w[3] = {G[7] - G[5], G[2] - G[6], G[3] - G[1]};
    double sym[3];  // (G + G^T) theta
    for (int m = 0; m < 3; m++)
        sym[m] = (G[3 * m] + G[m]) * t[0] + (G[3 * m + 1] + G[3 + m]) * t[1] + (G[3 * m + 2] + G[6 + m]) * t[2];
    const double tr = G[0] + G[4] + G[8];
    const double wt = w[0] * t[0] + w[1] * t[1] + w[2] * t[2];
    const double tgt = 0.5 * (sym[0] * t[0] + sym[1] * t[1] + sym[2] * t[2]);
    const double c = 2.0 * da * wt + 2.0 * db * (tgt - s * tr) - 2.0 * b * tr;
    for (int k = 0; k < 3; k++) out[k] = c * t[k] + a * w[k] + b * sym[k];
}

// Rg_j = R(theta_j) for a root, else Rg_p R(theta_j);  tg_j = c_j for a root, else tg_p + Rg_p (c_j - c_p);
// M_j = Rg_j, b_j = tg_j - Rg_j c_j.  A parent sits in an earlier level, written before the barrier.
__global__ void __launch_bounds__(DEODR_B200_SKIN_MAX_JOINTS)
    k_forward_kinematics(DeodrSkeleton S, const double *__restrict__ rotations, double *table) {
    for (int l = 0; l < S.nb_levels; l++) {
        for (int q = S.level_offset[l] + threadIdx.x; q < S.level_offset[l + 1]; q += blockDim.x) {
            const int j = S.level_index[q], p = S.parents[j];
            const double t[3] = {rotations[3 * j], rotations[3 * j + 1], rotations[3 * j + 2]};
            const double c[3] = {S.centres[3 * j], S.centres[3 * j + 1], S.centres[3 * j + 2]};
            double R[9], Rg[9], tg[3];
            rotation(t, R);
            if (p < 0) {
                for (int m = 0; m < 9; m++) Rg[m] = R[m];
                for (int m = 0; m < 3; m++) tg[m] = c[m];
            } else {
                const double *P = table + (size_t)TABLE * p;
                const double d[3] = {c[0] - S.centres[3 * p], c[1] - S.centres[3 * p + 1], c[2] - S.centres[3 * p + 2]};
                for (int m = 0; m < 3; m++) {
                    for (int n = 0; n < 3; n++)
                        Rg[3 * m + n] = P[3 * m] * R[n] + P[3 * m + 1] * R[3 + n] + P[3 * m + 2] * R[6 + n];
                    tg[m] = P[9 + m] + (P[3 * m] * d[0] + P[3 * m + 1] * d[1] + P[3 * m + 2] * d[2]);
                }
            }
            double *T = table + (size_t)TABLE * j;
            for (int m = 0; m < 9; m++) T[m] = Rg[m];
            for (int m = 0; m < 3; m++) T[9 + m] = tg[m];
            for (int m = 0; m < 9; m++) T[12 + m] = Rg[m];
            for (int m = 0; m < 3; m++)
                T[21 + m] = tg[m] - (Rg[3 * m] * c[0] + Rg[3 * m + 1] * c[1] + Rg[3 * m + 2] * c[2]);
        }
        __syncthreads();
    }
}

// M_j v + b_j from the table's (M, b), read through the read-only cache
__device__ __forceinline__ void transform(const double *__restrict__ table, int j, const double v[3], double out[3]) {
    const double *T = table + (size_t)TABLE * j + 12;
    for (int m = 0; m < 3; m++)
        out[m] = __ldg(T + 3 * m) * v[0] + __ldg(T + 3 * m + 1) * v[1] + __ldg(T + 3 * m + 2) * v[2] + __ldg(T + 9 + m);
}

// v'_i = sum_k w_ik (M_j v_i + b_j), k ascending
__global__ void k_skin(DeodrSkeleton S, const double *__restrict__ vertices, const double *__restrict__ table,
                       double *__restrict__ skinned) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S.nb_vertices) return;
    const int K = S.nb_influences;
    const double v[3] = {vertices[3 * (size_t)i], vertices[3 * (size_t)i + 1], vertices[3 * (size_t)i + 2]};
    double s[3] = {0.0, 0.0, 0.0};
    for (int k = 0; k < K; k++) {
        const size_t e = (size_t)i * K + k;
        const double w = S.skin_weight[e];
        double x[3];
        transform(table, S.skin_index[e], v, x);
        for (int m = 0; m < 3; m++) s[m] += w * x[m];
    }
    for (int m = 0; m < 3; m++) skinned[3 * (size_t)i + m] = s[m];
}

// vertices_b_i = grad_in_i + sum_k w_ik M_j^T g_i;  weights_b_ik = g_i . (M_j v_i + b_j)
__global__ void k_skin_vertices_b(DeodrSkeleton S, const double *__restrict__ vertices,
                                  const double *__restrict__ table, const double *__restrict__ skinned_b,
                                  const double *grad_in, double *vertices_b, double *__restrict__ weights_b) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S.nb_vertices) return;
    const int K = S.nb_influences;
    const double g[3] = {skinned_b[3 * (size_t)i], skinned_b[3 * (size_t)i + 1], skinned_b[3 * (size_t)i + 2]};
    double v[3] = {0.0, 0.0, 0.0};
    if (weights_b)
        for (int m = 0; m < 3; m++) v[m] = vertices[3 * (size_t)i + m];
    double s[3] = {0.0, 0.0, 0.0};
    for (int k = 0; k < K; k++) {
        const size_t e = (size_t)i * K + k;
        const int j = S.skin_index[e];
        const double w = S.skin_weight[e];
        const double *M = table + (size_t)TABLE * j + 12;
        for (int n = 0; n < 3; n++)
            s[n] += w * (__ldg(M + n) * g[0] + __ldg(M + 3 + n) * g[1] + __ldg(M + 6 + n) * g[2]);
        if (weights_b) {
            double x[3];
            transform(table, j, v, x);
            weights_b[e] = g[0] * x[0] + g[1] * x[1] + g[2] * x[2];
        }
    }
    for (int m = 0; m < 3; m++) {
        const double base = grad_in ? grad_in[3 * (size_t)i + m] : 0.0;
        vertices_b[3 * (size_t)i + m] = base + s[m];
    }
}

// One CTA per chunk of CHUNK consecutive entries i*K+k of a joint's CSR row: the chunk's sums
//   M_b = sum w_ik g_i v_i^T,  b_b = sum w_ik g_i
// reduced in a fixed order (a shuffle tree per warp, then the warps in order) into partials[chunk][12].
__global__ void __launch_bounds__(BLOCK) k_skin_joint_partials(DeodrSkeleton S, const double *__restrict__ vertices,
                                                               const double *__restrict__ skinned_b,
                                                               double *__restrict__ partials) {
    __shared__ double warp_sums[SUMS][BLOCK / 32];
    const int c = blockIdx.x;
    // the last joint whose first chunk is <= c (joints without chunks come before it)
    int lo = 0, hi = S.nb_joints - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (S.chunk_offset[mid] <= c) lo = mid; else hi = mid - 1;
    }
    const int j = lo;
    const int e = S.joint_offset[j] + (c - S.chunk_offset[j]) * CHUNK + threadIdx.x;
    double x[SUMS];
    for (int m = 0; m < SUMS; m++) x[m] = 0.0;
    if (e < S.joint_offset[j + 1]) {
        const int entry = S.joint_entry[e];
        const size_t i = (size_t)(entry / S.nb_influences);
        const double w = S.skin_weight[entry];
        const double wg[3] = {w * skinned_b[3 * i], w * skinned_b[3 * i + 1], w * skinned_b[3 * i + 2]};
        const double v[3] = {vertices[3 * i], vertices[3 * i + 1], vertices[3 * i + 2]};
        for (int m = 0; m < 3; m++) {
            for (int n = 0; n < 3; n++) x[3 * m + n] = wg[m] * v[n];
            x[9 + m] = wg[m];
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int m = 0; m < SUMS; m++) {
        double y = x[m];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) y += __shfl_down_sync(0xffffffffu, y, o);
        if (lane == 0) warp_sums[m][warp] = y;
    }
    __syncthreads();
    if (threadIdx.x < SUMS) {
        double t = 0.0;
        for (int w = 0; w < BLOCK / 32; w++) t += warp_sums[threadIdx.x][w];
        partials[(size_t)c * SUMS + threadIdx.x] = t;
    }
}

// One CTA of up to FK_B_THREADS threads.  First every joint's (M_b, b_b): one warp per joint sums its chunk partials
// in a fixed order, lane-strided over the chunks, then a shuffle tree (not chunk by chunk, but the same order every
// call), and turns them into (Rg_b, tg_b) = (M_b - b_b c_j^T, b_b) in acc[j].  Then the levels from the deepest to the
// roots: joint j adds its children's contributions (children CSR order) to acc[j], writes
//   rotations_b_j = rotation_b(theta_j, Rg_p^T Rg_b)     (Rg_b itself for a root)
// and replaces acc[j] by its contribution to its parent, (Rg_b R_j^T + tg_b (c_j - c_p)^T, tg_b).
__global__ void __launch_bounds__(FK_B_THREADS)
    k_forward_kinematics_b(DeodrSkeleton S, const double *__restrict__ rotations, const double *__restrict__ table,
                           const double *__restrict__ partials, double *acc, double *__restrict__ rotations_b) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
    for (int j = warp; j < S.nb_joints; j += warps) {
        const int c0 = S.chunk_offset[j], c1 = S.chunk_offset[j + 1];
        double x[SUMS];
        for (int m = 0; m < SUMS; m++) x[m] = 0.0;
        for (int c = c0 + lane; c < c1; c += 32)
            for (int m = 0; m < SUMS; m++) x[m] += partials[(size_t)c * SUMS + m];
#pragma unroll
        for (int m = 0; m < SUMS; m++)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) x[m] += __shfl_down_sync(0xffffffffu, x[m], o);
        if (lane == 0) {
            const double *cj = S.centres + 3 * j;
            double *A = acc + (size_t)SUMS * j;
            for (int m = 0; m < 3; m++) {
                for (int n = 0; n < 3; n++) A[3 * m + n] = x[3 * m + n] - x[9 + m] * cj[n];
                A[9 + m] = x[9 + m];
            }
        }
    }
    __syncthreads();
    for (int l = S.nb_levels - 1; l >= 0; l--) {
        for (int q = S.level_offset[l] + threadIdx.x; q < S.level_offset[l + 1]; q += blockDim.x) {
            const int j = S.level_index[q], p = S.parents[j];
            double *A = acc + (size_t)SUMS * j;
            double G[9], tb[3];
            for (int m = 0; m < 9; m++) G[m] = A[m];
            for (int m = 0; m < 3; m++) tb[m] = A[9 + m];
            for (int q2 = S.child_offset[j]; q2 < S.child_offset[j + 1]; q2++) {
                const double *B = acc + (size_t)SUMS * S.child_index[q2];
                for (int m = 0; m < 9; m++) G[m] += B[m];
                for (int m = 0; m < 3; m++) tb[m] += B[9 + m];
            }
            const double t[3] = {rotations[3 * j], rotations[3 * j + 1], rotations[3 * j + 2]};
            double Rb[9];
            if (p < 0) {
                for (int m = 0; m < 9; m++) Rb[m] = G[m];
            } else {
                const double *P = table + (size_t)TABLE * p;  // Rg_p
                for (int m = 0; m < 3; m++)
                    for (int n = 0; n < 3; n++)
                        Rb[3 * m + n] = P[m] * G[n] + P[3 + m] * G[3 + n] + P[6 + m] * G[6 + n];
                double R[9];
                rotation(t, R);
                const double d[3] = {S.centres[3 * j] - S.centres[3 * p], S.centres[3 * j + 1] - S.centres[3 * p + 1],
                                     S.centres[3 * j + 2] - S.centres[3 * p + 2]};
                for (int m = 0; m < 3; m++) {
                    for (int n = 0; n < 3; n++)
                        A[3 * m + n] = G[3 * m] * R[3 * n] + G[3 * m + 1] * R[3 * n + 1] + G[3 * m + 2] * R[3 * n + 2] +
                                       tb[m] * d[n];
                    A[9 + m] = tb[m];
                }
            }
            double out[3];
            rotation_b(t, Rb, out);
            for (int m = 0; m < 3; m++) rotations_b[3 * j + m] = out[m];
        }
        __syncthreads();
    }
}

int check_skeleton(const DeodrSkeleton *S) {
    if (!S) return set_error(DEODR_B200_EINVAL, "bad argument: skeleton == NULL");
    if (!S->parents || !S->centres || !S->level_offset || !S->level_index || !S->child_offset || !S->child_index ||
        !S->skin_index || !S->skin_weight || !S->joint_offset || !S->joint_entry || !S->chunk_offset)
        return set_error(DEODR_B200_EINVAL, "bad argument: a skeleton array is NULL");
    if (S->nb_joints < 1 || S->nb_joints > DEODR_B200_SKIN_MAX_JOINTS || S->nb_vertices < 1 || S->nb_influences < 1 ||
        S->nb_influences > DEODR_B200_SKIN_MAX_INFLUENCES || S->nb_levels < 1 || S->nb_levels > S->nb_joints ||
        S->nb_chunks < 0)
        return set_error(DEODR_B200_EINVAL, "bad argument: skeleton sizes");
    if ((int64_t)S->nb_vertices * S->nb_influences > 0x7fffffff)
        return set_error(DEODR_B200_EUNSUPPORTED, "V * K must fit in int32");
    return DEODR_B200_OK;
}

int block_of_joints(int J) { return (J + 31) / 32 * 32; }

}  // namespace

extern "C" {

int deodr_b200_skin(const DeodrSkeleton *skeleton, const double *vertices, const double *rotations, double *transforms,
                    double *skinned, void *stream) {
    if (int rc = check_skeleton(skeleton)) return rc;
    if (!vertices || !rotations || !transforms || !skinned) return set_error(DEODR_B200_EINVAL, "bad argument");
    const cudaStream_t s = (cudaStream_t)stream;
    k_forward_kinematics<<<1, block_of_joints(skeleton->nb_joints), 0, s>>>(*skeleton, rotations, transforms);
    CUDA_TRY(cudaGetLastError());
    k_skin<<<grid_of(skeleton->nb_vertices), BLOCK, 0, s>>>(*skeleton, vertices, transforms, skinned);
    CUDA_TRY(cudaGetLastError());
    return DEODR_B200_OK;
}

int deodr_b200_skin_b(const DeodrSkeleton *skeleton, const double *vertices, const double *rotations,
                      const double *transforms, const double *skinned_b, const double *grad_in, double *vertices_b,
                      double *weights_b, double *rotations_b, double *scratch, void *stream) {
    if (int rc = check_skeleton(skeleton)) return rc;
    if (!vertices || !rotations || !transforms || !skinned_b || !vertices_b || !rotations_b || !scratch)
        return set_error(DEODR_B200_EINVAL, "bad argument");
    const DeodrSkeleton &S = *skeleton;
    const cudaStream_t s = (cudaStream_t)stream;
    double *partials = scratch, *acc = scratch + (size_t)SUMS * S.nb_chunks;
    k_skin_vertices_b<<<grid_of(S.nb_vertices), BLOCK, 0, s>>>(S, vertices, transforms, skinned_b, grad_in, vertices_b,
                                                               weights_b);
    CUDA_TRY(cudaGetLastError());
    if (S.nb_chunks > 0) {
        k_skin_joint_partials<<<S.nb_chunks, BLOCK, 0, s>>>(S, vertices, skinned_b, partials);
        CUDA_TRY(cudaGetLastError());
    }
    const int fk_threads = min(block_of_joints(S.nb_joints), FK_B_THREADS);
    k_forward_kinematics_b<<<1, fk_threads, 0, s>>>(S, rotations, transforms, partials, acc, rotations_b);
    CUDA_TRY(cudaGetLastError());
    return DEODR_B200_OK;
}

}  // extern "C"
