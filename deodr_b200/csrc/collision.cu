// deodr_b200: self-collision energy with its gradient, and self-intersection detection (include/deodr_b200.h,
// "Self-collision").
//
// One call runs, on the caller's stream:
//   k_bounds      bounding box of the finite vertices (fixed grid reduction) -> the grid: origin, cell size, cells per axis
//   k_count       cells of every primitive: a vertex 1, a face or an edge every cell of its inflated bounding box
//   scan          CUB exclusive sum of the counts -> entry offsets; the total goes to pinned memory (the verdict)
//   k_fill        (cell << 2 | type, id) entries, at the offsets, when the total fits the plan's capacity
//   sort          CUB stable radix sort of the entries by key: ids ascending inside every (cell, type)
//   k_vertex      one thread per vertex: its vertex-triangle pairs as the point (energy, point gradient, minimum)
//   k_face        one thread per face: its corners' shares of the same pairs, into per-corner slots [3F,3]
//   k_edge        one thread per edge: its edge-edge pairs, counted at the first cell the two edges share; its two
//                 ends' shares into slots [2E,3], half of every pair's energy
//   k_gather      one thread per vertex: grad_in + point share + corner slots + end slots in CSR order; the energy and
//                 the minimum as fixed-order grid reductions
// Every kernel after k_fill returns at once when the total exceeded the capacity; the host reads the verdict after the
// sort is enqueued, grows the capacity and runs again.  No fp64 atomics: results are reproducible bit for bit.
// The distances round every product and sum on its own (no fused multiply-add), as the fp64 restatement does.
#include <cuda_runtime.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <utility>

#include "../../include/deodr_b200.h"
#include "reduce.cuh"
#include "workspace.h"

namespace {

constexpr int MAX_AXIS = 1024;          // cells per axis
constexpr int64_t MAX_GRID = 1 << 21;   // cells in all: keys (cell << 2 | type) fit in 23 bits
constexpr int KEY_BITS = 24;            // the sort looks at these bits; the padding key 0xffffffff sorts last
enum { T_VERTEX = 0, T_FACE = 1, T_EDGE = 2 };

struct Grid {
    double origin[3];
    double inv_h;
    int n[3];
    int nonfinite;  // a vertex in a face has a non-finite coordinate
};

// the state's scratch: bounds partials, the minimum's partials, the grid, the grid_sum scratch (zeroed at allocation)
struct CollisionScratch {
    Scratch sum;
    double bounds[6 * MAX_CTAS];
    int flags[MAX_CTAS];
    double mins[MAX_CTAS];
    unsigned done;
    Grid grid;
};

// ---- rounded fp64 arithmetic (no contraction) ------------------------------------------------------------------------
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dvd(double a, double b) { return __ddiv_rn(a, b); }

struct V3 {
    double x, y, z;
};
__device__ __forceinline__ V3 load3(const double *v, int i) {
    const double *p = v + 3 * (size_t)i;
    return {p[0], p[1], p[2]};
}
__device__ __forceinline__ V3 vsub(V3 a, V3 b) { return {sub(a.x, b.x), sub(a.y, b.y), sub(a.z, b.z)}; }
__device__ __forceinline__ V3 vadd(V3 a, V3 b) { return {add(a.x, b.x), add(a.y, b.y), add(a.z, b.z)}; }
__device__ __forceinline__ V3 vscale(V3 a, double s) { return {mul(a.x, s), mul(a.y, s), mul(a.z, s)}; }
__device__ __forceinline__ double dot(V3 a, V3 b) { return add(add(mul(a.x, b.x), mul(a.y, b.y)), mul(a.z, b.z)); }
__device__ __forceinline__ V3 cross(V3 a, V3 b) {
    return {sub(mul(a.y, b.z), mul(a.z, b.y)), sub(mul(a.z, b.x), mul(a.x, b.z)), sub(mul(a.x, b.y), mul(a.y, b.x))};
}
__device__ __forceinline__ bool finite3(V3 a) { return isfinite(a.x) && isfinite(a.y) && isfinite(a.z); }
__device__ __forceinline__ double clamp01(double x) { return x < 0.0 ? 0.0 : (x > 1.0 ? 1.0 : x); }

// Ericson's ClosestPtPointTriangle: the closest point q = sum w_i (a, b, c)_i; returns diff = p - q.
__device__ V3 closest_point_triangle(V3 p, V3 a, V3 b, V3 c, double w[3]) {
    const V3 ab = vsub(b, a), ac = vsub(c, a), ap = vsub(p, a);
    const double d1 = dot(ab, ap), d2 = dot(ac, ap);
    if (d1 <= 0.0 && d2 <= 0.0) {
        w[0] = 1.0; w[1] = 0.0; w[2] = 0.0;
        return ap;
    }
    const V3 bp = vsub(p, b);
    const double d3 = dot(ab, bp), d4 = dot(ac, bp);
    if (d3 >= 0.0 && d4 <= d3) {
        w[0] = 0.0; w[1] = 1.0; w[2] = 0.0;
        return bp;
    }
    const double vc = sub(mul(d1, d4), mul(d3, d2));
    if (vc <= 0.0 && d1 >= 0.0 && d3 <= 0.0) {
        const double v = dvd(d1, sub(d1, d3));
        w[0] = sub(1.0, v); w[1] = v; w[2] = 0.0;
        return vsub(p, vadd(a, vscale(ab, v)));
    }
    const V3 cp = vsub(p, c);
    const double d5 = dot(ab, cp), d6 = dot(ac, cp);
    if (d6 >= 0.0 && d5 <= d6) {
        w[0] = 0.0; w[1] = 0.0; w[2] = 1.0;
        return cp;
    }
    const double vb = sub(mul(d5, d2), mul(d1, d6));
    if (vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0) {
        const double t = dvd(d2, sub(d2, d6));
        w[0] = sub(1.0, t); w[1] = 0.0; w[2] = t;
        return vsub(p, vadd(a, vscale(ac, t)));
    }
    const double va = sub(mul(d3, d6), mul(d5, d4));
    const double e43 = sub(d4, d3), e56 = sub(d5, d6);
    if (va <= 0.0 && e43 >= 0.0 && e56 >= 0.0) {
        const double t = dvd(e43, add(e43, e56));
        w[0] = 0.0; w[1] = sub(1.0, t); w[2] = t;
        return vsub(p, vadd(b, vscale(vsub(c, b), t)));
    }
    const double den = dvd(1.0, add(add(va, vb), vc));
    const double v = mul(vb, den), t = mul(vc, den);
    w[0] = sub(sub(1.0, v), t); w[1] = v; w[2] = t;
    return vsub(p, vadd(vadd(a, vscale(ab, v)), vscale(ac, t)));
}

// Ericson's ClosestPtSegmentSegment with EPSILON = 0: returns diff = c1 - c2, and s, t.
__device__ V3 closest_segment_segment(V3 p1, V3 q1, V3 p2, V3 q2, double &s, double &t) {
    const V3 d1 = vsub(q1, p1), d2 = vsub(q2, p2), r = vsub(p1, p2);
    const double a = dot(d1, d1), e = dot(d2, d2), f = dot(d2, r);
    if (a <= 0.0 && e <= 0.0) {
        s = 0.0; t = 0.0;
    } else if (a <= 0.0) {
        s = 0.0;
        t = clamp01(dvd(f, e));
    } else {
        const double c = dot(d1, r);
        if (e <= 0.0) {
            t = 0.0;
            s = clamp01(dvd(-c, a));
        } else {
            const double b = dot(d1, d2);
            const double denom = sub(mul(a, e), mul(b, b));
            s = denom != 0.0 ? clamp01(dvd(sub(mul(b, f), mul(c, e)), denom)) : 0.0;
            t = dvd(add(mul(b, s), f), e);
            if (t < 0.0) {
                t = 0.0;
                s = clamp01(dvd(-c, a));
            } else if (t > 1.0) {
                t = 1.0;
                s = clamp01(dvd(sub(b, c), a));
            }
        }
    }
    return vsub(vadd(p1, vscale(d1, s)), vadd(p2, vscale(d2, t)));
}

__device__ __forceinline__ double norm_of(V3 d) { return __dsqrt_rn(dot(d, d)); }

// ---- topology --------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool is_neighbour(const DeodrCollisionMesh &m, int x, int y) {
    int lo = m.neighbour_offset[x], hi = m.neighbour_offset[x + 1];
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const int v = m.neighbour_index[mid];
        if (v == y) return true;
        if (v < y) lo = mid + 1;
        else hi = mid;
    }
    return false;
}
__device__ __forceinline__ bool near(const DeodrCollisionMesh &m, int x, int y) { return x == y || is_neighbour(m, x, y); }

__device__ __forceinline__ bool vt_excluded(const DeodrCollisionMesh &m, int v, const uint32_t f[3]) {
    return near(m, (int)f[0], v) || near(m, (int)f[1], v) || near(m, (int)f[2], v);
}
__device__ __forceinline__ bool ee_excluded(const DeodrCollisionMesh &m, int a, int b, int c, int d) {
    return near(m, a, c) || near(m, a, d) || near(m, b, c) || near(m, b, d);
}
__device__ __forceinline__ bool in_a_face(const DeodrCollisionMesh &m, int v) {
    return m.corner_offset[v + 1] > m.corner_offset[v];
}

// ---- grid ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int cell_of(const Grid &g, int axis, double x) {
    const double q = floor(mul(sub(x, g.origin[axis]), g.inv_h));
    if (!(q >= 0.0)) return 0;  // NaN too
    return q >= (double)(g.n[axis] - 1) ? g.n[axis] - 1 : (int)q;
}
__device__ __forceinline__ uint32_t key_of(const Grid &g, int i, int j, int k, int type) {
    return ((uint32_t)((i * g.n[1] + j) * g.n[2] + k) << 2) | (uint32_t)type;
}

struct Box {
    int lo[3], hi[3];
};
// cells of the bounding box of `n` points inflated by r (plus a relative margin, so that a point closer than r in
// exact arithmetic always falls inside); false when a point is not finite
__device__ bool box_of(const Grid &g, const V3 *pts, int n, double r, Box &b) {
    double lo[3] = {pts[0].x, pts[0].y, pts[0].z}, hi[3] = {pts[0].x, pts[0].y, pts[0].z};
    for (int i = 0; i < n; i++) {
        if (!finite3(pts[i])) return false;
        const double c[3] = {pts[i].x, pts[i].y, pts[i].z};
        for (int a = 0; a < 3; a++) {
            lo[a] = fmin(lo[a], c[a]);
            hi[a] = fmax(hi[a], c[a]);
        }
    }
    for (int a = 0; a < 3; a++) {
        const double rl = r * (1.0 + 0x1p-20) + fabs(lo[a]) * 0x1p-48, rh = r * (1.0 + 0x1p-20) + fabs(hi[a]) * 0x1p-48;
        b.lo[a] = cell_of(g, a, lo[a] - rl);
        b.hi[a] = cell_of(g, a, hi[a] + rh);
    }
    return true;
}
__device__ __forceinline__ int64_t box_cells(const Box &b) {
    return (int64_t)(b.hi[0] - b.lo[0] + 1) * (b.hi[1] - b.lo[1] + 1) * (b.hi[2] - b.lo[2] + 1);
}

// The bounding boxes of a[0..na) and b[0..nb) are farther apart than r along an axis (with box_of's margins, so
// that a pair closer than r in exact arithmetic is never rejected): a cheap test before the exclusion and the distance.
__device__ __forceinline__ bool boxes_apart(const V3 *a, int na, const V3 *b, int nb, double r) {
    double lo[2][3], hi[2][3], big = 0.0;
    for (int s = 0; s < 2; s++) {
        const V3 *p = s ? b : a;
        const int n = s ? nb : na;
        lo[s][0] = hi[s][0] = p[0].x; lo[s][1] = hi[s][1] = p[0].y; lo[s][2] = hi[s][2] = p[0].z;
        for (int i = 1; i < n; i++) {
            const double c[3] = {p[i].x, p[i].y, p[i].z};
            for (int k = 0; k < 3; k++) {
                lo[s][k] = fmin(lo[s][k], c[k]);
                hi[s][k] = fmax(hi[s][k], c[k]);
            }
        }
        for (int k = 0; k < 3; k++) big = fmax(big, fmax(fabs(lo[s][k]), fabs(hi[s][k])));
    }
    const double rr = r * (1.0 + 0x1p-20) + big * 0x1p-48;
    for (int k = 0; k < 3; k++)
        if (lo[1][k] - hi[0][k] > rr || lo[0][k] - hi[1][k] > rr) return true;
    return false;
}

// first entry with key >= k among n sorted keys
__device__ __forceinline__ int lower_bound(const uint32_t *keys, int n, uint32_t k) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (keys[mid] < k) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

struct Entries {
    const uint32_t *keys;
    const int32_t *ids;
    int cap;
    const int64_t *total;  // the scan's total (device); > cap: the plan overflowed
};
__device__ __forceinline__ bool overflowed(const Entries &en) { return *en.total > (int64_t)en.cap; }

// r of the faces: the thickness (vertex-triangle); of the edges: half of it (their boxes, each inflated by r / 2,
// overlap exactly when one inflated by r overlaps the other)
__device__ __forceinline__ double face_r(double delta) { return delta; }
__device__ __forceinline__ double edge_r(double delta) { return 0.5 * delta; }

__device__ __forceinline__ bool face_points(const DeodrCollisionMesh &m, const double *vertices, int f, uint32_t c[3],
                                            V3 p[3]) {
    for (int k = 0; k < 3; k++) {
        c[k] = m.faces[3 * (size_t)f + k];
        p[k] = load3(vertices, (int)c[k]);
    }
    const V3 n = cross(vsub(p[1], p[0]), vsub(p[2], p[0]));
    return !(n.x == 0.0 && n.y == 0.0 && n.z == 0.0);
}

// ---- kernels ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_min(double x) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x = fmin(x, __shfl_down_sync(0xffffffffu, x, o));
    return x;
}
__device__ __forceinline__ double warp_max(double x) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x = fmax(x, __shfl_down_sync(0xffffffffu, x, o));
    return x;
}

// Bounding box of the finite vertices that are in a face (min and max do not depend on the order), then the grid.
__global__ void __launch_bounds__(NT) k_bounds(DeodrCollisionMesh m, const double *__restrict__ vertices, double h0,
                                               CollisionScratch *s) {
    double v[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
    int bad = 0;
    for (int i = blockIdx.x * NT + threadIdx.x; i < m.nb_vertices; i += gridDim.x * NT) {
        if (!in_a_face(m, i)) continue;
        const V3 p = load3(vertices, i);
        if (!finite3(p)) {
            bad = 1;
            continue;
        }
        v[0] = fmin(v[0], p.x); v[1] = fmin(v[1], p.y); v[2] = fmin(v[2], p.z);
        v[3] = fmax(v[3], p.x); v[4] = fmax(v[4], p.y); v[5] = fmax(v[5], p.z);
    }
    __shared__ double part[6][NT / 32];
    __shared__ int any_bad;
    __shared__ bool last;
    if (threadIdx.x == 0) any_bad = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = 0; k < 6; k++) {
        const double x = k < 3 ? warp_min(v[k]) : warp_max(v[k]);
        if (lane == 0) part[k][warp] = x;
    }
    if (bad) atomicOr(&any_bad, 1);
    __syncthreads();
    if (threadIdx.x < 6) {
        const int k = threadIdx.x;
        double x = part[k][0];
        for (int w = 1; w < NT / 32; w++) x = k < 3 ? fmin(x, part[k][w]) : fmax(x, part[k][w]);
        s->bounds[k * MAX_CTAS + blockIdx.x] = x;
    }
    if (threadIdx.x == 0) s->flags[blockIdx.x] = any_bad;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        last = atomicAdd(&s->done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last || threadIdx.x != 0) return;
    __threadfence();
    double b[6];
    int nonfinite = 0;
    for (int k = 0; k < 6; k++) {
        double x = __ldcg(s->bounds + k * MAX_CTAS);
        for (int c = 1; c < (int)gridDim.x; c++) {
            const double y = __ldcg(s->bounds + k * MAX_CTAS + c);
            x = k < 3 ? fmin(x, y) : fmax(x, y);
        }
        b[k] = x;
    }
    for (int c = 0; c < (int)gridDim.x; c++) nonfinite |= __ldcg(s->flags + c);
    Grid g;
    g.nonfinite = nonfinite;
    if (!(b[0] <= b[3])) {  // no finite vertex: one cell
        for (int a = 0; a < 3; a++) {
            g.origin[a] = 0.0;
            g.n[a] = 1;
        }
        g.inv_h = 0.0;
    } else {
        double ext[3], h = h0;
        for (int a = 0; a < 3; a++) {
            g.origin[a] = b[a];
            ext[a] = b[a + 3] - b[a];
            h = fmax(h, ext[a] / (MAX_AXIS - 1));
        }
        for (int it = 0;; it++) {  // grow the cells until the grid has at most MAX_GRID of them
            int64_t total = 1;
            for (int a = 0; a < 3; a++) {
                const double q = floor(ext[a] / h);  // NaN when ext and h are both infinite: one cell
                g.n[a] = !(q >= 0.0) ? 1 : (q < (double)(MAX_AXIS - 1) ? (int)q + 1 : MAX_AXIS);
                total *= g.n[a];
            }
            if (total <= MAX_GRID || it == 64) break;
            h *= 1.25;
        }
        g.inv_h = isfinite(h) ? 1.0 / h : 0.0;
    }
    s->grid = g;
    s->done = 0;
}

// counts [V + F + E]: cells of every primitive (0 for a primitive left out)
__global__ void k_count(DeodrCollisionMesh m, const double *__restrict__ vertices, double r, int with_edges,
                        const CollisionScratch *__restrict__ s, int64_t *__restrict__ counts) {
    const int V = m.nb_vertices, F = m.nb_faces, E = with_edges ? m.nb_edges : 0;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V + F + E) return;
    const Grid g = s->grid;
    int64_t n = 0;
    if (i < V) {
        n = with_edges && in_a_face(m, i) && finite3(load3(vertices, i)) ? 1 : 0;
    } else if (i < V + F) {
        uint32_t c[3];
        V3 p[3];
        const bool area = face_points(m, vertices, i - V, c, p);
        Box b;
        if ((area || !with_edges) && box_of(g, p, 3, r, b)) n = box_cells(b);
    } else {
        const int e = i - V - F;
        const V3 p[2] = {load3(vertices, m.edges[2 * e]), load3(vertices, m.edges[2 * e + 1])};
        Box b;
        if (box_of(g, p, 2, 0.5 * r, b)) n = box_cells(b);
    }
    counts[i] = n;
}

__global__ void k_fill(DeodrCollisionMesh m, const double *__restrict__ vertices, double r, int with_edges,
                       const CollisionScratch *__restrict__ s, const int64_t *__restrict__ counts,
                       const int64_t *__restrict__ offsets, int64_t total_index, int cap, uint32_t *__restrict__ keys,
                       int32_t *__restrict__ ids) {
    const int V = m.nb_vertices, F = m.nb_faces, E = with_edges ? m.nb_edges : 0;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V + F + E || offsets[total_index] > cap || counts[i] == 0) return;
    const Grid g = s->grid;
    int64_t o = offsets[i];
    if (i < V) {
        const V3 p = load3(vertices, i);
        keys[o] = key_of(g, cell_of(g, 0, p.x), cell_of(g, 1, p.y), cell_of(g, 2, p.z), T_VERTEX);
        ids[o] = i;
        return;
    }
    Box b;
    int type, id;
    if (i < V + F) {
        uint32_t c[3];
        V3 p[3];
        face_points(m, vertices, i - V, c, p);
        box_of(g, p, 3, r, b);
        type = T_FACE;
        id = i - V;
    } else {
        id = i - V - F;
        const V3 p[2] = {load3(vertices, m.edges[2 * id]), load3(vertices, m.edges[2 * id + 1])};
        box_of(g, p, 2, 0.5 * r, b);
        type = T_EDGE;
    }
    for (int x = b.lo[0]; x <= b.hi[0]; x++)
        for (int y = b.lo[1]; y <= b.hi[1]; y++)
            for (int z = b.lo[2]; z <= b.hi[2]; z++) {
                keys[o] = key_of(g, x, y, z, type);
                ids[o] = id;
                o++;
            }
}

// One thread per vertex: its pairs as the point of a vertex-triangle pair.
__global__ void __launch_bounds__(NT) k_vertex(DeodrCollisionMesh m, const double *__restrict__ vertices, double delta,
                                               double weight, const CollisionScratch *__restrict__ s, Entries en,
                                               double *__restrict__ point_b, double *__restrict__ energy_v,
                                               double *__restrict__ min_v) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= m.nb_vertices || overflowed(en)) return;
    const Grid g = s->grid;
    double e = 0.0, dmin = delta, gx = 0.0, gy = 0.0, gz = 0.0;
    const V3 p = load3(vertices, v);
    if (in_a_face(m, v) && finite3(p)) {
        const uint32_t key = key_of(g, cell_of(g, 0, p.x), cell_of(g, 1, p.y), cell_of(g, 2, p.z), T_FACE);
        for (int k = lower_bound(en.keys, en.cap, key); k < en.cap && en.keys[k] == key; k++) {
            const int f = en.ids[k];
            uint32_t c[3];
            V3 q[3];
            face_points(m, vertices, f, c, q);
            if (boxes_apart(&p, 1, q, 3, delta) || vt_excluded(m, v, c)) continue;
            double w[3];
            const V3 diff = closest_point_triangle(p, q[0], q[1], q[2], w);
            const double d = norm_of(diff);
            if (!(d < delta)) continue;
            const double t = sub(delta, d);
            e = add(e, mul(t, t));
            dmin = fmin(dmin, d);
            if (d > 0.0) {
                const double cf = mul(mul(2.0, weight), t);
                gx = sub(gx, mul(cf, dvd(diff.x, d)));
                gy = sub(gy, mul(cf, dvd(diff.y, d)));
                gz = sub(gz, mul(cf, dvd(diff.z, d)));
            }
        }
    }
    point_b[3 * (size_t)v] = gx;
    point_b[3 * (size_t)v + 1] = gy;
    point_b[3 * (size_t)v + 2] = gz;
    energy_v[v] = e;
    min_v[v] = dmin;
}

// One thread per face: its corners' shares of its vertex-triangle pairs (the same pairs k_vertex finds).
__global__ void __launch_bounds__(NT) k_face(DeodrCollisionMesh m, const double *__restrict__ vertices, double delta,
                                             double weight, const CollisionScratch *__restrict__ s, Entries en,
                                             double *__restrict__ corner_b) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= m.nb_faces || overflowed(en)) return;
    const Grid g = s->grid;
    double acc[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
    uint32_t c[3];
    V3 q[3];
    Box b;
    if (face_points(m, vertices, f, c, q) && box_of(g, q, 3, face_r(delta), b)) {
        for (int x = b.lo[0]; x <= b.hi[0]; x++)
            for (int y = b.lo[1]; y <= b.hi[1]; y++)
                for (int z = b.lo[2]; z <= b.hi[2]; z++) {
                    const uint32_t key = key_of(g, x, y, z, T_VERTEX);
                    for (int k = lower_bound(en.keys, en.cap, key); k < en.cap && en.keys[k] == key; k++) {
                        const int v = en.ids[k];
                        const V3 p = load3(vertices, v);
                        if (boxes_apart(&p, 1, q, 3, delta) || vt_excluded(m, v, c)) continue;
                        double w[3];
                        const V3 diff = closest_point_triangle(p, q[0], q[1], q[2], w);
                        const double d = norm_of(diff);
                        if (!(d < delta) || !(d > 0.0)) continue;
                        const double cf = mul(mul(2.0, weight), sub(delta, d));
                        const double n[3] = {dvd(diff.x, d), dvd(diff.y, d), dvd(diff.z, d)};
#pragma unroll
                        for (int i = 0; i < 3; i++)
#pragma unroll
                            for (int j = 0; j < 3; j++) acc[i][j] = add(acc[i][j], mul(mul(cf, w[i]), n[j]));
                    }
                }
    }
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) corner_b[9 * (size_t)f + 3 * i + j] = acc[i][j];
}

// One thread per edge: its edge-edge pairs, each counted at the first cell the two edges' boxes share.
__global__ void __launch_bounds__(NT) k_edge(DeodrCollisionMesh m, const double *__restrict__ vertices, double delta,
                                             double weight, const CollisionScratch *__restrict__ s, Entries en,
                                             double *__restrict__ end_b, double *__restrict__ energy_e,
                                             double *__restrict__ min_e) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m.nb_edges || overflowed(en)) return;
    const Grid g = s->grid;
    const int a = m.edges[2 * e], b = m.edges[2 * e + 1];
    const V3 pa = load3(vertices, a), pb = load3(vertices, b);
    double en_sum = 0.0, dmin = delta;
    double acc[2][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
    const V3 pts[2] = {pa, pb};
    Box bx;
    if (box_of(g, pts, 2, edge_r(delta), bx)) {
        for (int x = bx.lo[0]; x <= bx.hi[0]; x++)
            for (int y = bx.lo[1]; y <= bx.hi[1]; y++)
                for (int z = bx.lo[2]; z <= bx.hi[2]; z++) {
                    const uint32_t key = key_of(g, x, y, z, T_EDGE);
                    for (int k = lower_bound(en.keys, en.cap, key); k < en.cap && en.keys[k] == key; k++) {
                        const int o = en.ids[k];
                        if (o == e) continue;
                        const int c = m.edges[2 * o], d_ = m.edges[2 * o + 1];
                        const V3 pc = load3(vertices, c), pd = load3(vertices, d_);
                        const V3 opts[2] = {pc, pd};
                        Box ob;
                        box_of(g, opts, 2, edge_r(delta), ob);
                        if (x != max(bx.lo[0], ob.lo[0]) || y != max(bx.lo[1], ob.lo[1]) || z != max(bx.lo[2], ob.lo[2]))
                            continue;  // not the first shared cell
                        if (boxes_apart(pts, 2, opts, 2, delta) || ee_excluded(m, a, b, c, d_)) continue;
                        const bool first = e < o;
                        double sp, tp;
                        const V3 diff = first ? closest_segment_segment(pa, pb, pc, pd, sp, tp)
                                              : closest_segment_segment(pc, pd, pa, pb, sp, tp);
                        const double d = norm_of(diff);
                        if (!(d < delta)) continue;
                        const double t = sub(delta, d);
                        en_sum = add(en_sum, mul(t, t));
                        dmin = fmin(dmin, d);
                        if (!(d > 0.0)) continue;
                        // this edge's parameter and sign: -c n for the first segment, +c n for the second
                        const double u = first ? sp : tp;
                        const double cf = mul(mul(2.0, weight), t);
                        const double sc = first ? -cf : cf;
                        const double n[3] = {dvd(diff.x, d), dvd(diff.y, d), dvd(diff.z, d)};
                        const double wt[2] = {sub(1.0, u), u};
#pragma unroll
                        for (int i = 0; i < 2; i++)
#pragma unroll
                            for (int j = 0; j < 3; j++) acc[i][j] = add(acc[i][j], mul(mul(sc, wt[i]), n[j]));
                    }
                }
    }
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) end_b[6 * (size_t)e + 3 * i + j] = acc[i][j];
    energy_e[e] = mul(0.5, en_sum);
    min_e[e] = dmin;
}

// One thread per vertex (grid-stride over max(V, E) items): the gradient in CSR order, and the energy and minimum.
__global__ void __launch_bounds__(NT) k_gather(DeodrCollisionMesh m, double delta, double weight,
                                               CollisionScratch *s, Entries en, const double *__restrict__ point_b,
                                               const double *__restrict__ corner_b, const double *__restrict__ end_b,
                                               const double *__restrict__ energy_v, const double *__restrict__ min_v,
                                               const double *__restrict__ energy_e, const double *__restrict__ min_e,
                                               const double *grad_in, double *grad, double *energy,
                                               double *min_distance) {
    if (overflowed(en)) return;
    const int V = m.nb_vertices, E = m.nb_edges, N = V > E ? V : E;
    double e = 0.0, dmin = delta;
    for (int i = blockIdx.x * NT + threadIdx.x; i < N; i += gridDim.x * NT) {
        if (i < V) {
            double g[3];
            for (int j = 0; j < 3; j++) g[j] = add(grad_in ? grad_in[3 * (size_t)i + j] : 0.0, point_b[3 * (size_t)i + j]);
            for (int k = m.corner_offset[i]; k < m.corner_offset[i + 1]; k++) {
                const double *c = corner_b + 3 * (size_t)m.corner_index[k];
                for (int j = 0; j < 3; j++) g[j] = add(g[j], c[j]);
            }
            for (int k = m.end_offset[i]; k < m.end_offset[i + 1]; k++) {
                const double *c = end_b + 3 * (size_t)m.end_index[k];
                for (int j = 0; j < 3; j++) g[j] = add(g[j], c[j]);
            }
            for (int j = 0; j < 3; j++) grad[3 * (size_t)i + j] = g[j];
            e = add(e, energy_v[i]);
            dmin = fmin(dmin, min_v[i]);
        }
        if (i < E) {
            e = add(e, energy_e[i]);
            dmin = fmin(dmin, min_e[i]);
        }
    }
    __shared__ double wmin[NT / 32];
    dmin = warp_min(dmin);
    if ((threadIdx.x & 31) == 0) wmin[threadIdx.x >> 5] = dmin;
    __syncthreads();
    if (threadIdx.x == 0) {
        double x = wmin[0];
        for (int w = 1; w < NT / 32; w++) x = fmin(x, wmin[w]);
        s->mins[blockIdx.x] = x;  // made visible by grid_sum's fence in this thread
    }
    const double v[1] = {e};
    __shared__ double tot[1];
    if (grid_sum<1>(v, &s->sum, tot) && threadIdx.x == 0) {
        double x = delta;
        for (int c = 0; c < (int)gridDim.x; c++) x = fmin(x, __ldcg(s->mins + c));
        const bool bad = s->grid.nonfinite != 0;
        *energy = bad ? NAN : mul(weight, tot[0]);
        *min_distance = bad ? NAN : x;
    }
}

// ---- self-intersections ----------------------------------------------------------------------------------------------
__device__ __forceinline__ double orient(V3 a, V3 b, V3 c, V3 d) { return dot(cross(vsub(b, a), vsub(c, a)), vsub(d, a)); }
__device__ __forceinline__ int sgn(double x) { return (x > 0.0) - (x < 0.0); }

// the edge (p, q) properly crosses the triangle (a, b, c)
__device__ bool edge_crosses(V3 p, V3 q, V3 a, V3 b, V3 c) {
    const int sp = sgn(orient(a, b, c, p)), sq = sgn(orient(a, b, c, q));
    if (sp == 0 || sq == 0 || sp == sq) return false;
    const int s1 = sgn(orient(p, q, a, b)), s2 = sgn(orient(p, q, b, c)), s3 = sgn(orient(p, q, c, a));
    return s1 != 0 && s1 == s2 && s2 == s3;
}
__device__ __forceinline__ bool faces_cross(const V3 (&x)[3], const V3 (&y)[3]) {
#pragma unroll
    for (int k = 0; k < 3; k++)
        if (edge_crosses(x[k], x[(k + 1) % 3], y[0], y[1], y[2]) || edge_crosses(y[k], y[(k + 1) % 3], x[0], x[1], x[2]))
            return true;
    return false;
}

// One thread per face i: the faces j > i it crosses, each found at the first cell the two boxes share.  With pairs ==
// NULL it counts them into counts[i]; otherwise it writes them from offsets[i] while they fit.
__global__ void __launch_bounds__(NT) k_intersections(DeodrCollisionMesh m, const double *__restrict__ vertices,
                                                      const CollisionScratch *__restrict__ s, Entries en,
                                                      int64_t *__restrict__ counts, const int64_t *__restrict__ offsets,
                                                      const int64_t *__restrict__ pair_total, int32_t *__restrict__ pairs,
                                                      int64_t capacity) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= m.nb_faces || overflowed(en)) return;
    if (pairs && *pair_total > capacity) return;
    const Grid g = s->grid;
    uint32_t c[3];
    V3 p[3];
    face_points(m, vertices, f, c, p);
    int64_t n = 0, o = pairs ? offsets[f] : 0;
    Box b;
    if (box_of(g, p, 3, 0.0, b)) {
        for (int x = b.lo[0]; x <= b.hi[0]; x++)
            for (int y = b.lo[1]; y <= b.hi[1]; y++)
                for (int z = b.lo[2]; z <= b.hi[2]; z++) {
                    const uint32_t key = key_of(g, x, y, z, T_FACE);
                    for (int k = lower_bound(en.keys, en.cap, key); k < en.cap && en.keys[k] == key; k++) {
                        const int h = en.ids[k];
                        if (h <= f) continue;
                        uint32_t d[3];
                        V3 q[3];
                        face_points(m, vertices, h, d, q);
                        Box ob;
                        box_of(g, q, 3, 0.0, ob);
                        if (x != max(b.lo[0], ob.lo[0]) || y != max(b.lo[1], ob.lo[1]) || z != max(b.lo[2], ob.lo[2]))
                            continue;
                        bool shared = false;
#pragma unroll
                        for (int i = 0; i < 3; i++)
#pragma unroll
                            for (int j = 0; j < 3; j++) shared |= c[i] == d[j];
                        if (shared || !faces_cross(p, q)) continue;
                        if (pairs) {
                            pairs[2 * o] = f;
                            pairs[2 * o + 1] = h;
                            o++;
                        } else {
                            n++;
                        }
                    }
                }
    }
    if (!pairs) counts[f] = n;
}

// ---- host ------------------------------------------------------------------------------------------------------------

int grid_of(int64_t n) { return (int)((n + NT - 1) / NT); }

}  // namespace

// The collision state of a workspace: the plan (entry capacity) and its buffers, kept from call to call.
struct CollisionState {
    int64_t cap = 0;            // entries the buffers hold
    DevBuf scratch;             // CollisionScratch, zeroed once
    DevBuf counts, offsets;     // [N + 1] int64
    DevBuf keys, ids, keys_alt, ids_alt;
    DevBuf cub_temp;
    DevBuf point_b, corner_b, end_b, energy_v, min_v, energy_e, min_e;
    DevBuf pair_counts, pair_offsets;
    int64_t *host_words = nullptr;  // pinned: [0] entries, [1] pairs
    cudaEvent_t verdict = nullptr;
};

void deodr_collision_destroy(DeodrWorkspace *ws) {
    if (!ws || !ws->collision) return;
    CollisionState *c = ws->collision;
    for (DevBuf *b : {&c->scratch, &c->counts, &c->offsets, &c->keys, &c->ids, &c->keys_alt, &c->ids_alt, &c->cub_temp,
                      &c->point_b, &c->corner_b, &c->end_b, &c->energy_v, &c->min_v, &c->energy_e, &c->min_e,
                      &c->pair_counts, &c->pair_offsets})
        b->release();
    if (c->host_words) cudaFreeHost(c->host_words);
    if (c->verdict) cudaEventDestroy(c->verdict);
    delete c;
    ws->collision = nullptr;
}

namespace {

int state_of(DeodrWorkspace *ws, CollisionState **out) {
    if (!ws->collision) {
        CollisionState *c = new CollisionState();
        ws->collision = c;
        CUDA_TRY(cudaHostAlloc(&c->host_words, 2 * sizeof(int64_t), cudaHostAllocDefault));
        CUDA_TRY(cudaEventCreateWithFlags(&c->verdict, cudaEventDisableTiming));
        if (int rc = c->scratch.ensure(sizeof(CollisionScratch), &ws->bytes)) return rc;
        CUDA_TRY(cudaMemset(c->scratch.ptr, 0, c->scratch.bytes));
    }
    *out = ws->collision;
    return DEODR_B200_OK;
}

int check_mesh(DeodrWorkspace *ws, const DeodrCollisionMesh *m, const double *vertices) {
    if (!ws || !m || !vertices) return set_error(DEODR_B200_EINVAL, "bad argument: NULL workspace, mesh or vertices");
    if (m->nb_faces <= 0 || m->nb_vertices <= 0 || m->nb_edges <= 0)
        return set_error(DEODR_B200_EINVAL, "bad argument: empty mesh");
    if (!m->faces || !m->edges || !m->neighbour_offset || !m->neighbour_index || !m->corner_offset ||
        !m->corner_index || !m->end_offset || !m->end_index)
        return set_error(DEODR_B200_EINVAL, "bad argument: NULL mesh array");
    if ((int64_t)m->nb_vertices + m->nb_faces + m->nb_edges > 0x7fffffff)
        return set_error(DEODR_B200_EUNSUPPORTED, "V + F + E must fit in int32");
    return DEODR_B200_OK;
}

// Bounds, counts, scan and (when the plan has room) the sorted entries; then the pinned copy of the entry total,
// which the caller reads after enqueueing the rest.  Returns the entries in `en`.
int build_grid(DeodrWorkspace *ws, CollisionState *c, const DeodrCollisionMesh &m, const double *vertices, double r,
               double h0, int with_edges, cudaStream_t st, Entries &en) {
    const int64_t N = (int64_t)m.nb_vertices + m.nb_faces + (with_edges ? m.nb_edges : 0);
    if (int rc = c->counts.ensure((N + 1) * sizeof(int64_t), &ws->bytes)) return rc;
    if (int rc = c->offsets.ensure((N + 1) * sizeof(int64_t), &ws->bytes)) return rc;
    CollisionScratch *s = c->scratch.as<CollisionScratch>();
    const int ctas = (int)std::min<int64_t>(std::max(grid_of(m.nb_vertices), 1), MAX_CTAS);
    k_bounds<<<ctas, NT, 0, st>>>(m, vertices, h0, s);
    k_count<<<grid_of(N), NT, 0, st>>>(m, vertices, r, with_edges, s, c->counts.as<int64_t>());
    CUDA_TRY(cudaMemsetAsync(c->counts.as<int64_t>() + N, 0, sizeof(int64_t), st));
    size_t scan_bytes = 0, sort_bytes = 0;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, c->counts.as<int64_t>(), c->offsets.as<int64_t>(),
                                           (int)(N + 1), st));
    cub::DoubleBuffer<uint32_t> kb(c->keys.as<uint32_t>(), c->keys_alt.as<uint32_t>());
    cub::DoubleBuffer<int32_t> vb(c->ids.as<int32_t>(), c->ids_alt.as<int32_t>());
    if (c->cap > 0)
        CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, kb, vb, (int)c->cap, 0, KEY_BITS, st));
    if (int rc = c->cub_temp.ensure(std::max<size_t>(std::max(scan_bytes, sort_bytes), 1), &ws->bytes)) return rc;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(c->cub_temp.ptr, scan_bytes, c->counts.as<int64_t>(),
                                           c->offsets.as<int64_t>(), (int)(N + 1), st));
    const int64_t *total = c->offsets.as<int64_t>() + N;
    CUDA_TRY(cudaMemcpyAsync(c->host_words, total, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaEventRecord(c->verdict, st));
    if (c->cap > 0) {
        CUDA_TRY(cudaMemsetAsync(c->keys.ptr, 0xff, c->cap * sizeof(uint32_t), st));
        k_fill<<<grid_of(N), NT, 0, st>>>(m, vertices, r, with_edges, s, c->counts.as<int64_t>(),
                                          c->offsets.as<int64_t>(), N, (int)c->cap, c->keys.as<uint32_t>(),
                                          c->ids.as<int32_t>());
        CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->cub_temp.ptr, sort_bytes, kb, vb, (int)c->cap, 0, KEY_BITS, st));
    }
    CUDA_TRY(cudaGetLastError());
    en.keys = kb.Current();
    en.ids = vb.Current();
    en.cap = (int)c->cap;
    en.total = total;
    return DEODR_B200_OK;
}

// Reads the verdict word; grows the plan and asks for a rerun when the entries did not fit.
int read_verdict(DeodrWorkspace *ws, CollisionState *c, bool *rerun) {
    CUDA_TRY(cudaEventSynchronize(c->verdict));
    const int64_t total = c->host_words[0];
    *rerun = total > c->cap || c->cap == 0;
    if (!*rerun) return DEODR_B200_OK;
    const int64_t want = std::max<int64_t>(total + total / 4, 1024);
    if (want >= 0x7fffffff) return set_error(DEODR_B200_EUNSUPPORTED, "the self-collision grid needs 2^31 entries or more");
    for (DevBuf *b : {&c->keys, &c->keys_alt})
        if (int rc = b->ensure(want * sizeof(uint32_t), &ws->bytes)) return rc;
    for (DevBuf *b : {&c->ids, &c->ids_alt})
        if (int rc = b->ensure(want * sizeof(int32_t), &ws->bytes)) return rc;
    c->cap = want;
    return DEODR_B200_OK;
}

}  // namespace

extern "C" {

int deodr_b200_self_collision(DeodrWorkspace *ws, const DeodrCollisionMesh *mesh, const double *vertices,
                              double thickness, double weight, double cell_size, const double *grad_in, double *grad,
                              double *energy, double *min_distance, void *stream) {
    if (int rc = check_mesh(ws, mesh, vertices)) return rc;
    if (!grad || !energy || !min_distance) return set_error(DEODR_B200_EINVAL, "bad argument: NULL output");
    if (!(thickness > 0.0) || !std::isfinite(thickness))
        return set_error(DEODR_B200_EINVAL, "bad argument: thickness must be > 0 and finite");
    if (!(weight >= 0.0) || !std::isfinite(weight))
        return set_error(DEODR_B200_EINVAL, "bad argument: weight must be >= 0 and finite");
    if (!std::isfinite(cell_size)) return set_error(DEODR_B200_EINVAL, "bad argument: cell_size must be finite");
    const DeodrCollisionMesh m = *mesh;
    const int V = m.nb_vertices, F = m.nb_faces, E = m.nb_edges;
    cudaStream_t st = (cudaStream_t)stream;
    CollisionState *c;
    if (int rc = state_of(ws, &c)) return rc;
    for (auto [b, bytes] : {std::pair<DevBuf *, size_t>{&c->point_b, 3 * (size_t)V}, {&c->corner_b, 9 * (size_t)F},
                            {&c->end_b, 6 * (size_t)E}, {&c->energy_v, (size_t)V}, {&c->min_v, (size_t)V},
                            {&c->energy_e, (size_t)E}, {&c->min_e, (size_t)E}})
        if (int rc = b->ensure(bytes * sizeof(double), &ws->bytes)) return rc;
    const double h0 = std::max(cell_size, thickness);
    CollisionScratch *s = c->scratch.as<CollisionScratch>();
    for (int pass = 0; pass < 3; pass++) {
        Entries en;
        if (int rc = build_grid(ws, c, m, vertices, thickness, h0, 1, st, en)) return rc;
        if (en.cap > 0) {
            k_vertex<<<grid_of(V), NT, 0, st>>>(m, vertices, thickness, weight, s, en, c->point_b.as<double>(),
                                                c->energy_v.as<double>(), c->min_v.as<double>());
            k_face<<<grid_of(F), NT, 0, st>>>(m, vertices, thickness, weight, s, en, c->corner_b.as<double>());
            k_edge<<<grid_of(E), NT, 0, st>>>(m, vertices, thickness, weight, s, en, c->end_b.as<double>(),
                                              c->energy_e.as<double>(), c->min_e.as<double>());
            const int ctas = (int)std::min<int64_t>(grid_of(std::max(V, E)), MAX_CTAS);
            k_gather<<<ctas, NT, 0, st>>>(m, thickness, weight, s, en, c->point_b.as<double>(),
                                          c->corner_b.as<double>(), c->end_b.as<double>(), c->energy_v.as<double>(),
                                          c->min_v.as<double>(), c->energy_e.as<double>(), c->min_e.as<double>(),
                                          grad_in, grad, energy, min_distance);
            CUDA_TRY(cudaGetLastError());
        }
        bool rerun;
        if (int rc = read_verdict(ws, c, &rerun)) return rc;
        if (!rerun) return DEODR_B200_OK;
    }
    return set_error(DEODR_B200_ECUDA, "self-collision: the plan did not settle");
}

int deodr_b200_self_intersections(DeodrWorkspace *ws, const DeodrCollisionMesh *mesh, const double *vertices,
                                  double cell_size, int32_t *pairs, int64_t capacity, int64_t *count, void *stream) {
    if (int rc = check_mesh(ws, mesh, vertices)) return rc;
    if (!count || capacity < 0 || (capacity > 0 && !pairs)) return set_error(DEODR_B200_EINVAL, "bad argument: pairs");
    if (!(cell_size > 0.0) || !std::isfinite(cell_size))
        return set_error(DEODR_B200_EINVAL, "bad argument: cell_size must be > 0 and finite");
    const DeodrCollisionMesh m = *mesh;
    const int F = m.nb_faces;
    cudaStream_t st = (cudaStream_t)stream;
    CollisionState *c;
    if (int rc = state_of(ws, &c)) return rc;
    if (int rc = c->pair_counts.ensure((F + 1) * sizeof(int64_t), &ws->bytes)) return rc;
    if (int rc = c->pair_offsets.ensure((F + 1) * sizeof(int64_t), &ws->bytes)) return rc;
    const CollisionScratch *s = c->scratch.as<CollisionScratch>();
    for (int pass = 0; pass < 3; pass++) {
        Entries en;
        if (int rc = build_grid(ws, c, m, vertices, 0.0, cell_size, 0, st, en)) return rc;
        if (en.cap > 0) {
            int64_t *pc = c->pair_counts.as<int64_t>(), *po = c->pair_offsets.as<int64_t>();
            k_intersections<<<grid_of(F), NT, 0, st>>>(m, vertices, s, en, pc, nullptr, nullptr, nullptr, 0);
            CUDA_TRY(cudaMemsetAsync(pc + F, 0, sizeof(int64_t), st));
            size_t bytes = 0;
            CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, bytes, pc, po, F + 1, st));
            if (bytes > c->cub_temp.bytes) {  // the scan's scratch: the sort's is no longer needed here
                if (int rc = c->cub_temp.ensure(bytes, &ws->bytes)) return rc;
            }
            CUDA_TRY(cub::DeviceScan::ExclusiveSum(c->cub_temp.ptr, bytes, pc, po, F + 1, st));
            if (capacity > 0)
                k_intersections<<<grid_of(F), NT, 0, st>>>(m, vertices, s, en, nullptr, po, po + F, pairs, capacity);
            CUDA_TRY(cudaMemcpyAsync(c->host_words + 1, po + F, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaGetLastError());
        }
        bool rerun;
        if (int rc = read_verdict(ws, c, &rerun)) return rc;
        if (!rerun) {
            CUDA_TRY(cudaStreamSynchronize(st));  // the pair count, copied behind the scan
            *count = c->host_words[1];
            return DEODR_B200_OK;
        }
    }
    return set_error(DEODR_B200_ECUDA, "self-intersections: the plan did not settle");
}

}  // extern "C"
