// Exact (fp64, reference-operation-order) geometry of the raster hot path: triangle stencil setup, per-row spans,
// z planes, silhouette-edge band setup and spans.  Everything that decides WHICH pixel is covered and WHAT z it gets
// lives here, so that the z-buffer / owner id can be bit-identical to the reference
// (C++/DifferentiableRenderer.h, "DR.h" below).
//
// The functions are __host__ __device__: the CUDA kernels (kernels.cu) call them on the device, and the CPU
// emulation harness under tests/emul (test infrastructure, never shipped) calls the very same code on the host to
// check it against the oracle without a GPU.
//
// No FMA contraction is allowed in this file: on the device every product/sum goes through __dmul_rn/__dadd_rn
// (never fused by ptxas); the host harness is compiled with -ffp-contract=off.
#pragma once

#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define DEODR_HD __host__ __device__ __forceinline__
#else
#define DEODR_HD inline
#endif

#if defined(__CUDA_ARCH__)
#define DMUL(a, b) __dmul_rn((a), (b))
#define DADD(a, b) __dadd_rn((a), (b))
#define DSUB(a, b) __dsub_rn((a), (b))
#define DDIV(a, b) __ddiv_rn((a), (b))
#define DSQRT(a) __dsqrt_rn((a))
#else
#define DMUL(a, b) ((a) * (b))
#define DADD(a, b) ((a) + (b))
#define DSUB(a, b) ((a) - (b))
#define DDIV(a, b) ((a) / (b))
#define DSQRT(a) sqrt((a))
#endif

namespace deodr {

// a*b - c*d with two roundings on the products and one on the difference (never fused)
DEODR_HD double diff_of_products(double a, double b, double c, double d) { return DSUB(DMUL(a, b), DMUL(c, d)); }

// DR.h:92-117: T = transposed cofactors of S times 1/det; det = (S0*T0 + S1*T3) + S2*T6.
DEODR_HD void inv3x3(const double *S, double *T) {
    T[0] = diff_of_products(S[4], S[8], S[7], S[5]);
    T[3] = -diff_of_products(S[3], S[8], S[6], S[5]);
    T[6] = diff_of_products(S[3], S[7], S[6], S[4]);
    T[1] = -diff_of_products(S[1], S[8], S[7], S[2]);
    T[4] = diff_of_products(S[0], S[8], S[6], S[2]);
    T[7] = -diff_of_products(S[0], S[7], S[6], S[1]);
    T[2] = diff_of_products(S[1], S[5], S[4], S[2]);
    T[5] = -diff_of_products(S[0], S[5], S[3], S[2]);
    T[8] = diff_of_products(S[0], S[4], S[3], S[1]);
    double det = DADD(DADD(DMUL(S[0], T[0]), DMUL(S[1], T[3])), DMUL(S[2], T[6]));
    double inv_det = DDIV(1.0, det);
    for (int k = 0; k < 9; k++) T[k] = DMUL(T[k], inv_det);
}

// Vertices beyond the `short` range (more than 32767 pixels from the origin).  The reference's casts wrap there
// (x86: cvttsd2si to int32, low 16 bits kept; 0x80000000 for anything outside int32), and a triangle with one far
// vertex is still drawn in part.  DEODR_EXACT_SHORT_WRAP=1 reproduces that bit for bit (on the CPU emulation against
// the compiled reference up to 1e15 px, tests/test_emul.py; on an H100, tests/test_gpu_edge_cases.py, where that build
// passes every `pytest -m gpu` test the default one passes); the default (0) is identical below the limit and culls such
// triangles beyond it (INTEGRATION.md section 5).  Both builds convert alike (to_short / to_int_trunc below), so they
// differ only in tri_bounds / tri_geom: same ptxas figures except k_small_tri_bwd<3, false> (63 registers in the exact
// build, 64 in the default), and the same bench.py c5 speed within run-to-run noise (DESIGN.md section 9).  Making it the default
// changes which pixels far triangles cover: a behaviour change of its own, not made here.
#ifndef DEODR_EXACT_SHORT_WRAP
#define DEODR_EXACT_SHORT_WRAP 0
#endif

// (short) conversion of the reference: double -> int32 (truncation) -> low 16 bits, sign-extended.
// In every build: the host and the device must agree on a vertex at 2^31 px or +inf (tests/test_gpu_edge_cases.py).
DEODR_HD int to_short(double v) {
    // cvttsd2si gives 0x80000000 (low 16 bits: 0) outside int32; cvt.rzi.s32.f64 saturates: only the positive side
    // differs in the low 16 bits (0x7fffffff -> -1).  (NaN: 0x80000000 there, 0 here: both 0.)
    if (v >= 2147483648.0) return 0;
#if defined(__CUDA_ARCH__)
    int i = __double2int_rz(v);
#else
    int i = (int)v;
#endif
    return (int)(int16_t)(i & 0xffff);
}

// (int) conversion as the reference's compiler performs it (cvttsd2si): INT_MIN for NaN and anything outside int32.
// (cvt.rzi.s32.f64 gives INT_MAX from 2^31 up: the band of an edge with such an end point would reach the last
// image row on the device, where the reference's is empty.)
DEODR_HD int to_int_trunc(double v) {
    if (!(v > -2147483649.0 && v < 2147483648.0)) return (int)0x80000000;
#if defined(__CUDA_ARCH__)
    return __double2int_rz(v);
#else
    return (int)v;
#endif
}

// Largest x in [x_min, x_max] such that pred(x') holds for every x' in (x_min, x]; pred is monotone in x'
// (a rounded product with a fixed factor is monotone), so the reference's incremental loops of DR.h:461-476 and
// DR.h:501-516 are equivalent to this bisection.  mode: 0 '<=', 1 '>=', 2 '<', 3 '>'.
DEODR_HD int monotone_search(double a, double b, int x_min, int x_max, int mode) {
    int lo = x_min, hi = x_max;  // invariant: pred holds on (x_min, lo]; fails at hi+1 (or hi == x_max)
    while (lo < hi) {
        int mid = lo + ((hi - lo + 1) >> 1);  // candidate x, tests x' = mid (the loop tests (x+1) with x = mid-1)
        double p = DMUL((double)mid, b);
        bool ok = mode == 0 ? (p <= a) : mode == 1 ? (p >= a) : mode == 2 ? (p < a) : (p > a);
        if (ok) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// ---- floor(RN(a / b)) without the fp64 division in the common case ------------------------------------------
// The reference computes (short)floor(a / b) with an IEEE division (DR.h:449).  An fp64 division costs ~40 issue slots
// on the GPU and two of them are needed per (triangle, row); the quotient is only used through its floor.  We get a
// candidate from an fp32 division (|error| < 0.01 in the admitted range |a/b| < 32768) and settle it with the exact
// predicate G(x) = [RN(a/b) >= x], x integer:
//   * RN is monotone and x is representable, so a/b >= x  ==>  RN(a/b) >= x;
//   * a/b >= x is decided EXACTLY by the sign of g = fma(-x, b, a) (a correctly rounded value has the sign of the
//     exact one);
//   * if a/b < x, RN(a/b) can still round up to x only when x - a/b <= ulp(x)/2, i.e. |g| <= 2^-53 |x b|; inside a
//     4x wider band (and for non-finite / tiny operands) we fall back to the real division.
// Result: bit-identical to the reference for every input (tests/test_rmath.py drives both on adversarial inputs).
DEODR_HD int floor_quotient_exact(double a, double b) { return to_short(floor(DDIV(a, b))); }

#if defined(__CUDA_ARCH__)
#define DEODR_FMA(x, y, z) __fma_rn((x), (y), (z))
#else
#define DEODR_FMA(x, y, z) fma((x), (y), (z))
#endif

// 1: RN(a/b) >= x, 0: RN(a/b) < x, -1: too close to call
DEODR_HD int quotient_ge(double a, double b, int x) {
    const double xd = (double)x;
    const double g = DEODR_FMA(-xd, b, a);  // a - x*b, one rounding
    const bool real_ge = b > 0 ? (g >= 0) : (g <= 0);
    if (real_ge) return 1;
    return fabs(g) > 4.5e-16 * fabs(xd * b) ? 0 : -1;
}

DEODR_HD int floor_quotient(double a, double b) {
    const float af = (float)a, bf = (float)b;
    const float qf = af / bf;
    // operands must be comfortably inside the normal fp32 range for the 0.01 error bound to hold
    if (!(fabsf(qf) < 33000.0f) || !(fabsf(bf) > 1e-30f) || !(fabsf(af) > 1e-30f || a == 0.0) ||
        !(fabsf(af) < 1e30f) || !(fabsf(bf) < 1e30f))
        return floor_quotient_exact(a, b);
    const int c = (int)floorf(qf);
    const int up = quotient_ge(a, b, c + 1);
    if (up < 0) return floor_quotient_exact(a, b);
    if (up) return to_short((double)(c + 1));
    const int at = quotient_ge(a, b, c);
    if (at < 0) return floor_quotient_exact(a, b);
    return to_short((double)(at ? c : c - 1));
}

// (short)(double)i for an int i: the reference's pass through `short` without the two conversions
DEODR_HD int wrap16(int i) { return (int)(int16_t)(i & 0xffff); }

// floor_quotient as straight-line code (no branches: several independent quotients interleave in the pipeline).
// Returns true when the result is not settled and floor_quotient_exact must be used instead; same decisions as
// floor_quotient.
DEODR_HD bool floor_quotient_try(double a, double b, int *out) {
    const float af = (float)a, bf = (float)b;
    const float qf = af / bf;
    const bool ok = (fabsf(qf) < 33000.0f) && (fabsf(bf) > 1e-30f) && (fabsf(af) > 1e-30f || a == 0.0) &&
                    (fabsf(af) < 1e30f) && (fabsf(bf) < 1e30f);
    const int c = ok ? (int)floorf(qf) : 0;
    const double c1 = (double)(c + 1), c0 = (double)c;
    const double g1 = DEODR_FMA(-c1, b, a), g0 = DEODR_FMA(-c0, b, a);
    const bool up_ge = b > 0 ? (g1 >= 0) : (g1 <= 0), at_ge = b > 0 ? (g0 >= 0) : (g0 <= 0);
    const bool up_far = fabs(g1) > 4.5e-16 * fabs(c1 * b), at_far = fabs(g0) > 4.5e-16 * fabs(c0 * b);
    *out = wrap16(up_ge ? c + 1 : (at_ge ? c : c - 1));
    return !ok || (!up_ge && (!up_far || (!at_ge && !at_far)));
}

// DR.h:440-479: min(x_max, max(x_min, floor(a/b))) with the robust fall-back.  Result passes through `short`.
DEODR_HD int floor_div_clamped(double a, double b, int x_min, int x_max) {
    if (DMUL(fabs(b), 32767.0) > DADD(fabs(a), fabs(b))) {
        int x = floor_quotient(a, b);
        if (x < x_min) x = to_short((double)x_min);
        if (x > x_max) x = to_short((double)x_max);
        return x;
    }
    return monotone_search(a, b, x_min, x_max, b > 0 ? 0 : 1);
}

// DR.h:481-519.  ceil(RN(q)) = -floor(RN(-q)) (rounding to nearest is symmetric).
DEODR_HD int ceil_div_clamped(double a, double b, int x_min, int x_max) {
    if (DMUL(fabs(b), 32767.0) > DADD(fabs(a), fabs(b))) {
        int x = to_short((double)(-floor_quotient(-a, b)));
        if (x < x_min) x = to_short((double)x_min);
        if (x > x_max) x = to_short((double)x_max);
        return x;
    }
    return monotone_search(a, b, x_min, x_max, b > 0 ? 2 : 3);
}

// the reference formulation with the real division, kept for the equivalence tests
DEODR_HD int floor_div_clamped_reference(double a, double b, int x_min, int x_max) {
    if (DMUL(fabs(b), 32767.0) > DADD(fabs(a), fabs(b))) {
        int x = to_short(floor(DDIV(a, b)));
        if (x < x_min) x = to_short((double)x_min);
        if (x > x_max) x = to_short((double)x_max);
        return x;
    }
    return monotone_search(a, b, x_min, x_max, b > 0 ? 0 : 1);
}
DEODR_HD int ceil_div_clamped_reference(double a, double b, int x_min, int x_max) {
    if (DMUL(fabs(b), 32767.0) > DADD(fabs(a), fabs(b))) {
        int x = to_short(ceil(DDIV(a, b)));
        if (x < x_min) x = to_short((double)x_min);
        if (x > x_max) x = to_short((double)x_max);
        return x;
    }
    return monotone_search(a, b, x_min, x_max, b > 0 ? 2 : 3);
}

// ------------------------------------------------------------------------------------------------ triangles

// DR.h:391-398 on the caller-supplied (un-offset) vertices; only the sign is used.
DEODR_HD double signed_area(const double V[3][2], bool clockwise) {
    double ux = DSUB(V[1][0], V[0][0]), uy = DSUB(V[1][1], V[0][1]);
    double vx = DSUB(V[2][0], V[0][0]), vy = DSUB(V[2][1], V[0][1]);
    return DMUL(DMUL(0.5, DSUB(DMUL(ux, vy), DMUL(vx, uy))), clockwise ? 1.0 : -1.0);
}

// Raster record of one triangle: what the tile kernel keeps in shared memory.
struct TriGeom {
    double eq[3][3];  // edge equations a x + b y + c  (DR.h:373-389)
    double zp[3];     // z (or 1/z when perspective_correct) plane: zp[0] x + zp[1] y + zp[2]
    int16_t x_min, x_max;
    int16_t y_begin[2], y_end[2];
    uint8_t left[2], right[2];
};

DEODR_HD void edge_equation(double e[3], const double v1[2], const double v2[2], bool cw) {
    if (cw) { e[0] = DSUB(v1[1], v2[1]); e[1] = DSUB(v2[0], v1[0]); }
    else    { e[0] = DSUB(v2[1], v1[1]); e[1] = DSUB(v1[0], v2[0]); }
    e[2] = DMUL(-0.5, DADD(DMUL(e[0], DADD(v1[0], v2[0])), DMUL(e[1], DADD(v1[1], v2[1]))));
}

// three compare-exchanges of DR.h:400-426; only what the caller needs: sorted values and the index of min / max
DEODR_HD void order3(const double v[3], double sv[3], int idx[3]) {
    sv[0] = v[0]; sv[1] = v[1]; sv[2] = v[2];
    idx[0] = 0; idx[1] = 1; idx[2] = 2;
    if (sv[0] > sv[1]) { double t = sv[0]; sv[0] = sv[1]; sv[1] = t; int i = idx[0]; idx[0] = idx[1]; idx[1] = i; }
    if (sv[0] > sv[2]) { double t = sv[0]; sv[0] = sv[2]; sv[2] = t; int i = idx[0]; idx[0] = idx[2]; idx[2] = i; }
    if (sv[1] > sv[2]) { double t = sv[1]; sv[1] = sv[2]; sv[2] = t; int i = idx[1]; idx[1] = idx[2]; idx[2] = i; }
}

// Integer bounds of DR.h:676-711 alone (what the binning needs): x_min / x_max and the first / last row of the two
// halves' union.  Identical to the fields tri_geom() derives, without the matrix inverse.
DEODR_HD void tri_bounds(const double V[3][2], bool strict, int *x_min, int *x_max, int *y_first, int *y_last) {
    double x_lo = fmin(fmin(V[0][0], V[1][0]), V[2][0]), x_hi = fmax(fmax(V[0][0], V[1][0]), V[2][0]);
    double y_lo = fmin(fmin(V[0][1], V[1][1]), V[2][1]), y_hi = fmax(fmax(V[0][1], V[1][1]), V[2][1]);
    *x_min = strict ? to_short(floor(x_lo)) : to_short(ceil(x_lo));
    *x_max = to_short(floor(x_hi));
#if DEODR_EXACT_SHORT_WRAP
    // rows of the two halves (DR.h:686-711), every bound through the reference's `short`: their union is [b0, e1] as
    // long as nothing wrapped; with a vertex beyond +-32767 one half can be empty while the other is not
    double y_mid = fmax(fmin(V[0][1], V[1][1]), fmin(fmax(V[0][1], V[1][1]), V[2][1]));
    // (32768 = (short)32767 + 1 starts the reference's `short` row counter, DR.h:925, at -32768)
    int b0 = strict ? wrap16(to_short(floor(y_lo)) + 1) : to_short(ceil(y_lo)), e0 = to_short(floor(y_mid));
    int b1 = strict ? wrap16(to_short(floor(y_mid)) + 1) : to_short(ceil(y_mid)), e1 = to_short(floor(y_hi));
    int first = 32767, last = -32768;
    if (b0 <= e0) { first = b0; last = e0; }
    if (b1 <= e1) { if (b1 < first) first = b1; if (e1 > last) last = e1; }
    *y_first = first;
    *y_last = last;
#else
    int yb = strict ? to_short(floor(y_lo)) + 1 : to_short(ceil(y_lo));
    *y_first = yb > 32767 ? 32767 : yb;
    *y_last = to_short(floor(y_hi));
#endif
}

// DR.h:633-739 (stencil) + DR.h:787 / 775 (z plane).  V already has the pixel-centre offset removed.
// Minv (xy1_to_bary) is returned for callers that need the reference's planes; pass nullptr otherwise.
DEODR_HD void tri_geom(const double V[3][2], const double Zv[3], bool strict, bool persp, TriGeom *g, double *Minv_out) {
    double M[9], Minv[9];
    for (int v = 0; v < 3; v++) { M[v] = V[v][0]; M[3 + v] = V[v][1]; M[6 + v] = 1.0; }
    inv3x3(M, Minv);
    bool cw = signed_area(V, true) > 0;
    edge_equation(g->eq[0], V[0], V[1], cw);
    edge_equation(g->eq[1], V[1], V[2], cw);
    edge_equation(g->eq[2], V[2], V[0], cw);
    double xu[3] = {V[0][0], V[1][0], V[2][0]}, yu[3] = {V[0][1], V[1][1], V[2][1]}, xs[3], ys[3];
    int xo[3], yo[3];
    order3(xu, xs, xo);
    order3(yu, ys, yo);
    g->x_min = (int16_t)(strict ? to_short(floor(xs[0])) : to_short(ceil(xs[0])));
    g->x_max = (int16_t)to_short(floor(xs[2]));
    // NB: "(short)floor(y) + 1" is computed in int and then stored in an int: no 16-bit wrap of the +1
    int yb0 = strict ? to_short(floor(ys[0])) + 1 : to_short(ceil(ys[0]));
    int yb1 = strict ? to_short(floor(ys[1])) + 1 : to_short(ceil(ys[1]));
#if DEODR_EXACT_SHORT_WRAP
    // 32768 = (short)32767 + 1 starts the reference's `short` row counter (DR.h:925) at -32768: rows from 0
    g->y_begin[0] = (int16_t)wrap16(yb0);
    g->y_begin[1] = (int16_t)wrap16(yb1);
#else
    // the +1 can only leave the int16 range at 32768, far outside any image: saturate for storage
    g->y_begin[0] = (int16_t)(yb0 > 32767 ? 32767 : yb0);
    g->y_begin[1] = (int16_t)(yb1 > 32767 ? 32767 : yb1);
#endif
    g->y_end[0] = (int16_t)to_short(floor(ys[1]));
    g->y_end[1] = (int16_t)to_short(floor(ys[2]));
    int id = yo[0];
    if (g->eq[id][0] > 0) { g->right[0] = (uint8_t)((id + 2) % 3); g->left[0] = (uint8_t)id; }
    else                  { g->right[0] = (uint8_t)id;             g->left[0] = (uint8_t)((id + 2) % 3); }
    id = yo[2];
    if (g->eq[id][0] < 0) { g->right[1] = (uint8_t)id;             g->left[1] = (uint8_t)((id + 2) % 3); }
    else                  { g->right[1] = (uint8_t)((id + 2) % 3); g->left[1] = (uint8_t)id; }
    double zv[3] = {Zv[0], Zv[1], Zv[2]};
    if (persp) for (int i = 0; i < 3; i++) zv[i] = DDIV(1.0, Zv[i]);
    // mul_vect_matrix3x3 DR.h:272-280: ((0 + Minv[i] z0) + Minv[3+i] z1) + Minv[6+i] z2
    for (int i = 0; i < 3; i++)
        g->zp[i] = DADD(DADD(DADD(0.0, DMUL(Minv[i], zv[0])), DMUL(Minv[3 + i], zv[1])), DMUL(Minv[6 + i], zv[2]));
    if (Minv_out) for (int i = 0; i < 9; i++) Minv_out[i] = Minv[i];
}

// DR.h:864-906 for one half.  Returns an empty span as x_begin > x_end.
// (formulation that follows the reference line by line; kept for the equivalence test)
DEODR_HD void tri_half_span_reference(const TriGeom &g, int half, int y, int width, bool strict, int *x_begin, int *x_end) {
    const double *l = g.eq[g.left[half]], *r = g.eq[g.right[half]];
    int x_min = g.x_min, x_max = g.x_max;
    if (x_min < 0) x_min = 0;
    if (x_max > width - 1) x_max = width - 1;
    int xb = x_min, xe = x_max;
    double num = -DADD(DMUL(l[1], (double)y), l[2]);
    int tmp = strict ? to_short((double)(1 + floor_div_clamped(num, l[0], x_min - 1, x_max)))
                     : ceil_div_clamped(num, l[0], x_min - 1, x_max);
    if (tmp > xb) xb = tmp;
    num = -DADD(DMUL(r[1], (double)y), r[2]);
    tmp = floor_div_clamped(num, r[0], x_min - 1, x_max);
    if (tmp < xe) xe = tmp;
    *x_begin = xb;
    *x_end = xe;
}

// Same result; the left and right bounds are clamped against the same [x_min - 1, x_max], so their two quotients are
// computed side by side (branch-free candidates, rare exact fall-back afterwards): half the dependent chain.
DEODR_HD void tri_half_span(const TriGeom &g, int half, int y, int width, bool strict, int *x_begin, int *x_end) {
    const double *l = g.eq[g.left[half]], *r = g.eq[g.right[half]];
    int x_min = g.x_min, x_max = g.x_max;
    if (x_min < 0) x_min = 0;
    if (x_max > width - 1) x_max = width - 1;
    const int lo = x_min - 1, hi = x_max;
    const double yd = (double)y;
    const double nl = -DADD(DMUL(l[1], yd), l[2]), nr = -DADD(DMUL(r[1], yd), r[2]);
    const bool normal_l = DMUL(fabs(l[0]), 32767.0) > DADD(fabs(nl), fabs(l[0]));
    const bool normal_r = DMUL(fabs(r[0]), 32767.0) > DADD(fabs(nr), fabs(r[0]));
    const double al = strict ? nl : -nl;  // ceil(RN(q)) = -floor(RN(-q))
    int ql, qr;
    const bool unsettled_l = floor_quotient_try(al, l[0], &ql), unsettled_r = floor_quotient_try(nr, r[0], &qr);
    if (normal_l && unsettled_l) ql = floor_quotient_exact(al, l[0]);
    if (normal_r && unsettled_r) qr = floor_quotient_exact(nr, r[0]);
    int xl, xr;
    if (normal_l) {
        xl = strict ? ql : wrap16(-ql);
        if (xl < lo) xl = wrap16(lo);
        if (xl > hi) xl = wrap16(hi);
    } else {
        xl = monotone_search(nl, l[0], lo, hi, strict ? (l[0] > 0 ? 0 : 1) : (l[0] > 0 ? 2 : 3));
    }
    if (normal_r) {
        xr = qr;
        if (xr < lo) xr = wrap16(lo);
        if (xr > hi) xr = wrap16(hi);
    } else {
        xr = monotone_search(nr, r[0], lo, hi, r[0] > 0 ? 0 : 1);
    }
    const int tmp = strict ? wrap16(1 + xl) : xl;
    *x_begin = tmp > x_min ? tmp : x_min;
    *x_end = xr < x_max ? xr : x_max;
}

// Coverage of row y = union of the (at most two) halves containing the row.  In non-strict mode the row of the
// middle vertex can belong to both halves (DR.h:697-711); the reference then draws both spans, and since the z of a
// pixel does not depend on the half the result is the union.  Both spans share the long-edge bound, so the union is
// an interval.
DEODR_HD void tri_row_span(const TriGeom &g, int y, int width, int height, bool strict, int *x_begin, int *x_end) {
    // SIMT note: the half is selected as DATA (index h) so that a warp whose lanes sit in different halves still runs
    // the expensive span body once; the second body only runs for rows that belong to both halves (rare).
    int lo0 = g.y_begin[0] < 0 ? 0 : g.y_begin[0], hi0 = g.y_end[0] > height - 1 ? height - 1 : g.y_end[0];
    int lo1 = g.y_begin[1] < 0 ? 0 : g.y_begin[1], hi1 = g.y_end[1] > height - 1 ? height - 1 : g.y_end[1];
    const bool in0 = y >= lo0 && y <= hi0, in1 = y >= lo1 && y <= hi1;
    int xb = 1, xe = 0;
    if (in0 || in1) {
        tri_half_span(g, in0 ? 0 : 1, y, width, strict, &xb, &xe);
        if (in0 && in1) {
            int b, e;
            tri_half_span(g, 1, y, width, strict, &b, &e);
            if (b <= e) {
                if (xb > xe) { xb = b; xe = e; }
                else { if (b < xb) xb = b; if (e > xe) xe = e; }
            }
        }
    }
    *x_begin = xb;
    *x_end = xe;
}

// rows that can be covered (both halves), clipped to the image; empty as y0 > y1
DEODR_HD void tri_row_range(const TriGeom &g, int height, int *y0, int *y1) {
    int a = g.y_begin[0] < g.y_begin[1] ? g.y_begin[0] : g.y_begin[1];
    int b = g.y_end[0] > g.y_end[1] ? g.y_end[0] : g.y_end[1];
    if (a < 0) a = 0;
    if (b > height - 1) b = height - 1;
    *y0 = a;
    *y1 = b;
}

// DR.h:934 + 960 (and 946-947 with perspective_correct): Z0y = ((0 + zp0*0) + zp1*y) + zp2 ; Z = Z0y + zp0*x.
// For finite planes (0 + zp0*0) is +0, so Z0y = zp1*y + zp2 exactly.
DEODR_HD double plane_row(const double *p, int y) { return DADD(DADD(DADD(0.0, DMUL(p[0], 0.0)), DMUL(p[1], (double)y)), DMUL(p[2], 1.0)); }
DEODR_HD double plane_at(const double *p, double row0, int x) { return DADD(row0, DMUL(p[0], (double)x)); }
DEODR_HD double tri_z(const TriGeom &g, int x, int y, bool persp) {
    double z = plane_at(g.zp, plane_row(g.zp, y), x);
    return persp ? DDIV(1.0, z) : z;
}

// The reference evaluates Z = (((0 + zp0*0) + zp1*y) + zp2*1) + zp0*x (DR.h:934, 960).  For a finite zp0 the first
// term is +0 and adding it only matters for the sign of an exactly-zero result; for an infinite zp0 it is NaN and so
// is Z.  plane_z() drops the no-op terms (2 DMUL + 2 DADD per pixel instead of 4 + 4) and stays bit-identical by
// (a) storing NaN for an infinite zp0 at record creation (canonical_plane) and (b) re-evaluating the full expression
// when the short one returns zero.
DEODR_HD void canonical_plane(const double *zp, double *out) {
    out[0] = (zp[0] - zp[0] == 0.0 || zp[0] != zp[0]) ? zp[0] : (zp[0] - zp[0]);  // +-inf -> NaN
    out[1] = zp[1];
    out[2] = zp[2];
}

DEODR_HD double plane_z(const double *zp, double xd, double yd, int x, int y) {
    double z = DADD(DADD(DMUL(zp[1], yd), zp[2]), DMUL(zp[0], xd));
    if (z == 0.0) z = plane_at(zp, plane_row(zp, y), x);
    return z;
}

// ---------------------------------------------------------------------------------------------- silhouette edges

struct EdgeGeom {
    double ineq[12];  // rows 0,1: edge barycentrics b0,b1; row 2: T = distance/sigma; row 3: 1 - T  (DR.h:1420-1435)
    double zp[3];     // z plane along the edge (DR.h:1577 / 1564)
    int y_begin, y_end;
};

// DR.h:1437-1459: rows of the sigma-wide band (note the sequential update of the bound between the two vertices).
DEODR_HD void edge_row_range(const double V[2][2], int height, double sigma, int *y_begin, int *y_end) {
    int yb = height - 1;
    for (int k = 0; k < 2; k++)
        if (DSUB(V[k][1], sigma) < (double)yb) yb = to_int_trunc(floor(DSUB(V[k][1], sigma))) + 1;
    if (yb < 0) yb = 0;
    int ye = 0;
    for (int k = 0; k < 2; k++)
        if (DADD(V[k][1], sigma) > (double)ye) ye = to_int_trunc(floor(DADD(V[k][1], sigma)));
    if (ye > height - 1) ye = height - 1;
    *y_begin = yb;
    *y_end = ye;
}

// DR.h:1366-1460 + the z plane.  V = the two end points (offset removed), Zv their depths.
// E / Einv / nt / inv_norm are returned for the adjoint (pass nullptr when not needed).
DEODR_HD void edge_geom(const double V[2][2], const double Zv[2], int height, double sigma, bool cw, bool persp,
                        EdgeGeom *g, double *E_out, double *Einv_out, double *nt_out) {
    double n[2], E[9], Einv[9];
    if (cw) { n[0] = DSUB(V[0][1], V[1][1]); n[1] = DSUB(V[1][0], V[0][0]); }
    else    { n[0] = DSUB(V[1][1], V[0][1]); n[1] = DSUB(V[0][0], V[1][0]); }
    double inv_norm = DDIV(1.0, DSQRT(DADD(DMUL(n[0], n[0]), DMUL(n[1], n[1]))));
    if (nt_out) { nt_out[0] = n[0]; nt_out[1] = n[1]; nt_out[2] = inv_norm; }
    n[0] = DMUL(n[0], inv_norm);
    n[1] = DMUL(n[1], inv_norm);
    E[0] = V[0][0]; E[1] = V[1][0]; E[2] = n[0];
    E[3] = V[0][1]; E[4] = V[1][1]; E[5] = n[1];
    E[6] = 1.0; E[7] = 1.0; E[8] = 0.0;
    inv3x3(E, Einv);
    double inv_sigma = DDIV(1.0, sigma);
    for (int k = 0; k < 6; k++) g->ineq[k] = Einv[k];
    for (int k = 0; k < 3; k++) g->ineq[6 + k] = DMUL(inv_sigma, Einv[6 + k]);
    g->ineq[9] = -g->ineq[6];
    g->ineq[10] = -g->ineq[7];
    g->ineq[11] = DSUB(1.0, g->ineq[8]);
    edge_row_range(V, height, sigma, &g->y_begin, &g->y_end);
    double zv[2] = {Zv[0], Zv[1]};
    if (persp) { zv[0] = DDIV(1.0, Zv[0]); zv[1] = DDIV(1.0, Zv[1]); }
    // mul_matrix(1,2,3) DR.h:296-309: (0 + z0*Einv[k]) + z1*Einv[3+k]
    for (int k = 0; k < 3; k++) g->zp[k] = DADD(DADD(0.0, DMUL(zv[0], Einv[k])), DMUL(zv[1], Einv[3 + k]));
    if (E_out) for (int k = 0; k < 9; k++) { E_out[k] = E[k]; Einv_out[k] = Einv[k]; }
}

// DR.h:2620-2648: the four half-planes are applied in sequence, each clamped against the running bounds.
// (formulation that follows the reference line by line; kept for the equivalence test)
DEODR_HD void edge_row_span_reference(const EdgeGeom &g, int width, int y, int *x_begin, int *x_end) {
    int xb = 0, xe = width - 1;
    for (int k = 0; k < 4; k++) {
        const double *q = g.ineq + 3 * k;
        double num = -DADD(DMUL(q[1], (double)y), q[2]);
        if (q[0] < 0) {
            int t = floor_div_clamped(num, q[0], xb - 1, xe + 1);
            if (t < xe) xe = t;
        } else {
            int t = to_short((double)(1 + floor_div_clamped(num, q[0], xb - 1, xe + 1)));
            if (t > xb) xb = t;
        }
    }
    *x_begin = xb;
    *x_end = xe;
}

// Same result with the four quotients computed side by side first (they do not depend on the running bounds; only
// the clamps and the rare incremental fall-back do), which shortens the dependent chain ~4x.
DEODR_HD void edge_row_span(const EdgeGeom &g, int width, int y, int *x_begin, int *x_end) {
    const double yd = (double)y;
    double num[4];
    int fq[4];
    bool normal[4], unsettled[4];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < 4; k++) {
        const double *q = g.ineq + 3 * k;
        num[k] = -DADD(DMUL(q[1], yd), q[2]);
        normal[k] = DMUL(fabs(q[0]), 32767.0) > DADD(fabs(num[k]), fabs(q[0]));
        unsettled[k] = floor_quotient_try(num[k], q[0], &fq[k]);
    }
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < 4; k++)
        if (normal[k] && unsettled[k]) fq[k] = floor_quotient_exact(num[k], g.ineq[3 * k]);
    int xb = 0, xe = width - 1;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < 4; k++) {
        const double q0 = g.ineq[3 * k];
        const int lo = xb - 1, hi = xe + 1;
        int x;
        if (normal[k]) {
            x = fq[k];
            if (x < lo) x = wrap16(lo);
            if (x > hi) x = wrap16(hi);
        } else {
            x = monotone_search(num[k], q0, lo, hi, q0 > 0 ? 0 : 1);
        }
        if (q0 < 0) {
            if (x < xe) xe = x;
        } else {
            const int t = wrap16(1 + x);
            if (t > xb) xb = t;
        }
    }
    *x_begin = xb;
    *x_end = xe;
}

DEODR_HD int lowest_bit(uint32_t m) {
#if defined(__CUDA_ARCH__)
    return __ffs((int)m) - 1;
#else
    return __builtin_ctz(m);
#endif
}

DEODR_HD int lowest_bit64(unsigned long long m) {
#if defined(__CUDA_ARCH__)
    return __ffsll((long long)m) - 1;
#else
    return __builtin_ctzll(m);
#endif
}

DEODR_HD int highest_bit64(unsigned long long m) {
#if defined(__CUDA_ARCH__)
    return 63 - __clzll((long long)m);
#else
    return 63 - __builtin_clzll(m);
#endif
}

// sort key: radix-ascending order of this key == descending order of the depth sum (DR.h:2656-2662, 2781)
DEODR_HD uint64_t depth_desc_key(double s) {
#if defined(__CUDA_ARCH__)
    uint64_t b = (uint64_t)__double_as_longlong(s);
#else
    union { double d; uint64_t u; } cvt; cvt.d = s; uint64_t b = cvt.u;
#endif
    uint64_t asc = (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
    return ~asc;
}

}  // namespace deodr
