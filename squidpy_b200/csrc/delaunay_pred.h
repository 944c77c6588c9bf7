// delaunay_pred.h — exact orientation and in-circle predicates on float64 coordinates, after Shewchuk, "Adaptive Precision
// Floating-Point Arithmetic and Fast Robust Geometric Predicates" (Discrete Comput. Geom. 18, 1997).  A floating-point
// evaluation is returned when its proven error bound (the paper's stage-A bounds) decides the sign; otherwise the determinant
// is evaluated exactly with expansion arithmetic (two-sum, two-product via FMA, zero-eliminating expansion sums and scaling).
// Compiles as CUDA device/host code and as plain C++ (tests build it with g++ -ffp-contract=off).  The in-circle terms are of
// degree 4 and their expansion tails reach about 2^-212 of the leading term, so no term may overflow and no tail may
// underflow: coordinates must be 0 or of magnitude in [COORD_MIN, COORD_MAX] = [2^-120, 2^120]; the callers check this.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define DP_HD __host__ __device__ __forceinline__
#else
#define DP_HD inline
#endif

namespace dpred {

// 2^120: a degree-4 term of coordinates or their differences stays below 2^490, far from overflow.
constexpr double COORD_MAX = 1.329227995784916e36;
// 2^-120: the smallest term, a product of four differences of at least 2^-172 each, carries tails down to about 2^-900, far
// above the smallest normal double (2^-1022).
constexpr double COORD_MIN = 7.52316384526264e-37;

// all arithmetic below is written so that no multiply-add may be contracted: the device build uses -fmad=false and the host
// build -ffp-contract=off; fma() is only called explicitly, where the exact product error is wanted
DP_HD void two_sum(double a, double b, double& x, double& y) {
    x = a + b;
    const double bv = x - a, av = x - bv;
    y = (a - av) + (b - bv);
}

DP_HD void two_prod(double a, double b, double& x, double& y) {
    x = a * b;
    y = fma(a, b, -x);
}

// h = e + f (nonoverlapping expansions in increasing magnitude), zero components dropped; returns the length of h
DP_HD int expansion_sum(int elen, const double* e, int flen, const double* f, double* h) {
    double Q, Qnew, hh, enow, fnow;
    int ei = 0, fi = 0, hi = 0;
    if (elen == 0) {
        for (int i = 0; i < flen; ++i) h[i] = f[i];
        return flen;
    }
    if (flen == 0) {
        for (int i = 0; i < elen; ++i) h[i] = e[i];
        return elen;
    }
    enow = e[0], fnow = f[0];
    if ((fnow > enow) == (fnow > -enow)) {
        Q = enow, enow = ++ei < elen ? e[ei] : 0.0;
    } else {
        Q = fnow, fnow = ++fi < flen ? f[fi] : 0.0;
    }
    while (ei < elen && fi < flen) {
        if ((fnow > enow) == (fnow > -enow)) {
            two_sum(Q, enow, Qnew, hh);
            enow = ++ei < elen ? e[ei] : 0.0;
        } else {
            two_sum(Q, fnow, Qnew, hh);
            fnow = ++fi < flen ? f[fi] : 0.0;
        }
        Q = Qnew;
        if (hh != 0.0) h[hi++] = hh;
    }
    while (ei < elen) {
        two_sum(Q, enow, Qnew, hh);
        enow = ++ei < elen ? e[ei] : 0.0;
        Q = Qnew;
        if (hh != 0.0) h[hi++] = hh;
    }
    while (fi < flen) {
        two_sum(Q, fnow, Qnew, hh);
        fnow = ++fi < flen ? f[fi] : 0.0;
        Q = Qnew;
        if (hh != 0.0) h[hi++] = hh;
    }
    if (Q != 0.0 || hi == 0) h[hi++] = Q;
    return hi;
}

// h = e * b, zero components dropped
DP_HD int scale_expansion(int elen, const double* e, double b, double* h) {
    double Q, sum, hh, p1, p0;
    int hi = 0;
    two_prod(e[0], b, Q, hh);
    if (hh != 0.0) h[hi++] = hh;
    for (int i = 1; i < elen; ++i) {
        two_prod(e[i], b, p1, p0);
        two_sum(Q, p0, sum, hh);
        if (hh != 0.0) h[hi++] = hh;
        two_sum(p1, sum, Q, hh);
        if (hh != 0.0) h[hi++] = hh;
    }
    if (Q != 0.0 || hi == 0) h[hi++] = Q;
    return hi;
}

DP_HD int sign_of(double v) { return (v > 0.0) - (v < 0.0); }

// a0 * b1 - b0 * a1 exactly (at most 4 components)
DP_HD int cross2(double a0, double a1, double b0, double b1, double* h) {
    double p[2], q[2];
    two_prod(a0, b1, p[1], p[0]);
    two_prod(b0, a1, q[1], q[0]);
    q[0] = -q[0], q[1] = -q[1];
    return expansion_sum(2, p, 2, q, h);
}

// sign of (a - c) x (b - c): > 0 when a, b, c turn counter-clockwise
DP_HD int orient2d(const double* pa, const double* pb, const double* pc) {
    const double detleft = (pa[0] - pc[0]) * (pb[1] - pc[1]);
    const double detright = (pa[1] - pc[1]) * (pb[0] - pc[0]);
    const double det = detleft - detright;
    const double eps = 1.1102230246251565e-16;  // 2^-53
    const double errbound = (3.0 + 16.0 * eps) * eps * (fabs(detleft) + fabs(detright));
    if (det > errbound || -det > errbound) return sign_of(det);
    // exact: ab + bc + ca of the untranslated coordinates
    double ab[4], bc[4], ca[4], t8[8], d[12];
    const int l1 = cross2(pa[0], pa[1], pb[0], pb[1], ab);
    const int l2 = cross2(pb[0], pb[1], pc[0], pc[1], bc);
    const int l3 = cross2(pc[0], pc[1], pa[0], pa[1], ca);
    const int l4 = expansion_sum(l1, ab, l2, bc, t8);
    const int l5 = expansion_sum(l4, t8, l3, ca, d);
    return sign_of(d[l5 - 1]);
}

// x * x * e + y * y * e (the lifted coordinate times a 12-component expansion), into h (at most 96 components)
DP_HD int lift_times(int elen, const double* e, double x, double y, double s, double* h) {
    double t24[24], x48[48], y48[48];
    int lx = scale_expansion(elen, e, x, t24);
    lx = scale_expansion(lx, t24, s * x, x48);
    int ly = scale_expansion(elen, e, y, t24);
    ly = scale_expansion(ly, t24, s * y, y48);
    return expansion_sum(lx, x48, ly, y48, h);
}

// Always inlined: an out-of-line device build of this function (sm_90a, -O3) returned wrong signs on the H100, while the
// inlined and the -G builds agree with the host build.
DP_HD int incircle_exact(const double* pa, const double* pb, const double* pc, const double* pd) {
    double ab[4], bc[4], cd[4], da[4], ac[4], bd[4], t8[8], abc[12], bcd[12], cda[12], dab[12];
    const int lab = cross2(pa[0], pa[1], pb[0], pb[1], ab);
    const int lbc = cross2(pb[0], pb[1], pc[0], pc[1], bc);
    const int lcd = cross2(pc[0], pc[1], pd[0], pd[1], cd);
    const int lda = cross2(pd[0], pd[1], pa[0], pa[1], da);
    const int lac = cross2(pa[0], pa[1], pc[0], pc[1], ac);
    const int lbd = cross2(pb[0], pb[1], pd[0], pd[1], bd);
    int t = expansion_sum(lcd, cd, lda, da, t8);
    const int lcda = expansion_sum(t, t8, lac, ac, cda);
    t = expansion_sum(lda, da, lab, ab, t8);
    const int ldab = expansion_sum(t, t8, lbd, bd, dab);
    for (int i = 0; i < 4; ++i) bd[i] = -bd[i], ac[i] = -ac[i];
    t = expansion_sum(lab, ab, lbc, bc, t8);
    const int labc = expansion_sum(t, t8, lac, ac, abc);
    t = expansion_sum(lbc, bc, lcd, cd, t8);
    const int lbcd = expansion_sum(t, t8, lbd, bd, bcd);
    double d1[96], d2[96], s1[192], s2[192], det[384];
    int l1 = lift_times(lbcd, bcd, pa[0], pa[1], 1.0, d1);
    int l2 = lift_times(lcda, cda, pb[0], pb[1], -1.0, d2);
    const int ls1 = expansion_sum(l1, d1, l2, d2, s1);
    l1 = lift_times(ldab, dab, pc[0], pc[1], 1.0, d1);
    l2 = lift_times(labc, abc, pd[0], pd[1], -1.0, d2);
    const int ls2 = expansion_sum(l1, d1, l2, d2, s2);
    const int ld = expansion_sum(ls1, s1, ls2, s2, det);
    return sign_of(det[ld - 1]);
}

// sign of the in-circle determinant: > 0 when d lies inside the circle through a, b, c (counter-clockwise), 0 on it
DP_HD int incircle(const double* pa, const double* pb, const double* pc, const double* pd) {
    const double adx = pa[0] - pd[0], bdx = pb[0] - pd[0], cdx = pc[0] - pd[0];
    const double ady = pa[1] - pd[1], bdy = pb[1] - pd[1], cdy = pc[1] - pd[1];
    const double bdxcdy = bdx * cdy, cdxbdy = cdx * bdy, alift = adx * adx + ady * ady;
    const double cdxady = cdx * ady, adxcdy = adx * cdy, blift = bdx * bdx + bdy * bdy;
    const double adxbdy = adx * bdy, bdxady = bdx * ady, clift = cdx * cdx + cdy * cdy;
    const double det = alift * (bdxcdy - cdxbdy) + blift * (cdxady - adxcdy) + clift * (adxbdy - bdxady);
    const double permanent = (fabs(bdxcdy) + fabs(cdxbdy)) * alift + (fabs(cdxady) + fabs(adxcdy)) * blift + (fabs(adxbdy) + fabs(bdxady)) * clift;
    const double eps = 1.1102230246251565e-16;
    const double errbound = (10.0 + 96.0 * eps) * eps * permanent;
    if (det > errbound || -det > errbound) return sign_of(det);
    return incircle_exact(pa, pb, pc, pd);
}

// In-circle with the symbolic perturbation of the lifted coordinate: x^2 + y^2 of point p is raised by eps^(N - p) for an
// infinitesimal eps, so a point of larger index is perturbed by more.  Exactly cocircular quadruples then take the sign of the
// first non-zero coefficient of the perturbation polynomial, in decreasing index order; with a, b, c counter-clockwise the
// coefficient of d is -orient(a, b, c) != 0, so the result is never 0.  It depends only on the four points and the cyclic order
// of (a, b, c), so every point that evaluates a quadruple gets the same answer.
DP_HD int incircle_sos(const double* pa, const double* pb, const double* pc, const double* pd, int64_t ia, int64_t ib, int64_t ic, int64_t id) {
    const int s = incircle(pa, pb, pc, pd);
    if (s != 0) return s;
    const double* P[4] = {pa, pb, pc, pd};
    const int64_t I[4] = {ia, ib, ic, id};
    bool used[4] = {false, false, false, false};
    for (int step = 0; step < 4; ++step) {
        int w = -1;
        for (int k = 0; k < 4; ++k)
            if (!used[k] && (w < 0 || I[k] > I[w])) w = k;
        used[w] = true;
        int c;
        if (w == 0) c = orient2d(pd, pb, pc);
        else if (w == 1) c = orient2d(pd, pc, pa);
        else if (w == 2) c = orient2d(pd, pa, pb);
        else c = -orient2d(pa, pb, pc);
        if (c != 0) return c;
    }
    (void)P;
    return 0;
}

}  // namespace dpred
