// delaunay.cu — the Delaunay triangulation of 2-D points as one CSR row per observation (sm_90a), for DelaunayBuilder
// (the reference builds it with scipy.spatial.Delaunay, src/squidpy/gr/neighbors.py:272-332).
//
// Every point builds its own star — the cyclic, counter-clockwise list of its Delaunay neighbours — by Bowyer–Watson insertion
// restricted to that star: a triangle (i, a, b) of the star conflicts with a point l iff l lies inside its circumcircle
// (dpred::incircle_sos > 0); a hull gap is a ghost vertex G, and the ghost triangles (i, a, G) / (i, G, b) conflict with l iff l
// lies strictly on the outer side of the hull edge i-a / b-i, or strictly inside that edge.  The triangles of the star that
// conflict with l are consecutive; inserting l replaces the neighbours strictly inside that run by l.  The result does not
// depend on the insertion order, so the star is exact once every point that could conflict has been offered:
//   pass 1  one thread per point walks the rings of the PointGrid around it (graph.cu) and stops once the star has no ghost and
//           the unvisited points are farther than twice its largest circumradius (the circle through i of radius R lies within
//           2R of i).  Floating point only decides when to stop looking, with slack; what is kept is decided by exact predicates.
//   pass 2  one CTA per point pass 1 could not certify (hull points, stars that grow past the ring budget or the register
//           capacity) walks the same rings without a budget: the threads test each ring's cells against the star's conflict
//           region (circumdiscs and outer half-planes), test the points of the cells that hit exactly, and thread 0 inserts the
//           conflicting ones nearest first; the walk stops on pass 1's certificate or when the grid is exhausted.  The star
//           lives in global memory and may reach n - 1 neighbours.
// Exact duplicates are collapsed first: the lowest index of each group is the vertex, the other copies get empty rows.
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>
#include <limits.h>
#include <math.h>

#include <algorithm>

#include "delaunay.cuh"
#include "delaunay_pred.h"

namespace {

constexpr int DT_CAP1 = 32;      // star capacity of pass 1 (per thread, local memory)
constexpr int DT_PEND = 8;       // collinear candidates pass 1 holds back until its star has a first triangle
constexpr int DT_RINGS = 4;      // ring budget of pass 1
constexpr int DT_P2_THREADS = 256;
constexpr int DT_P2_BUF = 2048;  // conflicting points collected per scan of pass 2
constexpr int32_t GHOST = -1;

struct Pts {
    const double* xy;  // original order, interleaved
    const int32_t* rep;
    DP_HD void get(int32_t j, double* p) const {
        p[0] = xy[2 * (int64_t)j];
        p[1] = xy[2 * (int64_t)j + 1];
    }
};

// l strictly inside the segment a-b, for collinear a, b, l
__device__ __forceinline__ bool strictly_between(const double* a, const double* b, const double* l) {
    if (a[0] != b[0]) return (a[0] < l[0] && l[0] < b[0]) || (b[0] < l[0] && l[0] < a[0]);
    return (a[1] < l[1] && l[1] < b[1]) || (b[1] < l[1] && l[1] < a[1]);
}

// does l conflict with the star triangle (i, p, q)?  (p or q may be the ghost)
__device__ __forceinline__ bool conflicts(const Pts& P, int32_t i, const double* qi, int32_t p, int32_t q, int32_t l, const double* pl) {
    if (l == p || l == q) return false;
    double a[2], b[2];
    if (p == GHOST) {
        P.get(q, b);
        const int o = dpred::orient2d(qi, pl, b);
        return o > 0 || (o == 0 && strictly_between(qi, b, pl));
    }
    P.get(p, a);
    if (q == GHOST) {
        const int o = dpred::orient2d(qi, a, pl);
        return o > 0 || (o == 0 && strictly_between(qi, a, pl));
    }
    P.get(q, b);
    return dpred::incircle_sos(qi, a, b, pl, i, p, q, l) > 0;
}

// Bowyer–Watson step on the star s[0 .. m) of i: returns the new length, m if l does not conflict, -1 past `cap`, -2 if every
// triangle conflicts (impossible for a valid star; reported, never silently kept).
__device__ int star_insert(const Pts& P, int32_t i, const double* qi, int32_t* s, int m, int cap, int32_t l) {
    double pl[2];
    P.get(l, pl);
    int start = -1, end = -1;
    bool c0 = false, prev = false, any = false, all = true;
    for (int k = 0; k < m; ++k) {
        const bool c = conflicts(P, i, qi, s[k], s[k + 1 < m ? k + 1 : 0], l, pl);
        if (k == 0) c0 = c;
        if (c && k > 0 && !prev) start = k;
        if (!c && k > 0 && prev) end = k - 1;
        any |= c, all &= c, prev = c;
    }
    if (!any) return m;
    if (all) return -2;
    if (c0 && !prev) start = 0;
    if (prev && !c0) end = m - 1;
    const int removed = (end - start + m) % m;  // neighbours strictly inside the run of conflicting triangles
    const int nm = m - removed + 1;
    if (nm > cap) return -1;
    if (start <= end) {  // remove s[start + 1 .. end], put l at start + 1
        const int shift = 1 - removed;
        if (shift > 0)
            for (int k = m - 1; k > end; --k) s[k + shift] = s[k];
        else if (shift < 0)
            for (int k = end + 1; k < m; ++k) s[k + shift] = s[k];
        s[start + 1] = l;
    } else {  // the run wraps: keep s[end + 1 .. start], then l
        const int keep = start - end;
        for (int k = 0; k < keep; ++k) s[k] = s[end + 1 + k];
        s[keep] = l;
    }
    return nm;
}

// squared circumradius of (i, a, b), INFINITY when it cannot be bounded reliably in floating point
__device__ __forceinline__ double circum_r2(const double* qi, const double* a, const double* b, double* cx, double* cy) {
    const double ax = a[0] - qi[0], ay = a[1] - qi[1], bx = b[0] - qi[0], by = b[1] - qi[1];
    const double t1 = ax * by, t2 = ay * bx, D = 2.0 * (t1 - t2);
    if (!(fabs(D) > 2e-6 * (fabs(t1) + fabs(t2)))) return INFINITY;
    const double na = ax * ax + ay * ay, nb = bx * bx + by * by;
    const double ux = (by * na - ay * nb) / D, uy = (ax * nb - bx * na) / D;
    *cx = qi[0] + ux, *cy = qi[1] + uy;
    return (ux * ux + uy * uy) * (1.0 + 1e-6);
}

}  // namespace

// rep[i]: the lowest index of the points with exactly i's coordinates (they share i's cell)
__global__ void dt_dedup_kernel(const double2* __restrict__ pts, const int32_t* __restrict__ idx_sorted, const int32_t* __restrict__ cell_start,
                                int64_t n, GridGeom gm, int32_t* __restrict__ rep) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n) return;
    const double2 q = pts[s];
    const int32_t qi = idx_sorted[s];
    const int64_t c = (int64_t)grid_cell_coord(q.y, gm.y0, gm.inv_cell, gm.gy) * gm.gx + grid_cell_coord(q.x, gm.x0, gm.inv_cell, gm.gx);
    int32_t r = qi;
    for (int32_t t = cell_start[c]; t < cell_start[c + 1]; ++t) {
        const double2 p = pts[t];
        if (p.x == q.x && p.y == q.y) r = min(r, idx_sorted[t]);
    }
    rep[qi] = r;
}

// first[0]: the lowest index whose coordinates differ from point 0's (INT_MAX if none)
// range[0] = 1 if a coordinate lies outside the range the predicates are exact for (DT_COORD_MAX, DT_COORD_MIN, see delaunay_pred.h)
__global__ void dt_first_distinct_kernel(const double* __restrict__ xy, int64_t n, int* __restrict__ first, int* __restrict__ range) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        if (xy[2 * i] != xy[0] || xy[2 * i + 1] != xy[1]) atomicMin(first, (int)i);
        for (int d = 0; d < 2; ++d) {
            const double v = fabs(xy[2 * i + d]);
            if (v > dpred::COORD_MAX || (v != 0.0 && v < dpred::COORD_MIN)) atomicOr(range, 1);
        }
    }
}

// flag = 1 iff some point is off the line through point 0 and point first[0]: at least three distinct, non-collinear points
__global__ void dt_noncollinear_kernel(const double* __restrict__ xy, int64_t n, const int* __restrict__ first, int* __restrict__ flag) {
    const int f = *first;
    if (f == INT_MAX) return;
    const double a[2] = {xy[0], xy[1]}, b[2] = {xy[2 * (int64_t)f], xy[2 * (int64_t)f + 1]};
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double c[2] = {xy[2 * i], xy[2 * i + 1]};
        if (dpred::orient2d(a, b, c) != 0) {
            *flag = 1;
            return;
        }
    }
}

// Pass 1: one thread per point (in cell order).  cnt[i] = degree and nb[i * CAP1 ..] the neighbours, or i queued for pass 2.
__global__ void __launch_bounds__(128) dt_pass1_kernel(const double2* __restrict__ pts, const int32_t* __restrict__ idx_sorted,
                                                       const int32_t* __restrict__ cell_start, int64_t n, GridGeom gm, Pts P,
                                                       int64_t* __restrict__ cnt, int32_t* __restrict__ nb, int32_t* __restrict__ queue,
                                                       int* __restrict__ n_queue) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n) return;
    const int32_t i = idx_sorted[s];
    if (P.rep[i] != i) {
        cnt[i] = 0;
        return;
    }
    const double2 q2 = pts[s];
    const double qi[2] = {q2.x, q2.y};
    const int cx = grid_cell_coord(qi[0], gm.x0, gm.inv_cell, gm.gx), cy = grid_cell_coord(qi[1], gm.y0, gm.inv_cell, gm.gy);
    int32_t st[DT_CAP1];
    int32_t pend[DT_PEND];
    int m = 0, np = 0;
    bool ok = true, done = false;
    for (int r = 0; r <= DT_RINGS && ok && !done; ++r) {
        for (int yy = cy - r; yy <= cy + r && ok; ++yy) {
            if (yy < 0 || yy >= gm.gy) continue;
            const int step = (yy == cy - r || yy == cy + r) ? 1 : 2 * r;
            for (int xx = cx - r; xx <= cx + r && ok; xx += (step > 0 ? step : 1)) {
                if (xx >= 0 && xx < gm.gx) {
                    const int64_t c = (int64_t)yy * gm.gx + xx;
                    for (int32_t t = cell_start[c]; t < cell_start[c + 1] && ok; ++t) {
                        const int32_t j = idx_sorted[t];
                        if (j == i || P.rep[j] != j) continue;
                        if (m == 0) {
                            st[0] = j, m = 1;
                        } else if (m == 1) {  // no triangle yet: wait for a point off the line i-st[0]
                            double a[2];
                            P.get(st[0], a);
                            const double b[2] = {pts[t].x, pts[t].y};
                            const int o = dpred::orient2d(qi, a, b);
                            if (o == 0) {
                                if (np == DT_PEND) ok = false;
                                else pend[np++] = j;
                                continue;
                            }
                            const int32_t a0 = st[0];
                            st[0] = o > 0 ? a0 : j, st[1] = o > 0 ? j : a0, st[2] = GHOST, m = 3;
                            for (int u = 0; u < np && ok; ++u) {
                                m = star_insert(P, i, qi, st, m, DT_CAP1, pend[u]);
                                ok = m > 0;
                            }
                        } else {
                            m = star_insert(P, i, qi, st, m, DT_CAP1, j);
                            ok = m > 0;
                        }
                    }
                }
                if (r == 0) break;
            }
        }
        if (!ok || m < 3) continue;
        const double lb = grid_unvisited_bound(gm, make_double2(qi[0], qi[1]), cx, cy, r);
        if (lb < 0.0) {  // every point has been offered
            done = true;
            break;
        }
        double r2max = 0.0;
        for (int k = 0; k < m && r2max < INFINITY; ++k) {
            const int32_t p = st[k], q = st[k + 1 < m ? k + 1 : 0];
            if (p == GHOST || q == GHOST) {
                r2max = INFINITY;
                break;
            }
            double a[2], b[2], ux, uy;
            P.get(p, a), P.get(q, b);
            r2max = fmax(r2max, circum_r2(qi, a, b, &ux, &uy));
        }
        if (4.0 * r2max < lb) done = true;
    }
    if (!(ok && done && m >= 3)) {
        queue[atomicAdd(n_queue, 1)] = i;
        cnt[i] = -1;
        return;
    }
    int d = 0;
    for (int k = 0; k < m; ++k)
        if (st[k] != GHOST) nb[(int64_t)i * DT_CAP1 + d++] = st[k];
    cnt[i] = d;
}

// The conflict region of star triangle k in a form the box test reads cheaply: a disc (kind 0: centre, squared radius), an outer
// half-plane (kind 1: origin u, edge direction e) or everything (kind 2: no reliable floating-point disc)
struct RegionTerm {
    double a, b, c, d;
    int kind;
};

__device__ RegionTerm region_term(const Pts& P, const double* qi, int32_t p, int32_t q) {
    RegionTerm t{0.0, 0.0, 0.0, 0.0, 2};
    double a[2], b[2];
    if (q == GHOST) {
        P.get(p, a);
        t = RegionTerm{qi[0], qi[1], a[0] - qi[0], a[1] - qi[1], 1};
    } else if (p == GHOST) {
        P.get(q, b);
        t = RegionTerm{b[0], b[1], qi[0] - b[0], qi[1] - b[1], 1};
    } else {
        P.get(p, a), P.get(q, b);
        double cx, cy;
        const double r2 = circum_r2(qi, a, b, &cx, &cy);
        if (r2 < INFINITY) t = RegionTerm{cx, cy, r2, 0.0, 0};
    }
    return t;
}

// conservative: may the box [x0, x1] x [y0, y1] hold a point of the region?
__device__ __forceinline__ bool term_hits(const RegionTerm& t, double x0, double y0, double x1, double y1) {
    if (t.kind == 0) {
        const double dx = fmax(fmax(x0 - t.a, t.a - x1), 0.0), dy = fmax(fmax(y0 - t.b, t.b - y1), 0.0);
        return dx * dx + dy * dy <= t.c;
    }
    if (t.kind == 1) {
        const double xs[2] = {x0, x1}, ys[2] = {y0, y1};
        for (int i = 0; i < 2; ++i)
            for (int j = 0; j < 2; ++j) {
                const double wx = xs[i] - t.a, wy = ys[j] - t.b;
                if (t.c * wy - t.d * wx >= -1e-9 * (fabs(t.c) + fabs(t.d)) * (fabs(wx) + fabs(wy))) return true;
            }
        return false;
    }
    return true;
}

constexpr int DT_TERMS = 256;  // conflict-region terms pass 2 keeps in shared memory

// Pass 2: one CTA per queued point, walking the rings of cells around it as pass 1 does but without a ring budget or a star
// capacity.  The threads test ring r's cells against the conflict region of the current star (every point while the star has
// no first triangle), test the points of the cells that hit exactly, and the conflicting ones are sorted by distance and
// inserted by thread 0.  The walk stops when pass 1's certificate holds or the grid is exhausted, so a point costs the cells
// within twice its largest circumradius (all cells for hull points).  Stars in global scratch (n entries per CTA); the
// finished star goes to the pool.
__device__ __forceinline__ bool ring_cell(int r, int e, int cx, int cy, int* xx, int* yy) {
    if (r == 0) {
        *xx = cx, *yy = cy;
    } else if (e < 2 * r + 1) {
        *xx = cx - r + e, *yy = cy - r;
    } else if (e < 4 * r + 2) {
        *xx = cx - r + (e - 2 * r - 1), *yy = cy + r;
    } else {
        const int k = e - 4 * r - 2;
        *xx = (k & 1) ? cx + r : cx - r, *yy = cy - r + 1 + (k >> 1);
    }
    return true;
}

__global__ void __launch_bounds__(DT_P2_THREADS) dt_pass2_kernel(const double2* __restrict__ pts, const int32_t* __restrict__ idx_sorted,
                                                                 const int32_t* __restrict__ cell_start, int64_t n, GridGeom gm, Pts P,
                                                                 const int32_t* __restrict__ queue, int n_queue, int32_t* __restrict__ scratch,
                                                                 int64_t* __restrict__ cnt, int64_t* __restrict__ pool_off,
                                                                 int32_t* __restrict__ pool, unsigned long long* __restrict__ pool_fill,
                                                                 int* __restrict__ err) {
    __shared__ int32_t buf[DT_P2_BUF];
    __shared__ int s_hits, s_m, s_err, s_r, s_done;
    __shared__ RegionTerm s_terms[DT_TERMS];
    __shared__ double s_key[DT_P2_BUF];
    __shared__ int32_t s_sorted[DT_P2_BUF];
    int32_t* st = scratch + (int64_t)blockIdx.x * n;
    const double bx1 = gm.x0 + gm.gx * gm.cell, by1 = gm.y0 + gm.gy * gm.cell;
    const double slack = 1e-9 * gm.cell + 1e-12 * (fabs(gm.x0) + fabs(gm.y0) + fabs(bx1) + fabs(by1));
    const int rmax = gm.gx > gm.gy ? gm.gx : gm.gy;
    for (int w = blockIdx.x; w < n_queue; w += gridDim.x) {
        const int32_t i = queue[w];
        double qi[2];
        P.get(i, qi);
        const int cx = grid_cell_coord(qi[0], gm.x0, gm.inv_cell, gm.gx), cy = grid_cell_coord(qi[1], gm.y0, gm.inv_cell, gm.gy);
        if (threadIdx.x == 0) s_m = 0, s_err = 0, s_r = 0, s_done = 0;
        __syncthreads();
        for (int round = 0;; ++round) {
            if (threadIdx.x == 0) {
                s_hits = 0;
                if (round == (1 << 22)) s_err = 4;  // a walk never needs this many rounds
            }
            __syncthreads();
            if (s_err || s_done) break;
            const int m = s_m, r = s_r;
            const bool seeded = m >= 3, cached = seeded && m <= DT_TERMS;
            if (cached)
                for (int k = threadIdx.x; k < m; k += blockDim.x) s_terms[k] = region_term(P, qi, st[k], st[k + 1 < m ? k + 1 : 0]);
            __syncthreads();
            const int n_ring = r == 0 ? 1 : 8 * r;
            for (int e = threadIdx.x; e < n_ring; e += blockDim.x) {
                int xx, yy;
                ring_cell(r, e, cx, cy, &xx, &yy);
                if (xx < 0 || xx >= gm.gx || yy < 0 || yy >= gm.gy) continue;
                const int64_t c = (int64_t)yy * gm.gx + xx;
                const int32_t b0 = cell_start[c], b1 = cell_start[c + 1];
                if (b0 == b1) continue;
                if (seeded) {
                    const double x0 = gm.x0 + xx * gm.cell - slack, x1 = gm.x0 + (xx + 1) * gm.cell + slack;
                    const double y0 = gm.y0 + yy * gm.cell - slack, y1 = gm.y0 + (yy + 1) * gm.cell + slack;
                    bool hit = false;
                    for (int k = 0; k < m && !hit; ++k)
                        hit = cached ? term_hits(s_terms[k], x0, y0, x1, y1) : term_hits(region_term(P, qi, st[k], st[k + 1 < m ? k + 1 : 0]), x0, y0, x1, y1);
                    if (!hit) continue;
                }
                for (int32_t t = b0; t < b1; ++t) {
                    const int32_t l = idx_sorted[t];
                    if (l == i || P.rep[l] != l) continue;
                    const double pl[2] = {pts[t].x, pts[t].y};
                    bool cf = !seeded;
                    for (int k = 0; k < m && !cf; ++k) cf = conflicts(P, i, qi, st[k], st[k + 1 < m ? k + 1 : 0], l, pl);
                    if (cf) {
                        const int slot = atomicAdd(&s_hits, 1);
                        if (slot < DT_P2_BUF) buf[slot] = l;
                    }
                }
            }
            __syncthreads();
            const int hits = s_hits;
            // nearest first (by squared distance, then index): any order gives the same star, this one keeps it small
            const int nh = hits < DT_P2_BUF ? hits : DT_P2_BUF;
            for (int k = threadIdx.x; k < nh; k += blockDim.x) {
                double p[2];
                P.get(buf[k], p);
                const double dx = p[0] - qi[0], dy = p[1] - qi[1];
                s_key[k] = dx * dx + dy * dy;
            }
            __syncthreads();
            for (int k = threadIdx.x; k < nh; k += blockDim.x) {
                const double kk = s_key[k];
                const int32_t kv = buf[k];
                int rank = 0;
                for (int u = 0; u < nh; ++u) rank += s_key[u] < kk || (s_key[u] == kk && buf[u] < kv);
                s_sorted[rank] = kv;
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                int mm = s_m;
                const bool was_seeded = mm >= 3;
                for (int k = 0; k < nh && mm >= 0; ++k) {
                    const int32_t l = s_sorted[k];
                    if (mm == 0) {
                        st[0] = l, mm = 1;
                    } else if (mm == 1) {  // the first triangle: the first point off the line through i and st[0]
                        double a[2], b[2];
                        P.get(st[0], a), P.get(l, b);
                        const int o = dpred::orient2d(qi, a, b);
                        if (o == 0) continue;
                        const int32_t a0 = st[0];
                        st[0] = o > 0 ? a0 : l, st[1] = o > 0 ? l : a0, st[2] = GHOST, mm = 3;
                    } else {
                        mm = star_insert(P, i, qi, st, mm, (int)n, l);
                    }
                }
                if (mm < 0) {
                    s_err = mm == -2 ? 2 : 1;
                } else {
                    s_m = mm;
                    if (mm >= 3 && !was_seeded) {
                        s_r = 0;  // the first triangle: offer the rings seen so far again (points skipped while seeding)
                    } else if (hits <= DT_P2_BUF || mm < 3) {  // else the same ring again: it held more conflicting points than one round takes
                        const double lb = grid_unvisited_bound(gm, make_double2(qi[0], qi[1]), cx, cy, r);
                        if (lb < 0.0 || r >= rmax) {
                            s_done = 1;
                            if (mm < 3) s_err = 3;
                        } else if (mm >= 3) {
                            double r2max = 0.0;
                            for (int k = 0; k < mm && r2max < INFINITY; ++k) {
                                const int32_t p = st[k], q = st[k + 1 < mm ? k + 1 : 0];
                                if (p == GHOST || q == GHOST) {
                                    r2max = INFINITY;
                                } else {
                                    double a[2], b[2], ux, uy;
                                    P.get(p, a), P.get(q, b);
                                    r2max = fmax(r2max, circum_r2(qi, a, b, &ux, &uy));
                                }
                            }
                            s_done = 4.0 * r2max < lb;
                        }
                        s_r = r + 1;
                    }
                }
            }
            __syncthreads();
        }
        if (s_err) {
            if (threadIdx.x == 0) atomicCAS(err, 0, s_err);
            __syncthreads();
            continue;
        }
        __shared__ unsigned long long s_off;
        const int m = s_m;
        if (threadIdx.x == 0) {
            int d = 0;
            for (int k = 0; k < m; ++k) d += st[k] != GHOST;
            s_off = atomicAdd(pool_fill, (unsigned long long)d);
            cnt[i] = d;
            pool_off[w] = (int64_t)s_off;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int o = 0;
            for (int k = 0; k < m; ++k)
                if (st[k] != GHOST) pool[s_off + o++] = st[k];
        }
        __syncthreads();
    }
}

// rows into CSR (unsorted within a row; a segmented sort follows)
__global__ void dt_fill_kernel(int64_t n, const int64_t* __restrict__ cnt1, const int32_t* __restrict__ nb, const int32_t* __restrict__ slot,
                               const int64_t* __restrict__ pool_off, const int32_t* __restrict__ pool, const int64_t* __restrict__ indptr,
                               int32_t* __restrict__ out) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t o = indptr[i], d = indptr[i + 1] - o;
        const int32_t* src = slot[i] >= 0 ? pool + pool_off[slot[i]] : nb + i * DT_CAP1;
        for (int64_t k = 0; k < d; ++k) out[o + k] = src[k];
    }
}

__global__ void dt_slot_kernel(const int32_t* __restrict__ queue, int n_queue, int32_t* __restrict__ slot) {
    for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < n_queue; w += gridDim.x * blockDim.x) slot[queue[w]] = w;
}

int delaunay_csr(sqb_ctx* c, PointGrid& g, int64_t n, DevBuf<int64_t>& indptr, DevBuf<int32_t>& idx, int64_t* nnz, int64_t* pass_counts) {
    SQB_CHECK(n < 2147483647LL, SQB_ERR_UNSUPPORTED, "Delaunay: n=%lld points do not fit int32 indices", (long long)n);
    const unsigned gb = sqb_grid_rows(c, n, 256);
    DevBuf<int32_t> rep(c->stream), nb(c->stream), queue(c->stream), slot(c->stream), scratch(c->stream), pool(c->stream);
    DevBuf<int64_t> cnt(c->stream), pool_off(c->stream);
    DevBuf<int> flags(c->stream);
    DevBuf<unsigned long long> fill(c->stream);
    DevBuf<uint8_t> tmp(c->stream);
    SQB_TRY(rep.alloc(n));
    SQB_TRY(flags.alloc(5));  // first distinct, non-collinear, queue length, pass-2 error, coordinate range
    const int init[5] = {INT_MAX, 0, 0, 0, 0};
    SQB_CUDA(cudaMemcpyAsync(flags.p, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        dt_first_distinct_kernel<<<gb, 256, 0, c->stream>>>(g.d_xy.p, n, flags.p, flags.p + 4);
        dt_noncollinear_kernel<<<gb, 256, 0, c->stream>>>(g.d_xy.p, n, flags.p, flags.p + 1);
        dt_dedup_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, c->stream>>>(g.d_pts.p, g.d_idx_sorted.p, g.d_cell_start.p, n, g.gm, rep.p);
    }
    SQB_POST_LAUNCH();
    int hflags[5];
    SQB_CUDA(cudaMemcpyAsync(hflags, flags.p, sizeof(hflags), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    SQB_CHECK(hflags[4] == 0, SQB_ERR_INVALID, "Delaunay: coordinates must be 0 or of magnitude between 2^-120 and 2^120 (exact predicates)");
    SQB_CHECK(hflags[1] == 1, SQB_ERR_INVALID, "QhullError: the Delaunay triangulation needs at least three distinct points that are not all collinear");
    const Pts P{g.d_xy.p, rep.p};
    SQB_TRY(cnt.alloc(n + 1));
    SQB_TRY(nb.alloc((size_t)n * DT_CAP1));
    SQB_TRY(queue.alloc(n));
    SQB_CUDA(cudaMemsetAsync(cnt.p + n, 0, sizeof(int64_t), c->stream));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        dt_pass1_kernel<<<(unsigned)ceil_div64(n, 128), 128, 0, c->stream>>>(g.d_pts.p, g.d_idx_sorted.p, g.d_cell_start.p, n, g.gm, P, cnt.p, nb.p,
                                                                             queue.p, flags.p + 2);
    }
    SQB_POST_LAUNCH();
    int n_queue = 0;
    SQB_CUDA(cudaMemcpyAsync(&n_queue, flags.p + 2, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    SQB_TRY(slot.alloc(n));
    SQB_CUDA(cudaMemsetAsync(slot.p, 0xff, n * sizeof(int32_t), c->stream));
    SQB_TRY(pool_off.alloc(n_queue > 0 ? n_queue : 1));
    if (n_queue > 0) {
        // at most 1 GiB of star scratch (n entries per CTA), at most two CTAs per SM
        const int64_t per = (int64_t)n * (int64_t)sizeof(int32_t);
        int64_t ctas = std::min<int64_t>(n_queue, 2LL * c->sm_count);
        ctas = std::max<int64_t>(1, std::min<int64_t>(ctas, (1LL << 30) / per));
        SQB_TRY(scratch.alloc((size_t)(ctas * n)));
        SQB_TRY(pool.alloc((size_t)6 * n));  // the degrees of all Delaunay vertices sum to below 6n
        SQB_TRY(fill.alloc(1));
        SQB_CUDA(cudaMemsetAsync(fill.p, 0, sizeof(unsigned long long), c->stream));
        {
            SqbLaunchScope scope(c, SQB_K_MISC);
            dt_pass2_kernel<<<(unsigned)ctas, DT_P2_THREADS, 0, c->stream>>>(g.d_pts.p, g.d_idx_sorted.p, g.d_cell_start.p, n, g.gm, P, queue.p,
                                                                             n_queue, scratch.p, cnt.p, pool_off.p, pool.p, fill.p, flags.p + 3);
            dt_slot_kernel<<<sqb_grid_rows(c, n_queue, 256), 256, 0, c->stream>>>(queue.p, n_queue, slot.p);
        }
        SQB_POST_LAUNCH();
        int perr = 0;
        SQB_CUDA(cudaMemcpyAsync(&perr, flags.p + 3, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaStreamSynchronize(c->stream));
        SQB_CHECK(perr == 0, SQB_ERR_INVALID, "Delaunay: a star could not be completed (code %d)", perr);
        scratch.release();
    } else {
        SQB_TRY(pool.alloc(1));
    }
    SQB_TRY(indptr.alloc(n + 1));
    size_t bytes = 0;
    SQB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, cnt.p, indptr.p, (int)(n + 1), c->stream));
    SQB_TRY(tmp.alloc(bytes > 0 ? bytes : 1));
    SQB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, cnt.p, indptr.p, (int)(n + 1), c->stream));
    int64_t m = 0;
    SQB_CUDA(cudaMemcpyAsync(&m, indptr.p + n, sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    SQB_CHECK(m < INT_MAX, SQB_ERR_UNSUPPORTED, "Delaunay: %lld entries exceed 2^31 - 1", (long long)m);
    DevBuf<int32_t> unsorted(c->stream);
    SQB_TRY(unsorted.alloc(m > 0 ? m : 1));
    SQB_TRY(idx.alloc(m > 0 ? m : 1));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        dt_fill_kernel<<<gb, 256, 0, c->stream>>>(n, cnt.p, nb.p, slot.p, pool_off.p, pool.p, indptr.p, unsorted.p);
    }
    SQB_POST_LAUNCH();
    if (m > 0) {
        bytes = 0;
        SQB_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, bytes, unsorted.p, idx.p, (int)m, (int)n, indptr.p, indptr.p + 1, c->stream));
        SQB_TRY(tmp.alloc(bytes > 0 ? bytes : 1));
        SQB_CUDA(cub::DeviceSegmentedSort::SortKeys(tmp.p, bytes, unsorted.p, idx.p, (int)m, (int)n, indptr.p, indptr.p + 1, c->stream));
        c->launches += 1;
    }
    *nnz = m;
    if (pass_counts) {  // duplicates count as finished by pass 1 (their rows are empty)
        pass_counts[0] = n - n_queue;
        pass_counts[1] = n_queue;
    }
    return SQB_OK;
}

// ---- distances in the coordinates' dtype: numpy's norm(coords[rows] - coords[indices], axis=1) -------------------------------
template <typename T>
__global__ void dt_dist_kernel(const double* __restrict__ xy, const int64_t* __restrict__ indptr, const int32_t* __restrict__ idx, int64_t n,
                               double* __restrict__ dist) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const T xi = (T)xy[2 * i], yi = (T)xy[2 * i + 1];
        for (int64_t t = indptr[i]; t < indptr[i + 1]; ++t) {
            const int32_t j = idx[t];
            const T dx = xi - (T)xy[2 * (int64_t)j], dy = yi - (T)xy[2 * (int64_t)j + 1];
            T d;
            if constexpr (sizeof(T) == 4)
                d = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
            else
                d = __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
            dist[t] = (double)d;
        }
    }
}

int delaunay_dist(sqb_ctx* c, const double* xy, const int64_t* indptr, const int32_t* idx, int64_t n, bool f32, double* dist) {
    SqbLaunchScope scope(c, SQB_K_MISC);
    if (f32)
        dt_dist_kernel<float><<<sqb_grid_rows(c, n, 256), 256, 0, c->stream>>>(xy, indptr, idx, n, dist);
    else
        dt_dist_kernel<double><<<sqb_grid_rows(c, n, 256), 256, 0, c->stream>>>(xy, indptr, idx, n, dist);
    SQB_POST_LAUNCH();
    return SQB_OK;
}

extern "C" {

int sqb_delaunay_2d(sqb_ctx* ctx, const double* xy, int64_t n, int64_t* out_indptr, int32_t* out_idx, int64_t capacity, int64_t* nnz_out,
                    int64_t* out_pass_counts) {
    SQB_CHECK(ctx && xy && out_indptr && nnz_out, SQB_ERR_INVALID, "sqb_delaunay_2d: null argument");
    SQB_CHECK(n >= 0 && n < 2147483647LL, SQB_ERR_UNSUPPORTED, "sqb_delaunay_2d: n=%lld out of range", (long long)n);
    double x0 = INFINITY, y0 = INFINITY, x1 = -INFINITY, y1 = -INFINITY;
    for (int64_t i = 0; i < n; ++i) {
        const double x = xy[2 * i], y = xy[2 * i + 1];
        SQB_CHECK(isfinite(x) && isfinite(y), SQB_ERR_INVALID, "coordinates of observation %lld are not finite", (long long)i);
        x0 = x < x0 ? x : x0, x1 = x > x1 ? x : x1, y0 = y < y0 ? y : y0, y1 = y > y1 ? y : y1;
    }
    SQB_CHECK(n >= 3, SQB_ERR_INVALID, "QhullError: the Delaunay triangulation needs at least three distinct points that are not all collinear");
    sqb_ctx* c = ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    PointGrid g(c->stream);
    g.gm = grid_geometry(x0, y0, x1, y1, n, 0.0, DT_PTS_PER_CELL);
    SQB_TRY(g.d_xy.alloc(2 * n));
    SQB_CUDA(cudaMemcpyAsync(g.d_xy.p, xy, 2 * n * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    SQB_TRY(grid_bucket(c, n, &g));
    DevBuf<int64_t> indptr(c->stream);
    DevBuf<int32_t> idx(c->stream);
    int64_t nnz = 0;
    SQB_TRY(delaunay_csr(c, g, n, indptr, idx, &nnz, out_pass_counts));
    *nnz_out = nnz;
    SQB_CUDA(cudaMemcpyAsync(out_indptr, indptr.p, (n + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    if (out_idx && capacity >= nnz && nnz > 0)
        SQB_CUDA(cudaMemcpyAsync(out_idx, idx.p, nnz * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    return SQB_OK;
}

}  // extern "C"
