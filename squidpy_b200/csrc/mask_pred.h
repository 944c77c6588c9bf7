// mask_pred.h — is a segment within a polygon?  shapely's LineString.within(P), DE-9IM T*F**F***, decided by exact orientation
// signs (dpred::orient2d) and coordinate comparisons only; no intersection point is ever constructed.  Compiles as CUDA
// device/host code and as plain C++ (tests build it with g++ -ffp-contract=off).  Coordinates must be 0 or of magnitude in
// [dpred::COORD_MIN, dpred::COORD_MAX]; the callers check this.
//
// P is given by its boundary edges, every ring of every polygon, each DIRECTED so that P's interior lies on its left (shells
// counter-clockwise, holes clockwise) and of non-zero length.  Every vertex of a ring starts exactly one of its edges.  P is
// assumed valid: rings touch each other at points only, never along an edge.
//
// A segment [p, q] (p != q) is within P iff no point of it is in P's exterior and some point of the open segment is in P's
// interior.  Cut at p, q and every boundary vertex on the open segment ("events"), the segment falls into open pieces that
// either run along a boundary edge or touch no boundary at all, unless an edge crosses it properly (interiors meeting at one
// point): then, a valid boundary having exterior on one side there, the segment is not within.  Each piece is classified at an
// event at one of its ends: the class of p (q) when that end is p (q) off the boundary, else the direction test below.  Taking
// both directions at every event covers every piece without sorting the events.
//
// Direction test at a boundary point v towards d: the boundary near v is a fan of rays from v (one per edge ending at v, two per
// edge passing through it).  The points v + t (d - v) for small t > 0 lie along the boundary when a ray points along d;
// otherwise they lie in the sector clockwise of the first ray counter-clockwise from d, which is exterior when that ray leaves v
// along its edge (interior on the edge's left, i.e. counter-clockwise of the ray) and interior when it arrives at v.
//
// A zero-length segment (p == q) is its point: within iff the point is in P's interior.
#pragma once
#include "delaunay_pred.h"

namespace mpred {

enum { EXTERIOR = 0, BOUNDARY = 1, INTERIOR = 2 };

struct Edge {
    double ax, ay, bx, by;  // directed a -> b, P's interior on the left
};

// > 0 when (a, b, c) turn counter-clockwise
DP_HD int orient(double ax, double ay, double bx, double by, double cx, double cy) {
    const double a[2] = {ax, ay}, b[2] = {bx, by}, c[2] = {cx, cy};
    return dpred::orient2d(a, b, c);
}

// c inside the closed bounding box of [a, b]: for collinear points, c on the closed segment
DP_HD bool in_box(double ax, double ay, double bx, double by, double cx, double cy) {
    return (ax <= bx ? (ax <= cx && cx <= bx) : (bx <= cx && cx <= ax)) && (ay <= by ? (ay <= cy && cy <= by) : (by <= cy && cy <= ay));
}

DP_HD bool on_edge(const Edge& e, double px, double py) {
    return in_box(e.ax, e.ay, e.bx, e.by, px, py) && orient(e.ax, e.ay, e.bx, e.by, px, py) == 0;
}

// Point against the edges that may contain it or cross the horizontal ray to its right (all edges whose closed y-range holds
// py suffice): BOUNDARY when on an edge, else INTERIOR by an odd number of half-open crossings of the ray.
template <typename EdgeAt>
DP_HD int classify_point(double px, double py, int64_t m, EdgeAt edge) {
    bool inside = false;
    for (int64_t k = 0; k < m; ++k) {
        const Edge e = edge(k);
        if ((e.ay > py) != (e.by > py)) {  // the edge straddles the ray's line, half-open at its lower end
            const int o = orient(e.ax, e.ay, e.bx, e.by, px, py);
            if (o == 0) return BOUNDARY;  // on the line through a non-horizontal edge, within its y-range: on the edge
            if (e.by > e.ay ? o > 0 : o < 0) inside = !inside;  // p left of the upward edge: the crossing lies right of p
        } else if (on_edge(e, px, py)) {
            return BOUNDARY;
        }
    }
    return inside ? INTERIOR : EXTERIOR;
}

// The directed edges of one ring of m vertices (interleaved x, y; a closing copy of the first vertex and repeated consecutive
// vertices are dropped) into out (at most m): counter-clockwise for a shell, clockwise for a hole, so that P's interior lies on
// every edge's left.  The orientation is that of the lexicographically smallest vertex, a convex corner of a simple ring.
// scratch: 2 m doubles.  Returns the number of edges, 0 for a ring of fewer than three distinct vertices.
DP_HD int64_t ring_edges(const double* xy, int64_t m, bool hole, double* scratch, Edge* out) {
    int64_t k = 0;
    for (int64_t i = 0; i < m; ++i) {
        const double x = xy[2 * i], y = xy[2 * i + 1];
        if (k > 0 && scratch[2 * k - 2] == x && scratch[2 * k - 1] == y) continue;
        scratch[2 * k] = x, scratch[2 * k + 1] = y, ++k;
    }
    while (k > 1 && scratch[2 * k - 2] == scratch[0] && scratch[2 * k - 1] == scratch[1]) --k;
    if (k < 3) return 0;
    int64_t lo = 0;
    for (int64_t i = 1; i < k; ++i)
        if (scratch[2 * i] < scratch[2 * lo] || (scratch[2 * i] == scratch[2 * lo] && scratch[2 * i + 1] < scratch[2 * lo + 1])) lo = i;
    const int64_t pv = (lo + k - 1) % k, nx = (lo + 1) % k;
    const bool ccw = orient(scratch[2 * pv], scratch[2 * pv + 1], scratch[2 * lo], scratch[2 * lo + 1], scratch[2 * nx], scratch[2 * nx + 1]) > 0;
    const bool flip = ccw == hole;
    for (int64_t i = 0; i < k; ++i) {
        const int64_t j = (i + 1) % k;
        const int64_t s = flip ? j : i, t = flip ? i : j;
        out[i] = Edge{scratch[2 * s], scratch[2 * s + 1], scratch[2 * t], scratch[2 * t + 1]};
    }
    return k;
}

// sign of a coordinate difference, by comparison
DP_HD int cmp(double a, double b) { return (a > b) - (a < b); }

// The class of the points just after v towards d (v on the boundary, d != v): INTERIOR, EXTERIOR, or BOUNDARY when a ray from v
// points along d.  Edges are added one at a time, in any order and with repeats; every edge containing v must be among them,
// the others are ignored.
struct Fan {
    double vx, vy, dx, dy;
    int sdx, sdy;
    bool found = false, along = false, best_out = false;
    int best_half = 0;  // half 0 holds the angles (0, pi) counter-clockwise from d, half 1 [pi, 2 pi)
    double bx = 0.0, by = 0.0;  // the first ray counter-clockwise from d so far
    DP_HD Fan(double vx_, double vy_, double dx_, double dy_) : vx(vx_), vy(vy_), dx(dx_), dy(dy_), sdx(cmp(dx_, vx_)), sdy(cmp(dy_, vy_)) {}
    DP_HD void add(const Edge& e) {
        const bool at_a = e.ax == vx && e.ay == vy, at_b = e.bx == vx && e.by == vy;
        if (!at_a && !at_b && !on_edge(e, vx, vy)) return;
        // rays: towards b leaving v along the edge (out), towards a arriving at v (in)
        for (int r = 0; r < 2; ++r) {
            const bool out = r == 0;
            if (out ? at_b : at_a) continue;
            const double rx = out ? e.bx : e.ax, ry = out ? e.by : e.ay;
            const int c = orient(vx, vy, dx, dy, rx, ry);
            int half;
            if (c == 0) {
                if (sdx != 0 ? cmp(rx, vx) == sdx : cmp(ry, vy) == sdy) {
                    along = true;
                    continue;
                }
                half = 1;  // opposite to d: angle pi
            } else {
                half = c > 0 ? 0 : 1;
            }
            if (!found || half < best_half || (half == best_half && orient(vx, vy, rx, ry, bx, by) > 0))
                found = true, best_out = out, best_half = half, bx = rx, by = ry;
        }
    }
    // EXTERIOR without rays: v is not on the boundary, never the case for the callers
    DP_HD int cls() const { return along ? BOUNDARY : (!found || best_out) ? EXTERIOR : INTERIOR; }
};

// Accumulates the verdicts of one piece class: bad once a piece (or point) is exterior, in once a piece is interior.
struct Verdict {
    bool bad = false, in = false;
    DP_HD void add(int cls) {
        bad |= cls == EXTERIOR;
        in |= cls == INTERIOR;
    }
};

// The pieces at the end point p (class cp, not EXTERIOR) of [p, q]: its own class off the boundary, else the direction test.
template <typename NearAt>
DP_HD void endpoint_pieces(double px, double py, int cp, double qx, double qy, NearAt near, Verdict& v) {
    if (cp == INTERIOR) {
        v.in = true;
        return;
    }
    Fan f(px, py, qx, qy);
    near(px, py, [&](int64_t m, auto edge) {
        for (int64_t k = 0; k < m; ++k) f.add(edge(k));
    });
    v.add(f.cls());
}

// One boundary edge against [p, q]: a proper crossing makes the segment not within; its start vertex on the open segment is
// an event whose two pieces are classified.  (The end vertex is the start of the ring's next edge.)
template <typename NearAt>
DP_HD void edge_pieces(const Edge& e, double px, double py, double qx, double qy, NearAt near, Verdict& v) {
    const int o1 = orient(px, py, qx, qy, e.ax, e.ay), o2 = orient(px, py, qx, qy, e.bx, e.by);
    if (o1 * o2 > 0) return;  // both on one side of the segment's line
    if (o1 * o2 < 0) {
        const int o3 = orient(e.ax, e.ay, e.bx, e.by, px, py), o4 = orient(e.ax, e.ay, e.bx, e.by, qx, qy);
        if (o3 * o4 < 0) {
            v.bad = true;
            return;
        }
    }
    if (o1 == 0 && in_box(px, py, qx, qy, e.ax, e.ay) && !(e.ax == px && e.ay == py) && !(e.ax == qx && e.ay == qy)) {
        Fan fq(e.ax, e.ay, qx, qy), fp(e.ax, e.ay, px, py);
        near(e.ax, e.ay, [&](int64_t m, auto edge) {
            for (int64_t k = 0; k < m; ++k) {
                const Edge g = edge(k);
                fq.add(g), fp.add(g);
            }
        });
        v.add(fq.cls());
        v.add(fp.cls());
    }
}

// Is [p, q] within P?  cp / cq: the classes of p and q (classify_point).  scan(f) calls f(m, edge) for groups of edges that
// together hold every edge meeting the closed segment (repeats allowed); near(x, y, f) does the same for the edges containing
// the point (x, y).  A point's fan is gathered over all of near's groups before it is classified.
template <typename Scan, typename NearAt>
DP_HD bool segment_within(double px, double py, int cp, double qx, double qy, int cq, Scan scan, NearAt near) {
    if (px == qx && py == qy) return cp == INTERIOR;
    if (cp == EXTERIOR || cq == EXTERIOR) return false;
    Verdict v;
    endpoint_pieces(px, py, cp, qx, qy, near, v);
    endpoint_pieces(qx, qy, cq, px, py, near, v);
    if (v.bad) return false;
    scan([&](int64_t m, auto edge) {
        for (int64_t k = 0; k < m && !v.bad; ++k) edge_pieces(edge(k), px, py, qx, qy, near, v);
    });
    return !v.bad && v.in;
}

}  // namespace mpred
