"""Rational oracle of ``mask_graph``'s predicate: shapely's ``LineString.within(P)`` (DE-9IM ``T*F**F***``) for a polygon with
holes or a MultiPolygon, in ``fractions.Fraction``.

The segment is cut at every parameter where it meets a boundary edge (crossing points and the ends of collinear overlaps),
then every cut point and the midpoint of every piece between them is located by exact point-in-polygon (on an edge, or by
the parity of the crossings of a horizontal ray, with the crossing abscissae computed exactly).  The segment is within P iff no
located point is exterior and some piece midpoint is interior.  A zero-length segment is its point: within iff interior.
Nothing here is shared with ``csrc/mask_pred.h``."""

from __future__ import annotations

from fractions import Fraction as F

EXTERIOR, BOUNDARY, INTERIOR = 0, 1, 2


def polygon_rings(geom) -> list[list[tuple[float, float]]]:
    """Every ring (shells and holes) of a ``__geo_interface__`` Polygon / MultiPolygon, as lists of (x, y)."""
    gi = geom.__geo_interface__ if hasattr(geom, "__geo_interface__") else geom
    polys = [gi["coordinates"]] if gi["type"] == "Polygon" else list(gi["coordinates"])
    return [[(float(v[0]), float(v[1])) for v in ring] for poly in polys for ring in poly]


def boundary_edges(rings) -> list[tuple[tuple[F, F], tuple[F, F]]]:
    out = []
    for ring in rings:
        pts = [(F(x), F(y)) for x, y in ring]
        for k in range(len(pts)):
            a, b = pts[k], pts[(k + 1) % len(pts)]
            if a != b:
                out.append((a, b))
    return out


def _cross(ox, oy, ax, ay, bx, by):
    return (ax - ox) * (by - oy) - (ay - oy) * (bx - ox)


def locate(p, edges) -> int:
    px, py = p
    for (ax, ay), (bx, by) in edges:
        if _cross(ax, ay, bx, by, px, py) == 0 and min(ax, bx) <= px <= max(ax, bx) and min(ay, by) <= py <= max(ay, by):
            return BOUNDARY
    odd = False
    for (ax, ay), (bx, by) in edges:
        if (ay <= py < by) or (by <= py < ay):
            x = ax + (py - ay) * (bx - ax) / (by - ay)
            if x > px:
                odd = not odd
    return INTERIOR if odd else EXTERIOR


def _cut_parameters(p, q, edges) -> list[F]:
    (px, py), (qx, qy) = p, q
    dx, dy = qx - px, qy - py
    ts = {F(0), F(1)}
    for (ax, ay), (bx, by) in edges:
        ex, ey = bx - ax, by - ay
        den = dx * ey - dy * ex
        if den != 0:
            t = ((ax - px) * ey - (ay - py) * ex) / den
            u = ((ax - px) * dy - (ay - py) * dx) / den
            if 0 <= t <= 1 and 0 <= u <= 1:
                ts.add(t)
        elif (ax - px) * dy - (ay - py) * dx == 0:  # collinear: the edge's ends projected on the segment
            n2 = dx * dx + dy * dy
            for cx, cy in ((ax, ay), (bx, by)):
                t = ((cx - px) * dx + (cy - py) * dy) / n2
                if 0 <= t <= 1:
                    ts.add(t)
    return sorted(ts)


def segment_within(p, q, edges) -> bool:
    p = (F(p[0]), F(p[1]))
    q = (F(q[0]), F(q[1]))
    if p == q:
        return locate(p, edges) == INTERIOR
    ts = _cut_parameters(p, q, edges)

    def at(t):
        return (p[0] + t * (q[0] - p[0]), p[1] + t * (q[1] - p[1]))

    if any(locate(at(t), edges) == EXTERIOR for t in ts):
        return False
    mids = [locate(at((t0 + t1) / 2), edges) for t0, t1 in zip(ts, ts[1:])]
    return EXTERIOR not in mids and INTERIOR in mids


def mask_flags(coords, rows, cols, geom) -> list[bool]:
    """Within-flags of the segments coords[rows[k]] -> coords[cols[k]]."""
    edges = boundary_edges(polygon_rings(geom))
    return [segment_within(coords[i], coords[j], edges) for i, j in zip(rows, cols)]
