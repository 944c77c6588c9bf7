// graph.cuh — the point grid and neighbour searches of graph.cu, shared with the device-coordinate builders of graph_device.cu.
#pragma once
#include "common.cuh"

struct GridGeom {
    double x0, y0, inv_cell, cell;
    int gx, gy;
};

struct PointGrid {
    explicit PointGrid(cudaStream_t s) : d_xy(s), d_pts(s), d_idx_sorted(s), d_cell_start(s) {}
    GridGeom gm;
    DevBuf<double> d_xy;  // interleaved x, y (float64) of the n points
    DevBuf<double2> d_pts;
    DevBuf<int32_t> d_idx_sorted, d_cell_start;
};

__device__ __forceinline__ int grid_cell_coord(double v, double v0, double inv, int g) {
    int c = (int)floor((v - v0) * inv);
    return c < 0 ? 0 : (c >= g ? g - 1 : c);
}

// Lower bound on the squared distance from q to every point of the grid outside the visited square of cells
// [cx - r, cx + r] x [cy - r, cy + r]: the minimum over the square's sides that still have cells beyond them of (separation
// along that axis)^2 + (distance from q to the grid box along the other axis)^2.  It holds for queries outside the box too
// (their cell is clamped to the box), where r cells alone would be a loose bound.  Both terms are shrunk by a slack
// proportional to the box's coordinates: the cell assignment of a point is a rounded computation.  Returns -1 when no cell
// is left (the walk is complete).
__device__ __forceinline__ double grid_unvisited_bound(const GridGeom gm, double2 q, int cx, int cy, int r) {
    const double bx1 = gm.x0 + gm.gx * gm.cell, by1 = gm.y0 + gm.gy * gm.cell;
    const double slack = 1e-12 * (fabs(gm.x0) + fabs(gm.y0) + fabs(bx1) + fabs(by1));
    const double ox = fmax(fmax(gm.x0 - q.x, q.x - bx1) - slack, 0.0), oy = fmax(fmax(gm.y0 - q.y, q.y - by1) - slack, 0.0);
    const double oy2 = __dmul_rn(oy, oy), ox2 = __dmul_rn(ox, ox);
    double lb = INFINITY;
    bool left = false;
    if (cx + r + 1 < gm.gx) {
        const double s = fmax(gm.x0 + (cx + r + 1) * gm.cell - q.x - slack, 0.0);
        lb = fmin(lb, s * s + oy2), left = true;
    }
    if (cx - r - 1 >= 0) {
        const double s = fmax(q.x - (gm.x0 + (cx - r) * gm.cell) - slack, 0.0);
        lb = fmin(lb, s * s + oy2), left = true;
    }
    if (cy + r + 1 < gm.gy) {
        const double s = fmax(gm.y0 + (cy + r + 1) * gm.cell - q.y - slack, 0.0);
        lb = fmin(lb, s * s + ox2), left = true;
    }
    if (cy - r - 1 >= 0) {
        const double s = fmax(q.y - (gm.y0 + (cy - r) * gm.cell) - slack, 0.0);
        lb = fmin(lb, s * s + ox2), left = true;
    }
    return left ? lb : -1.0;
}

// Grid geometry from the bounding box of n points: square cells of edge `cell_hint` (or sized for `pts_per_cell` points per
// cell when the hint is 0), coarsened until the grid has at most ~4n + 16 cells.
GridGeom grid_geometry(double x0, double y0, double x1, double y1, int64_t n, double cell_hint, double pts_per_cell);
// Buckets the n points of g->d_xy (already on the device, in stream order) into the cells of g->gm.
int grid_bucket(sqb_ctx* c, int64_t n, PointGrid* g);
// Points per cell the kNN search sizes its grid for.
static inline double knn_pts_per_cell(int k) { return k <= 8 ? 2.5 : (double)k / 3.0; }
// Exact kNN of every point (self excluded): n x k ascending neighbour indices and float64 distances (device arrays).
int knn_launch(sqb_ctx* c, const PointGrid& g, int64_t n, int k, int32_t* idx, double* dist);
// np.median of m device distances: sorts them into `sorted` and copies the two middle order statistics to med[0..1] (the copy
// completes in stream order; the median is (med[0] + med[1]) / 2).
int median_enqueue(sqb_ctx* c, const double* dist, int64_t m, DevBuf<double>& sorted, DevBuf<uint8_t>& tmp, double* med);
// Cells the radius search visits on every side of a point's cell.
static inline int radius_reach(double radius, const GridGeom& gm) { return (int)ceil(radius / gm.cell * (1.0 + 1e-12)); }
// Radius search: with idx == nullptr, counts[i] = neighbours of point i; else the rows at indptr[i], ascending columns.
int radius_launch(sqb_ctx* c, const PointGrid& g, int64_t n, double radius, int64_t* counts, const int64_t* indptr, int32_t* idx,
                  double* dist);
