// graph.cu — spatial neighbour graphs from 2-D coordinates on the GPU (sm_90a): exact k-nearest neighbours and fixed-radius
// neighbours over a uniform cell grid.
//
// Replaces the scikit-learn KD-tree queries of the reference's graph builders (src/squidpy/gr/neighbors.py):
//   KNNBuilder.build_graph        :192-209   NearestNeighbors(n_neighbors=k).fit(coords).kneighbors()   (the query point itself
//   GridBuilder._base_adjacency   :395-419   the same + the `dist < 1.3 * median(dists)` cut                is excluded)
//   RadiusBuilder.build_graph     :253-270   NearestNeighbors(radius=r).fit(coords).radius_neighbors()
// Arithmetic is sklearn's for euclidean distances in low dimension (kd_tree): d2 = dx*dx + dy*dy accumulated in float64 without
// contraction, candidates compared by d2, the reported distance is sqrt(d2) — so distances are bit-identical.  Ties at the
// k-th distance (lattices!) are broken by the smaller observation index here; sklearn's tie order is unspecified, which
// only matters for KNNBuilder on exactly regular coordinates (GridBuilder's distance cut removes the tied far candidates).
// Layout: points are bucketed into square cells (counting sort by cell id: cub radix sort of (cell, index) pairs), coordinates
// are gathered into cell order so that a query streams its 3x3 / 5x5 ... rings of cells from contiguous memory; one thread per
// query, the k best (d2, index) pairs in registers.  The search of a point stops after ring r as soon as its k-th distance
// is below r cells (nothing unseen can be closer).
#include <algorithm>
#include <cmath>
#include <limits>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <map>
#include <math.h>
#include <vector>

#include "graph.cuh"

__device__ __forceinline__ int grid_cell_coord(double v, double v0, double inv, int g) {
    int c = (int)floor((v - v0) * inv);
    return c < 0 ? 0 : (c >= g ? g - 1 : c);
}

__global__ void graph_cell_id_kernel(const double* __restrict__ xy, int64_t n, GridGeom gm, uint32_t* __restrict__ cell,
                                     int32_t* __restrict__ idx) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int cx = grid_cell_coord(xy[2 * i], gm.x0, gm.inv_cell, gm.gx), cy = grid_cell_coord(xy[2 * i + 1], gm.y0, gm.inv_cell, gm.gy);
    cell[i] = (uint32_t)cy * (uint32_t)gm.gx + (uint32_t)cx;
    idx[i] = (int32_t)i;
}

// sorted (cell, index) pairs -> coordinates in cell order + first position of every cell (cell_start[c] .. cell_start[c+1])
__global__ void graph_gather_kernel(const double* __restrict__ xy, const uint32_t* __restrict__ cell_sorted,
                                    const int32_t* __restrict__ idx_sorted, int64_t n, int64_t n_cells, double2* __restrict__ pts,
                                    int32_t* __restrict__ cell_start) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n) return;
    const int32_t i = idx_sorted[s];
    pts[s] = make_double2(xy[2 * (int64_t)i], xy[2 * (int64_t)i + 1]);
    const uint32_t c = cell_sorted[s];
    const uint32_t prev = s > 0 ? cell_sorted[s - 1] : 0xffffffffu;
    if (s == 0 || c != prev) {
        // cells between the previous occupied cell and this one are empty: they start here too
        for (int64_t e = (s == 0 ? 0 : (int64_t)prev + 1); e <= (int64_t)c; ++e) cell_start[e] = (int32_t)s;
    }
    if (s == n - 1)
        for (int64_t e = (int64_t)c + 1; e <= n_cells; ++e) cell_start[e] = (int32_t)n;
}

// ---- exact kNN -------------------------------------------------------------------------------------------------------
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

// The ring walk of the exact kNN searches: the k smallest d2 from q to the points of one grid (points pts[cell_start[c] ..
// cell_start[c + 1]) of cell c) in bd[0 .. k), in DESCENDING order: bd[0] is the k-th smallest, so the list is only ever read at
// constant indices and stays in registers.  BY_INDEX (graph search): the point with index qi is skipped and ties at the k-th
// distance go to the smaller index, kept in bi.  Without it (distance histograms) no point is skipped, only the multiset of
// the k distances is kept and bi is not written.
template <int KMAX, bool BY_INDEX>
__device__ __forceinline__ void grid_knn_walk(const double2* __restrict__ pts, const int32_t* __restrict__ idx_sorted,
                                              const int32_t* __restrict__ cell_start, const GridGeom gm, double2 q, int32_t qi, int k,
                                              double (&bd)[KMAX], int32_t (&bi)[KMAX]) {
    const int cx = grid_cell_coord(q.x, gm.x0, gm.inv_cell, gm.gx), cy = grid_cell_coord(q.y, gm.y0, gm.inv_cell, gm.gy);
#pragma unroll
    for (int t = 0; t < KMAX; ++t) {
        bd[t] = INFINITY;
        if (BY_INDEX) bi[t] = 0x7fffffff;
    }
    const int rmax = gm.gx > gm.gy ? gm.gx : gm.gy;
    for (int r = 0; r <= rmax; ++r) {
        // ring r: the cells at Chebyshev distance exactly r from (cx, cy)
        for (int yy = cy - r; yy <= cy + r; ++yy) {
            if (yy < 0 || yy >= gm.gy) continue;
            const bool edge_row = (yy == cy - r) || (yy == cy + r);
            const int step = edge_row ? 1 : 2 * r;  // interior rows of the ring: only the two end columns
            for (int xx = cx - r; xx <= cx + r; xx += (step > 0 ? step : 1)) {
                if (xx < 0 || xx >= gm.gx) continue;
                const int64_t c = (int64_t)yy * gm.gx + xx;
                const int32_t b = cell_start[c], e = cell_start[c + 1];
                for (int32_t t = b; t < e; ++t) {
                    int32_t j = 0;
                    if (BY_INDEX) {
                        j = idx_sorted[t];
                        if (j == qi) continue;  // the query point itself is not its own neighbour (kneighbors() without X)
                    }
                    const double2 p = pts[t];
                    const double dx = q.x - p.x, dy = q.y - p.y;
                    const double d2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
                    if (d2 < bd[0] || (BY_INDEX && d2 == bd[0] && j < bi[0])) {
                        // drop the k-th entry, shift the larger ones down and put (d2, j) in place
                        bool placed = false;
#pragma unroll
                        for (int u = 0; u < KMAX; ++u) {
                            if (u < k && !placed) {
                                const double nd = (u + 1 < KMAX && u + 1 < k) ? bd[u + 1 < KMAX ? u + 1 : u] : -INFINITY;
                                const int32_t ni = (BY_INDEX && u + 1 < KMAX && u + 1 < k) ? bi[u + 1 < KMAX ? u + 1 : u] : 0;
                                if (nd > d2 || (BY_INDEX && nd == d2 && ni > j)) {
                                    bd[u] = nd;
                                    if (BY_INDEX) bi[u] = ni;
                                } else {
                                    bd[u] = d2;
                                    if (BY_INDEX) bi[u] = j;
                                    placed = true;
                                }
                            }
                        }
                    }
                }
                if (r == 0) break;
            }
        }
        // every unvisited point is at least sqrt(lb) away: stop once the k-th distance is below that
        const double lb = grid_unvisited_bound(gm, q, cx, cy, r);
        if (lb < 0.0 || bd[0] < lb) break;
    }
}

template <int KMAX>
__global__ void __launch_bounds__(128) graph_knn_kernel(const double2* __restrict__ pts, const int32_t* __restrict__ idx_sorted,
                                                        const int32_t* __restrict__ cell_start, int64_t n, GridGeom gm, int k,
                                                        int32_t* __restrict__ out_idx, double* __restrict__ out_dist) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n) return;
    const double2 q = pts[s];
    const int32_t qi = idx_sorted[s];
    double bd[KMAX];
    int32_t bi[KMAX];
    grid_knn_walk<KMAX, true>(pts, idx_sorted, cell_start, gm, q, qi, k, bd, bi);
    // rows of a CSR matrix hold ascending column indices: order the k neighbours by index (k is small)
    for (int a = 1; a < k; ++a) {
        const double vd = bd[a];
        const int32_t vi = bi[a];
        int b = a - 1;
        while (b >= 0 && bi[b] > vi) {
            bd[b + 1] = bd[b];
            bi[b + 1] = bi[b];
            --b;
        }
        bd[b + 1] = vd;
        bi[b + 1] = vi;
    }
    for (int t = 0; t < k; ++t) {
        out_idx[(int64_t)qi * k + t] = bi[t];
        out_dist[(int64_t)qi * k + t] = __dsqrt_rn(bd[t]);
    }
}

// ---- fixed radius -------------------------------------------------------------------------------------------------------
// pass 1 (out_idx == nullptr): neighbours per point;  pass 2: ascending column indices + distances at indptr[i]
__global__ void __launch_bounds__(128) graph_radius_kernel(const double2* __restrict__ pts, const int32_t* __restrict__ idx_sorted,
                                                           const int32_t* __restrict__ cell_start, int64_t n, GridGeom gm, double radius,
                                                           int reach_cells, int64_t* __restrict__ counts,
                                                           const int64_t* __restrict__ indptr, int32_t* __restrict__ out_idx,
                                                           double* __restrict__ out_dist) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n) return;
    const double2 q = pts[s];
    const int32_t qi = idx_sorted[s];
    const int cx = grid_cell_coord(q.x, gm.x0, gm.inv_cell, gm.gx), cy = grid_cell_coord(q.y, gm.y0, gm.inv_cell, gm.gy);
    int64_t cnt = 0;
    const int64_t base = out_idx ? indptr[qi] : 0;
    const double r2 = __dmul_rn(radius, radius);
    for (int yy = cy - reach_cells; yy <= cy + reach_cells; ++yy) {
        if (yy < 0 || yy >= gm.gy) continue;
        for (int xx = cx - reach_cells; xx <= cx + reach_cells; ++xx) {
            if (xx < 0 || xx >= gm.gx) continue;
            const int64_t c = (int64_t)yy * gm.gx + xx;
            for (int32_t t = cell_start[c]; t < cell_start[c + 1]; ++t) {
                const int32_t j = idx_sorted[t];
                if (j == qi) continue;
                const double2 p = pts[t];
                const double dx = q.x - p.x, dy = q.y - p.y;
                const double d2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
                if (d2 <= r2) {  // sklearn's kd_tree compares the reduced distance with radius * radius
                    if (out_idx) {
                        out_idx[base + cnt] = j;
                        out_dist[base + cnt] = __dsqrt_rn(d2);
                    }
                    ++cnt;
                }
            }
        }
    }
    if (!out_idx) {
        counts[qi] = cnt;
        return;
    }
    // ascending column order inside the row (insertion sort: rows are short)
    for (int64_t a = 1; a < cnt; ++a) {
        const int32_t vi = out_idx[base + a];
        const double vd = out_dist[base + a];
        int64_t b = a - 1;
        while (b >= 0 && out_idx[base + b] > vi) {
            out_idx[base + b + 1] = out_idx[base + b];
            out_dist[base + b + 1] = out_dist[base + b];
            --b;
        }
        out_idx[base + b + 1] = vi;
        out_dist[base + b + 1] = vd;
    }
}

// ================================================================================================
GridGeom grid_geometry(double x0, double y0, double x1, double y1, int64_t n, double cell_hint, double pts_per_cell) {
    const double w = x1 - x0, h = y1 - y0;
    double cell = cell_hint;
    if (!(cell > 0.0)) {
        const double area = (w > 0 ? w : 1.0) * (h > 0 ? h : 1.0);
        cell = sqrt(area * pts_per_cell / (double)n);
        if (w <= 0 || h <= 0) cell = ((w > h ? w : h) > 0 ? (w > h ? w : h) : 1.0) * pts_per_cell / (double)n;
    }
    if (!(cell > 0.0)) cell = 1.0;
    const double max_cells = 4.0 * (double)n + 16.0;
    for (;;) {
        const double gx = floor(w / cell) + 1.0, gy = floor(h / cell) + 1.0;
        if (gx * gy <= max_cells && gx < 2.0e9 && gy < 2.0e9) break;
        cell *= 1.5;
    }
    GridGeom gm;
    gm.x0 = x0, gm.y0 = y0, gm.cell = cell, gm.inv_cell = 1.0 / cell;
    gm.gx = (int)(floor(w / cell) + 1.0), gm.gy = (int)(floor(h / cell) + 1.0);
    return gm;
}

int grid_bucket(sqb_ctx* c, int64_t n, PointGrid* g) {
    const GridGeom gm = g->gm;
    const int64_t n_cells = (int64_t)gm.gx * gm.gy;
    DevBuf<uint32_t> cell_a(c->stream), cell_b(c->stream);
    DevBuf<int32_t> idx_a(c->stream);
    DevBuf<uint8_t> tmp(c->stream);
    SQB_TRY(g->d_pts.alloc(n));
    SQB_TRY(g->d_idx_sorted.alloc(n));
    SQB_TRY(g->d_cell_start.alloc(n_cells + 1));
    SQB_TRY(cell_a.alloc(n));
    SQB_TRY(cell_b.alloc(n));
    SQB_TRY(idx_a.alloc(n));
    c->launches += 1;
    graph_cell_id_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, c->stream>>>(g->d_xy.p, n, gm, cell_a.p, idx_a.p);
    SQB_POST_LAUNCH();
    int bits = 1;
    while (bits < 32 && ((uint64_t)(n_cells - 1) >> bits) != 0) ++bits;
    size_t tmp_bytes = 0;
    SQB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, cell_a.p, cell_b.p, idx_a.p, g->d_idx_sorted.p, (int)n, 0, bits, c->stream));
    SQB_TRY(tmp.alloc(tmp_bytes > 0 ? tmp_bytes : 1));
    SQB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, cell_a.p, cell_b.p, idx_a.p, g->d_idx_sorted.p, (int)n, 0, bits, c->stream));
    c->launches += 2;
    graph_gather_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, c->stream>>>(g->d_xy.p, cell_b.p, g->d_idx_sorted.p, n, n_cells, g->d_pts.p, g->d_cell_start.p);
    SQB_POST_LAUNCH();
    return SQB_OK;
}

// host coordinates: bounding box and finiteness on the host, then upload and bucket
static int build_grid(sqb_ctx* c, const double* xy, int64_t n, double cell_hint, double pts_per_cell, PointGrid* g) {
    double x0 = INFINITY, y0 = INFINITY, x1 = -INFINITY, y1 = -INFINITY;
    for (int64_t i = 0; i < n; ++i) {
        const double x = xy[2 * i], y = xy[2 * i + 1];
        SQB_CHECK(isfinite(x) && isfinite(y), SQB_ERR_INVALID, "coordinates of observation %lld are not finite", (long long)i);
        x0 = x < x0 ? x : x0, x1 = x > x1 ? x : x1, y0 = y < y0 ? y : y0, y1 = y > y1 ? y : y1;
    }
    g->gm = grid_geometry(x0, y0, x1, y1, n, cell_hint, pts_per_cell);
    SQB_TRY(g->d_xy.alloc(2 * n));
    SQB_CUDA(cudaMemcpyAsync(g->d_xy.p, xy, 2 * n * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    return grid_bucket(c, n, g);
}

int knn_launch(sqb_ctx* c, const PointGrid& g, int64_t n, int k, int32_t* idx, double* dist) {
    SqbLaunchScope scope(c, SQB_K_MISC);
    const unsigned grid = (unsigned)ceil_div64(n, 128);
    if (k <= 8)
        graph_knn_kernel<8><<<grid, 128, 0, c->stream>>>(g.d_pts.p, g.d_idx_sorted.p, g.d_cell_start.p, n, g.gm, k, idx, dist);
    else if (k <= 16)
        graph_knn_kernel<16><<<grid, 128, 0, c->stream>>>(g.d_pts.p, g.d_idx_sorted.p, g.d_cell_start.p, n, g.gm, k, idx, dist);
    else if (k <= 32)
        graph_knn_kernel<32><<<grid, 128, 0, c->stream>>>(g.d_pts.p, g.d_idx_sorted.p, g.d_cell_start.p, n, g.gm, k, idx, dist);
    else
        graph_knn_kernel<64><<<grid, 128, 0, c->stream>>>(g.d_pts.p, g.d_idx_sorted.p, g.d_cell_start.p, n, g.gm, k, idx, dist);
    SQB_POST_LAUNCH();
    return SQB_OK;
}

int median_enqueue(sqb_ctx* c, const double* dist, int64_t m, DevBuf<double>& sorted, DevBuf<uint8_t>& tmp, double* med) {
    // np.median of all m distances: radix sort, the middle element (odd count) or the mean of the two middle ones
    size_t tmp_bytes = 0;
    SQB_TRY(sorted.alloc((size_t)m));
    SQB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, dist, sorted.p, (int)m, 0, 64, c->stream));
    SQB_TRY(tmp.alloc(tmp_bytes > 0 ? tmp_bytes : 1));
    SQB_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, tmp_bytes, dist, sorted.p, (int)m, 0, 64, c->stream));
    c->launches += 1;
    SQB_CUDA(cudaMemcpyAsync(&med[0], sorted.p + (m - 1) / 2, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaMemcpyAsync(&med[1], sorted.p + m / 2, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    return SQB_OK;
}

int radius_launch(sqb_ctx* c, const PointGrid& g, int64_t n, double radius, int64_t* counts, const int64_t* indptr, int32_t* idx,
                  double* dist) {
    SqbLaunchScope scope(c, SQB_K_MISC);
    graph_radius_kernel<<<(unsigned)ceil_div64(n, 128), 128, 0, c->stream>>>(g.d_pts.p, g.d_idx_sorted.p, g.d_cell_start.p, n, g.gm, radius,
                                                                             radius_reach(radius, g.gm), counts, indptr, idx, dist);
    SQB_POST_LAUNCH();
    return SQB_OK;
}

// ---- nearest-neighbour distance histograms (Ripley's F and G) -----------------------------------------------------------
// Every reference set is bucketed into its own grid; the grids are concatenated (set s owns the global cells cell_off ..
// cell_off + gx * gy), so one radix sort of (global cell, pool index) buckets all of them.
struct NnSet {
    GridGeom gm;
    int64_t cell_off;   // first global cell of the set's grid
    int64_t ref_begin;  // pool index of the set's first point
    int64_t entry_off;  // first entry of the set in the concatenated bucketing input
};

// One CTA's share of a task: queries q0 .. q1 of the pool against set `set`, k distances each, into histogram row `row`.
struct NnBlock {
    int32_t q0, q1, set, row, k, pad;
};

#define NN_THREADS 128
#define NN_QPB 1024            // queries per block descriptor (NN_QPB / NN_THREADS per thread)
#define NN_SHARED_BINS 8192    // histograms of up to this many bins are kept in shared memory per block

__global__ void nnd_cell_id_kernel(const double* __restrict__ xy, const NnSet* __restrict__ sets, int n_sets, int64_t n_entries,
                                   uint32_t* __restrict__ cell, int32_t* __restrict__ idx) {
    const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (e >= n_entries) return;
    int lo = 0, hi = n_sets - 1;  // the last set whose entry_off <= e
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (sets[mid].entry_off <= e) lo = mid; else hi = mid - 1;
    }
    const NnSet st = sets[lo];
    const int64_t i = st.ref_begin + (e - st.entry_off);
    const int cx = grid_cell_coord(xy[2 * i], st.gm.x0, st.gm.inv_cell, st.gm.gx);
    const int cy = grid_cell_coord(xy[2 * i + 1], st.gm.y0, st.gm.inv_cell, st.gm.gy);
    cell[e] = (uint32_t)(st.cell_off + (int64_t)cy * st.gm.gx + cx);
    idx[e] = (int32_t)i;
}

// np.histogram(sqrt(d2), bins=e) for ascending edges e[0 .. S) (numpy's cumulative searchsorted: side 'left' for every edge but
// the last, 'right' for the last): d = sqrt(d2) falls into bin i = #{j < S - 1 : e[j] <= d} - 1 when e[0] <= d <= e[S - 1], and
// is dropped otherwise.  The comparisons are made on d2 against thresholds of the host (nnd_thresholds): thr[j] = min{t : sqrt(t)
// >= e[j]} for j < S - 1 and thr[S - 1] = max{t : sqrt(t) <= e[S - 1]}, so that e[j] <= sqrt(d2) <=> thr[j] <= d2 and
// sqrt(d2) <= e[S - 1] <=> d2 <= thr[S - 1] exactly (sqrt is correctly rounded and monotone).  Returns -1 for a dropped value.
__device__ __forceinline__ int nnd_bin(double d2, const double* __restrict__ thr, int S) {
    if (!(d2 >= thr[0]) || !(d2 <= thr[S - 1])) return -1;
    int lo = 0, hi = S - 1;  // first j in [0, S - 1) with thr[j] > d2, or S - 1
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (thr[mid] > d2) hi = mid; else lo = mid + 1;
    }
    return lo - 1;
}

template <int KMAX, bool SHARED>
__global__ void __launch_bounds__(NN_THREADS, 1) nnd_hist_kernel(const double2* __restrict__ pool, const double2* __restrict__ pts,
                                                              const int32_t* __restrict__ cell_start, const NnSet* __restrict__ sets,
                                                              const NnBlock* __restrict__ blocks, const double* __restrict__ thr, int S,
                                                              unsigned long long* __restrict__ out) {
    extern __shared__ uint32_t s_hist[];
    const NnBlock blk = blocks[blockIdx.x];
    const int nb = S - 1;
    if (SHARED) {
        for (int b = threadIdx.x; b < nb; b += NN_THREADS) s_hist[b] = 0u;
        __syncthreads();
    }
    const NnSet st = sets[blk.set];
    const int32_t* cs = cell_start + st.cell_off;
    for (int32_t qi = blk.q0 + threadIdx.x; qi < blk.q1; qi += NN_THREADS) {
        double bd[KMAX];
        int32_t bi[KMAX];
        grid_knn_walk<KMAX, false>(pts, nullptr, cs, st.gm, pool[qi], -1, blk.k, bd, bi);
#pragma unroll
        for (int u = 0; u < KMAX; ++u) {
            if (u < blk.k) {
                const int b = nnd_bin(bd[u], thr, S);
                if (b >= 0) {
                    if (SHARED)
                        atomicAdd(&s_hist[b], 1u);
                    else
                        atomicAdd(&out[(int64_t)blk.row * nb + b], 1ULL);
                }
            }
        }
    }
    if (SHARED) {
        __syncthreads();
        unsigned long long* row = out + (int64_t)blocks[blockIdx.x].row * nb;
        for (int b = threadIdx.x; b < nb; b += NN_THREADS) {
            const uint32_t v = s_hist[b];
            if (v) atomicAdd(&row[b], (unsigned long long)v);
        }
    }
}

template <int KMAX>
static int nnd_launch(sqb_ctx* c, int64_t nblk, const double2* pool, const double2* pts, const int32_t* cell_start, const NnSet* sets,
                      const NnBlock* blocks, const double* thr, int S, unsigned long long* out) {
    if (nblk == 0) return SQB_OK;
    SqbLaunchScope scope(c, SQB_K_MISC);
    if (S - 1 <= NN_SHARED_BINS)
        nnd_hist_kernel<KMAX, true><<<(unsigned)nblk, NN_THREADS, (size_t)(S - 1) * sizeof(uint32_t), c->stream>>>(pool, pts, cell_start, sets,
                                                                                                                 blocks, thr, S, out);
    else
        nnd_hist_kernel<KMAX, false><<<(unsigned)nblk, NN_THREADS, 0, c->stream>>>(pool, pts, cell_start, sets, blocks, thr, S, out);
    SQB_POST_LAUNCH();
    return SQB_OK;
}

// The d2 thresholds of nnd_bin for the edges e[0 .. S).
static void nnd_thresholds(const double* e, int S, double* thr) {
    const double inf = std::numeric_limits<double>::infinity();
    for (int j = 0; j < S - 1; ++j) {  // min{t >= 0 : sqrt(t) >= e[j]}
        const double r = e[j];
        if (r <= 0.0 || std::isinf(r)) {
            thr[j] = r <= 0.0 ? 0.0 : inf;
            continue;
        }
        double t = r * r;
        while (std::sqrt(t) < r) t = std::nextafter(t, inf);  // r * r overflowed: t reaches inf, sqrt(inf) >= r
        while (t > 0.0 && std::sqrt(std::nextafter(t, 0.0)) >= r) t = std::nextafter(t, 0.0);
        thr[j] = t;
    }
    const double r = e[S - 1];  // max{t : sqrt(t) <= e[S - 1]}
    if (r < 0.0 || std::isinf(r)) {
        thr[S - 1] = r < 0.0 ? -1.0 : inf;
        return;
    }
    double t = r * r;
    while (std::sqrt(t) > r) t = std::nextafter(t, 0.0);
    for (;;) {
        const double u = std::nextafter(t, inf);
        if (std::isfinite(u) && std::sqrt(u) <= r)
            t = u;
        else
            break;
    }
    thr[S - 1] = t;
}

static int nnd_kclass(int k) { return k <= 2 ? 0 : k <= 8 ? 1 : k <= 16 ? 2 : k <= 32 ? 3 : 4; }

extern "C" {

int sqb_knn_2d(sqb_ctx* ctx, const double* xy, int64_t n, int k, int32_t* out_idx, double* out_dist, double* median_out) {
    SQB_CHECK(ctx && xy && out_idx && out_dist, SQB_ERR_INVALID, "sqb_knn_2d: null argument");
    SQB_CHECK(n >= 2 && n < 2147483647LL, SQB_ERR_INVALID, "sqb_knn_2d: n=%lld out of range", (long long)n);
    SQB_CHECK(k >= 1 && k <= 64, SQB_ERR_UNSUPPORTED, "sqb_knn_2d: n_neighbors=%d outside [1, 64]", k);
    // scikit-learn's message for kneighbors() on the training set itself
    SQB_CHECK(k < n, SQB_ERR_INVALID, "Expected n_neighbors <= n_samples_fit, but n_neighbors = %d, n_samples_fit = %lld, n_samples = %lld", k + 1,
              (long long)n, (long long)n);
    SQB_CHECK((int64_t)n * k < 2147483647LL, SQB_ERR_UNSUPPORTED, "sqb_knn_2d: n * k does not fit int32");
    sqb_ctx* c = ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    PointGrid g(c->stream);
    SQB_TRY(build_grid(c, xy, n, 0.0, knn_pts_per_cell(k), &g));
    DevBuf<int32_t> d_idx(c->stream);
    DevBuf<double> d_dist(c->stream), d_sorted(c->stream);
    DevBuf<uint8_t> tmp(c->stream);
    SQB_TRY(d_idx.alloc((size_t)n * k));
    SQB_TRY(d_dist.alloc((size_t)n * k));
    SQB_TRY(knn_launch(c, g, n, k, d_idx.p, d_dist.p));
    double med[2] = {0.0, 0.0};
    if (median_out) SQB_TRY(median_enqueue(c, d_dist.p, n * k, d_sorted, tmp, med));
    SQB_CUDA(cudaMemcpyAsync(out_idx, d_idx.p, (size_t)n * k * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaMemcpyAsync(out_dist, d_dist.p, (size_t)n * k * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    if (median_out) *median_out = (med[0] + med[1]) / 2.0;  // numpy: mean of the two middle values (the same value twice if odd)
    return SQB_OK;
}

int sqb_radius_2d(sqb_ctx* ctx, const double* xy, int64_t n, double radius, int64_t* out_indptr, int32_t* out_idx, double* out_dist,
                  int64_t capacity, int64_t* nnz_out) {
    SQB_CHECK(ctx && xy && out_indptr && nnz_out, SQB_ERR_INVALID, "sqb_radius_2d: null argument");
    SQB_CHECK(n >= 1 && n < 2147483647LL, SQB_ERR_INVALID, "sqb_radius_2d: n=%lld out of range", (long long)n);
    SQB_CHECK(radius >= 0.0 && isfinite(radius), SQB_ERR_INVALID, "sqb_radius_2d: radius must be finite and non-negative");
    sqb_ctx* c = ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    PointGrid g(c->stream);
    SQB_TRY(build_grid(c, xy, n, radius > 0.0 ? radius : 0.0, 2.5, &g));
    DevBuf<int64_t> d_cnt(c->stream), d_ptr(c->stream);
    DevBuf<uint8_t> tmp(c->stream);
    SQB_TRY(d_cnt.alloc(n + 1));
    SQB_TRY(d_ptr.alloc(n + 1));
    SQB_CUDA(cudaMemsetAsync(d_cnt.p, 0, (n + 1) * sizeof(int64_t), c->stream));
    SQB_TRY(radius_launch(c, g, n, radius, d_cnt.p, nullptr, nullptr, nullptr));
    size_t tmp_bytes = 0;
    SQB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_cnt.p, d_ptr.p, (int)(n + 1), c->stream));
    SQB_TRY(tmp.alloc(tmp_bytes > 0 ? tmp_bytes : 1));
    SQB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tmp_bytes, d_cnt.p, d_ptr.p, (int)(n + 1), c->stream));
    SQB_CUDA(cudaMemcpyAsync(out_indptr, d_ptr.p, (n + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    const int64_t nnz = out_indptr[n];
    *nnz_out = nnz;
    if (!out_idx || !out_dist || capacity < nnz) return SQB_OK;  // first call of the two-call protocol: the caller allocates nnz entries
    if (nnz > 0) {
        DevBuf<int32_t> d_idx(c->stream);
        DevBuf<double> d_dist(c->stream);
        SQB_TRY(d_idx.alloc((size_t)nnz));
        SQB_TRY(d_dist.alloc((size_t)nnz));
        SQB_TRY(radius_launch(c, g, n, radius, nullptr, d_ptr.p, d_idx.p, d_dist.p));
        SQB_CUDA(cudaMemcpyAsync(out_idx, d_idx.p, (size_t)nnz * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaMemcpyAsync(out_dist, d_dist.p, (size_t)nnz * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaStreamSynchronize(c->stream));
    }
    return SQB_OK;
}

int sqb_nn_dist_hist_f64(sqb_ctx* ctx, const double* pts, int64_t n_pts, const int64_t* tasks, int64_t n_tasks, const double* support, int S,
                         int n_rows, int shard_index, int shard_count, int64_t* out) {
    SQB_CHECK(ctx && pts && support && out && (tasks || n_tasks == 0), SQB_ERR_INVALID, "sqb_nn_dist_hist_f64: null argument");
    SQB_CHECK(n_pts >= 0 && n_pts < 2147483647LL, SQB_ERR_INVALID, "sqb_nn_dist_hist_f64: n_pts=%lld out of range", (long long)n_pts);
    SQB_CHECK(n_tasks >= 0, SQB_ERR_INVALID, "sqb_nn_dist_hist_f64: n_tasks=%lld out of range", (long long)n_tasks);
    SQB_CHECK(S >= 2 && S <= (1 << 24), SQB_ERR_INVALID, "sqb_nn_dist_hist_f64: S=%d out of range [2,%d]", S, 1 << 24);
    SQB_CHECK(n_rows >= 1, SQB_ERR_INVALID, "sqb_nn_dist_hist_f64: n_rows=%d out of range", n_rows);
    SQB_CHECK(shard_count >= 1 && shard_index >= 0 && shard_index < shard_count, SQB_ERR_INVALID, "sqb_nn_dist_hist_f64: bad shard %d/%d",
              shard_index, shard_count);
    SQB_CHECK((int64_t)n_rows * (S - 1) < (1LL << 40), SQB_ERR_INVALID, "sqb_nn_dist_hist_f64: output too large");
    for (int s = 0; s < S; ++s) {
        SQB_CHECK(!(support[s] != support[s]), SQB_ERR_INVALID, "sqb_nn_dist_hist_f64: support[%d] is NaN", s);
        SQB_CHECK(s == 0 || support[s] >= support[s - 1], SQB_ERR_INVALID, "sqb_nn_dist_hist_f64: support must be ascending (support[%d])", s);
    }
    for (int64_t i = 0; i < n_pts; ++i)
        SQB_CHECK(std::isfinite(pts[2 * i]) && std::isfinite(pts[2 * i + 1]), SQB_ERR_INVALID, "sqb_nn_dist_hist_f64: point %lld is not finite",
                  (long long)i);
    // reference sets: one grid per distinct (ref_begin, ref_end), sized for the largest k searched in it
    std::map<std::pair<int64_t, int64_t>, int> set_of;
    std::vector<std::pair<int64_t, int64_t>> ranges;
    std::vector<int> set_k, task_set(n_tasks);
    for (int64_t t = 0; t < n_tasks; ++t) {
        const int64_t* tk = tasks + 6 * t;
        const int64_t rb = tk[0], re = tk[1], qb = tk[2], qe = tk[3], k = tk[4], row = tk[5];
        SQB_CHECK(0 <= rb && rb <= re && re <= n_pts && 0 <= qb && qb <= qe && qe <= n_pts, SQB_ERR_INVALID,
                  "sqb_nn_dist_hist_f64: task %lld has a range outside [0, %lld]", (long long)t, (long long)n_pts);
        SQB_CHECK(k >= 1 && k <= 64, SQB_ERR_UNSUPPORTED, "sqb_nn_dist_hist_f64: task %lld: k=%lld outside [1, 64]", (long long)t, (long long)k);
        SQB_CHECK(k <= re - rb, SQB_ERR_INVALID, "Expected n_neighbors <= n_samples_fit, but n_neighbors = %lld, n_samples_fit = %lld (task %lld)",
                  (long long)k, (long long)(re - rb), (long long)t);
        SQB_CHECK(row >= 0 && row < n_rows, SQB_ERR_INVALID, "sqb_nn_dist_hist_f64: task %lld: row %lld outside [0, %d)", (long long)t,
                  (long long)row, n_rows);
        auto it = set_of.find({rb, re});
        if (it == set_of.end()) {
            it = set_of.emplace(std::make_pair(rb, re), (int)ranges.size()).first;
            ranges.push_back({rb, re});
            set_k.push_back(0);
        }
        task_set[t] = it->second;
        set_k[it->second] = std::max(set_k[it->second], (int)k);
    }
    const int n_sets = (int)ranges.size();
    std::vector<NnSet> sets(n_sets);
    int64_t n_entries = 0, n_cells = 0;
    for (int s = 0; s < n_sets; ++s) {
        const int64_t rb = ranges[s].first, re = ranges[s].second;
        double x0 = INFINITY, y0 = INFINITY, x1 = -INFINITY, y1 = -INFINITY;
        for (int64_t i = rb; i < re; ++i) {
            const double x = pts[2 * i], y = pts[2 * i + 1];
            x0 = x < x0 ? x : x0, x1 = x > x1 ? x : x1, y0 = y < y0 ? y : y0, y1 = y > y1 ? y : y1;
        }
        sets[s].gm = grid_geometry(x0, y0, x1, y1, re - rb, 0.0, knn_pts_per_cell(set_k[s]));
        sets[s].cell_off = n_cells;
        sets[s].ref_begin = rb;
        sets[s].entry_off = n_entries;
        n_cells += (int64_t)sets[s].gm.gx * sets[s].gm.gy;
        n_entries += re - rb;
    }
    SQB_CHECK(n_entries < 2147483647LL && n_cells < 2147483647LL, SQB_ERR_UNSUPPORTED,
              "sqb_nn_dist_hist_f64: %lld reference points in %lld cells do not fit int32", (long long)n_entries, (long long)n_cells);
    // query blocks in task order, dealt to the shards round robin; grouped by the kernel's k class
    std::vector<NnBlock> blocks[5];
    int64_t nblk_all = 0;
    for (int64_t t = 0; t < n_tasks; ++t) {
        const int64_t* tk = tasks + 6 * t;
        for (int64_t q0 = tk[2]; q0 < tk[3]; q0 += NN_QPB, ++nblk_all) {
            if (nblk_all % shard_count != shard_index) continue;
            NnBlock b;
            b.q0 = (int32_t)q0, b.q1 = (int32_t)std::min<int64_t>(q0 + NN_QPB, tk[3]), b.set = task_set[t], b.row = (int32_t)tk[5];
            b.k = (int32_t)tk[4], b.pad = 0;
            blocks[nnd_kclass(b.k)].push_back(b);
        }
    }
    const size_t out_n = (size_t)n_rows * (S - 1);
    int64_t nblk = 0;
    for (auto& v : blocks) nblk += (int64_t)v.size();
    if (nblk == 0) {
        std::fill(out, out + out_n, (int64_t)0);
        return SQB_OK;
    }
    sqb_ctx* c = ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    PointGrid g(c->stream);  // d_xy: the pool; d_pts / d_idx_sorted / d_cell_start: every reference set in cell order
    DevBuf<NnSet> d_sets(c->stream);
    DevBuf<NnBlock> d_blocks(c->stream);
    DevBuf<double> d_thr(c->stream);
    DevBuf<unsigned long long> d_out(c->stream);
    SQB_TRY(g.d_xy.alloc(2 * (size_t)std::max<int64_t>(n_pts, 1)));
    SQB_TRY(d_sets.alloc(n_sets));
    SQB_TRY(d_blocks.alloc(nblk));
    SQB_TRY(d_thr.alloc(S));
    SQB_TRY(d_out.alloc(out_n));
    SQB_CUDA(cudaMemcpyAsync(g.d_xy.p, pts, 2 * n_pts * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    SQB_CUDA(cudaMemcpyAsync(d_sets.p, sets.data(), n_sets * sizeof(NnSet), cudaMemcpyHostToDevice, c->stream));
    {
        int64_t off = 0;
        for (auto& v : blocks) {
            if (!v.empty()) SQB_CUDA(cudaMemcpyAsync(d_blocks.p + off, v.data(), v.size() * sizeof(NnBlock), cudaMemcpyHostToDevice, c->stream));
            off += (int64_t)v.size();
        }
    }
    std::vector<double> thr(S);
    nnd_thresholds(support, S, thr.data());
    SQB_CUDA(cudaMemcpyAsync(d_thr.p, thr.data(), S * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    SQB_CUDA(cudaMemsetAsync(d_out.p, 0, out_n * sizeof(unsigned long long), c->stream));
    {
        DevBuf<uint32_t> cell_a(c->stream), cell_b(c->stream);
        DevBuf<int32_t> idx_a(c->stream);
        DevBuf<uint8_t> tmp(c->stream);
        const int64_t ne = std::max<int64_t>(n_entries, 1);
        SQB_TRY(g.d_pts.alloc(ne));
        SQB_TRY(g.d_idx_sorted.alloc(ne));
        SQB_TRY(g.d_cell_start.alloc(n_cells + 1));
        SQB_TRY(cell_a.alloc(ne));
        SQB_TRY(cell_b.alloc(ne));
        SQB_TRY(idx_a.alloc(ne));
        if (n_entries > 0) {
            c->launches += 1;
            nnd_cell_id_kernel<<<(unsigned)ceil_div64(n_entries, 256), 256, 0, c->stream>>>(g.d_xy.p, d_sets.p, n_sets, n_entries, cell_a.p, idx_a.p);
            SQB_POST_LAUNCH();
            int bits = 1;
            while (bits < 32 && ((uint64_t)(n_cells - 1) >> bits) != 0) ++bits;
            size_t tmp_bytes = 0;
            SQB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, cell_a.p, cell_b.p, idx_a.p, g.d_idx_sorted.p, (int)n_entries, 0, bits,
                                                     c->stream));
            SQB_TRY(tmp.alloc(tmp_bytes > 0 ? tmp_bytes : 1));
            SQB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, cell_a.p, cell_b.p, idx_a.p, g.d_idx_sorted.p, (int)n_entries, 0, bits,
                                                     c->stream));
            c->launches += 2;
            graph_gather_kernel<<<(unsigned)ceil_div64(n_entries, 256), 256, 0, c->stream>>>(g.d_xy.p, cell_b.p, g.d_idx_sorted.p, n_entries, n_cells,
                                                                                            g.d_pts.p, g.d_cell_start.p);
            SQB_POST_LAUNCH();
        }
    }
    const double2* pool = reinterpret_cast<const double2*>(g.d_xy.p);
    const int64_t n_cls[5] = {(int64_t)blocks[0].size(), (int64_t)blocks[1].size(), (int64_t)blocks[2].size(), (int64_t)blocks[3].size(),
                              (int64_t)blocks[4].size()};
    const NnBlock* b = d_blocks.p;
    SQB_TRY(nnd_launch<2>(c, n_cls[0], pool, g.d_pts.p, g.d_cell_start.p, d_sets.p, b, d_thr.p, S, d_out.p));
    b += n_cls[0];
    SQB_TRY(nnd_launch<8>(c, n_cls[1], pool, g.d_pts.p, g.d_cell_start.p, d_sets.p, b, d_thr.p, S, d_out.p));
    b += n_cls[1];
    SQB_TRY(nnd_launch<16>(c, n_cls[2], pool, g.d_pts.p, g.d_cell_start.p, d_sets.p, b, d_thr.p, S, d_out.p));
    b += n_cls[2];
    SQB_TRY(nnd_launch<32>(c, n_cls[3], pool, g.d_pts.p, g.d_cell_start.p, d_sets.p, b, d_thr.p, S, d_out.p));
    b += n_cls[3];
    SQB_TRY(nnd_launch<64>(c, n_cls[4], pool, g.d_pts.p, g.d_cell_start.p, d_sets.p, b, d_thr.p, S, d_out.p));
    static_assert(sizeof(unsigned long long) == sizeof(int64_t), "counts are copied as int64");
    SQB_CUDA(cudaMemcpyAsync(out, d_out.p, out_n * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    return SQB_OK;
}

}  // extern "C"
