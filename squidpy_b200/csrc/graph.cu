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
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <math.h>

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
template <int KMAX>
__global__ void __launch_bounds__(128) graph_knn_kernel(const double2* __restrict__ pts, const int32_t* __restrict__ idx_sorted,
                                                        const int32_t* __restrict__ cell_start, int64_t n, GridGeom gm, int k,
                                                        int32_t* __restrict__ out_idx, double* __restrict__ out_dist) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n) return;
    const double2 q = pts[s];
    const int32_t qi = idx_sorted[s];
    const int cx = grid_cell_coord(q.x, gm.x0, gm.inv_cell, gm.gx), cy = grid_cell_coord(q.y, gm.y0, gm.inv_cell, gm.gy);
    double bd[KMAX];
    int32_t bi[KMAX];
#pragma unroll
    for (int t = 0; t < KMAX; ++t) {
        bd[t] = INFINITY;
        bi[t] = 0x7fffffff;
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
                    const int32_t j = idx_sorted[t];
                    if (j == qi) continue;  // the query point itself is not its own neighbour (kneighbors() without X)
                    const double2 p = pts[t];
                    const double dx = q.x - p.x, dy = q.y - p.y;
                    const double d2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
                    if (d2 < bd[k - 1] || (d2 == bd[k - 1] && j < bi[k - 1])) {
                        // insert (d2, j) into the ascending list of the k best
                        double cd = d2;
                        int32_t ci = j;
#pragma unroll
                        for (int u = 0; u < KMAX; ++u) {
                            if (u < k && (cd < bd[u] || (cd == bd[u] && ci < bi[u]))) {
                                const double td = bd[u];
                                const int32_t ti = bi[u];
                                bd[u] = cd;
                                bi[u] = ci;
                                cd = td;
                                ci = ti;
                            }
                        }
                    }
                }
                if (r == 0) break;
            }
        }
        // everything not yet visited lies beyond r cells; slightly shrunk bound: cell assignment is a rounded computation
        const double reach = (double)r * gm.cell * (1.0 - 1e-12);
        if (bd[k - 1] < reach * reach) break;
    }
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

}  // extern "C"
