// mask.cu — mask_graph: keep or drop the entries of a spatial graph by whether their segments lie within a polygon
// (sqb_mask_graph, include/squidpy_b200.h; the predicate is mask_pred.h).
//
// The polygon's rings become directed boundary edges on the host (mask_pred.h's ring_edges), bucketed twice over a uniform grid
// on their bounding box: per cell, every edge whose path (walked along its major axis, one cell of margin around it) may touch
// the cell; per row of cells ("band"), every edge whose y-range meets the row.  A band holds every edge a horizontal ray from a
// point of that row can cross or a point there can lie on (the row of a coordinate is monotone in it), so one kernel classifies
// each observation exactly once against its band.  One thread per stored entry (i, j) of adj then decides the segment
// coords[i] -> coords[j] from the two classes where they settle it (an exterior end point, or a zero-length segment) and
// otherwise tests the edges of the cells the segment's walk covers; the walks of a segment and of an edge meeting it share the
// cell holding their contact point.  dst's entries take the verdict of adj's entry at the same (row, col), and both matrices
// lose their removed entries and their zeros (scipy's eliminate_zeros) in one scan and compaction each.
#include <math.h>

#include <algorithm>
#include <tuple>
#include <vector>

#include "caller_graph.cuh"
#include "mask_pred.h"

using mpred::Edge;

namespace {

struct MaskGrid {
    double x0 = 0, y0 = 0, x1 = -1, y1 = -1, cell = 1, inv = 1;  // x1 < x0: no edges, every point is exterior
    int gx = 1, gy = 1;
};

__host__ __device__ __forceinline__ int grid_cell(double v, double v0, double inv, int g) {
    const double t = floor((v - v0) * inv);
    return t < 0.0 ? 0 : (t >= (double)g ? g - 1 : (int)t);
}

// f(cx, cy) for every cell of the walk of [a, b]: the columns (rows, for a steep segment) from one before its first to one past
// its last, and within each the rows (columns) its line passes over that stretch, one more on either side.  The margins absorb
// the rounding of the walk, so the cell of every point of the segment is visited.
template <typename F>
__host__ __device__ void grid_walk(const MaskGrid& g, double ax, double ay, double bx, double by, F f) {
    const bool steep = fabs(by - ay) > fabs(bx - ax);
    // major axis u, minor axis w
    double ua = steep ? ay : ax, wa = steep ? ax : ay, ub = steep ? by : bx, wb = steep ? bx : by;
    if (ub < ua) {
        double t = ua;
        ua = ub, ub = t;
        t = wa, wa = wb, wb = t;
    }
    const double u0 = steep ? g.y0 : g.x0, w0 = steep ? g.x0 : g.y0;
    const int gu = steep ? g.gy : g.gx, gw = steep ? g.gx : g.gy;
    const double s = ub > ua ? (wb - wa) / (ub - ua) : 0.0;
    const int c0 = max(grid_cell(ua, u0, g.inv, gu) - 1, 0), c1 = min(grid_cell(ub, u0, g.inv, gu) + 1, gu - 1);
    for (int c = c0; c <= c1; ++c) {
        const double ul = fmin(fmax(u0 + c * g.cell, ua), ub), uh = fmin(fmax(u0 + (c + 1) * g.cell, ua), ub);
        const double wl = wa + (ul - ua) * s, wh = wa + (uh - ua) * s;
        const int r0 = max(grid_cell(fmin(wl, wh), w0, g.inv, gw) - 1, 0), r1 = min(grid_cell(fmax(wl, wh), w0, g.inv, gw) + 1, gw - 1);
        for (int r = r0; r <= r1; ++r) steep ? f(r, c) : f(c, r);
    }
}

// the polygon on the device
struct MaskPoly {
    MaskGrid g;
    const Edge* edges;
    const int32_t *cell_ptr, *cell_idx;  // gx * gy cells, row-major by y
    const int32_t *band_ptr, *band_idx;  // gy rows
};

__device__ __forceinline__ Edge load_edge(const Edge* e) {
    const double2 a = __ldg(reinterpret_cast<const double2*>(e)), b = __ldg(reinterpret_cast<const double2*>(e) + 1);
    return Edge{a.x, a.y, b.x, b.y};
}

constexpr unsigned kIndexBad = 1u, kDuplicate = 2u, kCoordRange = 4u;

// Observation i: its float64 coordinates (xy of dtype T with element strides sr, sc), range checks, and its class.
template <typename T>
__global__ void __launch_bounds__(256) mask_points(const T* __restrict__ xy, int64_t n, int64_t sr, int64_t sc, MaskPoly P,
                                                   double2* __restrict__ pts, uint8_t* __restrict__ cls,
                                                   unsigned long long* __restrict__ first_nonfinite, unsigned* __restrict__ err) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double x = (double)xy[i * sr], y = (double)xy[i * sr + sc];
        pts[i] = make_double2(x, y);
        if (!(isfinite(x) && isfinite(y))) {
            atomicMin(first_nonfinite, (unsigned long long)i);
            cls[i] = mpred::EXTERIOR;
            continue;
        }
        const double ax = fabs(x), ay = fabs(y);
        if (ax > dpred::COORD_MAX || (ax != 0.0 && ax < dpred::COORD_MIN) || ay > dpred::COORD_MAX || (ay != 0.0 && ay < dpred::COORD_MIN))
            atomicOr(err, kCoordRange);
        int c = mpred::EXTERIOR;
        if (x >= P.g.x0 && x <= P.g.x1 && y >= P.g.y0 && y <= P.g.y1) {
            const int r = grid_cell(y, P.g.y0, P.g.inv, P.g.gy);
            const int32_t* band = P.band_idx + P.band_ptr[r];
            c = mpred::classify_point(x, y, P.band_ptr[r + 1] - P.band_ptr[r], [&](int64_t k) { return load_edge(P.edges + band[k]); });
        }
        cls[i] = (uint8_t)c;
    }
}

// the row of entry e: the last r with ptr[r] <= e (ptr of n + 1 entries, e < ptr[n])
__device__ __forceinline__ int64_t row_of(const uint32_t* __restrict__ ptr, int64_t n, int64_t e) {
    int64_t lo = 0, hi = n;  // ptr[lo] <= e < ptr[hi]
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if ((int64_t)ptr[mid] <= e)
            lo = mid;
        else
            hi = mid;
    }
    return lo;
}

// raises kDuplicate when column j of entry e occurs earlier in its row (the scan runs only where the row is not ascending)
__device__ __forceinline__ void check_repeat(const int32_t* __restrict__ col, int64_t start, int64_t e, int32_t j, unsigned* err) {
    if (e > start && col[e - 1] >= j)
        for (int64_t k = start; k < e; ++k)
            if (col[k] == j) {
                atomicOr(err, kDuplicate);
                return;
            }
}

// Entry e = (i, j) of adj: removed[e] = whether the mask drops it, keep[e] = !removed and a non-zero value (bits & nz_mask).
template <typename U>
__global__ void __launch_bounds__(256) mask_adj(const uint32_t* __restrict__ ptr, const int32_t* __restrict__ col, const U* __restrict__ val,
                                                U nz_mask, int64_t n, int64_t nnz, const double2* __restrict__ pts,
                                                const uint8_t* __restrict__ cls, MaskPoly P, int negative, uint8_t* __restrict__ removed,
                                                uint32_t* __restrict__ keep, unsigned* __restrict__ err) {
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = row_of(ptr, n, e);
        const int32_t j = col[e];
        check_repeat(col, ptr[i], e, j, err);
        const double2 p = pts[i], q = pts[j];
        const auto scan_cells = [&](double ax, double ay, double bx, double by, auto f) {
            grid_walk(P.g, ax, ay, bx, by, [&](int cx, int cy) {
                const int64_t cell = (int64_t)cy * P.g.gx + cx;
                const int32_t* list = P.cell_idx + P.cell_ptr[cell];
                f((int64_t)(P.cell_ptr[cell + 1] - P.cell_ptr[cell]), [&](int64_t k) { return load_edge(P.edges + list[k]); });
            });
        };
        const bool within = mpred::segment_within(
            p.x, p.y, cls[i], q.x, q.y, cls[j], [&](auto f) { scan_cells(p.x, p.y, q.x, q.y, f); },
            [&](double x, double y, auto f) { scan_cells(x, y, x, y, f); });
        const bool rm = negative ? within : !within;
        removed[e] = rm;
        keep[e] = !rm && (val[e] & nz_mask) != 0;
    }
}

// Entry e = (i, c) of dst: removed when adj's entry (i, c) is; keep[e] = !removed and a non-zero value.
template <typename U>
__global__ void __launch_bounds__(256) mask_dst(const uint32_t* __restrict__ ptr, const int32_t* __restrict__ col, const U* __restrict__ val,
                                                U nz_mask, int64_t n, int64_t nnz, const uint32_t* __restrict__ aptr,
                                                const int32_t* __restrict__ acol, const uint8_t* __restrict__ aremoved,
                                                uint32_t* __restrict__ keep, unsigned* __restrict__ err) {
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = row_of(ptr, n, e);
        const int32_t c = col[e];
        check_repeat(col, ptr[i], e, c, err);
        const int64_t a0 = aptr[i], a1 = aptr[i + 1], same = a0 + (e - (int64_t)ptr[i]);  // adj's entry when the rows align
        int64_t at = -1;
        if (same < a1 && acol[same] == c)
            at = same;
        else
            for (int64_t k = a0; k < a1; ++k)
                if (acol[k] == c) {
                    at = k;
                    break;
                }
        const bool rm = at >= 0 && aremoved[at];
        keep[e] = !rm && (val[e] & nz_mask) != 0;
    }
}

// indices of a caller's CSR as int32; an index outside [0, n) raises kIndexBad and is written as 0
template <typename II>
__global__ void __launch_bounds__(256) mask_indices(const II* __restrict__ ix, int64_t nnz, int64_t n, int32_t* __restrict__ col,
                                                    unsigned* __restrict__ err) {
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t j = (int64_t)ix[e];
        const bool ok = j >= 0 && j < n;
        if (!ok) atomicOr(err, kIndexBad);
        col[e] = ok ? (int32_t)j : 0;
    }
}

// the kept entries at their ranks, and the compacted indptr
template <typename U>
__global__ void __launch_bounds__(256) mask_compact(const uint32_t* __restrict__ keep, const uint32_t* __restrict__ rank,
                                                    const int32_t* __restrict__ col, const U* __restrict__ val, int64_t nnz,
                                                    int32_t* __restrict__ out_col, U* __restrict__ out_val) {
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
        if (!keep[e]) continue;
        const uint32_t q = rank[e];
        out_col[q] = col[e];
        out_val[q] = val[e];
    }
}

__global__ void __launch_bounds__(256) mask_indptr(const uint32_t* __restrict__ ptr, const uint32_t* __restrict__ rank, int64_t n, int64_t nnz,
                                                   uint32_t total, int32_t* __restrict__ out) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r <= n; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = ptr[r];
        out[r] = (int32_t)(s < nnz ? rank[s] : total);
    }
}

// A graph as the kernels read it: validated uint32 indptr, int32 columns, the values as stored (vbytes each).
struct MGraph {
    explicit MGraph(cudaStream_t s) : ptr(s), col(s), val(s) {}
    DevBuf<uint32_t> ptr;
    DevBuf<int32_t> col;
    DevBuf<uint8_t> val;
    int64_t nnz = 0;
    int code = 0, vbytes = 0;
};

// f(SqbType<U>(), nz_mask): the storage type of a value dtype code and the bits that make a value non-zero (a float's sign
// bit alone is -0.0, a zero; NaN is non-zero)
template <typename F>
int with_storage(int code, F&& f) {
    switch (code) {
        case 0: return f(SqbType<uint32_t>(), (uint32_t)0x7FFFFFFFu);
        case 1: return f(SqbType<uint64_t>(), (uint64_t)0x7FFFFFFFFFFFFFFFull);
        case 3: return f(SqbType<uint32_t>(), ~(uint32_t)0);
        case 4: return f(SqbType<uint64_t>(), ~(uint64_t)0);
        case 5: return f(SqbType<uint8_t>(), (uint8_t)0xFF);
    }
    return SQB_ERR_INVALID;
}

int load_graph(sqb_ctx* c, const SqbGraphArgs& a, MGraph& g, unsigned* err, const char* where) {
    SQB_TRY(sqb_check_graph_args(a, 31, where));
    SQB_CHECK(!a.csc, SQB_ERR_INVALID, "%s: a CSC graph is not supported; pass it as CSR", where);
    SQB_CHECK(a.data_dtype == 0 || a.data_dtype == 1 || a.data_dtype == 3 || a.data_dtype == 4 || a.data_dtype == 5, SQB_ERR_INVALID,
              "%s: data_dtype must be 0 (f32), 1 (f64), 3 (i32), 4 (i64) or 5 (bool)", where);
    g.nnz = a.nnz, g.code = a.data_dtype, g.vbytes = sqb_graph_value_bytes(a.data_dtype);
    SQB_TRY(g.ptr.alloc(a.n + 1));
    SQB_TRY(g.col.alloc(a.nnz));
    SQB_TRY(g.val.alloc(a.nnz * g.vbytes));
    return sqb_with_caller_csr(c, a.n, a.nnz, a.indptr, a.indptr_bits, a.indices, a.index_bits, a.data, g.vbytes, a.device_input, a.producer_stream,
                               [&](const void* ip, const void* ix, const void* dv) {
                                   return sqb_dispatch_index(a.indptr_bits, a.index_bits, where, [&](auto tp, auto tx) -> int {
                                       using IP = typename decltype(tp)::type;
                                       using II = typename decltype(tx)::type;
                                       SQB_TRY(sqb_check_indptr(c, SQB_K_MISC, reinterpret_cast<const IP*>(ip), a.n, a.nnz, g.ptr.p, where));
                                       if (a.nnz == 0) return SQB_OK;
                                       {
                                           SqbLaunchScope scope(c, SQB_K_MISC);
                                           mask_indices<II><<<sqb_grid_rows(c, a.nnz, 256), 256, 0, c->stream>>>(
                                               reinterpret_cast<const II*>(ix), a.nnz, a.n, g.col.p, err);
                                           SQB_POST_LAUNCH();
                                       }
                                       SQB_CUDA(cudaMemcpyAsync(g.val.p, dv, a.nnz * g.vbytes, cudaMemcpyDeviceToDevice, c->stream));
                                       return SQB_OK;
                                   });
                               });
}

// the masked graph: keep flags -> ranks -> compacted columns, values and indptr
struct MaskCsr {
    explicit MaskCsr(cudaStream_t s) : ptr(s), col(s), val(s) {}
    DevBuf<int32_t> ptr, col;
    DevBuf<uint8_t> val;
    int64_t nnz = 0;
    int vbytes = 0;
};

int compact(sqb_ctx* c, const MGraph& g, int64_t n, const uint32_t* keep, MaskCsr& out) {
    out.vbytes = g.vbytes;
    SQB_TRY(out.ptr.alloc(n + 1));
    uint32_t total = 0;
    DevBuf<uint32_t> rank(c->stream);
    if (g.nnz > 0) {
        SQB_TRY(rank.alloc(g.nnz));
        SQB_TRY(sqb_exclusive_scan(c, keep, rank.p, g.nnz, &total));
    }
    out.nnz = total;
    SQB_TRY(out.col.alloc(total));
    SQB_TRY(out.val.alloc((size_t)total * g.vbytes));
    if (g.nnz > 0)
        SQB_TRY(with_storage(g.code, [&](auto tu, auto) -> int {
            using U = typename decltype(tu)::type;
            SqbLaunchScope scope(c, SQB_K_MISC);
            mask_compact<U><<<sqb_grid_rows(c, g.nnz, 256), 256, 0, c->stream>>>(keep, rank.p, g.col.p, reinterpret_cast<const U*>(g.val.p), g.nnz,
                                                                                 out.col.p, reinterpret_cast<U*>(out.val.p));
            SQB_POST_LAUNCH();
            return SQB_OK;
        }));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        mask_indptr<<<sqb_grid_rows(c, n + 1, 256), 256, 0, c->stream>>>(g.ptr.p, rank.p, n, g.nnz, total, out.ptr.p);
        SQB_POST_LAUNCH();
    }
    return SQB_OK;
}

bool coord_ok(double v) {
    const double a = fabs(v);
    return isfinite(v) && (a == 0.0 || (a >= dpred::COORD_MIN && a <= dpred::COORD_MAX));
}

// The grid of the edges' bounding box: about two cells per edge, at most 2048 per side, and cells no smaller than 2^-30 of the
// largest coordinate, so that the walks' rounding stays far below a cell.
MaskGrid make_grid(const std::vector<Edge>& edges) {
    MaskGrid g;
    if (edges.empty()) return g;
    g.x0 = g.y0 = INFINITY, g.x1 = g.y1 = -INFINITY;
    for (const Edge& e : edges) {
        g.x0 = std::min({g.x0, e.ax, e.bx}), g.x1 = std::max({g.x1, e.ax, e.bx});
        g.y0 = std::min({g.y0, e.ay, e.by}), g.y1 = std::max({g.y1, e.ay, e.by});
    }
    const double w = g.x1 - g.x0, h = g.y1 - g.y0, big = std::max({fabs(g.x0), fabs(g.x1), fabs(g.y0), fabs(g.y1)});
    double cell = std::sqrt(w * h / (2.0 * (double)edges.size()));
    cell = std::max({cell, std::max(w, h) / 2047.0, big * 0x1p-30});
    if (!(cell > 0.0)) cell = 1.0;
    g.cell = cell, g.inv = 1.0 / cell;
    g.gx = std::min((int)(w / cell) + 1, 2048), g.gy = std::min((int)(h / cell) + 1, 2048);
    return g;
}

// CSR lists (ptr of m + 1, idx) from (bucket, edge) pairs produced by visit(f) with f(bucket, edge), called twice
template <typename V>
void bucket_lists(int64_t m, V visit, std::vector<int32_t>& ptr, std::vector<int32_t>& idx) {
    ptr.assign(m + 1, 0);
    visit([&](int64_t b, int32_t) { ++ptr[b + 1]; });
    for (int64_t b = 0; b < m; ++b) ptr[b + 1] += ptr[b];
    idx.resize(std::max<int64_t>(ptr[m], 1));
    std::vector<int32_t> fill(ptr.begin(), ptr.end() - 1);
    visit([&](int64_t b, int32_t k) { idx[fill[b]++] = k; });
}

}  // namespace

struct sqb_masked {
    explicit sqb_masked(sqb_ctx* ctx) : c(ctx), adj(ctx->stream), dst(ctx->stream) {}
    sqb_ctx* c;
    int64_t n = 0;
    MaskCsr adj, dst;
};

extern "C" {

int sqb_mask_graph(sqb_ctx* ctx, int64_t n, int64_t adj_nnz, const void* adj_indptr, int adj_indptr_bits, const void* adj_indices,
                   int adj_index_bits, const void* adj_data, int adj_dtype, int64_t dst_nnz, const void* dst_indptr, int dst_indptr_bits,
                   const void* dst_indices, int dst_index_bits, const void* dst_data, int dst_dtype, int graph_device, uintptr_t graph_stream,
                   const void* xy, int xy_dtype, int64_t stride_row, int64_t stride_col, int xy_device, uintptr_t xy_stream, const double* ring_xy,
                   const int64_t* ring_ptr, const uint8_t* ring_hole, int64_t n_rings, int negative, sqb_masked** out, int64_t* adj_nnz_out,
                   int64_t* dst_nnz_out) {
    const char* where = "sqb_mask_graph";
    SQB_CHECK(ctx && out && adj_nnz_out && dst_nnz_out && (xy || n == 0), SQB_ERR_INVALID, "%s: null argument", where);
    SQB_CHECK(xy_dtype == 0 || xy_dtype == 1, SQB_ERR_INVALID, "%s: xy_dtype must be 0 (f32) or 1 (f64)", where);
    SQB_CHECK(n_rings >= 0 && (n_rings == 0 || (ring_xy && ring_ptr && ring_hole)), SQB_ERR_INVALID, "%s: null polygon argument", where);
    *out = nullptr;
    sqb_ctx* c = ctx;
    SQB_CUDA(cudaSetDevice(c->device));

    // the polygon: directed edges, their grid and its cell and band lists (host)
    std::vector<Edge> edges;
    {
        std::vector<double> scratch;
        for (int64_t r = 0; r < n_rings; ++r) {
            const int64_t b = ring_ptr[r], m = ring_ptr[r + 1] - b;
            SQB_CHECK(b >= 0 && m >= 0, SQB_ERR_INVALID, "%s: ring_ptr must not decrease", where);
            for (int64_t k = 0; k < 2 * m; ++k)
                SQB_CHECK(coord_ok(ring_xy[2 * b + k]), SQB_ERR_INVALID,
                          "polygon vertices must be finite and 0 or of magnitude in [2^-120, 2^120]");
            scratch.resize(2 * m + 2);
            const size_t at = edges.size();
            edges.resize(at + m);
            edges.resize(at + mpred::ring_edges(ring_xy + 2 * b, m, ring_hole[r] != 0, scratch.data(), edges.data() + at));
        }
    }
    const MaskGrid grid = make_grid(edges);
    std::vector<int32_t> cell_ptr, cell_idx, band_ptr, band_idx;
    bucket_lists((int64_t)grid.gx * grid.gy, [&](auto f) {
        for (int32_t k = 0; k < (int32_t)edges.size(); ++k) {
            const Edge& e = edges[k];
            grid_walk(grid, e.ax, e.ay, e.bx, e.by, [&](int cx, int cy) { f((int64_t)cy * grid.gx + cx, k); });
        }
    }, cell_ptr, cell_idx);
    bucket_lists(grid.gy, [&](auto f) {
        for (int32_t k = 0; k < (int32_t)edges.size(); ++k) {
            const Edge& e = edges[k];
            const int r0 = grid_cell(std::min(e.ay, e.by), grid.y0, grid.inv, grid.gy), r1 = grid_cell(std::max(e.ay, e.by), grid.y0, grid.inv, grid.gy);
            for (int r = r0; r <= r1; ++r) f(r, k);
        }
    }, band_ptr, band_idx);
    DevBuf<Edge> d_edges(c->stream);
    DevBuf<int32_t> d_cell_ptr(c->stream), d_cell_idx(c->stream), d_band_ptr(c->stream), d_band_idx(c->stream);
    const auto upload = [&](auto& buf, const auto& v) -> int {
        SQB_TRY(buf.alloc(std::max<size_t>(v.size(), 1)));
        if (!v.empty()) SQB_CUDA(cudaMemcpyAsync(buf.p, v.data(), v.size() * sizeof(v[0]), cudaMemcpyHostToDevice, c->stream));
        return SQB_OK;
    };
    SQB_TRY(upload(d_edges, edges));
    SQB_TRY(upload(d_cell_ptr, cell_ptr));
    SQB_TRY(upload(d_cell_idx, cell_idx));
    SQB_TRY(upload(d_band_ptr, band_ptr));
    SQB_TRY(upload(d_band_idx, band_idx));
    const MaskPoly P{grid, d_edges.p, d_cell_ptr.p, d_cell_idx.p, d_band_ptr.p, d_band_idx.p};

    // the graphs, as uint32 indptr / int32 columns / stored values in the library's buffers
    DevBuf<unsigned> err(c->stream);
    DevBuf<unsigned long long> first_nonfinite(c->stream);
    SQB_TRY(err.alloc(1));
    SQB_TRY(first_nonfinite.alloc(1));
    SQB_CUDA(cudaMemsetAsync(err.p, 0, sizeof(unsigned), c->stream));
    SQB_CUDA(cudaMemsetAsync(first_nonfinite.p, 0xFF, sizeof(unsigned long long), c->stream));
    MGraph adj(c->stream), dst(c->stream);
    const SqbGraphArgs aa{n, adj_nnz, adj_indptr, adj_indices, adj_data, adj_indptr_bits, adj_index_bits, adj_dtype, 0, graph_device, graph_stream};
    const SqbGraphArgs da{n, dst_nnz, dst_indptr, dst_indices, dst_data, dst_indptr_bits, dst_index_bits, dst_dtype, 0, graph_device, graph_stream};
    SQB_TRY(load_graph(c, aa, adj, err.p, "sqb_mask_graph (connectivities)"));
    SQB_TRY(load_graph(c, da, dst, err.p, "sqb_mask_graph (distances)"));

    // the observations: float64 coordinates and classes
    DevBuf<double2> pts(c->stream);
    DevBuf<uint8_t> cls(c->stream);
    SQB_TRY(pts.alloc(n));
    SQB_TRY(cls.alloc(n));
    const auto classify = [&](const void* p, int code, int64_t sr, int64_t sc) -> int {
        SqbLaunchScope scope(c, SQB_K_MISC);
        if (code == 1)
            mask_points<double><<<sqb_grid_rows(c, n, 256), 256, 0, c->stream>>>(static_cast<const double*>(p), n, sr, sc, P, pts.p, cls.p,
                                                                                  first_nonfinite.p, err.p);
        else
            mask_points<float><<<sqb_grid_rows(c, n, 256), 256, 0, c->stream>>>(static_cast<const float*>(p), n, sr, sc, P, pts.p, cls.p,
                                                                                 first_nonfinite.p, err.p);
        SQB_POST_LAUNCH();
        return SQB_OK;
    };
    if (xy_device) {
        SQB_TRY(sqb_read_caller_buffers(c, xy_stream, [&]() -> int {
            SQB_TRY(classify(xy, xy_dtype, stride_row, stride_col));
            SQB_CUDA(cudaStreamSynchronize(c->stream));  // the caller's coordinates are no longer read
            return SQB_OK;
        }));
    } else {
        SQB_CHECK(xy_dtype == 1 && stride_row == 2 && stride_col == 1, SQB_ERR_INVALID, "%s: host coordinates must be C-contiguous float64", where);
        DevBuf<double> h(c->stream);
        SQB_TRY(h.alloc(2 * n));
        SQB_TRY(sqb_h2d(c, h.p, xy, 2 * n * sizeof(double)));
        SQB_TRY(classify(h.p, 1, 2, 1));
    }

    // the verdicts: adj by its segments, dst by adj's entry at the same position
    DevBuf<uint8_t> removed(c->stream);
    DevBuf<uint32_t> keep_a(c->stream), keep_d(c->stream);
    SQB_TRY(removed.alloc(adj.nnz));
    SQB_TRY(keep_a.alloc(adj.nnz));
    SQB_TRY(keep_d.alloc(dst.nnz));
    if (adj.nnz > 0)
        SQB_TRY(with_storage(adj.code, [&](auto tu, auto mask) -> int {
            using U = typename decltype(tu)::type;
            SqbLaunchScope scope(c, SQB_K_MISC);
            mask_adj<U><<<sqb_grid_rows(c, adj.nnz, 256), 256, 0, c->stream>>>(adj.ptr.p, adj.col.p, reinterpret_cast<const U*>(adj.val.p), mask, n,
                                                                                adj.nnz, pts.p, cls.p, P, negative, removed.p, keep_a.p, err.p);
            SQB_POST_LAUNCH();
            return SQB_OK;
        }));
    if (dst.nnz > 0)
        SQB_TRY(with_storage(dst.code, [&](auto tu, auto mask) -> int {
            using U = typename decltype(tu)::type;
            SqbLaunchScope scope(c, SQB_K_MISC);
            mask_dst<U><<<sqb_grid_rows(c, dst.nnz, 256), 256, 0, c->stream>>>(dst.ptr.p, dst.col.p, reinterpret_cast<const U*>(dst.val.p), mask, n,
                                                                                dst.nnz, adj.ptr.p, adj.col.p, removed.p, keep_d.p, err.p);
            SQB_POST_LAUNCH();
            return SQB_OK;
        }));
    unsigned flags = 0;
    unsigned long long bad = 0;
    SQB_CUDA(cudaMemcpyAsync(&flags, err.p, sizeof(unsigned), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaMemcpyAsync(&bad, first_nonfinite.p, sizeof(bad), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    SQB_CHECK(bad == ~0ull, SQB_ERR_INVALID, "coordinates of observation %lld are not finite", (long long)bad);
    SQB_CHECK(!(flags & kCoordRange), SQB_ERR_INVALID, "coordinates must be 0 or of magnitude in [2^-120, 2^120]");
    SQB_CHECK(!(flags & kIndexBad), SQB_ERR_INVALID, "%s: index out of range [0, %lld)", where, (long long)n);
    SQB_CHECK(!(flags & kDuplicate), SQB_ERR_INVALID, "%s: the graph stores a (row, col) entry more than once; sum duplicates first", where);

    sqb_masked* m = new sqb_masked(c);
    m->n = n;
    int rc = compact(c, adj, n, keep_a.p, m->adj);
    if (rc == SQB_OK) rc = compact(c, dst, n, keep_d.p, m->dst);
    if (rc == SQB_OK) rc = cudaStreamSynchronize(c->stream) == cudaSuccess ? SQB_OK : SQB_ERR_CUDA;
    if (rc != SQB_OK) {
        delete m;
        return rc;
    }
    *out = m;
    *adj_nnz_out = m->adj.nnz;
    *dst_nnz_out = m->dst.nnz;
    return SQB_OK;
}

int sqb_mask_export(sqb_masked* m, int32_t* adj_indptr, int32_t* adj_indices, void* adj_data, int32_t* dst_indptr, int32_t* dst_indices,
                    void* dst_data, uintptr_t consumer_stream) {
    SQB_CHECK(m && adj_indptr && dst_indptr, SQB_ERR_INVALID, "sqb_mask_export: null argument");
    SQB_CHECK((adj_indices && adj_data) || m->adj.nnz == 0, SQB_ERR_INVALID, "sqb_mask_export: null connectivities buffer");
    SQB_CHECK((dst_indices && dst_data) || m->dst.nnz == 0, SQB_ERR_INVALID, "sqb_mask_export: null distances buffer");
    sqb_ctx* c = m->c;
    SQB_CUDA(cudaSetDevice(c->device));
    SQB_TRY(sqb_wait_producer(c, consumer_stream));
    const auto copy = [&](void* to, const void* from, size_t bytes) -> int {
        if (bytes) SQB_CUDA(cudaMemcpyAsync(to, from, bytes, cudaMemcpyDefault, c->stream));
        return SQB_OK;
    };
    for (const auto& [g, ip, ix, v] : {std::make_tuple(&m->adj, adj_indptr, adj_indices, adj_data), std::make_tuple(&m->dst, dst_indptr, dst_indices, dst_data)}) {
        SQB_TRY(copy(ip, g->ptr.p, (m->n + 1) * sizeof(int32_t)));
        SQB_TRY(copy(ix, g->col.p, g->nnz * sizeof(int32_t)));
        SQB_TRY(copy(v, g->val.p, g->nnz * g->vbytes));
    }
    SQB_CUDA(cudaStreamSynchronize(c->stream));  // the buffers are complete when the call returns
    return SQB_OK;
}

int sqb_mask_free(sqb_masked* m) {
    if (!m) return SQB_OK;
    SQB_CUDA(cudaSetDevice(m->c->device));
    delete m;
    return SQB_OK;
}

}  // extern "C"
