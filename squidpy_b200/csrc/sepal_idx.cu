// sepal_idx.cu — the saturation tables of sepal (`_compute_idxs`, src/squidpy/gr/_sepal.py:308-361) from a caller's graph
// and coordinates, on the host or in device memory, built on the device (sqb_sepal_idxs).
//
// The graph is loaded as stored (caller_graph.cuh: a CSC becomes scipy's tocsr).  An entry counts when its value is not 0
// (scipy's eliminate_zeros: NaN counts, -0.0 and False do not).  One warp per row counts a row's entries (its degree) and,
// once the maximum degree has been checked on the host, writes the row's tables: a saturated row (degree == max_neighs)
// its columns in storage order, an unsaturated one its first saturated column, found by a ballot over each 32 entries.
// Unsaturated rows without a saturated neighbour ("orphans") take the saturated node nearest in L1 distance:
//     argmin_j (|x_o - x_j| + |y_o - y_j|)  over the saturated nodes j in ascending order, in float64,
// numpy's argmin of scikit-learn's (scipy's cityblock) distance row: the lowest position wins ties and the first NaN wins
// outright.  Each candidate is a key k = 0 for NaN, else bits(d) + 1 (d >= 0, so the bit patterns order like the values),
// and the argmin is the least (k, j): a minimum of an order-free reduction, so the tiled brute force below is exact whatever
// the tiling.  Its cost is orphans x n_sat distance evaluations; no orphans x n_sat matrix is stored.
#include <math.h>

#include "caller_graph.cuh"

namespace {

constexpr int kOrphTile = 8;     // orphans per thread of a search block (coordinates and running minimum in registers)
constexpr int kSearchT = 256;    // threads of a search block
constexpr int kMinChunk = 2048;  // least saturated nodes per search block

__device__ __forceinline__ unsigned lanes_below(int lane) { return (1u << lane) - 1u; }

// deg[i] = the entries of row i whose value is not 0; is_sat[i] = deg[i] == k; *max_deg = the largest degree.
__global__ void __launch_bounds__(256) si_degree(const uint32_t* __restrict__ ptr, const double* __restrict__ val, int64_t n, int k,
                                                 uint32_t* __restrict__ is_sat, unsigned* __restrict__ max_deg) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    unsigned most = 0;
    for (int64_t i = warp; i < n; i += nwarps) {
        unsigned deg = 0;
        for (uint32_t e0 = ptr[i]; e0 < ptr[i + 1]; e0 += 32) {
            const uint32_t e = e0 + lane;
            deg += __popc(__ballot_sync(~0u, e < ptr[i + 1] && val[e] != 0.0));
        }
        if (lane == 0) is_sat[i] = deg == (unsigned)k;
        most = max(most, deg);
    }
    if (lane == 0 && most) atomicMax(max_deg, most);
}

// Row i's tables.  sat_rank[i]: the saturated rows before i.  Saturated: sat[r] = i, sat_idx[r, :] = its counted columns in
// storage order.  Unsaturated (rank q = i - sat_rank[i]): unsat[q] = i, unsat_idx[q] = its first counted column that is
// saturated, or -1 with q appended to orphans.
__global__ void __launch_bounds__(256) si_tables(const uint32_t* __restrict__ ptr, const int32_t* __restrict__ col, const double* __restrict__ val,
                                                 int64_t n, int k, const uint32_t* __restrict__ is_sat, const uint32_t* __restrict__ sat_rank,
                                                 int32_t* __restrict__ sat, int32_t* __restrict__ sat_idx, int32_t* __restrict__ unsat,
                                                 int32_t* __restrict__ unsat_idx, int32_t* __restrict__ orphans, unsigned* __restrict__ n_orph) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = warp; i < n; i += nwarps) {
        const uint32_t lo = ptr[i], hi = ptr[i + 1];
        const int64_t r = sat_rank[i];
        if (is_sat[i]) {
            if (lane == 0) sat[r] = (int32_t)i;
            int32_t* out = sat_idx + r * k;
            unsigned at = 0;
            for (uint32_t e0 = lo; e0 < hi; e0 += 32) {
                const uint32_t e = e0 + lane;
                const bool nz = e < hi && val[e] != 0.0;
                const unsigned m = __ballot_sync(~0u, nz);
                if (nz) out[at + __popc(m & lanes_below(lane))] = col[e];
                at += __popc(m);
            }
            continue;
        }
        const int64_t q = i - r;
        int32_t first = -1;
        for (uint32_t e0 = lo; e0 < hi && first < 0; e0 += 32) {
            const uint32_t e = e0 + lane;
            const bool hit = e < hi && val[e] != 0.0 && is_sat[col[e]];
            const unsigned m = __ballot_sync(~0u, hit);
            if (m) first = __shfl_sync(~0u, e < hi ? col[e] : 0, __ffs(m) - 1);
        }
        if (lane == 0) {
            unsat[q] = (int32_t)i;
            unsat_idx[q] = first;
            if (first < 0) orphans[atomicAdd(n_orph, 1u)] = (int32_t)q;
        }
    }
}

// pts[p] = the float64 coordinates of observation rows[p] (rows[via[p]] when via is not null); bit 0 of *nonfinite when one
// of them is NaN or infinite.
template <typename XT>
__global__ void __launch_bounds__(256) si_gather(const XT* __restrict__ xy, int64_t sr, int64_t sc, const int32_t* __restrict__ rows,
                                                 const int32_t* __restrict__ via, int64_t m, double2* __restrict__ pts,
                                                 unsigned* __restrict__ nonfinite) {
    bool bad = false;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < m; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = rows[via ? via[p] : p];
        const double x = (double)xy[i * sr], y = (double)xy[i * sr + sc];
        bad |= !isfinite(x) || !isfinite(y);
        pts[p] = make_double2(x, y);
    }
    if (bad) atomicOr(nonfinite, 1u);
}

// The order of a candidate: NaN first, then ascending distance (d >= 0, +inf last).
__device__ __forceinline__ unsigned long long dist_key(double d) {
    return isnan(d) ? 0ull : (unsigned long long)__double_as_longlong(d) + 1ull;
}

__device__ __forceinline__ void take_min(unsigned long long& k, int32_t& j, unsigned long long k2, int32_t j2) {
    if (k2 < k || (k2 == k && j2 < j)) k = k2, j = j2;
}

// Block (tile, chunk): the least (key, j) of orphans tile * kOrphTile + t against the saturated nodes of the chunk, into
// part[(tile * kOrphTile + t) * n_chunks + chunk].
__global__ void __launch_bounds__(kSearchT) si_nearest(const double2* __restrict__ opts, int64_t n_orph, const double2* __restrict__ spts,
                                                       int64_t n_sat, int64_t chunk_len, int n_chunks, ulonglong2* __restrict__ part) {
    __shared__ unsigned long long s_k[kSearchT / 32][kOrphTile];
    __shared__ int32_t s_j[kSearchT / 32][kOrphTile];
    const int64_t o0 = (int64_t)blockIdx.x * kOrphTile;
    double ox[kOrphTile], oy[kOrphTile];
    unsigned long long bk[kOrphTile];
    int32_t bj[kOrphTile];
#pragma unroll
    for (int t = 0; t < kOrphTile; ++t) {
        const double2 o = opts[min(o0 + t, n_orph - 1)];  // a padding slot repeats the last orphan and is not written
        ox[t] = o.x, oy[t] = o.y;
        bk[t] = ~0ull, bj[t] = INT32_MAX;
    }
    const int64_t j0 = (int64_t)blockIdx.y * chunk_len, j1 = min(j0 + chunk_len, n_sat);
    for (int64_t j = j0 + threadIdx.x; j < j1; j += kSearchT) {  // ascending j per thread: a strict < keeps the first
        const double2 s = spts[j];
#pragma unroll
        for (int t = 0; t < kOrphTile; ++t) {
            const unsigned long long kk = dist_key(__dadd_rn(fabs(__dsub_rn(ox[t], s.x)), fabs(__dsub_rn(oy[t], s.y))));
            if (kk < bk[t]) bk[t] = kk, bj[t] = (int32_t)j;
        }
    }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int t = 0; t < kOrphTile; ++t) {
        for (int off = 16; off; off >>= 1) take_min(bk[t], bj[t], __shfl_down_sync(~0u, bk[t], off), __shfl_down_sync(~0u, bj[t], off));
        if (lane == 0) s_k[w][t] = bk[t], s_j[w][t] = bj[t];
    }
    __syncthreads();
    if (threadIdx.x < kOrphTile && o0 + threadIdx.x < n_orph) {
        const int t = threadIdx.x;
        unsigned long long k = s_k[0][t];
        int32_t j = s_j[0][t];
        for (int v = 1; v < kSearchT / 32; ++v) take_min(k, j, s_k[v][t], s_j[v][t]);
        part[(o0 + t) * n_chunks + blockIdx.y] = make_ulonglong2(k, (unsigned long long)(uint32_t)j);
    }
}

// unsat_idx[orphans[o]] = sat[the least (key, j) over the chunks of orphan o].
__global__ void __launch_bounds__(256) si_finish(const ulonglong2* __restrict__ part, int64_t n_orph, int n_chunks, const int32_t* __restrict__ orphans,
                                                 const int32_t* __restrict__ sat, int32_t* __restrict__ unsat_idx) {
    for (int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; o < n_orph; o += (int64_t)gridDim.x * blockDim.x) {
        unsigned long long k = ~0ull;
        int32_t j = INT32_MAX;
        for (int c = 0; c < n_chunks; ++c) take_min(k, j, part[o * n_chunks + c].x, (int32_t)part[o * n_chunks + c].y);
        unsat_idx[orphans[o]] = sat[j];
    }
}

}  // namespace

extern "C" int sqb_sepal_idxs(sqb_ctx* c, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices, int index_bits,
                              const void* data, int data_dtype, int csc, int device_input, uintptr_t producer_stream, const void* xy,
                              int xy_dtype, int64_t stride_row, int64_t stride_col, int xy_device, uintptr_t xy_stream, int max_neighs,
                              int64_t* max_degree, int32_t* sat, int32_t* sat_idx, int32_t* unsat, int32_t* unsat_idx, int64_t* n_sat,
                              int64_t* n_unsat, int* nonfinite) {
    static const char* where = "sqb_sepal_idxs";
    SQB_CHECK(c, SQB_ERR_INVALID, "%s: null ctx", where);
    const SqbGraphArgs ga{n, nnz, indptr, indices, data, indptr_bits, index_bits, data_dtype, csc != 0, device_input, producer_stream};
    SQB_TRY(sqb_check_graph_args(ga, 31, where));
    SQB_CHECK(max_degree && sat && sat_idx && unsat && unsat_idx && n_sat && n_unsat && nonfinite, SQB_ERR_INVALID, "%s: null argument", where);
    SQB_CHECK(nnz == 0 || sqb_graph_value_bytes(data_dtype), SQB_ERR_INVALID, "%s: data_dtype must be 0 (f32), 1 (f64), 3 (i32), 4 (i64) or 5 (bool)",
              where);
    SQB_CHECK(max_neighs >= 1 && max_neighs <= 1024, SQB_ERR_INVALID, "%s: max_neighs=%d out of range [1, 1024]", where, max_neighs);
    SQB_CHECK(xy_dtype == 0 || xy_dtype == 1, SQB_ERR_INVALID, "%s: xy_dtype must be 0 (f32) or 1 (f64)", where);
    SQB_CHECK(xy_device || (xy_dtype == 1 && stride_row == 2 && stride_col == 1), SQB_ERR_INVALID, "%s: host coordinates must be C-contiguous float64",
              where);
    *max_degree = 0, *n_sat = 0, *n_unsat = 0, *nonfinite = 0;
    SQB_CUDA(cudaSetDevice(c->device));
    SqbGraph g(c->stream);
    SQB_TRY(sqb_load_graph(c, ga, SqbGraphForm::STORED, 0, g, where));

    // degrees, and the maximum the caller checks before anything is built
    DevBuf<uint32_t> is_sat(c->stream), rank(c->stream);
    DevBuf<unsigned> counters(c->stream);  // max degree, orphans, non-finite flag
    SQB_TRY(is_sat.alloc(n));
    SQB_TRY(rank.alloc(n));
    SQB_TRY(counters.alloc(3));
    SQB_CUDA(cudaMemsetAsync(counters.p, 0, 3 * sizeof(unsigned), c->stream));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        si_degree<<<sqb_grid_rows(c, n * 32, 256), 256, 0, c->stream>>>(g.ptr.p, g.val.p, n, max_neighs, is_sat.p, counters.p);
        SQB_POST_LAUNCH();
    }
    unsigned most = 0;
    SQB_CUDA(cudaMemcpyAsync(&most, counters.p, sizeof(unsigned), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    *max_degree = most;
    if (most != (unsigned)max_neighs) return SQB_OK;

    // the tables
    uint32_t ns = 0;
    SQB_TRY(sqb_exclusive_scan(c, is_sat.p, rank.p, n, &ns));
    const int64_t nu = n - ns;
    DevBuf<int32_t> d_sat(c->stream), d_sat_idx(c->stream), d_unsat(c->stream), d_unsat_idx(c->stream), orphans(c->stream);
    SQB_TRY(d_sat.alloc(ns));
    SQB_TRY(d_sat_idx.alloc((size_t)ns * max_neighs));
    SQB_TRY(d_unsat.alloc(nu));
    SQB_TRY(d_unsat_idx.alloc(nu));
    SQB_TRY(orphans.alloc(nu));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        si_tables<<<sqb_grid_rows(c, n * 32, 256), 256, 0, c->stream>>>(g.ptr.p, g.col.p, g.val.p, n, max_neighs, is_sat.p, rank.p, d_sat.p, d_sat_idx.p,
                                                                         d_unsat.p, d_unsat_idx.p, orphans.p, counters.p + 1);
        SQB_POST_LAUNCH();
    }
    unsigned n_orph = 0;
    SQB_CUDA(cudaMemcpyAsync(&n_orph, counters.p + 1, sizeof(unsigned), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    g.col.release();
    g.val.release();
    is_sat.release();
    rank.release();

    // the orphans' nearest saturated nodes (ns >= 1: some row has degree max_neighs)
    if (n_orph > 0) {
        DevBuf<double2> spts(c->stream), opts(c->stream);
        SQB_TRY(spts.alloc(ns));
        SQB_TRY(opts.alloc(n_orph));
        const auto gather = [&](const void* p, int code, int64_t sr, int64_t sc) -> int {
            const auto run = [&](auto tx, const int32_t* rows, const int32_t* via, int64_t m, double2* pts) -> int {
                using XT = typename decltype(tx)::type;
                SqbLaunchScope scope(c, SQB_K_MISC);
                si_gather<XT><<<sqb_grid_rows(c, m, 256), 256, 0, c->stream>>>(static_cast<const XT*>(p), sr, sc, rows, via, m, pts, counters.p + 2);
                SQB_POST_LAUNCH();
                return SQB_OK;
            };
            const auto both = [&](auto tx) -> int {
                SQB_TRY(run(tx, d_sat.p, nullptr, ns, spts.p));
                return run(tx, d_unsat.p, orphans.p, n_orph, opts.p);
            };
            return code == 1 ? both(SqbType<double>()) : both(SqbType<float>());
        };
        if (xy_device) {
            SQB_TRY(sqb_read_caller_buffers(c, xy_stream, [&]() -> int {
                SQB_TRY(gather(xy, xy_dtype, stride_row, stride_col));
                SQB_CUDA(cudaStreamSynchronize(c->stream));  // the caller's coordinates are no longer read
                return SQB_OK;
            }));
        } else {
            DevBuf<double> h(c->stream);
            SQB_TRY(h.alloc(2 * n));
            SQB_TRY(sqb_h2d(c, h.p, xy, 2 * n * sizeof(double)));
            SQB_TRY(gather(h.p, 1, 2, 1));
        }
        const int64_t tiles = ceil_div64(n_orph, kOrphTile);
        const int64_t want = ceil_div64(4 * (int64_t)c->sm_count, tiles);  // chunks that fill the GPU with a few blocks per SM
        const int n_chunks = (int)std::max<int64_t>(1, std::min<int64_t>(want, ceil_div64(ns, kMinChunk)));
        const int64_t chunk_len = ceil_div64(ns, n_chunks);
        DevBuf<ulonglong2> part(c->stream);
        SQB_TRY(part.alloc((size_t)n_orph * n_chunks));
        {
            SqbLaunchScope scope(c, SQB_K_MISC);
            si_nearest<<<dim3((unsigned)tiles, (unsigned)n_chunks), kSearchT, 0, c->stream>>>(opts.p, n_orph, spts.p, ns, chunk_len, n_chunks, part.p);
            SQB_POST_LAUNCH();
        }
        {
            SqbLaunchScope scope(c, SQB_K_MISC);
            si_finish<<<sqb_grid_rows(c, n_orph, 256), 256, 0, c->stream>>>(part.p, n_orph, n_chunks, orphans.p, d_sat.p, d_unsat_idx.p);
            SQB_POST_LAUNCH();
        }
    }
    unsigned bad = 0;
    SQB_CUDA(cudaMemcpyAsync(&bad, counters.p + 2, sizeof(unsigned), cudaMemcpyDeviceToHost, c->stream));
    if (ns) SQB_CUDA(cudaMemcpyAsync(sat, d_sat.p, ns * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    if (ns) SQB_CUDA(cudaMemcpyAsync(sat_idx, d_sat_idx.p, (size_t)ns * max_neighs * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    if (nu) SQB_CUDA(cudaMemcpyAsync(unsat, d_unsat.p, nu * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    if (nu) SQB_CUDA(cudaMemcpyAsync(unsat_idx, d_unsat_idx.p, nu * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    *n_sat = ns, *n_unsat = nu, *nonfinite = bad != 0;
    return SQB_OK;
}
