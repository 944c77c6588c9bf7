// centrality.cu — centrality_scores on H100 (sm_90a): group degree, group closeness and local clustering over the
// undirected neighbour graph.
//
// Replaces, in src/squidpy/gr/_nhood.py, _build_graph (:432-454), rustworkx's group_degree_centrality /
// group_closeness_centrality (:309-312) and _local_clustering (:457-491).  Every result is an integer count (the clustering
// coefficient one float64 division of two of them), so nothing depends on summation order.
//
// 1. Canonicalise (one path for host and device input: a host CSR is uploaded as given first).  The graph is A + Aᵀ with
//    values summed in A's dtype, diagonal and zero sums dropped.  Every stored entry (i -> j), i != j, gives two records,
//    (i, j) from A and (j, i) from Aᵀ, keyed (row << 33 | col << 1 | from_transpose) and radix-sorted with the entry index
//    as payload (stable: storage order within a key).  The head of each (row, col) run sums the run's values the way scipy's
//    csr_plus_csr does — A's duplicates in storage order, Aᵀ's likewise, then the two partial sums — and keeps the pair when
//    the sum is non-zero (NaN is non-zero).  The kept records, compacted, are the sorted duplicate-free symmetric CSR.
// 2. Degree and closeness: a bit-parallel BFS from every cluster at once.  Node v holds W = ceil(C / 64) words of visited
//    and frontier bits, one bit per cluster; at level l every node ORs its neighbours' frontier words and masks out what it
//    has visited.  The bits set at level l are the nodes at distance l from the cluster: level 1 is N(S) \ S (the degree
//    numerator), and l * (count at level l) summed over levels is the closeness denominator.  Counts are aggregated per
//    warp (ballot + popc) and per block (shared memory) before one global atomic per cluster and block.
// 3. Clustering: 2 T(v) = sum over u in N(v) of |N(u) ∩ N(v)| by merging sorted neighbour lists (one warp per node, one
//    lane per neighbour), cc[v] = 2 T(v) / (k (k - 1)) in float64, 0 for k < 2.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace {

constexpr uint64_t kDiagKey = ~0ull;  // a diagonal entry: sorts after every record and is never kept

// Two records per stored entry (one warp per row).  A column index outside [0, n) raises bit 2 of *err.
template <typename IP, typename II>
__global__ void __launch_bounds__(256) cent_expand(const IP* __restrict__ indptr, const II* __restrict__ indices, int64_t n,
                                                   uint64_t* __restrict__ keys, uint32_t* __restrict__ ids, unsigned* __restrict__ err) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    unsigned bad = 0;
    for (int64_t i = warp; i < n; i += nwarps) {
        const int64_t beg = (int64_t)indptr[i], end = (int64_t)indptr[i + 1];
        for (int64_t e = beg + lane; e < end; e += 32) {
            const int64_t j = (int64_t)indices[e];
            const bool ok = j >= 0 && j < n;
            bad |= !ok;
            const bool edge = ok && j != i;
            const uint64_t k0 = edge ? ((uint64_t)i << 33) | ((uint64_t)j << 1) : kDiagKey;
            const uint64_t k1 = edge ? ((uint64_t)j << 33) | ((uint64_t)i << 1) | 1u : kDiagKey;
            reinterpret_cast<ulonglong2*>(keys)[e] = make_ulonglong2(k0, k1);
            reinterpret_cast<uint2*>(ids)[e] = make_uint2((uint32_t)e, (uint32_t)e);
        }
    }
    if (bad) atomicOr(err, 2u);
}

// The sum of A's dtype.  Integers wrap at int_bits (the caller's dtype width; narrower integers arrive widened), bool
// (one byte) sums as logical or, floats in their own precision.
template <typename VT>
struct ValueSum {
    using Acc = typename std::conditional<std::is_floating_point<VT>::value, VT, uint64_t>::type;
    __device__ static Acc zero() { return (Acc)0; }
    __device__ static Acc add(Acc a, VT v) {
        if constexpr (std::is_same<VT, uint8_t>::value)
            return a | (uint64_t)(v != 0);
        else if constexpr (std::is_floating_point<VT>::value)
            return a + v;
        else
            return a + (uint64_t)(int64_t)v;
    }
    __device__ static Acc combine(Acc a, Acc b) {
        if constexpr (std::is_same<VT, uint8_t>::value)
            return a | b;
        else
            return a + b;
    }
    __device__ static bool nonzero(Acc s, int int_bits) {
        if constexpr (std::is_floating_point<VT>::value)
            return s != (Acc)0;  // NaN != 0
        else
            return int_bits >= 64 ? s != 0 : (s & ((1ull << int_bits) - 1)) != 0;
    }
};

// keep[p] = 1 at the head of a (row, col) run whose summed value is non-zero.
template <typename VT>
__global__ void __launch_bounds__(256) cent_reduce(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ ids,
                                                   const VT* __restrict__ data, int64_t m, int int_bits, uint32_t* __restrict__ keep) {
    using S = ValueSum<VT>;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < m; p += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t k = keys[p];
        uint32_t flag = 0;
        if (k != kDiagKey && (p == 0 || (keys[p - 1] >> 1) != (k >> 1))) {
            typename S::Acc sa = S::zero(), st = S::zero();  // entries of A, entries of its transpose
            for (int64_t q = p; q < m && (keys[q] >> 1) == (k >> 1); ++q) {
                if (keys[q] & 1)
                    st = S::add(st, data[ids[q]]);
                else
                    sa = S::add(sa, data[ids[q]]);
            }
            flag = S::nonzero(S::combine(sa, st), int_bits);
        }
        keep[p] = flag;
    }
}

// Compaction of the kept heads: column and row of every kept record at its rank.
__global__ void __launch_bounds__(256) cent_scatter(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ keep,
                                                    const uint32_t* __restrict__ rank, int64_t m, int32_t* __restrict__ col,
                                                    int32_t* __restrict__ row) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < m; p += (int64_t)gridDim.x * blockDim.x) {
        if (!keep[p]) continue;
        const uint64_t k = keys[p];
        col[rank[p]] = (int32_t)((k >> 1) & 0xFFFFFFFFull);
        row[rank[p]] = (int32_t)(k >> 33);
    }
}

// indptr of the canonical CSR from the sorted rows of its e records: indptr[r] = first record of row >= r.
__global__ void __launch_bounds__(256) cent_indptr(const int32_t* __restrict__ row, int64_t e, int64_t n, uint32_t* __restrict__ indptr) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p <= e; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = p < e ? row[p] : n;
        const int64_t rp = p == 0 ? -1 : row[p - 1];
        for (int64_t q = rp + 1; q <= r; ++q) indptr[q] = (uint32_t)p;
    }
}

// Level 0: every labelled node is visited by, and on the frontier of, its own cluster.  Word-major: word w of node v at
// w * n + v.
__global__ void __launch_bounds__(256) cent_bfs_init(const int32_t* __restrict__ codes, int64_t n, int W, uint64_t* __restrict__ vis,
                                                     uint64_t* __restrict__ front) {
    for (int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; v < n; v += (int64_t)gridDim.x * blockDim.x) {
        const int32_t c = codes[v];
        for (int w = 0; w < W; ++w) {
            const uint64_t bit = (c >= 0 && (c >> 6) == w) ? 1ull << (c & 63) : 0ull;
            vis[(int64_t)w * n + v] = bit;
            front[(int64_t)w * n + v] = bit;
        }
    }
}

// One BFS level for word blockIdx.y.  A node that every non-empty cluster of the word has reached (full) reads nothing.
// Counts of newly set bits: ballot + popc per warp, shared-memory sums per block, one global atomic per (block, cluster).
// *last: the deepest level that set a bit.
__global__ void __launch_bounds__(256) cent_bfs_level(const uint32_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                                                      int64_t n, const uint64_t* __restrict__ full, uint64_t* __restrict__ vis,
                                                      const uint64_t* __restrict__ front, uint64_t* __restrict__ next, int level,
                                                      unsigned long long* __restrict__ dist, unsigned long long* __restrict__ reach1,
                                                      unsigned* __restrict__ last) {
    __shared__ unsigned s_cnt[64];
    if (threadIdx.x < 64) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const int w = blockIdx.y;
    const uint64_t fw = full[w];
    const uint64_t* fr = front + (int64_t)w * n;
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    // warp-uniform trip count: lanes past n carry no bits
    for (int64_t base = blockIdx.x * (int64_t)blockDim.x + (threadIdx.x & ~31); base < n; base += stride) {
        const int64_t v = base + lane;
        uint64_t nw = 0;
        if (v < n) {
            const uint64_t vw = vis[(int64_t)w * n + v];
            if ((vw & fw) != fw) {
                uint64_t acc = 0;
                for (uint32_t a = indptr[v], b = indptr[v + 1]; a < b; ++a) acc |= fr[indices[a]];
                nw = acc & ~vw;
                if (nw) vis[(int64_t)w * n + v] = vw | nw;
            }
            next[(int64_t)w * n + v] = nw;
        }
        const uint32_t lo = __reduce_or_sync(0xFFFFFFFFu, (uint32_t)nw), hi = __reduce_or_sync(0xFFFFFFFFu, (uint32_t)(nw >> 32));
        for (uint64_t bits = ((uint64_t)hi << 32) | lo; bits; bits &= bits - 1) {
            const int b = __ffsll((long long)bits) - 1;
            const unsigned cnt = __popc(__ballot_sync(0xFFFFFFFFu, (nw >> b) & 1));
            if (lane == 0) atomicAdd(&s_cnt[b], cnt);
        }
    }
    __syncthreads();
    if (threadIdx.x < 64) {
        const unsigned cnt = s_cnt[threadIdx.x];
        if (cnt) {
            const int64_t c = (int64_t)w * 64 + threadIdx.x;
            atomicAdd(&dist[c], (unsigned long long)level * cnt);
            if (level == 1) atomicAdd(&reach1[c], (unsigned long long)cnt);
            atomicMax(last, (unsigned)level);
        }
    }
}

// cc[v] = 2 T(v) / (k (k - 1)) (0 when k < 2): one warp per node, one lane per neighbour u merging N(u) with N(v).
__global__ void __launch_bounds__(256) cent_clustering(const uint32_t* __restrict__ indptr, const int32_t* __restrict__ indices, int64_t n,
                                                       double* __restrict__ cc) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t v = warp; v < n; v += nwarps) {
        const uint32_t vs = indptr[v], ve = indptr[v + 1];
        const int64_t k = (int64_t)ve - vs;
        unsigned long long t2 = 0;
        if (k >= 2) {
            for (uint32_t a = vs + lane; a < ve; a += 32) {
                const int32_t u = indices[a];
                uint32_t i = vs, j = indptr[u];
                const uint32_t ue = indptr[u + 1];
                while (i < ve && j < ue) {
                    const int32_t x = indices[i], y = indices[j];
                    t2 += x == y;
                    i += x <= y;
                    j += y <= x;
                }
            }
            for (int o = 16; o; o >>= 1) t2 += __shfl_xor_sync(0xFFFFFFFFu, t2, o);
        }
        if (lane == 0) cc[v] = k < 2 ? 0.0 : (double)t2 / (double)(k * (k - 1));
    }
}

// Value bytes of the ABI's dtype codes (DTYPE_CODES of _device.py plus 5 = bool); 0 for codes the function does not take.
int value_bytes(int code) {
    switch (code) {
        case 0: return 4;
        case 1: return 8;
        case 3: return 4;
        case 4: return 8;
        case 5: return 1;
    }
    return 0;
}

struct Canon {
    DevBuf<uint32_t> indptr;
    DevBuf<int32_t> indices;
    int64_t e = 0;
    explicit Canon(cudaStream_t s) : indptr(s), indices(s) {}
};

template <typename IP, typename II>
int canonicalise(sqb_ctx* c, int64_t n, int64_t nnz, const void* indptr, const void* indices, const void* data, int data_dtype,
                 int int_bits, Canon& out) {
    static const char* where = "sqb_centrality_scores";
    const IP* ip = reinterpret_cast<const IP*>(indptr);
    const II* ix = reinterpret_cast<const II*>(indices);
    SQB_TRY(sqb_check_indptr(c, SQB_K_MISC, ip, n, nnz, nullptr, where));
    SQB_TRY(out.indptr.alloc(n + 1));
    if (nnz == 0) {
        SQB_CUDA(cudaMemsetAsync(out.indptr.p, 0, (n + 1) * sizeof(uint32_t), c->stream));
        SQB_TRY(out.indices.alloc(1));
        out.e = 0;
        return SQB_OK;
    }
    const int64_t m = 2 * nnz;
    DevBuf<uint64_t> keys(c->stream), keys_s(c->stream);
    DevBuf<uint32_t> ids(c->stream), ids_s(c->stream), keep(c->stream), rank(c->stream);
    DevBuf<unsigned> err(c->stream);
    SQB_TRY(keys.alloc(m));
    SQB_TRY(keys_s.alloc(m));
    SQB_TRY(ids.alloc(m));
    SQB_TRY(ids_s.alloc(m));
    SQB_TRY(err.alloc(1));
    SQB_CUDA(cudaMemsetAsync(err.p, 0, sizeof(unsigned), c->stream));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        cent_expand<IP, II><<<sqb_grid_rows(c, n * 32, 256), 256, 0, c->stream>>>(ip, ix, n, keys.p, ids.p, err.p);
        SQB_POST_LAUNCH();
    }
    int nbits = 1;
    while (nbits < 31 && ((int64_t)1 << nbits) < n) ++nbits;
    const int end_bit = 33 + nbits;  // (row < 2^nbits) << 33 | col << 1 | dir; the diagonal key has all these bits set
    size_t tmp_bytes = 0, scan_bytes = 0;
    SQB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys.p, keys_s.p, ids.p, ids_s.p, (int)m, 0, end_bit, c->stream));
    SQB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, keep.p, rank.p, (int)m, c->stream));
    DevBuf<uint8_t> tmp(c->stream);
    SQB_TRY(tmp.alloc(tmp_bytes > scan_bytes ? tmp_bytes : scan_bytes));
    SQB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, keys.p, keys_s.p, ids.p, ids_s.p, (int)m, 0, end_bit, c->stream));
    keys.release();
    ids.release();
    SQB_TRY(keep.alloc(m));
    SQB_TRY(rank.alloc(m));
    SQB_TRY(sqb_dispatch_value<true>(data_dtype, where, "data_dtype", [&](auto vt) -> int {
        using VT = typename decltype(vt)::type;
        if constexpr (std::is_same<VT, __half>::value) {
            sqb_set_error("%s: float16 graph values are not supported", where);
            return SQB_ERR_INVALID;
        } else {
            SqbLaunchScope scope(c, SQB_K_MISC);
            cent_reduce<VT><<<sqb_grid_rows(c, m, 256), 256, 0, c->stream>>>(keys_s.p, ids_s.p, reinterpret_cast<const VT*>(data), m,
                                                                              int_bits, keep.p);
            SQB_POST_LAUNCH();
            return SQB_OK;
        }
    }));
    SQB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, scan_bytes, keep.p, rank.p, (int)m, c->stream));
    uint32_t tail[2] = {0, 0};
    unsigned flag = 0;
    SQB_CUDA(cudaMemcpyAsync(&tail[0], rank.p + m - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaMemcpyAsync(&tail[1], keep.p + m - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaMemcpyAsync(&flag, err.p, sizeof(unsigned), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    SQB_CHECK(!(flag & 2u), SQB_ERR_INVALID, "%s: column index out of range [0, %lld)", where, (long long)n);
    out.e = (int64_t)tail[0] + tail[1];
    SQB_TRY(out.indices.alloc(out.e));
    DevBuf<int32_t> rows(c->stream);
    SQB_TRY(rows.alloc(out.e));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        cent_scatter<<<sqb_grid_rows(c, m, 256), 256, 0, c->stream>>>(keys_s.p, keep.p, rank.p, m, out.indices.p, rows.p);
        SQB_POST_LAUNCH();
    }
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        cent_indptr<<<sqb_grid_rows(c, out.e + 1, 256), 256, 0, c->stream>>>(rows.p, out.e, n, out.indptr.p);
        SQB_POST_LAUNCH();
    }
    return SQB_OK;
}

// The measures on the canonical graph.  Integer outputs are per cluster: reach1 = |N(S) \ S|, dist = sum of hop distances
// from S over the nodes it reaches; levels = the deepest BFS level that reached a node.
int measures_run(sqb_ctx* c, int64_t n, const Canon& g, const int32_t* h_codes, int n_cls, int measures, int64_t* out_reach1,
                 int64_t* out_dist, double* out_cc, int64_t* out_levels) {
    if (measures & 4) {
        DevBuf<double> cc(c->stream);
        SQB_TRY(cc.alloc(n));
        {
            SqbLaunchScope scope(c, SQB_K_MISC);
            cent_clustering<<<sqb_grid_rows(c, n * 32, 256), 256, 0, c->stream>>>(g.indptr.p, g.indices.p, n, cc.p);
            SQB_POST_LAUNCH();
        }
        SQB_CUDA(cudaMemcpyAsync(out_cc, cc.p, n * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaStreamSynchronize(c->stream));
    }
    if (!(measures & 3)) return SQB_OK;
    const int W = (n_cls + 63) / 64;
    std::vector<uint64_t> full(W, 0);
    for (int64_t v = 0; v < n; ++v)
        if (h_codes[v] >= 0) full[h_codes[v] >> 6] |= 1ull << (h_codes[v] & 63);
    DevBuf<int32_t> codes(c->stream);
    DevBuf<uint64_t> vis(c->stream), fa(c->stream), fb(c->stream), d_full(c->stream);
    DevBuf<unsigned long long> sums(c->stream);  // dist [64 W] | reach1 [64 W]
    DevBuf<unsigned> last(c->stream);
    SQB_TRY(codes.alloc(n));
    SQB_TRY(vis.alloc((size_t)W * n));
    SQB_TRY(fa.alloc((size_t)W * n));
    SQB_TRY(fb.alloc((size_t)W * n));
    SQB_TRY(d_full.alloc(W));
    SQB_TRY(sums.alloc((size_t)128 * W));
    SQB_TRY(last.alloc(1));
    SQB_CUDA(cudaMemcpyAsync(codes.p, h_codes, n * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    SQB_CUDA(cudaMemcpyAsync(d_full.p, full.data(), W * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
    SQB_CUDA(cudaMemsetAsync(sums.p, 0, (size_t)128 * W * sizeof(unsigned long long), c->stream));
    SQB_CUDA(cudaMemsetAsync(last.p, 0, sizeof(unsigned), c->stream));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        cent_bfs_init<<<sqb_grid_rows(c, n, 256), 256, 0, c->stream>>>(codes.p, n, W, vis.p, fa.p);
        SQB_POST_LAUNCH();
    }
    const dim3 grid(sqb_grid_rows(c, n, 256), (unsigned)W);
    unsigned long long* dist = sums.p;
    unsigned long long* reach1 = sums.p + (size_t)64 * W;
    // Levels are launched in batches between read-backs of the deepest level reached: a level after the last one that set
    // a bit finds an empty frontier and changes nothing.  Degree alone needs level 1 only.
    const int max_levels = (measures & 2) ? (int)(n < 0x7FFFFFFF ? n : 0x7FFFFFFF) : 1;
    int level = 0, batch = 8;
    unsigned reached = 0;
    while (level < max_levels) {
        const int stop = level + batch < max_levels ? level + batch : max_levels;
        for (; level < stop; ++level) {
            SqbLaunchScope scope(c, SQB_K_MISC);
            cent_bfs_level<<<grid, 256, 0, c->stream>>>(g.indptr.p, g.indices.p, n, d_full.p, vis.p, fa.p, fb.p, level + 1, dist, reach1, last.p);
            SQB_POST_LAUNCH();
            std::swap(fa.p, fb.p);
        }
        SQB_CUDA(cudaMemcpyAsync(&reached, last.p, sizeof(unsigned), cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaStreamSynchronize(c->stream));
        if ((int)reached < level) break;
        if (batch < 256) batch *= 2;
    }
    std::vector<unsigned long long> h((size_t)128 * W);
    SQB_CUDA(cudaMemcpyAsync(h.data(), sums.p, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    for (int k = 0; k < n_cls; ++k) {
        if (out_dist) out_dist[k] = (int64_t)h[k];
        if (out_reach1) out_reach1[k] = (int64_t)h[(size_t)64 * W + k];
    }
    if (out_levels) *out_levels = (measures & 2) ? (int64_t)reached : -1;
    return SQB_OK;
}

}  // namespace

extern "C" int sqb_centrality_scores(sqb_ctx* c, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices,
                                     int index_bits, const void* data, int data_dtype, int int_bits, int device_input,
                                     const int32_t* codes, int n_cls, int measures, int64_t* out_reach1, int64_t* out_dist,
                                     double* out_cc, int64_t* out_levels, uintptr_t producer_stream) {
    static const char* where = "sqb_centrality_scores";
    SQB_CHECK(c, SQB_ERR_INVALID, "%s: null ctx", where);
    SQB_CHECK(n >= 1 && n < 0x7FFFFFFFLL, SQB_ERR_INVALID, "%s: n=%lld out of range [1, 2^31 - 1)", where, (long long)n);
    SQB_CHECK(nnz >= 0 && nnz < (1LL << 30), SQB_ERR_INVALID, "%s: nnz=%lld out of range [0, 2^30)", where, (long long)nnz);
    SQB_CHECK(indptr && ((indices && data) || nnz == 0) && codes, SQB_ERR_INVALID, "%s: null argument", where);
    SQB_CHECK(n_cls >= 1 && n_cls <= 64 * 65535, SQB_ERR_INVALID, "%s: n_cls=%d out of range [1, 4194240]", where, n_cls);
    SQB_CHECK(measures >= 1 && measures <= 7, SQB_ERR_INVALID, "%s: measures=%d must be a non-empty mask of 1 | 2 | 4", where, measures);
    SQB_CHECK(!(measures & 1) || out_reach1, SQB_ERR_INVALID, "%s: null out_reach1", where);
    SQB_CHECK(!(measures & 2) || out_dist, SQB_ERR_INVALID, "%s: null out_dist", where);
    SQB_CHECK(!(measures & 4) || out_cc, SQB_ERR_INVALID, "%s: null out_cc", where);
    SQB_CHECK(int_bits == 8 || int_bits == 16 || int_bits == 32 || int_bits == 64, SQB_ERR_INVALID, "%s: int_bits must be 8, 16, 32 or 64", where);
    SQB_CHECK(nnz == 0 || value_bytes(data_dtype), SQB_ERR_INVALID, "%s: data_dtype must be 0 (f32), 1 (f64), 3 (i32), 4 (i64) or 5 (bool)", where);
    for (int64_t v = 0; v < n; ++v)
        SQB_CHECK(codes[v] >= -1 && codes[v] < n_cls, SQB_ERR_INVALID, "%s: codes[%lld]=%d out of range [-1, %d)", where, (long long)v, codes[v], n_cls);
    SQB_CUDA(cudaSetDevice(c->device));
    Canon g(c->stream);
    const auto canon = [&](const void* ip, const void* ix, const void* dv) {
        return sqb_dispatch_index(indptr_bits, index_bits, where, [&](auto tp, auto tx) {
            return canonicalise<typename decltype(tp)::type, typename decltype(tx)::type>(c, n, nnz, ip, ix, dv, data_dtype, int_bits, g);
        });
    };
    if (device_input) {
        SQB_TRY(sqb_read_caller_buffers(c, producer_stream, [&]() -> int {
            SQB_TRY(canon(indptr, indices, data));
            SQB_CUDA(cudaStreamSynchronize(c->stream));  // the caller's buffers are no longer read
            return SQB_OK;
        }));
    } else {
        SQB_CHECK(indptr_bits == 32 || indptr_bits == 64, SQB_ERR_INVALID, "%s: indptr_bits / index_bits must be 32 or 64", where);
        SQB_CHECK(index_bits == 32 || index_bits == 64, SQB_ERR_INVALID, "%s: indptr_bits / index_bits must be 32 or 64", where);
        DevBuf<uint8_t> d_ip(c->stream), d_ix(c->stream), d_v(c->stream);
        const size_t ip_bytes = (size_t)(n + 1) * (indptr_bits / 8), ix_bytes = (size_t)nnz * (index_bits / 8),
                     v_bytes = (size_t)nnz * value_bytes(data_dtype);
        SQB_TRY(d_ip.alloc(ip_bytes));
        SQB_TRY(d_ix.alloc(ix_bytes));
        SQB_TRY(d_v.alloc(v_bytes));
        SQB_TRY(sqb_h2d(c, d_ip.p, indptr, ip_bytes));
        if (nnz > 0) {
            SQB_TRY(sqb_h2d(c, d_ix.p, indices, ix_bytes));
            SQB_TRY(sqb_h2d(c, d_v.p, data, v_bytes));
        }
        SQB_TRY(canon(d_ip.p, d_ix.p, d_v.p));
    }
    return measures_run(c, n, g, codes, n_cls, measures, out_reach1, out_dist, out_cc, out_levels);
}
