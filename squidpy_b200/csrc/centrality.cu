// centrality.cu — centrality_scores on H100 (sm_90a): group degree, group closeness and local clustering over the
// undirected neighbour graph.
//
// Replaces, in src/squidpy/gr/_nhood.py, _build_graph (:432-454), rustworkx's group_degree_centrality /
// group_closeness_centrality (:309-312) and _local_clustering (:457-491).  Every result is an integer count (the clustering
// coefficient one float64 division of two of them), so nothing depends on summation order.
//
// 1. The caller's graph (host or device) becomes the sorted, duplicate-free CSR of A + Aᵀ without the diagonal and the zero
//    sums: the SYMMETRIC form of caller_graph.cuh.
// 2. Degree and closeness: a bit-parallel BFS from every cluster at once.  Node v holds W = ceil(C / 64) words of visited
//    and frontier bits, one bit per cluster; at level l every node ORs its neighbours' frontier words and masks out what it
//    has visited.  The bits set at level l are the nodes at distance l from the cluster: level 1 is N(S) \ S (the degree
//    numerator), and l * (count at level l) summed over levels is the closeness denominator.  Counts are aggregated per
//    warp (ballot + popc) and per block (shared memory) before one global atomic per cluster and block.
// 3. Clustering: 2 T(v) = sum over u in N(v) of |N(u) ∩ N(v)| by merging sorted neighbour lists (one warp per node, one
//    lane per neighbour), cc[v] = 2 T(v) / (k (k - 1)) in float64, 0 for k < 2.
#include "caller_graph.cuh"

namespace {

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

// The measures on the canonical graph.  Integer outputs are per cluster: reach1 = |N(S) \ S|, dist = sum of hop distances
// from S over the nodes it reaches; levels = the deepest BFS level that reached a node.
int measures_run(sqb_ctx* c, int64_t n, const SqbGraph& g, const int32_t* h_codes, int n_cls, int measures, int64_t* out_reach1,
                 int64_t* out_dist, double* out_cc, int64_t* out_levels) {
    if (measures & 4) {
        DevBuf<double> cc(c->stream);
        SQB_TRY(cc.alloc(n));
        {
            SqbLaunchScope scope(c, SQB_K_MISC);
            cent_clustering<<<sqb_grid_rows(c, n * 32, 256), 256, 0, c->stream>>>(g.ptr.p, g.col.p, n, cc.p);
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
            cent_bfs_level<<<grid, 256, 0, c->stream>>>(g.ptr.p, g.col.p, n, d_full.p, vis.p, fa.p, fb.p, level + 1, dist, reach1, last.p);
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
    const SqbGraphArgs ga{n, nnz, indptr, indices, data, indptr_bits, index_bits, data_dtype, 0, device_input, producer_stream};
    SQB_TRY(sqb_check_graph_args(ga, 30, where));  // 2 nnz records
    SQB_CHECK(codes, SQB_ERR_INVALID, "%s: null argument", where);
    SQB_CHECK(n_cls >= 1 && n_cls <= 64 * 65535, SQB_ERR_INVALID, "%s: n_cls=%d out of range [1, 4194240]", where, n_cls);
    SQB_CHECK(measures >= 1 && measures <= 7, SQB_ERR_INVALID, "%s: measures=%d must be a non-empty mask of 1 | 2 | 4", where, measures);
    SQB_CHECK(!(measures & 1) || out_reach1, SQB_ERR_INVALID, "%s: null out_reach1", where);
    SQB_CHECK(!(measures & 2) || out_dist, SQB_ERR_INVALID, "%s: null out_dist", where);
    SQB_CHECK(!(measures & 4) || out_cc, SQB_ERR_INVALID, "%s: null out_cc", where);
    SQB_CHECK(int_bits == 8 || int_bits == 16 || int_bits == 32 || int_bits == 64, SQB_ERR_INVALID, "%s: int_bits must be 8, 16, 32 or 64", where);
    SQB_CHECK(nnz == 0 || sqb_graph_value_bytes(data_dtype), SQB_ERR_INVALID, "%s: data_dtype must be 0 (f32), 1 (f64), 3 (i32), 4 (i64) or 5 (bool)", where);
    for (int64_t v = 0; v < n; ++v)
        SQB_CHECK(codes[v] >= -1 && codes[v] < n_cls, SQB_ERR_INVALID, "%s: codes[%lld]=%d out of range [-1, %d)", where, (long long)v, codes[v], n_cls);
    SQB_CUDA(cudaSetDevice(c->device));
    SqbGraph g(c->stream);
    SQB_TRY(sqb_load_graph(c, ga, SqbGraphForm::SYMMETRIC, int_bits, g, where));
    return measures_run(c, n, g, codes, n_cls, measures, out_reach1, out_dist, out_cc, out_levels);
}
