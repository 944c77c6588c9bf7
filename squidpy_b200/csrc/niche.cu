// niche.cu — the embeddings of calculate_niche on H100 (sm_90a): neighbourhood profiles, UTAG feature propagation and
// CellCharter hop aggregates.  Everything after the embedding (scaling, PCA, the kNN graph, leiden, the GMM) stays with
// scanpy / scikit-learn, as in the reference.
//
// Replaces, in src/squidpy/gr/_niche.py:
//   sqb_niche_profile     <- _NhoodProfileEmbedder._calculate_neighborhood_profile and the hop loop of get_embedding
//                            (:1117-1169, :1176-1214)
//   sqb_niche_aggregate   <- _UtagEmbedder.get_embedding up to sc.tl.pca (:1259-1260), and _CellcharterEmbedder.get_embedding
//                            up to sc.tl.pca (:1336-1355) with _setdiag, _hop, _normalize and _aggregate (:1002-1054)
//
// Graph input (host or device CSR / CSC, int32 / int64 indices, float32 / float64 / int32 / int64 values) becomes a
// device CSR in the STORED or CANONICAL form of caller_graph.cuh.  A float32 graph's values are float32 numbers and every
// operation on them rounds to float32.
//
// Arithmetic is written as separate multiplies and adds (__fmul_rn / __fadd_rn, __dmul_rn / __dadd_rn): scipy's sparse
// products do not contract to FMA, and the float32 results are bit-exact only in their order.
#include <cub/device/device_segmented_sort.cuh>

#include <algorithm>

#include "caller_graph.cuh"

namespace {

// The graph checks of both entry points.  Boolean graphs are refused: scipy multiplies and adds them as logical and / or,
// which path sums do not reproduce.
int check_graph(const SqbGraphArgs& a, const char* where) {
    SQB_TRY(sqb_check_graph_args(a, 31, where));
    SQB_CHECK(a.nnz == 0 || (a.data_dtype != 5 && sqb_graph_value_bytes(a.data_dtype)), SQB_ERR_INVALID,
              "%s: data_dtype must be 0 (f32), 1 (f64), 3 (i32) or 4 (i64)", where);
    return SQB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Sparse x dense products
// ---------------------------------------------------------------------------------------------------------------------
// Row i of Y (columns [0, m) at out + i * ld): sum over the stored entries e of row i, in storage order (reverse: backwards),
// of v_e * X[col_e, :], accumulated in TA, v_e = val[e] (or rscale[i] when val is null).  skip_zero drops entries whose
// value is 0, as scipy drops zero products from a sparse product.  VAR: the output is N (X∘X) - (N X)², X∘X squared in TX.
// One warp per row, one lane per column of a 32-column slice.
template <typename TA, typename TX, typename TO, bool VAR>
__global__ void __launch_bounds__(256) niche_spmm(const uint32_t* __restrict__ ptr, const int32_t* __restrict__ col,
                                                  const double* __restrict__ val, const double* __restrict__ rscale, int reverse,
                                                  int skip_zero, const TX* __restrict__ X, int64_t n, int64_t m, TO* __restrict__ out,
                                                  int64_t ld) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = warp; i < n; i += nwarps) {
        const int64_t beg = ptr[i], end = ptr[i + 1];
        const TA rs = rscale ? (TA)rscale[i] : (TA)0;
        for (int64_t c0 = 0; c0 < m; c0 += 32) {
            const int64_t cc = c0 + lane;
            const bool on = cc < m;
            TA acc = (TA)0, acc2 = (TA)0;
            for (int64_t t = 0; t < end - beg; ++t) {
                const int64_t e = reverse ? end - 1 - t : beg + t;
                const TA v = val ? (TA)val[e] : rs;
                if (skip_zero && v == (TA)0) continue;
                if (on) {
                    const TX x = X[(int64_t)col[e] * m + cc];
                    acc = add_rn<TA>(acc, mul_rn<TA>(v, (TA)x));
                    if constexpr (VAR) acc2 = add_rn<TA>(acc2, mul_rn<TA>(v, (TA)mul_rn<TX>(x, x)));
                }
            }
            if (on) {
                if constexpr (VAR)
                    out[i * ld + cc] = (TO)add_rn<TA>(acc2, -mul_rn<TA>(acc, acc));
                else
                    out[i * ld + cc] = (TO)acc;
            }
        }
    }
}

template <typename TX, typename TO>
__global__ void __launch_bounds__(256) niche_copy_block(const TX* __restrict__ X, int64_t n, int64_t m, TO* __restrict__ out, int64_t ld) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n * m; p += (int64_t)gridDim.x * blockDim.x)
        out[(p / m) * ld + p % m] = (TO)X[p];
}

// A CSR X as a dense row-major n x m matrix (zeroed first); duplicates add up in storage order.
template <typename TX, typename IP, typename II>
__global__ void __launch_bounds__(256) niche_densify(const IP* __restrict__ ip, const II* __restrict__ ix, const TX* __restrict__ xv, int64_t n,
                                                     int64_t m, TX* __restrict__ X, unsigned* __restrict__ err) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        for (int64_t e = (int64_t)ip[i]; e < (int64_t)ip[i + 1]; ++e) {
            const int64_t j = (int64_t)ix[e];
            if (j < 0 || j >= m) {
                atomicOr(err, 2u);
                continue;
            }
            X[i * m + j] = add_rn<TX>(X[i * m + j], xv[e]);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Neighbourhood profiles
// ---------------------------------------------------------------------------------------------------------------------
// P[i, c] = sum over the row's entries j (ascending) with codes[j] = c of A[i, j], in float64.  One thread per row.
__global__ void __launch_bounds__(256) niche_profile_hop1(const uint32_t* __restrict__ ptr, const int32_t* __restrict__ col,
                                                          const double* __restrict__ val, const int32_t* __restrict__ codes, int64_t n,
                                                          int C, double* __restrict__ P) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        double* row = P + i * C;
        for (int c = 0; c < C; ++c) row[c] = 0.0;
        for (uint32_t e = ptr[i]; e < ptr[i + 1]; ++e) {
            const int32_t c = codes[col[e]];
            if (c >= 0) row[c] = __dadd_rn(row[c], val[e]);
        }
    }
}

// Hop k's share of the embedding: p = P (abs) or P / (row total) with NaN -> 0; out = p (one hop), w * p (first of
// several), out + w * p (later hops); the last hop divides by wsum unless abs.
__global__ void __launch_bounds__(256) niche_profile_fold(const double* __restrict__ P, int64_t n, int C, int abs_nhood, int k,
                                                          int distance, double w, double wsum, double* __restrict__ out) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double* p = P + i * C;
        double* o = out + i * C;
        double t = 0.0;
        if (!abs_nhood)
            for (int c = 0; c < C; ++c)
                if (p[c] == p[c]) t = __dadd_rn(t, p[c]);  // pandas' sum skips NaN
        for (int c = 0; c < C; ++c) {
            double v = p[c];
            if (!abs_nhood) {
                v = __ddiv_rn(v, t);
                if (v != v) v = 0.0;
            }
            if (distance > 1) {
                v = __dmul_rn(w, v);
                if (k > 0) v = __dadd_rn(o[c], v);
                if (k == distance - 1 && !abs_nhood) v = __ddiv_rn(v, wsum);
            }
            o[c] = v;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// UTAG: sklearn.preprocessing.normalize(A, norm="l1", axis=1)
// ---------------------------------------------------------------------------------------------------------------------
// Row sum of |v| in float64 in storage order; a row summing to 0 is left as it is; v / sum in float64, rounded to the
// graph's value type (float32 rows: the float64 quotient rounded once to float32).
template <typename W>
__global__ void __launch_bounds__(256) niche_l1_rows(const uint32_t* __restrict__ ptr, double* __restrict__ val, int64_t n) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        double s = 0.0;
        for (uint32_t e = ptr[i]; e < ptr[i + 1]; ++e) s = __dadd_rn(s, fabs(val[e]));
        if (s == 0.0) continue;
        for (uint32_t e = ptr[i]; e < ptr[i + 1]; ++e) val[e] = (double)(W)__ddiv_rn(val[e], s);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// CellCharter hops
// ---------------------------------------------------------------------------------------------------------------------
// hop_1 (FILL = 0: counts, 1: entries) from the canonical A: the diagonal and zero values removed (_setdiag(A, 0)).
// visited_0: the canonical A with its diagonal set to 1, inserted where absent (_setdiag(A, 1)).
template <bool FILL>
__global__ void __launch_bounds__(256) niche_hop1(const uint32_t* __restrict__ ptr, const int32_t* __restrict__ col,
                                                  const double* __restrict__ val, int64_t n, uint32_t* __restrict__ h_cnt,
                                                  uint32_t* __restrict__ v_cnt, const uint32_t* __restrict__ h_ptr,
                                                  const uint32_t* __restrict__ v_ptr, int32_t* __restrict__ h_col,
                                                  double* __restrict__ h_val, int32_t* __restrict__ v_col, double* __restrict__ v_val) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        uint32_t nh = 0, nv = 0;
        bool diag_done = false;
        for (uint32_t e = ptr[i]; e < ptr[i + 1]; ++e) {
            const int32_t j = col[e];
            if (!diag_done && j >= i) {
                if (FILL) v_col[v_ptr[i] + nv] = (int32_t)i, v_val[v_ptr[i] + nv] = 1.0;
                ++nv;
                diag_done = true;
            }
            if (j == i) continue;
            if (FILL) v_col[v_ptr[i] + nv] = j, v_val[v_ptr[i] + nv] = val[e];
            ++nv;
            if (val[e] != 0.0) {
                if (FILL) h_col[h_ptr[i] + nh] = j, h_val[h_ptr[i] + nh] = val[e];
                ++nh;
            }
        }
        if (!diag_done) {
            if (FILL) v_col[v_ptr[i] + nv] = (int32_t)i, v_val[v_ptr[i] + nv] = 1.0;
            ++nv;
        }
        if (!FILL) h_cnt[i] = nh, v_cnt[i] = nv;
    }
}

// numpy's pairwise float sum (the add reduction of np.add.reduceat, which _normalize's sum(axis=1) is): fewer than 8
// terms sequentially from -0.0, up to 128 in eight interleaved partial sums, beyond that halves at a multiple of 8.
template <typename W>
__device__ W pairwise_sum(const double* a, int64_t n) {
    if (n < 8) {
        W r = (W)-0.0;
        for (int64_t i = 0; i < n; ++i) r = add_rn<W>(r, (W)a[i]);
        return r;
    }
    if (n <= 128) {
        W r[8];
        for (int j = 0; j < 8; ++j) r[j] = (W)a[j];
        int64_t i = 8;
        for (; i < n - (n % 8); i += 8)
            for (int j = 0; j < 8; ++j) r[j] = add_rn<W>(r[j], (W)a[i + j]);
        W res = add_rn<W>(add_rn<W>(add_rn<W>(r[0], r[1]), add_rn<W>(r[2], r[3])), add_rn<W>(add_rn<W>(r[4], r[5]), add_rn<W>(r[6], r[7])));
        for (; i < n; ++i) res = add_rn<W>(res, (W)a[i]);
        return res;
    }
    int64_t n2 = n / 2;
    n2 -= n2 % 8;
    return add_rn<W>(pairwise_sum<W>(a, n2), pairwise_sum<W>(a + n2, n - n2));
}

// _normalize(hop_1): deg = a_0 + pairwise(a_1..) in the value type, dinv = 1 / deg with +inf -> 0, entries dinv * a_ij.
template <typename W>
__global__ void __launch_bounds__(256) niche_norm_hop1(const uint32_t* __restrict__ ptr, double* __restrict__ val, int64_t n) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t b = ptr[i], e = ptr[i + 1];
        if (b == e) continue;
        const W deg = add_rn<W>((W)val[b], pairwise_sum<W>(val + b + 1, (int64_t)(e - b - 1)));
        W dinv = (W)1 / deg;
        if (dinv == (W)INFINITY) dinv = (W)0;
        for (uint32_t p = b; p < e; ++p) val[p] = (double)mul_rn<W>(dinv, (W)val[p]);
    }
}

// _normalize(hop_k), k >= 2 (boolean entries): dinv = 1 / (entry count) in float64, 0 for an empty row.
__global__ void __launch_bounds__(256) niche_norm_bool(const uint32_t* __restrict__ ptr, int64_t n, double* __restrict__ dinv) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t d = ptr[i + 1] - ptr[i];
        dinv[i] = d ? 1.0 / (double)d : 0.0;
    }
}

// Upper bound on the distinct columns of row i of (H @ A) ∪ V: the summed A-degrees of H's columns plus V's row length.
__global__ void __launch_bounds__(256) niche_hop_bound(const uint32_t* __restrict__ h_ptr, const int32_t* __restrict__ h_col,
                                                       const uint32_t* __restrict__ a_ptr, const uint32_t* __restrict__ v_ptr, int64_t n,
                                                       int64_t* __restrict__ ub) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t s = v_ptr[i + 1] - v_ptr[i];
        for (uint32_t e = h_ptr[i]; e < h_ptr[i + 1]; ++e) s += a_ptr[h_col[e] + 1] - a_ptr[h_col[e]];
        ub[i] = s;
    }
}

constexpr int kWarps = 4;       // warps per block of the hop kernel
constexpr int kSlots = 512;     // shared-memory hash slots per warp
constexpr int kShortRow = 256;  // rows whose bound exceeds this use a table in global memory

template <typename W>
struct HashTable {
    int32_t* key;
    W* m;  // path sum of (H @ A)[i, key]
    W* v;  // visited[i, key]
    uint8_t* st;  // bit 0: reached by H @ A, bit 1: stored in visited
    int cap;  // a power of two
};

template <typename W>
__device__ __forceinline__ int ht_slot(HashTable<W>& t, int32_t k) {
    int s = (int)(((uint32_t)k * 2654435761u) & (uint32_t)(t.cap - 1));
    while (true) {
        const int32_t prev = atomicCAS(&t.key[s], -1, k);
        if (prev == -1 || prev == k) return s;
        s = (s + 1) & (t.cap - 1);
    }
}

// One row of hop_k = (H @ A) > visited and visited' = visited + hop_k (_hop, :1014-1027), one warp per row of `rows`.
// H's entries are taken in storage order (ascending columns), each one's row of A across the lanes (distinct columns), so
// every path sum adds its terms in the order scipy's SpGEMM does.  The row's hash table is the warp's shared-memory one, or,
// when g_off is given, the table of g_cap[r] slots at pool + g_off[r].  FILL = 0 counts hop_k's and visited's entries;
// FILL = 1 writes both in table order (hop_k is sorted afterwards).
template <typename W, bool FILL>
__global__ void __launch_bounds__(kWarps * 32) niche_hop(const int32_t* __restrict__ rows, int64_t n_rows, const uint32_t* __restrict__ h_ptr,
                                                         const int32_t* __restrict__ h_col, const double* __restrict__ h_val,
                                                         const uint32_t* __restrict__ a_ptr, const int32_t* __restrict__ a_col,
                                                         const double* __restrict__ a_val, const uint32_t* __restrict__ v_ptr,
                                                         const int32_t* __restrict__ v_col, const double* __restrict__ v_val,
                                                         const int64_t* __restrict__ g_off, const int32_t* __restrict__ g_cap,
                                                         uint8_t* __restrict__ pool, uint32_t* __restrict__ o_hcnt, uint32_t* __restrict__ o_vcnt,
                                                         const uint32_t* __restrict__ o_hptr, const uint32_t* __restrict__ o_vptr,
                                                         int32_t* __restrict__ o_hcol, int32_t* __restrict__ o_vcol,
                                                         double* __restrict__ o_vval) {
    __shared__ int32_t s_key[kWarps][kSlots];
    __shared__ W s_m[kWarps][kSlots];
    __shared__ W s_v[kWarps][kSlots];
    __shared__ uint8_t s_st[kWarps][kSlots];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n_rows; r += nwarps) {
        const int64_t i = rows[r];
        HashTable<W> t;
        if (!g_off) {
            t = {s_key[wib], s_m[wib], s_v[wib], s_st[wib], kSlots};
        } else {
            const int cap = g_cap[r];
            uint8_t* base = pool + g_off[r];
            t.key = reinterpret_cast<int32_t*>(base);
            t.m = reinterpret_cast<W*>(base + (size_t)cap * 4);
            t.v = reinterpret_cast<W*>(base + (size_t)cap * (4 + sizeof(W)));
            t.st = base + (size_t)cap * (4 + 2 * sizeof(W));
            t.cap = cap;
        }
        for (int s = lane; s < t.cap; s += 32) t.key[s] = -1, t.m[s] = (W)0, t.v[s] = (W)0, t.st[s] = 0;
        __syncwarp();
        for (uint32_t e = h_ptr[i]; e < h_ptr[i + 1]; ++e) {
            const int32_t j = h_col[e];
            const W h = h_val ? (W)h_val[e] : (W)1;
            for (uint32_t q = a_ptr[j] + lane; q < a_ptr[j + 1]; q += 32) {
                const int s = ht_slot(t, a_col[q]);
                t.m[s] = add_rn<W>(t.m[s], mul_rn<W>(h, (W)a_val[q]));
                t.st[s] |= 1;
            }
            __syncwarp();
        }
        for (uint32_t q = v_ptr[i] + lane; q < v_ptr[i + 1]; q += 32) {
            const int s = ht_slot(t, v_col[q]);
            t.v[s] = (W)v_val[q];
            t.st[s] |= 2;
        }
        __syncwarp();
        uint32_t nh = 0, nv = 0;
        for (int s0 = 0; s0 < t.cap; s0 += 32) {
            const int s = s0 + lane;
            const bool occ = t.key[s] >= 0;
            const bool hop = occ && t.m[s] > t.v[s];
            const bool vis = occ && (hop || (t.st[s] & 2));
            const unsigned bh = __ballot_sync(0xFFFFFFFFu, hop), bv = __ballot_sync(0xFFFFFFFFu, vis);
            const unsigned below = (1u << lane) - 1;
            if (FILL) {
                if (hop) o_hcol[o_hptr[i] + nh + __popc(bh & below)] = t.key[s];
                if (vis) {
                    const uint32_t q = o_vptr[i] + nv + __popc(bv & below);
                    o_vcol[q] = t.key[s];
                    o_vval[q] = (double)add_rn<W>(t.v[s], hop ? (W)1 : (W)0);
                }
            }
            nh += __popc(bh);
            nv += __popc(bv);
        }
        if (!FILL && lane == 0) o_hcnt[i] = nh, o_vcnt[i] = nv;
        __syncwarp();
    }
}

// hop_k and visited' from hop_{k-1} (h_val null: boolean), A and visited.  Rows whose bound fits half a shared-memory table
// run in one launch; the others get tables of at least twice their bound in global memory, in batches whose tables fit
// a quarter of the free device memory, so the scratch never exceeds that whatever the graph.  hop_k's rows are sorted by
// a segmented radix sort at the end.
template <typename W>
int next_hop(sqb_ctx* c, int64_t n, const uint32_t* h_ptr, const int32_t* h_col, const double* h_val, const SqbGraph& a, const uint32_t* v_ptr,
             const int32_t* v_col, const double* v_val, DevBuf<uint32_t>& o_hptr, DevBuf<int32_t>& o_hcol, DevBuf<uint32_t>& o_vptr,
             DevBuf<int32_t>& o_vcol, DevBuf<double>& o_vval) {
    DevBuf<int64_t> ub(c->stream);
    SQB_TRY(ub.alloc(n));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        niche_hop_bound<<<sqb_grid_rows(c, n, 256), 256, 0, c->stream>>>(h_ptr, h_col, a.ptr.p, v_ptr, n, ub.p);
        SQB_POST_LAUNCH();
    }
    std::vector<int64_t> h_ub(n);
    SQB_CUDA(cudaMemcpyAsync(h_ub.data(), ub.p, n * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    ub.release();
    size_t free_b = 0, total_b = 0;
    SQB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const size_t budget = std::max<size_t>(free_b / 4, (size_t)64 << 20);
    const size_t slot_bytes = 4 + 2 * sizeof(W) + 1;
    // rows: the short rows, then the long ones batch by batch; per long row its table's offset in its batch and its size
    std::vector<int32_t> rows;
    std::vector<int32_t> long_rows, cap_of;
    std::vector<int64_t> off_of;
    std::vector<int64_t> batch_begin{0};
    size_t batch_bytes = 0, pool_bytes = 0;
    for (int64_t i = 0; i < n; ++i) {
        if (h_ub[i] <= kShortRow) {
            rows.push_back((int32_t)i);
            continue;
        }
        SQB_CHECK(h_ub[i] < (1LL << 29), SQB_ERR_UNSUPPORTED, "sqb_niche_aggregate: a hop row may reach %lld columns (limit 2^29)",
                  (long long)h_ub[i]);
        int cap = 64;
        while (cap < 2 * h_ub[i]) cap *= 2;
        const size_t bytes = ((size_t)cap * slot_bytes + 15) & ~(size_t)15;
        if (batch_bytes > 0 && batch_bytes + bytes > budget) {
            batch_begin.push_back((int64_t)long_rows.size());
            batch_bytes = 0;
        }
        long_rows.push_back((int32_t)i);
        cap_of.push_back(cap);
        off_of.push_back((int64_t)batch_bytes);
        batch_bytes += bytes;
        pool_bytes = std::max(pool_bytes, batch_bytes);
    }
    batch_begin.push_back((int64_t)long_rows.size());
    const int64_t n_short = (int64_t)rows.size(), n_long = (int64_t)long_rows.size();
    rows.insert(rows.end(), long_rows.begin(), long_rows.end());
    DevBuf<int32_t> d_rows(c->stream), d_cap(c->stream);
    DevBuf<int64_t> d_off(c->stream);
    DevBuf<uint8_t> pool(c->stream);
    SQB_TRY(d_rows.alloc(n));
    SQB_TRY(sqb_h2d(c, d_rows.p, rows.data(), n * sizeof(int32_t)));
    if (n_long) {
        SQB_TRY(d_cap.alloc(n_long));
        SQB_TRY(d_off.alloc(n_long));
        SQB_TRY(pool.alloc(pool_bytes));
        SQB_TRY(sqb_h2d(c, d_cap.p, cap_of.data(), n_long * sizeof(int32_t)));
        SQB_TRY(sqb_h2d(c, d_off.p, off_of.data(), n_long * sizeof(int64_t)));
    }
    DevBuf<uint32_t> hcnt(c->stream), vcnt(c->stream);
    SQB_TRY(hcnt.alloc(n + 1));
    SQB_TRY(vcnt.alloc(n + 1));
    SQB_CUDA(cudaMemsetAsync(hcnt.p + n, 0, sizeof(uint32_t), c->stream));
    SQB_CUDA(cudaMemsetAsync(vcnt.p + n, 0, sizeof(uint32_t), c->stream));
    // one pass (FILL = 0 counts, 1 writes) over the short rows and every batch of long rows
    const auto pass = [&](auto fill) -> int {
        constexpr bool FILL = decltype(fill)::value;
        const auto launch = [&](const int32_t* rw, int64_t nr, const int64_t* go, const int32_t* gc) -> int {
            if (nr == 0) return SQB_OK;
            SqbLaunchScope scope(c, SQB_K_MISC);
            niche_hop<W, FILL><<<sqb_grid_rows(c, nr * 32, kWarps * 32), kWarps * 32, 0, c->stream>>>(
                rw, nr, h_ptr, h_col, h_val, a.ptr.p, a.col.p, a.val.p, v_ptr, v_col, v_val, go, gc, pool.p, FILL ? nullptr : hcnt.p,
                FILL ? nullptr : vcnt.p, FILL ? o_hptr.p : nullptr, FILL ? o_vptr.p : nullptr, FILL ? o_hcol.p : nullptr,
                FILL ? o_vcol.p : nullptr, FILL ? o_vval.p : nullptr);
            SQB_POST_LAUNCH();
            return SQB_OK;
        };
        SQB_TRY(launch(d_rows.p, n_short, nullptr, nullptr));
        for (size_t b = 0; b + 1 < batch_begin.size(); ++b) {
            const int64_t lo = batch_begin[b], hi = batch_begin[b + 1];
            SQB_TRY(launch(d_rows.p + n_short + lo, hi - lo, d_off.p + lo, d_cap.p + lo));
        }
        return SQB_OK;
    };
    SQB_TRY(pass(std::false_type()));
    SQB_TRY(o_hptr.alloc(n + 1));
    SQB_TRY(o_vptr.alloc(n + 1));
    uint32_t nh = 0, nv = 0;
    SQB_TRY(sqb_exclusive_scan(c, hcnt.p, o_hptr.p, n + 1, &nh));
    SQB_TRY(sqb_exclusive_scan(c, vcnt.p, o_vptr.p, n + 1, &nv));
    DevBuf<int32_t> unsorted(c->stream);
    SQB_TRY(unsorted.alloc(nh));
    SQB_TRY(o_hcol.alloc(nh));
    SQB_TRY(o_vcol.alloc(nv));
    SQB_TRY(o_vval.alloc(nv));
    std::swap(unsorted.p, o_hcol.p);  // the fill pass writes into `unsorted`
    std::swap(unsorted.n, o_hcol.n);
    SQB_TRY(pass(std::true_type()));
    std::swap(unsorted.p, o_hcol.p);
    std::swap(unsorted.n, o_hcol.n);
    pool.release();
    if (nh > 0) {
        size_t bytes = 0;
        SQB_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, bytes, unsorted.p, o_hcol.p, (int)nh, (int)n, o_hptr.p, o_hptr.p + 1, c->stream));
        DevBuf<uint8_t> tmp(c->stream);
        SQB_TRY(tmp.alloc(bytes));
        SQB_CUDA(cub::DeviceSegmentedSort::SortKeys(tmp.p, bytes, unsorted.p, o_hcol.p, (int)nh, (int)n, o_hptr.p, o_hptr.p + 1, c->stream));
    }
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    return SQB_OK;
}

// Launches niche_spmm for the accumulation type TA and writes columns [off, off + m) of the n x ld output (type TO).
template <typename TA, typename TX, typename TO>
int spmm(sqb_ctx* c, const uint32_t* ptr, const int32_t* col, const double* val, const double* rscale, int reverse, int skip_zero,
         bool variance, const TX* X, int64_t n, int64_t m, TO* out, int64_t ld) {
    SqbLaunchScope scope(c, SQB_K_MISC);
    const unsigned grid = sqb_grid_rows(c, n * 32, 256);
    if (variance)
        niche_spmm<TA, TX, TO, true><<<grid, 256, 0, c->stream>>>(ptr, col, val, rscale, reverse, skip_zero, X, n, m, out, ld);
    else
        niche_spmm<TA, TX, TO, false><<<grid, 256, 0, c->stream>>>(ptr, col, val, rscale, reverse, skip_zero, X, n, m, out, ld);
    SQB_POST_LAUNCH();
    return SQB_OK;
}

// The aggregation of one graph over X (dense on the device): UTAG (mode 0) or the CellCharter blocks (modes 1 mean, 2 variance).
template <typename W, typename TX, typename TO>
int aggregate_run(sqb_ctx* c, SqbGraph& g, const TX* X, int64_t m, int mode, int distance, TO* d_out, int64_t* out_hop_nnz) {
    const int64_t n = g.n;
    // float32 accumulation only when both the graph's normalised values and X are float32 (scipy's upcast)
    using T1 = typename std::conditional<std::is_same<W, float>::value && std::is_same<TX, float>::value, float, double>::type;
    if (mode == 0) {
        {
            SqbLaunchScope scope(c, SQB_K_MISC);
            niche_l1_rows<W><<<sqb_grid_rows(c, n, 256), 256, 0, c->stream>>>(g.ptr.p, g.val.p, n);
            SQB_POST_LAUNCH();
        }
        return spmm<T1, TX, TO>(c, g.ptr.p, g.col.p, g.val.p, nullptr, 0, 0, false, X, n, m, d_out, m);
    }
    const bool var = mode == 2;
    const int64_t ld = (int64_t)(distance + 1) * m;
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        niche_copy_block<TX, TO><<<sqb_grid_rows(c, n * m, 256), 256, 0, c->stream>>>(X, n, m, d_out, ld);
        SQB_POST_LAUNCH();
    }
    DevBuf<uint32_t> hcnt(c->stream), vcnt(c->stream), h_ptr(c->stream), v_ptr(c->stream);
    DevBuf<int32_t> h_col(c->stream), v_col(c->stream);
    DevBuf<double> h_val(c->stream), v_val(c->stream), n1(c->stream), dinv(c->stream);
    SQB_TRY(hcnt.alloc(n + 1));
    SQB_TRY(vcnt.alloc(n + 1));
    SQB_CUDA(cudaMemsetAsync(hcnt.p + n, 0, sizeof(uint32_t), c->stream));
    SQB_CUDA(cudaMemsetAsync(vcnt.p + n, 0, sizeof(uint32_t), c->stream));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        niche_hop1<false><<<sqb_grid_rows(c, n, 256), 256, 0, c->stream>>>(g.ptr.p, g.col.p, g.val.p, n, hcnt.p, vcnt.p, nullptr, nullptr,
                                                                          nullptr, nullptr, nullptr, nullptr);
        SQB_POST_LAUNCH();
    }
    SQB_TRY(h_ptr.alloc(n + 1));
    SQB_TRY(v_ptr.alloc(n + 1));
    uint32_t nh = 0, nv = 0;
    SQB_TRY(sqb_exclusive_scan(c, hcnt.p, h_ptr.p, n + 1, &nh));
    SQB_TRY(sqb_exclusive_scan(c, vcnt.p, v_ptr.p, n + 1, &nv));
    SQB_TRY(h_col.alloc(nh));
    SQB_TRY(h_val.alloc(nh));
    SQB_TRY(v_col.alloc(nv));
    SQB_TRY(v_val.alloc(nv));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        niche_hop1<true><<<sqb_grid_rows(c, n, 256), 256, 0, c->stream>>>(g.ptr.p, g.col.p, g.val.p, n, nullptr, nullptr, h_ptr.p, v_ptr.p,
                                                                         h_col.p, h_val.p, v_col.p, v_val.p);
        SQB_POST_LAUNCH();
    }
    out_hop_nnz[0] = nh;
    // hop 1: _normalize gives dinv * a in the value type, stored by scipy's SpGEMM in reverse column order
    SQB_TRY(n1.alloc(nh));
    SQB_CUDA(cudaMemcpyAsync(n1.p, h_val.p, (size_t)nh * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        niche_norm_hop1<W><<<sqb_grid_rows(c, n, 256), 256, 0, c->stream>>>(h_ptr.p, n1.p, n);
        SQB_POST_LAUNCH();
    }
    SQB_TRY((spmm<T1, TX, TO>(c, h_ptr.p, h_col.p, n1.p, nullptr, 1, 1, var, X, n, m, d_out + m, ld)));
    n1.release();
    SQB_TRY(dinv.alloc(n));
    for (int k = 2; k <= distance; ++k) {
        DevBuf<uint32_t> nh_ptr(c->stream), nv_ptr(c->stream);
        DevBuf<int32_t> nh_col(c->stream), nv_col(c->stream);
        DevBuf<double> nv_val(c->stream);
        SQB_TRY(next_hop<W>(c, n, h_ptr.p, h_col.p, k == 2 ? h_val.p : nullptr, g, v_ptr.p, v_col.p, v_val.p, nh_ptr, nh_col, nv_ptr, nv_col,
                            nv_val));
        h_ptr = std::move(nh_ptr);
        h_col = std::move(nh_col);
        v_ptr = std::move(nv_ptr);
        v_col = std::move(nv_col);
        v_val = std::move(nv_val);
        uint32_t e = 0;
        SQB_CUDA(cudaMemcpyAsync(&e, h_ptr.p + n, sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaStreamSynchronize(c->stream));
        out_hop_nnz[k - 1] = e;
        {
            SqbLaunchScope scope(c, SQB_K_MISC);
            niche_norm_bool<<<sqb_grid_rows(c, n, 256), 256, 0, c->stream>>>(h_ptr.p, n, dinv.p);
            SQB_POST_LAUNCH();
        }
        SQB_TRY((spmm<double, TX, TO>(c, h_ptr.p, h_col.p, nullptr, dinv.p, 0, 0, var, X, n, m, d_out + (int64_t)k * m, ld)));
    }
    return SQB_OK;
}

struct XArgs {
    const void *x, *indptr, *indices;
    int64_t nnz, m;
    int format, indptr_bits, index_bits, f32, device_input;
    uintptr_t producer_stream;
};

// X as a dense row-major n x m device matrix of TX: a dense device X is read in place, everything else lands in dx.
template <typename TX>
int x_on_device(sqb_ctx* c, int64_t n, const XArgs& x, DevBuf<uint8_t>& dx, const TX** out, const char* where) {
    if (x.format == 0 && x.device_input) {
        *out = reinterpret_cast<const TX*>(x.x);
        return SQB_OK;
    }
    SQB_TRY(dx.alloc((size_t)n * x.m * sizeof(TX)));
    TX* X = reinterpret_cast<TX*>(dx.p);
    *out = X;
    if (x.format == 0) return sqb_h2d(c, X, x.x, (size_t)n * x.m * sizeof(TX));
    SQB_CUDA(cudaMemsetAsync(X, 0, (size_t)n * x.m * sizeof(TX), c->stream));
    const auto densify = [&](const void* ip, const void* ix, const void* xv) {
        return sqb_dispatch_index(x.indptr_bits, x.index_bits, where, [&](auto tp, auto tx) -> int {
            using IP = typename decltype(tp)::type;
            using II = typename decltype(tx)::type;
            SQB_TRY(sqb_check_indptr(c, SQB_K_MISC, reinterpret_cast<const IP*>(ip), n, x.nnz, nullptr, where));
            DevBuf<unsigned> err(c->stream);
            SQB_TRY(err.alloc(1));
            SQB_CUDA(cudaMemsetAsync(err.p, 0, sizeof(unsigned), c->stream));
            {
                SqbLaunchScope scope(c, SQB_K_MISC);
                niche_densify<TX, IP, II><<<sqb_grid_rows(c, n, 256), 256, 0, c->stream>>>(
                    reinterpret_cast<const IP*>(ip), reinterpret_cast<const II*>(ix), reinterpret_cast<const TX*>(xv), n, x.m, X, err.p);
                SQB_POST_LAUNCH();
            }
            unsigned flag = 0;
            SQB_CUDA(cudaMemcpyAsync(&flag, err.p, sizeof(unsigned), cudaMemcpyDeviceToHost, c->stream));
            SQB_CUDA(cudaStreamSynchronize(c->stream));
            SQB_CHECK(!flag, SQB_ERR_INVALID, "%s: X column index out of range [0, %lld)", where, (long long)x.m);
            return SQB_OK;
        });
    };
    // a device X: sqb_niche_aggregate has waited for its producer stream already
    return sqb_with_caller_csr(c, n, x.nnz, x.indptr, x.indptr_bits, x.indices, x.index_bits, x.x, sizeof(TX), x.device_input, 0, densify);
}

}  // namespace

extern "C" int sqb_niche_profile(sqb_ctx* c, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices, int index_bits,
                                 const void* data, int data_dtype, int csc, int device_input, uintptr_t producer_stream,
                                 const int32_t* codes, int n_cls, int distance, const double* weights, double weight_sum, int abs_nhood,
                                 double* out) {
    static const char* where = "sqb_niche_profile";
    SQB_CHECK(c, SQB_ERR_INVALID, "%s: null ctx", where);
    const SqbGraphArgs ga{n, nnz, indptr, indices, data, indptr_bits, index_bits, data_dtype, csc, device_input, producer_stream};
    SQB_TRY(check_graph(ga, where));
    SQB_CHECK(codes && out, SQB_ERR_INVALID, "%s: null argument", where);
    SQB_CHECK(n_cls >= 1, SQB_ERR_INVALID, "%s: n_cls=%d must be at least 1", where, n_cls);
    SQB_CHECK(distance >= 1 && (distance == 1 || weights), SQB_ERR_INVALID, "%s: distance=%d must be >= 1 (with weights when > 1)", where,
              distance);
    for (int64_t v = 0; v < n; ++v)
        SQB_CHECK(codes[v] >= -1 && codes[v] < n_cls, SQB_ERR_INVALID, "%s: codes[%lld]=%d out of range [-1, %d)", where, (long long)v, codes[v],
                  n_cls);
    SQB_CUDA(cudaSetDevice(c->device));
    SqbGraph g(c->stream);
    SQB_TRY(sqb_load_graph(c, ga, SqbGraphForm::CANONICAL, 0, g, where));
    const size_t cells = (size_t)n * n_cls;
    DevBuf<int32_t> d_codes(c->stream);
    DevBuf<double> P(c->stream), Q(c->stream), O(c->stream);
    SQB_TRY(d_codes.alloc(n));
    SQB_TRY(P.alloc(cells));
    SQB_TRY(O.alloc(cells));
    if (distance > 1) SQB_TRY(Q.alloc(cells));
    SQB_TRY(sqb_h2d(c, d_codes.p, codes, n * sizeof(int32_t)));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        niche_profile_hop1<<<sqb_grid_rows(c, n, 256), 256, 0, c->stream>>>(g.ptr.p, g.col.p, g.val.p, d_codes.p, n, n_cls, P.p);
        SQB_POST_LAUNCH();
    }
    for (int k = 0; k < distance; ++k) {
        if (k > 0) {  // P_{k+1} = A P_k
            SQB_TRY((spmm<double, double, double>(c, g.ptr.p, g.col.p, g.val.p, nullptr, 0, 0, false, P.p, n, n_cls, Q.p, n_cls)));
            std::swap(P.p, Q.p);
        }
        SqbLaunchScope scope(c, SQB_K_MISC);
        niche_profile_fold<<<sqb_grid_rows(c, n, 256), 256, 0, c->stream>>>(P.p, n, n_cls, abs_nhood, k, distance, distance > 1 ? weights[k] : 1.0,
                                                                           weight_sum, O.p);
        SQB_POST_LAUNCH();
    }
    SQB_CUDA(cudaMemcpyAsync(out, O.p, cells * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    return SQB_OK;
}

extern "C" int sqb_niche_aggregate(sqb_ctx* c, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices, int index_bits,
                                   const void* data, int data_dtype, int csc, int device_input, uintptr_t producer_stream, const void* x,
                                   const void* x_indptr, const void* x_indices, int64_t x_nnz, int x_format, int x_indptr_bits,
                                   int x_index_bits, int x_f32, int64_t m, int x_device, uintptr_t x_stream, int mode, int distance,
                                   int out_f32, void* out, int64_t* out_hop_nnz) {
    static const char* where = "sqb_niche_aggregate";
    SQB_CHECK(c, SQB_ERR_INVALID, "%s: null ctx", where);
    const SqbGraphArgs ga{n, nnz, indptr, indices, data, indptr_bits, index_bits, data_dtype, csc, device_input, producer_stream};
    SQB_TRY(check_graph(ga, where));
    SQB_CHECK(mode >= 0 && mode <= 2, SQB_ERR_INVALID, "%s: mode=%d must be 0 (utag), 1 (mean) or 2 (variance)", where, mode);
    SQB_CHECK(mode == 0 || (distance >= 1 && out_hop_nnz), SQB_ERR_INVALID, "%s: distance must be >= 1 with out_hop_nnz", where);
    SQB_CHECK(m >= 1 && out && (x || (x_format == 1 && x_nnz == 0)), SQB_ERR_INVALID, "%s: null argument or m < 1", where);
    SQB_CHECK(x_format == 0 || (x_format == 1 && x_indptr && (x_indices || x_nnz == 0)), SQB_ERR_INVALID, "%s: x_format must be 0 (dense) or 1 (CSR)",
              where);
    const bool w_f32 = data_dtype == 0 || nnz == 0;
    const bool t1_f32 = w_f32 && x_f32;
    SQB_CHECK(!out_f32 || (t1_f32 && (mode == 0 || distance == 1)), SQB_ERR_INVALID,
              "%s: a float32 output needs float32 graph values and X, and no hop beyond the first", where);
    SQB_CUDA(cudaSetDevice(c->device));
    SqbGraph g(c->stream);
    // UTAG reads the graph in storage order (normalize keeps it); CellCharter starts from its canonical form (tolil)
    SQB_TRY(sqb_load_graph(c, ga, mode != 0 ? SqbGraphForm::CANONICAL : SqbGraphForm::STORED, 0, g, where));
    const XArgs xa{x, x_indptr, x_indices, x_nnz, m, x_format, x_indptr_bits, x_index_bits, x_f32, x_device, x_stream};
    const int64_t cols = mode == 0 ? m : (int64_t)(distance + 1) * m;
    const size_t out_bytes = (size_t)n * cols * (out_f32 ? 4 : 8);
    DevBuf<uint8_t> dx(c->stream), d_out(c->stream);
    SQB_TRY(d_out.alloc(out_bytes));
    const auto body = [&]() -> int {
        const auto with_x = [&](auto tx) -> int {
            using TX = typename decltype(tx)::type;
            const TX* X = nullptr;
            SQB_TRY(x_on_device<TX>(c, n, xa, dx, &X, where));
            const auto with_out = [&](auto to) -> int {
                using TO = typename decltype(to)::type;
                TO* o = reinterpret_cast<TO*>(d_out.p);
                return w_f32 ? aggregate_run<float, TX, TO>(c, g, X, m, mode, distance, o, out_hop_nnz)
                             : aggregate_run<double, TX, TO>(c, g, X, m, mode, distance, o, out_hop_nnz);
            };
            return out_f32 ? with_out(SqbType<float>()) : with_out(SqbType<double>());
        };
        SQB_TRY(x_f32 ? with_x(SqbType<float>()) : with_x(SqbType<double>()));
        SQB_CUDA(cudaStreamSynchronize(c->stream));  // the caller's X is no longer read
        return SQB_OK;
    };
    if (x_device)
        SQB_TRY(sqb_read_caller_buffers(c, x_stream, body));
    else
        SQB_TRY(body());
    SQB_CUDA(cudaMemcpyAsync(out, d_out.p, out_bytes, cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    return SQB_OK;
}
