// caller_graph.cu — a caller's n x n graph as a device CSR in one of the forms of caller_graph.cuh, for the entry points
// that take a neighbour graph and rebuild it (sqb_centrality_scores, sqb_niche_*).
//
// Every stored entry becomes a record (two for SYMMETRIC: (i, j) from A and (j, i) from Aᵀ): a 64-bit key
// row << (nbits + 1) | col << 1 | from_transpose, with n <= 2^nbits, and the entry index as payload.  A stable radix sort on
// the row bits (STORED) or the row and column bits (CANONICAL, SYMMETRIC) keeps storage order within a key.  The head of
// each run of equal (row, col) reduces the run (the reducer of its form) and sets its keep flag; the kept heads, compacted
// by an exclusive scan of the flags, are the CSR.  A CSR used as stored needs no records: its columns and values are
// written in place of them.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "caller_graph.cuh"

namespace {

// A diagonal entry of SYMMETRIC: all ones over the sorted bits, it sorts after every record and is never kept.  No
// off-diagonal key is all ones there: row = col = 2^nbits - 1 is the diagonal.
constexpr uint64_t kDiagKey = ~0ull;

// One warp per major index m: the records of its stored entries (keys and ids), their values as float64 (val, or null)
// and, for a CSR used as stored, their columns instead of records (col non-null).  An index outside [0, n) raises bit 2 of
// *err; its entry is written with index 0.
template <typename IP, typename II, typename VT>
__global__ void __launch_bounds__(256) cgraph_expand(const IP* __restrict__ ip, const II* __restrict__ ix, const VT* __restrict__ data,
                                                     int64_t n, int csc, int sym, int nbits, uint64_t* __restrict__ keys,
                                                     uint32_t* __restrict__ ids, int32_t* __restrict__ col, double* __restrict__ val,
                                                     unsigned* __restrict__ err) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    unsigned bad = 0;
    for (int64_t m = warp; m < n; m += nwarps) {
        for (int64_t e = (int64_t)ip[m] + lane; e < (int64_t)ip[m + 1]; e += 32) {
            const int64_t j = (int64_t)ix[e];
            const bool ok = j >= 0 && j < n;
            bad |= !ok;
            const int64_t jj = ok ? j : 0;
            if (val) val[e] = sqb_cvt<double>(data[e]);
            if (col) {
                col[e] = (int32_t)jj;
                continue;
            }
            const uint64_t r = csc ? jj : m, c = csc ? m : jj;
            if (sym) {
                const bool edge = r != c;
                const uint64_t k0 = edge ? (r << (nbits + 1)) | (c << 1) : kDiagKey;
                const uint64_t k1 = edge ? (c << (nbits + 1)) | (r << 1) | 1u : kDiagKey;
                reinterpret_cast<ulonglong2*>(keys)[e] = make_ulonglong2(k0, k1);
                reinterpret_cast<uint2*>(ids)[e] = make_uint2((uint32_t)e, (uint32_t)e);
            } else {
                keys[e] = (r << (nbits + 1)) | (c << 1);
                ids[e] = (uint32_t)e;
            }
        }
    }
    if (bad) atomicOr(err, 2u);
}

// Reducers of a run: first(id, from_transpose) starts it, add(...) takes each later record, keep(run, p) is the head's keep
// flag.  kMerge false: every record is a run of its own.
//
// STORED / CANONICAL: the float64 values summed in W in storage order, from the first one; every run is kept, its sum
// written to out[p].
template <typename W, bool MERGE>
struct SumValues {
    static constexpr bool kMerge = MERGE;
    using Run = W;
    const double* val;
    double* out;
    __device__ W first(uint32_t id, bool) const { return (W)val[id]; }
    __device__ W add(W s, uint32_t id, bool) const { return add_rn<W>(s, (W)val[id]); }
    __device__ uint32_t keep(W s, int64_t p) const {
        out[p] = (double)s;
        return 1;
    }
};

// SYMMETRIC: A's entries and Aᵀ's summed apart in A's dtype, then combined.  Integers wrap at int_bits (the caller's dtype
// width; narrower integers arrive widened), bool (one byte) sums as logical or, floats in their own precision.  A run is
// kept when its sum is non-zero (NaN is non-zero).
template <typename VT>
struct SumSymmetric {
    static constexpr bool kMerge = true;
    using Acc = typename std::conditional<std::is_floating_point<VT>::value, VT, uint64_t>::type;
    struct Run {
        Acc a, t;  // entries of A, entries of its transpose
    };
    const VT* data;
    int int_bits;
    __device__ static Acc sum(Acc a, VT v) {
        if constexpr (std::is_same<VT, uint8_t>::value)
            return a | (uint64_t)(v != 0);
        else if constexpr (std::is_floating_point<VT>::value)
            return a + v;
        else
            return a + (uint64_t)(int64_t)v;
    }
    __device__ Run add(Run s, uint32_t id, bool t) const {
        if (t)
            s.t = sum(s.t, data[id]);
        else
            s.a = sum(s.a, data[id]);
        return s;
    }
    __device__ Run first(uint32_t id, bool t) const { return add(Run{(Acc)0, (Acc)0}, id, t); }
    __device__ uint32_t keep(Run s, int64_t) const {
        if constexpr (std::is_same<VT, uint8_t>::value)
            return (s.a | s.t) != 0;
        else if constexpr (std::is_floating_point<VT>::value)
            return s.a + s.t != (Acc)0;  // NaN != 0
        else
            return int_bits >= 64 ? s.a + s.t != 0 : ((s.a + s.t) & ((1ull << int_bits) - 1)) != 0;
    }
};

// keep[p]: the head of a run of equal (row, col) reduced by R (0 elsewhere and for the diagonal key).
template <typename R>
__global__ void __launch_bounds__(256) cgraph_runs(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ ids, int64_t m, R r,
                                                   uint32_t* __restrict__ keep) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < m; p += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t k = keys[p];
        uint32_t flag = 0;
        if (k != kDiagKey && (!R::kMerge || p == 0 || (keys[p - 1] >> 1) != (k >> 1))) {
            typename R::Run s = r.first(ids[p], k & 1);
            if (R::kMerge)
                for (int64_t q = p + 1; q < m && (keys[q] >> 1) == (k >> 1); ++q) s = r.add(s, ids[q], keys[q] & 1);
            flag = r.keep(s, p);
        }
        keep[p] = flag;
    }
}

// The kept records at their ranks: row, column and (val non-null) the run's value.
__global__ void __launch_bounds__(256) cgraph_compact(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ keep,
                                                      const uint32_t* __restrict__ rank, const double* __restrict__ run_val, int64_t m,
                                                      int nbits, int32_t* __restrict__ row, int32_t* __restrict__ col,
                                                      double* __restrict__ val) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < m; p += (int64_t)gridDim.x * blockDim.x) {
        if (!keep[p]) continue;
        const uint64_t k = keys[p];
        const uint32_t q = rank[p];
        row[q] = (int32_t)(k >> (nbits + 1));
        col[q] = (int32_t)((k >> 1) & ((1ull << nbits) - 1));
        if (val) val[q] = run_val[p];
    }
}

// indptr of a CSR from the ascending rows of its e entries: indptr[r] = the first entry of a row >= r.
__global__ void __launch_bounds__(256) cgraph_indptr(const int32_t* __restrict__ row, int64_t e, int64_t n, uint32_t* __restrict__ indptr) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p <= e; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = p < e ? row[p] : n;
        const int64_t rp = p == 0 ? -1 : row[p - 1];
        for (int64_t q = rp + 1; q <= r; ++q) indptr[q] = (uint32_t)p;
    }
}

// f(SqbType<VT>()) for the graph's value dtype; float16 values are refused (and bool unless WITH_BOOL).
template <bool WITH_BOOL, typename F>
int dispatch_values(int code, const char* where, F&& f) {
    return sqb_dispatch_value<WITH_BOOL>(code, where, "data_dtype", [&](auto tv) -> int {
        if constexpr (std::is_same<typename decltype(tv)::type, __half>::value) {
            sqb_set_error("%s: float16 graph values are not supported", where);
            return SQB_ERR_INVALID;
        } else {
            return f(tv);
        }
    });
}

template <typename IP, typename II>
int load(sqb_ctx* c, const SqbGraphArgs& a, const void* indptr, const void* indices, const void* data, SqbGraphForm form, int int_bits,
         SqbGraph& g, const char* where) {
    const int64_t n = a.n, nnz = a.nnz;
    const IP* ip = reinterpret_cast<const IP*>(indptr);
    const bool sym = form == SqbGraphForm::SYMMETRIC, as_stored = form == SqbGraphForm::STORED && !a.csc;
    g.n = n;
    SQB_TRY(g.ptr.alloc(n + 1));
    SQB_TRY(sqb_check_indptr(c, SQB_K_MISC, ip, n, nnz, g.ptr.p, where));
    if (nnz == 0) {
        g.e = 0;
        SQB_TRY(g.col.alloc(1));
        if (!sym) SQB_TRY(g.val.alloc(1));
        return SQB_OK;
    }
    const int64_t m = sym ? 2 * nnz : nnz;  // records
    int nbits = 1;
    while (nbits < 31 && ((int64_t)1 << nbits) < n) ++nbits;
    DevBuf<uint64_t> keys(c->stream);
    DevBuf<uint32_t> ids(c->stream), keep(c->stream), rank(c->stream);
    DevBuf<int32_t> col(c->stream);
    DevBuf<double> val(c->stream), run_val(c->stream);
    DevBuf<unsigned> err(c->stream);
    if (as_stored) {
        SQB_TRY(col.alloc(nnz));
    } else {
        SQB_TRY(keys.alloc(m));
        SQB_TRY(ids.alloc(m));
    }
    if (!sym) SQB_TRY(val.alloc(nnz));
    SQB_TRY(err.alloc(1));
    SQB_CUDA(cudaMemsetAsync(err.p, 0, sizeof(unsigned), c->stream));
    const auto expand = [&](auto tv) -> int {
        using VT = typename decltype(tv)::type;
        SqbLaunchScope scope(c, SQB_K_MISC);
        cgraph_expand<IP, II, VT><<<sqb_grid_rows(c, n * 32, 256), 256, 0, c->stream>>>(
            ip, reinterpret_cast<const II*>(indices), reinterpret_cast<const VT*>(data), n, a.csc, sym, nbits, keys.p, ids.p, col.p, val.p, err.p);
        SQB_POST_LAUNCH();
        return SQB_OK;
    };
    // SYMMETRIC reads the values in its reducer, in their own type; a bool value becomes 1.0 / 0.0
    SQB_TRY(sym ? expand(SqbType<double>()) : dispatch_values<true>(a.data_dtype, where, expand));
    uint32_t e = (uint32_t)nnz;
    if (!as_stored) {
        DevBuf<uint64_t> keys_s(c->stream);
        DevBuf<uint32_t> ids_s(c->stream);
        SQB_TRY(keys_s.alloc(m));
        SQB_TRY(ids_s.alloc(m));
        const int begin_bit = form == SqbGraphForm::STORED ? nbits + 1 : 1, end_bit = 2 * nbits + 1;
        size_t bytes = 0;
        SQB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys.p, keys_s.p, ids.p, ids_s.p, (int)m, begin_bit, end_bit, c->stream));
        {
            DevBuf<uint8_t> tmp(c->stream);
            SQB_TRY(tmp.alloc(bytes));
            SQB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, bytes, keys.p, keys_s.p, ids.p, ids_s.p, (int)m, begin_bit, end_bit, c->stream));
        }
        keys = std::move(keys_s);
        ids = std::move(ids_s);
        SQB_TRY(keep.alloc(m));
        SQB_TRY(rank.alloc(m));
        if (!sym) SQB_TRY(run_val.alloc(m));
        const auto runs = [&](auto r) -> int {
            SqbLaunchScope scope(c, SQB_K_MISC);
            cgraph_runs<<<sqb_grid_rows(c, m, 256), 256, 0, c->stream>>>(keys.p, ids.p, m, r, keep.p);
            SQB_POST_LAUNCH();
            return SQB_OK;
        };
        if (sym)
            SQB_TRY(dispatch_values<true>(a.data_dtype, where, [&](auto tv) {
                using VT = typename decltype(tv)::type;
                return runs(SumSymmetric<VT>{reinterpret_cast<const VT*>(data), int_bits});
            }));
        else if (form == SqbGraphForm::STORED)
            SQB_TRY(runs(SumValues<double, false>{val.p, run_val.p}));  // float32 values are exact in float64
        else if (a.data_dtype == 0)
            SQB_TRY(runs(SumValues<float, true>{val.p, run_val.p}));
        else
            SQB_TRY(runs(SumValues<double, true>{val.p, run_val.p}));
        ids.release();
        val.release();
        SQB_TRY(sqb_exclusive_scan(c, keep.p, rank.p, m, &e));
    }
    unsigned flag = 0;
    SQB_CUDA(cudaMemcpyAsync(&flag, err.p, sizeof(unsigned), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    SQB_CHECK(!(flag & 2u), SQB_ERR_INVALID, "%s: index out of range [0, %lld)", where, (long long)n);
    g.e = e;
    if (as_stored) {
        g.col = std::move(col);
        g.val = std::move(val);
        return SQB_OK;
    }
    DevBuf<int32_t> rows(c->stream);
    SQB_TRY(rows.alloc(e));
    SQB_TRY(g.col.alloc(e));
    if (!sym) SQB_TRY(g.val.alloc(e));
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        cgraph_compact<<<sqb_grid_rows(c, m, 256), 256, 0, c->stream>>>(keys.p, keep.p, rank.p, run_val.p, m, nbits, rows.p, g.col.p, g.val.p);
        SQB_POST_LAUNCH();
    }
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        cgraph_indptr<<<sqb_grid_rows(c, (int64_t)e + 1, 256), 256, 0, c->stream>>>(rows.p, e, n, g.ptr.p);
        SQB_POST_LAUNCH();
    }
    return SQB_OK;
}

}  // namespace

int sqb_graph_value_bytes(int code) {
    switch (code) {
        case 0: return 4;
        case 1: return 8;
        case 3: return 4;
        case 4: return 8;
        case 5: return 1;
    }
    return 0;
}

int sqb_check_graph_args(const SqbGraphArgs& a, int nnz_log2, const char* where) {
    SQB_CHECK(a.n >= 1 && a.n < 0x7FFFFFFFLL, SQB_ERR_INVALID, "%s: n=%lld out of range [1, 2^31 - 1)", where, (long long)a.n);
    SQB_CHECK(a.nnz >= 0 && a.nnz < (1LL << nnz_log2), SQB_ERR_INVALID, "%s: nnz=%lld out of range [0, 2^%d)", where, (long long)a.nnz, nnz_log2);
    SQB_CHECK(a.indptr && ((a.indices && a.data) || a.nnz == 0), SQB_ERR_INVALID, "%s: null graph argument", where);
    SQB_CHECK((a.indptr_bits == 32 || a.indptr_bits == 64) && (a.index_bits == 32 || a.index_bits == 64), SQB_ERR_INVALID,
              "%s: indptr_bits / index_bits must be 32 or 64", where);
    return SQB_OK;
}

int sqb_load_graph(sqb_ctx* c, const SqbGraphArgs& a, SqbGraphForm form, int int_bits, SqbGraph& g, const char* where) {
    return sqb_with_caller_csr(c, a.n, a.nnz, a.indptr, a.indptr_bits, a.indices, a.index_bits, a.data, sqb_graph_value_bytes(a.data_dtype),
                               a.device_input, a.producer_stream, [&](const void* ip, const void* ix, const void* dv) {
                                   return sqb_dispatch_index(a.indptr_bits, a.index_bits, where, [&](auto tp, auto tx) {
                                       return load<typename decltype(tp)::type, typename decltype(tx)::type>(c, a, ip, ix, dv, form, int_bits, g,
                                                                                                             where);
                                   });
                               });
}

int sqb_exclusive_scan(sqb_ctx* c, const uint32_t* in, uint32_t* out, int64_t m, uint32_t* total) {
    size_t bytes = 0;
    SQB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, (int)m, c->stream));
    DevBuf<uint8_t> tmp(c->stream);
    SQB_TRY(tmp.alloc(bytes));
    SQB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, in, out, (int)m, c->stream));
    uint32_t tail[2] = {0, 0};
    SQB_CUDA(cudaMemcpyAsync(&tail[0], out + m - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaMemcpyAsync(&tail[1], in + m - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    *total = tail[0] + tail[1];
    return SQB_OK;
}

namespace {

__global__ void cgraph_iota(int32_t* __restrict__ out, int64_t m) {
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < m; k += (int64_t)gridDim.x * blockDim.x) out[k] = (int32_t)k;
}

// column ranges [cbeg[j], cend[j]) of the entries sorted by column (both zeroed first: an empty column stays empty)
__global__ void cgraph_col_bounds(const int32_t* __restrict__ key, int64_t m, int32_t* __restrict__ cbeg, int32_t* __restrict__ cend) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < m; p += (int64_t)gridDim.x * blockDim.x) {
        const int32_t j = key[p];
        if (p == 0 || key[p - 1] != j) cbeg[j] = (int32_t)p;
        if (p == m - 1 || key[p + 1] != j) cend[j] = (int32_t)(p + 1);
    }
}

}  // namespace

int sqb_col_order(sqb_ctx* c, int kclass, const int32_t* idx, int64_t m, int64_t n, DevBuf<int32_t>& perm, DevBuf<int32_t>& cbeg,
                  DevBuf<int32_t>& cend) {
    SQB_TRY(cbeg.alloc(n));
    SQB_TRY(cend.alloc(n));
    SQB_TRY(perm.alloc(m > 0 ? m : 1));
    SQB_CUDA(cudaMemsetAsync(cbeg.p, 0, n * sizeof(int32_t), c->stream));
    SQB_CUDA(cudaMemsetAsync(cend.p, 0, n * sizeof(int32_t), c->stream));
    if (m == 0) return SQB_OK;
    DevBuf<int32_t> keys(c->stream), iota(c->stream);
    DevBuf<uint8_t> tmp(c->stream);
    SQB_TRY(keys.alloc(m));
    SQB_TRY(iota.alloc(m));
    {
        SqbLaunchScope scope(c, kclass);
        cgraph_iota<<<sqb_grid_rows(c, m, 256), 256, 0, c->stream>>>(iota.p, m);
        SQB_POST_LAUNCH();
    }
    int bits = 1;
    while (bits < 31 && ((uint64_t)(n - 1) >> bits) != 0) ++bits;
    size_t bytes = 0;
    SQB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, idx, keys.p, iota.p, perm.p, (int)m, 0, bits, c->stream));
    SQB_TRY(tmp.alloc(bytes > 0 ? bytes : 1));
    SQB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, bytes, idx, keys.p, iota.p, perm.p, (int)m, 0, bits, c->stream));
    c->launches += 1;
    SqbLaunchScope scope(c, kclass);
    cgraph_col_bounds<<<sqb_grid_rows(c, m, 256), 256, 0, c->stream>>>(keys.p, m, cbeg.p, cend.p);
    SQB_POST_LAUNCH();
    return SQB_OK;
}
