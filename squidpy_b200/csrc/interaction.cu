// interaction.cu — interaction_matrix on H100 (sm_90a): cluster x cluster sums over the stored entries of a CSR graph.
//
// Replaces the reference's numba loop `_interaction_matrix` (src/squidpy/gr/_nhood.py:412-429) together with the NaN masking
// of `interaction_matrix` (:386-395): observations without a label (code < 0) are removed from rows AND columns, which for
// the sums is the same as skipping every stored entry with an unlabelled end point (no sub-matrix is built).  Every result
// equals the reference's bit for bit, and does not change from run to run:
//   counts (weights = false):    out[a][b] = number of stored entries (i -> j) with code(i) = a, code(j) = b      (int64 atomics)
//   integer / bool values:       their sum in int64, wrapping modulo 2^64 like numba's int64 `+=`                 (uint64 atomics)
//   float values, float64 sums:  the reference adds output[a, b] += v in float64, rows ascending and each row's entries in
//                                storage order.  Where every partial sum is exact (all values finite multiples of 2^q with
//                                sum |v| <= 2^(53+q): binary connectivities, for one) any order gives those bits, and the
//                                entries are added by atomics (the fast path).  Otherwise (the ordered path) every labelled
//                                entry gets the key (cell, row of the graph); a stable radix sort of the keys in storage
//                                order puts each cell's entries in the reference's order, and one warp per cell adds them
//                                in a single __dadd_rn chain from +0.0.  Cells run in parallel; only a cell's own chain is serial.
// For a CSC graph (the CSR arrays of its transpose) the rows of the graph are the arrays' column indices: the stable sort on
// (cell, graph row) gives columns ascending within a row and duplicates in storage order, the order of the graph's tocsr().
// HBM-bound: the CSR is streamed once (8-12 bytes per stored entry); the label gather hits L2.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"

// MODE of interaction_kernel: what a stored entry adds to its bin
enum { IM_COUNT = 0, IM_FLOAT = 1, IM_INT = 2 };

// IP / II: index types of indptr / indices (uint32 for the host path's staged copy, int32 / int64 for a caller's device
// CSR read in place).  A column index outside [0, n) is skipped and raises bit 2 of *err (null: host input, validated on
// the host); a code >= C is skipped too (bit 4).  indptr must have been validated: the kernel follows it.
// IM_FLOAT adds float64 values by atomics: exact only where every partial sum is (interaction_fast_ok).
template <typename IP, typename II, typename VT, int MODE>
__global__ void __launch_bounds__(256) interaction_kernel(const IP* __restrict__ indptr, const II* __restrict__ indices,
                                                          const VT* __restrict__ data, const int32_t* __restrict__ codes, int64_t n,
                                                          int C, int use_smem, double* __restrict__ out_w,
                                                          unsigned long long* __restrict__ out_c, unsigned* __restrict__ err) {
    extern __shared__ unsigned char sqb_inter_smem[];
    double* s_w = reinterpret_cast<double*>(sqb_inter_smem);
    unsigned long long* s_c = reinterpret_cast<unsigned long long*>(sqb_inter_smem);
    const int CC = C * C;
    if (use_smem) {
        for (int i = threadIdx.x; i < CC; i += blockDim.x) {
            if (MODE == IM_FLOAT)
                s_w[i] = 0.0;
            else
                s_c[i] = 0ull;
        }
        __syncthreads();
    }
    // one warp per row: lanes stride over the row's entries (coalesced index / value loads)
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = warp; i < n; i += nwarps) {
        const int32_t a = codes[i];  // warp uniform
        if (a >= C) {
            if (err && lane == 0) atomicOr(err, 4u);
            continue;
        }
        if (a < 0 && !err) continue;  // unlabelled row; device input still has its column indices validated
        const int64_t beg = (int64_t)indptr[i], end = (int64_t)indptr[i + 1];
        for (int64_t e = beg + lane; e < end; e += 32) {
            const int64_t j = (int64_t)indices[e];
            if (j < 0 || j >= n) {
                if (err) atomicOr(err, 2u);
                continue;
            }
            if (a < 0) continue;
            const int32_t b = codes[j];
            if ((unsigned)b >= (unsigned)C) continue;  // no label (< 0); >= C is flagged by row j
            const int bin = a * C + b;
            if (MODE == IM_FLOAT) {
                const double v = sqb_cvt<double>(data[e]);
                if (use_smem)
                    atomicAdd(&s_w[bin], v);
                else
                    atomicAdd(&out_w[bin], v);
            } else {
                // int64 values wrap modulo 2^64 in two's complement, as numba's int64 sums do
                const unsigned long long v = MODE == IM_COUNT ? 1ull : (unsigned long long)sqb_cvt<int64_t>(data[e]);
                if (use_smem)
                    atomicAdd(&s_c[bin], v);
                else
                    atomicAdd(&out_c[bin], v);
            }
        }
    }
    if (use_smem) {
        __syncthreads();
        for (int i = threadIdx.x; i < CC; i += blockDim.x) {
            if (MODE == IM_FLOAT) {
                const double v = s_w[i];
                if (v != 0.0) atomicAdd(&out_w[i], v);
            } else {
                const unsigned long long v = s_c[i];
                if (v != 0ull) atomicAdd(&out_c[i], v);
            }
        }
    }
}

// grid / shared memory of interaction_kernel for n rows and C classes
struct InterLaunch {
    unsigned blocks;
    size_t smem;
    int use_smem;
    InterLaunch(const sqb_ctx* c, int64_t n, int C) {
        const size_t CC = (size_t)C * C;
        use_smem = CC * 8 <= 48 * 1024;
        smem = use_smem ? CC * 8 : 0;
        int64_t b = ceil_div64(n * 32, 256);
        const int64_t max_blocks = (int64_t)c->sm_count * 8;
        if (b > max_blocks) b = max_blocks;
        if (b < 1) b = 1;
        blocks = (unsigned)b;
    }
};

// ---- float values: the exactness test of the fast path ----------------------------------------------------------------
// Over the nnz stored values (as float64): stat[0] = min q with every non-zero value a multiple of 2^q, stat[1] = max h with
// some |v| < 2^h not holding for h - 1, stat[2] = 1 if a value is NaN or ±inf.  Exponents are stored + 2048 (unsigned).
template <typename VT>
__global__ void __launch_bounds__(256) interaction_exp_kernel(const VT* __restrict__ data, int64_t nnz, unsigned* __restrict__ stat) {
    unsigned lo = 0xFFFFFFFFu, hi = 0u, bad = 0u;
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long bits = (unsigned long long)__double_as_longlong(sqb_cvt<double>(data[e])) & 0x7FFFFFFFFFFFFFFFull;
        const int E = (int)(bits >> 52);
        const unsigned long long M = bits & 0xFFFFFFFFFFFFFull;
        if (E == 0x7FF) {
            bad = 1u;
        } else if (E == 0) {  // zero or subnormal M * 2^-1074
            if (M) {
                lo = min(lo, (unsigned)(2048 - 1074 + __ffsll((long long)M) - 1));
                hi = max(hi, (unsigned)(2048 - 1074 + 64 - __clzll((long long)M)));
            }
        } else {  // (2^52 + M) * 2^(E - 1075) < 2^(E - 1022)
            lo = min(lo, (unsigned)(2048 + E - 1075 + (M ? __ffsll((long long)M) - 1 : 52)));
            hi = max(hi, (unsigned)(2048 + E - 1022));
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        lo = min(lo, __shfl_xor_sync(0xFFFFFFFFu, lo, o));
        hi = max(hi, __shfl_xor_sync(0xFFFFFFFFu, hi, o));
        bad |= __shfl_xor_sync(0xFFFFFFFFu, bad, o);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMin(&stat[0], lo);
        atomicMax(&stat[1], hi);
        if (bad) atomicOr(&stat[2], 1u);
    }
}

// True when adding any subset of the nnz values in any order gives the exact sum: every value finite and a multiple of 2^q,
// nnz * max|v| <= 2^(53 + q) (every partial sum is then an integer multiple of 2^q below 2^53 * 2^q, a float64) and below
// 2^1024 (no overflow).
static bool interaction_fast_ok(const unsigned stat[3], int64_t nnz) {
    if (stat[2]) return false;
    if (stat[0] == 0xFFFFFFFFu) return true;  // every value is ±0
    int t = 0;
    while (t < 63 && (1ll << t) < nnz) ++t;  // nnz <= 2^t
    const int q = (int)stat[0] - 2048, h = (int)stat[1] - 2048;
    return h + t <= 53 + q && h + t <= 1024;
}

// ---- float values: the ordered path -----------------------------------------------------------------------------------
// key[e] = (cell << row_bits) | graph row of entry e (row_bits 0: the arrays are the graph's CSR and storage order is
// already row order), sentinel CC << row_bits for an entry with an unlabelled end point; val[e] = its value as float64;
// cnt[cell] += 1.  Index and code checks as in interaction_kernel.
template <typename IP, typename II, typename VT>
__global__ void __launch_bounds__(256) interaction_key_kernel(const IP* __restrict__ indptr, const II* __restrict__ indices,
                                                              const VT* __restrict__ data, const int32_t* __restrict__ codes, int64_t n,
                                                              int C, int row_bits, unsigned long long* __restrict__ key,
                                                              double* __restrict__ val, unsigned* __restrict__ cnt,
                                                              unsigned* __restrict__ err) {
    const unsigned long long sentinel = (unsigned long long)C * C << row_bits;
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = warp; i < n; i += nwarps) {
        const int32_t a = codes[i];
        if (a >= C && err && lane == 0) atomicOr(err, 4u);
        const int64_t beg = (int64_t)indptr[i], end = (int64_t)indptr[i + 1];
        for (int64_t e = beg + lane; e < end; e += 32) {
            const int64_t j = (int64_t)indices[e];
            unsigned long long k = sentinel;
            if (j < 0 || j >= n) {
                if (err) atomicOr(err, 2u);
            } else if ((unsigned)a < (unsigned)C) {
                const int32_t b = codes[j];
                if ((unsigned)b < (unsigned)C) {
                    const unsigned cell = (unsigned)(a * C + b);
                    k = (unsigned long long)cell << row_bits | (row_bits ? (unsigned long long)j : 0ull);
                    atomicAdd(&cnt[cell], 1u);
                }
            }
            key[e] = k;
            val[e] = sqb_cvt<double>(data[e]);
        }
    }
}

// out[cell] = +0.0 + v_0 + v_1 + ... over the cell's sorted values val[off[cell] .. off[cell + 1]), one __dadd_rn at a
// time.  One warp per cell: the lanes stage a tile of values in shared memory, lane 0 adds them in order.
constexpr int IM_TILE = 512;
__global__ void __launch_bounds__(256) interaction_chain_kernel(const double* __restrict__ val, const unsigned* __restrict__ off, int CC,
                                                                double* __restrict__ out) {
    __shared__ double tile[8][IM_TILE];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    double* s = tile[w];
    for (int64_t cell = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; cell < CC; cell += ((int64_t)gridDim.x * blockDim.x) >> 5) {
        const int64_t beg = off[cell], end = off[cell + 1];
        double acc = 0.0;
        for (int64_t t = beg; t < end; t += IM_TILE) {
            const int m = (int)min((int64_t)IM_TILE, end - t);
            for (int k = lane; k < m; k += 32) s[k] = val[t + k];
            __syncwarp();
            if (lane == 0) {
#pragma unroll 8
                for (int k = 0; k < m; ++k) acc = __dadd_rn(acc, s[k]);
            }
            __syncwarp();
        }
        if (lane == 0) out[cell] = acc;
    }
}

static int bit_width(uint64_t x) {
    int b = 0;
    while (x >> b) ++b;
    return b;
}

// ---- one graph on the device, any index and value type -----------------------------------------------------------------
// d_out (CC entries, zeroed): int64 counts (data null) or integer sums, float64 float sums.  csc: the arrays are the CSR
// of the graph's transpose (their column indices are the graph's rows).  Returns after the kernels are enqueued, except
// that float values take one synchronisation to choose between the fast and the ordered path.
template <typename IP, typename II>
static int inter_sum(sqb_ctx* c, int64_t n, int64_t nnz, const IP* ip, const II* ix, const void* data, int data_dtype, int csc,
                     const int32_t* d_codes, int C, unsigned long long* d_out, unsigned* d_err, const char* where) {
    const InterLaunch L(c, n, C);
    double* ow = reinterpret_cast<double*>(d_out);
    auto atomics = [&](auto vt, auto mode) -> int {
        using VT = typename decltype(vt)::type;
        SqbLaunchScope scope(c, SQB_K_MISC);
        interaction_kernel<IP, II, VT, decltype(mode)::value><<<L.blocks, 256, L.smem, c->stream>>>(
            ip, ix, reinterpret_cast<const VT*>(data), d_codes, n, C, L.use_smem, ow, d_out, d_err);
        SQB_POST_LAUNCH();
        return SQB_OK;
    };
    if (data_dtype < 0) return atomics(SqbType<float>(), std::integral_constant<int, IM_COUNT>());
    return sqb_dispatch_value<true>(data_dtype, where, "data_dtype", [&](auto vt) -> int {
        using VT = typename decltype(vt)::type;
        if constexpr (std::is_integral<VT>::value) {
            return atomics(vt, std::integral_constant<int, IM_INT>());
        } else {
            const VT* v = reinterpret_cast<const VT*>(data);
            if (nnz == 0) return SQB_OK;
            DevBuf<unsigned> d_stat(c->stream);
            SQB_TRY(d_stat.alloc(3));
            const unsigned init[3] = {0xFFFFFFFFu, 0u, 0u};
            unsigned stat[3];
            SQB_CUDA(cudaMemcpyAsync(d_stat.p, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
            {
                SqbLaunchScope scope(c, SQB_K_MISC);
                interaction_exp_kernel<VT><<<sqb_grid_rows(c, nnz, 256), 256, 0, c->stream>>>(v, nnz, d_stat.p);
                SQB_POST_LAUNCH();
            }
            SQB_CUDA(cudaMemcpyAsync(stat, d_stat.p, sizeof(stat), cudaMemcpyDeviceToHost, c->stream));
            SQB_CUDA(cudaStreamSynchronize(c->stream));
            if (interaction_fast_ok(stat, nnz)) return atomics(vt, std::integral_constant<int, IM_FLOAT>());
            // the ordered path
            const int CC = C * C;
            const int row_bits = csc ? bit_width((uint64_t)(n - 1)) : 0;
            const int end_bit = bit_width((uint64_t)CC) + row_bits;
            DevBuf<unsigned long long> key(c->stream), key_s(c->stream);
            DevBuf<double> val(c->stream), val_s(c->stream);
            DevBuf<unsigned> cnt(c->stream), off(c->stream);
            DevBuf<uint8_t> tmp(c->stream);
            SQB_TRY(key.alloc(nnz));
            SQB_TRY(key_s.alloc(nnz));
            SQB_TRY(val.alloc(nnz));
            SQB_TRY(val_s.alloc(nnz));
            SQB_TRY(cnt.alloc(CC + 1));
            SQB_TRY(off.alloc(CC + 1));
            SQB_CUDA(cudaMemsetAsync(cnt.p, 0, (CC + 1) * sizeof(unsigned), c->stream));
            {
                SqbLaunchScope scope(c, SQB_K_MISC);
                interaction_key_kernel<IP, II, VT><<<L.blocks, 256, 0, c->stream>>>(ip, ix, v, d_codes, n, C, row_bits, key.p, val.p, cnt.p,
                                                                                     d_err);
                SQB_POST_LAUNCH();
            }
            size_t sort_bytes = 0, scan_bytes = 0;
            SQB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, key.p, key_s.p, val.p, val_s.p, (int)nnz, 0, end_bit, c->stream));
            SQB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, cnt.p, off.p, CC + 1, c->stream));
            SQB_TRY(tmp.alloc(std::max(sort_bytes, scan_bytes)));
            SQB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, sort_bytes, key.p, key_s.p, val.p, val_s.p, (int)nnz, 0, end_bit, c->stream));
            SQB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, scan_bytes, cnt.p, off.p, CC + 1, c->stream));
            c->launches += 2;
            {
                SqbLaunchScope scope(c, SQB_K_MISC);
                interaction_chain_kernel<<<sqb_grid_rows(c, (int64_t)CC * 32, 256), 256, 0, c->stream>>>(val_s.p, off.p, CC, ow);
                SQB_POST_LAUNCH();
            }
            return SQB_OK;
        }
    });
}

// The ABI's data_dtype: -1 counts (weights = false), else the value code of sqb_dispatch_value<true>; integer and bool codes
// (3, 4, 5) write int64 sums to out_counts, float codes float64 sums to out_weighted.
static bool inter_int_out(int data_dtype) { return data_dtype < 0 || data_dtype >= 3; }

extern "C" int sqb_interaction_matrix(sqb_ctx* c, int64_t n, int64_t nnz, const uint32_t* indptr, const uint32_t* indices,
                                      const void* data, int data_dtype, const int32_t* codes, int n_cls, double* out_weighted,
                                      int64_t* out_counts) {
    static const char* where = "sqb_interaction_matrix";
    SQB_CHECK(c, SQB_ERR_INVALID, "%s: null ctx", where);
    SQB_CHECK(n >= 1 && n < 0x7FFFFFFFLL, SQB_ERR_INVALID, "%s: n=%lld out of range", where, (long long)n);
    SQB_CHECK(nnz >= 0 && nnz < 0xFFFFFFFFLL, SQB_ERR_INVALID, "%s: nnz=%lld does not fit uint32", where, (long long)nnz);
    SQB_CHECK(indptr && (indices || nnz == 0) && codes && (data_dtype < 0 || data || nnz == 0), SQB_ERR_INVALID, "%s: null argument", where);
    SQB_CHECK(n_cls >= 1 && n_cls <= 4096, SQB_ERR_INVALID, "%s: n_cls=%d out of range [1, 4096]", where, n_cls);
    SQB_CHECK(data_dtype >= -1 && data_dtype <= 5 && data_dtype != 2, SQB_ERR_INVALID,
              "%s: data_dtype must be -1 (counts), 0 (f32), 1 (f64), 3 (i32), 4 (i64) or 5 (bool)", where);
    SQB_CHECK(inter_int_out(data_dtype) ? out_counts != nullptr : out_weighted != nullptr, SQB_ERR_INVALID, "%s: null output", where);
    SQB_CHECK(indptr[0] == 0 && (int64_t)indptr[n] == nnz, SQB_ERR_INVALID, "%s: indptr inconsistent with nnz", where);
    for (int64_t i = 0; i < n; ++i) {
        SQB_CHECK(indptr[i] <= indptr[i + 1], SQB_ERR_INVALID, "%s: indptr not monotone at row %lld", where, (long long)i);
        SQB_CHECK(codes[i] < n_cls, SQB_ERR_INVALID, "%s: codes[%lld]=%d >= n_cls=%d", where, (long long)i, codes[i], n_cls);
    }
    for (int64_t e = 0; e < nnz; ++e)
        SQB_CHECK((int64_t)indices[e] < n, SQB_ERR_INVALID, "%s: column index %u at entry %lld out of range", where, indices[e], (long long)e);
    SQB_CUDA(cudaSetDevice(c->device));
    const int CC = n_cls * n_cls;
    static const size_t vsize[6] = {4, 8, 2, 4, 8, 1};
    const size_t vs = data_dtype < 0 ? 0 : vsize[data_dtype];
    DevBuf<uint32_t> d_ptr(c->stream), d_idx(c->stream);
    DevBuf<uint8_t> d_val(c->stream);
    DevBuf<int32_t> d_codes(c->stream);
    DevBuf<unsigned long long> d_out(c->stream);  // 8 bytes per bin: double or uint64
    SQB_TRY(d_ptr.alloc(n + 1));
    SQB_TRY(d_idx.alloc(nnz > 0 ? nnz : 1));
    SQB_TRY(d_val.alloc(vs && nnz > 0 ? nnz * vs : 1));
    SQB_TRY(d_codes.alloc(n));
    SQB_TRY(d_out.alloc(CC));
    SQB_CUDA(cudaMemcpyAsync(d_ptr.p, indptr, (n + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    if (nnz > 0) SQB_TRY(sqb_h2d(c, d_idx.p, indices, nnz * sizeof(uint32_t)));
    if (vs && nnz > 0) SQB_TRY(sqb_h2d(c, d_val.p, data, nnz * vs));
    SQB_CUDA(cudaMemcpyAsync(d_codes.p, codes, n * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    SQB_CUDA(cudaMemsetAsync(d_out.p, 0, (size_t)CC * 8, c->stream));
    SQB_TRY((inter_sum<uint32_t, uint32_t>(c, n, nnz, d_ptr.p, d_idx.p, d_val.p, data_dtype, 0, d_codes.p, n_cls, d_out.p, nullptr, where)));
    void* out = inter_int_out(data_dtype) ? (void*)out_counts : (void*)out_weighted;
    SQB_CUDA(cudaMemcpyAsync(out, d_out.p, (size_t)CC * 8, cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    return SQB_OK;
}

// ---- device-resident graph (sqb_interaction_matrix_device) ----------------------------------------------------------
// The caller's CSR is read in place by the kernels above: no copy.  indptr is validated first (one synchronisation);
// column indices and codes are validated by the kernels as they go, and a flagged result is discarded.
extern "C" int sqb_interaction_matrix_device(sqb_ctx* c, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices,
                                             int index_bits, int csc, const void* data, int data_dtype, const int32_t* codes, int n_cls,
                                             double* out_weighted, int64_t* out_counts, uintptr_t producer_stream) {
    static const char* where = "sqb_interaction_matrix_device";
    SQB_CHECK(c, SQB_ERR_INVALID, "%s: null ctx", where);
    SQB_CHECK(n >= 1 && n < 0x7FFFFFFFLL, SQB_ERR_INVALID, "%s: n=%lld out of range", where, (long long)n);
    SQB_CHECK(nnz >= 0 && nnz < 0xFFFFFFFFLL, SQB_ERR_INVALID, "%s: nnz=%lld does not fit uint32", where, (long long)nnz);
    SQB_CHECK(indptr && (indices || nnz == 0) && codes && (data_dtype < 0 || data || nnz == 0), SQB_ERR_INVALID, "%s: null argument", where);
    SQB_CHECK(n_cls >= 1 && n_cls <= 4096, SQB_ERR_INVALID, "%s: n_cls=%d out of range [1, 4096]", where, n_cls);
    SQB_CHECK(data_dtype >= -1 && data_dtype <= 5, SQB_ERR_INVALID, "%s: data_dtype must be -1 (counts) or a value code in [0, 5]", where);
    SQB_CHECK(inter_int_out(data_dtype) ? out_counts != nullptr : out_weighted != nullptr, SQB_ERR_INVALID, "%s: null output", where);
    SQB_CUDA(cudaSetDevice(c->device));
    const int CC = n_cls * n_cls;
    DevBuf<int32_t> d_codes(c->stream);
    DevBuf<unsigned long long> d_out(c->stream);  // 8 bytes per bin: double or uint64
    DevBuf<unsigned> d_err(c->stream);
    unsigned flag = 0;
    return sqb_read_caller_buffers(c, producer_stream, [&]() -> int {
        SQB_TRY(d_codes.alloc(n));
        SQB_TRY(d_out.alloc(CC));
        SQB_TRY(d_err.alloc(1));
        SQB_CUDA(cudaMemcpyAsync(d_codes.p, codes, n * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        SQB_CUDA(cudaMemsetAsync(d_out.p, 0, (size_t)CC * 8, c->stream));
        SQB_CUDA(cudaMemsetAsync(d_err.p, 0, sizeof(unsigned), c->stream));
        SQB_TRY(sqb_dispatch_index(indptr_bits, index_bits, where, [&](auto ip, auto ix) -> int {
            using IP = typename decltype(ip)::type;
            using II = typename decltype(ix)::type;
            const IP* p = reinterpret_cast<const IP*>(indptr);
            SQB_TRY(sqb_check_indptr(c, SQB_K_MISC, p, n, nnz, nullptr, where));
            return inter_sum<IP, II>(c, n, nnz, p, reinterpret_cast<const II*>(indices), data, data_dtype, csc, d_codes.p, n_cls, d_out.p,
                                     d_err.p, where);
        }));
        void* out = inter_int_out(data_dtype) ? (void*)out_counts : (void*)out_weighted;
        SQB_CUDA(cudaMemcpyAsync(out, d_out.p, (size_t)CC * 8, cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaMemcpyAsync(&flag, d_err.p, sizeof(unsigned), cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaStreamSynchronize(c->stream));  // the caller's buffers are no longer read
        SQB_CHECK(!(flag & 2u), SQB_ERR_INVALID, "%s: column index out of range [0, %lld)", where, (long long)n);
        SQB_CHECK(!(flag & 4u), SQB_ERR_INVALID, "%s: a code is >= n_cls=%d", where, n_cls);
        return SQB_OK;
    });
}
