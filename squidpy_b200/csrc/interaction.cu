// interaction.cu — interaction_matrix on H100 (sm_90a): cluster x cluster sums over the stored entries of a CSR graph.
//
// Replaces the reference's numba loop `_interaction_matrix` (src/squidpy/gr/_nhood.py:412-429) together with the NaN masking
// of `interaction_matrix` (:386-395): observations without a label (code < 0) are removed from rows AND columns, which for
// the sums is the same as skipping every stored entry with an unlabelled end point (no sub-matrix is built).
//   weights = false: out[a][b] = number of stored entries (i -> j) with code(i) = a, code(j) = b          (int64, exact)
//   weights = true : out[a][b] = sum of their values, accumulated in float64                             (order free:
//                    exact for integer-valued weights, |rel err| ~1e-16 * entries otherwise)
// HBM-bound: the CSR is streamed once (8-12 bytes per stored entry); the label gather hits L2.
#include "common.cuh"

// IP / II: index types of indptr / indices (uint32 for the host path's staged copy, int32 / int64 for a caller's device
// CSR read in place).  A column index outside [0, n) is skipped and raises bit 2 of *err (null: host input, validated on
// the host); a code >= C is skipped too (bit 4).  indptr must have been validated: the kernel follows it.
template <typename IP, typename II, typename VT, bool WEIGHTED>
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
            if (WEIGHTED)
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
            if (WEIGHTED) {
                const double v = sqb_cvt<double>(data[e]);
                if (use_smem)
                    atomicAdd(&s_w[bin], v);
                else
                    atomicAdd(&out_w[bin], v);
            } else {
                if (use_smem)
                    atomicAdd(&s_c[bin], 1ull);
                else
                    atomicAdd(&out_c[bin], 1ull);
            }
        }
    }
    if (use_smem) {
        __syncthreads();
        for (int i = threadIdx.x; i < CC; i += blockDim.x) {
            if (WEIGHTED) {
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

extern "C" int sqb_interaction_matrix(sqb_ctx* c, int64_t n, int64_t nnz, const uint32_t* indptr, const uint32_t* indices,
                                      const void* data, int data_dtype, const int32_t* codes, int n_cls, double* out_weighted,
                                      int64_t* out_counts) {
    SQB_CHECK(c, SQB_ERR_INVALID, "sqb_interaction_matrix: null ctx");
    SQB_CHECK(n >= 1 && n < 0x7FFFFFFFLL, SQB_ERR_INVALID, "sqb_interaction_matrix: n=%lld out of range", (long long)n);
    SQB_CHECK(nnz >= 0 && nnz < 0xFFFFFFFFLL, SQB_ERR_INVALID, "sqb_interaction_matrix: nnz=%lld does not fit uint32", (long long)nnz);
    SQB_CHECK(indptr && (indices || nnz == 0) && codes, SQB_ERR_INVALID, "sqb_interaction_matrix: null argument");
    SQB_CHECK(n_cls >= 1 && n_cls <= 4096, SQB_ERR_INVALID, "sqb_interaction_matrix: n_cls=%d out of range [1, 4096]", n_cls);
    const bool weighted = data != nullptr;
    SQB_CHECK(!weighted || data_dtype == 0 || data_dtype == 1, SQB_ERR_INVALID, "sqb_interaction_matrix: data_dtype must be 0 (f32) or 1 (f64)");
    SQB_CHECK(weighted ? out_weighted != nullptr : out_counts != nullptr, SQB_ERR_INVALID, "sqb_interaction_matrix: null output");
    SQB_CHECK(indptr[0] == 0 && (int64_t)indptr[n] == nnz, SQB_ERR_INVALID, "sqb_interaction_matrix: indptr inconsistent with nnz");
    for (int64_t i = 0; i < n; ++i) {
        SQB_CHECK(indptr[i] <= indptr[i + 1], SQB_ERR_INVALID, "sqb_interaction_matrix: indptr not monotone at row %lld", (long long)i);
        SQB_CHECK(codes[i] < n_cls, SQB_ERR_INVALID, "sqb_interaction_matrix: codes[%lld]=%d >= n_cls=%d", (long long)i, codes[i], n_cls);
    }
    for (int64_t e = 0; e < nnz; ++e)
        SQB_CHECK((int64_t)indices[e] < n, SQB_ERR_INVALID, "sqb_interaction_matrix: column index %u at entry %lld out of range", indices[e],
                  (long long)e);
    SQB_CUDA(cudaSetDevice(c->device));
    const int CC = n_cls * n_cls;
    const size_t vsize = weighted ? (data_dtype == 0 ? 4 : 8) : 0;
    DevBuf<uint32_t> d_ptr(c->stream), d_idx(c->stream);
    DevBuf<uint8_t> d_val(c->stream);
    DevBuf<int32_t> d_codes(c->stream);
    DevBuf<unsigned long long> d_out(c->stream);  // 8 bytes per bin: double or uint64
    SQB_TRY(d_ptr.alloc(n + 1));
    SQB_TRY(d_idx.alloc(nnz > 0 ? nnz : 1));
    SQB_TRY(d_val.alloc(weighted && nnz > 0 ? nnz * vsize : 1));
    SQB_TRY(d_codes.alloc(n));
    SQB_TRY(d_out.alloc(CC));
    SQB_CUDA(cudaMemcpyAsync(d_ptr.p, indptr, (n + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    if (nnz > 0) SQB_TRY(sqb_h2d(c, d_idx.p, indices, nnz * sizeof(uint32_t)));
    if (weighted && nnz > 0) SQB_TRY(sqb_h2d(c, d_val.p, data, nnz * vsize));
    SQB_CUDA(cudaMemcpyAsync(d_codes.p, codes, n * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    SQB_CUDA(cudaMemsetAsync(d_out.p, 0, (size_t)CC * 8, c->stream));
    {
        const InterLaunch L(c, n, n_cls);
        SqbLaunchScope scope(c, SQB_K_MISC);
        double* ow = reinterpret_cast<double*>(d_out.p);
        if (!weighted)
            interaction_kernel<uint32_t, uint32_t, float, false><<<L.blocks, 256, L.smem, c->stream>>>(d_ptr.p, d_idx.p, nullptr, d_codes.p, n, n_cls, L.use_smem, ow, d_out.p, nullptr);
        else if (data_dtype == 0)
            interaction_kernel<uint32_t, uint32_t, float, true><<<L.blocks, 256, L.smem, c->stream>>>(d_ptr.p, d_idx.p, reinterpret_cast<const float*>(d_val.p), d_codes.p, n, n_cls, L.use_smem, ow, d_out.p, nullptr);
        else
            interaction_kernel<uint32_t, uint32_t, double, true><<<L.blocks, 256, L.smem, c->stream>>>(d_ptr.p, d_idx.p, reinterpret_cast<const double*>(d_val.p), d_codes.p, n, n_cls, L.use_smem, ow, d_out.p, nullptr);
        SQB_POST_LAUNCH();
    }
    SQB_CUDA(cudaMemcpyAsync(weighted ? (void*)out_weighted : (void*)out_counts, d_out.p, (size_t)CC * 8, cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    return SQB_OK;
}

// ---- device-resident graph (sqb_interaction_matrix_device) ----------------------------------------------------------
// The caller's CSR is read in place by interaction_kernel<IP, II, VT>: no copy.  indptr is validated first (one
// synchronisation); column indices and codes are validated by the kernel as it goes, and a flagged result is discarded.
template <typename IP, typename II>
static int inter_device_typed(sqb_ctx* c, int64_t n, int64_t nnz, const void* indptr, const void* indices, bool weighted, const void* data,
                              int data_dtype, const int32_t* d_codes, int n_cls, unsigned long long* d_out, unsigned* d_err) {
    static const char* where = "sqb_interaction_matrix_device";
    const IP* ip = reinterpret_cast<const IP*>(indptr);
    const II* ix = reinterpret_cast<const II*>(indices);
    SQB_TRY(sqb_check_indptr(c, SQB_K_MISC, ip, n, nnz, nullptr, where));
    const InterLaunch L(c, n, n_cls);
    double* ow = reinterpret_cast<double*>(d_out);
    auto launch = [&](auto vt, auto w) -> int {
        using VT = typename decltype(vt)::type;
        SqbLaunchScope scope(c, SQB_K_MISC);
        interaction_kernel<IP, II, VT, decltype(w)::value><<<L.blocks, 256, L.smem, c->stream>>>(
            ip, ix, reinterpret_cast<const VT*>(data), d_codes, n, n_cls, L.use_smem, ow, d_out, d_err);
        SQB_POST_LAUNCH();
        return SQB_OK;
    };
    if (!weighted) return launch(SqbType<float>(), std::false_type());
    return sqb_dispatch_value<true>(data_dtype, where, "data_dtype", [&](auto vt) { return launch(vt, std::true_type()); });
}

extern "C" int sqb_interaction_matrix_device(sqb_ctx* c, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices,
                                             int index_bits, const void* data, int data_dtype, const int32_t* codes, int n_cls,
                                             double* out_weighted, int64_t* out_counts, uintptr_t producer_stream) {
    static const char* where = "sqb_interaction_matrix_device";
    SQB_CHECK(c, SQB_ERR_INVALID, "%s: null ctx", where);
    SQB_CHECK(n >= 1 && n < 0x7FFFFFFFLL, SQB_ERR_INVALID, "%s: n=%lld out of range", where, (long long)n);
    SQB_CHECK(nnz >= 0 && nnz < 0xFFFFFFFFLL, SQB_ERR_INVALID, "%s: nnz=%lld does not fit uint32", where, (long long)nnz);
    const bool weighted = out_weighted != nullptr;  // data may be null only when there are no entries
    SQB_CHECK(indptr && (indices || nnz == 0) && codes && (!weighted || data || nnz == 0), SQB_ERR_INVALID, "%s: null argument", where);
    SQB_CHECK(n_cls >= 1 && n_cls <= 4096, SQB_ERR_INVALID, "%s: n_cls=%d out of range [1, 4096]", where, n_cls);
    SQB_CHECK(weighted || out_counts != nullptr, SQB_ERR_INVALID, "%s: null output", where);
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
        SQB_TRY(sqb_dispatch_index(indptr_bits, index_bits, where, [&](auto ip, auto ix) {
            return inter_device_typed<typename decltype(ip)::type, typename decltype(ix)::type>(c, n, nnz, indptr, indices, weighted, data,
                                                                                                data_dtype, d_codes.p, n_cls, d_out.p, d_err.p);
        }));
        SQB_CUDA(cudaMemcpyAsync(weighted ? (void*)out_weighted : (void*)out_counts, d_out.p, (size_t)CC * 8, cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaMemcpyAsync(&flag, d_err.p, sizeof(unsigned), cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaStreamSynchronize(c->stream));  // the caller's buffers are no longer read
        SQB_CHECK(!(flag & 2u), SQB_ERR_INVALID, "%s: column index out of range [0, %lld)", where, (long long)n);
        SQB_CHECK(!(flag & 4u), SQB_ERR_INVALID, "%s: a code is >= n_cls=%d", where, n_cls);
        return SQB_OK;
    });
}
