// dense.cu — a dense block gathered from a caller's device-resident expression matrix (sm_90a), and the observed statistics
// of ligrec on it.
//
// sqb_dense_gather_device reads the caller's X in place (CSR, CSC or strided dense, values f32 / f64 / f16 / int32 / int64)
// and writes the selected rows x selected columns into a context-owned dense matrix: observations x genes row-major (what
// ligrec_group_means_kernel reads) or genes x observations (what sepal_kernel reads).  One pass per call: one warp per
// stored row (CSR) or column (CSC) of the selection, writing through the row / column maps; one thread per output cell for
// dense input.  Values are converted to float64 exactly (the host's astype(float64)) or kept in their own type.
//
// Duplicates: a per-output-cell bitmap (atomicOr) finds two stored entries that land in the same gathered cell; such input is
// rejected.  scipy's toarray() sums them on the host, so this is the one input on which host and device differ; duplicates in
// rows or columns that are not gathered are never read.
//
// ligrec_observed_kernel: the per-cluster mean of every gathered gene as pandas' groupby(...).mean() computes it — a Kahan
// sum per (cluster, gene) in cell order, whose NaN compensation is reset (so +-inf inputs give +-inf), divided by the count
// — plus the number of positive values (the expression-fraction mask).  Lane = gene, cells walked in order, accumulators
// [cluster][lane] in shared memory; __dadd_rn / __dsub_rn / __ddiv_rn keep the compiler from contracting or reassociating.
#include <math.h>

#include "common.cuh"

namespace {

enum { DG_ERR_INDEX = 2u, DG_ERR_DUP = 4u };

template <typename T>
__device__ __forceinline__ T dg_nan0(T v) { return v; }  // integers have no NaN
__device__ __forceinline__ float dg_nan0(float v) { return v != v ? 0.0f : v; }
__device__ __forceinline__ double dg_nan0(double v) { return v != v ? 0.0 : v; }
__device__ __forceinline__ __half dg_nan0(__half v) { return __hisnan(v) ? __float2half(0.0f) : v; }

template <typename VT>
__device__ __forceinline__ void dg_store(void* out, int64_t cell, VT v, bool nan0, bool keep) {
    if (nan0) v = dg_nan0(v);
    if (keep)
        reinterpret_cast<VT*>(out)[cell] = v;
    else
        reinterpret_cast<double*>(out)[cell] = sqb_cvt<double>(v);
}

// CSR (major = observations) or CSC (major = genes): one warp per selected major segment.  maj_map / min_map: the output index
// of every input row / column, or -1.  Every index read is checked against [0, n_minor).
template <typename IP, typename II, typename VT>
__global__ void __launch_bounds__(256, 1) dg_sparse_kernel(const IP* __restrict__ indptr, const II* __restrict__ indices,
                                                        const VT* __restrict__ vals, int64_t n_major, int64_t n_minor,
                                                        const int32_t* __restrict__ maj_map, const int32_t* __restrict__ min_map,
                                                        int csr, int layout, int64_t n_obs_out, int64_t n_genes_out, int nan0,
                                                        int keep, void* __restrict__ out, unsigned* __restrict__ bitmap,
                                                        unsigned* __restrict__ err) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t s = warp; s < n_major; s += nwarps) {
        const int32_t mo = maj_map[s];  // warp uniform
        if (mo < 0) continue;
        const int64_t beg = (int64_t)indptr[s], end = (int64_t)indptr[s + 1];
        for (int64_t e = beg + lane; e < end; e += 32) {
            const int64_t j = (int64_t)indices[e];
            if (j < 0 || j >= n_minor) {
                atomicOr(err, DG_ERR_INDEX);
                continue;
            }
            const int32_t no = min_map[j];
            if (no < 0) continue;
            const int64_t obs = csr ? mo : no, gene = csr ? no : mo;
            const int64_t cell = layout == 0 ? obs * n_genes_out + gene : gene * n_obs_out + obs;
            const unsigned bit = 1u << (cell & 31);
            if (atomicOr(bitmap + (cell >> 5), bit) & bit) {
                atomicOr(err, DG_ERR_DUP);
                continue;
            }
            dg_store(out, cell, vals[e], nan0, keep);
        }
    }
}

// strided dense input (rows = observations): one thread per output cell, written in output order
template <typename VT>
__global__ void __launch_bounds__(256, 1) dg_dense_kernel(const VT* __restrict__ x, int64_t stride_row, int64_t stride_col,
                                                       const int64_t* __restrict__ rows, const int32_t* __restrict__ cols,
                                                       int layout, int64_t n_obs_out, int64_t n_genes_out, int nan0, int keep,
                                                       void* __restrict__ out) {
    const int64_t total = n_obs_out * n_genes_out;
    for (int64_t cell = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; cell < total; cell += (int64_t)gridDim.x * blockDim.x) {
        const int64_t obs = layout == 0 ? cell / n_genes_out : cell % n_obs_out;
        const int64_t gene = layout == 0 ? cell % n_genes_out : cell / n_obs_out;
        dg_store(out, cell, x[rows[obs] * stride_row + (int64_t)cols[gene] * stride_col], nan0, keep);
    }
}

const size_t kDtypeSize[5] = {4, 8, 2, 4, 8};

}  // namespace

// ---- ligrec observed statistics ---------------------------------------------------------------------------------------
// wpb warps per block, each owning 32 genes; shared memory per warp: sum and compensation [n_cls][32] (double) and the
// positive count [n_cls][32] (int).
__global__ void __launch_bounds__(128, 1) ligrec_observed_kernel(const double* __restrict__ data, const int32_t* __restrict__ codes,
                                                              int64_t n_cells, int n_genes, int n_cls, const double* __restrict__ sizes,
                                                              double* __restrict__ mean, long long* __restrict__ npos) {
    extern __shared__ double lo_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double* __restrict__ s_sum = lo_smem + (size_t)warp * n_cls * 32 * 2 + lane;
    double* __restrict__ s_comp = s_sum + (size_t)n_cls * 32;
    int* __restrict__ s_pos = reinterpret_cast<int*>(lo_smem + (size_t)(blockDim.x >> 5) * n_cls * 32 * 2) + (size_t)warp * n_cls * 32 + lane;
    for (int k = 0; k < n_cls; ++k) s_sum[k * 32] = 0.0, s_comp[k * 32] = 0.0, s_pos[k * 32] = 0;
    const int g = (blockIdx.x * (blockDim.x >> 5) + warp) * 32 + lane;
    const bool ok = g < n_genes;
    const double* __restrict__ col = data + (ok ? g : 0);
    for (int64_t c = 0; c < n_cells; ++c) {
        const int k = codes[c] * 32;
        const double v = col[c * n_genes];
        const double sum = s_sum[k];
        const double y = __dsub_rn(v, s_comp[k]);
        const double t = __dadd_rn(sum, y);
        const double comp = __dsub_rn(__dsub_rn(t, sum), y);
        s_comp[k] = isnan(comp) ? 0.0 : comp;
        s_sum[k] = t;
        s_pos[k] += v > 0.0 ? 1 : 0;
    }
    if (ok)
        for (int k = 0; k < n_cls; ++k) {
            mean[(size_t)k * n_genes + g] = __ddiv_rn(s_sum[k * 32], sizes[k]);
            npos[(size_t)k * n_genes + g] = s_pos[k * 32];
        }
}

extern "C" {

int sqb_dense_gather_device(sqb_ctx* ctx, int format, const void* x, const void* indptr, int indptr_bits, const void* indices,
                            int index_bits, int64_t nnz, int x_dtype, int64_t n_rows, int64_t n_cols, int64_t stride_row,
                            int64_t stride_col, const int64_t* rows, int64_t n_rows_out, const int32_t* cols, int64_t n_cols_out,
                            int layout, int flags, uintptr_t producer_stream, sqb_dense** out) {
    static const char* where = "sqb_dense_gather_device";
    SQB_CHECK(ctx && out && cols && (x || (format != 0 && nnz == 0)), SQB_ERR_INVALID, "%s: null argument", where);
    SQB_CHECK(format >= 0 && format <= 2, SQB_ERR_INVALID, "%s: format must be 0 (dense), 1 (CSR) or 2 (CSC)", where);
    SQB_CHECK(layout == 0 || layout == 1, SQB_ERR_INVALID, "%s: layout must be 0 or 1", where);
    SQB_CHECK((flags & ~3) == 0, SQB_ERR_INVALID, "%s: unknown flags %d", where, flags);
    SQB_CHECK(n_rows >= 1 && n_rows < 2147483647LL && n_cols >= 1 && n_cols < 2147483647LL, SQB_ERR_INVALID, "%s: bad shape (%lld, %lld)",
              where, (long long)n_rows, (long long)n_cols);
    if (!rows) n_rows_out = n_rows;
    SQB_CHECK(n_rows_out >= 1 && n_rows_out <= n_rows && n_cols_out >= 1 && n_cols_out <= n_cols, SQB_ERR_INVALID,
              "%s: %lld rows x %lld columns selected of (%lld, %lld)", where, (long long)n_rows_out, (long long)n_cols_out, (long long)n_rows,
              (long long)n_cols);
    if (format != 0) {
        SQB_CHECK(indptr && (indices || nnz == 0), SQB_ERR_INVALID, "%s: null sparse arrays", where);
        SQB_CHECK(nnz >= 0, SQB_ERR_INVALID, "%s: nnz=%lld", where, (long long)nnz);
    }
    // row / column maps on the host: input index -> output index or -1
    std::vector<int32_t> rmap, cmap((size_t)n_cols, -1);
    std::vector<int64_t> rlist;
    for (int64_t k = 0; k < n_cols_out; ++k) {
        SQB_CHECK(cols[k] >= 0 && cols[k] < n_cols && cmap[cols[k]] < 0, SQB_ERR_INVALID, "%s: column %d is out of range or selected twice",
                  where, cols[k]);
        cmap[cols[k]] = (int32_t)k;
    }
    if (rows) {
        for (int64_t k = 0; k < n_rows_out; ++k)
            SQB_CHECK(rows[k] >= 0 && rows[k] < n_rows && (k == 0 || rows[k] > rows[k - 1]), SQB_ERR_INVALID,
                      "%s: the selected rows must be ascending indices in [0, %lld)", where, (long long)n_rows);
    }
    if (format == 0) {
        rlist.resize((size_t)n_rows_out);
        for (int64_t k = 0; k < n_rows_out; ++k) rlist[k] = rows ? rows[k] : k;
    } else {
        rmap.assign((size_t)n_rows, rows ? -1 : 0);
        for (int64_t k = 0; k < n_rows_out; ++k) rmap[rows ? rows[k] : k] = (int32_t)k;
    }
    sqb_ctx* c = ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    const bool keep = flags & 2, nan0 = flags & 1;
    std::unique_ptr<sqb_dense> d(new sqb_dense(c));
    d->n_obs = n_rows_out, d->n_genes = n_cols_out, d->layout = layout, d->dtype = keep ? x_dtype : 1, d->nan_zero = nan0;
    const int64_t cells = n_rows_out * n_cols_out;
    DevBuf<int32_t> d_rmap(c->stream), d_cmap(c->stream);
    DevBuf<int64_t> d_rlist(c->stream);
    DevBuf<unsigned> d_bits(c->stream), d_err(c->stream);
    unsigned flag = 0;
    auto gather = [&](auto vt) -> int {
        using VT = typename decltype(vt)::type;
        SQB_TRY(d->buf.alloc((size_t)cells * kDtypeSize[d->dtype]));
        SQB_TRY(d_cmap.alloc(format == 0 ? n_cols_out : n_cols));
        if (format == 0) {
            SQB_TRY(d_rlist.alloc(n_rows_out));
            SQB_CUDA(cudaMemcpyAsync(d_cmap.p, cols, n_cols_out * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
            SQB_CUDA(cudaMemcpyAsync(d_rlist.p, rlist.data(), n_rows_out * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
            SqbLaunchScope scope(c, SQB_K_MISC);
            dg_dense_kernel<VT><<<sqb_grid_rows(c, cells, 256), 256, 0, c->stream>>>(reinterpret_cast<const VT*>(x), stride_row, stride_col,
                                                                                     d_rlist.p, d_cmap.p, layout, n_rows_out, n_cols_out,
                                                                                     nan0, keep, d->buf.p);
            SQB_POST_LAUNCH();
            SQB_CUDA(cudaStreamSynchronize(c->stream));  // the caller's buffer is no longer read
            return SQB_OK;
        }
        const bool csr = format == 1;
        const int64_t n_major = csr ? n_rows : n_cols, n_minor = csr ? n_cols : n_rows;
        SQB_TRY(d_rmap.alloc(n_rows));
        SQB_TRY(d_bits.alloc((size_t)ceil_div64(cells, 32)));
        SQB_TRY(d_err.alloc(1));
        SQB_CUDA(cudaMemcpyAsync(d_rmap.p, rmap.data(), n_rows * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        SQB_CUDA(cudaMemcpyAsync(d_cmap.p, cmap.data(), n_cols * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        SQB_CUDA(cudaMemsetAsync(d->buf.p, 0, (size_t)cells * kDtypeSize[d->dtype], c->stream));
        SQB_CUDA(cudaMemsetAsync(d_bits.p, 0, (size_t)ceil_div64(cells, 32) * sizeof(unsigned), c->stream));
        SQB_CUDA(cudaMemsetAsync(d_err.p, 0, sizeof(unsigned), c->stream));
        SQB_TRY(sqb_dispatch_index(indptr_bits, index_bits, where, [&](auto ipt, auto ixt) -> int {
            using IP = typename decltype(ipt)::type;
            using II = typename decltype(ixt)::type;
            const IP* ip = reinterpret_cast<const IP*>(indptr);
            SQB_TRY(sqb_check_indptr(c, SQB_K_MISC, ip, n_major, nnz, nullptr, where));  // the gather follows it
            SqbLaunchScope scope(c, SQB_K_MISC);
            dg_sparse_kernel<IP, II, VT><<<sqb_grid_rows(c, n_major * 32, 256), 256, 0, c->stream>>>(
                ip, reinterpret_cast<const II*>(indices), reinterpret_cast<const VT*>(x), n_major, n_minor, csr ? d_rmap.p : d_cmap.p,
                csr ? d_cmap.p : d_rmap.p, csr, layout, n_rows_out, n_cols_out, nan0, keep, d->buf.p, d_bits.p, d_err.p);
            SQB_POST_LAUNCH();
            return SQB_OK;
        }));
        SQB_CUDA(cudaMemcpyAsync(&flag, d_err.p, sizeof(unsigned), cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaStreamSynchronize(c->stream));  // the caller's buffers are no longer read
        SQB_CHECK(!(flag & DG_ERR_INDEX), SQB_ERR_INVALID, "%s: index out of range [0, %lld)", where, (long long)n_minor);
        SQB_CHECK(!(flag & DG_ERR_DUP), SQB_ERR_INVALID,
                  "%s: two stored entries fall into the same gathered cell (duplicate entries; sum them first, e.g. scipy's "
                  "sum_duplicates())",
                  where);
        return SQB_OK;
    };
    SQB_TRY(sqb_read_caller_buffers(c, producer_stream, [&] { return sqb_dispatch_value(x_dtype, where, "x_dtype", gather); }));
    *out = d.release();
    return SQB_OK;
}

int sqb_dense_download(sqb_dense* d, void* out) {
    SQB_CHECK(d && out, SQB_ERR_INVALID, "sqb_dense_download: null argument");
    sqb_ctx* c = d->ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    SQB_CUDA(cudaMemcpyAsync(out, d->buf.p, (size_t)d->n_obs * d->n_genes * kDtypeSize[d->dtype], cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    return SQB_OK;
}

int sqb_dense_free(sqb_dense* d) {
    if (!d) return SQB_OK;
    cudaSetDevice(d->ctx->device);
    delete d;
    return SQB_OK;
}

int sqb_ligrec_observed(sqb_dense* d, const int32_t* codes, int n_cls, double* mean_out, int64_t* npos_out, int64_t* sizes_out) {
    static const char* where = "sqb_ligrec_observed";
    SQB_CHECK(d && codes && mean_out && npos_out && sizes_out, SQB_ERR_INVALID, "%s: null argument", where);
    SQB_CHECK(d->layout == 0 && d->dtype == 1 && d->nan_zero, SQB_ERR_INVALID,
              "%s: the matrix must be gathered as observations x genes float64 with NaN written as 0", where);
    SQB_CHECK(d->n_genes < 2147483647LL, SQB_ERR_INVALID, "%s: too many genes", where);
    sqb_ctx* c = d->ctx;
    SQB_CHECK(n_cls >= 1, SQB_ERR_INVALID, "%s: n_cls=%d", where, n_cls);
    const size_t per_warp = (size_t)n_cls * 32 * (2 * sizeof(double) + sizeof(int));
    SQB_CHECK(per_warp <= c->smem_optin, SQB_ERR_UNSUPPORTED, "%s: %d clusters exceed the shared-memory accumulators", where, n_cls);
    const int64_t n = d->n_obs, G = d->n_genes;
    std::vector<double> sizes((size_t)n_cls, 0.0);
    for (int64_t k = 0; k < n_cls; ++k) sizes_out[k] = 0;
    for (int64_t i = 0; i < n; ++i) {
        SQB_CHECK(codes[i] >= 0 && codes[i] < n_cls, SQB_ERR_INVALID, "%s: code %d out of range [0, %d)", where, codes[i], n_cls);
        sizes_out[codes[i]] += 1;
    }
    for (int k = 0; k < n_cls; ++k) sizes[k] = (double)sizes_out[k];
    int wpb = (int)(c->smem_optin / per_warp);
    wpb = wpb > 4 ? 4 : wpb;
    const size_t smem = per_warp * wpb;
    SQB_CUDA(cudaSetDevice(c->device));
    DevBuf<int32_t> d_codes(c->stream);
    DevBuf<double> d_sizes(c->stream), d_mean(c->stream);
    DevBuf<long long> d_npos(c->stream);
    auto body = [&]() -> int {
        SQB_TRY(d_codes.alloc(n));
        SQB_TRY(d_sizes.alloc(n_cls));
        SQB_TRY(d_mean.alloc((size_t)n_cls * G));
        SQB_TRY(d_npos.alloc((size_t)n_cls * G));
        SQB_CUDA(cudaMemcpyAsync(d_codes.p, codes, n * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        SQB_CUDA(cudaMemcpyAsync(d_sizes.p, sizes.data(), n_cls * sizeof(double), cudaMemcpyHostToDevice, c->stream));
        if (smem > 48 * 1024) SQB_CUDA(cudaFuncSetAttribute(ligrec_observed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        {
            SqbLaunchScope scope(c, SQB_K_MISC);
            ligrec_observed_kernel<<<(unsigned)ceil_div64(G, 32 * wpb), 32 * wpb, smem, c->stream>>>(
                reinterpret_cast<const double*>(d->buf.p), d_codes.p, n, (int)G, n_cls, d_sizes.p, d_mean.p, d_npos.p);
            SQB_POST_LAUNCH();
        }
        SQB_CUDA(cudaMemcpyAsync(mean_out, d_mean.p, (size_t)n_cls * G * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaMemcpyAsync(npos_out, d_npos.p, (size_t)n_cls * G * sizeof(long long), cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaStreamSynchronize(c->stream));
        return SQB_OK;
    };
    const int rc = body();
    if (rc != SQB_OK) cudaStreamSynchronize(c->stream);
    return rc;
}

}  // extern "C"
