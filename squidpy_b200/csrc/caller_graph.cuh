// caller_graph.cuh — a caller's n x n graph (host or device CSR / CSC) as a device CSR (caller_graph.cu).
#pragma once
#include "common.cuh"

// The ABI arguments of a caller's graph: CSR arrays (a CSC's are the CSR of its transpose), int32 / int64 indices
// (indptr_bits / index_bits), values of the dtype code data_dtype, on the host or (device_input) in device memory written
// on producer_stream.
struct SqbGraphArgs {
    int64_t n, nnz;
    const void *indptr, *indices, *data;
    int indptr_bits, index_bits, data_dtype, csc, device_input;
    uintptr_t producer_stream;
};

// Bytes per value of the dtype codes a graph may have (0 f32, 1 f64, 3 i32, 4 i64, 5 bool); 0 for the others.
int sqb_graph_value_bytes(int code);

// n in [1, 2^31 - 1), nnz in [0, 2^nnz_log2), the graph's pointers, 32- or 64-bit index arrays.  Each entry point checks
// its value dtypes itself.
int sqb_check_graph_args(const SqbGraphArgs& a, int nnz_log2, const char* where);

// Runs body(indptr, indices, data) over a caller's CSR arrays in device memory: host arrays are uploaded first (sqb_h2d into
// stream-bound buffers), device arrays are read in place once the stream has waited for the producer stream
// (sqb_read_caller_buffers).  Returns once the caller's arrays are no longer read.
template <typename F>
int sqb_with_caller_csr(sqb_ctx* c, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices, int index_bits,
                        const void* data, size_t value_bytes, int device_input, uintptr_t producer_stream, F&& body) {
    if (device_input)
        return sqb_read_caller_buffers(c, producer_stream, [&]() -> int {
            SQB_TRY(body(indptr, indices, data));
            SQB_CUDA(cudaStreamSynchronize(c->stream));  // the caller's buffers are no longer read
            return SQB_OK;
        });
    DevBuf<uint8_t> d_ip(c->stream), d_ix(c->stream), d_v(c->stream);
    const size_t ip_bytes = (size_t)(n + 1) * (indptr_bits / 8), ix_bytes = (size_t)nnz * (index_bits / 8), v_bytes = (size_t)nnz * value_bytes;
    SQB_TRY(d_ip.alloc(ip_bytes));
    SQB_TRY(d_ix.alloc(ix_bytes));
    SQB_TRY(d_v.alloc(v_bytes));
    SQB_TRY(sqb_h2d(c, d_ip.p, indptr, ip_bytes));
    if (nnz > 0) {
        SQB_TRY(sqb_h2d(c, d_ix.p, indices, ix_bytes));
        SQB_TRY(sqb_h2d(c, d_v.p, data, v_bytes));
    }
    return body(d_ip.p, d_ix.p, d_v.p);
}

// The three device forms of a caller's graph A.
//   STORED     A's entries as stored, values as below: a CSR as given (uint32 indptr), a CSC as a CSR by a stable sort on the
//              row (rows by ascending column, then storage order: scipy's tocsr), duplicates not merged.
//   CANONICAL  sorted by (row, column), duplicates summed in storage order in W (float for float32 values, double otherwise)
//              over their float64 conversions; every sum is kept, zeros included.
//   SYMMETRIC  A + Aᵀ without the diagonal and without values (indices only).  Each (row, column) sums A's entries, then
//              Aᵀ's, then the two (scipy's csr_plus_csr), in A's dtype: integers wrap at int_bits, bool is a logical or,
//              floats add in their own precision.  Only non-zero sums are kept (NaN is non-zero).
// STORED and CANONICAL values are in float64 slots; a float32 graph's are float32 numbers, a bool graph's 1.0 / 0.0.
enum class SqbGraphForm { STORED, CANONICAL, SYMMETRIC };

struct SqbGraph {
    int64_t n = 0, e = 0;
    DevBuf<uint32_t> ptr;  // n + 1
    DevBuf<int32_t> col;   // e (at least one slot)
    DevBuf<double> val;    // e, STORED and CANONICAL only
    explicit SqbGraph(cudaStream_t s) : ptr(s), col(s), val(s) {}
};

// The caller's graph (checked by sqb_check_graph_args, data_dtype one its entry point takes) as a device CSR of the given
// form; int_bits: the width integer sums wrap at (SYMMETRIC).  A malformed indptr or an index outside [0, n) raises
// SQB_ERR_INVALID.  Returns once the caller's arrays are no longer read.
int sqb_load_graph(sqb_ctx* c, const SqbGraphArgs& a, SqbGraphForm form, int int_bits, SqbGraph& g, const char* where);

// out[i] = in[0] + ... + in[i - 1] for i < m, and *total = the sum of all m (one synchronisation).  cub's launches are not
// counted in c->launches.
int sqb_exclusive_scan(sqb_ctx* c, const uint32_t* in, uint32_t* out, int64_t m, uint32_t* total);

// A stable transpose of the m column indices idx of a CSR with n columns: its entries sorted by column, row order kept within
// a column.  perm[p] is the entry at sorted position p (at least one slot), [cbeg[j], cend[j]) the positions of column j
// (0, 0 when it is empty).  The kernels count under launch class kclass.
int sqb_col_order(sqb_ctx* c, int kclass, const int32_t* idx, int64_t m, int64_t n, DevBuf<int32_t>& perm, DevBuf<int32_t>& cbeg,
                  DevBuf<int32_t>& cend);

// Column sums in row order over sqb_col_order's permutation, each added from 0 one entry after another: csum[j] over the
// float64 values wd and colT[j] over the values w in their own type, as scipy's W.sum(axis=0) adds them.  Either output may
// be null (with its input); that sum is skipped.
template <typename T>
__global__ void sqb_col_sums_kernel(const int32_t* __restrict__ cbeg, const int32_t* __restrict__ cend, const int32_t* __restrict__ perm,
                                    const double* __restrict__ wd, const T* __restrict__ w, int64_t n, double* __restrict__ csum,
                                    T* __restrict__ colT) {
    for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
        double s = 0.0;
        T t = (T)0;
        for (int32_t p = cbeg[j]; p < cend[j]; ++p) {
            const int32_t e = perm[p];
            if (csum) s = __dadd_rn(s, wd[e]);
            if (colT) t = t + w[e];
        }
        if (csum) csum[j] = s;
        if (colT) colT[j] = t;
    }
}
