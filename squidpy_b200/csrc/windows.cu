// windows.cu — which sliding windows contain each observation, on the GPU (sm_90a).
//
// Replaces the per-window boolean masks of the reference's tl.sliding_window (src/squidpy/tl/_sliding_window.py:130-158):
// `x_start <= x <= x_end and y_start <= y <= y_end` over every observation for every window, a cost that grows as windows x
// observations.  A library's windows are the product of its x windows and its y windows (_calculate_window_corners,
// :224-242), and along one axis both the starts (an np.arange with a positive step) and the ends (start + window_size, clipped
// to the maximum) are non-decreasing.  The windows of an axis that contain v are therefore one contiguous index range:
//   hi = the last i with start[i] <= v,   lo = the first i with end[i] >= v,
// both found by binary search, and the observation lies in window (ix, iy) iff lo_x <= ix <= hi_x and lo_y <= iy <= hi_y.
// The host turns the four numbers into the reference's labels or columns; the edges themselves are computed on the host with
// the reference's numpy calls and only compared here, in the dtype numpy compares them in (float64, or int64 when every
// edge and coordinate is an integer), so no edge is ever recomputed on the device.
#include <cmath>

#include "common.cuh"

#define WR_THREADS 256

// Number of entries of the non-decreasing a[0 .. m) that are <= v (LE) or < v (!LE); 0 for a NaN v.
template <bool LE, typename T>
__device__ __forceinline__ int32_t wr_count(const T* __restrict__ a, int32_t m, T v) {
    int32_t lo = 0, hi = m;
    while (lo < hi) {
        const int32_t mid = (lo + hi) >> 1;
        const T e = __ldg(a + mid);
        if (LE ? e <= v : e < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// One thread per observation: out[i] = {lo_x, hi_x, lo_y, hi_y}; {0, -1, 0, -1} for an observation of no library.
template <typename T>
__global__ void __launch_bounds__(WR_THREADS) wr_ranges_kernel(const T* __restrict__ xy, const int32_t* __restrict__ lib, int64_t n,
                                                               const int64_t* __restrict__ off, const T* __restrict__ starts,
                                                               const T* __restrict__ ends, int4* __restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t l = lib[i];
    int4 r = make_int4(0, -1, 0, -1);
    if (l >= 0) {
        const int64_t bx = off[2 * l], by = off[2 * l + 1], e = off[2 * l + 2];
        const T x = xy[2 * i], y = xy[2 * i + 1];
        r.x = wr_count<false>(ends + bx, (int32_t)(by - bx), x);
        r.y = wr_count<true>(starts + bx, (int32_t)(by - bx), x) - 1;
        r.z = wr_count<false>(ends + by, (int32_t)(e - by), y);
        r.w = wr_count<true>(starts + by, (int32_t)(e - by), y) - 1;
    }
    out[i] = r;
}

template <typename T>
static int wr_run(sqb_ctx* c, const T* xy, int64_t n, const int32_t* lib, int n_libs, const int64_t* off, const T* starts, const T* ends,
                  int32_t* out) {
    static const char* where = "sqb_window_ranges";
    const int64_t n_edges = off[2 * (int64_t)n_libs];
    for (int64_t s = 0; s < 2 * (int64_t)n_libs; ++s)  // every range first: the edge arrays end at the last offset
        SQB_CHECK(off[s] <= off[s + 1] && off[s + 1] - off[s] < 2147483647LL, SQB_ERR_INVALID,
                  "%s: edge_off[%lld .. %lld] = %lld .. %lld is not a range of fewer than 2^31 - 1 edges", where, (long long)s,
                  (long long)s + 1, (long long)off[s], (long long)off[s + 1]);
    for (int64_t s = 0; s < 2 * (int64_t)n_libs; ++s) {
        for (int64_t k = off[s] + 1; k < off[s + 1]; ++k)
            SQB_CHECK(starts[k - 1] <= starts[k] && ends[k - 1] <= ends[k], SQB_ERR_INVALID,
                      "%s: the edges of library %lld, axis %lld decrease (or are NaN) at %lld", where, (long long)(s / 2), (long long)(s % 2),
                      (long long)(k - off[s]));
    }
    for (int64_t i = 0; i < n; ++i)
        SQB_CHECK(lib[i] >= -1 && lib[i] < n_libs, SQB_ERR_INVALID, "%s: lib[%lld] = %d is outside [-1, %d)", where, (long long)i, lib[i], n_libs);
    if (n == 0) return SQB_OK;
    SQB_CUDA(cudaSetDevice(c->device));
    DevBuf<T> d_xy(c->stream), d_starts(c->stream), d_ends(c->stream);
    DevBuf<int32_t> d_lib(c->stream);
    DevBuf<int64_t> d_off(c->stream);
    DevBuf<int4> d_out(c->stream);
    SQB_TRY(d_xy.alloc(2 * (size_t)n));
    SQB_TRY(d_lib.alloc((size_t)n));
    SQB_TRY(d_off.alloc(2 * (size_t)n_libs + 1));
    SQB_TRY(d_starts.alloc((size_t)n_edges));
    SQB_TRY(d_ends.alloc((size_t)n_edges));
    SQB_TRY(d_out.alloc((size_t)n));
    SQB_TRY(sqb_h2d(c, d_xy.p, xy, 2 * (size_t)n * sizeof(T)));
    SQB_TRY(sqb_h2d(c, d_lib.p, lib, (size_t)n * sizeof(int32_t)));
    SQB_CUDA(cudaMemcpyAsync(d_off.p, off, (2 * (size_t)n_libs + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
    if (n_edges > 0) {
        SQB_CUDA(cudaMemcpyAsync(d_starts.p, starts, (size_t)n_edges * sizeof(T), cudaMemcpyHostToDevice, c->stream));
        SQB_CUDA(cudaMemcpyAsync(d_ends.p, ends, (size_t)n_edges * sizeof(T), cudaMemcpyHostToDevice, c->stream));
    }
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        wr_ranges_kernel<T><<<(unsigned)ceil_div64(n, WR_THREADS), WR_THREADS, 0, c->stream>>>(d_xy.p, d_lib.p, n, d_off.p, d_starts.p,
                                                                                              d_ends.p, d_out.p);
        SQB_POST_LAUNCH();
    }
    SQB_CUDA(cudaMemcpyAsync(out, d_out.p, (size_t)n * sizeof(int4), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    return SQB_OK;
}

extern "C" int sqb_window_ranges(sqb_ctx* ctx, const void* xy, int xy_dtype, int64_t n, const int32_t* lib, int n_libs, const int64_t* edge_off,
                                 const void* starts, const void* ends, int32_t* out) {
    static const char* where = "sqb_window_ranges";
    SQB_CHECK(ctx && edge_off && (n == 0 || (xy && lib && out)), SQB_ERR_INVALID, "%s: null argument", where);
    SQB_CHECK(n >= 0 && n < 2147483648LL, SQB_ERR_INVALID, "%s: n=%lld outside [0, 2^31)", where, (long long)n);
    SQB_CHECK(n_libs >= 0 && n_libs < (1 << 30), SQB_ERR_INVALID, "%s: n_libs=%d outside [0, 2^30)", where, n_libs);
    SQB_CHECK(xy_dtype == 0 || xy_dtype == 1, SQB_ERR_INVALID, "%s: xy_dtype=%d is not 0 (float64) or 1 (int64)", where, xy_dtype);
    SQB_CHECK(edge_off[0] == 0, SQB_ERR_INVALID, "%s: edge_off[0] = %lld, expected 0", where, (long long)edge_off[0]);
    SQB_CHECK(edge_off[2 * (int64_t)n_libs] == 0 || (starts && ends), SQB_ERR_INVALID, "%s: null edge array", where);
    if (xy_dtype == 0)
        return wr_run<double>(ctx, (const double*)xy, n, lib, n_libs, edge_off, (const double*)starts, (const double*)ends, out);
    return wr_run<int64_t>(ctx, (const int64_t*)xy, n, lib, n_libs, edge_off, (const int64_t*)starts, (const int64_t*)ends, out);
}
