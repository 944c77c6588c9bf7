// common.cuh — shared host/device plumbing for libsquidpy_b200 (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/squidpy_b200.h"

// ---------------------------------------------------------------------------------------------
// error handling: every C-ABI entry point returns 0 on success or a negative sqb_status; the message is
// kept in a thread-local buffer readable through sqb_last_error().
// ---------------------------------------------------------------------------------------------
void sqb_set_error(const char* fmt, ...);

#define SQB_CUDA(call)                                                                              \
    do {                                                                                            \
        cudaError_t _e = (call);                                                                    \
        if (_e != cudaSuccess) {                                                                    \
            sqb_set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__,  \
                          cudaGetErrorString(_e));                                                  \
            return SQB_ERR_CUDA;                                                                    \
        }                                                                                           \
    } while (0)

#define SQB_CHECK(cond, code, ...)   \
    do {                             \
        if (!(cond)) {               \
            sqb_set_error(__VA_ARGS__); \
            return (code);           \
        }                            \
    } while (0)

#define SQB_TRY(expr)           \
    do {                        \
        int _rc = (expr);       \
        if (_rc != SQB_OK) return _rc; \
    } while (0)

// kernel classes for the per-class launch accounting / event timing (sqb_ctx_profile_get)
enum {
    SQB_K_NHOOD_FILL = 0,
    SQB_K_NHOOD_SHUFFLE = 1,
    SQB_K_NHOOD_TRANSPOSE = 2,
    SQB_K_NHOOD_COUNT = 3,
    SQB_K_AUTOCORR_PREP = 4,
    SQB_K_AUTOCORR_MAIN = 5,
    SQB_K_AUTOCORR_FINAL = 6,
    SQB_K_PAIRS = 7,
    SQB_K_MISC = 8,
    SQB_K_NCLASS = 16
};

struct sqb_ctx;

// A device buffer that owns its allocation: the destructor frees it, so a buffer is freed when the local or the handle
// holding it goes away, on every return path.  release() frees it earlier on purpose.  Buffers move but do not copy.
// A default-constructed buffer uses synchronous cudaMalloc / cudaFree.  A buffer constructed with a stream uses the
// stream-ordered allocator (cudaMallocAsync / cudaFreeAsync on that stream, from the device's default memory pool, whose
// release threshold sqb_ctx_create raises so freed blocks are reused): creating and destroying a handle per API call then
// costs microseconds instead of ~1 ms of device synchronisation per buffer.  Its free is enqueued on the stream, so a
// stream-bound buffer must be destroyed before its stream is.
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    cudaStream_t stream = nullptr;
    bool async = false;
    DevBuf() = default;
    explicit DevBuf(cudaStream_t s) : stream(s), async(true) {}
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n), stream(o.stream), async(o.async) { o.p = nullptr, o.n = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) {
            release();
            p = o.p, n = o.n, stream = o.stream, async = o.async;
            o.p = nullptr, o.n = 0;
        }
        return *this;
    }
    ~DevBuf() { release(); }
    int alloc(size_t count) {
        if (count <= n && p) return SQB_OK;
        release();
        if (count == 0) count = 1;
        cudaError_t e = async ? cudaMallocAsync((void**)&p, count * sizeof(T), stream) : cudaMalloc((void**)&p, count * sizeof(T));
        if (e != cudaSuccess) {
            p = nullptr;
            n = 0;
            sqb_set_error("device allocation of %zu bytes failed: %s", count * sizeof(T), cudaGetErrorString(e));
            return SQB_ERR_OOM;
        }
        n = count;
        return SQB_OK;
    }
    void release() {
        if (p) {
            if (async)
                cudaFreeAsync(p, stream);
            else
                cudaFree(p);
        }
        p = nullptr;
        n = 0;
    }
};

struct sqb_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int sm_count = 132;
    size_t l2_bytes = (size_t)50 << 20;
    size_t smem_optin = 0;   // max opt-in dynamic shared memory per block
    size_t smem_per_sm = 0;  // shared memory per SM, shared by its resident blocks
    size_t smem_reserved = 0;  // shared memory the system reserves for every resident block
    int64_t launches = 0;
    bool profile = false;
    double k_ms[SQB_K_NCLASS] = {0};
    int64_t k_n[SQB_K_NCLASS] = {0};
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaEvent_t ev_in0 = nullptr, ev_in1 = nullptr;  // profile events of a launch timed inside another launch's scope
    // Second stream at the device's greatest priority, owned by the context: the region replay's last round runs on it, so
    // that the block scheduler places its CTAs before those of the transpose the context stream runs beside it (nhood.cu,
    // launch_shuffle_part).  fork (fired once every CTA of the whole rounds has begun) / join order it with the context stream.
    cudaStream_t tail = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    // Large scratch buffers that live as long as the context (GB-sized cudaMalloc/cudaFree per API call would
    // otherwise dominate the host-facing latency).  Work on one ctx is stream ordered, so handles can share them.
    DevBuf<uint8_t> scratch[4];
    // pinned staging ring for large host-to-device copies of pageable caller memory (sqb_h2d)
    static constexpr int kStage = 16;
    void* stage[kStage] = {};
    cudaEvent_t stage_ev[kStage] = {};
    bool stage_used[kStage] = {};
};

// A dense matrix gathered from a caller's device X (sqb_dense_gather_device, dense.cu): n_obs x n_genes row-major (layout 0)
// or n_genes x n_obs row-major (layout 1), float64 (dtype 1) or the input's own value type (DTYPE_CODES of _device.py).
struct sqb_dense {
    explicit sqb_dense(sqb_ctx* c) : ctx(c) {}
    sqb_ctx* ctx;
    DevBuf<uint8_t> buf{ctx->stream};  // in ctx->stream order (ctx is declared first: this initialiser reads it)
    int64_t n_obs = 0, n_genes = 0;
    int layout = 0, dtype = 1;
    bool nan_zero = false;  // NaN entries were written as 0.0
};

// Host-to-device copy of caller-owned (pageable) memory on the ctx stream.  Large copies go through a ring of pinned
// staging buffers filled by several host threads while the previous chunk is on the bus: a plain cudaMemcpyAsync from
// pageable memory is bounded by the host's single-threaded page-locking copy.
// The source has been read completely when the call returns; the copy itself completes in stream order.
int sqb_h2d(sqb_ctx* c, void* dst, const void* src, size_t bytes);
int sqb_h2d_gather(sqb_ctx* c, void* dst, const void* src, size_t elem, const int64_t* start, const int64_t* cnt,
                   const int64_t* out_ptr, int64_t rows);

// Device-resident caller arrays: make the context's stream wait for the caller's producer stream before it reads them
// (CUDA Array Interface v3 `stream`: 0 none, 1 legacy default stream, 2 per-thread default stream, else a cudaStream_t).
int sqb_wait_producer(sqb_ctx* c, uintptr_t producer);

// Launch accounting.  In profile mode each launch is bracketed by events on the ctx stream and the elapsed
// time accumulated per kernel class (the launch is synchronised; never used inside a timed bench region
// except for the dedicated roofline pass).  A scope opened inside another one passes inner = true: it takes the second
// pair of events, and its time overlaps the outer scope's.
struct SqbLaunchScope {
    sqb_ctx* c;
    int kclass;
    cudaEvent_t e0, e1;
    SqbLaunchScope(sqb_ctx* ctx, int k, bool inner = false)
        : c(ctx), kclass(k), e0(inner ? ctx->ev_in0 : ctx->ev0), e1(inner ? ctx->ev_in1 : ctx->ev1) {
        if (c->profile) cudaEventRecord(e0, c->stream);
    }
    ~SqbLaunchScope() {
        c->launches += 1;
        c->k_n[kclass] += 1;
        if (c->profile) {
            cudaEventRecord(e1, c->stream);
            cudaEventSynchronize(e1);
            float ms = 0.f;
            cudaEventElapsedTime(&ms, e0, e1);
            c->k_ms[kclass] += ms;
        }
    }
};

#define SQB_POST_LAUNCH()                                                                     \
    do {                                                                                      \
        cudaError_t _e = cudaGetLastError();                                                  \
        if (_e != cudaSuccess) {                                                              \
            sqb_set_error("kernel launch failed at %s:%d: %s", __FILE__, __LINE__,            \
                          cudaGetErrorString(_e));                                            \
            return SQB_ERR_CUDA;                                                              \
        }                                                                                     \
    } while (0)

static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// The indptr (n + 1 entries, int32 or int64) of a caller's device CSR must run from 0 at row 0 to nnz at row n without
// decreasing; bit 1 of *err otherwise.  Kernels that follow it may run only after *err has been read back as 0.
// dst (or null) receives the validated indptr as uint32 (nnz < 2^32 - 1; an invalid entry is written as 0).
template <typename IP>
__global__ void sqb_check_indptr_kernel(const IP* __restrict__ ptr, int64_t n, int64_t nnz, uint32_t* __restrict__ dst,
                                        unsigned* __restrict__ err) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r <= n; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t v = (int64_t)ptr[r];
        const bool bad = v < 0 || v > nnz || (r == 0 && v != 0) || (r == n && v != nnz) || (r < n && (int64_t)ptr[r + 1] < v);
        if (bad) atomicOr(err, 1u);
        if (dst) dst[r] = bad ? 0u : (uint32_t)v;
    }
}
static inline unsigned sqb_grid_rows(const sqb_ctx* c, int64_t rows, int threads) {
    const int64_t b = ceil_div64(rows, threads), cap = (int64_t)c->sm_count * 8;
    return (unsigned)(b < 1 ? 1 : b > cap ? cap : b);
}

// ---------------------------------------------------------------------------------------------
// Caller arrays in device memory (the *_device entry points): the ABI's type codes, the indptr check, and the way out of an
// entry point that reads them.
// ---------------------------------------------------------------------------------------------
// A stored value in the type XT a kernel works in: float16 goes through float32 (exact), the one-byte bool of interaction
// graphs is 1 for any non-zero byte, everything else is a plain conversion (int64 rounds to nearest, like numpy's astype).
template <typename XT, typename VT>
__device__ __forceinline__ XT sqb_cvt(VT v) {
    if constexpr (std::is_same<VT, __half>::value)
        return (XT)__half2float(v);
    else if constexpr (std::is_same<VT, uint8_t>::value)
        return v != 0 ? (XT)1 : (XT)0;
    else
        return (XT)v;
}

// A product or sum rounded on its own (never contracted to an FMA), in float or double.
template <typename T>
__device__ __forceinline__ T mul_rn(T a, T b) {
    if constexpr (std::is_same<T, float>::value)
        return __fmul_rn(a, b);
    else
        return __dmul_rn(a, b);
}
template <typename T>
__device__ __forceinline__ T add_rn(T a, T b) {
    if constexpr (std::is_same<T, float>::value)
        return __fadd_rn(a, b);
    else
        return __dadd_rn(a, b);
}

// The type a dispatch below hands to its callback: SqbType<T>::type.
template <typename T>
struct SqbType {
    using type = T;
};

// indptr_bits / index_bits of a caller's CSR (32 or 64 each) -> f(SqbType<IP>(), SqbType<II>()), IP / II int32_t or int64_t.
template <typename F>
int sqb_dispatch_index(int indptr_bits, int index_bits, const char* where, F&& f) {
    SQB_CHECK((indptr_bits == 32 || indptr_bits == 64) && (index_bits == 32 || index_bits == 64), SQB_ERR_INVALID,
              "%s: indptr_bits / index_bits must be 32 or 64", where);
    const auto with_ip = [&](auto ip) { return index_bits == 32 ? f(ip, SqbType<int32_t>()) : f(ip, SqbType<int64_t>()); };
    return indptr_bits == 64 ? with_ip(SqbType<int64_t>()) : with_ip(SqbType<int32_t>());
}

// The value dtype code of the ABI (DTYPE_CODES of _device.py: 0 f32, 1 f64, 2 f16, 3 i32, 4 i64) -> f(SqbType<VT>()).
// WITH_BOOL adds code 5, the one-byte bool of interaction graphs; callers without it compile no bool instances.
// name: the code's argument name in the error message.
template <bool WITH_BOOL = false, typename F>
int sqb_dispatch_value(int code, const char* where, const char* name, F&& f) {
    switch (code) {
        case 0: return f(SqbType<float>());
        case 1: return f(SqbType<double>());
        case 2: return f(SqbType<__half>());
        case 3: return f(SqbType<int32_t>());
        case 4: return f(SqbType<int64_t>());
    }
    if constexpr (WITH_BOOL)
        if (code == 5) return f(SqbType<uint8_t>());
    sqb_set_error("%s: %s must be 0 (f32), 1 (f64), 2 (f16), 3 (i32)%s", where, name, WITH_BOOL ? ", 4 (i64) or 5 (bool)" : " or 4 (i64)");
    return SQB_ERR_INVALID;
}

// Checks a caller's indptr (n + 1 entries) against nnz with sqb_check_indptr_kernel and reads the verdict back (one
// synchronisation): SQB_ERR_INVALID unless it runs from 0 to nnz without decreasing.  Kernels that follow indptr may run
// only after SQB_OK.  dst (or null) receives the kernel's uint32 copy; kclass is the launch's class.
template <typename IP>
int sqb_check_indptr(sqb_ctx* c, int kclass, const IP* ptr, int64_t n, int64_t nnz, uint32_t* dst, const char* where) {
    DevBuf<unsigned> err(c->stream);
    SQB_TRY(err.alloc(1));
    SQB_CUDA(cudaMemsetAsync(err.p, 0, sizeof(unsigned), c->stream));
    {
        SqbLaunchScope scope(c, kclass);
        sqb_check_indptr_kernel<IP><<<sqb_grid_rows(c, n + 1, 256), 256, 0, c->stream>>>(ptr, n, nnz, dst, err.p);
        SQB_POST_LAUNCH();
    }
    unsigned flag = 0;
    SQB_CUDA(cudaMemcpyAsync(&flag, err.p, sizeof(unsigned), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    SQB_CHECK(flag == 0, SQB_ERR_INVALID, "%s: indptr inconsistent with nnz=%lld (it must run from 0 to nnz without decreasing)", where,
              (long long)nnz);
    return SQB_OK;
}

// Runs body() for an entry point that reads caller-owned device buffers: the context's stream first waits for the caller's
// producer stream (sqb_wait_producer; 0: none), and when body fails the stream is synchronised, so that the caller's buffers
// are no longer read when the entry point returns.  body synchronises on its own way to success.
template <typename F>
int sqb_read_caller_buffers(sqb_ctx* c, uintptr_t producer, F&& body) {
    SQB_TRY(sqb_wait_producer(c, producer));
    const int rc = body();
    if (rc != SQB_OK) cudaStreamSynchronize(c->stream);  // the caller's buffers are no longer read
    return rc;
}
