// capi.cu — context management and error plumbing of the C ABI (include/squidpy_b200.h).
#include <sched.h>
#include <stdarg.h>
#include <stdlib.h>

#include <algorithm>
#include <thread>

#include "common.cuh"

// Host threads the staging copies may use: the CPUs this PROCESS may run on (the affinity mask -- a GPU box often grants a
// container 2 of its 128 logical CPUs, which std::thread::hardware_concurrency() does not see), shared between the ranks of a
// torchrun launch, one per ~8 CPUs (a thread fills ~10 GB/s of pinned buffers), at least 1.
static int sqb_host_threads(int at_most) {
    int cpus = 0;
    cpu_set_t set;
    CPU_ZERO(&set);
    if (sched_getaffinity(0, sizeof(set), &set) == 0) cpus = CPU_COUNT(&set);
    if (cpus <= 0) cpus = (int)std::thread::hardware_concurrency();
    int ranks = 1;
    if (const char* lws = getenv("LOCAL_WORLD_SIZE")) ranks = std::max(1, atoi(lws));
    cpus = std::max(1, cpus / ranks);
    int t = cpus >= 16 ? cpus / 8 : std::min(cpus, 2);
    return std::max(1, std::min(t, at_most));
}

static thread_local char g_err[1024] = "";

void sqb_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// ---------------------------------------------------------------------------------------------
// staged host-to-device copy (see common.cuh)
// ---------------------------------------------------------------------------------------------
static const size_t kStageBytes = (size_t)16 << 20;   // per ring buffer
static const size_t kStageMin = (size_t)256 << 20;    // smaller copies go straight through cudaMemcpyAsync

int sqb_h2d(sqb_ctx* c, void* dst, const void* src, size_t bytes) {
    if (bytes == 0) return SQB_OK;
    cudaPointerAttributes attr;
    const bool pinned_src = cudaPointerGetAttributes(&attr, src) == cudaSuccess && attr.type == cudaMemoryTypeHost;
    cudaGetLastError();
    static const bool staged_on = []() {
        const char* e = getenv("SQB_STAGED_H2D");  // 0 switches the staging ring off (plain cudaMemcpyAsync from pageable memory)
        return !(e && atoi(e) == 0);
    }();
    if (bytes < kStageMin || pinned_src || !staged_on) {
        SQB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c->stream));
        return SQB_OK;
    }
    for (int b = 0; b < sqb_ctx::kStage; ++b) {
        if (!c->stage[b]) {
            SQB_CUDA(cudaHostAlloc(&c->stage[b], kStageBytes, cudaHostAllocDefault));
            SQB_CUDA(cudaEventCreateWithFlags(&c->stage_ev[b], cudaEventDisableTiming));
        }
    }
    // T host threads, two pinned buffers each: thread t copies the chunks t, t + T, ... into its buffers and queues their DMA
    // on the ctx stream itself (chunks go to disjoint destination ranges, so their order on the stream does not matter).
    // Several threads are needed to keep a PCIe x16 link busy.
    int T = sqb_host_threads(sqb_ctx::kStage / 2);
    const size_t chunks = (bytes + kStageBytes - 1) / kStageBytes;
    if ((size_t)T > chunks) T = (int)chunks;
    std::vector<cudaError_t> errs((size_t)T, cudaSuccess);
    std::vector<std::thread> pool;
    const int device = c->device;
    for (int t = 0; t < T; ++t) {
        pool.emplace_back([=, &errs]() {
            cudaError_t e = cudaSetDevice(device);
            for (size_t k = (size_t)t, it = 0; k < chunks && e == cudaSuccess; k += (size_t)T, ++it) {
                const int b = 2 * t + (int)(it & 1);
                const size_t off = k * kStageBytes, len = std::min(kStageBytes, bytes - off);
                if (c->stage_used[b]) e = cudaEventSynchronize(c->stage_ev[b]);  // the DMA that last read this buffer is done
                if (e != cudaSuccess) break;
                memcpy(c->stage[b], (const char*)src + off, len);
                e = cudaMemcpyAsync((char*)dst + off, c->stage[b], len, cudaMemcpyHostToDevice, c->stream);
                if (e == cudaSuccess) e = cudaEventRecord(c->stage_ev[b], c->stream);
                c->stage_used[b] = true;
            }
            errs[t] = e;
        });
    }
    for (auto& th : pool) th.join();
    for (int t = 0; t < T; ++t) SQB_CUDA(errs[t]);
    return SQB_OK;
}

// Gathering variant: copies the pieces [start[r], start[r] + cnt[r]) (elements of elem bytes) of src, r = 0..rows-1, back to
// back to dst.  The pieces are packed into the pinned ring by several host threads (each stage = a run of whole rows).
int sqb_h2d_gather(sqb_ctx* c, void* dst, const void* src, size_t elem, const int64_t* start, const int64_t* cnt,
                   const int64_t* out_ptr, int64_t rows) {
    if (rows <= 0 || out_ptr[rows] == 0) return SQB_OK;
    for (int b = 0; b < sqb_ctx::kStage; ++b) {
        if (!c->stage[b]) {
            SQB_CUDA(cudaHostAlloc(&c->stage[b], kStageBytes, cudaHostAllocDefault));
            SQB_CUDA(cudaEventCreateWithFlags(&c->stage_ev[b], cudaEventDisableTiming));
        }
    }
    int threads = sqb_host_threads(8);
    const int64_t cap = (int64_t)(kStageBytes / elem);
    int64_t r0 = 0;
    for (int k = 0; r0 < rows; ++k) {
        // rows [r0, r1) whose pieces fit one stage (a single longer piece is split below by the caller's contract: cnt <= cap)
        int64_t r1 = r0;
        while (r1 < rows && out_ptr[r1 + 1] - out_ptr[r0] <= cap) ++r1;
        SQB_CHECK(r1 > r0, SQB_ERR_UNSUPPORTED, "sqb_h2d_gather: a single row of %lld elements exceeds the staging buffer",
                  (long long)cnt[r0]);
        const int b = k % sqb_ctx::kStage;
        if (c->stage_used[b]) SQB_CUDA(cudaEventSynchronize(c->stage_ev[b]));
        char* stage = (char*)c->stage[b];
        const int64_t base = out_ptr[r0];
        const int64_t nr = r1 - r0;
        const int used = (int)std::min<int64_t>(threads, nr);
        std::thread pool[16];
        for (int t = 0; t < used; ++t) {
            const int64_t a = r0 + nr * t / used, e = r0 + nr * (t + 1) / used;
            pool[t] = std::thread([=]() {
                for (int64_t r = a; r < e; ++r)
                    if (cnt[r] > 0) memcpy(stage + (size_t)(out_ptr[r] - base) * elem, (const char*)src + (size_t)start[r] * elem, (size_t)cnt[r] * elem);
            });
        }
        for (int t = 0; t < used; ++t) pool[t].join();
        const size_t len = (size_t)(out_ptr[r1] - base) * elem;
        if (len > 0) SQB_CUDA(cudaMemcpyAsync((char*)dst + (size_t)base * elem, stage, len, cudaMemcpyHostToDevice, c->stream));
        SQB_CUDA(cudaEventRecord(c->stage_ev[b], c->stream));
        c->stage_used[b] = true;
        r0 = r1;
    }
    return SQB_OK;
}

int sqb_wait_producer(sqb_ctx* c, uintptr_t producer) {
    if (producer == 0) return SQB_OK;
    cudaStream_t s = producer == 1 ? cudaStreamLegacy : producer == 2 ? cudaStreamPerThread : (cudaStream_t)producer;
    if (s == c->stream) return SQB_OK;
    cudaEvent_t ev;
    SQB_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    cudaError_t e = cudaEventRecord(ev, s);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(c->stream, ev, 0);
    cudaEventDestroy(ev);  // released once the recorded work completes
    SQB_CUDA(e);
    return SQB_OK;
}

extern "C" {

int sqb_abi_version(void) { return SQB_ABI_VERSION; }

const char* sqb_last_error(void) { return g_err; }

int sqb_device_count(int* count) {
    SQB_CHECK(count, SQB_ERR_INVALID, "sqb_device_count: null argument");
    SQB_CUDA(cudaGetDeviceCount(count));
    return SQB_OK;
}

int sqb_ctx_create(int device, void* stream, sqb_ctx** out) {
    SQB_CHECK(out, SQB_ERR_INVALID, "sqb_ctx_create: null out");
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        sqb_set_error("no CUDA device available (%s); squidpy_b200 has no CPU fallback", cudaGetErrorString(e));
        return SQB_ERR_CUDA;
    }
    SQB_CHECK(device >= 0 && device < ndev, SQB_ERR_INVALID, "sqb_ctx_create: device %d not in [0,%d)", device, ndev);
    SQB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    SQB_CUDA(cudaGetDeviceProperties(&prop, device));
    SQB_CHECK(prop.major == 9 && prop.minor == 0, SQB_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a (H100) only",
              device, prop.major, prop.minor);
    sqb_ctx* c = new sqb_ctx();
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    c->smem_optin = prop.sharedMemPerBlockOptin;
    c->smem_per_sm = prop.sharedMemPerMultiprocessor;
    c->smem_reserved = prop.reservedSharedMemPerBlock;
    c->l2_bytes = (size_t)prop.l2CacheSize;
    if (stream) {
        c->stream = (cudaStream_t)stream;
        c->own_stream = false;
    } else {
        e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
        if (e != cudaSuccess) {
            delete c;
            sqb_set_error("cudaStreamCreate: %s", cudaGetErrorString(e));
            return SQB_ERR_CUDA;
        }
        c->own_stream = true;
    }
    cudaEventCreate(&c->ev0);
    cudaEventCreate(&c->ev1);
    cudaEventCreate(&c->ev_in0);
    cudaEventCreate(&c->ev_in1);
    {
        int least = 0, greatest = 0;
        e = cudaDeviceGetStreamPriorityRange(&least, &greatest);
        if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&c->tail, cudaStreamNonBlocking, greatest);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming);
        if (e != cudaSuccess) {
            sqb_ctx_destroy(c);
            sqb_set_error("sqb_ctx_create: second stream: %s", cudaGetErrorString(e));
            return SQB_ERR_CUDA;
        }
    }
    {  // keep freed blocks of the stream-ordered allocator in the pool (handles are created and destroyed per API call)
        cudaMemPool_t pool = nullptr;
        if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
            unsigned long long thr = ~0ULL;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
        }
        cudaGetLastError();
    }
    // Optional L2 fetch granularity override (SQB_L2_FETCH=32|64|128); the driver default is kept unless it is set.
    {
        const char* env = getenv("SQB_L2_FETCH");
        if (env && atoi(env) > 0) {
            cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)atoi(env));
            cudaGetLastError();
        }
    }
    *out = c;
    return SQB_OK;
}

int sqb_ctx_destroy(sqb_ctx* c) {
    if (!c) return SQB_OK;
    cudaSetDevice(c->device);
    if (c->ev0) cudaEventDestroy(c->ev0);
    if (c->ev1) cudaEventDestroy(c->ev1);
    if (c->ev_in0) cudaEventDestroy(c->ev_in0);
    if (c->ev_in1) cudaEventDestroy(c->ev_in1);
    if (c->ev_fork) cudaEventDestroy(c->ev_fork);
    if (c->ev_join) cudaEventDestroy(c->ev_join);
    if (c->tail) {
        cudaStreamSynchronize(c->tail);
        cudaStreamDestroy(c->tail);
    }
    if (c->stream) cudaStreamSynchronize(c->stream);
    for (auto& s : c->scratch) s.release();
    for (int b = 0; b < sqb_ctx::kStage; ++b) {
        if (c->stage_ev[b]) cudaEventDestroy(c->stage_ev[b]);
        if (c->stage[b]) cudaFreeHost(c->stage[b]);
    }
    if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
    delete c;
    return SQB_OK;
}

int sqb_ctx_sync(sqb_ctx* c) {
    SQB_CHECK(c, SQB_ERR_INVALID, "sqb_ctx_sync: null ctx");
    SQB_CUDA(cudaSetDevice(c->device));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    return SQB_OK;
}

int sqb_ctx_stream(sqb_ctx* c, void** stream) {
    SQB_CHECK(c && stream, SQB_ERR_INVALID, "sqb_ctx_stream: null argument");
    *stream = (void*)c->stream;
    return SQB_OK;
}

int sqb_ctx_sm_count(sqb_ctx* c, int* sm_count) {
    SQB_CHECK(c && sm_count, SQB_ERR_INVALID, "sqb_ctx_sm_count: null argument");
    *sm_count = c->sm_count;
    return SQB_OK;
}

int sqb_ctx_launch_count(sqb_ctx* c, int64_t* launches) {
    SQB_CHECK(c && launches, SQB_ERR_INVALID, "sqb_ctx_launch_count: null argument");
    *launches = c->launches;
    return SQB_OK;
}

int sqb_ctx_profile(sqb_ctx* c, int enable) {
    SQB_CHECK(c, SQB_ERR_INVALID, "sqb_ctx_profile: null ctx");
    c->profile = enable != 0;
    return SQB_OK;
}

int sqb_ctx_profile_reset(sqb_ctx* c) {
    SQB_CHECK(c, SQB_ERR_INVALID, "sqb_ctx_profile_reset: null ctx");
    for (int k = 0; k < SQB_K_NCLASS; ++k) {
        c->k_ms[k] = 0.0;
        c->k_n[k] = 0;
    }
    return SQB_OK;
}

int sqb_ctx_profile_get(sqb_ctx* c, int kclass, double* ms, int64_t* launches) {
    SQB_CHECK(c && ms && launches, SQB_ERR_INVALID, "sqb_ctx_profile_get: null argument");
    SQB_CHECK(kclass >= 0 && kclass < SQB_K_NCLASS, SQB_ERR_INVALID, "sqb_ctx_profile_get: bad class %d", kclass);
    *ms = c->k_ms[kclass];
    *launches = c->k_n[kclass];
    return SQB_OK;
}

int sqb_host_alloc(size_t bytes, void** ptr) {
    SQB_CHECK(ptr, SQB_ERR_INVALID, "sqb_host_alloc: null argument");
    SQB_CUDA(cudaHostAlloc(ptr, bytes > 0 ? bytes : 1, cudaHostAllocPortable));
    return SQB_OK;
}

int sqb_host_free(void* ptr) {
    if (ptr) SQB_CUDA(cudaFreeHost(ptr));
    return SQB_OK;
}

int sqb_pointer_device(const void* p, int* device) {
    SQB_CHECK(device, SQB_ERR_INVALID, "sqb_pointer_device: null argument");
    cudaPointerAttributes attr;
    const cudaError_t e = cudaPointerGetAttributes(&attr, p);
    if (e == cudaErrorInvalidValue) {  // a host pointer CUDA has never seen
        cudaGetLastError();
        *device = -1;
        return SQB_OK;
    }
    SQB_CUDA(e);
    *device = (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged) ? attr.device : -1;
    return SQB_OK;
}

}  // extern "C"
