// graph_device.cu — spatial neighbour graphs from coordinates already in GPU memory, built AND post-processed on the device
// (sm_90a).  The result stays on the device as two CSR matrices (connectivities, distances) with int32 indptr / indices and
// ascending columns in every row.
//
// Replaces, for device coordinates, the host steps of the builders (src/squidpy/gr/neighbors.py):
//   KNNBuilder / RadiusBuilder / GridBuilder.build_graph   :192-209, :253-270, :365-419   (search, cut, ring expansion, diagonals)
//   GraphBuilder.build -> _filter_by_radius_interval /       :80-135, :423-452             (interval and percentile pruning,
//     _apply_percentile / _apply_transform                   :455-477                       eliminate_zeros, spectral / cosine)
//   GraphBuilderCSR.combine                                  :138-156                       (library_key block diagonal)
//   DelaunayBuilder.build_graph                              :318-332                       (Delaunay graph, delaunay.cu)
// Every value equals the host path's bit for bit (squidpy_b200/gr/_build.py; DESIGN.md §3.4 has the argument per step):
//  * entries are those of the host's CSR after eliminate_zeros: the host's explicit zeros (setdiag, pruning) only matter to
//    the percentile, whose order statistics include them here too (the n diagonal zeros lead the sorted distances);
//  * percentile: numpy's `linear` method evaluated from the two order statistics around (m - 1) * q / 100;
//  * spectral: column sums of ones are exact counts; deg = sqrt(1 / count) and deg[i] * deg[j] * w in float32, in that order;
//  * cosine: sklearn's row normalisation (float32 squares summed in double, float32 / double) and scipy's csr_matmat
//    (products v * b added into each output column in row-walk order, float32, zero sums dropped): the products of a row
//    are generated in walk order and stably sorted by column, so each column's sum runs in the same order;
//  * rings: the host's matrix-power loop gives entry (i, j) the directed graph distance d(i, j) of the cut graph for
//    1 <= d <= n_rings; here one level at a time: the entries of level d expand along the cut graph, a stable sort by
//    (row, column) puts each candidate after the entry already present, and the first of each run is kept.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <limits.h>
#include <math.h>

#include <vector>

#include "delaunay.cuh"

enum { GD_KNN = 0, GD_GRID = 1, GD_RADIUS = 2, GD_DELAUNAY = 3 };
enum { GD_NONE = 0, GD_SPECTRAL = 1, GD_COSINE = 2 };
enum { DST_DIST = 0, DST_ADJ = 1, DST_VAL = 2 };  // distances value: the distance (f64), the connectivity (f32), the table value (f32)

namespace {

struct Csr {
    explicit Csr(cudaStream_t s) : ptr(s), idx(s), vf(s), vd(s) {}
    DevBuf<int32_t> ptr, idx;
    DevBuf<float> vf;   // float32 values
    DevBuf<double> vd;  // float64 values (distances of kNN / radius graphs)
    int64_t nnz = 0;
    bool f64 = false;
};

struct Params {
    int kind, k, n_rings, set_diag, interval, transform;
    double radius, lo, hi, percentile;  // percentile NaN: none
};

struct Coords {  // the caller's (n, 2) array: element strides, dtype 0 float32 / 1 float64
    const void* p;
    int dtype;
    int64_t s0, s1;
};

struct AsmParams {
    int cut_on;
    double cut;
    int interval;
    double lo, hi, thr;
    int diag;
    float diag_adj;
    int dst_mode;
};

inline unsigned blocks_for(const sqb_ctx* c, int64_t n) { return sqb_grid_rows(c, n, 256); }

#define GD_LAUNCH(...)                                 \
    do {                                               \
        {                                              \
            SqbLaunchScope _scope(c, SQB_K_MISC);      \
            __VA_ARGS__;                               \
        }                                              \
        SQB_POST_LAUNCH();                             \
    } while (0)

int read_back(sqb_ctx* c, void* host, const void* dev, size_t bytes) {
    SQB_CUDA(cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    return SQB_OK;
}

template <typename T>
int exclusive_scan(sqb_ctx* c, DevBuf<uint8_t>& tmp, const T* in, T* out, int64_t count) {
    size_t bytes = 0;
    SQB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, (int)count, c->stream));
    SQB_TRY(tmp.alloc(bytes > 0 ? bytes : 1));
    SQB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, in, out, (int)count, c->stream));
    c->launches += 1;
    return SQB_OK;
}

// stable radix sort of (key, value) pairs over key bits [0, end_bit)
template <typename K, typename V>
int sort_pairs(sqb_ctx* c, DevBuf<uint8_t>& tmp, const K* kin, K* kout, const V* vin, V* vout, int64_t m, int end_bit) {
    size_t bytes = 0;
    SQB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, kin, kout, vin, vout, (int)m, 0, end_bit, c->stream));
    SQB_TRY(tmp.alloc(bytes > 0 ? bytes : 1));
    SQB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, bytes, kin, kout, vin, vout, (int)m, 0, end_bit, c->stream));
    c->launches += 1;
    return SQB_OK;
}

int key_bits(int64_t n) {  // (row << 32 | column) keys of rows < n
    int b = 1;
    while (b < 31 && ((uint64_t)(n - 1) >> b) != 0) ++b;
    return 32 + b;
}

// np.percentile(values, q) (method 'linear') of m sorted values from the two order statistics it reads; get(i) is the i-th
int percentile_linear(double q_pct, int64_t m, double* thr, int (*get)(void*, int64_t, double*), void* env) {
    const double q = q_pct / 100.0;
    const double vi = (double)(m - 1) * q;
    double prev = floor(vi);
    int64_t ip = (int64_t)prev, in = ip + 1;
    if (vi >= (double)(m - 1)) ip = in = m - 1, prev = -1.0;  // numpy's index -1 (the last value); gamma is computed from it
    const double gamma = vi - prev;
    double a, b;
    SQB_TRY(get(env, ip, &a));
    SQB_TRY(get(env, in, &b));
    const double diff = b - a;
    double r = a + diff * gamma;
    if (gamma >= 0.5) r = b - diff * (1.0 - gamma);
    *thr = r;
    return SQB_OK;
}

// The same for float32 values, in numpy's float32 arithmetic (NEP 50: the Python-float percentile and the Python-int counts
// are cast to float32): q = float32(p) / 100, the virtual index (m - 1) * q, its fraction and the interpolation all in float32.
int percentile_linear_f32(double q_pct, int64_t m, double* thr, int (*get)(void*, int64_t, double*), void* env) {
    const float q = (float)q_pct / 100.0f;
    const float vi = (float)(m - 1) * q;
    int64_t ip = (int64_t)floorf(vi), in = ip + 1;
    float gamma = vi - (float)ip;
    if (vi >= (float)(m - 1)) ip = in = m - 1, gamma = (float)((double)vi + 1.0);  // numpy's index -1
    double a, b;
    SQB_TRY(get(env, ip, &a));
    SQB_TRY(get(env, in, &b));
    const float fa = (float)a, fb = (float)b, diff = fb - fa;
    float r = fa + diff * gamma;
    if (gamma >= 0.5f) r = fb - diff * (1.0f - gamma);
    *thr = (double)r;
    return SQB_OK;
}

}  // namespace

// ---- kernels ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void gd_gather_kernel(const T* __restrict__ xy, int64_t s0, int64_t s1, const int32_t* __restrict__ rows, int64_t n,
                                 double* __restrict__ out) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = rows ? (int64_t)rows[i] : i;
        out[2 * i] = (double)xy[r * s0];
        out[2 * i + 1] = (double)xy[r * s0 + s1];
    }
}

// per-block bounding box (x0, y0, x1, y1) of the finite points and the first non-finite observation (LLONG_MAX: none)
__global__ void __launch_bounds__(256) gd_bbox_kernel(const double* __restrict__ xy, int64_t n, double* __restrict__ box,
                                                      long long* __restrict__ bad) {
    __shared__ double s[4][256];
    __shared__ long long sb[256];
    double x0 = INFINITY, y0 = INFINITY, x1 = -INFINITY, y1 = -INFINITY;
    long long b = LLONG_MAX;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double x = xy[2 * i], y = xy[2 * i + 1];
        if (!(isfinite(x) && isfinite(y))) {
            b = i < b ? i : b;
        } else {
            x0 = fmin(x0, x), y0 = fmin(y0, y), x1 = fmax(x1, x), y1 = fmax(y1, y);
        }
    }
    const int t = threadIdx.x;
    s[0][t] = x0, s[1][t] = y0, s[2][t] = x1, s[3][t] = y1, sb[t] = b;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (t < w) {
            s[0][t] = fmin(s[0][t], s[0][t + w]), s[1][t] = fmin(s[1][t], s[1][t + w]);
            s[2][t] = fmax(s[2][t], s[2][t + w]), s[3][t] = fmax(s[3][t], s[3][t + w]);
            sb[t] = sb[t + w] < sb[t] ? sb[t + w] : sb[t];
        }
        __syncthreads();
    }
    if (t == 0) {
        for (int q = 0; q < 4; ++q) box[4 * blockIdx.x + q] = s[q][0];
        bad[blockIdx.x] = sb[0];
    }
}

__global__ void gd_knn_ptr_kernel(int64_t* __restrict__ ptr, int64_t n, int k) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= n; i += (int64_t)gridDim.x * blockDim.x) ptr[i] = i * k;
}

// the distances the percentile sees besides the diagonal zeros: interval-pruned entries are zero
__global__ void gd_masked_kernel(const double* __restrict__ d, int64_t m, int interval, double lo, double hi, double* __restrict__ out) {
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < m; t += (int64_t)gridDim.x * blockDim.x) {
        const double v = d[t];
        out[t] = interval && (v < lo || v > hi) ? 0.0 : v;
    }
}

// One thread per row of a base table (ascending columns, no diagonal): the entries of the connectivities and distances after
// the host's diagonal handling, pruning and eliminate_zeros.  Count pass (ia == nullptr): entries per row; fill pass: the rows.
__global__ void gd_assemble_kernel(const int64_t* __restrict__ bptr, const int32_t* __restrict__ bidx, const double* __restrict__ bval, int64_t n,
                                   AsmParams p, int32_t* __restrict__ cnt_a, int32_t* __restrict__ cnt_d, const int32_t* __restrict__ pa,
                                   int32_t* __restrict__ ia, float* __restrict__ va, const int32_t* __restrict__ pd, int32_t* __restrict__ id,
                                   float* __restrict__ vdf, double* __restrict__ vdd) {
    const bool fill = ia != nullptr;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int32_t na = 0, nd = 0;
        const int32_t oa = fill ? pa[i] : 0, od = fill ? pd[i] : 0;
        auto emit = [&](int32_t j, float a, double d) {
            if (a != 0.0f) {
                if (fill) ia[oa + na] = j, va[oa + na] = a;
                ++na;
            }
            if (d != 0.0) {
                if (fill) {
                    id[od + nd] = j;
                    if (vdd)
                        vdd[od + nd] = d;
                    else
                        vdf[od + nd] = (float)d;
                }
                ++nd;
            }
        };
        bool diag_done = !p.diag;
        for (int64_t t = bptr[i]; t < bptr[i + 1]; ++t) {
            const int32_t j = bidx[t];
            const double v = bval[t];
            if (!diag_done && j > i) {
                emit((int32_t)i, p.diag_adj, 0.0);
                diag_done = true;
            }
            if (p.cut_on && !(v < p.cut)) continue;  // GridBuilder: `dist < 1.3 * median` (neighbors.py:408-409)
            float a = 1.0f;
            double d = v;
            if (p.interval && (v < p.lo || v > p.hi)) a = 0.0f, d = 0.0;
            if (d > p.thr) a = 0.0f, d = 0.0;
            emit(j, a, p.dst_mode == DST_DIST ? d : p.dst_mode == DST_ADJ ? (double)a : v);
        }
        if (!diag_done) emit((int32_t)i, p.diag_adj, 0.0);
        if (!fill) cnt_a[i] = na, cnt_d[i] = nd;
    }
}

__global__ void gd_colcount_kernel(const int32_t* __restrict__ idx, int64_t m, int32_t* __restrict__ cnt) {
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < m; t += (int64_t)gridDim.x * blockDim.x) atomicAdd(&cnt[idx[t]], 1);
}

// D^-1/2 A D^-1/2 of a matrix of ones: column sums are exact counts (below 2^24); every step rounded like numpy's float32
__global__ void gd_spectral_kernel(const int32_t* __restrict__ ptr, const int32_t* __restrict__ idx, int64_t n, const int32_t* __restrict__ colcnt,
                                   float* __restrict__ val) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float di = __fsqrt_rn(__fdiv_rn(1.0f, (float)colcnt[i]));
        for (int32_t t = ptr[i]; t < ptr[i + 1]; ++t) {
            const float dj = __fsqrt_rn(__fdiv_rn(1.0f, (float)colcnt[idx[t]]));
            val[t] = __fmul_rn(__fmul_rn(di, dj), val[t]);
        }
    }
}

// sklearn's inplace_csr_row_normalize_l2: float32 squares summed in double, every value divided by the double norm
__global__ void gd_rownorm_kernel(const int32_t* __restrict__ ptr, int64_t n, const float* __restrict__ x, float* __restrict__ xn) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        double s = 0.0;
        for (int32_t t = ptr[i]; t < ptr[i + 1]; ++t) s = __dadd_rn(s, (double)__fmul_rn(x[t], x[t]));
        const bool zero = s == 0.0;
        s = __dsqrt_rn(s);
        for (int32_t t = ptr[i]; t < ptr[i + 1]; ++t) xn[t] = zero ? x[t] : __double2float_rn(__ddiv_rn((double)x[t], s));
    }
}

// (row, column) keys of a CSR's entries; transposed: (column, row)
__global__ void gd_keys_kernel(const int32_t* __restrict__ ptr, const int32_t* __restrict__ idx, int64_t n, int transposed, uint64_t* __restrict__ keys) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        for (int32_t t = ptr[i]; t < ptr[i + 1]; ++t)
            keys[t] = transposed ? ((uint64_t)(uint32_t)idx[t] << 32) | (uint64_t)i : ((uint64_t)i << 32) | (uint32_t)idx[t];
}

// row pointer of m sorted (row << 32 | column) keys
template <typename P>
__global__ void gd_ptr_from_keys_kernel(const uint64_t* __restrict__ keys, int64_t m, int64_t n, P* __restrict__ ptr) {
    for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < m; q += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = (int64_t)(keys[q] >> 32);
        const int64_t prev = q > 0 ? (int64_t)(keys[q - 1] >> 32) : -1;
        for (int64_t e = prev + 1; e <= r; ++e) ptr[e] = (P)q;
        if (q == m - 1)
            for (int64_t e = r + 1; e <= n; ++e) ptr[e] = (P)m;
    }
}

// cosine: products of row i of Xn with the rows of B = Xn^T it meets, in csr_matmat's walk order
__global__ void gd_prod_count_kernel(const int32_t* __restrict__ ptr, const int32_t* __restrict__ idx, int64_t n, const int32_t* __restrict__ bptr,
                                     int64_t* __restrict__ cnt) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t s = 0;
        for (int32_t t = ptr[i]; t < ptr[i + 1]; ++t) s += bptr[idx[t] + 1] - bptr[idx[t]];
        cnt[i] = s;
    }
}

__global__ void gd_prod_fill_kernel(const int32_t* __restrict__ ptr, const int32_t* __restrict__ idx, const float* __restrict__ xn, int64_t n,
                                    const int32_t* __restrict__ bptr, const uint64_t* __restrict__ bkeys, const float* __restrict__ bval,
                                    const int64_t* __restrict__ lptr, uint64_t* __restrict__ keys, float* __restrict__ prod) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t o = lptr[i];
        for (int32_t t = ptr[i]; t < ptr[i + 1]; ++t) {
            const int32_t j = idx[t];
            const float v = xn[t];
            for (int32_t q = bptr[j]; q < bptr[j + 1]; ++q, ++o) {
                keys[o] = ((uint64_t)i << 32) | (bkeys[q] & 0xffffffffull);
                prod[o] = __fmul_rn(v, bval[q]);
            }
        }
    }
}

// per row: the column-sorted products summed in order per column (from 0, float32); non-zero sums are the row's entries
__global__ void gd_prod_reduce_kernel(const int64_t* __restrict__ lptr, const uint64_t* __restrict__ keys, const float* __restrict__ prod, int64_t n,
                                      int32_t* __restrict__ cnt, const int32_t* __restrict__ optr, int32_t* __restrict__ oidx,
                                      float* __restrict__ oval) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int32_t o = optr ? optr[i] : 0, m = 0;
        int64_t q = lptr[i];
        const int64_t e = lptr[i + 1];
        while (q < e) {
            const uint32_t col = (uint32_t)(keys[q] & 0xffffffffull);
            float s = 0.0f;
            for (; q < e && (uint32_t)(keys[q] & 0xffffffffull) == col; ++q) s = __fadd_rn(s, prod[q]);
            if (s != 0.0f) {
                if (oidx) oidx[o + m] = (int32_t)col, oval[o + m] = s;
                ++m;
            }
        }
        if (!oidx) cnt[i] = m;
    }
}

// rings: the entries of the cut graph as level-1 keys
__global__ void gd_ring_init_kernel(const int32_t* __restrict__ ptr, const int32_t* __restrict__ idx, int64_t n, uint64_t* __restrict__ keys,
                                    float* __restrict__ lvl) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        for (int32_t t = ptr[i]; t < ptr[i + 1]; ++t) keys[t] = ((uint64_t)i << 32) | (uint32_t)idx[t], lvl[t] = 1.0f;
}

__global__ void gd_ring_count_kernel(const uint64_t* __restrict__ keys, const float* __restrict__ lvl, int64_t m, float level,
                                     const int32_t* __restrict__ bptr, int64_t* __restrict__ cnt) {
    for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < m; q += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t j = (uint32_t)(keys[q] & 0xffffffffull);
        cnt[q] = lvl[q] == level ? bptr[j + 1] - bptr[j] : 0;
    }
}

// the present entries first, then the neighbours of every level-`level` entry's column as level + 1 candidates
__global__ void gd_ring_expand_kernel(const uint64_t* __restrict__ keys, const float* __restrict__ lvl, int64_t m, float level,
                                      const int32_t* __restrict__ bptr, const int32_t* __restrict__ bidx, const int64_t* __restrict__ eptr,
                                      uint64_t* __restrict__ okeys, float* __restrict__ olvl) {
    for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < m; q += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t key = keys[q];
        okeys[q] = key, olvl[q] = lvl[q];
        if (lvl[q] != level) continue;
        const uint64_t row = key & 0xffffffff00000000ull;
        const uint32_t j = (uint32_t)(key & 0xffffffffull);
        int64_t o = m + eptr[q];
        for (int32_t t = bptr[j]; t < bptr[j + 1]; ++t, ++o) okeys[o] = row | (uint32_t)bidx[t], olvl[o] = level + 1.0f;
    }
}

// first entry of every run of equal sorted keys, the diagonal excluded
__global__ void gd_ring_first_kernel(const uint64_t* __restrict__ keys, int64_t m, int32_t* __restrict__ flag) {
    for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < m; q += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t key = keys[q];
        flag[q] = (q == 0 || keys[q - 1] != key) && (key >> 32) != (key & 0xffffffffull);
    }
}

__global__ void gd_ring_compact_kernel(const uint64_t* __restrict__ keys, const float* __restrict__ lvl, const int32_t* __restrict__ flag,
                                       const int32_t* __restrict__ pos, int64_t m, uint64_t* __restrict__ okeys, float* __restrict__ olvl) {
    for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < m; q += (int64_t)gridDim.x * blockDim.x)
        if (flag[q]) okeys[pos[q]] = keys[q], olvl[pos[q]] = lvl[q];
}

__global__ void gd_split_keys_kernel(const uint64_t* __restrict__ keys, const float* __restrict__ lvl, int64_t m, int32_t* __restrict__ idx,
                                     double* __restrict__ val) {
    for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < m; q += (int64_t)gridDim.x * blockDim.x)
        idx[q] = (int32_t)(keys[q] & 0xffffffffull), val[q] = (double)lvl[q];
}

// library blocks -> one matrix: row r of a block is output row grow[r]; its columns map through grow as well (ascending)
__global__ void gd_block_count_kernel(const int32_t* __restrict__ ptr, const int32_t* __restrict__ grow, int64_t nb, int32_t* __restrict__ cnt) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < nb; r += (int64_t)gridDim.x * blockDim.x) cnt[grow[r]] = ptr[r + 1] - ptr[r];
}

template <typename V>
__global__ void gd_block_fill_kernel(const int32_t* __restrict__ ptr, const int32_t* __restrict__ idx, const V* __restrict__ val,
                                     const int32_t* __restrict__ grow, int64_t nb, const int32_t* __restrict__ optr, int32_t* __restrict__ oidx,
                                     V* __restrict__ oval) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < nb; r += (int64_t)gridDim.x * blockDim.x) {
        const int32_t o = optr[grow[r]] - ptr[r];
        for (int32_t t = ptr[r]; t < ptr[r + 1]; ++t) oidx[o + t] = grow[idx[t]], oval[o + t] = val[t];
    }
}

// ---- host steps --------------------------------------------------------------------------------------------------------
struct sqb_graph {
    explicit sqb_graph(sqb_ctx* ctx) : c(ctx), adj(ctx->stream), dst(ctx->stream) {}
    sqb_ctx* c;
    int64_t n = 0;
    Csr adj, dst;
};

namespace {

// count pass -> per-row pointers of both matrices -> fill pass
int assemble(sqb_ctx* c, const int64_t* bptr, const int32_t* bidx, const double* bval, int64_t n, const AsmParams& p, bool dst_f64, Csr* adj,
             Csr* dst) {
    DevBuf<int32_t> ca(c->stream), cd(c->stream);
    DevBuf<uint8_t> tmp(c->stream);
    SQB_TRY(ca.alloc(n + 1));
    SQB_TRY(cd.alloc(n + 1));
    SQB_TRY(adj->ptr.alloc(n + 1));
    SQB_TRY(dst->ptr.alloc(n + 1));
    SQB_CUDA(cudaMemsetAsync(ca.p + n, 0, sizeof(int32_t), c->stream));
    SQB_CUDA(cudaMemsetAsync(cd.p + n, 0, sizeof(int32_t), c->stream));
    GD_LAUNCH(gd_assemble_kernel<<<blocks_for(c, n), 256, 0, c->stream>>>(bptr, bidx, bval, n, p, ca.p, cd.p, nullptr, nullptr, nullptr, nullptr,
                                                                           nullptr, nullptr, nullptr));
    SQB_TRY(exclusive_scan(c, tmp, ca.p, adj->ptr.p, n + 1));
    SQB_TRY(exclusive_scan(c, tmp, cd.p, dst->ptr.p, n + 1));
    int32_t na = 0, nd = 0;
    SQB_TRY(read_back(c, &na, adj->ptr.p + n, sizeof(int32_t)));
    SQB_TRY(read_back(c, &nd, dst->ptr.p + n, sizeof(int32_t)));
    adj->nnz = na, dst->nnz = nd, adj->f64 = false, dst->f64 = dst_f64;
    SQB_TRY(adj->idx.alloc(na));
    SQB_TRY(adj->vf.alloc(na));
    SQB_TRY(dst->idx.alloc(nd));
    SQB_TRY(dst_f64 ? dst->vd.alloc(nd) : dst->vf.alloc(nd));
    GD_LAUNCH(gd_assemble_kernel<<<blocks_for(c, n), 256, 0, c->stream>>>(bptr, bidx, bval, n, p, nullptr, nullptr, adj->ptr.p, adj->idx.p, adj->vf.p,
                                                                           dst->ptr.p, dst->idx.p, dst_f64 ? nullptr : dst->vf.p,
                                                                           dst_f64 ? dst->vd.p : nullptr));
    return SQB_OK;
}

// Xn Xn^T of the row-normalised connectivities (sklearn's cosine_similarity(adj, dense_output=False))
int cosine(sqb_ctx* c, int64_t n, Csr* adj) {
    const int64_t m = adj->nnz;
    DevBuf<float> xn(c->stream), bval(c->stream), prod(c->stream), pout(c->stream);
    DevBuf<uint64_t> keys(c->stream), bkeys(c->stream), lkeys(c->stream), lkeys_s(c->stream);
    DevBuf<int32_t> bptr(c->stream), cnt(c->stream);
    DevBuf<int64_t> lcnt(c->stream), lptr(c->stream);
    DevBuf<uint8_t> tmp(c->stream);
    Csr out(c->stream);
    const unsigned gb = blocks_for(c, n);
    SQB_TRY(xn.alloc(m));
    GD_LAUNCH(gd_rownorm_kernel<<<gb, 256, 0, c->stream>>>(adj->ptr.p, n, adj->vf.p, xn.p));
    // B = Xn^T as CSR with ascending columns (scipy converts the CSC transpose to sorted CSR)
    SQB_TRY(keys.alloc(m));
    SQB_TRY(bkeys.alloc(m));
    SQB_TRY(bval.alloc(m));
    SQB_TRY(bptr.alloc(n + 1));
    GD_LAUNCH(gd_keys_kernel<<<gb, 256, 0, c->stream>>>(adj->ptr.p, adj->idx.p, n, 1, keys.p));
    if (m > 0) SQB_TRY(sort_pairs(c, tmp, keys.p, bkeys.p, xn.p, bval.p, m, key_bits(n)));
    SQB_CUDA(cudaMemsetAsync(bptr.p, 0, (n + 1) * sizeof(int32_t), c->stream));
    if (m > 0) GD_LAUNCH(gd_ptr_from_keys_kernel<int32_t><<<blocks_for(c, m), 256, 0, c->stream>>>(bkeys.p, m, n, bptr.p));
    // the products of every row in walk order, then stably sorted by (row, column)
    SQB_TRY(lcnt.alloc(n + 1));
    SQB_TRY(lptr.alloc(n + 1));
    SQB_CUDA(cudaMemsetAsync(lcnt.p + n, 0, sizeof(int64_t), c->stream));
    GD_LAUNCH(gd_prod_count_kernel<<<gb, 256, 0, c->stream>>>(adj->ptr.p, adj->idx.p, n, bptr.p, lcnt.p));
    SQB_TRY(exclusive_scan(c, tmp, lcnt.p, lptr.p, n + 1));
    int64_t L = 0;
    SQB_TRY(read_back(c, &L, lptr.p + n, sizeof(int64_t)));
    SQB_CHECK(L < INT_MAX, SQB_ERR_UNSUPPORTED, "cosine transform: %lld products exceed 2^31 - 1", (long long)L);
    SQB_TRY(lkeys.alloc(L));
    SQB_TRY(lkeys_s.alloc(L));
    SQB_TRY(prod.alloc(L));
    SQB_TRY(pout.alloc(L));
    GD_LAUNCH(gd_prod_fill_kernel<<<gb, 256, 0, c->stream>>>(adj->ptr.p, adj->idx.p, xn.p, n, bptr.p, bkeys.p, bval.p, lptr.p, lkeys.p, prod.p));
    if (L > 0) SQB_TRY(sort_pairs(c, tmp, lkeys.p, lkeys_s.p, prod.p, pout.p, L, key_bits(n)));
    // column sums in order; zero sums dropped (csr_matmat)
    SQB_TRY(cnt.alloc(n + 1));
    SQB_TRY(out.ptr.alloc(n + 1));
    SQB_CUDA(cudaMemsetAsync(cnt.p + n, 0, sizeof(int32_t), c->stream));
    GD_LAUNCH(gd_prod_reduce_kernel<<<gb, 256, 0, c->stream>>>(lptr.p, lkeys_s.p, pout.p, n, cnt.p, nullptr, nullptr, nullptr));
    SQB_TRY(exclusive_scan(c, tmp, cnt.p, out.ptr.p, n + 1));
    int32_t nnz = 0;
    SQB_TRY(read_back(c, &nnz, out.ptr.p + n, sizeof(int32_t)));
    SQB_TRY(out.idx.alloc(nnz));
    SQB_TRY(out.vf.alloc(nnz));
    GD_LAUNCH(gd_prod_reduce_kernel<<<gb, 256, 0, c->stream>>>(lptr.p, lkeys_s.p, pout.p, n, nullptr, out.ptr.p, out.idx.p, out.vf.p));
    out.nnz = nnz;
    std::swap(*adj, out);
    return SQB_OK;
}

// Entries (i, j) of graph distance 1 .. n_rings from i in the cut graph `cut`, as a base table (int64 pointers, ring numbers)
int rings(sqb_ctx* c, int64_t n, const Csr& cut, int n_rings, DevBuf<int64_t>& tptr, DevBuf<int32_t>& tidx, DevBuf<double>& tval) {
    DevBuf<uint64_t> keys(c->stream), ekeys(c->stream), skeys(c->stream);
    DevBuf<float> lvl(c->stream), elvl(c->stream), slvl(c->stream);
    DevBuf<int64_t> ecnt(c->stream), eptr(c->stream);
    DevBuf<int32_t> flag(c->stream), pos(c->stream);
    DevBuf<uint8_t> tmp(c->stream);
    int64_t m = cut.nnz;
    SQB_TRY(keys.alloc(m));
    SQB_TRY(lvl.alloc(m));
    GD_LAUNCH(gd_ring_init_kernel<<<blocks_for(c, n), 256, 0, c->stream>>>(cut.ptr.p, cut.idx.p, n, keys.p, lvl.p));
    for (int level = 1; level < n_rings && m > 0; ++level) {
        SQB_TRY(ecnt.alloc(m + 1));
        SQB_TRY(eptr.alloc(m + 1));
        SQB_CUDA(cudaMemsetAsync(ecnt.p + m, 0, sizeof(int64_t), c->stream));
        GD_LAUNCH(gd_ring_count_kernel<<<blocks_for(c, m), 256, 0, c->stream>>>(keys.p, lvl.p, m, (float)level, cut.ptr.p, ecnt.p));
        SQB_TRY(exclusive_scan(c, tmp, ecnt.p, eptr.p, m + 1));
        int64_t e = 0;
        SQB_TRY(read_back(c, &e, eptr.p + m, sizeof(int64_t)));
        if (e == 0) break;
        const int64_t t = m + e;
        SQB_CHECK(t < INT_MAX, SQB_ERR_UNSUPPORTED, "n_rings=%d: %lld candidate entries exceed 2^31 - 1", n_rings, (long long)t);
        SQB_TRY(ekeys.alloc(t));
        SQB_TRY(elvl.alloc(t));
        SQB_TRY(skeys.alloc(t));
        SQB_TRY(slvl.alloc(t));
        SQB_TRY(flag.alloc(t + 1));
        SQB_TRY(pos.alloc(t + 1));
        GD_LAUNCH(gd_ring_expand_kernel<<<blocks_for(c, m), 256, 0, c->stream>>>(keys.p, lvl.p, m, (float)level, cut.ptr.p, cut.idx.p, eptr.p,
                                                                                  ekeys.p, elvl.p));
        SQB_TRY(sort_pairs(c, tmp, ekeys.p, skeys.p, elvl.p, slvl.p, t, key_bits(n)));
        SQB_CUDA(cudaMemsetAsync(flag.p + t, 0, sizeof(int32_t), c->stream));
        GD_LAUNCH(gd_ring_first_kernel<<<blocks_for(c, t), 256, 0, c->stream>>>(skeys.p, t, flag.p));
        SQB_TRY(exclusive_scan(c, tmp, flag.p, pos.p, t + 1));
        int32_t mm = 0;
        SQB_TRY(read_back(c, &mm, pos.p + t, sizeof(int32_t)));
        SQB_TRY(keys.alloc(mm));
        SQB_TRY(lvl.alloc(mm));
        GD_LAUNCH(gd_ring_compact_kernel<<<blocks_for(c, t), 256, 0, c->stream>>>(skeys.p, slvl.p, flag.p, pos.p, t, keys.p, lvl.p));
        m = mm;
    }
    SQB_TRY(tptr.alloc(n + 1));
    SQB_TRY(tidx.alloc(m));
    SQB_TRY(tval.alloc(m));
    SQB_CUDA(cudaMemsetAsync(tptr.p, 0, (n + 1) * sizeof(int64_t), c->stream));
    if (m > 0) {
        GD_LAUNCH(gd_ptr_from_keys_kernel<int64_t><<<blocks_for(c, m), 256, 0, c->stream>>>(keys.p, m, n, tptr.p));
        GD_LAUNCH(gd_split_keys_kernel<<<blocks_for(c, m), 256, 0, c->stream>>>(keys.p, lvl.p, m, tidx.p, tval.p));
    }
    return SQB_OK;
}

struct PctEnv {
    sqb_ctx* c;
    const double* sorted;
    int64_t zeros;  // the n diagonal zeros precede the sorted distances
};

int pct_get(void* env, int64_t i, double* v) {
    const PctEnv* e = (const PctEnv*)env;
    if (i < e->zeros) {
        *v = 0.0;
        return SQB_OK;
    }
    return read_back(e->c, v, e->sorted + (i - e->zeros), sizeof(double));
}

// One graph (or one library's block), before its transform, from the rows `rows` (device, or null: all n) of the caller's
// coordinates.  Its temporaries are freed when it returns.
int build_untransformed(sqb_ctx* c, const Coords& xy, const int32_t* rows, int64_t n, const Params& P, Csr* adj, Csr* dst) {
    const bool knn = P.kind == GD_KNN || P.kind == GD_GRID;
    if (P.kind == GD_DELAUNAY) {
        SQB_CHECK(n >= 3, SQB_ERR_INVALID,
                  "QhullError: the Delaunay triangulation needs at least three distinct points that are not all collinear");
    } else if (knn) {  // the checks and messages of sqb_knn_2d / sqb_radius_2d, in their order
        SQB_CHECK(n >= 2 && n < 2147483647LL, SQB_ERR_INVALID, "sqb_knn_2d: n=%lld out of range", (long long)n);
        SQB_CHECK(P.k >= 1 && P.k <= 64, SQB_ERR_UNSUPPORTED, "sqb_knn_2d: n_neighbors=%d outside [1, 64]", P.k);
        SQB_CHECK(P.k < n, SQB_ERR_INVALID, "Expected n_neighbors <= n_samples_fit, but n_neighbors = %d, n_samples_fit = %lld, n_samples = %lld",
                  P.k + 1, (long long)n, (long long)n);
        SQB_CHECK((int64_t)n * P.k < 2147483647LL, SQB_ERR_UNSUPPORTED, "sqb_knn_2d: n * k does not fit int32");
    } else {
        SQB_CHECK(n >= 1 && n < 2147483647LL, SQB_ERR_INVALID, "sqb_radius_2d: n=%lld out of range", (long long)n);
    }
    PointGrid g(c->stream);
    DevBuf<double> box(c->stream), dist(c->stream), sorted(c->stream), bval(c->stream);
    DevBuf<long long> bad(c->stream);
    DevBuf<int32_t> idx(c->stream);
    DevBuf<int64_t> bptr(c->stream), cnt(c->stream);
    DevBuf<uint8_t> tmp(c->stream);
    // coordinates: gathered into float64 (n, 2), bounding box and the first non-finite observation in one reduction
    SQB_TRY(g.d_xy.alloc(2 * n));
    const unsigned gb = blocks_for(c, n);
    if (xy.dtype == 0)
        GD_LAUNCH(gd_gather_kernel<float><<<gb, 256, 0, c->stream>>>((const float*)xy.p, xy.s0, xy.s1, rows, n, g.d_xy.p));
    else
        GD_LAUNCH(gd_gather_kernel<double><<<gb, 256, 0, c->stream>>>((const double*)xy.p, xy.s0, xy.s1, rows, n, g.d_xy.p));
    SQB_TRY(box.alloc(4 * (size_t)gb));
    SQB_TRY(bad.alloc(gb));
    GD_LAUNCH(gd_bbox_kernel<<<gb, 256, 0, c->stream>>>(g.d_xy.p, n, box.p, bad.p));
    std::vector<double> hbox(4 * (size_t)gb);
    std::vector<long long> hbad(gb);
    SQB_CUDA(cudaMemcpyAsync(hbox.data(), box.p, hbox.size() * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SQB_TRY(read_back(c, hbad.data(), bad.p, hbad.size() * sizeof(long long)));
    double x0 = INFINITY, y0 = INFINITY, x1 = -INFINITY, y1 = -INFINITY;
    long long first_bad = LLONG_MAX;
    for (unsigned b = 0; b < gb; ++b) {
        x0 = fmin(x0, hbox[4 * b]), y0 = fmin(y0, hbox[4 * b + 1]), x1 = fmax(x1, hbox[4 * b + 2]), y1 = fmax(y1, hbox[4 * b + 3]);
        first_bad = hbad[b] < first_bad ? hbad[b] : first_bad;
    }
    SQB_CHECK(first_bad == LLONG_MAX, SQB_ERR_INVALID, "coordinates of observation %lld are not finite", first_bad);
    g.gm = P.kind == GD_DELAUNAY ? grid_geometry(x0, y0, x1, y1, n, 0.0, DT_PTS_PER_CELL)
           : knn                 ? grid_geometry(x0, y0, x1, y1, n, 0.0, knn_pts_per_cell(P.k))
                                 : grid_geometry(x0, y0, x1, y1, n, P.radius > 0.0 ? P.radius : 0.0, 2.5);
    SQB_TRY(grid_bucket(c, n, &g));
    // the neighbour table as rows of ascending columns: bptr / idx / dist
    int64_t m;
    SQB_TRY(bptr.alloc(n + 1));
    if (P.kind == GD_DELAUNAY) {
        SQB_TRY(delaunay_csr(c, g, n, bptr, idx, &m, nullptr));
        SQB_TRY(dist.alloc(m));
        if (m > 0) SQB_TRY(delaunay_dist(c, g.d_xy.p, bptr.p, idx.p, n, xy.dtype == 0, dist.p));
    } else if (knn) {
        m = n * P.k;
        SQB_TRY(idx.alloc(m));
        SQB_TRY(dist.alloc(m));
        SQB_TRY(knn_launch(c, g, n, P.k, idx.p, dist.p));
        GD_LAUNCH(gd_knn_ptr_kernel<<<gb, 256, 0, c->stream>>>(bptr.p, n, P.k));
    } else {
        SQB_TRY(cnt.alloc(n + 1));
        SQB_CUDA(cudaMemsetAsync(cnt.p, 0, (n + 1) * sizeof(int64_t), c->stream));
        SQB_TRY(radius_launch(c, g, n, P.radius, cnt.p, nullptr, nullptr, nullptr));
        SQB_TRY(exclusive_scan(c, tmp, cnt.p, bptr.p, n + 1));
        SQB_TRY(read_back(c, &m, bptr.p + n, sizeof(int64_t)));
        SQB_TRY(idx.alloc(m));
        SQB_TRY(dist.alloc(m));
        if (m > 0) SQB_TRY(radius_launch(c, g, n, P.radius, nullptr, bptr.p, idx.p, dist.p));
    }
    SQB_CHECK(m + n < INT_MAX, SQB_ERR_UNSUPPORTED, "the graph has %lld entries; int32 indices hold at most 2^31 - 1", (long long)(m + n));
    AsmParams ap{};
    ap.thr = INFINITY;
    if (P.kind == GD_GRID) {
        double med[2] = {0.0, 0.0};
        SQB_TRY(median_enqueue(c, dist.p, m, sorted, tmp, med));
        SQB_CUDA(cudaStreamSynchronize(c->stream));
        ap.cut_on = 1, ap.cut = (med[0] + med[1]) / 2.0 * 1.3;
        if (P.n_rings == 1) {
            ap.diag = P.set_diag, ap.diag_adj = 1.0f, ap.dst_mode = DST_ADJ;
            return assemble(c, bptr.p, idx.p, dist.p, n, ap, false, adj, dst);
        }
        // neighbors.py:372-386 on the cut graph; the diagonal follows below.  Each graph is freed once the next is built.
        DevBuf<int64_t> tptr(c->stream);
        DevBuf<int32_t> tidx(c->stream);
        DevBuf<double> tval(c->stream);
        {
            Csr cut(c->stream);
            {
                Csr cut_dst(c->stream);
                ap.dst_mode = DST_ADJ;
                SQB_TRY(assemble(c, bptr.p, idx.p, dist.p, n, ap, false, &cut, &cut_dst));
            }
            SQB_TRY(rings(c, n, cut, P.n_rings, tptr, tidx, tval));
        }
        AsmParams rp{};
        rp.thr = INFINITY, rp.diag = P.set_diag, rp.diag_adj = 1.0f, rp.dst_mode = DST_VAL;
        return assemble(c, tptr.p, tidx.p, tval.p, n, rp, false, adj, dst);
    }
    ap.diag = P.set_diag || P.interval || !isnan(P.percentile);  // _Builder._diagonals
    ap.diag_adj = P.set_diag ? 1.0f : 0.0f;
    ap.interval = P.interval, ap.lo = P.lo, ap.hi = P.hi, ap.dst_mode = DST_DIST;
    // float32 Delaunay distances are compared with the bounds cast to float32, as numpy compares a float32 array with a
    // Python float; the float32 values themselves are exact in float64
    const bool f32 = P.kind == GD_DELAUNAY && xy.dtype == 0;
    if (f32) ap.lo = (double)(float)P.lo, ap.hi = (double)(float)P.hi;
    if (!isnan(P.percentile)) {
        SQB_TRY(bval.alloc(m));
        SQB_TRY(sorted.alloc(m));
        if (m > 0) {
            GD_LAUNCH(gd_masked_kernel<<<blocks_for(c, m), 256, 0, c->stream>>>(dist.p, m, P.interval, ap.lo, ap.hi, bval.p));
            size_t bytes = 0;
            SQB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, bytes, bval.p, sorted.p, (int)m, 0, 64, c->stream));
            SQB_TRY(tmp.alloc(bytes > 0 ? bytes : 1));
            SQB_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, bytes, bval.p, sorted.p, (int)m, 0, 64, c->stream));
            c->launches += 1;
        }
        PctEnv env{c, sorted.p, n};
        SQB_TRY((f32 ? percentile_linear_f32 : percentile_linear)(P.percentile, m + n, &ap.thr, pct_get, &env));
    }
    return assemble(c, bptr.p, idx.p, dist.p, n, ap, !f32, adj, dst);
}

// One graph (or one library's block) with its transform
int build_block(sqb_ctx* c, const Coords& xy, const int32_t* rows, int64_t n, const Params& P, Csr* adj, Csr* dst) {
    SQB_TRY(build_untransformed(c, xy, rows, n, P, adj, dst));
    if (P.transform == GD_SPECTRAL && adj->nnz > 0) {
        DevBuf<int32_t> colcnt(c->stream);
        SQB_TRY(colcnt.alloc(n));
        SQB_CUDA(cudaMemsetAsync(colcnt.p, 0, n * sizeof(int32_t), c->stream));
        GD_LAUNCH(gd_colcount_kernel<<<blocks_for(c, adj->nnz), 256, 0, c->stream>>>(adj->idx.p, adj->nnz, colcnt.p));
        GD_LAUNCH(gd_spectral_kernel<<<blocks_for(c, n), 256, 0, c->stream>>>(adj->ptr.p, adj->idx.p, n, colcnt.p, adj->vf.p));
    } else if (P.transform == GD_COSINE) {
        SQB_TRY(cosine(c, n, adj));
    }
    return SQB_OK;
}

// the library blocks as one matrix of n_out rows
int combine(sqb_ctx* c, int64_t n_out, const std::vector<Csr>& blocks, const std::vector<DevBuf<int32_t>>& grow, const std::vector<int64_t>& nb,
            Csr* out) {
    DevBuf<int32_t> cnt(c->stream);
    DevBuf<uint8_t> tmp(c->stream);
    SQB_TRY(cnt.alloc(n_out + 1));
    SQB_TRY(out->ptr.alloc(n_out + 1));
    SQB_CUDA(cudaMemsetAsync(cnt.p, 0, (n_out + 1) * sizeof(int32_t), c->stream));
    int64_t total = 0;
    for (size_t b = 0; b < blocks.size(); ++b) {
        total += blocks[b].nnz;
        GD_LAUNCH(gd_block_count_kernel<<<blocks_for(c, nb[b]), 256, 0, c->stream>>>(blocks[b].ptr.p, grow[b].p, nb[b], cnt.p));
    }
    SQB_CHECK(total < INT_MAX, SQB_ERR_UNSUPPORTED, "the graph has %lld entries; int32 indices hold at most 2^31 - 1", (long long)total);
    SQB_TRY(exclusive_scan(c, tmp, cnt.p, out->ptr.p, n_out + 1));
    out->nnz = total, out->f64 = !blocks.empty() && blocks[0].f64;
    SQB_TRY(out->idx.alloc(total));
    SQB_TRY(out->f64 ? out->vd.alloc(total) : out->vf.alloc(total));
    for (size_t b = 0; b < blocks.size(); ++b) {
        const Csr& k = blocks[b];
        if (out->f64)
            GD_LAUNCH(gd_block_fill_kernel<double><<<blocks_for(c, nb[b]), 256, 0, c->stream>>>(k.ptr.p, k.idx.p, k.vd.p, grow[b].p, nb[b], out->ptr.p,
                                                                                               out->idx.p, out->vd.p));
        else
            GD_LAUNCH(gd_block_fill_kernel<float><<<blocks_for(c, nb[b]), 256, 0, c->stream>>>(k.ptr.p, k.idx.p, k.vf.p, grow[b].p, nb[b], out->ptr.p,
                                                                                              out->idx.p, out->vf.p));
    }
    return SQB_OK;
}

}  // namespace

extern "C" {

int sqb_graph_build_device(sqb_ctx* c, const void* xy, int xy_dtype, int64_t n, int64_t stride_row, int64_t stride_col, uintptr_t producer_stream,
                           int kind, int n_neighbors, int n_rings, double radius, int interval, double radius_min, double radius_max, int set_diag,
                           double percentile, int transform, const int64_t* lib_ptr, const int32_t* lib_rows, int n_libs, sqb_graph** out,
                           int64_t* n_out, int64_t* adj_nnz, int64_t* dst_nnz, int* dst_f64) {
    static const char* where = "sqb_graph_build_device";
    SQB_CHECK(c && out && n_out && adj_nnz && dst_nnz && dst_f64, SQB_ERR_INVALID, "%s: null argument", where);
    *out = nullptr;
    SQB_CHECK(xy || n == 0, SQB_ERR_INVALID, "%s: null coordinates", where);
    SQB_CHECK(xy_dtype == 0 || xy_dtype == 1, SQB_ERR_INVALID, "%s: xy_dtype must be 0 (float32) or 1 (float64)", where);
    SQB_CHECK(n >= 0 && n < 2147483647LL, SQB_ERR_INVALID, "%s: n=%lld out of range", where, (long long)n);
    SQB_CHECK(kind >= GD_KNN && kind <= GD_DELAUNAY, SQB_ERR_INVALID, "%s: kind must be 0 (kNN), 1 (grid), 2 (radius) or 3 (Delaunay)", where);
    SQB_CHECK(transform >= GD_NONE && transform <= GD_COSINE, SQB_ERR_INVALID, "%s: transform must be 0 (none), 1 (spectral) or 2 (cosine)", where);
    SQB_CHECK(kind != GD_GRID || n_rings >= 1, SQB_ERR_INVALID, "%s: n_rings must be positive", where);
    SQB_CHECK(kind != GD_RADIUS || (radius >= 0.0 && isfinite(radius)), SQB_ERR_INVALID, "sqb_radius_2d: radius must be finite and non-negative");
    SQB_CHECK(isnan(percentile) || (percentile >= 0.0 && percentile <= 100.0), SQB_ERR_INVALID, "Percentiles must be in the range [0, 100]");
    SQB_CHECK(n_libs >= 0 && (n_libs == 0 || (lib_ptr && lib_rows)), SQB_ERR_INVALID, "%s: library index lists missing", where);
    Params P{kind, n_neighbors, n_rings, set_diag ? 1 : 0, (kind == GD_RADIUS || kind == GD_DELAUNAY) && interval ? 1 : 0, transform, radius, radius_min, radius_max,
             kind == GD_GRID ? NAN : percentile};
    // libraries: ascending, distinct rows of [0, n); output row = rank among all listed rows (the host's argsort of the blocks)
    std::vector<int32_t> rank;
    if (n_libs > 0) {
        SQB_CHECK(lib_ptr[0] == 0 && lib_ptr[n_libs] <= n, SQB_ERR_INVALID, "%s: library pointers must run from 0 to at most n", where);
        rank.assign((size_t)n, -1);
        for (int b = 0; b < n_libs; ++b) {
            SQB_CHECK(lib_ptr[b + 1] >= lib_ptr[b], SQB_ERR_INVALID, "%s: library pointers must not decrease", where);
            for (int64_t t = lib_ptr[b]; t < lib_ptr[b + 1]; ++t) {
                const int32_t r = lib_rows[t];
                SQB_CHECK(r >= 0 && r < n && rank[r] < 0 && (t == lib_ptr[b] || r > lib_rows[t - 1]), SQB_ERR_INVALID,
                          "%s: the rows of a library must be ascending, distinct observations of [0, n)", where);
                rank[r] = 0;
            }
        }
        int32_t next = 0;
        for (auto& r : rank)
            if (r == 0) r = next++;
    }
    SQB_CUDA(cudaSetDevice(c->device));
    SQB_TRY(sqb_wait_producer(c, producer_stream));
    const Coords co{xy, xy_dtype, stride_row, stride_col};
    std::unique_ptr<sqb_graph> g(new sqb_graph(c));
    if (n_libs == 0) {
        g->n = n;
        SQB_TRY(build_block(c, co, nullptr, n, P, &g->adj, &g->dst));
    } else {
        g->n = lib_ptr[n_libs];
        std::vector<Csr> ba, bd;
        std::vector<DevBuf<int32_t>> rows, grow;
        std::vector<int64_t> nb(n_libs);
        for (int b = 0; b < n_libs; ++b) {
            ba.emplace_back(c->stream), bd.emplace_back(c->stream), rows.emplace_back(c->stream), grow.emplace_back(c->stream);
            nb[b] = lib_ptr[b + 1] - lib_ptr[b];
            std::vector<int32_t> gr(nb[b] > 0 ? nb[b] : 1);
            for (int64_t r = 0; r < nb[b]; ++r) gr[r] = rank[lib_rows[lib_ptr[b] + r]];
            SQB_TRY(rows[b].alloc(nb[b]));
            SQB_TRY(grow[b].alloc(nb[b]));
            SQB_CUDA(cudaMemcpyAsync(rows[b].p, lib_rows + lib_ptr[b], nb[b] * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
            SQB_CUDA(cudaMemcpyAsync(grow[b].p, gr.data(), nb[b] * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
            SQB_CUDA(cudaStreamSynchronize(c->stream));  // gr is released at the end of this iteration
            SQB_TRY(build_block(c, co, rows[b].p, nb[b], P, &ba[b], &bd[b]));
        }
        SQB_TRY(combine(c, g->n, ba, grow, nb, &g->adj));
        SQB_TRY(combine(c, g->n, bd, grow, nb, &g->dst));
    }
    SQB_CUDA(cudaStreamSynchronize(c->stream));  // surfaces an asynchronous fault of the build here
    *n_out = g->n, *adj_nnz = g->adj.nnz, *dst_nnz = g->dst.nnz, *dst_f64 = g->dst.f64 ? 1 : 0;
    *out = g.release();
    return SQB_OK;
}

int sqb_graph_export(sqb_graph* g, int32_t* adj_indptr, int32_t* adj_indices, float* adj_data, int32_t* dst_indptr, int32_t* dst_indices,
                     void* dst_data, uintptr_t consumer_stream) {
    SQB_CHECK(g && adj_indptr && dst_indptr, SQB_ERR_INVALID, "sqb_graph_export: null argument");
    SQB_CHECK((adj_indices && adj_data) || g->adj.nnz == 0, SQB_ERR_INVALID, "sqb_graph_export: null connectivities buffer");
    SQB_CHECK((dst_indices && dst_data) || g->dst.nnz == 0, SQB_ERR_INVALID, "sqb_graph_export: null distances buffer");
    sqb_ctx* c = g->c;
    SQB_CUDA(cudaSetDevice(c->device));
    SQB_TRY(sqb_wait_producer(c, consumer_stream));  // the stream that allocated the buffers
    const int64_t n = g->n;
    auto copy = [&](void* dst, const void* src, size_t bytes) -> int {
        if (bytes) SQB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, c->stream));
        return SQB_OK;
    };
    SQB_TRY(copy(adj_indptr, g->adj.ptr.p, (n + 1) * sizeof(int32_t)));
    SQB_TRY(copy(dst_indptr, g->dst.ptr.p, (n + 1) * sizeof(int32_t)));
    SQB_TRY(copy(adj_indices, g->adj.idx.p, g->adj.nnz * sizeof(int32_t)));
    SQB_TRY(copy(adj_data, g->adj.vf.p, g->adj.nnz * sizeof(float)));
    SQB_TRY(copy(dst_indices, g->dst.idx.p, g->dst.nnz * sizeof(int32_t)));
    SQB_TRY(g->dst.f64 ? copy(dst_data, g->dst.vd.p, g->dst.nnz * sizeof(double)) : copy(dst_data, g->dst.vf.p, g->dst.nnz * sizeof(float)));
    SQB_CUDA(cudaStreamSynchronize(c->stream));  // the graph is complete when the call returns
    return SQB_OK;
}

int sqb_graph_free(sqb_graph* g) {
    if (!g) return SQB_OK;
    SQB_CUDA(cudaSetDevice(g->c->device));
    delete g;
    return SQB_OK;
}

}  // extern "C"
