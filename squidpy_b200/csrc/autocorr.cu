// autocorr.cu — Moran's I / Geary's C for every feature over a sparse weight matrix W (sm_90a).
//
// Replaces the scanpy.metrics.morans_i / gearys_c call of the reference (src/squidpy/gr/_ppatterns.py:216 and,
// per permutation, :267-272).  Arithmetic follows scanpy's published kernels, float64 throughout:
//     I = N/S0 * sum_i z_i * sum_j w_ij z_j / sum_i z_i^2,   z = x - mean(x)
//     C = (N-1) * sum_ij w_ij (x_i - x_j)^2 / (2 * S0 * sum_i (x_i - mean)^2)
//
// SPARSE X (AnnData's native CSR, the path BASELINE configs[2] is quoted on) — work proportional to the non-zeros:
//   The feature matrix is kept as CSR *by feature* with observation indices ascending inside a feature and every
//   segment padded to a multiple of 4 entries (16-byte vector loads).  One CTA walks one feature at a time:
//     1. the feature's stored observations S are marked in a shared-memory bitmap; word w of the bitmap also holds the
//        rank of its first stored observation (entries are sorted, so the rank is the entry's position): a lookup
//        "is j stored, and what is x_j" is ONE 8-byte shared-memory read, + popc + one cached read of the value;
//     2. for every stored observation i the row of W is fetched (packed 64/128-byte rows, 8/16 lanes per row, one
//        slot each) and  acc_i = sum_j w_ij z_j  is formed with z_j = x_j - m for stored j and -m otherwise;
//     3. the rows of W that belong to unstored observations are never touched; their contribution follows from the
//        column sums c_j = sum_i w_ij:   sum_{i not in S} (Wz)_i = c'z - sum_{i in S} (Wz)_i,
//           z'Wz   = A - m * (D - m*(S0 - E) - B)        A = sum_S z_i acc_i, B = sum_S acc_i,
//                                                         D = sum_S c_j z_j,   E = sum_S c_j
//           sum z^2 = sum_S z_i^2 + (N - |S|) m^2
//        Geary likewise:
//           sum_ij w_ij (x_i-x_j)^2 = sum_{i in S} sum_j w_ij [(x_i-x_j)^2 - [j in S] x_j^2] + sum_{j in S} c_j x_j^2.
//        The correction terms are NOT centred: Moran's carries m^2 * (S0 - E), Geary's two sums of size S0 * m^2.  When
//        every observation is stored they are 0 in exact arithmetic and rounding noise times m^2 in float64, which swamps
//        the result once m >> std(x).  A feature stored at every observation (|S| = N: uniform per CTA, and true for every
//        row permutation) therefore takes num = A for Moran, and for Geary every value is shifted by m (the terms are
//        translation invariant, so they become centred); the other features keep the formulas above, instruction for
//        instruction.  Features stored at all but a few observations keep the uncentred terms (~1e-11 of the result).
//     4. constant feature -> NaN: the definition is 0/0, and the rounded mean of a constant is not always the constant (then
//        every z is the same tiny delta and I comes out ~1, C 0).  It is decided by exact comparison, not by sum z^2 == 0:
//        stored at every observation with all values equal (found by the rank sort at load time; sum z^2 is then taken as
//        its exact value, 0), or every stored value 0 (m = 0 exactly, so sum z^2 is 0 already).
//   A row permutation of W (g[idx, :], the permutation variant) changes neither c nor S0; D, E, sum z^2, m and the
//   Geary column term are kept per feature from the unpermuted pass.
//   Reductions are fixed-order (entry -> lane assignment, shuffle tree, sequential combine over warps) and one CTA
//   owns a feature whatever the grid size: results are bit-reproducible run to run and GPU to GPU.
// DENSE X keeps the tile formulation of round 1: features in tiles of 32 (lane = feature), a dense [N][32] slab per
//   tile, W streamed once per tile.  Every term is centred there; a feature whose values are all equal (found next to the
//   column sums) is NaN.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cuda_fp16.h>

#include <stdlib.h>

#include <algorithm>
#include <climits>
#include <thread>

#include "caller_graph.cuh"

#define TILE 32

// =====================================================================================================
// dense path (features x obs or obs x features, row-major)
// =====================================================================================================
// ---- dense features x obs (row-major) -> dense tile (transpose through shared memory) -------------------
template <typename XT>
__global__ void ac_transpose_kernel(const XT* __restrict__ x, int64_t g0, int64_t n_feat, int64_t n, XT* __restrict__ D) {
    __shared__ XT tile[TILE][33];
    const int64_t tl = blockIdx.y;
    const int64_t c0 = (int64_t)blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
    for (int r = ty; r < TILE; r += 8) {
        const int64_t g = g0 + tl * TILE + r;
        const int64_t c = c0 + tx;
        tile[r][tx] = (g < n_feat && c < n) ? x[g * n + c] : (XT)0;
    }
    __syncthreads();
    XT* __restrict__ Dt = D + tl * n * TILE;
    for (int r = ty; r < 32; r += 8) {
        const int64_t c = c0 + r;
        if (c < n) Dt[c * TILE + tx] = tile[tx][r];
    }
}

// ---- column sums of a dense tile (fixed order): partial[tile][warp][lane] --------------------------------
// pdiff[tile][warp][lane]: does any value of the warp's range differ from the feature's first value (constant features)
template <typename XT>
__global__ void ac_colsum_kernel(const XT* __restrict__ D, int64_t pitch, int64_t tile_stride, int64_t n,
                                 int64_t obs_per_warp, double* __restrict__ partial, int* __restrict__ pdiff, int64_t g0,
                                 int64_t n_feat) {
    const int lane = threadIdx.x & 31;
    const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t tl = blockIdx.y;
    const bool valid = g0 + tl * TILE + lane < n_feat;
    const XT* __restrict__ Dt = D + tl * tile_stride;
    int64_t r0 = w * obs_per_warp, r1 = r0 + obs_per_warp;
    if (r1 > n) r1 = n;
    double s = 0.0;
    int differs = 0;
    if (valid) {
        const XT x0 = Dt[lane];
        for (int64_t r = r0; r < r1; ++r) {
            const XT x = Dt[r * pitch + lane];
            s += (double)x;
            differs |= x != x0;
        }
    }
    partial[(tl * nw + w) * TILE + lane] = s;
    pdiff[(tl * nw + w) * TILE + lane] = differs;
}

// sums[tile][lane] = column sum; varies[tile][lane] = 0 when every value of the feature is equal
__global__ void ac_colsum_final_kernel(const double* __restrict__ partial, const int* __restrict__ pdiff, int64_t nw,
                                       double* __restrict__ sums, int* __restrict__ varies) {
    const int lane = threadIdx.x;
    const int64_t tl = blockIdx.x;
    double s = 0.0;
    int d = 0;
    for (int64_t w = 0; w < nw; ++w) {
        s += partial[(tl * nw + w) * TILE + lane];
        d |= pdiff[(tl * nw + w) * TILE + lane];
    }
    sums[tl * TILE + lane] = s;
    varies[tl * TILE + lane] = d;
}

// ---- dense SpMM-style kernel -----------------------------------------------------------------------------
// MODE 0: Moran (num = sum_r z_r * sum_e w_e z_{j_e}), MODE 1: Geary (num = sum_r sum_e w_e (x_r - x_{j_e})^2).
// den = sum_r z_r^2 in both modes.  lane = feature; warp = contiguous observation range.
template <typename XT, int MODE>
__global__ void __launch_bounds__(256) ac_main_kernel(const int32_t* __restrict__ wp, const int32_t* __restrict__ wi,
                                                      const double* __restrict__ wd, const XT* __restrict__ D,
                                                      int64_t pitch, int64_t tile_stride, int64_t n, int64_t obs_per_warp,
                                                      const double* __restrict__ sums, const int64_t* __restrict__ row_perm,
                                                      double* __restrict__ pnum, double* __restrict__ pden, int64_t g0,
                                                      int64_t n_feat) {
    const int lane = threadIdx.x & 31;
    const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t tl = blockIdx.y;
    const bool valid = g0 + tl * TILE + lane < n_feat;
    const XT* __restrict__ Dt = D + tl * tile_stride + lane;
    const double mean = sums[tl * TILE + lane] / (double)n;
    int64_t r0 = w * obs_per_warp, r1 = r0 + obs_per_warp;
    if (r1 > n) r1 = n;
    double num = 0.0, den = 0.0;
    if (valid) {
        for (int64_t r = r0; r < r1; ++r) {
            const int64_t src = row_perm ? row_perm[r] : r;
            const int32_t beg = wp[src], end = wp[src + 1];
            const double xr = (double)Dt[r * pitch];
            const double zr = xr - mean;
            double acc = 0.0;
#pragma unroll 4
            for (int32_t e = beg; e < end; ++e) {
                const double xj = (double)Dt[(int64_t)wi[e] * pitch];
                if (MODE == 0) {
                    acc = fma(wd[e], xj - mean, acc);
                } else {
                    const double d = xr - xj;
                    acc = fma(wd[e], d * d, acc);
                }
            }
            if (MODE == 0)
                num = fma(acc, zr, num);
            else
                num += acc;
            den = fma(zr, zr, den);
        }
    }
    // fixed-order combine of the 8 warps of this CTA -> one partial per (tile, CTA)
    __shared__ double s_num[8][TILE], s_den[8][TILE];
    s_num[threadIdx.x >> 5][lane] = num;
    s_den[threadIdx.x >> 5][lane] = den;
    __syncthreads();
    if (threadIdx.x < TILE) {
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            a += s_num[k][lane];
            b += s_den[k][lane];
        }
        pnum[(tl * gridDim.x + blockIdx.x) * TILE + lane] = a;
        pden[(tl * gridDim.x + blockIdx.x) * TILE + lane] = b;
    }
}

template <int MODE>
__global__ void __launch_bounds__(256) ac_final_kernel(const double* __restrict__ pnum, const double* __restrict__ pden,
                                                       const int* __restrict__ varies, int64_t nparts, int64_t n, double s0,
                                                       int64_t g0, int64_t n_feat, double* __restrict__ out) {
    // 8 warps sum contiguous ranges of the per-CTA partials (lane = feature), then warp 0 combines them in order
    __shared__ double s_num[8][TILE], s_den[8][TILE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t tl = blockIdx.x;
    const int64_t chunk = (nparts + 7) / 8;
    int64_t p0 = warp * chunk, p1 = p0 + chunk;
    if (p1 > nparts) p1 = nparts;
    double num = 0.0, den = 0.0;
    for (int64_t w = p0; w < p1; ++w) {
        num += pnum[(tl * nparts + w) * TILE + lane];
        den += pden[(tl * nparts + w) * TILE + lane];
    }
    s_num[warp][lane] = num;
    s_den[warp][lane] = den;
    __syncthreads();
    const int64_t g = g0 + tl * TILE + lane;
    if (warp != 0 || g >= n_feat) return;
    num = 0.0;
    den = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        num += s_num[k][lane];
        den += s_den[k][lane];
    }
    double r;
    if (den == 0.0 || !varies[tl * TILE + lane]) {
        r = __longlong_as_double(0x7ff8000000000000LL);  // constant feature -> NaN (0/0; the rounded mean need not be the value)
    } else if (MODE == 0) {
        r = (double)n / s0 * num / den;
    } else {
        r = ((double)(n - 1) * num) / (2.0 * s0 * den);
    }
    out[g] = r;
}

// =====================================================================================================
// sparse path
// =====================================================================================================
#define AC_T 256          // threads per CTA of the per-feature kernels
#define AC_NW (AC_T / 32)

enum { AC_ERR_INDEX = 1, AC_ERR_DUP = 2, AC_ERR_PERM = 8, AC_W_NONCANON = 16, AC_W_NONFINITE = 32 };

// ---- input validation / transposition (load time) ----------------------------------------------------
// Output feature of input column c, or -1 to skip it (range errors raise *err unless err is null).  colmap == null: the shard [col_lo, col_lo + n_feat) of the columns,
// anything outside is an error; else colmap[c] for c in [0, n_cols).
__device__ __forceinline__ int64_t ac_map_col(int64_t c, int64_t n_feat, int32_t col_lo, const int32_t* __restrict__ colmap,
                                              int64_t n_cols, int* __restrict__ err) {
    if (colmap) {
        if (c < 0 || c >= n_cols) {
            if (err) atomicOr(err, AC_ERR_INDEX);
            return -1;
        }
        return colmap[c];
    }
    c -= col_lo;
    if (c < 0 || c >= n_feat) {
        if (err) atomicOr(err, AC_ERR_INDEX);
        return -1;
    }
    return c;
}

// per-column entry counts of a CSR-by-observation matrix; out-of-range column -> error flag.
// Shared-memory histogram per CTA when n_feat fits (hist_smem), else global atomics.
template <typename II>
__global__ void ac_colcount_kernel(const II* __restrict__ xi, int64_t nnz, int64_t n_feat, int32_t col_lo,
                                   const int32_t* __restrict__ colmap, int64_t n_cols, int hist_smem,
                                   unsigned int* __restrict__ cnt, int* __restrict__ err) {
    extern __shared__ unsigned int s_hist[];
    if (hist_smem)
        for (int64_t c = threadIdx.x; c < n_feat; c += blockDim.x) s_hist[c] = 0;
    __syncthreads();
    const int64_t per = (nnz + gridDim.x - 1) / gridDim.x;
    const int64_t e0 = blockIdx.x * per, e1 = e0 + per < nnz ? e0 + per : nnz;
    for (int64_t e = e0 + threadIdx.x; e < e1; e += blockDim.x) {
        const int64_t c = ac_map_col((int64_t)xi[e], n_feat, col_lo, colmap, n_cols, err);
        if (c < 0) continue;
        if (hist_smem)
            atomicAdd(&s_hist[c], 1u);
        else
            atomicAdd(&cnt[c], 1u);
    }
    if (!hist_smem) return;
    __syncthreads();
    for (int64_t c = threadIdx.x; c < n_feat; c += blockDim.x) {
        const unsigned int v = s_hist[c];
        if (v) atomicAdd(&cnt[c], v);
    }
}

// ptr[g] = exclusive prefix of cnt, pad[g] = exclusive prefix of cnt rounded up to 4, cursor[g] = ptr[g]
// (single CTA; n_feat + 1 outputs)
__global__ void __launch_bounds__(1024) ac_scan_counts_kernel(const unsigned int* __restrict__ cnt, int64_t n_feat,
                                                              int64_t* __restrict__ ptr, int64_t* __restrict__ pad,
                                                              unsigned long long* __restrict__ cursor) {
    __shared__ int64_t s_a[32], s_b[32];
    __shared__ int64_t s_run[2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_run[0] = s_run[1] = 0;
    __syncthreads();
    for (int64_t base = 0; base <= n_feat; base += 1024) {
        const int64_t g = base + threadIdx.x;
        const int64_t c = g < n_feat ? (int64_t)cnt[g] : 0;
        int64_t a = c, b = (c + 3) & ~(int64_t)3;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int64_t ta = __shfl_up_sync(0xffffffffu, a, d), tb = __shfl_up_sync(0xffffffffu, b, d);
            if (lane >= d) {
                a += ta;
                b += tb;
            }
        }
        if (lane == 31) {
            s_a[warp] = a;
            s_b[warp] = b;
        }
        __syncthreads();
        if (warp == 0) {
            int64_t va = s_a[lane], vb = s_b[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int64_t ta = __shfl_up_sync(0xffffffffu, va, d), tb = __shfl_up_sync(0xffffffffu, vb, d);
                if (lane >= d) {
                    va += ta;
                    vb += tb;
                }
            }
            s_a[lane] = va - s_a[lane];  // exclusive over warps
            s_b[lane] = vb - s_b[lane];
        }
        __syncthreads();
        const int64_t ea = s_run[0] + s_a[warp] + a - c, eb = s_run[1] + s_b[warp] + b - ((c + 3) & ~(int64_t)3);
        if (g <= n_feat) {
            if (ptr) ptr[g] = ea;
            pad[g] = eb;
            if (cursor) cursor[g] = (unsigned long long)ea;
        }
        __syncthreads();
        if (threadIdx.x == 1023) {
            s_run[0] = ea + c;
            s_run[1] = eb + ((c + 3) & ~(int64_t)3);
        }
        __syncthreads();
    }
}

// segments of the selected features of a caller's CSR by feature: feature k is input row inv[k]
template <typename IP>
__global__ void ac_select_segs_kernel(const IP* __restrict__ ptr, const int32_t* __restrict__ inv, int64_t n_out,
                                      int64_t* __restrict__ beg, int64_t* __restrict__ end, unsigned int* __restrict__ cnt,
                                      int64_t n, int* __restrict__ err) {
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n_out; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t a = (int64_t)ptr[inv[k]], b = (int64_t)ptr[inv[k] + 1];  // validated non-decreasing
        beg[k] = a;
        end[k] = b;
        int64_t d = b - a;
        if (d > n) {
            atomicOr(err, AC_ERR_DUP);
            d = n;
        }
        cnt[k] = (unsigned int)d;
    }
}

// CSR by observation -> unsorted segments by feature (atomic cursor; the rank sort below orders them)
template <typename IP, typename II, typename VT, typename XT>
__global__ void ac_coltranspose_kernel(const IP* __restrict__ xp, const II* __restrict__ xi,
                                       const VT* __restrict__ xv, int64_t n_obs, int64_t n_feat, int32_t col_lo,
                                       const int32_t* __restrict__ colmap, int64_t n_cols,
                                       unsigned long long* __restrict__ cursor, int32_t* __restrict__ oi, XT* __restrict__ ov) {
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; r < n_obs; r += nw) {
        const int64_t e1 = (int64_t)xp[r + 1];
        for (int64_t e = (int64_t)xp[r] + lane; e < e1; e += 32) {
            const int64_t c = ac_map_col((int64_t)xi[e], n_feat, col_lo, colmap, n_cols, nullptr);  // flagged by the count kernel
            if (c < 0) continue;
            const unsigned long long pos = atomicAdd(&cursor[c], 1ULL);
            oi[pos] = (int32_t)r;
            ov[pos] = sqb_cvt<XT>(xv[e]);
        }
    }
}

// Dense gather of the selected features of a strided device array (element strides s_obs / s_feat, any sign) into the layout
// sqb_autocorr_load_dense produces: obs_major = 1 -> [n_obs][n_out], 0 -> [n_out][n_obs]; feature k is input feature inv[k].
template <typename VT, typename XT>
__global__ void ac_gather_dense_kernel(const VT* __restrict__ x, int64_t n_obs, int64_t n_out, int64_t s_obs, int64_t s_feat,
                                       const int32_t* __restrict__ inv, int obs_major, XT* __restrict__ out) {
    const int64_t total = n_obs * n_out;
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = obs_major ? t / n_out : t % n_obs;
        const int64_t k = obs_major ? t - r * n_out : t / n_obs;
        out[t] = sqb_cvt<XT>(x[r * s_obs + (int64_t)inv[k] * s_feat]);
    }
}

// ---- bitmap + rank structure ------------------------------------------------------------------------------
// S[w] = { bits of the observations 32w .. 32w+31 stored for the feature, rank of the first of them }
__device__ __forceinline__ void ac_zero_words(uint2* S, int nwords) {
    for (int w = threadIdx.x; w < nwords; w += AC_T) S[w] = make_uint2(0u, 0u);
}

// exclusive prefix of popc(S[w].x) into S[w].y; returns the total through s_tmp[32] (all threads must call)
__device__ __forceinline__ unsigned int ac_scan_words(uint2* S, int nwords, unsigned int* s_tmp) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int chunk = (nwords + AC_T - 1) / AC_T;
    int w0 = threadIdx.x * chunk, w1 = w0 + chunk;
    if (w0 > nwords) w0 = nwords;
    if (w1 > nwords) w1 = nwords;
    unsigned int cnt = 0;
    for (int w = w0; w < w1; ++w) cnt += __popc(S[w].x);
    unsigned int inc = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned int t = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += t;
    }
    if (lane == 31) s_tmp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        const unsigned int v = lane < AC_NW ? s_tmp[lane] : 0u;
        unsigned int s = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned int t = __shfl_up_sync(0xffffffffu, s, d);
            if (lane >= d) s += t;
        }
        if (lane < AC_NW) s_tmp[lane] = s - v;
        if (lane == AC_NW - 1) s_tmp[AC_NW] = s;
    }
    __syncthreads();
    unsigned int run = inc - cnt + s_tmp[warp];
    for (int w = w0; w < w1; ++w) {
        const unsigned int b = S[w].x;
        S[w].y = run;
        run += __popc(b);
    }
    const unsigned int total = s_tmp[AC_NW];
    __syncthreads();
    return total;
}

// One CTA per feature: order the (observation, value) pairs of a segment by observation (rank = number of stored
// observations below), write them to the padded segment, pad with index -1 / value 0.  Out-of-range or repeated
// observation indices raise the error flag.  Segment g is in_idx / in_val [in_beg[g], in_end[g]).  seg_const[g] = 1 when the
// feature is stored at every observation with every value equal.
template <typename II, typename VT, typename XT>
__global__ void __launch_bounds__(AC_T) ac_rank_sort_kernel(const int64_t* __restrict__ in_beg, const int64_t* __restrict__ in_end,
                                                             const II* __restrict__ in_idx, const VT* __restrict__ in_val,
                                                             const int64_t* __restrict__ out_start,
                                                             int32_t* __restrict__ out_idx, XT* __restrict__ out_val,
                                                             int32_t* __restrict__ seg_len, int32_t* __restrict__ seg_const,
                                                             int64_t n, int64_t n_feat,
                                                             int nwords, uint2* __restrict__ s_global, int* __restrict__ err) {
    extern __shared__ __align__(16) unsigned char ac_smem[];
    __shared__ unsigned int s_tmp[AC_NW + 1];
    uint2* S = s_global ? s_global + (size_t)blockIdx.x * nwords : reinterpret_cast<uint2*>(ac_smem);
    ac_zero_words(S, nwords);
    __syncthreads();
    for (int64_t g = blockIdx.x; g < n_feat; g += gridDim.x) {
        const int64_t rb = in_beg[g];
        int64_t len64 = in_end[g] - rb;
        if (len64 < 0) len64 = 0;
        if (len64 > n) {  // more entries than observations: some observation repeats
            if (threadIdx.x == 0) atomicOr(err, AC_ERR_DUP);
            len64 = n;
        }
        const int len = (int)len64;
        const int64_t os = out_start[g];
        for (int e = threadIdx.x; e < len; e += AC_T) {
            const int64_t i = (int64_t)in_idx[rb + e];
            if (i < 0 || i >= n) {
                atomicOr(err, AC_ERR_INDEX);
                continue;
            }
            const unsigned int bit = 1u << (i & 31);
            if (atomicOr(&S[i >> 5].x, bit) & bit) atomicOr(err, AC_ERR_DUP);
        }
        __syncthreads();
        ac_scan_words(S, nwords, s_tmp);
        for (int e = threadIdx.x; e < len; e += AC_T) {
            const int64_t i = (int64_t)in_idx[rb + e];
            if (i < 0 || i >= n) continue;
            const uint2 s = S[i >> 5];
            const unsigned int bit = 1u << (i & 31);
            const int64_t pos = os + s.y + __popc(s.x & (bit - 1u));
            out_idx[pos] = (int32_t)i;
            out_val[pos] = sqb_cvt<XT>(in_val[rb + e]);
        }
        const int lenp = (len + 3) & ~3;
        for (int e = len + threadIdx.x; e < lenp; e += AC_T) {
            out_idx[os + e] = -1;
            out_val[os + e] = (XT)0;
        }
        // stored at every observation with all values equal: a constant feature (0/0), whatever its rounded mean is
        int differs = 0;
        if (len == n)
            for (int e = threadIdx.x; e < len; e += AC_T) differs |= sqb_cvt<XT>(in_val[rb + e]) != sqb_cvt<XT>(in_val[rb]);
        const int varies = __syncthreads_or(differs);
        if (threadIdx.x == 0) {
            seg_len[g] = len;
            seg_const[g] = len == n && !varies;
        }
        __syncthreads();
        ac_zero_words(S, nwords);
        __syncthreads();
    }
}

// ---- W preprocessing ---------------------------------------------------------------------------------------
// packed rows: LPR slots of 8 bytes {column (int32, -1 = empty), weight (float32)}
template <int LPR>
__global__ void ac_pack_rows_kernel(const int32_t* __restrict__ wp, const int32_t* __restrict__ wi, const double* __restrict__ wd,
                                    int64_t n, uint2* __restrict__ rows) {
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n * LPR; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = t / LPR;
        const int32_t e = wp[r] + (int)(t % LPR);
        rows[t] = e < wp[r + 1] ? make_uint2((unsigned int)wi[e], __float_as_uint((float)wd[e])) : make_uint2(0xffffffffu, 0u);
    }
}

// compact rows (FMT 3): 8 slots of 4 bytes = 7 columns (-1 = empty) + the float32 weight ALL entries of the row share (the
// row-normalised binary graph of the standard pipeline): one 32-byte sector per row instead of a 64-byte line
__global__ void ac_pack_rows32_kernel(const int32_t* __restrict__ wp, const int32_t* __restrict__ wi, const double* __restrict__ wd,
                                      int64_t n, uint32_t* __restrict__ rows) {
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n * 8; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = t >> 3;
        const int s = (int)(t & 7);
        const int32_t b = wp[r], e = wp[r + 1];
        if (s < 7) rows[t] = b + s < e ? (uint32_t)wi[b + s] : 0xffffffffu;
        else rows[t] = e > b ? __float_as_uint((float)wd[b]) : 0u;
    }
}

// row permutation: int64 host layout -> int32, validated on the device (bitmap of seen sources)
__global__ void ac_perm_prepare_kernel(const int64_t* __restrict__ in, int64_t n, int32_t* __restrict__ out,
                                       unsigned int* __restrict__ seen, int* __restrict__ err) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = in[r];
        if (s < 0 || s >= n) {
            atomicOr(err, AC_ERR_PERM);
            out[r] = 0;
            continue;
        }
        const unsigned int bit = 1u << (s & 31);
        if (atomicOr(&seen[s >> 5], bit) & bit) atomicOr(err, AC_ERR_PERM);
        out[r] = (int32_t)s;
    }
}

// ---- the per-feature kernel ---------------------------------------------------------------------------------
struct AcSparseParams {
    int64_t n, n_feat;
    int nwords;
    uint2* s_global;  // bitmap scratch in global memory (nwords per CTA) when it does not fit shared memory, else null
    const int64_t* seg_start;
    const int32_t* seg_len;
    const int32_t* seg_const;  // 1: stored at every observation, every value equal (set by the rank sort)
    const int32_t* order;  // features by decreasing length (longest first), or null
    const int32_t* xi;
    const void* xv;
    // W
    const uint2* rows;  // packed rows (FMT 0 / 1)
    const int32_t* wp;  // CSR (FMT 2)
    const int32_t* wi;
    const double* wd;
    const double* csum;
    double s0;
    const int32_t* perm;  // PERM: n_perm row permutations [n_perm][n] (one feature pass serves all of them), else null
    int n_perm;           // PERM: permutations per launch; outputs go to out[b * n_feat + g]
    double* aux;          // [5][n_feat]: mean, sum z^2 over stored, D, E, Geary column term (written by unpermuted runs; the
                          // column term depends on the mode, so permuted runs read it only after one of their own mode)
    double* out;
    int* counter;  // dynamic feature queue
};

// fixed-order block reduction of NQ doubles; result valid in thread 0
template <int NQ>
__device__ __forceinline__ void ac_block_reduce(double (&q)[NQ], double (*s_red)[AC_NW]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < NQ; ++k) {
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) q[k] += __shfl_xor_sync(0xffffffffu, q[k], d);
        if (lane == 0) s_red[k][warp] = q[k];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < NQ; ++k) {
            double t = 0.0;
#pragma unroll
            for (int w = 0; w < AC_NW; ++w) t += s_red[k][w];
            q[k] = t;
        }
    }
}

// FMT 0: packed rows, 8 lanes per row (<= 8 entries);  FMT 1: packed rows, 16 lanes per row (<= 16 entries);
// FMT 2: CSR rows, 8 lanes per row (any length; float64 weights);  FMT 3: compact rows, 8 lanes per row (<= 7 entries of one
// common float32 weight: 32 bytes per row).
template <typename XT, int MODE, int FMT, bool PERM, int GRP>
__global__ void __launch_bounds__(AC_T, GRP == 8 ? 3 : 4) ac_sparse_kernel(const __grid_constant__ AcSparseParams p) {
    constexpr int LPR = FMT == 1 ? 16 : 8;
    constexpr int RPW = 32 / LPR;        // rows per warp step
    constexpr int NSUB = 32 / RPW;       // warp steps per block of 32 entries
    // GRP = warp steps handled together: GRP independent row loads / look-ups / value loads in flight per warp
    extern __shared__ __align__(16) unsigned char ac_smem[];
    __shared__ double s_red[6][AC_NW];
    __shared__ double s_mean;
    __shared__ int s_next;
    uint2* S = p.s_global ? p.s_global + (size_t)blockIdx.x * p.nwords : reinterpret_cast<uint2*>(ac_smem);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int slot = lane % LPR, sub = lane / LPR;
    const double dn = (double)p.n;
    ac_zero_words(S, p.nwords);
    __syncthreads();
    for (;;) {
        if (threadIdx.x == 0) s_next = atomicAdd(p.counter, 1);
        __syncthreads();
        const int k = s_next;
        if (k >= p.n_feat) break;
        const int g = p.order ? p.order[k] : k;
        const int64_t b = p.seg_start[g];
        const int len = p.seg_len[g];
        const bool full = len == p.n;  // every observation stored: no correction term (see the header)
        const int32_t* __restrict__ xi = p.xi + b;
        const XT* __restrict__ xv = reinterpret_cast<const XT*>(p.xv) + b;
        const int len4 = (len + 3) >> 2;
        // ---- phase 1: mark the stored observations, rank of the first one of every word, sum of the values ----
        double q[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll 2
        for (int v = threadIdx.x; v < len4; v += AC_T) {
            const int4 iv = __ldg(reinterpret_cast<const int4*>(xi) + v);
            const int prev = v > 0 ? __ldg(xi + 4 * v - 1) : -1;
            const int ii[4] = {iv.x, iv.y, iv.z, iv.w};
            if (!PERM) {
                double xs[4];
                if (sizeof(XT) == 4) {
                    const float4 f = __ldg(reinterpret_cast<const float4*>(xv) + v);
                    xs[0] = f.x, xs[1] = f.y, xs[2] = f.z, xs[3] = f.w;
                } else {
                    const double2 d0 = __ldg(reinterpret_cast<const double2*>(xv) + 2 * v);
                    const double2 d1 = __ldg(reinterpret_cast<const double2*>(xv) + 2 * v + 1);
                    xs[0] = d0.x, xs[1] = d0.y, xs[2] = d1.x, xs[3] = d1.y;
                }
                q[0] += ((xs[0] + xs[1]) + xs[2]) + xs[3];  // pads hold 0
            }
            int cur_w = prev >= 0 ? prev >> 5 : -1;  // word of the previous entry
            int open_w = -1;
            unsigned int mask = 0;
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const int i = ii[t];
                if (i < 0) break;
                const int w = i >> 5;
                if (w != open_w) {
                    if (open_w >= 0) atomicOr(&S[open_w].x, mask);
                    open_w = w;
                    mask = 0;
                }
                mask |= 1u << (i & 31);
                if (w != cur_w) {
                    S[w].y = (unsigned int)(4 * v + t);  // first stored observation of this word
                    cur_w = w;
                }
            }
            if (open_w >= 0) atomicOr(&S[open_w].x, mask);
        }
        double m;
        if (!PERM) {
            double q1[1] = {q[0]};
            ac_block_reduce<1>(q1, s_red);  // contains a __syncthreads after the shuffles
            if (threadIdx.x == 0) s_mean = q1[0] / dn;
            __syncthreads();
            m = s_mean;
            q[0] = 0.0;
            // ---- phase 1b (unpermuted pass only): the column-sum terms D = sum c z, E = sum c, sum z^2, Geary's sum c x^2 ----
#pragma unroll 2
            for (int v = threadIdx.x; v < len4; v += AC_T) {
                const int4 iv = __ldg(reinterpret_cast<const int4*>(xi) + v);
                const int ii[4] = {iv.x, iv.y, iv.z, iv.w};
                double xs[4], cs[4];
                if (sizeof(XT) == 4) {
                    const float4 f = __ldg(reinterpret_cast<const float4*>(xv) + v);
                    xs[0] = f.x, xs[1] = f.y, xs[2] = f.z, xs[3] = f.w;
                } else {
                    const double2 d0 = __ldg(reinterpret_cast<const double2*>(xv) + 2 * v);
                    const double2 d1 = __ldg(reinterpret_cast<const double2*>(xv) + 2 * v + 1);
                    xs[0] = d0.x, xs[1] = d0.y, xs[2] = d1.x, xs[3] = d1.y;
                }
#pragma unroll
                for (int t = 0; t < 4; ++t) cs[t] = ii[t] >= 0 ? __ldg(p.csum + ii[t]) : 0.0;
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    if (ii[t] < 0) continue;
                    const double zi = xs[t] - m;
                    q[2] = fma(cs[t], zi, q[2]);
                    q[3] += cs[t];
                    q[4] = fma(zi, zi, q[4]);
                    const double xg = MODE == 1 && full ? zi : xs[t];  // Geary's shift (gs below): aux depends on the mode
                    q[5] = fma(cs[t], xg * xg, q[5]);
                }
            }
        } else {
            m = p.aux[g];
            __syncthreads();
        }
        // Geary's terms are translation invariant: a feature stored everywhere is shifted by m (every term centred, nothing of
        // size S0 * m^2 cancels); the others keep x, whose unstored values are the 0 the column-sum term assumes
        const double gs = full ? m : 0.0;
        // ---- phase 2: walk the rows of W of the stored observations; q[0], q[1] = slot accumulators ----
        // Moran: q[0] += z_i * w z_j, q[1] += w z_j;   Geary: q[0] += w ((x_i - x_j)^2 - [j stored] x_j^2)
        // PERM: the bitmap of the feature is built once and walked once per row permutation of the batch
        for (int pb = 0; pb < (PERM ? p.n_perm : 1); ++pb) {
        const int32_t* __restrict__ perm = PERM ? p.perm + (int64_t)pb * p.n : nullptr;
        if (PERM) q[0] = q[1] = 0.0;
        int nxt_i = -1;
        XT nxt_x = (XT)0;
        {
            const int e = warp * 32 + lane;
            if (e < len) {
                nxt_i = __ldg(xi + e);
                nxt_x = __ldg(xv + e);
            }
        }
        for (int base = warp * 32; base < len; base += AC_NW * 32) {
            const int my_i = nxt_i;
            const XT my_x = nxt_x;
            {  // prefetch this warp's next block of 32 entries
                const int e = base + AC_NW * 32 + lane;
                nxt_i = -1;
                nxt_x = (XT)0;
                if (e < len) {
                    nxt_i = __ldg(xi + e);
                    nxt_x = __ldg(xv + e);
                }
            }
#pragma unroll
            for (int s0 = 0; s0 < NSUB; s0 += GRP) {
                int ri[GRP];
                double rx[GRP];
                if (FMT != 2) {
                    // stage 1: the row slots; stage 2: bitmap lookups; stage 3: values of the hits; stage 4: accumulate.
                    // No branches: an empty slot / a missing row has weight 0, column 0 and a suppressed value load.
                    uint2 rs[GRP];
#pragma unroll
                    for (int s = 0; s < GRP; ++s) {
                        const int src = (s0 + s) * RPW + sub;
                        ri[s] = __shfl_sync(0xffffffffu, my_i, src);
                        rx[s] = (double)__shfl_sync(0xffffffffu, my_x, src);
                        rs[s] = make_uint2(0xffffffffu, 0u);
                        if (FMT == 3) {  // 7 columns + the row's weight: 4 bytes per lane, the weight comes from lane 7 of the row
                            unsigned int cw = 0xffffffffu;
                            if (ri[s] >= 0) {
                                const int64_t r = PERM ? (int64_t)__ldg(perm + ri[s]) : (int64_t)ri[s];
                                cw = __ldg(reinterpret_cast<const unsigned int*>(p.rows) + r * 8 + slot);
                            }
                            const unsigned int wb = __shfl_sync(0xffffffffu, cw, (lane & ~7) | 7);
                            rs[s] = make_uint2(slot == 7 ? 0xffffffffu : cw, wb);
                        } else if (ri[s] >= 0) {
                            const int64_t r = PERM ? (int64_t)__ldg(perm + ri[s]) : (int64_t)ri[s];
                            rs[s] = __ldg(p.rows + r * LPR + slot);
                        }
                    }
                    bool hit[GRP];
                    unsigned int rank[GRP];
#pragma unroll
                    for (int s = 0; s < GRP; ++s) {
                        const int j = (int)rs[s].x;
                        const int jj = j >= 0 ? j : 0;
                        const uint2 w = S[jj >> 5];
                        const unsigned int bit = 1u << (jj & 31);
                        hit[s] = j >= 0 && (w.x & bit) != 0u;
                        rank[s] = w.y + __popc(w.x & (bit - 1u));
                    }
                    XT xj[GRP];
#pragma unroll
                    for (int s = 0; s < GRP; ++s) xj[s] = hit[s] ? __ldg(xv + rank[s]) : (XT)0;
#pragma unroll
                    for (int s = 0; s < GRP; ++s) {
                        const double w = (int)rs[s].x >= 0 ? (double)__uint_as_float(rs[s].y) : 0.0;
                        const double xjd = (double)xj[s];
                        if (MODE == 0) {
                            const double t = w * (hit[s] ? xjd - m : -m);
                            q[0] = fma(rx[s] - m, t, q[0]);
                            q[1] += t;
                        } else {
                            const double d = rx[s] - xjd;
                            const double xg = xjd - gs;
                            q[0] = fma(w, d * d - xg * xg, q[0]);  // xj == 0 when not stored
                        }
                    }
                } else {
#pragma unroll
                    for (int s = 0; s < GRP; ++s) {
                        const int src = (s0 + s) * RPW + sub;
                        ri[s] = __shfl_sync(0xffffffffu, my_i, src);
                        rx[s] = (double)__shfl_sync(0xffffffffu, my_x, src);
                    }
#pragma unroll
                    for (int s = 0; s < GRP; ++s) {
                        if (ri[s] < 0) continue;
                        const int64_t r = PERM ? (int64_t)__ldg(perm + ri[s]) : (int64_t)ri[s];
                        const int rbeg = __ldg(p.wp + r), rend = __ldg(p.wp + r + 1);
                        const double zi = rx[s] - m;
                        for (int ew = rbeg + slot; ew < rend; ew += LPR) {
                            const int j = __ldg(p.wi + ew);
                            const double w = __ldg(p.wd + ew);
                            const uint2 sw = S[j >> 5];
                            const unsigned int bit = 1u << (j & 31);
                            const bool h = (sw.x & bit) != 0u;
                            const double xjd = h ? (double)__ldg(xv + (sw.y + __popc(sw.x & (bit - 1u)))) : 0.0;
                            if (MODE == 0) {
                                const double t = w * (h ? xjd - m : -m);
                                q[0] = fma(zi, t, q[0]);
                                q[1] += t;
                            } else {
                                const double d = rx[s] - xjd;
                                const double xg = xjd - gs;
                                q[0] = fma(w, d * d - xg * xg, q[0]);
                            }
                        }
                    }
                }
            }
        }
        // ---- phase 3: combine, finish the feature, clear the touched words ----
        if (!PERM) {
            ac_block_reduce<6>(q, s_red);
        } else {
            double q2[2] = {q[0], q[1]};
            ac_block_reduce<2>(q2, s_red);
            q[0] = q2[0];
            q[1] = q2[1];
        }
        if (threadIdx.x == 0) {
            double D, E, Z2, CX;
            if (!PERM) {
                D = q[2], E = q[3], Z2 = p.seg_const[g] ? 0.0 : q[4], CX = q[5];  // a constant's sum z^2 is exactly 0 (aux keeps it)
                p.aux[g] = m;
                p.aux[p.n_feat + g] = Z2;
                p.aux[2 * p.n_feat + g] = D;
                p.aux[3 * p.n_feat + g] = E;
                p.aux[4 * p.n_feat + g] = CX;
            } else {
                Z2 = p.aux[p.n_feat + g];
                D = p.aux[2 * p.n_feat + g];
                E = p.aux[3 * p.n_feat + g];
                CX = p.aux[4 * p.n_feat + g];
            }
            const double den = Z2 + (dn - (double)len) * m * m;
            double r;
            if (den == 0.0) {
                r = __longlong_as_double(0x7ff8000000000000LL);  // constant feature -> NaN (0/0)
            } else if (MODE == 0) {
                const double num = full ? q[0] : q[0] - m * (D - m * (p.s0 - E) - q[1]);
                r = dn / p.s0 * num / den;
            } else {
                const double num = q[0] + CX;
                r = ((dn - 1.0) * num) / (2.0 * p.s0 * den);
            }
            p.out[(int64_t)pb * p.n_feat + g] = r;
        }
        if (PERM) __syncthreads();  // s_red is reused by the next permutation of the batch
        }  // permutations of the batch
#pragma unroll 4
        for (int v = threadIdx.x; v < len4; v += AC_T) {
            const int4 iv = __ldg(reinterpret_cast<const int4*>(xi) + v);
            if (iv.x >= 0) S[iv.x >> 5] = make_uint2(0u, 0u);
            if (iv.y >= 0) S[iv.y >> 5] = make_uint2(0u, 0u);
            if (iv.z >= 0) S[iv.z >> 5] = make_uint2(0u, 0u);
            if (iv.w >= 0) S[iv.w >> 5] = make_uint2(0u, 0u);
        }
        __syncthreads();
    }
}

// ================================================================================================
// Every buffer of a handle is allocated, used and freed in ctx->stream order, from the device pool: a handle is created and
// destroyed per API call, and GB-sized cudaMalloc / cudaFree pairs would synchronise the device every time.  The buffers'
// initialisers read ctx, which is declared first.
struct sqb_autocorr {
    explicit sqb_autocorr(sqb_ctx* c) : ctx(c) {}
    sqb_ctx* ctx;
    int64_t n = 0, nnz = 0;
    double s0 = 0.0;
    int s0_branch = 0;  // how S0 was summed: 0 the exact integer sum of w / g (parallel), 1 one ordered thread
    int w_fmt = 2;  // 0 packed 8 lanes, 1 packed 16 lanes, 2 CSR, 3 compact (7 columns + one common weight in 32 bytes)
    DevBuf<int32_t> d_wp{ctx->stream}, d_wi{ctx->stream};
    DevBuf<double> d_wd{ctx->stream}, d_csum{ctx->stream};
    DevBuf<uint2> d_rows{ctx->stream};
    // loaded X
    int kind = 0;     // 0 none, 1 dense feat x obs, 2 dense obs x feat (zero copy tiles), 3 sparse (padded CSR by feature)
    int x_dtype = 0;  // 0 f32, 1 f64
    int64_t n_feat = 0;
    DevBuf<uint8_t> d_x{ctx->stream};   // dense matrix or padded sparse values
    DevBuf<int64_t> d_xp{ctx->stream};  // padded segment starts (n_feat + 1)
    DevBuf<int32_t> d_xi{ctx->stream}, d_len{ctx->stream}, d_const{ctx->stream}, d_order{ctx->stream};
    DevBuf<uint8_t> d_tile{ctx->stream};
    DevBuf<double> d_sums{ctx->stream}, d_partial{ctx->stream}, d_pnum{ctx->stream}, d_pden{ctx->stream}, d_out{ctx->stream}, d_aux{ctx->stream},
        d_out_perms{ctx->stream};
    DevBuf<int> d_pdiff{ctx->stream}, d_varies{ctx->stream};  // dense path: constant-feature flags (per warp, per feature)
    DevBuf<int64_t> d_perm{ctx->stream};
    DevBuf<int32_t> d_perm32{ctx->stream};
    DevBuf<unsigned int> d_seen{ctx->stream};
    DevBuf<uint2> d_bitmap{ctx->stream};  // global-memory bitmap scratch (large n)
    DevBuf<int> d_flags{ctx->stream};     // [0] error flags, [1] feature queue counter
    bool aux_valid = false;  // d_aux holds the invariants of the loaded X, written by an unpermuted run of mode aux_mode
    int aux_mode = 0;
    int tiles_per_launch = 8;  // dense path: 256 features per launch
    bool ran = false;
};

static int xsize(int dt) { return dt == 0 ? 4 : 8; }

static const char* ac_err_text(int f) {
    if (f & AC_ERR_INDEX) return "index out of range";
    if (f & AC_ERR_DUP) return "an observation is stored twice for one feature (sum duplicates first)";
    if (f & AC_ERR_PERM) return "row_perm is not a permutation";
    return "invalid input";
}

// bitmap placement: shared memory when 8 bytes per 32 observations fit, else one global scratch slice per CTA
struct AcGeom {
    int nwords = 0;
    size_t smem = 0;
    int ctas = 0;
    bool global = false;
};

static int ac_geometry(sqb_autocorr* h, const void* kernel, AcGeom* g) {
    sqb_ctx* c = h->ctx;
    g->nwords = (int)ceil_div64(h->n, 32);
    const size_t need = (size_t)g->nwords * sizeof(uint2);
    const size_t avail = c->smem_optin > 4096 ? c->smem_optin - 4096 : 0;  // static shared memory of the kernels
    g->global = need > avail;
    g->smem = g->global ? 0 : need;
    if (!g->global && g->smem > 48 * 1024) SQB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g->smem));
    int per_sm = 0;
    SQB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, AC_T, g->smem));
    if (per_sm < 1) per_sm = 1;
    g->ctas = per_sm * c->sm_count;
    if (g->global) SQB_TRY(h->d_bitmap.alloc((size_t)g->ctas * g->nwords));
    return SQB_OK;
}

template <typename XT, int MODE, int FMT, bool PERM, int GRP>
static int ac_sparse_launch_g(sqb_autocorr* h, const AcSparseParams& base) {
    sqb_ctx* c = h->ctx;
    const void* kernel = (const void*)ac_sparse_kernel<XT, MODE, FMT, PERM, GRP>;
    AcGeom geo;
    SQB_TRY(ac_geometry(h, kernel, &geo));
    AcSparseParams p = base;
    p.nwords = geo.nwords;
    p.s_global = geo.global ? h->d_bitmap.p : nullptr;
    int64_t ctas = geo.ctas;
    if (ctas > h->n_feat) ctas = h->n_feat;
    SQB_CUDA(cudaMemsetAsync(h->d_flags.p + 1, 0, sizeof(int), c->stream));
    SqbLaunchScope scope(c, SQB_K_AUTOCORR_MAIN);
    ac_sparse_kernel<XT, MODE, FMT, PERM, GRP><<<(unsigned)ctas, AC_T, geo.smem, c->stream>>>(p);
    SQB_POST_LAUNCH();
    return SQB_OK;
}

template <typename XT, int MODE, int FMT, bool PERM>
static int ac_sparse_launch(sqb_autocorr* h, const AcSparseParams& base) {
    // 8 row groups in flight per warp
    return ac_sparse_launch_g<XT, MODE, FMT, PERM, 8>(h, base);
}

template <typename XT, int MODE, bool PERM>
static int ac_sparse_fmt(sqb_autocorr* h, const AcSparseParams& p) {
    switch (h->w_fmt) {
        case 0: return ac_sparse_launch<XT, MODE, 0, PERM>(h, p);
        case 1: return ac_sparse_launch<XT, MODE, 1, PERM>(h, p);
        case 3: return ac_sparse_launch<XT, MODE, 3, PERM>(h, p);
        default: return ac_sparse_launch<XT, MODE, 2, PERM>(h, p);
    }
}

// one pass over all features; d_perm32 == nullptr: unpermuted (also refreshes the per-feature invariants)
static int ac_run_sparse(sqb_autocorr* h, int mode, const int32_t* d_perm32, double* d_out, int n_perm = 1) {
    AcSparseParams p;
    memset(&p, 0, sizeof(p));
    p.n = h->n;
    p.n_feat = h->n_feat;
    p.seg_start = h->d_xp.p;
    p.seg_len = h->d_len.p;
    p.seg_const = h->d_const.p;
    p.order = h->d_order.p;
    p.xi = h->d_xi.p;
    p.xv = h->d_x.p;
    p.rows = h->d_rows.p;
    p.wp = h->d_wp.p;
    p.wi = h->d_wi.p;
    p.wd = h->d_wd.p;
    p.csum = h->d_csum.p;
    p.s0 = h->s0;
    p.perm = d_perm32;
    p.n_perm = n_perm;
    p.aux = h->d_aux.p;
    p.out = d_out;
    p.counter = h->d_flags.p + 1;
    const bool f32 = h->x_dtype == 0;
    if (!d_perm32) {
        int rc;
        if (mode == 0)
            rc = f32 ? ac_sparse_fmt<float, 0, false>(h, p) : ac_sparse_fmt<double, 0, false>(h, p);
        else
            rc = f32 ? ac_sparse_fmt<float, 1, false>(h, p) : ac_sparse_fmt<double, 1, false>(h, p);
        if (rc == SQB_OK) {
            h->aux_valid = true;
            h->aux_mode = mode;
        }
        return rc;
    }
    if (mode == 0) return f32 ? ac_sparse_fmt<float, 0, true>(h, p) : ac_sparse_fmt<double, 0, true>(h, p);
    return f32 ? ac_sparse_fmt<float, 1, true>(h, p) : ac_sparse_fmt<double, 1, true>(h, p);
}

template <typename XT>
static int ac_run_dense(sqb_autocorr* h, int mode, const int64_t* d_perm) {
    sqb_ctx* c = h->ctx;
    const int64_t n = h->n, G = h->n_feat;
    const int64_t ntiles = ceil_div64(G, TILE);
    const int TPL = (int)(ntiles < h->tiles_per_launch ? ntiles : h->tiles_per_launch);
    // warps: contiguous observation ranges, >= 32 observations per warp
    int64_t ctas = (int64_t)c->sm_count * 4;
    int64_t nw = ctas * 8;
    int64_t obs_per_warp = ceil_div64(n, nw);
    if (obs_per_warp < 32) obs_per_warp = 32;
    nw = ceil_div64(n, obs_per_warp);
    ctas = ceil_div64(nw, 8);
    nw = ctas * 8;
    SQB_TRY(h->d_sums.alloc((size_t)TPL * TILE));
    SQB_TRY(h->d_partial.alloc((size_t)TPL * nw * TILE));
    SQB_TRY(h->d_pdiff.alloc((size_t)TPL * nw * TILE));
    SQB_TRY(h->d_varies.alloc((size_t)TPL * TILE));
    SQB_TRY(h->d_pnum.alloc((size_t)TPL * nw * TILE));
    SQB_TRY(h->d_pden.alloc((size_t)TPL * nw * TILE));
    const bool zero_copy = (h->kind == 2);
    if (!zero_copy) SQB_TRY(h->d_tile.alloc((size_t)TPL * n * TILE * sizeof(XT)));
    XT* Dbuf = reinterpret_cast<XT*>(h->d_tile.p);
    const XT* X = reinterpret_cast<const XT*>(h->d_x.p);
    for (int64_t t0 = 0; t0 < ntiles; t0 += TPL) {
        const int nt = (int)(ntiles - t0 < TPL ? ntiles - t0 : TPL);
        const int64_t g0 = t0 * TILE;
        const XT* D;
        int64_t pitch, tile_stride;
        if (zero_copy) {
            D = X + g0;
            pitch = G;
            tile_stride = TILE;
        } else {
            D = Dbuf;
            pitch = TILE;
            tile_stride = n * TILE;
            SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
            dim3 grid((unsigned)ceil_div64(n, 32), (unsigned)nt);
            ac_transpose_kernel<XT><<<grid, 256, 0, c->stream>>>(X, g0, G, n, Dbuf);
            SQB_POST_LAUNCH();
        }
        {
            SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
            dim3 grid((unsigned)ctas, (unsigned)nt);
            ac_colsum_kernel<XT><<<grid, 256, 0, c->stream>>>(D, pitch, tile_stride, n, obs_per_warp, h->d_partial.p, h->d_pdiff.p, g0, G);
            SQB_POST_LAUNCH();
        }
        {
            SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
            ac_colsum_final_kernel<<<nt, 32, 0, c->stream>>>(h->d_partial.p, h->d_pdiff.p, nw, h->d_sums.p, h->d_varies.p);
            SQB_POST_LAUNCH();
        }
        {
            SqbLaunchScope scope(c, SQB_K_AUTOCORR_MAIN);
            dim3 grid((unsigned)ctas, (unsigned)nt);
            if (mode == 0)
                ac_main_kernel<XT, 0><<<grid, 256, 0, c->stream>>>(h->d_wp.p, h->d_wi.p, h->d_wd.p, D, pitch, tile_stride, n,
                                                                   obs_per_warp, h->d_sums.p, d_perm, h->d_pnum.p,
                                                                   h->d_pden.p, g0, G);
            else
                ac_main_kernel<XT, 1><<<grid, 256, 0, c->stream>>>(h->d_wp.p, h->d_wi.p, h->d_wd.p, D, pitch, tile_stride, n,
                                                                   obs_per_warp, h->d_sums.p, d_perm, h->d_pnum.p,
                                                                   h->d_pden.p, g0, G);
            SQB_POST_LAUNCH();
        }
        {
            SqbLaunchScope scope(c, SQB_K_AUTOCORR_FINAL);
            if (mode == 0)
                ac_final_kernel<0><<<nt, 256, 0, c->stream>>>(h->d_pnum.p, h->d_pden.p, h->d_varies.p, ctas, n, h->s0, g0, G, h->d_out.p);
            else
                ac_final_kernel<1><<<nt, 256, 0, c->stream>>>(h->d_pnum.p, h->d_pden.p, h->d_varies.p, ctas, n, h->s0, g0, G, h->d_out.p);
            SQB_POST_LAUNCH();
        }
    }
    return SQB_OK;
}

// read the error flag word (synchronises the stream)
static int ac_check_flags(sqb_autocorr* h, const char* where) {
    sqb_ctx* c = h->ctx;
    int f = 0;
    SQB_CUDA(cudaMemcpyAsync(&f, h->d_flags.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    if (f != 0) {
        SQB_CUDA(cudaMemsetAsync(h->d_flags.p, 0, sizeof(int), c->stream));
        sqb_set_error("%s: %s", where, ac_err_text(f));
        return SQB_ERR_INVALID;
    }
    return SQB_OK;
}

// raw segments by feature (segment g = [d_beg[g], d_end[g]) of idx / val on the device, any order inside a segment) ->
// padded, ordered layout; nnz >= the entries of all segments
template <typename II, typename VT, typename XT>
static int ac_build_segments(sqb_autocorr* h, const int64_t* d_beg, const int64_t* d_end, const unsigned int* d_cnt, int64_t* d_pad,
                             const II* d_idx, const VT* d_val, int64_t nnz, int64_t n_feat) {
    sqb_ctx* c = h->ctx;
    const int64_t cap = nnz + 4 * n_feat + 4;
    SQB_TRY(h->d_xi.alloc((size_t)cap));
    SQB_TRY(h->d_x.alloc((size_t)cap * sizeof(XT)));
    SQB_TRY(h->d_len.alloc((size_t)n_feat));
    SQB_TRY(h->d_const.alloc((size_t)n_feat));
    SQB_TRY(h->d_order.alloc((size_t)n_feat));
    SQB_TRY(h->d_aux.alloc((size_t)5 * n_feat));
    SQB_TRY(h->d_out.alloc((size_t)n_feat));
    const void* kernel = (const void*)ac_rank_sort_kernel<II, VT, XT>;
    AcGeom geo;
    SQB_TRY(ac_geometry(h, kernel, &geo));
    int64_t ctas = geo.ctas < n_feat ? geo.ctas : n_feat;
    {
        SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
        ac_rank_sort_kernel<II, VT, XT><<<(unsigned)ctas, AC_T, geo.smem, c->stream>>>(
            d_beg, d_end, d_idx, d_val, d_pad, h->d_xi.p, reinterpret_cast<XT*>(h->d_x.p), h->d_len.p, h->d_const.p, h->n, n_feat, geo.nwords,
            geo.global ? h->d_bitmap.p : nullptr, h->d_flags.p);
        SQB_POST_LAUNCH();
    }
    // features by decreasing length: the queue hands out the long ones first (LPT), the tail of the grid stays short
    {
        DevBuf<unsigned int> keys_out(c->stream);
        DevBuf<int32_t> iota(c->stream);
        DevBuf<uint8_t> tmp(c->stream);
        SQB_TRY(keys_out.alloc(n_feat));
        SQB_TRY(iota.alloc(n_feat));
        std::vector<int32_t> hi((size_t)n_feat);
        for (int64_t g = 0; g < n_feat; ++g) hi[g] = (int32_t)g;
        SQB_CUDA(cudaMemcpyAsync(iota.p, hi.data(), n_feat * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        size_t tmp_bytes = 0;
        SQB_CUDA(cub::DeviceRadixSort::SortPairsDescending(nullptr, tmp_bytes, d_cnt, keys_out.p, iota.p, h->d_order.p, (int)n_feat, 0, 32,
                                                           c->stream));
        SQB_TRY(tmp.alloc(tmp_bytes > 0 ? tmp_bytes : 1));
        SQB_CUDA(cub::DeviceRadixSort::SortPairsDescending(tmp.p, tmp_bytes, d_cnt, keys_out.p, iota.p, h->d_order.p, (int)n_feat, 0, 32,
                                                           c->stream));
        SQB_CUDA(cudaStreamSynchronize(c->stream));  // hi must outlive the copy
        c->launches += 2;
    }
    // the padded starts now belong to the handle
    SQB_TRY(h->d_xp.alloc((size_t)n_feat + 1));
    SQB_CUDA(cudaMemcpyAsync(h->d_xp.p, d_pad, (n_feat + 1) * sizeof(int64_t), cudaMemcpyDeviceToDevice, c->stream));
    return SQB_OK;
}

// ---- loading X: CSR relayout (host and device-resident), device-resident dense X ---------------------------------------
// col_map[f] in [0, n_out) or -1 for every input feature f; every output feature must come from exactly one input feature.
// inv[k] = the input feature of output feature k.
static int ac_invert_col_map(const int32_t* col_map, int64_t n_cols, int64_t n_out, std::vector<int32_t>& inv, const char* where) {
    SQB_CHECK(n_cols >= 1 && n_cols < 2147483647LL && n_out >= 1 && n_out <= n_cols, SQB_ERR_INVALID,
              "%s: n_out=%lld, n_cols=%lld out of range", where, (long long)n_out, (long long)n_cols);
    inv.assign((size_t)n_out, -1);
    for (int64_t f = 0; f < n_cols; ++f) {
        const int32_t k = col_map[f];
        if (k == -1) continue;
        SQB_CHECK(k >= 0 && k < n_out && inv[k] < 0, SQB_ERR_INVALID, "%s: col_map[%lld] = %d is not -1 or an unused index in [0, %lld)",
                  where, (long long)f, k, (long long)n_out);
        inv[k] = (int32_t)f;
    }
    for (int64_t k = 0; k < n_out; ++k)
        SQB_CHECK(inv[k] >= 0, SQB_ERR_INVALID, "%s: output feature %lld is not in col_map", where, (long long)k);
    return SQB_OK;
}

// A CSR of X in device memory (indptr IP, indices II, values VT: the caller's, read in place, or the host path's upload) -> the
// padded layout by feature (values XT).  indptr is validated (one synchronisation) before any kernel follows it, so no read
// leaves [0, nnz).  Layout 0 (rows = features): output feature k is input row inv[k].  Layout 1 (rows = observations): input
// column j goes to output feature col_map[j] (n_cols entries, -1: skipped), or, with col_map null, to j - col_lo, any column
// outside [col_lo, col_lo + n_out) being an error.  Synchronises on success.
template <typename IP, typename II, typename VT, typename XT>
static int ac_relayout_csr(sqb_autocorr* h, const IP* xp, const II* xi, const VT* xv, int layout, int64_t n_cols, const int32_t* col_map,
                           int32_t col_lo, const std::vector<int32_t>& inv, int64_t n_out, const char* where) {
    sqb_ctx* c = h->ctx;
    const int64_t n = h->n;
    const int64_t rows = layout == 0 ? n_cols : n;
    DevBuf<int32_t> map(c->stream), t_idx(c->stream);
    DevBuf<XT> t_val(c->stream);
    DevBuf<int64_t> beg(c->stream), end(c->stream), t_ptr(c->stream), pad(c->stream);
    DevBuf<unsigned int> cnt(c->stream);
    DevBuf<unsigned long long> cursor(c->stream);
    SQB_CUDA(cudaMemsetAsync(h->d_flags.p, 0, 2 * sizeof(int), c->stream));
    IP last = 0;
    SQB_CUDA(cudaMemcpyAsync(&last, xp + rows, sizeof(IP), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    const int64_t nnz = (int64_t)last;
    SQB_TRY(sqb_check_indptr(c, SQB_K_AUTOCORR_PREP, xp, rows, nnz, nullptr, where));
    SQB_CHECK(nnz == 0 || (xi && xv), SQB_ERR_INVALID, "%s: null X arrays", where);
    SQB_TRY(cnt.alloc(n_out + 1));
    SQB_TRY(pad.alloc(n_out + 1));
    SQB_TRY(t_ptr.alloc(n_out + 1));
    if (layout == 0) {
        SQB_TRY(map.alloc(n_out));
        SQB_TRY(beg.alloc(n_out));
        SQB_TRY(end.alloc(n_out));
        SQB_CUDA(cudaMemcpyAsync(map.p, inv.data(), n_out * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
        ac_select_segs_kernel<IP><<<c->sm_count * 2, 256, 0, c->stream>>>(xp, map.p, n_out, beg.p, end.p, cnt.p, n, h->d_flags.p);
        SQB_POST_LAUNCH();
    } else {
        if (col_map) {
            SQB_TRY(map.alloc(n_cols));
            SQB_CUDA(cudaMemcpyAsync(map.p, col_map, n_cols * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        }
        SQB_TRY(cursor.alloc(n_out + 1));
        SQB_CUDA(cudaMemsetAsync(cnt.p, 0, (n_out + 1) * sizeof(unsigned int), c->stream));
        if (nnz > 0) {
            SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
            const size_t hist_bytes = (size_t)n_out * sizeof(unsigned int);
            const int hist_smem = hist_bytes <= 160 * 1024 ? 1 : 0;
            if (hist_smem && hist_bytes > 48 * 1024)
                SQB_CUDA(cudaFuncSetAttribute(ac_colcount_kernel<II>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hist_bytes));
            ac_colcount_kernel<II><<<c->sm_count * (hist_smem ? 1 : 8), 1024, hist_smem ? hist_bytes : 0, c->stream>>>(
                xi, nnz, n_out, col_lo, map.p, n_cols, hist_smem, cnt.p, h->d_flags.p);
            SQB_POST_LAUNCH();
        }
    }
    {
        SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
        ac_scan_counts_kernel<<<1, 1024, 0, c->stream>>>(cnt.p, n_out, t_ptr.p, pad.p, layout == 0 ? nullptr : cursor.p);
        SQB_POST_LAUNCH();
    }
    // entries of the selected features: the relaid-out copy is sized by them, not by the whole matrix
    int64_t sel = 0;
    SQB_CUDA(cudaMemcpyAsync(&sel, t_ptr.p + n_out, sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    if (layout == 0) {
        SQB_TRY((ac_build_segments<II, VT, XT>(h, beg.p, end.p, cnt.p, pad.p, xi, xv, sel, n_out)));
    } else {
        SQB_TRY(t_idx.alloc(sel));
        SQB_TRY(t_val.alloc(sel));
        if (sel > 0) {
            SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
            ac_coltranspose_kernel<IP, II, VT, XT><<<c->sm_count * 8, 256, 0, c->stream>>>(xp, xi, xv, n, n_out, col_lo, map.p, n_cols,
                                                                                          cursor.p, t_idx.p, t_val.p);
            SQB_POST_LAUNCH();
        }
        SQB_TRY((ac_build_segments<int32_t, XT, XT>(h, t_ptr.p, t_ptr.p + 1, cnt.p, pad.p, t_idx.p, t_val.p, sel, n_out)));
    }
    return ac_check_flags(h, where);  // synchronises: the inputs are no longer read
}

// Host CSR of X (int64 indptr, int32 indices, values XT): uploaded, then re-laid out as device input is.  sub_start / sub_cnt
// (layout 1 only): upload only the piece [sub_start[r], +sub_cnt[r]) of every observation's row (the columns col_lo .. col_lo +
// n_feat of rows with ascending indices); xp then is the indptr of the pieces.
template <typename XT>
static int ac_load_csr_host(sqb_autocorr* h, const int64_t* xp, const int32_t* xi, const void* xv, int layout, int64_t n_feat,
                            int32_t col_lo = 0, const int64_t* sub_start = nullptr, const int64_t* sub_cnt = nullptr) {
    sqb_ctx* c = h->ctx;
    const int64_t rows = layout == 0 ? n_feat : h->n, nnz = xp[rows];
    DevBuf<int64_t> d_ptr(c->stream);
    DevBuf<int32_t> d_idx(c->stream);
    DevBuf<XT> d_val(c->stream);
    SQB_TRY(d_ptr.alloc(rows + 1));
    SQB_TRY(d_idx.alloc(nnz));
    SQB_TRY(d_val.alloc(nnz));
    SQB_CUDA(cudaMemcpyAsync(d_ptr.p, xp, (rows + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
    if (nnz > 0) {  // a failed upload is reported as SQB_ERR_CUDA, whatever the copy returned
        const bool failed = sub_start ? sqb_h2d_gather(c, d_idx.p, xi, sizeof(int32_t), sub_start, sub_cnt, xp, rows) ||
                                            sqb_h2d_gather(c, d_val.p, xv, sizeof(XT), sub_start, sub_cnt, xp, rows)
                                      : sqb_h2d(c, d_idx.p, xi, nnz * sizeof(int32_t)) || sqb_h2d(c, d_val.p, xv, (size_t)nnz * sizeof(XT));
        if (failed) return SQB_ERR_CUDA;
    }
    std::vector<int32_t> inv(layout == 0 ? n_feat : 0);  // layout 0: every row is a feature, in order
    for (int64_t k = 0; k < (int64_t)inv.size(); ++k) inv[k] = (int32_t)k;
    return ac_relayout_csr<int64_t, int32_t, XT, XT>(h, d_ptr.p, d_idx.p, d_val.p, layout, n_feat, nullptr, col_lo, inv, n_feat,
                                                     "sqb_autocorr_load_csr");
}

// The value type of the loaded X: float32 stays float32, everything else becomes float64 (the host path's dtype rule).
template <typename VT>
using AcX = std::conditional_t<std::is_same<VT, float>::value, float, double>;

template <typename VT, typename XT>
static int ac_gather_dense(sqb_autocorr* h, const void* x, int64_t n_out, int64_t s_obs, int64_t s_feat, const int32_t* d_inv,
                           int obs_major) {
    sqb_ctx* c = h->ctx;
    SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
    ac_gather_dense_kernel<VT, XT><<<c->sm_count * 8, 256, 0, c->stream>>>((const VT*)x, h->n, n_out, s_obs, s_feat, d_inv, obs_major,
                                                                          reinterpret_cast<XT*>(h->d_x.p));
    SQB_POST_LAUNCH();
    return SQB_OK;
}

// =====================================================================================================
// W build: one device pass serves the host upload (sqb_autocorr_create) and a caller's device CSR (sqb_autocorr_create_device).
// Every quantity equals, bit for bit, what the host computes for the same W (tests/autocorr_w_ref.py is the specification):
//   wd = (double)w;  S0 = the sequential float64 sum of wd in entry order;  csum[j] = the sequential float64 sum of column j in
//   row order (a stable radix sort of the entries by column);  the packed-row format of the per-feature kernel.
// S0 is one dependent chain.  Every weight is a multiple of g = the smallest lowest set bit among the weights; when
// sum |w| < 2^53 g every partial sum is a representable multiple of g, so the chain is exact and equals the integer sum of w / g,
// which is summed in parallel (a row-normalised float32 graph always qualifies).  Otherwise one thread walks the chain.
// Device input also gets sklearn's l1 row normalisation and the moments s0, s1, s2 of _g_moments in W's dtype, in scipy's
// operation order: numpy's pairwise summation (np.sum), np.add.reduceat per row (the first value plus the pairwise sum of the
// rest), a sequential sum per column, and the zero-free values of W^T + W (a symmetric matrix: its canonical CSC order is the
// row-major order of a row merge of W with its transpose).
// =====================================================================================================
#define AC_PW_BLOCK 128  // numpy's PW_BLOCKSIZE

static inline unsigned ac_grid(const sqb_ctx* c, int64_t items, int threads = 256) { return sqb_grid_rows(c, items, threads); }

// caller's column indices -> int32; an index outside [0, n) raises AC_ERR_INDEX, a row whose indices do not strictly increase
// AC_W_NONCANON.  wp has been validated.
template <typename II>
__global__ void ac_w_indices_kernel(const int32_t* __restrict__ wp, const II* __restrict__ in, int64_t n, int32_t* __restrict__ out,
                                    int* __restrict__ err) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        int64_t prev = -1;
        int f = 0;
        for (int32_t e = wp[r]; e < wp[r + 1]; ++e) {
            const int64_t j = (int64_t)in[e];
            if (j < 0 || j >= n) {
                f |= AC_ERR_INDEX;
                out[e] = 0;
                continue;
            }
            if (j <= prev) f |= AC_W_NONCANON;
            prev = j;
            out[e] = (int32_t)j;
        }
        if (f) atomicOr(err, f);
    }
}

// sklearn's normalize(norm="l1", axis=1) of a float32 / float64 CSR (normalise = 0: a plain copy): per row a sequential float64
// sum of |w| in entry order; a row whose sum is 0 is kept; every value becomes (T)((double)w / sum).  normalize rejects NaN and
// infinite values: with normalise, one raises AC_W_NONFINITE.
template <typename T>
__global__ void ac_w_l1_kernel(const int32_t* __restrict__ wp, const T* __restrict__ in, int64_t n, int normalise, T* __restrict__ out,
                               int* __restrict__ err) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const int32_t b = wp[r], e1 = wp[r + 1];
        double s = 0.0;
        bool finite = true;
        if (normalise)
            for (int32_t e = b; e < e1; ++e) {
                finite &= isfinite((double)in[e]);
                s = __dadd_rn(s, fabs((double)in[e]));
            }
        if (!finite) atomicOr(err, AC_W_NONFINITE);
        for (int32_t e = b; e < e1; ++e) out[e] = normalise && s != 0.0 ? (T)__ddiv_rn((double)in[e], s) : in[e];
    }
}

// exponent of the lowest set bit of a finite non-zero double
__device__ __forceinline__ int ac_lowbit_exp(double d) {
    int e;
    const double m = frexp(d, &e);  // d = m 2^e, 0.5 <= |m| < 1
    const unsigned long long sig = (unsigned long long)fabs(ldexp(m, 53));
    return e - 53 + __ffsll((long long)sig) - 1;
}

// wd = (double)w and the statistics of W: st[0] longest row, st[1] some float32 row holds two different weights, st[2] the
// smallest lowest-bit exponent, st[3] a non-finite weight; part[block] = sum |w| rounded upward (an upper bound)
template <typename T>
__global__ void __launch_bounds__(256) ac_w_stats_kernel(const int32_t* __restrict__ wp, const T* __restrict__ w, int64_t n,
                                                         double* __restrict__ wd, int* __restrict__ st, double* __restrict__ part) {
    __shared__ double s_sum[256];
    double acc = 0.0;
    int maxdeg = 0, nonuni = 0, lb = INT_MAX, nonfin = 0;
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const int32_t b = wp[r], e1 = wp[r + 1];
        maxdeg = max(maxdeg, (int)(e1 - b));
        for (int32_t e = b; e < e1; ++e) {
            const T v = w[e];
            const double d = (double)v;
            wd[e] = d;
            if (sizeof(T) == 4 && e > b && __float_as_uint((float)v) != __float_as_uint((float)w[b])) nonuni = 1;
            if (!isfinite(d)) {
                nonfin = 1;
            } else if (d != 0.0) {
                lb = min(lb, ac_lowbit_exp(d));
                acc = __dadd_ru(acc, fabs(d));
            }
        }
    }
    if (maxdeg) atomicMax(&st[0], maxdeg);
    if (nonuni) atomicOr(&st[1], 1);
    if (lb != INT_MAX) atomicMin(&st[2], lb);
    if (nonfin) atomicOr(&st[3], 1);
    s_sum[threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int k = 0; k < blockDim.x; ++k) t = __dadd_ru(t, s_sum[k]);
        part[blockIdx.x] = t;
    }
}

__global__ void ac_w_bound_kernel(const double* __restrict__ part, int np, double* __restrict__ out) {
    double t = 0.0;
    for (int k = 0; k < np; ++k) t = __dadd_ru(t, part[k]);
    *out = t;
}

// S0 as the integer sum of w / 2^g (every term an integer below 2^53 in magnitude, and so is every partial sum)
__global__ void __launch_bounds__(256) ac_w_s0_int_kernel(const double* __restrict__ wd, int64_t nnz, int g, unsigned long long* __restrict__ acc) {
    long long loc = 0;
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x)
        loc += (long long)ldexp(wd[e], -g);
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) loc += __shfl_xor_sync(0xffffffffu, loc, d);
    if ((threadIdx.x & 31) == 0 && loc != 0) atomicAdd(acc, (unsigned long long)loc);
}

// S0 as the host computes it: one ordered chain.  One lane adds, from shared memory, while warps 1.. stage the next tile from
// global memory: the loop runs at the latency of the dependent additions, not of global loads.
#define AC_SEQ_TILE 2048
__global__ void __launch_bounds__(256) ac_w_s0_seq_kernel(const double* __restrict__ wd, int64_t nnz, double* __restrict__ out) {
    __shared__ double buf[2][AC_SEQ_TILE];
    const int64_t ntiles = (nnz + AC_SEQ_TILE - 1) / AC_SEQ_TILE;
    for (int64_t i = threadIdx.x; i < AC_SEQ_TILE && i < nnz; i += blockDim.x) buf[0][i] = wd[i];
    __syncthreads();
    double s = 0.0;
    for (int64_t t = 0; t < ntiles; ++t) {
        const int64_t base = t * AC_SEQ_TILE;
        if (threadIdx.x == 0) {
            const double* __restrict__ b = buf[t & 1];
            const int len = (int)(nnz - base < AC_SEQ_TILE ? nnz - base : AC_SEQ_TILE);
            int k = 0;
            for (; k + 8 <= len; k += 8) {
                double v[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) v[j] = b[k + j];
#pragma unroll
                for (int j = 0; j < 8; ++j) s = __dadd_rn(s, v[j]);
            }
            for (; k < len; ++k) s = __dadd_rn(s, b[k]);
        } else if (threadIdx.x >= 32 && t + 1 < ntiles) {
            const int64_t nb = base + AC_SEQ_TILE;
            const int64_t len = nnz - nb < AC_SEQ_TILE ? nnz - nb : AC_SEQ_TILE;
            for (int64_t i = threadIdx.x - 32; i < len; i += blockDim.x - 32) buf[(t + 1) & 1][i] = wd[nb + i];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = s;
}

// ---- numpy's pairwise summation ---------------------------------------------------------------------------
// A block of at most 128 values: a plain loop below 8, else eight strided accumulators combined as
// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) and the tail added in order.  (numpy starts the short loop from -0.0 and np.sum adds the
// result to +0.0: the sign of a zero never reaches a non-zero sum, and the caller adds +0.0 last.)
template <typename T>
__device__ T ac_pw_leaf(const T* __restrict__ a, int64_t n) {
    if (n < 8) {
        T r = (T)0;
        for (int64_t i = 0; i < n; ++i) r = r + a[i];
        return r;
    }
    T r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    int64_t i = 8;
    for (; i < n - (n % 8); i += 8)
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = r[j] + a[i + j];
    T res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res = res + a[i];
    return res;
}

// a whole pairwise tree on one thread (rows of W)
template <typename T>
__device__ T ac_pw_seq(const T* __restrict__ a, int64_t n) {
    if (n <= AC_PW_BLOCK) return ac_pw_leaf(a, n);
    int64_t h = n / 2;
    h -= h % 8;
    return ac_pw_seq(a, h) + ac_pw_seq(a + h, n - h);
}

// node p of level L of the tree over n values (left = 0 bit, most significant first): false when the path ends in a leaf above L
// and p is not the first index under it
__device__ __forceinline__ bool ac_pw_node(int64_t n, int L, int64_t p, int64_t* off, int64_t* len) {
    int64_t o = 0;
    for (int l = 0; l < L; ++l) {
        if (n <= AC_PW_BLOCK) {
            *off = o, *len = n;
            return (p & ((1LL << (L - l)) - 1)) == 0;
        }
        int64_t h = n / 2;
        h -= h % 8;
        if ((p >> (L - 1 - l)) & 1) {
            o += h;
            n -= h;
        } else {
            n = h;
        }
    }
    *off = o, *len = n;
    return true;
}

template <typename T>
__global__ void ac_pw_leaves_kernel(const T* __restrict__ a, int64_t n, int depth, T* __restrict__ res) {
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < (1LL << depth); t += (int64_t)gridDim.x * blockDim.x) {
        int64_t off, len;
        if (ac_pw_node(n, depth, t, &off, &len)) res[t] = ac_pw_leaf(a + off, len);
    }
}

// level L: every inner node = its left subtree's sum + its right subtree's (kept at the first index under each node)
template <typename T>
__global__ void ac_pw_level_kernel(int64_t n, int depth, int L, T* __restrict__ res) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < (1LL << L); p += (int64_t)gridDim.x * blockDim.x) {
        int64_t off, len;
        if (ac_pw_node(n, L, p, &off, &len) && len > AC_PW_BLOCK)
            res[p << (depth - L)] = res[(2 * p) << (depth - L - 1)] + res[(2 * p + 1) << (depth - L - 1)];
    }
}

static int ac_pw_depth(int64_t n) {  // the right half is never the shorter one: its path is the deepest
    int d = 0;
    while (n > AC_PW_BLOCK) {
        int64_t h = n / 2;
        h -= h % 8;
        n -= h;
        ++d;
    }
    return d;
}

// *out (device) = pairwise sum of a[0, n) in T, leaves in parallel, then one launch per level of the tree
template <typename T>
static int ac_pairwise(sqb_ctx* c, const T* a, int64_t n, T* out) {
    if (n == 0) {
        SQB_CUDA(cudaMemsetAsync(out, 0, sizeof(T), c->stream));
        return SQB_OK;
    }
    const int depth = ac_pw_depth(n);
    DevBuf<T> res(c->stream);
    SQB_TRY(res.alloc((size_t)1 << depth));
    {
        SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
        ac_pw_leaves_kernel<T><<<ac_grid(c, (int64_t)1 << depth), 256, 0, c->stream>>>(a, n, depth, res.p);
        SQB_POST_LAUNCH();
    }
    for (int L = depth - 1; L >= 0; --L) {
        SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
        ac_pw_level_kernel<T><<<ac_grid(c, (int64_t)1 << L), 256, 0, c->stream>>>(n, depth, L, res.p);
        SQB_POST_LAUNCH();
    }
    SQB_CUDA(cudaMemcpyAsync(out, res.p, sizeof(T), cudaMemcpyDeviceToDevice, c->stream));
    return SQB_OK;
}

// (W.sum(1) + W.sum(0).T)^2 per row: the row sum is np.add.reduceat's (first value + the pairwise sum of the rest; 0 if empty)
template <typename T>
__global__ void ac_w_rowcol_sq_kernel(const int32_t* __restrict__ wp, const T* __restrict__ w, const T* __restrict__ colT, int64_t n,
                                      int32_t* __restrict__ rowof, T* __restrict__ out) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const int32_t b = wp[r], e1 = wp[r + 1];
        T rs = (T)0;
        if (e1 > b) rs = e1 - b > 1 ? w[b] + ac_pw_seq(w + b + 1, (int64_t)(e1 - b - 1)) : w[b];
        const T v = rs + colT[r];
        out[r] = v * v;
        for (int32_t e = b; e < e1; ++e) rowof[e] = (int32_t)r;
    }
}

// row i of W^T + W: merge of row i of W (ascending columns) with column i of W (ascending rows, the sorted entries); the squares
// of the non-zero sums that are themselves non-zero (scipy drops zeros from both the sum and the product).  cnt: count pass
// (out null) or write pass at out + off[i].
template <typename T>
__global__ void ac_w_sym_kernel(const int32_t* __restrict__ wp, const int32_t* __restrict__ wi, const T* __restrict__ w,
                                const int32_t* __restrict__ cbeg, const int32_t* __restrict__ cend, const int32_t* __restrict__ perm,
                                const int32_t* __restrict__ rowof, int64_t n, unsigned long long* __restrict__ cnt,
                                const unsigned long long* __restrict__ off, T* __restrict__ out) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int32_t a = wp[i];
        const int32_t ae = wp[i + 1];
        int32_t b = cbeg[i];
        const int32_t be = cend[i];
        unsigned long long k = 0, o = out ? off[i] : 0;
        while (a < ae || b < be) {
            const int32_t ja = a < ae ? wi[a] : INT_MAX;
            const int32_t jb = b < be ? rowof[perm[b]] : INT_MAX;
            T t;
            if (ja == jb) {
                t = w[a++] + w[perm[b++]];
            } else if (ja < jb) {
                t = w[a++];
            } else {
                t = w[perm[b++]];
            }
            if (t == (T)0) continue;
            const T sq = t * t;
            if (sq == (T)0) continue;
            if (out) out[o + k] = sq;
            ++k;
        }
        if (!out) cnt[i] = k;
    }
}

// The rest of a handle's W once h->d_wp / h->d_wi hold a validated CSR (n, nnz set) and w its values (float or double, already
// normalised): d_wd, S0, d_csum, the packed rows; with moments (3 doubles, host) s0, s1, s2 of _g_moments in T.  Synchronises.
template <typename T>
static int ac_build_w(sqb_autocorr* h, const T* w, double* moments) {
    sqb_ctx* c = h->ctx;
    const int64_t n = h->n, nnz = h->nnz;
    const unsigned gs = (unsigned)c->sm_count * 4;
    SQB_TRY(h->d_wd.alloc(nnz > 0 ? nnz : 1));
    SQB_TRY(h->d_csum.alloc(n));
    DevBuf<int> st(c->stream);
    DevBuf<double> part(c->stream), bound(c->stream);
    SQB_TRY(st.alloc(4));
    SQB_TRY(part.alloc(gs));
    SQB_TRY(bound.alloc(1));
    const int st0[4] = {0, 0, INT_MAX, 0};
    SQB_CUDA(cudaMemcpyAsync(st.p, st0, sizeof(st0), cudaMemcpyHostToDevice, c->stream));
    {
        SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
        ac_w_stats_kernel<T><<<gs, 256, 0, c->stream>>>(h->d_wp.p, w, n, h->d_wd.p, st.p, part.p);
        SQB_POST_LAUNCH();
    }
    {
        SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
        ac_w_bound_kernel<<<1, 1, 0, c->stream>>>(part.p, (int)gs, bound.p);
        SQB_POST_LAUNCH();
    }
    int sth[4];
    double bnd = 0.0;
    SQB_CUDA(cudaMemcpyAsync(sth, st.p, sizeof(sth), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaMemcpyAsync(&bnd, bound.p, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    const int maxdeg = sth[0], g = sth[2];
    const bool exact = !sth[3] && (g == INT_MAX || bnd < ldexp(1.0, 53 + g));
    h->s0_branch = exact ? 0 : 1;
    DevBuf<unsigned long long> acc(c->stream);
    DevBuf<double> d_s0(c->stream);
    if (exact) {
        SQB_TRY(acc.alloc(1));
        SQB_CUDA(cudaMemsetAsync(acc.p, 0, sizeof(unsigned long long), c->stream));
        if (g != INT_MAX) {
            SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
            ac_w_s0_int_kernel<<<ac_grid(c, nnz), 256, 0, c->stream>>>(h->d_wd.p, nnz, g, acc.p);
            SQB_POST_LAUNCH();
        }
    } else {
        SQB_TRY(d_s0.alloc(1));
        SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
        ac_w_s0_seq_kernel<<<1, 256, 0, c->stream>>>(h->d_wd.p, nnz, d_s0.p);
        SQB_POST_LAUNCH();
    }
    // stable transpose: the entries sorted by column keep their row order
    DevBuf<int32_t> perm(c->stream), cbeg(c->stream), cend(c->stream), rowof(c->stream);
    DevBuf<T> colT(c->stream);
    DevBuf<uint8_t> tmp(c->stream);
    if (moments) SQB_TRY(colT.alloc(n));
    SQB_TRY(sqb_col_order(c, SQB_K_AUTOCORR_PREP, h->d_wi.p, nnz, n, perm, cbeg, cend));
    {
        SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
        sqb_col_sums_kernel<T><<<ac_grid(c, n), 256, 0, c->stream>>>(cbeg.p, cend.p, perm.p, h->d_wd.p, w, n, h->d_csum.p,
                                                                      moments ? colT.p : nullptr);
        SQB_POST_LAUNCH();
    }
    // rows of at most 7 entries that all carry the same float32 weight (a row-normalised binary graph) take the compact format;
    // packed rows hold float32 weights: only for float32 W (lossless); float64 W walks the CSR
    const bool f32 = sizeof(T) == 4;
    const bool uniform7 = f32 && maxdeg <= 7 && nnz > 0 && !sth[1];
    h->w_fmt = uniform7 ? 3 : (f32 && maxdeg <= 8) ? 0 : (f32 && maxdeg <= 16) ? 1 : 2;
    if (h->w_fmt != 2) {
        const int lpr = h->w_fmt == 3 ? 4 : h->w_fmt == 0 ? 8 : 16;  // uint2 units per row
        SQB_TRY(h->d_rows.alloc((size_t)n * lpr));
        SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
        if (h->w_fmt == 3)
            ac_pack_rows32_kernel<<<c->sm_count * 4, 256, 0, c->stream>>>(h->d_wp.p, h->d_wi.p, h->d_wd.p, n, reinterpret_cast<uint32_t*>(h->d_rows.p));
        else if (h->w_fmt == 0)
            ac_pack_rows_kernel<8><<<c->sm_count * 4, 256, 0, c->stream>>>(h->d_wp.p, h->d_wi.p, h->d_wd.p, n, h->d_rows.p);
        else
            ac_pack_rows_kernel<16><<<c->sm_count * 4, 256, 0, c->stream>>>(h->d_wp.p, h->d_wi.p, h->d_wd.p, n, h->d_rows.p);
        SQB_POST_LAUNCH();
    }
    DevBuf<T> mom(c->stream), sq_rc(c->stream), sq_sym(c->stream);
    DevBuf<unsigned long long> scnt(c->stream), soff(c->stream);
    if (moments) {
        SQB_TRY(mom.alloc(3));
        SQB_TRY(sq_rc.alloc(n));
        SQB_TRY(rowof.alloc(nnz > 0 ? nnz : 1));
        SQB_TRY(scnt.alloc(n + 1));
        SQB_TRY(soff.alloc(n + 1));
        SQB_TRY(ac_pairwise<T>(c, w, nnz, mom.p));  // s0 = W.sum() = np.sum(W.data)
        {
            SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
            ac_w_rowcol_sq_kernel<T><<<ac_grid(c, n), 256, 0, c->stream>>>(h->d_wp.p, w, colT.p, n, rowof.p, sq_rc.p);
            SQB_POST_LAUNCH();
        }
        SQB_TRY(ac_pairwise<T>(c, sq_rc.p, n, mom.p + 2));  // s2
        SQB_CUDA(cudaMemsetAsync(scnt.p + n, 0, sizeof(unsigned long long), c->stream));
        {
            SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
            ac_w_sym_kernel<T><<<ac_grid(c, n), 256, 0, c->stream>>>(h->d_wp.p, h->d_wi.p, w, cbeg.p, cend.p, perm.p, rowof.p, n, scnt.p,
                                                                     nullptr, nullptr);
            SQB_POST_LAUNCH();
        }
        size_t bytes = 0;
        SQB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, scnt.p, soff.p, (int)(n + 1), c->stream));
        SQB_TRY(tmp.alloc(bytes > 0 ? bytes : 1));
        SQB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, scnt.p, soff.p, (int)(n + 1), c->stream));
        c->launches += 1;
        unsigned long long m = 0;
        SQB_CUDA(cudaMemcpyAsync(&m, soff.p + n, sizeof(m), cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaStreamSynchronize(c->stream));
        SQB_TRY(sq_sym.alloc(m > 0 ? m : 1));
        {
            SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
            ac_w_sym_kernel<T><<<ac_grid(c, n), 256, 0, c->stream>>>(h->d_wp.p, h->d_wi.p, w, cbeg.p, cend.p, perm.p, rowof.p, n, nullptr,
                                                                     soff.p, sq_sym.p);
            SQB_POST_LAUNCH();
        }
        SQB_TRY(ac_pairwise<T>(c, sq_sym.p, (int64_t)m, mom.p + 1));  // s1 = (W^T + W).multiply(W^T + W).sum() / 2
    }
    unsigned long long s0_int = 0;
    T mh[3] = {(T)0, (T)0, (T)0};
    if (exact) SQB_CUDA(cudaMemcpyAsync(&s0_int, acc.p, sizeof(s0_int), cudaMemcpyDeviceToHost, c->stream));
    else SQB_CUDA(cudaMemcpyAsync(&h->s0, d_s0.p, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    if (moments) SQB_CUDA(cudaMemcpyAsync(mh, mom.p, sizeof(mh), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    if (exact) h->s0 = g == INT_MAX ? 0.0 : ldexp((double)(long long)s0_int, g);
    if (moments) {  // np.sum adds the pairwise sum to +0.0; s1 is halved in T
        moments[0] = (double)((T)0 + mh[0]);
        moments[1] = (double)(((T)0 + mh[1]) / (T)2);
        moments[2] = (double)((T)0 + mh[2]);
    }
    return SQB_OK;
}

// W's values from the caller's device array into the handle's build: normalised (or copied) into a buffer of W's own dtype
template <typename T>
static int ac_create_from_device(sqb_autocorr* h, const void* data, int transformation, double* moments) {
    sqb_ctx* c = h->ctx;
    DevBuf<T> w(c->stream);
    SQB_TRY(w.alloc(h->nnz > 0 ? h->nnz : 1));
    {
        SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
        ac_w_l1_kernel<T><<<ac_grid(c, h->n), 256, 0, c->stream>>>(h->d_wp.p, (const T*)data, h->n, transformation, w.p, h->d_flags.p);
        SQB_POST_LAUNCH();
    }
    if (transformation) {  // sklearn's normalize raises on NaN / infinite weights: the host path reports it
        int f = 0;
        SQB_CUDA(cudaMemcpyAsync(&f, h->d_flags.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaStreamSynchronize(c->stream));
        SQB_CHECK(!(f & AC_W_NONFINITE), SQB_ERR_LAYOUT, "sqb_autocorr_create_device: W holds NaN or infinite weights to normalise");
    }
    return ac_build_w<T>(h, w.p, moments);
}

extern "C" {

int sqb_autocorr_create(sqb_ctx* ctx, int64_t n, int64_t nnz, const int32_t* w_indptr, const int32_t* w_indices,
                        const void* w_data, int w_dtype, sqb_autocorr** out) {
    SQB_CHECK(ctx && out && w_indptr, SQB_ERR_INVALID, "sqb_autocorr_create: null argument");
    SQB_CHECK(n >= 2 && n < 2147483647LL, SQB_ERR_INVALID, "sqb_autocorr_create: n=%lld out of range", (long long)n);
    SQB_CHECK(nnz >= 0 && nnz < 2147483647LL, SQB_ERR_INVALID, "sqb_autocorr_create: nnz=%lld does not fit int32", (long long)nnz);
    SQB_CHECK(w_dtype == 0 || w_dtype == 1, SQB_ERR_INVALID, "sqb_autocorr_create: w_dtype must be 0 (f32) or 1 (f64)");
    SQB_CHECK(w_indptr[0] == 0 && (int64_t)w_indptr[n] == nnz, SQB_ERR_INVALID, "sqb_autocorr_create: inconsistent indptr");
    SQB_CHECK(nnz == 0 || (w_indices && w_data), SQB_ERR_INVALID, "sqb_autocorr_create: null W arrays");
    // host validation (messages of the host path); the build itself is the device pass sqb_autocorr_create_device runs
    for (int64_t r = 0; r < n; ++r) {
        const int64_t d = (int64_t)w_indptr[r + 1] - (int64_t)w_indptr[r];
        SQB_CHECK(d >= 0 && w_indptr[r + 1] <= nnz, SQB_ERR_INVALID, "sqb_autocorr_create: indptr decreases at row %lld", (long long)r);
    }
    for (int64_t e = 0; e < nnz; ++e) {
        const int32_t j = w_indices[e];
        SQB_CHECK(j >= 0 && j < n, SQB_ERR_INVALID, "sqb_autocorr_create: column index %d out of range at entry %lld", j, (long long)e);
    }
    SQB_CUDA(cudaSetDevice(ctx->device));
    std::unique_ptr<sqb_autocorr> h(new sqb_autocorr(ctx));
    h->n = n;
    h->nnz = nnz;
    SQB_TRY(h->d_wp.alloc(n + 1));
    SQB_TRY(h->d_wi.alloc(nnz > 0 ? nnz : 1));
    SQB_TRY(h->d_flags.alloc(2));
    SQB_CUDA(cudaMemsetAsync(h->d_flags.p, 0, 2 * sizeof(int), ctx->stream));
    const size_t vbytes = (size_t)nnz * (w_dtype == 0 ? sizeof(float) : sizeof(double));
    DevBuf<uint8_t> wv(ctx->stream);
    SQB_TRY(wv.alloc(vbytes > 0 ? vbytes : 1));
    SQB_CUDA(cudaMemcpyAsync(h->d_wp.p, w_indptr, (n + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    if (nnz > 0) SQB_CUDA(cudaMemcpyAsync(h->d_wi.p, w_indices, nnz * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    if (nnz > 0) SQB_CUDA(cudaMemcpyAsync(wv.p, w_data, vbytes, cudaMemcpyHostToDevice, ctx->stream));
    if (w_dtype == 0)
        SQB_TRY(ac_build_w<float>(h.get(), reinterpret_cast<const float*>(wv.p), nullptr));
    else
        SQB_TRY(ac_build_w<double>(h.get(), reinterpret_cast<const double*>(wv.p), nullptr));
    *out = h.release();
    return SQB_OK;
}

int sqb_autocorr_create_device(sqb_ctx* ctx, int64_t n, int64_t nnz, const void* indptr, int indptr_bits, const void* indices, int index_bits,
                               const void* data, int value_code, int transformation, uintptr_t producer_stream, double* out_moments,
                               sqb_autocorr** out) {
    static const char* where = "sqb_autocorr_create_device";
    SQB_CHECK(ctx && out && indptr && out_moments, SQB_ERR_INVALID, "%s: null argument", where);
    SQB_CHECK(n >= 2 && n < 2147483647LL, SQB_ERR_INVALID, "%s: n=%lld out of range", where, (long long)n);
    SQB_CHECK(nnz >= 0 && nnz < 2147483647LL, SQB_ERR_INVALID, "%s: nnz=%lld does not fit int32", where, (long long)nnz);
    SQB_CHECK(value_code == 0 || value_code == 1, SQB_ERR_INVALID, "%s: value_code must be 0 (f32) or 1 (f64)", where);
    SQB_CHECK(nnz == 0 || (indices && data), SQB_ERR_INVALID, "%s: null W arrays", where);
    SQB_CUDA(cudaSetDevice(ctx->device));
    std::unique_ptr<sqb_autocorr> h(new sqb_autocorr(ctx));
    h->n = n;
    h->nnz = nnz;
    SQB_TRY(h->d_wp.alloc(n + 1));
    SQB_TRY(h->d_wi.alloc(nnz > 0 ? nnz : 1));
    SQB_TRY(h->d_flags.alloc(2));
    SQB_CUDA(cudaMemsetAsync(h->d_flags.p, 0, 2 * sizeof(int), ctx->stream));
    SQB_TRY(sqb_read_caller_buffers(ctx, producer_stream, [&]() -> int {
        return sqb_dispatch_index(indptr_bits, index_bits, where, [&](auto ipt, auto ixt) -> int {
            using IP = typename decltype(ipt)::type;
            using II = typename decltype(ixt)::type;
            // indptr first (one synchronisation): nothing follows it before it is known to run from 0 to nnz
            SQB_TRY(sqb_check_indptr(ctx, SQB_K_AUTOCORR_PREP, (const IP*)indptr, n, nnz, reinterpret_cast<uint32_t*>(h->d_wp.p), where));
            {
                SqbLaunchScope scope(ctx, SQB_K_AUTOCORR_PREP);
                ac_w_indices_kernel<II><<<ac_grid(ctx, n), 256, 0, ctx->stream>>>(h->d_wp.p, (const II*)indices, n, h->d_wi.p, h->d_flags.p);
                SQB_POST_LAUNCH();
            }
            int f = 0;
            SQB_CUDA(cudaMemcpyAsync(&f, h->d_flags.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
            SQB_CUDA(cudaStreamSynchronize(ctx->stream));
            SQB_CHECK(!(f & AC_ERR_INDEX), SQB_ERR_INVALID, "%s: %s", where, ac_err_text(AC_ERR_INDEX));
            SQB_CHECK(!(f & AC_W_NONCANON), SQB_ERR_LAYOUT, "%s: the column indices of a row are not strictly increasing", where);
            return value_code == 0 ? ac_create_from_device<float>(h.get(), data, transformation, out_moments)
                                   : ac_create_from_device<double>(h.get(), data, transformation, out_moments);
        });
    }));
    *out = h.release();
    return SQB_OK;
}

int sqb_autocorr_w_info(sqb_autocorr* h, int* w_format, int* s0_branch) {
    SQB_CHECK(h && w_format && s0_branch, SQB_ERR_INVALID, "sqb_autocorr_w_info: null argument");
    *w_format = h->w_fmt;
    *s0_branch = h->s0_branch;
    return SQB_OK;
}

int sqb_autocorr_destroy(sqb_autocorr* h) {
    if (!h) return SQB_OK;
    cudaSetDevice(h->ctx->device);
    delete h;
    return SQB_OK;
}

int sqb_autocorr_load_dense(sqb_autocorr* h, const void* x, int x_dtype, int layout, int64_t n_features) {
    SQB_CHECK(h && x, SQB_ERR_INVALID, "sqb_autocorr_load_dense: null argument");
    SQB_CHECK(x_dtype == 0 || x_dtype == 1, SQB_ERR_INVALID, "sqb_autocorr_load_dense: x_dtype must be 0 or 1");
    SQB_CHECK(layout == 0 || layout == 1, SQB_ERR_INVALID, "sqb_autocorr_load_dense: layout must be 0 or 1");
    SQB_CHECK(n_features >= 1, SQB_ERR_INVALID, "sqb_autocorr_load_dense: n_features must be positive");
    sqb_ctx* c = h->ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    const size_t bytes = (size_t)n_features * h->n * xsize(x_dtype);
    // zero-copy tiles read up to 31 elements past the last feature of a row: pad the allocation
    SQB_TRY(h->d_x.alloc(bytes + 64 * 8));
    SQB_TRY(h->d_out.alloc((size_t)n_features));
    SQB_TRY(sqb_h2d(c, h->d_x.p, x, bytes));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    h->kind = layout == 0 ? 1 : 2;
    h->x_dtype = x_dtype;
    h->n_feat = n_features;
    h->ran = false;
    h->aux_valid = false;
    return SQB_OK;
}

int sqb_autocorr_load_csr(sqb_autocorr* h, const int64_t* x_indptr, const int32_t* x_indices, const void* x_data, int x_dtype,
                          int layout, int64_t n_features) {
    SQB_CHECK(h && x_indptr, SQB_ERR_INVALID, "sqb_autocorr_load_csr: null argument");
    SQB_CHECK(x_dtype == 0 || x_dtype == 1, SQB_ERR_INVALID, "sqb_autocorr_load_csr: x_dtype must be 0 or 1");
    SQB_CHECK(layout == 0 || layout == 1, SQB_ERR_INVALID, "sqb_autocorr_load_csr: layout must be 0 or 1");
    SQB_CHECK(n_features >= 1 && n_features < 2147483647LL, SQB_ERR_INVALID, "sqb_autocorr_load_csr: n_features out of range");
    sqb_ctx* c = h->ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    const int64_t rows = layout == 0 ? n_features : h->n;
    const int64_t nnz = x_indptr[rows];
    SQB_CHECK(x_indptr[0] == 0 && nnz >= 0, SQB_ERR_INVALID, "sqb_autocorr_load_csr: bad indptr");
    SQB_CHECK(nnz == 0 || (x_indices && x_data), SQB_ERR_INVALID, "sqb_autocorr_load_csr: null X arrays");
    h->kind = 0;
    h->aux_valid = false;
    h->ran = false;
    // index range, indptr monotonicity and duplicate observations are checked on the device while the matrix is
    // re-laid out (no host pass over the non-zeros)
    if (x_dtype == 0)
        SQB_TRY(ac_load_csr_host<float>(h, x_indptr, x_indices, x_data, layout, n_features));
    else
        SQB_TRY(ac_load_csr_host<double>(h, x_indptr, x_indices, x_data, layout, n_features));
    h->kind = 3;
    h->x_dtype = x_dtype;
    h->n_feat = n_features;
    return SQB_OK;
}

int sqb_autocorr_load_csr_cols(sqb_autocorr* h, const int64_t* x_indptr, const int32_t* x_indices, const void* x_data, int x_dtype,
                               int64_t n_features_total, int64_t col_lo, int64_t col_hi) {
    SQB_CHECK(h && x_indptr, SQB_ERR_INVALID, "sqb_autocorr_load_csr_cols: null argument");
    SQB_CHECK(x_dtype == 0 || x_dtype == 1, SQB_ERR_INVALID, "sqb_autocorr_load_csr_cols: x_dtype must be 0 or 1");
    SQB_CHECK(0 <= col_lo && col_lo < col_hi && col_hi <= n_features_total && n_features_total < 2147483647LL, SQB_ERR_INVALID,
              "sqb_autocorr_load_csr_cols: bad column range [%lld, %lld) of %lld", (long long)col_lo, (long long)col_hi,
              (long long)n_features_total);
    sqb_ctx* c = h->ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    const int64_t n = h->n;
    const int64_t nnz_all = x_indptr[n];
    SQB_CHECK(x_indptr[0] == 0 && nnz_all >= 0, SQB_ERR_INVALID, "sqb_autocorr_load_csr_cols: bad indptr");
    SQB_CHECK(nnz_all == 0 || (x_indices && x_data), SQB_ERR_INVALID, "sqb_autocorr_load_csr_cols: null X arrays");
    // per observation: the run of entries with col_lo <= column < col_hi (rows hold ascending columns: two binary searches)
    std::vector<int64_t> start((size_t)n), cnt((size_t)n), ptr((size_t)n + 1);
    {
        int threads = (int)std::thread::hardware_concurrency() / 8;
        threads = threads < 2 ? 2 : (threads > 16 ? 16 : threads);
        std::vector<std::thread> pool;
        std::vector<int> bad((size_t)threads, 0);
        for (int t = 0; t < threads; ++t) {
            pool.emplace_back([&, t]() {
                for (int64_t r = n * t / threads; r < n * (t + 1) / threads; ++r) {
                    const int64_t a = x_indptr[r], b = x_indptr[r + 1];
                    if (a > b || a < 0 || b > nnz_all) {
                        bad[t] = 1;
                        start[r] = 0;
                        cnt[r] = 0;
                        continue;
                    }
                    const int32_t* lo = std::lower_bound(x_indices + a, x_indices + b, (int32_t)col_lo);
                    const int32_t* hi = std::lower_bound(lo, x_indices + b, (int32_t)col_hi);
                    start[r] = lo - x_indices;
                    cnt[r] = hi - lo;
                }
            });
        }
        for (auto& th : pool) th.join();
        for (int t = 0; t < threads; ++t) SQB_CHECK(!bad[t], SQB_ERR_INVALID, "sqb_autocorr_load_csr_cols: indptr is not non-decreasing");
    }
    ptr[0] = 0;
    for (int64_t r = 0; r < n; ++r) ptr[r + 1] = ptr[r] + cnt[r];
    h->kind = 0;
    h->aux_valid = false;
    h->ran = false;
    // the device checks that every uploaded column lies in [col_lo, col_hi) (an unsorted row shows up there or as a
    // duplicate) while it re-lays the slice out
    const int64_t nf = col_hi - col_lo;
    if (x_dtype == 0)
        SQB_TRY(ac_load_csr_host<float>(h, ptr.data(), x_indices, x_data, 1, nf, (int32_t)col_lo, start.data(), cnt.data()));
    else
        SQB_TRY(ac_load_csr_host<double>(h, ptr.data(), x_indices, x_data, 1, nf, (int32_t)col_lo, start.data(), cnt.data()));
    h->kind = 3;
    h->x_dtype = x_dtype;
    h->n_feat = nf;
    return SQB_OK;
}

int sqb_autocorr_load_csr_device(sqb_autocorr* h, const void* indptr, int indptr_bits, const void* indices, int index_bits,
                                 const void* data, int data_dtype, int layout, int64_t n_cols, const int32_t* col_map, int64_t n_out,
                                 uintptr_t producer_stream) {
    static const char* where = "sqb_autocorr_load_csr_device";
    SQB_CHECK(h && indptr && col_map, SQB_ERR_INVALID, "%s: null argument", where);
    SQB_CHECK(layout == 0 || layout == 1, SQB_ERR_INVALID, "%s: layout must be 0 or 1", where);
    std::vector<int32_t> inv;
    SQB_TRY(ac_invert_col_map(col_map, n_cols, n_out, inv, where));
    sqb_ctx* c = h->ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    h->kind = 0;
    h->aux_valid = false;
    h->ran = false;
    SQB_TRY(sqb_read_caller_buffers(c, producer_stream, [&] {
        return sqb_dispatch_index(indptr_bits, index_bits, where, [&](auto ipt, auto ixt) {
            using IP = typename decltype(ipt)::type;
            using II = typename decltype(ixt)::type;
            return sqb_dispatch_value(data_dtype, where, "data_dtype", [&](auto vt) {
                using VT = typename decltype(vt)::type;
                return ac_relayout_csr<IP, II, VT, AcX<VT>>(h, (const IP*)indptr, (const II*)indices, (const VT*)data, layout, n_cols, col_map, 0,
                                                            inv, n_out, where);
            });
        });
    }));
    h->kind = 3;
    h->x_dtype = data_dtype == 0 ? 0 : 1;
    h->n_feat = n_out;
    return SQB_OK;
}

int sqb_autocorr_load_dense_device(sqb_autocorr* h, const void* x, int x_dtype, int64_t rows, int64_t cols, int64_t stride_row,
                                   int64_t stride_col, int layout, const int32_t* col_map, int64_t n_out, uintptr_t producer_stream) {
    static const char* where = "sqb_autocorr_load_dense_device";
    SQB_CHECK(h && x && col_map, SQB_ERR_INVALID, "%s: null argument", where);
    SQB_CHECK(layout == 0 || layout == 1, SQB_ERR_INVALID, "%s: layout must be 0 or 1", where);
    const int64_t n_obs = layout == 1 ? rows : cols, n_cols = layout == 1 ? cols : rows;
    SQB_CHECK(n_obs == h->n, SQB_ERR_INVALID, "%s: expected %lld observations, found %lld", where, (long long)h->n, (long long)n_obs);
    const int64_t s_obs = layout == 1 ? stride_row : stride_col, s_feat = layout == 1 ? stride_col : stride_row;
    std::vector<int32_t> inv;
    SQB_TRY(ac_invert_col_map(col_map, n_cols, n_out, inv, where));
    sqb_ctx* c = h->ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    h->kind = 0;
    h->aux_valid = false;
    h->ran = false;
    const int xt = x_dtype == 0 ? 0 : 1;
    // zero-copy tiles read up to 31 elements past the last feature of a row: pad the allocation (as sqb_autocorr_load_dense)
    SQB_TRY(h->d_x.alloc((size_t)n_out * h->n * xsize(xt) + 64 * 8));
    SQB_TRY(h->d_out.alloc((size_t)n_out));
    DevBuf<int32_t> map(c->stream);
    SQB_TRY(map.alloc(n_out));
    SQB_TRY(sqb_read_caller_buffers(c, producer_stream, [&]() -> int {
        SQB_CUDA(cudaMemcpyAsync(map.p, inv.data(), n_out * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        SQB_TRY(sqb_dispatch_value(x_dtype, where, "x_dtype", [&](auto vt) {
            using VT = typename decltype(vt)::type;
            return ac_gather_dense<VT, AcX<VT>>(h, x, n_out, s_obs, s_feat, map.p, layout);
        }));
        SQB_CUDA(cudaStreamSynchronize(c->stream));  // the caller's buffer is no longer read
        return SQB_OK;
    }));
    h->kind = layout == 0 ? 1 : 2;
    h->x_dtype = xt;
    h->n_feat = n_out;
    return SQB_OK;
}

// upload + validate one or more row permutations (int64 host layout); d_perm (int64) and d_perm32 hold them afterwards
static int ac_upload_perms(sqb_autocorr* h, const int64_t* row_perm, int64_t count) {
    sqb_ctx* c = h->ctx;
    const int64_t n = h->n;
    const int64_t words = ceil_div64(n, 32);
    SQB_TRY(h->d_perm.alloc((size_t)(n * count)));
    SQB_TRY(h->d_perm32.alloc((size_t)(n * count)));
    SQB_TRY(h->d_seen.alloc((size_t)(words * count)));
    SQB_TRY(sqb_h2d(c, h->d_perm.p, row_perm, (size_t)(n * count) * sizeof(int64_t)));
    SQB_CUDA(cudaMemsetAsync(h->d_seen.p, 0, (size_t)(words * count) * sizeof(unsigned int), c->stream));
    for (int64_t k = 0; k < count; ++k) {
        SqbLaunchScope scope(c, SQB_K_AUTOCORR_PREP);
        ac_perm_prepare_kernel<<<c->sm_count * 2, 256, 0, c->stream>>>(h->d_perm.p + k * n, n, h->d_perm32.p + k * n, h->d_seen.p + k * words,
                                                                       h->d_flags.p);
        SQB_POST_LAUNCH();
    }
    return SQB_OK;
}

// the per-feature invariants a permuted sparse run reads are those of an unpermuted run of the same mode
static bool ac_aux_ready(const sqb_autocorr* h, int mode) { return h->aux_valid && h->aux_mode == mode; }

static int ac_run_one(sqb_autocorr* h, int mode, int64_t perm_index /* -1: none */, double* d_out) {
    if (h->kind == 3) {
        if (perm_index >= 0 && !ac_aux_ready(h, mode)) SQB_TRY(ac_run_sparse(h, mode, nullptr, h->d_out.p));
        return ac_run_sparse(h, mode, perm_index >= 0 ? h->d_perm32.p + perm_index * h->n : nullptr, d_out);
    }
    const int64_t* dp = perm_index >= 0 ? h->d_perm.p + perm_index * h->n : nullptr;
    SQB_TRY(h->x_dtype == 0 ? ac_run_dense<float>(h, mode, dp) : ac_run_dense<double>(h, mode, dp));
    if (d_out != h->d_out.p)
        SQB_CUDA(cudaMemcpyAsync(d_out, h->d_out.p, h->n_feat * sizeof(double), cudaMemcpyDeviceToDevice, h->ctx->stream));
    return SQB_OK;
}

int sqb_autocorr_run_async(sqb_autocorr* h, int mode, const int64_t* row_perm) {
    SQB_CHECK(h, SQB_ERR_INVALID, "sqb_autocorr_run_async: null handle");
    SQB_CHECK(h->kind != 0, SQB_ERR_STATE, "sqb_autocorr_run_async: load X first");
    SQB_CHECK(mode == 0 || mode == 1, SQB_ERR_INVALID, "sqb_autocorr_run_async: mode must be 0 (moran) or 1 (geary)");
    sqb_ctx* c = h->ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    if (row_perm) {
        SQB_TRY(ac_upload_perms(h, row_perm, 1));
        SQB_TRY(ac_check_flags(h, "sqb_autocorr_run_async"));
    }
    int rc = ac_run_one(h, mode, row_perm ? 0 : -1, h->d_out.p);
    if (rc == SQB_OK) h->ran = true;
    return rc;
}

int sqb_autocorr_download(sqb_autocorr* h, double* out) {
    SQB_CHECK(h && out, SQB_ERR_INVALID, "sqb_autocorr_download: null argument");
    SQB_CHECK(h->ran, SQB_ERR_STATE, "sqb_autocorr_download: nothing has run");
    sqb_ctx* c = h->ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    SQB_CUDA(cudaMemcpyAsync(out, h->d_out.p, h->n_feat * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    return SQB_OK;
}

int sqb_autocorr_run_perms(sqb_autocorr* h, int mode, const int64_t* row_perms, int64_t n_perms, double* out) {
    SQB_CHECK(h && row_perms && out, SQB_ERR_INVALID, "sqb_autocorr_run_perms: null argument");
    SQB_CHECK(h->kind != 0, SQB_ERR_STATE, "sqb_autocorr_run_perms: load X first");
    SQB_CHECK(mode == 0 || mode == 1, SQB_ERR_INVALID, "sqb_autocorr_run_perms: mode must be 0 (moran) or 1 (geary)");
    SQB_CHECK(n_perms >= 1, SQB_ERR_INVALID, "sqb_autocorr_run_perms: n_perms must be positive");
    sqb_ctx* c = h->ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    const int64_t G = h->n_feat;
    // permutations are staged in batches of <= 32 (8 bytes + 4 bytes + 1 bit per entry on the device)
    const int64_t batch = n_perms < 32 ? n_perms : 32;
    SQB_TRY(h->d_out_perms.alloc((size_t)(batch * G)));
    for (int64_t p0 = 0; p0 < n_perms; p0 += batch) {
        const int64_t pb = n_perms - p0 < batch ? n_perms - p0 : batch;
        SQB_TRY(ac_upload_perms(h, row_perms + p0 * h->n, pb));
        if (h->kind == 3) {  // sparse X: one launch scores the whole batch (the feature's bitmap is built once per batch)
            if (!ac_aux_ready(h, mode)) SQB_TRY(ac_run_sparse(h, mode, nullptr, h->d_out.p));
            SQB_TRY(ac_run_sparse(h, mode, h->d_perm32.p, h->d_out_perms.p, (int)pb));
        } else {
            for (int64_t k = 0; k < pb; ++k) SQB_TRY(ac_run_one(h, mode, k, h->d_out_perms.p + k * G));
        }
        SQB_CUDA(cudaMemcpyAsync(out + p0 * G, h->d_out_perms.p, (size_t)(pb * G) * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        SQB_TRY(ac_check_flags(h, "sqb_autocorr_run_perms"));  // synchronises
    }
    return SQB_OK;
}

int sqb_autocorr_dense(sqb_autocorr* h, int mode, const void* x, int x_dtype, int layout, int64_t n_features,
                       const int64_t* row_perm, double* out) {
    SQB_TRY(sqb_autocorr_load_dense(h, x, x_dtype, layout, n_features));
    SQB_TRY(sqb_autocorr_run_async(h, mode, row_perm));
    return sqb_autocorr_download(h, out);
}

int sqb_autocorr_csr(sqb_autocorr* h, int mode, const int64_t* x_indptr, const int32_t* x_indices, const void* x_data,
                     int x_dtype, int layout, int64_t n_features, const int64_t* row_perm, double* out) {
    SQB_TRY(sqb_autocorr_load_csr(h, x_indptr, x_indices, x_data, x_dtype, layout, n_features));
    SQB_TRY(sqb_autocorr_run_async(h, mode, row_perm));
    return sqb_autocorr_download(h, out);
}

}  // extern "C"
