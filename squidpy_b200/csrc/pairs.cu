// pairs.cu — tiled all-pairs radial histograms (sm_90a): co_occurrence counts (float32) and Ripley-L pair
// counts (float64).
//
// Replaces  _occur_count                      src/squidpy/gr/_ppatterns.py:283-310   (float32, ordered pairs i != j,
//                                             cumulative in r, per (label_i, label_j))
//      and  KDTree.two_point_correlation      src/squidpy/gr/_ripley.py:218-223       (float64, ordered pairs incl. i == j,
//                                             cumulative in r, per cluster; euclidean, manhattan or chebyshev)
// Points are grouped by label on the host (stable counting sort), so every tile of the pair matrix belongs to
// ONE (label_a, label_b) cell and only an L-bin radial histogram is needed per tile.  Each warp keeps a
// lane-private histogram column in shared memory (bank == lane: no conflicts, no atomics); a pair is binned
// once (first threshold it satisfies) and the cumulative sum over r is taken on the host.  Symmetry is used:
// only tiles with group_a <= group_b (and block_i <= block_j inside a group) are evaluated; d2 is exactly
// symmetric in floating point because negation is exact.  Not HBM bound: every point is re-used ~N/tile
// times from shared memory; the bound is FP32/INT issue rate (no tensor cores — there is no contraction here).
#include <algorithm>
#include <cmath>
#include <limits>
#include <type_traits>

#include "common.cuh"

struct PairTile {
    int32_t i0, i1, j0, j1;
    int32_t slot;    // output histogram slot
    int32_t weight;  // 1, or 2 for off-diagonal tiles inside one group (each unordered pair = 2 ordered pairs)
    int32_t diag;    // 1: i-range == j-range, skip i == j, all ordered pairs enumerated
    int32_t pad;
};

template <typename FT>
struct Vec2;
template <>
struct Vec2<float> {
    typedef float2 type;
};
template <>
struct Vec2<double> {
    typedef double2 type;
};

// d2 exactly as the reference computes it
template <typename FT, int FMA>
__device__ __forceinline__ FT sqb_d2(FT dx, FT dy);
template <>
__device__ __forceinline__ float sqb_d2<float, 1>(float dx, float dy) {
    return __fmaf_rn(dy, dy, __fmul_rn(dx, dx));  // numba fastmath on x86-64+FMA: vmulss dx,dx ; vfmadd231ss dy,dy
}
template <>
__device__ __forceinline__ float sqb_d2<float, 0>(float dx, float dy) {
    return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
}
template <>
__device__ __forceinline__ double sqb_d2<double, 0>(double dx, double dy) {
    return __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));  // sklearn euclidean_dist: d += tmp*tmp, no contraction
}
template <>
__device__ __forceinline__ double sqb_d2<double, 1>(double dx, double dy) {
    return __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
}

// Ripley-L pair distance in the kernel's compare space (float64 only).  METRIC 0: squared euclidean, compared with squared
// thresholds; 1 manhattan |dx| + |dy| and 2 chebyshev max(|dx|, |dy|), compared with the radii themselves.  These are
// scikit-learn's EuclideanDistance / ManhattanDistance / ChebyshevDistance in float64 (0 + |dx| + |dy| == |dx| + |dy|, and
// max(0, |dx|, |dy|) == max(|dx|, |dy|)).  All are exactly symmetric in (i, j): |a - b| == |b - a| in round-to-nearest.
template <typename FT, int FMA, int METRIC>
__device__ __forceinline__ FT sqb_pair_dist(FT dx, FT dy) {
    static_assert(METRIC == 0 || std::is_same<FT, double>::value, "manhattan / chebyshev pair counts are float64 only");
    if constexpr (METRIC == 0)
        return sqb_d2<FT, FMA>(dx, dy);
    else if constexpr (METRIC == 1)
        return __dadd_rn(fabs(dx), fabs(dy));
    else
        return fmax(fabs(dx), fabs(dy));
}

#define PAIRS_THREADS 256
#define PAIRS_IPT 4
#define PAIRS_JCHUNK 1024
#define PAIRS_NC 1024

// LANEPRIV: hist[warp][bin][lane] (conflict-free, plain read-modify-write); else hist[warp][bin] with atomics.
// Launch bounds: a minimum of 1 block per SM lets ptxas give the manhattan / chebyshev kernels the 64-72 registers they
// need without spilling; 0 (no minimum) leaves the euclidean and co-occurrence kernels as ptxas allocates them by default.
template <typename FT, int FMA, int METRIC, bool LANEPRIV>
__global__ void __launch_bounds__(PAIRS_THREADS, METRIC == 0 ? 0 : 1) pairs_kernel(const typename Vec2<FT>::type* __restrict__ pts,
                                                              const PairTile* __restrict__ tiles, int64_t ntiles,
                                                              int shard_index, int shard_count, const FT* __restrict__ thr,
                                                              int L, const int* __restrict__ lut, FT lut_scale,
                                                              unsigned long long* __restrict__ out) {
    typedef typename Vec2<FT>::type V2;
    extern __shared__ unsigned char smem_raw[];
    // layout: V2 s_pts[JCHUNK] | FT s_thr[L+1] | int s_lut[NC] | uint32 hist[...]
    V2* s_pts = reinterpret_cast<V2*>(smem_raw);
    FT* s_thr = reinterpret_cast<FT*>(s_pts + PAIRS_JCHUNK);
    int* s_lut = reinterpret_cast<int*>(s_thr + (L + 1 + 1) / 2 * 2);
    uint32_t* hist_all = reinterpret_cast<uint32_t*>(s_lut + PAIRS_NC);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int hstride = LANEPRIV ? L * 32 : L;
    uint32_t* hist = hist_all + warp * hstride;

    for (int i = tid; i < L; i += PAIRS_THREADS) s_thr[i] = thr[i];
    if (tid == 0) s_thr[L] = (FT)INFINITY;
    for (int i = tid; i < PAIRS_NC; i += PAIRS_THREADS) s_lut[i] = lut[i];
    __syncthreads();
    const FT thr_max = s_thr[L - 1];

    for (int64_t tt = blockIdx.x; ; tt += gridDim.x) {
        const int64_t t = tt * shard_count + shard_index;
        if (t >= ntiles) break;
        const PairTile tile = tiles[t];
        for (int i = lane; i < hstride; i += 32) hist[i] = 0;
        __syncwarp();
        FT xi[PAIRS_IPT], yi[PAIRS_IPT];
        int gi[PAIRS_IPT];
#pragma unroll
        for (int q = 0; q < PAIRS_IPT; ++q) {
            gi[q] = tile.i0 + tid + q * PAIRS_THREADS;
            if (gi[q] < tile.i1) {
                const V2 p = pts[gi[q]];
                xi[q] = p.x;
                yi[q] = p.y;
            } else {
                gi[q] = -1;
                // NaN never satisfies d2 <= thr.  Both coordinates must stay NaN: fmax (METRIC 2) returns its non-NaN
                // operand, so one finite axis would give a padded lane a real distance.
                xi[q] = (FT)NAN;
                yi[q] = (FT)NAN;
            }
        }
        for (int jb = tile.j0; jb < tile.j1; jb += PAIRS_JCHUNK) {
            const int cnt = min(PAIRS_JCHUNK, tile.j1 - jb);
            __syncthreads();
            for (int k = tid; k < cnt; k += PAIRS_THREADS) s_pts[k] = pts[jb + k];
            __syncthreads();
            for (int jj = 0; jj < cnt; ++jj) {
                const V2 pj = s_pts[jj];
                const int gj = jb + jj;
#pragma unroll
                for (int q = 0; q < PAIRS_IPT; ++q) {
                    const FT d2 = sqb_pair_dist<FT, FMA, METRIC>(xi[q] - pj.x, yi[q] - pj.y);
                    if (d2 <= thr_max && !(tile.diag && gj == gi[q])) {
                        int cell = (int)(d2 * lut_scale) - 1;
                        cell = max(0, min(cell, PAIRS_NC - 1));
                        int b = s_lut[cell];
                        while (s_thr[b] < d2) ++b;
                        if (LANEPRIV)
                            hist[b * 32 + lane] += 1u;
                        else
                            atomicAdd(&hist[b], 1u);
                    }
                }
            }
        }
        __syncwarp();
        // flush this warp's histogram
        if (LANEPRIV) {
            for (int b = 0; b < L; ++b) {
                uint32_t v = hist[b * 32 + lane];
#pragma unroll
                for (int d = 16; d >= 1; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
                if (lane == 0 && v) atomicAdd(&out[(int64_t)tile.slot * L + b], (unsigned long long)v * tile.weight);
            }
        } else {
            for (int b = lane; b < L; b += 32) {
                const uint32_t v = hist[b];
                if (v) atomicAdd(&out[(int64_t)tile.slot * L + b], (unsigned long long)v * tile.weight);
            }
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------------
template <typename FT>
static int pairs_run(sqb_ctx* c, const FT* xy /* interleaved, grouped */, int64_t n, const std::vector<int64_t>& gptr,
                     bool cross_groups, const FT* thr, int L, int use_fma, int metric, int shard_index, int shard_count,
                     std::vector<unsigned long long>& hout /* nslots*L */, int nslots_k) {
    typedef typename Vec2<FT>::type V2;
    const int k = (int)gptr.size() - 1;
    // ---- tiles ----
    const int TI = PAIRS_THREADS * PAIRS_IPT;  // 1024
    const int TJX = 4096;
    std::vector<PairTile> tiles;
    for (int a = 0; a < k; ++a) {
        const int64_t a0 = gptr[a], a1 = gptr[a + 1];
        // same group: square blocks, upper triangle
        for (int64_t bi = a0; bi < a1; bi += TI) {
            for (int64_t bj = bi; bj < a1; bj += TI) {
                PairTile t;
                t.i0 = (int32_t)bi;
                t.i1 = (int32_t)std::min<int64_t>(bi + TI, a1);
                t.j0 = (int32_t)bj;
                t.j1 = (int32_t)std::min<int64_t>(bj + TI, a1);
                t.slot = cross_groups ? a * nslots_k + a : a;
                t.diag = (bi == bj);
                t.weight = t.diag ? 1 : 2;
                t.pad = 0;
                tiles.push_back(t);
            }
        }
        if (!cross_groups) continue;
        for (int b = a + 1; b < k; ++b) {
            const int64_t b0 = gptr[b], b1 = gptr[b + 1];
            for (int64_t bi = a0; bi < a1; bi += TI) {
                for (int64_t bj = b0; bj < b1; bj += TJX) {
                    PairTile t;
                    t.i0 = (int32_t)bi;
                    t.i1 = (int32_t)std::min<int64_t>(bi + TI, a1);
                    t.j0 = (int32_t)bj;
                    t.j1 = (int32_t)std::min<int64_t>(bj + TJX, b1);
                    t.slot = a * nslots_k + b;
                    t.diag = 0;
                    t.weight = 1;
                    t.pad = 0;
                    tiles.push_back(t);
                }
            }
        }
    }
    const int64_t nslots = cross_groups ? (int64_t)nslots_k * nslots_k : k;
    hout.assign((size_t)nslots * L, 0ULL);
    const int64_t ntiles = (int64_t)tiles.size();
    if (ntiles == 0 || n == 0) return SQB_OK;

    // ---- LUT: lut[c] = #{thr < lower edge of cell c}, cells uniform in d2 over [0, thr_max] ----
    const double tmax = (double)thr[L - 1];
    const FT scale = (tmax > 0.0 && std::isfinite(tmax)) ? (FT)((double)PAIRS_NC / tmax) : (FT)0;
    std::vector<int> lut(PAIRS_NC);
    {
        int b = 0;
        for (int cidx = 0; cidx < PAIRS_NC; ++cidx) {
            // conservative lower edge: anything that maps to cell >= cidx+1 after the device's "-1" has d2*scale >= cidx+1,
            // so d2 >= (cidx + 1) / scale * (1 - eps); use cidx / scale, one full cell of slack
            const double edge = (double)scale > 0.0 ? (double)cidx / (double)scale : 0.0;
            while (b < L && (double)thr[b] < edge) ++b;
            lut[cidx] = b;
        }
    }
    DevBuf<V2> d_pts;
    DevBuf<PairTile> d_tiles;
    DevBuf<FT> d_thr;
    DevBuf<int> d_lut;
    DevBuf<unsigned long long> d_out;
    SQB_TRY(d_pts.alloc(n));
    SQB_TRY(d_tiles.alloc(ntiles));
    SQB_TRY(d_thr.alloc(L));
    SQB_TRY(d_lut.alloc(PAIRS_NC));
    SQB_TRY(d_out.alloc((size_t)nslots * L));
    SQB_CUDA(cudaMemcpyAsync(d_pts.p, xy, n * sizeof(V2), cudaMemcpyHostToDevice, c->stream));
    SQB_CUDA(cudaMemcpyAsync(d_tiles.p, tiles.data(), ntiles * sizeof(PairTile), cudaMemcpyHostToDevice, c->stream));
    SQB_CUDA(cudaMemcpyAsync(d_thr.p, thr, L * sizeof(FT), cudaMemcpyHostToDevice, c->stream));
    SQB_CUDA(cudaMemcpyAsync(d_lut.p, lut.data(), PAIRS_NC * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    SQB_CUDA(cudaMemsetAsync(d_out.p, 0, (size_t)nslots * L * sizeof(unsigned long long), c->stream));
    const size_t base_smem = PAIRS_JCHUNK * sizeof(V2) + (size_t)((L + 2) / 2 * 2) * sizeof(FT) + PAIRS_NC * sizeof(int);
    const size_t priv_smem = base_smem + (size_t)(PAIRS_THREADS / 32) * L * 32 * 4;
    const size_t shared_smem = base_smem + (size_t)(PAIRS_THREADS / 32) * L * 4;
    const bool lanepriv = priv_smem + 1024 <= c->smem_optin;
    const size_t smem = lanepriv ? priv_smem : shared_smem;
    SQB_CHECK(smem + 1024 <= c->smem_optin, SQB_ERR_UNSUPPORTED, "pairs: %d radial bins need %zu bytes of shared memory (> %zu)", L, smem,
              c->smem_optin);
    int ctas_per_sm = (int)std::max<size_t>(1, std::min<size_t>(8, (c->smem_optin + 1024) / (smem + 1024)));
    int64_t my_tiles = (ntiles - shard_index + shard_count - 1) / shard_count;
    int64_t grid = std::min<int64_t>((int64_t)c->sm_count * ctas_per_sm, std::max<int64_t>(my_tiles, 1));
    {
        SqbLaunchScope scope(c, SQB_K_PAIRS);
#define PAIRS_LAUNCH(FMAV, METRIC, LP)                                                                                \
    do {                                                                                                              \
        auto kern = pairs_kernel<FT, FMAV, METRIC, LP>;                                                               \
        SQB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                \
        kern<<<(unsigned)grid, PAIRS_THREADS, smem, c->stream>>>(d_pts.p, d_tiles.p, ntiles, shard_index, shard_count, \
                                                                 d_thr.p, L, d_lut.p, scale, d_out.p);                \
    } while (0)
        if constexpr (std::is_same<FT, double>::value) {
            if (metric == 1) {
                if (lanepriv)
                    PAIRS_LAUNCH(0, 1, true);
                else
                    PAIRS_LAUNCH(0, 1, false);
            } else if (metric == 2) {
                if (lanepriv)
                    PAIRS_LAUNCH(0, 2, true);
                else
                    PAIRS_LAUNCH(0, 2, false);
            }
        }
        if (metric == 0) {
            if (use_fma) {
                if (lanepriv)
                    PAIRS_LAUNCH(1, 0, true);
                else
                    PAIRS_LAUNCH(1, 0, false);
            } else {
                if (lanepriv)
                    PAIRS_LAUNCH(0, 0, true);
                else
                    PAIRS_LAUNCH(0, 0, false);
            }
        }
#undef PAIRS_LAUNCH
        SQB_POST_LAUNCH();
    }
    SQB_CUDA(cudaMemcpyAsync(hout.data(), d_out.p, (size_t)nslots * L * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    return SQB_OK;
}

extern "C" {

int sqb_cooc_counts(sqb_ctx* ctx, const float* x, const float* y, int64_t n, const int32_t* labs, int k, const float* thr,
                    int L, int use_fma, int shard_index, int shard_count, int64_t* out) {
    SQB_CHECK(ctx && x && y && labs && thr && out, SQB_ERR_INVALID, "sqb_cooc_counts: null argument");
    SQB_CHECK(n >= 0 && n < 2147483647LL, SQB_ERR_INVALID, "sqb_cooc_counts: n=%lld out of range", (long long)n);
    SQB_CHECK(k >= 1 && k <= 4096, SQB_ERR_INVALID, "sqb_cooc_counts: k=%d out of range [1,4096]", k);
    SQB_CHECK(L >= 1 && L <= 4096, SQB_ERR_INVALID, "sqb_cooc_counts: L=%d out of range [1,4096]", L);
    SQB_CHECK(shard_count >= 1 && shard_index >= 0 && shard_index < shard_count, SQB_ERR_INVALID, "sqb_cooc_counts: bad shard %d/%d",
              shard_index, shard_count);
    for (int r = 0; r < L; ++r) {
        SQB_CHECK(!(thr[r] != thr[r]), SQB_ERR_INVALID, "sqb_cooc_counts: thr[%d] is NaN", r);
        SQB_CHECK(r == 0 || thr[r] >= thr[r - 1], SQB_ERR_INVALID, "sqb_cooc_counts: thresholds must be ascending (thr[%d])", r);
    }
    SQB_CUDA(cudaSetDevice(ctx->device));
    // group by label (stable counting sort)
    std::vector<int64_t> gptr(k + 1, 0);
    for (int64_t i = 0; i < n; ++i) {
        SQB_CHECK(labs[i] >= 0 && labs[i] < k, SQB_ERR_INVALID, "sqb_cooc_counts: labs[%lld]=%d outside [0,%d)", (long long)i, labs[i], k);
        gptr[labs[i] + 1]++;
    }
    for (int a = 0; a < k; ++a) gptr[a + 1] += gptr[a];
    std::vector<float> xy((size_t)(n > 0 ? n : 1) * 2);
    {
        std::vector<int64_t> cur(gptr.begin(), gptr.end() - 1);
        for (int64_t i = 0; i < n; ++i) {
            const int64_t p = cur[labs[i]]++;
            xy[2 * p] = x[i];
            xy[2 * p + 1] = y[i];
        }
    }
    std::vector<unsigned long long> h;
    SQB_TRY(pairs_run<float>(ctx, xy.data(), n, gptr, true, thr, L, use_fma, 0, shard_index, shard_count, h, k));
    // first-bin histogram -> cumulative counts, mirrored to both (a,b) and (b,a)
    for (int a = 0; a < k; ++a) {
        for (int b = a; b < k; ++b) {
            unsigned long long run = 0;
            for (int r = 0; r < L; ++r) {
                run += h[((size_t)a * k + b) * L + r];
                out[((size_t)a * k + b) * L + r] = (int64_t)run;
                out[((size_t)b * k + a) * L + r] = (int64_t)run;
            }
        }
    }
    return SQB_OK;
}

int sqb_pair_counts_f64(sqb_ctx* ctx, const double* pts, const int64_t* group_ptr, int n_groups, const double* support, int S,
                        int metric, int shard_index, int shard_count, int64_t* out) {
    SQB_CHECK(ctx && pts && group_ptr && support && out, SQB_ERR_INVALID, "sqb_pair_counts_f64: null argument");
    SQB_CHECK(n_groups >= 1 && n_groups <= 1000000, SQB_ERR_INVALID, "sqb_pair_counts_f64: n_groups=%d out of range", n_groups);
    SQB_CHECK(S >= 1 && S <= 4096, SQB_ERR_INVALID, "sqb_pair_counts_f64: S=%d out of range [1,4096]", S);
    SQB_CHECK(metric >= 0 && metric <= 2, SQB_ERR_INVALID, "sqb_pair_counts_f64: metric=%d is not 0 (euclidean), 1 (manhattan) or 2 (chebyshev)",
              metric);
    SQB_CHECK(shard_count >= 1 && shard_index >= 0 && shard_index < shard_count, SQB_ERR_INVALID, "sqb_pair_counts_f64: bad shard %d/%d",
              shard_index, shard_count);
    SQB_CHECK(group_ptr[0] == 0, SQB_ERR_INVALID, "sqb_pair_counts_f64: group_ptr[0] must be 0");
    std::vector<int64_t> gptr(group_ptr, group_ptr + n_groups + 1);
    for (int g = 0; g < n_groups; ++g)
        SQB_CHECK(gptr[g + 1] >= gptr[g], SQB_ERR_INVALID, "sqb_pair_counts_f64: group_ptr must be non-decreasing");
    const int64_t n = gptr[n_groups];
    SQB_CHECK(n < 2147483647LL, SQB_ERR_INVALID, "sqb_pair_counts_f64: too many points");
    // euclidean thresholds in d2 space: T_s = max{ t : sqrt(t) <= r_s }  (sqrt is monotone and correctly rounded), so that
    // (sqrt(d2) <= r_s)  <=>  (d2 <= T_s) exactly.  Manhattan and chebyshev compare the distance itself: T_s = r_s.
    std::vector<double> T(S);
    for (int s = 0; s < S; ++s) {
        const double r = support[s];
        SQB_CHECK(!(r != r), SQB_ERR_INVALID, "sqb_pair_counts_f64: support[%d] is NaN", s);
        SQB_CHECK(s == 0 || r >= support[s - 1], SQB_ERR_INVALID, "sqb_pair_counts_f64: support must be ascending (support[%d])", s);
        if (metric != 0) {
            T[s] = r;  // a negative radius counts nothing: every distance is >= 0
            continue;
        }
        if (r < 0.0) {
            T[s] = -1.0;  // nothing satisfies sqrt(d2) <= negative
            continue;
        }
        double t = r * r;
        if (!std::isfinite(t)) {
            T[s] = std::numeric_limits<double>::max();
            continue;
        }
        while (std::sqrt(t) > r) t = std::nextafter(t, -1.0);
        while (true) {
            const double u = std::nextafter(t, std::numeric_limits<double>::infinity());
            if (std::isfinite(u) && std::sqrt(u) <= r)
                t = u;
            else
                break;
        }
        T[s] = t;
    }
    SQB_CUDA(cudaSetDevice(ctx->device));
    std::vector<unsigned long long> h;
    SQB_TRY(pairs_run<double>(ctx, pts, n, gptr, false, T.data(), S, 0, metric, shard_index, shard_count, h, n_groups));
    for (int g = 0; g < n_groups; ++g) {
        unsigned long long run = 0;
        const int64_t m = gptr[g + 1] - gptr[g];
        // self pairs (distance 0 <= every non-negative radius) are added by shard 0 only
        for (int s = 0; s < S; ++s) {
            run += h[(size_t)g * S + s];
            int64_t v = (int64_t)run;
            if (shard_index == 0 && support[s] >= 0.0) v += m;
            out[(size_t)g * S + s] = v;
        }
    }
    return SQB_OK;
}

}  // extern "C"
