// sepal.cu — Sepal diffusion scores (sm_90a): for every gene simulate diffusion on the regular spot lattice until the entropy
// of the concentration field stops changing; the score is the (virtual) time that took.
//
// Replaces `_diffusion` / `_diffusion_genes` of the reference (src/squidpy/gr/_sepal.py:186-289): per iteration
//     nhood[j] = sum_k conc[sat_idx[j, k]]                         (saturated nodes: all max_neighs neighbours present)
//     d2[j]    = hex ? (2 nhood[j] - 12 conc[sat[j]]) / 3 : nhood[j] - 4 conc[sat[j]]
//     conc[sat] += d2 dt;  conc[unsat] += d2[nearest saturated node] dt;  conc = max(conc, 0)
//     ent = -sum_sat p log p / n_sat,  p = conc / sum(conc > 0);   stop when |ent - ent_prev| <= thresh  (ent_prev starts at 1)
// One CTA owns one gene at a time (genes are independent; up to 30 000 dependent iterations each): the concentration and the
// increment vector live in shared memory (2 x 8 bytes per spot; global scratch beyond ~14 000 spots), the neighbour tables are
// re-read through L1 every iteration, two block barriers + one fixed-order block reduction of (sum x, sum x log x) per
// iteration (ent = log S - sum(x log x) / S is the same entropy with one pass instead of two).  float64 throughout.
// The reference's entropy clamps p = x / S to at least eps before the log; this one does not.  For one entry with p < eps the
// two terms differ by p (log eps - log p) <= eps / e ~ 8.2e-17 (the maximum, at p = eps / e), so after the division by n_sat the
// entropies differ by at most 8.2e-17 times the clamped fraction of the saturated spots: the clamp can move a stop only where
// |ent change| lies within ~1.6e-16 of thresh, a decision float64 rounding alone already leaves open.
// tests/test_gpu_sepal_exact.py pins the stopping iteration exactly, on both sides of the shared-memory rule, against a
// float64 / long-double restatement of the reference on every gene whose decisions are well conditioned.  The reference
// itself compiles with numba fastmath (re-associated sums, approximate log), so against its own output a stop can differ by
// one or two steps on genes whose entropy change crosses the threshold very slowly.
#include <math.h>

#include "common.cuh"

#define SEPAL_T 512
#define SEPAL_NW (SEPAL_T / 32)

struct SepalParams {
    const double* vals;  // [n_genes][n]
    int64_t n_genes, n;
    const int32_t* sat;
    const int32_t* sat_idx;  // [n_sat][K]
    int n_sat, K;
    const int32_t* unsat;
    const int32_t* unsat_idx;
    int n_unsat;
    int use_hex, n_iter;
    double dt, thresh;
    double* out;       // [n_genes]: dt * first converged iteration, NaN if none
    double* g_scratch;  // 2 * n doubles per CTA when the field does not fit shared memory, else null
    int* counter;
};

__global__ void __launch_bounds__(SEPAL_T) sepal_kernel(const __grid_constant__ SepalParams p) {
    extern __shared__ double sp_smem[];
    __shared__ double s_red[2][SEPAL_NW];
    __shared__ double s_ent;
    __shared__ int s_next, s_stop;
    double* conc = p.g_scratch ? p.g_scratch + (size_t)blockIdx.x * 2 * p.n : sp_smem;
    double* dcdt = conc + p.n;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double eps = 2.220446049250313e-16;
    for (;;) {
        if (threadIdx.x == 0) s_next = atomicAdd(p.counter, 1);
        __syncthreads();
        const int g = s_next;
        if (g >= p.n_genes) break;
        for (int64_t i = threadIdx.x; i < p.n; i += SEPAL_T) {
            conc[i] = p.vals[(size_t)g * p.n + i];
            dcdt[i] = 0.0;
        }
        __syncthreads();
        double prev_ent = 1.0;
        int result = -1;
        for (int it = 0; it < p.n_iter; ++it) {
            // increments of the saturated nodes from the current field
            for (int j = threadIdx.x; j < p.n_sat; j += SEPAL_T) {
                const int32_t* __restrict__ nb = p.sat_idx + (size_t)j * p.K;
                double nh = 0.0;
                for (int k = 0; k < p.K; ++k) nh += conc[__ldg(nb + k)];
                const int s = __ldg(p.sat + j);
                const double c = conc[s];
                dcdt[s] = p.use_hex ? (2.0 * nh - 12.0 * c) / 3.0 : nh - 4.0 * c;
            }
            __syncthreads();
            double sx = 0.0, sxl = 0.0;
            for (int j = threadIdx.x; j < p.n_sat; j += SEPAL_T) {
                const int s = __ldg(p.sat + j);
                double v = conc[s] + dcdt[s] * p.dt;
                v = v < 0.0 ? 0.0 : v;
                conc[s] = v;
                if (v > 0.0) {
                    sx += v;
                    sxl += v * log(v);
                }
            }
            for (int j = threadIdx.x; j < p.n_unsat; j += SEPAL_T) {
                const int u = __ldg(p.unsat + j);
                double v = conc[u] + dcdt[__ldg(p.unsat_idx + j)] * p.dt;
                conc[u] = v < 0.0 ? 0.0 : v;
            }
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) {
                sx += __shfl_xor_sync(0xffffffffu, sx, d);
                sxl += __shfl_xor_sync(0xffffffffu, sxl, d);
            }
            if (lane == 0) {
                s_red[0][warp] = sx;
                s_red[1][warp] = sxl;
            }
            __syncthreads();  // also: every conc update of this iteration is visible before the next one reads neighbours
            if (threadIdx.x == 0) {
                double S = 0.0, L = 0.0;
                for (int w = 0; w < SEPAL_NW; ++w) {
                    S += s_red[0][w];
                    L += s_red[1][w];
                }
                // -sum p log p with p = x / S  ==  log S - sum(x log x) / S;  S < eps -> 0 like the reference
                const double ent = (S < eps ? 0.0 : log(S) - L / S) / (double)p.n_sat;
                s_stop = fabs(ent - prev_ent) <= p.thresh ? 1 : 0;
                s_ent = ent;
            }
            __syncthreads();
            prev_ent = s_ent;
            if (s_stop) {
                result = it;
                break;
            }
        }
        if (threadIdx.x == 0) p.out[g] = result >= 0 ? p.dt * (double)result : __longlong_as_double(0x7ff8000000000000LL);
        __syncthreads();
    }
}

// the host-side argument checks shared by both entry points
static int sepal_check(const int32_t* sat, int64_t n_sat, const int32_t* sat_idx, int max_neighs, const int32_t* unsat,
                       const int32_t* unsat_idx, int64_t n_unsat, int64_t n_genes, int64_t n, int n_iter) {
    SQB_CHECK(max_neighs == 4 || max_neighs == 6, SQB_ERR_INVALID, "Expected `max_neighs` to be either `4` or `6`, found `%d`.", max_neighs);
    SQB_CHECK(n_genes >= 1 && n >= 1 && n < 2147483647LL && n_sat >= 1 && n_sat <= n && n_unsat >= 0 && n_iter >= 1, SQB_ERR_INVALID,
              "sqb_sepal: bad sizes");
    for (int64_t j = 0; j < n_sat; ++j) SQB_CHECK(sat[j] >= 0 && sat[j] < n, SQB_ERR_INVALID, "sqb_sepal: node index out of range");
    for (int64_t j = 0; j < n_sat * max_neighs; ++j) SQB_CHECK(sat_idx[j] >= 0 && sat_idx[j] < n, SQB_ERR_INVALID, "sqb_sepal: neighbour index out of range");
    for (int64_t j = 0; j < n_unsat; ++j)
        SQB_CHECK(unsat[j] >= 0 && unsat[j] < n && unsat_idx[j] >= 0 && unsat_idx[j] < n, SQB_ERR_INVALID, "sqb_sepal: node index out of range");
    return SQB_OK;
}

// sqb_sepal over genes x observations float64 values already on the device (d_vals: the host copy of sqb_sepal, or a gathered
// sqb_dense); the arguments have been checked
static int sepal_impl(sqb_ctx* c, const double* d_vals, int64_t n_genes, int64_t n, const int32_t* sat, int64_t n_sat, const int32_t* sat_idx,
                      int max_neighs, const int32_t* unsat, const int32_t* unsat_idx, int64_t n_unsat, int n_iter, double dt, double thresh,
                      double* out) {
    const size_t need = (size_t)2 * n * sizeof(double);
    const bool global = need + 1024 > c->smem_optin;
    const size_t smem = global ? 0 : need;
    if (!global && smem > 48 * 1024) SQB_CUDA(cudaFuncSetAttribute(sepal_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 1;
    SQB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sepal_kernel, SEPAL_T, smem));
    if (per_sm < 1) per_sm = 1;
    int64_t ctas = (int64_t)per_sm * c->sm_count;
    if (ctas > n_genes) ctas = n_genes;
    DevBuf<double> d_out, d_scr;
    DevBuf<int32_t> d_sat, d_idx, d_unsat, d_uidx;
    DevBuf<int> d_cnt;
    SQB_TRY(d_out.alloc(n_genes));
    SQB_TRY(d_sat.alloc(n_sat));
    SQB_TRY(d_idx.alloc((size_t)n_sat * max_neighs));
    SQB_TRY(d_unsat.alloc(n_unsat > 0 ? n_unsat : 1));
    SQB_TRY(d_uidx.alloc(n_unsat > 0 ? n_unsat : 1));
    SQB_TRY(d_cnt.alloc(1));
    if (global) SQB_TRY(d_scr.alloc((size_t)ctas * 2 * n));
    auto body = [&]() -> int {
        SQB_CUDA(cudaMemsetAsync(d_cnt.p, 0, sizeof(int), c->stream));
        SQB_CUDA(cudaMemcpyAsync(d_sat.p, sat, n_sat * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        SQB_CUDA(cudaMemcpyAsync(d_idx.p, sat_idx, (size_t)n_sat * max_neighs * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        if (n_unsat > 0) SQB_CUDA(cudaMemcpyAsync(d_unsat.p, unsat, n_unsat * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        if (n_unsat > 0) SQB_CUDA(cudaMemcpyAsync(d_uidx.p, unsat_idx, n_unsat * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        {
            SepalParams p;
            p.vals = d_vals, p.n_genes = n_genes, p.n = n, p.sat = d_sat.p, p.sat_idx = d_idx.p, p.n_sat = (int)n_sat, p.K = max_neighs;
            p.unsat = d_unsat.p, p.unsat_idx = d_uidx.p, p.n_unsat = (int)n_unsat, p.use_hex = max_neighs == 6, p.n_iter = n_iter, p.dt = dt, p.thresh = thresh;
            p.out = d_out.p, p.g_scratch = global ? d_scr.p : nullptr, p.counter = d_cnt.p;
            SqbLaunchScope scope(c, SQB_K_MISC);
            sepal_kernel<<<(unsigned)ctas, SEPAL_T, smem, c->stream>>>(p);
            SQB_POST_LAUNCH();
        }
        SQB_CUDA(cudaMemcpyAsync(out, d_out.p, n_genes * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        SQB_CUDA(cudaStreamSynchronize(c->stream));
        return SQB_OK;
    };
    const int rc = body();
    if (rc != SQB_OK) cudaStreamSynchronize(c->stream);
    return rc;
}

extern "C" {

int sqb_sepal(sqb_ctx* ctx, const double* vals, int64_t n_genes, int64_t n, const int32_t* sat, int64_t n_sat, const int32_t* sat_idx,
              int max_neighs, const int32_t* unsat, const int32_t* unsat_idx, int64_t n_unsat, int n_iter, double dt, double thresh,
              double* out) {
    SQB_CHECK(ctx && vals && sat && sat_idx && out && (n_unsat == 0 || (unsat && unsat_idx)), SQB_ERR_INVALID, "sqb_sepal: null argument");
    SQB_TRY(sepal_check(sat, n_sat, sat_idx, max_neighs, unsat, unsat_idx, n_unsat, n_genes, n, n_iter));
    sqb_ctx* c = ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    DevBuf<double> d_vals;
    SQB_TRY(d_vals.alloc((size_t)n_genes * n));
    int rc = sqb_h2d(c, d_vals.p, vals, (size_t)n_genes * n * sizeof(double));
    if (rc == SQB_OK)
        rc = sepal_impl(c, d_vals.p, n_genes, n, sat, n_sat, sat_idx, max_neighs, unsat, unsat_idx, n_unsat, n_iter, dt, thresh, out);
    else
        cudaStreamSynchronize(c->stream);
    return rc;
}

int sqb_sepal_dense(const sqb_dense* x, const int32_t* sat, int64_t n_sat, const int32_t* sat_idx, int max_neighs, const int32_t* unsat,
                    const int32_t* unsat_idx, int64_t n_unsat, int n_iter, double dt, double thresh, double* out) {
    SQB_CHECK(x && sat && sat_idx && out && (n_unsat == 0 || (unsat && unsat_idx)), SQB_ERR_INVALID, "sqb_sepal_dense: null argument");
    SQB_CHECK(x->layout == 1 && x->dtype == 1, SQB_ERR_INVALID, "sqb_sepal_dense: expected a float64 genes x observations matrix");
    SQB_TRY(sepal_check(sat, n_sat, sat_idx, max_neighs, unsat, unsat_idx, n_unsat, x->n_genes, x->n_obs, n_iter));
    sqb_ctx* c = x->ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    return sepal_impl(c, reinterpret_cast<const double*>(x->buf.p), x->n_genes, x->n_obs, sat, n_sat, sat_idx, max_neighs, unsat, unsat_idx,
                      n_unsat, n_iter, dt, thresh, out);
}

}  // extern "C"
