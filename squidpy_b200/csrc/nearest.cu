// nearest.cu — exact distance from every query point to its nearest point of a reference set, on the GPU (sm_90a), for the
// three metric classes of scikit-learn's KDTree (euclidean, manhattan, chebyshev).
//
// Replaces `KDTree(anchor_coord, metric=DistanceMetric.get_metric(metric)).query(batch_coord)` of the reference's
// tl.var_by_distance (src/squidpy/tl/_var_by_distance.py:129-134).  Anchor sets are usually spatially coherent (a vessel, a
// region, a layer), so a search whose cost grows with the empty space between a query and the anchors (the grid ring walk of
// graph.cu) is the wrong structure here: this file builds a bounding-volume hierarchy per reference set instead.
//
// Layout.  Every reference set and every distinct query range is a "group".  Each point of a group gets a 32-bit Morton key of
// its position in the group's bounding box, with the group index above it; one cub radix sort orders all groups at once.  A
// reference set's sorted points are cut into leaves of NB_LEAF consecutive points; above them an implicit complete binary tree
// (heap numbering: root 1, children 2i and 2i + 1, the L leaves at L .. 2L - 1 with L a power of two, empty leaves padded with
// an empty box) stores the min / max of the exact coordinates below each node, built bottom-up.  Queries run one thread each,
// in the Morton order of their query range, so the lanes of a warp walk similar paths: nearer child first, a short stack of
// the farther children, a node pruned when its lower bound is >= the best distance so far.
//
// Exactness.  Distances are scikit-learn's reduced distances in float64: dx*dx + dy*dy without contraction (sqrt taken once at
// the end), |dx| + |dy|, max(|dx|, |dy|).  A box's lower bound combines the per-axis gaps max(x0 - qx, qx - x1, 0) the same way.
// Boxes hold exact point coordinates and rounded subtraction is monotone, so for every point p of a box the computed gap never
// exceeds the computed |p.x - qx|; products, sums and max are monotone too, so the bound never exceeds the computed distance of
// any point below the node and the pruning needs no slack.  Only the minimum value is returned: ties need no rule.
#include <algorithm>
#include <cmath>
#include <cub/device/device_radix_sort.cuh>
#include <map>
#include <vector>

#include "common.cuh"

#define NB_LEAF 16          // points per leaf
#define NB_THREADS 128      // queries per block
#define NB_STACK 32         // deferred nodes per query: one per tree level (n < 2^31 points: at most 27 levels above the leaves)

struct alignas(16) NbBox {
    double x0, y0, x1, y1;
};

// A group of the Morton sort: pool points begin .. begin + (entries of the group) at entries entry_off ..
struct NbGroup {
    double x0, y0, sx, sy;  // bounding box origin and the scale to [0, 65535] per axis
    int64_t begin, entry_off;
};

// A reference set: its sorted points are entries entry_off .. entry_off + m, its tree nodes node_off + 1 .. node_off + 2L - 1.
struct NbSet {
    int64_t entry_off, node_off, leaf_off;
    int32_t m, L;
};

// NB_THREADS consecutive sorted queries (entries e0 .. e0 + n) of one task against reference set `set`.
struct NbBlock {
    int32_t set, e0, n, pad;
    int64_t out_off;  // out[out_off + pool index]
};

__device__ __forceinline__ uint32_t nb_spread16(uint32_t v) {
    v &= 0xffffu;
    v = (v | (v << 8)) & 0x00ff00ffu;
    v = (v | (v << 4)) & 0x0f0f0f0fu;
    v = (v | (v << 2)) & 0x33333333u;
    v = (v | (v << 1)) & 0x55555555u;
    return v;
}

__device__ __forceinline__ uint32_t nb_quant(double v, double v0, double s) {
    const double t = (v - v0) * s;
    return t <= 0.0 ? 0u : t >= 65535.0 ? 65535u : (uint32_t)t;
}

__global__ void nb_key_kernel(const double2* __restrict__ pool, const NbGroup* __restrict__ groups, int n_groups, int64_t n_entries,
                              uint64_t* __restrict__ key, int32_t* __restrict__ idx) {
    const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (e >= n_entries) return;
    int lo = 0, hi = n_groups - 1;  // the last group whose entry_off <= e
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (groups[mid].entry_off <= e) lo = mid; else hi = mid - 1;
    }
    const NbGroup g = groups[lo];
    const int64_t i = g.begin + (e - g.entry_off);
    const double2 p = pool[i];
    const uint32_t m = nb_spread16(nb_quant(p.x, g.x0, g.sx)) | (nb_spread16(nb_quant(p.y, g.y0, g.sy)) << 1);
    key[e] = ((uint64_t)lo << 32) | m;
    idx[e] = (int32_t)i;
}

__global__ void nb_gather_kernel(const double2* __restrict__ pool, const int32_t* __restrict__ idx, int64_t n_entries, double2* __restrict__ sxy) {
    const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (e < n_entries) sxy[e] = pool[idx[e]];
}

// The set owning global leaf slot g (the sets' leaf slots are concatenated: set s owns leaf_off .. leaf_off + L).
__device__ __forceinline__ int nb_set_of_slot(const NbSet* __restrict__ sets, int n_sets, int64_t g) {
    int lo = 0, hi = n_sets - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (sets[mid].leaf_off <= g) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void nb_leaf_kernel(const double2* __restrict__ sxy, const NbSet* __restrict__ sets, int n_sets, int64_t n_slots,
                               NbBox* __restrict__ boxes) {
    const int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (g >= n_slots) return;
    const NbSet st = sets[nb_set_of_slot(sets, n_sets, g)];
    const int64_t j = g - st.leaf_off;
    NbBox b{INFINITY, INFINITY, -INFINITY, -INFINITY};  // an empty leaf: every bound is +inf, so it is always pruned
    const int64_t e1 = min((j + 1) * NB_LEAF, (int64_t)st.m);
    for (int64_t e = j * NB_LEAF; e < e1; ++e) {
        const double2 p = sxy[st.entry_off + e];
        b.x0 = fmin(b.x0, p.x), b.y0 = fmin(b.y0, p.y), b.x1 = fmax(b.x1, p.x), b.y1 = fmax(b.y1, p.y);
    }
    boxes[st.node_off + st.L + j] = b;
}

// Level `level` above the leaves: the node over leaf slots j .. j + 2^level of every set tall enough.
__global__ void nb_level_kernel(const NbSet* __restrict__ sets, int n_sets, int64_t n_slots, int level, NbBox* __restrict__ boxes) {
    const int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (g >= n_slots) return;
    const NbSet st = sets[nb_set_of_slot(sets, n_sets, g)];
    const int64_t j = g - st.leaf_off;
    if ((j & ((1LL << level) - 1)) != 0 || (st.L >> level) == 0) return;
    const int64_t node = (st.L + j) >> level;
    const NbBox a = boxes[st.node_off + 2 * node], c = boxes[st.node_off + 2 * node + 1];
    boxes[st.node_off + node] = NbBox{fmin(a.x0, c.x0), fmin(a.y0, c.y0), fmax(a.x1, c.x1), fmax(a.y1, c.y1)};
}

// scikit-learn's reduced distance of the metric from the coordinate differences (or box gaps) dx, dy.
template <int METRIC>
__device__ __forceinline__ double nb_rdist(double dx, double dy) {
    if (METRIC == 0) return __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
    if (METRIC == 1) return __dadd_rn(fabs(dx), fabs(dy));
    return fmax(fabs(dx), fabs(dy));
}

template <int METRIC>
__device__ __forceinline__ double nb_bound(const NbBox& b, double qx, double qy) {
    const double gx = fmax(fmax(__dsub_rn(b.x0, qx), __dsub_rn(qx, b.x1)), 0.0);
    const double gy = fmax(fmax(__dsub_rn(b.y0, qy), __dsub_rn(qy, b.y1)), 0.0);
    return nb_rdist<METRIC>(gx, gy);
}

template <int METRIC>
__global__ void __launch_bounds__(NB_THREADS) nb_query_kernel(const double2* __restrict__ sxy, const int32_t* __restrict__ idx,
                                                              const NbSet* __restrict__ sets, const NbBox* __restrict__ boxes,
                                                              const NbBlock* __restrict__ blocks, double* __restrict__ out) {
    const NbBlock blk = blocks[blockIdx.x];
    if ((int)threadIdx.x >= blk.n) return;
    const int64_t e = (int64_t)blk.e0 + threadIdx.x;
    const double2 q = sxy[e];
    const NbSet st = sets[blk.set];
    const NbBox* bx = boxes + st.node_off;
    const double2* pts = sxy + st.entry_off;
    int stack[NB_STACK];
    int sp = 0;
    int node = 1;
    double best = INFINITY;
    for (;;) {
        if (node >= st.L) {  // a leaf: its points are NB_LEAF consecutive sorted entries
            const int p0 = (node - st.L) * NB_LEAF, p1 = min(p0 + NB_LEAF, st.m);
            for (int p = p0; p < p1; ++p) {
                const double2 r = pts[p];
                best = fmin(best, nb_rdist<METRIC>(__dsub_rn(q.x, r.x), __dsub_rn(q.y, r.y)));
            }
        } else {
            const double la = nb_bound<METRIC>(bx[2 * node], q.x, q.y), lb = nb_bound<METRIC>(bx[2 * node + 1], q.x, q.y);
            const int near = la <= lb ? 2 * node : 2 * node + 1;
            const double lnear = la <= lb ? la : lb, lfar = la <= lb ? lb : la;
            if (lfar < best) stack[sp++] = near ^ 1;
            if (lnear < best) {
                node = near;
                continue;
            }
        }
        node = 0;
        while (sp > 0) {
            const int n = stack[--sp];
            if (nb_bound<METRIC>(bx[n], q.x, q.y) < best) {
                node = n;
                break;
            }
        }
        if (node == 0) break;
    }
    out[blk.out_off + idx[e]] = METRIC == 0 ? sqrt(best) : best;
}

template <int METRIC>
static int nb_query_launch(sqb_ctx* c, int64_t nblk, const double2* sxy, const int32_t* idx, const NbSet* sets, const NbBox* boxes,
                           const NbBlock* blocks, double* out) {
    SqbLaunchScope scope(c, SQB_K_MISC);
    nb_query_kernel<METRIC><<<(unsigned)nblk, NB_THREADS, 0, c->stream>>>(sxy, idx, sets, boxes, blocks, out);
    SQB_POST_LAUNCH();
    return SQB_OK;
}

// Bounding box of pool points [b, e) and the Morton scale of the group.
static NbGroup nb_group(const double* pts, int64_t b, int64_t e, int64_t entry_off) {
    double x0 = INFINITY, y0 = INFINITY, x1 = -INFINITY, y1 = -INFINITY;
    for (int64_t i = b; i < e; ++i) {
        const double x = pts[2 * i], y = pts[2 * i + 1];
        x0 = std::min(x0, x), x1 = std::max(x1, x), y0 = std::min(y0, y), y1 = std::max(y1, y);
    }
    NbGroup g;
    g.x0 = x0, g.y0 = y0;
    g.sx = x1 > x0 ? 65535.0 / (x1 - x0) : 0.0;
    g.sy = y1 > y0 ? 65535.0 / (y1 - y0) : 0.0;
    if (!std::isfinite(g.sx)) g.sx = 0.0;  // an extent too small to invert: every point in one Morton cell (order only)
    if (!std::isfinite(g.sy)) g.sy = 0.0;
    g.begin = b, g.entry_off = entry_off;
    return g;
}

extern "C" {

int sqb_nn_min_dist_f64(sqb_ctx* ctx, const double* pts, int64_t n_pts, const int64_t* tasks, int64_t n_tasks, int metric, int64_t n_out,
                        double* out) {
    SQB_CHECK(ctx && (pts || n_pts == 0) && (tasks || n_tasks == 0) && (out || n_out == 0), SQB_ERR_INVALID, "sqb_nn_min_dist_f64: null argument");
    SQB_CHECK(n_pts >= 0 && n_pts < 2147483648LL, SQB_ERR_INVALID, "sqb_nn_min_dist_f64: n_pts=%lld outside [0, 2^31)", (long long)n_pts);
    SQB_CHECK(n_tasks >= 0 && n_out >= 0, SQB_ERR_INVALID, "sqb_nn_min_dist_f64: negative n_tasks or n_out");
    SQB_CHECK(metric >= 0 && metric <= 2, SQB_ERR_INVALID, "sqb_nn_min_dist_f64: metric=%d is not 0 (euclidean), 1 (manhattan) or 2 (chebyshev)",
              metric);
    for (int64_t i = 0; i < n_pts; ++i)
        SQB_CHECK(std::isfinite(pts[2 * i]) && std::isfinite(pts[2 * i + 1]), SQB_ERR_INVALID, "sqb_nn_min_dist_f64: point %lld is not finite",
                  (long long)i);
    // groups: the distinct reference ranges (sets), then the distinct query ranges
    std::map<std::pair<int64_t, int64_t>, int> set_of, qry_of;
    std::vector<std::pair<int64_t, int64_t>> set_rng, qry_rng, out_rng;
    std::vector<int> task_set(n_tasks), task_qry(n_tasks);
    for (int64_t t = 0; t < n_tasks; ++t) {
        const int64_t* tk = tasks + 5 * t;
        const int64_t rb = tk[0], re = tk[1], qb = tk[2], qe = tk[3], ob = tk[4];
        SQB_CHECK(0 <= rb && rb <= re && re <= n_pts && 0 <= qb && qb <= qe && qe <= n_pts, SQB_ERR_INVALID,
                  "sqb_nn_min_dist_f64: task %lld has a range outside [0, %lld]", (long long)t, (long long)n_pts);
        SQB_CHECK(re > rb, SQB_ERR_INVALID, "sqb_nn_min_dist_f64: task %lld has an empty reference range", (long long)t);
        SQB_CHECK(0 <= ob && ob <= n_out - (qe - qb), SQB_ERR_INVALID, "sqb_nn_min_dist_f64: task %lld writes outside [0, %lld)", (long long)t,
                  (long long)n_out);
        if (qe > qb) out_rng.push_back({ob, ob + (qe - qb)});
        auto s = set_of.emplace(std::make_pair(rb, re), (int)set_rng.size());
        if (s.second) set_rng.push_back({rb, re});
        task_set[t] = s.first->second;
        auto q = qry_of.emplace(std::make_pair(qb, qe), (int)qry_rng.size());
        if (q.second) qry_rng.push_back({qb, qe});
        task_qry[t] = q.first->second;
    }
    std::sort(out_rng.begin(), out_rng.end());
    for (size_t i = 1; i < out_rng.size(); ++i)
        SQB_CHECK(out_rng[i].first >= out_rng[i - 1].second, SQB_ERR_INVALID, "sqb_nn_min_dist_f64: output ranges overlap at %lld",
                  (long long)out_rng[i].first);
    // positions no task writes are NaN
    {
        int64_t pos = 0;
        for (const auto& r : out_rng) {
            std::fill(out + pos, out + r.first, NAN);
            pos = r.second;
        }
        std::fill(out + pos, out + n_out, NAN);
    }
    const int n_sets = (int)set_rng.size();
    std::vector<NbGroup> groups;
    std::vector<NbSet> sets(n_sets);
    int64_t n_entries = 0, n_slots = 0, n_nodes = 0;
    int max_level = 0;
    for (int s = 0; s < n_sets; ++s) {
        const int64_t m = set_rng[s].second - set_rng[s].first;
        groups.push_back(nb_group(pts, set_rng[s].first, set_rng[s].second, n_entries));
        int64_t L = 1;
        int lev = 0;
        while (L * NB_LEAF < m) L <<= 1, ++lev;
        sets[s].entry_off = n_entries, sets[s].node_off = n_nodes, sets[s].leaf_off = n_slots;
        sets[s].m = (int32_t)m, sets[s].L = (int32_t)L;
        n_entries += m, n_slots += L, n_nodes += 2 * L;
        max_level = std::max(max_level, lev);
    }
    std::vector<int64_t> qry_entry(qry_rng.size());
    for (size_t r = 0; r < qry_rng.size(); ++r) {
        groups.push_back(nb_group(pts, qry_rng[r].first, qry_rng[r].second, n_entries));
        qry_entry[r] = n_entries;
        n_entries += qry_rng[r].second - qry_rng[r].first;
    }
    SQB_CHECK(n_entries < 2147483648LL, SQB_ERR_UNSUPPORTED, "sqb_nn_min_dist_f64: %lld reference and query points do not fit int32",
              (long long)n_entries);
    std::vector<NbBlock> blocks;
    for (int64_t t = 0; t < n_tasks; ++t) {
        const int64_t* tk = tasks + 5 * t;
        const int64_t nq = tk[3] - tk[2];
        for (int64_t i = 0; i < nq; i += NB_THREADS) {
            NbBlock b;
            b.set = task_set[t], b.e0 = (int32_t)(qry_entry[task_qry[t]] + i), b.n = (int32_t)std::min<int64_t>(NB_THREADS, nq - i), b.pad = 0;
            b.out_off = tk[4] - tk[2];
            blocks.push_back(b);
        }
    }
    if (blocks.empty()) return SQB_OK;
    sqb_ctx* c = ctx;
    SQB_CUDA(cudaSetDevice(c->device));
    const int n_groups = (int)groups.size();
    DevBuf<double> d_pool(c->stream), d_out(c->stream);
    DevBuf<NbGroup> d_groups(c->stream);
    DevBuf<NbSet> d_sets(c->stream);
    DevBuf<NbBlock> d_blocks(c->stream);
    DevBuf<NbBox> d_boxes(c->stream);
    DevBuf<double2> d_sxy(c->stream);
    DevBuf<int32_t> d_idx(c->stream);
    SQB_TRY(d_pool.alloc(2 * (size_t)n_pts));
    SQB_TRY(d_out.alloc((size_t)n_out));
    SQB_TRY(d_groups.alloc(n_groups));
    SQB_TRY(d_sets.alloc(n_sets));
    SQB_TRY(d_blocks.alloc(blocks.size()));
    SQB_TRY(d_boxes.alloc((size_t)n_nodes));
    SQB_TRY(d_sxy.alloc((size_t)n_entries));
    SQB_TRY(d_idx.alloc((size_t)n_entries));
    SQB_TRY(sqb_h2d(c, d_pool.p, pts, 2 * (size_t)n_pts * sizeof(double)));
    SQB_CUDA(cudaMemcpyAsync(d_groups.p, groups.data(), n_groups * sizeof(NbGroup), cudaMemcpyHostToDevice, c->stream));
    SQB_CUDA(cudaMemcpyAsync(d_sets.p, sets.data(), n_sets * sizeof(NbSet), cudaMemcpyHostToDevice, c->stream));
    SQB_CUDA(cudaMemcpyAsync(d_blocks.p, blocks.data(), blocks.size() * sizeof(NbBlock), cudaMemcpyHostToDevice, c->stream));
    const double2* pool = reinterpret_cast<const double2*>(d_pool.p);
    const unsigned eb = (unsigned)ceil_div64(n_entries, 256);
    {  // Morton sort of every group at once
        DevBuf<uint64_t> key_a(c->stream), key_b(c->stream);
        DevBuf<int32_t> idx_a(c->stream);
        DevBuf<uint8_t> tmp(c->stream);
        SQB_TRY(key_a.alloc((size_t)n_entries));
        SQB_TRY(key_b.alloc((size_t)n_entries));
        SQB_TRY(idx_a.alloc((size_t)n_entries));
        {
            SqbLaunchScope scope(c, SQB_K_MISC);
            nb_key_kernel<<<eb, 256, 0, c->stream>>>(pool, d_groups.p, n_groups, n_entries, key_a.p, idx_a.p);
            SQB_POST_LAUNCH();
        }
        int bits = 1;
        while (bits < 31 && ((uint64_t)(n_groups - 1) >> bits) != 0) ++bits;
        size_t tmp_bytes = 0;
        SQB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, key_a.p, key_b.p, idx_a.p, d_idx.p, (int)n_entries, 0, 32 + bits, c->stream));
        SQB_TRY(tmp.alloc(tmp_bytes > 0 ? tmp_bytes : 1));
        SQB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, key_a.p, key_b.p, idx_a.p, d_idx.p, (int)n_entries, 0, 32 + bits, c->stream));
        c->launches += 1;
    }
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        nb_gather_kernel<<<eb, 256, 0, c->stream>>>(pool, d_idx.p, n_entries, d_sxy.p);
        SQB_POST_LAUNCH();
    }
    const unsigned sb = (unsigned)ceil_div64(n_slots, 256);
    {
        SqbLaunchScope scope(c, SQB_K_MISC);
        nb_leaf_kernel<<<sb, 256, 0, c->stream>>>(d_sxy.p, d_sets.p, n_sets, n_slots, d_boxes.p);
        SQB_POST_LAUNCH();
    }
    for (int level = 1; level <= max_level; ++level) {
        SqbLaunchScope scope(c, SQB_K_MISC);
        nb_level_kernel<<<sb, 256, 0, c->stream>>>(d_sets.p, n_sets, n_slots, level, d_boxes.p);
        SQB_POST_LAUNCH();
    }
    const int64_t nblk = (int64_t)blocks.size();
    if (metric == 0)
        SQB_TRY(nb_query_launch<0>(c, nblk, d_sxy.p, d_idx.p, d_sets.p, d_boxes.p, d_blocks.p, d_out.p));
    else if (metric == 1)
        SQB_TRY(nb_query_launch<1>(c, nblk, d_sxy.p, d_idx.p, d_sets.p, d_boxes.p, d_blocks.p, d_out.p));
    else
        SQB_TRY(nb_query_launch<2>(c, nblk, d_sxy.p, d_idx.p, d_sets.p, d_boxes.p, d_blocks.p, d_out.p));
    for (const auto& r : out_rng)
        SQB_CUDA(cudaMemcpyAsync(out + r.first, d_out.p + r.first, (size_t)(r.second - r.first) * sizeof(double), cudaMemcpyDeviceToHost,
                                 c->stream));
    SQB_CUDA(cudaStreamSynchronize(c->stream));
    return SQB_OK;
}

}  // extern "C"
