// delaunay.cuh — the Delaunay triangulation of delaunay.cu, shared with the device-coordinate builder of graph_device.cu.
#pragma once
#include "graph.cuh"

// Points per cell of the grid the triangulation walks.
constexpr double DT_PTS_PER_CELL = 2.5;
// The Delaunay graph of the n points bucketed in g (grid sized with DT_PTS_PER_CELL): indptr (n + 1) and the ascending
// neighbours of every row in idx (*nnz entries).  QhullError-style SQB_ERR_INVALID when fewer than three distinct points or
// all distinct points collinear.  pass_counts (host int64[2], or null): points finished by pass 1 and by pass 2.
int delaunay_csr(sqb_ctx* c, PointGrid& g, int64_t n, DevBuf<int64_t>& indptr, DevBuf<int32_t>& idx, int64_t* nnz, int64_t* pass_counts);
// dist[t] = |xy[i] - xy[idx[t]]| for the entries of row i, computed in float32 (f32) or float64 like numpy's norm.
int delaunay_dist(sqb_ctx* c, const double* xy, const int64_t* indptr, const int32_t* idx, int64_t n, bool f32, double* dist);
