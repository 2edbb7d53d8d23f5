// K1 radius-graph build, CSR helpers, K2 edge features.
//
// Radius graph: one warp per target agent; the 32 lanes sweep the sources of the agent's own graph in
// ascending order, a ballot + popc gives each hit its rank, so the output is (target asc, source asc)
// without any sort and without atomics.  Positions are read straight from the state rows (coalesced,
// L2-resident: a 4096+128-node graph is 68 KB).  Bit-exactness against the CPU reference:
//   metric 0 (SimpleCar -> torch_cluster.radius_graph, reference gcbf/env/simple_car.py:32-33,249-252):
//       d2 = 0; d2 = d2 + (dx*dx) for each dim, NO fma contraction;  hit = d2 < r*r
//   metric 1 (DubinsCar / SimpleDrone, gcbf/env/dubins_car.py:730-746, simple_drone.py:316-333):
//       torch.norm on CPU accumulates acc = fma(d, d, acc) per dim, then sqrt (measured against torch
//       2.11 CPU: 0 mismatches in 4e6 pairs);  hit = sqrtf(acc) < r, diagonal excluded.
// The pair rule and the edge-feature map g(s) live in graph_core.h (shared with the probe graphs of field.cu).
#include "common.cuh"
#include "graph_core.h"

namespace gcbf {

using graph::pair_hit;
using graph::edge_feat;

template <bool FILL>
__global__ void radius_graph_kernel(const float* __restrict__ states, int ld, int pos_dim, int num_graphs, int N,
                                    int n, float r, int metric, int32_t* __restrict__ counts,
                                    const int32_t* __restrict__ rowptr, int64_t* __restrict__ edge_index,
                                    int64_t E) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= num_graphs * n) return;
  const int g = warp / n, il = warp % n;
  const int64_t base = (int64_t)g * N;
  float pi[3] = {0.f, 0.f, 0.f};
  for (int d = 0; d < pos_dim; ++d) pi[d] = __ldg(states + (base + il) * ld + d);
  const float r2 = __fmul_rn(r, r);
  int total = 0;
  int64_t out = FILL ? (int64_t)rowptr[warp] : 0;
  for (int j0 = 0; j0 < N; j0 += 32) {
    const int j = j0 + lane;
    bool hit = false;
    if (j < N && j != il) {
      float pj[3] = {0.f, 0.f, 0.f};
      for (int d = 0; d < pos_dim; ++d) pj[d] = __ldg(states + (base + j) * ld + d);
      hit = pair_hit(pi, pj, pos_dim, r, r2, metric);
    }
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (FILL) {
      if (hit) {
        const int64_t pos = out + __popc(m & ((1u << lane) - 1u));
        edge_index[pos] = base + j;           // source j
        edge_index[E + pos] = base + il;      // target i
      }
      out += __popc(m);
    } else {
      total += __popc(m);
    }
  }
  if (!FILL && lane == 0) counts[warp] = total;
}

// single-block exclusive scan of `count` int32 values (in place: data[i] <- sum_{k<i}, data[count] <- total)
__global__ void exclusive_scan_kernel(int32_t* __restrict__ data, int count) {
  __shared__ int32_t warp_tot[32];
  __shared__ int32_t carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int base = 0; base < count; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const int32_t v = (i < count) ? data[i] : 0;
    int32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int32_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_tot[wid] = x;
    __syncthreads();
    if (wid == 0) {
      int32_t t = (lane < (int)(blockDim.x >> 5)) ? warp_tot[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int32_t y = __shfl_up_sync(0xffffffffu, t, o);
        if (lane >= o) t += y;
      }
      warp_tot[lane] = t;  // inclusive scan of warp totals
    }
    __syncthreads();
    const int32_t carry = carry_s;
    const int32_t warp_off = (wid == 0) ? 0 : warp_tot[wid - 1];
    if (i < count) data[i] = carry + warp_off + x - v;
    __syncthreads();
    if (threadIdx.x == 0) carry_s = carry + warp_tot[(blockDim.x >> 5) - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) data[count] = carry_s;
}

cudaError_t exclusive_scan_i32(int32_t* data, int count, cudaStream_t st) {
  exclusive_scan_kernel<<<1, 1024, 0, st>>>(data, count);
  return cudaGetLastError();
}

// rowptr[i] = first edge e with dst[e] >= i  (binary search; dst is non-decreasing)
__global__ void rowptr_kernel(const int64_t* __restrict__ dst, int64_t E, int num_nodes, int32_t* __restrict__ rowptr,
                              int32_t* __restrict__ unsorted_flag) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= num_nodes) {
    int64_t lo = 0, hi = E;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (dst[mid] < i) lo = mid + 1; else hi = mid;
    }
    rowptr[i] = (int32_t)lo;
  }
  // sortedness / range check, grid-stride over edges
  for (int64_t e = i; e < E; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t d = dst[e];
    if (d < 0 || d >= num_nodes || (e + 1 < E && dst[e + 1] < d)) *unsorted_flag = 1;
  }
}

template <int ENV, int SD, int ED>
__global__ void edge_attr_fwd_kernel(const float* __restrict__ states, int ld, const int64_t* __restrict__ ei,
                                     int64_t E, float* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int64_t src = ei[e], dst = ei[E + e];
  float ss[SD], sd[SD], fs[ED], fd[ED];
#pragma unroll
  for (int k = 0; k < SD; ++k) { ss[k] = __ldg(states + src * ld + k); sd[k] = __ldg(states + dst * ld + k); }
  edge_feat<ENV>(ss, fs);
  edge_feat<ENV>(sd, fd);
#pragma unroll
  for (int k = 0; k < ED; ++k) out[e * ED + k] = __fsub_rn(fs[k], fd[k]);
}

// d_states[src] += J_g(s_src)^T d_e ; d_states[dst] -= J_g(s_dst)^T d_e
template <int ENV, int SD, int ED>
__global__ void edge_attr_bwd_kernel(const float* __restrict__ states, int ld, const int64_t* __restrict__ ei,
                                     int64_t E, const float* __restrict__ d_e, float* __restrict__ d_states) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int64_t node[2] = {ei[e], ei[E + e]};
  float g[ED];
#pragma unroll
  for (int k = 0; k < ED; ++k) g[k] = d_e[e * ED + k];
#pragma unroll
  for (int side = 0; side < 2; ++side) {
    const float sgn = side == 0 ? 1.f : -1.f;
    float ds[SD];
    if (ENV == GCBF_ENV_DUBINS_CAR) {
      const float th = __ldg(states + node[side] * ld + 2), v = __ldg(states + node[side] * ld + 3);
      const float c = cosf(th), s = sinf(th);
      ds[0] = g[0]; ds[1] = g[1];
      ds[2] = g[2] + g[3] * (-v * s) + g[4] * (v * c);
      ds[3] = g[3] * c + g[4] * s;
    } else {
#pragma unroll
      for (int k = 0; k < SD; ++k) ds[k] = g[k];
    }
#pragma unroll
    for (int k = 0; k < SD; ++k) atomicAdd(d_states + node[side] * ld + k, sgn * ds[k]);
  }
}

__global__ void edge_input_kernel(const float* __restrict__ x, int node_dim, const float* __restrict__ ea, int edge_dim,
                                  const int64_t* __restrict__ ei, int64_t E, float* __restrict__ out, int ld_out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t e = idx / ld_out;
  const int c = (int)(idx % ld_out);
  if (e >= E) return;
  float v = 0.f;
  if (c < node_dim) v = __ldg(x + ei[E + e] * node_dim + c);                       // x_i (target)
  else if (c < 2 * node_dim) v = __ldg(x + ei[e] * node_dim + (c - node_dim));     // x_j (source)
  else if (c < 2 * node_dim + edge_dim) v = ea[e * edge_dim + (c - 2 * node_dim)];
  out[idx] = v;
}

}  // namespace gcbf

using namespace gcbf;

extern "C" int gcbf_radius_graph_count(const float* states, int ld_state, int pos_dim, int num_graphs,
                                       int nodes_per_graph, int num_agents, float radius, int metric,
                                       int32_t* rowptr, void* stream) {
  GCBF_REQUIRE(states && rowptr, "gcbf_radius_graph_count: null pointer");
  GCBF_REQUIRE(pos_dim >= 1 && pos_dim <= 3 && ld_state >= pos_dim, "gcbf_radius_graph_count: pos_dim=%d ld=%d", pos_dim, ld_state);
  GCBF_REQUIRE(num_graphs >= 0 && nodes_per_graph >= num_agents && num_agents >= 0, "gcbf_radius_graph_count: bad sizes");
  GCBF_REQUIRE(metric == 0 || metric == 1, "gcbf_radius_graph_count: metric %d", metric);
  cudaStream_t st = as_stream(stream);
  const int64_t na = (int64_t)num_graphs * num_agents;
  GCBF_REQUIRE(na < (1ll << 31), "gcbf_radius_graph_count: too many agents");
  if (na > 0) {
    radius_graph_kernel<false><<<ceil_div(na * 32, 256), 256, 0, st>>>(states, ld_state, pos_dim, num_graphs,
                                                                      nodes_per_graph, num_agents, radius, metric,
                                                                      rowptr, nullptr, nullptr, 0);
    GCBF_LAUNCH_OK();
  }
  exclusive_scan_kernel<<<1, 1024, 0, st>>>(rowptr, (int)na);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

extern "C" int gcbf_radius_graph_fill(const float* states, int ld_state, int pos_dim, int num_graphs,
                                      int nodes_per_graph, int num_agents, float radius, int metric,
                                      const int32_t* rowptr, int64_t* edge_index, int64_t num_edges, void* stream) {
  GCBF_REQUIRE(states && rowptr && (edge_index || num_edges == 0), "gcbf_radius_graph_fill: null pointer");
  GCBF_REQUIRE(pos_dim >= 1 && pos_dim <= 3 && (metric == 0 || metric == 1), "gcbf_radius_graph_fill: bad pos_dim/metric");
  const int64_t na = (int64_t)num_graphs * num_agents;
  if (na == 0 || num_edges == 0) return GCBF_OK;
  radius_graph_kernel<true><<<ceil_div(na * 32, 256), 256, 0, as_stream(stream)>>>(
      states, ld_state, pos_dim, num_graphs, nodes_per_graph, num_agents, radius, metric, nullptr, rowptr,
      edge_index, num_edges);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

extern "C" int gcbf_rowptr_from_targets(const int64_t* edge_dst, int64_t num_edges, int num_nodes, int32_t* rowptr,
                                        int32_t* unsorted_flag, void* stream) {
  GCBF_REQUIRE(rowptr && unsorted_flag && (edge_dst || num_edges == 0) && num_nodes >= 0, "gcbf_rowptr_from_targets: bad arguments");
  GCBF_REQUIRE(num_edges < (1ll << 31), "gcbf_rowptr_from_targets: E too large for int32 CSR");
  cudaStream_t st = as_stream(stream);
  GCBF_CUDA_OK(cudaMemsetAsync(unsorted_flag, 0, sizeof(int32_t), st));
  const int64_t work = imax64(num_nodes + 1, imin64(num_edges, 1 << 20));
  rowptr_kernel<<<ceil_div(work, 256), 256, 0, st>>>(edge_dst, num_edges, num_nodes, rowptr, unsorted_flag);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

extern "C" int gcbf_edge_attr_fwd(int env, const float* states, int ld_state, const int64_t* edge_index,
                                  int64_t num_edges, float* edge_attr, void* stream) {
  GCBF_REQUIRE(states && (num_edges == 0 || (edge_index && edge_attr)), "gcbf_edge_attr_fwd: null pointer");
  if (num_edges == 0) return GCBF_OK;
  cudaStream_t st = as_stream(stream);
  const int grid = ceil_div(num_edges, 256);
  switch (env) {
    case GCBF_ENV_SIMPLE_CAR: edge_attr_fwd_kernel<GCBF_ENV_SIMPLE_CAR, 4, 4><<<grid, 256, 0, st>>>(states, ld_state, edge_index, num_edges, edge_attr); break;
    case GCBF_ENV_DUBINS_CAR: edge_attr_fwd_kernel<GCBF_ENV_DUBINS_CAR, 4, 5><<<grid, 256, 0, st>>>(states, ld_state, edge_index, num_edges, edge_attr); break;
    case GCBF_ENV_SIMPLE_DRONE: edge_attr_fwd_kernel<GCBF_ENV_SIMPLE_DRONE, 6, 6><<<grid, 256, 0, st>>>(states, ld_state, edge_index, num_edges, edge_attr); break;
    default: GCBF_REQUIRE(false, "gcbf_edge_attr_fwd: unknown env %d", env);
  }
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

namespace gcbf {

// Deterministic form of the same scatter for callers that know the node count: every edge writes its two contributions to
// scratch, then one thread per node adds them in edge order -- target side from the node's contiguous run of the (target-sorted)
// edge list, source side from a counting sort of the edges by source -- so d_states does not depend on the order edges run in.
template <int ENV, int SD, int ED>
__global__ void edge_attr_contrib_kernel(const float* __restrict__ states, int ld, const int64_t* __restrict__ ei, int64_t E,
                                         const float* __restrict__ d_e, float* __restrict__ contrib, int32_t* __restrict__ src_count) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int64_t node[2] = {ei[e], ei[E + e]};
  float g[ED];
#pragma unroll
  for (int k = 0; k < ED; ++k) g[k] = d_e[e * ED + k];
#pragma unroll
  for (int side = 0; side < 2; ++side) {
    const float sgn = side == 0 ? 1.f : -1.f;
    float ds[SD];
    if (ENV == GCBF_ENV_DUBINS_CAR) {
      const float th = __ldg(states + node[side] * ld + 2), v = __ldg(states + node[side] * ld + 3);
      const float c = cosf(th), s = sinf(th);
      ds[0] = g[0]; ds[1] = g[1];
      ds[2] = g[2] + g[3] * (-v * s) + g[4] * (v * c);
      ds[3] = g[3] * c + g[4] * s;
    } else {
#pragma unroll
      for (int k = 0; k < SD; ++k) ds[k] = g[k];
    }
#pragma unroll
    for (int k = 0; k < SD; ++k) contrib[(side * E + e) * SD + k] = sgn * ds[k];
  }
  atomicAdd(src_count + node[0], 1);
}

__global__ void edge_src_fill_kernel(const int64_t* __restrict__ ei, int64_t E, int32_t* __restrict__ cursor, int32_t* __restrict__ ids) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < E) ids[atomicAdd(cursor + ei[e], 1)] = (int32_t)e;
}

template <int SD>
__global__ void edge_attr_gather_kernel(const int64_t* __restrict__ ei, int64_t E, int num_nodes, const float* __restrict__ contrib,
                                        const int32_t* __restrict__ src_off, int32_t* __restrict__ ids, float* __restrict__ d_states, int ld) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= num_nodes) return;
  float acc[SD];
#pragma unroll
  for (int k = 0; k < SD; ++k) acc[k] = 0.f;
  // source side: this node's edges in ascending edge order (the fill order above is arbitrary)
  const int b = src_off[n], t = src_off[n + 1];
  for (int i = b + 1; i < t; ++i) {
    const int32_t v = ids[i];
    int j = i - 1;
    while (j >= b && ids[j] > v) { ids[j + 1] = ids[j]; --j; }
    ids[j + 1] = v;
  }
  for (int i = b; i < t; ++i)
#pragma unroll
    for (int k = 0; k < SD; ++k) acc[k] += contrib[(int64_t)ids[i] * SD + k];
  // target side: the contiguous run of edges whose target is n
  const int64_t* dst = ei + E;
  int64_t lo = 0, hi = E;
  while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (dst[mid] < n) lo = mid + 1; else hi = mid; }
  for (int64_t e = lo; e < E && dst[e] == n; ++e)
#pragma unroll
    for (int k = 0; k < SD; ++k) acc[k] += contrib[(E + e) * SD + k];
#pragma unroll
  for (int k = 0; k < SD; ++k) d_states[(int64_t)n * ld + k] += acc[k];
}

template <int ENV, int SD, int ED>
static int edge_attr_bwd_ordered_t(const float* states, int ld, const int64_t* ei, int64_t E, int num_nodes, const float* d_e,
                                   float* d_states, cudaStream_t st) {
  // scratch: contributions [2][E][SD] floats, source offsets [N + 1], fill cursors [N], edge ids [E]
  const size_t cbytes = (size_t)2 * E * SD * 4, obytes = ((size_t)num_nodes + 1) * 4;
  uint8_t* buf = nullptr;
  GCBF_CUDA_OK(scratch_alloc((void**)&buf, cbytes + 2 * obytes + (size_t)E * 4, st));
  float* contrib = reinterpret_cast<float*>(buf);
  int32_t* off = reinterpret_cast<int32_t*>(buf + cbytes);
  int32_t* cursor = reinterpret_cast<int32_t*>(buf + cbytes + obytes);
  int32_t* ids = reinterpret_cast<int32_t*>(buf + cbytes + 2 * obytes);
  GCBF_CUDA_OK(cudaMemsetAsync(off, 0, obytes, st));
  edge_attr_contrib_kernel<ENV, SD, ED><<<ceil_div(E, 256), 256, 0, st>>>(states, ld, ei, E, d_e, contrib, off);
  GCBF_LAUNCH_OK();
  GCBF_CUDA_OK(exclusive_scan_i32(off, num_nodes, st));
  GCBF_CUDA_OK(cudaMemcpyAsync(cursor, off, (size_t)num_nodes * 4, cudaMemcpyDeviceToDevice, st));
  edge_src_fill_kernel<<<ceil_div(E, 256), 256, 0, st>>>(ei, E, cursor, ids);
  GCBF_LAUNCH_OK();
  edge_attr_gather_kernel<SD><<<ceil_div(num_nodes, 128), 128, 0, st>>>(ei, E, num_nodes, contrib, off, ids, d_states, ld);
  GCBF_LAUNCH_OK();
  GCBF_CUDA_OK(scratch_free(buf, st));
  return GCBF_OK;
}

int edge_attr_bwd_ordered(int env, const float* states, int ld_state, const int64_t* edge_index, int64_t num_edges, int num_nodes,
                          const float* d_edge_attr, float* d_states, cudaStream_t st) {
  if (num_edges == 0) return GCBF_OK;
  switch (env) {
    case GCBF_ENV_SIMPLE_CAR: return edge_attr_bwd_ordered_t<GCBF_ENV_SIMPLE_CAR, 4, 4>(states, ld_state, edge_index, num_edges, num_nodes, d_edge_attr, d_states, st);
    case GCBF_ENV_DUBINS_CAR: return edge_attr_bwd_ordered_t<GCBF_ENV_DUBINS_CAR, 4, 5>(states, ld_state, edge_index, num_edges, num_nodes, d_edge_attr, d_states, st);
    case GCBF_ENV_SIMPLE_DRONE: return edge_attr_bwd_ordered_t<GCBF_ENV_SIMPLE_DRONE, 6, 6>(states, ld_state, edge_index, num_edges, num_nodes, d_edge_attr, d_states, st);
    default: set_error("edge_attr_bwd_ordered: unknown env %d", env); return GCBF_E_INVALID;
  }
}

}  // namespace gcbf

extern "C" int gcbf_edge_attr_bwd(int env, const float* states, int ld_state, const int64_t* edge_index,
                                  int64_t num_edges, const float* d_edge_attr, float* d_states, void* stream) {
  GCBF_REQUIRE(states && d_states && (num_edges == 0 || (edge_index && d_edge_attr)), "gcbf_edge_attr_bwd: null pointer");
  if (num_edges == 0) return GCBF_OK;
  cudaStream_t st = as_stream(stream);
  const int grid = ceil_div(num_edges, 256);
  switch (env) {
    case GCBF_ENV_SIMPLE_CAR: edge_attr_bwd_kernel<GCBF_ENV_SIMPLE_CAR, 4, 4><<<grid, 256, 0, st>>>(states, ld_state, edge_index, num_edges, d_edge_attr, d_states); break;
    case GCBF_ENV_DUBINS_CAR: edge_attr_bwd_kernel<GCBF_ENV_DUBINS_CAR, 4, 5><<<grid, 256, 0, st>>>(states, ld_state, edge_index, num_edges, d_edge_attr, d_states); break;
    case GCBF_ENV_SIMPLE_DRONE: edge_attr_bwd_kernel<GCBF_ENV_SIMPLE_DRONE, 6, 6><<<grid, 256, 0, st>>>(states, ld_state, edge_index, num_edges, d_edge_attr, d_states); break;
    default: GCBF_REQUIRE(false, "gcbf_edge_attr_bwd: unknown env %d", env);
  }
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

extern "C" int gcbf_edge_input_fwd(const float* x, int node_dim, const float* edge_attr, int edge_dim,
                                   const int64_t* edge_index, int64_t num_edges, float* out, int ld_out, void* stream) {
  GCBF_REQUIRE(ld_out >= 2 * node_dim + edge_dim, "gcbf_edge_input_fwd: ld_out %d too small", ld_out);
  GCBF_REQUIRE(num_edges == 0 || (x && edge_attr && edge_index && out), "gcbf_edge_input_fwd: null pointer");
  if (num_edges == 0) return GCBF_OK;
  edge_input_kernel<<<ceil_div(num_edges * ld_out, 256), 256, 0, as_stream(stream)>>>(x, node_dim, edge_attr, edge_dim,
                                                                                     edge_index, num_edges, out, ld_out);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}
