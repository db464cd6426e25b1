// Batch structure kernels: graph offsets of a PyG-collated batch and the per-node message-passing
// adjacency (incoming / outgoing edge lists sorted by (edge_type, neighbour)).
//
// The reference hands RGCNConv a flat [2,E] edge_index and lets torch-scatter do an atomic
// scatter-mean per layer (third-party PyG 1.4.2; call site models.py:201).  Here the batch is turned
// ONCE per step into a destination-sorted CSR that all 4 forward and 4 backward layer passes reuse
// as a deterministic segment-reduce (no float atomics anywhere).
#include "common.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int BP_THREADS = 1024;

// node_ptr[b] = first node with batch >= b ; edge_ptr[b] = first edge whose source lies in graph >= b.  A batch id
// outside [0, B) or below its predecessor, and an edge source outside [0, N) or in a graph before its predecessor's,
// set IGMC_ERR_BAD_BATCH (node_ptr / edge_ptr are then undefined).
__global__ void k_batch_ptrs(const int64_t* __restrict__ batch, const int64_t* __restrict__ edge_src,
                             int N, int E, int B, int32_t* __restrict__ node_ptr,
                             int32_t* __restrict__ edge_ptr, int* err) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < N) {
    const int64_t cur = batch[t];
    const int64_t prev = t == 0 ? -1 : batch[t - 1];
    if (cur < 0 || cur < prev || cur >= B) igmc_set_err(err, IGMC_ERR_BAD_BATCH);
    for (int64_t b = prev + 1; b <= cur && b < B; ++b) node_ptr[b] = t;
    if (t == N - 1)
      for (int64_t b = cur + 1; b <= B; ++b) node_ptr[b] = N;
  }
  if (N == 0 && t == 0)
    for (int b = 0; b <= B; ++b) node_ptr[b] = 0;
  if (t < E) {
    const int64_t s = edge_src[t];
    const int64_t cur = (s >= 0 && s < N) ? batch[s] : -1;
    int64_t prev = -1;
    if (t > 0) {
      const int64_t sp = edge_src[t - 1];
      prev = (sp >= 0 && sp < N) ? batch[sp] : -1;
    }
    if (cur < 0 || cur < prev) igmc_set_err(err, IGMC_ERR_BAD_BATCH);
    for (int64_t b = prev + 1; b <= cur && b < B; ++b) edge_ptr[b] = t;
    if (t == E - 1)
      for (int64_t b = (cur < 0 ? 0 : cur + 1); b <= B; ++b) edge_ptr[b] = E;
  }
  if (E == 0 && t == 0)
    for (int b = 0; b <= B; ++b) edge_ptr[b] = 0;
}

// One direction of the adjacency of graph g.  key: node whose list the edge joins (dst for
// incoming), nbr: the other endpoint.  An edge with an endpoint outside the graph or a type outside 0..255 (the 8-bit
// type field of a list entry) sets IGMC_ERR_BAD_BATCH and joins no list.
__device__ __forceinline__ bool edge_ok(int64_t k, int64_t o, int64_t type, int n) {
  return k >= 0 && k < n && o >= 0 && o < n && type >= 0 && type <= 255;
}

__device__ void build_lists(const int64_t* __restrict__ key_row, const int64_t* __restrict__ nbr_row,
                            const int64_t* __restrict__ edge_type, int nb, int n, int eb, int ne,
                            int32_t* __restrict__ ptr_out, uint32_t* __restrict__ adj_out,
                            int32_t* __restrict__ eid_out, uint64_t* __restrict__ tmp, int* cnt, int* fill,
                            int* ws, int* err) {
  const int tid = threadIdx.x, nt = blockDim.x, warp = tid >> 5, nwarps = nt >> 5;
  for (int v = tid; v <= n; v += nt) cnt[v] = 0;
  __syncthreads();
  for (int e = tid; e < ne; e += nt) {
    const int64_t k = key_row[eb + e] - nb, o = nbr_row[eb + e] - nb;
    if (!edge_ok(k, o, edge_type[eb + e], n)) { igmc_set_err(err, IGMC_ERR_BAD_BATCH); continue; }
    atomicAdd(&cnt[(int)k], 1);
  }
  __syncthreads();
  block_scan_chunks(
      n, ws, [&](int v) { return cnt[v]; },
      [&](int v, int ex) {
        fill[v] = ex;
        ptr_out[nb + v] = eb + ex;
      });
  __syncthreads();
  // unordered placement; fill[v] ends at the list end
  for (int e = tid; e < ne; e += nt) {
    const int64_t k = key_row[eb + e] - nb, o = nbr_row[eb + e] - nb, type = edge_type[eb + e];
    if (!edge_ok(k, o, type, n)) continue;
    const int slot = atomicAdd(&fill[(int)k], 1);
    tmp[eb + slot] = list_key((uint32_t)type, (uint32_t)o, (uint32_t)e);
  }
  __syncthreads();
  // deterministic order: rank-sort every list by its key (lists are short: mean degree ~20)
  for (int v = warp; v < n; v += nwarps) {
    const int k = cnt[v], beg = eb + fill[v] - k;
    rank_sort_list(tmp + beg, k, adj_out + beg, eid_out + beg, eb);
  }
  __syncthreads();
}

__global__ void __launch_bounds__(BP_THREADS)
k_batch_prepare(const int64_t* __restrict__ edge_index, int64_t row_stride, const int64_t* __restrict__ edge_type,
                const int32_t* __restrict__ node_ptr, const int32_t* __restrict__ edge_ptr, int B, int n_cap,
                igmc_adj_t A, int* err) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int* cnt = reinterpret_cast<int*>(smem_raw);  // [n_cap+1]
  int* fill = cnt + (n_cap + 1);                // [n_cap+1]
  __shared__ int ws[34];
  const int g = blockIdx.x;
  const int nb = node_ptr[g], n = node_ptr[g + 1] - nb;
  const int eb = edge_ptr[g], ne = edge_ptr[g + 1] - eb;
  if (g == B - 1 && threadIdx.x == 0) {
    A.in_ptr[node_ptr[B]] = edge_ptr[B];
    if (!A.symmetric) A.out_ptr[node_ptr[B]] = edge_ptr[B];
  }
  if (n > n_cap || n > 65535) {
    if (threadIdx.x == 0) igmc_set_err(err, IGMC_ERR_SMEM_NODES);
    return;
  }
  const int64_t* src = edge_index;
  const int64_t* dst = edge_index + row_stride;
  build_lists(dst, src, edge_type, nb, n, eb, ne, A.in_ptr, A.in_adj, A.in_eid, A.tmp, cnt, fill, ws, err);
  if (!A.symmetric)
    build_lists(src, dst, edge_type, nb, n, eb, ne, A.out_ptr, A.out_adj, A.out_eid, A.tmp, cnt, fill, ws, err);
}

}  // namespace

extern "C" int igmc_batch_ptrs(const int64_t* batch, const int64_t* edge_src, int N, int E, int B,
                               int32_t* node_ptr, int32_t* edge_ptr, int* err, void* stream) {
  const int work = N > E ? N : E;
  const int blocks = work > 0 ? (work + 255) / 256 : 1;
  k_batch_ptrs<<<blocks, 256, 0, (cudaStream_t)stream>>>(batch, edge_src, N, E, B, node_ptr, edge_ptr, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_batch_prepare(const int64_t* edge_index, int64_t edge_row_stride, const int64_t* edge_type,
                                  const int32_t* node_ptr, const int32_t* edge_ptr, int B, int n_cap,
                                  const igmc_adj_t* A, int* err, void* stream) {
  if (B <= 0) return 0;
  const size_t smem = 2 * (size_t)(n_cap + 1) * sizeof(int);
  if (smem > 200 * 1024) return -3;
  cudaFuncSetAttribute(k_batch_prepare, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  k_batch_prepare<<<B, BP_THREADS, smem, (cudaStream_t)stream>>>(edge_index, edge_row_stride, edge_type, node_ptr,
                                                                  edge_ptr, B, n_cap, *A, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
