// Explanation path: the score change from removing each rating of a pair's enclosing subgraph (igmc_b200/recommend.py,
// explain_pairs).
//
// The run has two passes over the inference engine's pipeline.  The base pass scores the P pairs as predict_pairs does
// and counts each subgraph's undirected edges; the occlusion pass scores T = sum of those counts copies of the pairs,
// copy (q, j) with both directed edges of pair q's rating j dropped through the model kernels' injected edge_keep mask:
//   k_explain_count     after a base batch's extraction: num_edges[tag] = the graph's undirected edge count
//   k_explain_offsets   one CTA: exclusive int64 prefix of num_edges, offsets[P] = T
//   k_occlusion_pairs   one CTA: positions [cursor, cursor + B) -> (pair q, edge j) by binary search over offsets, the
//                       pairs for igmc_extract_batch (idx = NULL), tag = position; then cursor += B
//   k_occlusion_mask    one CTA per graph of an extracted occlusion batch: edge_keep of its edges (all ones but edge j's
//                       two directed copies) and that rating's global (user, item, label) at its position
//   k_order_keys / sort / k_order_gather   delta = occluded - score[q], per-pair segmented radix sort on
//                       (~orderable(|delta|) << 32) | j, then all of each segment or its first m entries
// Every copy of pair q samples its subgraph with the same pair id, so it is the same subgraph and edge j is the same
// rating in every copy.  The sort key is a strict total order, so nothing depends on batch boundaries.
// Attribution (attribute_pairs) reuses the count, offsets and order: its gradient pass extracts the P pairs again and
// k_edge_grad_scatter sums each rating's two directed-edge gradients of igmc_edge_grad (csrc/rgcn_l2.cu) into its
// position; igmc_occlusion_order then orders those values as they are (score = NULL).
// Node explanations (explain_nodes / attribute_nodes) run the same passes with a pair's non-target nodes as positions:
//   k_node_count          after a base batch's extraction: num_nodes[tag] = the graph's node count - 2
//   k_node_occlusion_mask an occlusion batch's edge_keep drops every rating of the node at position j
//                         (k_occlusion_pairs' edge_j is the node position) and records its id, label and rating count
//   k_node_grad_scatter   the sum of each node's ratings' igmc_edge_grad values, in its in-list order, at its position
#include <algorithm>

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_segmented_radix_sort.cuh>

#include "common.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int SCAN_THREADS = 512;
constexpr int PAIR_THREADS = 512;
constexpr int MASK_THREADS = 256;
constexpr int ORDER_THREADS = 256;

__global__ void k_explain_count(const int32_t* __restrict__ edge_ptr, const int64_t* __restrict__ tag, int B,
                                int32_t* __restrict__ num_edges) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  const long long t = tag[i];
  if (t >= 0) num_edges[t] = (edge_ptr[i + 1] - edge_ptr[i]) >> 1;
}

__global__ void __launch_bounds__(SCAN_THREADS)
k_explain_offsets(const int32_t* __restrict__ num_edges, long long P, int64_t* __restrict__ offsets) {
  using Scan = cub::BlockScan<long long, SCAN_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  long long carry = 0;
  for (long long base = 0; base < P; base += SCAN_THREADS) {
    const long long i = base + threadIdx.x;
    const long long v = i < P ? (long long)num_edges[i] : 0;
    long long ex, tot;
    Scan(tmp).ExclusiveSum(v, ex, tot);
    if (i < P) offsets[i] = carry + ex;
    carry += tot;
    __syncthreads();   // tmp is reused by the next chunk
  }
  if (threadIdx.x == 0) offsets[P] = carry;
}

__global__ void __launch_bounds__(PAIR_THREADS)
k_occlusion_pairs(igmc_csr_t G, const int32_t* __restrict__ pair_u, const int32_t* __restrict__ pair_v,
                  const int64_t* __restrict__ offsets, int P, int64_t* __restrict__ cursor, int B,
                  int32_t* __restrict__ links_u, int32_t* __restrict__ links_v, int64_t* __restrict__ pair_id,
                  int64_t* __restrict__ tag, int32_t* __restrict__ edge_j, int* err) {
  __shared__ long long s_pos;
  if (threadIdx.x == 0) s_pos = *cursor;
  __syncthreads();
  const long long pos = s_pos, T = offsets[P];
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    long long c = pos + i;
    const bool real = c < T;
    if (!real) c = T - 1;       // tail batch: a valid duplicate of the last position, marked -1
    const int q = owner(offsets, P, c);
    int u = pair_u[q], v = pair_v[q];
    if (u < 0 || u >= G.num_users || v < 0 || v >= G.num_items) {
      igmc_set_err(err, IGMC_ERR_CANDIDATES);
      u = 0;
      v = 0;
    }
    links_u[i] = u;
    links_v[i] = v;
    pair_id[i] = (int64_t)u * G.num_items + v;
    tag[i] = real ? c : -1;
    edge_j[i] = (int32_t)(c - offsets[q]);
  }
  __syncthreads();
  if (threadIdx.x == 0) *cursor = pos + B;
}

// global user, item and label of the rating whose user -> item edge is a (an extracted batch's edge_index, row stride
// row_stride) at position c
__device__ __forceinline__ void record_rating(const int64_t* __restrict__ edge_index, long long row_stride,
                                              const int64_t* __restrict__ edge_type, const int32_t* __restrict__ node_gid,
                                              int a, long long c, int32_t* __restrict__ out_user,
                                              int32_t* __restrict__ out_item, int32_t* __restrict__ out_rating) {
  out_user[c] = node_gid[edge_index[a]];
  out_item[c] = node_gid[edge_index[row_stride + a]];
  out_rating[c] = (int32_t)edge_type[a];
}

// graph i of an extracted occlusion batch; its edge_index is [u|v ; v|u], so undirected edge j is the directed pair
// edge_ptr[i] + j (user -> item) and edge_ptr[i] + m + j (item -> user), m = the graph's undirected edge count
__global__ void __launch_bounds__(MASK_THREADS)
k_occlusion_mask(const int32_t* __restrict__ edge_ptr, const int64_t* __restrict__ edge_index, long long row_stride,
                 const int64_t* __restrict__ edge_type, const int32_t* __restrict__ node_gid,
                 const int64_t* __restrict__ tag, const int32_t* __restrict__ edge_j, uint8_t* __restrict__ edge_keep,
                 int32_t* __restrict__ out_user, int32_t* __restrict__ out_item, int32_t* __restrict__ out_rating,
                 int* err) {
  const int i = blockIdx.x;
  const int e0 = edge_ptr[i], e1 = edge_ptr[i + 1], m = (e1 - e0) >> 1;
  const long long c = tag[i];
  const int j = edge_j[i];
  bool drop = c >= 0;
  if (drop && (j < 0 || j >= m)) {   // the subgraph is not the one the base pass counted
    if (threadIdx.x == 0) igmc_set_err(err, IGMC_ERR_CANDIDATES);
    drop = false;
  }
  const int a = e0 + j, b = a + m;
  for (int e = e0 + threadIdx.x; e < e1; e += blockDim.x) edge_keep[e] = (drop && (e == a || e == b)) ? 0 : 1;
  if (drop && threadIdx.x == 0)
    record_rating(edge_index, row_stride, edge_type, node_gid, a, c, out_user, out_item, out_rating);
}

// graph i of an attribution batch with tag q >= 0: rating j's value is the sum of its two directed edges' gradients,
// out[offsets[q] + j] = (checkpoint k = 0 ? 0 : out) + that sum, divided by K after the last checkpoint k = K - 1
__global__ void __launch_bounds__(MASK_THREADS)
k_edge_grad_scatter(const int32_t* __restrict__ edge_ptr, const int64_t* __restrict__ edge_index, long long row_stride,
                    const int64_t* __restrict__ edge_type, const int32_t* __restrict__ node_gid,
                    const int64_t* __restrict__ tag, const float* __restrict__ edge_grad,
                    const int64_t* __restrict__ offsets, int k, int K, float* __restrict__ out,
                    int32_t* __restrict__ out_user, int32_t* __restrict__ out_item, int32_t* __restrict__ out_rating,
                    int* err) {
  const int i = blockIdx.x;
  const long long q = tag[i];
  if (q < 0) return;
  const int e0 = edge_ptr[i], m = (edge_ptr[i + 1] - e0) >> 1;
  const long long o = offsets[q];
  if (offsets[q + 1] - o != m) {   // the subgraph is not the one the base pass counted
    if (threadIdx.x == 0) igmc_set_err(err, IGMC_ERR_CANDIDATES);
    return;
  }
  for (int j = threadIdx.x; j < m; j += blockDim.x) {
    float v = edge_grad[e0 + j] + edge_grad[e0 + m + j];
    if (k > 0) v = out[o + j] + v;
    if (k == K - 1) v = v / (float)K;
    out[o + j] = v;
    if (k == 0) record_rating(edge_index, row_stride, edge_type, node_gid, e0 + j, o + j, out_user, out_item, out_rating);
  }
}

// ---- node explanations (explain_nodes / attribute_nodes) ----
// A pair's positions are the non-target nodes of its subgraph (node_label >= 2) in node order: position j is the j-th.

__global__ void k_node_count(const int32_t* __restrict__ node_ptr, const int64_t* __restrict__ tag, int B,
                             int32_t* __restrict__ num_nodes) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  const long long t = tag[i];
  if (t >= 0) num_nodes[t] = max(node_ptr[i + 1] - node_ptr[i] - 2, 0);
}

// f(n, j) for every non-target node n of the nodes [n0, n1), j its position; one chunk of MASK_THREADS nodes at a time.
// Every thread of the CTA must call it.
template <class F>
__device__ __forceinline__ void foreach_position(const uint8_t* __restrict__ node_label, int n0, int n1, F f) {
  using Scan = cub::BlockScan<int, MASK_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  int carry = 0;
  for (int base = n0; base < n1; base += MASK_THREADS) {
    const int n = base + threadIdx.x;
    const int flag = n < n1 && node_label[n] >= 2;
    int ex, tot;
    Scan(tmp).ExclusiveSum(flag, ex, tot);
    if (flag) f(n, carry + ex);
    carry += tot;
    __syncthreads();   // tmp is reused by the next chunk
  }
}

// graph i of an extracted occlusion batch: edge_keep of its edges (0 on every directed edge with node p = position j
// as an endpoint: both copies of each of p's ratings) and p's global id, label and rating count at position c
__global__ void __launch_bounds__(MASK_THREADS)
k_node_occlusion_mask(const int32_t* __restrict__ node_ptr, const int32_t* __restrict__ edge_ptr,
                      const int64_t* __restrict__ edge_index, long long row_stride,
                      const uint8_t* __restrict__ node_label, const int32_t* __restrict__ node_gid,
                      const int64_t* __restrict__ tag, const int32_t* __restrict__ node_j,
                      uint8_t* __restrict__ edge_keep, int32_t* __restrict__ out_node, int32_t* __restrict__ out_label,
                      int32_t* __restrict__ out_ratings, int* err) {
  using Reduce = cub::BlockReduce<int, MASK_THREADS>;
  __shared__ typename Reduce::TempStorage rtmp;
  __shared__ int s_p;
  const int i = blockIdx.x;
  const int e0 = edge_ptr[i], e1 = edge_ptr[i + 1];
  const long long c = tag[i];
  const int j = node_j[i];
  if (threadIdx.x == 0) s_p = -1;
  __syncthreads();
  if (c >= 0) foreach_position(node_label, node_ptr[i], node_ptr[i + 1], [&](int n, int jn) { if (jn == j) s_p = n; });
  __syncthreads();
  const int p = s_p;
  if (c >= 0 && p < 0 && threadIdx.x == 0) igmc_set_err(err, IGMC_ERR_CANDIDATES);   // not the base pass's subgraph
  int hits = 0;
  for (int e = e0 + threadIdx.x; e < e1; e += blockDim.x) {
    const bool hit = p >= 0 && (edge_index[e] == p || edge_index[row_stride + e] == p);
    edge_keep[e] = hit ? 0 : 1;
    hits += hit;
  }
  const int total = Reduce(rtmp).Sum(hits);   // thread 0: two directed edges per rating
  if (p >= 0 && threadIdx.x == 0) {
    out_node[c] = node_gid[p];
    out_label[c] = node_label[p];
    out_ratings[c] = total >> 1;
  }
}

// graph i of an attribution batch with tag q >= 0: node n at position j gets the sum, in n's in-list order, of its
// ratings' values edge_grad[a] + edge_grad[a + m] (a the rating's user -> item edge); out[offsets[q] + j] =
// (checkpoint k = 0 ? 0 : out) + that sum, divided by K after the last checkpoint k = K - 1
__global__ void __launch_bounds__(MASK_THREADS)
k_node_grad_scatter(const int32_t* __restrict__ node_ptr, const int32_t* __restrict__ edge_ptr,
                    const uint8_t* __restrict__ node_label, const int32_t* __restrict__ node_gid,
                    const int32_t* __restrict__ in_ptr, const int32_t* __restrict__ in_eid,
                    const int64_t* __restrict__ tag, const float* __restrict__ edge_grad,
                    const int64_t* __restrict__ offsets, int k, int K, float* __restrict__ out,
                    int32_t* __restrict__ out_node, int32_t* __restrict__ out_label, int32_t* __restrict__ out_ratings,
                    int* err) {
  const int i = blockIdx.x;
  const long long q = tag[i];
  if (q < 0) return;
  const int n0 = node_ptr[i], n1 = node_ptr[i + 1], e0 = edge_ptr[i], m = (edge_ptr[i + 1] - e0) >> 1;
  const long long o = offsets[q], cnt = offsets[q + 1] - o;
  if (cnt != max(n1 - n0 - 2, 0)) {   // the subgraph is not the one the base pass counted
    if (threadIdx.x == 0) igmc_set_err(err, IGMC_ERR_CANDIDATES);
    return;
  }
  foreach_position(node_label, n0, n1, [&](int n, int j) {
    if (j >= cnt) {   // more non-target nodes than nodes - 2: labels unlike an extracted subgraph's
      igmc_set_err(err, IGMC_ERR_CANDIDATES);
      return;
    }
    const int a0 = in_ptr[n], a1 = in_ptr[n + 1];
    float v = 0.f;
    for (int a = a0; a < a1; ++a) {
      const int e = in_eid[a];
      const int r = e - e0 < m ? e : e - m;
      const float g = edge_grad[r] + edge_grad[r + m];
      v = a == a0 ? g : v + g;
    }
    if (k > 0) v = out[o + j] + v;
    if (k == K - 1) v = v / (float)K;
    out[o + j] = v;
    if (k == 0) {
      out_node[o + j] = node_gid[n];
      out_label[o + j] = node_label[n];
      out_ratings[o + j] = a1 - a0;
    }
  });
}

// |delta| descending, NaN after every number: an ascending key on ~o, o = 0 for NaN, else the bits of |delta| + 1
// (the bits of a non-negative float ascend with its value; +0 and -0 are one value)
__device__ __forceinline__ uint32_t orderable_abs(float d) {
  return isnan(d) ? 0u : __float_as_uint(fabsf(d)) + 1u;
}

__global__ void k_order_keys(const float* __restrict__ score, const float* __restrict__ occluded,
                             const int64_t* __restrict__ offsets, int P, int T, uint64_t* __restrict__ keys,
                             int32_t* __restrict__ pos, float* __restrict__ delta) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < T; c += gridDim.x * blockDim.x) {
    const int q = owner(offsets, P, c);
    const float d = score ? __fsub_rn(occluded[c], score[q]) : occluded[c];
    const uint32_t j = (uint32_t)(c - offsets[q]);
    keys[c] = ((uint64_t)~orderable_abs(d) << 32) | j;
    pos[c] = c;
    delta[c] = d;
  }
}

// m = 0: out[i] = entry srt[i] for every i < T.  m > 0: out[q * m + t] = the t-th entry of pair q's sorted segment, or
// padding (user / item / rating -1, delta 0) past its end.
__global__ void k_order_gather(const int32_t* __restrict__ srt, const int64_t* __restrict__ offsets, int P, int T,
                               int m, const int32_t* __restrict__ user, const int32_t* __restrict__ item,
                               const int32_t* __restrict__ rating, const float* __restrict__ delta,
                               int32_t* __restrict__ out_user, int32_t* __restrict__ out_item,
                               int32_t* __restrict__ out_rating, float* __restrict__ out_delta) {
  const long long n = m ? (long long)P * m : T;
  for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < n;
       o += (long long)gridDim.x * blockDim.x) {
    long long i = o;
    if (m) {
      const long long q = o / m, t = o - q * m;
      i = offsets[q] + t < offsets[q + 1] ? offsets[q] + t : -1;
    }
    if (i < 0) {
      out_user[o] = -1;
      out_item[o] = -1;
      out_rating[o] = -1;
      out_delta[o] = 0.f;
    } else {
      const int c = srt[i];
      out_user[o] = user[c];
      out_item[o] = item[c];
      out_rating[o] = rating[c];
      out_delta[o] = delta[c];
    }
  }
}

// the carve-up of igmc_occlusion_order's workspace: keys in / out [T], positions in / out [T], delta [T], CUB scratch
struct OrderLayout {
  uint64_t *keys, *keys_out;
  int32_t *pos, *pos_out;
  float* delta;
  void* temp;
  size_t temp_bytes, total;
};

OrderLayout order_layout(void* base, int P, int T, cudaStream_t st) {
  OrderLayout L = {};
  const size_t k = align256((size_t)T * 8), p = align256((size_t)T * 4);
  unsigned char* b = static_cast<unsigned char*>(base);
  if (b) {
    L.keys = reinterpret_cast<uint64_t*>(b);
    L.keys_out = reinterpret_cast<uint64_t*>(b + k);
    L.pos = reinterpret_cast<int32_t*>(b + 2 * k);
    L.pos_out = reinterpret_cast<int32_t*>(b + 2 * k + p);
    L.delta = reinterpret_cast<float*>(b + 2 * k + 2 * p);
    L.temp = b + 2 * k + 3 * p;
  }
  cub::DeviceSegmentedRadixSort::SortPairs(nullptr, L.temp_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                           (const int32_t*)nullptr, (int32_t*)nullptr, T, P,
                                           (const int64_t*)nullptr, (const int64_t*)nullptr, 0, 64, st);
  L.total = 2 * k + 3 * p + align256(L.temp_bytes);
  return L;
}

bool order_shape_ok(long long P, long long T) { return P >= 0 && T >= 0 && P < (1ll << 31) - 1 && T < (1ll << 31) - 1; }

int grid_for(long long n, int threads) { return (int)std::max(1ll, std::min((n + threads - 1) / threads, 4096ll)); }

}  // namespace

extern "C" int igmc_explain_count(const int32_t* edge_ptr, const int64_t* tag, int B, int32_t* num_edges,
                                  void* stream) {
  if (!edge_ptr || !tag || !num_edges || B <= 0) return -1;
  k_explain_count<<<(B + 255) / 256, 256, 0, (cudaStream_t)stream>>>(edge_ptr, tag, B, num_edges);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_explain_offsets(const int32_t* num_edges, int num_pairs, int64_t* offsets, void* stream) {
  if (!offsets || num_pairs < 0 || (num_pairs > 0 && !num_edges)) return -1;
  k_explain_offsets<<<1, SCAN_THREADS, 0, (cudaStream_t)stream>>>(num_edges, num_pairs, offsets);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_occlusion_pairs(const igmc_csr_t* G, const int32_t* pair_u, const int32_t* pair_v,
                                    const int64_t* offsets, int num_pairs, int64_t* cursor, int B, int32_t* links_u,
                                    int32_t* links_v, int64_t* pair_id, int64_t* tag, int32_t* edge_j, int* err,
                                    void* stream) {
  if (!G || !pair_u || !pair_v || !offsets || !cursor || num_pairs <= 0 || B <= 0) return -1;
  if (!links_u || !links_v || !pair_id || !tag || !edge_j) return -1;
  k_occlusion_pairs<<<1, PAIR_THREADS, 0, (cudaStream_t)stream>>>(*G, pair_u, pair_v, offsets, num_pairs, cursor, B,
                                                                   links_u, links_v, pair_id, tag, edge_j, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_occlusion_mask(const igmc_batch_out_t* O, int B, const int64_t* tag, const int32_t* edge_j,
                                   uint8_t* edge_keep, int32_t* user, int32_t* item, int32_t* rating, int* err,
                                   void* stream) {
  if (!O || !O->edge_ptr || !O->edge_index || !O->edge_type || !O->node_gid || B <= 0) return -1;
  if (!tag || !edge_j || !edge_keep || !user || !item || !rating) return -1;
  k_occlusion_mask<<<B, MASK_THREADS, 0, (cudaStream_t)stream>>>(O->edge_ptr, O->edge_index, O->edge_cap,
                                                                  O->edge_type, O->node_gid, tag, edge_j, edge_keep,
                                                                  user, item, rating, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_edge_grad_scatter(const igmc_batch_out_t* O, int B, const int64_t* tag, const float* edge_grad,
                                      const int64_t* offsets, int k, int K, float* out, int32_t* user, int32_t* item,
                                      int32_t* rating, int* err, void* stream) {
  if (!O || !O->edge_ptr || !O->edge_index || !O->edge_type || !O->node_gid || B <= 0) return -1;
  if (!tag || !edge_grad || !offsets || !out || !user || !item || !rating || K < 1 || k < 0 || k >= K) return -1;
  k_edge_grad_scatter<<<B, MASK_THREADS, 0, (cudaStream_t)stream>>>(O->edge_ptr, O->edge_index, O->edge_cap,
                                                                     O->edge_type, O->node_gid, tag, edge_grad, offsets,
                                                                     k, K, out, user, item, rating, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_explain_node_count(const int32_t* node_ptr, const int64_t* tag, int B, int32_t* num_nodes,
                                       void* stream) {
  if (!node_ptr || !tag || !num_nodes || B <= 0) return -1;
  k_node_count<<<(B + 255) / 256, 256, 0, (cudaStream_t)stream>>>(node_ptr, tag, B, num_nodes);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_node_occlusion_mask(const igmc_batch_out_t* O, int B, const int64_t* tag, const int32_t* node_j,
                                        uint8_t* edge_keep, int32_t* node, int32_t* label, int32_t* ratings, int* err,
                                        void* stream) {
  if (!O || !O->node_ptr || !O->edge_ptr || !O->edge_index || !O->node_label || !O->node_gid || B <= 0) return -1;
  if (!tag || !node_j || !edge_keep || !node || !label || !ratings) return -1;
  k_node_occlusion_mask<<<B, MASK_THREADS, 0, (cudaStream_t)stream>>>(O->node_ptr, O->edge_ptr, O->edge_index,
                                                                       O->edge_cap, O->node_label, O->node_gid, tag,
                                                                       node_j, edge_keep, node, label, ratings, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_node_grad_scatter(const igmc_batch_out_t* O, int B, const int64_t* tag, const float* edge_grad,
                                      const int64_t* offsets, int k, int K, float* out, int32_t* node, int32_t* label,
                                      int32_t* ratings, int* err, void* stream) {
  if (!O || !O->node_ptr || !O->edge_ptr || !O->node_label || !O->node_gid || !O->adj_in_ptr || !O->adj_eid || B <= 0)
    return -1;
  if (!tag || !edge_grad || !offsets || !out || !node || !label || !ratings || K < 1 || k < 0 || k >= K) return -1;
  k_node_grad_scatter<<<B, MASK_THREADS, 0, (cudaStream_t)stream>>>(O->node_ptr, O->edge_ptr, O->node_label,
                                                                     O->node_gid, O->adj_in_ptr, O->adj_eid, tag,
                                                                     edge_grad, offsets, k, K, out, node, label,
                                                                     ratings, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_occlusion_order_ws_bytes(int num_pairs, int64_t num_positions, int64_t* bytes) {
  if (!bytes || !order_shape_ok(num_pairs, num_positions)) return -1;
  *bytes = (int64_t)order_layout(nullptr, num_pairs, (int)num_positions, 0).total;
  return 0;
}

extern "C" int igmc_occlusion_order(const float* score, const float* occluded, const int64_t* offsets, int num_pairs,
                                    int64_t num_positions, const int32_t* user, const int32_t* item,
                                    const int32_t* rating, int m, void* ws, int64_t ws_bytes, int32_t* out_user,
                                    int32_t* out_item, int32_t* out_rating, float* out_delta, void* stream) {
  if (!order_shape_ok(num_pairs, num_positions) || m < 0 || m > IGMC_TOPK_MAX) return -1;
  const int P = num_pairs, T = (int)num_positions;
  if (P == 0 || (T == 0 && m == 0)) return 0;
  if (!offsets || !out_user || !out_item || !out_rating || !out_delta || !ws) return -1;
  if (T > 0 && (!occluded || !user || !item || !rating)) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  const OrderLayout L = order_layout(ws, P, T, st);
  if ((int64_t)L.total > ws_bytes) return -2;
  if (T > 0) {
    k_order_keys<<<grid_for(T, ORDER_THREADS), ORDER_THREADS, 0, st>>>(score, occluded, offsets, P, T, L.keys, L.pos,
                                                                       L.delta);
    IGMC_CUDA_CHECK_LAUNCH();
    size_t tb = L.temp_bytes;
    if (cub::DeviceSegmentedRadixSort::SortPairs(L.temp, tb, L.keys, L.keys_out, L.pos, L.pos_out, T, P, offsets,
                                                 offsets + 1, 0, 64, st) != cudaSuccess)
      return -3;
  }
  const long long n = m ? (long long)P * m : T;
  k_order_gather<<<grid_for(n, ORDER_THREADS), ORDER_THREADS, 0, st>>>(L.pos_out, offsets, P, T, m, user, item, rating,
                                                                       L.delta, out_user, out_item, out_rating,
                                                                       out_delta);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
