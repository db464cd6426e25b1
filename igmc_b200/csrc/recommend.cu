// Inference path: candidate pairs on the device and streaming per-user top-k (igmc_b200/recommend.py).
//
// A trained model scores (user, item) pairs it has no rating for and ranks them.  The host names the query users and
// (optionally) a candidate item list once; from then on every batch is produced, scored and merged on the device:
//   k_candidate_plan   one CTA: per query user the candidate count and its exclusive prefix user_off[U+1]; with a
//                      candidate list and exclude_rated, also the positions in the list of the user's rated items
//   k_lists_rows       per-user candidate rows (after a segmented sort): one CTA per row counts, then writes, the valid,
//                      distinct, (with exclude_rated) unrated items; k_lists_scan turns the counts into user_off
//   k_candidate_pairs  one CTA: the pairs of global candidate positions [cursor, cursor + B) for igmc_extract_batch
//                      (idx = NULL), then cursor += B - a captured graph replays with no host input
//   k_topk_merge       one CTA per per-user segment of the batch: fp32 checkpoint mean + merge into the running
//                      [U, k] (score, item) list
//   k_score_scatter    explicit pairs: the fp32 checkpoint mean stored at the pair's index
//   k_item_query_pairs item-side runs (query items, candidate users): the candidate kernels run on the transposed view
//                      of the graph, and this post-pass turns their (item, user) pairs back into (user, item) ones
// No float atomics: the ranking order (score descending, item ascending, NaN last, empty slots after everything) is a
// strict total order on distinct items, so the top-k of a user does not depend on where batch boundaries fall.
#include <cub/device/device_segmented_radix_sort.cuh>

#include "common.cuh"
#include "topk_merge.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int LIST_THREADS = 256;
constexpr int PLAN_THREADS = 1024;
constexpr int PAIR_THREADS = 512;
constexpr int MERGE_THREADS = 256;

__device__ __forceinline__ long long warp_incl_scan_ll(long long v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    long long t = __shfl_up_sync(IGMC_FULL, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

// block-wide exclusive scan of one int64 per thread; `ws` >= 33 long longs of shared scratch; ends with a barrier
__device__ __forceinline__ long long block_excl_scan_ll(long long v, long long* ws, long long* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  long long incl = warp_incl_scan_ll(v, lane);
  if (lane == 31) ws[w] = incl;
  __syncthreads();
  if (w == 0) {
    long long s = lane < nw ? ws[lane] : 0;
    long long inc = warp_incl_scan_ll(s, lane);
    ws[lane] = inc - s;
    if (lane == 31) ws[32] = inc;
  }
  __syncthreads();
  long long excl = ws[w] + incl - v;
  *total = ws[32];
  __syncthreads();
  return excl;
}

// position of `item` in the ascending list a[0..n), or -1
__device__ __forceinline__ int find_sorted(const int32_t* __restrict__ a, int n, int item) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < item) lo = mid + 1; else hi = mid;
  }
  return (lo < n && a[lo] == item) ? lo : -1;
}

__global__ void __launch_bounds__(PLAN_THREADS) k_candidate_plan(igmc_csr_t G, igmc_candidates_t Cd, int* err) {
  __shared__ long long ws[33];
  const int U = Cd.num_query;
  const bool lists = Cd.cand != nullptr && Cd.exclude_rated;
  long long carry = 0, carry_r = 0;
  for (int base = 0; base < U; base += blockDim.x) {
    const int j = base + threadIdx.x;
    long long cnt = 0, hits = 0;
    if (j < U) {
      const int u = Cd.users[j];
      if (u < 0 || u >= G.num_users) {
        igmc_set_err(err, IGMC_ERR_CANDIDATES);
      } else {
        const int r0 = G.row_ptr[u], r1 = G.row_ptr[u + 1];
        if (Cd.cand == nullptr) {
          cnt = Cd.exclude_rated ? (long long)G.num_items - (r1 - r0) : G.num_items;
        } else if (!Cd.exclude_rated) {
          cnt = Cd.num_cand;
        } else {
          for (int e = r0; e < r1; ++e) hits += find_sorted(Cd.cand, Cd.num_cand, G.col_idx[e]) >= 0;
          cnt = Cd.num_cand - hits;
        }
      }
    }
    long long tot, tot_r = 0;
    const long long off = block_excl_scan_ll(cnt, ws, &tot);
    long long off_r = 0;
    if (lists) off_r = block_excl_scan_ll(hits, ws, &tot_r);
    if (j < U) {
      Cd.user_off[j] = carry + off;
      if (lists) Cd.rated_off[j] = carry_r + off_r;
    }
    carry += tot;
    carry_r += tot_r;
  }
  if (threadIdx.x == 0) {
    Cd.user_off[U] = carry;
    if (lists) Cd.rated_off[U] = carry_r;
  }
  if (!lists) return;
  __syncthreads();
  // the rated positions of every user, ascending (rows and the candidate list are both ascending)
  for (int j = threadIdx.x; j < U; j += blockDim.x) {
    const int u = Cd.users[j];
    if (u < 0 || u >= G.num_users) continue;
    long long o = Cd.rated_off[j];
    for (int e = G.row_ptr[u]; e < G.row_ptr[u + 1]; ++e) {
      const int p = find_sorted(Cd.cand, Cd.num_cand, G.col_idx[e]);
      if (p >= 0) Cd.rated_pos[o++] = p;
    }
  }
}

__global__ void k_segment_offsets(int32_t* __restrict__ off, int U, int width) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j <= U; j += gridDim.x * blockDim.x) off[j] = j * width;
}

// one CTA per query slot j over its sorted row srt[j*width, (j+1)*width): the items kept are in [0, num_items), not
// equal to their predecessor and (exclude_rated) not rated by the user.  Counting pass (WRITE = false): the count goes
// to user_off[j] and ids outside [-1, num_items) set the error; writing pass: the kept items, ascending, from lists[
// user_off[j]] on.
template <bool WRITE>
__global__ void __launch_bounds__(LIST_THREADS)
k_lists_rows(igmc_csr_t G, igmc_candidates_t Cd, const int32_t* __restrict__ srt, int width, int32_t* __restrict__ lists,
             int* err) {
  __shared__ long long ws[33];
  const int j = blockIdx.x;
  const int u = Cd.users[j];
  const bool user_ok = u >= 0 && u < G.num_users;
  if (!user_ok) {
    if (!WRITE && threadIdx.x == 0) {
      igmc_set_err(err, IGMC_ERR_CANDIDATES);
      Cd.user_off[j] = 0;
    }
    return;
  }
  const int32_t* row = srt + (size_t)j * width;
  const int32_t* rated = G.col_idx + G.row_ptr[u];
  const int nr = G.row_ptr[u + 1] - G.row_ptr[u];
  const long long out0 = WRITE ? Cd.user_off[j] : 0;
  long long carry = 0;
  for (int c0 = 0; c0 < width; c0 += blockDim.x) {
    const int t = c0 + threadIdx.x;
    bool keep = false;
    if (t < width) {
      const int x = row[t];
      if (!WRITE && (x < -1 || x >= G.num_items)) igmc_set_err(err, IGMC_ERR_CANDIDATES);
      keep = x >= 0 && x < G.num_items && (t == 0 || row[t - 1] != x) &&
             !(Cd.exclude_rated && find_sorted(rated, nr, x) >= 0);
    }
    long long tot;
    const long long off = block_excl_scan_ll(keep ? 1 : 0, ws, &tot);
    if (WRITE && keep) lists[out0 + carry + off] = row[t];
    carry += tot;
  }
  if (!WRITE && threadIdx.x == 0) Cd.user_off[j] = carry;
}

// user_off[0..U) holds the per-user counts: turn it into their exclusive prefix, user_off[U] = the total
__global__ void __launch_bounds__(PLAN_THREADS) k_lists_scan(igmc_candidates_t Cd) {
  __shared__ long long ws[33];
  const int U = Cd.num_query;
  long long carry = 0;
  for (int base = 0; base < U; base += blockDim.x) {
    const int j = base + threadIdx.x;
    const long long cnt = j < U ? Cd.user_off[j] : 0;
    long long tot;
    const long long off = block_excl_scan_ll(cnt, ws, &tot);
    if (j < U) Cd.user_off[j] = carry + off;
    carry += tot;
  }
  if (threadIdx.x == 0) Cd.user_off[U] = carry;
}

__global__ void __launch_bounds__(PAIR_THREADS)
k_candidate_pairs(igmc_csr_t G, igmc_candidates_t Cd, int64_t* __restrict__ cursor, int B,
                  int32_t* __restrict__ links_u, int32_t* __restrict__ links_v, int64_t* __restrict__ pair_id,
                  int64_t* __restrict__ tag, int* err) {
  __shared__ long long s_pos;
  if (threadIdx.x == 0) s_pos = *cursor;
  __syncthreads();
  const long long pos = s_pos, P = Cd.num_pairs;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    long long g = pos + i;
    const bool real = g < P;
    if (!real) g = P - 1;       // tail batch: a valid duplicate of the last pair, marked slot -1
    int u, v;
    long long t;
    if (Cd.users == nullptr) {  // explicit pairs: tag = pair index
      u = Cd.pair_u[g];
      v = Cd.pair_v[g];
      t = g;
    } else {
      // query slot j: the last j with user_off[j] <= g (users without candidates share their offset with the next)
      int lo = 0, hi = Cd.num_query;
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (Cd.user_off[mid] <= g) lo = mid; else hi = mid;
      }
      const long long c = g - Cd.user_off[lo];
      u = Cd.users[lo];
      long long p = c;
      if (Cd.per_user) {
        p = Cd.user_off[lo] + c;    // the user's own list in cand; its rated items are already gone
      } else if (Cd.exclude_rated) {
        // candidate rank c -> list position c + t, t = number of rated positions r_q with r_q - q <= c
        const int32_t* r;
        long long n;
        if (Cd.cand) {
          r = Cd.rated_pos + Cd.rated_off[lo];
          n = Cd.rated_off[lo + 1] - Cd.rated_off[lo];
        } else {
          r = G.col_idx + G.row_ptr[u];
          n = G.row_ptr[u + 1] - G.row_ptr[u];
        }
        p = c + rank_skip(r, n, c);
      }
      const long long lim = Cd.per_user ? P : Cd.cand ? Cd.num_cand : G.num_items;
      if (p < 0 || p >= lim) {
        igmc_set_err(err, IGMC_ERR_CANDIDATES);
        p = 0;
      }
      v = Cd.cand ? Cd.cand[p] : (int)p;
      t = lo;
    }
    if (u < 0 || u >= G.num_users || v < 0 || v >= G.num_items) {
      igmc_set_err(err, IGMC_ERR_CANDIDATES);
      u = 0;
      v = 0;
    }
    links_u[i] = u;
    links_v[i] = v;
    pair_id[i] = (int64_t)u * G.num_items + v;
    tag[i] = real ? t : -1;
  }
  __syncthreads();
  if (threadIdx.x == 0) *cursor = pos + B;
}

__global__ void __launch_bounds__(MERGE_THREADS)
k_topk_merge(const float* __restrict__ preds, int K, int B, const int64_t* __restrict__ tag,
             const int32_t* __restrict__ items, int k, float* __restrict__ top_score, int64_t* __restrict__ top_item) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int i0 = blockIdx.x;
  const long long slot = tag[i0];
  if (slot < 0 || (i0 > 0 && tag[i0 - 1] == slot)) return;   // not the first entry of a user's segment
  int& s_end = *reinterpret_cast<int*>(smem_raw);              // the segment's end, then the lists at MERGE_HEAD
  if (threadIdx.x == 0) s_end = B;
  __syncthreads();
  for (int i = i0 + 1 + threadIdx.x; i < B; i += blockDim.x)
    if (tag[i] != slot) atomicMin(&s_end, i);
  __syncthreads();
  const int m = s_end - i0, n = k + m;
  long long* I = reinterpret_cast<long long*>(smem_raw + MERGE_HEAD);
  float* S = reinterpret_cast<float*>(I + n);
  float* ts = top_score + (size_t)slot * k;
  int64_t* ti = top_item + (size_t)slot * k;
  for (int t = threadIdx.x; t < k; t += blockDim.x) {   // the running list: ranked, empty slots last
    S[t] = ts[t];
    I[t] = ti[t];
  }
  for (int t = threadIdx.x; t < m; t += blockDim.x) {   // this batch's candidates of the user
    S[k + t] = ckpt_mean(preds, K, B, i0 + t);
    I[k + t] = items[i0 + t];
  }
  __syncthreads();
  rank_merge(S, I, k, n, 1.f, ts, ti);
}

__global__ void __launch_bounds__(MERGE_THREADS)
k_score_scatter(const float* __restrict__ preds, int K, int B, const int64_t* __restrict__ tag,
                float* __restrict__ scores) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  const long long t = tag[i];
  if (t >= 0) scores[t] = ckpt_mean(preds, K, B, i);
}

// pairs igmc_candidate_pairs wrote over the transposed view (links_u = the query item, links_v = the candidate user):
// swapped back, with the pair id (user, item) samples its subgraph with
__global__ void __launch_bounds__(LIST_THREADS)
k_item_query_pairs(int num_items, int B, int32_t* __restrict__ links_u, int32_t* __restrict__ links_v,
                   int64_t* __restrict__ pair_id, int* err) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
    int v = links_u[i], u = links_v[i];
    if (v < 0 || v >= num_items || u < 0) {
      igmc_set_err(err, IGMC_ERR_CANDIDATES);
      u = 0;
      v = 0;
    }
    links_u[i] = u;
    links_v[i] = v;
    pair_id[i] = (int64_t)u * num_items + v;
  }
}

}  // namespace

extern "C" int igmc_candidate_plan(const igmc_csr_t* G, const igmc_candidates_t* Cd, int* err, void* stream) {
  if (!G || !Cd || !Cd->users || !Cd->user_off || Cd->num_query < 0) return -1;
  if (Cd->cand && Cd->exclude_rated && (!Cd->rated_off || !Cd->rated_pos)) return -1;
  k_candidate_plan<<<1, PLAN_THREADS, 0, (cudaStream_t)stream>>>(*G, *Cd, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

namespace {

// the carve-up of igmc_candidate_lists' workspace: sorted rows [U * width], segment offsets [U + 1], CUB scratch
struct ListsLayout {
  int32_t *srt, *seg;
  void* temp;
  size_t temp_bytes, total;
};

ListsLayout lists_layout(void* base, int U, int width, cudaStream_t st) {
  ListsLayout L = {};
  unsigned char* b = static_cast<unsigned char*>(base);
  const size_t a = align256((size_t)U * width * 4), s = align256(((size_t)U + 1) * 4);
  L.srt = b ? reinterpret_cast<int32_t*>(b) : nullptr;
  L.seg = b ? reinterpret_cast<int32_t*>(b + a) : nullptr;
  cub::DeviceSegmentedRadixSort::SortKeys(nullptr, L.temp_bytes, (const int32_t*)nullptr, (int32_t*)nullptr,
                                          U * width, U, (const int32_t*)nullptr, (const int32_t*)nullptr, 0, 32, st);
  L.temp = b ? b + a + s : nullptr;
  L.total = a + s + align256(L.temp_bytes);
  return L;
}

bool lists_shape_ok(int U, int width) { return U >= 0 && width >= 0 && (long long)U * width < (1ll << 31) - 1; }

}  // namespace

extern "C" int igmc_candidate_lists_ws_bytes(int num_query, int width, int64_t* bytes) {
  if (!bytes || !lists_shape_ok(num_query, width)) return -1;
  *bytes = (int64_t)lists_layout(nullptr, num_query, width, 0).total;
  return 0;
}

extern "C" int igmc_candidate_lists(const igmc_csr_t* G, const igmc_candidates_t* Cd, const int32_t* rows, int width,
                                    int32_t* lists, void* ws, int64_t ws_bytes, int* err, void* stream) {
  if (!G || !Cd || !Cd->users || !Cd->user_off || !lists_shape_ok(Cd->num_query, width)) return -1;
  const int U = Cd->num_query;
  cudaStream_t st = (cudaStream_t)stream;
  if (U == 0 || width == 0) {
    cudaMemsetAsync(Cd->user_off, 0, ((size_t)U + 1) * sizeof(int64_t), st);
    IGMC_CUDA_CHECK_LAUNCH();
    return 0;
  }
  if (!rows || !lists || !ws) return -1;
  const ListsLayout L = lists_layout(ws, U, width, st);
  if ((int64_t)L.total > ws_bytes) return -2;
  k_segment_offsets<<<(U + 1 + 255) / 256, 256, 0, st>>>(L.seg, U, width);
  IGMC_CUDA_CHECK_LAUNCH();
  size_t tb = L.temp_bytes;
  if (cub::DeviceSegmentedRadixSort::SortKeys(L.temp, tb, rows, L.srt, U * width, U, L.seg, L.seg + 1, 0, 32, st) !=
      cudaSuccess)
    return -3;
  k_lists_rows<false><<<U, LIST_THREADS, 0, st>>>(*G, *Cd, L.srt, width, lists, err);
  IGMC_CUDA_CHECK_LAUNCH();
  k_lists_scan<<<1, PLAN_THREADS, 0, st>>>(*Cd);
  IGMC_CUDA_CHECK_LAUNCH();
  k_lists_rows<true><<<U, LIST_THREADS, 0, st>>>(*G, *Cd, L.srt, width, lists, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_candidate_pairs(const igmc_csr_t* G, const igmc_candidates_t* Cd, int64_t* cursor, int B,
                                    int32_t* links_u, int32_t* links_v, int64_t* pair_id, int64_t* tag, int* err,
                                    void* stream) {
  if (!G || !Cd || !cursor || B <= 0 || Cd->num_pairs <= 0) return -1;
  if (Cd->users ? !Cd->user_off : (!Cd->pair_u || !Cd->pair_v)) return -1;
  if (Cd->per_user && (!Cd->users || !Cd->cand)) return -1;
  k_candidate_pairs<<<1, PAIR_THREADS, 0, (cudaStream_t)stream>>>(*G, *Cd, cursor, B, links_u, links_v, pair_id, tag,
                                                                   err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_item_query_pairs(int num_items, int B, int32_t* links_u, int32_t* links_v, int64_t* pair_id,
                                     int* err, void* stream) {
  if (num_items < 1 || B <= 0 || !links_u || !links_v || !pair_id) return -1;
  k_item_query_pairs<<<(B + LIST_THREADS - 1) / LIST_THREADS, LIST_THREADS, 0, (cudaStream_t)stream>>>(
      num_items, B, links_u, links_v, pair_id, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_topk_fits(int k, int B) {
  if (k < 1 || k > IGMC_TOPK_MAX || B < 1) return 0;
  return merge_smem(k, B) <= 227 * 1024 ? 1 : 0;
}

extern "C" int igmc_topk_merge(const float* preds, int K, int B, const int64_t* tag, const int32_t* items, int k,
                               float* top_score, int64_t* top_item, void* stream) {
  if (K < 1 || B <= 0 || k < 1 || k > IGMC_TOPK_MAX) return -1;
  if (!igmc_topk_fits(k, B)) return -2;
  const size_t smem = merge_smem(k, B);
  if (smem > 48 * 1024)
    cudaFuncSetAttribute(k_topk_merge, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  k_topk_merge<<<B, MERGE_THREADS, smem, (cudaStream_t)stream>>>(preds, K, B, tag, items, k, top_score, top_item);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_score_scatter(const float* preds, int K, int B, const int64_t* tag, float* scores, void* stream) {
  if (K < 1 || B <= 0) return -1;
  k_score_scatter<<<(B + MERGE_THREADS - 1) / MERGE_THREADS, MERGE_THREADS, 0, (cudaStream_t)stream>>>(preds, K, B,
                                                                                                     tag, scores);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
