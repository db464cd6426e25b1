// Cached top-k lists kept exact across rating-graph updates (igmc_b200/recommend.py: RecommendationCache).
//
// With h = 1 a rating edit (a, b) can change the enclosing subgraph of (u, v) only when u = a, v = b, or u rated b and
// a rated v; every other pair keeps its score bit for bit (DESIGN.md §19).  A repair rescores just those pairs:
//   k_rp_candmask  one CTA: the bitmap of the candidate items (a shared list, or every item)
//   k_rp_mark      one CTA per slot of a chunk: the slot's row of the user-by-item bitmap (integer atomicOr), its
//                  rated items cleared (exclude_rated), masked by the candidates; the rescore and candidate counts
//   k_rp_scan      one CTA: the chunk's counts onto user_off (int64, carried over the chunks) and the two totals
//   k_rp_write     one CTA per slot of a chunk: the marked items, ascending, at user_off[j] (a popcount scan)
//   k_cache_invalidate  one thread per slot: the rescored items out of the cached prefix, and the threshold key
//   k_cache_settle      one CTA: the exact depth of every merged list under the threshold, the padding past it, and
//                       the ascending list of slots that fall back to a full re-rank
// No float atomics and one writer per output: runs are bit-identical.  Twins: igmc_b200/recommend.py::
// rescore_plan_host, cache_invalidate_host, cache_settle_host.
#include "common.cuh"
#include "topk_merge.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int MARK_THREADS = 256;
constexpr int SCAN_THREADS = 1024;
constexpr int SLOT_THREADS = 256;
constexpr long long RESCORE_WS_DEFAULT = 256ll << 20;

__host__ __device__ __forceinline__ int bitmap_words(int num_items) { return (num_items + 31) >> 5; }

// the bits of word w that name items below num_items
__device__ __forceinline__ uint32_t word_mask(int w, int num_items) {
  const int rest = num_items - (w << 5);
  return rest >= 32 ? 0xffffffffu : (1u << rest) - 1u;
}

// igmc_rescore_plan's workspace for chunks of `chunk` slots: the candidate bitmap, per slot two counts, the bitmap rows
struct PlanLayout {
  uint32_t* cmask;
  int* cnt;
  uint32_t* bits;
};

size_t plan_fixed(int W) { return align256((size_t)W * 4) + 512; }
size_t plan_per_slot(int W) { return (size_t)W * 4 + 8; }

PlanLayout plan_layout(void* base, int W, int chunk) {
  unsigned char* b = static_cast<unsigned char*>(base);
  PlanLayout L;
  L.cmask = reinterpret_cast<uint32_t*>(b);
  L.cnt = reinterpret_cast<int*>(b + align256((size_t)W * 4));
  L.bits = reinterpret_cast<uint32_t*>(b + align256((size_t)W * 4) + align256((size_t)chunk * 8));
  return L;
}

// the slots a workspace of ws_bytes holds at once (0: not even one)
long long plan_chunk(long long ws_bytes, int W, int U) {
  const long long room = ws_bytes - (long long)plan_fixed(W);
  if (room < (long long)plan_per_slot(W)) return 0;
  return min((long long)max(U, 1), room / (long long)plan_per_slot(W));
}

__global__ void __launch_bounds__(SCAN_THREADS)
k_rp_candmask(const int32_t* __restrict__ cand, int num_cand, int num_items, uint32_t* __restrict__ cmask, int* err) {
  const int W = bitmap_words(num_items);
  for (int w = threadIdx.x; w < W; w += blockDim.x) cmask[w] = cand ? 0u : word_mask(w, num_items);
  if (!cand) return;
  __syncthreads();
  for (int t = threadIdx.x; t < num_cand; t += blockDim.x) {
    const int v = cand[t];
    if (v < 0 || v >= num_items) {
      igmc_set_err(err, IGMC_ERR_CANDIDATES);
      continue;
    }
    atomicOr(&cmask[v >> 5], 1u << (v & 31));
  }
}

// slot j = j0 + blockIdx.x, user u: bit v of its row is set for v = b_i, and for every v in row(a_i) when u rated
// b_i; a_i = u sets every bit.  Then the rated items of u are cleared (exclude_rated) and the row is masked by the
// candidates.  cnt[2t] = the marked candidates, cnt[2t+1] = the slot's candidates; full[j] = 1 when they are equal.
__global__ void __launch_bounds__(MARK_THREADS)
k_rp_mark(igmc_csr_t G, const int32_t* __restrict__ users, int j0, const int32_t* __restrict__ edit_u,
          const int32_t* __restrict__ edit_v, int E, int exclude_rated, const uint32_t* __restrict__ cmask,
          uint32_t* __restrict__ bits, int* __restrict__ cnt, uint8_t* __restrict__ full, int* err) {
  __shared__ int ws[33];
  __shared__ int s_all;
  const int t = blockIdx.x, j = j0 + t, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int W = bitmap_words(G.num_items);
  uint32_t* row = bits + (size_t)t * W;
  for (int w = threadIdx.x; w < W; w += blockDim.x) row[w] = 0u;
  if (threadIdx.x == 0) s_all = 0;
  const int u = users[j];
  const bool user_ok = u >= 0 && u < G.num_users;
  if (!user_ok && threadIdx.x == 0) igmc_set_err(err, IGMC_ERR_CANDIDATES);
  __syncthreads();
  const int r0 = user_ok ? G.row_ptr[u] : 0, nr = user_ok ? G.row_ptr[u + 1] - r0 : 0;
  if (user_ok) {
    for (int i = warp; i < E; i += blockDim.x >> 5) {
      const int a = edit_u[i], b = edit_v[i];
      if (a < 0 || a >= G.num_users || b < 0 || b >= G.num_items) {
        if (lane == 0) igmc_set_err(err, IGMC_ERR_CANDIDATES);
        continue;
      }
      if (a == u) {
        if (lane == 0) s_all = 1;
        continue;
      }
      if (lane == 0) atomicOr(&row[b >> 5], 1u << (b & 31));
      if (find_sorted(G.col_idx + r0, nr, b) < 0) continue;   // u did not rate b: no bridge through (a, b)
      for (int e = G.row_ptr[a] + lane; e < G.row_ptr[a + 1]; e += 32) {
        const int v = G.col_idx[e];
        atomicOr(&row[v >> 5], 1u << (v & 31));
      }
    }
  }
  __syncthreads();
  if (s_all)
    for (int w = threadIdx.x; w < W; w += blockDim.x) row[w] = word_mask(w, G.num_items);
  __syncthreads();
  int rated = 0;   // u's rated items among the candidates
  if (exclude_rated) {
    for (int e = threadIdx.x; e < nr; e += blockDim.x) {
      const int v = G.col_idx[r0 + e];
      atomicAnd(&row[v >> 5], ~(1u << (v & 31)));
      rated += (cmask[v >> 5] >> (v & 31)) & 1u;
    }
  }
  __syncthreads();
  int marked = 0, cands = 0;
  for (int w = threadIdx.x; w < W; w += blockDim.x) {
    const uint32_t x = row[w] & cmask[w];
    row[w] = x;
    marked += __popc(x);
    cands += user_ok ? __popc(cmask[w]) : 0;
  }
  marked = block_sum_i(marked, ws);
  cands = block_sum_i(cands, ws) - block_sum_i(rated, ws);
  if (threadIdx.x == 0) {
    cnt[2 * t] = marked;
    cnt[2 * t + 1] = cands;
    full[j] = marked == cands;
  }
}

// slots [j0, j0 + n): user_off[j] = user_off[j0] (0 for the first chunk) + the exclusive prefix of the marked counts,
// user_off[j0 + n] the running total; totals = (user_off[j0 + n], the running candidate total)
__global__ void __launch_bounds__(SCAN_THREADS)
k_rp_scan(int j0, int n, const int* __restrict__ cnt, int64_t* __restrict__ user_off, int64_t* __restrict__ totals) {
  __shared__ long long ws[33];
  long long carry = j0 ? user_off[j0] : 0, carry_c = j0 ? totals[1] : 0;
  __syncthreads();
  for (int base = 0; base < n; base += blockDim.x) {
    const int t = base + threadIdx.x;
    long long tot, tot_c;
    const long long off = block_excl_scan_ll(t < n ? cnt[2 * t] : 0, ws, &tot);
    block_excl_scan_ll(t < n ? cnt[2 * t + 1] : 0, ws, &tot_c);
    if (t < n) user_off[j0 + t] = carry + off;
    carry += tot;
    carry_c += tot_c;
  }
  if (threadIdx.x == 0) {
    user_off[j0 + n] = carry;
    totals[0] = carry;
    totals[1] = carry_c;
  }
}

// slot j0 + blockIdx.x: the set bits of its row, ascending, from out[user_off[j]] on (positions past out_cap set the
// error word and are not written)
__global__ void __launch_bounds__(MARK_THREADS)
k_rp_write(int j0, int num_items, const uint32_t* __restrict__ bits, const int64_t* __restrict__ user_off,
           int32_t* __restrict__ out, long long out_cap, int* err) {
  __shared__ int ws[33];
  const int t = blockIdx.x, W = bitmap_words(num_items);
  const uint32_t* row = bits + (size_t)t * W;
  const long long o0 = user_off[j0 + t];
  block_scan_chunks(
      W, ws, [&](int w) { return __popc(row[w]); },
      [&](int w, int prefix) {
        uint32_t x = row[w];
        long long o = o0 + prefix;
        while (x) {
          const int bit = __ffs(x) - 1;
          x &= x - 1;
          if (o < out_cap) out[o] = (w << 5) + bit;
          else igmc_set_err(err, IGMC_ERR_CANDIDATES);
          ++o;
        }
      });
}

// one thread per slot: the prefix (the leading entries with an item >= 0) without the slot's rescored items (a fully
// rescored slot keeps nothing), compacted in order and padded; the threshold key = the old last prefix entry, item -1 (none) for a complete or fully
// rescored slot, -2 for an empty prefix of a slot that is not complete
__global__ void __launch_bounds__(SLOT_THREADS)
k_cache_invalidate(int U, int D, const int64_t* __restrict__ user_off, const int32_t* __restrict__ resc,
                   const uint8_t* __restrict__ full, const uint8_t* __restrict__ complete, float* __restrict__ top_s,
                   int64_t* __restrict__ top_i, float* __restrict__ thr_s, int64_t* __restrict__ thr_i) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= U) return;
  float* s = top_s + (size_t)j * D;
  int64_t* it = top_i + (size_t)j * D;
  int n = 0;
  while (n < D && it[n] >= 0) ++n;
  if (complete[j] || full[j]) {
    thr_i[j] = -1;
    thr_s[j] = -INFINITY;
  } else if (n == 0) {
    thr_i[j] = -2;
    thr_s[j] = -INFINITY;
  } else {
    thr_i[j] = it[n - 1];
    thr_s[j] = s[n - 1];
  }
  if (full[j]) n = 0;   // every candidate is rescored, and the user's own edits may have taken some out of the set
  const int32_t* seg = resc + user_off[j];
  const long long m = user_off[j + 1] - user_off[j];
  int w = 0;
  for (int e = 0; e < n; ++e) {
    const long long v = it[e];
    long long lo = 0, hi = m;
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (seg[mid] < v) lo = mid + 1; else hi = mid;
    }
    if (lo < m && seg[lo] == v) continue;
    const float x = s[e];
    s[w] = x;
    it[w] = v;
    ++w;
  }
  for (int e = w; e < D; ++e) {
    s[e] = -INFINITY;
    it[e] = -1;
  }
}

// one CTA: per slot the exact depth of its merged list (threshold none: every entry; -2: none; else the leading
// entries not ranked after the threshold), the padding past it, complete[j] = (no threshold and fewer than D
// entries), and the slots with a threshold and fewer than k exact entries listed ascending in redo, their count in
// *redo_count
__global__ void __launch_bounds__(SCAN_THREADS)
k_cache_settle(int U, int D, int k, const float* __restrict__ thr_s, const int64_t* __restrict__ thr_i,
               float* __restrict__ top_s, int64_t* __restrict__ top_i, uint8_t* __restrict__ complete,
               int32_t* __restrict__ redo, int32_t* __restrict__ redo_count) {
  __shared__ int ws[33];
  int need = 0;   // the flag of the slot this thread settled last (block_scan_chunks: in(j), then out(j) by one thread)
  const int total = block_scan_chunks(
      U, ws,
      [&](int j) {
        float* s = top_s + (size_t)j * D;
        int64_t* it = top_i + (size_t)j * D;
        const long long ti = thr_i[j];
        const float ts = thr_s[j];
        int d = 0;
        if (ti != -2)
          while (d < D && it[d] >= 0 && (ti == -1 || !ranks_before(ts, ti, s[d], it[d], 1.f))) ++d;
        for (int e = d; e < D; ++e) {
          s[e] = -INFINITY;
          it[e] = -1;
        }
        complete[j] = ti == -1 && d < D;
        need = ti != -1 && d < k;
        return need;
      },
      [&](int j, int prefix) {
        if (need) redo[prefix] = j;
      });
  if (threadIdx.x == 0) *redo_count = total;
}

}  // namespace

extern "C" int igmc_rescore_plan_ws_bytes(int num_query, int num_items, int64_t bound, int64_t* bytes, int* chunk) {
  if (!bytes || num_query < 0 || num_items < 1) return -1;
  const int W = bitmap_words(num_items);
  const long long want = (long long)plan_fixed(W) + (long long)max(num_query, 1) * (long long)plan_per_slot(W);
  const long long b = min(want, max(bound > 0 ? (long long)bound : RESCORE_WS_DEFAULT,
                                    (long long)(plan_fixed(W) + plan_per_slot(W))));
  *bytes = b;
  if (chunk) *chunk = (int)plan_chunk(b, W, num_query);
  return 0;
}

extern "C" int igmc_rescore_plan(const igmc_csr_t* G, const int32_t* users, int num_query, const int32_t* edit_u,
                                 const int32_t* edit_v, int num_edits, const int32_t* cand, int num_cand,
                                 int exclude_rated, void* ws, int64_t ws_bytes, int64_t* user_off, int32_t* out,
                                 int64_t out_cap, uint8_t* full, int64_t* totals, int* err, void* stream) {
  if (!G || G->num_items < 1 || num_query < 0 || num_edits < 0 || num_cand < 0 || out_cap < 0) return -1;
  if (!user_off || !totals || (num_query > 0 && (!users || !full || !ws)) || (num_edits > 0 && (!edit_u || !edit_v)))
    return -1;
  if (cand && num_cand == 0) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  if (num_query == 0) {
    cudaMemsetAsync(user_off, 0, sizeof(int64_t), st);
    cudaMemsetAsync(totals, 0, 2 * sizeof(int64_t), st);
    IGMC_CUDA_CHECK_LAUNCH();
    return 0;
  }
  const int W = bitmap_words(G->num_items);
  const long long chunk = plan_chunk(ws_bytes, W, num_query);
  if (chunk < 1) return -2;
  if (out_cap > 0 && !out) return -1;
  const PlanLayout L = plan_layout(ws, W, (int)chunk);
  k_rp_candmask<<<1, SCAN_THREADS, 0, st>>>(cand, num_cand, G->num_items, L.cmask, err);
  IGMC_CUDA_CHECK_LAUNCH();
  for (int j0 = 0; j0 < num_query; j0 += (int)chunk) {
    const int n = (int)min(chunk, (long long)(num_query - j0));
    k_rp_mark<<<n, MARK_THREADS, 0, st>>>(*G, users, j0, edit_u, edit_v, num_edits, exclude_rated, L.cmask, L.bits,
                                          L.cnt, full, err);
    IGMC_CUDA_CHECK_LAUNCH();
    k_rp_scan<<<1, SCAN_THREADS, 0, st>>>(j0, n, L.cnt, user_off, totals);
    IGMC_CUDA_CHECK_LAUNCH();
    k_rp_write<<<n, MARK_THREADS, 0, st>>>(j0, G->num_items, L.bits, user_off, out, out_cap, err);
    IGMC_CUDA_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int igmc_cache_invalidate(int num_query, int depth, const int64_t* user_off, const int32_t* resc,
                                     const uint8_t* full, const uint8_t* complete, float* top_score,
                                     int64_t* top_item, float* thr_score, int64_t* thr_item, void* stream) {
  if (num_query < 0 || depth < 1 || depth > IGMC_TOPK_MAX) return -1;
  if (num_query == 0) return 0;
  if (!user_off || !full || !complete || !top_score || !top_item || !thr_score || !thr_item) return -1;
  k_cache_invalidate<<<(num_query + SLOT_THREADS - 1) / SLOT_THREADS, SLOT_THREADS, 0, (cudaStream_t)stream>>>(
      num_query, depth, user_off, resc, full, complete, top_score, top_item, thr_score, thr_item);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_cache_settle(int num_query, int depth, int k, const float* thr_score, const int64_t* thr_item,
                                 float* top_score, int64_t* top_item, uint8_t* complete, int32_t* redo,
                                 int32_t* redo_count, void* stream) {
  if (num_query < 0 || depth < 1 || depth > IGMC_TOPK_MAX || k < 1 || k > depth || !redo_count) return -1;
  if (num_query > 0 && (!thr_score || !thr_item || !top_score || !top_item || !complete || !redo)) return -1;
  k_cache_settle<<<1, SCAN_THREADS, 0, (cudaStream_t)stream>>>(num_query, depth, k, thr_score, thr_item, top_score,
                                                               top_item, complete, redo, redo_count);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
