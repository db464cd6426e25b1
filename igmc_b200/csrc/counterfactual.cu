// Counterfactual explanations of a recommendation (igmc_b200/recommend.py: counterfactual).
//
// Query (u, X, Y): the smallest set R of u's own ratings, found greedily, whose removal puts item X behind the rival Y.
// A run is a base pass and at most max_removals trial passes over the inference engine's pipeline.  Every trial is
// scored exactly: its two pairs (u, X) and (u, Y) are extracted in session mode with u's row without the trial's
// removals as the target row, so a score is bit for bit the score on the graph with those ratings deleted.
//   k_cf_pairs   one CTA: positions [cursor, cursor + B) -> (trial, side), the pairs for igmc_extract_sessions and
//                each slot's trial-row length, scanned into the slots' row pointers; then cursor += B
//   k_cf_rows    one CTA per slot: u's graph row without R and without the trial's candidate, in row order
//   k_cf_select  one CTA per query after a pass: the best trial by a fixed-order block reduction, appended to R
// The candidate of trial c is the c-th position of u's row not in R, found by the rank-skip search of
// igmc_candidate_pairs over R kept ascending.  The selection order is a strict total order (items are distinct within a
// row), so nothing depends on batch boundaries or on the other queries of the run.
// Twins: igmc_b200/recommend.py::counterfactual_pairs_host / counterfactual_select_host.
#include "common.cuh"
#include "topk_merge.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int PAIR_THREADS = 512;
constexpr int ROW_THREADS = 256;
constexpr int SELECT_THREADS = 256;   // a power of two: the selection's tree reduction halves it

// slot i of a pass: position p = pos + i of the 2T positions (past them: the last one again, tag -1)
struct Slot {
  int u, v, len;
  long long tag;
};

__device__ __forceinline__ Slot cf_slot(const igmc_csr_t& G, const igmc_counterfactual_t& Q,
                                        const int64_t* __restrict__ offsets, int step, long long p, long long P2,
                                        int* err) {
  Slot s = {0, 0, 0, -1};
  if (P2 <= 0) {   // a pass without trials is never launched
    igmc_set_err(err, IGMC_ERR_CANDIDATES);
    return s;
  }
  const bool real = p < P2;
  if (!real) p = P2 - 1;
  const long long trial = p >> 1;
  const int q = owner(offsets, Q.num_query, trial);
  int u = Q.users[q], v = (p & 1) ? Q.rivals[q] : Q.items[q];
  if (u < 0 || u >= G.num_users || v < 0 || v >= G.num_items) {
    igmc_set_err(err, IGMC_ERR_CANDIDATES);
    u = 0;
    v = 0;
  }
  const int kept = G.row_ptr[u + 1] - G.row_ptr[u] - Q.size[q];
  if (step > 0 && trial - offsets[q] >= kept) igmc_set_err(err, IGMC_ERR_CANDIDATES);   // not the plan's row
  s.u = u;
  s.v = v;
  s.len = max(kept - (step > 0 ? 1 : 0), 0);
  s.tag = real ? p : -1;
  return s;
}

__global__ void __launch_bounds__(PAIR_THREADS)
k_cf_pairs(igmc_csr_t G, igmc_counterfactual_t Q, const int64_t* __restrict__ offsets, int step,
           int64_t* __restrict__ cursor, int B, int32_t* __restrict__ links_u, int32_t* __restrict__ links_v,
           int64_t* __restrict__ pair_id, int64_t* __restrict__ tag, int32_t* __restrict__ row_users,
           int32_t* __restrict__ row_ptr, int row_cap, int32_t* __restrict__ sess, int* err) {
  __shared__ long long s_pos;
  __shared__ int ws[33];
  if (threadIdx.x == 0) s_pos = *cursor;
  __syncthreads();
  const long long pos = s_pos, P2 = 2 * offsets[Q.num_query];
  const int total = block_scan_chunks(
      B, ws,
      [&](int i) {
        const Slot s = cf_slot(G, Q, offsets, step, pos + i, P2, err);
        links_u[i] = s.u;
        links_v[i] = s.v;
        pair_id[i] = (int64_t)s.u * G.num_items + s.v;
        tag[i] = s.tag;
        row_users[i] = s.u;
        sess[i] = i;
        return s.len;
      },
      [&](int i, int prefix) { row_ptr[i] = prefix; });
  if (threadIdx.x == 0) {
    row_ptr[B] = total;
    if (total > row_cap) igmc_set_err(err, IGMC_ERR_CANDIDATES);
    *cursor = pos + B;
  }
}

// slot g's trial row; runs after k_cf_pairs, so the slot's position is *cursor - B + g
__global__ void __launch_bounds__(ROW_THREADS)
k_cf_rows(igmc_csr_t G, igmc_counterfactual_t Q, const int64_t* __restrict__ offsets, int step,
          const int64_t* __restrict__ cursor, int B, const int32_t* __restrict__ row_users,
          const int32_t* __restrict__ row_ptr, int row_cap, int32_t* __restrict__ row_col,
          uint8_t* __restrict__ row_rating) {
  __shared__ int32_t sr[IGMC_COUNTERFACTUAL_MAX];
  const int g = blockIdx.x;
  const long long P2 = 2 * offsets[Q.num_query];
  const int o0 = row_ptr[g], len = row_ptr[g + 1] - o0;
  if (P2 <= 0 || o0 + len > row_cap) return;   // k_cf_pairs set the error word
  const long long p = *cursor - B + g;
  const long long trial = (p < P2 ? p : P2 - 1) >> 1;
  const int q = owner(offsets, Q.num_query, trial);
  const int n = min(Q.size[q], Q.max_removals);
  for (int t = threadIdx.x; t < n; t += blockDim.x) sr[t] = Q.removed[(size_t)q * Q.max_removals + t];
  __syncthreads();
  const long long c = trial - offsets[q];
  const long long cand = step > 0 ? c + rank_skip(sr, n, c) : -1;
  const int u = row_users[g], r0 = G.row_ptr[u], deg = G.row_ptr[u + 1] - r0;
  for (int k = threadIdx.x; k < deg; k += blockDim.x) {
    if (k == cand) continue;
    int lo = 0, hi = n;   // the removed positions below k
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (sr[mid] < k) lo = mid + 1; else hi = mid;
    }
    if (lo < n && sr[lo] == k) continue;
    const long long o = k - lo - (cand >= 0 && cand < k ? 1 : 0);
    if (o < len) {
      row_col[o0 + o] = G.col_idx[r0 + k];
      row_rating[o0 + o] = G.rating[r0 + k];
    }
  }
}

// one trial of the selection: c < 0 is no trial, after every other
struct Trial {
  int flip;       // X behind Y under the trial
  float margin;   // s(u, X) - s(u, Y)
  int item, c;
};

// the selection order: flips first, then margin ascending with NaN after every number, then item ascending
__device__ __forceinline__ bool trial_before(const Trial& a, const Trial& b) {
  if (a.c < 0) return false;
  if (b.c < 0) return true;
  if (a.flip != b.flip) return a.flip > b.flip;
  const bool an = isnan(a.margin), bn = isnan(b.margin);
  if (an != bn) return bn;
  if (!an && a.margin != b.margin) return a.margin < b.margin;
  return a.item < b.item;
}

__global__ void __launch_bounds__(SELECT_THREADS)
k_cf_select(igmc_csr_t G, igmc_counterfactual_t Q, const int64_t* __restrict__ offsets,
            const float* __restrict__ scores, int step, int32_t* __restrict__ count, uint8_t* __restrict__ found,
            int32_t* __restrict__ out_item, int32_t* __restrict__ out_rating, float* __restrict__ score,
            float* __restrict__ rival_score, int* err) {
  __shared__ int32_t sr[IGMC_COUNTERFACTUAL_MAX];
  __shared__ Trial red[SELECT_THREADS];
  const int q = blockIdx.x, M = Q.max_removals;
  const long long o = offsets[q], n = offsets[q + 1] - o;
  const int u = Q.users[q], X = Q.items[q], Y = Q.rivals[q];
  const bool bad = u < 0 || u >= G.num_users || X < 0 || X >= G.num_items || Y < 0 || Y >= G.num_items;
  const int t = Q.size[q];
  const int r0 = bad ? 0 : G.row_ptr[u], deg = bad ? 0 : G.row_ptr[u + 1] - r0;
  if (n <= 0 || bad || (step > 0 && (t >= M || n != deg - t))) {   // no trials, or not the plan's
    if (threadIdx.x == 0) {
      if (n > 0) igmc_set_err(err, IGMC_ERR_CANDIDATES);
      count[q] = 0;
    }
    return;
  }
  float* sc = score + (size_t)q * (M + 1);
  float* rv = rival_score + (size_t)q * (M + 1);
  if (step == 0) {
    if (threadIdx.x == 0) {
      const float sx = scores[2 * o], sy = scores[2 * o + 1];
      sc[0] = sx;
      rv[0] = sy;
      const bool behind = ranks_before(sy, Y, sx, X, 1.f);
      found[q] = behind;
      count[q] = behind ? 0 : deg;
    }
    return;
  }
  for (int j = threadIdx.x; j < t; j += blockDim.x) sr[j] = Q.removed[(size_t)q * M + j];
  __syncthreads();
  Trial best = {0, 0.f, 0, -1};
  for (long long c = threadIdx.x; c < n; c += blockDim.x) {
    const long long pos = c + rank_skip(sr, t, c);
    const float sx = scores[2 * (o + c)], sy = scores[2 * (o + c) + 1];
    const Trial cur = {ranks_before(sy, Y, sx, X, 1.f) ? 1 : 0, __fsub_rn(sx, sy), G.col_idx[r0 + pos], (int)c};
    if (trial_before(cur, best)) best = cur;
  }
  red[threadIdx.x] = best;
  __syncthreads();
  for (int w = SELECT_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w && trial_before(red[threadIdx.x + w], red[threadIdx.x])) red[threadIdx.x] = red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const Trial b = red[0];
    const int pos = (int)(b.c + rank_skip(sr, t, b.c));
    int32_t* r = Q.removed + (size_t)q * M;   // insert pos, keeping R ascending
    int j = t;
    for (; j > 0 && sr[j - 1] > pos; --j) r[j] = sr[j - 1];
    r[j] = pos;
    out_item[(size_t)q * M + t] = b.item;
    out_rating[(size_t)q * M + t] = G.rating[r0 + pos];
    sc[t + 1] = scores[2 * (o + b.c)];
    rv[t + 1] = scores[2 * (o + b.c) + 1];
    Q.size[q] = t + 1;
    found[q] = (uint8_t)b.flip;
    count[q] = (b.flip || t + 1 == M || deg == t + 1) ? 0 : deg - t - 1;
  }
}

bool query_ok(const igmc_counterfactual_t* Q) {
  return Q && Q->users && Q->items && Q->rivals && Q->size && Q->removed && Q->num_query > 0 &&
         Q->max_removals >= 1 && Q->max_removals <= IGMC_COUNTERFACTUAL_MAX;
}

}  // namespace

extern "C" int igmc_counterfactual_pairs(const igmc_csr_t* G, const igmc_counterfactual_t* Q, const int64_t* offsets,
                                         int step, int64_t* cursor, int B, int32_t* links_u, int32_t* links_v,
                                         int64_t* pair_id, int64_t* tag, int32_t* row_users, int32_t* row_ptr,
                                         int32_t* row_col, uint8_t* row_rating, int row_cap, int32_t* sess, int* err,
                                         void* stream) {
  if (!G || !query_ok(Q) || !offsets || !cursor || B <= 0 || step < 0 || row_cap < 0) return -1;
  if (!links_u || !links_v || !pair_id || !tag || !row_users || !row_ptr || !sess) return -1;
  if (row_cap > 0 && (!row_col || !row_rating)) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  k_cf_pairs<<<1, PAIR_THREADS, 0, st>>>(*G, *Q, offsets, step, cursor, B, links_u, links_v, pair_id, tag, row_users,
                                         row_ptr, row_cap, sess, err);
  IGMC_CUDA_CHECK_LAUNCH();
  k_cf_rows<<<B, ROW_THREADS, 0, st>>>(*G, *Q, offsets, step, cursor, B, row_users, row_ptr, row_cap, row_col,
                                       row_rating);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_counterfactual_select(const igmc_csr_t* G, const igmc_counterfactual_t* Q, const int64_t* offsets,
                                          const float* trial_scores, int step, int32_t* count, uint8_t* found,
                                          int32_t* out_item, int32_t* out_rating, float* score, float* rival_score,
                                          int* err, void* stream) {
  if (!G || !query_ok(Q) || !offsets || !trial_scores || step < 0) return -1;
  if (!count || !found || !out_item || !out_rating || !score || !rival_score) return -1;
  k_cf_select<<<Q->num_query, SELECT_THREADS, 0, (cudaStream_t)stream>>>(*G, *Q, offsets, trial_scores, step, count,
                                                                          found, out_item, out_rating, score,
                                                                          rival_score, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
