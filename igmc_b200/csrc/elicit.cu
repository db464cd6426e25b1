// Question impact for rating sessions (igmc_b200/recommend.py: elicit, question_impact).
//
// A question asks session s about an item q not in its row; its answers are the rating labels a = 0..A-1.  Each
// (s, q, a) is scored exactly: the session's targets t are extracted in session mode with s's row plus (q, a) as the
// target row, so a score is bit for bit predict_sessions of a session with s's edits and the edit (q, a + 1).
// A unit (s, q) takes U = A * W consecutive batch positions, answer major (position i: answer i / W, target slot
// i % W); a batch of B positions holds G = B / U units and positions G*U..B-1 are padding:
//   k_el_pairs  one CTA: the B positions -> (users[s], target, pair id, tag, trial row), and the exclusive scan of the
//               G*A trial-row lengths deg(s) + 1 into row_ptr
//   k_el_rows   one CTA per trial row g*A + a: s's session row with (q, a) inserted at q's sorted position
//   k_el_stats  one thread per unit after the forward: impact and answer_mean in fp64, rounded once
// Twins: igmc_b200/recommend.py::elicit_pairs_host / elicit_stats_host.
#include "common.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int PAIR_THREADS = 512;
constexpr int ROW_THREADS = 128;
constexpr int STATS_THREADS = 128;

// unit g of the batch: its session and question (ids outside the sessions / items set the error word and read as 0)
__device__ __forceinline__ void unit_at(const igmc_sessions_t& S, int num_items, const int32_t* __restrict__ unit_s,
                                        const int32_t* __restrict__ unit_q, int g, int* s, int* q, int* err) {
  *s = unit_s[g];
  *q = unit_q[g];
  if (*s < 0 || *s >= S.num_sessions || *q < 0 || *q >= num_items) {
    igmc_set_err(err, IGMC_ERR_CANDIDATES);
    *s = 0;
    *q = 0;
  }
}

__global__ void __launch_bounds__(PAIR_THREADS)
k_el_pairs(igmc_sessions_t S, int num_items, int A, const int32_t* __restrict__ targets, int W, int per_session,
           const int32_t* __restrict__ unit_s, const int32_t* __restrict__ unit_q, const int64_t* __restrict__ unit_tag,
           int B, int32_t* __restrict__ links_u, int32_t* __restrict__ links_v, int64_t* __restrict__ pair_id,
           int64_t* __restrict__ tag, int32_t* __restrict__ row_ptr, int row_cap, int32_t* __restrict__ sess,
           int* err) {
  __shared__ int ws[33];
  const int U = A * W, G = B / U;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const bool real = i < G * U;
    const int g = real ? i / U : 0, a = real ? (i % U) / W : 0;
    int s, q;
    unit_at(S, num_items, unit_s, unit_q, g, &s, &q, err);
    int t = real ? targets[(size_t)(per_session ? s : 0) * W + i % W] : -1;
    if (t < -1 || t >= num_items) {
      igmc_set_err(err, IGMC_ERR_CANDIDATES);
      t = -1;
    }
    const int u = S.users[s], v = t >= 0 ? t : q;   // an empty slot or the tail: a valid pair, tag -1
    links_u[i] = u;
    links_v[i] = v;
    pair_id[i] = (int64_t)u * num_items + v;
    tag[i] = t >= 0 ? unit_tag[g] : -1;
    sess[i] = g * A + a;
  }
  const int total = block_scan_chunks(
      G * A, ws,
      [&](int r) {
        int s, q;
        unit_at(S, num_items, unit_s, unit_q, r / A, &s, &q, err);
        return S.row_ptr[s + 1] - S.row_ptr[s] + 1;
      },
      [&](int r, int prefix) { row_ptr[r] = min(prefix, row_cap); });   // rows past row_cap are cut short
  if (threadIdx.x == 0) {
    row_ptr[G * A] = min(total, row_cap);
    if (total > row_cap) igmc_set_err(err, IGMC_ERR_CANDIDATES);
  }
}

// trial row r = g * A + a: session row s with (q, a) inserted before the first item > q
__global__ void __launch_bounds__(ROW_THREADS)
k_el_rows(igmc_sessions_t S, int num_items, int A, const int32_t* __restrict__ unit_s,
          const int32_t* __restrict__ unit_q, const int32_t* __restrict__ row_ptr, int32_t* __restrict__ row_users,
          int32_t* __restrict__ row_col, uint8_t* __restrict__ row_rating, int* err) {
  const int r = blockIdx.x, a = r % A;
  int s, q;
  unit_at(S, num_items, unit_s, unit_q, r / A, &s, &q, nullptr);   // k_el_pairs set the error word
  const int o0 = row_ptr[r], len = row_ptr[r + 1] - o0;
  const int r0 = S.row_ptr[s], deg = S.row_ptr[s + 1] - r0;
  int lo = 0, hi = deg;   // q's position: the items below it
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (S.col_idx[r0 + mid] < q) lo = mid + 1; else hi = mid;
  }
  if (threadIdx.x == 0) {
    row_users[r] = S.users[s];
    if (lo < deg && S.col_idx[r0 + lo] == q) igmc_set_err(err, IGMC_ERR_CANDIDATES);   // already rated
    if (lo < len) {
      row_col[o0 + lo] = q;
      row_rating[o0 + lo] = (uint8_t)a;
    }
  }
  for (int k = threadIdx.x; k < deg; k += blockDim.x) {
    const int o = k < lo ? k : k + 1;
    if (o < len) {
      row_col[o0 + o] = S.col_idx[r0 + k];
      row_rating[o0 + o] = S.rating[r0 + k];
    }
  }
}

// unit g: x_a(w) = the fp32 checkpoint mean of position g*U + a*W + w for the real slots w (tag >= 0); in fp64, in
// slot order and without fma contraction: impact = sum_w (max_a x - min_a x) / n, answer_mean[a] = sum_w x_a(w) / n,
// each rounded once.  A NaN score makes the impact NaN (and its answer's mean, by the sum).
__global__ void __launch_bounds__(STATS_THREADS)
k_el_stats(const float* __restrict__ preds, int K, int B, int A, int W, const int64_t* __restrict__ tag,
           float* __restrict__ key, float* __restrict__ impact, float* __restrict__ answer_mean) {
  const int U = A * W, G = B / U;
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const int i0 = g * U;
  long long t = -1;
  int n = 0;
  double sum = 0.0;
  bool nan = false;
  for (int w = 0; w < W; ++w) {
    if (tag[i0 + w] < 0) continue;
    t = tag[i0 + w];
    ++n;
    double mx = 0.0, mn = 0.0;
    for (int a = 0; a < A; ++a) {
      const float x = ckpt_mean(preds, K, B, i0 + a * W + w);
      nan |= isnan(x);
      mx = a == 0 ? (double)x : fmax(mx, (double)x);
      mn = a == 0 ? (double)x : fmin(mn, (double)x);
    }
    sum = __dadd_rn(sum, __dsub_rn(mx, mn));
  }
  const float imp = nan ? __int_as_float(0x7fc00000) : (float)__ddiv_rn(sum, (double)max(n, 1));
  if (key) key[g] = imp;
  if (t < 0 || !impact) return;
  impact[t] = imp;
  for (int a = 0; a < A; ++a) {
    double m = 0.0;
    for (int w = 0; w < W; ++w)
      if (tag[i0 + w] >= 0) m = __dadd_rn(m, (double)ckpt_mean(preds, K, B, i0 + a * W + w));
    answer_mean[(size_t)t * A + a] = (float)__ddiv_rn(m, (double)n);
  }
}

bool layout_ok(int A, int W, int B) { return A >= 1 && A <= 256 && W >= 1 && (long long)A * W <= B; }

}  // namespace

extern "C" int igmc_elicit_pairs(const igmc_sessions_t* S, int num_items, int A, const int32_t* targets, int W,
                                 int per_session, const int32_t* unit_s, const int32_t* unit_q,
                                 const int64_t* unit_tag, int B, int32_t* links_u, int32_t* links_v, int64_t* pair_id,
                                 int64_t* tag, int32_t* row_users, int32_t* row_ptr, int32_t* row_col,
                                 uint8_t* row_rating, int row_cap, int32_t* sess, int* err, void* stream) {
  if (!S || !S->users || !S->row_ptr || !S->col_idx || !S->rating || S->num_sessions < 1 || num_items < 1 ||
      !layout_ok(A, W, B))
    return -1;
  if (!targets || !unit_s || !unit_q || !unit_tag || !links_u || !links_v || !pair_id || !tag || !row_users ||
      !row_ptr || !sess || row_cap < 0)
    return -1;
  if (row_cap > 0 && (!row_col || !row_rating)) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  k_el_pairs<<<1, PAIR_THREADS, 0, st>>>(*S, num_items, A, targets, W, per_session, unit_s, unit_q, unit_tag, B,
                                         links_u, links_v, pair_id, tag, row_ptr, row_cap, sess, err);
  IGMC_CUDA_CHECK_LAUNCH();
  k_el_rows<<<B / (A * W) * A, ROW_THREADS, 0, st>>>(*S, num_items, A, unit_s, unit_q, row_ptr, row_users, row_col,
                                                      row_rating, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_elicit_stats(const float* preds, int K, int B, int A, int W, const int64_t* tag, float* key,
                                 float* impact, float* answer_mean, void* stream) {
  if (!preds || K < 1 || !layout_ok(A, W, B) || !tag) return -1;
  if (!key && (!impact || !answer_mean)) return -1;
  const int G = B / (A * W);
  k_el_stats<<<(G + STATS_THREADS - 1) / STATS_THREADS, STATS_THREADS, 0, (cudaStream_t)stream>>>(
      preds, K, B, A, W, tag, key, impact, answer_mean);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
