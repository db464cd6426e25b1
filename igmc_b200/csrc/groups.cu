// Group recommendation (igmc_b200/recommend.py: recommend_groups, predict_groups).
//
// A group is up to IGMC_GROUP_MAX users; its score of an item aggregates its members' own pair scores, each bit for bit
// predict_pairs' score (pair id member * num_items + item).  So a group run is an ordinary candidate stream over group
// slots whose units (group, item) expand to one batch position per member:
//   k_gr_offsets  one CTA: per group the summed member degrees and their exclusive scan (the union's upper bound), in
//                 64 bits and saturated at cap
//   k_gr_flags    one CTA per group: every entry of the concatenated member rows flagged when no earlier member rated
//                 the item, and the group's exclusive scan of the flags
//   k_gr_scan     one CTA: row_ptr = the exclusive scan of the union sizes
//   k_gr_write    one CTA per group: each flagged item written at its rank in the union (integer counting, one writer)
//   k_gr_pairs    the B positions of a batch of B / M units: member-major units, empty slots and the tail padding
//   k_gr_stats    one thread per unit after the forward: mean in fp64 / min / max over the real members
// Twins: igmc_b200/recommend.py::group_rows_host / group_pairs_host / group_stats_host.
#include "common.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int ROW_THREADS = 256;
constexpr int PAIR_THREADS = 256;
constexpr int STATS_THREADS = 128;

// member j of group g: a user id, or -1 for an empty slot (an id outside [-1, num_users) sets the error word when
// err != NULL and reads as -1)
__device__ __forceinline__ int member_at(const int32_t* __restrict__ members, int M, int num_users, int g, int j,
                                         int* err) {
  const int m = members[(size_t)g * M + j];
  if (m < -1 || m >= num_users) {
    if (err) igmc_set_err(err, IGMC_ERR_CANDIDATES);
    return -1;
  }
  return m;
}

// the group's member rows in shared memory: start r0[j], length and the prefix cum[j] of the lengths (cum[M] = n).  Up
// to IGMC_GROUP_MAX rows of up to 2^31 - 1 entries each: the prefix is kept in 64 bits, and group_entries only lets a
// group whose n fits the int32 workspace through, so every position below n is an int.
struct GroupRows {
  int r0[IGMC_GROUP_MAX];
  long long cum[IGMC_GROUP_MAX + 1];
};

__device__ __forceinline__ void load_rows(const igmc_csr_t& G, const int32_t* __restrict__ members, int M, int g,
                                          GroupRows& s) {
  if (threadIdx.x < M) {
    const int m = member_at(members, M, G.num_users, g, threadIdx.x, nullptr);
    s.r0[threadIdx.x] = m >= 0 ? G.row_ptr[m] : 0;
    s.cum[threadIdx.x + 1] = m >= 0 ? G.row_ptr[m + 1] - G.row_ptr[m] : 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    s.cum[0] = 0;
    for (int j = 0; j < M; ++j) s.cum[j + 1] += s.cum[j];
  }
  __syncthreads();
}

// entry e of the concatenated rows: its member (the last j with cum[j] <= e) and item
__device__ __forceinline__ int entry_at(const igmc_csr_t& G, const GroupRows& s, int M, int e, int* j) {
  int lo = 0, hi = M;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (s.cum[mid] <= e) lo = mid; else hi = mid;
  }
  *j = lo;
  return G.col_idx[s.r0[lo] + (int)(e - s.cum[lo])];
}

// the group's entries when they fit the workspace (else none: k_gr_offsets set the error word)
__device__ __forceinline__ int group_entries(const GroupRows& s, int M, const int32_t* __restrict__ off, int g,
                                             int cap) {
  return (long long)off[g] + s.cum[M] <= cap ? (int)s.cum[M] : 0;
}

// per group its summed member degrees and their exclusive scan, both in 64 bits (a group's sum reaches 64 * (2^31 - 1))
// and the scan saturated at cap + 1: off[g] = min(prefix, cap), so a group whose entries end past cap reads none
__global__ void __launch_bounds__(ROW_THREADS)
k_gr_offsets(igmc_csr_t G, const int32_t* __restrict__ members, int num_groups, int M, int cap,
             int32_t* __restrict__ off, int* err) {
  __shared__ long long ws[33];
  long long carry = 0;
  for (int base = 0; base < num_groups; base += blockDim.x) {
    const int g = base + threadIdx.x;
    long long n = 0, tot;
    if (g < num_groups)
      for (int j = 0; j < M; ++j) {
        const int m = member_at(members, M, G.num_users, g, j, err);
        if (m >= 0) n += G.row_ptr[m + 1] - G.row_ptr[m];
      }
    const long long ex = block_excl_scan_ll(n, ws, &tot);
    if (g < num_groups) off[g] = (int)min(carry + ex, (long long)cap);
    carry = min(carry + tot, (long long)cap + 1);
  }
  if (threadIdx.x == 0) {
    off[num_groups] = (int)min(carry, (long long)cap);
    if (carry > cap) igmc_set_err(err, IGMC_ERR_CANDIDATES);
  }
}

__global__ void __launch_bounds__(ROW_THREADS)
k_gr_flags(igmc_csr_t G, const int32_t* __restrict__ members, int M, int cap, const int32_t* __restrict__ off,
           int32_t* __restrict__ cnt, int32_t* __restrict__ pre) {
  __shared__ GroupRows s;
  __shared__ int ws[33];
  const int g = blockIdx.x;
  load_rows(G, members, M, g, s);
  const int n = group_entries(s, M, off, g, cap), o = off[g];
  const int total = block_scan_chunks(
      n, ws,
      [&](int e) {
        int j;
        const int x = entry_at(G, s, M, e, &j);
        for (int q = 0; q < j; ++q)
          if (find_sorted(G.col_idx + s.r0[q], (int)(s.cum[q + 1] - s.cum[q]), x) >= 0) return 0;
        return 1;
      },
      [&](int e, int prefix) { pre[o + e] = prefix; });
  if (threadIdx.x == 0) cnt[g] = total;
}

__global__ void __launch_bounds__(ROW_THREADS)
k_gr_scan(const int32_t* __restrict__ cnt, int num_groups, int32_t* __restrict__ row_ptr) {
  __shared__ int ws[33];
  const int total =
      block_scan_chunks(num_groups, ws, [&](int g) { return cnt[g]; }, [&](int g, int prefix) { row_ptr[g] = prefix; });
  if (threadIdx.x == 0) row_ptr[num_groups] = total;
}

// flagged entry e holding item x: its rank in the union is the number of flagged entries with an item below x, summed
// over the member rows (each row ascending: its entries below x are a prefix)
__global__ void __launch_bounds__(ROW_THREADS)
k_gr_write(igmc_csr_t G, const int32_t* __restrict__ members, int M, int cap, const int32_t* __restrict__ off,
           const int32_t* __restrict__ cnt, const int32_t* __restrict__ pre, const int32_t* __restrict__ row_ptr,
           int32_t* __restrict__ col_idx) {
  __shared__ GroupRows s;
  const int g = blockIdx.x;
  load_rows(G, members, M, g, s);
  const int n = group_entries(s, M, off, g, cap), o = off[g], c = cnt[g], base = row_ptr[g];
  auto before = [&](int e) { return e < n ? pre[o + e] : c; };   // flagged entries before e
  for (int e = threadIdx.x; e < n; e += blockDim.x) {
    if (before(e + 1) == before(e)) continue;
    int j;
    const int x = entry_at(G, s, M, e, &j);
    int rank = 0;
    for (int q = 0; q < M; ++q) {
      const int32_t* r = G.col_idx + s.r0[q];
      const int c0 = (int)s.cum[q];
      int lo = 0, hi = (int)(s.cum[q + 1] - s.cum[q]);
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (r[mid] < x) lo = mid + 1; else hi = mid;
      }
      rank += before(c0 + lo) - before(c0);
    }
    col_idx[base + rank] = x;
  }
}

__global__ void __launch_bounds__(PAIR_THREADS)
k_gr_pairs(const int32_t* __restrict__ members, int num_groups, int M, int num_users, int num_items,
           const int32_t* __restrict__ unit_g, const int32_t* __restrict__ unit_v, const int64_t* __restrict__ unit_tag,
           int B, int32_t* __restrict__ links_u, int32_t* __restrict__ links_v, int64_t* __restrict__ pair_id,
           int64_t* __restrict__ tag, int* err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  const int Gu = B / M;
  const bool real = i < Gu * M;
  const int u0 = real ? i / M : 0, j = real ? i % M : 0;
  int grp = unit_g[u0], v = unit_v[u0];
  if (grp < 0 || grp >= num_groups || v < 0 || v >= num_items) {
    igmc_set_err(err, IGMC_ERR_CANDIDATES);
    grp = 0;
    v = 0;
  }
  const int m = member_at(members, M, num_users, grp, j, err);
  const int lead = member_at(members, M, num_users, grp, 0, nullptr);
  const int u = m >= 0 ? m : lead >= 0 ? lead : 0;   // an empty slot or the tail: a valid pair, tag -1
  links_u[i] = u;
  links_v[i] = v;
  pair_id[i] = (int64_t)u * num_items + v;
  tag[i] = real && m >= 0 ? unit_tag[u0] : -1;
}

// unit g: x_j = the fp32 checkpoint mean of position g*M + j for the real members (tag >= 0), in member order.  mean:
// sum_j x_j in fp64 without fma contraction, / n, rounded once; min / max: the first smallest / largest x_j (strict
// compares).  A NaN x_j makes the key NaN.
__global__ void __launch_bounds__(STATS_THREADS)
k_gr_stats(const float* __restrict__ preds, int K, int B, int M, int aggregate, const int64_t* __restrict__ tag,
           float* __restrict__ key, float* __restrict__ score, float* __restrict__ member_score) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= B / M) return;
  const int i0 = g * M;
  long long t = -1;
  int n = 0;
  double sum = 0.0;
  float best = 0.f;
  bool nan = false;
  for (int j = 0; j < M; ++j) {
    if (tag[i0 + j] < 0) continue;
    t = tag[i0 + j];
    const float x = ckpt_mean(preds, K, B, i0 + j);
    nan |= isnan(x);
    if (aggregate == IGMC_GROUP_AGG_MEAN)
      sum = __dadd_rn(sum, (double)x);
    else if (n == 0 || (aggregate == IGMC_GROUP_AGG_MIN ? x < best : x > best))
      best = x;
    ++n;
  }
  const float k = nan ? __int_as_float(0x7fc00000)
                      : aggregate == IGMC_GROUP_AGG_MEAN ? (float)__ddiv_rn(sum, (double)max(n, 1)) : best;
  if (key) key[g] = k;
  if (t < 0 || !score) return;
  score[t] = k;
  for (int j = 0; j < M; ++j)
    member_score[t * M + j] = tag[i0 + j] >= 0 ? ckpt_mean(preds, K, B, i0 + j) : __int_as_float(0x7fc00000);
}

bool width_ok(int M) { return M >= 1 && M <= IGMC_GROUP_MAX; }

}  // namespace

extern "C" int igmc_group_rows(const igmc_csr_t* G, const int32_t* members, int num_groups, int width,
                               int32_t* row_ptr, int32_t* col_idx, int cap, int32_t* ws, int* err, void* stream) {
  if (!G || !G->row_ptr || !G->col_idx || !members || num_groups < 1 || !width_ok(width) || !row_ptr || !ws ||
      cap < 0 || (cap > 0 && !col_idx))
    return -1;
  cudaStream_t st = (cudaStream_t)stream;
  int32_t *off = ws, *cnt = ws + num_groups + 1, *pre = cnt + num_groups;
  k_gr_offsets<<<1, ROW_THREADS, 0, st>>>(*G, members, num_groups, width, cap, off, err);
  IGMC_CUDA_CHECK_LAUNCH();
  k_gr_flags<<<num_groups, ROW_THREADS, 0, st>>>(*G, members, width, cap, off, cnt, pre);
  IGMC_CUDA_CHECK_LAUNCH();
  k_gr_scan<<<1, ROW_THREADS, 0, st>>>(cnt, num_groups, row_ptr);
  IGMC_CUDA_CHECK_LAUNCH();
  k_gr_write<<<num_groups, ROW_THREADS, 0, st>>>(*G, members, width, cap, off, cnt, pre, row_ptr, col_idx);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_group_pairs(const int32_t* members, int num_groups, int width, int num_users, int num_items,
                                const int32_t* unit_g, const int32_t* unit_v, const int64_t* unit_tag, int B,
                                int32_t* links_u, int32_t* links_v, int64_t* pair_id, int64_t* tag, int* err,
                                void* stream) {
  if (!members || num_groups < 1 || !width_ok(width) || width > B || num_users < 1 || num_items < 1) return -1;
  if (!unit_g || !unit_v || !unit_tag || !links_u || !links_v || !pair_id || !tag) return -1;
  k_gr_pairs<<<(B + PAIR_THREADS - 1) / PAIR_THREADS, PAIR_THREADS, 0, (cudaStream_t)stream>>>(
      members, num_groups, width, num_users, num_items, unit_g, unit_v, unit_tag, B, links_u, links_v, pair_id, tag,
      err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_group_stats(const float* preds, int K, int B, int width, int aggregate, const int64_t* tag,
                                float* key, float* score, float* member_score, void* stream) {
  if (!preds || K < 1 || !width_ok(width) || width > B || !tag) return -1;
  if (aggregate < IGMC_GROUP_AGG_MEAN || aggregate > IGMC_GROUP_AGG_MAX) return -1;
  if (!key && (!score || !member_score)) return -1;
  const int Gu = B / width;
  k_gr_stats<<<(Gu + STATS_THREADS - 1) / STATS_THREADS, STATS_THREADS, 0, (cudaStream_t)stream>>>(
      preds, K, B, width, aggregate, tag, key, score, member_score);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
