// Online fine-tuning (igmc_b200/train_eval.py: OnlineTrainer): the training pairs of a step drawn from the device rating
// graph itself, and a ring of recently rated pairs that a share of every batch is drawn from.
//
//   igmc_online_recent_append  appends the (user, item) of a delta's rated entries (value > 0) to the ring, in input
//                              order, the newest over the oldest; the append count stays on the device
//   igmc_online_draw           one step's B pairs, labels, pair ids and seeds, for igmc_extract_batch with idx = NULL
//
// The draw reads only device state (the graph, the ring, its count and the optimizer's step counter), so one captured
// CUDA graph serves every step.  Twin: igmc_b200/train_eval.py::online_draw_host / recent_append_host.
#include "common.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int DRAW_THREADS = 128;
constexpr int APPEND_THREADS = 1024;
constexpr int DRAW_HOP_TAG = 7;   // sample_state's hop slot for the draw: extraction uses hops 1..IGMC_MAX_HOP only

// slot j's keys: round 0 chooses window or graph (and the window entry), round 1 is the uniform draw
__device__ __forceinline__ uint64_t draw_key(uint64_t seed, int j, int round) {
  return sample_state(seed, j, round, DRAW_HOP_TAG);
}

// position of v in row u's ascending columns, or -1
__device__ __forceinline__ int find_in_row(const igmc_csr_t& G, int u, int v) {
  int lo = G.row_ptr[u], hi = G.row_ptr[u + 1];
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const int c = G.col_idx[mid];
    if (c == v) return mid;
    if (c < v) lo = mid + 1; else hi = mid;
  }
  return -1;
}

__global__ void k_online_draw(igmc_csr_t G, const int32_t* __restrict__ ring_u, const int32_t* __restrict__ ring_v,
                              int capacity, const int64_t* __restrict__ total, long long recent_thresh,
                              const int64_t* __restrict__ step_count, int step_ahead, uint64_t sample_seed,
                              uint64_t drop_seed, int B, int32_t* __restrict__ links_u, int32_t* __restrict__ links_v,
                              int32_t* __restrict__ label, int64_t* __restrict__ pair_id, uint64_t* __restrict__ seeds,
                              int* err) {
  const uint64_t s = (uint64_t)step_count[0] + (uint64_t)step_ahead;
  const uint64_t seed = splitmix64(sample_seed + s);
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j == 0) {
    seeds[0] = seed;
    seeds[1] = splitmix64(drop_seed + s);
    seeds[2] = splitmix64(drop_seed + s + 1);
  }
  if (j >= B) return;
  const int nnz = G.row_ptr[G.num_users];
  if (nnz <= 0) {
    igmc_set_err(err, IGMC_ERR_ONLINE);
    links_u[j] = links_v[j] = label[j] = 0;
    pair_id[j] = 0;
    return;
  }
  const long long n = total[0];
  const int W = n < (long long)capacity ? (int)n : capacity;
  int u = -1, v = 0, pos = -1;
  const uint64_t key = draw_key(seed, j, 0);
  if (W > 0 && (long long)(key >> 32) < recent_thresh) {
    const int e = (int)(((key & 0xffffffffull) * (uint64_t)W) >> 32);
    u = ring_u[e];
    v = ring_v[e];
    if (u >= 0 && u < G.num_users && v >= 0 && v < G.num_items) pos = find_in_row(G, u, v);
  }
  if (pos < 0) {   // the graph's ratings, uniformly: the user whose row holds position pos
    pos = (int)__umul64hi(draw_key(seed, j, 1), (uint64_t)nnz);
    int lo = 0, hi = G.num_users;   // upper_bound(row_ptr[0..num_users], pos) - 1: the last row starting at or before pos
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (G.row_ptr[mid + 1] <= pos) lo = mid + 1; else hi = mid;
    }
    u = lo;
    v = G.col_idx[pos];
  }
  links_u[j] = u;
  links_v[j] = v;
  label[j] = G.rating[pos];
  pair_id[j] = (int64_t)u * G.num_items + v;
}

// single CTA: rank the rated entries in input order (chunked block scan) and store the last `capacity` of them
__global__ void __launch_bounds__(APPEND_THREADS)
k_online_append(const int32_t* __restrict__ users, const int32_t* __restrict__ items, const int32_t* __restrict__ values,
                int D, int32_t* __restrict__ ring_u, int32_t* __restrict__ ring_v, int capacity,
                int64_t* __restrict__ total, int* err) {
  __shared__ int ws[33];
  auto keep = [&](int i) -> int {
    const int x = values[i];
    return (users[i] >= 0 && items[i] >= 0 && x > 0 && x <= 256) ? 1 : 0;
  };
  const int kept = block_scan_chunks(D, ws, [&](int i) -> int {   // pass 1: validate and count
    const int x = values[i];
    if (users[i] < 0 || items[i] < 0 || x < 0 || x > 256) igmc_set_err(err, IGMC_ERR_GRAPH_UPDATE);
    return keep(i);
  }, [](int, int) {});
  const long long base = total[0];
  const int first = kept > capacity ? kept - capacity : 0;   // earlier ones would be overwritten within this call
  block_scan_chunks(D, ws, keep, [&](int i, int rank) {        // pass 2: one writer per ring slot
    if (!keep(i) || rank < first) return;
    const int slot = (int)((base + rank) % capacity);
    ring_u[slot] = users[i];
    ring_v[slot] = items[i];
  });
  if (threadIdx.x == 0) total[0] = base + kept;
}

}  // namespace

extern "C" int igmc_online_draw(const igmc_csr_t* G, const int32_t* ring_u, const int32_t* ring_v, int capacity,
                                const int64_t* total, int64_t recent_thresh, const int64_t* step_count, int step_ahead,
                                uint64_t sample_seed, uint64_t drop_seed, int B, int32_t* links_u, int32_t* links_v,
                                int32_t* label, int64_t* pair_id, uint64_t* seeds, int* err, void* stream) {
  if (!G || !G->row_ptr || !G->col_idx || !G->rating || G->num_users < 0 || G->num_items < 0) return -1;
  if (!ring_u || !ring_v || capacity < 1 || !total) return -2;
  if (recent_thresh < 0 || recent_thresh > (int64_t(1) << 32)) return -3;
  if (!step_count || step_ahead < 0) return -4;
  if (B < 1 || !links_u || !links_v || !label || !pair_id || !seeds || !err) return -5;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  k_online_draw<<<(B + DRAW_THREADS - 1) / DRAW_THREADS, DRAW_THREADS, 0, st>>>(
      *G, ring_u, ring_v, capacity, total, (long long)recent_thresh, step_count, step_ahead, sample_seed, drop_seed, B,
      links_u, links_v, label, pair_id, seeds, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_online_recent_append(const int32_t* users, const int32_t* items, const int32_t* values, int D,
                                         int32_t* ring_u, int32_t* ring_v, int capacity, int64_t* total, int* err,
                                         void* stream) {
  if (D < 0 || (D > 0 && (!users || !items || !values))) return -1;
  if (!ring_u || !ring_v || capacity < 1 || !total || !err) return -2;
  if (D == 0) return 0;
  k_online_append<<<1, APPEND_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(users, items, values, D, ring_u, ring_v,
                                                                            capacity, total, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
