// Rating sessions (igmc_b200/recommend.py: RatingSessions): per session s the rating row of user users[s] with the
// session's edits applied, as one device CSR of S rows, without changing the graph.
//
// An edit (session s, item v, value) uses RatingGraph.update's encoding: value = label + 1 inserts or overwrites, 0
// deletes (an absent rating: nothing), the last occurrence of (s, v) wins.  Session s starts from the graph row of
// users[s] when users[s] < G.num_users, from an empty row otherwise (a new user).  The row is exactly the row
// RatingGraph.update would leave for that user; it is graph_update.cu's merge restricted to one row per session, and
// shares its device code (row_merge.cuh).  Two entry points, one host sync between them:
//   igmc_session_plan    validate; stable sort by (s, v) carrying the input position; keep the last of each run;
//                        classify against the base row (binary search); exclusive scan of the packed counts; per session
//                        the run of edits and the new length; int64 scan to the row pointers; the header (total length,
//                        longest row)
//   igmc_session_apply   merge every session's row from its base row and its run, a warp per session; int32 row_ptr
// Every output element has exactly one writer; the result does not depend on the order threads run in.
//
// igmc_session_pairs maps the pairs igmc_candidate_pairs writes over the session rows (query slot = session) to the
// session user's real id.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "row_merge.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int THREADS = 256;

size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

struct Layout {
  long long *key, *skey, *pk, *scan, *len, *ptr;
  int32_t *pos, *spos, *ds, *de;
  uint8_t *cls, *lab;
  void* temp;
  size_t temp_bytes, total;
};

Layout layout(void* base, int S, int D, int num_items, cudaStream_t st) {
  Layout L = {};
  size_t off = 0;
  unsigned char* b = static_cast<unsigned char*>(base);
  auto take = [&](size_t bytes) -> void* {
    void* p = b ? b + off : nullptr;
    off += align256(bytes);
    return p;
  };
  const size_t d = (size_t)D, d1 = d + 1, s1 = (size_t)S + 1;
  L.key = (long long*)take(d * 8);
  L.skey = (long long*)take(d * 8);
  L.pk = (long long*)take(d1 * 8);
  L.scan = (long long*)take(d1 * 8);
  L.pos = (int32_t*)take(d * 4);
  L.spos = (int32_t*)take(d * 4);
  L.cls = (uint8_t*)take(d);
  L.lab = (uint8_t*)take(d);
  L.ds = (int32_t*)take(s1 * 4);
  L.de = (int32_t*)take(s1 * 4);
  L.len = (long long*)take(s1 * 8);
  L.ptr = (long long*)take(s1 * 8);
  size_t t = 0, s = 0;
  if (D > 0) {
    cub::DeviceRadixSort::SortPairs(nullptr, s, (long long*)nullptr, (long long*)nullptr, (int32_t*)nullptr,
                                    (int32_t*)nullptr, D, 0,
                                    bits_for((unsigned long long)S * (unsigned long long)num_items), st);
    t = s > t ? s : t;
    cub::DeviceScan::ExclusiveSum(nullptr, s, (long long*)nullptr, (long long*)nullptr, D + 1, st);
    t = s > t ? s : t;
  }
  cub::DeviceScan::ExclusiveSum(nullptr, s, (long long*)nullptr, (long long*)nullptr, S + 1, st);
  t = s > t ? s : t;
  L.temp_bytes = t;
  L.temp = take(t);
  L.total = off;
  return L;
}

int grid_for(long long n) {
  long long g = (n + THREADS - 1) / THREADS;
  return (int)(g < 1 ? 1 : g > 65535 * 8 ? 65535 * 8 : g);
}

// the sort key s * num_items + v of every edit; invalid edits (and invalid user ids) set the error and key 0
__global__ void k_session_keys(const int32_t* __restrict__ users, int S, const int32_t* __restrict__ sess,
                               const int32_t* __restrict__ items, const int32_t* __restrict__ val, int D,
                               int num_items, long long* __restrict__ key, int32_t* __restrict__ pos, int* err) {
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < D; i += stride) {
    int a = sess[i], b = items[i];
    const int x = val[i];
    if (a < 0 || a >= S || b < 0 || b >= num_items || x < 0 || x > 256) {
      igmc_set_err(err, IGMC_ERR_SESSIONS);
      a = 0;
      b = 0;
    }
    key[i] = (long long)a * num_items + b;
    pos[i] = i;
  }
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < S; s += stride)
    if (users[s] < 0) igmc_set_err(err, IGMC_ERR_SESSIONS);
}

// sorted edit i: kept when it is the last of its (s, v) run, classified against the base row of session s
__global__ void k_session_classify(igmc_csr_t G, const int32_t* __restrict__ users, const int32_t* __restrict__ val,
                                   int D, int num_items, const long long* __restrict__ skey,
                                   const int32_t* __restrict__ spos, uint8_t* __restrict__ cls,
                                   uint8_t* __restrict__ lab, long long* __restrict__ pk) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < D; i += gridDim.x * blockDim.x) {
    const long long k = skey[i];
    const int s = (int)(k / num_items), b = (int)(k % num_items);
    uint8_t c = C_NOOP, l = 0;
    if (i == D - 1 || skey[i + 1] != k) {
      const int u = users[s];
      int p = -1;
      if (u >= 0 && u < G.num_users) {
        const int r0 = G.row_ptr[u], r1 = G.row_ptr[u + 1];
        const int q = find_col(G.col_idx, r0, r1, b);
        if (q < r1 && G.col_idx[q] == b) p = q;
      }
      c = classify(val[spos[i]], p, G.rating, &l);
    }
    cls[i] = c;
    lab[i] = l;
    pk[i] = pack_count(c);
  }
}

__device__ __forceinline__ void base_row(const igmc_csr_t& G, int u, int* o0, int* o1) {
  const bool old = u >= 0 && u < G.num_users;
  *o0 = old ? G.row_ptr[u] : 0;
  *o1 = old ? G.row_ptr[u + 1] : 0;
}

// new length of every session row: base length + the run's net count; len[S] = 0 closes the scan; the block maxima
// go into header[1] (integer max: order-free)
__global__ void k_session_lengths(igmc_csr_t G, const int32_t* __restrict__ users, int S,
                                  const int32_t* __restrict__ ds, const int32_t* __restrict__ de,
                                  const long long* __restrict__ scan, long long* __restrict__ len,
                                  int64_t* __restrict__ header) {
  __shared__ int ws[33];
  for (int base = blockIdx.x * blockDim.x; base <= S; base += gridDim.x * blockDim.x) {
    const int s = base + threadIdx.x;
    long long l = 0;
    if (s < S) {
      int o0, o1;
      base_row(G, users[s], &o0, &o1);
      l = o1 - o0;
      if (scan && de[s] > ds[s]) l += net(scan[de[s]]) - net(scan[ds[s]]);
    }
    if (s <= S) len[s] = l;
    int m = (int)(l < 0x7fffffff ? l : 0x7fffffff);
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(IGMC_FULL, m, o));
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
      int bm = 0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) bm = max(bm, ws[w]);
      if (bm > 0) atomicMax((unsigned long long*)&header[1], (unsigned long long)bm);
    }
    __syncthreads();
  }
}

__global__ void k_session_total(const long long* __restrict__ ptr, int S, int64_t* header) { header[0] = ptr[S]; }

// one warp per session: merge_row of its base row and its run of edits
__global__ void k_session_merge(igmc_csr_t G, const int32_t* __restrict__ users, int S,
                                const long long* __restrict__ ptr_new, const int32_t* __restrict__ ds,
                                const int32_t* __restrict__ de, const long long* __restrict__ skey, int num_items,
                                const uint8_t* __restrict__ cls, const uint8_t* __restrict__ lab,
                                const long long* __restrict__ scan, int32_t* __restrict__ out_idx,
                                uint8_t* __restrict__ out_rating) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < S; s += warps) {
    int o0, o1;
    base_row(G, users[s], &o0, &o1);
    merge_row<true>(G.col_idx, G.rating, o0, o1, ds[s], de[s], ptr_new[s], skey, num_items, cls, lab, nullptr, scan,
                    out_idx, out_rating, lane);
  }
}

__global__ void k_session_store_ptr(const long long* __restrict__ src, int n, int32_t* __restrict__ dst) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += gridDim.x * blockDim.x) dst[i] = (int32_t)src[i];
}

// pairs over the session rows: links_u holds the session index; it becomes sess[i], and links_u / pair_id the
// session user's id and its pair id u * num_items + v
__global__ void k_session_pairs(const int32_t* __restrict__ users, int S, int num_items, int B,
                                int32_t* __restrict__ links_u, const int32_t* __restrict__ links_v,
                                int64_t* __restrict__ pair_id, int32_t* __restrict__ sess, int* err) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
    int s = links_u[i];
    if (s < 0 || s >= S) {
      igmc_set_err(err, IGMC_ERR_CANDIDATES);
      s = 0;
    }
    const int u = users[s];
    sess[i] = s;
    links_u[i] = u;
    pair_id[i] = (int64_t)u * num_items + links_v[i];
  }
}

}  // namespace

extern "C" int igmc_session_ws_bytes(int num_sessions, int D, int num_items, int64_t* bytes) {
  if (num_sessions < 1 || D < 0 || num_items < 1 || !bytes) return -1;
  *bytes = (int64_t)layout(nullptr, num_sessions, D, num_items, 0).total;
  return 0;
}

extern "C" int igmc_session_plan(const igmc_csr_t* G, const int32_t* users, int num_sessions, const int32_t* sess,
                                 const int32_t* items, const int32_t* values, int D, void* ws, int64_t ws_bytes,
                                 int64_t* header, int* err, void* stream) {
  const int S = num_sessions;
  if (!G || !users || S < 1 || D < 0 || !ws || !header || G->num_items < 1) return -1;
  if (D > 0 && (!sess || !items || !values)) return -1;
  if ((unsigned long long)S * (unsigned long long)G->num_items >= (1ull << 62)) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  const Layout L = layout(ws, S, D, G->num_items, st);
  if ((int64_t)L.total > ws_bytes) return -2;
  cudaMemsetAsync(header, 0, 2 * sizeof(int64_t), st);
  cudaMemsetAsync(L.ds, 0, ((size_t)S + 1) * 4, st);
  cudaMemsetAsync(L.de, 0, ((size_t)S + 1) * 4, st);
  const int g = grid_for(D > S ? D : S);
  k_session_keys<<<g, THREADS, 0, st>>>(users, S, sess, items, values, D, G->num_items, L.key, L.pos, err);
  size_t tb;
  if (D > 0) {
    cudaMemsetAsync(L.pk + D, 0, 8, st);
    tb = L.temp_bytes;
    if (cub::DeviceRadixSort::SortPairs(L.temp, tb, L.key, L.skey, L.pos, L.spos, D, 0,
                                        bits_for((unsigned long long)S * (unsigned long long)G->num_items),
                                        st) != cudaSuccess)
      return -3;
    k_session_classify<<<grid_for(D), THREADS, 0, st>>>(*G, users, values, D, G->num_items, L.skey, L.spos, L.cls,
                                                        L.lab, L.pk);
    tb = L.temp_bytes;
    if (cub::DeviceScan::ExclusiveSum(L.temp, tb, L.pk, L.scan, D + 1, st) != cudaSuccess) return -3;
    k_runs<<<grid_for(D), THREADS, 0, st>>>(L.skey, D, G->num_items, L.ds, L.de);
  }
  k_session_lengths<<<grid_for(S + 1), THREADS, 0, st>>>(*G, users, S, L.ds, L.de, D > 0 ? L.scan : nullptr, L.len,
                                                         header);
  tb = L.temp_bytes;
  if (cub::DeviceScan::ExclusiveSum(L.temp, tb, L.len, L.ptr, S + 1, st) != cudaSuccess) return -3;
  k_session_total<<<1, 1, 0, st>>>(L.ptr, S, header);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_session_apply(const igmc_csr_t* G, const int32_t* users, int num_sessions, int D, void* ws,
                                  int64_t ws_bytes, int32_t* row_ptr, int32_t* col_idx, uint8_t* rating,
                                  void* stream) {
  const int S = num_sessions;
  if (!G || !users || S < 1 || D < 0 || !ws || !row_ptr || !col_idx || !rating || G->num_items < 1) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  const Layout L = layout(ws, S, D, G->num_items, st);
  if ((int64_t)L.total > ws_bytes) return -2;
  k_session_merge<<<grid_for((long long)S * 32), THREADS, 0, st>>>(*G, users, S, L.ptr, L.ds, L.de, L.skey,
                                                                    G->num_items, L.cls, L.lab, L.scan, col_idx,
                                                                    rating);
  k_session_store_ptr<<<grid_for(S + 1), THREADS, 0, st>>>(L.ptr, S, row_ptr);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_session_pairs(const igmc_sessions_t* Sv, int num_items, int B, int32_t* links_u,
                                  const int32_t* links_v, int64_t* pair_id, int32_t* sess, int* err, void* stream) {
  if (!Sv || !Sv->users || B <= 0 || num_items < 1 || !links_u || !links_v || !pair_id || !sess) return -1;
  k_session_pairs<<<(B + THREADS - 1) / THREADS, THREADS, 0, (cudaStream_t)stream>>>(
      Sv->users, Sv->num_sessions, num_items, B, links_u, links_v, pair_id, sess, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
