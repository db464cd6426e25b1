// In-place update of the device rating graph (igmc_b200/util_functions.py: RatingGraph.update).
//
// A delta of D entries (u, v, value) - value = rating label + 1 inserts or overwrites, value 0 deletes - is applied to
// the CSR (row_ptr, col_idx, rating) and the CSC (col_ptr, row_idx) of an igmc_csr_t without changing its pointers.
// The arrays afterwards are exactly those RatingGraph(A_updated) builds.  Two entry points, one host sync between them:
//   igmc_graph_update_plan    validate; stable sort by (u, v) carrying the input position; keep the last entry of each
//                             equal-key run; classify the kept entries against the current rows (binary search);
//                             exclusive scans of the packed (inserted, deleted) counts in (u, v) and, through a second
//                             stable sort of the same entries by (v, u), in column order; per row / column the run of
//                             delta entries and the new length (the run's count difference, no atomics); int64 scans to
//                             the new row_ptr / col_ptr; the header (new nnz, shape, max degrees, counts)
//   igmc_graph_update_apply   merge every new row (column) from its surviving old entries and its inserted entries into
//                             scratch, a warp per row; then copy the scratch back into the graph's own arrays
// Every output element has exactly one writer; the result does not depend on the order threads run in.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "row_merge.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int THREADS = 256;

// the carve-up of the caller's workspace; the same for the size query, the plan and the apply
struct Layout {
  // per delta entry
  long long *key_uv, *skey_uv, *key_vu, *skey_vu, *pk_uv, *pk_vu, *scan_uv, *scan_vu;
  int32_t *pos, *spos, *perm_c;
  uint8_t *cls, *lab;
  // per row / column (capacity) and per rating (capacity)
  int32_t *row_ds, *row_de, *col_ds, *col_de;
  long long *len_r, *len_c, *ptr_r, *ptr_c;
  int32_t *new_col_idx, *new_row_idx;
  uint8_t *new_rating;
  void* temp;
  size_t temp_bytes, total;
};

Layout layout(void* base, int D, int cap_users, int cap_items, int cap_nnz, cudaStream_t st) {
  Layout L = {};
  size_t off = 0;
  unsigned char* b = static_cast<unsigned char*>(base);
  auto take = [&](size_t bytes) -> void* {
    void* p = b ? b + off : nullptr;
    off += align256(bytes);
    return p;
  };
  const size_t d = (size_t)D, d1 = d + 1, u1 = (size_t)cap_users + 1, i1 = (size_t)cap_items + 1;
  L.key_uv = (long long*)take(d * 8);
  L.skey_uv = (long long*)take(d * 8);
  L.key_vu = (long long*)take(d * 8);
  L.skey_vu = (long long*)take(d * 8);
  L.scan_uv = (long long*)take(d1 * 8);
  L.scan_vu = (long long*)take(d1 * 8);
  L.pk_uv = (long long*)take(d1 * 8);
  L.pk_vu = (long long*)take(d1 * 8);
  L.pos = (int32_t*)take(d * 4);
  L.spos = (int32_t*)take(d * 4);
  L.perm_c = (int32_t*)take(d * 4);
  L.cls = (uint8_t*)take(d);
  L.lab = (uint8_t*)take(d);
  L.row_ds = (int32_t*)take(u1 * 4);
  L.row_de = (int32_t*)take(u1 * 4);
  L.col_ds = (int32_t*)take(i1 * 4);
  L.col_de = (int32_t*)take(i1 * 4);
  L.len_r = (long long*)take(u1 * 8);
  L.len_c = (long long*)take(i1 * 8);
  L.ptr_r = (long long*)take(u1 * 8);
  L.ptr_c = (long long*)take(i1 * 8);
  L.new_col_idx = (int32_t*)take((size_t)cap_nnz * 4 + 4);
  L.new_row_idx = (int32_t*)take((size_t)cap_nnz * 4 + 4);
  L.new_rating = (uint8_t*)take((size_t)cap_nnz + 4);
  // CUB scratch: the largest of the two sorts and the four scans
  const unsigned long long nk = (unsigned long long)cap_users * (unsigned long long)cap_items;
  size_t t = 0, s = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, s, (long long*)nullptr, (long long*)nullptr, (int32_t*)nullptr,
                                  (int32_t*)nullptr, D, 0, bits_for(nk), st);
  t = s > t ? s : t;
  cub::DeviceScan::ExclusiveSum(nullptr, s, (long long*)nullptr, (long long*)nullptr, D + 1, st);
  t = s > t ? s : t;
  cub::DeviceScan::ExclusiveSum(nullptr, s, (long long*)nullptr, (long long*)nullptr, cap_users + 1, st);
  t = s > t ? s : t;
  cub::DeviceScan::ExclusiveSum(nullptr, s, (long long*)nullptr, (long long*)nullptr, cap_items + 1, st);
  t = s > t ? s : t;
  L.temp_bytes = t;
  L.temp = take(t);
  L.total = off;
  return L;
}

// ---- plan ----------------------------------------------------------------------------------------------------------
__global__ void k_keys(const int32_t* __restrict__ u, const int32_t* __restrict__ v, const int32_t* __restrict__ val,
                       int D, int cap_users, int cap_items, long long* __restrict__ key, int32_t* __restrict__ pos,
                       int* err) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < D; i += gridDim.x * blockDim.x) {
    int a = u[i], b = v[i];
    const int x = val[i];
    if (a < 0 || a >= cap_users || b < 0 || b >= cap_items || x < 0 || x > 256) {
      igmc_set_err(err, IGMC_ERR_GRAPH_UPDATE);
      a = 0;
      b = 0;
    }
    key[i] = (long long)a * cap_items + b;
    pos[i] = i;
  }
}

// entry i of the (u, v) order: keep the last of each equal-key run (the stable sort kept input order), classify it
// against row u of G, its (v, u) sort key and the block's counts
__global__ void k_classify(igmc_csr_t G, const int32_t* __restrict__ val, int D, int cap_items,
                           const long long* __restrict__ skey, const int32_t* __restrict__ spos,
                           uint8_t* __restrict__ cls, uint8_t* __restrict__ lab, long long* __restrict__ pk,
                           long long* __restrict__ key_vu, int32_t* __restrict__ pos, int cap_users,
                           igmc_graph_update_header_t* H) {
  __shared__ int ws[33];
  for (int base = blockIdx.x * blockDim.x; base < D; base += gridDim.x * blockDim.x) {
    const int i = base + threadIdx.x;
    int ins = 0, chg = 0, del = 0;
    if (i < D) {
      const long long k = skey[i];
      const int a = (int)(k / cap_items), b = (int)(k % cap_items);
      uint8_t c = C_NOOP, l = 0;
      if (i == D - 1 || skey[i + 1] != k) {
        int p = -1;
        if (a < G.num_users && b < G.num_items) {
          const int r0 = G.row_ptr[a], r1 = G.row_ptr[a + 1];
          const int q = find_col(G.col_idx, r0, r1, b);
          if (q < r1 && G.col_idx[q] == b) p = q;
        }
        c = classify(val[spos[i]], p, G.rating, &l);
      }
      cls[i] = c;
      lab[i] = l;
      pk[i] = pack_count(c);
      key_vu[i] = (long long)b * cap_users + a;
      pos[i] = i;
      ins = c == C_INSERT;
      chg = c == C_CHANGE;
      del = c == C_DELETE;
    }
    // integer counts: exact, so the order of the per-block adds does not matter
    ins = block_sum_i(ins, ws);
    chg = block_sum_i(chg, ws);
    del = block_sum_i(del, ws);
    if (threadIdx.x == 0) {
      if (ins) atomicAdd((unsigned long long*)&H->inserted, (unsigned long long)ins);
      if (chg) atomicAdd((unsigned long long*)&H->changed, (unsigned long long)chg);
      if (del) atomicAdd((unsigned long long*)&H->removed, (unsigned long long)del);
    }
  }
}

// column order: the packed counts of entry perm_c[i] of the (u, v) order (pk[D] = 0 closes the scan)
__global__ void k_gather_col(const int32_t* __restrict__ perm_c, const long long* __restrict__ pk, int D,
                             long long* __restrict__ pk_vu) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= D; i += gridDim.x * blockDim.x)
    pk_vu[i] = i < D ? pk[perm_c[i]] : 0;
}

// new length of every row (column) r < cap: old length (0 at or past the current shape) + the run's net count, 0 past
// the new shape; the block maxima go into the header (integer max: order-free)
__global__ void k_lengths(const int32_t* __restrict__ ptr, int n_old, int cap, const long long* __restrict__ skey,
                          int D, int stride, int n_req, const int32_t* __restrict__ ds,
                          const int32_t* __restrict__ de, const long long* __restrict__ scan,
                          long long* __restrict__ len, int64_t* n_new_out, int64_t* max_out) {
  __shared__ int ws[33];
  const int n_new = max(max(n_old, n_req), (int)(skey[D - 1] / stride) + 1);
  for (int base = blockIdx.x * blockDim.x; base <= cap; base += gridDim.x * blockDim.x) {
    const int r = base + threadIdx.x;
    long long l = 0;
    if (r < n_new) {
      if (r < n_old) l = ptr[r + 1] - ptr[r];
      if (de[r] > ds[r]) l += net(scan[de[r]]) - net(scan[ds[r]]);
    }
    if (r <= cap) len[r] = l;
    // degrees stay below 2^31 (checked against the int32 nnz in k_finalize)
    int m = (int)(l < 0x7fffffff ? l : 0x7fffffff);
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(IGMC_FULL, m, o));
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
      int bm = 0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) bm = max(bm, ws[w]);
      if (bm > 0) atomicMax((unsigned long long*)max_out, (unsigned long long)bm);
    }
    __syncthreads();
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *n_new_out = n_new;
}

__global__ void k_finalize(const long long* __restrict__ ptr_r, int cap_users, int cap_nnz, const int* err,
                           igmc_graph_update_header_t* H) {
  const long long nnz = ptr_r[cap_users];
  H->nnz = nnz;
  H->status = nnz > 0x7fffffffll ? IGMC_GRAPH_UPDATE_OVER_INT32
              : nnz > (long long)cap_nnz ? IGMC_GRAPH_UPDATE_OVER_CAPACITY : 0;
  H->err = err ? *err : 0;
}

// ---- apply ----------------------------------------------------------------------------------------------------------
// One warp per new row (column) r: merge_row of its old entries and its delta run.
template <bool RATING>
__global__ void k_merge(const int32_t* __restrict__ ptr, const int32_t* __restrict__ idx,
                        const uint8_t* __restrict__ rating, int n_old, int n_new,
                        const long long* __restrict__ ptr_new, const int32_t* __restrict__ ds,
                        const int32_t* __restrict__ de, const long long* __restrict__ skey, int stride,
                        const uint8_t* __restrict__ cls, const uint8_t* __restrict__ lab,
                        const int32_t* __restrict__ perm, const long long* __restrict__ scan,
                        int32_t* __restrict__ out_idx, uint8_t* __restrict__ out_rating) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n_new; r += warps) {
    const int o0 = r < n_old ? ptr[r] : 0, o1 = r < n_old ? ptr[r + 1] : 0;
    merge_row<RATING>(idx, rating, o0, o1, ds[r], de[r], ptr_new[r], skey, stride, cls, lab, perm, scan, out_idx,
                      out_rating, lane);
  }
}

bool caps_ok(const igmc_csr_t* G, int nnz, int cap_users, int cap_items, int cap_nnz) {
  return G && nnz >= 0 && cap_users >= G->num_users && cap_items >= G->num_items && cap_nnz >= nnz &&
         G->num_users >= 0 && G->num_items >= 0 && cap_users >= 1 && cap_items >= 1;
}

}  // namespace

extern "C" int igmc_graph_update_ws_bytes(int D, int cap_users, int cap_items, int cap_nnz, int64_t* bytes) {
  if (D <= 0 || cap_users < 1 || cap_items < 1 || cap_nnz < 0 || !bytes) return -1;
  *bytes = (int64_t)layout(nullptr, D, cap_users, cap_items, cap_nnz, 0).total;
  return 0;
}

extern "C" int igmc_graph_update_plan(const igmc_csr_t* G, int nnz, int cap_users, int cap_items, int cap_nnz,
                                      const int32_t* users, const int32_t* items, const int32_t* values, int D,
                                      int shape_users, int shape_items, void* ws, int64_t ws_bytes,
                                      igmc_graph_update_header_t* header, int* err, void* stream) {
  if (!caps_ok(G, nnz, cap_users, cap_items, cap_nnz) || D <= 0 || !users || !items || !values || !ws || !header)
    return -1;
  if (shape_users > cap_users || shape_items > cap_items) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  const Layout L = layout(ws, D, cap_users, cap_items, cap_nnz, st);
  if ((int64_t)L.total > ws_bytes) return -2;
  igmc_graph_update_header_t* H = header;
  cudaMemsetAsync(H, 0, sizeof(*H), st);
  cudaMemsetAsync(L.row_ds, 0, ((size_t)cap_users + 1) * 4, st);
  cudaMemsetAsync(L.row_de, 0, ((size_t)cap_users + 1) * 4, st);
  cudaMemsetAsync(L.col_ds, 0, ((size_t)cap_items + 1) * 4, st);
  cudaMemsetAsync(L.col_de, 0, ((size_t)cap_items + 1) * 4, st);
  cudaMemsetAsync(L.pk_uv + D, 0, 8, st);
  const int bits = bits_for((unsigned long long)cap_users * (unsigned long long)cap_items);
  const int g = grid_for(D, THREADS);
  size_t tb = L.temp_bytes;
  k_keys<<<g, THREADS, 0, st>>>(users, items, values, D, cap_users, cap_items, L.key_uv, L.pos, err);
  if (cub::DeviceRadixSort::SortPairs(L.temp, tb, L.key_uv, L.skey_uv, L.pos, L.spos, D, 0, bits, st) != cudaSuccess)
    return -3;
  k_classify<<<g, THREADS, 0, st>>>(*G, values, D, cap_items, L.skey_uv, L.spos, L.cls, L.lab, L.pk_uv, L.key_vu,
                                    L.pos, cap_users, H);
  tb = L.temp_bytes;
  if (cub::DeviceScan::ExclusiveSum(L.temp, tb, L.pk_uv, L.scan_uv, D + 1, st) != cudaSuccess) return -3;
  // the column side: the same classified entries, stably ordered by (v, u); perm_c maps to the (u, v) position
  tb = L.temp_bytes;
  if (cub::DeviceRadixSort::SortPairs(L.temp, tb, L.key_vu, L.skey_vu, L.pos, L.perm_c, D, 0, bits, st) != cudaSuccess)
    return -3;
  k_gather_col<<<grid_for(D + 1, THREADS), THREADS, 0, st>>>(L.perm_c, L.pk_uv, D, L.pk_vu);
  tb = L.temp_bytes;
  if (cub::DeviceScan::ExclusiveSum(L.temp, tb, L.pk_vu, L.scan_vu, D + 1, st) != cudaSuccess) return -3;
  k_runs<<<g, THREADS, 0, st>>>(L.skey_uv, D, cap_items, L.row_ds, L.row_de);
  k_runs<<<g, THREADS, 0, st>>>(L.skey_vu, D, cap_users, L.col_ds, L.col_de);
  k_lengths<<<grid_for(cap_users + 1, THREADS), THREADS, 0, st>>>(G->row_ptr, G->num_users, cap_users, L.skey_uv, D,
                                                                  cap_items, shape_users, L.row_ds, L.row_de,
                                                                  L.scan_uv, L.len_r, &H->num_users, &H->max_row_deg);
  k_lengths<<<grid_for(cap_items + 1, THREADS), THREADS, 0, st>>>(G->col_ptr, G->num_items, cap_items, L.skey_vu, D,
                                                                  cap_users, shape_items, L.col_ds, L.col_de,
                                                                  L.scan_vu, L.len_c, &H->num_items, &H->max_col_deg);
  tb = L.temp_bytes;
  if (cub::DeviceScan::ExclusiveSum(L.temp, tb, L.len_r, L.ptr_r, cap_users + 1, st) != cudaSuccess) return -3;
  tb = L.temp_bytes;
  if (cub::DeviceScan::ExclusiveSum(L.temp, tb, L.len_c, L.ptr_c, cap_items + 1, st) != cudaSuccess) return -3;
  k_finalize<<<1, 1, 0, st>>>(L.ptr_r, cap_users, cap_nnz, err, H);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_graph_update_apply(const igmc_csr_t* G, int nnz, int cap_users, int cap_items, int cap_nnz, int D,
                                       void* ws, int64_t ws_bytes, int new_nnz, int new_users, int new_items,
                                       void* stream) {
  if (!caps_ok(G, nnz, cap_users, cap_items, cap_nnz) || D <= 0 || !ws) return -1;
  if (new_nnz < 0 || new_nnz > cap_nnz || new_users < G->num_users || new_users > cap_users ||
      new_items < G->num_items || new_items > cap_items)
    return -1;
  cudaStream_t st = (cudaStream_t)stream;
  const Layout L = layout(ws, D, cap_users, cap_items, cap_nnz, st);
  if ((int64_t)L.total > ws_bytes) return -2;
  k_merge<true><<<grid_for((long long)new_users * 32, THREADS), THREADS, 0, st>>>(
      G->row_ptr, G->col_idx, G->rating, G->num_users, new_users, L.ptr_r, L.row_ds, L.row_de, L.skey_uv, cap_items,
      L.cls, L.lab, nullptr, L.scan_uv, L.new_col_idx, L.new_rating);
  k_merge<false><<<grid_for((long long)new_items * 32, THREADS), THREADS, 0, st>>>(
      G->col_ptr, G->row_idx, nullptr, G->num_items, new_items, L.ptr_c, L.col_ds, L.col_de, L.skey_vu, cap_users,
      L.cls, L.lab, L.perm_c, L.scan_vu, L.new_row_idx, nullptr);
  IGMC_CUDA_CHECK_LAUNCH();
  // copy-back: the graph keeps its five device pointers
  if (new_nnz > 0) {
    cudaMemcpyAsync((void*)G->col_idx, L.new_col_idx, (size_t)new_nnz * 4, cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync((void*)G->rating, L.new_rating, (size_t)new_nnz, cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync((void*)G->row_idx, L.new_row_idx, (size_t)new_nnz * 4, cudaMemcpyDeviceToDevice, st);
  }
  k_store_ptr<<<grid_for(new_users + 1, THREADS), THREADS, 0, st>>>(L.ptr_r, new_users, (int32_t*)G->row_ptr);
  k_store_ptr<<<grid_for(new_items + 1, THREADS), THREADS, 0, st>>>(L.ptr_c, new_items, (int32_t*)G->col_ptr);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
