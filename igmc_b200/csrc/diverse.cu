// Diversified recommendation lists (igmc_b200/recommend.py: recommend_diverse, item_similarity).
//
// The similarity of items a and b is the cosine of their binary rating columns, c_ab / sqrt(d_a d_b), with c_ab the
// number of users who rated both.  Only the items of the query users' pools are ever compared, so the counts are kept
// for their union alone:
//   k_dv_mark    one thread per pool entry: the item's bit set in an item bitmap (integer atomicOr)
//   k_dv_scan    one CTA: the popcount scan of the bitmap gives each marked item its dense index (map) and the union list
//   k_dv_count   one CTA per user row: the row's union entries compacted in tiles, every pair i < j of them adds 1 to
//                the upper-triangle table (integer atomicAdd: the counts are exact and bit-identical across runs)
//   k_dv_select  one CTA per query user, one thread per pool entry: k greedy steps of the penalised key
//   k_dv_cosine  one thread per entry of item_similarity's matrix
// Twins: igmc_b200/recommend.py::item_union_host / cocount_host / item_cosine_host / diverse_select_host.
#include "common.cuh"
#include "topk_merge.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int MARK_THREADS = 256;
constexpr int SCAN_THREADS = 256;
constexpr int COUNT_THREADS = 256;
constexpr int COUNT_TILE = 1024;          // row entries compacted per tile (rows longer than this run tile by tile)
constexpr int SELECT_THREADS = IGMC_TOPK_MAX;
constexpr int COSINE_THREADS = 256;
constexpr long long DIVERSE_WS_DEFAULT = 256ll << 20;

__host__ __device__ __forceinline__ long long tri_entries(long long nu) { return nu * (nu - 1) / 2; }

// the table entry of union indices i < j: row i of the upper triangle starts at i * (2 nu - i - 1) / 2
__device__ __forceinline__ long long tri_at(int i, int j, int nu) {
  return (long long)i * (2ll * nu - i - 1) / 2 + (j - i - 1);
}

// sim(a, b) = c / sqrt(d_a * d_b) in fp64, every operation correctly rounded, rounded once to fp32; 0 when d_a d_b = 0
__device__ __forceinline__ float item_cosine(uint32_t c, int da, int db) {
  if (da == 0 || db == 0) return 0.f;
  return __double2float_rn(__ddiv_rn((double)c, __dsqrt_rn(__dmul_rn((double)da, (double)db))));
}

// c of union indices i, j of items with degrees: the item's own degree on the diagonal
__device__ __forceinline__ uint32_t cocount(const uint32_t* __restrict__ T, int nu, int i, int j, int deg_i) {
  if (i == j) return (uint32_t)deg_i;
  return i < j ? T[tri_at(i, j, nu)] : T[tri_at(j, i, nu)];
}

__device__ __forceinline__ int col_deg(const igmc_csr_t& G, long long v) { return G.col_ptr[v + 1] - G.col_ptr[v]; }

__global__ void __launch_bounds__(MARK_THREADS)
k_dv_mark(const int64_t* __restrict__ items, long long n, int num_items, uint32_t* __restrict__ bitmap, int* err) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const long long v = items[e];
  if (v == -1) return;
  if (v < -1 || v >= num_items) {
    igmc_set_err(err, IGMC_ERR_CANDIDATES);
    return;
  }
  atomicOr(bitmap + (v >> 5), 1u << (v & 31));
}

__global__ void __launch_bounds__(SCAN_THREADS)
k_dv_scan(const uint32_t* __restrict__ bitmap, int num_items, int32_t* __restrict__ map, int32_t* __restrict__ list,
          int32_t* __restrict__ nu) {
  __shared__ int ws[33];
  const int W = (num_items + 31) >> 5;
  const int total = block_scan_chunks(
      W, ws, [&](int w) { return __popc(bitmap[w]); },
      [&](int w, int prefix) {
        const uint32_t b = bitmap[w];
        for (int t = 0; t < 32 && w * 32 + t < num_items; ++t) {
          const int v = w * 32 + t;
          if ((b >> t) & 1u) {
            const int r = prefix + __popc(b & ((1u << t) - 1u));
            map[v] = r;
            list[r] = v;
          } else {
            map[v] = -1;
          }
        }
      });
  if (threadIdx.x == 0) *nu = total;
}

// the union indices of row entries [0, n) in order, compacted into s; returns their count (every thread)
__device__ __forceinline__ int compact_tile(const int32_t* __restrict__ row, int n, const int32_t* __restrict__ map,
                                            int* s, int* ws) {
  const int c = block_scan_chunks(
      n, ws, [&](int e) { return map[row[e]] >= 0 ? 1 : 0; },
      [&](int e, int prefix) {
        const int i = map[row[e]];
        if (i >= 0) s[prefix] = i;
      });
  __syncthreads();
  return c;
}

// pairs (sa[x], sb[y]) with y > x when the tiles are the same (same), every y otherwise: one warp per x, lanes over y
__device__ __forceinline__ void count_pairs(const int* sa, int na, const int* sb, int nb, bool same, int nu,
                                            uint32_t* __restrict__ T) {
  const int lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int x = threadIdx.x >> 5; x < na; x += nw) {
    const int i = sa[x];
    const long long base = (long long)i * (2ll * nu - i - 1) / 2 - i - 1;
    for (int y = (same ? x + 1 : 0) + lane; y < nb; y += 32) atomicAdd(T + base + sb[y], 1u);
  }
}

// Each row is ascending and the map keeps item order, so a pair of entries at row positions p < q has union indices
// i < j: tile a against itself and every later tile b counts each pair of the row exactly once.
__global__ void __launch_bounds__(COUNT_THREADS)
k_dv_count(igmc_csr_t G, const int32_t* __restrict__ map, int nu, uint32_t* __restrict__ T) {
  __shared__ int sa[COUNT_TILE], sb[COUNT_TILE];
  __shared__ int ws[33];
  for (int w = blockIdx.x; w < G.num_users; w += gridDim.x) {
    const int32_t* row = G.col_idx + G.row_ptr[w];
    const int len = G.row_ptr[w + 1] - G.row_ptr[w];
    for (int a0 = 0; a0 < len; a0 += COUNT_TILE) {
      const int na = compact_tile(row + a0, min(COUNT_TILE, len - a0), map, sa, ws);
      if (na == 0) continue;
      count_pairs(sa, na, sa, na, true, nu, T);
      for (int b0 = a0 + COUNT_TILE; b0 < len; b0 += COUNT_TILE) {
        const int nb = compact_tile(row + b0, min(COUNT_TILE, len - b0), map, sb, ws);
        count_pairs(sa, na, sb, nb, false, nu, T);
        __syncthreads();
      }
      __syncthreads();
    }
  }
}

// Query q's pool is row q of pool_item / pool_score [Q, P]; thread j holds entry j.  Step s chooses, among the unchosen
// real entries, the first under ranks_before of key_j = score_j - penalty * m_j (id: the pool position), then raises
// every m_j to its sim with the chosen item.
__global__ void __launch_bounds__(SELECT_THREADS)
k_dv_select(igmc_csr_t G, const int64_t* __restrict__ pool_item, const float* __restrict__ pool_score, int P, int k,
            float penalty, const int32_t* __restrict__ map, int nu, const uint32_t* __restrict__ T,
            int64_t* __restrict__ out_item, float* __restrict__ out_score, float* __restrict__ out_key, int* err) {
  __shared__ float s_key[SELECT_THREADS / 32];
  __shared__ int s_id[SELECT_THREADS / 32];
  __shared__ int s_win, s_idx, s_deg;
  const int q = blockIdx.x, j = threadIdx.x, lane = j & 31, warp = j >> 5, nw = blockDim.x >> 5;
  const size_t o = (size_t)q * k;
  long long v = -1;
  float score = 0.f;
  int idx = -1, deg = 0;
  bool bad = false;
  if (j < P) {
    v = pool_item[(size_t)q * P + j];
    score = pool_score[(size_t)q * P + j];
    if (v < -1 || v >= G.num_items) {
      bad = true;
    } else if (v >= 0) {
      idx = map[v];
      deg = col_deg(G, v);
      bad = idx < 0 || idx >= nu;
    }
  }
  if (__syncthreads_or(bad)) {
    if (j == 0) igmc_set_err(err, IGMC_ERR_CANDIDATES);
    for (int s = j; s < k; s += blockDim.x) {
      out_item[o + s] = -1;
      out_score[o + s] = -INFINITY;
      out_key[o + s] = -INFINITY;
    }
    return;
  }
  bool live = v >= 0;
  float m = 0.f;
  for (int s = 0; s < k; ++s) {
    const float key = __fsub_rn(score, __fmul_rn(penalty, m));
    float bv = key;
    int bi = live ? j : -1;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      const float ov = __shfl_xor_sync(IGMC_FULL, bv, d);
      const int oi = __shfl_xor_sync(IGMC_FULL, bi, d);
      if (ranks_before(ov, oi, bv, bi, 1.f)) {
        bv = ov;
        bi = oi;
      }
    }
    if (lane == 0) {
      s_key[warp] = bv;
      s_id[warp] = bi;
    }
    __syncthreads();
    if (j == 0) {
      float wv = s_key[0];
      int wi = s_id[0];
      for (int x = 1; x < nw; ++x)
        if (ranks_before(s_key[x], s_id[x], wv, wi, 1.f)) {
          wv = s_key[x];
          wi = s_id[x];
        }
      s_win = wi;
    }
    __syncthreads();
    const int c = s_win;
    if (c < 0) {
      if (j == 0) {
        out_item[o + s] = -1;
        out_score[o + s] = -INFINITY;
        out_key[o + s] = -INFINITY;
      }
      continue;
    }
    if (j == c) {
      out_item[o + s] = v;
      out_score[o + s] = score;
      out_key[o + s] = key;
      live = false;
      s_idx = idx;
      s_deg = deg;
    }
    __syncthreads();
    if (live) {
      const float sim = item_cosine(cocount(T, nu, idx, s_idx, deg), deg, s_deg);
      m = sim > m ? sim : m;
    }
  }
}

__global__ void __launch_bounds__(COSINE_THREADS)
k_dv_cosine(igmc_csr_t G, const int64_t* __restrict__ items, int Q, const int32_t* __restrict__ map, int nu,
            const uint32_t* __restrict__ T, float* __restrict__ out, int* err) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)Q * Q) return;
  const long long a = items[e / Q], b = items[e % Q];
  const int ia = a >= 0 && a < G.num_items ? map[a] : -1, ib = b >= 0 && b < G.num_items ? map[b] : -1;
  if (ia < 0 || ib < 0 || ia >= nu || ib >= nu) {
    igmc_set_err(err, IGMC_ERR_CANDIDATES);
    out[e] = 0.f;
    return;
  }
  const int da = col_deg(G, a);
  out[e] = item_cosine(cocount(T, nu, ia, ib, da), da, col_deg(G, b));
}

}  // namespace

extern "C" int igmc_diverse_ws_bytes(int num_query, int pool, int num_items, int64_t bound, int64_t* table_bytes,
                                     int* chunk) {
  if (!table_bytes || num_query < 1 || pool < 1 || num_items < 1) return -1;
  const long long cap = bound > 0 ? (long long)bound : DIVERSE_WS_DEFAULT;
  auto bytes_of = [&](long long users) {
    return tri_entries(min(users * pool, (long long)num_items)) * (long long)sizeof(uint32_t);
  };
  long long c = num_query;
  if (bytes_of(c) > cap) {   // the largest chunk whose worst-case union fits the bound, at least one query
    long long lo = 1, hi = c;
    while (hi - lo > 1) {
      const long long mid = (lo + hi) >> 1;
      if (bytes_of(mid) <= cap) lo = mid; else hi = mid;
    }
    c = lo;
  }
  *table_bytes = bytes_of(c);
  if (chunk) *chunk = (int)c;
  return 0;
}

extern "C" int igmc_item_union(const int64_t* items, int64_t n, int num_items, uint32_t* bitmap, int32_t* map,
                               int32_t* list, int32_t* nu, int* err, void* stream) {
  if (n < 0 || num_items < 1 || (n > 0 && !items) || !bitmap || !map || !list || !nu) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(bitmap, 0, (size_t)((num_items + 31) >> 5) * sizeof(uint32_t), st);
  IGMC_CUDA_CHECK_LAUNCH();
  if (n > 0) {
    k_dv_mark<<<(unsigned)((n + MARK_THREADS - 1) / MARK_THREADS), MARK_THREADS, 0, st>>>(items, n, num_items, bitmap,
                                                                                          err);
    IGMC_CUDA_CHECK_LAUNCH();
  }
  k_dv_scan<<<1, SCAN_THREADS, 0, st>>>(bitmap, num_items, map, list, nu);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_cocount(const igmc_csr_t* G, const int32_t* map, int nu, uint32_t* table, int64_t table_cap,
                            void* stream) {
  if (!G || !G->row_ptr || !G->col_idx || !map || nu < 0 || nu > G->num_items) return -1;
  const long long need = tri_entries(nu);
  if (need > table_cap) return -2;
  if (need == 0) return 0;
  if (!table) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(table, 0, (size_t)need * sizeof(uint32_t), st);
  IGMC_CUDA_CHECK_LAUNCH();
  if (G->num_users > 0) {
    k_dv_count<<<min(G->num_users, 65535), COUNT_THREADS, 0, st>>>(*G, map, nu, table);
    IGMC_CUDA_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int igmc_diverse_select(const igmc_csr_t* G, const int64_t* pool_item, const float* pool_score,
                                   int num_query, int pool, int k, float penalty, const int32_t* map, int nu,
                                   const uint32_t* table, int64_t* out_item, float* out_score, float* out_key,
                                   int* err, void* stream) {
  if (!G || !G->col_ptr || num_query < 0 || pool < 1 || pool > IGMC_TOPK_MAX || k < 1 || k > pool) return -1;
  if (!(penalty >= 0.f) || isinf(penalty)) return -1;
  if (num_query == 0) return 0;
  if (!pool_item || !pool_score || !map || nu < 0 || (nu > 1 && !table) || !out_item || !out_score || !out_key)
    return -1;
  k_dv_select<<<num_query, SELECT_THREADS, 0, (cudaStream_t)stream>>>(*G, pool_item, pool_score, pool, k, penalty, map,
                                                                      nu, table, out_item, out_score, out_key, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_item_cosine(const igmc_csr_t* G, const int64_t* items, int Q, const int32_t* map, int nu,
                                const uint32_t* table, float* out, int* err, void* stream) {
  if (!G || !G->col_ptr || Q < 0 || nu < 0) return -1;
  if (Q == 0) return 0;
  if (!items || !map || (nu > 1 && !table) || !out) return -1;
  const long long n = (long long)Q * Q;
  k_dv_cosine<<<(unsigned)((n + COSINE_THREADS - 1) / COSINE_THREADS), COSINE_THREADS, 0, (cudaStream_t)stream>>>(
      *G, items, Q, map, nu, table, out, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
