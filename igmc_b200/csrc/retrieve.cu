// Candidate retrieval by bridge count (igmc_b200/recommend.py: corated_items).
//
// With h = 1 the enclosing subgraph of an unrated pair (u, v) holds u's star, v's star and the "bridge" edges (u', i):
// u' rated v, u rated i, u' != u, u' rated i.  Their number is the number of 3-paths u - i - u' - v,
//   paths[v] = sum over u' != u of |N(u) & N(u')| * [u' rated v].
// Without a bridge the two targets lie in disconnected stars and the model sees no signal joining them, so the items
// with the most bridges are the candidates worth scoring.  One CTA per query user (a fixed grid loops over the users
// when the histograms live in global memory):
//   pass 1 (push)  w[u'] += 1 for every i in row(u), u' in col(i), u' != u      integer atomics, sum deg(i) updates
//   pass 2 (pull)  paths[v] = sum over u' in col(v) of w[u']                     a warp per item, one writer, nnz reads
//   select         radix select of the M-th largest count (8 bits a pass), ties at the threshold in ascending item
//                  order, then a bitonic sort of the chosen (~paths, item) keys: paths descending, item ascending
// Integer arithmetic only and every output has one writer: two runs are bit-identical.
#include "common.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int THREADS = 512;
constexpr int WARPS = THREADS / 32;
constexpr int GLOBAL_CTAS = 264;                  // two per H100 SM when the histograms live in global memory
constexpr size_t SMEM_LIMIT = 200 * 1024;         // dynamic shared memory of the shared-memory regime

__host__ __device__ __forceinline__ size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

__host__ __device__ __forceinline__ int pow2_at_least(int n) {
  int p = 1;
  while (p < n) p <<= 1;
  return p;
}

// bytes of one CTA's histograms and sort keys: w [num_users], paths [num_items], keys [pow2 >= m]
size_t row_bytes(int num_users, int num_items, int m) {
  return align256((size_t)num_users * 4) + align256((size_t)num_items * 4) + (size_t)pow2_at_least(m) * 8;
}

bool fits_shared(int num_users, int num_items, int m) { return row_bytes(num_users, num_items, m) <= SMEM_LIMIT; }

// exclusive prefix over the block of one 0/1 flag per thread; `wsum` >= WARPS + 1 ints of shared scratch.  Returns the
// flags set in threads before this one; *total the block's sum.  Ends with a barrier.
__device__ __forceinline__ int block_excl_count(bool f, int* wsum, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned b = __ballot_sync(IGMC_FULL, f);
  if (lane == 0) wsum[w] = __popc(b);
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int q = 0; q < WARPS; ++q) {
      const int c = wsum[q];
      wsum[q] = s;
      s += c;
    }
    wsum[WARPS] = s;
  }
  __syncthreads();
  const int r = wsum[w] + __popc(b & ((1u << lane) - 1u));
  *total = wsum[WARPS];
  __syncthreads();
  return r;
}

// SESS: query j is session j of Q (igmc_sessions_t): N(u) is its session row, u = Q.users[j] its real id (a new
// user, u >= num_users, is in no column of G and is never looked up in w)
template <bool SESS>
__device__ __forceinline__ void
corated(const igmc_csr_t& G, const int32_t* __restrict__ users, int U, int m, int exclude_rated, int in_shared,
        unsigned char* __restrict__ ws, size_t ws_row, int32_t* __restrict__ out_items, int32_t* __restrict__ out_paths,
        int* err, const igmc_sessions_t& Q) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ int hist[256];
  __shared__ int wsum[WARPS + 1];
  __shared__ int s_sel;
  unsigned char* base = in_shared ? smem_raw : ws + (size_t)blockIdx.x * ws_row;
  const int nu = G.num_users, ni = G.num_items;
  unsigned* w = reinterpret_cast<unsigned*>(base);
  unsigned* paths = reinterpret_cast<unsigned*>(base + align256((size_t)nu * 4));
  unsigned long long* keys =
      reinterpret_cast<unsigned long long*>(base + align256((size_t)nu * 4) + align256((size_t)ni * 4));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  for (int j = blockIdx.x; j < U; j += gridDim.x) {
    int32_t* oi = out_items + (size_t)j * m;
    int32_t* op = out_paths + (size_t)j * m;
    const int u = SESS ? Q.users[j] : users[j];
    if (!SESS && (u < 0 || u >= nu)) {
      if (threadIdx.x == 0) igmc_set_err(err, IGMC_ERR_CANDIDATES);
      for (int r = threadIdx.x; r < m; r += THREADS) {
        oi[r] = -1;
        op[r] = 0;
      }
      continue;
    }
    for (int x = threadIdx.x; x < nu; x += THREADS) w[x] = 0;
    __syncthreads();
    // pass 1: user overlap, a warp per rated item
    const int32_t* qi = SESS ? Q.col_idx : G.col_idx;
    const int r0 = SESS ? Q.row_ptr[j] : G.row_ptr[u], r1 = SESS ? Q.row_ptr[j + 1] : G.row_ptr[u + 1];
    for (int e = r0 + warp; e < r1; e += WARPS) {
      const int i = qi[e];
      for (int q = G.col_ptr[i] + lane; q < G.col_ptr[i + 1]; q += 32) {
        const int v = G.row_idx[q];
        if (v != u) atomicAdd(&w[v], 1u);
      }
    }
    __syncthreads();
    // pass 2: item scores, a warp per item
    for (int v = warp; v < ni; v += WARPS) {
      unsigned s = 0;
      for (int q = G.col_ptr[v] + lane; q < G.col_ptr[v + 1]; q += 32) s += w[G.row_idx[q]];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(IGMC_FULL, s, o);
      if (lane == 0) paths[v] = s;
    }
    __syncthreads();
    if (exclude_rated)
      for (int e = r0 + threadIdx.x; e < r1; e += THREADS) paths[qi[e]] = 0;
    // select: threshold T and the number `need` of ties at T to take (ascending item order); every count > T is taken
    unsigned prefix = 0, mask = 0;
    int need = m;
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int b = threadIdx.x; b < 256; b += THREADS) hist[b] = 0;
      __syncthreads();
      for (int v = threadIdx.x; v < ni; v += THREADS) {
        const unsigned p = paths[v];
        if (p != 0 && (p & mask) == prefix) atomicAdd(&hist[(p >> shift) & 255], 1);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        int above = 0, d = 255;
        for (; d >= 0; --d) {
          if (above + hist[d] >= need) break;
          above += hist[d];
        }
        // d < 0 only on the first pass, when fewer than m items have a bridge: take every one of them
        s_sel = d < 0 ? -1 : (d | ((need - above) << 8));
      }
      __syncthreads();
      const int sel = s_sel;
      __syncthreads();
      if (sel < 0) {
        prefix = 1;
        mask = 0;
        need = m;
        break;
      }
      prefix |= (unsigned)(sel & 255) << shift;
      mask |= 255u << shift;
      need = sel >> 8;
    }
    // with mask == 0 every nonzero count is taken (there are at most m of them); else counts > prefix and the first
    // `need` items whose count equals prefix
    const unsigned T = prefix;
    int ties = 0, nsel = 0;
    for (int c0 = 0; c0 < ni; c0 += THREADS) {
      const int v = c0 + threadIdx.x;
      const unsigned p = v < ni ? paths[v] : 0u;
      const bool tie = mask != 0 && p == T;
      int tot;
      const int tr = ties + block_excl_count(tie, wsum, &tot);
      ties += tot;
      const bool take = p != 0 && (mask == 0 || p > T || (tie && tr < need));
      const int pos = nsel + block_excl_count(take, wsum, &tot);
      if (take) keys[pos] = ((unsigned long long)(~p) << 32) | (unsigned)v;
      nsel += tot;
    }
    const int n2 = pow2_at_least(nsel > 0 ? nsel : 1);
    for (int x = nsel + threadIdx.x; x < n2; x += THREADS) keys[x] = ~0ull;
    __syncthreads();
    for (int k = 2; k <= n2; k <<= 1) {
      for (int jj = k >> 1; jj > 0; jj >>= 1) {
        for (int x = threadIdx.x; x < n2; x += THREADS) {
          const int y = x ^ jj;
          if (y > x) {
            const unsigned long long a = keys[x], b = keys[y];
            if ((a > b) == ((x & k) == 0)) {
              keys[x] = b;
              keys[y] = a;
            }
          }
        }
        __syncthreads();
      }
    }
    for (int r = threadIdx.x; r < m; r += THREADS) {
      if (r < nsel) {
        const unsigned long long key = keys[r];
        oi[r] = (int32_t)(key & 0xffffffffull);
        op[r] = (int32_t)(~(unsigned)(key >> 32));
      } else {
        oi[r] = -1;
        op[r] = 0;
      }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(THREADS)
k_corated(igmc_csr_t G, const int32_t* __restrict__ users, int U, int m, int exclude_rated, int in_shared,
          unsigned char* __restrict__ ws, size_t ws_row, int32_t* __restrict__ out_items,
          int32_t* __restrict__ out_paths, int* err) {
  corated<false>(G, users, U, m, exclude_rated, in_shared, ws, ws_row, out_items, out_paths, err, igmc_sessions_t{});
}

__global__ void __launch_bounds__(THREADS)
k_corated_sess(igmc_csr_t G, igmc_sessions_t Q, int m, int exclude_rated, int in_shared,
               unsigned char* __restrict__ ws, size_t ws_row, int32_t* __restrict__ out_items,
               int32_t* __restrict__ out_paths, int* err) {
  corated<true>(G, nullptr, Q.num_sessions, m, exclude_rated, in_shared, ws, ws_row, out_items, out_paths, err, Q);
}

}  // namespace

extern "C" int igmc_corated_ws_bytes(int num_users, int num_items, int num_query, int m, int64_t* bytes) {
  if (!bytes || num_users < 0 || num_items < 1 || num_query < 0 || m < 1 || m > num_items) return -1;
  if (fits_shared(num_users, num_items, m) || num_query == 0) {
    *bytes = 0;
    return 0;
  }
  const int ctas = num_query < GLOBAL_CTAS ? num_query : GLOBAL_CTAS;
  *bytes = (int64_t)ctas * (int64_t)row_bytes(num_users, num_items, m);
  return 0;
}

extern "C" int igmc_corated_items(const igmc_csr_t* G, const int32_t* users, int num_query, int m, int exclude_rated,
                                  void* ws, int64_t ws_bytes, int32_t* items, int32_t* paths, int* err,
                                  void* stream) {
  if (!G || num_query < 0 || m < 1 || m > G->num_items) return -1;
  if (num_query == 0) return 0;
  if (!users || !items || !paths) return -1;
  const int nu = G->num_users, ni = G->num_items;
  const size_t row = row_bytes(nu, ni, m);
  const bool shared = fits_shared(nu, ni, m);
  int grid = num_query;
  if (!shared) {
    grid = num_query < GLOBAL_CTAS ? num_query : GLOBAL_CTAS;
    if (!ws || ws_bytes < (int64_t)grid * (int64_t)row) return -2;
  }
  const size_t smem = shared ? row : 0;
  // opted in at every size: the static histogram and scan words count against the default 48 KB as well
  cudaFuncSetAttribute(k_corated, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  k_corated<<<grid, THREADS, smem, (cudaStream_t)stream>>>(*G, users, num_query, m, exclude_rated ? 1 : 0,
                                                           shared ? 1 : 0, static_cast<unsigned char*>(ws), row, items,
                                                           paths, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_corated_sessions(const igmc_csr_t* G, const igmc_sessions_t* S, int m, int exclude_rated,
                                     void* ws, int64_t ws_bytes, int32_t* items, int32_t* paths, int* err,
                                     void* stream) {
  if (!G || !S || S->num_sessions < 0 || m < 1 || m > G->num_items) return -1;
  const int U = S->num_sessions;
  if (U == 0) return 0;
  if (!S->users || !S->row_ptr || !items || !paths) return -1;
  const int nu = G->num_users, ni = G->num_items;
  const size_t row = row_bytes(nu, ni, m);
  const bool shared = fits_shared(nu, ni, m);
  int grid = U;
  if (!shared) {
    grid = U < GLOBAL_CTAS ? U : GLOBAL_CTAS;
    if (!ws || ws_bytes < (int64_t)grid * (int64_t)row) return -2;
  }
  const size_t smem = shared ? row : 0;
  // opted in at every size: the static histogram and scan words count against the default 48 KB as well
  cudaFuncSetAttribute(k_corated_sess, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  k_corated_sess<<<grid, THREADS, smem, (cudaStream_t)stream>>>(*G, *S, m, exclude_rated ? 1 : 0, shared ? 1 : 0,
                                                                static_cast<unsigned char*>(ws), row, items, paths,
                                                                err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
