// Shared device helpers for the IGMC hot-path kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define IGMC_WARP 32
#define IGMC_FULL 0xffffffffu

// ---- error codes written to the device-side error word -------------------------------------
enum {
  IGMC_OK = 0,
  IGMC_ERR_NODE_CAP = 1,    // a subgraph side exceeded the node-list capacity
  IGMC_ERR_EDGE_CAP = 2,    // batch edge capacity exceeded
  IGMC_ERR_NODE_TOTAL = 3,  // batch node capacity exceeded
  IGMC_ERR_SMEM_NODES = 4,  // subgraph larger than the model kernel's shared-memory plan
  IGMC_ERR_BAD_BATCH = 5,   // edges not grouped by graph / node ids outside their graph
  IGMC_ERR_NODE_ID16 = 6,   // subgraph of more than 65 535 nodes: beyond the 16-bit neighbour field of the lists
  IGMC_ERR_CANDIDATES = 7,  // inference candidates: a user / item id outside the rating matrix or an inconsistent plan
  IGMC_ERR_GRAPH_UPDATE = 8,  // graph update: an id outside the capacity or a value outside 0..256
  IGMC_ERR_SESSIONS = 9,    // rating sessions: a session / item id out of range, a negative user or a value outside 0..256
  IGMC_ERR_ONLINE = 10,     // online training draw: the rating graph has no ratings
  IGMC_ERR_LABEL = 11,      // extraction: a stored rating label or a pair label outside 0..num_classes-1
};

__device__ __forceinline__ void igmc_set_err(int* err, int code) {
  if (err) atomicCAS(err, 0, code);
}

// workspace carve-ups: every sub-array starts on a 256-byte boundary
__host__ __device__ __forceinline__ size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

// ---- "raw" per-CTA gradient rows of the relation-space kernels (csrc/rgcn_rs.cu -> csrc/optim.cu) -------------
// layer l: [ dW_r : R x inp x 32 | d root : inp x 32 | d bias : 32 ],  inp = in rounded up to 4 (in = in_dim0 for
// layer 0, 32 after).  The (att, basis) chain rule is linear in dW_r, so it is applied ONCE to the sum over CTAs
// (k_grad_reduce_raw) instead of in every CTA.
__host__ __device__ __forceinline__ int igmc_raw_layer_floats(int R, int inp) { return (R + 1) * inp * 32 + 32; }
__host__ __device__ __forceinline__ int igmc_raw_off(int R, int in0, int l) {
  const int in0p = (in0 + 3) & ~3;
  return l == 0 ? 0 : igmc_raw_layer_floats(R, in0p) + (l - 1) * igmc_raw_layer_floats(R, 32);
}
__host__ __device__ __forceinline__ int igmc_raw_count(int R, int in0, int L) { return igmc_raw_off(R, in0, L); }

// ---- counter-based hashing (bit-exact twin: oracle/extract_np.py::splitmix64/hash_keys) ----
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// per (seed, pair, side, hop) stream state
__host__ __device__ __forceinline__ uint64_t sample_state(uint64_t seed, int64_t pair_id, int side, int hop) {
  uint64_t tag = (uint64_t)pair_id * 16ull + (uint64_t)hop * 2ull + (uint64_t)side;
  return splitmix64(seed ^ splitmix64(tag));
}
__host__ __device__ __forceinline__ uint32_t sample_key(uint64_t state, int node) {
  return (uint32_t)(splitmix64(state + (uint64_t)(uint32_t)node) >> 32);
}

// edge-dropout draw for directed edge `eid` of the current step: keep iff hash >= thresh (thresh = p * 2^32,
// keep_thresh in csrc/lists.cuh).  thresh 0xFFFFFFFF is p >= 1 (an fp32 p < 1 gives at most 2^32 - 256) and keeps
// nothing: the hash is clamped to 0xFFFFFFFE, which changes no compare against a smaller threshold (a separate test of
// thresh would add spills to the train kernels; the clamp adds none).  Twin: igmc_b200/models.py::edge_keep_reference.
__host__ __device__ __forceinline__ bool edge_keep(uint64_t seed, uint32_t eid, uint32_t thresh) {
  const uint32_t h = (uint32_t)(splitmix64(seed + (uint64_t)eid) >> 32);
  return (h < 0xFFFFFFFEu ? h : 0xFFFFFFFEu) >= thresh;
}

// fp32 mean of the K checkpoint predictions of batch entry i (preds row stride B), summed in checkpoint order
__device__ __forceinline__ float ckpt_mean(const float* __restrict__ preds, int K, int B, int i) {
  float a = preds[i];
  for (int q = 1; q < K; ++q) a = __fadd_rn(a, preds[(size_t)q * B + i]);
  return K > 1 ? __fdiv_rn(a, (float)K) : a;
}

// Rank-skip search over ascending excluded positions r[0..n): the number t of them with r[q] - q <= c, so that the c-th
// position not in r is c + t (r[q] - q counts the positions below r[q] that are not excluded, non-decreasing in q)
__device__ __forceinline__ long long rank_skip(const int32_t* __restrict__ r, long long n, long long c) {
  long long a = 0, b = n;
  while (a < b) {
    const long long mid = (a + b) >> 1;
    if ((long long)r[mid] - mid <= c) a = mid + 1; else b = mid;
  }
  return a;
}

// the pair that owns position c of a run of per-pair positions: the last q in [0, P) with offsets[q] <= c (pairs
// without positions share their offset with the next pair and own none)
__device__ __forceinline__ int owner(const int64_t* __restrict__ offsets, int P, long long c) {
  int lo = 0, hi = P;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (offsets[mid] <= c) lo = mid; else hi = mid;
  }
  return lo;
}

// ---- warp / block primitives -----------------------------------------------------------------
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(IGMC_FULL, v, o);
  return v;
}
__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(IGMC_FULL, v, o);
  return v;
}
__device__ __forceinline__ int warp_incl_scan_i(int v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(IGMC_FULL, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

// Block-wide exclusive scan of one int per thread.  `ws` is >= 33 ints of shared scratch.
// Returns the exclusive prefix; *total receives the block sum.  Ends with a barrier so `ws`
// can be reused immediately.
__device__ __forceinline__ int block_excl_scan_i(int v, int* ws, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  int incl = warp_incl_scan_i(v, lane);
  if (lane == 31) ws[w] = incl;
  __syncthreads();
  if (w == 0) {
    int s = lane < nw ? ws[lane] : 0;
    int inc = warp_incl_scan_i(s, lane);
    ws[lane] = inc - s;
    if (lane == 31) ws[32] = inc;
  }
  __syncthreads();
  int excl = ws[w] + incl - v;
  *total = ws[32];
  __syncthreads();
  return excl;
}

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

// Block-wide exclusive scan of in(k), k < n, in chunks of one value per thread: out(k, prefix) for every k < n, called
// by the thread that called in(k).  Returns the total.  Every thread of the block calls it.
template <class In, class Out>
__device__ __forceinline__ int block_scan_chunks(int n, int* ws, In in, Out out) {
  int running = 0;
  for (int base = 0; base < n; base += blockDim.x) {
    const int k = base + threadIdx.x;
    const int v = k < n ? in(k) : 0;
    int tot;
    const int ex = block_excl_scan_i(v, ws, &tot);
    if (k < n) out(k, running + ex);
    running += tot;
  }
  return running;
}

// Sum of one float per thread of a 256-thread block in a fixed order; `red` is 8 floats of shared scratch.  Starts
// with a barrier, so consecutive calls may share red; it does not end with one.
__device__ __forceinline__ float block_sum_f256(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum_f(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float s = 0.f;
  for (int w = 0; w < 8; ++w) s += red[w];
  return s;
}

__device__ __forceinline__ int block_sum_i(int v, int* ws) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum_i(v);
  if (lane == 0) ws[w] = v;
  __syncthreads();
  int s = 0;
  if (w == 0) {
    s = lane < nw ? ws[lane] : 0;
    s = warp_sum_i(s);
    if (lane == 0) ws[32] = s;
  }
  __syncthreads();
  s = ws[32];
  __syncthreads();
  return s;
}

// ---- message-passing list entries (igmc_adj_t: neighbour | type << 16 and an edge id), built by the extractor and
// by igmc_batch_prepare.  A list is sorted by (type, neighbour, edge id): the order of this 64-bit key.
__device__ __forceinline__ uint64_t list_key(uint32_t type, uint32_t nbr, uint32_t eid) {
  return ((uint64_t)type << 56) | ((uint64_t)nbr << 32) | (uint64_t)eid;
}
// Warp-wide rank sort of the k keys at key[0..k) (lists are short): the entry of rank r goes to adj[r] / eid[r], its
// edge id offset by eid_base.
__device__ __forceinline__ void rank_sort_list(const uint64_t* __restrict__ key, int k, uint32_t* __restrict__ adj,
                                               int32_t* __restrict__ eid, int eid_base) {
  for (int i = threadIdx.x & 31; i < k; i += 32) {
    const uint64_t x = key[i];
    int rank = 0;
    for (int q = 0; q < k; ++q) rank += (key[q] < x) ? 1 : 0;
    adj[rank] = (uint32_t)((x >> 32) & 0xffffu) | ((uint32_t)(x >> 56) << 16);
    eid[rank] = eid_base + (int32_t)(uint32_t)(x & 0xffffffffu);
  }
}

// ---- async-proxy bulk copies (TMA, 1-D) + mbarrier completion --------------------------------------
// One thread arms the barrier with the byte count (mbar_expect_tx) and issues cp.async.bulk; every consumer
// spins on mbar_wait(parity).  A barrier initialised with count 1 completes a phase when that one arrival AND all
// announced bytes have landed.  Sizes / addresses must be multiples of 16 bytes.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {}
}
// generic-proxy accesses of shared memory made before this fence are ordered before later async-proxy (TMA) writes
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

__device__ __forceinline__ long long igmc_globaltimer() {
  long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ int igmc_smid() {
  int s;
  asm volatile("mov.u32 %0, %smid;" : "=r"(s));
  return s;
}

// ---- programmatic dependent launch (PDL): a kernel launched with the programmatic-serialization attribute may start
// while its predecessor in the stream still runs; pdl_wait() blocks until the predecessor has completed and its
// writes are visible, pdl_trigger() lets the successor's CTAs be scheduled as soon as SMs free up.  Both are no-ops
// for launches without the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

#define IGMC_CUDA_CHECK_LAUNCH()                      \
  do {                                                \
    cudaError_t e__ = cudaGetLastError();             \
    if (e__ != cudaSuccess) return (int)e__ + 1000;   \
  } while (0)

// Launches `kern` on `grid` CTAs of `threads` threads in thread-block clusters of `cluster` CTAs along x, with `smem`
// bytes of dynamic shared memory.  `pdl`: programmatic stream serialization, so the kernel may start under the tail of
// the previous kernel of the stream (it must pdl_wait() before reading that kernel's results).  Returns 0 or the CUDA
// error + 1000.
template <class Kern, class... Args>
int launch_cluster(Kern kern, int grid, int threads, size_t smem, int cluster, bool pdl, cudaStream_t st,
                   Args... args) {
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = cluster;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  if (pdl) {
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.numAttrs = 2;
  }
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, args...);
  return e != cudaSuccess ? (int)e + 1000 : 0;
}
