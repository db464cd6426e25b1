// Monte-Carlo-dropout draws of predicted ratings (igmc_b200/recommend.py: predict_draws, and recommend /
// recommend_users / recommend_sessions with draws=S).
//
// Draw s of pair (u, v) is a training-mode forward of the pair's enclosing subgraph under the model's own dropout:
// each directed edge kept with probability 1 - adj_dropout, each of the 128 hidden units before lin2 kept with
// probability 0.5 and scaled by 2.  The masks come from counter hashes keyed by (draw_seed, pair id, s, local index),
// never by a batch position, and reach the unchanged model kernels through their injected edge_keep / hidden_keep.
// A batch of B graphs holds G = B / S pairs times S consecutive draws, pair major; graphs G*S..B-1 are padding:
//   k_draws_expand  the G pairs of igmc_candidate_pairs -> B positions (u, v, pair id, tag, draw index)
//   k_draws_mask    one CTA per extracted graph: edge_keep of its edges and hidden_keep of its 128 units
//   k_draws_stats   one thread per pair: its S draws (fp32 checkpoint means) -> value / mean / std by tag, or the
//                   ranking key mean + beta * std that igmc_topk_merge consumes
// Twins: igmc_b200/recommend.py::draws_expand_host / draws_mask_host / draws_stats_host.
#include "common.cuh"
#include "lists.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int EXPAND_THREADS = 256;
constexpr int MASK_THREADS = 128;
constexpr int STATS_THREADS = 128;
// sample_state's hop slot of the draw streams (side 0: edges, side 1: hidden units).  Extraction uses hops
// 1..IGMC_MAX_HOP and the online training draw hop 7.
constexpr int DRAWS_HOP_TAG = 4;

// the stream of draw s of a pair: one state per (seed, pair id, draw, edges / hidden units)
__device__ __forceinline__ uint64_t draw_state(uint64_t seed, int64_t pid, int s, int side) {
  return splitmix64(sample_state(seed, pid, side, DRAWS_HOP_TAG) + (uint64_t)(uint32_t)s);
}

__global__ void __launch_bounds__(EXPAND_THREADS)
k_draws_expand(int S, int B, const int32_t* __restrict__ pu, const int32_t* __restrict__ pv,
               const int64_t* __restrict__ ppid, const int64_t* __restrict__ ptag, int32_t* __restrict__ links_u,
               int32_t* __restrict__ links_v, int64_t* __restrict__ pair_id, int64_t* __restrict__ tag,
               int32_t* __restrict__ draw) {
  const int G = B / S;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
    const bool real = i < G * S;
    const int g = real ? i / S : 0;   // padding: a valid copy of pair 0, tag -1
    links_u[i] = pu[g];
    links_v[i] = pv[g];
    pair_id[i] = ppid[g];
    tag[i] = real ? ptag[g] : -1;
    draw[i] = real ? i - g * S : 0;
  }
}

__global__ void __launch_bounds__(MASK_THREADS)
k_draws_mask(const int32_t* __restrict__ edge_ptr, const int64_t* __restrict__ pair_id, const int64_t* __restrict__ tag,
             const int32_t* __restrict__ draw, float adj_dropout, uint64_t seed, uint8_t* __restrict__ ekeep,
             uint8_t* __restrict__ hkeep) {
  const int i = blockIdx.x;
  const uint32_t thresh = keep_thresh(adj_dropout);
  const int e0 = edge_ptr[i], e1 = edge_ptr[i + 1];
  const bool pad = tag[i] < 0;
  const uint64_t se = draw_state(seed, pair_id[i], draw[i], 0), sh = draw_state(seed, pair_id[i], draw[i], 1);
  for (int e = e0 + threadIdx.x; e < e1; e += blockDim.x)
    ekeep[e] = (pad || edge_keep(se, (uint32_t)(e - e0), thresh)) ? 1 : 0;
  for (int o = threadIdx.x; o < IGMC_LIN1_OUT; o += blockDim.x)
    hkeep[(size_t)i * IGMC_LIN1_OUT + o] = (pad || edge_keep(sh, (uint32_t)o, keep_thresh(0.5f))) ? 1 : 0;
}

// pair g of the batch: its S draws x_s (fp32 checkpoint means of positions g*S + s), mean and the unbiased std in
// fp64 in draw order (no contraction into fma), each rounded once to fp32
__global__ void __launch_bounds__(STATS_THREADS)
k_draws_stats(const float* __restrict__ preds, int K, int B, int S, const int64_t* __restrict__ tag, double beta,
              float* __restrict__ value, float* __restrict__ mean_out, float* __restrict__ std_out,
              float* __restrict__ key) {
  const int G = B / S;
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const int i0 = g * S;
  const long long t = tag[i0];
  double sum = 0.0;
  for (int s = 0; s < S; ++s) {
    const float x = ckpt_mean(preds, K, B, i0 + s);
    sum = __dadd_rn(sum, (double)x);
    if (value && t >= 0) value[t * S + s] = x;
  }
  const double mean = __ddiv_rn(sum, (double)S);
  double sd = 0.0;
  if (S > 1) {
    double ss = 0.0;
    for (int s = 0; s < S; ++s) {
      const double d = __dsub_rn((double)ckpt_mean(preds, K, B, i0 + s), mean);
      ss = __dadd_rn(ss, __dmul_rn(d, d));
    }
    sd = __dsqrt_rn(__ddiv_rn(ss, (double)(S - 1)));
  }
  if (key) key[g] = (float)__dadd_rn(mean, __dmul_rn(beta, sd));
  if (t >= 0 && mean_out) {
    mean_out[t] = (float)mean;
    std_out[t] = (float)sd;
  }
}

}  // namespace

extern "C" int igmc_draws_expand(int S, int B, const int32_t* pair_u, const int32_t* pair_v, const int64_t* pair_pid,
                                 const int64_t* pair_tag, int32_t* links_u, int32_t* links_v, int64_t* pair_id,
                                 int64_t* tag, int32_t* draw, void* stream) {
  if (S < 1 || S > IGMC_DRAWS_MAX || B < S) return -1;
  if (!pair_u || !pair_v || !pair_pid || !pair_tag || !links_u || !links_v || !pair_id || !tag || !draw) return -1;
  k_draws_expand<<<(B + EXPAND_THREADS - 1) / EXPAND_THREADS, EXPAND_THREADS, 0, (cudaStream_t)stream>>>(
      S, B, pair_u, pair_v, pair_pid, pair_tag, links_u, links_v, pair_id, tag, draw);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_draws_mask(const igmc_batch_out_t* O, int B, const int64_t* pair_id, const int64_t* tag,
                               const int32_t* draw, float adj_dropout, uint64_t draw_seed, uint8_t* edge_keep,
                               uint8_t* hidden_keep, void* stream) {
  if (!O || !O->edge_ptr || B <= 0 || !pair_id || !tag || !draw || !edge_keep || !hidden_keep) return -1;
  if (!(adj_dropout >= 0.f && adj_dropout <= 1.f)) return -2;
  k_draws_mask<<<B, MASK_THREADS, 0, (cudaStream_t)stream>>>(O->edge_ptr, pair_id, tag, draw, adj_dropout, draw_seed,
                                                              edge_keep, hidden_keep);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_draws_stats(const float* preds, int K, int B, int S, const int64_t* tag, double beta, float* value,
                                float* mean, float* std, float* key, void* stream) {
  if (!preds || K < 1 || S < 1 || S > IGMC_DRAWS_MAX || B < S || !tag) return -1;
  if (!key && (!value || !mean || !std)) return -1;
  if (!(beta - beta == 0.0)) return -2;   // beta must be finite
  const int G = B / S;
  k_draws_stats<<<(G + STATS_THREADS - 1) / STATS_THREADS, STATS_THREADS, 0, (cudaStream_t)stream>>>(
      preds, K, B, S, tag, beta, value, mean, std, key);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
