// SortPooling + 1-D convolution readout of DGCNN_RS, one CTA per graph, everything of a graph in shared memory.
//
// Replaces (reference call sites): global_sort_pool (models.py:155; PyG 1.4.2, SURVEY.md A.4), Conv1d(1,16,97,97) /
// ReLU / MaxPool1d(2,2) / Conv1d(16,32,5,1) / ReLU / flatten / lin1 / ReLU / Dropout / lin2 (models.py:156-165) and
// their autograd.  The sort is a rank computation (n <= a few hundred nodes: n^2/256 compares per thread), order =
// last channel descending, ties by node index (torch's sort leaves ties unspecified).  All reductions have a fixed
// order: results are bitwise run-to-run deterministic.  HBM traffic per graph: the k pooled rows of concat_states,
// the saved activations (c1*k + c1*t1 + dense_dim floats) and, through L2, lin1.weight.
#include "lists.cuh"

namespace {

constexpr int SP_THREADS = 1024;   // 50 CTAs of work per batch: parallelism has to come from inside the CTA
constexpr int SP_WARPS = SP_THREADS / 32;
constexpr int L1O = IGMC_LIN1_OUT;

__host__ __device__ __forceinline__ int al4(int x) { return (x + 3) & ~3; }
__host__ __device__ __forceinline__ int odd(int x) { return x | 1; }   // odd row stride: conflict-free column walks

struct FwdCarve {
  int keys, X, w1, act1, pool, w2, flat, hid, total;
};
__host__ __device__ __forceinline__ FwdCarve fwd_carve(const igmc_sortpool_t& P, int n_cap) {
  FwdCarve c;
  int o = 0;
  c.keys = o; o += al4(n_cap);
  c.X = o;    o += al4(P.k * odd(P.width));
  c.w1 = o;   o += al4(P.c1 * P.width + P.c1);
  c.act1 = o; o += al4(P.c1 * P.k);
  c.pool = o; o += al4(P.c1 * P.t1);
  c.w2 = o;   o += al4(P.c2 * P.c1 * P.kw2 + P.c2);
  c.flat = o; o += al4(P.dense_dim);
  c.hid = o;  o += L1O;
  c.total = o;
  return c;
}

struct BwdCarve {
  int X, w1, act1, pool, w2, dout2, dp, dout1, dhid, total;
};
__host__ __device__ __forceinline__ BwdCarve bwd_carve(const igmc_sortpool_t& P) {
  BwdCarve c;
  int o = 0;
  c.X = o;     o += al4(P.k * odd(P.width));
  c.w1 = o;    o += al4(P.c1 * P.width);
  c.act1 = o;  o += al4(P.c1 * P.k);
  c.pool = o;  o += al4(P.c1 * P.t1);
  c.w2 = o;    o += al4(P.c2 * P.c1 * P.kw2);
  c.dout2 = o; o += al4(P.dense_dim);
  c.dp = o;    o += al4(P.c1 * P.t1);
  c.dout1 = o; o += al4(P.c1 * P.k);
  c.dhid = o;  o += L1O;
  c.total = o;
  return c;
}

// pooled rows X[t][0..width) of graph g (row stride XS), zero rows for padding positions
__device__ __forceinline__ void gather_pooled(const igmc_sortpool_t& P, const float* __restrict__ states,
                                              const int32_t* __restrict__ perm_g, float* __restrict__ X, int XS) {
  for (int idx = threadIdx.x; idx < P.k * P.width; idx += SP_THREADS) {
    const int t = idx / P.width, j = idx - t * P.width;
    const int v = perm_g[t];
    X[t * XS + j] = v >= 0 ? __ldg(states + (size_t)v * P.state_stride + j) : 0.f;
  }
}

__global__ void __launch_bounds__(SP_THREADS)
k_sortpool_forward(igmc_sortpool_t P, const float* __restrict__ params, const float* __restrict__ states,
                   const int32_t* __restrict__ node_ptr, int n_cap, igmc_dropout_t D, int training,
                   igmc_sortpool_saved_t S, const float* __restrict__ y, float loss_scale, float* __restrict__ dpred,
                   float* __restrict__ sqerr, int* err) {
  extern __shared__ __align__(16) float smem[];
  const FwdCarve cv = fwd_carve(P, n_cap);
  float* keys = smem + cv.keys;
  float* X = smem + cv.X;
  float* w1 = smem + cv.w1;
  float* b1 = w1 + P.c1 * P.width;
  float* act1 = smem + cv.act1;
  float* pool = smem + cv.pool;
  float* w2 = smem + cv.w2;
  float* b2 = w2 + P.c2 * P.c1 * P.kw2;
  float* flat = smem + cv.flat;
  float* hid_s = smem + cv.hid;
  const int g = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nb = node_ptr[g], n = node_ptr[g + 1] - nb;
  const int k = P.k, W = P.width, XS = odd(W);
  if (n > n_cap) {
    if (tid == 0) igmc_set_err(err, IGMC_ERR_SMEM_NODES);
    return;
  }
  // ---- SortPooling: rank of every node by (last channel desc, index asc) ----
  for (int v = tid; v < n; v += SP_THREADS) keys[v] = __ldg(states + (size_t)(nb + v) * P.state_stride + W - 1);
  for (int i = tid; i < P.c1 * W; i += SP_THREADS) w1[i] = params[P.off_conv1_w + i];
  for (int i = tid; i < P.c1; i += SP_THREADS) b1[i] = params[P.off_conv1_b + i];
  for (int i = tid; i < P.c2 * P.c1 * P.kw2; i += SP_THREADS) w2[i] = params[P.off_conv2_w + i];
  for (int i = tid; i < P.c2; i += SP_THREADS) b2[i] = params[P.off_conv2_b + i];
  int32_t* perm_g = S.perm + (size_t)g * k;
  for (int t = tid; t < k; t += SP_THREADS) perm_g[t] = -1;
  __syncthreads();
  for (int v = tid; v < n; v += SP_THREADS) {
    const float kv = keys[v];
    int r = 0;
    for (int u = 0; u < n; ++u) {
      const float ku = keys[u];
      r += (ku > kv) || (ku == kv && u < v);
    }
    S.rank[nb + v] = r;
    if (r < k) perm_g[r] = nb + v;
  }
  __syncthreads();   // perm_g is read back by this block only: block-level visibility of global writes
  gather_pooled(P, states, perm_g, X, XS);
  __syncthreads();
  // ---- Conv1d(1, c1, width, stride width) + ReLU: act1[c][t] ----
  for (int idx = tid; idx < P.c1 * k; idx += SP_THREADS) {
    const int c = idx / k, t = idx - c * k;
    const float* xr = X + t * XS;
    const float* wr = w1 + c * W;
    float s0 = b1[c], s1 = 0.f;
    int j = 0;
    for (; j + 2 <= W; j += 2) { s0 = fmaf(wr[j], xr[j], s0); s1 = fmaf(wr[j + 1], xr[j + 1], s1); }
    if (j < W) s0 = fmaf(wr[j], xr[j], s0);
    const float a = fmaxf(s0 + s1, 0.f);
    act1[idx] = a;
    S.act1[(size_t)g * P.c1 * k + idx] = a;
  }
  __syncthreads();
  // ---- MaxPool1d(2, 2) ----
  for (int idx = tid; idx < P.c1 * P.t1; idx += SP_THREADS) {
    const int c = idx / P.t1, t = idx - c * P.t1;
    const float m = fmaxf(act1[c * k + 2 * t], act1[c * k + 2 * t + 1]);
    pool[idx] = m;
    S.pool[(size_t)g * P.c1 * P.t1 + idx] = m;
  }
  __syncthreads();
  // ---- Conv1d(c1, c2, kw2, 1) + ReLU, flattened channel-major ----
  for (int idx = tid; idx < P.c2 * P.t2; idx += SP_THREADS) {
    const int c2 = idx / P.t2, t = idx - c2 * P.t2;
    float s = b2[c2];
    const float* wr = w2 + c2 * P.c1 * P.kw2;
    for (int c = 0; c < P.c1; ++c) {
      const float* pr = pool + c * P.t1 + t;
      for (int j = 0; j < P.kw2; ++j) s = fmaf(wr[c * P.kw2 + j], pr[j], s);
    }
    const float a = fmaxf(s, 0.f);
    flat[idx] = a;
    S.flat[(size_t)g * P.dense_dim + idx] = a;
  }
  __syncthreads();
  // ---- lin1 + ReLU + Dropout (warp per output, coalesced weight rows) ----
  const float* W1 = params + P.off_lin1_w;
  const uint64_t seed = D.seed_dev ? *D.seed_dev : D.seed;
  for (int o = warp; o < L1O; o += SP_WARPS) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    const float* wr = W1 + (size_t)o * P.dense_dim;
    int i = lane;
    for (; i + 96 < P.dense_dim; i += 128) {   // four independent L2 loads in flight per lane
      const float a0 = __ldg(wr + i), a1 = __ldg(wr + i + 32), a2 = __ldg(wr + i + 64), a3 = __ldg(wr + i + 96);
      s0 = fmaf(a0, flat[i], s0);
      s1 = fmaf(a1, flat[i + 32], s1);
      s2 = fmaf(a2, flat[i + 64], s2);
      s3 = fmaf(a3, flat[i + 96], s3);
    }
    for (; i < P.dense_dim; i += 32) s0 = fmaf(__ldg(wr + i), flat[i], s0);
    const float s = warp_sum_f((s0 + s1) + (s2 + s3));
    if (lane == 0)   // dropout models.py:163
      readout_hidden(s + params[P.off_lin1_b + o], g, o, D, seed, training, hid_s, S);
  }
  __syncthreads();
  if (warp == 0)   // x[:, 0]  models.py:165 (no multiply_by: the factor 1 is exact)
    readout_lin2(P, params, hid_s, 1.f, g, y, loss_scale, S.pred, sqerr, dpred, lane);
}

__global__ void __launch_bounds__(SP_THREADS)
k_sortpool_backward(igmc_sortpool_t P, const float* __restrict__ params, const float* __restrict__ states,
                    const int32_t* __restrict__ node_ptr, int n_cap, igmc_sortpool_saved_t S,
                    const float* __restrict__ dpred, float* __restrict__ dstate, int* err) {
  extern __shared__ __align__(16) float smem[];
  const BwdCarve cv = bwd_carve(P);
  float* X = smem + cv.X;
  float* w1 = smem + cv.w1;
  float* act1 = smem + cv.act1;
  float* pool = smem + cv.pool;
  float* w2 = smem + cv.w2;
  float* dout2 = smem + cv.dout2;
  float* dp = smem + cv.dp;
  float* dout1 = smem + cv.dout1;
  float* dhid_s = smem + cv.dhid;
  const int g = blockIdx.x, tid = threadIdx.x;
  const int nb = node_ptr[g], n = node_ptr[g + 1] - nb;
  const int k = P.k, W = P.width, XS = odd(W), c1 = P.c1, c2 = P.c2, kw2 = P.kw2, t1 = P.t1, t2 = P.t2;
  if (n > n_cap) {
    if (tid == 0) igmc_set_err(err, IGMC_ERR_SMEM_NODES);
    return;
  }
  const int GP = c1 * W + c1 + c2 * c1 * kw2 + c2;
  float* gp = S.gpart + (size_t)g * GP;
  float* gp_w1 = gp, *gp_b1 = gp + c1 * W, *gp_w2 = gp_b1 + c1, *gp_b2 = gp_w2 + c2 * c1 * kw2;

  // d hid (lin2, dropout, relu) ; operands of the later phases -> shared
  readout_dhid(P, params, S, dpred, g, dhid_s, S.dhid, true, tid, SP_THREADS);
  for (int i = tid; i < c1 * W; i += SP_THREADS) w1[i] = params[P.off_conv1_w + i];
  for (int i = tid; i < c2 * c1 * kw2; i += SP_THREADS) w2[i] = params[P.off_conv2_w + i];
  for (int i = tid; i < c1 * k; i += SP_THREADS) act1[i] = S.act1[(size_t)g * c1 * k + i];
  for (int i = tid; i < c1 * t1; i += SP_THREADS) pool[i] = S.pool[(size_t)g * c1 * t1 + i];
  gather_pooled(P, states, S.perm + (size_t)g * k, X, XS);
  __syncthreads();
  // d flat = lin1.weight^T d hid, through the ReLU of conv2
  {
    const float* W1 = params + P.off_lin1_w;
    for (int i = tid; i < P.dense_dim; i += SP_THREADS) {
      float s4[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int o = 0; o < L1O; o += 8) {   // eight independent L2 loads in flight
        float w[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) w[u] = __ldg(W1 + (size_t)(o + u) * P.dense_dim + i);
#pragma unroll
        for (int u = 0; u < 8; ++u) s4[u] = fmaf(w[u], dhid_s[o + u], s4[u]);
      }
      const float s = ((s4[0] + s4[1]) + (s4[2] + s4[3])) + ((s4[4] + s4[5]) + (s4[6] + s4[7]));
      dout2[i] = S.flat[(size_t)g * P.dense_dim + i] > 0.f ? s : 0.f;
    }
  }
  __syncthreads();
  // d conv2.weight[c2][c][j] = sum_t dout2[c2][t] pool[c][t+j] ; d conv2.bias[c2] = sum_t dout2[c2][t]
  for (int idx = tid; idx < c2 * c1 * kw2; idx += SP_THREADS) {
    const int q = idx / kw2, j = idx - q * kw2, cc2 = q / c1, c = q - cc2 * c1;
    const float* dr = dout2 + cc2 * t2;
    const float* pr = pool + c * t1 + j;
    float s = 0.f;
    for (int t = 0; t < t2; ++t) s = fmaf(dr[t], pr[t], s);
    gp_w2[idx] = s;
  }
  for (int cc2 = tid; cc2 < c2; cc2 += SP_THREADS) {
    float s = 0.f;
    for (int t = 0; t < t2; ++t) s += dout2[cc2 * t2 + t];
    gp_b2[cc2] = s;
  }
  // d pool[c][t'] = sum_{c2, j} conv2.weight[c2][c][j] dout2[c2][t'-j]
  for (int idx = tid; idx < c1 * t1; idx += SP_THREADS) {
    const int c = idx / t1, t = idx - c * t1;
    float s = 0.f;
    for (int cc2 = 0; cc2 < c2; ++cc2) {
      const float* wr = w2 + (cc2 * c1 + c) * kw2;
      const float* dr = dout2 + cc2 * t2;
      for (int j = 0; j < kw2; ++j) {
        const int tt = t - j;
        if (tt >= 0 && tt < t2) s = fmaf(wr[j], dr[tt], s);
      }
    }
    dp[idx] = s;
  }
  __syncthreads();
  // d act1 through MaxPool (first maximum takes the gradient) and the ReLU of conv1
  for (int idx = tid; idx < c1 * k; idx += SP_THREADS) {
    const int c = idx / k, t = idx - c * k, tp = t >> 1;
    float d = 0.f;
    if (tp < t1) {
      const float a0 = act1[c * k + 2 * tp], a1 = act1[c * k + 2 * tp + 1];
      const int arg = a1 > a0 ? 1 : 0;
      if ((t & 1) == arg && act1[idx] > 0.f) d = dp[c * t1 + tp];
    }
    dout1[idx] = d;
  }
  __syncthreads();
  // d conv1.weight[c][j] = sum_t dout1[c][t] X[t][j] ; d conv1.bias[c]
  for (int idx = tid; idx < c1 * W; idx += SP_THREADS) {
    const int c = idx / W, j = idx - c * W;
    const float* dr = dout1 + c * k;
    float s = 0.f;
    for (int t = 0; t < k; ++t) s = fmaf(dr[t], X[t * XS + j], s);
    gp_w1[idx] = s;
  }
  for (int c = tid; c < c1; c += SP_THREADS) {
    float s = 0.f;
    for (int t = 0; t < k; ++t) s += dout1[c * k + t];
    gp_b1[c] = s;
  }
  // d concat_states: pooled rows get conv1.weight^T dout1[:, rank], every other entry of the graph is zero
  for (int idx = tid; idx < n * P.state_stride; idx += SP_THREADS) {
    const int v = idx / P.state_stride, j = idx - v * P.state_stride;
    float s = 0.f;
    if (j < W) {
      const int r = S.rank[nb + v];
      if (r < k)
        for (int c = 0; c < c1; ++c) s = fmaf(w1[c * W + j], dout1[c * k + r], s);
    }
    dstate[(size_t)(nb + v) * P.state_stride + j] = s;
  }
}

// one thread per readout parameter: fixed-order sums over the graphs of the batch
__global__ void __launch_bounds__(256)
k_sortpool_grad(igmc_sortpool_t P, int B, igmc_sortpool_saved_t S, const float* __restrict__ dpred, float grad_scale,
                float* __restrict__ grad) {
  const int p = P.param_begin + blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P.param_end) return;
  const int GP = P.c1 * P.width + P.c1 + P.c2 * P.c1 * P.kw2 + P.c2;
  const int n_w1 = P.c1 * P.width, n_w2 = P.c2 * P.c1 * P.kw2;
  int q = -1;
  if (p >= P.off_conv1_w && p < P.off_conv1_w + n_w1) q = p - P.off_conv1_w;
  else if (p >= P.off_conv1_b && p < P.off_conv1_b + P.c1) q = n_w1 + (p - P.off_conv1_b);
  else if (p >= P.off_conv2_w && p < P.off_conv2_w + n_w2) q = n_w1 + P.c1 + (p - P.off_conv2_w);
  else if (p >= P.off_conv2_b && p < P.off_conv2_b + P.c2) q = n_w1 + P.c1 + n_w2 + (p - P.off_conv2_b);
  float s = 0.f;
  if (q >= 0) {
    for (int g = 0; g < B; ++g) s += S.gpart[(size_t)g * GP + q];
  } else {
    readout_param_grad_sum(P, p, P.dense_dim, B, S.dhid, S.flat, S.hid, dpred, s);
  }
  grad[p] = s * grad_scale;   // alignment padding between parameters gets 0
}

int check_plan(const igmc_sortpool_t* P) {
  if (P->k < 2 * P->kw2 || P->width < 1 || P->width > P->state_stride) return -20;
  if (P->t1 != P->k / 2 || P->t2 != P->t1 - P->kw2 + 1 || P->t2 < 1 || P->dense_dim != P->c2 * P->t2) return -21;
  if (P->c1 < 1 || P->c2 < 1 || P->kw2 < 1) return -22;
  return 0;
}

}  // namespace

extern "C" int igmc_sortpool_plan(const igmc_sortpool_t* P, int n_cap, int backward) {
  int rc = check_plan(P);
  if (rc) return rc;
  const size_t b = (size_t)(backward ? bwd_carve(*P).total : fwd_carve(*P, n_cap).total) * sizeof(float);
  return b > 227 * 1024 ? -3 : (int)b;
}

extern "C" int igmc_sortpool_forward(const igmc_sortpool_t* P, const float* params, const float* states,
                                     const int32_t* node_ptr, int B, int n_cap, const igmc_dropout_t* D, int training,
                                     const igmc_sortpool_saved_t* S, const float* y, float loss_scale, float* dpred,
                                     float* sqerr, int* err, void* stream) {
  if (B <= 0) return 0;
  const int smem = igmc_sortpool_plan(P, n_cap, 0);
  if (smem < 0) return smem;
  cudaFuncSetAttribute(k_sortpool_forward, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  k_sortpool_forward<<<B, SP_THREADS, smem, (cudaStream_t)stream>>>(*P, params, states, node_ptr, n_cap, *D, training,
                                                                   *S, y, loss_scale, dpred, sqerr, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_sortpool_backward(const igmc_sortpool_t* P, const float* params, const float* states,
                                      const int32_t* node_ptr, int B, int n_cap, const igmc_sortpool_saved_t* S,
                                      const float* dpred, float* dstate, float grad_scale, float* grad, int* err,
                                      void* stream) {
  if (B <= 0) return 0;
  const int smem = igmc_sortpool_plan(P, n_cap, 1);
  if (smem < 0) return smem;
  cudaStream_t st = (cudaStream_t)stream;
  cudaFuncSetAttribute(k_sortpool_backward, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  k_sortpool_backward<<<B, SP_THREADS, smem, st>>>(*P, params, states, node_ptr, n_cap, *S, dpred, dstate, err);
  IGMC_CUDA_CHECK_LAUNCH();
  const int np = P->param_end - P->param_begin;
  k_sortpool_grad<<<(np + 255) / 256, 256, 0, st>>>(*P, B, *S, dpred, grad_scale, grad);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
