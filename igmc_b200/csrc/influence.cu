// Per-pair gradients and training-data influence (TracIn-CP, DESIGN §13).
//
//   k_pair_seed        d l / d lin2 output per graph: 2 (f - y[tag]) multiply_by (loss seed) or multiply_by (score seed)
//   k_pair_grad_rows   conv block of every graph's gradient from parameter-layout partial rows (plan 0, L2 plan)
//   k_pair_grad_raw    the same from the raw rows of the cluster plans, (att, basis) chain rule per graph
//   k_pair_readout     lin1 / lin2 gradients materialised (pair_gradients) and / or the graph's factor row
//   k_self_influence   eta * ||g||^2 added to self[tag] (conv block squared + the readout's factor form)
//   k_infl_partial     split-K FFMA tiles of <G_b, G_t> over the conv block, fixed K chunk per split
//   k_infl_finish      fixed-order sum of the splits + the readout's factor terms, S = S + eta * value
//   k_infl_topk        per test pair: merge a batch's values into the running proponent / opponent lists
//
// Every sum has one writer and a fixed order, and no launch shape depends on the batch size except the number of
// tiles: runs are bit-identical across batch sizes, graph replay and repetitions.
#include <cmath>

#include "common.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int HID = IGMC_HIDDEN;
constexpr int L1O = IGMC_LIN1_OUT;
constexpr int INFL_KC = 256;       // conv-block entries per split of the influence GEMM (independent of B and T)
constexpr int TILE = 64;           // output tile of the influence GEMM: 64 training x 64 test pairs
constexpr int KS = 32;             // k-slice held in shared memory

// factor row of one pair: dhid [128] | feat [F] | hid [128] | dpred, F = 2 * 32 * L
__host__ __device__ __forceinline__ int factor_count(int L) { return L1O + 2 * HID * L + L1O + 1; }

__global__ void k_pair_seed(const float* __restrict__ pred, const float* __restrict__ y, const int64_t* __restrict__ tag,
                            int B, float multiply_by, float* __restrict__ dpred) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= B) return;
  const long long t = tag[g];
  float d = 0.f;
  if (t >= 0) {
    if (y) {
      const float diff = pred[g] - y[t];
      d = 2.f * diff * multiply_by;   // readout_lin2 (lists.cuh) at loss_scale 1
    } else {
      d = multiply_by;
    }
  }
  dpred[g] = d;
}

// destination row of graph g: g itself, or (scatter) its tag; -1 = nothing to write
__device__ __forceinline__ long long dest_row(const int64_t* __restrict__ tag, int scatter, int g) {
  const long long t = tag[g];
  return scatter ? t : (long long)g;
}

// blockIdx.y = graph g, thread = parameter p < conv_param_count: the sum of g's `CL` rows in rank order
__global__ void __launch_bounds__(256)
k_pair_grad_rows(int PC, int CL, const float* __restrict__ gpart, const int64_t* __restrict__ tag, int scatter,
                 float* __restrict__ out, int ld) {
  const int g = blockIdx.y, p = blockIdx.x * 256 + threadIdx.x;
  if (p >= PC) return;
  const long long row = dest_row(tag, scatter, g);
  if (row < 0) return;
  float s = 0.f;
  if (tag[g] >= 0)
    for (int c = 0; c < CL; ++c) s += gpart[((size_t)g * CL + c) * PC + p];
  out[(size_t)row * ld + p] = s;
}

// block (l, g): layer l of graph g from its CL raw rows.  Per input row k: dWs[r][j] (and d root, d bias at k = 0) =
// the sum of the rows in rank order; d basis[b][k][j] = sum_r att[r,b] dWs[r][j]; d att[r,b] += <dWs[r], basis[b][k]>
// over k in order (thread (r, b) owns the sum).
__global__ void __launch_bounds__(256)
k_pair_grad_raw(igmc_model_t M, const float* __restrict__ params, int CL, const float* __restrict__ gpart,
                const int64_t* __restrict__ tag, int scatter, float* __restrict__ out, int ld) {
  const int l = blockIdx.x, g = blockIdx.y, tid = threadIdx.x;
  const long long row = dest_row(tag, scatter, g);
  if (row < 0) return;
  const bool real = tag[g] >= 0;
  const int R = M.num_relations, NB = M.num_bases, in0 = M.in_dim0;
  const int in = l == 0 ? in0 : HID, inp = (in + 3) & ~3;
  const int RC = igmc_raw_count(R, in0, M.num_layers);
  const float* gp = gpart + (size_t)g * CL * RC + igmc_raw_off(R, in0, l);
  float* o = out + (size_t)row * ld;
  __shared__ float dWs[13][HID];      // R <= 12 relation rows + root
  __shared__ float att[12 * IGMC_MAX_BASES];
  __shared__ float bs[IGMC_MAX_BASES][HID];
  if (tid < R * NB) att[tid] = params[M.off_att[l] + tid];
  float datt = 0.f;                   // thread tid < R * NB: d att[r][b], r = tid / NB
  for (int k = 0; k < in; ++k) {
    __syncthreads();
    for (int t = tid; t < (R + 1) * HID; t += 256) {
      const int c = t >> 5, j = t & 31;
      float s = 0.f;
      if (real)
        for (int q = 0; q < CL; ++q) s += gp[(size_t)q * RC + (c * inp + k) * HID + j];
      dWs[c][j] = s;
    }
    if (tid < NB * HID) bs[tid >> 5][tid & 31] = params[M.off_basis[l] + ((tid >> 5) * in + k) * HID + (tid & 31)];
    __syncthreads();
    if (tid < NB * HID) {
      const int b = tid >> 5, j = tid & 31;
      float s = 0.f;
      for (int r = 0; r < R; ++r) s = fmaf(att[r * NB + b], dWs[r][j], s);
      o[M.off_basis[l] + (b * in + k) * HID + j] = s;
    } else if (tid < (NB + 1) * HID) {
      const int j = tid & 31;
      o[M.off_root[l] + k * HID + j] = dWs[R][j];
    }
    if (tid < R * NB) {
      const int r = tid / NB, b = tid - r * NB;
      float s = 0.f;
      for (int j = 0; j < HID; ++j) s = fmaf(dWs[r][j], bs[b][j], s);
      datt += s;
    }
  }
  if (tid < R * NB) o[M.off_att[l] + tid] = datt;
  if (tid < HID) {
    float s = 0.f;
    if (real)
      for (int q = 0; q < CL; ++q) s += gp[(size_t)q * RC + (R + 1) * inp * HID + tid];
    o[M.off_bias[l] + tid] = s;
  }
}

// blockIdx.y = graph g.  full: the lin1 / lin2 entries of out (stride ld = param_count) from the factors; fac: the
// graph's factor row.  Padding graphs write zeros.
__global__ void __launch_bounds__(256)
k_pair_readout(igmc_model_t M, const float* __restrict__ dhid, const float* __restrict__ feat,
               const float* __restrict__ hid, const float* __restrict__ dpred, const int64_t* __restrict__ tag,
               int scatter, float* __restrict__ out, int ld, float* __restrict__ fac) {
  const int g = blockIdx.y;
  const long long row = dest_row(tag, scatter, g);
  if (row < 0) return;
  const bool real = tag[g] >= 0;
  const int F = 2 * HID * M.num_layers, PC = M.conv_param_count;
  const int q = blockIdx.x * 256 + threadIdx.x;
  if (out) {
    const int p = PC + q;
    if (p < M.param_count) {
      float s = 0.f;
      if (p >= M.off_lin1_w && p < M.off_lin1_w + L1O * F) {
        const int r = p - M.off_lin1_w, oo = r / F, i = r - oo * F;
        s = dhid[(size_t)g * L1O + oo] * feat[(size_t)g * F + i];
      } else if (p >= M.off_lin1_b && p < M.off_lin1_b + L1O) {
        s = dhid[(size_t)g * L1O + p - M.off_lin1_b];
      } else if (p >= M.off_lin2_w && p < M.off_lin2_w + L1O) {
        s = dpred[g] * hid[(size_t)g * L1O + p - M.off_lin2_w];
      } else if (p == M.off_lin2_b) {
        s = dpred[g];
      }
      out[(size_t)row * ld + p] = real ? s : 0.f;
    }
  }
  const int FW = factor_count(M.num_layers);
  if (fac && q < FW) {
    float v;
    if (q < L1O) v = dhid[(size_t)g * L1O + q];
    else if (q < L1O + F) v = feat[(size_t)g * F + q - L1O];
    else if (q < L1O + F + L1O) v = hid[(size_t)g * L1O + q - L1O - F];
    else v = dpred[g];
    fac[(size_t)row * FW + q] = real ? v : 0.f;
  }
}

__device__ __forceinline__ float block_sum_256(float v, float* red) {   // fixed order; ends with a barrier
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum_f(v);
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float s = 0.f;
  for (int w = 0; w < 8; ++w) s += red[w];
  __syncthreads();
  return s;
}

// the readout's share of <G_a, G_b> from two factor rows (lin1: rank-1 dhid (x) feat, plus its bias; lin2: dpred hid,
// plus its bias): (dhid_a . dhid_b)(feat_a . feat_b + 1) + dpred_a dpred_b (hid_a . hid_b + 1).  One warp, lane-strided
// partial sums and the shuffle tree: the same bits wherever it is called from.
__device__ __forceinline__ float readout_dot(const float* __restrict__ fa, const float* __restrict__ fb, int F,
                                             int lane) {
  float dd = 0.f, ff = 0.f, hh = 0.f;
  for (int i = lane; i < L1O; i += 32) dd = fmaf(fa[i], fb[i], dd);
  for (int i = lane; i < F; i += 32) ff = fmaf(fa[L1O + i], fb[L1O + i], ff);
  for (int i = lane; i < L1O; i += 32) hh = fmaf(fa[L1O + F + i], fb[L1O + F + i], hh);
  dd = warp_sum_f(dd);
  ff = warp_sum_f(ff);
  hh = warp_sum_f(hh);
  const float pa = fa[2 * L1O + F], pb = fb[2 * L1O + F];
  return fmaf(dd, ff + 1.f, pa * pb * (hh + 1.f));
}

// block g: self[tag[g]] += eta * ||G_g||^2 (conv rows of stride PC + the factor form of the readout)
__global__ void __launch_bounds__(256)
k_self_influence(int PC, int L, const float* __restrict__ conv, const float* __restrict__ fac,
                 const int64_t* __restrict__ tag, float eta, float* __restrict__ self_out) {
  const int g = blockIdx.x;
  const long long t = tag[g];
  if (t < 0) return;
  __shared__ float red[8];
  __shared__ float s_ro;
  const float* cr = conv + (size_t)g * PC;
  float s = 0.f;
  for (int p = threadIdx.x; p < PC; p += 256) s = fmaf(cr[p], cr[p], s);
  const int FW = factor_count(L);
  if (threadIdx.x < 32) {
    const float* f = fac + (size_t)g * FW;
    const float ro = readout_dot(f, f, 2 * HID * L, threadIdx.x);
    if (threadIdx.x == 0) s_ro = ro;
  }
  const float c = block_sum_256(s, red);
  if (threadIdx.x == 0) self_out[t] = fmaf(eta, c + s_ro, self_out[t]);
}

// blockIdx = (training tile, test tile, split): part[split][b][t] = sum over the split's conv entries
// [split * INFL_KC, +INFL_KC) of Gb[b][p] Gt[t][p], in ascending p (one fmaf chain per output)
__global__ void __launch_bounds__(256)
k_infl_partial(int PC, int B, int T, const float* __restrict__ Gb, const float* __restrict__ Gt,
               float* __restrict__ part) {
  __shared__ float As[KS][TILE + 4];
  __shared__ float Bs[KS][TILE + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int b0 = blockIdx.x * TILE, t0 = blockIdx.y * TILE, split = blockIdx.z;
  const int k0 = split * INFL_KC, k1 = min(k0 + INFL_KC, PC);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int ks = k0; ks < k1; ks += KS) {
#pragma unroll
    for (int q = 0; q < TILE * KS / 256; ++q) {   // 64 rows x 32 k of each side, coalesced along k
      const int e = tid + 256 * q, r = e >> 5, kk = e & 31, p = ks + kk;
      As[kk][r] = (b0 + r < B && p < k1) ? __ldg(Gb + (size_t)(b0 + r) * PC + p) : 0.f;
      Bs[kk][r] = (t0 + r < T && p < k1) ? __ldg(Gt + (size_t)(t0 + r) * PC + p) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < KS; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int b = b0 + ty + 16 * i, t = t0 + tx + 16 * j;
      if (b < B && t < T) part[((size_t)split * B + b) * T + t] = acc[i][j];
    }
}

// one warp per (b, t): the splits summed lane-strided + shuffle tree, the readout's factor terms, S = S + eta * value
// (first: S = eta * value)
__global__ void __launch_bounds__(256)
k_infl_finish(int L, int B, int T, int splits, const float* __restrict__ part, const float* __restrict__ fb,
              const float* __restrict__ ft, float eta, int first, float* __restrict__ S) {
  const int w = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= B * T) return;
  const int b = w / T, t = w - b * T;
  float s = 0.f;
  for (int q = lane; q < splits; q += 32) s += part[((size_t)q * B + b) * T + t];
  s = warp_sum_f(s);
  const int FW = factor_count(L);
  const float ro = readout_dot(fb + (size_t)b * FW, ft + (size_t)t * FW, 2 * HID * L, lane);
  if (lane == 0) S[w] = fmaf(eta, s + ro, first ? 0.f : S[w]);
}

// a ranks before b under key sign * value: key descending, index ascending, NaN after every number, empty slots
// (index < 0) last
__device__ __forceinline__ bool infl_before(float as, long long ai, float bs, long long bi, float sign) {
  if (ai < 0) return false;
  if (bi < 0) return true;
  const float ak = sign * as, bk = sign * bs;
  const bool an = isnan(ak), bn = isnan(bk);
  if (an || bn) return (an && bn) ? ai < bi : bn;
  return ak > bk || (ak == bk && ai < bi);
}

// block t: S[:, t] (index tag[b], padding skipped) merged into the running lists of test pair t by rank counting,
// proponents (sign +1) then opponents (sign -1)
__global__ void __launch_bounds__(256)
k_infl_topk(const float* __restrict__ S, int B, int T, const int64_t* __restrict__ tag, int k,
            float* __restrict__ pro_v, int64_t* __restrict__ pro_i, float* __restrict__ con_v,
            int64_t* __restrict__ con_i) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int t = blockIdx.x, n = k + B;
  long long* I = reinterpret_cast<long long*>(smem_raw);
  float* V = reinterpret_cast<float*>(I + n);
  for (int side = 0; side < 2; ++side) {
    const float sign = side ? -1.f : 1.f;
    float* tv = (side ? con_v : pro_v) + (size_t)t * k;
    int64_t* ti = (side ? con_i : pro_i) + (size_t)t * k;
    __syncthreads();
    for (int e = threadIdx.x; e < k; e += blockDim.x) {
      V[e] = tv[e];
      I[e] = ti[e];
    }
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
      V[k + b] = S[(size_t)b * T + t];
      I[k + b] = tag[b];
    }
    __syncthreads();
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
      const float ev = V[e];
      const long long ei = I[e];
      if (e >= k && ei < 0) continue;
      int r;
      if (e < k) {
        r = e;
      } else {
        int lo = 0, hi = k;   // the running list is ranked
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (infl_before(V[mid], I[mid], ev, ei, sign)) lo = mid + 1; else hi = mid;
        }
        r = lo;
      }
      if (r >= k) continue;
      for (int x = k; x < n && r < k; ++x)
        if (x != e && infl_before(V[x], I[x], ev, ei, sign)) ++r;
      if (r < k) {
        tv[r] = ev;
        ti[r] = ei;
      }
    }
  }
}

int infl_splits(int PC) { return (PC + INFL_KC - 1) / INFL_KC; }

}  // namespace

extern "C" int igmc_pair_factor_count(const igmc_model_t* M) { return factor_count(M->num_layers); }

extern "C" int igmc_pair_seed(const float* pred, const float* y, const int64_t* tag, int B, float multiply_by,
                              float* dpred, void* stream) {
  if (B < 0 || (B > 0 && (!pred || !tag || !dpred))) return -20;
  if (B == 0) return 0;
  k_pair_seed<<<(B + 255) / 256, 256, 0, (cudaStream_t)stream>>>(pred, y, tag, B, multiply_by, dpred);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_pair_grad(const igmc_model_t* M, const float* params, int B, int rows_per_graph,
                              const float* gpart, int raw_rows, const float* dhid, const float* feat, const float* hid,
                              const float* dpred, const int64_t* tag, int scatter, float* grad, int full, float* fac,
                              void* stream) {
  if (!M || B < 0 || rows_per_graph < 1) return -20;
  if (M->readout != 0) return -16;   // an external readout sums its gradient over the batch
  if (B == 0) return 0;
  if (!gpart || !dhid || !feat || !hid || !dpred || !tag || (!grad && !fac)) return -20;
  cudaStream_t st = (cudaStream_t)stream;
  const int PC = M->conv_param_count, ld = full ? M->param_count : PC;
  if (grad) {
    if (raw_rows) {
      if (M->num_relations > 12) return -16;
      k_pair_grad_raw<<<dim3(M->num_layers, B), 256, 0, st>>>(*M, params, rows_per_graph, gpart, tag, scatter, grad,
                                                               ld);
    } else {
      k_pair_grad_rows<<<dim3((PC + 255) / 256, B), 256, 0, st>>>(PC, rows_per_graph, gpart, tag, scatter, grad, ld);
    }
    IGMC_CUDA_CHECK_LAUNCH();
  }
  const int ro = full && grad ? M->param_count - PC : 0, FW = fac ? factor_count(M->num_layers) : 0;
  const int n = ro > FW ? ro : FW;
  if (n > 0) {
    k_pair_readout<<<dim3((n + 255) / 256, B), 256, 0, st>>>(*M, dhid, feat, hid, dpred, tag, scatter,
                                                              full ? grad : nullptr, ld, fac);
    IGMC_CUDA_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int igmc_self_influence(const igmc_model_t* M, int B, const float* conv, const float* fac,
                                   const int64_t* tag, float eta, float* self_out, void* stream) {
  if (!M || B < 0 || (B > 0 && (!conv || !fac || !tag || !self_out))) return -20;
  if (B == 0) return 0;
  k_self_influence<<<B, 256, 0, (cudaStream_t)stream>>>(M->conv_param_count, M->num_layers, conv, fac, tag, eta,
                                                        self_out);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_influence_ws_bytes(const igmc_model_t* M, int B, int T, int64_t* bytes) {
  if (!M || B < 0 || T < 0 || !bytes) return -20;
  *bytes = (int64_t)infl_splits(M->conv_param_count) * B * T * (int64_t)sizeof(float);
  return 0;
}

extern "C" int igmc_influence_accum(const igmc_model_t* M, int B, int T, const float* conv_b, const float* fac_b,
                                    const float* conv_t, const float* fac_t, float eta, int first, void* ws,
                                    int64_t ws_bytes, float* S, void* stream) {
  if (!M || B < 0 || T < 0) return -20;
  if (B == 0 || T == 0) return 0;
  if (!conv_b || !fac_b || !conv_t || !fac_t || !ws || !S) return -20;
  const int PC = M->conv_param_count, splits = infl_splits(PC);
  if (ws_bytes < (int64_t)splits * B * T * (int64_t)sizeof(float)) return -18;
  cudaStream_t st = (cudaStream_t)stream;
  float* part = static_cast<float*>(ws);
  k_infl_partial<<<dim3((B + TILE - 1) / TILE, (T + TILE - 1) / TILE, splits), 256, 0, st>>>(PC, B, T, conv_b, conv_t,
                                                                                           part);
  IGMC_CUDA_CHECK_LAUNCH();
  const int warps = B * T;
  k_infl_finish<<<(warps + 7) / 8, 256, 0, st>>>(M->num_layers, B, T, splits, part, fac_b, fac_t, eta, first, S);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_influence_topk(const float* S, int B, int T, const int64_t* tag, int k, float* pro_value,
                                   int64_t* pro_index, float* con_value, int64_t* con_index, void* stream) {
  if (B < 0 || T < 0 || k < 1 || k > IGMC_TOPK_MAX) return -20;
  if (B == 0 || T == 0) return 0;
  if (!S || !tag || !pro_value || !pro_index || !con_value || !con_index) return -20;
  if (!igmc_topk_fits(k, B)) return -20;
  const size_t smem = (size_t)(k + B) * (sizeof(long long) + sizeof(float));
  if (smem > 48 * 1024)
    cudaFuncSetAttribute(k_infl_topk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  k_infl_topk<<<T, 256, smem, (cudaStream_t)stream>>>(S, B, T, tag, k, pro_value, pro_index, con_value, con_index);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
