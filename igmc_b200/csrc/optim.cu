// Gradient assembly (per-CTA partial rows -> flat bucket), adjacent-rating regulariser and Adam.
//
// Replaces autograd's accumulation + `loss += ARR * sum((w[1:]-w[:-1])**2)` (train_eval.py:167-174)
// + `torch.optim.Adam.step` (train_eval.py:54,177) with TWO launches on the flat parameter bucket, which is
// also what the one NCCL all-reduce per step operates on.
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "lists.cuh"

namespace {

constexpr int HID = IGMC_HIDDEN;

// dW_r[kj] of the adjacent-rating regulariser for one (layer, kj), W_r composed from att and the basis bs (stride KJ
// between bases)
__device__ __forceinline__ float arr_dw_kj(const float* __restrict__ att, const float* __restrict__ bs, int NB, int KJ,
                                           int R, int r, int kj, float* pair) {
  const auto w = [&](int rr) {
    return compose_w(NB, [&](int b) { return att[rr * NB + b]; }, [&](int b) { return bs[b * KJ + kj]; });
  };
  return arr_dw(w, R, r, pair);
}

// Blocks [0, PB): one thread per parameter.
//   conv params = fixed-order sum of the per-CTA partial rows (+ the ARR term for basis entries, thread-local);
//   lin1/lin2 from the saved readout factors; att entries are left to the ARR blocks when arr != 0.
// Blocks [PB, PB + L*R) (arr != 0): block (l, r) owns att[l][r][:]:  sum of the partial rows + arr * <dW_r, basis[b]>,
//   and the regulariser value of the pair (r, r+1).  The last of them to finish writes the loss
//   (sum_g sqerr * loss_scale + arr * sum of the pair values, in fixed order).
__global__ void __launch_bounds__(256)
k_grad_reduce(igmc_model_t M, const float* __restrict__ params, int B, int rows, int PB,
              const float* __restrict__ gpart, const float* __restrict__ dhid, const float* __restrict__ feat,
              const float* __restrict__ hid, const float* __restrict__ dpred, const float* __restrict__ sqerr,
              float loss_scale, float arr, float grad_scale, float* __restrict__ grad, float* __restrict__ loss_out,
              float* __restrict__ reg_ws) {
  const int PC = M.conv_param_count, F = 2 * HID * M.num_layers;
  const int R = M.num_relations, NB = M.num_bases;
  if ((int)blockIdx.x < PB) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < M.param_count) {
      float s = 0.f;
      bool skip = false;
      if (p < PC) {
        for (int g = 0; g < rows; ++g) s += gpart[(size_t)g * PC + p];
        if (arr != 0.f) {
          for (int l = 0; l < M.num_layers; ++l) {
            const int in = l == 0 ? M.in_dim0 : HID, KJ = in * HID;
            const int q = p - M.off_basis[l];
            if (q >= 0 && q < NB * KJ) {   // basis[b][kj]:  += arr * sum_r att[r,b] dW_r[kj]
              const int b = q / KJ, kj = q - b * KJ;
              const float* att = params + M.off_att[l];
              float t = 0.f;
              for (int r = 0; r < R; ++r)
                t = fmaf(att[r * NB + b], arr_dw_kj(att, params + M.off_basis[l], NB, KJ, R, r, kj, nullptr), t);
              s = fmaf(arr, t, s);
            }
            const int qa = p - M.off_att[l];
            if (qa >= 0 && qa < R * NB) skip = true;   // written by the ARR block (l, r)
          }
        }
      } else if (M.readout != 0) {
        skip = true;   // readout parameters belong to the external readout's gradient kernel
      } else {
        readout_param_grad_sum(M, p, F, B, dhid, feat, hid, dpred, s);
      }
      if (!skip) grad[p] = s * grad_scale;
    }
    if (arr == 0.f && blockIdx.x == 0 && threadIdx.x == 0 && loss_out) {
      float s = 0.f;
      if (sqerr)
        for (int g = 0; g < B; ++g) s += sqerr[g];
      loss_out[0] = s * loss_scale;
    }
    return;
  }
  // ---- ARR block (l, r) ----
  const int lr = blockIdx.x - PB, l = lr / R, r = lr - l * R;
  const int in = l == 0 ? M.in_dim0 : HID, KJ = in * HID;
  const int tid = threadIdx.x;
  extern __shared__ float sm_arr[];                 // att [R*NB] | basis [NB*KJ] | dW_r [KJ]
  float* att = sm_arr;
  float* bs = att + ((R * NB + 3) & ~3);
  float* dw = bs + NB * KJ;
  __shared__ float red[8];
  __shared__ int s_last;
  for (int i = tid; i < R * NB; i += 256) att[i] = params[M.off_att[l] + i];
  for (int i = tid; i < NB * KJ; i += 256) bs[i] = params[M.off_basis[l] + i];
  __syncthreads();
  float pair_sum = 0.f;
  for (int kj = tid; kj < KJ; kj += 256) {
    float pr;
    dw[kj] = arr_dw_kj(att, bs, NB, KJ, R, r, kj, &pr);
    pair_sum += pr;
  }
  __syncthreads();
  for (int b = 0; b < NB; ++b) {
    float s = 0.f;
    for (int kj = tid; kj < KJ; kj += 256) s = fmaf(dw[kj], bs[b * KJ + kj], s);
    const float dot = block_sum_f256(s, red);
    // column sum of the partial rows for att[l][r][b]
    float c = 0.f;
    for (int g = tid; g < rows; g += 256) c += gpart[(size_t)g * PC + M.off_att[l] + r * NB + b];
    const float col = block_sum_f256(c, red);
    if (tid == 0) grad[M.off_att[l] + r * NB + b] = (col + arr * dot) * grad_scale;
  }
  const float reg = block_sum_f256(pair_sum, red);
  if (tid == 0) {
    reg_ws[lr] = reg;
    __threadfence();
    int* ticket = reinterpret_cast<int*>(reg_ws + IGMC_MAX_LAYERS * 256);
    s_last = (atomicAdd(ticket, 1) == (int)(gridDim.x - PB) - 1);
  }
  __syncthreads();
  if (s_last && tid == 0) {
    __threadfence();
    float s = 0.f;
    for (int q = 0; q < (int)(gridDim.x - PB); ++q) s += __ldcg(reg_ws + q);
    float mse = 0.f;
    if (sqerr)
      for (int g = 0; g < B; ++g) mse += sqerr[g];
    if (loss_out) loss_out[0] = mse * loss_scale + arr * s;
    *reinterpret_cast<int*>(reg_ws + IGMC_MAX_LAYERS * 256) = 0;   // re-arm for the next step
  }
}

// ---- raw rows of the cluster plans (csrc/rgcn_rs.cu): [rows][igmc_raw_count] with per layer dW_r | d root | d bias ----
// Blocks [0, NA): block (l, k) owns row k of every dW_r of layer l (kj = k*32 + lane):
//   dWs[r][j] = sum over the partial rows (8 warps = 8 interleaved row subsets, added in fixed order)
//               + arr * d reg / d W_r[k][j]
//   d basis[b][k][j] = sum_r att[r,b] dWs[r][j]                       (complete: written to grad)
//   d att[r,b]      += sum_j dWs[r][j] basis[b][k][j]                 (partial over k: scratch, summed by the layer's
//                                                                      last block in k order)
//   reg             += sum_{r<R-1} sum_j (W_{r+1}[k][j] - W_r[k][j])^2   (same)
// Blocks [NA, NA + PB): one thread per parameter for d root / d bias (row sums) and lin1 / lin2 (saved factors).
// The last layer-finaliser writes the loss.  Every sum has a fixed order: bitwise deterministic.
constexpr int RW_ATT = 0;                                   // [L][32][64] partial <dW_r, basis[b]> per (l, k)
constexpr int RW_REGP = IGMC_MAX_LAYERS * 32 * 64;          // [L][32] partial regulariser values
constexpr int RW_REGL = RW_REGP + IGMC_MAX_LAYERS * 32;     // [L] per-layer regulariser
constexpr int RW_TICK = RW_REGL + IGMC_MAX_LAYERS;          // ints: [L] layer tickets, [1] global ticket

// per-warp partial sums of NC columns of the raw rows g == warp (mod 8) -> ps[c][warp][lane]; fixed order
template <int NCT, int UR>
__device__ __forceinline__ void sum_rows(const float* __restrict__ gp, int rows, int RC, int R, int inp, int k, int NC,
                                         int warp, int lane, float (*ps)[8][HID]) {
  int off[NCT];
  float acc[NCT];
#pragma unroll
  for (int c = 0; c < NCT; ++c) {
    off[c] = c < NC ? (c <= R ? (c * inp + k) * HID : (R + 1) * inp * HID) : 0;
    acc[c] = 0.f;
  }
  int g0 = warp;
  for (; g0 + 8 * (UR - 1) < rows; g0 += 8 * UR) {   // full batches: no guards, every load independent
    float v[UR][NCT];
#pragma unroll
    for (int u = 0; u < UR; ++u) {
      const float* gr = gp + (size_t)(g0 + 8 * u) * RC;
#pragma unroll
      for (int c = 0; c < NCT; ++c) v[u][c] = __ldcg(gr + off[c]);
    }
#pragma unroll
    for (int u = 0; u < UR; ++u)
#pragma unroll
      for (int c = 0; c < NCT; ++c) acc[c] += v[u][c];
  }
  if (g0 < rows) {   // last, partial batch: still ONE round of loads (rows past the end read row g0 and add +0)
    float v[UR][NCT];
#pragma unroll
    for (int u = 0; u < UR; ++u) {
      const bool in_range = g0 + 8 * u < rows;
      const float* gr = gp + (size_t)(in_range ? g0 + 8 * u : g0) * RC;
#pragma unroll
      for (int c = 0; c < NCT; ++c) v[u][c] = __ldcg(gr + off[c]);
    }
#pragma unroll
    for (int u = 0; u < UR; ++u) {
      const bool in_range = g0 + 8 * u < rows;
#pragma unroll
      for (int c = 0; c < NCT; ++c) acc[c] += in_range ? v[u][c] : 0.f;
    }
  }
#pragma unroll
  for (int c = 0; c < NCT; ++c)
    if (c < NC) ps[c][warp][lane] = acc[c];
}

// the step's loss from the per-layer regulariser values and the squared errors (one warp; lane-strided partial sums +
// shuffle tree: the same bits wherever it is called from)
__device__ __forceinline__ float loss_from_parts(const float* __restrict__ reg_ws, const float* __restrict__ sqerr, int B,
                                                 int L, float loss_scale, float arr, int lane);

template <bool LOSS_INSIDE>
__device__ __forceinline__ void reduce_raw_block(const igmc_model_t& M, const float* __restrict__ params, int B, int rows,
                                                 int NA, const float* __restrict__ gpart, const float* __restrict__ dhid,
                                                 const float* __restrict__ feat, const float* __restrict__ hid,
                                                 const float* __restrict__ dpred, const float* __restrict__ sqerr,
                                                 float loss_scale, float arr, float grad_scale, float* __restrict__ grad,
                                                 float* __restrict__ loss_out, float* __restrict__ reg_ws) {
  const int R = M.num_relations, NB = M.num_bases, L = M.num_layers, in0 = M.in_dim0;
  const int RC = igmc_raw_count(R, in0, L), F = 2 * HID * L;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if ((int)blockIdx.x >= NA) {   // readout parameters (lin1 / lin2) from the saved factors
    const int p = M.conv_param_count + ((int)blockIdx.x - NA) * 256 + tid;
    if (p >= M.param_count) return;
    float s = 0.f;
    if (readout_param_grad_sum(M, p, F, B, dhid, feat, hid, dpred, s)) grad[p] = s * grad_scale;
    return;
  }
  // ---- block (l, k): row k of dW_0..dW_{R-1} and of d root; block (l, 0) also d bias ----
  int l = 0, k = (int)blockIdx.x;
  if (k >= in0) { l = 1 + (k - in0) / HID; k = (k - in0) % HID; }
  const int in = l == 0 ? in0 : HID, inp = (in + 3) & ~3;
  constexpr int MAXC = 14;                            // R <= 12 relation rows + root + bias
  __shared__ float att[IGMC_MAX_BASES * 16];          // [R][NB]
  __shared__ float bs[IGMC_MAX_BASES][HID];           // basis[b][k][:]
  __shared__ float ps[MAXC][8][HID];                  // per-warp partial row sums
  __shared__ float dWs[12][HID];
  __shared__ float Wc[12][HID];
  __shared__ float red[8];
  __shared__ int s_last;
  // (R * NB <= 48 and NB * 32 <= 128 values: one per thread; loaded now, parked in registers under the row sums)
  const float att_v = tid < R * NB ? params[M.off_att[l] + tid] : 0.f;
  const float bs_v = tid < NB * HID ? params[M.off_basis[l] + ((tid >> 5) * in + k) * HID + (tid & 31)] : 0.f;
  const int NC = R + 1 + (k == 0 ? 1 : 0);
  {
    // column c of this block inside a raw row: c <= R: row k of dW_c / d root; c == R + 1: d bias.
    // warp w sums the partial rows g == w (mod 8); loads are issued in batches (UR rows x NCT columns in flight per
    // thread) BEFORE any of them is consumed - the row sums are L2-latency bound
    const float* gp = gpart + (size_t)igmc_raw_off(R, in0, l) + lane;
    if (NC <= 7) sum_rows<7, 7>(gp, rows, RC, R, inp, k, NC, warp, lane, ps);   // 100 rows: two rounds of 49 loads
    else sum_rows<14, 4>(gp, rows, RC, R, inp, k, NC, warp, lane, ps);
  }
  if (tid < R * NB) att[tid] = att_v;
  if (tid < NB * HID) bs[tid >> 5][tid & 31] = bs_v;
  __syncthreads();
  for (int t = tid; t < NC * HID; t += 256) {
    const int c = t >> 5, j = t & 31;
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += ps[c][w][j];
    if (c < R) {
      dWs[c][j] = s;
      Wc[c][j] = compose_w(NB, [&](int b) { return att[c * NB + b]; }, [&](int b) { return bs[b][j]; });
    } else if (c == R) {
      grad[M.off_root[l] + k * HID + j] = s * grad_scale;
    } else {
      grad[M.off_bias[l] + j] = s * grad_scale;
    }
  }
  __syncthreads();
  float pair_sum = 0.f;
  if (arr != 0.f) {
    for (int t = tid; t < R * HID; t += 256) {
      const int r = t >> 5, j = t & 31;
      float pr;
      const float dw = arr_dw([&](int rr) { return Wc[rr][j]; }, R, r, &pr);
      pair_sum += pr;
      dWs[r][j] = fmaf(arr, dw, dWs[r][j]);
    }
  }
  const float regp = block_sum_f256(pair_sum, red);   // barriers inside: dWs is complete afterwards
  __syncthreads();
  // d basis[b][k][:]
  for (int t = tid; t < NB * HID; t += 256) {
    const int b = t >> 5, j = t & 31;
    float s = 0.f;
    for (int r = 0; r < R; ++r) s = fmaf(att[r * NB + b], dWs[r][j], s);
    grad[M.off_basis[l] + (b * in + k) * HID + j] = s * grad_scale;
  }
  // partial d att[r,b] over this k
  float* wsa = reg_ws + RW_ATT + ((size_t)l * 32 + k) * 64;
  for (int pr = warp; pr < R * NB; pr += 8) {
    const int r = pr / NB, b = pr - r * NB;
    const float s = warp_sum_f(dWs[r][lane] * bs[b][lane]);
    if (lane == 0) wsa[pr] = s;
  }
  int* tick = reinterpret_cast<int*>(reg_ws + RW_TICK);
  if (tid == 0) reg_ws[RW_REGP + l * 32 + k] = regp;
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_last = (atomicAdd(&tick[l], 1) == in - 1);
  }
  __syncthreads();
  if (!s_last) return;
  // ---- last block of layer l: d att[l] and the layer's regulariser value (warp per value, lane = k; the shuffle tree
  //      fixes the order) ----
  __threadfence();
  {
    constexpr int MAXV = (12 * IGMC_MAX_BASES + 1 + 7) / 8;   // values per warp at R = 12
    float pv[MAXV];
#pragma unroll
    for (int q = 0; q < MAXV; ++q) {   // one round of L2 latency for all of the warp's values
      const int pr = warp + 8 * q;
      const float* src = pr < R * NB ? reg_ws + RW_ATT + (size_t)l * 32 * 64 + pr : reg_ws + RW_REGP + l * 32;
      const int strd = pr < R * NB ? 64 : 1;
      pv[q] = (pr < R * NB + 1 && lane < in) ? __ldcg(src + (size_t)lane * strd) : 0.f;
    }
#pragma unroll
    for (int q = 0; q < MAXV; ++q) {
      const int pr = warp + 8 * q;
      if (pr < R * NB + 1) {   // (uniform over the warp)
        const float s = warp_sum_f(pv[q]);
        if (lane == 0) {
          if (pr < R * NB) grad[M.off_att[l] + pr] = s * grad_scale;
          else reg_ws[RW_REGL + l] = s;
        }
      }
    }
  }
  __syncthreads();
  if (!LOSS_INSIDE) {   // the caller computes the loss behind its own grid barrier (k_reduce_allreduce_adam)
    if (tid == 0) tick[l] = 0;   // re-arm
    return;
  }
  if (tid == 0) {
    tick[l] = 0;   // re-arm
    __threadfence();
    s_last = (atomicAdd(&tick[IGMC_MAX_LAYERS], 1) == L - 1);
  }
  __syncthreads();
  if (!s_last || warp != 0) return;
  // last layer to finish: the loss
  __threadfence();
  const float loss = loss_from_parts(reg_ws, sqerr, B, L, loss_scale, arr, lane);
  if (lane == 0) {
    if (loss_out) loss_out[0] = loss;
    tick[IGMC_MAX_LAYERS] = 0;
  }
}

__device__ __forceinline__ float loss_from_parts(const float* __restrict__ reg_ws, const float* __restrict__ sqerr, int B,
                                                 int L, float loss_scale, float arr, int lane) {
  float reg = lane < L ? __ldcg(reg_ws + RW_REGL + lane) : 0.f;
  float mse = 0.f;
  if (sqerr)
    for (int g = lane; g < B; g += 32) mse += __ldcg(sqerr + g);
  reg = warp_sum_f(reg);
  mse = warp_sum_f(mse);
  return mse * loss_scale + arr * reg;
}

__global__ void __launch_bounds__(256)
k_grad_reduce_raw(igmc_model_t M, const float* __restrict__ params, int B, int rows, int NA,
                  const float* __restrict__ gpart, const float* __restrict__ dhid, const float* __restrict__ feat,
                  const float* __restrict__ hid, const float* __restrict__ dpred, const float* __restrict__ sqerr,
                  float loss_scale, float arr, float grad_scale, float* __restrict__ grad, float* __restrict__ loss_out,
                  float* __restrict__ reg_ws) {
  reduce_raw_block<true>(M, params, B, rows, NA, gpart, dhid, feat, hid, dpred, sqerr, loss_scale, arr, grad_scale, grad,
                         loss_out, reg_ws);
}

// ---- torch.optim.Adam (torch 1.4 semantics) --------------------------------------------------------------------
// bias correction 1 - beta^step, in double from log beta (computed on the host)
__device__ __forceinline__ float adam_bias_correction(int64_t step, double log_beta) {
  return (float)(1.0 - exp((double)step * log_beta));
}

// one element: gradient g (already scaled), weight decay, moments m / v, parameter p
__device__ __forceinline__ void adam_update(float* __restrict__ params, float* __restrict__ m, float* __restrict__ v,
                                            int i, float g, float lr, float b1, float b2, float bc1, float bc2,
                                            float eps, float wd) {
  const float p = params[i];
  if (wd != 0.f) g = fmaf(wd, p, g);
  const float mi = b1 * m[i] + (1.f - b1) * g;
  const float vi = b2 * v[i] + (1.f - b2) * g * g;
  m[i] = mi;
  v[i] = vi;
  const float denom = sqrtf(vi) / sqrtf(bc2) + eps;
  params[i] = p - (lr / bc1) * (mi / denom);
}

// ---- system-scope flags for the peer exchange ----------------------------------------------------------------
__device__ __forceinline__ void st_release_sys(int* p, int v) {
  asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// gpu-scope twins for a single-rank exchange (world == 1: the flags only release this GPU's own blocks; a system-scope
// fence per block costs microseconds on the critical path of every step)
__device__ __forceinline__ void st_release_dev(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_acquire_dev(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float ld_relaxed_sys(const float* p) {
  float v;
  asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}

// ONE launch for  gradient assembly (+ARR)  ->  data-parallel all-reduce  ->  Adam:
//   phase 1  every block assembles its part of this rank's gradient into the rank's exchange buffer (parity t & 1)
//   phase 2  grid barrier; the last block publishes "step t ready" to every peer's flag array (st.release.sys over
//            NVLink); every block then waits until all ranks (itself included) have published step t
//   phase 3  one-shot all-reduce: each thread sums its elements over the ranks' buffers in rank order (peer loads
//            through NVLink / NVSwitch; identical order on every rank -> bit-identical parameters everywhere) and
//            applies the torch-Adam update
// Two parities are enough: a rank overwrites parity p in step t + 2 only after it has seen every peer's flag t + 1,
// which a peer raises after its step-t kernel (and thus its reads of parity p) has finished.
// Spinning inside the grid is safe only while every block is resident at once: igmc_reduce_update refuses a grid larger
// than the device holds (two blocks per SM: 264 on an H100; the 4-layer IGMC needs 230, 5 to 8 layers need 294 to 486
// and train through the separate kernels instead: igmc_reduce_update_grid tells the caller beforehand).
__global__ void __launch_bounds__(256, 2)   // <= 128 registers: two blocks per SM
k_reduce_allreduce_adam(igmc_model_t M, float* __restrict__ params, int B, int rows, int NA,
                        const float* __restrict__ gpart, const float* __restrict__ dhid, const float* __restrict__ feat,
                        const float* __restrict__ hid, const float* __restrict__ dpred, const float* __restrict__ sqerr,
                        float loss_scale, float arr, igmc_comm_t C, float* __restrict__ exp_avg,
                        float* __restrict__ exp_avg_sq, int64_t* __restrict__ step_count, float lr_val,
                        const float* __restrict__ lr_dev, float b1, float b2, double log_b1, double log_b2, float eps,
                        float wd, float grad_mul, float* __restrict__ loss_out, float* __restrict__ loss_acc,
                        float loss_weight, float* __restrict__ reg_ws, float* __restrict__ grad_copy,
                        float* __restrict__ loss_ring, int ring_mask, float* __restrict__ wprep) {
  const int tid = threadIdx.x;
  pdl_wait();   // launched as a programmatic dependent of the backward: its partial rows are complete from here on
  const int64_t t64 = C.state[0] + 1;               // the exchange step this launch executes
  const int t = (int)t64;
  const int64_t step_i = step_count[0] + 1;
  __shared__ float s_bc[2];
  if (tid >= 254)   // bias corrections (off the critical path: before the gradient assembly)
    s_bc[tid - 254] = adam_bias_correction(step_i, tid == 255 ? log_b2 : log_b1);
  float* gl = C.grad[C.rank] + (size_t)(t & 1) * C.stride;
  reduce_raw_block<false>(M, params, B, rows, NA, gpart, dhid, feat, hid, dpred, sqerr, loss_scale, arr, 1.0f, gl,
                          loss_out, reg_ws);
  int* tick = reinterpret_cast<int*>(C.state + 1);  // [0] phase-1 ticket, [1] phase-3 ticket
  __shared__ int s_pub;
  __syncthreads();
  const bool solo = C.world == 1;   // no peers: device-scope ordering is enough
  if (tid == 0) {
    if (solo) __threadfence(); else __threadfence_system();
    s_pub = (atomicAdd(&tick[0], 1) == (int)gridDim.x - 1);
    if (s_pub) tick[0] = 0;
  }
  __syncthreads();
  // the last block publishes "step t ready", one thread per destination rank (the stores travel in parallel)
  if (s_pub && tid < C.world) {
    if (solo) {
      __threadfence();
      st_release_dev(C.flag[0] + C.rank, t);
    } else {
      __threadfence_system();
      st_release_sys(C.flag[tid] + C.rank, t);   // includes the own flag
    }
  }
  // every block: one thread per source rank polls its arrival flag
  if (tid < C.world) {
    if (solo) while (ld_acquire_dev(C.flag[C.rank]) - t < 0) {}
    else while (ld_acquire_sys(C.flag[C.rank] + tid) - t < 0) {}
  }
  __syncthreads();
  const float lr = lr_dev ? *lr_dev : lr_val;
  const float bc1 = s_bc[0], bc2 = s_bc[1];
  const size_t poff = (size_t)(t & 1) * C.stride;
  for (int i = blockIdx.x * 256 + tid; i < M.param_count; i += gridDim.x * 256) {
    float gv[IGMC_MAX_RANKS];
#pragma unroll
    for (int r = 0; r < IGMC_MAX_RANKS; ++r) gv[r] = r < C.world ? ld_relaxed_sys(C.grad[r] + poff + i) : 0.f;
    float g = 0.f;
#pragma unroll
    for (int r = 0; r < IGMC_MAX_RANKS; ++r) g += gv[r];   // rank order; absent ranks add +0
    if (grad_copy) grad_copy[i] = g;
    adam_update(params, exp_avg, exp_avg_sq, i, g * grad_mul, lr, b1, b2, bc1, bc2, eps, wd);
  }
  if (blockIdx.x == 0 && tid < 32 && loss_out) {
    // the step's loss, off the critical path (every layer's regulariser value is complete behind the grid barrier)
    const float lv = loss_from_parts(reg_ws, sqerr, B, M.num_layers, loss_scale, arr, tid);
    if (tid == 0) {
      loss_out[0] = lv;
      if (loss_acc) loss_acc[0] += lv * loss_weight;
      // the step's result for the host: slot (step number mod ring size) of a mapped pinned-host ring, no copy launch
      if (loss_ring) loss_ring[(int)(step_i & (int64_t)ring_mask)] = lv;
    }
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    if (atomicAdd(&tick[1], 1) == (int)gridDim.x - 1) {
      tick[1] = 0;
      step_count[0] = step_i;
      C.state[0] = t64;
      if (wprep) {   // second grid barrier: every block's parameter slice is written - release the weight preparation
        __threadfence();
        *reinterpret_cast<volatile int*>(&tick[2]) = t;
      }
    }
    if (wprep)
      while (*reinterpret_cast<volatile int*>(&tick[2]) - t < 0) {}
    __threadfence();
  }
  if (!wprep) return;
  __syncthreads();
  // ---- phase 4: the prepared weights of the NEXT step's kernels (what igmc_prep_weights launches).  Rows of slab
  //      (0, 1) do not exist (layer 0 has no data gradient): active row a -> row a (a < 32) / a + 32 ----
  for (int a = blockIdx.x; a < (M.num_layers * 2 - 1) * 32; a += gridDim.x) {
    const int row = a < 32 ? a : a + 32;
    const int ld = row >> 5;
    wprep_write_row(M, params, wprep, ld >> 1, ld & 1, row & 31);
  }
}

// torch.optim.Adam step; the last block to finish increments the device-side step counter.
__global__ void k_adam(float* __restrict__ params, const float* __restrict__ grad, float* __restrict__ m,
                       float* __restrict__ v, int64_t* __restrict__ step_count, int* __restrict__ ticket, int n,
                       float lr_val, const float* __restrict__ lr_dev, float b1, float b2, double log_b1, double log_b2,
                       float eps, float wd, float grad_mul, const float* __restrict__ loss_in,
                       float* __restrict__ loss_acc, float loss_weight) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0 && loss_acc) loss_acc[0] += loss_in[0] * loss_weight;   // epoch loss bookkeeping (train_eval.py:176)
  const int64_t step_i = step_count[0] + 1;
  __shared__ float s_bc[2];
  if (threadIdx.x < 2)   // bias corrections, once per block
    s_bc[threadIdx.x] = adam_bias_correction(step_i, threadIdx.x ? log_b2 : log_b1);
  __syncthreads();
  if (i < n)
    adam_update(params, m, v, i, grad[i] * grad_mul, lr_dev ? *lr_dev : lr_val, b1, b2, s_bc[0], s_bc[1], eps, wd);
  __syncthreads();   // every thread of the block has read step_count
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(ticket, 1) == (int)gridDim.x - 1) {
      step_count[0] = step_i;
      *ticket = 0;
    }
  }
}

// grid of k_reduce_allreduce_adam: one block per layer input row of the gradient assembly plus the blocks of the
// readout parameters
int reduce_update_rows(const igmc_model_t* M) { return M->in_dim0 + (M->num_layers - 1) * HID; }
int reduce_update_blocks(const igmc_model_t* M) {
  return reduce_update_rows(M) + (M->param_count - M->conv_param_count + 255) / 256;
}

// blocks of k_reduce_allreduce_adam the current device runs at once (queried once per process)
int reduce_update_resident(int* resident) {
  static int cached = 0;
  if (!cached) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_reduce_allreduce_adam, 256, 0);
    if (e != cudaSuccess) return (int)e + 1000;
    cached = sms * per_sm;
  }
  *resident = cached;
  return 0;
}

}  // namespace

extern "C" int igmc_reduce_update_grid(const igmc_model_t* M, int* blocks, int* resident) {
  if (!M || !blocks) return -20;
  *blocks = reduce_update_blocks(M);
  return resident ? reduce_update_resident(resident) : 0;
}

extern "C" int igmc_grad_reduce(const igmc_model_t* M, const float* params, int B, int gpart_rows, const float* gpart,
                                int raw_rows, const float* dhid, const float* feat, const float* hid,
                                const float* dpred, const float* sqerr, float loss_scale, float arr, float grad_scale,
                                float* grad, float* loss_out, float* reg_ws, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int PB = (M->param_count + 255) / 256;
  if (raw_rows) {
    if (!reg_ws) return -18;
    if (M->num_relations > 12) return -16;
    const int NA = M->in_dim0 + (M->num_layers - 1) * HID;
    const int PBr = M->readout != 0 ? 0 : (M->param_count - M->conv_param_count + 255) / 256;
    k_grad_reduce_raw<<<NA + PBr, 256, 0, st>>>(*M, params, B, gpart_rows, NA, gpart, dhid, feat, hid, dpred, sqerr,
                                               loss_scale, arr, grad_scale, grad, loss_out, reg_ws);
    IGMC_CUDA_CHECK_LAUNCH();
    return 0;
  }
  int blocks = PB;
  size_t smem = 0;
  if (arr != 0.f) {
    if (!reg_ws) return -18;
    blocks += M->num_layers * M->num_relations;
    smem = (size_t)(((M->num_relations * M->num_bases + 3) & ~3) + (M->num_bases + 1) * HID * HID) * sizeof(float);
  }
  k_grad_reduce<<<blocks, 256, smem, st>>>(*M, params, B, gpart_rows, PB, gpart, dhid, feat, hid, dpred, sqerr,
                                          loss_scale, arr, grad_scale, grad, loss_out, reg_ws);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_adam_step(float* params, const float* grad, float* exp_avg, float* exp_avg_sq,
                              int64_t* step_count, int n, float lr, const float* lr_dev, float beta1, float beta2,
                              float eps, float weight_decay, float grad_mul, const float* loss_in, float* loss_acc,
                              float loss_weight, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  // step_count points at [int64 step | int32 ticket]: the word after the counter is the kernel's completion ticket
  int* ticket = reinterpret_cast<int*>(step_count + 1);
  k_adam<<<(n + 255) / 256, 256, 0, st>>>(params, grad, exp_avg, exp_avg_sq, step_count, ticket, n, lr, lr_dev, beta1,
                                          beta2, log((double)beta1), log((double)beta2), eps, weight_decay, grad_mul,
                                          loss_in, loss_acc, loss_weight);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_reduce_update(const igmc_model_t* M, float* params, int B, int gpart_rows, const float* gpart,
                                  const float* dhid, const float* feat, const float* hid, const float* dpred,
                                  const float* sqerr, float loss_scale, float arr, const igmc_comm_t* comm,
                                  float* exp_avg, float* exp_avg_sq, int64_t* step_count, float lr, const float* lr_dev,
                                  float beta1, float beta2, float eps, float weight_decay, float grad_mul,
                                  float* loss_out, float* loss_acc, float loss_weight, float* reg_ws, float* grad_copy,
                                  float* loss_ring, int ring_size, float* wprep, void* stream) {
  if (loss_ring && (ring_size < 1 || (ring_size & (ring_size - 1)))) return -20;   // power of two
  if (!comm || !reg_ws || comm->world < 1 || comm->world > IGMC_MAX_RANKS || comm->rank < 0 || comm->rank >= comm->world)
    return -20;
  if (comm->stride < M->param_count || !comm->state) return -20;
  for (int r = 0; r < comm->world; ++r)
    if (!comm->grad[r] || !comm->flag[r]) return -20;
  if (M->num_relations > 12) return -16;
  if (M->readout != 0) return -16;   // external readouts write their own gradient slice: use the separate kernels
  const int NA = reduce_update_rows(M), blocks = reduce_update_blocks(M);
  int resident = 0;
  const int rc = reduce_update_resident(&resident);
  if (rc) return rc;
  if (blocks > resident) return -21;   // the grid barrier would wait for blocks that cannot be scheduled
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(blocks);
  cfg.blockDim = dim3(256);
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;   // scheduled under the backward's tail (pdl_wait)
  at[0].val.programmaticStreamSerializationAllowed = 1;
  static int pdl = -1;
  if (pdl < 0) {
    const char* e = getenv("IGMC_PDL");
    pdl = e ? atoi(e) : 0;   // off by default (same reason as the backward, csrc/rgcn_rs.cu)
  }
  cfg.attrs = at;
  cfg.numAttrs = (pdl & 2) ? 1 : 0;   // IGMC_PDL bit 1 (bit 0: the backward, csrc/rgcn_rs.cu)
  cudaError_t e = cudaLaunchKernelEx(&cfg, k_reduce_allreduce_adam, *M, params, B, gpart_rows, NA, gpart, dhid, feat, hid,
                                     dpred, sqerr, loss_scale, arr, *comm, exp_avg, exp_avg_sq, step_count, lr, lr_dev,
                                     beta1, beta2, log((double)beta1), log((double)beta2), eps, weight_decay, grad_mul,
                                     loss_out, loss_acc, loss_weight, reg_ws, grad_copy, loss_ring, ring_size - 1, wprep);
  if (e != cudaSuccess) return (int)e + 1000;
  return 0;
}

// ---- exchange buffers: device memory every rank of the node maps (CUDA IPC); NCCL / gloo only carry the 64-byte
// handles once at start-up ----
extern "C" int igmc_comm_alloc(int64_t bytes, void** dev_ptr, unsigned char* handle64) {
  if (bytes <= 0 || !dev_ptr || !handle64) return -20;
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, (size_t)bytes);
  if (e != cudaSuccess) return (int)e + 1000;
  e = cudaMemset(p, 0, (size_t)bytes);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) { cudaFree(p); return (int)e + 1000; }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
  memcpy(handle64, &h, 64);
  *dev_ptr = p;
  return 0;
}
extern "C" int igmc_comm_open(const unsigned char* handle64, void** dev_ptr) {
  if (!handle64 || !dev_ptr) return -20;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) return (int)e + 1000;
  *dev_ptr = p;
  return 0;
}
extern "C" int igmc_comm_close(void* peer_ptr) {
  cudaError_t e = cudaIpcCloseMemHandle(peer_ptr);
  return e == cudaSuccess ? 0 : (int)e + 1000;
}
extern "C" int igmc_comm_free(void* dev_ptr) {
  cudaError_t e = cudaFree(dev_ptr);
  return e == cudaSuccess ? 0 : (int)e + 1000;
}

extern "C" int igmc_build_info(void) {
#ifdef IGMC_SM_ARCH
  return IGMC_SM_ARCH;
#else
  return 0;
#endif
}
