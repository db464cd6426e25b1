// Device pieces shared by the model kernels: csrc/rgcn.cu (plan 0), csrc/rgcn_l2.cu (L2 plan), csrc/rgcn_rs.cu
// (relation-space / cluster plans) and csrc/sortpool.cu (DGCNN_RS readout), and by the gradient kernels.
//   - the step's dropout draws: edge dropout (EdgeKeep) and the hidden dropout before lin2 (hidden_scale)
//   - a warp-wide walk over one node's (type, neighbour)-sorted list and the type-run segment reduce on it
//   - the readout head: lin1 / ReLU / dropout / save, lin2 / loss, their backward (d hid, d feat) and the lin1 / lin2
//     parameter gradients from the saved factors (csrc/optim.cu, csrc/influence.cu too)
//   - W_r from att and basis, the adjacent-rating regulariser's d W_r, and the per-step weight preparation (the wprep
//     slab layout) of the cluster plans (csrc/optim.cu too)
//   - the basis-space weight staging and weight-gradient row store of plan 0 and the L2 plan
// Each is one computation in one place: a kernel that calls it computes bit-for-bit what the others do.
#pragma once
#include "common.cuh"
#include "../../include/igmc_b200.h"

namespace {

// Activation tiles [n][32] live in shared memory with an XOR swizzle of the column by the row in 4-float groups:
// a row stays one contiguous 128 B line (lane = channel: conflict-free, float4 groups intact) and a fixed channel
// over 8 consecutive rows hits 8 different banks (column reads of the dense phases).
__device__ __forceinline__ int hix(int v, int c) { return (v << 5) + (c ^ ((v & 7) << 2)); }
__host__ __device__ __forceinline__ int a4(int x) { return (x + 3) & ~3; }

// ---- dropout draws of the step ---------------------------------------------------------------------------------
constexpr uint32_t DROPPED = 0xFFFFFFFFu;

// keep threshold p * 2^32 of a hash draw, 0xFFFFFFFF for p >= 1, which edge_keep reads as "drop everything".  Twin:
// igmc_b200/models.py::_keep_threshold.
__device__ __forceinline__ uint32_t keep_thresh(float p) {
  const double t = (double)p * 4294967296.0;
  return t >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)t;
}

struct EdgeKeep {
  bool active;
  const uint8_t* mask;
  uint64_t seed;
  uint32_t thresh;
  __device__ __forceinline__ bool keep(int e) const {
    return mask ? (mask[e] != 0) : edge_keep(seed, (uint32_t)e, thresh);
  }
};

__device__ __forceinline__ EdgeKeep make_keep(const igmc_dropout_t& D, int training) {
  EdgeKeep K;
  K.mask = D.edge_keep;
  K.seed = D.seed_dev ? *D.seed_dev : D.seed;
  K.active = training && (D.adj_dropout > 0.0f || D.edge_keep != nullptr);
  K.thresh = keep_thresh(D.adj_dropout);
  return K;
}

// F.dropout before lin2 (models.py:212): factor of unit o of graph g, 0 or 1/(1-p) in training, else 1.  The draw is
// an edge_keep draw of index g*128 + o on the step seed ^ 0x5bd1e995a5a5a5a5 (twin: models.py::hidden_keep_reference),
// so p >= 1 keeps no unit and every factor is 0; an injected D.hidden_keep mask stands for p = 0.5.
__device__ __forceinline__ float hidden_scale(const igmc_dropout_t& D, uint64_t seed, int training, int g, int o) {
  float scale = 1.f;
  if (training && (D.hidden_dropout > 0.f || D.hidden_keep)) {
    bool keep;
    if (D.hidden_keep) keep = D.hidden_keep[(size_t)g * IGMC_LIN1_OUT + o] != 0;
    else keep = edge_keep(seed ^ 0x5bd1e995a5a5a5a5ull, (uint32_t)(g * IGMC_LIN1_OUT + o), keep_thresh(D.hidden_dropout));
    const float p = D.hidden_keep ? 0.5f : D.hidden_dropout;
    scale = keep ? 1.f / (1.f - p) : 0.f;
  }
  return scale;
}

// ---- list walking ------------------------------------------------------------------------------------------------
// Walks list [p0,p1) of one node with the whole warp; body(nbr, type) is called warp-uniformly for
// every kept entry, in list order.  `mirror`: the entry describes edge nbr->x but the caller wants
// the reverse edge x->nbr of a symmetric batch, whose id is the mirror image inside the graph.
// WITH_ID: body(nbr, type, e) also gets that directed edge's id e (the id the keep draw reads).
template <bool WITH_ID = false, class Body>
__device__ __forceinline__ int list_foreach(const uint32_t* __restrict__ adj, const int32_t* __restrict__ eid,
                                            int p0, int p1, const EdgeKeep& K, bool mirror, int eb, int m_half,
                                            int lane, Body&& body) {
  int kept = 0;
  for (int c = p0; c < p1; c += 32) {
    const int p = c + lane;
    uint32_t ent = DROPPED;
    int e = -1;
    if (p < p1) {
      ent = adj[p];
      if (WITH_ID || K.active) {
        e = eid[p];
        if (mirror) { const int el = e - eb; e = eb + (el < m_half ? el + m_half : el - m_half); }
        if (K.active && !K.keep(e)) ent = DROPPED;
      }
    }
    const int cnt = min(32, p1 - c);
    for (int q = 0; q < cnt; ++q) {
      const uint32_t en = __shfl_sync(IGMC_FULL, ent, q);
      if (en == DROPPED) continue;
      ++kept;
      if constexpr (WITH_ID) body((int)(en & 0xffffu), (int)((en >> 16) & 0xffu), __shfl_sync(IGMC_FULL, e, q));
      else body((int)(en & 0xffffu), (int)((en >> 16) & 0xffu));
    }
  }
  return kept;
}

// Per-relation mean (igmc_saved_t.rel_inv_deg): out[r] = 1/max(kept entries of type r, 1) for r < R, for one node's
// list.  Lists are sorted by type, so every type is one run.  Warp-wide; returns the kept count.
__device__ __forceinline__ int rel_inv_deg_row(const uint32_t* __restrict__ adj, const int32_t* __restrict__ eid,
                                               int p0, int p1, const EdgeKeep& K, int eb, int m_half, int lane, int R,
                                               float* __restrict__ out) {
  for (int r = lane; r < R; r += 32) out[r] = 1.f;
  __syncwarp();
  int cur = -1, cnt = 0;
  const int kept = list_foreach(adj, eid, p0, p1, K, false, eb, m_half, lane, [&](int, int ty) {
    if (ty != cur) {
      if (cur >= 0 && lane == 0) out[cur] = 1.f / (float)cnt;
      cur = ty;
      cnt = 0;
    }
    ++cnt;
  });
  if (cur >= 0 && lane == 0) out[cur] = 1.f / (float)cnt;
  return kept;
}

// Type-run segment reduce over kept list entries: acc[b] = sum_runs att[type][b] * sum_run feat(nbr, type);
// MEAN: every run divided by its length (the forward's mean per relation, igmc_saved_t.rel_inv_deg)
template <int NB, bool MEAN = false, class Feat>
__device__ __forceinline__ int gather_runs(const uint32_t* __restrict__ adj, const int32_t* __restrict__ eid, int p0,
                                           int p1, const EdgeKeep& K, bool mirror, int eb, int m_half, int lane,
                                           Feat&& feat, const float* __restrict__ att_s, float (&acc)[NB]) {
  float run = 0.f;
  int cur = -1, cnt = 0;
#pragma unroll
  for (int b = 0; b < NB; ++b) acc[b] = 0.f;
  auto flush = [&]() {
    float rv = run;
    if (MEAN) rv *= 1.f / (float)cnt;
#pragma unroll
    for (int b = 0; b < NB; ++b) acc[b] = fmaf(att_s[cur * NB + b], rv, acc[b]);
  };
  const int kept = list_foreach(adj, eid, p0, p1, K, mirror, eb, m_half, lane, [&](int nbr, int ty) {
    if (ty != cur) {
      if (cur >= 0) flush();
      run = 0.f;
      cur = ty;
      cnt = 0;
    }
    run += feat(nbr, ty);
    ++cnt;
  });
  if (cur >= 0) flush();
  return kept;
}

// ---- readout head (models.py:205-215 IGMC, 160-165 DGCNN_RS) ---------------------------------------------------
// `M` is the model or readout descriptor (igmc_model_t / igmc_sortpool_t: the lin1 / lin2 offsets into params), `S`
// the saved tensors of the step (igmc_saved_t / igmc_sortpool_saved_t: hid, hid_gscale).
// relu(lin1 pre-activation) of unit o of graph g, hidden dropout, and what the backward needs: hid = h * scale (to
// shared hid_s and S.hid), S.hid_gscale = d hid / d pre-activation
template <class Saved>
__device__ __forceinline__ void readout_hidden(float pre, int g, int o, const igmc_dropout_t& D, uint64_t seed,
                                               int training, float* hid_s, const Saved& S) {
  const float h = fmaxf(pre, 0.f);
  const float scale = hidden_scale(D, seed, training, g, o);
  hid_s[o] = h * scale;
  S.hid[(size_t)g * IGMC_LIN1_OUT + o] = h * scale;
  S.hid_gscale[(size_t)g * IGMC_LIN1_OUT + o] = h > 0.f ? scale : 0.f;
}

// lin1 of the readout row feat_s[F] (shared memory) of graph g, then readout_hidden.  Eight outputs per warp and pass
// (16 warps x 8 = all 128 in one pass of L2 latency); each output is one per-lane fmaf chain over i = lane, lane + 32,
// .. and one warp_sum_f.
template <class Model, class Saved>
__device__ __forceinline__ void readout_lin1(const Model& M, const float* params, const float* feat_s, int F, int g,
                                             const igmc_dropout_t& D, uint64_t seed, int training, float* hid_s,
                                             const Saved& S, int warp, int nwarps, int lane) {
  constexpr int OW = 8;
  const float* W1 = params + M.off_lin1_w;
  for (int ob = warp * OW; ob < IGMC_LIN1_OUT; ob += nwarps * OW) {
    float s4[OW];
#pragma unroll
    for (int u = 0; u < OW; ++u) s4[u] = 0.f;
    const float bias_o = lane < OW ? __ldg(params + M.off_lin1_b + ob + lane) : 0.f;   // independent of the dot products
#pragma unroll 4   // 32 independent L2 loads in flight per lane (the loop is latency bound)
    for (int i = lane; i < F; i += 32) {
      const float f = feat_s[i];
#pragma unroll
      for (int u = 0; u < OW; ++u) s4[u] = fmaf(__ldg(W1 + (size_t)(ob + u) * F + i), f, s4[u]);
    }
#pragma unroll
    for (int u = 0; u < OW; ++u) s4[u] = warp_sum_f(s4[u]);
#pragma unroll
    for (int u = 0; u < OW; ++u)
      if (lane == u) readout_hidden(s4[u] + bias_o, g, ob + u, D, seed, training, hid_s, S);
  }
}

// lin2 and the loss of graph g on one warp: pred = (lin2 . hid + b) * multiply_by; with targets y also the squared
// error and dpred = d (loss_scale * mse) / d lin2 output
template <class Model>
__device__ __forceinline__ void readout_lin2(const Model& M, const float* params, const float* hid_s,
                                             float multiply_by, int g, const float* y, float loss_scale, float* pred,
                                             float* sqerr, float* dpred, int lane) {
  float s = 0.f;
  const float b2 = __ldg(params + M.off_lin2_b), yg = y ? __ldg(y + g) : 0.f;   // issued with the weight loads
  for (int o = lane; o < IGMC_LIN1_OUT; o += 32) s = fmaf(params[M.off_lin2_w + o], hid_s[o], s);
  s = warp_sum_f(s);
  if (lane == 0) {
    const float out = (s + b2) * multiply_by;
    pred[g] = out;
    if (y) {
      const float diff = out - yg;
      if (sqerr) sqerr[g] = diff * diff;
      if (dpred) dpred[g] = 2.f * diff * loss_scale * multiply_by;
    }
  }
}

// d hid = dpred[g] * lin2.weight * S.hid_gscale[g] (lin2, dropout and ReLU backward) -> dhid_s [128] and, if
// `store`, row g of dhid_out
template <class Model, class Saved>
__device__ __forceinline__ void readout_dhid(const Model& M, const float* params, const Saved& S, const float* dpred,
                                             int g, float* dhid_s, float* dhid_out, bool store, int tid, int NT) {
  const float dp = dpred[g];
  for (int o = tid; o < IGMC_LIN1_OUT; o += NT) {
    const float d = dp * params[M.off_lin2_w + o] * S.hid_gscale[(size_t)g * IGMC_LIN1_OUT + o];
    dhid_s[o] = d;
    if (store) dhid_out[(size_t)g * IGMC_LIN1_OUT + o] = d;
  }
}

// One partial of d feat[i] = sum_o lin1.weight[o][i] d hid[o]: slot t = part * F + i (nothing for t >= parts * F)
// sums every parts-th o from `part` on, in order, into out[t].  With parts = 1 and out = d feat this is the whole
// sum of column i; with more slices the caller adds the parts of a column in slice order after a barrier.
template <class Model>
__device__ __forceinline__ void readout_dfeat_part(const Model& M, const float* params, const float* dhid_s, int F,
                                                   int parts, int t, float* out) {
  const float* W1 = params + M.off_lin1_w;
  const int i = t % F, part = t / F;
  if (part < parts) {
    float s = 0.f;
#pragma unroll 32   // independent L2 loads in flight (latency bound)
    for (int o = part; o < IGMC_LIN1_OUT; o += parts) s = fmaf(__ldg(W1 + (size_t)o * F + i), dhid_s[o], s);
    out[part * F + i] = s;
  }
}

// The gradient of readout parameter p as a function of the saved factors of the graphs (dhid [g][128], feat [g][F],
// hid [g][128], dpred [g]):
//   lin1.weight[o][i]: sum_g dhid[g][o] feat[g][i]      lin1.bias[o]: sum_g dhid[g][o]
//   lin2.weight[o]:    sum_g dpred[g] hid[g][o]         lin2.bias:    sum_g dpred[g]
// Calls prod(x, sx, y, sy) for a product term x[g * sx] * y[g * sy] or one(x, sx) for a single factor x[g * sx], and
// returns false (calling neither) when p is not a lin1 / lin2 entry.
template <class Model, class Prod, class One>
__device__ __forceinline__ bool readout_param_grad(const Model& M, int p, int F, const float* dhid, const float* feat,
                                                   const float* hid, const float* dpred, Prod&& prod, One&& one) {
  constexpr int L1O = IGMC_LIN1_OUT;
  if (p >= M.off_lin1_w && p < M.off_lin1_w + L1O * F) {
    const int q = p - M.off_lin1_w, o = q / F, i = q - o * F;
    prod(dhid + o, L1O, feat + i, F);
  } else if (p >= M.off_lin1_b && p < M.off_lin1_b + L1O) {
    one(dhid + (p - M.off_lin1_b), L1O);
  } else if (p >= M.off_lin2_w && p < M.off_lin2_w + L1O) {
    prod(dpred, 1, hid + (p - M.off_lin2_w), L1O);
  } else if (p == M.off_lin2_b) {
    one(dpred, 1);
  } else {
    return false;
  }
  return true;
}

// readout_param_grad summed over the batch's B graphs in ascending g into s (which starts at +0)
template <class Model>
__device__ __forceinline__ bool readout_param_grad_sum(const Model& M, int p, int F, int B, const float* dhid,
                                                       const float* feat, const float* hid, const float* dpred,
                                                       float& s) {
  return readout_param_grad(
      M, p, F, dhid, feat, hid, dpred,
      [&](const float* x, int sx, const float* y, int sy) {
#pragma unroll 25   // 50 independent L2 loads in flight (latency bound)
        for (int g = 0; g < B; ++g) s = fmaf(x[(size_t)g * sx], y[(size_t)g * sy], s);
      },
      [&](const float* x, int sx) {
#pragma unroll 25
        for (int g = 0; g < B; ++g) s += x[(size_t)g * sx];
      });
}

// ---- per-step weight preparation (csrc/rgcn_rs.cu consumes it) ---------------------------------------------------
// W_r[k][j] = sum_b att[r,b] basis[b][k][j] as one fmaf chain over ascending b; att(b) and basis(b) read the two
// factors of term b, all of them before the first fmaf
template <class Att, class Basis>
__device__ __forceinline__ float compose_w(int NB, Att&& att, Basis&& basis) {
  float av[IGMC_MAX_BASES], bv[IGMC_MAX_BASES];
#pragma unroll
  for (int b = 0; b < IGMC_MAX_BASES; ++b) {
    av[b] = b < NB ? att(b) : 0.f;
    bv[b] = b < NB ? basis(b) : 0.f;
  }
  float w = 0.f;
#pragma unroll
  for (int b = 0; b < IGMC_MAX_BASES; ++b)
    if (b < NB) w = fmaf(av[b], bv[b], w);
  return w;
}

// d reg / d W_r at one entry of the adjacent-rating regulariser reg = sum_{r<R-1} ||W_{r+1} - W_r||^2:
// 2 (W_r - W_{r-1}) [r > 0] - 2 (W_{r+1} - W_r) [r < R-1], W(r) giving the entry of W_r.  `pair` (optional) receives
// (W_{r+1} - W_r)^2, the entry's share of the pair (r, r+1) (+0 for r = R-1).
template <class W>
__device__ __forceinline__ float arr_dw(W&& w, int R, int r, float* pair) {
  const float w0 = w(r);
  float dw = 0.f, d = 0.f;
  if (r > 0) dw += 2.f * (w0 - w(r - 1));
  if (r < R - 1) {
    d = w(r + 1) - w0;
    dw -= 2.f * d;
  }
  if (pair) *pair = d * d;
  return dw;
}

// Prepared weights: slab(l, dir) = Bn[n][KS] (n = output channel, 32 rows):
//   dir 0 (forward, B of  [AGG | h] . [W_r ; root]):   Bn[n][r*inp+k] = W_r[k][n],  Bn[n][K1p+k] = root[k][n]
//   dir 1 (backward, B of [Q | dpre] . [W_r^T ; root^T], layers >= 1):  Bn[k][r*32+j] = W_r[k][j],  Bn[k][R*32+j] = root[k][j]
// Rows are n-major / K-contiguous so the mma B fragments load conflict-free.  Row geometry of a layer whose input width
// rounded up to 4 is inp: the relation columns [0, K1 = R * inp) padded to K1p, the root columns [K1p, K1p + inp) padded
// to inpp, 4 more floats: KS per row.
__host__ __device__ __forceinline__ int a8(int x) { return (x + 7) & ~7; }
struct WprepRow {
  int K1, K1p, inpp;
  __host__ __device__ __forceinline__ int KS() const { return K1p + inpp + 4; }
};
__host__ __device__ __forceinline__ WprepRow wprep_row(int R, int inp) {
  WprepRow g;
  g.K1 = R * inp;
  g.K1p = a8(g.K1);
  g.inpp = a8(inp);
  return g;
}
// floats of one slab: 32 rows of a 32-wide layer's KS = (R + 1) * 32 + 4 (the widest; a slab of layer 0 uses a
// prefix).  Twin: igmc_b200/models.py IGMC._wprep_buf.
__host__ __device__ __forceinline__ size_t wprep_slab(int R) {
  return (size_t)IGMC_HIDDEN * ((size_t)(R + 1) * IGMC_HIDDEN + 4);
}

// Row n of slab (l, dir) from the parameters, a 256-thread block striding over its KS floats.  params are read through
// L2 (__ldcg): the update kernel calls this on parameters other blocks of the same launch have just written.
__device__ __forceinline__ void wprep_write_row(const igmc_model_t& M, const float* params, float* wprep, int l,
                                                int dir, int n) {
  constexpr int HID = IGMC_HIDDEN;
  const int R = M.num_relations, NB = M.num_bases;
  const int in = l == 0 ? M.in_dim0 : HID, inp = a4(in);
  const WprepRow G = wprep_row(R, inp);
  const float* bs = params + M.off_basis[l];
  const float* at = params + M.off_att[l];
  const float* rt = params + M.off_root[l];
  float* out = wprep + ((size_t)l * 2 + dir) * wprep_slab(R) + (size_t)n * G.KS();
  for (int kk = threadIdx.x; kk < G.KS(); kk += 256) {
    float w = 0.f;
    if (kk < G.K1) {
      const int r = kk / inp, q = kk - r * inp;
      if (q < in) {
        // dir 0: W_r[k=q][n] ; dir 1: W_r[k=n][j=q]
        const int k = dir == 0 ? q : n, j = dir == 0 ? n : q;
        w = compose_w(NB, [&](int b) { return __ldcg(at + r * NB + b); },
                      [&](int b) { return __ldcg(bs + (b * in + k) * HID + j); });
      }
    } else if (kk >= G.K1p && kk < G.K1p + inp) {
      const int q = kk - G.K1p;
      if (q < in) w = dir == 0 ? __ldcg(rt + q * HID + n) : __ldcg(rt + n * HID + q);
    }
    out[kk] = w;
  }
}

// ---- basis-space weights of plan 0 and the L2 plan --------------------------------------------------------------
// layer l's [basis ; root] rows -> Wc [(NB+1)*in][32] (rows NB*in.. are root), att -> att_s, bias -> bias_s
template <int NB, int NT>
__device__ __forceinline__ void stage_layer(const igmc_model_t& M, const float* __restrict__ params, int l, int in,
                                            float* Wc, float* att_s, float* bias_s, int tid) {
  constexpr int HID = IGMC_HIDDEN;
  const float* bs = params + M.off_basis[l];
  const float* rt = params + M.off_root[l];
  const int K1 = NB * in;
  for (int idx = tid; idx < K1 * HID; idx += NT) Wc[idx] = bs[idx];
  for (int idx = tid; idx < in * HID; idx += NT) Wc[K1 * HID + idx] = rt[idx];
  for (int idx = tid; idx < M.num_relations * NB; idx += NT) att_s[idx] = params[M.off_att[l] + idx];
  if (tid < HID) bias_s[tid] = params[M.off_bias[l] + tid];
}

// the transposed [basis ; root] of a 32-wide layer l for the data gradient: basis[b][k][j] -> Wt[b*32+j][k],
// root[k][j] -> Wt[NB*32+j][k], row stride WS
template <int NB, int NT, int WS>
__device__ __forceinline__ void stage_layer_t(const igmc_model_t& M, const float* __restrict__ params, int l,
                                              float* Wt, int tid) {
  constexpr int HID = IGMC_HIDDEN;
  const float* bs = params + M.off_basis[l];
  const float* rt = params + M.off_root[l];
  for (int idx = tid; idx < NB * HID * HID; idx += NT) {
    const int j = idx & 31, k = (idx >> 5) & 31, b = idx >> 10;
    Wt[(b * HID + j) * WS + k] = bs[idx];
  }
  for (int idx = tid; idx < HID * HID; idx += NT) {
    const int j = idx & 31, k = idx >> 5;
    Wt[(NB * HID + j) * WS + k] = rt[idx];
  }
}

// basis of layer l (input width in) for the d att pass: basis[b][k][j] -> W2[j][b*32+k], row stride NB*32+4
template <int NB, int NT>
__device__ __forceinline__ void stage_basis_w2(const igmc_model_t& M, const float* __restrict__ params, int l, int in,
                                               float* W2, int tid) {
  constexpr int HID = IGMC_HIDDEN, ZS = NB * HID + 4;
  const float* bs = params + M.off_basis[l];
  for (int idx = tid; idx < NB * in * HID; idx += NT) {
    const int j = idx & 31, k = (idx >> 5) % in, b = (idx >> 5) / in;
    W2[j * ZS + b * HID + k] = bs[idx];
  }
}

// weight-gradient rows of layer l in parameter layout: thread (kg, c0) holds d basis[i][kg][c0..c0+3] (acc[i], i < NB),
// d root[kg][c0..] (acc[NB]) and, for kg = 0, d bias[c0..] (accb)
template <int NB>
__device__ __forceinline__ void store_wgrad_rows(const igmc_model_t& M, int l, int in, int kg, int c0,
                                                 const float (&acc)[NB + 1][4], const float (&accb)[4],
                                                 float* __restrict__ gp) {
  constexpr int HID = IGMC_HIDDEN;
  if (kg >= in) return;
#pragma unroll
  for (int i = 0; i < NB; ++i)
    *reinterpret_cast<float4*>(gp + M.off_basis[l] + (i * in + kg) * HID + c0) =
        make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
  *reinterpret_cast<float4*>(gp + M.off_root[l] + kg * HID + c0) =
      make_float4(acc[NB][0], acc[NB][1], acc[NB][2], acc[NB][3]);
  if (kg == 0) *reinterpret_cast<float4*>(gp + M.off_bias[l] + c0) = make_float4(accb[0], accb[1], accb[2], accb[3]);
}

}  // namespace
