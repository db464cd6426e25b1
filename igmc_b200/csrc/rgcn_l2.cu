// L2 plan: the generic (basis-space) message passing of csrc/rgcn.cu for enclosing subgraphs of any size up to
// 65 535 nodes.  The other plans keep a whole subgraph's node features in shared memory, which caps the subgraph size;
// here they live in global memory (L2-resident at these sizes) and shared memory holds only a node tile, the layer's
// weights, att and the readout, so its size does not depend on n.
//
// One thread-block cluster of c CTAs (c = 1, 2, 4, 8) per subgraph; CTA `rank` owns the contiguous destination range
// own_range(n, c, rank).  Forward: layer l is written straight into S.states[:, 32l:32l+32] and gathered from there
// by layer l+1 (layer 0 gathers the one-hot of node_label).  Backward: two [node_cap][32] global buffers hold d pre_l
// and d h_{l-1} and swap roles every layer.  Rows written by another CTA of the cluster during the same launch are read
// with ld.global.cg (__ldcg) after a barrier.cluster arrive.release / wait.acquire, never through the non-coherent
// path.  Gradients: every CTA writes one partial row in parameter layout (gpart[B*c][conv_param_count], as plan 0)
// that igmc_grad_reduce sums in a fixed order.  No float atomics: results are run-to-run deterministic.
#include "lists.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int TM = 64;              // destination-node tile of the dense phases
constexpr int WS = 36;              // row stride of the transposed weights in backward
constexpr int HID = IGMC_HIDDEN;
constexpr int L1O = IGMC_LIN1_OUT;
constexpr int MAX_NODES = 65535;    // the neighbour field of an adjacency entry is 16 bits

__device__ __forceinline__ void cluster_sync_rel_acq() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

__device__ __forceinline__ void own_range(int n, int csize, int rank, int& v0, int& v1) {
  const int per = (n + csize - 1) / csize;
  v0 = min(n, rank * per);
  v1 = min(n, v0 + per);
}

// h_{l-1}[v][c]: one-hot of the node label for l = 0, else layer l-1 of concat_states (possibly another CTA's row)
struct PrevLayer {
  const uint8_t* label;
  const float* states;
  int l, in0, CW;
  __device__ __forceinline__ float operator()(int v, int c) const {
    if (l == 0) return (c == (int)label[v] && c < in0) ? 1.f : 0.f;
    return __ldcg(states + (size_t)v * CW + (l - 1) * HID + c);
  }
};

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
template <int NB, bool PR>
__global__ void __launch_bounds__(THREADS)
k_l2_forward(igmc_model_t M, const float* __restrict__ params, const uint8_t* __restrict__ node_label,
             const int32_t* __restrict__ node_ptr, const int32_t* __restrict__ edge_ptr, igmc_adj_t A, int csize,
             igmc_dropout_t D, int training, igmc_saved_t S, const float* __restrict__ y, float loss_scale,
             float* __restrict__ dpred, float* __restrict__ sqerr, int* err) {
  extern __shared__ __align__(16) float smem[];
  constexpr int ZS = (NB + 1) * HID + 4;   // tile row: [Z (NB*in) | h_{l-1} (in)]
  const int L = M.num_layers, R = M.num_relations, CW = HID * L, F = 2 * CW;
  float* Zs = smem;
  float* Wc = Zs + TM * ZS;                // [basis ; root] rows
  float* att_s = Wc + (NB + 1) * HID * HID;
  float* bias_s = att_s + a4(R * NB);
  float* feat_s = bias_s + HID;
  float* hid_s = feat_s + a4(F);
  __shared__ int s_t[2];

  const int g = blockIdx.x / csize, rank = blockIdx.x % csize;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nb = node_ptr[g], n = node_ptr[g + 1] - nb;
  const int eb = edge_ptr[g], m_half = (edge_ptr[g + 1] - eb) >> 1;
  if (n > MAX_NODES) {   // (the whole cluster returns: no CTA waits at a barrier)
    if (tid == 0) igmc_set_err(err, IGMC_ERR_NODE_ID16);
    return;
  }
  const EdgeKeep K = make_keep(D, training);
  const int in0 = M.in_dim0;
  int v0, v1;
  own_range(n, csize, rank, v0, v1);

  // target rows (models.py:205-206): every CTA of the cluster scans the labels, so all of them agree
  if (tid == 0) { s_t[0] = 0x7fffffff; s_t[1] = 0x7fffffff; }
  __syncthreads();
  for (int v = tid; v < n; v += THREADS) {
    const int lab = node_label[nb + v];
    if (lab == 0) atomicMin(&s_t[0], v);
    if (lab == 1) atomicMin(&s_t[1], v);
  }
  __syncthreads();
  const int tu = s_t[0], ti = s_t[1];
  if (M.readout == 0 && (tu >= n || ti >= n)) {
    if (tid == 0) igmc_set_err(err, IGMC_ERR_BAD_BATCH);
    return;
  }

  for (int l = 0; l < L; ++l) {
    const int in = l == 0 ? in0 : HID;
    const int K1 = NB * in;
    const PrevLayer hp{node_label + nb, S.states + (size_t)nb * CW, l, in0, CW};
    stage_layer<NB, THREADS>(M, params, l, in, Wc, att_s, bias_s, tid);
    __syncthreads();
    for (int t0 = v0; t0 < v1; t0 += TM) {
      const int tend = min(t0 + TM, v1);
      // ---- phase G: basis-space aggregate of the tile's nodes (warp per destination node) + their own rows ----
      for (int v = t0 + warp; v < tend; v += WARPS) {
        float z[NB];
        const int kept = gather_runs<NB, PR>(A.in_adj, A.in_eid, A.in_ptr[nb + v], A.in_ptr[nb + v + 1], K, false, eb,
                                             m_half, lane, [&](int u, int) { return hp(u, lane); }, att_s, z);
        const float id = 1.f / (float)max(kept, 1);   // kept in-degree: the same for every layer
        if (l == 0 && lane == 0) S.inv_deg[nb + v] = id;
        if (PR && l == 0)   // per-relation table for the backward (the runs above are means already)
          rel_inv_deg_row(A.in_adj, A.in_eid, A.in_ptr[nb + v], A.in_ptr[nb + v + 1], K, eb, m_half, lane, R,
                          S.rel_inv_deg + (size_t)(nb + v) * R);
        float* zr = Zs + (v - t0) * ZS;
#pragma unroll
        for (int b = 0; b < NB; ++b) {
          if (!PR) z[b] *= id;
          if (lane < in) zr[b * in + lane] = z[b];
          if (S.zsave) S.zsave[((size_t)l * S.node_cap + nb + v) * (NB * HID) + b * HID + lane] = z[b];
        }
        if (lane < in) zr[K1 + lane] = hp(v, lane);
      }
      __syncthreads();
      // ---- phase T: [Z | h] . [basis ; root] + bias, tanh (thread = 2 nodes x 4 channels) ----
      {
        const int r0 = (tid >> 3) * 2, c0 = (tid & 7) * 4;
        float a0[4], a1[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) { a0[c] = bias_s[c0 + c]; a1[c] = a0[c]; }
        const float* z0 = Zs + r0 * ZS;
        const float* z1 = z0 + ZS;
        for (int kk = 0; kk < K1 + in; ++kk) {
          const float x0 = z0[kk], x1 = z1[kk];
          const float4 w = *reinterpret_cast<const float4*>(Wc + kk * HID + c0);
          a0[0] = fmaf(x0, w.x, a0[0]); a0[1] = fmaf(x0, w.y, a0[1]); a0[2] = fmaf(x0, w.z, a0[2]); a0[3] = fmaf(x0, w.w, a0[3]);
          a1[0] = fmaf(x1, w.x, a1[0]); a1[1] = fmaf(x1, w.y, a1[1]); a1[2] = fmaf(x1, w.z, a1[2]); a1[3] = fmaf(x1, w.w, a1[3]);
        }
        const int va = t0 + r0, vb = va + 1;
        if (va < tend)
          *reinterpret_cast<float4*>(S.states + (size_t)(nb + va) * CW + l * HID + c0) =
              make_float4(tanhf(a0[0]), tanhf(a0[1]), tanhf(a0[2]), tanhf(a0[3]));
        if (vb < tend)
          *reinterpret_cast<float4*>(S.states + (size_t)(nb + vb) * CW + l * HID + c0) =
              make_float4(tanhf(a1[0]), tanhf(a1[1]), tanhf(a1[2]), tanhf(a1[3]));
      }
      __syncthreads();
    }
    cluster_sync_rel_acq();   // layer l of every CTA's nodes is in L2 before any CTA gathers it
  }

  if (M.readout != 0 || rank != 0) return;   // concat_states only (csrc/sortpool.cu takes over) / readout on rank 0
  // ---- readout: concat rows of the target user and item (models.py:205-207) ----
  for (int c = tid; c < F; c += THREADS) {
    const int node = c < CW ? tu : ti;
    const float v = __ldcg(S.states + (size_t)(nb + node) * CW + (c < CW ? c : c - CW));
    feat_s[c] = v;
    S.feat[(size_t)g * F + c] = v;
  }
  if (tid == 0) { S.target[2 * g] = nb + tu; S.target[2 * g + 1] = nb + ti; }
  __syncthreads();
  readout_lin1(M, params, feat_s, F, g, D, K.seed, training, hid_s, S, warp, WARPS, lane);
  __syncthreads();
  if (warp == 0)
    readout_lin2(M, params, hid_s, M.multiply_by, g, y, loss_scale, S.pred, sqerr,
                 dpred, lane);
}

// Per-edge score gradient of layer l at own node v (warp-wide; the EG mode of k_l2_backward).  dz[b] = dZ'[v,b,lane]
// (1/deg(v) applied; under PR not), so t = <h_{l-1}[j], sum_b att[r,b] dZ'[v,b]> is s/deg(v) (PR: s).  A first walk
// sums t over the segment (one per-lane partial, a warp sum per segment; PR: per type run, its mean kept in mean_r[r]),
// a second forms each entry's t again and writes t - mean (PR: (t - mean_r) / |N_r(v)|) into edge_grad[e]: stored
// when `first` (the top layer), added otherwise.  A segment of one entry gives exactly 0: both walks round the same
// products and sum them in the same order.
template <int NB, bool PR, class H>
__device__ __forceinline__ void edge_terms(const igmc_adj_t& A, const EdgeKeep& K, int nb, int v, int eb, int m_half,
                                           int lane, int R, const H& hp, const float* __restrict__ att_s,
                                           const float (&dz)[NB], const float* __restrict__ rinv, float* mean_r,
                                           bool first, float* __restrict__ edge_grad) {
  const int p0 = A.in_ptr[nb + v], p1 = A.in_ptr[nb + v + 1];
  auto term = [&](int nbr, int ty) {
    float p = 0.f;
#pragma unroll
    for (int b = 0; b < NB; ++b) p = fmaf(att_s[ty * NB + b], dz[b], p);
    return hp(nbr, lane) * p;
  };
  float part = 0.f;
  int cur = -1, cnt = 0;
  auto flush = [&]() {
    const float s = warp_sum_f(part);
    if (lane == 0) mean_r[cur] = s / (float)cnt;
  };
  const int kept = list_foreach(A.in_adj, A.in_eid, p0, p1, K, false, eb, m_half, lane, [&](int nbr, int ty) {
    if (PR && ty != cur) {
      if (cur >= 0) flush();
      part = 0.f;
      cur = ty;
      cnt = 0;
    }
    part += term(nbr, ty);
    ++cnt;
  });
  if (kept == 0) return;
  float mean = 0.f;
  if (PR) flush();
  else mean = warp_sum_f(part) / (float)kept;
  __syncwarp();
  list_foreach<true>(A.in_adj, A.in_eid, p0, p1, K, false, eb, m_half, lane, [&](int nbr, int ty, int e) {
    const float t = warp_sum_f(term(nbr, ty));
    const float d = PR ? (t - mean_r[ty]) * __ldcg(rinv + (size_t)v * R + ty) : t - mean;
    if (lane == 0) edge_grad[e] = first ? d : edge_grad[e] + d;
  });
  __syncwarp();   // mean_r is read before the warp's next node overwrites it
}

// ------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------
// EG (igmc_edge_grad): no parameter gradients.  Passes (0) and (1) and the dZ' tile run as in training; pass (3)'s
// in-list walk forms, per directed edge j->v of type r, s/|seg| - mean over the segment, s = <h_{l-1}[j] W_r, dpre[v]>
// (segment: v's in-list, or its type run under PR), and adds it into gpart[edge id] (there: edge_grad[edge_ptr[B]])
// layer by layer.  Every edge is an in-edge of one own node of one CTA: one writer per element, in a fixed order.
template <int NB, bool PR, bool EG = false>
__global__ void __launch_bounds__(THREADS)
k_l2_backward(igmc_model_t M, const float* __restrict__ params, const uint8_t* __restrict__ node_label,
              const int32_t* __restrict__ node_ptr, const int32_t* __restrict__ edge_ptr, igmc_adj_t A, int csize,
              igmc_dropout_t D, igmc_saved_t S, const float* __restrict__ dpred, float* __restrict__ gpart,
              float* __restrict__ dhid_out, float* __restrict__ dbuf, int* err) {
  extern __shared__ __align__(16) float smem[];
  constexpr int ZB = (NB + 2) * HID + 4;   // tile row: [Z or G or dZ' (NB*32) | d pre (32) | h_{l-1} (32)]
  constexpr int ZS2 = NB * HID + 4;        // row stride of basis^T in the d att pass
  constexpr int WT = (NB + 1) * HID * WS > HID * ZS2 ? (NB + 1) * HID * WS : HID * ZS2;
  const int L = M.num_layers, R = M.num_relations, CW = HID * L, F = 2 * CW;
  float* Zs = smem;
  float* Wt = Zs + TM * ZB;                // transposed [basis ; root] | basis as W2[j][b*32+k]
  float* att_s = Wt + WT;
  float* dfeat = att_s + a4(R * NB);
  float* dhid_s = dfeat + a4(F);
  double* datt_w = reinterpret_cast<double*>(dhid_s + L1O);   // [WARPS][R*NB], fp64: the sums over a large
                                                                 // subgraph cancel to a small fraction of their terms

  const int g = blockIdx.x / csize, rank = blockIdx.x % csize;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nb = node_ptr[g], n = node_ptr[g + 1] - nb;
  const int eb = edge_ptr[g], m_half = (edge_ptr[g + 1] - eb) >> 1;
  if (n > MAX_NODES) {
    if (tid == 0) igmc_set_err(err, IGMC_ERR_NODE_ID16);
    return;
  }
  const EdgeKeep K = make_keep(D, 1);
  const bool sym = A.symmetric != 0;
  const int32_t* optr = sym ? A.in_ptr : A.out_ptr;
  const uint32_t* oadj = sym ? A.in_adj : A.out_adj;
  const int32_t* oeid = sym ? A.in_eid : A.out_eid;
  const int in0 = M.in_dim0;
  const bool ext = M.readout != 0;   // d concat_states comes from an external readout (S.dstate)
  const int tu = ext ? -1 : S.target[2 * g] - nb, ti = ext ? -1 : S.target[2 * g + 1] - nb;
  float* gp = gpart + (size_t)blockIdx.x * M.conv_param_count;
  const float* invdeg = S.inv_deg + nb;
  const float* rinv = PR ? S.rel_inv_deg + (size_t)nb * R : nullptr;   // [n][R] 1/|N_r(v)| (PR mode)
  const float* states = S.states + (size_t)nb * CW;
  int v0, v1;
  own_range(n, csize, rank, v0, v1);

  // ---- readout backward: d hid, d feat (models.py:211-213) ----
  if (!ext) {
    readout_dhid(M, params, S, dpred, g, dhid_s, dhid_out, !EG && rank == 0, tid, THREADS);
    __syncthreads();
    for (int i = tid; i < F; i += THREADS) readout_dfeat_part(M, params, dhid_s, F, 1, i, dfeat);
  }
  __syncthreads();
  // d loss / d h_l[v][c] from the readout: S.dstate (external readout) and the two target rows
  auto seed = [&](int l, int v, int c) {
    float gval = 0.f;
    if (ext) gval = S.dstate[(size_t)(nb + v) * CW + l * HID + c];
    if (v == tu) gval += dfeat[l * HID + c];
    if (v == ti) gval += dfeat[CW + l * HID + c];
    return gval;
  };

  for (int l = L - 1; l >= 0; --l) {
    const int in = l == 0 ? in0 : HID;
    float* X = dbuf + (size_t)((L - 1 - l) & 1) * S.node_cap * HID + (size_t)nb * HID;   // d h_l -> d pre_l
    float* Y = dbuf + (size_t)((L - l) & 1) * S.node_cap * HID + (size_t)nb * HID;       // d h_{l-1}
    const PrevLayer hp{node_label + nb, states, l, in0, CW};
    // (0) d pre = d h * (1 - h^2) of the own nodes, in place
    for (int idx = tid; idx < (v1 - v0) * HID; idx += THREADS) {
      const int v = v0 + (idx >> 5), c = idx & 31;
      const float dh = l == L - 1 ? seed(l, v, c) : __ldcg(X + (size_t)v * HID + c);
      const float h = __ldcg(states + (size_t)v * CW + l * HID + c);
      X[(size_t)v * HID + c] = dh * (1.f - h * h);
    }
    for (int idx = tid; idx < R * NB; idx += THREADS) att_s[idx] = params[M.off_att[l] + idx];
    if (!EG)
      for (int idx = tid; idx < WARPS * R * NB; idx += THREADS) datt_w[idx] = 0.f;
    // d pre_l of every node of the subgraph is in L2 from here on.  (Y, written below, was last read by the previous
    // layer's pass (1) of the other CTAs, which they finished before arriving here.)
    cluster_sync_rel_acq();

    // (1) data gradient: d h_{l-1} = readout rows + [G | dpre] . [basis ; root]^T, G = out-list aggregate of dpre/deg
    if (l > 0) {
      stage_layer_t<NB, THREADS, WS>(M, params, l, Wt, tid);
      __syncthreads();
      for (int t0 = v0; t0 < v1; t0 += TM) {
        const int tend = min(t0 + TM, v1);
        for (int u = t0 + warp; u < tend; u += WARPS) {
          float gz[NB];
          gather_runs<NB>(oadj, oeid, optr[nb + u], optr[nb + u + 1], K, sym, eb, m_half, lane,
                          [&](int w, int ty) {
                            return __ldcg(X + (size_t)w * HID + lane) *
                                   (PR ? __ldcg(rinv + (size_t)w * R + ty) : __ldcg(invdeg + w));
                          }, att_s, gz);
          float* zr = Zs + (u - t0) * ZB;
#pragma unroll
          for (int b = 0; b < NB; ++b) zr[b * HID + lane] = gz[b];
          zr[NB * HID + lane] = __ldcg(X + (size_t)u * HID + lane);
        }
        __syncthreads();
        {
          const int r0 = (tid >> 3) * 2, c0 = (tid & 7) * 4;
          float a0[4] = {0.f, 0.f, 0.f, 0.f}, a1[4] = {0.f, 0.f, 0.f, 0.f};
          const float* z0 = Zs + r0 * ZB;
          const float* z1 = z0 + ZB;
          for (int kk = 0; kk < (NB + 1) * HID; ++kk) {
            const float x0 = z0[kk], x1 = z1[kk];
            const float4 w = *reinterpret_cast<const float4*>(Wt + kk * WS + c0);
            a0[0] = fmaf(x0, w.x, a0[0]); a0[1] = fmaf(x0, w.y, a0[1]); a0[2] = fmaf(x0, w.z, a0[2]); a0[3] = fmaf(x0, w.w, a0[3]);
            a1[0] = fmaf(x1, w.x, a1[0]); a1[1] = fmaf(x1, w.y, a1[1]); a1[2] = fmaf(x1, w.z, a1[2]); a1[3] = fmaf(x1, w.w, a1[3]);
          }
          const int va = t0 + r0, vb = va + 1;
          if (va < tend) {
            float4 t;
            t.x = seed(l - 1, va, c0) + a0[0]; t.y = seed(l - 1, va, c0 + 1) + a0[1];
            t.z = seed(l - 1, va, c0 + 2) + a0[2]; t.w = seed(l - 1, va, c0 + 3) + a0[3];
            *reinterpret_cast<float4*>(Y + (size_t)va * HID + c0) = t;
          }
          if (vb < tend) {
            float4 t;
            t.x = seed(l - 1, vb, c0) + a1[0]; t.y = seed(l - 1, vb, c0 + 1) + a1[1];
            t.z = seed(l - 1, vb, c0 + 2) + a1[2]; t.w = seed(l - 1, vb, c0 + 3) + a1[3];
            *reinterpret_cast<float4*>(Y + (size_t)vb * HID + c0) = t;
          }
        }
        __syncthreads();
      }
    }

    // (2) weight gradients d[basis ; root] = [Z | h_{l-1}]^T . dpre (K = own nodes), d bias = sum_v dpre, and
    // (3) d att[r,b] = sum_v sum_{in-runs of type r} < sum_run h_{l-1}[src,:] , dZ'[v,b,:] >,
    //     dZ'[v,b,k] = 1/deg(v) * sum_j dpre[v,j] basis[b][k][j]  - one pass over the own-node tiles
    {
      stage_basis_w2<NB, THREADS>(M, params, l, in, Wt, tid);
      const int kg = tid >> 3, c0 = (tid & 7) * 4;   // thread: row kg, channels c0..c0+3
      float acc[NB + 1][4];
      float accb[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int i = 0; i <= NB; ++i)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[i][c] = 0.f;
      double* dw = datt_w + warp * (R * NB);
      for (int t0 = v0; t0 < v1; t0 += TM) {
        const int tend = min(t0 + TM, v1), rows = tend - t0;
        if (!EG)
          for (int idx = tid; idx < rows * (NB * HID); idx += THREADS) {
            const int r = idx / (NB * HID), c = idx - r * (NB * HID);
            Zs[r * ZB + c] = S.zsave[((size_t)l * S.node_cap + nb + t0 + r) * (NB * HID) + c];
          }
        for (int idx = tid; idx < rows * HID; idx += THREADS) {
          const int r = idx >> 5, c = idx & 31;
          Zs[r * ZB + NB * HID + c] = __ldcg(X + (size_t)(t0 + r) * HID + c);
          if (!EG) Zs[r * ZB + (NB + 1) * HID + c] = hp(t0 + r, c);
        }
        __syncthreads();
        if (!EG && kg < in) {
          for (int r = 0; r < rows; ++r) {
            const float* zr = Zs + r * ZB;
            const float4 d = *reinterpret_cast<const float4*>(zr + NB * HID + c0);
#pragma unroll
            for (int i = 0; i < NB; ++i) {
              const float zv = zr[i * HID + kg];
              acc[i][0] = fmaf(zv, d.x, acc[i][0]); acc[i][1] = fmaf(zv, d.y, acc[i][1]);
              acc[i][2] = fmaf(zv, d.z, acc[i][2]); acc[i][3] = fmaf(zv, d.w, acc[i][3]);
            }
            const float hv = zr[(NB + 1) * HID + kg];
            acc[NB][0] = fmaf(hv, d.x, acc[NB][0]); acc[NB][1] = fmaf(hv, d.y, acc[NB][1]);
            acc[NB][2] = fmaf(hv, d.z, acc[NB][2]); acc[NB][3] = fmaf(hv, d.w, acc[NB][3]);
            if (kg == 0) { accb[0] += d.x; accb[1] += d.y; accb[2] += d.z; accb[3] += d.w; }
          }
        }
        __syncthreads();
        {
          // dZ' of the tile's nodes over the Z columns (thread: node r = tid/4, columns [cg*8NB, (cg+1)*8NB))
          const int r = tid >> 2, cg = tid & 3;
          constexpr int CPT = 8 * NB;
          float a[CPT];
#pragma unroll
          for (int c = 0; c < CPT; ++c) a[c] = 0.f;
          if (r < rows) {
            const float* dr = Zs + r * ZB + NB * HID;
            for (int j = 0; j < HID; ++j) {
              const float x = dr[j];
              const float* w = Wt + j * ZS2 + cg * CPT;
#pragma unroll
              for (int c = 0; c < CPT; c += 4) {
                const float4 w4 = *reinterpret_cast<const float4*>(w + c);
                a[c] = fmaf(x, w4.x, a[c]); a[c + 1] = fmaf(x, w4.y, a[c + 1]);
                a[c + 2] = fmaf(x, w4.z, a[c + 2]); a[c + 3] = fmaf(x, w4.w, a[c + 3]);
              }
            }
          }
          __syncthreads();   // every thread of the row has read d pre before the row's Z columns are overwritten
          if (r < rows) {
            const float id = PR ? 1.f : __ldcg(invdeg + t0 + r);   // (PR: 1/|N_r(v)| is applied per run below)
#pragma unroll
            for (int c = 0; c < CPT; ++c) Zs[r * ZB + cg * CPT + c] = a[c] * id;
          }
        }
        __syncthreads();
        for (int v = t0 + warp; v < tend; v += WARPS) {
          float dz[NB];
#pragma unroll
          for (int b = 0; b < NB; ++b) dz[b] = (lane < in) ? Zs[(v - t0) * ZB + b * HID + lane] : 0.f;
          if constexpr (EG) {
            edge_terms<NB, PR>(A, K, nb, v, eb, m_half, lane, R, hp, att_s, dz, rinv,
                               reinterpret_cast<float*>(datt_w) + warp * R, l == L - 1, gpart);
            continue;
          }
          float run = 0.f;
          int cur = -1, cnt = 0;
          auto flush = [&]() {
            const float rv = PR ? run * (1.f / (float)cnt) : run;
#pragma unroll
            for (int b = 0; b < NB; ++b) {
              const float p = warp_sum_f(rv * dz[b]);
              if (lane == 0) dw[cur * NB + b] += (double)p;
            }
          };
          list_foreach(A.in_adj, A.in_eid, A.in_ptr[nb + v], A.in_ptr[nb + v + 1], K, false, eb, m_half, lane,
                       [&](int nbr, int ty) {
                         if (ty != cur) {
                           if (cur >= 0) flush();
                           run = 0.f;
                           cur = ty;
                           cnt = 0;
                         }
                         run += hp(nbr, lane);
                         ++cnt;
                       });
          if (cur >= 0) flush();
        }
        __syncthreads();
      }
      if (!EG) {
        store_wgrad_rows<NB>(M, l, in, kg, c0, acc, accb, gp);
        __syncthreads();
        for (int idx = tid; idx < R * NB; idx += THREADS) {
          double s = 0.0;
          for (int w = 0; w < WARPS; ++w) s += datt_w[w * (R * NB) + idx];
          gp[M.off_att[l] + idx] = (float)s;
        }
      }
      __syncthreads();
    }
  }
}

size_t fwd_smem(int R, int NB, int L) {
  const size_t ZS = (NB + 1) * HID + 4, F = 2 * HID * L;
  const size_t fl = TM * ZS + (size_t)(NB + 1) * HID * HID + ((R * NB + 3) & ~3) + HID + ((F + 3) & ~3) + L1O;
  return fl * sizeof(float);
}
size_t bwd_smem(int R, int NB, int L) {
  const size_t ZB = (NB + 2) * HID + 4, ZS2 = NB * HID + 4, F = 2 * HID * L;
  size_t wt = (size_t)(NB + 1) * HID * WS;
  if (HID * ZS2 > wt) wt = HID * ZS2;
  const size_t fl = TM * ZB + wt + ((R * NB + 3) & ~3) + ((F + 3) & ~3) + L1O + 2 * (size_t)WARPS * R * NB;
  return fl * sizeof(float);
}

}  // namespace

// bytes of dynamic shared memory of the L2 plan's forward / backward kernel (independent of the subgraph size)
size_t l2_smem_bytes(const igmc_model_t* M, int backward) {
  return backward ? bwd_smem(M->num_relations, M->num_bases, M->num_layers)
                  : fwd_smem(M->num_relations, M->num_bases, M->num_layers);
}

int l2_forward(const igmc_model_t* M, const float* params, const uint8_t* node_label, const int32_t* node_ptr,
               const int32_t* edge_ptr, const igmc_adj_t* A, int B, int csize, const igmc_dropout_t* D, int training,
               const igmc_saved_t* S, const float* y, float loss_scale, float* dpred, float* sqerr, int* err,
               cudaStream_t st) {
  const size_t smem = l2_smem_bytes(M, 0);
  auto kern = M->num_bases == 4 ? (S->rel_inv_deg ? k_l2_forward<4, true> : k_l2_forward<4, false>)
                                : (S->rel_inv_deg ? k_l2_forward<2, true> : k_l2_forward<2, false>);
  return launch_cluster(kern, B * csize, THREADS, smem, csize, false, st, *M, params, node_label, node_ptr, edge_ptr, *A,
                        csize, *D, training, *S, y, loss_scale, dpred, sqerr, err);
}

int l2_backward(const igmc_model_t* M, const float* params, const uint8_t* node_label, const int32_t* node_ptr,
                const int32_t* edge_ptr, const igmc_adj_t* A, int B, int csize, const igmc_dropout_t* D,
                const igmc_saved_t* S, const float* dpred, float* gpart, float* dhid, float* dbuf, int* err,
                cudaStream_t st) {
  const size_t smem = l2_smem_bytes(M, 1);
  auto kern = M->num_bases == 4 ? (S->rel_inv_deg ? k_l2_backward<4, true> : k_l2_backward<4, false>)
                                : (S->rel_inv_deg ? k_l2_backward<2, true> : k_l2_backward<2, false>);
  return launch_cluster(kern, B * csize, THREADS, smem, csize, false, st, *M, params, node_label, node_ptr, edge_ptr, *A,
                        csize, *D, *S, dpred, gpart, dhid, dbuf, err);
}

int l2_edge_grad(const igmc_model_t* M, const float* params, const uint8_t* node_label, const int32_t* node_ptr,
                 const int32_t* edge_ptr, const igmc_adj_t* A, int B, int csize, const igmc_dropout_t* D,
                 const igmc_saved_t* S, const float* dpred, float* edge_grad, float* dbuf, int* err, cudaStream_t st) {
  const size_t smem = l2_smem_bytes(M, 1);
  auto kern = M->num_bases == 4
                  ? (S->rel_inv_deg ? k_l2_backward<4, true, true> : k_l2_backward<4, false, true>)
                  : (S->rel_inv_deg ? k_l2_backward<2, true, true> : k_l2_backward<2, false, true>);
  return launch_cluster(kern, B * csize, THREADS, smem, csize, false, st, *M, params, node_label, node_ptr, edge_ptr, *A,
                        csize, *D, *S, dpred, edge_grad, (float*)nullptr, dbuf, err);
}
