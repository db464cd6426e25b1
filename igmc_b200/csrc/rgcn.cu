// Fused relational message passing for IGMC: one CTA per enclosing subgraph, node features resident
// in shared memory for all layers.
//
// Replaces (reference call sites): dropout_adj (models.py:193-198), 4x tanh(RGCNConv) (models.py:200-202;
// PyG 1.4.2 RGCNConv = index_select of a per-edge [in,out] weight + bmm + scatter_mean, SURVEY.md A.1),
// concat + target-row readout + lin1/relu/dropout/lin2 (models.py:203-215) and their autograd.
//
// Formulation (never materialises the per-edge weight):  with W_r = sum_b att[r,b] basis[b],
//   Z[v,b,:]  = 1/deg(v) * sum_{(u->v, type r) kept} att[r,b] * h[u,:]          (segment reduce, run per type)
//   pre[v,:]  = [Z[v] | h[v]] . [basis ; root] + bias ,   h'[v] = tanh(pre[v])     (dense K=(NB+1)*in GEMM tile)
// deg(v) = number of kept incoming edges of ANY type (aggr='mean').  PR = true (PyG >= 1.6 RGCNConv, selected by
// igmc_saved_t.rel_inv_deg) moves the mean inside the relation sum: each type run is divided by its own length, and
// the backward weighs an out-list entry u->d of type r by 1/|N_r(d)| instead of 1/deg(d).  Backward is the same pair of
// passes on the transposed lists with [basis ; root]^T, plus K=n weight-gradient GEMM tiles.
// All reductions have a fixed order: results are run-to-run deterministic.
#include "lists.cuh"

namespace {

constexpr int MP_THREADS = 256;
constexpr int MP_WARPS = MP_THREADS / 32;
constexpr int TM = 64;   // node tile of the dense phases
constexpr int WS = 36;   // row stride of transposed weights in backward
constexpr int HID = IGMC_HIDDEN;
constexpr int L1O = IGMC_LIN1_OUT;

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
template <int NB, bool PR>
__global__ void __launch_bounds__(MP_THREADS)
k_forward(igmc_model_t M, const float* __restrict__ params, const uint8_t* __restrict__ node_label,
          const int32_t* __restrict__ node_ptr, const int32_t* __restrict__ edge_ptr, igmc_adj_t A, int n_cap,
          igmc_dropout_t D, int training, igmc_saved_t S, const float* __restrict__ y, float loss_scale,
          float* __restrict__ dpred, float* __restrict__ sqerr, int* err) {
  extern __shared__ __align__(16) float smem[];
  constexpr int ZS = NB * HID + 4;
  const int L = M.num_layers, R = M.num_relations, CW = HID * L, F = 2 * CW;
  float* HA = smem;
  float* HB = HA + (size_t)n_cap * HID;
  float* Zs = HB + (size_t)n_cap * HID;
  float* Wc = Zs + TM * ZS;
  float* att_s = Wc + (NB + 1) * HID * HID;
  float* bias_s = att_s + a4(R * NB);
  float* invdeg = bias_s + HID;
  float* feat_s = invdeg + a4(n_cap);
  float* hid_s = feat_s + a4(F);
  __shared__ int s_t[2];

  const int g = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nb = node_ptr[g], n = node_ptr[g + 1] - nb;
  const int eb = edge_ptr[g], m_half = (edge_ptr[g + 1] - eb) >> 1;
  if (n > n_cap) {
    if (tid == 0) igmc_set_err(err, IGMC_ERR_SMEM_NODES);
    return;
  }
  const EdgeKeep K = make_keep(D, training);
  const int in0 = M.in_dim0;

  // h_0 = one-hot(node label) (util_functions.py:286) padded to 32 columns; target rows
  if (tid == 0) { s_t[0] = 0x7fffffff; s_t[1] = 0x7fffffff; }
  __syncthreads();
  for (int idx = tid; idx < n * HID; idx += MP_THREADS) {
    const int v = idx >> 5, c = idx & 31;
    const int lab = node_label[nb + v];
    HA[hix(v, c)] = (c == lab && c < in0) ? 1.f : 0.f;
    if (c == 0 && lab == 0) atomicMin(&s_t[0], v);   // users = x[:,0]==1 (models.py:205)
    if (c == 0 && lab == 1) atomicMin(&s_t[1], v);   // items = x[:,1]==1 (models.py:206)
  }
  // kept in-degree (same for every layer: dropout_adj is applied once, models.py:193); per relation too in PR mode
  for (int v = warp; v < n; v += MP_WARPS) {
    const int p0 = A.in_ptr[nb + v], p1 = A.in_ptr[nb + v + 1];
    int kept = p1 - p0;
    if (PR)
      kept = rel_inv_deg_row(A.in_adj, A.in_eid, p0, p1, K, eb, m_half, lane, R, S.rel_inv_deg + (size_t)(nb + v) * R);
    else if (K.active)
      kept = list_foreach(A.in_adj, A.in_eid, p0, p1, K, false, eb, m_half, lane, [](int, int) {});
    if (lane == 0) {
      const float id = 1.f / (float)max(kept, 1);
      invdeg[v] = id;
      S.inv_deg[nb + v] = id;
    }
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
    stage_layer<NB, MP_THREADS>(M, params, l, in, Wc, att_s, bias_s, tid);   // [basis ; root] rows, att, bias
    __syncthreads();
    for (int t0 = 0; t0 < n; t0 += TM) {
      const int tend = min(t0 + TM, n);
      // ---- phase G: basis-space aggregate of the tile's nodes (warp per destination node) ----
      for (int v = t0 + warp; v < tend; v += MP_WARPS) {
        float z[NB];
        gather_runs<NB, PR>(A.in_adj, A.in_eid, A.in_ptr[nb + v], A.in_ptr[nb + v + 1], K, false, eb, m_half, lane,
                            [&](int u, int) { return HA[hix(u, lane)]; }, att_s, z);
        const float id = invdeg[v];
#pragma unroll
        for (int b = 0; b < NB; ++b) {
          if (!PR) z[b] *= id;   // (PR: every relation's run is already a mean)
          if (lane < in) Zs[(v - t0) * ZS + b * in + lane] = z[b];
          if (S.zsave)
            S.zsave[((size_t)l * S.node_cap + nb + v) * (NB * HID) + b * HID + lane] = z[b];
        }
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
        for (int kk = 0; kk < K1; ++kk) {
          const float x0 = z0[kk], x1 = z1[kk];
          const float4 w = *reinterpret_cast<const float4*>(Wc + kk * HID + c0);
          a0[0] = fmaf(x0, w.x, a0[0]); a0[1] = fmaf(x0, w.y, a0[1]); a0[2] = fmaf(x0, w.z, a0[2]); a0[3] = fmaf(x0, w.w, a0[3]);
          a1[0] = fmaf(x1, w.x, a1[0]); a1[1] = fmaf(x1, w.y, a1[1]); a1[2] = fmaf(x1, w.z, a1[2]); a1[3] = fmaf(x1, w.w, a1[3]);
        }
        const int v0 = t0 + r0, v1 = v0 + 1;
        const int q0 = min(v0, n - 1), q1 = min(v1, n - 1);
        for (int k = 0; k < in; ++k) {
          const float x0 = HA[hix(q0, k)], x1 = HA[hix(q1, k)];
          const float4 w = *reinterpret_cast<const float4*>(Wc + (K1 + k) * HID + c0);
          a0[0] = fmaf(x0, w.x, a0[0]); a0[1] = fmaf(x0, w.y, a0[1]); a0[2] = fmaf(x0, w.z, a0[2]); a0[3] = fmaf(x0, w.w, a0[3]);
          a1[0] = fmaf(x1, w.x, a1[0]); a1[1] = fmaf(x1, w.y, a1[1]); a1[2] = fmaf(x1, w.z, a1[2]); a1[3] = fmaf(x1, w.w, a1[3]);
        }
        if (v0 < tend) {
          float4 o = make_float4(tanhf(a0[0]), tanhf(a0[1]), tanhf(a0[2]), tanhf(a0[3]));
          *reinterpret_cast<float4*>(HB + hix(v0, c0)) = o;
          *reinterpret_cast<float4*>(S.states + (size_t)(nb + v0) * CW + l * HID + c0) = o;
        }
        if (v1 < tend) {
          float4 o = make_float4(tanhf(a1[0]), tanhf(a1[1]), tanhf(a1[2]), tanhf(a1[3]));
          *reinterpret_cast<float4*>(HB + hix(v1, c0)) = o;
          *reinterpret_cast<float4*>(S.states + (size_t)(nb + v1) * CW + l * HID + c0) = o;
        }
      }
      __syncthreads();
    }
    float* t = HA; HA = HB; HB = t;
  }

  if (M.readout != 0) return;   // concat_states only: an external readout (csrc/sortpool.cu) takes over
  // ---- readout: concat rows of the target user and item (models.py:205-207) ----
  for (int c = tid; c < F; c += MP_THREADS) {
    const int node = c < CW ? tu : ti;
    const float v = S.states[(size_t)(nb + node) * CW + (c < CW ? c : c - CW)];
    feat_s[c] = v;
    S.feat[(size_t)g * F + c] = v;
  }
  if (tid == 0) { S.target[2 * g] = nb + tu; S.target[2 * g + 1] = nb + ti; }
  __syncthreads();
  readout_lin1(M, params, feat_s, F, g, D, K.seed, training, hid_s, S, warp, MP_WARPS, lane);
  __syncthreads();
  if (warp == 0)
    readout_lin2(M, params, hid_s, M.multiply_by, g, y, loss_scale, S.pred, sqerr,
                 dpred, lane);
}

// ------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------
template <int NB, bool PR>
__global__ void __launch_bounds__(MP_THREADS)
k_backward(igmc_model_t M, const float* __restrict__ params, const uint8_t* __restrict__ node_label,
           const int32_t* __restrict__ node_ptr, const int32_t* __restrict__ edge_ptr, igmc_adj_t A, int n_cap,
           igmc_dropout_t D, igmc_saved_t S, const float* __restrict__ dpred, float* __restrict__ gpart,
           float* __restrict__ dhid_out, int* err) {
  extern __shared__ __align__(16) float smem[];
  constexpr int ZS = NB * HID + 4;
  const int L = M.num_layers, R = M.num_relations, CW = HID * L, F = 2 * CW;
  float* GA = smem;                               // d h_l  -> d pre_l
  float* GB = GA + (size_t)n_cap * HID;           // d h_{l-1}
  float* HP = GB + (size_t)n_cap * HID;           // h_{l-1}
  float* Zs = HP + (size_t)n_cap * HID;           // tile scratch [TM][ZS]
  float* Wt = Zs + TM * ZS;                       // transposed weights, (NB+1)*32 rows x WS  |  W2 [32][ZS]
  float* att_s = Wt + (NB + 1) * HID * WS;
  float* invdeg = att_s + a4(R * NB);
  float* dfeat = invdeg + a4(n_cap);
  float* dhid_s = dfeat + a4(F);
  float* datt_w = dhid_s + L1O;                   // [MP_WARPS][R*NB]

  const int g = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nb = node_ptr[g], n = node_ptr[g + 1] - nb;
  const int eb = edge_ptr[g], m_half = (edge_ptr[g + 1] - eb) >> 1;
  if (n > n_cap) {
    if (tid == 0) igmc_set_err(err, IGMC_ERR_SMEM_NODES);
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
  float* gp = gpart + (size_t)g * M.conv_param_count;

  // ---- readout backward: d hid, d feat (models.py:211-213) ----
  if (!ext)
    readout_dhid(M, params, S, dpred, g, dhid_s, dhid_out, true, tid, MP_THREADS);
  for (int v = tid; v < n; v += MP_THREADS) invdeg[v] = S.inv_deg[nb + v];
  __syncthreads();
  if (!ext)
    for (int i = tid; i < F; i += MP_THREADS) readout_dfeat_part(M, params, dhid_s, F, 1, i, dfeat);
  __syncthreads();
  // d h_L : only the two target rows receive gradient from the IGMC readout
  for (int idx = tid; idx < n * HID; idx += MP_THREADS) {
    const int v = idx >> 5, c = idx & 31;
    float gval = 0.f;
    if (ext) gval = S.dstate[(size_t)(nb + v) * CW + (L - 1) * HID + c];
    if (v == tu) gval += dfeat[(L - 1) * HID + c];
    if (v == ti) gval += dfeat[CW + (L - 1) * HID + c];
    GA[hix(v, c)] = gval;
  }
  __syncthreads();

  for (int l = L - 1; l >= 0; --l) {
    const int in = l == 0 ? in0 : HID;
    // (0) d pre = d h * (1 - h^2) ; h_{l-1} ; d h_{l-1} seeded with the readout rows
    for (int idx = tid; idx < n * HID; idx += MP_THREADS) {
      const int v = idx >> 5, c = idx & 31;
      const float h = S.states[(size_t)(nb + v) * CW + l * HID + c];
      GA[hix(v, c)] *= (1.f - h * h);
      float hp, gval = 0.f;
      if (l > 0) {
        hp = S.states[(size_t)(nb + v) * CW + (l - 1) * HID + c];
        if (ext) gval = S.dstate[(size_t)(nb + v) * CW + (l - 1) * HID + c];
        if (v == tu) gval += dfeat[(l - 1) * HID + c];
        if (v == ti) gval += dfeat[CW + (l - 1) * HID + c];
      } else {
        hp = (c == (int)node_label[nb + v] && c < in0) ? 1.f : 0.f;
      }
      HP[hix(v, c)] = hp;
      GB[hix(v, c)] = gval;
    }
    for (int idx = tid; idx < R * NB; idx += MP_THREADS) att_s[idx] = params[M.off_att[l] + idx];
    for (int idx = tid; idx < MP_WARPS * R * NB; idx += MP_THREADS) datt_w[idx] = 0.f;
    __syncthreads();

    // (1) data gradient: d h_{l-1} += [G | dpre] . [basis ; root]^T , G = out-list aggregate of dpre/deg
    if (l > 0) {
      stage_layer_t<NB, MP_THREADS, WS>(M, params, l, Wt, tid);
      __syncthreads();
      const float* rinv = PR ? S.rel_inv_deg + (size_t)nb * R : nullptr;   // 1/|N_r(d)| of the destination d
      for (int t0 = 0; t0 < n; t0 += TM) {
        const int tend = min(t0 + TM, n);
        for (int u = t0 + warp; u < tend; u += MP_WARPS) {
          float gz[NB];
          gather_runs<NB>(oadj, oeid, optr[nb + u], optr[nb + u + 1], K, sym, eb, m_half, lane,
                          [&](int d, int ty) {
                            return GA[hix(d, lane)] * (PR ? __ldg(rinv + d * R + ty) : invdeg[d]);
                          }, att_s, gz);
#pragma unroll
          for (int b = 0; b < NB; ++b) Zs[(u - t0) * ZS + b * HID + lane] = gz[b];
        }
        __syncthreads();
        {
          const int r0 = (tid >> 3) * 2, c0 = (tid & 7) * 4;
          float a0[4] = {0.f, 0.f, 0.f, 0.f}, a1[4] = {0.f, 0.f, 0.f, 0.f};
          const float* z0 = Zs + r0 * ZS;
          const float* z1 = z0 + ZS;
          for (int kk = 0; kk < NB * HID; ++kk) {
            const float x0 = z0[kk], x1 = z1[kk];
            const float4 w = *reinterpret_cast<const float4*>(Wt + kk * WS + c0);
            a0[0] = fmaf(x0, w.x, a0[0]); a0[1] = fmaf(x0, w.y, a0[1]); a0[2] = fmaf(x0, w.z, a0[2]); a0[3] = fmaf(x0, w.w, a0[3]);
            a1[0] = fmaf(x1, w.x, a1[0]); a1[1] = fmaf(x1, w.y, a1[1]); a1[2] = fmaf(x1, w.z, a1[2]); a1[3] = fmaf(x1, w.w, a1[3]);
          }
          const int v0 = t0 + r0, v1 = v0 + 1;
          const int q0 = min(v0, n - 1), q1 = min(v1, n - 1);
          for (int j = 0; j < HID; ++j) {
            const float x0 = GA[hix(q0, j)], x1 = GA[hix(q1, j)];
            const float4 w = *reinterpret_cast<const float4*>(Wt + (NB * HID + j) * WS + c0);
            a0[0] = fmaf(x0, w.x, a0[0]); a0[1] = fmaf(x0, w.y, a0[1]); a0[2] = fmaf(x0, w.z, a0[2]); a0[3] = fmaf(x0, w.w, a0[3]);
            a1[0] = fmaf(x1, w.x, a1[0]); a1[1] = fmaf(x1, w.y, a1[1]); a1[2] = fmaf(x1, w.z, a1[2]); a1[3] = fmaf(x1, w.w, a1[3]);
          }
          if (v0 < tend) {
            float4* o = reinterpret_cast<float4*>(GB + hix(v0, c0));
            float4 t = *o; t.x += a0[0]; t.y += a0[1]; t.z += a0[2]; t.w += a0[3]; *o = t;
          }
          if (v1 < tend) {
            float4* o = reinterpret_cast<float4*>(GB + hix(v1, c0));
            float4 t = *o; t.x += a1[0]; t.y += a1[1]; t.z += a1[2]; t.w += a1[3]; *o = t;
          }
        }
        __syncthreads();
      }
    }

    // (2) weight gradients: d[basis ; root] = [Z | h_{l-1}]^T . dpre  (K = n), d bias = sum_v dpre
    {
      const int kg = tid >> 3, c0 = (tid & 7) * 4;   // thread: rows {kg + 32 i}, channels c0..c0+3
      float acc[NB + 1][4];
      float accb[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int i = 0; i <= NB; ++i)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[i][c] = 0.f;
      for (int t0 = 0; t0 < n; t0 += TM) {
        const int tend = min(t0 + TM, n), rows = tend - t0;
        for (int idx = tid; idx < rows * (NB * HID); idx += MP_THREADS) {
          const int r = idx / (NB * HID), c = idx - r * (NB * HID);
          Zs[r * ZS + c] = S.zsave[((size_t)l * S.node_cap + nb + t0 + r) * (NB * HID) + c];
        }
        __syncthreads();
        if (kg < in) {
          for (int r = 0; r < rows; ++r) {
            const float4 d = *reinterpret_cast<const float4*>(GA + hix(t0 + r, c0));
#pragma unroll
            for (int i = 0; i < NB; ++i) {
              const float zv = Zs[r * ZS + i * HID + kg];
              acc[i][0] = fmaf(zv, d.x, acc[i][0]); acc[i][1] = fmaf(zv, d.y, acc[i][1]);
              acc[i][2] = fmaf(zv, d.z, acc[i][2]); acc[i][3] = fmaf(zv, d.w, acc[i][3]);
            }
            const float hv = HP[hix(t0 + r, kg)];
            acc[NB][0] = fmaf(hv, d.x, acc[NB][0]); acc[NB][1] = fmaf(hv, d.y, acc[NB][1]);
            acc[NB][2] = fmaf(hv, d.z, acc[NB][2]); acc[NB][3] = fmaf(hv, d.w, acc[NB][3]);
            if (kg == 0) { accb[0] += d.x; accb[1] += d.y; accb[2] += d.z; accb[3] += d.w; }
          }
        }
        __syncthreads();
      }
      store_wgrad_rows<NB>(M, l, in, kg, c0, acc, accb, gp);
    }

    // (3) d att[r,b] = sum_v sum_{in-runs of type r} < sum_run h_{l-1}[src,:] , dZ'[v,b,:] >,
    //     dZ'[v,b,k] = 1/deg(v) * sum_j dpre[v,j] basis[b][k][j]
    {
      stage_basis_w2<NB, MP_THREADS>(M, params, l, in, Wt, tid);
      __syncthreads();
      for (int t0 = 0; t0 < n; t0 += TM) {
        const int tend = min(t0 + TM, n);
        {
          // thread: node r = tid/4, columns [cg*8NB, (cg+1)*8NB) ; only k < in are meaningful
          const int r = tid >> 2, cg = tid & 3;
          constexpr int CPT = 8 * NB;
          float a[CPT];
#pragma unroll
          for (int c = 0; c < CPT; ++c) a[c] = 0.f;
          const int v = t0 + r;
          if (v < tend) {
            for (int j = 0; j < HID; ++j) {
              const float x = GA[hix(v, j)];
              const float* w = Wt + j * ZS + cg * CPT;
#pragma unroll
              for (int c = 0; c < CPT; c += 4) {
                const float4 w4 = *reinterpret_cast<const float4*>(w + c);
                a[c] = fmaf(x, w4.x, a[c]); a[c + 1] = fmaf(x, w4.y, a[c + 1]);
                a[c + 2] = fmaf(x, w4.z, a[c + 2]); a[c + 3] = fmaf(x, w4.w, a[c + 3]);
              }
            }
            const float id = PR ? 1.f : invdeg[v];   // (PR: the 1/|N_r(v)| factor is applied per run below)
#pragma unroll
            for (int c = 0; c < CPT; ++c) Zs[r * ZS + cg * CPT + c] = a[c] * id;
          }
        }
        __syncthreads();
        for (int v = t0 + warp; v < tend; v += MP_WARPS) {
          float dz[NB];
#pragma unroll
          for (int b = 0; b < NB; ++b) dz[b] = (lane < in) ? Zs[(v - t0) * ZS + b * HID + lane] : 0.f;
          float run = 0.f;
          int cur = -1, cnt = 0;
          float* dw = datt_w + warp * (R * NB);
          auto flush = [&]() {
            const float rv = PR ? run * (1.f / (float)cnt) : run;
#pragma unroll
            for (int b = 0; b < NB; ++b) {
              const float p = warp_sum_f(rv * dz[b]);
              if (lane == 0) dw[cur * NB + b] += p;
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
                         run += HP[hix(nbr, lane)];
                         ++cnt;
                       });
          if (cur >= 0) flush();
        }
        __syncthreads();
      }
      for (int idx = tid; idx < R * NB; idx += MP_THREADS) {
        float s = 0.f;
        for (int w = 0; w < MP_WARPS; ++w) s += datt_w[w * (R * NB) + idx];
        gp[M.off_att[l] + idx] = s;
      }
    }
    __syncthreads();
    float* t = GA; GA = GB; GB = t;
  }
}

size_t fwd_smem_bytes(int n_cap, int R, int NB, int L) {
  const size_t ZS = NB * HID + 4, F = 2 * HID * L;
  size_t fl = 2 * (size_t)n_cap * HID + TM * ZS + (size_t)(NB + 1) * HID * HID + ((R * NB + 3) & ~3) + HID +
              ((n_cap + 3) & ~3) + ((F + 3) & ~3) + L1O;
  return fl * sizeof(float);
}
size_t bwd_smem_bytes(int n_cap, int R, int NB, int L) {
  const size_t ZS = NB * HID + 4, F = 2 * HID * L;
  size_t wt = (size_t)(NB + 1) * HID * WS;
  if (HID * ZS > wt) wt = HID * ZS;
  size_t fl = 3 * (size_t)n_cap * HID + TM * ZS + wt + ((R * NB + 3) & ~3) + ((n_cap + 3) & ~3) +
              ((F + 3) & ~3) + L1O + (size_t)MP_WARPS * R * NB;
  return fl * sizeof(float);
}

int check_model(const igmc_model_t* M) {
  if (M->num_layers < 1 || M->num_layers > IGMC_MAX_LAYERS) return -10;
  if (M->num_bases != 2 && M->num_bases != 4) return -11;
  if (M->num_relations < 1 || M->num_relations > 256) return -12;
  if (M->in_dim0 < 1 || M->in_dim0 > HID) return -13;
  if (M->readout != 0 && M->readout != 1) return -19;
  return 0;
}

}  // namespace

// relation-space / cluster kernels (csrc/rgcn_rs.cu)
int rs_supported(const igmc_model_t* M);
int rs_plan(const igmc_model_t* M, int n_cap, int cluster, int backward, int* threads, size_t* smem, int* lcap, int* chunk);
int rs_forward(const igmc_model_t* M, const float* params, const uint8_t* node_label, const int32_t* node_ptr,
               const int32_t* edge_ptr, const igmc_adj_t* A, int B, int n_cap, const igmc_dropout_t* D, int training,
               const igmc_saved_t* S, const float* y, float loss_scale, float* dpred, float* sqerr, int cluster,
               const igmc_stage_t* stage, int* err, cudaStream_t st);
int rs_backward(const igmc_model_t* M, const float* params, const uint8_t* node_label, const int32_t* node_ptr,
                const int32_t* edge_ptr, const igmc_adj_t* A, int B, int n_cap, const igmc_dropout_t* D,
                const igmc_saved_t* S, const float* dpred, float* gpart, float* dhid, int cluster,
                const igmc_stage_t* stage, int* err, cudaStream_t st);
int rs_stage_plan(const igmc_model_t* M, int n_cap, int cluster, int backward, igmc_stage_t* img);
int rs_stage_lists(const igmc_model_t* M, const int32_t* node_ptr, const int32_t* edge_ptr, const igmc_adj_t* A, int B,
                   int n_cap, const igmc_dropout_t* D, int training, const igmc_stage_t* fwd, const igmc_stage_t* bwd,
                   cudaStream_t st);

int rs_prep_weights(const igmc_model_t* M, const float* params, float* wprep, cudaStream_t st);
int rs_train(const igmc_model_t* M, const float* params, const uint8_t* node_label, const int32_t* node_ptr,
             const int32_t* edge_ptr, const igmc_adj_t* A, int B, int n_cap, const igmc_dropout_t* D,
             const igmc_saved_t* S, const float* y, float loss_scale, float* dpred, float* sqerr, float* gpart,
             float* dhid, int cluster, const igmc_stage_t* stage_f, const igmc_stage_t* stage_b, int* err,
             cudaStream_t st);
int rs_gate_wait(int* gate, int target, int timeout_us, cudaStream_t st);

// L2 plan (csrc/rgcn_l2.cu)
size_t l2_smem_bytes(const igmc_model_t* M, int backward);
int l2_forward(const igmc_model_t* M, const float* params, const uint8_t* node_label, const int32_t* node_ptr,
               const int32_t* edge_ptr, const igmc_adj_t* A, int B, int csize, const igmc_dropout_t* D, int training,
               const igmc_saved_t* S, const float* y, float loss_scale, float* dpred, float* sqerr, int* err,
               cudaStream_t st);
int l2_backward(const igmc_model_t* M, const float* params, const uint8_t* node_label, const int32_t* node_ptr,
                const int32_t* edge_ptr, const igmc_adj_t* A, int B, int csize, const igmc_dropout_t* D,
                const igmc_saved_t* S, const float* dpred, float* gpart, float* dhid, float* dbuf, int* err,
                cudaStream_t st);
int l2_edge_grad(const igmc_model_t* M, const float* params, const uint8_t* node_label, const int32_t* node_ptr,
                 const int32_t* edge_ptr, const igmc_adj_t* A, int B, int csize, const igmc_dropout_t* D,
                 const igmc_saved_t* S, const float* dpred, float* edge_grad, float* dbuf, int* err, cudaStream_t st);

// CTAs per subgraph of an IGMC_PLAN_L2(c) value, 0 for every other plan value
static int l2_csize(int cluster) {
  const int c = cluster - IGMC_PLAN_L2_BASE;
  return (c == 1 || c == 2 || c == 4 || c == 8) ? c : 0;
}

extern "C" int igmc_gate_wait(int32_t* gate, int target, int timeout_us, void* stream) {
  if (!gate || target < 0 || timeout_us < 0) return -21;
  return rs_gate_wait(gate, target, timeout_us, (cudaStream_t)stream);
}

extern "C" int igmc_prep_weights(const igmc_model_t* M, const float* params, float* wprep, void* stream) {
  int rc = check_model(M);
  if (rc) return rc;
  if (!rs_supported(M)) return -16;
  return rs_prep_weights(M, params, wprep, (cudaStream_t)stream);
}

extern "C" int igmc_model_plan(const igmc_model_t* M, int n_cap, int cluster, int backward) {
  int rc = check_model(M);
  if (rc) return rc;
  if (l2_csize(cluster)) {
    if (n_cap > IGMC_L2_MAX_NODES) return -3;
    const size_t b = l2_smem_bytes(M, backward);
    return b > 227 * 1024 ? -3 : (int)b;
  }
  if (cluster == 0) {
    const size_t b = backward ? bwd_smem_bytes(n_cap, M->num_relations, M->num_bases, M->num_layers)
                              : fwd_smem_bytes(n_cap, M->num_relations, M->num_bases, M->num_layers);
    return b > 227 * 1024 ? -3 : (int)b;
  }
  if (cluster < 1 || cluster > 4) return -15;
  if (!rs_supported(M)) return -16;
  int threads, lcap, chunk;
  size_t smem;
  rc = rs_plan(M, n_cap, cluster, backward, &threads, &smem, &lcap, &chunk);
  return rc ? rc : (int)smem;
}

extern "C" int igmc_stage_plan(const igmc_model_t* M, int n_cap, int cluster, int backward, igmc_stage_t* img) {
  int rc = check_model(M);
  if (rc) return rc;
  if (cluster < 1 || cluster > 4) return -15;
  if (!rs_supported(M)) return -16;
  return rs_stage_plan(M, n_cap, cluster, backward, img);
}

extern "C" int igmc_stage_lists(const igmc_model_t* M, const int32_t* node_ptr, const int32_t* edge_ptr,
                                const igmc_adj_t* A, int B, int n_cap, const igmc_dropout_t* D, int training,
                                const igmc_stage_t* fwd, const igmc_stage_t* bwd, int* err, void* stream) {
  (void)err;
  if (B <= 0) return 0;
  int rc = check_model(M);
  if (rc) return rc;
  if (!rs_supported(M)) return -16;
  return rs_stage_lists(M, node_ptr, edge_ptr, A, B, n_cap, D, training, fwd, bwd, (cudaStream_t)stream);
}

extern "C" int igmc_raw_grad_count(const igmc_model_t* M) {
  int rc = check_model(M);
  if (rc) return rc;
  return igmc_raw_count(M->num_relations, M->in_dim0, M->num_layers);
}

extern "C" int igmc_forward(const igmc_model_t* M, const float* params, const uint8_t* node_label,
                            const int32_t* node_ptr, const int32_t* edge_ptr, const igmc_adj_t* A, int B, int n_cap,
                            const igmc_dropout_t* D, int training, const igmc_saved_t* S, const float* y,
                            float loss_scale, float* dpred, float* sqerr, int cluster, const igmc_stage_t* stage,
                            int* err, void* stream) {
  if (B <= 0) return 0;
  int rc = check_model(M);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (const int c = l2_csize(cluster)) {   // (before the relation-space branch: every cluster > 0 goes there)
    if (n_cap > IGMC_L2_MAX_NODES) return -3;
    return l2_forward(M, params, node_label, node_ptr, edge_ptr, A, B, c, D, training, S, y, loss_scale, dpred, sqerr,
                      err, st);
  }
  if (cluster > 0) {
    if (!rs_supported(M)) return -16;
    if (!S->wprep) return -17;
    return rs_forward(M, params, node_label, node_ptr, edge_ptr, A, B, n_cap, D, training, S, y, loss_scale, dpred,
                      sqerr, cluster, stage, err, st);
  }
  const size_t smem = fwd_smem_bytes(n_cap, M->num_relations, M->num_bases, M->num_layers);
  if (smem > 227 * 1024) return -3;
  auto kern = M->num_bases == 4 ? (S->rel_inv_deg ? k_forward<4, true> : k_forward<4, false>)
                                : (S->rel_inv_deg ? k_forward<2, true> : k_forward<2, false>);
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  kern<<<B, MP_THREADS, smem, st>>>(*M, params, node_label, node_ptr, edge_ptr, *A, n_cap, *D, training, *S, y,
                                    loss_scale, dpred, sqerr, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_forward_backward(const igmc_model_t* M, const float* params, const uint8_t* node_label,
                                     const int32_t* node_ptr, const int32_t* edge_ptr, const igmc_adj_t* A, int B,
                                     int n_cap, const igmc_dropout_t* D, const igmc_saved_t* S, const float* y,
                                     float loss_scale, float* dpred, float* sqerr, float* gpart, float* dhid,
                                     int cluster, const igmc_stage_t* stage_fwd, const igmc_stage_t* stage_bwd,
                                     int* err, void* stream) {
  if (B <= 0) return 0;
  int rc = check_model(M);
  if (rc) return rc;
  if (cluster <= 0 || l2_csize(cluster) || M->readout != 0 || !rs_supported(M)) return -16;   // relation-space plans,
                                                                                                // IGMC readout
  if (!S->wprep || !S->zsave || !y || !dpred) return -17;
  return rs_train(M, params, node_label, node_ptr, edge_ptr, A, B, n_cap, D, S, y, loss_scale, dpred, sqerr, gpart, dhid,
                  cluster, stage_fwd, stage_bwd, err, (cudaStream_t)stream);
}

extern "C" int igmc_backward(const igmc_model_t* M, const float* params, const uint8_t* node_label,
                             const int32_t* node_ptr, const int32_t* edge_ptr, const igmc_adj_t* A, int B, int n_cap,
                             const igmc_dropout_t* D, const igmc_saved_t* S, const float* dpred, float* gpart,
                             float* dhid, int cluster, const igmc_stage_t* stage, int* err, void* stream) {
  if (B <= 0) return 0;
  int rc = check_model(M);
  if (rc) return rc;
  if (!S->zsave) return -14;
  if (M->readout != 0 && !S->dstate) return -17;
  cudaStream_t st = (cudaStream_t)stream;
  if (const int c = l2_csize(cluster)) {
    if (n_cap > IGMC_L2_MAX_NODES) return -3;
    if (!S->l2_scratch) return -17;
    return l2_backward(M, params, node_label, node_ptr, edge_ptr, A, B, c, D, S, dpred, gpart, dhid, S->l2_scratch,
                       err, st);
  }
  if (cluster > 0) {
    if (!rs_supported(M)) return -16;
    if (!S->wprep) return -17;
    return rs_backward(M, params, node_label, node_ptr, edge_ptr, A, B, n_cap, D, S, dpred, gpart, dhid, cluster, stage,
                       err, st);
  }
  const size_t smem = bwd_smem_bytes(n_cap, M->num_relations, M->num_bases, M->num_layers);
  if (smem > 227 * 1024) return -3;
  auto kern = M->num_bases == 4 ? (S->rel_inv_deg ? k_backward<4, true> : k_backward<4, false>)
                                : (S->rel_inv_deg ? k_backward<2, true> : k_backward<2, false>);
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  kern<<<B, MP_THREADS, smem, st>>>(*M, params, node_label, node_ptr, edge_ptr, *A, n_cap, *D, *S, dpred, gpart, dhid,
                                    err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

extern "C" int igmc_edge_grad(const igmc_model_t* M, const float* params, const uint8_t* node_label,
                              const int32_t* node_ptr, const int32_t* edge_ptr, const igmc_adj_t* A, int B, int n_cap,
                              const igmc_dropout_t* D, const igmc_saved_t* S, const float* dpred, float* edge_grad,
                              int cluster, int* err, void* stream) {
  if (B <= 0) return 0;
  int rc = check_model(M);
  if (rc) return rc;
  const int c = l2_csize(cluster);
  if (!c) return -16;
  if (D->adj_dropout > 0.f || D->edge_keep) return -18;   // every edge kept: each one gets its gradient
  if (M->readout != 0 && !S->dstate) return -17;
  if (!S->l2_scratch || !dpred || !edge_grad) return -17;
  if (n_cap > IGMC_L2_MAX_NODES) return -3;
  return l2_edge_grad(M, params, node_label, node_ptr, edge_ptr, A, B, c, D, S, dpred, edge_grad, S->l2_scratch, err,
                      (cudaStream_t)stream);
}
