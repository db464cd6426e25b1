// Batched enclosing-subgraph extraction (h = 1..3) over the device-resident rating CSR/CSC.
//
// Replaces, for a whole mini-batch in two launches, the reference's per-pair Python path
//   MyDynamicDataset.get            util_functions.py:138-145
//   subgraph_extraction_labeling    util_functions.py:208-247   (BFS, sampling, labels, induced sub-matrix)
//   construct_pyg_graph / one_hot   util_functions.py:280-297, 307-311
//   PyG Batch.from_data_list        (third party; SURVEY.md Appendix A.3)
// and emits the already-collated batch in canonical form (SURVEY.md §8c): per side the target
// first, then the fringe in ascending global id; undirected edges sorted by (u_local, v_local).
//
// Layout: one CTA per (user,item) pair.
//   k_extract_select_count : fringe discovery from CSC column j / CSR row i (coalesced int32
//       loads), uniform k-subset sampling by 4-pass radix-select over counter-hash keys
//       (no storage, any degree), item-id -> local-id table in shared memory, per-user-row
//       match count (warp per row).
//   k_extract_fill         : cross-graph prefix (each CTA sums its predecessors' counts),
//       second row scan with warp-ballot ordered compaction, writes x / labels / batch / y /
//       edge_index (int64, PyG order [u|v ; v|u]) / edge_type / node_ptr / edge_ptr.
// HBM-bound integer work: no tensor cores; int32 index + uint8 rating per nonzero.
#include <cstdlib>

#include "common.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr int EX_THREADS = 1024;
constexpr uint16_t NONE16 = 0xFFFF;

// Select the node list of one side and hop from the sorted candidate list `nbr`: with `emit_target` (hop 1)
// out[0] = target and out[1..] = the (sampled) fringe ascending, the target itself excluded from the candidates;
// without (hops >= 2: `out` points behind the nodes found so far) out[0..] = the (sampled) fringe ascending.
__device__ void select_side(const int32_t* __restrict__ nbr, int len, int target, bool emit_target, int mnph,
                            double ratio, uint64_t state, int32_t* __restrict__ outp, int cap, int* n_out,
                            int* hist, int* ws, int* sh, int* err) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const int base_ = emit_target ? 1 : 0;
  int32_t* out = outp + base_ - 1;          // the code below writes the fringe at out[1 + ...]
  if (tid == 0) sh[0] = -1;
  __syncthreads();
  if (emit_target)
    for (int p = tid; p < len; p += nt)
      if (nbr[p] == target) sh[0] = p;  // sorted, duplicate-free list: at most one hit
  __syncthreads();
  const int pos = sh[0];
  const int d = len - (pos >= 0 ? 1 : 0);
  int k = d;
  if (ratio < 1.0) k = (int)(ratio * (double)d);   // int(sample_ratio*len(fringe)), ref :223-224
  if (mnph >= 0 && mnph < k) k = mnph;             // strict '<', ref :226,:228
  if (k + base_ > cap) {
    if (tid == 0) { igmc_set_err(err, IGMC_ERR_NODE_CAP); if (emit_target) outp[0] = target; *n_out = base_; }
    __syncthreads();
    return;
  }
  if (tid == 0) { if (emit_target) outp[0] = target; *n_out = base_ + k; }
  if (k == d) {  // no sampling: ordered copy minus the target
    for (int p = tid; p < len; p += nt) {
      if (p == pos) continue;
      out[1 + p - ((pos >= 0 && p > pos) ? 1 : 0)] = nbr[p];
    }
    __syncthreads();
    return;
  }
  if (k == 0) { __syncthreads(); return; }

  // ---- radix-select the k-th smallest 32-bit key (ties resolved by ascending node id) ----
  uint32_t prefix = 0, mask = 0;
  int remaining = k;
  for (int pass = 3; pass >= 0; --pass) {
    for (int b = tid; b < 256; b += nt) hist[b] = 0;
    __syncthreads();
    for (int p = tid; p < len; p += nt) {
      if (p == pos) continue;
      uint32_t key = sample_key(state, nbr[p]);
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> (8 * pass)) & 255u], 1);
    }
    __syncthreads();
    if (tid < 32) {
      int s = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) s += hist[8 * tid + i];
      int incl = warp_incl_scan_i(s, tid);
      int excl = incl - s;
      if (excl < remaining && remaining <= incl) {
        int c = excl, b = 8 * tid + 7;
        for (int i = 0; i < 8; ++i) {
          int hc = hist[8 * tid + i];
          if (c + hc >= remaining) { b = 8 * tid + i; break; }
          c += hc;
        }
        sh[1] = b;
        sh[2] = remaining - c;
      }
    }
    __syncthreads();
    prefix |= (uint32_t)sh[1] << (8 * pass);
    mask |= 255u << (8 * pass);
    remaining = sh[2];
    __syncthreads();
  }
  const uint32_t tau = prefix;  // keys < tau are all taken; `remaining` ties (key == tau) are taken
  // ordered compaction with two barriers: every warp owns one contiguous range of the list (a multiple of 32 entries),
  // counts its (strict | tie << 16) selections, all warps scan the <= 32 per-warp totals, then each warp writes its
  // range with ballot ranks.  (A block scan per 1024-entry chunk cost 3 barriers per chunk: 17 % of the kernel.)
  {
    const int lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    const int chunks = (len + 31) >> 5, per = (chunks + nw - 1) / nw;
    const int c0 = warp * per, c1 = min(chunks, c0 + per);
    int cs = 0, ct = 0;
    for (int c = c0; c < c1; ++c) {
      const int p = (c << 5) + lane;
      int strict = 0, tie = 0;
      if (p < len && p != pos) {
        const uint32_t key = sample_key(state, nbr[p]);
        strict = key < tau;
        tie = key == tau;
      }
      cs += __popc(__ballot_sync(IGMC_FULL, strict));
      ct += __popc(__ballot_sync(IGMC_FULL, tie));
    }
    if (lane == 0) { hist[warp] = cs; hist[32 + warp] = ct; }   // (the radix histogram is free again)
    __syncthreads();
    int sb = 0, tb = 0;
    for (int w = 0; w < warp; ++w) { sb += hist[w]; tb += hist[32 + w]; }
    const unsigned lt = (1u << lane) - 1u;
    for (int c = c0; c < c1; ++c) {
      const int p = (c << 5) + lane;
      int strict = 0, tie = 0, node = 0;
      if (p < len && p != pos) {
        node = nbr[p];
        const uint32_t key = sample_key(state, node);
        strict = key < tau;
        tie = key == tau;
      }
      const unsigned bs = __ballot_sync(IGMC_FULL, strict), bt = __ballot_sync(IGMC_FULL, tie);
      const int s_here = sb + __popc(bs & lt), t_here = tb + __popc(bt & lt);
      if (strict || (tie && t_here < remaining)) out[1 + s_here + min(t_here, remaining)] = node;
      sb += __popc(bs);
      tb += __popc(bt);
    }
  }
  __syncthreads();
}

// ---- hops >= 2 (util_functions.py:216-235): bitmaps over one side's ids in shared memory -------------------------
// cand |= union of the CSR rows (CSC columns) of `nodes`  (warp per node, coalesced index reads)
__device__ void mark_neighbours(const int32_t* __restrict__ ptr, const int32_t* __restrict__ idx,
                                const int32_t* __restrict__ nodes, int cnt, uint32_t* cand) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int a = warp; a < cnt; a += nwarps) {
    const int v = nodes[a];
    for (int p = ptr[v] + lane; p < ptr[v + 1]; p += 32) {
      const int t = idx[p];
      atomicOr(&cand[t >> 5], 1u << (t & 31));
    }
  }
}
// fringe = cand & ~visited; visited |= fringe; list = ids of the fringe ascending.  Returns its length (block-wide).
__device__ int fringe_to_list(uint32_t* cand, uint32_t* vis, int words, int32_t* list, int* ws) {
  const int tid = threadIdx.x, nt = blockDim.x;
  int running = 0;
  for (int base = 0; base < words; base += nt) {
    const int w = base + tid;
    uint32_t f = 0;
    if (w < words) {
      f = cand[w] & ~vis[w];
      vis[w] |= f;
    }
    int tot;
    const int ex = block_excl_scan_i(__popc(f), ws, &tot);
    int o = running + ex;
    while (f) {
      const int b = __ffs(f) - 1;
      list[o++] = (w << 5) + b;
      f &= f - 1;
    }
    running += tot;
  }
  __syncthreads();
  return running;
}

__device__ __forceinline__ void resolve_pair(const igmc_pairs_t& P, int g, int* i, int* j, int* lab, int64_t* pid) {
  const int64_t src = P.idx ? P.idx[g] : (int64_t)g;
  *i = P.links_u[src];
  *j = P.links_v[src];
  *lab = P.links_label ? P.links_label[src] : 0;
  *pid = P.pair_id ? P.pair_id[g] : src;
}

// A rating label (stored, or the pair's) as an index of class_values and of the model's relations: outside 0..R-1 it
// sets IGMC_ERR_LABEL (when `who` is 0: callers pass their thread index to flag once per CTA) and reads as 0, so that
// no later kernel indexes a relation table past R.
__device__ __forceinline__ int checked_label(int lab, int R, int who, int* err) {
  if ((unsigned)lab < (unsigned)R) return lab;
  if (who == 0) igmc_set_err(err, IGMC_ERR_LABEL);
  return 0;
}

// Session mode (igmc_extract_sessions, SESS = true): graph g takes its target user's row from session row sess[g];
// every other row and column comes from G.  Plain mode passes an empty SessArg and never reads it.
struct SessArg {
  igmc_sessions_t S;
  const int32_t* sess;   // [B] session of graph g
};

// the target row (ptr into its column ids, its ratings, its length) of graph g in session mode
struct TargetRow {
  const int32_t* col;
  const uint8_t* rat;
  int len;
};

// The row local user a (global id u) reads: in session mode the target user's (a = 0) is its session row, every other
// row is G's.  Plain mode never reads `tr`.
template <bool SESS>
struct UserRows {
  const igmc_csr_t& G;
  TargetRow tr;
  __device__ __forceinline__ bool own(int a) const { return SESS && a == 0; }
  __device__ __forceinline__ const int32_t* col(int a) const { return own(a) ? tr.col : G.col_idx; }
  __device__ __forceinline__ const uint8_t* rat(int a) const { return own(a) ? tr.rat : G.rating; }
  __device__ __forceinline__ int begin(int a, int u) const { return own(a) ? 0 : G.row_ptr[u]; }
  __device__ __forceinline__ int end(int a, int u) const { return own(a) ? tr.len : G.row_ptr[u + 1]; }
};
template <bool SESS>
__device__ __forceinline__ UserRows<SESS> user_rows(const igmc_csr_t& G, const SessArg& A, int g) {
  UserRows<SESS> rows = {G, {}};
  if (SESS) {
    const int q = A.sess[g];
    const int s = A.S.row_ptr[q];
    rows.tr = {A.S.col_idx + s, A.S.rating + s, A.S.row_ptr[q + 1] - s};
  }
  return rows;
}

// Hop-1 node lists of graph g (target first) into gu / gv and their lengths into *s_nu / *s_nv: the injected lists, or
// the (sampled) users who rated item j and items user i rated.  Ends with a barrier on the injected branch only.
template <bool SESS>
__device__ __forceinline__ void hop1_lists(const UserRows<SESS>& rows, const int32_t* inj_nodes_u,
                                           const int32_t* inj_nodes_v, const int32_t* inj_n_u, const int32_t* inj_n_v,
                                           int g, int i, int j, int mnph, double ratio, uint64_t seed, int64_t pid,
                                           int cap, int32_t* gu, int32_t* gv, int* s_nu, int* s_nv, int* hist, int* ws,
                                           int* sh, int* err) {
  const int tid = threadIdx.x, nt = blockDim.x;
  if (!SESS && inj_nodes_u) {
    const int nu = inj_n_u[g], nv = inj_n_v[g];
    if (nu > cap || nv > cap) {
      if (tid == 0) { igmc_set_err(err, IGMC_ERR_NODE_CAP); *s_nu = 1; *s_nv = 1; gu[0] = i; gv[0] = j; }
    } else {
      for (int t = tid; t < nu; t += nt) gu[t] = inj_nodes_u[(size_t)g * cap + t];
      for (int t = tid; t < nv; t += nt) gv[t] = inj_nodes_v[(size_t)g * cap + t];
      if (tid == 0) { *s_nu = nu; *s_nv = nv; }
    }
    __syncthreads();
  } else {
    const igmc_csr_t& G = rows.G;
    // user fringe = users who rated item j (CSC column j); item fringe = items rated by user i (its row)
    select_side(G.row_idx + G.col_ptr[j], G.col_ptr[j + 1] - G.col_ptr[j], i, true, mnph, ratio,
                sample_state(seed, pid, 0, 1), gu, cap, s_nu, hist, ws, sh, err);
    const int s = rows.begin(0, i);
    select_side(rows.col(0) + s, rows.end(0, i) - s, j, true, mnph, ratio, sample_state(seed, pid, 1, 1), gv, cap, s_nv,
                hist, ws, sh, err);
  }
}

// Node and edge bases of graph g: block-wide sums over its predecessors q < g of count(q) = (nodes, edges).
template <class Count>
__device__ __forceinline__ int2 graph_bases(int g, int* ws, Count count) {
  int ns = 0, es = 0;
  for (int q = threadIdx.x; q < g; q += blockDim.x) {
    const int2 c = count(q);
    ns += c.x;
    es += c.y;
  }
  const int nb = block_sum_i(ns, ws);
  return make_int2(nb, block_sum_i(es, ws));
}

// The batch offsets of graph g (n nodes from Nbase, e directed edges from Ebase): node_ptr / edge_ptr, and from the
// last graph the totals and the end of adj_in_ptr.  Returns false, the error set, when the graph does not fit the batch.
__device__ __forceinline__ bool batch_offsets(const igmc_batch_out_t& O, int g, int B, int Nbase, int n, int Ebase,
                                              int e, int* err) {
  if (threadIdx.x == 0) {
    if (g == B - 1) {
      O.counts[0] = Nbase + n;
      O.counts[1] = Ebase + e;
      O.node_ptr[B] = Nbase + n;
      O.edge_ptr[B] = Ebase + e;
      if (O.adj_in_ptr && Nbase + n <= O.node_cap) O.adj_in_ptr[Nbase + n] = Ebase + e;
    }
    O.node_ptr[g] = Nbase;
    O.edge_ptr[g] = Ebase;
  }
  if (Nbase + n > O.node_cap || Ebase + e > O.edge_cap) {
    if (threadIdx.x == 0) igmc_set_err(err, (Nbase + n > O.node_cap) ? IGMC_ERR_NODE_TOTAL : IGMC_ERR_EDGE_CAP);
    return false;
  }
  return true;
}

// one node row of the batch: label, graph, global id and the one-hot x
__device__ __forceinline__ void store_node(const igmc_batch_out_t& O, size_t row, int label, int g, int gid) {
  O.node_label[row] = (uint8_t)label;
  O.batch[row] = g;
  O.node_gid[row] = gid;
  if (O.x)
    for (int f = 0; f < O.feat_dim; ++f) O.x[row * O.feat_dim + f] = (f == label) ? 1.0f : 0.0f;
}

template <bool SESS>
__global__ void __launch_bounds__(EX_THREADS)
k_extract_select_count(igmc_csr_t G, igmc_pairs_t P, int B, int mnph, double ratio, uint64_t seed_val,
                       const uint64_t* __restrict__ seed_dev, int cap,
                       const int32_t* __restrict__ inj_nodes_u, const int32_t* __restrict__ inj_nodes_v,
                       const int32_t* __restrict__ inj_n_u, const int32_t* __restrict__ inj_n_v,
                       int32_t* __restrict__ nodes_u, int32_t* __restrict__ nodes_v,
                       int32_t* __restrict__ n_u, int32_t* __restrict__ n_v,
                       int32_t* __restrict__ row_cnt, int32_t* __restrict__ m_cnt, int32_t* __restrict__ col_cnt,
                       int h, int32_t* __restrict__ hop_off, int* err, SessArg A) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int* colcnt = reinterpret_cast<int*>(smem_raw);                 // [cap]
  uint16_t* tab = reinterpret_cast<uint16_t*>(colcnt + cap);      // [num_items]
  // h > 1 only: visited / candidate bitmaps and the ascending fringe list, behind the item table
  const int wu = (G.num_users + 31) >> 5, wv = (G.num_items + 31) >> 5;
  uint32_t* vis_u = reinterpret_cast<uint32_t*>(smem_raw + (((size_t)cap * 4 + (size_t)G.num_items * 2 + 15) & ~(size_t)15));
  uint32_t* vis_v = vis_u + wu;
  uint32_t* cand = vis_v + wv;
  int32_t* flist = reinterpret_cast<int32_t*>(cand + max(wu, wv));
  __shared__ int hist[256];
  __shared__ int ws[34];
  __shared__ int sh[4];
  __shared__ int s_nu, s_nv, s_m;
  const int g = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
  const uint64_t seed = seed_dev ? *seed_dev : seed_val;
  int i, j, lab;
  int64_t pid;
  resolve_pair(P, g, &i, &j, &lab, &pid);
  const UserRows<SESS> rows = user_rows<SESS>(G, A, g);
  int32_t* gu = nodes_u + (size_t)g * cap;
  int32_t* gv = nodes_v + (size_t)g * cap;
  if (tid == 0) s_m = 0;
  hop1_lists<SESS>(rows, inj_nodes_u, inj_nodes_v, inj_n_u, inj_n_v, g, i, j, mnph, ratio, seed, pid, cap, gu, gv,
                   &s_nu, &s_nv, hist, ws, sh, err);
  __syncthreads();
  if (hop_off && tid == 0) {   // nodes within distance d per side: [users 0..3 | items 0..3]
    int32_t* ho = hop_off + (size_t)g * 2 * (IGMC_MAX_HOP + 1);
    ho[0] = 1; ho[IGMC_MAX_HOP + 1] = 1;
    for (int d = 1; d <= IGMC_MAX_HOP; ++d) { ho[d] = s_nu; ho[IGMC_MAX_HOP + 1 + d] = s_nv; }
  }
  if (h > 1 && (SESS || !inj_nodes_u)) {
    // visited = the targets and the WHOLE hop-1 fringes (the reference marks a fringe visited before it samples it,
    // util_functions.py:220-221)
    for (int w = tid; w < wu + wv; w += nt) vis_u[w] = 0;   // vis_u and vis_v are contiguous
    __syncthreads();
    // (a session's new user, i >= num_users, is in no column of G: it needs no visited bit and has none)
    if (tid == 0) {
      if (!SESS || i < G.num_users) atomicOr(&vis_u[i >> 5], 1u << (i & 31));
      atomicOr(&vis_v[j >> 5], 1u << (j & 31));
    }
    for (int p = G.col_ptr[j] + tid; p < G.col_ptr[j + 1]; p += nt) { const int t = G.row_idx[p]; atomicOr(&vis_u[t >> 5], 1u << (t & 31)); }
    {
      const int32_t* ci = rows.col(0);
      const int e = rows.end(0, i);
      for (int p = rows.begin(0, i) + tid; p < e; p += nt) {
        const int t = ci[p];
        atomicOr(&vis_v[t >> 5], 1u << (t & 31));
      }
    }
    __syncthreads();
    int lo_u = 1, hi_u = s_nu, lo_v = 1, hi_v = s_nv;
    for (int d = 2; d <= h; ++d) {
      // both new fringes come from the PREVIOUS fringes (tuple assignment, util_functions.py:217)
      for (int w = tid; w < wv; w += nt) cand[w] = 0;
      __syncthreads();
      mark_neighbours(G.row_ptr, G.col_idx, gu + lo_u, hi_u - lo_u, cand);
      __syncthreads();
      int len = fringe_to_list(cand, vis_v, wv, flist, ws);
      select_side(flist, len, -1, false, mnph, ratio, sample_state(seed, pid, 1, d), gv + hi_v, cap - hi_v, &s_nv,
                  hist, ws, sh, err);
      __syncthreads();
      const int add_v = s_nv;
      for (int w = tid; w < wu; w += nt) cand[w] = 0;
      __syncthreads();
      mark_neighbours(G.col_ptr, G.row_idx, gv + lo_v, hi_v - lo_v, cand);
      __syncthreads();
      len = fringe_to_list(cand, vis_u, wu, flist, ws);
      select_side(flist, len, -1, false, mnph, ratio, sample_state(seed, pid, 0, d), gu + hi_u, cap - hi_u, &s_nu,
                  hist, ws, sh, err);
      __syncthreads();
      const int add_u = s_nu;
      if (add_u == 0 && add_v == 0) break;        // util_functions.py:230-231
      lo_u = hi_u; hi_u += add_u; lo_v = hi_v; hi_v += add_v;
      if (hop_off && tid == 0) {
        int32_t* ho = hop_off + (size_t)g * 2 * (IGMC_MAX_HOP + 1);
        for (int dd = d; dd <= IGMC_MAX_HOP; ++dd) { ho[dd] = hi_u; ho[IGMC_MAX_HOP + 1 + dd] = hi_v; }
      }
      __syncthreads();
    }
    if (tid == 0) { s_nu = hi_u; s_nv = hi_v; }
    __syncthreads();
  }
  const int nu = s_nu, nv = s_nv;
  // item-id -> local-id table
  for (int t = tid; t < G.num_items; t += nt) tab[t] = NONE16;
  for (int b = tid; b < nv; b += nt) colcnt[b] = 0;
  __syncthreads();
  for (int b = tid; b < nv; b += nt) tab[gv[b]] = (uint16_t)b;
  __syncthreads();
  // per-row match count (warp per user row); bit31 = row contains the target item j
  for (int a = warp; a < nu; a += nwarps) {
    const int u = gu[a];
    const int32_t* ci = rows.col(a);
    const int s = rows.begin(a, u), e = rows.end(a, u);
    int cnt = 0, hasj = 0;
    for (int p = s + lane; p < e; p += 32) {
      const uint16_t b = tab[ci[p]];
      if (b != NONE16) {
        if (b == 0) { hasj = 1; if (a != 0) { ++cnt; atomicAdd(&colcnt[0], 1); } }   // (0,0) = target edge: dropped (ref :238)
        else { ++cnt; atomicAdd(&colcnt[b], 1); }
      }
    }
    cnt = warp_sum_i(cnt);
    hasj = __any_sync(IGMC_FULL, hasj);
    if (lane == 0) {
      row_cnt[(size_t)g * cap + a] = cnt | (hasj ? (int)0x80000000 : 0);
      atomicAdd(&s_m, cnt);
    }
  }
  __syncthreads();
  for (int b = tid; b < nv; b += nt) col_cnt[(size_t)g * cap + b] = colcnt[b];
  if (tid == 0) { n_u[g] = nu; n_v[g] = nv; m_cnt[g] = s_m; }
}

template <bool SESS>
__global__ void __launch_bounds__(EX_THREADS)
k_extract_fill(igmc_csr_t G, igmc_pairs_t P, int B, int cap,
               const int32_t* __restrict__ nodes_u, const int32_t* __restrict__ nodes_v,
               const int32_t* __restrict__ n_u, const int32_t* __restrict__ n_v,
               const int32_t* __restrict__ row_cnt, const int32_t* __restrict__ m_cnt,
               const int32_t* __restrict__ col_cnt, int h, const int32_t* __restrict__ hop_off,
               const float* __restrict__ class_values, int R, igmc_batch_out_t O, int* err, SessArg A) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int* rowoff = reinterpret_cast<int*>(smem_raw);                 // [cap]
  int* colfill = rowoff + cap;                                    // [cap] running fill pointer of the item lists
  uint16_t* tab = reinterpret_cast<uint16_t*>(colfill + cap);     // [num_items]
  __shared__ int ws[34];
  const int g = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
  const int2 base = graph_bases(g, ws, [&](int q) { return make_int2(n_u[q] + n_v[q], m_cnt[q]); });
  const int Nbase = base.x, Mbase = base.y;
  const int nu = n_u[g], nv = n_v[g], m = m_cnt[g], n = nu + nv;
  const int32_t* gu = nodes_u + (size_t)g * cap;
  const int32_t* gv = nodes_v + (size_t)g * cap;
  const bool want_adj = O.adj_in_ptr != nullptr;
  if (!batch_offsets(O, g, B, Nbase, n, 2 * Mbase, 2 * m, err)) return;
  int i, j, lab;
  int64_t pid;
  resolve_pair(P, g, &i, &j, &lab, &pid);
  lab = checked_label(lab, R, tid, err);
  if (tid == 0) {
    O.y[g] = class_values[lab];
    O.graph_nu[g] = nu;
  }
  // node labels: user at distance d -> 2d, item -> 2d+1 (ref :245); h=1: 0 / 1 targets, 2 / 3 the others
  int hu[IGMC_MAX_HOP + 1], hv[IGMC_MAX_HOP + 1];   // nodes within distance d, per side
#pragma unroll
  for (int d = 0; d <= IGMC_MAX_HOP; ++d) {
    hu[d] = (h > 1 && hop_off) ? hop_off[(size_t)g * 2 * (IGMC_MAX_HOP + 1) + d] : (d == 0 ? 1 : nu);
    hv[d] = (h > 1 && hop_off) ? hop_off[(size_t)g * 2 * (IGMC_MAX_HOP + 1) + IGMC_MAX_HOP + 1 + d] : (d == 0 ? 1 : nv);
  }
  for (int t = tid; t < n; t += nt) {
    int label;
    if (t < nu) {
      int d = 0;
#pragma unroll
      for (int q = 0; q < IGMC_MAX_HOP; ++q) d += (t >= hu[q]) ? 1 : 0;
      label = 2 * d;
    } else {
      int d = 0;
#pragma unroll
      for (int q = 0; q < IGMC_MAX_HOP; ++q) d += (t - nu >= hv[q]) ? 1 : 0;
      label = 2 * d + 1;
    }
    store_node(O, (size_t)Nbase + t, label, g, t < nu ? gu[t] : gv[t - nu]);
  }
  // exclusive scan of the per-row match counts; user a: in-edges from its items
  block_scan_chunks(
      nu, ws, [&](int a) { return row_cnt[(size_t)g * cap + a] & 0x7fffffff; },
      [&](int a, int ex) {
        rowoff[a] = ex;
        if (want_adj) O.adj_in_ptr[Nbase + a] = 2 * Mbase + ex;
      });
  if (want_adj)   // item b: in-edges from users, stored after the m user-side entries of this graph
    block_scan_chunks(
        nv, ws, [&](int b) { return col_cnt[(size_t)g * cap + b]; },
        [&](int b, int ex) {
          colfill[b] = ex;
          O.adj_in_ptr[Nbase + nu + b] = 2 * Mbase + m + ex;
        });
  for (int t = tid; t < G.num_items; t += nt) tab[t] = NONE16;
  __syncthreads();
  for (int b = tid; b < nv; b += nt) tab[gv[b]] = (uint16_t)b;
  __syncthreads();
  int64_t* ei0 = O.edge_index;
  int64_t* ei1 = O.edge_index + O.edge_cap;
  const unsigned lt_mask = (1u << lane) - 1u;
  const UserRows<SESS> rows = user_rows<SESS>(G, A, g);
  for (int a = warp; a < nu; a += nwarps) {
    const int u = gu[a];
    const int32_t* ci = rows.col(a);
    const uint8_t* rt = rows.rat(a);
    const int s = rows.begin(a, u), e = rows.end(a, u);
    const int jfirst = (a != 0 && (row_cnt[(size_t)g * cap + a] < 0)) ? 1 : 0;  // j sorts first (v_local 0)
    const int base = rowoff[a];
    int seen = 0;
    // h > 1: local item ids ascend with (hop, global id), the row is in global-id order -> a match's rank is the
    // number of matches of earlier hops plus its position among the matches of its own hop
    int hop_base[IGMC_MAX_HOP + 1] = {0, 0, 0, 0}, hop_seen[IGMC_MAX_HOP + 1] = {0, 0, 0, 0};
    if (h > 1) {
      int c[IGMC_MAX_HOP + 1] = {0, 0, 0, 0};
      for (int p0 = s; p0 < e; p0 += 32) {
        const int p = p0 + lane;
        uint16_t b = NONE16;
        if (p < e) b = tab[ci[p]];
        const bool m_ = (b != NONE16) && b != 0;
#pragma unroll
        for (int d = 1; d <= IGMC_MAX_HOP; ++d)
          c[d] += __popc(__ballot_sync(IGMC_FULL, m_ && (int)b >= hv[d - 1] && (int)b < hv[d]));
      }
      hop_base[1] = 0;
#pragma unroll
      for (int d = 2; d <= IGMC_MAX_HOP; ++d) hop_base[d] = hop_base[d - 1] + c[d - 1];
    }
    for (int p0 = s; p0 < e; p0 += 32) {
      const int p = p0 + lane;
      uint16_t b = NONE16;
      if (p < e) b = tab[ci[p]];
      const bool match = (b != NONE16) && !(a == 0 && b == 0);
      const bool isj = match && b == 0;
      const unsigned bal = __ballot_sync(IGMC_FULL, match && !isj);
      int hrank = 0;
      if (h > 1) {
#pragma unroll
        for (int d = 1; d <= IGMC_MAX_HOP; ++d) {
          const bool in_d = match && !isj && (int)b >= hv[d - 1] && (int)b < hv[d];
          const unsigned bd = __ballot_sync(IGMC_FULL, in_d);
          if (in_d) hrank = hop_base[d] + hop_seen[d] + __popc(bd & lt_mask);
          hop_seen[d] += __popc(bd);
        }
      }
      if (match) {
        const int rank = isj ? 0 : (h > 1 ? jfirst + hrank : jfirst + seen + __popc(bal & lt_mask));
        const int64_t r = checked_label(rt[p], R, 0, err);
        const size_t e1 = (size_t)2 * Mbase + base + rank, e2 = e1 + m;
        const int64_t un = Nbase + a, vn = Nbase + nu + b;
        ei0[e1] = un; ei1[e1] = vn; O.edge_type[e1] = r;
        ei0[e2] = vn; ei1[e2] = un; O.edge_type[e2] = r;
        if (want_adj) {
          // user a's list (slots [rowoff[a], +cnt)): in-edge item->user is the mirrored copy e2
          O.adj_tmp[e1] = list_key((uint32_t)r, (uint32_t)(nu + b), (uint32_t)e2);
          // item b's list: in-edge user->item is e1; unordered placement
          const int slot = atomicAdd(&colfill[b], 1);
          O.adj_tmp[(size_t)2 * Mbase + m + slot] = list_key((uint32_t)r, (uint32_t)a, (uint32_t)e1);
        }
      }
      seen += __popc(bal);
    }
  }
  if (want_adj) {   // deterministic lists sorted by (type, neighbour): rank-sort (lists are short)
    __syncthreads();
    for (int v = warp; v < n; v += nwarps) {
      int k;
      size_t beg;
      if (v < nu) {
        k = row_cnt[(size_t)g * cap + v] & 0x7fffffff;
        beg = (size_t)2 * Mbase + rowoff[v];
      } else {
        k = col_cnt[(size_t)g * cap + (v - nu)];
        beg = (size_t)2 * Mbase + m + (colfill[v - nu] - k);
      }
      rank_sort_list(O.adj_tmp + beg, k, O.adj_in + beg, O.adj_eid + beg, 0);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// h = 1 fast path: ONE launch, one 512-thread CTA per pair (two CTAs per SM, so that a batch sits next to the model
// kernels' one-per-SM CTAs), every row entry read once.
//   A  node lists (select_side, as above)
//   B  the concatenated user rows are cut into 128-entry tiles handed round-robin to the warps (balanced whatever
//      the row lengths; four independent index loads in flight per lane).  A matching entry (item in the subgraph,
//      looked up in the shared-memory item table) is packed as  u_local << 20 | v_local << 8 | rating  and appended
//      to the graph's scratch slot at a cursor position reserved per tile; edges to the target item (which sort first
//      in their row) are kept per row instead.  Per-row counts by shared atomics; a bitmap over the user rows per
//      (item, rating) replaces every per-item counter.
//   C  canonical rank of an entry = exclusive prefix of the tile counts + index in its tile (+ the row's target-item
//      edges before it): block scans, then the cross-graph node / edge offsets by look-back on the counts the
//      lower-numbered CTAs publish (no second launch, no host sync).
//   D  the entries go to their canonical positions in a shared-memory copy and in the API arrays (edge_index,
//      edge_type; both directions); message-passing lists sorted by (rating, neighbour): a user's list is its
//      contiguous run of the canonical order, stably split by rating with warp ballots; an entry's position in its
//      item's list is a population count over the (item, rating) bitmaps.  No sort, no O(k^2) ranking.
// Same outputs, bit for bit, as the generic two-kernel path (tests/test_gpu_extract.py runs both).
// ------------------------------------------------------------------------------------------------------------------
constexpr int FX_THREADS = 512;
constexpr int FX_TILE = 128;
constexpr int FX_TCAP = 2048;        // tiles per pair: the user rows of one subgraph hold <= 262144 entries
constexpr int FX_CANO = 12288;       // canonical edges kept in shared memory (more: second half of the scratch slot)
constexpr int FX_MAXCAP = 4095;      // local ids travel in 12 bits
constexpr int FX_MAXR = 32;          // rating classes (lane = class in the ballot split)

__device__ __forceinline__ void st_release_gpu(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

struct FastSmem {   // carve-up of the dynamic shared memory (ints unless noted); `words` = bitmap words per (item, rating)
  int *rp, *rowstart, *rowcnt, *rowoff, *jbefore, *hj, *colcnt, *coloff, *cur, *tilebase, *stage_off;
  uint32_t *bm, *cano;
  uint16_t* tab;
};
__host__ __device__ __forceinline__ size_t fast_smem_ints(int cap, int R, int words) {
  return (size_t)cap * 4 + (size_t)(cap + 1) * 4 + (size_t)cap * R + (size_t)cap * R * words + (FX_TCAP + 1) + FX_TCAP +
         FX_CANO;
}


// List length of item b from the (item, rating) bitmaps; S.cur[b * R + r] gets the first slot of rating r's sub-list.
__device__ __forceinline__ int item_list(const FastSmem& S, int b, int R, int words) {
  int run = 0;
  for (int r = 0; r < R; ++r) {
    S.cur[b * R + r] = run;
    const uint32_t* w = S.bm + ((size_t)b * R + r) * words;
    for (int x = 0; x < words; ++x) run += __popc(w[x]);
  }
  S.colcnt[b] = run;
  return run;
}

template <bool SESS>
__global__ void __launch_bounds__(FX_THREADS, 2)
k_extract_fast(igmc_csr_t G, igmc_pairs_t P, int B, int mnph, double ratio, uint64_t seed_val,
               const uint64_t* __restrict__ seed_dev, int cap, const int32_t* __restrict__ inj_nodes_u,
               const int32_t* __restrict__ inj_nodes_v, const int32_t* __restrict__ inj_n_u,
               const int32_t* __restrict__ inj_n_v, igmc_extract_ws_t W, int R, int words, int slot_e,
               const float* __restrict__ class_values, igmc_batch_out_t O, int* err, SessArg A) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FastSmem S;
  {
    int* p = reinterpret_cast<int*>(smem_raw);
    S.rp = p; p += cap;
    S.rowcnt = p; p += cap;
    S.hj = p; p += cap;
    S.colcnt = p; p += cap;
    S.rowstart = p; p += cap + 1;
    S.rowoff = p; p += cap + 1;
    S.jbefore = p; p += cap + 1;
    S.coloff = p; p += cap + 1;
    S.cur = p; p += cap * R;
    S.bm = reinterpret_cast<uint32_t*>(p); p += (size_t)cap * R * words;
    S.tilebase = p; p += FX_TCAP + 1;
    S.stage_off = p; p += FX_TCAP;
    S.cano = reinterpret_cast<uint32_t*>(p); p += FX_CANO;
    S.tab = reinterpret_cast<uint16_t*>(p);
  }
  __shared__ int hist[256];
  __shared__ int ws[34];
  __shared__ int sh[4];
  __shared__ int s_nu, s_nv, s_cursor;
  const int g = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  const uint64_t seed = seed_dev ? *seed_dev : seed_val;
  int* flags = W.sync;   // [B] "counts published" flags + [1] completion ticket (all zero between launches)
  // debug aid (the hop table is unused for h = 1): low 32 bits of the CTA's start / end wall clock and its SM
  if (tid == 0 && W.hop_off) {
    W.hop_off[(size_t)g * 2 * (IGMC_MAX_HOP + 1) + 5] = (int)(igmc_globaltimer() & 0x7fffffff);
    W.hop_off[(size_t)g * 2 * (IGMC_MAX_HOP + 1) + 7] = igmc_smid();
  }
  int i, j, lab;
  int64_t pid;
  resolve_pair(P, g, &i, &j, &lab, &pid);
  lab = checked_label(lab, R, tid, err);
  const UserRows<SESS> rows = user_rows<SESS>(G, A, g);
  int32_t* gu = W.nodes_u + (size_t)g * cap;
  int32_t* gv = W.nodes_v + (size_t)g * cap;

  // ---- A: node lists ----
  hop1_lists<SESS>(rows, inj_nodes_u, inj_nodes_v, inj_n_u, inj_n_v, g, i, j, mnph, ratio, seed, pid, cap, gu, gv,
                   &s_nu, &s_nv, hist, ws, sh, err);
  __syncthreads();
  const int nu = s_nu, nv = s_nv, n = nu + nv;

  // ---- B: one balanced scan of the user rows ----
  for (int t = tid; t < G.num_items; t += nt) S.tab[t] = NONE16;
  for (int t = tid; t < nv * R * words; t += nt) S.bm[t] = 0u;
  for (int a = tid; a < nu; a += nt) { S.rowcnt[a] = 0; S.hj[a] = 0; }
  if (tid == 0) s_cursor = 0;
  {   // row pointers and the flat prefix of the row lengths
    const int total = block_scan_chunks(
        nu, ws,
        [&](int a) {
          const int u = gu[a];
          S.rp[a] = rows.begin(a, u);
          return rows.end(a, u) - S.rp[a];
        },
        [&](int a, int ex) { S.rowstart[a] = ex; });
    if (tid == 0) S.rowstart[nu] = total;
  }
  __syncthreads();
  for (int b = tid; b < nv; b += nt) S.tab[gv[b]] = (uint16_t)b;
  __syncthreads();
  const int D = S.rowstart[nu];
  const int T = (D + FX_TILE - 1) / FX_TILE;
  uint32_t* stage = reinterpret_cast<uint32_t*>(O.adj_tmp + (size_t)g * slot_e);   // [2 * slot_e] u32 of scratch
  if (T > FX_TCAP) {   // the host sizes the plan so that this cannot happen; never run past the tables
    if (tid == 0) igmc_set_err(err, IGMC_ERR_EDGE_CAP);
  } else {
    for (int tile = warp; tile < T; tile += nwarps) {
      const int q0 = tile * FX_TILE;
      int lo = 0, hi = nu - 1;   // row of entry q0 (uniform over the warp)
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (S.rowstart[mid] <= q0) lo = mid; else hi = mid - 1;
      }
      int ar[4], col[4];
      uint32_t rat[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int q = q0 + 32 * u + lane;
        int a = lo;
        col[u] = -1;
        rat[u] = 0;
        if (q < D) {
          while (q >= S.rowstart[a + 1]) ++a;
          const int p = S.rp[a] + (q - S.rowstart[a]);
          col[u] = __ldg(rows.col(a) + p);
          rat[u] = __ldg(rows.rat(a) + p);   // fetched with the index (1 B per entry): no second dependent L2 latency
        }
        ar[u] = a;
      }
      uint32_t word[4];
      unsigned bal[4];
      int cnt = 0;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        uint16_t b = NONE16;
        if (col[u] >= 0) b = S.tab[col[u]];
        const bool match = (b != NONE16) && !(ar[u] == 0 && b == 0);   // (target user, target item): removed (ref :238)
        uint32_t r = 0;
        if (match) {
          r = rat[u];
          r = checked_label((int)r, R, 0, err);
          atomicAdd(&S.rowcnt[ar[u]], 1);
          atomicOr(&S.bm[((size_t)b * R + r) * words + (ar[u] >> 5)], 1u << (ar[u] & 31));
          if (b == 0) S.hj[ar[u]] = 1 | (int)(r << 8);
        }
        const bool nonj = match && b != 0;
        word[u] = nonj ? (((uint32_t)ar[u] << 20) | ((uint32_t)b << 8) | r) : 0xFFFFFFFFu;
        bal[u] = __ballot_sync(IGMC_FULL, nonj);
        cnt += __popc(bal[u]);
      }
      int off = 0;
      if (lane == 0) {
        if (cnt) off = atomicAdd(&s_cursor, cnt);
        S.stage_off[tile] = off;
        S.tilebase[tile] = cnt;
      }
      off = __shfl_sync(IGMC_FULL, off, 0);
      if (off + cnt <= 2 * slot_e) {   // never write past the scratch slot (the overflow is reported below)
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (word[u] != 0xFFFFFFFFu) stage[off + __popc(bal[u] & lt_mask)] = word[u];
          off += __popc(bal[u]);
        }
      }
    }
  }
  __syncthreads();

  // ---- C: prefixes ----
  // rows: edge offsets and the number of target-item edges in earlier rows, one packed scan (counts < 2^20);
  // tiles: staged entries -> exclusive prefix, in place; items: list offsets from the (item, rating) bitmaps
  const int TTc = T > FX_TCAP ? 0 : T;
  if (nu <= nt && nv <= nt && TTc <= nt) {
    // the common case (every table fits one value per thread): the three exclusive scans share one set of barriers
    int v0 = tid < nu ? (S.rowcnt[tid] | ((S.hj[tid] & 1) << 20)) : 0;
    int v1 = tid < TTc ? S.tilebase[tid] : 0;
    int v2 = tid < nv ? item_list(S, tid, R, words) : 0;
    int i0 = warp_incl_scan_i(v0, lane), i1 = warp_incl_scan_i(v1, lane), i2 = warp_incl_scan_i(v2, lane);
    if (lane == 31) { hist[warp] = i0; hist[32 + warp] = i1; hist[64 + warp] = i2; }
    __syncthreads();
    if (warp < 3) {
      const int sv = lane < nwarps ? hist[32 * warp + lane] : 0;
      const int inc = warp_incl_scan_i(sv, lane);
      hist[96 + 32 * warp + lane] = inc - sv;
      if (lane == 31) hist[192 + warp] = inc;
    }
    __syncthreads();
    const int e0 = hist[96 + warp] + i0 - v0, e1 = hist[128 + warp] + i1 - v1, e2 = hist[160 + warp] + i2 - v2;
    if (tid < nu) { S.rowoff[tid] = e0 & 0xFFFFF; S.jbefore[tid] = e0 >> 20; }
    if (tid < TTc) S.tilebase[tid] = e1;
    if (tid < nv) S.coloff[tid] = e2;
    if (tid == 0) {
      S.rowoff[nu] = hist[192] & 0xFFFFF; S.jbefore[nu] = hist[192] >> 20;
      S.tilebase[TTc] = hist[193];
    }
    __syncthreads();
  } else {
    const int rtot = block_scan_chunks(
        nu, ws, [&](int a) { return S.rowcnt[a] | ((S.hj[a] & 1) << 20); },
        [&](int a, int ex) { S.rowoff[a] = ex & 0xFFFFF; S.jbefore[a] = ex >> 20; });
    if (tid == 0) { S.rowoff[nu] = rtot & 0xFFFFF; S.jbefore[nu] = rtot >> 20; }
    const int ttot = block_scan_chunks(
        TTc, ws, [&](int t) { return S.tilebase[t]; }, [&](int t, int ex) { S.tilebase[t] = ex; });
    if (tid == 0) S.tilebase[TTc] = ttot;
    for (int b = tid; b < nv; b += nt) item_list(S, b, R, words);
    __syncthreads();
    block_scan_chunks(nv, ws, [&](int b) { return S.colcnt[b]; }, [&](int b, int ex) { S.coloff[b] = ex; });
  }
  const int m = S.rowoff[nu];
  // publish this graph's counts, then sum the predecessors' (they run at the same time; lower block ids are
  // dispatched first, so waiting on them cannot deadlock)
  if (tid == 0) {
    W.n_u[g] = nu; W.n_v[g] = nv; W.m_cnt[g] = m;
    __threadfence();
    st_release_gpu(&flags[g], 1);
  }
  const int2 base = graph_bases(g, ws, [&](int q) {
    while (ld_acquire_gpu(&flags[q]) == 0) {}
    return make_int2(__ldcg(W.n_u + q) + __ldcg(W.n_v + q), __ldcg(W.m_cnt + q));
  });
  const int Nbase = base.x, Mbase = base.y;
  bool fits = batch_offsets(O, g, B, Nbase, n, 2 * Mbase, 2 * m, err);
  if (fits && (T > FX_TCAP || m > slot_e)) {   // the tile table (reported above) or the scratch slot overflowed
    if (tid == 0) igmc_set_err(err, IGMC_ERR_EDGE_CAP);
    fits = false;
  }
  if (fits) {
    // ---- D: outputs ----
    if (tid == 0) { O.y[g] = class_values[lab]; O.graph_nu[g] = nu; }
    for (int t = tid; t < n; t += nt) {
      const int label = t < nu ? (t == 0 ? 0 : 2) : (t == nu ? 1 : 3);   // ref :245 with h = 1
      const size_t row = (size_t)Nbase + t;
      store_node(O, row, label, g, t < nu ? gu[t] : gv[t - nu]);
      O.adj_in_ptr[row] = t < nu ? 2 * Mbase + S.rowoff[t] : 2 * Mbase + m + S.coloff[t - nu];
    }
    // canonical (row-major, target item first) order: in shared memory, or (large subgraphs) in the upper half of
    // the scratch slot, read back past L1
    const bool cs = m <= FX_CANO;
    uint32_t* cano = cs ? S.cano : stage + slot_e;
    auto cld = [&](int q) -> uint32_t { return cs ? S.cano[q] : __ldcg(stage + slot_e + q); };
    int64_t* ei0 = O.edge_index;
    int64_t* ei1 = O.edge_index + O.edge_cap;
    auto emit = [&](uint32_t w, int pos) {
      cano[pos] = w;
      const int a = (int)(w >> 20), b = (int)((w >> 8) & 0xFFFu);
      const int64_t r = (int64_t)(w & 0xFFu);
      const size_t e1 = (size_t)2 * Mbase + pos, e2 = e1 + m;
      const int64_t un = Nbase + a, vn = Nbase + nu + b;
      ei0[e1] = un; ei1[e1] = vn; O.edge_type[e1] = r;
      ei0[e2] = vn; ei1[e2] = un; O.edge_type[e2] = r;
    };
    for (int tile = warp; tile < T; tile += nwarps) {
      const int base = S.tilebase[tile], cnt = S.tilebase[tile + 1] - base, so = S.stage_off[tile];
      for (int k = lane; k < cnt; k += 32) {
        const uint32_t w = __ldcg(stage + so + k);
        const int a = (int)(w >> 20);
        emit(w, base + k + S.jbefore[a] + (S.hj[a] & 1));
      }
    }
    for (int a = tid; a < nu; a += nt)
      if (S.hj[a] & 1) emit(((uint32_t)a << 20) | (uint32_t)(S.hj[a] >> 8), S.rowoff[a]);
    __syncthreads();
    // user lists: the row's run of the canonical order, stably split by rating (lane r keeps rating r's counter)
    for (int a = warp; a < nu; a += nwarps) {
      const int ro = S.rowoff[a], cnt = S.rowoff[a + 1] - ro;
      int tc = 0;
      for (int c0 = 0; c0 < cnt; c0 += 32) {
        const int k = c0 + lane;
        const int r = k < cnt ? (int)(cld(ro + k) & 0xFFu) : -1;
        for (int t = 0; t < R; ++t) {
          const unsigned mk = __ballot_sync(IGMC_FULL, r == t);
          if (lane == t) tc += __popc(mk);
        }
      }
      int run = warp_incl_scan_i(tc, lane) - tc;   // first slot of rating `lane`
      const size_t beg = (size_t)2 * Mbase + ro;
      for (int c0 = 0; c0 < cnt; c0 += 32) {
        const int k = c0 + lane;
        const uint32_t w = k < cnt ? cld(ro + k) : 0u;
        const int r = k < cnt ? (int)(w & 0xFFu) : -1;
        int slot = 0;
        for (int t = 0; t < R; ++t) {
          const unsigned mk = __ballot_sync(IGMC_FULL, r == t);
          const int rt = __shfl_sync(IGMC_FULL, run, t);
          if (r == t) slot = rt + __popc(mk & lt_mask);
          if (lane == t) run += __popc(mk);
        }
        if (k < cnt) {
          O.adj_in[beg + slot] = (uint32_t)(nu + (int)((w >> 8) & 0xFFFu)) | ((uint32_t)r << 16);
          O.adj_eid[beg + slot] = 2 * Mbase + m + ro + k;          // the mirrored (item -> user) directed edge
        }
      }
    }
    // item lists: position = rating sub-list offset + number of earlier user rows holding the same (item, rating)
    for (int k = tid; k < m; k += nt) {
      const uint32_t w = cld(k);
      const int a = (int)(w >> 20), b = (int)((w >> 8) & 0xFFFu), r = (int)(w & 0xFFu);
      const uint32_t* bw = S.bm + ((size_t)b * R + r) * words;
      int rank = __popc(bw[a >> 5] & ((1u << (a & 31)) - 1u));
      for (int x = 0; x < (a >> 5); ++x) rank += __popc(bw[x]);
      const size_t o = (size_t)2 * Mbase + m + S.coloff[b] + S.cur[b * R + r] + rank;
      O.adj_in[o] = (uint32_t)a | ((uint32_t)r << 16);
      O.adj_eid[o] = 2 * Mbase + k;
    }
  }
  // the last CTA to finish re-arms the flags for the next launch
  __syncthreads();
  if (tid == 0) {
    if (W.hop_off) W.hop_off[(size_t)g * 2 * (IGMC_MAX_HOP + 1) + 6] = (int)(igmc_globaltimer() & 0x7fffffff);
    __threadfence();
    if (atomicAdd(&flags[B], 1) == B - 1) {
      for (int q = 0; q <= B; ++q) flags[q] = 0;
    }
  }
}

// Batch assembly from the static store (one CTA per output graph).
__global__ void __launch_bounds__(256)
k_assemble(igmc_store_t S, const int64_t* __restrict__ idx, int B, igmc_batch_out_t O, int* err) {
  __shared__ int ws[34];
  const int g = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int2 base = graph_bases(g, ws, [&](int q) {
    const int64_t s = idx[q];
    return make_int2(S.node_off[s + 1] - S.node_off[s], S.edge_off[s + 1] - S.edge_off[s]);
  });
  const int Nbase = base.x, Ebase = base.y;
  const int64_t s = idx[g];
  const int n0 = S.node_off[s], n = S.node_off[s + 1] - n0;
  const int e0 = S.edge_off[s], e = S.edge_off[s + 1] - e0;
  if (!batch_offsets(O, g, B, Nbase, n, Ebase, e, err)) return;
  if (tid == 0) { O.y[g] = S.y[s]; O.graph_nu[g] = S.graph_nu[s]; }
  const int32_t* aptr = S.adj_ptr + n0 + s;   // per graph n+1 entries -> offset n0 + s
  for (int t = tid; t < n; t += nt) {
    const size_t row = (size_t)Nbase + t;
    store_node(O, row, S.node_label[n0 + t], g, S.node_gid[n0 + t]);
    if (O.adj_in_ptr) O.adj_in_ptr[row] = Ebase + aptr[t];
  }
  int64_t* ei0 = O.edge_index;
  int64_t* ei1 = O.edge_index + O.edge_cap;
  for (int t = tid; t < e; t += nt) {
    const size_t k = (size_t)Ebase + t;
    ei0[k] = (int64_t)Nbase + S.edge_src[e0 + t];
    ei1[k] = (int64_t)Nbase + S.edge_dst[e0 + t];
    O.edge_type[k] = S.edge_type[e0 + t];
    if (O.adj_in_ptr) {
      O.adj_in[k] = S.adj_in[e0 + t];
      O.adj_eid[k] = Ebase + S.adj_eid[e0 + t];
    }
  }
}

}  // namespace

namespace {

// h = 1 fast path (one launch) whenever its tables fit: ids in 12 bits, <= 32 rating classes, the user rows of one
// subgraph within the tile table, two CTAs per SM worth of shared memory, scratch slot >= the edge bound.  `fast`: the
// workspace has the one-launch flags; `adjacency`: the batch wants the message-passing lists.  Returns the dynamic
// shared memory of k_extract_fast, 0 when the batch takes the generic path.
size_t fast_smem(int num_items, int B, int h, int cap, int num_classes, int max_row_deg, int edge_cap, bool fast,
                 bool adjacency) {
  static int fast_env = -1;
  if (fast_env < 0) {
    const char* e = getenv("IGMC_EXTRACT_FAST");
    fast_env = e ? atoi(e) : 1;
  }
  const int R = num_classes;
  const int words = (cap + 31) / 32;
  const int slot_e = edge_cap / B;
  const size_t smemF = fast_smem_ints(cap, R > 0 ? R : 1, words) * 4 + (((size_t)num_items * 2 + 15) & ~(size_t)15);
  const long long rows_max = (long long)cap * (long long)(max_row_deg > 0 ? max_row_deg : num_items);
  if (fast_env && h == 1 && fast && adjacency && R >= 1 && R <= FX_MAXR && cap <= FX_MAXCAP &&
      rows_max <= (long long)FX_TILE * FX_TCAP && smemF <= 110 * 1024 && slot_e >= 2)
    return smemF;
  return 0;
}

// generic two-kernel path (any hop count / capacity): 1024-thread CTAs - the kernels are latency-bound, and more
// threads per subgraph keep more independent loads in flight.
int generic_threads() {
  static int ex_threads = 0;
  if (!ex_threads) {
    const char* e = getenv("IGMC_EX_THREADS");
    ex_threads = e ? atoi(e) : 1024;
    if (ex_threads != 256 && ex_threads != 512 && ex_threads != 1024) ex_threads = 1024;
  }
  return ex_threads;
}

// the dynamic shared memory of the two generic kernels; false when the item table or the bitmaps do not fit
bool generic_smem(int num_users, int num_items, int h, int cap, size_t* smemA, size_t* smemB) {
  size_t a = (size_t)cap * sizeof(int) + (size_t)num_items * sizeof(uint16_t);
  if (h > 1) {   // visited / candidate bitmaps + the fringe list of the larger side
    const size_t wu = (num_users + 31) / 32, wv = (num_items + 31) / 32;
    a = ((a + 15) & ~(size_t)15) + (wu + wv + (wu > wv ? wu : wv)) * 4 +
        (size_t)(num_users > num_items ? num_users : num_items) * 4;
    if (a > 220 * 1024) return false;
  }
  *smemA = a;
  *smemB = 2 * (size_t)cap * sizeof(int) + (size_t)num_items * sizeof(uint16_t);
  return *smemB <= 220 * 1024;   // else the item table does not fit in shared memory
}

// The path a batch takes, decided once for igmc_extract_batch, igmc_extract_sessions and igmc_extract_plan.
struct ExtractPlan {
  size_t fast;           // dynamic shared memory of k_extract_fast, 0: the generic kernels
  size_t smemA, smemB;   // dynamic shared memory of the two generic kernels
  bool ok;               // false: neither path fits
};
ExtractPlan extract_plan(int num_users, int num_items, int B, int h, int cap, int num_classes, int max_row_deg,
                         int edge_cap, bool fast, bool adjacency) {
  ExtractPlan p = {fast_smem(num_items, B, h, cap, num_classes, max_row_deg, edge_cap, fast, adjacency), 0, 0, true};
  if (!p.fast) p.ok = generic_smem(num_users, num_items, h, cap, &p.smemA, &p.smemB);
  return p;
}

// The arguments of igmc_extract_batch and igmc_extract_sessions.  The kernels take them one by one: as one struct
// parameter (no __restrict__, sizes read from the struct) nvcc generates slower code, k_extract_fill ~9 % and the
// session k_extract_fast ~5 % slower on an H100 80GB HBM3 at 700 W.
struct ExtractArgs {
  igmc_csr_t G;
  igmc_pairs_t P;
  int B, h, mnph, cap;
  double ratio;
  uint64_t seed_val;
  const uint64_t* seed_dev;   // device word overriding seed_val, or null
  const int32_t *inj_nodes_u, *inj_nodes_v, *inj_n_u, *inj_n_v;   // test hook (plain mode): injected node lists
  igmc_extract_ws_t W;
  const float* class_values;
  int R;                      // rating classes
  igmc_batch_out_t O;
  int* err;
  SessArg A;                  // session mode only
};

// The launch behind both entries: the plan, then k_extract_fast or the two generic kernels.
template <bool SESS>
int launch_extract(const ExtractArgs& X, int max_row_deg, cudaStream_t st) {
  const ExtractPlan pl = extract_plan(X.G.num_users, X.G.num_items, X.B, X.h, X.cap, X.R, max_row_deg, X.O.edge_cap,
                                      X.W.sync != nullptr, X.O.adj_in_ptr != nullptr);
  const igmc_extract_ws_t& W = X.W;
  if (pl.fast) {
    cudaFuncSetAttribute(k_extract_fast<SESS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.fast);
    k_extract_fast<SESS><<<X.B, FX_THREADS, pl.fast, st>>>(
        X.G, X.P, X.B, X.mnph, X.ratio, X.seed_val, X.seed_dev, X.cap, X.inj_nodes_u, X.inj_nodes_v, X.inj_n_u,
        X.inj_n_v, W, X.R, (X.cap + 31) / 32, X.O.edge_cap / X.B, X.class_values, X.O, X.err, X.A);
    IGMC_CUDA_CHECK_LAUNCH();
    return 0;
  }
  if (!pl.ok) return -3;
  const int threads = generic_threads();
  cudaFuncSetAttribute(k_extract_select_count<SESS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smemA);
  cudaFuncSetAttribute(k_extract_fill<SESS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smemB);
  k_extract_select_count<SESS><<<X.B, threads, pl.smemA, st>>>(
      X.G, X.P, X.B, X.mnph, X.ratio, X.seed_val, X.seed_dev, X.cap, X.inj_nodes_u, X.inj_nodes_v, X.inj_n_u,
      X.inj_n_v, W.nodes_u, W.nodes_v, W.n_u, W.n_v, W.row_cnt, W.m_cnt, W.col_cnt, X.h, W.hop_off, X.err, X.A);
  IGMC_CUDA_CHECK_LAUNCH();
  k_extract_fill<SESS><<<X.B, threads, pl.smemB, st>>>(X.G, X.P, X.B, X.cap, W.nodes_u, W.nodes_v, W.n_u, W.n_v,
                                                        W.row_cnt, W.m_cnt, W.col_cnt, X.h, W.hop_off, X.class_values,
                                                        X.R, X.O, X.err, X.A);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}

}  // namespace

extern "C" int igmc_extract_plan(int num_users, int num_items, int B, int h, int cap, int num_classes,
                                 int max_row_deg, int edge_cap, int fast, int adjacency) {
  if (B <= 0) return 0;
  if (cap < 1 || cap > 65534) return -2;
  if (h < 1 || h > IGMC_MAX_HOP) return -4;
  const ExtractPlan p = extract_plan(num_users, num_items, B, h, cap, num_classes, max_row_deg, edge_cap, fast != 0,
                                     adjacency != 0);
  return p.fast ? (int)p.fast : p.ok ? 0 : -3;
}

extern "C" int igmc_extract_batch(const igmc_csr_t* G, const igmc_pairs_t* P, int B, int h, int max_nodes_per_hop,
                                  double sample_ratio, uint64_t seed, const uint64_t* seed_dev, int cap,
                                  const int32_t* inj_nodes_u, const int32_t* inj_nodes_v,
                                  const int32_t* inj_n_u, const int32_t* inj_n_v,
                                  const igmc_extract_ws_t* W, const float* class_values, int num_classes,
                                  int max_row_deg, const igmc_batch_out_t* O, int* err, void* stream) {
  if (B <= 0) return 0;
  if (cap < 1 || cap > 65534) return -2;
  if (h < 1 || h > IGMC_MAX_HOP) return -4;
  if (h > 1 && (inj_nodes_u || !W->hop_off)) return -4;   // injected node lists carry no hop boundaries
  const ExtractArgs X = {*G, *P, B, h, max_nodes_per_hop, cap, sample_ratio, seed, seed_dev,
                         inj_nodes_u, inj_nodes_v, inj_n_u, inj_n_v, *W, class_values, num_classes, *O, err, {}};
  return launch_extract<false>(X, max_row_deg, (cudaStream_t)stream);
}

extern "C" int igmc_extract_sessions(const igmc_csr_t* G, const igmc_sessions_t* S, const int32_t* sess,
                                     const igmc_pairs_t* P, int B, int h, int max_nodes_per_hop, double sample_ratio,
                                     uint64_t seed, const uint64_t* seed_dev, int cap, const igmc_extract_ws_t* W,
                                     const float* class_values, int num_classes, int max_row_deg,
                                     const igmc_batch_out_t* O, int* err, void* stream) {
  if (B <= 0) return 0;
  if (!S || !S->users || !S->row_ptr || !sess) return -1;
  if (cap < 1 || cap > 65534) return -2;
  if (h < 1 || h > IGMC_MAX_HOP) return -4;
  if (h > 1 && !W->hop_off) return -4;
  const ExtractArgs X = {*G, *P, B, h, max_nodes_per_hop, cap, sample_ratio, seed, seed_dev,
                         nullptr, nullptr, nullptr, nullptr, *W, class_values, num_classes, *O, err, {*S, sess}};
  return launch_extract<true>(X, max_row_deg, (cudaStream_t)stream);
}

extern "C" int igmc_assemble_batch(const igmc_store_t* S, const int64_t* idx, int B, const igmc_batch_out_t* O, int* err,
                                   void* stream) {
  if (B <= 0) return 0;
  k_assemble<<<B, 256, 0, (cudaStream_t)stream>>>(*S, idx, B, *O, err);
  IGMC_CUDA_CHECK_LAUNCH();
  return 0;
}
