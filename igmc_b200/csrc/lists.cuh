// Edge-list walking shared by the basis-space kernels (csrc/rgcn.cu, csrc/rgcn_l2.cu): the step's edge-dropout
// draws and a warp-wide walk over one node's (type, neighbour)-sorted list.
#pragma once
#include "common.cuh"
#include "../../include/igmc_b200.h"

namespace {

constexpr uint32_t DROPPED = 0xFFFFFFFFu;

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
  double t = (double)D.adj_dropout * 4294967296.0;
  K.thresh = t >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)t;
  return K;
}

// Walks list [p0,p1) of one node with the whole warp; body(nbr, type) is called warp-uniformly for
// every kept entry, in list order.  `mirror`: the entry describes edge nbr->x but the caller wants
// the reverse edge x->nbr of a symmetric batch, whose id is the mirror image inside the graph.
template <class Body>
__device__ __forceinline__ int list_foreach(const uint32_t* __restrict__ adj, const int32_t* __restrict__ eid,
                                            int p0, int p1, const EdgeKeep& K, bool mirror, int eb, int m_half,
                                            int lane, Body&& body) {
  int kept = 0;
  for (int c = p0; c < p1; c += 32) {
    const int p = c + lane;
    uint32_t ent = DROPPED;
    if (p < p1) {
      ent = adj[p];
      if (K.active) {
        int e = eid[p];
        if (mirror) { const int el = e - eb; e = eb + (el < m_half ? el + m_half : el - m_half); }
        if (!K.keep(e)) ent = DROPPED;
      }
    }
    const int cnt = min(32, p1 - c);
    for (int q = 0; q < cnt; ++q) {
      const uint32_t en = __shfl_sync(IGMC_FULL, ent, q);
      if (en == DROPPED) continue;
      ++kept;
      body((int)(en & 0xffffu), (int)((en >> 16) & 0xffu));
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

}  // namespace
