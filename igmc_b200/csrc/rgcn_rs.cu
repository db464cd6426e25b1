// v2 fused relational message passing: relation-space aggregate + dense transform, one thread-block
// CLUSTER per enclosing subgraph (1/2/4 CTAs split the destination nodes), up to 32 warps per CTA.
//
// Same math and C-ABI as csrc/rgcn.cu (which stays as the generic path for many relations); this is the
// fast path for num_relations <= RS_MAX_R.  Per layer (reference: tanh(RGCNConv) models.py:200-202,
// PyG 1.4.2 semantics SURVEY.md A.1), with W_r = sum_b att[r,b] basis[b] formed once per CTA in shared memory:
//   AGG[v,r,:] = sum_{(u->v) of type r, kept} h[u,:]      warp owns 4 destination nodes; 8-lane groups x float4,
//                                                          edge lists staged in shared memory, software-pipelined
//   h'[v]      = tanh( 1/deg(v) * sum_r AGG[v,r,:] W_r + h[v] root + bias )    lane = (node, 4 output channels)
// PR = true (PyG >= 1.6 RGCNConv, igmc_saved_t.rel_inv_deg): 1/|N_r(v)| per relation block in place of 1/deg(v).
// Node features of the WHOLE subgraph stay in shared memory; CTAs of a cluster store their rows of every layer into
// each other's shared memory with st.async, counted on the receiver's mbarrier.  Backward = same two passes on the
// out-lists with W_r^T,
// a K=n weight-gradient tile GEMM, and the (att,basis) chain rule applied to the per-CTA dW_r.
// No float atomics; every reduction has a fixed order (bitwise run-to-run deterministic).
#include <cooperative_groups.h>
#include <cstdlib>

#include "lists.cuh"

namespace cg = cooperative_groups;

namespace rs {

constexpr int HID = IGMC_HIDDEN;
constexpr int L1O = IGMC_LIN1_OUT;
constexpr int RS_MAX_R = 12;
constexpr int GN = 4;          // destination nodes per warp group (one 8-lane group each)
constexpr int TW = 32;         // node tile of the weight-gradient GEMM
constexpr int WP = 33;         // padded row stride of the transposition scratch

// entry of list position p, DROPPED if the (possibly mirrored) edge is dropped this step
__device__ __forceinline__ uint32_t load_entry(const uint32_t* __restrict__ adj, const int32_t* __restrict__ eid,
                                               int p, const EdgeKeep& K, bool mirror, int eb, int m_half) {
  uint32_t ent = __ldg(adj + p);
  if (K.active) {
    int e = __ldg(eid + p);
    if (mirror) { const int el = e - eb; e = eb + (el < m_half ? el + m_half : el - m_half); }
    if (!K.keep(e)) ent = DROPPED;
  }
  return ent;
}

// Edge lists of the own nodes [lo,hi): staged once per kernel in shared memory (dropped edges compacted out)
// and cut into SEGMENTS of at most SEG edges.  A segment is the unit of gather work of one 8-lane group and owns
// one staging row: the first segment of a node writes the node's row, further segments of a long list (the two
// target nodes are adjacent to every other node of their subgraph) write extra rows behind the chunk's node rows,
// which are then summed into the node row in segment order.  This bounds the gather critical path by SEG edges.
constexpr int SEG = 32;        // edges per segment
constexpr int XR = 16;         // extra staging rows per chunk
constexpr int XCH = 8;         // chunks that may use extra rows

// staged list entry: type << 24 | RUN_END | swizzled float offset of the neighbour's feature row
// ((nbr << 5) | ((nbr & 7) << 2), below 2^21), so that the edge loop gets a lane's address with one LOP3
// ((entry & ENT_OFF) ^ column) instead of re-deriving the swizzle.  RUN_END marks the last entry of a type run within
// its segment (set by stage_lists once the segments are known).
constexpr uint32_t ENT_OFF = 0x1fffffu;
constexpr uint32_t RUN_END = 1u << 21;
// seg_row of a staged segment: staging row | types present in the segment << 16 (rows are below 2^16, R <= 12)
constexpr int SEG_ROW = 0xffff;
__device__ __forceinline__ uint32_t enc_entry(uint32_t ent) {
  const uint32_t nbr = ent & 0xffffu;
  return ((ent >> 16) << 24) | (nbr << 5) | ((nbr & 7u) << 2);
}

struct Lists {
  const uint32_t* lst;   // staged entries (nullptr: not staged -> adj/eid are read per edge)
  const int* lptr;       // [n_own+1] list offsets (into lst when staged, else absolute positions in adj)
  const int* segbase;    // [n_own+1] first segment of every node
  const int* seg_p0;     // per segment: list range and staging row (relative to its chunk)
  const int* seg_p1;
  const int* seg_row;
  const int* seg_ord;    // segments of every chunk in order of decreasing length (the order they are handed out in)
  const int* ex;         // per node: first extra row (relative to crow) | number of extra segments << 16
  const uint32_t* adj;   // global fallback
  const int32_t* eid;
  bool mirror;
  int eb, m_half;
};

__host__ __device__ __forceinline__ int list_ints(int own_cap) { return 3 * (own_cap + 4) + 4 * (own_cap + XR * XCH); }
// A list image = IMG_HDR header ints (entries, segments, staged flag, own nodes) directly followed by the tables
// above.  Built either by the kernel itself (stage_lists) or once per batch by k_stage_lists (igmc_stage_lists), in
// which case the model kernels pull it into shared memory with bulk (TMA) copies.
constexpr int IMG_HDR = 4;
__host__ __device__ __forceinline__ int img_ints(int own_cap) { return IMG_HDR + ((list_ints(own_cap) + 3) & ~3); }

// pointers into a table block `ibuf` (the header sits at ibuf - IMG_HDR)
__device__ __forceinline__ Lists lists_view(int* ibuf, int own_cap, const uint32_t* lbuf, const uint32_t* adj,
                                            const int32_t* eid, bool mirror, int eb, int m_half) {
  Lists Ls;
  Ls.lptr = ibuf;
  Ls.segbase = ibuf + (own_cap + 4);
  Ls.ex = Ls.segbase + (own_cap + 4);
  Ls.seg_p0 = Ls.ex + (own_cap + 4);
  Ls.seg_p1 = Ls.seg_p0 + (own_cap + XR * XCH);
  Ls.seg_row = Ls.seg_p1 + (own_cap + XR * XCH);
  Ls.seg_ord = Ls.seg_row + (own_cap + XR * XCH);
  Ls.adj = adj; Ls.eid = eid; Ls.mirror = mirror; Ls.eb = eb; Ls.m_half = m_half;
  Ls.lst = ibuf[2 - IMG_HDR] ? lbuf : nullptr;
  return Ls;
}

// Block-wide; ends with a barrier.  `ibuf` has list_ints(own_cap) ints and is preceded by the IMG_HDR header ints
// (written here too).  invdeg_out/invdeg_glob (each optional) get 1/max(kept degree,1) of the own nodes.
__device__ __forceinline__ Lists stage_lists(const uint32_t* adj, const int32_t* eid, const int32_t* ptr, int nb, int lo,
                                             int hi, const EdgeKeep& K, bool mirror, int eb, int m_half, uint32_t* lbuf,
                                             int lcap, int* ibuf, int own_cap, int chunk, int* ws, float* invdeg_out,
                                             float* invdeg_glob) {
  const int tid = threadIdx.x, NT = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarps = NT >> 5;
  const int n_own = hi - lo;
  int* lptr = ibuf;
  int* segbase = lptr + (own_cap + 4);
  int* ex = segbase + (own_cap + 4);
  int* seg_p0 = ex + (own_cap + 4);
  int* seg_p1 = seg_p0 + (own_cap + XR * XCH);
  int* seg_row = seg_p1 + (own_cap + XR * XCH);
  int* seg_ord = seg_row + (own_cap + XR * XCH);
  Lists Ls;
  Ls.seg_ord = seg_ord;
  Ls.adj = adj; Ls.eid = eid; Ls.mirror = mirror; Ls.eb = eb; Ls.m_half = m_half;
  Ls.lptr = lptr; Ls.segbase = segbase; Ls.ex = ex; Ls.seg_p0 = seg_p0; Ls.seg_p1 = seg_p1; Ls.seg_row = seg_row;
  // ---- pass 1: kept entries per node ----
  if (K.active) {
    for (int i = warp; i < n_own; i += nwarps) {
      const int p0 = ptr[nb + lo + i], p1 = ptr[nb + lo + i + 1];
      int kept = 0;
      for (int p = p0 + lane; p < p1; p += 32) kept += load_entry(adj, eid, p, K, mirror, eb, m_half) != DROPPED;
      kept = warp_sum_i(kept);
      if (lane == 0) lptr[i + 1] = kept;
    }
  } else {
    for (int i = tid; i < n_own; i += NT) lptr[i + 1] = ptr[nb + lo + i + 1] - ptr[nb + lo + i];
  }
  if (tid == 0) lptr[0] = 0;
  __syncthreads();
  if (invdeg_out || invdeg_glob)
    for (int i = tid; i < n_own; i += NT) {
      const float id = 1.f / (float)max(lptr[i + 1], 1);
      if (invdeg_out) invdeg_out[lo + i] = id;
      if (invdeg_glob) invdeg_glob[nb + lo + i] = id;
    }
  // ---- segments per node (uncapped) and their prefix sums: offsets | extras << 16 ----
  int run_off = 0, run_ex = 0;
  for (int base = 0; base < n_own; base += NT) {
    const int i = base + tid;
    const int d = i < n_own ? lptr[i + 1] : 0;
    const int extras = i < n_own ? max(0, (d + SEG - 1) / SEG - 1) : 0;
    int tot_d, tot_e;
    const int ex_d = block_excl_scan_i(d, ws, &tot_d);
    const int ex_e = block_excl_scan_i(extras, ws, &tot_e);
    if (i < n_own) {
      segbase[i] = extras;                 // temporarily: uncapped extras
      ex[i] = run_ex + ex_e;               // temporarily: exclusive prefix of the uncapped extras
      lptr[i + 1] = run_off + ex_d + d;    // end offset of node i
    }
    run_off += tot_d;
    run_ex += tot_e;
  }
  __syncthreads();
  const int total = n_own > 0 ? lptr[n_own] : 0;
  const bool staged = total <= lcap;
  Ls.lst = staged ? lbuf : nullptr;
  // ---- cap the extra segments of every chunk at XR, second prefix sum for the segment ids ----
  int run_seg = 0;
  for (int base = 0; base < n_own; base += NT) {
    const int i = base + tid;
    int nseg = 0, x = 0;
    if (i < n_own) {
      const int ci = i / chunk, cfirst = ci * chunk;
      x = ex[i] - ex[cfirst];
      const int allowed = ci < XCH ? max(0, min(segbase[i], XR - x)) : 0;
      nseg = 1 + allowed;
    }
    int tot;
    const int exs = block_excl_scan_i(nseg, ws, &tot);
    __syncthreads();                       // every thread has read ex[] / segbase[] of this round
    if (i < n_own) {
      const int ci = i / chunk, c0 = ci * chunk, crow = min(chunk, n_own - c0);
      const int sb = run_seg + exs;
      // list offsets: staged lists are compacted (offset 0 = first own entry); unstaged use absolute positions
      const int l0 = staged ? lptr[i] : ptr[nb + lo + i];
      const int l1 = staged ? lptr[i + 1] : ptr[nb + lo + i + 1];
      for (int j = 0; j < nseg; ++j) {
        seg_p0[sb + j] = l0 + j * SEG;
        seg_p1[sb + j] = (j == nseg - 1) ? l1 : l0 + (j + 1) * SEG;
        seg_row[sb + j] = j == 0 ? (i - c0) : (crow + x + j - 1);
      }
      ex[i] = x | ((nseg - 1) << 16);
      segbase[i] = sb;
    }
    run_seg += tot;
    __syncthreads();
  }
  if (tid == 0) {
    segbase[n_own] = run_seg;
    int* hdr = ibuf - IMG_HDR;
    hdr[0] = total; hdr[1] = run_seg; hdr[2] = staged ? 1 : 0; hdr[3] = n_own;
  }
  // ---- pass 2: compacted copy of the entries ----
  if (staged) {
    if (K.active) {
      for (int i = warp; i < n_own; i += nwarps) {
        const int p0 = ptr[nb + lo + i], p1 = ptr[nb + lo + i + 1];
        int o = lptr[i];
        for (int c = p0; c < p1; c += 32) {
          const int p = c + lane;
          uint32_t ent = DROPPED;
          if (p < p1) ent = load_entry(adj, eid, p, K, mirror, eb, m_half);
          const unsigned bal = __ballot_sync(IGMC_FULL, ent != DROPPED);
          if (ent != DROPPED) lbuf[o + __popc(bal & ((1u << lane) - 1u))] = enc_entry(ent);
          o += __popc(bal);
        }
      }
    } else {
      const int e_lo = ptr[nb + lo];
      for (int i = tid; i < total; i += NT) lbuf[i] = enc_entry(__ldg(adj + e_lo + i));
    }
  }
  __syncthreads();
  // run structure of the staged segments (warp per segment): lists are sorted by (type, neighbour), so every type
  // is at most one run of a segment; its last entry gets RUN_END and the segment's row its type mask
  if (staged) {
    const int nseg = segbase[n_own];
    for (int sg = warp; sg < nseg; sg += nwarps) {
      const int p0 = seg_p0[sg], p1 = seg_p1[sg];
      uint32_t types = 0;
      for (int c = p0; c < p1; c += 32) {
        const int p = c + lane;
        const uint32_t e = p < p1 ? lbuf[p] : 0u, en = p + 1 < p1 ? lbuf[p + 1] : 0u;
        __syncwarp();   // every lane has read its successor before any flag is written
        if (p < p1) {
          types |= 1u << (e >> 24);
          if (p + 1 == p1 || (en >> 24) != (e >> 24)) lbuf[p] = e | RUN_END;
        }
      }
      types = __reduce_or_sync(IGMC_FULL, types);
      if (lane == 0) seg_row[sg] |= (int)(types << 16);
    }
  }
  // hand-out order: within every chunk, segments by decreasing length (rank sort, ties by index)
  {
    const int nseg = segbase[n_own];
    for (int sg = tid; sg < nseg; sg += NT) {
      int c0 = 0;
      while (c0 + chunk < n_own && segbase[c0 + chunk] <= sg) c0 += chunk;
      const int s0 = segbase[c0], s1 = segbase[min(c0 + chunk, n_own)];
      const int len = seg_p1[sg] - seg_p0[sg];
      int rank = 0;
      for (int t = s0; t < s1; ++t) {
        const int lt = seg_p1[t] - seg_p0[t];
        rank += (lt > len) || (lt == len && t < sg);
      }
      seg_ord[s0 + rank] = sg;
    }
  }
  __syncthreads();
  return Ls;
}

__device__ __forceinline__ float4 scale_row(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }

// Mean per relation (igmc_saved_t.rel_inv_deg): out[v*R + r] = 1/max(kept in-edges of type r at v, 1) for the own
// nodes v = lo + i, counted from the staged (compacted) in-lists, or from the global lists when they are not staged.
// Warp per node, lane r counts type r (R <= RS_MAX_R < 32).  Block-wide; the caller's next barrier publishes it.
__device__ __forceinline__ void rel_inv_deg_own(const Lists& Ls, const EdgeKeep& K, const int32_t* __restrict__ in_ptr,
                                                int nb, int lo, int n_own, int R, float* __restrict__ out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int i = warp; i < n_own; i += nwarps) {
    const int p0 = Ls.lst ? Ls.lptr[i] : in_ptr[nb + lo + i], p1 = Ls.lst ? Ls.lptr[i + 1] : in_ptr[nb + lo + i + 1];
    int cnt = 0;
    for (int c = p0; c < p1; c += 32) {
      const int p = c + lane;
      int ty = -1;
      if (p < p1) {
        if (Ls.lst) {
          ty = (int)(Ls.lst[p] >> 24);
        } else {
          const uint32_t e = load_entry(Ls.adj, Ls.eid, p, K, false, Ls.eb, Ls.m_half);
          if (e != DROPPED) ty = (int)((e >> 16) & 0xffu);
        }
      }
      for (int r = 0; r < R; ++r) {
        const int c_r = __popc(__ballot_sync(IGMC_FULL, ty == r));
        if (lane == r) cnt += c_r;
      }
    }
    if (lane < R) out[(size_t)(lo + i) * R + lane] = 1.f / (float)max(cnt, 1);
  }
}

// Relation-space aggregate of the segments [sg0, sg1) of one chunk into their staging rows
// stage[row][r*inp + k] (row stride SS): one 8-lane group per segment, float4 per lane.
// `K` is only consulted for unstaged lists (dropout draws evaluated per edge).
// Segments are handed out through a shared-memory ticket (`ticket`, zero on entry, reset by the caller after the
// barrier that follows) in order of decreasing length (Ls.seg_ord): the four groups of a warp run in lockstep, so
// segments of similar length taken at the same time keep their lanes busy (a warp-instruction of the edge loop had
// less than half of its lanes active with the node-order assignment).  Which group computes a segment does
// not change its result (own staging row, fixed summation order): the output stays bitwise deterministic.
// GL = lanes per segment (one float4 each): 8 for the 32-wide layers; 1 for a 4-wide input layer (one-hot labels) -
// there seven of the eight lanes of a group had nothing to do, now a warp works on 32 segments at a time.
// PR (backward of the mean per relation): every entry (nbr, type r) is weighed by rinv[nbr*R + r] = 1/|N_r(nbr)|,
// read through L2 (the table is written by the forward, possibly by a peer CTA of the same launch).
// RS (forward, staged lists): the run store of a node row whose list is one segment is scaled by the node's degree
// factor, so that the fold pass only visits rows with extra segments.  The product is the one the fold computed
// (run sum times the factor, both rounded once); zeroed blocks stay +0.  RS = 1: 1/deg of the segment's row
// (RunScale::inv[row]), RS = 2 (mean per relation): 1/|N_r(v)| of the run's type r (RunScale::inv[row*R + r], L2).
// Every other row (extra rows, rows of nodes with extras, RunScale::inv == nullptr) is stored as summed.
struct RunScale {
  const float* inv;   // degree factors of the chunk's rows (nullptr: no scaling)
  const int* ex;      // Lists::ex of the chunk's rows
  int crow;           // node rows of the chunk (staging rows >= crow are extra rows)
};
template <int GL, bool PR = false, int RS = 0>
__device__ __forceinline__ void gather_segments(const Lists& Ls, const EdgeKeep& K, int sg0, int sg1, int lane,
                                                const float* __restrict__ feat, float* __restrict__ stage, int SS,
                                                int inp, int R, int* ticket, const float* rinv = nullptr,
                                                RunScale rsc = RunScale{nullptr, nullptr, 0}) {
  const int q = lane & (GL - 1);
  const int fo = 4 * q;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  for (;;) {
    int t = 0;
    if (lane == 0) t = atomicAdd(ticket, 32 / GL);   // 32 / GL consecutive segments (similar lengths) per warp
    t = sg0 + __shfl_sync(IGMC_FULL, t, 0) + lane / GL;
    const bool valid = t < sg1;
    if (!__any_sync(IGMC_FULL, valid)) break;
    const int sg = valid ? Ls.seg_ord[t] : 0;
    float* rowb = stage;
    int p = 0, p1 = 0;
    float sc = 1.f;                  // RS = 1: factor of every run of the segment
    const float* scp = nullptr;      // RS = 2: factors of the row's relation blocks
    if (valid) {
      const int sr = Ls.seg_row[sg];
      rowb = stage + (size_t)(sr & SEG_ROW) * SS;
      if (RS && rsc.inv) {
        const int row = sr & SEG_ROW;
        if (row < rsc.crow && (rsc.ex[row] >> 16) == 0) {
          if (RS == 1) sc = rsc.inv[row];
          else scp = rsc.inv + (size_t)row * R;
        }
      }
      if (Ls.lst) {
        // every type present gets one plain store of its run below: zero only the blocks of the other types (a
        // lane owns column fo of every block) and the padding behind the last block
        if (fo < inp)
          for (uint32_t m = ~((uint32_t)sr >> 16) & ((1u << R) - 1u); m; m &= m - 1u)
            *reinterpret_cast<float4*>(rowb + (__ffs(m) - 1) * inp + fo) = z4;
        for (int i = R * inp + fo; i < SS; i += 4 * GL) *reinterpret_cast<float4*>(rowb + i) = z4;
      } else {
        for (int i = fo; i < SS; i += 4 * GL) *reinterpret_cast<float4*>(rowb + i) = z4;
      }
      if (fo < inp) { p = Ls.seg_p0[sg]; p1 = Ls.seg_p1[sg]; }
    }
    __syncwarp();
    float* row = rowb + fo;
    if (Ls.lst) {
      // each type run is summed in registers from zero, in list order, and written with one plain store at its
      // RUN_END entry (the last entry of a segment always carries it): the row equals the zeroed row plus the run
      const uint32_t* lst = Ls.lst;
      float4 acc = z4;
#define IGMC_HROW(e_) (PR ? scale_row(*reinterpret_cast<const float4*>(feat + (((e_) & ENT_OFF) ^ (uint32_t)fo)), \
                                      __ldcg(rinv + (int)(((e_) & ENT_OFF) >> 5) * R + (int)((e_) >> 24)))       \
                         : *reinterpret_cast<const float4*>(feat + (((e_) & ENT_OFF) ^ (uint32_t)fo)))
#define IGMC_STEP(e_, a_)                                                                             \
      do {                                                                                            \
        acc.x = __fadd_rn(acc.x, (a_).x); acc.y = __fadd_rn(acc.y, (a_).y);                           \
        acc.z = __fadd_rn(acc.z, (a_).z); acc.w = __fadd_rn(acc.w, (a_).w);                           \
        if ((e_) & RUN_END) {                                                                         \
          if (RS) {                                                                                   \
            const float s_ = (RS == 2 && scp) ? __ldcg(scp + (int)((e_) >> 24)) : sc;                 \
            acc = make_float4(__fmul_rn(acc.x, s_), __fmul_rn(acc.y, s_), __fmul_rn(acc.z, s_),       \
                              __fmul_rn(acc.w, s_));                                                  \
          }                                                                                           \
          *reinterpret_cast<float4*>(row + (int)((e_) >> 24) * inp) = acc;                            \
          acc = z4;                                                                                   \
        }                                                                                             \
      } while (0)
      // four edges in flight: the entry and source-row loads of a batch are independent
      for (; p + 4 <= p1; p += 4) {
        const uint32_t e0 = lst[p], e1 = lst[p + 1], e2 = lst[p + 2], e3 = lst[p + 3];
        const float4 a0 = IGMC_HROW(e0), a1 = IGMC_HROW(e1), a2 = IGMC_HROW(e2), a3 = IGMC_HROW(e3);
        IGMC_STEP(e0, a0); IGMC_STEP(e1, a1); IGMC_STEP(e2, a2); IGMC_STEP(e3, a3);
      }
      for (; p < p1; ++p) {
        const uint32_t e0 = lst[p];
        const float4 a0 = IGMC_HROW(e0);
        IGMC_STEP(e0, a0);
      }
#undef IGMC_STEP
#undef IGMC_HROW
    } else {
      for (; p < p1; ++p) {
        const uint32_t ent = load_entry(Ls.adj, Ls.eid, p, K, Ls.mirror, Ls.eb, Ls.m_half);
        if (ent == DROPPED) continue;
        const int src = (int)(ent & 0xffffu);
        float4 a = *reinterpret_cast<const float4*>(feat + (src << 5) + (fo ^ ((src & 7) << 2)));
        if (PR) a = scale_row(a, __ldcg(rinv + src * R + (int)((ent >> 16) & 0xffu)));
        float4* d = reinterpret_cast<float4*>(row + (int)((ent >> 16) & 0xffu) * inp);
        float4 t = *d;
        t.x += a.x; t.y += a.y; t.z += a.z; t.w += a.w;
        *d = t;
      }
    }
    __syncwarp();
  }
}

// ---- tensor-core tiles: mma.sync m16n8k8 TF32 with 3xTF32 error compensation (fp32-level accuracy) ----------
// D(16x8) += A(16x8, row) * B(8x8, col).  lane: g = lane>>2, t = lane&3
//   A: a0=(g,t) a1=(g+8,t) a2=(g,t+4) a3=(g+8,t+4)   B: b0=(k=t,n=g) b1=(k=t+4,n=g)   D: d0=(g,2t) d1=(g,2t+1) d2=(g+8,2t) d3=(g+8,2t+1)
__device__ __forceinline__ uint32_t f2tf32(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return u;
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// x = hi + lo:  hi = x with the 13 low mantissa bits cleared (exactly a tf32 value), lo = x - hi (exact in fp32;
// the tensor core reads its top 10 mantissa bits).  a*b ~= lo_a*hi_b + hi_a*lo_b + hi_a*hi_b  (small terms first);
// the dropped lo*lo term and the truncation of lo are O(2^-21) relative.  The split is a mask and a subtraction
// (cvt.rna.tf32 would round instead of truncate and costs more instructions per value).
__device__ __forceinline__ void mma_3xtf32(float (&d)[4], float (&dsm)[4], const float (&af)[4], const float (&bf)[2]) {
  uint32_t ah[4], al[4], bh[2], bl[2];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    ah[i] = __float_as_uint(af[i]) & 0xffffe000u;
    al[i] = __float_as_uint(af[i] - __uint_as_float(ah[i]));
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    bh[i] = __float_as_uint(bf[i]) & 0xffffe000u;
    bl[i] = __float_as_uint(bf[i] - __uint_as_float(bh[i]));
  }
  // the two cross terms go to a separate accumulator: shorter dependency chains (and the small terms are summed
  // among themselves before meeting the large one)
  mma_tf32(dsm, al, bh);
  mma_tf32(dsm, ah, bl);
  mma_tf32(d, ah, bh);
}

__device__ __forceinline__ void split_tf32(const float (&f)[4], uint32_t (&hi)[4], uint32_t (&lo)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    hi[i] = __float_as_uint(f[i]) & 0xffffe000u;
    lo[i] = __float_as_uint(f[i] - __uint_as_float(hi[i]));
  }
}
__device__ __forceinline__ void mma_3xtf32_a(float (&d)[4], float (&dsm)[4], const uint32_t (&ah)[4],
                                             const uint32_t (&al)[4], const float (&bf)[2]) {
  uint32_t bh[2], bl[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    bh[i] = __float_as_uint(bf[i]) & 0xffffe000u;
    bl[i] = __float_as_uint(bf[i] - __uint_as_float(bh[i]));
  }
  mma_tf32(dsm, al, bh);
  mma_tf32(dsm, ah, bl);
  mma_tf32(d, ah, bh);
}

// ---- fragments by ldmatrix: a 16 x 8 fp32 block read as four 8 x 8 b16 matrices (8 rows of 16 bytes each, each row
// address 16-byte aligned; lanes 8j .. 8j + 7 address the rows of matrix j).  Lane (g, t) = (L >> 2, L & 3) gets word
// t of row g of matrix j in register j, so
//   A (rows m of a K-contiguous block): lane L addresses row L & 15, floats 4 (L >> 4) .. +3 -> {a0, a1, a2, a3} of
//     mma m16n8k8;
//   B (rows n0 .. n0 + 15 of an n-major, K-contiguous slab): lane L addresses row (L & 7) + 8 (L >> 4), floats
//     4 ((L >> 3) & 1) .. +3 -> {b0, b1} of the tile n0, then {b0, b1} of the tile n0 + 8 (each pair in adjacent
//     registers, as the mma takes it).
// One LDSM replaces four 32-bit LDS.
__device__ __forceinline__ void ldsm_x4(float (&f)[4], uint32_t addr) {
  uint32_t r[4];
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
#pragma unroll
  for (int i = 0; i < 4; ++i) f[i] = __uint_as_float(r[i]);
}

// ---- two adjacent 16x8 tiles (columns n0, n0 + 8) of one 16-row block per warp: the A fragments are loaded and split
// ONCE for both (the tile loops are issue bound; one tile per warp repeated the A part in the four warps of a row
// block), and one ldmatrix.x4 of the B slab gives both tiles' B fragments of a k-step.  Per output element the sums
// and their order are those of one tile per warp: (d, e) take the even k-steps of the first span, (d2, e2) the odd
// ones and the second (root) span; e/e2 hold the 3xTF32 cross terms.
struct TileAcc { float d[4], d2[4], e[4], e2[4]; };
__device__ __forceinline__ void tile_zero(TileAcc& t) {
#pragma unroll
  for (int i = 0; i < 4; ++i) { t.d[i] = 0.f; t.d2[i] = 0.f; t.e[i] = 0.f; t.e2[i] = 0.f; }
}
// a: this lane's ldmatrix address in the A block (K-contiguous rows, k = 0);  b: the same in rows n0 .. n0 + 15 of
// the n-major slab.  K is a multiple of 8.
__device__ __forceinline__ void tiles_span(TileAcc (&T)[2], uint32_t a, uint32_t b, int K) {
  int k0 = 0;
  for (; k0 + 16 <= K; k0 += 16) {                  // two independent accumulator sets per iteration
    float af[4], ag[4], bf[4], bg[4];
    ldsm_x4(af, a + 4 * k0);
    ldsm_x4(ag, a + 4 * k0 + 32);
    ldsm_x4(bf, b + 4 * k0);
    ldsm_x4(bg, b + 4 * k0 + 32);
    uint32_t ah[4], al[4], gh[4], gl[4];
    split_tf32(af, ah, al);
    split_tf32(ag, gh, gl);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      mma_3xtf32_a(T[i].d, T[i].e, ah, al, {bf[2 * i], bf[2 * i + 1]});
      mma_3xtf32_a(T[i].d2, T[i].e2, gh, gl, {bg[2 * i], bg[2 * i + 1]});
    }
  }
  if (k0 < K) {                                     // 8-K tail (K = 8 mod 16: the 4-wide input layer at R = 5)
    float af[4], bf[4];
    ldsm_x4(af, a + 4 * k0);
    ldsm_x4(bf, b + 4 * k0);
    uint32_t ah[4], al[4];
    split_tf32(af, ah, al);
#pragma unroll
    for (int i = 0; i < 2; ++i) mma_3xtf32_a(T[i].d, T[i].e, ah, al, {bf[2 * i], bf[2 * i + 1]});
  }
}
// the second span (root / d pre rows), into (d2, e2).  a: this lane's ldmatrix address at k = 0 (already swizzled),
// xs: XOR applied to the k offset (hix swizzle bits 3-4; 0 = linear);  b as in tiles_span
__device__ __forceinline__ void tiles_span2(TileAcc (&T)[2], uint32_t a, int xs, uint32_t b, int K) {
  for (int k0 = 0; k0 < K; k0 += 8) {
    float af[4], bf[4];
    ldsm_x4(af, a + 4 * (k0 ^ xs));
    ldsm_x4(bf, b + 4 * k0);
    uint32_t ah[4], al[4];
    split_tf32(af, ah, al);
#pragma unroll
    for (int i = 0; i < 2; ++i) mma_3xtf32_a(T[i].d2, T[i].e2, ah, al, {bf[2 * i], bf[2 * i + 1]});
  }
}

__host__ __device__ __forceinline__ int a16(int x) { return (x + 15) & ~15; }

struct Split { int lo, hi; };
__device__ __forceinline__ Split own_range(int n, int rank, int CL) {
  const int per = ((n + CL - 1) / CL + GN - 1) / GN * GN;   // multiple of the warp group
  Split s;
  s.lo = min(n, rank * per);
  s.hi = min(n, s.lo + per);
  return s;
}
__host__ __device__ __forceinline__ int own_cap_of(int n_cap, int CL) { return ((n_cap + CL - 1) / CL + GN - 1) / GN * GN; }

#define IGMC_STAMP(i_) do { if (S.prof && threadIdx.x == 0) S.prof[(size_t)blockIdx.x * 64 + (i_)] = clock64(); } while (0)
// debug: wall-clock (globaltimer, ns) of a CTA's start / end and the SM it ran on - slots 50..52 of its prof row
#define IGMC_WALL(i_) do { if (S.prof && threadIdx.x == 0) { S.prof[(size_t)blockIdx.x * 64 + (i_)] = igmc_globaltimer(); \
                                                              S.prof[(size_t)blockIdx.x * 64 + ((i_) < 53 ? 52 : 55)] = igmc_smid(); } } while (0)

// per-step weight preparation (layout: wprep_slab in csrc/lists.cuh).  grid = L * 2 * 32 blocks: block (l, dir, n)
// writes row n of slab (l, dir); one thread per K position.
__global__ void __launch_bounds__(256)
k_prep_weights(igmc_model_t M, const float* __restrict__ params, float* __restrict__ wprep) {
  const int n = blockIdx.x & 31, ld = blockIdx.x >> 5, l = ld >> 1, dir = ld & 1;
  if (dir == 1 && l == 0) return;
  wprep_write_row(M, params, wprep, l, dir, n);
}

__device__ __forceinline__ void copy_f4(float* __restrict__ dst, const float* __restrict__ src, int nfloats) {
  const float4* s4 = reinterpret_cast<const float4*>(src);
  float4* d4 = reinterpret_cast<float4*>(dst);
  for (int i = threadIdx.x; i < (nfloats >> 2); i += blockDim.x) d4[i] = __ldg(s4 + i);
}

// split cluster barrier: work that does not touch peer-written shared memory goes between arrive and wait
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }

// ---- layer rows to the peer CTAs: every CTA stores its rows straight into the peers' buffers with st.async, which
// credits the bytes to an mbarrier of the receiving CTA (complete_tx, release at cluster scope).  The receiver arms
// its barrier with the bytes it expects, (n - n_own) rows x 128 B, and waits for them with acquire at cluster scope:
// no CTA-wide cluster barrier per layer, and a CTA waits only for the rows it reads.  The byte credit may reach the
// barrier before it is armed (the phase cannot complete before the receiver's own arrival).
__device__ __forceinline__ uint32_t mapa_u32(uint32_t a, int rank) {   // shared::cta address -> rank's shared::cluster
  uint32_t d;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(rank));
  return d;
}
// rank of the (pr + 1)-th other CTA of the cluster (pr + 1 < CL), without a division
__device__ __forceinline__ int peer_rank(int rank, int pr, int CL) {
  const int r = rank + pr + 1;
  return r >= CL ? r - CL : r;
}
// v -> the float2 at `dst` and 8 bytes credited to the barrier `bar`, both mapped into CTA `rank` of the cluster
// (the mapping is derived per store: addresses kept across the layer cost registers in the gather)
__device__ __forceinline__ void st_async_peer(const float* dst, float2 v, const uint64_t* bar, int rank) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v2.f32 [%0], {%1, %2}, [%3];"
               ::"r"(mapa_u32(smem_u32(dst), rank)), "f"(v.x), "f"(v.y), "r"(mapa_u32(smem_u32(bar), rank)));
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!ok);
}

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
// The forward of one subgraph as a device function (returns false when it bailed out on a data error, uniformly over
// the cluster): body of k_forward_rs, and first half of the fused train kernel k_train_rs.
template <int NTMAX, bool PR>
__device__ __forceinline__ bool forward_body(const igmc_model_t& M, const float* __restrict__ params,
                                             const uint8_t* __restrict__ node_label,
                                             const int32_t* __restrict__ node_ptr,
                                             const int32_t* __restrict__ edge_ptr, const igmc_adj_t& A, int n_cap,
                                             int lcap, int chunk, const igmc_dropout_t& D, int training,
                                             const igmc_saved_t& S, const float* __restrict__ y, float loss_scale,
                                             float* __restrict__ dpred, float* __restrict__ sqerr,
                                             const igmc_stage_t& IMG, int* err, float* smem) {
  cg::cluster_group cluster = cg::this_cluster();
  const int CL = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int g = blockIdx.x / CL;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5, NT = blockDim.x;
  const int L = M.num_layers, R = M.num_relations, CW = HID * L, F = 2 * CW;
  const int in0 = M.in_dim0, in0p = a4(in0);
  const int SSmax = R * HID + 4, KSmax = (R + 1) * HID + 4;
  const int own_cap = own_cap_of(n_cap, CL);
  float* Hbuf0 = smem;                               // [n_cap][32]
  float* Hbuf1 = Hbuf0 + (size_t)n_cap * HID;        // [n_cap][32]
  float* Wn = Hbuf1 + (size_t)n_cap * HID;           // [32][KS]
  float* stage = Wn + (size_t)HID * KSmax;           // [chunk + XR][SSmax]
  float* bias_s = stage + (size_t)(chunk + XR) * SSmax;
  float* invdeg = bias_s + HID;                      // [n_cap]
  float* feat_s = invdeg + a4(n_cap);
  float* hid_s = feat_s + a4(F);
  int* ibuf = reinterpret_cast<int*>(hid_s + L1O) + IMG_HDR;    // [header |] list offsets + segment table
  uint32_t* lbuf = reinterpret_cast<uint32_t*>(ibuf + a4(list_ints(own_cap)));   // [lcap]
  __shared__ int s_t[2];
  __shared__ int ws[34];
  // [0] list image, [1] weight slab of the current layer (TMA completion), [2 + (l & 1)] the peers' rows of layer l
  __shared__ __align__(8) uint64_t mbar[4];

  const int nb = node_ptr[g], n = node_ptr[g + 1] - nb;
  const int eb = edge_ptr[g], m_half = (edge_ptr[g + 1] - eb) >> 1;
  if (n > n_cap) {   // uniform over the cluster
    if (tid == 0) igmc_set_err(err, IGMC_ERR_SMEM_NODES);
    return false;
  }
  const EdgeKeep K = make_keep(D, training);
  const Split own = own_range(n, rank, CL);
  const int n_own = own.hi - own.lo;
  IGMC_STAMP(0);
  IGMC_WALL(50);
  if (S.gate && tid == 0) atomicAdd(S.gate, 1);   // "this CTA is resident" (igmc_gate_wait)
  pdl_trigger();   // a backward launched behind this kernel may take the SMs the first finished clusters free

  // weights of a layer: the [W_r ; root] slab prepared by igmc_prep_weights, one bulk (TMA) copy issued by a single
  // thread; every thread waits on mbar[1] (phase = layer parity) right before the layer's tensor-core tiles, so the
  // copy runs under the gather.  Callers guarantee (barrier) that nobody still reads Wn.
  auto load_weights = [&](int l) {
    const int KS = wprep_row(R, l == 0 ? in0p : HID).KS();
    if (tid == 0) {
      fence_proxy_async();
      mbar_expect_tx(&mbar[1], (uint32_t)(HID * KS * 4));
      bulk_g2s(Wn, S.wprep + (size_t)l * 2 * wprep_slab(R), (uint32_t)(HID * KS * 4), &mbar[1]);
    }
    if (tid < HID) bias_s[tid] = params[M.off_bias[l] + tid];
  };
  if (tid == 0) {
    s_t[0] = 0x7fffffff; s_t[1] = 0x7fffffff;
    for (int i = 0; i < 4; ++i) mbar_init(&mbar[i], 1);
    mbar_fence_init();
  }
  __syncthreads();
  // the peers store into this CTA's buffers and barriers from layer 0's tiles on: its barriers are initialised before
  // any of them passes the wait in front of the layer loop
  if (CL > 1) cluster_arrive_relaxed();
  const bool use_img = IMG.tab != nullptr;
  if (use_img && tid == 0) {   // pre-staged lists: header + tables, then the entries, straight into shared memory
    const int32_t* gt = IMG.tab + (size_t)blockIdx.x * IMG.tab_ints;
    const int total = __ldg(gt), staged = __ldg(gt + 2);
    const uint32_t tb = (uint32_t)IMG.tab_ints * 4u, eb4 = (staged && total > 0) ? (uint32_t)a4(total) * 4u : 0u;
    mbar_expect_tx(&mbar[0], tb + eb4);
    bulk_g2s(ibuf - IMG_HDR, gt, tb, &mbar[0]);
    if (eb4) bulk_g2s(lbuf, IMG.ent + (size_t)blockIdx.x * IMG.lcap, eb4, &mbar[0]);
  }
  load_weights(0);
  float* H = Hbuf0;
  float* Hn = Hbuf1;
  for (int idx = tid; idx < n * HID; idx += NT) {
    const int v = idx >> 5, c = idx & 31;
    const int lab = node_label[nb + v];
    H[hix(v, c)] = (c == lab && c < in0) ? 1.f : 0.f;
    if (c == 0 && lab == 0) atomicMin(&s_t[0], v);
    if (c == 0 && lab == 1) atomicMin(&s_t[1], v);
  }
  // in-lists of the own nodes -> shared memory; kept in-degree (dropout_adj is applied once, models.py:193)
  Lists Ls;
  if (use_img) {
    for (int i = tid; i < n_own; i += NT) {
      const float id = __ldg(IMG.inv_deg + nb + own.lo + i);
      invdeg[own.lo + i] = id;
      S.inv_deg[nb + own.lo + i] = id;
    }
    mbar_wait(&mbar[0], 0);
    Ls = lists_view(ibuf, own_cap, lbuf, A.in_adj, A.in_eid, false, eb, m_half);
    __syncthreads();
  } else {
    Ls = stage_lists(A.in_adj, A.in_eid, A.in_ptr, nb, own.lo, own.hi, K, false, eb, m_half, lbuf, lcap, ibuf, own_cap,
                     chunk, ws, invdeg, S.inv_deg);
  }
  float* rinv = PR ? S.rel_inv_deg + (size_t)nb * R : nullptr;   // [n][R] 1/|N_r(v)| (own rows written here)
  if (PR) rel_inv_deg_own(Ls, K, A.in_ptr, nb, own.lo, n_own, R, rinv);
  if (tid == 0) ws[33] = 0;   // segment ticket of gather_segments (made visible by the barrier at the top of the layer loop)
  const bool ext = M.readout != 0;   // concat_states only: an external readout (csrc/sortpool.cu) takes over
  const int tu = s_t[0], ti = s_t[1];
  if (!ext && (tu >= n || ti >= n)) {   // (uniform over the cluster)
    if (tid == 0) igmc_set_err(err, IGMC_ERR_BAD_BATCH);
    mbar_wait(&mbar[1], 0);   // do not exit under an in-flight bulk copy
    if (CL > 1) cluster_wait();
    return false;
  }
  if (S.prof && tid == 0) {   // debug: staging facts
    long long* pp = S.prof + (size_t)blockIdx.x * 64;
    pp[60] = Ls.lst != nullptr; pp[61] = n_own > 0 ? Ls.lptr[n_own] : 0; pp[62] = Ls.segbase[n_own]; pp[63] = lcap;
    pp[59] = chunk; pp[58] = n_own;
  }
  const int gq = lane >> 2, tq = lane & 3;
  // the peers' barriers are initialised (arrive after this CTA's initialisation above)
  if (CL > 1) cluster_wait();
  IGMC_STAMP(1);
  // Layer l's rows travel to the peers by st.async on their barrier mbar[2 + (l & 1)] (phase (l >> 1) & 1); every CTA
  // waits on its own barrier for the (n - n_own) rows of the peers at the end of the layer.  Write-after-read: a peer
  // stores only rows it owns, into the buffer this CTA gathers layer l - 1 from; it reaches layer l's tiles only after
  // it has received all of this CTA's layer l - 1 rows, which are pushed by the tiles of the last chunk, after every
  // gather of layer l - 1 (release of the byte credit, acquire of the peer's wait).  The same argument orders a
  // barrier's uses: layer l + 2's bytes can reach it only after this CTA's layer l + 1 gather, behind its layer l wait.
  // Nothing is stored into this CTA after its last layer's wait has seen every byte: it may exit (or re-carve its
  // shared memory for the backward) from there.
  for (int l = 0; l < L; ++l) {
    const int inp = l == 0 ? in0p : HID;
    const WprepRow wr = wprep_row(R, inp);
    const int K1 = wr.K1, K1p = wr.K1p, inpp = wr.inpp, SS = K1p + 4, KS = wr.KS();
    uint64_t* xbar = &mbar[2 + (l & 1)];
    if (CL > 1 && tid == 0) mbar_expect_tx(xbar, (uint32_t)(n - n_own) * 128u);
    __syncthreads();
    IGMC_STAMP(2 + 6 * l);
    // staged lists: the gather stores the rows of one-segment nodes already scaled by their degree factor, the fold
    // below only adds the extra rows of long lists.  Unstaged lists (gathered by read-modify-write) and layer 0 with a
    // saved aggregate over several chunks (written by the fold) keep the fold over every row.
    const bool run_scale = Ls.lst != nullptr && !(S.zsave && l == 0 && n_own > chunk);
    for (int c0 = 0; c0 < n_own; c0 += chunk) {
      const int crow = min(chunk, n_own - c0);
      // ---- aggregate: one 8-lane group per list segment ----
#define IGMC_STAMP_T(t_, i_) do { if (S.prof && l == 1 && threadIdx.x == (t_)) S.prof[(size_t)blockIdx.x * 64 + (i_)] = clock64(); } while (0)
      IGMC_STAMP_T(0, 39); IGMC_STAMP_T(992, 49);
      const RunScale rsc{run_scale ? (PR ? rinv + (size_t)(own.lo + c0) * R : invdeg + own.lo + c0) : nullptr,
                         Ls.ex + c0, crow};
      const int sg0 = Ls.segbase[c0], sg1 = Ls.segbase[c0 + crow];
      if (inp == 4) gather_segments<1, false, PR ? 2 : 1>(Ls, K, sg0, sg1, lane, H, stage, SS, inp, R, &ws[33], nullptr, rsc);
      else gather_segments<8, false, PR ? 2 : 1>(Ls, K, sg0, sg1, lane, H, stage, SS, inp, R, &ws[33], nullptr, rsc);
      IGMC_STAMP_T(0, 40); IGMC_STAMP_T(992, 43); IGMC_STAMP_T(480, 46);
      if (l == 0) IGMC_STAMP(32);
      __syncthreads();
      if (l == 0) IGMC_STAMP(33);
      if (tid == 0) ws[33] = 0;   // re-arm the segment ticket (the next gather is several barriers away)
      IGMC_STAMP_T(0, 41); IGMC_STAMP_T(992, 44);
      // ---- fold the extra segments of long lists into their node row, scale by 1/deg (PR: the relation block by
      //      1/|N_r(v)|), keep a copy for backward ----
      if (!run_scale) {
        const int kq = K1 >> 2, SS4 = SS >> 2;
        float4* st4 = reinterpret_cast<float4*>(stage);
        // flat over (row, float4): independent iterations; (r, k4) advance by NT = dr * kq + dk without a division
        const int dr = NT / kq, dk = NT - dr * kq;
        int r = tid / kq, k4 = tid - r * kq;
        for (int idx = tid; idx < crow * kq; idx += NT, r += dr, k4 += dk) {
          if (k4 >= kq) { k4 -= kq; ++r; }
          const int v = own.lo + c0 + r;
          const float id2 = PR ? __ldcg(rinv + (size_t)v * R + k4 / (inp >> 2)) : invdeg[v];
          const int e = Ls.ex[c0 + r], x0 = e & 0xffff, nex = e >> 16;
          float4 t = st4[(size_t)r * SS4 + k4];
          for (int j = 0; j < nex; ++j) {
            const float4 u = st4[(size_t)(crow + x0 + j) * SS4 + k4];
            t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
          }
          t.x *= id2; t.y *= id2; t.z *= id2; t.w *= id2;
          st4[(size_t)r * SS4 + k4] = t;
          if (S.zsave && l == 0 && n_own > chunk)   // (one chunk: copied out below, at the end of the layer)
            reinterpret_cast<float4*>(S.zsave + (size_t)(nb + v) * (size_t)K1)[k4] = t;
        }
      } else if (sg1 - sg0 > crow) {   // the chunk has extra segments (uniform: from the segment table)
        const int kq = K1 >> 2, SS4 = SS >> 2;
        float4* st4 = reinterpret_cast<float4*>(stage);
        for (int r = warp; r < crow; r += nwarps) {
          const int e = Ls.ex[c0 + r], x0 = e & 0xffff, nex = e >> 16;
          if (nex == 0) continue;
          const int v = own.lo + c0 + r;
          for (int k4 = lane; k4 < kq; k4 += 32) {
            const float id2 = PR ? __ldcg(rinv + (size_t)v * R + k4 / (inp >> 2)) : invdeg[v];
            float4 t = st4[(size_t)r * SS4 + k4];
            for (int j = 0; j < nex; ++j) {
              const float4 u = st4[(size_t)(crow + x0 + j) * SS4 + k4];
              t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
            }
            t.x *= id2; t.y *= id2; t.z *= id2; t.w *= id2;
            st4[(size_t)r * SS4 + k4] = t;
          }
        }
      }
      IGMC_STAMP_T(0, 42); IGMC_STAMP_T(992, 45);
      IGMC_STAMP(3 + 6 * l);
      if (!run_scale || sg1 - sg0 > crow) __syncthreads();
      IGMC_STAMP(4 + 6 * l);
      // ---- dense transform on tensor cores: out[16x8 tiles] = [AGG' | h] . [W_r ; root] ----
      if (c0 == 0) mbar_wait(&mbar[1], (uint32_t)(l & 1));   // this layer's weight slab has landed
      const int mt = (crow + 15) >> 4;
      for (int item = warp; item < mt * 2; item += nwarps) {   // warp = (16-row block, 16-column half)
        const int m0 = (item >> 1) << 4, nh = (item & 1) << 4;
        // this lane's ldmatrix row and float offset in the A block and in the B slab (ldsm_x4)
        const int ar = lane & 15, ac = (lane >> 4) << 2, br = (lane & 7) | ((lane >> 1) & 8), bc = (lane >> 1) & 4;
        TileAcc T[2];
        tile_zero(T[0]); tile_zero(T[1]);
        const uint32_t bs = smem_u32(Wn + (nh + br) * KS + bc);
        tiles_span(T, smem_u32(stage + (m0 + ar) * SS + ac), bs, K1p);
        const int r0 = c0 + m0 + gq, r1 = r0 + 8;           // rows relative to the own range
        const int vf = own.lo + min(c0 + m0 + ar, n_own - 1);  // this lane's ldmatrix row of H
        const int sw = (vf & 7) << 2;                       // hix(): column ^ swizzle, split into its bit 2 and bits 3-4
        tiles_span2(T, smem_u32(H + (vf << 5) + (ac ^ (sw & 4))), sw & 24, bs + 4 * K1p, inpp);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float d[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) d[q] = (T[i].d[q] + T[i].d2[q]) + (T[i].e[q] + T[i].e2[q]);
          const int cc = nh + 8 * i + 2 * tq;
          const float b0 = bias_s[cc], b1 = bias_s[cc + 1];
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int r = half ? r1 : r0;
            if (r < n_own) {
              const int v = own.lo + r;
              const float2 o = make_float2(tanhf(d[2 * half] + b0), tanhf(d[2 * half + 1] + b1));
              const int off = hix(v, cc);
              *reinterpret_cast<float2*>(Hn + off) = o;
#pragma unroll
              for (int pr = 0; pr < 3; ++pr)   // push the row slice to the other CTAs of the cluster
                if (pr + 1 < CL) st_async_peer(Hn + off, o, xbar, peer_rank(rank, pr, CL));
            }
          }
        }
      }
      IGMC_STAMP(5 + 6 * l);
      __syncthreads();
    }
    IGMC_STAMP(6 + 6 * l);
    if (n_own == 0) mbar_wait(&mbar[1], (uint32_t)(l & 1));   // keep the barrier phases in step (no tiles ran)
    // the next layer's weights do not depend on the peers (every read of Wn is behind the barrier above): load them
    // while the peers' rows land
    if (l + 1 < L) load_weights(l + 1);
    if (S.zsave && l == 0 && n_own <= chunk) {
      // layer 0's scaled aggregate for the backward (layers >= 1: the backward takes its weight gradients from its own
      // aggregate): the staging rows are untouched until the next gather, so the copy runs while the peers' rows land
      const int kq = K1 >> 2, SS4 = SS >> 2;
      const float4* st4 = reinterpret_cast<const float4*>(stage);
      const int dr = NT / kq, dk = NT - dr * kq;
      int r = tid / kq, k4 = tid - r * kq;
      for (int idx = tid; idx < n_own * kq; idx += NT, r += dr, k4 += dk) {
        if (k4 >= kq) { k4 -= kq; ++r; }
        reinterpret_cast<float4*>(S.zsave + (size_t)(nb + own.lo + r) * (size_t)K1)[k4] = st4[(size_t)r * SS4 + k4];
      }
      IGMC_STAMP(34);
    }
    float* t = H; H = Hn; Hn = t;
    // concat_states of the own rows -> global (local rows: no need to wait for the peers), overlapping the next
    // layer's gather; one coalesced 128 B row per 8 threads
    for (int idx = tid; idx < n_own * 8; idx += NT) {
      const int v = own.lo + (idx >> 3), c4 = (idx & 7) << 2;
      __stcg(reinterpret_cast<float4*>(S.states + (size_t)(nb + v) * CW + l * HID + c4),
             *reinterpret_cast<const float4*>(H + hix(v, c4)));
    }
    if (CL > 1) mbar_wait_cluster(xbar, (uint32_t)((l >> 1) & 1));   // the peers' rows of layer l have landed
    IGMC_STAMP(7 + 6 * l);
    // concat_states rows of the two target nodes (models.py:203-207), all rows are local now
    if (rank == 0 && !ext && tid < 2 * HID) {
      const int node = tid < HID ? tu : ti, c = tid & 31;
      feat_s[(tid < HID ? 0 : CW) + l * HID + c] = H[hix(node, c)];
    }
  }

  if (rank != 0 || ext) { IGMC_WALL(51); return true; }
  // ---- readout (models.py:205-215), one CTA of the cluster ----
  __syncthreads();
  IGMC_STAMP(27);
  for (int c = tid; c < F; c += NT) S.feat[(size_t)g * F + c] = feat_s[c];
  if (tid == 0) { S.target[2 * g] = nb + tu; S.target[2 * g + 1] = nb + ti; }
  readout_lin1(M, params, feat_s, F, g, D, K.seed, training, hid_s, S, warp, nwarps, lane);
  IGMC_STAMP(28);
  __syncthreads();
  IGMC_STAMP(29);
  if (warp == 0)
    readout_lin2(M, params, hid_s, M.multiply_by, g, y, loss_scale, S.pred, sqerr,
                 dpred, lane);
  IGMC_STAMP(2 + 6 * L);
  IGMC_WALL(51);
  return true;
}

template <int NTMAX, bool PR>
__global__ void __launch_bounds__(NTMAX, 1)
k_forward_rs(igmc_model_t M, const float* __restrict__ params, const uint8_t* __restrict__ node_label,
             const int32_t* __restrict__ node_ptr, const int32_t* __restrict__ edge_ptr, igmc_adj_t A, int n_cap,
             int lcap, int chunk, igmc_dropout_t D, int training, igmc_saved_t S, const float* __restrict__ y,
             float loss_scale, float* __restrict__ dpred, float* __restrict__ sqerr, igmc_stage_t IMG, int* err) {
  extern __shared__ __align__(16) float smem[];
  forward_body<NTMAX, PR>(M, params, node_label, node_ptr, edge_ptr, A, n_cap, lcap, chunk, D, training, S, y, loss_scale,
                      dpred, sqerr, IMG, err, smem);
}

// ------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------
constexpr int DPS_ = 40;   // row stride of the own-rows dpre / h_{l-1} copies (== 8 mod 32: conflict-free k-major fragments)

// 3xTF32 with the A operand split once (it is reused for several B tiles)

// weight-gradient tiles of one warp over the chunk's nodes: CNT column tiles share the A^T fragment of a k-step
template <int CNT>
__device__ __forceinline__ void wgrad_pass(const float* __restrict__ ha, const float* const (&bb)[4], const int (&bst)[4],
                                           int krows, float (&acc)[4][4], float (&acs)[4][4]) {
  for (int k0 = 0; k0 < krows; k0 += 8) {
    const float* a = ha + (size_t)k0 * DPS_;
    const float af[4] = {a[0], a[8], a[4 * DPS_], a[4 * DPS_ + 8]};
    uint32_t ah[4], al[4];
    split_tf32(af, ah, al);
#pragma unroll
    for (int i = 0; i < CNT; ++i) {
      const float* bp = bb[i] + (size_t)k0 * bst[i];
      const float bf[2] = {bp[0], bp[4 * bst[i]]};
      mma_3xtf32_a(acc[i], acs[i], ah, al, bf);
    }
  }
}

// Per layer l (top down), for the own nodes u of this CTA:
//   (0) dpre = d h_l (1 - h_l^2); gather source DPS = dpre / deg of ALL nodes (PR: dpre, the gather weighs every
//       entry (d, r) by 1/|N_r(d)| instead), DP = dpre of the own rows
//   (1) Q[u,r,:] = sum_{(u->d) of type r, kept} DPS[d,:]                  (gather over the out-lists, as forward)
//       d h_{l-1}[u] = [Q[u] | dpre[u]] . [W_r^T ; root^T]                (tensor cores) -> pushed to every CTA
//   (2) dW_r = sum_u h_{l-1}[u]^T Q[u,r,:],  d root = sum_u h_{l-1}[u]^T dpre[u],  d bias = sum_u dpre[u]
//       (tensor cores, K = own nodes; A = the h_{l-1} rows fetched by TMA under the gather)  -> raw partial row
//   Layer 0 has no data gradient; its dW_r come from the saved aggregate of the one-hot input (S.zsave).
// The (att, basis) chain rule is NOT applied here: it is linear and runs once on the sum (igmc_grad_reduce).
template <int NTMAX, bool PR>
__device__ __forceinline__ void backward_body(const igmc_model_t& M, const float* __restrict__ params,
                                              const uint8_t* __restrict__ node_label,
                                              const int32_t* __restrict__ node_ptr,
                                              const int32_t* __restrict__ edge_ptr, const igmc_adj_t& A, int n_cap,
                                              int lcap, int chunk, const igmc_dropout_t& D, const igmc_saved_t& S,
                                              const float* dpred /* written by this launch in k_train_rs */,
                                              float* __restrict__ gpart,
                                              float* __restrict__ dhid_out, const igmc_stage_t& IMG, int* err,
                                              float* smem) {
  cg::cluster_group cluster = cg::this_cluster();
  const int CL = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int g = blockIdx.x / CL;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5, NT = blockDim.x;
  const int L = M.num_layers, R = M.num_relations, CW = HID * L, F = 2 * CW;
  const int in0 = M.in_dim0, in0p = a4(in0);
  const int SSmax = R * HID + 4, KSmax = (R + 1) * HID + 4;
  const int own_cap = own_cap_of(n_cap, CL), own_cap16 = a16(own_cap);
  float* DH0 = smem;                                    // [2][n_cap][32]  d h_l of all nodes, double-buffered by layer
  float* DH1 = DH0 + (size_t)n_cap * HID;               //   parity: peers push d h_{l-1} into one while the other, turned
                                                        //   in place into dpre/deg (the gather source), is being read
  float* DP = DH1 + (size_t)n_cap * HID;                // [own_cap16][DPS_] dpre of the own rows (zero padded)
  float* Wn = DP + (size_t)own_cap16 * DPS_;            // [32][KS]   prepared weights of the data-gradient tiles
  float* stage = Wn + (size_t)HID * KSmax;              // [chunk + XR][SSmax] Q rows  |  layer 0: aggregate tile [rows][TS]
  float* Hs = stage + (size_t)(chunk + XR) * SSmax;     // [chunk][DPS_] h_{l-1} of the chunk's rows (TMA)
  float* invdeg = Hs + (size_t)chunk * DPS_;
  float* dfeat = invdeg + a4(n_cap);
  float* dhid_s = dfeat + a4(F);
  int* ibuf = reinterpret_cast<int*>(dhid_s + L1O) + IMG_HDR;   // [header |] list offsets + segment table
  uint32_t* lbuf = reinterpret_cast<uint32_t*>(ibuf + a4(list_ints(own_cap)));   // [lcap]
  __shared__ int ws[34];
  // TMA completion: [0] list image, [1] weight slab, [2] h_{l-1} rows;  [3 + (l & 1)] the peers' rows of d h_{l-1}
  __shared__ __align__(8) uint64_t mbar[5];

  const int nb = node_ptr[g], n = node_ptr[g + 1] - nb;
  const int eb = edge_ptr[g], m_half = (edge_ptr[g + 1] - eb) >> 1;
  if (n > n_cap) {
    if (tid == 0) igmc_set_err(err, IGMC_ERR_SMEM_NODES);
    return;
  }
  const EdgeKeep K = make_keep(D, 1);
  const bool sym = A.symmetric != 0;
  const Split own = own_range(n, rank, CL);
  const int n_own = own.hi - own.lo;
  const bool ext = M.readout != 0;   // d concat_states comes from an external readout (S.dstate)
  float* gp = gpart + ((size_t)g * CL + rank) * (size_t)igmc_raw_count(R, in0, L);
  pdl_trigger();   // the gradient-assembly kernel behind this one may be scheduled as SMs free up
  if (tid == 0) {
    for (int i = 0; i < 5; ++i) mbar_init(&mbar[i], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (CL > 1) cluster_arrive_relaxed();   // (waited for in front of the layer loop, before the first push)
  uint32_t wuse = 0, huse = 0;   // completed-phase counters of mbar[1] / mbar[2] (uniform over the block)
  // per-layer operand that does not depend on the peers: the [W_r^T ; root^T] slab of the data gradient (one bulk
  // copy by one thread; waited for right before the tiles).  Callers guarantee that nobody still reads Wn.
  auto load_weights = [&](int l) {
    if (tid == 0) {
      const uint32_t bytes = (uint32_t)(wprep_slab(R) * 4);
      fence_proxy_async();
      mbar_expect_tx(&mbar[1], bytes);
      bulk_g2s(Wn, S.wprep + ((size_t)l * 2 + 1) * wprep_slab(R), bytes, &mbar[1]);
    }
  };
  const bool use_img = IMG.tab != nullptr;
  if (use_img && tid == 0) {
    const int32_t* gt = IMG.tab + (size_t)blockIdx.x * IMG.tab_ints;
    const int total = __ldg(gt), staged = __ldg(gt + 2);
    const uint32_t tb = (uint32_t)IMG.tab_ints * 4u, eb4 = (staged && total > 0) ? (uint32_t)a4(total) * 4u : 0u;
    mbar_expect_tx(&mbar[0], tb + eb4);
    bulk_g2s(ibuf - IMG_HDR, gt, tb, &mbar[0]);
    if (eb4) bulk_g2s(lbuf, IMG.ent + (size_t)blockIdx.x * IMG.lcap, eb4, &mbar[0]);
  }
  if (L > 1) load_weights(L - 1);
  // stale staging rows are read as (discarded or zero-weighted) tile padding: keep them finite
  {
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float4* st4 = reinterpret_cast<float4*>(stage);
    const int tot4 = (int)((((size_t)(chunk + XR) * SSmax) + (size_t)chunk * DPS_) >> 2);   // stage + Hs are adjacent
    for (int i = tid; i < tot4; i += NT) st4[i] = z4;
  }
  // out-lists of the own nodes (symmetric batches: the in-lists with mirrored edge ids)
  Lists Ls;
  if (!use_img)
    Ls = stage_lists(sym ? A.in_adj : A.out_adj, sym ? A.in_eid : A.out_eid, sym ? A.in_ptr : A.out_ptr, nb, own.lo,
                     own.hi, K, sym, eb, m_half, lbuf, lcap, ibuf, own_cap, chunk, ws, nullptr, nullptr);
  // everything above only touches what existed before the forward ran (batch, list images, prepared weights): under
  // a programmatic dependent launch it overlaps the forward's tail.  From here on the forward's results are read.
  pdl_wait();
  IGMC_STAMP(0);
  IGMC_WALL(53);   // (the backward's wall-clock stamps use slots 53..55 so that one buffer holds both kernels')
  const int tu = ext ? -1 : S.target[2 * g] - nb, ti = ext ? -1 : S.target[2 * g + 1] - nb;

  // ---- readout backward (every CTA needs d feat to seed its target rows) ----
  if (!ext) readout_dhid(M, params, S, dpred, g, dhid_s, dhid_out, rank == 0, tid, NT);
  if (!PR)
    for (int v = tid; v < n; v += NT) invdeg[v] = __ldcg(S.inv_deg + nb + v);   // (peer rows: L2, see k_train_rs)
  // PR: 1/|N_r(d)| of every node d, read through L2 by the gather (peer rows, as inv_deg above)
  const float* rinv = PR ? S.rel_inv_deg + (size_t)nb * R : nullptr;
  __syncthreads();
  if (!ext) {
    // d feat: thread slice p of NT/F takes every (NT/F)-th o, partials in `stage`, summed in slice order
    const int parts = max(1, NT / F);
    readout_dfeat_part(M, params, dhid_s, F, parts, tid, stage);
    __syncthreads();
    for (int j = tid; j < F; j += NT) {
      float s = 0.f;
      for (int q = 0; q < parts; ++q) s += stage[q * F + j];
      dfeat[j] = s;
    }
  }
  __syncthreads();
  // d h_L : only the two target rows receive gradient from the readout
  {
    float* DHtop = ((L - 1) & 1) ? DH1 : DH0;
    for (int idx = tid; idx < n * HID; idx += NT) {
      const int v = idx >> 5, c = idx & 31;
      float dh = 0.f;
      if (ext) dh = __ldg(S.dstate + (size_t)(nb + v) * CW + (L - 1) * HID + c);
      if (v == tu) dh += dfeat[(L - 1) * HID + c];
      if (v == ti) dh += dfeat[CW + (L - 1) * HID + c];
      DHtop[hix(v, c)] = dh;
    }
  }
  if (use_img) {
    mbar_wait(&mbar[0], 0);
    Ls = lists_view(ibuf, own_cap, lbuf, sym ? A.in_adj : A.out_adj, sym ? A.in_eid : A.out_eid, sym, eb, m_half);
  }
  if (tid == 0) ws[33] = 0;   // segment ticket of gather_segments
  __syncthreads();

  const int gq = lane >> 2, tq = lane & 3;
  if (CL > 1) cluster_wait();   // the peers' barriers are initialised
  IGMC_STAMP(1);
  // d h_{l-1} travels as the forward's layer rows do (st.async on the receiver's barrier mbar[3 + (l & 1)], phase
  // ((L - 1 - l) >> 1) & 1, waited for at the end of layer l; layer 0 exchanges nothing).  Write-after-read: a peer
  // stores its own rows of d h_{l-1} into the buffer this CTA gathered layer l + 1 from, and only after it has received
  // all of this CTA's d h_l rows, pushed by the tiles of this CTA's last layer l + 1 chunk, behind every read of that
  // buffer (step (0) and the gathers).  After its layer 1 wait nothing is stored into this CTA any more.
  for (int l = L - 1; l >= 0; --l) {
    const int in = l == 0 ? in0 : HID, inp = l == 0 ? in0p : HID;
    const WprepRow wr = wprep_row(R, inp);
    const int K1 = wr.K1, K1p = wr.K1p, KRp = K1p + wr.inpp;
    const int sb = 2 + 8 * (L - 1 - l);
    float* DPS = (l & 1) ? DH1 : DH0;                    // d h_l on entry, dpre/deg after step (0)
    float* DHn = (l & 1) ? DH0 : DH1;                    // d h_{l-1} (written here and by the peers)
    float* gpl = gp + igmc_raw_off(R, in0, l);           // this layer's block of the raw partial row
    uint64_t* xbar = &mbar[3 + (l & 1)];
    if (CL > 1 && l > 0 && tid == 0) mbar_expect_tx(xbar, (uint32_t)(n - n_own) * 128u);
    // (0) d pre = d h (1 - h^2);  DPS = d pre / deg (gather source), DP = d pre of the own rows (padded with zeros)
    for (int idx = tid; idx < n * 8; idx += NT) {
      const int v = idx >> 3, c4 = (idx & 7) * 4;
      const float4 dh = *reinterpret_cast<const float4*>(DPS + hix(v, c4));
      const float4 h = __ldcg(reinterpret_cast<const float4*>(S.states + (size_t)(nb + v) * CW + l * HID + c4));
      const float4 dpre = make_float4(dh.x * (1.f - h.x * h.x), dh.y * (1.f - h.y * h.y), dh.z * (1.f - h.z * h.z),
                                      dh.w * (1.f - h.w * h.w));
      const float id = PR ? 1.f : invdeg[v];   // (PR: the factor depends on the relation - applied per entry in (1))
      *reinterpret_cast<float4*>(DPS + hix(v, c4)) = make_float4(dpre.x * id, dpre.y * id, dpre.z * id, dpre.w * id);
      if (v >= own.lo && v < own.hi) *reinterpret_cast<float4*>(DP + (size_t)(v - own.lo) * DPS_ + c4) = dpre;
    }
    for (int idx = tid; idx < (a16(n_own) - n_own) * 8; idx += NT) {
      const int r = n_own + (idx >> 3), c4 = (idx & 7) * 4;
      *reinterpret_cast<float4*>(DP + (size_t)r * DPS_ + c4) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    IGMC_STAMP(sb);
    // d bias = column sums of d pre over the own rows (last warp, lane = channel; the loads are independent)
    if (warp == nwarps - 1) {
      float accb = 0.f;
      for (int r_ = 0; r_ < n_own; ++r_) accb += DP[(size_t)r_ * DPS_ + lane];
      gpl[(R + 1) * inp * HID + lane] = accb;
    }

    if (l > 0) {
      const int SS = K1p + 4, KS = wr.KS();
      const int NTN = (R + 1) * 4;                        // 8-column tiles of [dW_r ... | d root]
      for (int c0 = 0; c0 < n_own; c0 += chunk) {
        const int crow = min(chunk, n_own - c0);
        // h_{l-1} of the chunk's rows -> Hs, one 128 B bulk copy per row issued by warp 0 (lands under the gather)
        if (warp == 0) {
          fence_proxy_async();
          if (lane == 0) mbar_expect_tx(&mbar[2], (uint32_t)crow * 128u);
          __syncwarp();
          for (int r_ = lane; r_ < crow; r_ += 32)
            bulk_g2s(Hs + (size_t)r_ * DPS_, S.states + (size_t)(nb + own.lo + c0 + r_) * CW + (l - 1) * HID, 128u,
                     &mbar[2]);
        }
        // (1) data gradient of the own nodes:  d h_{l-1}[u] = [Q[u] | dpre[u]] . [W_r^T ; root^T],
        //     Q[u,r,:] = sum_{(u->d) of type r, kept} dpre[d,:]/deg(d)         -> pushed to every CTA's DH
        gather_segments<8, PR>(Ls, K, Ls.segbase[c0], Ls.segbase[c0 + crow], lane, DPS, stage, SS, HID, R, &ws[33], rinv);
        __syncthreads();
        if (tid == 0) ws[33] = 0;
        {   // fold the extra segments of long lists into their node row
          const int kq = K1 >> 2, SS4 = SS >> 2;
          float4* st4 = reinterpret_cast<float4*>(stage);
          for (int r = warp; r < crow; r += nwarps) {
            const int e = Ls.ex[c0 + r], x0 = e & 0xffff, nex = e >> 16;
            if (nex == 0) continue;
            for (int k4 = lane; k4 < kq; k4 += 32) {
              float4 t = st4[(size_t)r * SS4 + k4];
              for (int j = 0; j < nex; ++j) {
                const float4 u = st4[(size_t)(crow + x0 + j) * SS4 + k4];
                t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
              }
              st4[(size_t)r * SS4 + k4] = t;
            }
          }
        }
        if (crow < chunk) {   // short (last) chunk: the K-padding rows of Hs must be zero (TMA fills rows < crow only)
          const int zr = a8(crow) - crow;
          for (int idx = tid; idx < zr * 8; idx += NT)
            *reinterpret_cast<float4*>(Hs + (size_t)(crow + (idx >> 3)) * DPS_ + ((idx & 7) << 2)) =
                make_float4(0.f, 0.f, 0.f, 0.f);
        }
        IGMC_STAMP(sb + 5);
        __syncthreads();
        IGMC_STAMP(sb + 6);
        if (c0 == 0) { mbar_wait(&mbar[1], wuse & 1u); ++wuse; }   // [W_r^T ; root^T] has landed
        const int mt = (crow + 15) >> 4;
        for (int item = warp; item < mt * 2; item += nwarps) {   // warp = (16-row block, 16-column half)
          const int m0 = (item >> 1) << 4, nh = (item & 1) << 4;
          const int ar = lane & 15, ac = (lane >> 4) << 2, br = (lane & 7) | ((lane >> 1) & 8), bc = (lane >> 1) & 4;
          TileAcc T[2];
          tile_zero(T[0]); tile_zero(T[1]);
          const uint32_t bs = smem_u32(Wn + (nh + br) * KS + bc);
          tiles_span(T, smem_u32(stage + (m0 + ar) * SS + ac), bs, K1p);
          const int r0 = c0 + m0 + gq, r1 = r0 + 8;
          tiles_span2(T, smem_u32(DP + min(c0 + m0 + ar, own_cap16 - 1) * DPS_ + ac), 0, bs + 4 * K1p, HID);
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            float d[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) d[q] = (T[i].d[q] + T[i].d2[q]) + (T[i].e[q] + T[i].e2[q]);
            const int cc = nh + 8 * i + 2 * tq;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              const int r = half ? r1 : r0;
              if (r < n_own) {
                const int u = own.lo + r;
                float2 o = make_float2(d[2 * half], d[2 * half + 1]);
                if (ext) {
                  const float2 sd = __ldg(reinterpret_cast<const float2*>(S.dstate + (size_t)(nb + u) * CW + (l - 1) * HID + cc));
                  o.x += sd.x; o.y += sd.y;
                }
                if (u == tu) { o.x += dfeat[(l - 1) * HID + cc]; o.y += dfeat[(l - 1) * HID + cc + 1]; }
                if (u == ti) { o.x += dfeat[CW + (l - 1) * HID + cc]; o.y += dfeat[CW + (l - 1) * HID + cc + 1]; }
                const int off = hix(u, cc);
                *reinterpret_cast<float2*>(DHn + off) = o;
#pragma unroll
                for (int pr = 0; pr < 3; ++pr)
                  if (pr + 1 < CL) st_async_peer(DHn + off, o, xbar, peer_rank(rank, pr, CL));
              }
            }
          }
        }
        IGMC_STAMP(sb + 1);
        // the weight-gradient tiles below touch neither peer memory nor the buffer the peers are writing (DHn)
        // (2) weight gradients over the chunk's rows:  D[k][(r,j) | j'] += sum_u h_{l-1}[u][k] [Q[u] | dpre[u]]
        //     M = 32 (k, two 16-row tiles), N = (R+1)*32, K = crow nodes; warp = (m tile, every (nwarps/2)-th n tile)
        mbar_wait(&mbar[2], huse & 1u); ++huse;            // the chunk's h_{l-1} rows have landed
        // a warp owns up to MAXI column tiles per pass; more (R > 7 at 16 warps) take further passes over the nodes
        for (int jp = warp >> 1; jp < NTN; jp += 4 * (nwarps >> 1)) {
          constexpr int MAXI = 4;
          const int m0 = (warp & 1) << 4, jn0 = jp, jstep = nwarps >> 1;
          float acc[MAXI][4], acs[MAXI][4];
#pragma unroll
          for (int i = 0; i < MAXI; ++i)
#pragma unroll
            for (int c = 0; c < 4; ++c) { acc[i][c] = 0.f; acs[i][c] = 0.f; }
          const int krows = a8(crow);                       // rows beyond crow: Hs is zero there, stage/DP are finite
          // B fragments (k = node, n = column of [Q | dpre]): base pointer and row stride of each of the warp's column
          // tiles, fixed over the node loop
          const float* bb[MAXI];
          int bst[MAXI];
          int cnt = 0;
#pragma unroll
          for (int i = 0; i < MAXI; ++i) {
            const int jn = jn0 + i * jstep, n0 = jn << 3;
            if (jn < NTN) cnt = i + 1;
            const bool q = n0 < K1 || jn >= NTN;
            bb[i] = jn >= NTN ? stage : q ? stage + (size_t)tq * SS + n0 + gq
                                          : DP + (size_t)(c0 + tq) * DPS_ + (n0 - K1) + gq;
            bst[i] = q ? SS : DPS_;
          }
          const float* ha = Hs + (size_t)tq * DPS_ + m0 + gq;   // A^T fragment: row = k (m0+g), col = node (k0+t)
          switch (cnt) {   // (uniform over the warp) one straight-line node loop per tile count
            case 4: wgrad_pass<4>(ha, bb, bst, krows, acc, acs); break;
            case 3: wgrad_pass<3>(ha, bb, bst, krows, acc, acs); break;
            case 2: wgrad_pass<2>(ha, bb, bst, krows, acc, acs); break;
            default: wgrad_pass<1>(ha, bb, bst, krows, acc, acs); break;
          }
#pragma unroll
          for (int i = 0; i < MAXI; ++i) {
            const int jn = jn0 + i * jstep;
            if (jn < NTN) {
              const int c = (jn << 3) + 2 * tq;             // column of [dW_0 .. dW_{R-1} | d root]
              const int k = m0 + gq;
              // raw layout: dW_r[k][j] at (r*32 + k)*32 + j, d root[k][j] at R*32*32 + k*32 + j
              float* o0 = gpl + (size_t)(((c >> 5) * HID + k) * HID + (c & 31));
              float* o1 = o0 + 8 * HID;
              float2 v0 = make_float2(acc[i][0] + acs[i][0], acc[i][1] + acs[i][1]);
              float2 v1 = make_float2(acc[i][2] + acs[i][2], acc[i][3] + acs[i][3]);
              if (c0 > 0) {   // later chunks accumulate into the row this thread wrote before (same thread, no race)
                const float2 p0 = *reinterpret_cast<const float2*>(o0), p1 = *reinterpret_cast<const float2*>(o1);
                v0.x += p0.x; v0.y += p0.y; v1.x += p1.x; v1.y += p1.y;
              }
              *reinterpret_cast<float2*>(o0) = v0;
              *reinterpret_cast<float2*>(o1) = v1;
            }
          }
        }
        IGMC_STAMP(sb + 7);
        __syncthreads();   // stage / Hs are free for the next chunk
      }
      if (n_own == 0) {   // nothing ran: keep the barrier phases in step and write the zero gradient block
        mbar_wait(&mbar[1], wuse & 1u); ++wuse;
        for (int i = tid; i < (R + 1) * HID * HID; i += NT) gpl[i] = 0.f;
      }
    } else {
      // layer 0: dW[kk][j] = sum_v A[v][kk] dpre[v][j],  A[v] = [ AGG'[v,r,k] (saved, 1/deg-scaled) | x[v,k] one-hot ]
      //          M = KRp rows, N = 32, K = own nodes
      const int TS = KRp + 8;                              // tile row stride (== 8 mod 32: conflict-free A^T frags)
      int trows = (int)(((size_t)(chunk + XR) * SSmax) / TS) & ~7;   // node rows of one tile pass
      if (trows > a8(n_own)) trows = a8(n_own);
      const int mt = (KRp + 15) >> 4;
      constexpr int MAXT = 4;
      float acc[MAXT][4], acs[MAXT][4];
#pragma unroll
      for (int i = 0; i < MAXT; ++i)
#pragma unroll
        for (int c = 0; c < 4; ++c) { acc[i][c] = 0.f; acs[i][c] = 0.f; }
      for (int t0 = 0; t0 < a8(n_own) && trows > 0; t0 += trows) {
        const int rows = min(trows, a8(n_own) - t0);        // multiple of 8, rows beyond n_own are zero
        {   // tile[r][0..K1) = saved aggregate, [K1..K1p) = 0, [K1p..KRp) = one-hot input; rows beyond n_own are zero
          const int kq = K1 >> 2, TS4 = TS >> 2;
          float4* t4 = reinterpret_cast<float4*>(stage);
          const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
          const float* zbase = S.zsave + (size_t)(nb + own.lo + t0) * (size_t)K1;
          for (int idx = tid; idx < rows * kq; idx += NT) {
            const int r_ = idx / kq, k4 = idx - r_ * kq;
            float4 val = z4;
            if (t0 + r_ < n_own) val = __ldcg(reinterpret_cast<const float4*>(zbase + (size_t)r_ * K1) + k4);
            t4[r_ * TS4 + k4] = val;
          }
          const int tail = KRp - K1;   // zero padding of the aggregate + the one-hot input columns
          for (int idx = tid; idx < rows * tail; idx += NT) {
            const int r_ = idx / tail, q = idx - r_ * tail, kk = K1 + q;
            float hv = 0.f;
            const int k = kk - K1p;
            if (k >= 0 && k < in && t0 + r_ < n_own) hv = (k == (int)node_label[nb + own.lo + t0 + r_]) ? 1.f : 0.f;
            stage[(size_t)r_ * TS + kk] = hv;
          }
        }
        __syncthreads();
        for (int k0 = 0; k0 < rows; k0 += 8) {
#pragma unroll
          for (int i = 0; i < MAXT; ++i) {
            const int tile = warp + i * nwarps;
            if (tile < mt * 4) {
              const int m0 = (tile >> 2) << 4, n0 = (tile & 3) << 3;
              const bool hi_ok = (m0 + 8) < KRp;               // KRp may be an odd multiple of 8
              const float* a = stage + (size_t)(k0 + tq) * TS + m0 + gq;
              const float* bp = DP + (size_t)(t0 + k0 + tq) * DPS_ + n0 + gq;
              const float af[4] = {a[0], hi_ok ? a[8] : 0.f, a[4 * TS], hi_ok ? a[4 * TS + 8] : 0.f};
              const float bf[2] = {bp[0], bp[4 * DPS_]};
              mma_3xtf32(acc[i], acs[i], af, bf);
            }
          }
        }
        __syncthreads();
      }
      // tile row kk -> raw row: kk < K1: dW (r*inp + k = kk); K1p <= kk < K1p + in: d root row kk - K1p
#pragma unroll
      for (int i = 0; i < MAXT; ++i) {
        const int tile = warp + i * nwarps;
        if (tile < mt * 4) {
          const int m0 = (tile >> 2) << 4, n0 = (tile & 3) << 3, cc = n0 + 2 * tq;
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int kk = m0 + gq + 8 * half;
            const float2 v = make_float2(acc[i][2 * half] + acs[i][2 * half], acc[i][2 * half + 1] + acs[i][2 * half + 1]);
            if (kk < K1) *reinterpret_cast<float2*>(gpl + (size_t)kk * HID + cc) = v;
            else if (kk >= K1p && kk < K1p + in) *reinterpret_cast<float2*>(gpl + (size_t)(K1 + kk - K1p) * HID + cc) = v;
          }
        }
      }
      IGMC_STAMP(sb + 2);
    }
    __syncthreads();
    IGMC_STAMP(sb + 3);
    // (3) every CTA's DH holds d h_{l-1} of all nodes once the pushes have landed; the next layer's weight slab is
    //     requested while they do (every read of Wn is behind the barrier above)
    if (l > 1) load_weights(l - 1);
    if (CL > 1 && l > 0) mbar_wait_cluster(xbar, (uint32_t)(((L - 1 - l) >> 1) & 1));   // (layer 0 exchanges nothing)
    IGMC_STAMP(sb + 4);
  }
  IGMC_WALL(54);
}

template <int NTMAX, bool PR>
__global__ void __launch_bounds__(NTMAX, 1)
k_backward_rs(igmc_model_t M, const float* __restrict__ params, const uint8_t* __restrict__ node_label,
              const int32_t* __restrict__ node_ptr, const int32_t* __restrict__ edge_ptr, igmc_adj_t A, int n_cap,
              int lcap, int chunk, igmc_dropout_t D, igmc_saved_t S, const float* __restrict__ dpred,
              float* __restrict__ gpart, float* __restrict__ dhid_out, igmc_stage_t IMG, int* err) {
  extern __shared__ __align__(16) float smem[];
  backward_body<NTMAX, PR>(M, params, node_label, node_ptr, edge_ptr, A, n_cap, lcap, chunk, D, S, dpred, gpart, dhid_out,
                       IMG, err, smem);
}

// Forward and backward of one subgraph in ONE kernel (training): the loss gradient of a subgraph depends on its own
// forward only (dpred[g] = 2 (out_g - y_g) / G), so a cluster goes straight from its readout into its backward - no
// second launch, and the spread of the forward times over the clusters is not paid twice (every cluster used to wait
// for the slowest forward before any backward could start).  The shared memory is re-carved for the backward; what the
// backward reads of the forward travels through global memory exactly as between the two separate kernels, ordered
// by a device fence + cluster barrier (the peer CTA wrote half of the states / inv_deg / rel_inv_deg rows, rank 0 the
// readout).
template <int NTMAX, bool PR>
__global__ void __launch_bounds__(NTMAX, 1)
k_train_rs(igmc_model_t M, const float* __restrict__ params, const uint8_t* __restrict__ node_label,
           const int32_t* __restrict__ node_ptr, const int32_t* __restrict__ edge_ptr, igmc_adj_t A, int n_cap,
           int lcap_f, int chunk_f, int lcap_b, int chunk_b, igmc_dropout_t D, igmc_saved_t S,
           const float* __restrict__ y, float loss_scale, float* __restrict__ dpred, float* __restrict__ sqerr,
           float* __restrict__ gpart, float* __restrict__ dhid_out, igmc_stage_t IMGF, igmc_stage_t IMGB, int* err) {
  extern __shared__ __align__(16) float smem[];
  const bool ok = forward_body<NTMAX, PR>(M, params, node_label, node_ptr, edge_ptr, A, n_cap, lcap_f, chunk_f, D, 1, S, y,
                                      loss_scale, dpred, sqerr, IMGF, err, smem);
  if (!ok) return;   // uniform over the cluster
  __threadfence();
  asm volatile("fence.proxy.async;" ::: "memory");   // the backward's bulk copies read state rows written above
  cg::this_cluster().sync();   // (a cluster of one CTA: a block barrier)
  backward_body<NTMAX, PR>(M, params, node_label, node_ptr, edge_ptr, A, n_cap, lcap_b, chunk_b, D, S, dpred, gpart,
                       dhid_out, IMGB, err, smem);
}

// ------------------------------------------------------------------------------------------------
// list images: what stage_lists builds, once per batch and off the model kernels' critical path
// grid = (B * CL, 2): blockIdx.y = 0 forward (in-lists, kept in-degree), 1 backward (out-lists / mirrored in-lists)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512)
k_stage_lists(const int32_t* __restrict__ node_ptr, const int32_t* __restrict__ edge_ptr, igmc_adj_t A, int n_cap,
              int CL, igmc_dropout_t D, int training, igmc_stage_t F, igmc_stage_t Bw) {
  extern __shared__ __align__(16) int smem_i[];
  __shared__ int ws[34];
  const int dir = blockIdx.y;
  const igmc_stage_t I = dir ? Bw : F;
  const int blk = blockIdx.x, g = blk / CL, rank = blk % CL;
  const int tid = threadIdx.x, NT = blockDim.x;
  const int own_cap = own_cap_of(n_cap, CL);
  int* ibuf = smem_i + IMG_HDR;
  uint32_t* lbuf = reinterpret_cast<uint32_t*>(ibuf + a4(list_ints(own_cap)));
  const int nb = node_ptr[g], n = node_ptr[g + 1] - nb;
  const int eb = edge_ptr[g], m_half = (edge_ptr[g + 1] - eb) >> 1;
  int32_t* gt = I.tab + (size_t)blk * I.tab_ints;
  if (n > n_cap) {   // the model kernels flag IGMC_ERR_SMEM_NODES and never look at the image
    if (tid < IMG_HDR) gt[tid] = 0;
    return;
  }
  const EdgeKeep K = make_keep(D, training);
  const bool sym = A.symmetric != 0;
  const Split own = own_range(n, rank, CL);
  if (dir == 0)
    stage_lists(A.in_adj, A.in_eid, A.in_ptr, nb, own.lo, own.hi, K, false, eb, m_half, lbuf, I.lcap, ibuf, own_cap,
                I.chunk, ws, nullptr, I.inv_deg);
  else
    stage_lists(sym ? A.in_adj : A.out_adj, sym ? A.in_eid : A.out_eid, sym ? A.in_ptr : A.out_ptr, nb, own.lo, own.hi,
                K, sym, eb, m_half, lbuf, I.lcap, ibuf, own_cap, I.chunk, ws, nullptr, nullptr);
  const int total = smem_i[0], staged = smem_i[2];
  for (int i = tid; i < I.tab_ints; i += NT) gt[i] = smem_i[i];
  if (staged) {
    uint32_t* ge = I.ent + (size_t)blk * I.lcap;
    for (int i = tid; i < a4(total); i += NT) ge[i] = i < total ? lbuf[i] : 0u;
  }
}

size_t fwd_base_fl(int n_cap, int R, int L, int CL) {   // everything except the stage rows and the list buffer
  const size_t F = 2 * HID * L;
  const size_t own_cap = (size_t)own_cap_of(n_cap, CL);
  return 2 * (size_t)n_cap * HID + wprep_slab(R) + HID + a4(n_cap) + a4((int)F) + L1O + img_ints((int)own_cap) +
         (size_t)XR * ((size_t)R * HID + 4);
}
size_t bwd_base_fl(int n_cap, int R, int L, int CL) {   // everything except the (stage + Hs) rows and the list buffer
  const size_t F = 2 * HID * L;
  const size_t own_cap = (size_t)own_cap_of(n_cap, CL), own_cap16 = (size_t)a16((int)own_cap);
  return 2 * (size_t)n_cap * HID + own_cap16 * DPS_ + wprep_slab(R) + a4(n_cap) + a4((int)F) + L1O +
         img_ints((int)own_cap) + (size_t)XR * ((size_t)R * HID + 4);
}

}  // namespace rs

// ---- host-side dispatch helpers used by rgcn.cu's extern "C" entry points ----------------------------------
int rs_supported(const igmc_model_t* M) { return M->num_relations <= rs::RS_MAX_R; }

// threads per CTA, dynamic shared memory, stage chunk rows and edge-list staging capacity for a plan
int rs_plan(const igmc_model_t* M, int n_cap, int cluster, int backward, int* threads, size_t* smem, int* lcap, int* chunk) {
  const size_t limit = 227 * 1024 - 1024;   // static shared memory of the kernels (scan scratch, mbarriers) counts too
  const int R = M->num_relations;
  const size_t SSmax = (size_t)R * rs::HID + 4;
  const size_t rowfl = SSmax + (backward ? rs::DPS_ : 0);   // a chunk row: staging row (+ its h_{l-1} row, backward)
  const size_t base = 4 * (backward ? rs::bwd_base_fl(n_cap, R, M->num_layers, cluster)
                                    : rs::fwd_base_fl(n_cap, R, M->num_layers, cluster));
  const int own16 = rs::a16(rs::own_cap_of(n_cap, cluster));
  // weight-gradient accumulators: ceil(8 (R+1) tiles / nwarps) per warp must be <= 4
  const int tiles = 4 * ((R + 1) * rs::HID / 16);
  // stage rows: as many as fit (multiple of 16, at least 16), leaving >= 4 KB for the edge lists
  if (base + 4096 + 16 * rowfl * 4 > limit) return -3;
  size_t rows = (limit - base - 4096) / (rowfl * 4);
  rows &= ~(size_t)15;
  if (rows > (size_t)own16) rows = own16;
  size_t left = limit - base - rows * rowfl * 4;
  size_t lc = (left / 4) & ~(size_t)3;
  // a list that does not fit is gathered through global memory (3-4x slower per layer): trade staging rows for list
  // capacity down to 32 rows when the caller knows how long the lists get
  const size_t hint = M->list_hint > 0 ? (size_t)(M->list_hint > 16384 ? 16384 : M->list_hint) : 0;
  while (lc < hint && rows > 32) {
    rows -= 16;
    left = limit - base - rows * rowfl * 4;
    lc = (left / 4) & ~(size_t)3;
  }
  if (lc > 16384) lc = 16384;
  {
    // 1024 threads (64 registers) or 512 threads (128 registers: no address rematerialisation, fewer instructions)
    static int nt_env = -1;
    if (nt_env < 0) {
      const char* e = getenv("IGMC_RS_THREADS");
      nt_env = e ? atoi(e) : 0;
    }
    // 512 threads x 128 registers for every R <= 12: beyond 4 weight-gradient column tiles per warp (R > 7) the tiles
    // run in a second pass over the nodes.  1024 threads leave 64 registers per thread, and the kernels spill there.
    int nt = 512;
    if (nt_env == 512 || nt_env == 1024) nt = nt_env;
    (void)tiles;
    *threads = nt;
  }
  *chunk = (int)rows;
  *lcap = (int)lc;
  *smem = base + rows * rowfl * 4 + lc * 4;
  return 0;
}

static int pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("IGMC_PDL");
    v = e ? atoi(e) : 0;   // off by default: a pre-launched grid that cannot be placed yet blocks the dispatch of the
                            // extraction kernel of the other stream
  }
  return v;
}

// the image a kernel is handed must have been built for exactly its plan
static int check_image(const igmc_stage_t* I, int n_cap, int cluster, int lcap, int chunk, igmc_stage_t* out) {
  igmc_stage_t none = {};
  *out = none;
  if (!I || !I->tab) return 0;
  if (I->cluster != cluster || I->chunk != chunk || I->lcap != lcap ||
      I->tab_ints != rs::img_ints(rs::own_cap_of(n_cap, cluster)) || !I->ent)
    return -19;
  *out = *I;
  return 0;
}

int rs_stage_plan(const igmc_model_t* M, int n_cap, int cluster, int backward, igmc_stage_t* img) {
  int threads, lcap, chunk;
  size_t smem;
  int rc = rs_plan(M, n_cap, cluster, backward, &threads, &smem, &lcap, &chunk);
  if (rc) return rc;
  img->tab_ints = rs::img_ints(rs::own_cap_of(n_cap, cluster));
  img->lcap = lcap;
  img->chunk = chunk;
  img->cluster = cluster;
  return 0;
}

int rs_stage_lists(const igmc_model_t* M, const int32_t* node_ptr, const int32_t* edge_ptr, const igmc_adj_t* A, int B,
                   int n_cap, const igmc_dropout_t* D, int training, const igmc_stage_t* fwd, const igmc_stage_t* bwd,
                   cudaStream_t st) {
  if (!fwd || !fwd->tab || !fwd->ent || !fwd->inv_deg) return -19;
  const int cluster = fwd->cluster;
  igmc_stage_t want;
  int rc = rs_stage_plan(M, n_cap, cluster, 0, &want);
  if (rc) return rc;
  if (want.tab_ints != fwd->tab_ints || want.lcap != fwd->lcap || want.chunk != fwd->chunk) return -19;
  const bool both = training && bwd && bwd->tab;
  igmc_stage_t bw = {};
  int lcmax = fwd->lcap;
  if (both) {
    rc = rs_stage_plan(M, n_cap, cluster, 1, &want);
    if (rc) return rc;
    if (want.tab_ints != bwd->tab_ints || want.lcap != bwd->lcap || want.chunk != bwd->chunk || bwd->cluster != cluster ||
        !bwd->ent)
      return -19;
    bw = *bwd;
    if (bw.lcap > lcmax) lcmax = bw.lcap;
  }
  const size_t smem = ((size_t)fwd->tab_ints + (size_t)lcmax) * 4;
  cudaFuncSetAttribute(rs::k_stage_lists, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  rs::k_stage_lists<<<dim3(B * cluster, both ? 2 : 1), 512, smem, st>>>(node_ptr, edge_ptr, *A, n_cap, cluster, *D,
                                                                        training, *fwd, bw);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e + 1000;
}

int rs_forward(const igmc_model_t* M, const float* params, const uint8_t* node_label, const int32_t* node_ptr,
               const int32_t* edge_ptr, const igmc_adj_t* A, int B, int n_cap, const igmc_dropout_t* D, int training,
               const igmc_saved_t* S, const float* y, float loss_scale, float* dpred, float* sqerr, int cluster,
               const igmc_stage_t* stage, int* err, cudaStream_t st) {
  int threads, lcap, chunk;
  size_t smem;
  int rc = rs_plan(M, n_cap, cluster, 0, &threads, &smem, &lcap, &chunk);
  if (rc) return rc;
  igmc_stage_t img;
  rc = check_image(stage, n_cap, cluster, lcap, chunk, &img);
  if (rc) return rc;
  if (img.tab && !img.inv_deg) return -19;
  const bool pr = S->rel_inv_deg != nullptr;
  auto kern = threads == 512 ? (pr ? rs::k_forward_rs<512, true> : rs::k_forward_rs<512, false>)
                             : (pr ? rs::k_forward_rs<1024, true> : rs::k_forward_rs<1024, false>);
  return launch_cluster(kern, B * cluster, threads, smem, cluster, false, st, *M, params, node_label, node_ptr, edge_ptr,
                        *A, n_cap, lcap, chunk, *D, training, *S, y, loss_scale, dpred, sqerr, img, err);
}

int rs_backward(const igmc_model_t* M, const float* params, const uint8_t* node_label, const int32_t* node_ptr,
                const int32_t* edge_ptr, const igmc_adj_t* A, int B, int n_cap, const igmc_dropout_t* D,
                const igmc_saved_t* S, const float* dpred, float* gpart, float* dhid, int cluster,
                const igmc_stage_t* stage, int* err, cudaStream_t st) {
  int threads, lcap, chunk;
  size_t smem;
  int rc = rs_plan(M, n_cap, cluster, 1, &threads, &smem, &lcap, &chunk);
  if (rc) return rc;
  igmc_stage_t img;
  rc = check_image(stage, n_cap, cluster, lcap, chunk, &img);
  if (rc) return rc;
  const bool pr = S->rel_inv_deg != nullptr;
  auto kern = threads == 512 ? (pr ? rs::k_backward_rs<512, true> : rs::k_backward_rs<512, false>)
                             : (pr ? rs::k_backward_rs<1024, true> : rs::k_backward_rs<1024, false>);
  // IGMC_PDL bit 0: the backward may start under the tail of the forward (bit 1: the update kernel, csrc/optim.cu)
  const bool pdl = pdl_enabled() & 1;
  return launch_cluster(kern, B * cluster, threads, smem, cluster, pdl, st, *M, params, node_label, node_ptr, edge_ptr,
                        *A, n_cap, lcap, chunk, *D, *S, dpred, gpart, dhid, img, err);
}

namespace rs {
// gate[0]: CTAs of gated forwards that have started, ever (never reset); gate[1]: the total this and all earlier gates
// expect.  Every gate is followed by exactly one forward that was handed the gate (the host arms it per launch), so
// the count catches up with the expectation once that forward is resident; un-gated forwards do not touch the counter
// and a timed-out gate does not desynchronise the pair (late arrivals still count towards the same total).
__global__ void k_gate_wait(int* gate, int target, long long timeout_ns) {
  if (threadIdx.x == 0) {
    const int expect = gate[1] + target;
    gate[1] = expect;
    const long long t0 = igmc_globaltimer();
    while (*reinterpret_cast<volatile int*>(gate) - expect < 0 && igmc_globaltimer() - t0 < timeout_ns) __nanosleep(64);
  }
}
}  // namespace rs

int rs_gate_wait(int* gate, int target, int timeout_us, cudaStream_t st) {
  rs::k_gate_wait<<<1, 32, 0, st>>>(gate, target, (long long)timeout_us * 1000);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e + 1000;
}

int rs_train(const igmc_model_t* M, const float* params, const uint8_t* node_label, const int32_t* node_ptr,
             const int32_t* edge_ptr, const igmc_adj_t* A, int B, int n_cap, const igmc_dropout_t* D,
             const igmc_saved_t* S, const float* y, float loss_scale, float* dpred, float* sqerr, float* gpart,
             float* dhid, int cluster, const igmc_stage_t* stage_f, const igmc_stage_t* stage_b, int* err,
             cudaStream_t st) {
  int tf, tb, lcf, lcb, chf, chb;
  size_t smf, smb;
  int rc = rs_plan(M, n_cap, cluster, 0, &tf, &smf, &lcf, &chf);
  if (rc) return rc;
  rc = rs_plan(M, n_cap, cluster, 1, &tb, &smb, &lcb, &chb);
  if (rc) return rc;
  if (tf != tb) return -3;
  igmc_stage_t imf, imb;
  rc = check_image(stage_f, n_cap, cluster, lcf, chf, &imf);
  if (rc) return rc;
  if (imf.tab && !imf.inv_deg) return -19;
  rc = check_image(stage_b, n_cap, cluster, lcb, chb, &imb);
  if (rc) return rc;
  const size_t smem = smf > smb ? smf : smb;
  const bool pr = S->rel_inv_deg != nullptr;
  auto kern = tf == 512 ? (pr ? rs::k_train_rs<512, true> : rs::k_train_rs<512, false>)
                        : (pr ? rs::k_train_rs<1024, true> : rs::k_train_rs<1024, false>);
  return launch_cluster(kern, B * cluster, tf, smem, cluster, false, st, *M, params, node_label, node_ptr, edge_ptr, *A,
                        n_cap, lcf, chf, lcb, chb, *D, *S, y, loss_scale, dpred, sqerr, gpart, dhid, imf, imb, err);
}

int rs_prep_weights(const igmc_model_t* M, const float* params, float* wprep, cudaStream_t st) {
  rs::k_prep_weights<<<M->num_layers * 2 * 32, 256, 0, st>>>(*M, params, wprep);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e + 1000;
}
