// The rank-counting merge shared by k_topk_merge (recommend.cu) and k_infl_topk (influence.cu): a running ranked
// list of k entries merged with one batch in shared memory, every entry placed by the number of entries ranked
// before it.
#pragma once

#include "common.cuh"

namespace {

constexpr int MERGE_HEAD = 16;   // the head of the merge's dynamic shared memory (k_topk_merge: the segment-end word)

// dynamic shared memory of one merge CTA (the kernels have no static shared memory): the head and (k + B) entries of an
// int64 id and an fp32 value
inline size_t merge_smem(int k, int B) { return MERGE_HEAD + (size_t)(k + B) * (sizeof(long long) + sizeof(float)); }

// a ranks before b under key sign * value: key descending, id ascending, NaN after every number (NaNs among
// themselves by id), empty slots (id < 0) last
__device__ __forceinline__ bool ranks_before(float av, long long ai, float bv, long long bi, float sign) {
  if (ai < 0) return false;
  if (bi < 0) return true;
  const float ak = sign * av, bk = sign * bv;
  const bool an = isnan(ak), bn = isnan(bk);
  if (an || bn) return (an && bn) ? ai < bi : bn;
  return ak > bk || (ak == bk && ai < bi);
}

// V / I [n] in shared memory: the running list [0, k) (ranked, empty slots last) and the batch [k, n) (entries with id
// < 0 skipped).  Every kept entry's rank is the number of entries ranked before it (distinct ids: a permutation), and
// the first k by rank are written to out_v / out_i.  The caller's block has filled V and I and passed a barrier.
__device__ __forceinline__ void rank_merge(const float* V, const long long* I, int k, int n, float sign,
                                           float* __restrict__ out_v, int64_t* __restrict__ out_i) {
  for (int e = threadIdx.x; e < n; e += blockDim.x) {
    const float ev = V[e];
    const long long ei = I[e];
    if (e >= k && ei < 0) continue;
    int r;
    if (e < k) {
      r = e;
    } else {
      int lo = 0, hi = k;   // the running list is ranked: binary search for the first entry not before e
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ranks_before(V[mid], I[mid], ev, ei, sign)) lo = mid + 1; else hi = mid;
      }
      r = lo;
    }
    for (int x = k; x < n && r < k; ++x)
      if (x != e && ranks_before(V[x], I[x], ev, ei, sign)) ++r;
    if (r < k) {
      out_v[r] = ev;
      out_i[r] = ei;
    }
  }
}

}  // namespace
