// Device code shared by the in-place graph update (graph_update.cu) and the rating-session rows (session.cu): the
// classification of a kept delta entry, the packed (inserted, deleted) counts, the binary search in a sorted row, the
// per-row runs of a sorted delta and the warp merge of one row with its run.
#pragma once

#include "common.cuh"

namespace {

enum : uint8_t { C_NOOP = 0, C_INSERT = 1, C_CHANGE = 2, C_DELETE = 3 };

// packed (inserted, deleted) count: inserted in the high 32 bits, deleted in the low 32 (D < 2^31: a scan never carries)
__device__ __forceinline__ long long pack_count(uint8_t c) {
  return c == C_INSERT ? (1ll << 32) : c == C_DELETE ? 1ll : 0ll;
}
__device__ __forceinline__ long long net(long long p) { return (p >> 32) - (p & 0xffffffffll); }

inline int bits_for(unsigned long long n) {   // radix-sort bits of keys in [0, n)
  int b = 0;
  while (b < 64 && (1ull << b) < n) ++b;
  return b > 0 ? b : 1;
}

// first position in the ascending a[lo, hi) whose value is not below c (hi if none)
__device__ __forceinline__ int find_col(const int32_t* __restrict__ a, int lo, int hi, int c) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < c) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// the class of the kept entry (value x) against the base row's entry p (-1: absent) and its new label
__device__ __forceinline__ uint8_t classify(int x, int p, const uint8_t* __restrict__ rating, uint8_t* l) {
  *l = 0;
  if (x > 0) {
    *l = (uint8_t)(x - 1);
    return p < 0 ? C_INSERT : (rating[p] != *l ? C_CHANGE : C_NOOP);
  }
  return p >= 0 ? C_DELETE : C_NOOP;
}

// the run [ds, de) of delta entries of every row (column) that has one; others keep the memset 0 / 0
__global__ void k_runs(const long long* __restrict__ skey, int D, int stride, int32_t* __restrict__ ds,
                       int32_t* __restrict__ de) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < D; i += gridDim.x * blockDim.x) {
    const long long r = skey[i] / stride;
    if (i == 0 || skey[i - 1] / stride != r) ds[r] = i;
    if (i == D - 1 || skey[i + 1] / stride != r) de[r] = i + 1;
  }
}

// One warp merges the old entries [o0, o1) of a row and its delta run [d0, d1) (ascending other-side id, only the
// last entry of an equal-id group is kept) into [n0, n0 + len).  Old entry j goes to n0 + (j - o0) + (inserted -
// deleted entries of the run with a smaller id) unless it is deleted; an inserted entry to n0 + (old entries with a
// smaller id) + the same count.
template <bool RATING>
__device__ __forceinline__ void merge_row(const int32_t* __restrict__ idx, const uint8_t* __restrict__ rating, int o0,
                                          int o1, int d0, int d1, long long n0, const long long* __restrict__ skey,
                                          int stride, const uint8_t* __restrict__ cls,
                                          const uint8_t* __restrict__ lab, const int32_t* __restrict__ perm,
                                          const long long* __restrict__ scan, int32_t* __restrict__ out_idx,
                                          uint8_t* __restrict__ out_rating, int lane) {
  auto other = [&](int p) { return (int)(skey[p] % stride); };
  auto clsof = [&](int p) { return perm ? cls[perm[p]] : cls[p]; };
  if (d0 == d1) {            // untouched row: shifted only
    for (int j = o0 + lane; j < o1; j += 32) {
      out_idx[n0 + (j - o0)] = idx[j];
      if (RATING) out_rating[n0 + (j - o0)] = rating[j];
    }
    return;
  }
  const long long base = scan[d0];
  for (int j = o0 + lane; j < o1; j += 32) {
    const int c = idx[j];
    int lo = d0, hi = d1;     // first delta entry with id >= c
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (other(mid) < c) lo = mid + 1; else hi = mid;
    }
    int last = lo;            // the kept (last) entry of the group with id c, if any
    while (last + 1 < d1 && other(last + 1) == c) ++last;
    uint8_t k = C_NOOP;
    if (last < d1 && other(last) == c) k = clsof(last);
    if (k == C_DELETE) continue;
    const long long o = n0 + (j - o0) + net(scan[lo] - base);
    out_idx[o] = c;
    if (RATING) out_rating[o] = k == C_CHANGE ? lab[last] : rating[j];
  }
  for (int p = d0 + lane; p < d1; p += 32) {
    if (clsof(p) != C_INSERT) continue;
    const int c = other(p);
    const int q = find_col(idx, o0, o1, c) - o0;
    const long long o = n0 + q + net(scan[p] - base);
    out_idx[o] = c;
    if (RATING) out_rating[o] = lab[p];
  }
}

}  // namespace
