// The guide blob view and the warp-cooperative transition, shared by the target-row kernels (sq_guide.cu) and the
// draft-row kernel (sq_draft_rows.cu).  Layout and step() in include/sequoia_b200.h.
#pragma once
#include "sq_common.cuh"

namespace sq {

// The parts of one guide blob (layout in include/sequoia_b200.h).
struct GuideView {
  int n, W, E;
  const int32_t* default_next;
  const int32_t* edge_off;
  const int32_t* edge_id;
  const int32_t* edge_next;
  const uint32_t* mask;
  __device__ __forceinline__ explicit GuideView(const int32_t* g) {
    n = g[0];
    W = g[1];
    E = g[2];
    default_next = g + SQ_GUIDE_HEADER;
    edge_off = default_next + n;
    edge_id = edge_off + n + 1;
    edge_next = edge_id + E;
    mask = reinterpret_cast<const uint32_t*>(edge_next + E);
  }
  __device__ __forceinline__ const uint32_t* row(int s) const { return mask + (int64_t)s * W; }
};

// step(s, t) for the whole warp (every lane gets the result).  All lanes must call it with the same s and t.
__device__ __forceinline__ int guide_step(const GuideView& g, int s, int64_t t, int V) {
  if (s < 0 || s >= g.n || t < 0 || t >= V) return -1;
  const int id = (int)t;
  const int lane = threadIdx.x & 31;
  // independent loads first: the allowed bit, the edge range, the default
  const uint32_t word = g.row(s)[id >> 5];
  int lo = g.edge_off[s], hi = g.edge_off[s + 1];
  const int dflt = g.default_next[s];
  if (!((word >> (id & 31)) & 1u)) return -1;
  while (hi - lo > 32) {                                // pivots at lo + lane*n/32: ascending, lane 0's is lo
    const int n = hi - lo;
    const int p = lo + (int)(((int64_t)lane * n) >> 5);
    const unsigned le = __ballot_sync(0xffffffffu, g.edge_id[p] <= id);
    if (le == 0u) return dflt;                          // below the first edge id
    const int L = 31 - __clz(le);                       // the last pivot <= id: t lies in [pivot L, pivot L+1)
    const int nlo = lo + (int)(((int64_t)L * n) >> 5);
    hi = L == 31 ? hi : lo + (int)(((int64_t)(L + 1) * n) >> 5);
    lo = nlo;
  }
  const int q = lo + lane;
  const unsigned hit = __ballot_sync(0xffffffffu, q < hi && g.edge_id[q] == id);
  if (hit == 0u) return dflt;
  return g.edge_next[lo + __ffs(hit) - 1];
}

__device__ __forceinline__ const int32_t* guide_of(const int64_t* table, const int32_t* st, int b) {
  if (st[ST_FROZEN] || !st[ST_GUIDED]) return nullptr;
  return reinterpret_cast<const int32_t*>(table[b]);
}

}  // namespace sq
