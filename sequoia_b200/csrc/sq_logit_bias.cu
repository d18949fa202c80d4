// Per-sequence allowed-token mask and logit bias on the (B*S, V) target rows of a batched tree
// (include/sequoia_b200.h, sq_logit_bias_rows_batch).  Stateless and tree-independent: every row of sequence b gets the
// same processing.  One launch, grid (chunks, S, B): CTA (c, k, b) owns ids [c*LB_CHUNK, (c+1)*LB_CHUNK) of row b*S + k.
//   1. Mask (has_mask[b]): the chunk in 8-entry groups (16-byte vectors when the rows are 16-byte aligned).  A group whose
//      8 mask bits are all set is not read; one whose bits are all clear is written as 8 x -inf without a read; a mixed one
//      is read, its disallowed entries set to -inf, and written back only if an entry changed.
//   2. Bias: the sequence's sorted (id, bias) entries that fall in the chunk, one thread per distinct id.  The chunk's
//      range [lo, hi) of entries is found by counting the ids below its ends with the whole CTA (one coalesced read of
//      the list instead of a chain of dependent binary-search loads), with __syncthreads_count, which also orders the
//      mask pass's writes of the same groups before the bias.  An entry is applied only if the id's mask bit is set (read
//      from the mask, never inferred from the logit), so no CTA reads what another writes.
#include "sq_common.cuh"

namespace sq {

constexpr int LB_THREADS = 256;
constexpr int LB_CHUNK = 4096;                          // ids per CTA: 2 groups of 8 per thread
constexpr int LB_GROUPS = LB_CHUNK / 8 / LB_THREADS;
constexpr int LB_IDS_PER_THREAD = SQ_MAX_LOGIT_BIAS / LB_THREADS;
constexpr uint16_t LB_NEG_INF = 0xFC00u;

__device__ __forceinline__ bool lb_allowed(const uint32_t* mask, int id) { return (mask[id >> 5] >> (id & 31)) & 1u; }

__global__ void __launch_bounds__(LB_THREADS)
    logit_bias_kernel(__half* __restrict__ logits, int64_t ld, int V, int S, const int32_t* __restrict__ state,
                      const uint32_t* __restrict__ allowed, int64_t allowed_words, const int32_t* __restrict__ has_mask,
                      const int32_t* __restrict__ bias_ids, const float* __restrict__ bias_vals,
                      const int32_t* __restrict__ n_bias, bool vec) {
  pdl_wait();
  pdl_trigger();
  const int c = blockIdx.x, k = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
  const bool masked = has_mask[b] != 0;
  const int nb = min(max(n_bias[b], 0), SQ_MAX_LOGIT_BIAS);
  if (state[b * ST_WORDS + ST_FROZEN] || (!masked && nb == 0)) return;
  const int c0 = c * LB_CHUNK, c1 = min(c0 + LB_CHUNK, V);
  __half* row = logits + ((int64_t)b * S + k) * ld;
  const uint32_t* mask = allowed + (int64_t)b * allowed_words;
  if (masked) {
#pragma unroll
    for (int g = 0; g < LB_GROUPS; ++g) {
      const int i = c0 + (g * LB_THREADS + tid) * 8;
      if (i >= c1) break;
      const uint32_t bits = (mask[i >> 5] >> (i & 31)) & 0xffu;   // (V % 8 == 0: a group never crosses V or a word)
      if (bits == 0xffu) continue;
      union {
        uint4 v;
        uint16_t h[8];
      } u;
      if (bits == 0u) {
#pragma unroll
        for (int e = 0; e < 8; ++e) u.h[e] = LB_NEG_INF;
      } else {
        if (vec) {
          u.v = *reinterpret_cast<const uint4*>(row + i);
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e) u.h[e] = reinterpret_cast<const uint16_t*>(row)[i + e];
        }
        bool changed = false;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          if (!((bits >> e) & 1u) && u.h[e] != LB_NEG_INF) {
            u.h[e] = LB_NEG_INF;
            changed = true;
          }
        }
        if (!changed) continue;
      }
      if (vec) {
        *reinterpret_cast<uint4*>(row + i) = u.v;
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) reinterpret_cast<uint16_t*>(row)[i + e] = u.h[e];
      }
    }
  }
  if (nb == 0) return;                                  // (uniform across the CTA: no thread waits below)
  const int32_t* ids = bias_ids + (int64_t)b * SQ_MAX_LOGIT_BIAS;
  const float* vals = bias_vals + (int64_t)b * SQ_MAX_LOGIT_BIAS;
  int mine[LB_IDS_PER_THREAD];
#pragma unroll
  for (int u = 0; u < LB_IDS_PER_THREAD; ++u) {
    const int j = u * LB_THREADS + tid;
    mine[u] = j < nb ? ids[j] : INT32_MAX;
  }
  int lo = 0, hi = 0;                                   // ascending ids: lower_bound(t) = the number of ids below t
#pragma unroll
  for (int u = 0; u < LB_IDS_PER_THREAD; ++u) {
    lo += __syncthreads_count(mine[u] < c0);
    hi += __syncthreads_count(mine[u] < c1);
  }
  for (int j = lo + tid; j < hi; j += LB_THREADS) {
    const int t = ids[j];
    if (t < 0 || t >= V || (j > lo && ids[j - 1] == t)) continue;   // a repeated id: its first entry applies them all
    if (masked && !lb_allowed(mask, t)) continue;
    float x = h2f(row[t]);
    if (!isfinite(x)) continue;
    for (int q = j; q < hi && ids[q] == t; ++q) {
      x = __fadd_rn(x, vals[q]);
      x = fminf(fmaxf(x, -65504.f), 65504.f);
      if (q + 1 < hi && ids[q + 1] == t) x = h2f(f2h(x));          // each entry rounds to fp16, as applied one by one
    }
    row[t] = f2h(x);
  }
}

}  // namespace sq

using namespace sq;

extern "C" int sq_logit_bias_rows_batch(sq_half* logits, int64_t ld, int V, int S, const int32_t* state,
                                        const uint32_t* allowed, int64_t allowed_words, const int32_t* has_mask,
                                        const int32_t* bias_ids, const float* bias_vals, const int32_t* n_bias, int B,
                                        void* stream) {
  SQ_CHECK_ARG(logits && state && allowed && has_mask && bias_ids && bias_vals && n_bias,
               "sq_logit_bias_rows_batch: null array");
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH, "sq_logit_bias_rows_batch: B=%d (1..%d)", B, SQ_MAX_BATCH);
  SQ_CHECK_ARG(V % 8 == 0 && V > 0 && V <= 131072, "sq_logit_bias_rows_batch: V=%d must be a multiple of 8, <= 131072",
               V);
  SQ_CHECK_ARG(ld >= V, "sq_logit_bias_rows_batch: ld=%lld < V=%d", (long long)ld, V);
  SQ_CHECK_ARG(S >= 1, "sq_logit_bias_rows_batch: S=%d", S);
  SQ_CHECK_ARG(allowed_words >= (V + 31) / 32, "sq_logit_bias_rows_batch: allowed_words=%lld < ceil(V/32)=%d",
               (long long)allowed_words, (V + 31) / 32);
  const bool vec = ((uintptr_t)logits & 15) == 0 && ld % 8 == 0;
  launch_k(logit_bias_kernel, dim3((V + LB_CHUNK - 1) / LB_CHUNK, S, B), dim3(LB_THREADS), 0, (cudaStream_t)stream,
           (__half*)logits, ld, V, S, state, allowed, allowed_words, has_mask, bias_ids, bias_vals, n_bias, vec);
  SQ_CHECK_LAUNCH("sq_logit_bias_rows_batch");
  return SQ_OK;
}
