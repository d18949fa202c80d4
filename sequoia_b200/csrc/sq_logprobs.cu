// Per-sequence logprobs of the tokens a batched verify step committed (include/sequoia_b200.h, sq_token_logprobs_batch).
// One 1024-thread CTA per committed position (grid x = path depth j, y = sequence b); a position the step did not commit
// exits after the dependency wait.  The CTA reads its target row three times (the first from HBM, the others mostly from
// L2), striped in 16-byte vectors, so one code path serves every V up to 131072:
//   1. the row max of the scaled values s_i = fp16(x_i / T) and the level-0 histogram (high byte) of the ranking keys;
//   2. sum exp(s_i - max) in fp32 and the level-1 histogram (low byte) inside the boundary bin;
//   3. the top-n candidates: every key above the boundary key (fewer than n), then the first of the keys equal to it in
//      index order (a block scan per tile of 8192 entries).
// The select is top_k_filter_kernel's two-level 256-bin histogram select (sq_sampling.cu) with the same key (topk_key),
// so the ids are exactly those the top-k filter would keep, ranked.  Counts are integers: no result depends on timing.
// sq_prompt_logprobs_ragged runs the same per-row body (lp_row) at T = 1 on the prompt rows of a first verify, one CTA per
// row of every listed sequence in one launch.
#include "sq_common.cuh"

namespace sq {

constexpr int LP_NT = 1024;
constexpr int LP_NW = LP_NT / 32;

// warp 0: the bin of the n-th key, scanning bins in descending order from `before` keys ranked above them.  sel[0] = the
// bin (-1 when the keys run out first), sel[1] = the keys ranked before it.  The caller syncs after.
__device__ __forceinline__ void lp_select_bin(const uint32_t* hist, uint32_t before, int n, int* sel) {
  const int lane = threadIdx.x & 31;
  uint32_t m[8], tot = 0u;
#pragma unroll
  for (int b = 0; b < 8; ++b) { m[b] = hist[255 - 8 * lane - b]; tot += m[b]; }
  uint32_t inc = tot;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t s = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += s;
  }
  uint32_t a = before + inc - tot;
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    if (a < (uint32_t)n && a + m[b] >= (uint32_t)n) { sel[0] = 255 - 8 * lane - b; sel[1] = (int)a; }   // unique
    a += m[b];
  }
}

// per-warp histograms -> hist (threads < 256), then the boundary bin; returns with hist / sel valid in every thread
__device__ __forceinline__ void lp_reduce_select(uint32_t (*whist)[256], uint32_t* hist, uint32_t before, int n, int* sel) {
  __syncthreads();
  if (threadIdx.x < 256) {
    uint32_t t = 0u;
#pragma unroll 8
    for (int w = 0; w < LP_NW; ++w) t += whist[w][threadIdx.x];
    hist[threadIdx.x] = t;
  }
  if (threadIdx.x == 0) sel[0] = -1;
  __syncthreads();
  if (threadIdx.x < 32) lp_select_bin(hist, before, n, sel);
  __syncthreads();
}

// One row's logprobs, by every thread (tid = threadIdx.x) of a 1024-thread CTA after the dependency wait: the
// log-softmax of s_i = fp16(x_i * inv_T) at token tokens[pos] into lp_token[pos], and the n best ids (topk_key order,
// ties by index) with their logprobs into lp_ids / lp_top[pos][0 .. n).  token_logprobs_kernel and prompt_logprobs_kernel
// share it, so one rule serves generated and prompt tokens.  (The caller reads tid before its early exits: that keeps
// token_logprobs_kernel's SASS what it was before the body moved here.)
__device__ __forceinline__ void lp_row(const __half* row, int V, float inv_T, int n,
                                       const int64_t* __restrict__ tokens, int64_t pos, float* __restrict__ lp_token,
                                       int32_t* __restrict__ lp_ids, float* __restrict__ lp_top, int tid) {
  __shared__ uint32_t whist[LP_NW][256];
  __shared__ uint32_t hist[256];
  __shared__ float red[LP_NW];
  __shared__ int sel[2];
  __shared__ int wtot[LP_NW];
  __shared__ int n_above;
  __shared__ uint32_t c_key[SQ_MAX_LOGPROBS];
  __shared__ int c_idx[SQ_MAX_LOGPROBS];
  const int lane = tid & 31, warp = tid >> 5;
  const uint4* row4 = reinterpret_cast<const uint4*>(row);
  const int nvec = V / 8;

  // pass 1: max of s, a +inf / NaN flag, level-0 histogram
  if (n > 0) {
    for (int i = tid; i < LP_NW * 256; i += LP_NT) (&whist[0][0])[i] = 0u;
    __syncthreads();
  }
  float m = -INFINITY;
  bool bad = false;
  for (int c = tid; c < nvec; c += LP_NT) {
    Pack8 x;
    x.u = row4[c];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float s = rnd16(h2f(x.h[e]) * inv_T);
      bad |= isnan(s) || s == INFINITY;
      m = fmaxf(m, s);
      if (n > 0) atomicAdd(&whist[warp][topk_key(x.h[e]) >> 8], 1u);
    }
  }
  bad = __syncthreads_or(bad);
  m = block_max<LP_NW>(m, red);
  int hi = -1;
  uint32_t before = 0u;
  if (n > 0) {
    lp_reduce_select(whist, hist, 0u, n, sel);
    hi = sel[0];
    before = (uint32_t)sel[1];
    for (int i = tid; i < LP_NW * 256; i += LP_NT) (&whist[0][0])[i] = 0u;
    __syncthreads();
  }
  // pass 2: the softmax sum, level-1 histogram
  const bool ok = !bad && m > -INFINITY;
  float sum = 0.f;
  for (int c = tid; c < nvec; c += LP_NT) {
    Pack8 x;
    x.u = row4[c];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      if (ok) sum += expf(rnd16(h2f(x.h[e]) * inv_T) - m);
      if (n > 0) {
        const uint32_t key = topk_key(x.h[e]);
        if ((int)(key >> 8) == hi) atomicAdd(&whist[warp][key & 255u], 1u);
      }
    }
  }
  sum = block_sum<LP_NW>(sum, red);
  const float log_sum = logf(sum);
  // the logprob of a raw fp16 value of this row
  auto lp_of = [&](__half h) -> float {
    return ok ? (rnd16(h2f(h) * inv_T) - m) - log_sum : __int_as_float(0x7fc00000);
  };
  if (tid == 0) {
    const int64_t t = tokens[pos];
    lp_token[pos] = (t >= 0 && t < V) ? lp_of(row[t]) : __int_as_float(0x7fc00000);
  }
  if (n == 0) return;
  lp_reduce_select(whist, hist, before, n, sel);
  const int key_b = (hi << 8) | sel[0];
  before = (uint32_t)sel[1];
  const int need = n - (int)before;                                            // tie members to take, by index
  if (tid == 0) n_above = 0;
  __syncthreads();
  // pass 3: candidates.  Tile t covers vectors [t * LP_NT, (t + 1) * LP_NT), thread tid one vector of it, so the scan
  // over threads is in index order.
  int base = 0;                                                                // tie members in earlier tiles
  for (int c0 = 0; c0 < nvec; c0 += LP_NT) {
    const int c = c0 + tid;
    Pack8 x;
    int cnt = 0;
    if (c < nvec) {
      x.u = row4[c];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const uint32_t key = topk_key(x.h[e]);
        if ((int)key > key_b) {
          const int q = atomicAdd(&n_above, 1);
          c_key[q] = key;
          c_idx[q] = c * 8 + e;
        }
        cnt += (int)key == key_b;
      }
    }
    int inc = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int s = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += s;
    }
    if (lane == 31) wtot[warp] = inc;
    __syncthreads();
    int wex = 0, tile = 0;
    for (int w = 0; w < LP_NW; ++w) {
      const int v = wtot[w];
      wex += w < warp ? v : 0;
      tile += v;
    }
    int r = base + wex + inc - cnt;                                            // tie rank of this thread's first member
    if (cnt > 0 && r < need) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if ((int)topk_key(x.h[e]) == key_b) {
          if (r < need) {
            c_key[before + r] = (uint32_t)key_b;
            c_idx[before + r] = c * 8 + e;
          }
          ++r;
        }
      }
    }
    base += tile;
    __syncthreads();                                                           // wtot is rewritten by the next tile
  }
  // rank the n candidates (keys descending, equal keys by ascending index) and write them
  if (tid < n) {
    const uint32_t k = c_key[tid];
    const int idx = c_idx[tid];
    int rank = 0;
    for (int q = 0; q < n; ++q) rank += c_key[q] > k || (c_key[q] == k && c_idx[q] < idx);
    lp_ids[pos * SQ_MAX_LOGPROBS + rank] = idx;
    lp_top[pos * SQ_MAX_LOGPROBS + rank] = lp_of(row[idx]);
  }
}

__global__ void __launch_bounds__(LP_NT)
    token_logprobs_kernel(const __half* __restrict__ logits, int64_t ld, int V, int S, const int64_t* __restrict__ tokens,
                          int64_t ld_seq, const int32_t* __restrict__ state, const int32_t* __restrict__ accept_idx,
                          int64_t ld_acc, const float* __restrict__ T, const int32_t* __restrict__ greedy,
                          const int32_t* __restrict__ n_top, float* __restrict__ lp_token, int32_t* __restrict__ lp_ids,
                          float* __restrict__ lp_top) {
  pdl_wait();
  pdl_trigger();
  const int j = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int32_t* st = state + b * ST_WORDS;
  if (st[ST_FROZEN] || n_top[b] < 0) return;
  const int P = st[ST_P_OLD], n_new = st[ST_N_NEW], a = P + n_new;
  const int M = st[ST_M] > 0 ? st[ST_M] : (int)min(ld_seq, (int64_t)INT32_MAX);
  const int committed = n_new + ((!st[ST_TERMINAL] && a < M) ? 1 : 0);      // finish_verify's bonus_ok
  if (j >= committed || P < 1 || (int64_t)P + j >= ld_seq) return;
  const int node = j == 0 ? 0 : accept_idx[b * ld_acc + j - 1] - (P - 1);
  if (node < 0 || node >= S) return;                                          // (not a walk's output)
  const int n = min(min(n_top[b], SQ_MAX_LOGPROBS), V);
  const float inv_T = greedy[b] ? 1.0f : 1.0f / T[b];                         // the walk's inv_temp
  const int64_t pos = (int64_t)b * ld_seq + P + j;
  lp_row(logits + ((int64_t)b * S + node) * ld, V, inv_T, n, tokens, pos, lp_token, lp_ids, lp_top, tid);
}

// Prompt logprobs (sq_prompt_logprobs_ragged): CTA (r, j) scores tokens[seq_j][r + 1] on logits row logits_row0_j + r at
// T = 1, position r + 1 of the outputs.
struct PromptLpParts {
  int seq[SQ_MAX_BATCH], row0[SQ_MAX_BATCH], n_rows[SQ_MAX_BATCH], n_top[SQ_MAX_BATCH];
};

__global__ void __launch_bounds__(LP_NT)
    prompt_logprobs_kernel(const __half* __restrict__ logits, int64_t ld, int V, PromptLpParts parts,
                           const int64_t* __restrict__ tokens, int64_t ld_seq, float* __restrict__ plp_token,
                           int32_t* __restrict__ plp_ids, float* __restrict__ plp_top) {
  pdl_wait();
  pdl_trigger();
  const int r = blockIdx.x, j = blockIdx.y;
  if (r >= parts.n_rows[j]) return;
  const int n = min(parts.n_top[j], V);
  const int64_t pos = (int64_t)parts.seq[j] * ld_seq + r + 1;
  lp_row(logits + ((int64_t)parts.row0[j] + r) * ld, V, 1.0f, n, tokens, pos, plp_token, plp_ids, plp_top, threadIdx.x);
}

}  // namespace sq

using namespace sq;

extern "C" int sq_token_logprobs_batch(const sq_half* logits, int64_t ld, int V, int S, int max_depth,
                                       const int64_t* tokens, int64_t ld_seq, const int32_t* state,
                                       const int32_t* accept_idx, int64_t ld_acc, const float* T, const int32_t* greedy,
                                       const int32_t* n_top, float* lp_token, int32_t* lp_ids, float* lp_top, int B,
                                       void* stream) {
  SQ_CHECK_ARG(logits && tokens && state && accept_idx && T && greedy && n_top && lp_token && lp_ids && lp_top,
               "sq_token_logprobs_batch: null array");
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH, "sq_token_logprobs_batch: B=%d (1..%d)", B, SQ_MAX_BATCH);
  SQ_CHECK_ARG(V % 8 == 0 && V > 0 && V <= 131072, "sq_token_logprobs_batch: V=%d must be a multiple of 8, <= 131072", V);
  SQ_CHECK_ARG(ld >= V && ld % 8 == 0, "sq_token_logprobs_batch: ld=%lld must be >= V=%d and a multiple of 8",
               (long long)ld, V);
  SQ_CHECK_ARG(((uintptr_t)logits & 15) == 0, "sq_token_logprobs_batch: logits must be 16-byte aligned");
  SQ_CHECK_ARG(S >= 1 && max_depth >= 0 && max_depth < S, "sq_token_logprobs_batch: S=%d with max_depth=%d", S,
               max_depth);
  SQ_CHECK_ARG(ld_seq >= 1, "sq_token_logprobs_batch: ld_seq=%lld", (long long)ld_seq);
  SQ_CHECK_ARG(ld_acc >= max_depth, "sq_token_logprobs_batch: ld_acc=%lld < max_depth=%d", (long long)ld_acc, max_depth);
  launch_k(token_logprobs_kernel, dim3(max_depth + 1, B), dim3(LP_NT), 0, (cudaStream_t)stream, (const __half*)logits, ld,
           V, S, tokens, ld_seq, state, accept_idx, ld_acc, T, greedy, n_top, lp_token, lp_ids, lp_top);
  SQ_CHECK_LAUNCH("sq_token_logprobs_batch");
  return SQ_OK;
}

extern "C" int sq_prompt_logprobs_ragged(const sq_half* logits, int64_t ld, int V, int64_t n_logit_rows,
                                         const sq_prompt_lp_part* parts, int n_parts, const int64_t* tokens,
                                         int64_t ld_seq, float* plp_token, int32_t* plp_ids, float* plp_top, int B,
                                         void* stream) {
  SQ_CHECK_ARG(logits && parts && tokens && plp_token && plp_ids && plp_top, "sq_prompt_logprobs_ragged: null array");
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH, "sq_prompt_logprobs_ragged: B=%d (1..%d)", B, SQ_MAX_BATCH);
  SQ_CHECK_ARG(V % 8 == 0 && V > 0 && V <= 131072, "sq_prompt_logprobs_ragged: V=%d must be a multiple of 8, <= 131072",
               V);
  SQ_CHECK_ARG(ld >= V && ld % 8 == 0, "sq_prompt_logprobs_ragged: ld=%lld must be >= V=%d and a multiple of 8",
               (long long)ld, V);
  SQ_CHECK_ARG(((uintptr_t)logits & 15) == 0, "sq_prompt_logprobs_ragged: logits must be 16-byte aligned");
  SQ_CHECK_ARG(n_parts >= 1 && n_parts <= B, "sq_prompt_logprobs_ragged: %d parts for %d sequences", n_parts, B);
  PromptLpParts pp{};
  unsigned seen = 0;
  int max_rows = 0;
  for (int j = 0; j < n_parts; ++j) {
    const sq_prompt_lp_part& p = parts[j];
    SQ_CHECK_ARG(p.seq >= 0 && p.seq < B, "sq_prompt_logprobs_ragged: part %d names sequence %d of %d", j, p.seq, B);
    SQ_CHECK_ARG(!(seen >> p.seq & 1u), "sq_prompt_logprobs_ragged: sequence %d listed twice", p.seq);
    SQ_CHECK_ARG(p.n_rows >= 1 && (int64_t)p.n_rows + 1 <= ld_seq,
                 "sq_prompt_logprobs_ragged: part %d has n_rows=%d (1..ld_seq-1, ld_seq=%lld)", j, p.n_rows,
                 (long long)ld_seq);
    SQ_CHECK_ARG(p.logits_row0 >= 0 && (int64_t)p.logits_row0 + p.n_rows <= n_logit_rows,
                 "sq_prompt_logprobs_ragged: part %d reads logits rows [%d, %lld) of %lld", j, p.logits_row0,
                 (long long)p.logits_row0 + p.n_rows, (long long)n_logit_rows);
    SQ_CHECK_ARG(p.n_top >= 0 && p.n_top <= SQ_MAX_LOGPROBS, "sq_prompt_logprobs_ragged: part %d has n_top=%d (0..%d)", j,
                 p.n_top, SQ_MAX_LOGPROBS);
    seen |= 1u << p.seq;
    pp.seq[j] = p.seq; pp.row0[j] = p.logits_row0; pp.n_rows[j] = p.n_rows; pp.n_top[j] = p.n_top;
    max_rows = max(max_rows, p.n_rows);
  }
  launch_k(prompt_logprobs_kernel, dim3(max_rows, n_parts), dim3(LP_NT), 0, (cudaStream_t)stream,
           (const __half*)logits, ld, V, pp, tokens, ld_seq, plp_token, plp_ids, plp_top);
  SQ_CHECK_LAUNCH("sq_prompt_logprobs_ragged");
  return SQ_OK;
}
