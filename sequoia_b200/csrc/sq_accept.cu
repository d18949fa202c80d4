// Device-side verification walk (Tree/SpecTree.py:137-157,196-227,261-271; Tree/GreedyTree.py:132-146,186-240).
// The reference walks the tree on the host with one D2H sync per tested child and ~6 tiny kernels each; here one
// 1024-thread CTA keeps the target distribution p and the temperature-scaled draft logits in registers, walks
// Successors (CSR), and then applies the whole post-processing (token / position compaction, bonus token, state for
// the next iteration), so a verify step needs no host round trip.  Latency / SFU-bound on one SM: ~2*V*2 bytes per
// visited parent from HBM, V exp + V div per tested child.
//
// fp16 rounding chain of the reference reproduced step by step (see sq_sampling.cu for the conventions):
//   p = fp16(softmax(fp16(t * 1/T)));  q = fp16(softmax(fp16(d * 1/T)));  accept iff p[tok] > fp16(r * q[tok])
//   residual: d = relu(fp16(p - q)); s = fp16(sum d); p = fp16(d / s);  rejected token's draft logit -> fp16 min
// The draft softmax is maintained incrementally: masking a token removes its exp from the running sum (the max only
// has to be recomputed if the masked token was the max).
#include <cstdlib>

#include "sq_common.cuh"
#include "sq_accept_common.cuh"

namespace sq {

constexpr int ANT = 1024;
constexpr int ANW = ANT / 32;
constexpr int ACH = 4;   // 16-byte chunks per thread: V <= 32768

__device__ __forceinline__ uint32_t a_ord16(__half h) {
  const uint32_t b = __half_as_ushort(h);
  return (b & 0x8000u) ? (~b & 0xFFFFu) : (b | 0x8000u);
}

// row striped over the block (chunk c = i*ANT + tid); out-of-range chunks read as -inf; scaled to fp16(x * inv_T)
__device__ __forceinline__ void a_load_scaled(const __half* __restrict__ row, int V, float inv_T, Pack8 (&x)[ACH]) {
  const int nvec = V / 8;
#pragma unroll
  for (int i = 0; i < ACH; ++i) {
    const int c = i * ANT + threadIdx.x;
    if (c < nvec) {
      x[i].u = reinterpret_cast<const uint4*>(row)[c];
#pragma unroll
      for (int j = 0; j < 8; ++j) x[i].h[j] = f2h(h2f(x[i].h[j]) * inv_T);
    } else {
      x[i].u = make_uint4(0xFC00FC00u, 0xFC00FC00u, 0xFC00FC00u, 0xFC00FC00u);
    }
  }
}

__device__ __forceinline__ void a_stats(const Pack8 (&x)[ACH], float* red, float& mx, float& sum) {
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < ACH; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) m = fmaxf(m, h2f(x[i].h[j]));
  mx = block_max<ANW>(m, red);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < ACH; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) s += __expf(h2f(x[i].h[j]) - mx);
  sum = block_sum<ANW>(s, red);
}

__global__ void __launch_bounds__(ANT) accept_stochastic_kernel(
    const __half* __restrict__ target_logits, int64_t ld_t, const __half* __restrict__ draft_logits, int64_t ld_d,
    const __half* __restrict__ r, const __half* __restrict__ noise, const int32_t* __restrict__ succ_off,
    const int32_t* __restrict__ succ, const int32_t* __restrict__ depth, int S, int V, float inv_T,
    int64_t* __restrict__ tokens, int64_t* __restrict__ position_ids, int32_t* __restrict__ accept_idx,
    int32_t* __restrict__ state, int max_target_seq, int policy) {
  __shared__ float red[ANW];
  __shared__ uint32_t redu[ANW];
  __shared__ int32_t sh_acc[1024];
  __shared__ float sh_etok;
  __shared__ int sh_flag;
  const int P = state[ST_P];
  const int nvec = V / 8;
  Pack8 p[ACH], xd[ACH];
  int cur = 0, n_new = 0;
  bool terminal = false;
  while (true) {
    // p = softmax(target_logits[cur] / T)   (SpecTree.py:198, computed lazily for visited parents only)
    a_load_scaled(target_logits + cur * ld_t, V, inv_T, p);
    {
      float mx, sum;
      a_stats(p, red, mx, sum);
#pragma unroll
      for (int i = 0; i < ACH; ++i)
#pragma unroll
        for (int e = 0; e < 8; ++e) p[i].h[e] = f2h(__fdividef(__expf(h2f(p[i].h[e]) - mx), sum));
    }
    const int c0 = succ_off[cur], c1 = succ_off[cur + 1];
    if (c0 == c1) break;                                     // leaf: residual = p   (SpecTree.py:143-144)
    a_load_scaled(draft_logits + cur * ld_d, V, inv_T, xd);
    float mxd, sumd;
    a_stats(xd, red, mxd, sumd);                             // q = softmax(draft_logits / T)  (:149)
    int accepted = -1;
    for (int ci = c0; ci < c1; ++ci) {
      const int child = succ[ci];
      const int slot = P - 1 + child;
      const int tok = (int)tokens[slot];
      const int tc = tok >> 3, te = tok & 7;
      const bool owner = (threadIdx.x == (tc % ANT));
      if (owner) {
        const int ti = tc / ANT;
        __half ptok = f2h(0.f), dtok = f2h(0.f);
#pragma unroll
        for (int i = 0; i < ACH; ++i)
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if (i == ti && e == te) { ptok = p[i].h[e]; dtok = xd[i].h[e]; }
        const float etok = __expf(h2f(dtok) - mxd);
        const float qtok = h2f(f2h(__fdividef(etok, sumd)));
        const float thr = rnd16(h2f(r[slot]) * qtok);        // r * q[token] in fp16
        const int acc = ((policy & SQ_ACCEPT_GE) ? (h2f(ptok) >= thr) : (h2f(ptok) > thr)) ? 1 : 0;   // strict > (:152)
        sh_flag = acc | ((!(policy & SQ_ACCEPT_KEEP_Q) && h2f(dtok) >= mxd) ? 2 : 0);   // bit 1: rejected token holds the max
        sh_etok = etok;
      }
      __syncthreads();
      const int flag = sh_flag;
      const float etok = sh_etok;
      __syncthreads();
      if (flag & 1) { accepted = child; break; }
      // p = get_residual(p, q)   (:155, utils.py:5-8)
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < ACH; ++i)
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float q = h2f(f2h(__fdividef(__expf(h2f(xd[i].h[e]) - mxd), sumd)));
          float d = rnd16(h2f(p[i].h[e]) - q);
          d = (d < 0.f) ? 0.f : d;                           // relu_; NaN propagates like torch
          p[i].h[e] = f2h(d);
          s += d;
        }
      const float tot = rnd16(block_sum<ANW>(s, red));
#pragma unroll
      for (int i = 0; i < ACH; ++i)
#pragma unroll
        for (int e = 0; e < 8; ++e) p[i].h[e] = f2h(h2f(p[i].h[e]) / tot);
      if (policy & SQ_ACCEPT_KEEP_Q) continue;               // SpecInfer policy: q is never edited
      // draft_logits[token] = fp16 min   (:156)  ->  scaled value -inf, exp 0
      if (owner) {
        const int ti = tc / ANT;
#pragma unroll
        for (int i = 0; i < ACH; ++i)
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if (i == ti && e == te) xd[i].h[e] = __ushort_as_half((unsigned short)0xFC00u);
      }
      if (flag & 2) a_stats(xd, red, mxd, sumd);             // rare: the max left the support
      else sumd -= etok;
    }
    if (accepted < 0) break;                                 // residual = p   (:157)
    const int slot = P - 1 + accepted;
    if (threadIdx.x == 0) sh_acc[n_new] = slot;
    ++n_new;
    const int64_t t = tokens[slot];
    if (t == 0 || t == 2) { terminal = true; break; }        // (:208)
    cur = accepted;
  }
  __syncthreads();
  bool nan_flag = false;
  int64_t bonus = -1;
  if (!terminal) {
    int has_nan = 0;
#pragma unroll
    for (int i = 0; i < ACH; ++i)
      if (i * ANT + threadIdx.x < nvec) {
#pragma unroll
        for (int e = 0; e < 8; ++e) has_nan |= __hisnan(p[i].h[e]) ? 1 : 0;
      }
    nan_flag = __syncthreads_or(has_nan) != 0;               // torch.isnan(residual).any()  (:219)
    if (nan_flag) {
      terminal = true;
    } else {
      // residual.multinomial(1): argmax(residual / Exp(1) noise)   (:222, torch's n=1 form)
      uint32_t best = 0u;
#pragma unroll
      for (int i = 0; i < ACH; ++i) {
        const int c = i * ANT + threadIdx.x;
        if (c < nvec) {
          Pack8 nz;
          nz.u = reinterpret_cast<const uint4*>(noise)[c];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const __half v = f2h(h2f(p[i].h[e]) / h2f(nz.h[e]));
            best = max(best, (a_ord16(v) << 16) | (0xFFFFu - (uint32_t)(c * 8 + e)));
          }
        }
      }
      best = __reduce_max_sync(0xffffffffu, best);
      if ((threadIdx.x & 31) == 0) redu[threadIdx.x >> 5] = best;
      __syncthreads();
      best = __reduce_max_sync(0xffffffffu, redu[threadIdx.x & 31]);
      bonus = (int64_t)(0xFFFFu - (best & 0xFFFFu));
    }
  }
  finish_verify(sh_acc, n_new, P, terminal, nan_flag, bonus, true, depth, S, tokens, position_ids, accept_idx, state,
                max_target_seq);
}

// BATCH: grid (B), one walk per sequence; target_token rows of S per sequence, the rest as in BatchArgs.
// MIXED (BATCH only): only the sequences with greedy[b] nonzero walk; the others' blocks exit as a frozen one does.
// STOP (BATCH only): stop mode, as in accept_stochastic_cluster_kernel: no fixed 0 / 2 end rule, then stop_cut with the
// rows of stop_ids / end_limit (nullptr in every other instance).
template <bool BATCH, bool MIXED = false, bool STOP = false>
__global__ void accept_greedy_kernel(const int64_t* __restrict__ target_token, const int32_t* __restrict__ succ_off,
                                     const int32_t* __restrict__ succ, const int32_t* __restrict__ depth, int S,
                                     int64_t* __restrict__ tokens, int64_t* __restrict__ position_ids,
                                     int32_t* __restrict__ accept_idx, int32_t* __restrict__ state,
                                     int max_target_seq, int64_t ld_seq, int64_t ld_acc,
                                     const int32_t* __restrict__ greedy, const int32_t* __restrict__ stop_ids,
                                     const int32_t* __restrict__ end_limit) {
  static_assert(BATCH || !MIXED, "a per-sequence policy needs the batched kernel");
  static_assert(BATCH || !STOP, "stop mode needs the batched kernel");
  __shared__ int32_t sh_acc[1024];
  __shared__ int sh_n, sh_term;
  __shared__ long long sh_bonus;
  const int b = seq_index<BATCH>(blockIdx.x);
  if (BATCH) {
    state += b * ST_WORDS;
    if (state[ST_FROZEN]) return;
    if (MIXED && !greedy[b]) return;
    target_token += (int64_t)b * S;
    tokens += b * ld_seq;
    position_ids += b * ld_seq;
    accept_idx += b * ld_acc;
  }
  __shared__ int32_t sh_stop[STOP ? SQ_MAX_STOP + 1 : 1];
  if constexpr (STOP) stop_row_load(sh_stop, stop_ids, end_limit, b);
  const int P = state[ST_P];
  if (threadIdx.x == 0) {
    int cur = 0, n_new = 0, term = 0;
    while (true) {                                           // GreedyTree.py:191-201
      const int64_t tt = target_token[cur];
      int acc = -1;
      for (int ci = succ_off[cur]; ci < succ_off[cur + 1]; ++ci) {
        const int child = succ[ci];
        if (tokens[P - 1 + child] == tt) { acc = child; break; }
      }
      if (acc < 0) break;
      const int slot = P - 1 + acc;
      sh_acc[n_new++] = slot;
      const int64_t t = tokens[slot];
      if (!STOP && (t == 0 || t == 2)) { term = 1; break; }
      cur = acc;
    }
    sh_n = n_new;
    sh_term = term;
    sh_bonus = term ? -1 : target_token[cur];                // GreedyTree.py:207
  }
  __syncthreads();
  finish_verify(sh_acc, sh_n, P, sh_term != 0, false, (int64_t)sh_bonus, false, depth, S, tokens, position_ids,
                accept_idx, state, max_target_seq);
  if constexpr (STOP) stop_cut(sh_stop, sh_n, P, sh_term != 0, tokens, state, max_target_seq);
}

}  // namespace sq

using namespace sq;

// SQ_ACCEPT_IMPL (read once): 1 = the cluster walk (default), 0 = the single-CTA cross-check walk
static int accept_impl() {
  static const int impl = [] { const char* e = getenv("SQ_ACCEPT_IMPL"); return e ? atoi(e) : 1; }();
  return impl;
}

extern "C" int sq_accept_stochastic(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits,
                                    int64_t ld_d, const sq_half* r, const sq_half* noise, const int32_t* succ_off,
                                    const int32_t* succ, const int32_t* depth, int S, int V, float T, int64_t* tokens,
                                    int64_t* position_ids, int32_t* accept_idx, int32_t* state, int max_target_seq,
                                    int policy, void* stream) {
  SQ_CHECK_ARG(S >= 1 && S <= 1024, "sq_accept_stochastic: S=%d unsupported", S);
  SQ_CHECK_ARG((policy & ~3) == 0, "sq_accept_stochastic: unknown policy bits %d", policy);
  if (accept_impl() == 1)   // product path: 8-CTA cluster kernel (sq_accept_cluster.cu); impl 0 = single-CTA cross-check
    return sq::launch_accept_cluster(target_logits, ld_t, draft_logits, ld_d, r, noise, succ_off, succ, depth, S, V, T,
                                     tokens, position_ids, accept_idx, state, max_target_seq, policy, stream);
  SQ_CHECK_ARG(V % 8 == 0 && V > 0 && V <= ANT * ACH * 8,
               "sq_accept_stochastic: V=%d unsupported by the single-CTA walk (SQ_ACCEPT_IMPL=0): multiple of 8, <= 32768",
               V);
  accept_stochastic_kernel<<<1, ANT, 0, (cudaStream_t)stream>>>(
      (const __half*)target_logits, ld_t, (const __half*)draft_logits, ld_d, (const __half*)r, (const __half*)noise,
      succ_off, succ, depth, S, V, 1.0f / T, tokens, position_ids, accept_idx, state, max_target_seq, policy);
  SQ_CHECK_LAUNCH("sq_accept_stochastic");
  return SQ_OK;
}

extern "C" int sq_accept_greedy(const int64_t* target_token, const int32_t* succ_off, const int32_t* succ,
                                const int32_t* depth, int S, int64_t* tokens, int64_t* position_ids,
                                int32_t* accept_idx, int32_t* state, int max_target_seq, void* stream) {
  SQ_CHECK_ARG(S >= 1 && S <= 1024, "sq_accept_greedy: S=%d unsupported", S);
  accept_greedy_kernel<false><<<1, 256, 0, (cudaStream_t)stream>>>(target_token, succ_off, succ, depth, S, tokens,
                                                                   position_ids, accept_idx, state, max_target_seq, 0, 0,
                                                                   nullptr, nullptr, nullptr);
  SQ_CHECK_LAUNCH("sq_accept_greedy");
  return SQ_OK;
}

// sq_accept_greedy_batch (greedy == nullptr), its mixed-policy form and (stop_ids != nullptr) the stop forms
static int accept_greedy_batch(const char* name, const int64_t* target_token, const int32_t* succ_off,
                               const int32_t* succ, const int32_t* depth, int S, int64_t* tokens, int64_t* position_ids,
                               int64_t ld_seq, int32_t* accept_idx, int64_t ld_acc, int32_t* state, int B,
                               int max_target_seq, const int32_t* greedy, void* stream,
                               const int32_t* stop_ids = nullptr, const int32_t* end_limit = nullptr) {
  SQ_CHECK_ARG(S >= 1 && S <= 1024, "%s: S=%d unsupported", name, S);
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH, "%s: B=%d (1..%d)", name, B, SQ_MAX_BATCH);
  SQ_CHECK_ARG(ld_acc >= S && ld_seq >= 1, "%s: accept_idx rows of %lld < S=%d", name, (long long)ld_acc, S);
  if (stop_ids && greedy)
    accept_greedy_kernel<true, true, true><<<B, 256, 0, (cudaStream_t)stream>>>(
        target_token, succ_off, succ, depth, S, tokens, position_ids, accept_idx, state, max_target_seq, ld_seq, ld_acc,
        greedy, stop_ids, end_limit);
  else if (stop_ids)
    accept_greedy_kernel<true, false, true><<<B, 256, 0, (cudaStream_t)stream>>>(
        target_token, succ_off, succ, depth, S, tokens, position_ids, accept_idx, state, max_target_seq, ld_seq, ld_acc,
        nullptr, stop_ids, end_limit);
  else if (greedy)
    accept_greedy_kernel<true, true><<<B, 256, 0, (cudaStream_t)stream>>>(
        target_token, succ_off, succ, depth, S, tokens, position_ids, accept_idx, state, max_target_seq, ld_seq, ld_acc,
        greedy, nullptr, nullptr);
  else
    accept_greedy_kernel<true><<<B, 256, 0, (cudaStream_t)stream>>>(target_token, succ_off, succ, depth, S, tokens,
                                                                    position_ids, accept_idx, state, max_target_seq,
                                                                    ld_seq, ld_acc, nullptr, nullptr, nullptr);
  SQ_CHECK_LAUNCH(name);
  return SQ_OK;
}

extern "C" int sq_accept_greedy_batch(const int64_t* target_token, const int32_t* succ_off, const int32_t* succ,
                                      const int32_t* depth, int S, int64_t* tokens, int64_t* position_ids, int64_t ld_seq,
                                      int32_t* accept_idx, int64_t ld_acc, int32_t* state, int B, int max_target_seq,
                                      void* stream) {
  return accept_greedy_batch("sq_accept_greedy_batch", target_token, succ_off, succ, depth, S, tokens, position_ids, ld_seq,
                             accept_idx, ld_acc, state, B, max_target_seq, nullptr, stream);
}

extern "C" int sq_accept_greedy_batch_mixed(const int64_t* target_token, const int32_t* succ_off, const int32_t* succ,
                                            const int32_t* depth, int S, int64_t* tokens, int64_t* position_ids,
                                            int64_t ld_seq, int32_t* accept_idx, int64_t ld_acc, int32_t* state,
                                            const int32_t* greedy, int B, int max_target_seq, void* stream) {
  SQ_CHECK_ARG(greedy != nullptr, "sq_accept_greedy_batch_mixed: null greedy array");
  return accept_greedy_batch("sq_accept_greedy_batch_mixed", target_token, succ_off, succ, depth, S, tokens, position_ids,
                             ld_seq, accept_idx, ld_acc, state, B, max_target_seq, greedy, stream);
}

// sq_accept_stochastic_batch (T_seq == nullptr), its per-sequence form, (greedy != nullptr) the mixed-policy form and
// (stop_ids != nullptr) the stop forms
static int accept_stochastic_batch(const char* name, const sq_half* target_logits, int64_t ld_t,
                                   const sq_half* draft_logits, int64_t ld_d, const int32_t* row_base,
                                   const int32_t* row_step, const sq_half* r, const sq_half* noise, int64_t ld_noise,
                                   const int32_t* succ_off, const int32_t* succ, const int32_t* depth, int S, int V,
                                   float T, const float* T_seq, int64_t* tokens, int64_t* position_ids, int64_t ld_seq,
                                   int32_t* accept_idx, int64_t ld_acc, int32_t* state, int B, int max_target_seq,
                                   int policy, void* stream, const int32_t* greedy = nullptr,
                                   const int32_t* stop_ids = nullptr, const int32_t* end_limit = nullptr) {
  SQ_CHECK_ARG(S >= 1 && S <= 1024, "%s: S=%d unsupported", name, S);
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH, "%s: B=%d (1..%d)", name, B, SQ_MAX_BATCH);
  SQ_CHECK_ARG((policy & ~(T_seq ? 3 | SQ_ACCEPT_SKIP_DEAD : 3)) == 0, "%s: unknown policy bits %d", name, policy);
  SQ_CHECK_ARG(row_base && row_step, "%s: null draft-row table", name);
  SQ_CHECK_ARG(ld_acc >= S && ld_noise >= V, "%s: accept_idx / noise rows too short", name);
  BatchArgs ba{B, ld_seq, ld_noise, ld_acc, row_base, row_step, greedy, stop_ids, end_limit};
  return sq::launch_accept_cluster(target_logits, ld_t, draft_logits, ld_d, r, noise, succ_off, succ, depth, S, V, T, tokens,
                                   position_ids, accept_idx, state, max_target_seq, policy, stream, &ba, T_seq);
}

extern "C" int sq_accept_stochastic_batch(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits,
                                          int64_t ld_d, const int32_t* row_base, const int32_t* row_step, const sq_half* r,
                                          const sq_half* noise, int64_t ld_noise, const int32_t* succ_off,
                                          const int32_t* succ, const int32_t* depth, int S, int V, float T,
                                          int64_t* tokens, int64_t* position_ids, int64_t ld_seq, int32_t* accept_idx,
                                          int64_t ld_acc, int32_t* state, int B, int max_target_seq, int policy,
                                          void* stream) {
  return accept_stochastic_batch("sq_accept_stochastic_batch", target_logits, ld_t, draft_logits, ld_d, row_base, row_step,
                                 r, noise, ld_noise, succ_off, succ, depth, S, V, T, nullptr, tokens, position_ids, ld_seq,
                                 accept_idx, ld_acc, state, B, max_target_seq, policy, stream);
}

extern "C" int sq_accept_stochastic_batch_per_seq(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits,
                                                  int64_t ld_d, const int32_t* row_base, const int32_t* row_step,
                                                  const sq_half* r, const sq_half* noise, int64_t ld_noise,
                                                  const int32_t* succ_off, const int32_t* succ, const int32_t* depth, int S,
                                                  int V, const float* T, int64_t* tokens, int64_t* position_ids,
                                                  int64_t ld_seq, int32_t* accept_idx, int64_t ld_acc, int32_t* state,
                                                  int B, int max_target_seq, int policy, void* stream) {
  SQ_CHECK_ARG(T != nullptr, "sq_accept_stochastic_batch_per_seq: null temperature array");
  return accept_stochastic_batch("sq_accept_stochastic_batch_per_seq", target_logits, ld_t, draft_logits, ld_d, row_base,
                                 row_step, r, noise, ld_noise, succ_off, succ, depth, S, V, 1.0f, T, tokens, position_ids,
                                 ld_seq, accept_idx, ld_acc, state, B, max_target_seq, policy, stream);
}

extern "C" int sq_accept_stochastic_batch_mixed(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits,
                                                int64_t ld_d, const int32_t* row_base, const int32_t* row_step,
                                                const sq_half* r, const sq_half* noise, int64_t ld_noise,
                                                const int32_t* succ_off, const int32_t* succ, const int32_t* depth, int S,
                                                int V, const float* T, const int32_t* greedy, int64_t* tokens,
                                                int64_t* position_ids, int64_t ld_seq, int32_t* accept_idx, int64_t ld_acc,
                                                int32_t* state, int B, int max_target_seq, int policy, void* stream) {
  SQ_CHECK_ARG(T != nullptr && greedy != nullptr, "sq_accept_stochastic_batch_mixed: null temperature or greedy array");
  return accept_stochastic_batch("sq_accept_stochastic_batch_mixed", target_logits, ld_t, draft_logits, ld_d, row_base,
                                 row_step, r, noise, ld_noise, succ_off, succ, depth, S, V, 1.0f, T, tokens, position_ids,
                                 ld_seq, accept_idx, ld_acc, state, B, max_target_seq, policy, stream, greedy);
}

extern "C" int sq_accept_stochastic_batch_stop(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits,
                                               int64_t ld_d, const int32_t* row_base, const int32_t* row_step,
                                               const sq_half* r, const sq_half* noise, int64_t ld_noise,
                                               const int32_t* succ_off, const int32_t* succ, const int32_t* depth, int S,
                                               int V, const float* T, const int32_t* greedy, const int32_t* stop_ids,
                                               const int32_t* end_limit, int64_t* tokens, int64_t* position_ids,
                                               int64_t ld_seq, int32_t* accept_idx, int64_t ld_acc, int32_t* state, int B,
                                               int max_target_seq, int policy, void* stream) {
  SQ_CHECK_ARG(T != nullptr, "sq_accept_stochastic_batch_stop: null temperature array");
  SQ_CHECK_ARG(stop_ids != nullptr && end_limit != nullptr, "sq_accept_stochastic_batch_stop: null stop_ids or end_limit");
  return accept_stochastic_batch("sq_accept_stochastic_batch_stop", target_logits, ld_t, draft_logits, ld_d, row_base,
                                 row_step, r, noise, ld_noise, succ_off, succ, depth, S, V, 1.0f, T, tokens, position_ids,
                                 ld_seq, accept_idx, ld_acc, state, B, max_target_seq, policy, stream, greedy, stop_ids,
                                 end_limit);
}

extern "C" int sq_accept_greedy_batch_stop(const int64_t* target_token, const int32_t* succ_off, const int32_t* succ,
                                           const int32_t* depth, int S, int64_t* tokens, int64_t* position_ids,
                                           int64_t ld_seq, int32_t* accept_idx, int64_t ld_acc, int32_t* state,
                                           const int32_t* greedy, const int32_t* stop_ids, const int32_t* end_limit, int B,
                                           int max_target_seq, void* stream) {
  SQ_CHECK_ARG(stop_ids != nullptr && end_limit != nullptr, "sq_accept_greedy_batch_stop: null stop_ids or end_limit");
  return accept_greedy_batch("sq_accept_greedy_batch_stop", target_token, succ_off, succ, depth, S, tokens, position_ids,
                             ld_seq, accept_idx, ld_acc, state, B, max_target_seq, greedy, stream, stop_ids, end_limit);
}
