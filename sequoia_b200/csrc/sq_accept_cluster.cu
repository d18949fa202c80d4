// Cluster version of the stochastic accept/reject walk (see sq_accept.cu for the algorithm and the reference citations).
// A thread-block cluster of 8 CTAs x 512 threads splits the vocabulary (one 16-byte chunk per thread); block-level
// partials are exchanged through distributed shared memory with ONE cluster barrier per tested child:
// every CTA speculatively computes its share of the residual sum while the CTA owning the tested token evaluates the
// accept rule, and both travel in the same exchange.  Per child: ~8 exp + 8 div per thread + 1 cluster.sync.
// NCH = 16-byte chunks per thread (V <= CL*CNT*8*NCH): 1 up to V = 32768, up to 4 (V <= 131072) for large vocabularies.
// CTA r owns chunks [r*cpb, (r+1)*cpb); thread t holds its CTA's chunks i*CNT + t.  With NCH > 1 the bonus keys carry
// CTA-local indices (< 16384) and are merged in rank order, so equal maxima still resolve to the lowest index.
#include <cooperative_groups.h>

#include <type_traits>

#include "sq_common.cuh"
#include "sq_accept_common.cuh"

namespace cg = cooperative_groups;

namespace sq {

constexpr int CL = 8;
constexpr int CNT = 512;
constexpr int CNW = CNT / 32;

struct Xch {                       // double-buffered exchange slots, one per source CTA
  float f[2][CL][4];
  uint32_t u[2][CL][2];
};

__device__ __forceinline__ uint32_t c_ord16(__half h) {
  const uint32_t b = __half_as_ushort(h);
  return (b & 0x8000u) ? (~b & 0xFFFFu) : (b | 0x8000u);
}

struct ClusterCtx {
  cg::cluster_group cluster;
  Xch* x;
  int rank;
  int ph;
  // publish (f0..f3, u0, u1) of this CTA to every CTA, barrier, then read all slots (fixed order => identical results)
  __device__ __forceinline__ void exchange(float f0, float f1, float f2, float f3, uint32_t u0, uint32_t u1) {
    if (threadIdx.x < CL) {
      Xch* remote = cluster.map_shared_rank(x, threadIdx.x);
      remote->f[ph][rank][0] = f0; remote->f[ph][rank][1] = f1;
      remote->f[ph][rank][2] = f2; remote->f[ph][rank][3] = f3;
      remote->u[ph][rank][0] = u0; remote->u[ph][rank][1] = u1;
    }
    cluster.sync();
  }
  __device__ __forceinline__ float fsum(int k) const {
    float s = 0.f;
#pragma unroll
    for (int r = 0; r < CL; ++r) s += x->f[ph][r][k];
    return s;
  }
  __device__ __forceinline__ float fmax_(int k) const {
    float s = -INFINITY;
#pragma unroll
    for (int r = 0; r < CL; ++r) s = fmaxf(s, x->f[ph][r][k]);
    return s;
  }
  __device__ __forceinline__ uint32_t uor(int k) const {
    uint32_t s = 0;
#pragma unroll
    for (int r = 0; r < CL; ++r) s |= x->u[ph][r][k];
    return s;
  }
  __device__ __forceinline__ uint32_t umax(int k) const {
    uint32_t s = 0;
#pragma unroll
    for (int r = 0; r < CL; ++r) s = max(s, x->u[ph][r][k]);
    return s;
  }
  __device__ __forceinline__ void next() { ph ^= 1; }
};

// BATCH: grid (CL, B), one cluster per sequence (see BatchArgs); a frozen sequence's cluster exits before its first
// exchange (the whole cluster reads the same word).
// PER_SEQ (BATCH only): `temp` is the (B,) temperature array and the walk of sequence b scales both the target and the
// draft rows by 1/T[b]; otherwise `temp` is the scalar 1/T.
// MIXED (PER_SEQ only): the cluster of a sequence with ba.greedy[b] nonzero exits where a frozen one does and writes
// nothing (its walk is the greedy kernel's).
// STOP (PER_SEQ only): stop mode.  The fixed 0 / 2 end rule is compiled out; rank 0 then cuts the committed tokens at the
// sequence's stop ids and length limit (ba.stop_ids / ba.end_limit, stop_cut) and writes ST_FINISH / ST_END.
// SKIP_DEAD (PER_SEQ only; policy bit SQ_ACCEPT_SKIP_DEAD): a child whose token is -inf in its parent's raw draft row is
// dead and skipped: no test, no residual, q unchanged.  Every CTA reads the same fp16 word, so the skip is uniform.
template <bool BATCH, int NCH, bool PER_SEQ = false, bool MIXED = false, bool STOP = false, bool SKIP_DEAD = false>
__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(CNT) accept_stochastic_cluster_kernel(
    const __half* __restrict__ target_logits, int64_t ld_t, const __half* __restrict__ draft_logits, int64_t ld_d,
    const __half* __restrict__ r, const __half* __restrict__ noise, const int32_t* __restrict__ succ_off,
    const int32_t* __restrict__ succ, const int32_t* __restrict__ depth, int S, int V, SeqParam<PER_SEQ> temp,
    int64_t* __restrict__ tokens, int64_t* __restrict__ position_ids, int32_t* __restrict__ accept_idx,
    int32_t* __restrict__ state, int max_target_seq, int policy, BatchArgs ba) {
  static_assert(BATCH || !PER_SEQ, "per-sequence parameters need the batched kernel");
  static_assert(PER_SEQ || !MIXED, "a per-sequence policy needs the per-sequence temperature");
  static_assert(PER_SEQ || !STOP, "stop mode needs the per-sequence walk");
  static_assert(PER_SEQ || !SKIP_DEAD, "dead children come from processed draft rows of a per-sequence batch");
  __shared__ Xch xch;
  __shared__ float red[CNW];
  __shared__ int32_t sh_acc[1024];
  __shared__ float sh_own[2];                    // owner thread -> block: {etok, flag bits as float}
  if constexpr (NCH > 1) pdl_wait();
  const int b = seq_index<BATCH>(blockIdx.y);
  if (BATCH) {
    state += b * ST_WORDS;
    if (state[ST_FROZEN]) return;
    if (MIXED && ba.greedy[b]) return;
    target_logits += (int64_t)b * S * ld_t;
    r += b * ba.ld_seq;
    noise += b * ba.ld_noise;
    tokens += b * ba.ld_seq;
    position_ids += b * ba.ld_seq;
    accept_idx += b * ba.ld_acc;
  }
  __shared__ int32_t sh_stop[STOP ? SQ_MAX_STOP + 1 : 1];
  if constexpr (STOP) stop_row_load(sh_stop, ba.stop_ids, ba.end_limit, b);
  const float inv_T = inv_temp(temp, b);
  ClusterCtx cx{cg::this_cluster(), &xch, 0, 0};
  cx.rank = (int)cx.cluster.block_rank();
  const int P = state[ST_P];
  const int nvec = V / 8;
  const int cpb = (nvec + CL - 1) / CL;          // chunks per CTA (<= CNT * NCH)
  int chunk[NCH];
  bool active[NCH];
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    chunk[i] = cx.rank * cpb + i * CNT + threadIdx.x;
    active[i] = i * CNT + threadIdx.x < cpb && chunk[i] < nvec;
  }
  const uint4 NEG_INF = make_uint4(0xFC00FC00u, 0xFC00FC00u, 0xFC00FC00u, 0xFC00FC00u);
  Pack8 p[NCH], xd[NCH];
  int cur = 0, n_new = 0;
  bool terminal = false;
  while (true) {
    const int c0 = succ_off[cur], c1 = succ_off[cur + 1];
    const bool leaf = (c0 == c1);
    // load + scale both rows; softmax statistics of both in two exchanges
    float m1 = -INFINITY, m2 = -INFINITY;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      p[i].u = active[i] ? reinterpret_cast<const uint4*>(target_logits + cur * ld_t)[chunk[i]] : NEG_INF;
      xd[i].u = (active[i] && !leaf) ? reinterpret_cast<const uint4*>(draft_logits + ba.row<BATCH>(cur, b) * ld_d)[chunk[i]]
                                     : NEG_INF;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        p[i].h[e] = f2h(h2f(p[i].h[e]) * inv_T);
        xd[i].h[e] = f2h(h2f(xd[i].h[e]) * inv_T);
        m1 = fmaxf(m1, h2f(p[i].h[e]));
        m2 = fmaxf(m2, h2f(xd[i].h[e]));
      }
    }
    m1 = block_max<CNW>(m1, red);
    m2 = block_max<CNW>(m2, red);
    cx.exchange(m1, m2, 0.f, 0.f, 0u, 0u);
    const float mxt = cx.fmax_(0);
    float mxd = cx.fmax_(1);
    cx.next();
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        s1 += __expf(h2f(p[i].h[e]) - mxt);
        s2 += __expf(h2f(xd[i].h[e]) - mxd);
      }
    s1 = block_sum<CNW>(s1, red);
    s2 = block_sum<CNW>(s2, red);
    cx.exchange(s1, s2, 0.f, 0.f, 0u, 0u);
    const float sumt = cx.fsum(0);
    float sumd = cx.fsum(1);
    cx.next();
#pragma unroll
    for (int i = 0; i < NCH; ++i)
#pragma unroll
      for (int e = 0; e < 8; ++e) p[i].h[e] = f2h(__fdividef(__expf(h2f(p[i].h[e]) - mxt), sumt));   // p = softmax(target/T)
    if (leaf) break;                                         // residual = p   (SpecTree.py:143-144)
    int accepted = -1;
    for (int ci = c0; ci < c1; ++ci) {
      const int child = succ[ci];
      const int slot = P - 1 + child;
      const int tok = (int)tokens[slot];
      if constexpr (SKIP_DEAD) {
        const __half raw = draft_logits[ba.row<BATCH>(cur, b) * ld_d + tok];
        if (__half_as_ushort(raw) == 0xFC00u) continue;      // dead: p and q stay as they are
      }
      const int tc = tok >> 3, te = tok & 7;
      // owner of the tested token: chunk own_i of this thread (-1: not this thread)
      int own_i;
      if constexpr (NCH == 1) own_i = ((tc / cpb == cx.rank) && (threadIdx.x == tc % cpb)) ? 0 : -1;
      else own_i = ((tc / cpb == cx.rank) && ((tc % cpb) % CNT == threadIdx.x)) ? (tc % cpb) / CNT : -1;
      if (threadIdx.x == 0) { sh_own[0] = 0.f; sh_own[1] = 0.f; }
      __syncthreads();
      // speculative residual share: d = relu(fp16(p - q)), partial sum
      Pack8 dtmp[NCH];
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < NCH; ++i)
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float q = h2f(f2h(__fdividef(__expf(h2f(xd[i].h[e]) - mxd), sumd)));
          float d = rnd16(h2f(p[i].h[e]) - q);
          d = (d < 0.f) ? 0.f : d;                           // relu_; NaN propagates like torch
          dtmp[i].h[e] = f2h(d);
          s += d;
          if (own_i == i && e == te) {
            const float etok = __expf(h2f(xd[i].h[e]) - mxd);
            const float thr = rnd16(h2f(r[slot]) * q);       // r * q[token] in fp16
            const float pv = h2f(p[i].h[e]);
            // strict > (SpecTree.py:152); the SpecInfer policy accepts on >= (SpecInferTree.py:158)
            const int acc = ((policy & SQ_ACCEPT_GE) ? (pv >= thr) : (pv > thr)) ? 1 : 0;
            sh_own[0] = etok;
            sh_own[1] = (float)(acc | ((!(policy & SQ_ACCEPT_KEEP_Q) && h2f(xd[i].h[e]) >= mxd) ? 2 : 0));
          }
        }
      s = block_sum<CNW>(s, red);                            // (contains the barriers that publish sh_own)
      cx.exchange(s, sh_own[0], 0.f, 0.f, (uint32_t)sh_own[1], 0u);
      const float tot = rnd16(cx.fsum(0));
      const float etok = cx.fsum(1);
      const uint32_t flag = cx.uor(0);
      cx.next();
      if (flag & 1u) { accepted = child; break; }
#pragma unroll
      for (int i = 0; i < NCH; ++i)
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          p[i].h[e] = f2h(h2f(dtmp[i].h[e]) / tot);          // get_residual (utils.py:5-8)
          if (own_i == i && e == te && !(policy & SQ_ACCEPT_KEEP_Q))
            xd[i].h[e] = __ushort_as_half((unsigned short)0xFC00u);   // draft_logits[token] = min (SpecTree.py:156)
        }
      if (policy & SQ_ACCEPT_KEEP_Q) continue;               // SpecInfer: q stays softmax(draft/T) for every child
      if (flag & 2u) {                                       // rare: the masked token held the max -> new statistics
        float m = -INFINITY;
#pragma unroll
        for (int i = 0; i < NCH; ++i)
#pragma unroll
          for (int e = 0; e < 8; ++e) m = fmaxf(m, h2f(xd[i].h[e]));
        m = block_max<CNW>(m, red);
        cx.exchange(m, 0.f, 0.f, 0.f, 0u, 0u);
        mxd = cx.fmax_(0);
        cx.next();
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < NCH; ++i)
#pragma unroll
          for (int e = 0; e < 8; ++e) ss += __expf(h2f(xd[i].h[e]) - mxd);
        ss = block_sum<CNW>(ss, red);
        cx.exchange(ss, 0.f, 0.f, 0.f, 0u, 0u);
        sumd = cx.fsum(0);
        cx.next();
      } else {
        sumd -= etok;
      }
    }
    if (accepted < 0) break;                                 // residual = p   (:157)
    const int slot = P - 1 + accepted;
    if (threadIdx.x == 0) sh_acc[n_new] = slot;
    ++n_new;
    const int64_t t = tokens[slot];
    if (!STOP && (t == 0 || t == 2)) { terminal = true; break; }   // (:208)
    cur = accepted;
  }
  bool nan_flag = false;
  int64_t bonus = -1;
  if (!terminal) {
    uint32_t has_nan = 0u, best = 0u;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      if (active[i]) {
        Pack8 nz;
        nz.u = reinterpret_cast<const uint4*>(noise)[chunk[i]];
        // key index field: the vocabulary index (NCH == 1), or the CTA-local one (< cpb * 8 <= 16384)
        const uint32_t ib = NCH == 1 ? (uint32_t)chunk[i] * 8 : (uint32_t)(i * CNT + threadIdx.x) * 8;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          has_nan |= __hisnan(p[i].h[e]) ? 1u : 0u;
          const __half v = f2h(h2f(p[i].h[e]) / h2f(nz.h[e]));   // multinomial(1) = argmax(residual / Exp(1))  (:222)
          best = max(best, (c_ord16(v) << 16) | (0xFFFFu - (ib + e)));
        }
      }
    }
    has_nan = __syncthreads_or((int)has_nan) ? 1u : 0u;
    best = __reduce_max_sync(0xffffffffu, best);
    __shared__ uint32_t redu[CNW];
    if ((threadIdx.x & 31) == 0) redu[threadIdx.x >> 5] = best;
    __syncthreads();
    best = __reduce_max_sync(0xffffffffu, (threadIdx.x & 31) < CNW ? redu[threadIdx.x & 31] : 0u);
    cx.exchange(0.f, 0.f, 0.f, 0.f, has_nan, best);
    nan_flag = cx.uor(0) != 0u;                              // torch.isnan(residual).any()  (:219)
    if constexpr (NCH == 1) {
      bonus = (int64_t)(0xFFFFu - (cx.umax(1) & 0xFFFFu));
    } else {                                                 // higher value, then the lower rank (strict >)
      uint32_t bk = 0u;
      int br = 0;
      for (int rr = 0; rr < CL; ++rr) {
        const uint32_t k = cx.x->u[cx.ph][rr][1];
        if ((k >> 16) > (bk >> 16)) { bk = k; br = rr; }
      }
      bonus = (int64_t)br * cpb * 8 + (int64_t)(0xFFFFu - (bk & 0xFFFFu));
    }
    cx.next();
    if (nan_flag) terminal = true;
  }
  if (cx.rank != 0) return;
  __syncthreads();
  // a guided sequence gathers its accepted slots before it writes the bonus, so its committed tokens stay in its guide
  const bool bonus_first = !(BATCH && state[ST_GUIDED]);
  finish_verify(sh_acc, n_new, P, terminal, nan_flag, bonus, bonus_first, depth, S, tokens, position_ids, accept_idx,
                state, max_target_seq);
  if constexpr (STOP) stop_cut(sh_stop, n_new, P, terminal, tokens, state, max_target_seq);
}

}  // namespace sq

using namespace sq;

template <int NCH, bool SKIP_DEAD>
static int launch_accept_batch(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits, int64_t ld_d,
                               const sq_half* r, const sq_half* noise, const int32_t* succ_off, const int32_t* succ,
                               const int32_t* depth, int S, int V, int64_t* tokens, int64_t* position_ids,
                               int32_t* accept_idx, int32_t* state, int max_target_seq, int policy, void* stream,
                               const BatchArgs* batch, const float* T_seq) {
  if (batch->stop_ids) {
    if (batch->greedy)
      accept_stochastic_cluster_kernel<true, NCH, true, true, true, SKIP_DEAD>
          <<<dim3(CL, batch->B), CNT, 0, (cudaStream_t)stream>>>(
              (const __half*)target_logits, ld_t, (const __half*)draft_logits, ld_d, (const __half*)r,
              (const __half*)noise, succ_off, succ, depth, S, V, T_seq, tokens, position_ids, accept_idx, state,
              max_target_seq, policy, *batch);
    else
      accept_stochastic_cluster_kernel<true, NCH, true, false, true, SKIP_DEAD>
          <<<dim3(CL, batch->B), CNT, 0, (cudaStream_t)stream>>>(
              (const __half*)target_logits, ld_t, (const __half*)draft_logits, ld_d, (const __half*)r,
              (const __half*)noise, succ_off, succ, depth, S, V, T_seq, tokens, position_ids, accept_idx, state,
              max_target_seq, policy, *batch);
    SQ_CHECK_LAUNCH("sq_accept_stochastic_batch_stop");
    return SQ_OK;
  }
  if (batch->greedy) {
    accept_stochastic_cluster_kernel<true, NCH, true, true, false, SKIP_DEAD>
        <<<dim3(CL, batch->B), CNT, 0, (cudaStream_t)stream>>>(
            (const __half*)target_logits, ld_t, (const __half*)draft_logits, ld_d, (const __half*)r, (const __half*)noise,
            succ_off, succ, depth, S, V, T_seq, tokens, position_ids, accept_idx, state, max_target_seq, policy, *batch);
    SQ_CHECK_LAUNCH("sq_accept_stochastic_batch_mixed");
    return SQ_OK;
  }
  accept_stochastic_cluster_kernel<true, NCH, true, false, false, SKIP_DEAD>
      <<<dim3(CL, batch->B), CNT, 0, (cudaStream_t)stream>>>(
          (const __half*)target_logits, ld_t, (const __half*)draft_logits, ld_d, (const __half*)r, (const __half*)noise,
          succ_off, succ, depth, S, V, T_seq, tokens, position_ids, accept_idx, state, max_target_seq, policy, *batch);
  SQ_CHECK_LAUNCH("sq_accept_stochastic_batch_per_seq");
  return SQ_OK;
}

template <int NCH>
static int launch_accept_nch(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits, int64_t ld_d,
                             const sq_half* r, const sq_half* noise, const int32_t* succ_off, const int32_t* succ,
                             const int32_t* depth, int S, int V, float T, int64_t* tokens, int64_t* position_ids,
                             int32_t* accept_idx, int32_t* state, int max_target_seq, int policy, void* stream,
                             const BatchArgs* batch, const float* T_seq) {
  if (batch && T_seq) {
    if (policy & SQ_ACCEPT_SKIP_DEAD)
      return launch_accept_batch<NCH, true>(target_logits, ld_t, draft_logits, ld_d, r, noise, succ_off, succ, depth, S,
                                            V, tokens, position_ids, accept_idx, state, max_target_seq, policy, stream,
                                            batch, T_seq);
    return launch_accept_batch<NCH, false>(target_logits, ld_t, draft_logits, ld_d, r, noise, succ_off, succ, depth, S, V,
                                           tokens, position_ids, accept_idx, state, max_target_seq, policy, stream, batch,
                                           T_seq);
  }
  if (batch) {
    accept_stochastic_cluster_kernel<true, NCH><<<dim3(CL, batch->B), CNT, 0, (cudaStream_t)stream>>>(
        (const __half*)target_logits, ld_t, (const __half*)draft_logits, ld_d, (const __half*)r, (const __half*)noise,
        succ_off, succ, depth, S, V, 1.0f / T, tokens, position_ids, accept_idx, state, max_target_seq, policy, *batch);
    SQ_CHECK_LAUNCH("sq_accept_stochastic_batch");
    return SQ_OK;
  }
  accept_stochastic_cluster_kernel<false, NCH><<<CL, CNT, 0, (cudaStream_t)stream>>>(
      (const __half*)target_logits, ld_t, (const __half*)draft_logits, ld_d, (const __half*)r, (const __half*)noise,
      succ_off, succ, depth, S, V, 1.0f / T, tokens, position_ids, accept_idx, state, max_target_seq, policy, BatchArgs{});
  SQ_CHECK_LAUNCH("sq_accept_stochastic(cluster)");
  return SQ_OK;
}

int sq::launch_accept_cluster(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits, int64_t ld_d,
                              const sq_half* r, const sq_half* noise, const int32_t* succ_off, const int32_t* succ,
                              const int32_t* depth, int S, int V, float T, int64_t* tokens, int64_t* position_ids,
                              int32_t* accept_idx, int32_t* state, int max_target_seq, int policy, void* stream,
                              const BatchArgs* batch, const float* T_seq) {
  SQ_CHECK_ARG(V % 8 == 0 && V > 0 && V <= CL * CNT * 8 * 4, "sq_accept_stochastic: V=%d unsupported (multiple of 8, "
               "<= %d)", V, CL * CNT * 8 * 4);
  const int nch = (V + CL * CNT * 8 - 1) / (CL * CNT * 8);
  auto go = [&](auto kern_nch) {
    return launch_accept_nch<decltype(kern_nch)::value>(target_logits, ld_t, draft_logits, ld_d, r, noise, succ_off, succ,
                                                        depth, S, V, T, tokens, position_ids, accept_idx, state,
                                                        max_target_seq, policy, stream, batch, T_seq);
  };
  if (nch == 1) return go(std::integral_constant<int, 1>{});
  if (nch == 2) return go(std::integral_constant<int, 2>{});
  return go(std::integral_constant<int, 4>{});
}
