// Constrained drafting: the per-sequence allowed set, logit bias, bad words and guide of a batched tree applied to its
// draft rows (include/sequoia_b200.h, sq_draft_rows_batch), so that the draft proposes only tokens the target rows can
// keep.  Draft row of node k, sequence b: row_base[k] + b * row_step[k].  One launch per tree level, grid (chunks, nk, B):
// CTA (c, j, b) owns ids [c*DR_CHUNK, (c+1)*DR_CHUNK) of node k = k0 + j's row.  Its result equals, bit for bit, the
// target-row sequence sq_logit_bias_rows_batch -> sq_ban_tokens_rows_batch -> sq_guide_mask_rows_batch on that row:
//   1. warp 0: node k's guide state, one transition (guide_step) from its parent's state in node_state (the committed
//      state for the root); chunk 0 writes it to node_state[b*S + k] for the next level.  Warp 1 stages the row's
//      generated context for the bad words (as ban_tokens_kernel does).
//   2. the chunk in 8-entry groups against the allowed set AND the state's mask (logit_bias_kernel's group pass: a group
//      whose bits are all set is not read, an all-clear one is written as -inf without a read, a mixed one is written back
//      only if an entry changed);
//   3. the banned ids that fall in the chunk become -inf (the end ids below min_end, the last ids of matching words);
//   4. the bias entries in the chunk: an entry whose logit is now -inf (masked or banned) is skipped as any non-finite
//      one, so the bias never overwrites what the mask, the ban or the guide set.  The ban and the guide write only -inf
//      and ignore what they overwrite; the bias changes only finite entries that neither touches.  So this order gives
//      the target rows' composition.
// Barriers separate 2, 3 and 4 (a group write-back in 2 may hold an entry 3 bans); no CTA touches another's ids.
#include "sq_common.cuh"
#include "sq_guide.cuh"

namespace sq {

constexpr int DR_THREADS = 256;
constexpr int DR_CHUNK = 4096;                          // ids per CTA: 2 groups of 8 per thread
constexpr int DR_GROUPS = DR_CHUNK / 8 / DR_THREADS;
constexpr int DR_IDS_PER_THREAD = SQ_MAX_LOGIT_BIAS / DR_THREADS;
constexpr uint16_t DR_NEG_INF = 0xFC00u;
static_assert(SQ_MAX_BAD_WORDS <= DR_THREADS && SQ_MAX_STOP <= DR_THREADS, "one thread per word and per end id");

constexpr int DR_CTX = SQ_MAX_BAD_WORD_LEN - 1;     // the longest prefix a word can have

// One warp (lane = its lane index) stages the last <= DR_CTX tokens of node k's generated context in ctx, oldest first
// (-1: an id outside [0, V)), and their count in *n_ctx: the tail of the path tokens (ancestors-or-self j >= 1 of node k
// in bits, the node's row of the tree bits, slots P-1+j), preceded by the tail of the committed tokens at positions
// L = prompt_len[b] .. P-1.  A block barrier must separate it from ban_word_id.
__device__ __forceinline__ void ban_stage_context(int* ctx, int* n_ctx, const int64_t* __restrict__ tok, int64_t ld_seq,
                                                  const uint32_t* __restrict__ bits, int tree_words, int S, int P,
                                                  const int32_t* __restrict__ prompt_len, int b, int V, int lane) {
  // lane l holds word l of the ancestor bits (node 0, the root, is committed, not a path token)
  const uint32_t mine = lane < tree_words ? bits[lane] & (lane == 0 ? ~1u : ~0u) : 0u;
  int incl = __popc(mine);
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  const int n_path = __shfl_sync(0xffffffffu, incl, 31);
  const int n_gen_comm = max(0, P - max(prompt_len[b], 0));    // committed tokens at positions >= L
  const int keep_path = min(n_path, DR_CTX);
  const int keep_comm = min(DR_CTX - keep_path, n_gen_comm);
  // committed tail: slots P - keep_comm .. P - 1 at ctx[0 .. keep_comm)
  if (lane < keep_comm) {
    const int64_t slot = (int64_t)P - keep_comm + lane;
    const int64_t t = slot < ld_seq ? tok[slot] : -1;
    ctx[lane] = (t >= 0 && t < V) ? (int)t : -1;
  }
  // path tail: path index p (slot order) >= n_path - keep_path goes to ctx[keep_comm + p - (n_path - keep_path)]
  const int first = n_path - keep_path;
  for (int wd = 0; wd < tree_words; ++wd) {
    const uint32_t word = __shfl_sync(0xffffffffu, mine, wd);
    const int base = __shfl_sync(0xffffffffu, incl, wd) - __popc(word);
    if ((word >> lane) & 1u) {
      const int p = base + __popc(word & ((1u << lane) - 1u));
      if (p >= first) {
        const int j = wd * 32 + lane;
        const int64_t slot = (int64_t)P - 1 + j;
        const int64_t t = (j < S && slot < ld_seq) ? tok[slot] : -1;
        ctx[keep_comm + p - first] = (t >= 0 && t < V) ? (int)t : -1;
      }
    }
  }
  if (lane == 0) *n_ctx = keep_comm + keep_path;
}

// The id that word wi of sequence b (words / word_len as sq_ban_tokens_rows_batch takes them) bans after the staged
// context ctx[0 .. n_ctx), or -1: its last id when its prefix ends the context and that id is in [0, V).
__device__ __forceinline__ int ban_word_id(const int* ctx, int n_ctx, const int32_t* __restrict__ words,
                                           const int32_t* __restrict__ word_len, int b, int wi, int V) {
  const int n = word_len[b * SQ_MAX_BAD_WORDS + wi];
  if (n < 1 || n > SQ_MAX_BAD_WORD_LEN || n - 1 > n_ctx) return -1;
  const int32_t* w = words + ((int64_t)b * SQ_MAX_BAD_WORDS + wi) * SQ_MAX_BAD_WORD_LEN;
  const int last = w[n - 1];
  if (last < 0 || last >= V) return -1;
  const int off = n_ctx - (n - 1);                      // the prefix w[0 .. n-2] against ctx[off .. n_ctx)
  bool match = true;
#pragma unroll
  for (int i = 0; i < DR_CTX; ++i) {
    if (i < n - 1) {
      const int c = ctx[off + i];
      match &= c >= 0 && c == w[i];
    }
  }
  return match ? last : -1;
}

struct DraftRowsArgs {
  __half* logits;
  int64_t ld;
  int V, S, k0, flags;
  const int32_t* row_base;
  const int32_t* row_step;
  const int32_t* state;
  // SQ_DRAFT_BIAS
  const uint32_t* allowed;
  int64_t allowed_words;
  const int32_t* has_mask;
  const int32_t* bias_ids;
  const float* bias_vals;
  const int32_t* n_bias;
  // SQ_DRAFT_BAN and SQ_DRAFT_GUIDE
  const int64_t* tokens;
  int64_t ld_seq;
  const uint32_t* tree_bits;
  int tree_words;
  // SQ_DRAFT_BAN
  const int32_t* prompt_len;
  const int32_t* depth;
  const int32_t* words;
  const int32_t* word_len;
  const int32_t* n_words;
  const int32_t* min_end;
  const int32_t* end_ids;
  // SQ_DRAFT_GUIDE
  const int64_t* guide_table;
  int32_t* node_state;
};

__global__ void __launch_bounds__(DR_THREADS) draft_rows_kernel(const DraftRowsArgs a, bool vec) {
  __shared__ int ctx[DR_CTX];
  __shared__ int n_ctx;
  __shared__ int sh_state;
  pdl_wait();
  pdl_trigger();
  const int c = blockIdx.x, k = a.k0 + blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
  const int32_t* st = a.state + b * ST_WORDS;
  if (st[ST_FROZEN]) return;
  const bool use_bias = a.flags & SQ_DRAFT_BIAS, use_ban = a.flags & SQ_DRAFT_BAN;
  const bool masked = use_bias && a.has_mask[b] != 0;
  const int nb = use_bias ? min(max(a.n_bias[b], 0), SQ_MAX_LOGIT_BIAS) : 0;
  const int nw = use_ban ? min(max(a.n_words[b], 0), SQ_MAX_BAD_WORDS) : 0;
  const int me = use_ban ? a.min_end[b] : 0;
  const int32_t* blob = (a.flags & SQ_DRAFT_GUIDE) ? guide_of(a.guide_table, st, b) : nullptr;
  if (!masked && nb == 0 && nw == 0 && me <= 0 && blob == nullptr) return;
  const int V = a.V, S = a.S, P = st[ST_P];
  const int64_t* tok = a.tokens + (int64_t)b * a.ld_seq;
  const uint32_t* bits = a.tree_bits + (int64_t)k * a.tree_words;
  if (blob != nullptr && tid < 32) {
    const GuideView g(blob);
    int s = st[ST_GUIDE_STATE];
    if (k > 0) {
      int par = 0;                                      // the highest ancestor-or-self bit below k (node 0 on every path)
      for (int w = (k - 1) >> 5; w >= 0; --w) {
        uint32_t m = bits[w];
        if (w == (k - 1) >> 5) m &= (k & 31) == 0 ? ~0u : ((1u << (k & 31)) - 1u);
        if (m) { par = w * 32 + 31 - __clz(m); break; }
      }
      const int slot = P - 1 + k;
      const int64_t t = slot < a.ld_seq ? tok[slot] : -1;
      s = guide_step(g, a.node_state[(int64_t)b * S + par], t, V);
    }
    if (tid == 0) {
      sh_state = s;
      if (c == 0) a.node_state[(int64_t)b * S + k] = s;
    }
  }
  if (nw > 0 && tid >= 32 && tid < 64)
    ban_stage_context(ctx, &n_ctx, tok, a.ld_seq, bits, a.tree_words, S, P, a.prompt_len, b, V, tid - 32);
  __syncthreads();
  const int c0 = c * DR_CHUNK, c1 = min(c0 + DR_CHUNK, V);
  __half* row = a.logits + ((int64_t)a.row_base[k] + (int64_t)b * a.row_step[k]) * a.ld;
  uint16_t* row16 = reinterpret_cast<uint16_t*>(row);
  const uint32_t* amask = masked ? a.allowed + (int64_t)b * a.allowed_words : nullptr;
  bool dead = false;
  const uint32_t* gmask = nullptr;
  if (blob != nullptr) {
    const GuideView g(blob);
    const int s = sh_state;
    dead = s < 0 || s >= g.n;
    gmask = dead ? nullptr : g.row(s);
  }
  if (masked || blob != nullptr) {
#pragma unroll
    for (int gi = 0; gi < DR_GROUPS; ++gi) {
      const int i = c0 + (gi * DR_THREADS + tid) * 8;
      if (i >= c1) break;
      uint32_t keep = 0xffu;                            // (V % 8 == 0: a group never crosses V or a word)
      if (masked) keep &= (amask[i >> 5] >> (i & 31)) & 0xffu;
      if (blob != nullptr) keep &= dead ? 0u : (gmask[i >> 5] >> (i & 31)) & 0xffu;
      if (keep == 0xffu) continue;
      union {
        uint4 v;
        uint16_t h[8];
      } u;
      if (keep == 0u) {
#pragma unroll
        for (int e = 0; e < 8; ++e) u.h[e] = DR_NEG_INF;
      } else {
        if (vec) {
          u.v = *reinterpret_cast<const uint4*>(row + i);
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e) u.h[e] = row16[i + e];
        }
        bool changed = false;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          if (!((keep >> e) & 1u) && u.h[e] != DR_NEG_INF) {
            u.h[e] = DR_NEG_INF;
            changed = true;
          }
        }
        if (!changed) continue;
      }
      if (vec) {
        *reinterpret_cast<uint4*>(row + i) = u.v;
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) row16[i + e] = u.h[e];
      }
    }
  }
  __syncthreads();                                      // the context is staged; the group write-backs are done
  if (tid < SQ_MAX_STOP && me > 0 && (int64_t)P + a.depth[k] < (int64_t)me) {   // (depth is read with the ban only)
    const int t = a.end_ids[b * SQ_MAX_STOP + tid];
    if (t >= c0 && t < c1) row16[t] = DR_NEG_INF;
  }
  if (tid < nw) {
    const int t = ban_word_id(ctx, n_ctx, a.words, a.word_len, b, tid, V);
    if (t >= c0 && t < c1) row16[t] = DR_NEG_INF;
  }
  if (nb == 0) return;                                  // (uniform across the CTA: no thread waits below)
  const int32_t* ids = a.bias_ids + (int64_t)b * SQ_MAX_LOGIT_BIAS;
  const float* vals = a.bias_vals + (int64_t)b * SQ_MAX_LOGIT_BIAS;
  int mine[DR_IDS_PER_THREAD];
#pragma unroll
  for (int u = 0; u < DR_IDS_PER_THREAD; ++u) {
    const int j = u * DR_THREADS + tid;
    mine[u] = j < nb ? ids[j] : INT32_MAX;
  }
  int lo = 0, hi = 0;                                   // (the counts' barriers also order the bans before the reads)
#pragma unroll
  for (int u = 0; u < DR_IDS_PER_THREAD; ++u) {
    lo += __syncthreads_count(mine[u] < c0);
    hi += __syncthreads_count(mine[u] < c1);
  }
  for (int j = lo + tid; j < hi; j += DR_THREADS) {
    const int t = ids[j];
    if (t < 0 || t >= V || (j > lo && ids[j - 1] == t)) continue;   // a repeated id: its first entry applies them all
    float x = h2f(row[t]);
    if (!isfinite(x)) continue;                         // (-inf here: masked, banned or outside the guide)
    for (int q = j; q < hi && ids[q] == t; ++q) {
      x = __fadd_rn(x, vals[q]);
      x = fminf(fmaxf(x, -65504.f), 65504.f);
      if (q + 1 < hi && ids[q + 1] == t) x = h2f(f2h(x));
    }
    row[t] = f2h(x);
  }
}

}  // namespace sq

using namespace sq;

extern "C" int sq_draft_rows_batch(sq_half* draft_logits, int64_t ld, int V, const int32_t* row_base,
                                   const int32_t* row_step, int k0, int nk, int S, const int32_t* state, int flags,
                                   const uint32_t* allowed, int64_t allowed_words, const int32_t* has_mask,
                                   const int32_t* bias_ids, const float* bias_vals, const int32_t* n_bias,
                                   const int64_t* tokens, int64_t ld_seq, const uint32_t* tree_bits, int tree_words,
                                   const int32_t* prompt_len, const int32_t* depth, const int32_t* words,
                                   const int32_t* word_len, const int32_t* n_words, const int32_t* min_end,
                                   const int32_t* end_ids, const int64_t* guide_table, int32_t* node_state, int B,
                                   void* stream) {
  SQ_CHECK_ARG(flags > 0 && (flags & ~(SQ_DRAFT_BIAS | SQ_DRAFT_BAN | SQ_DRAFT_GUIDE)) == 0,
               "sq_draft_rows_batch: flags=%d (a nonzero set of SQ_DRAFT_BIAS, SQ_DRAFT_BAN, SQ_DRAFT_GUIDE)", flags);
  SQ_CHECK_ARG(draft_logits && row_base && row_step && state, "sq_draft_rows_batch: null array");
  SQ_CHECK_ARG(!(flags & SQ_DRAFT_BIAS) || (allowed && has_mask && bias_ids && bias_vals && n_bias),
               "sq_draft_rows_batch: null logit-bias array");
  SQ_CHECK_ARG(!(flags & (SQ_DRAFT_BAN | SQ_DRAFT_GUIDE)) || (tokens && tree_bits),
               "sq_draft_rows_batch: null tokens or tree_bits");
  SQ_CHECK_ARG(!(flags & SQ_DRAFT_BAN) || (prompt_len && depth && words && word_len && n_words && min_end && end_ids),
               "sq_draft_rows_batch: null bad-words array");
  SQ_CHECK_ARG(!(flags & SQ_DRAFT_GUIDE) || (guide_table && node_state), "sq_draft_rows_batch: null guide array");
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH, "sq_draft_rows_batch: B=%d (1..%d)", B, SQ_MAX_BATCH);
  SQ_CHECK_ARG(V % 8 == 0 && V > 0 && V <= 131072, "sq_draft_rows_batch: V=%d must be a multiple of 8, <= 131072", V);
  SQ_CHECK_ARG(ld >= V, "sq_draft_rows_batch: ld=%lld < V=%d", (long long)ld, V);
  SQ_CHECK_ARG(S >= 1 && S <= 1024 && tree_words == (S + 31) / 32,
               "sq_draft_rows_batch: S=%d with tree_words=%d (S in 1..1024, tree_words = ceil(S/32))", S, tree_words);
  SQ_CHECK_ARG(nk >= 1 && ((k0 == 0 && nk == 1) || (k0 >= 1 && k0 + nk <= S)),
               "sq_draft_rows_batch: nodes [%d, %d) (the root alone, or a range in [1, S=%d))", k0, k0 + nk, S);
  SQ_CHECK_ARG(!(flags & SQ_DRAFT_BIAS) || allowed_words >= (V + 31) / 32,
               "sq_draft_rows_batch: allowed_words=%lld < ceil(V/32)=%d", (long long)allowed_words, (V + 31) / 32);
  SQ_CHECK_ARG(!(flags & (SQ_DRAFT_BAN | SQ_DRAFT_GUIDE)) || ld_seq >= 1, "sq_draft_rows_batch: ld_seq=%lld",
               (long long)ld_seq);
  DraftRowsArgs a{(__half*)draft_logits, ld, V, S, k0, flags, row_base, row_step, state, allowed, allowed_words,
                  has_mask, bias_ids, bias_vals, n_bias, tokens, ld_seq, tree_bits, tree_words, prompt_len, depth, words,
                  word_len, n_words, min_end, end_ids, guide_table, node_state};
  const bool vec = ((uintptr_t)draft_logits & 15) == 0 && ld % 8 == 0;
  launch_k(draft_rows_kernel, dim3((V + DR_CHUNK - 1) / DR_CHUNK, nk, B), dim3(DR_THREADS), 0, (cudaStream_t)stream, a,
           vec);
  SQ_CHECK_LAUNCH("sq_draft_rows_batch");
  return SQ_OK;
}
