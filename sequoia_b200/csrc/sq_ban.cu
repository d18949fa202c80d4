// Per-sequence bad words and min_tokens on the (B*S, V) target rows of a batched tree (include/sequoia_b200.h,
// sq_ban_tokens_rows_batch).  Stateless: each step decides the bans from tokens and state.  One launch, grid (S, B),
// one CTA per target row (node k of sequence b):
//   1. warp 0 stages the last <= BAN_CTX tokens of the row's generated context in shared memory, oldest first: the tail
//      of the path tokens (ancestors-or-self j >= 1 of node k, slots P-1+j, as penalty_rows_kernel finds them), preceded
//      by the tail of the committed tokens at positions L .. P-1;
//   2. thread w tests word w (its prefix against the staged tail) and writes -inf at its last id on a match; threads
//      0 .. SQ_MAX_STOP-1 write -inf at the end ids while the row's position P + depth[k] is below min_end[b].
// Only -inf is written, never read back, so two threads writing the same entry are harmless and no CTA reads what
// another writes.
#include "sq_common.cuh"

namespace sq {

constexpr int BAN_THREADS = SQ_MAX_BAD_WORDS;           // one thread per word
constexpr int BAN_CTX = SQ_MAX_BAD_WORD_LEN - 1;         // the longest prefix a word can have
constexpr uint16_t BAN_NEG_INF = 0xFC00u;
static_assert(SQ_MAX_STOP <= BAN_THREADS, "one thread per end id");

__global__ void __launch_bounds__(BAN_THREADS)
    ban_tokens_kernel(__half* __restrict__ logits, int64_t ld, int V, const int64_t* __restrict__ tokens, int64_t ld_seq,
                      const int32_t* __restrict__ state, const int32_t* __restrict__ prompt_len,
                      const int32_t* __restrict__ depth, const uint32_t* __restrict__ tree_bits, int tree_words, int S,
                      const int32_t* __restrict__ words, const int32_t* __restrict__ word_len,
                      const int32_t* __restrict__ n_words, const int32_t* __restrict__ min_end,
                      const int32_t* __restrict__ end_ids) {
  __shared__ int ctx[BAN_CTX];                          // the staged tail, oldest first (-1: an id outside [0, V))
  __shared__ int n_ctx;
  pdl_wait();
  pdl_trigger();
  const int k = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int nw = min(max(n_words[b], 0), SQ_MAX_BAD_WORDS);
  const int me = min_end[b];
  if (state[b * ST_WORDS + ST_FROZEN] || (nw == 0 && me <= 0)) return;
  const int P = state[b * ST_WORDS + ST_P];
  __half* row = logits + ((int64_t)b * S + k) * ld;
  uint16_t* row16 = reinterpret_cast<uint16_t*>(row);
  if (tid < SQ_MAX_STOP && (int64_t)P + depth[k] < (int64_t)me) {
    const int t = end_ids[b * SQ_MAX_STOP + tid];
    if (t >= 0 && t < V) row16[t] = BAN_NEG_INF;
  }
  if (nw == 0) return;                                  // (uniform across the CTA: no thread waits below)
  if (tid < 32) {
    const int64_t* tok = tokens + (int64_t)b * ld_seq;
    const uint32_t* bits = tree_bits + (int64_t)k * tree_words;
    // lane l holds word l of the ancestor bits (node 0, the root, is committed, not a path token)
    const uint32_t mine = tid < tree_words ? bits[tid] & (tid == 0 ? ~1u : ~0u) : 0u;
    int incl = __popc(mine);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (tid >= o) incl += v;
    }
    const int n_path = __shfl_sync(0xffffffffu, incl, 31);
    const int n_gen_comm = max(0, P - max(prompt_len[b], 0));    // committed tokens at positions >= L
    const int keep_path = min(n_path, BAN_CTX);
    const int keep_comm = min(BAN_CTX - keep_path, n_gen_comm);
    // committed tail: slots P - keep_comm .. P - 1 at ctx[0 .. keep_comm)
    if (tid < keep_comm) {
      const int64_t slot = (int64_t)P - keep_comm + tid;
      const int64_t t = slot < ld_seq ? tok[slot] : -1;
      ctx[tid] = (t >= 0 && t < V) ? (int)t : -1;
    }
    // path tail: path index p (slot order) >= n_path - keep_path goes to ctx[keep_comm + p - (n_path - keep_path)]
    const int first = n_path - keep_path;
    for (int wd = 0; wd < tree_words; ++wd) {
      const uint32_t word = __shfl_sync(0xffffffffu, mine, wd);
      const int base = __shfl_sync(0xffffffffu, incl, wd) - __popc(word);
      if ((word >> tid) & 1u) {
        const int p = base + __popc(word & ((1u << tid) - 1u));
        if (p >= first) {
          const int j = wd * 32 + tid;
          const int64_t slot = (int64_t)P - 1 + j;
          const int64_t t = (j < S && slot < ld_seq) ? tok[slot] : -1;
          ctx[keep_comm + p - first] = (t >= 0 && t < V) ? (int)t : -1;
        }
      }
    }
    if (tid == 0) n_ctx = keep_comm + keep_path;
  }
  __syncthreads();
  if (tid >= nw) return;
  const int n = word_len[b * SQ_MAX_BAD_WORDS + tid];
  if (n < 1 || n > SQ_MAX_BAD_WORD_LEN || n - 1 > n_ctx) return;
  const int32_t* w = words + ((int64_t)b * SQ_MAX_BAD_WORDS + tid) * SQ_MAX_BAD_WORD_LEN;
  const int last = w[n - 1];
  if (last < 0 || last >= V) return;
  const int off = n_ctx - (n - 1);                      // the prefix w[0 .. n-2] against ctx[off .. n_ctx)
  bool match = true;
#pragma unroll
  for (int i = 0; i < BAN_CTX; ++i) {
    if (i < n - 1) {
      const int c = ctx[off + i];
      match &= c >= 0 && c == w[i];
    }
  }
  if (match) row16[last] = BAN_NEG_INF;
}

}  // namespace sq

using namespace sq;

extern "C" int sq_ban_tokens_rows_batch(sq_half* logits, int64_t ld, int V, const int64_t* tokens, int64_t ld_seq,
                                        const int32_t* state, const int32_t* prompt_len, const int32_t* depth,
                                        const uint32_t* tree_bits, int tree_words, int S, const int32_t* words,
                                        const int32_t* word_len, const int32_t* n_words, const int32_t* min_end,
                                        const int32_t* end_ids, int B, void* stream) {
  SQ_CHECK_ARG(logits && tokens && state && prompt_len && depth && tree_bits && words && word_len && n_words && min_end &&
                   end_ids,
               "sq_ban_tokens_rows_batch: null array");
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH, "sq_ban_tokens_rows_batch: B=%d (1..%d)", B, SQ_MAX_BATCH);
  SQ_CHECK_ARG(V % 8 == 0 && V > 0 && V <= 131072, "sq_ban_tokens_rows_batch: V=%d must be a multiple of 8, <= 131072",
               V);
  SQ_CHECK_ARG(ld >= V, "sq_ban_tokens_rows_batch: ld=%lld < V=%d", (long long)ld, V);
  SQ_CHECK_ARG(S >= 1 && tree_words == (S + 31) / 32 && tree_words <= 32,
               "sq_ban_tokens_rows_batch: S=%d with tree_words=%d (must be ceil(S/32) <= 32)", S, tree_words);
  SQ_CHECK_ARG(ld_seq >= 1, "sq_ban_tokens_rows_batch: ld_seq=%lld", (long long)ld_seq);
  launch_k(ban_tokens_kernel, dim3(S, B), dim3(BAN_THREADS), 0, (cudaStream_t)stream, (__half*)logits, ld, V, tokens,
           ld_seq, state, prompt_len, depth, tree_bits, tree_words, S, words, word_len, n_words, min_end, end_ids);
  SQ_CHECK_LAUNCH("sq_ban_tokens_rows_batch");
  return SQ_OK;
}
