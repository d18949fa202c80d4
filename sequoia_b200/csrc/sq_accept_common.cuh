// Shared by the single-CTA and the cluster accept kernels.
#pragma once
#include "sq_common.cuh"

namespace sq {

// Per-sequence addressing of the batched walks (sequence b = blockIdx.y): tokens / position_ids / r rows of ld_seq
// elements, noise rows of ld_noise, accept_idx rows of ld_acc, target logits (B*S, V), and the draft-logit row of node k
// at row_base[k] + b * row_step[k].  greedy: the (B,) per-sequence policy of the mixed walks (nonzero = greedy), nullptr
// for every other batched walk.  stop_ids / end_limit: the stop walks' per-sequence stop ids and length limits
// (StopRow), nullptr for every other walk.
struct BatchArgs {
  int B;
  int64_t ld_seq, ld_noise, ld_acc;
  const int32_t* row_base;
  const int32_t* row_step;
  const int32_t* greedy = nullptr;
  const int32_t* stop_ids = nullptr;
  const int32_t* end_limit = nullptr;
  template <bool BATCH>
  __device__ __forceinline__ int64_t row(int node, int b) const {
    return BATCH ? (int64_t)row_base[node] + (int64_t)b * row_step[node] : node;
  }
};

// batch == nullptr: the single-sequence kernel.  T_seq (batches only): the (B,) temperature array, used instead of T.
int launch_accept_cluster(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits, int64_t ld_d,
                          const sq_half* r, const sq_half* noise, const int32_t* succ_off, const int32_t* succ,
                          const int32_t* depth, int S, int V, float T, int64_t* tokens, int64_t* position_ids,
                          int32_t* accept_idx, int32_t* state, int max_target_seq, int policy, void* stream,
                          const BatchArgs* batch = nullptr, const float* T_seq = nullptr);

// policy bits: SQ_ACCEPT_GE / SQ_ACCEPT_KEEP_Q from include/sequoia_b200.h

// Post-processing shared by both walks.  Runs with the whole block; thread 0 does the (short, ordered) serial part.
// sh_acc[0..n_new) = accepted absolute slots; publishes state[].
// bonus_first: SpecTree writes the bonus token at slot a BEFORE gathering tokens[accept_list] (SpecTree.py:222-224), so
// an accepted node that happens to live at slot a is returned as the bonus token -- reproduced here; GreedyTree
// gathers first (GreedyTree.py:205-207).
__device__ __forceinline__ void finish_verify(const int32_t* sh_acc, int n_new, int P, bool terminal, bool nan_flag, int64_t bonus,
                              bool bonus_first, const int32_t* __restrict__ depth, int S, int64_t* __restrict__ tokens,
                              int64_t* __restrict__ position_ids, int32_t* __restrict__ accept_idx,
                              int32_t* __restrict__ state, int max_target_seq) {
  const int a = P + n_new;
  // Buffer bound (the reference raises an IndexError / shape error at the equivalent slice assignments): tokens[a] needs
  // a < M, the re-laid tree positions need a + S - 1 < M.  M travels in the state word (set by the Tree constructor);
  // 0 = unknown -> fall back to max_target_seq, which callers size as the buffer length.
  const int M = state[ST_M] > 0 ? state[ST_M] : max_target_seq;
  const bool prepare = !terminal && (a + 1 <= max_target_seq) && (a + S <= M);
  const bool bonus_ok = !terminal && a < M;
  if (threadIdx.x == 0) {
    if (bonus_ok && bonus_first) tokens[a] = bonus;         // SpecTree.py:222
    for (int j = 0; j < n_new; ++j) {                       // tokens[:a] = tokens[accept_list]  (SpecTree.py:224)
      const int src = sh_acc[j];
      accept_idx[j] = src;
      tokens[P + j] = tokens[src];
    }
    if (bonus_ok && !bonus_first) tokens[a] = bonus;        // GreedyTree.py:207
    if (prepare) {                                          // prepare_for_next_iter (SpecTree.py:261-271)
      for (int j = 0; j < n_new; ++j) position_ids[P + j] = position_ids[sh_acc[j]];
      position_ids[a] = a;
    }
    state[ST_ACCEPT_LEN] = a;
    state[ST_TERMINAL] = terminal ? 1 : 0;
    state[ST_N_NEW] = n_new;
    state[ST_P_OLD] = P;
    state[ST_BONUS] = terminal ? -1 : (int32_t)bonus;
    state[ST_NAN] = nan_flag ? 1 : 0;
    state[ST_SKIPPED] = (!terminal && !prepare) ? 1 : 0;
    if (prepare) state[ST_P] = a + 1;
  }
  __syncthreads();   // the gather above reads old tree positions that the re-lay below overwrites
  if (prepare) {
    for (int k = 1 + threadIdx.x; k < S; k += blockDim.x) position_ids[a + k] = (int64_t)depth[k] + a;
  }
}

// Stop mode (the STOP instances behind the *_batch_stop entry points).  Sequence b's stop row is staged in shared memory
// once, after the kernel's PDL wait: words [0, SQ_MAX_STOP) its stop ids (-1 = unused), word SQ_MAX_STOP its absolute
// length limit E_b (<= 0 = none).  A block barrier must separate the load from stop_cut.
__device__ __forceinline__ void stop_row_load(int32_t* sh_stop, const int32_t* __restrict__ stop_ids,
                                              const int32_t* __restrict__ end_limit, int b) {
  if (threadIdx.x < SQ_MAX_STOP) sh_stop[threadIdx.x] = stop_ids[b * SQ_MAX_STOP + threadIdx.x];
  else if (threadIdx.x == SQ_MAX_STOP) sh_stop[SQ_MAX_STOP] = end_limit[b];
}

// The cut, after finish_verify, by thread 0 (which wrote the committed tokens itself).  The walk ran without an end rule,
// so its output is tokens[P .. n), n = a + 1 when finish_verify wrote the bonus token at a, else a (NaN, or no room).
// The first stop id at j ends the sequence at j + 1; E_b ends it when E_b <= n; the earlier end wins, the stop id on a tie.
__device__ __forceinline__ void stop_cut(const int32_t* sh_stop, int n_new, int P, bool terminal,
                                         const int64_t* __restrict__ tokens, int32_t* __restrict__ state,
                                         int max_target_seq) {
  if (threadIdx.x != 0) return;
  const int a = P + n_new;
  const int M = state[ST_M] > 0 ? state[ST_M] : max_target_seq;
  const int n = (!terminal && a < M) ? a + 1 : a;           // finish_verify's bonus_ok
  int end = 0, finish = 0;
  for (int j = P; j < n && finish == 0; ++j) {
    const int64_t t = tokens[j];
#pragma unroll
    for (int k = 0; k < SQ_MAX_STOP; ++k)
      if (t == sh_stop[k]) finish = 1;
    if (finish) end = j + 1;
  }
  const int E = sh_stop[SQ_MAX_STOP];
  if (E > 0 && E <= n && (finish == 0 || E < end)) { end = E; finish = 2; }
  state[ST_FINISH] = finish;
  state[ST_END] = end;
}

}  // namespace sq
