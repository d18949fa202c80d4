// Per-sequence repetition, frequency and presence penalties on the (B*S, V) target rows of a batched tree
// (include/sequoia_b200.h, sq_penalize_rows_batch).  Stateless: each step recomputes the counts from tokens and state.
//   1. penalty_list_kernel, one CTA per sequence: bitonic sort of the P committed ids in shared memory, keyed
//      (id << 1) | (slot >= L), then the distinct (id, c_all, c_out) list to the scratch.
//   2. penalty_rows_kernel, one CTA per target row (node k of sequence b): the row's path tokens (ancestors-or-self j >= 1
//      of node k, slots P-1+j) are staged in shared memory; a path token found in the list (binary search) adds its path
//      count to that entry, one absent from it is penalised at its first path occurrence; then the threads walk the list.
//      Every affected logit is read and written exactly once.
#include "sq_common.cuh"

namespace sq {

constexpr int PEN_SORT_THREADS = 1024;
constexpr int PEN_ROW_THREADS = 256;
constexpr int PEN_MAX_PATH = 32 * 32;                   // tree_words <= 32
constexpr uint32_t PEN_NO_KEY = 0xffffffffu;            // an id outside [0, V), or padding: sorts last

__device__ __forceinline__ bool pen_neutral(const float* rep, const float* freq, const float* pres, int b) {
  return rep[b] == 1.0f && freq[b] == 0.0f && pres[b] == 0.0f;
}

// scratch of sequence b: [count][ids: ld_seq][c_all: ld_seq][c_out: ld_seq]
template <typename T>
__device__ __forceinline__ T* pen_list(T* scratch, int64_t ld_seq, int b) {
  return scratch + (int64_t)b * (3 * ld_seq + 1);
}

// the penalised value of one logit: each operation one IEEE fp32 round-to-nearest (no FMA contraction), then clamped to
// the fp16 range and rounded.  Non-finite logits are left alone.
__device__ __forceinline__ void pen_apply(__half* p, int c_all, int c_out, float rho, float f, float pr) {
  float x = h2f(*p);
  if (!isfinite(x)) return;
  if (c_all > 0) x = x < 0.f ? __fmul_rn(x, rho) : __fdiv_rn(x, rho);
  if (c_out > 0) {
    x = __fsub_rn(x, __fmul_rn(f, (float)c_out));
    x = __fsub_rn(x, pr);
  }
  *p = f2h(fminf(fmaxf(x, -65504.f), 65504.f));
}

__global__ void __launch_bounds__(PEN_SORT_THREADS)
    penalty_list_kernel(const int64_t* __restrict__ tokens, int64_t ld_seq, const int32_t* __restrict__ state,
                        const int32_t* __restrict__ prompt_len, const float* __restrict__ rep,
                        const float* __restrict__ freq, const float* __restrict__ pres, int V,
                        int32_t* __restrict__ scratch) {
  __shared__ uint32_t key[SQ_PENALTY_MAX_LEN];
  __shared__ int start[SQ_PENALTY_MAX_LEN + 1];
  __shared__ int wsum[PEN_SORT_THREADS / 32];
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.x, tid = threadIdx.x;
  if (state[b * ST_WORDS + ST_FROZEN] || pen_neutral(rep, freq, pres, b)) return;
  const int P = min(max(state[b * ST_WORDS + ST_P], 0), (int)ld_seq);
  const int L = prompt_len[b];
  int n2 = 1;
  while (n2 < P) n2 <<= 1;
  const int64_t* tok = tokens + (int64_t)b * ld_seq;
  for (int i = tid; i < n2; i += PEN_SORT_THREADS) {
    const int64_t t = i < P ? tok[i] : -1;
    key[i] = (t >= 0 && t < V) ? ((uint32_t)t << 1 | (i >= L ? 1u : 0u)) : PEN_NO_KEY;
  }
  __syncthreads();
  for (int k = 2; k <= n2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < n2; i += PEN_SORT_THREADS) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const uint32_t a = key[i], c = key[ixj];
          if ((a > c) == ((i & k) == 0)) {
            key[i] = c;
            key[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  // run starts (the first key of each distinct id); thread t scans its 4 consecutive keys, then a block exclusive scan
  constexpr int IT = SQ_PENALTY_MAX_LEN / PEN_SORT_THREADS;
  bool first[IT];
  int mine = 0;
#pragma unroll
  for (int u = 0; u < IT; ++u) {
    const int i = tid * IT + u;
    first[u] = i < n2 && key[i] != PEN_NO_KEY && (i == 0 || (key[i] >> 1) != (key[i - 1] >> 1));
    mine += first[u];
  }
  const int lane = tid & 31, w = tid >> 5;
  int incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) wsum[w] = incl;
  __syncthreads();
  if (w == 0) {
    int s = wsum[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += v;
    }
    wsum[lane] = s;                                     // inclusive over warps
  }
  __syncthreads();
  const int n_distinct = wsum[PEN_SORT_THREADS / 32 - 1];
  int r = (w ? wsum[w - 1] : 0) + incl - mine;          // run index of this thread's first start
#pragma unroll
  for (int u = 0; u < IT; ++u) {
    if (first[u]) start[r++] = tid * IT + u;
  }
  if (tid == 0) {
    int n_valid = n2;                                   // the invalid keys sort last
    while (n_valid > 0 && key[n_valid - 1] == PEN_NO_KEY) --n_valid;
    start[n_distinct] = n_valid;
  }
  __syncthreads();
  int32_t* list = pen_list(scratch, ld_seq, b);
  int32_t *ids = list + 1, *c_all = ids + ld_seq, *c_out = c_all + ld_seq;
  if (tid == 0) list[0] = n_distinct;
  for (int q = tid; q < n_distinct; q += PEN_SORT_THREADS) {
    const int s = start[q], e = start[q + 1];
    ids[q] = (int)(key[s] >> 1);
    c_all[q] = e - s;
    // the output slots of an id are the last keys of its run (the low bit sorts them after the prompt slots)
    int lo = s, hi = e;                                 // first key with the output bit in [s, e)
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (key[mid] & 1u) hi = mid; else lo = mid + 1;
    }
    c_out[q] = e - lo;
  }
}

__global__ void __launch_bounds__(PEN_ROW_THREADS)
    penalty_rows_kernel(__half* __restrict__ logits, int64_t ld, int V, const int64_t* __restrict__ tokens, int64_t ld_seq,
                        const int32_t* __restrict__ state, const uint32_t* __restrict__ tree_bits, int tree_words, int S,
                        const float* __restrict__ rep, const float* __restrict__ freq, const float* __restrict__ pres,
                        const int32_t* __restrict__ scratch) {
  __shared__ int path[PEN_MAX_PATH];                    // the row's path tokens (-1: outside [0, V))
  __shared__ int pcount[SQ_PENALTY_MAX_LEN];            // path occurrences of list entry i
  __shared__ int n_path;
  pdl_wait();
  pdl_trigger();
  const int k = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  if (state[b * ST_WORDS + ST_FROZEN] || pen_neutral(rep, freq, pres, b)) return;
  const float rho = rep[b], f = freq[b], pr = pres[b];
  const int P = state[b * ST_WORDS + ST_P];
  const int64_t* tok = tokens + (int64_t)b * ld_seq;
  const int32_t* list = pen_list(scratch, ld_seq, b);
  const int n = list[0];
  const int32_t *ids = list + 1, *c_all = ids + ld_seq, *c_out = c_all + ld_seq;
  __half* row = logits + ((int64_t)b * S + k) * ld;
  if (tid < 32) {                                       // ancestors-or-self j >= 1 of node k, in slot order
    const uint32_t* bits = tree_bits + (int64_t)k * tree_words;
    int base = 0;
    for (int wd = 0; wd < tree_words; ++wd) {
      const uint32_t word = bits[wd] & (wd == 0 ? ~1u : ~0u);
      const int j = wd * 32 + tid;
      if ((word >> tid) & 1u) {
        const int64_t slot = (int64_t)P - 1 + j;
        const int64_t t = (j < S && slot < ld_seq) ? tok[slot] : -1;
        path[base + __popc(word & ((1u << tid) - 1u))] = (t >= 0 && t < V) ? (int)t : -1;
      }
      base += __popc(word);
    }
    if (tid == 0) n_path = base;
  }
  for (int i = tid; i < n; i += PEN_ROW_THREADS) pcount[i] = 0;
  __syncthreads();
  const int d = n_path;
  for (int p = tid; p < d; p += PEN_ROW_THREADS) {
    const int t = path[p];
    if (t < 0) continue;
    bool first = true;
    for (int q = 0; q < p && first; ++q) first = path[q] != t;
    if (!first) continue;
    int cnt = 0;
    for (int q = p; q < d; ++q) cnt += path[q] == t;
    int lo = 0, hi = n;                                 // the sorted list: first id >= t
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (ids[mid] < t) lo = mid + 1; else hi = mid;
    }
    if (lo < n && ids[lo] == t) pcount[lo] = cnt;       // (distinct tokens: distinct entries)
    else pen_apply(row + t, cnt, cnt, rho, f, pr);      // only on the path: every occurrence is output
  }
  __syncthreads();
  for (int i = tid; i < n; i += PEN_ROW_THREADS) {
    const int pc = pcount[i];
    pen_apply(row + ids[i], c_all[i] + pc, c_out[i] + pc, rho, f, pr);
  }
}

}  // namespace sq

using namespace sq;

extern "C" int sq_penalize_rows_batch(sq_half* logits, int64_t ld, int V, const int64_t* tokens, int64_t ld_seq,
                                      const int32_t* state, const int32_t* prompt_len, const uint32_t* tree_bits,
                                      int tree_words, int S, const float* rep, const float* freq, const float* pres,
                                      int32_t* scratch, int64_t scratch_words, int B, void* stream) {
  SQ_CHECK_ARG(logits && tokens && state && prompt_len && tree_bits && rep && freq && pres && scratch,
               "sq_penalize_rows_batch: null array");
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH, "sq_penalize_rows_batch: B=%d (1..%d)", B, SQ_MAX_BATCH);
  SQ_CHECK_ARG(V % 8 == 0 && V > 0 && V <= 131072, "sq_penalize_rows_batch: V=%d must be a multiple of 8, <= 131072", V);
  SQ_CHECK_ARG(ld >= V, "sq_penalize_rows_batch: ld=%lld < V=%d", (long long)ld, V);
  SQ_CHECK_ARG(S >= 1 && tree_words == (S + 31) / 32 && tree_words <= 32,
               "sq_penalize_rows_batch: S=%d with tree_words=%d (must be ceil(S/32) <= 32)", S, tree_words);
  SQ_CHECK_ARG(ld_seq >= 1 && ld_seq <= SQ_PENALTY_MAX_LEN,
               "sq_penalize_rows_batch: ld_seq=%lld (1..%d: the context a penalty counts is at most %d tokens)",
               (long long)ld_seq, SQ_PENALTY_MAX_LEN, SQ_PENALTY_MAX_LEN);
  SQ_CHECK_ARG(scratch_words >= (int64_t)B * (3 * ld_seq + 1),
               "sq_penalize_rows_batch: scratch of %lld words, needs B * (3 * ld_seq + 1) = %lld", (long long)scratch_words,
               (long long)B * (3 * ld_seq + 1));
  cudaStream_t st = (cudaStream_t)stream;
  launch_k(penalty_list_kernel, dim3(B), dim3(PEN_SORT_THREADS), 0, st, tokens, ld_seq, state, prompt_len, rep, freq,
           pres, V, scratch);
  SQ_CHECK_LAUNCH("sq_penalize_rows_batch");
  launch_k(penalty_rows_kernel, dim3(S, B), dim3(PEN_ROW_THREADS), 0, st, (__half*)logits, ld, V, tokens, ld_seq, state,
           tree_bits, tree_words, S, rep, freq, pres, (const int32_t*)scratch);
  SQ_CHECK_LAUNCH("sq_penalize_rows_batch");
  return SQ_OK;
}
