// Guided decoding: a per-sequence token automaton on the (B*S, V) target rows of a batched tree (include/sequoia_b200.h,
// sq_guide_*).  Unlike the stateless row processors, a guide carries state along the sequence: state word
// ST_GUIDE_STATE holds the state after the committed tokens and advances by at most max_depth + 1 transitions a step.
//   1. guide_states_kernel, grid (B): the state of every node of the tree, one level at a time (a node's state is one
//      transition from its parent's), one warp per node, into a (B, S) scratch.
//   2. guide_mask_kernel, grid (chunks, S, B): each row's state mask in 8-entry groups, as logit_bias_kernel applies an
//      allowed set (a group whose bits are all set is not read, an all-clear one is written without a read, a mixed one
//      is written back only if an entry changed).  A dead node (-1) gets an all -inf row.
//   3. guide_advance_kernel, grid (B) of one warp: the committed state through the step's committed tokens.
// A transition is warp-cooperative: the state's allowed bit, then a 32-ary search of its ascending edge ids (one round
// of 32 parallel loads narrows the range 32-fold), so a state with E edges costs about log32(E) dependent loads.
#include "sq_common.cuh"
#include "sq_guide.cuh"

namespace sq {

constexpr int GS_THREADS = 512;                         // 16 warps: the nodes of one tree level in one or a few rounds
constexpr int GM_THREADS = 256;
constexpr int GM_CHUNK = 4096;                          // ids per CTA: 2 groups of 8 per thread
constexpr int GM_GROUPS = GM_CHUNK / 8 / GM_THREADS;
constexpr uint16_t GUIDE_NEG_INF = 0xFC00u;

__global__ void __launch_bounds__(GS_THREADS)
    guide_states_kernel(const int64_t* __restrict__ table, const int64_t* __restrict__ tokens, int64_t ld_seq,
                        const int32_t* __restrict__ state, const int32_t* __restrict__ depth,
                        const uint32_t* __restrict__ tree_bits, int tree_words, int S, int V,
                        int32_t* __restrict__ node_state) {
  __shared__ int sh_state[1024];
  __shared__ int sh_parent[1024];
  __shared__ int sh_max_depth;
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int32_t* st = state + b * ST_WORDS;
  const int32_t* blob = guide_of(table, st, b);
  if (blob == nullptr) return;
  const GuideView g(blob);
  const int P = st[ST_P];
  const int64_t* tok = tokens + (int64_t)b * ld_seq;
  if (tid == 0) sh_max_depth = 0;
  __syncthreads();
  // the parent of node k: its highest ancestor-or-self bit below k (node 0 is every path's root)
  for (int k = tid; k < S; k += GS_THREADS) {
    int par = 0;
    if (k > 0) {
      const uint32_t* bits = tree_bits + (int64_t)k * tree_words;
      for (int w = (k - 1) >> 5; w >= 0; --w) {
        uint32_t m = bits[w];
        if (w == (k - 1) >> 5) m &= (k & 31) == 0 ? ~0u : ((1u << (k & 31)) - 1u);   // bits below k only
        if (m) { par = w * 32 + 31 - __clz(m); break; }
      }
      atomicMax(&sh_max_depth, depth[k]);
    }
    sh_parent[k] = par;
  }
  const int root = st[ST_GUIDE_STATE];
  if (tid == 0) sh_state[0] = root;
  __syncthreads();
  const int md = sh_max_depth;
  for (int d = 1; d <= md; ++d) {                       // level d reads level d-1's states only
    for (int k = 1 + warp; k < S; k += GS_THREADS / 32) {
      if (depth[k] != d) continue;                      // (uniform across the warp)
      const int slot = P - 1 + k;
      const int64_t t = slot < ld_seq ? tok[slot] : -1;
      const int s = guide_step(g, sh_state[sh_parent[k]], t, V);
      if (lane == 0) sh_state[k] = s;
    }
    __syncthreads();
  }
  for (int k = tid; k < S; k += GS_THREADS) node_state[(int64_t)b * S + k] = sh_state[k];
}

__global__ void __launch_bounds__(GM_THREADS)
    guide_mask_kernel(__half* __restrict__ logits, int64_t ld, int V, int S, const int32_t* __restrict__ state,
                      const int64_t* __restrict__ table, const int32_t* __restrict__ node_state, bool vec) {
  pdl_wait();
  pdl_trigger();
  const int c = blockIdx.x, k = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
  const int32_t* blob = guide_of(table, state + b * ST_WORDS, b);
  if (blob == nullptr) return;
  const GuideView g(blob);
  const int s = node_state[(int64_t)b * S + k];
  const bool dead = s < 0 || s >= g.n;
  const uint32_t* mask = dead ? nullptr : g.row(s);
  const int c0 = c * GM_CHUNK, c1 = min(c0 + GM_CHUNK, V);
  __half* row = logits + ((int64_t)b * S + k) * ld;
#pragma unroll
  for (int gi = 0; gi < GM_GROUPS; ++gi) {
    const int i = c0 + (gi * GM_THREADS + tid) * 8;
    if (i >= c1) break;
    const uint32_t bits = dead ? 0u : (mask[i >> 5] >> (i & 31)) & 0xffu;   // (V % 8 == 0: a group never crosses V)
    if (bits == 0xffu) continue;
    union {
      uint4 v;
      uint16_t h[8];
    } u;
    if (bits == 0u) {
#pragma unroll
      for (int e = 0; e < 8; ++e) u.h[e] = GUIDE_NEG_INF;
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
        if (!((bits >> e) & 1u) && u.h[e] != GUIDE_NEG_INF) {
          u.h[e] = GUIDE_NEG_INF;
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

__global__ void __launch_bounds__(32)
    guide_advance_kernel(const int64_t* __restrict__ table, const int64_t* __restrict__ tokens, int64_t ld_seq,
                         int32_t* __restrict__ state, int V) {
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.x;
  int32_t* st = state + b * ST_WORDS;
  const int32_t* blob = guide_of(table, st, b);
  if (blob == nullptr) return;
  int s = st[ST_GUIDE_STATE];
  if (s < 0) return;
  const GuideView g(blob);
  const int a = st[ST_ACCEPT_LEN];
  const int M = st[ST_M] > 0 ? st[ST_M] : (int)(ld_seq < INT32_MAX ? ld_seq : INT32_MAX);
  int n = (!st[ST_TERMINAL] && a < M) ? a + 1 : a;      // the walk's committed length (finish_verify's bonus_ok)
  if (st[ST_FINISH]) n = st[ST_END];                    // the stop walks' cut
  if ((int64_t)n > ld_seq) n = (int)ld_seq;
  const int64_t* tok = tokens + (int64_t)b * ld_seq;
  int pos = max(st[ST_GUIDE_POS], 0);
  for (; pos < n; ++pos) {
    const int nx = guide_step(g, s, tok[pos], V);
    if (nx < 0) break;
    s = nx;
  }
  __syncwarp();
  if (threadIdx.x == 0) {
    const bool died = pos < n;
    st[ST_GUIDE_STATE] = died ? -1 : s;
    st[ST_GUIDE_POS] = died ? pos : max(n, st[ST_GUIDE_POS]);
  }
}

}  // namespace sq

using namespace sq;

#define SQ_GUIDE_COMMON_ARGS(name)                                                                                      \
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH, name ": B=%d (1..%d)", B, SQ_MAX_BATCH);                                    \
  SQ_CHECK_ARG(V % 8 == 0 && V > 0 && V <= 131072, name ": V=%d must be a multiple of 8, <= 131072", V)

extern "C" int sq_guide_states_batch(const int64_t* guide_table, const int64_t* tokens, int64_t ld_seq,
                                     const int32_t* state, const int32_t* depth, const uint32_t* tree_bits,
                                     int tree_words, int S, int V, int32_t* node_state, int B, void* stream) {
  SQ_CHECK_ARG(guide_table && tokens && state && depth && tree_bits && node_state, "sq_guide_states_batch: null array");
  SQ_GUIDE_COMMON_ARGS("sq_guide_states_batch");
  SQ_CHECK_ARG(S >= 1 && S <= 1024 && tree_words == (S + 31) / 32,
               "sq_guide_states_batch: S=%d with tree_words=%d (S in 1..1024, tree_words = ceil(S/32))", S, tree_words);
  SQ_CHECK_ARG(ld_seq >= 1, "sq_guide_states_batch: ld_seq=%lld", (long long)ld_seq);
  launch_k(guide_states_kernel, dim3(B), dim3(GS_THREADS), 0, (cudaStream_t)stream, guide_table, tokens, ld_seq, state,
           depth, tree_bits, tree_words, S, V, node_state);
  SQ_CHECK_LAUNCH("sq_guide_states_batch");
  return SQ_OK;
}

extern "C" int sq_guide_mask_rows_batch(sq_half* logits, int64_t ld, int V, int S, const int32_t* state,
                                        const int64_t* guide_table, const int32_t* node_state, int B, void* stream) {
  SQ_CHECK_ARG(logits && state && guide_table && node_state, "sq_guide_mask_rows_batch: null array");
  SQ_GUIDE_COMMON_ARGS("sq_guide_mask_rows_batch");
  SQ_CHECK_ARG(ld >= V, "sq_guide_mask_rows_batch: ld=%lld < V=%d", (long long)ld, V);
  SQ_CHECK_ARG(S >= 1, "sq_guide_mask_rows_batch: S=%d", S);
  const bool vec = ((uintptr_t)logits & 15) == 0 && ld % 8 == 0;
  launch_k(guide_mask_kernel, dim3((V + GM_CHUNK - 1) / GM_CHUNK, S, B), dim3(GM_THREADS), 0, (cudaStream_t)stream,
           (__half*)logits, ld, V, S, state, guide_table, node_state, vec);
  SQ_CHECK_LAUNCH("sq_guide_mask_rows_batch");
  return SQ_OK;
}

extern "C" int sq_guide_advance_batch(const int64_t* guide_table, const int64_t* tokens, int64_t ld_seq, int32_t* state,
                                      int V, int B, void* stream) {
  SQ_CHECK_ARG(guide_table && tokens && state, "sq_guide_advance_batch: null array");
  SQ_GUIDE_COMMON_ARGS("sq_guide_advance_batch");
  SQ_CHECK_ARG(ld_seq >= 1, "sq_guide_advance_batch: ld_seq=%lld", (long long)ld_seq);
  launch_k(guide_advance_kernel, dim3(B), dim3(32), 0, (cudaStream_t)stream, guide_table, tokens, ld_seq, state, V);
  SQ_CHECK_LAUNCH("sq_guide_advance_batch");
  return SQ_OK;
}
