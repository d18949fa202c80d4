// Draft-side sampling kernels (utils.py:5-32): temperature softmax, exponential-race sampling without
// replacement / top-k, residual distribution, row argmax.  One 1024-thread CTA per vocabulary row; the row lives in
// registers (16-byte striped loads, fully coalesced); reductions are warp-shuffle / redux + one shared-memory hop.
// HBM-bound by bytes (V*2 logits + V*2 rand per row) but in practice SFU/latency-bound: few rows, one SM each.
//
// fp16 rounding chain of the reference, reproduced step by step:
//   xt = fp16(x * (1/T))        torch's CUDA div-by-scalar multiplies by the fp32 reciprocal
//   q  = fp16(exp(xt - max) / sum)            softmax computes in fp32, rounds once
//   sc = fp16(fp16(log(u)) / q)               rand.log() and the division are separate fp16 ops
// exp uses ex2.approx (rel. error ~1e-6, far below the fp16 rounding that follows); log stays full precision
// because log(u) for u close to 1 decides the top ranks.
//
// Large vocabularies (WIDE = true, 32768 < V <= 131072; all but softmax_T): one thread-block cluster of ceil(V / 32768) CTAs per row.  CTA r
// owns the vocabulary slice [r*32768, (r+1)*32768) and runs the per-CTA code above on it (local indices, so keys keep
// their 16-bit index field); the row max, the softmax sum, the top-p histograms and the top-k / argmax candidates cross
// slices through distributed shared memory.  Every value is pushed into the slot of its source rank in the receiving
// CTAs, then one cluster barrier; partials are combined in rank order, so results do not depend on timing.  Slices are in
// index order, so candidates merged by (key, rank, local index) still resolve ties to the lower vocabulary index.
// WIDE = false is the single-CTA kernel, unchanged.
#include <cooperative_groups.h>

#include "sq_common.cuh"

namespace cg = cooperative_groups;

namespace sq {

constexpr int NT = 1024;
constexpr int NW = NT / 32;
constexpr int CH = 4;          // 16-byte chunks per thread: V <= NT*CH*8 = 32768
constexpr int SLICE = NT * CH * 8;      // vocabulary entries per CTA
constexpr int MAX_SLICES = 4;           // WIDE: V <= 131072
constexpr int WIDE_KMAX = 256;          // WIDE top-k: k_max bound (candidate buffer of the merging CTA)

// WIDE row geometry: the row (blockIdx.x / cluster size) and this CTA's slice.  The cluster rank and size are read from
// their special registers where needed rather than held in registers across the kernel.
struct Slice {
  int row, base, V;
  __device__ __forceinline__ int rank() const { return (int)cg::this_cluster().block_rank(); }
  __device__ __forceinline__ int n() const { return (int)cg::this_cluster().num_blocks(); }
};
__device__ __forceinline__ Slice slice_of(int V) {
  cg::cluster_group cl = cg::this_cluster();
  const int r = (int)cl.block_rank(), n = (int)cl.num_blocks();
  return Slice{(int)blockIdx.x / n, r * SLICE, min(SLICE, V - r * SLICE)};
}

// Block-uniform v -> slots[s.rank()] of every CTA of the cluster, then a cluster barrier (also a block barrier).  Each call
// site owns its slots, so no slot is written twice and a CTA may leave after its last exchange.
template <typename T>
__device__ __forceinline__ void cl_publish(T v, T* slots, const Slice& s) {
  cg::cluster_group cl = cg::this_cluster();
  if ((int)threadIdx.x < s.n()) *cl.map_shared_rank(&slots[s.rank()], (int)threadIdx.x) = v;
  cl.sync();
}
__device__ __forceinline__ float cl_max(float v, float* slots, const Slice& s) {
  cl_publish(v, slots, s);
  float m = -INFINITY;
  for (int r = 0; r < s.n(); ++r) m = fmaxf(m, slots[r]);
  return m;
}
__device__ __forceinline__ float cl_sum(float v, float* slots, const Slice& s) {
  cl_publish(v, slots, s);
  float t = 0.f;
  for (int r = 0; r < s.n(); ++r) t += slots[r];
  return t;
}

// slice-local key (ord16 << 16 | 0xFFFF - local index) of rank r -> row-wide key ordered by (value, lower rank, lower
// index); 0 stays 0 (no candidate)
__device__ __forceinline__ uint64_t wide_key(uint32_t key, int rank) {
  return key ? ((uint64_t)(key >> 16) << 32) | ((uint64_t)(MAX_SLICES - 1 - rank) << 16) | (key & 0xFFFFu) : 0ull;
}
__device__ __forceinline__ int64_t wide_index(uint64_t k) {
  const int rank = MAX_SLICES - 1 - (int)((k >> 16) & 0xFFFFu);
  return (int64_t)rank * SLICE + (int64_t)(0xFFFFu - (uint32_t)(k & 0xFFFFu));
}

__device__ __forceinline__ uint32_t block_max_u32(uint32_t v, uint32_t* red) {
  v = __reduce_max_sync(0xffffffffu, v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  return __reduce_max_sync(0xffffffffu, red[l]);   // NW == 32
}

// Loads the row striped: chunk c = i*NT + tid holds elements [8c, 8c+8).  Out-of-range chunks read as -inf.
__device__ __forceinline__ void load_row(const __half* __restrict__ row, int V, Pack8 (&x)[CH]) {
  const int nvec = V / 8;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = i * NT + threadIdx.x;
    if (c < nvec) x[i].u = reinterpret_cast<const uint4*>(row)[c];
    else x[i].u = make_uint4(0xFC00FC00u, 0xFC00FC00u, 0xFC00FC00u, 0xFC00FC00u);
  }
}

// in place: x <- fp16(x * inv_T); returns the row max and sum(exp(xt - max)) (fp32)
__device__ __forceinline__ void scale_and_stats(Pack8 (&x)[CH], float inv_T, float* red, float& mx, float& sum) {
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < CH; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      x[i].h[j] = f2h(h2f(x[i].h[j]) * inv_T);
      m = fmaxf(m, h2f(x[i].h[j]));
    }
  mx = block_max<NW>(m, red);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < CH; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) s += __expf(h2f(x[i].h[j]) - mx);
  sum = block_sum<NW>(s, red);
}

// scale_and_stats over the whole row of a WIDE cluster (xs: two exchange slot sets)
__device__ __forceinline__ void scale_and_stats_wide(Pack8 (&x)[CH], float inv_T, float* red, float (&xs)[2][MAX_SLICES],
                                                     const Slice& sl, float& mx, float& sum) {
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < CH; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      x[i].h[j] = f2h(h2f(x[i].h[j]) * inv_T);
      m = fmaxf(m, h2f(x[i].h[j]));
    }
  mx = cl_max(block_max<NW>(m, red), xs[0], sl);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < CH; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) s += __expf(h2f(x[i].h[j]) - mx);
  sum = cl_sum(block_sum<NW>(s, red), xs[1], sl);
}

__device__ __forceinline__ __half softmax_val(__half xt, float mx, float inv_sum_unused, float sum) {
  return f2h(__fdividef(__expf(h2f(xt) - mx), sum));
}

// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT) softmax_T_kernel(const __half* __restrict__ logits, int64_t ld_in,
                                                        __half* __restrict__ out, int64_t ld_out, int V, float inv_T) {
  __shared__ float red[NW];
  Pack8 x[CH];
  load_row(logits + blockIdx.x * ld_in, V, x);
  float mx, sum;
  scale_and_stats(x, inv_T, red, mx, sum);
  const int nvec = V / 8;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = i * NT + threadIdx.x;
    if (c < nvec) {
      Pack8 o;
#pragma unroll
      for (int j = 0; j < 8; ++j) o.h[j] = softmax_val(x[i].h[j], mx, 0.f, sum);
      reinterpret_cast<uint4*>(out + blockIdx.x * ld_out)[c] = o.u;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// WIDE top-k, after every CTA pushed its k_need best slice-local keys (0 = none) to gk[rank * k_need + i] of rank 0: the
// merging CTA ranks the n * k_need candidates (rank = number of larger row-wide keys) and writes the first k_need.
__device__ __forceinline__ void wide_topk_merge(const uint64_t* gk, int n, int k_need, int j, int k_max, int nb, int base,
                                                int64_t* __restrict__ positions, int64_t* __restrict__ tokens) {
  const int total = n * k_need;
  for (int q = threadIdx.x; q < total; q += NT) {
    const uint64_t mine = gk[q];
    if (mine == 0ull) continue;
    int rank = 0;
    for (int i = 0; i < total; ++i) rank += (gk[i] > mine) ? 1 : 0;
    if (rank < k_need) {
      const int64_t idx = wide_index(mine);
      if (positions) positions[(int64_t)j * k_max + rank] = idx;
      if (tokens && rank < nb) tokens[base + rank] = idx;
    }
  }
}

// BATCH: grid (n_parents, B); sequence b reads the logits row drow_base[node] + b * drow_step[node] of parent node `node`,
// its rand rows at rand + b * ld_rand_seq, writes tokens + b * ld_seq, and does nothing when frozen.
// WIDE: grid (n * n_parents, B), clusters of n = ceil(V / SLICE) CTAs; the whole cluster reads the same frozen word and
// k_need, so it takes every exit together.
// PER_SEQ (BATCH only): `temp` is the (B,) temperature array and mode 0 uses T[b]; otherwise `temp` is the scalar 1/T.
// MIXED (PER_SEQ only): `mode` is the (B,) int32 `greedy` array: sequence b draws as mode 1 when greedy[b] is nonzero, else
// as mode 0 at T[b].  b is the grid's y index, so the choice is uniform per block (per cluster when WIDE).
template <bool MIXED>
using ModeArg = typename std::conditional<MIXED, const int32_t*, int>::type;
__device__ __forceinline__ int seq_mode(int mode, int) { return mode; }
__device__ __forceinline__ int seq_mode(const int32_t* greedy, int b) { return greedy[b] ? 1 : 0; }

template <bool BATCH, bool WIDE, bool PER_SEQ = false, bool MIXED = false>
__global__ void __launch_bounds__(NT) sample_level_kernel(
    const __half* __restrict__ logits, int64_t ld_logits, const __half* __restrict__ rand, int64_t ld_rand,
    const int32_t* __restrict__ parent_rows, const int32_t* __restrict__ child_first,
    const int32_t* __restrict__ n_branch, int k_max, int V, SeqParam<PER_SEQ> temp, ModeArg<MIXED> mode,
    int64_t* __restrict__ positions, int64_t* __restrict__ tokens, const int32_t* __restrict__ state,
    const int32_t* __restrict__ drow_base, const int32_t* __restrict__ drow_step, int64_t ld_rand_seq, int64_t ld_seq) {
  static_assert(BATCH || !PER_SEQ, "per-sequence parameters need the batched kernel");
  static_assert(PER_SEQ || !MIXED, "a per-sequence policy needs the per-sequence temperature");
  __shared__ float red[NW];
  __shared__ uint32_t redu[NW];
  Slice sl{};
  if constexpr (WIDE) {
    pdl_wait();
    sl = slice_of(V);
  }
  const int j = WIDE ? sl.row : blockIdx.x;
  const int b = seq_index<BATCH>(blockIdx.y);
  if (BATCH) {
    state += b * ST_WORDS;
    if (state[ST_FROZEN]) return;
    tokens += b * ld_seq;
  }
  const int nb = n_branch ? n_branch[j] : 0;
  const int k_need = positions ? k_max : min(nb, k_max);   // children this row actually needs (block-uniform)
  if (k_need == 0) return;
  const int prow = parent_rows ? parent_rows[j] : j;
  const int64_t lrow = BATCH ? (int64_t)drow_base[prow] + (int64_t)b * drow_step[prow] : prow;
  if (BATCH && rand) rand += b * ld_rand_seq;
  if constexpr (WIDE) {                  // from here on: this CTA's slice, slice-local indices
    logits += sl.base;
    if (rand) rand += sl.base;
    V = sl.V;
  }
  const int nvec = V / 8;
  uint32_t key[CH * 8];
  {
    Pack8 x[CH];
    load_row(logits + lrow * ld_logits, V, x);
    if (seq_mode(mode, b) == 0) {
      const float inv_T = inv_temp(temp, b);
      float mx, sum;
      if constexpr (WIDE) {
        __shared__ float xs[2][MAX_SLICES];
        scale_and_stats_wide(x, inv_T, red, xs, sl, mx, sum);
      } else {
        scale_and_stats(x, inv_T, red, mx, sum);
      }
#pragma unroll
      for (int i = 0; i < CH; ++i) {
        const int c = i * NT + threadIdx.x;
        Pack8 u;
        if (c < nvec) u.u = reinterpret_cast<const uint4*>(rand + prow * ld_rand)[c];
        else u.u = make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float q = h2f(softmax_val(x[i].h[e], mx, 0.f, sum));
          const float lg = rnd16(logf(h2f(u.h[e])));                 // rand.log() in fp16
          const __half sc = f2h(__fdividef(lg, q));                  // / sampling_q in fp16
          key[i * 8 + e] = (c < nvec) ? ((ord16(sc) << 16) | (0xFFFFu - (uint32_t)(c * 8 + e))) : 0u;
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < CH; ++i) {
        const int c = i * NT + threadIdx.x;
#pragma unroll
        for (int e = 0; e < 8; ++e)
          key[i * 8 + e] = (c < nvec) ? ((ord16(x[i].h[e]) << 16) | (0xFFFFu - (uint32_t)(c * 8 + e))) : 0u;
      }
    }
  }
  // top-k over unique (score, index) keys; ties on the score resolve to the lower index
  uint32_t best = 0u;
#pragma unroll
  for (int e = 0; e < CH * 8; ++e) best = max(best, key[e]);
  const int base = tokens ? row_base(state, child_first[j]) : 0;
  // WIDE: the k_need best keys of this slice go to the merging CTA (rank 0) instead of the outputs
  uint64_t* gk = nullptr;
  if constexpr (WIDE) {
    __shared__ uint64_t gk_buf[MAX_SLICES * WIDE_KMAX];
    gk = gk_buf;
  }
  cg::cluster_group cl = cg::this_cluster();
  // Fast path (k <= 32): the k-th largest of the 32 warp maxima is a lower bound of the k-th largest key (at least k keys
  // reach it), and usually only a few more do: collect the keys >= that threshold in shared memory and rank them directly
  // (rank = number of larger candidates) -- three block barriers instead of two per selected child.
  if (k_need <= 32) {
    __shared__ uint32_t cand[NT];
    __shared__ int cnt;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t wmax = __reduce_max_sync(0xffffffffu, best);
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();                       // (also orders the last read of `redu`/`red` by scale_and_stats)
    if (lane == 0) redu[warp] = wmax;
    __syncthreads();
    uint32_t v = redu[lane], thr = 0u;     // NW == 32
    for (int r = 0; r < k_need; ++r) {
      thr = __reduce_max_sync(0xffffffffu, v);
      if (v == thr) v = 0u;
    }
    if (best >= thr && best != 0u) {       // (valid keys are never 0; thr == 0 only when few warps hold valid keys)
#pragma unroll
      for (int e = 0; e < CH * 8; ++e)
        if (key[e] >= thr && key[e] != 0u) {
          const int p = atomicAdd(&cnt, 1);
          if (p < NT) cand[p] = key[e];
        }
    }
    __syncthreads();
    const int C = cnt;
    if (C <= NT) {
      if ((int)threadIdx.x < C) {
        const uint32_t mine = cand[threadIdx.x];
        int rank = 0;
        for (int i = 0; i < C; ++i) rank += (cand[i] > mine) ? 1 : 0;
        if (rank < k_need) {
          if constexpr (WIDE) {
            *cl.map_shared_rank(&gk[sl.rank() * k_need + rank], 0) = wide_key(mine, sl.rank());
          } else {
            const int64_t idx = (int64_t)(0xFFFFu - (mine & 0xFFFFu));
            if (positions) positions[(int64_t)j * k_max + rank] = idx;
            if (tokens && rank < nb) tokens[base + rank] = idx;
          }
        }
      }
      if constexpr (WIDE) {
        for (int q = C + threadIdx.x; q < k_need; q += NT) *cl.map_shared_rank(&gk[sl.rank() * k_need + q], 0) = 0ull;
        cl.sync();
        if (sl.rank() == 0) wide_topk_merge(gk, sl.n(), k_need, j, k_max, nb, base, positions, tokens);
      }
      return;
    }
    // (more than NT keys reach the threshold -- e.g. an index-sorted row in top-k mode: fall through to the round loop)
  }
  for (int rnd = 0; rnd < k_need; ++rnd) {
    const uint32_t top = block_max_u32(best, redu);
    if constexpr (WIDE) {                 // a short last slice may run out of keys: push 0 (no candidate)
      if (top == 0u) {
        if (threadIdx.x == 0) *cl.map_shared_rank(&gk[sl.rank() * k_need + rnd], 0) = 0ull;
        continue;
      }
    }
    if (best == top) {                    // unique owner (keys embed the index)
      if constexpr (WIDE) {
        *cl.map_shared_rank(&gk[sl.rank() * k_need + rnd], 0) = wide_key(top, sl.rank());
      } else {
        const int64_t idx = (int64_t)(0xFFFFu - (top & 0xFFFFu));
        if (positions) positions[(int64_t)j * k_max + rnd] = idx;
        if (tokens && rnd < nb) tokens[base + rnd] = idx;
      }
      best = 0u;
#pragma unroll
      for (int e = 0; e < CH * 8; ++e) {
        if (key[e] == top) key[e] = 0u;
        best = max(best, key[e]);
      }
    }
  }
  if constexpr (WIDE) {
    cl.sync();
    if (sl.rank() == 0) wide_topk_merge(gk, sl.n(), k_need, j, k_max, nb, base, positions, tokens);
  }
}

// ---------------------------------------------------------------------------------------------
// Sampling WITH replacement (SpecInferTree.py:100-105: softmax(l/T).multinomial(k, replacement=True)) by exact integer
// inverse-CDF.  Every fp16 probability is an integer multiple of 2^-24, so w = q * 2^24 is an exact uint32 weight, the
// prefix sums are exact (order-independent) and draw c is the first index whose inclusive prefix exceeds
// (word_c * total) >> 32.  The oracle's `multinomial_words` does the same arithmetic: given equal q rows the draws agree
// bit for bit.  The striped row layout (chunk c = i*NT + tid = elements [8c, 8c+8)) is already in index order, so the
// CDF needs one 4-wide block scan of the per-chunk sums.
__global__ void __launch_bounds__(NT) sample_replace_kernel(
    const __half* __restrict__ logits, int64_t ld_logits, const int64_t* __restrict__ words,
    const int32_t* __restrict__ parent_rows, const int32_t* __restrict__ child_first,
    const int32_t* __restrict__ n_branch, int k_max, int V, float inv_T, int64_t* __restrict__ positions,
    int64_t* __restrict__ tokens, const int32_t* __restrict__ state) {
  __shared__ float red[NW];
  __shared__ uint32_t wtot[CH][NW];
  const int j = blockIdx.x;
  const int prow = parent_rows ? parent_rows[j] : j;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t w[CH * 8];
  uint32_t cs[CH], excl[CH];
  {
    Pack8 x[CH];
    load_row(logits + prow * ld_logits, V, x);
    float mx, sum;
    scale_and_stats(x, inv_T, red, mx, sum);
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      cs[i] = 0u;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float q = h2f(softmax_val(x[i].h[e], mx, 0.f, sum));        // fp16 q; padding chunks are exp(-inf) = 0
        w[i * 8 + e] = (uint32_t)(q * 16777216.f);                        // exact
        cs[i] += w[i * 8 + e];
      }
    }
  }
  // inclusive warp scans of the 4 chunk sums, then the warp totals
  uint32_t inc[CH];
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    uint32_t v = cs[i];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += t;
    }
    inc[i] = v;
    if (lane == 31) wtot[i][warp] = v;
  }
  __syncthreads();
  uint32_t total = 0u;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    uint32_t v = wtot[i][lane];                   // NW == 32
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += t;
    }
    const uint32_t before = __shfl_sync(0xffffffffu, v, (warp + 31) & 31);   // inclusive total of warps < warp
    excl[i] = total + (warp ? before : 0u) + inc[i] - cs[i];
    total += __shfl_sync(0xffffffffu, v, 31);
  }
  const int count = n_branch ? n_branch[j] : k_max;
  const int wbase = child_first ? child_first[j] : j * k_max;
  const int tbase = tokens ? row_base(state, child_first[j]) : 0;
  for (int c = 0; c < count; ++c) {
    const uint32_t word = (uint32_t)words[wbase + c];
    const uint32_t t = (uint32_t)(((uint64_t)word * (uint64_t)total) >> 32);
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      if (t >= excl[i] && t - excl[i] < cs[i]) {  // unique owner chunk
        uint32_t run = excl[i];
        int idx = -1;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          run += w[i * 8 + e];
          if (idx < 0 && run > t) idx = (i * NT + (int)threadIdx.x) * 8 + e;
        }
        if (positions) positions[(int64_t)j * k_max + c] = idx;
        if (tokens) tokens[tbase + c] = idx;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
template <bool WIDE>
__global__ void __launch_bounds__(NT) residual_kernel(const __half* __restrict__ p, const __half* __restrict__ q,
                                                       __half* __restrict__ out, int V) {
  __shared__ float red[NW];
  Slice sl{};
  if constexpr (WIDE) {                  // grid = one cluster over the row
    pdl_wait();
    sl = slice_of(V);
    p += sl.base;
    q += sl.base;
    out += sl.base;
    V = sl.V;
  }
  Pack8 a[CH], b[CH];
  load_row(p, V, a);
  load_row(q, V, b);
  const int nvec = V / 8;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < CH; ++i)
    if (i * NT + threadIdx.x < nvec) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float d = rnd16(h2f(a[i].h[e]) - h2f(b[i].h[e]));
        d = (d < 0.f) ? 0.f : d;                                   // relu_ (NaN propagates like torch)
        a[i].h[e] = f2h(d);
        s += d;
      }
    }
  float tot;
  if constexpr (WIDE) {
    __shared__ float xs[MAX_SLICES];
    tot = rnd16(cl_sum(block_sum<NW>(s, red), xs, sl));
  } else {
    tot = rnd16(block_sum<NW>(s, red));                            // .sum() of an fp16 tensor -> fp16
  }
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = i * NT + threadIdx.x;
    if (c < nvec) {
      Pack8 o;
#pragma unroll
      for (int e = 0; e < 8; ++e) o.h[e] = f2h(h2f(a[i].h[e]) / tot);
      reinterpret_cast<uint4*>(out)[c] = o.u;
    }
  }
}

// ---------------------------------------------------------------------------------------------
template <bool WIDE>
__global__ void __launch_bounds__(NT) argmax_rows_kernel(const __half* __restrict__ logits, int64_t ld, int V,
                                                          int64_t* __restrict__ out) {
  __shared__ uint32_t redu[NW];
  Slice sl{};
  Pack8 x[CH];
  if constexpr (WIDE) {
    pdl_wait();
    sl = slice_of(V);
    V = sl.V;
    load_row(logits + sl.row * ld + sl.base, V, x);
  } else {
    load_row(logits + blockIdx.x * ld, V, x);
  }
  const int nvec = V / 8;
  uint32_t best = 0u;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = i * NT + threadIdx.x;
    if (c < nvec) {
#pragma unroll
      for (int e = 0; e < 8; ++e) best = max(best, (ord16(x[i].h[e]) << 16) | (0xFFFFu - (uint32_t)(c * 8 + e)));
    }
  }
  const uint32_t top = block_max_u32(best, redu);
  if constexpr (WIDE) {                  // equal maxima in several slices: the lowest rank, i.e. the lowest index, wins
    __shared__ uint64_t gk[MAX_SLICES];
    cl_publish(wide_key(top, sl.rank()), gk, sl);
    if (sl.rank() == 0 && threadIdx.x == 0) {
      uint64_t m = 0ull;
      for (int r = 0; r < sl.n(); ++r) m = max(m, gk[r]);
      out[sl.row] = wide_index(m);
    }
  } else {
    if (threadIdx.x == 0) out[blockIdx.x] = (int64_t)(0xFFFFu - (top & 0xFFFFu));
  }
}


// ---------------------------------------------------------------------------------------------
// get_sampling_logits (utils.py:65-77): nucleus (top-p) filter, in place.  The reference sorts the row, takes
// cumsum(softmax(sorted / T)) in fp16 and removes every token whose PREDECESSOR's cumulative probability exceeds top_p
// (the first sorted token is always kept).  No sort here: the fp16 probabilities are integer multiples of 2^-24, so
// "mass of all tokens ranked before token i" is an exact integer S(i) that a two-level histogram over the 16-bit
// order-preserving key of fp16(logit / T) yields directly (high byte, then low byte inside the boundary bin; per-warp
// private histograms, integer atomics => order-independent, deterministic).  Token i is removed iff
// fp16(S(i) * 2^-24) > fp16(top_p) -- the comparison torch performs.  Tokens with the SAME fp16 logit tie: they are
// ranked by ascending index (a stable descending sort), resolved with a block scan over the boundary key only.
// (torch's cumsum adds the same fp16 terms in fp32 in scan order; the exact sum differs from it by < 2^-20 relative, far
// below the fp16 rounding of the comparison.)
__device__ __forceinline__ bool topp_pred(uint32_t S, float tp) { return h2f(f2h((float)S * (1.0f / 16777216.f))) > tp; }

// WIDE: the histograms are summed over the cluster (every CTA then selects the same boundary bins, so all take the same
// exits), and the boundary tie group is ranked across slices by an exclusive prefix of the per-slice counts in rank order.
// PER_SEQ: `temp` / `top_p` are (B,) arrays and row r belongs to sequence r / rows_per_seq; a row whose top_p >= 1 is left
// untouched (the whole cluster reads the same value).  Otherwise `temp` is the scalar 1/T and `top_p` fp16(top_p) < 1.
template <bool WIDE, bool PER_SEQ = false>
__global__ void __launch_bounds__(NT) top_p_filter_kernel(__half* __restrict__ logits, int64_t ld, int V,
                                                           SeqParam<PER_SEQ> temp, SeqParam<PER_SEQ> top_p,
                                                           int rows_per_seq) {
  __shared__ float red[NW];
  __shared__ uint32_t whist[NW][256];
  __shared__ uint32_t hist[256];
  __shared__ int sel[2];            // boundary bin, mass ranked before it
  __shared__ uint32_t wtot[CH][NW];
  Slice sl{};
  __half* row;
  if constexpr (WIDE || PER_SEQ) pdl_wait();
  if constexpr (WIDE) {
    sl = slice_of(V);
    row = logits + sl.row * ld + sl.base;
    V = sl.V;
  } else {
    row = logits + blockIdx.x * ld;
  }
  float inv_T, tp;
  if constexpr (PER_SEQ) {
    const int seq = (WIDE ? sl.row : (int)blockIdx.x) / rows_per_seq;
    if (top_p[seq] >= 1.0f) return;                  // utils.py:68: only when top_p < 1
    inv_T = inv_temp(temp, seq);
    tp = rnd16(top_p[seq]);                          // torch compares in the tensor's dtype (fp16)
  } else {
    inv_T = temp;
    tp = top_p;
  }
  const int nvec = V / 8;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  Pack8 xt[CH];
  load_row(row, V, xt);
  float mx, sum;
  if constexpr (WIDE) {
    __shared__ float xs[2][MAX_SLICES];
    scale_and_stats_wide(xt, inv_T, red, xs, sl, mx, sum);
  } else {
    scale_and_stats(xt, inv_T, red, mx, sum);
  }
  uint32_t before = 0u;             // mass ranked before the current boundary bin
  int hi = -1, key_b = -1;
  for (int level = 0; level < 2; ++level) {
    for (int i = threadIdx.x; i < NW * 256; i += NT) (&whist[0][0])[i] = 0u;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < CH; ++i)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const uint32_t k = ord16(xt[i].h[e]);
        const uint32_t w = (uint32_t)(h2f(softmax_val(xt[i].h[e], mx, 0.f, sum)) * 16777216.f);
        if (w != 0u && (level == 0 || (int)(k >> 8) == hi)) atomicAdd(&whist[warp][level == 0 ? (k >> 8) : (k & 255u)], w);
      }
    __syncthreads();
    if constexpr (WIDE) {
      __shared__ uint32_t ghist[2][MAX_SLICES][256];
      cg::cluster_group cl = cg::this_cluster();
      if (threadIdx.x < 256) {
        uint32_t t = 0u;
#pragma unroll 8
        for (int w = 0; w < NW; ++w) t += whist[w][threadIdx.x];
        for (int r = 0; r < sl.n(); ++r) *cl.map_shared_rank(&ghist[level][sl.rank()][threadIdx.x], r) = t;
      }
      cl.sync();
      if (threadIdx.x < 256) {
        uint32_t t = 0u;
        for (int r = 0; r < sl.n(); ++r) t += ghist[level][r][threadIdx.x];
        hist[threadIdx.x] = t;
      }
    } else {
      if (threadIdx.x < 256) {
        uint32_t t = 0u;
#pragma unroll 8
        for (int w = 0; w < NW; ++w) t += whist[w][threadIdx.x];
        hist[threadIdx.x] = t;
      }
    }
    if (threadIdx.x == 0) sel[0] = -1;
    __syncthreads();
    if (warp == 0) {
      // lane l owns bins 255-8l .. 248-8l (descending order of value); exclusive scan over the lanes
      uint32_t m[8], tot = 0u;
#pragma unroll
      for (int b = 0; b < 8; ++b) { m[b] = hist[255 - 8 * lane - b]; tot += m[b]; }
      uint32_t inc = tot;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
      }
      uint32_t a = before + inc - tot;
#pragma unroll
      for (int b = 0; b < 8; ++b) {
        if (!topp_pred(a, tp) && topp_pred(a + m[b], tp)) { sel[0] = 255 - 8 * lane - b; sel[1] = (int)a; }   // unique
        a += m[b];
      }
    }
    __syncthreads();
    const int bb = sel[0];
    if (bb < 0) return;             // the whole row stays below top_p: nothing to remove (block-uniform)
    before = (uint32_t)sel[1];
    if (level == 0) hi = bb; else key_b = (hi << 8) | bb;
    __syncthreads();
  }
  // ties on the boundary key: the first t_keep of them (ascending index) stay
  uint32_t w_b = 0u;
  int cs[CH], excl[CH];
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    cs[i] = 0;
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if ((int)ord16(xt[i].h[e]) == key_b) {
        ++cs[i];
        w_b = (uint32_t)(h2f(softmax_val(xt[i].h[e], mx, 0.f, sum)) * 16777216.f);
      }
  }
  w_b = __reduce_max_sync(0xffffffffu, w_b);
  if (lane == 0) red[warp] = __uint_as_float(w_b);
  int inc[CH];
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    int v = cs[i];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += t;
    }
    inc[i] = v;
    if (lane == 31) wtot[i][warp] = (uint32_t)v;
  }
  __syncthreads();
  w_b = __reduce_max_sync(0xffffffffu, __float_as_uint(red[lane]));          // NW == 32: every warp gets the bin's weight
  int total = 0;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    int v = (int)wtot[i][lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += t;
    }
    const int prev = __shfl_sync(0xffffffffu, v, (warp + 31) & 31);
    excl[i] = total + (warp ? prev : 0) + inc[i] - cs[i];
    total += __shfl_sync(0xffffffffu, v, 31);
  }
  if constexpr (WIDE) {             // tie members in lower slices rank first; w_b from a slice that holds the key
    __shared__ uint32_t gcnt[MAX_SLICES], gw[MAX_SLICES];
    cg::cluster_group cl = cg::this_cluster();
    if ((int)threadIdx.x < sl.n()) {
      *cl.map_shared_rank(&gcnt[sl.rank()], (int)threadIdx.x) = (uint32_t)total;
      *cl.map_shared_rank(&gw[sl.rank()], (int)threadIdx.x) = w_b;
    }
    cl.sync();
    int below = 0;
    total = 0;
    for (int r = 0; r < sl.n(); ++r) {
      if (r < sl.rank()) below += (int)gcnt[r];
      total += (int)gcnt[r];
      w_b = max(w_b, gw[r]);
    }
#pragma unroll
    for (int i = 0; i < CH; ++i) excl[i] += below;
  }
  // smallest t with pred(before + t * w_b): tie ranks >= t are removed (pred(before) is false, pred at t = total true)
  int lo = 0, hi_t = total;
  while (lo < hi_t) {
    const int mid = (lo + hi_t) >> 1;
    if (topp_pred(before + (uint32_t)mid * w_b, tp)) hi_t = mid; else lo = mid + 1;
  }
  const int t_keep = lo;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = i * NT + threadIdx.x;
    if (c >= nvec) continue;
    bool any = false;
    bool rm[8];
    int rank = excl[i];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = (int)ord16(xt[i].h[e]);
      rm[e] = (k < key_b) || (k == key_b && rank >= t_keep);
      if (k == key_b) ++rank;
      any |= rm[e];
    }
    if (any) {
      Pack8 x;
      x.u = reinterpret_cast<const uint4*>(row)[c];
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (rm[e]) x.h[e] = __ushort_as_half((unsigned short)0xFC00u);     // -inf
      reinterpret_cast<uint4*>(row)[c] = x.u;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Top-k filter, in place: exactly k tokens of the row keep their logit and every other one becomes -inf.  The ranking is a
// stable descending sort of the raw fp16 logits (value descending, equal values by ascending index), so the kept set does
// not depend on the temperature.  No sort: top_p_filter_kernel's two-level histogram select with token COUNTS in place of
// probability masses -- level 0 finds the high byte of the k-th key, level 1 its low byte inside that bin.  Counts are
// integers, so the result does not depend on the order of the atomics.  Keys above the boundary key stay, keys below it are
// removed, and of the tokens equal to it the first k - (count ranked before it) by index stay.
// WIDE: as top_p_filter_kernel (cluster-summed histograms; the boundary tie group ranked across slices in rank order).
// PER_SEQ: `top_k` is the (B,) int32 array and row r belongs to sequence r / rows_per_seq; a row whose k <= 0 or k >= V is
// left untouched (the whole cluster reads the same k).  Otherwise `top_k` is the scalar k, 0 < k < V.
template <bool PER_SEQ>
using SeqInt = typename std::conditional<PER_SEQ, const int32_t*, int>::type;

template <bool WIDE, bool PER_SEQ = false>
__global__ void __launch_bounds__(NT) top_k_filter_kernel(__half* __restrict__ logits, int64_t ld, int V,
                                                           SeqInt<PER_SEQ> top_k, int rows_per_seq) {
  __shared__ uint32_t whist[NW][256];
  __shared__ uint32_t hist[256];
  __shared__ int sel[2];            // boundary bin, count ranked before it
  __shared__ uint32_t wtot[CH][NW];
  pdl_wait();
  Slice sl{};
  __half* row;
  if constexpr (WIDE) sl = slice_of(V);
  int k;
  if constexpr (PER_SEQ) {
    k = top_k[(WIDE ? sl.row : (int)blockIdx.x) / rows_per_seq];
    if (k <= 0 || k >= V) return;
  } else {
    k = top_k;
  }
  if constexpr (WIDE) {
    row = logits + sl.row * ld + sl.base;
    V = sl.V;
  } else {
    row = logits + blockIdx.x * ld;
  }
  const int nvec = V / 8;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  Pack8 x[CH];
  load_row(row, V, x);
  uint32_t before = 0u;             // tokens ranked before the current boundary bin
  int hi = -1, key_b = -1;
  for (int level = 0; level < 2; ++level) {
    for (int i = threadIdx.x; i < NW * 256; i += NT) (&whist[0][0])[i] = 0u;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < CH; ++i)
      if (i * NT + (int)threadIdx.x < nvec) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const uint32_t key = topk_key(x[i].h[e]);
          if (level == 0 || (int)(key >> 8) == hi) atomicAdd(&whist[warp][level == 0 ? (key >> 8) : (key & 255u)], 1u);
        }
      }
    __syncthreads();
    uint32_t t = 0u;
    if (threadIdx.x < 256) {
#pragma unroll 8
      for (int w = 0; w < NW; ++w) t += whist[w][threadIdx.x];
    }
    if constexpr (WIDE) {
      __shared__ uint32_t ghist[2][MAX_SLICES][256];
      cg::cluster_group cl = cg::this_cluster();
      if (threadIdx.x < 256)
        for (int r = 0; r < sl.n(); ++r) *cl.map_shared_rank(&ghist[level][sl.rank()][threadIdx.x], r) = t;
      cl.sync();
      if (threadIdx.x < 256) {
        t = 0u;
        for (int r = 0; r < sl.n(); ++r) t += ghist[level][r][threadIdx.x];
      }
    }
    if (threadIdx.x < 256) hist[threadIdx.x] = t;
    if (threadIdx.x == 0) sel[0] = -1;
    __syncthreads();
    if (warp == 0) {
      // lane l owns bins 255-8l .. 248-8l (descending order of value); exclusive scan over the lanes
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
        if (a < (uint32_t)k && a + m[b] >= (uint32_t)k) { sel[0] = 255 - 8 * lane - b; sel[1] = (int)a; }   // unique
        a += m[b];
      }
    }
    __syncthreads();
    const int bb = sel[0];
    if (bb < 0) return;             // (0 < k < V always finds a bin; block- and cluster-uniform all the same)
    before = (uint32_t)sel[1];
    if (level == 0) hi = bb; else key_b = (hi << 8) | bb;
    __syncthreads();
  }
  // ties on the boundary key: the first k - before of them (ascending index) stay
  int cs[CH], excl[CH];
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    cs[i] = 0;
    if (i * NT + (int)threadIdx.x < nvec) {
#pragma unroll
      for (int e = 0; e < 8; ++e) cs[i] += ((int)topk_key(x[i].h[e]) == key_b) ? 1 : 0;
    }
  }
  int inc[CH];
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    int v = cs[i];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int s = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += s;
    }
    inc[i] = v;
    if (lane == 31) wtot[i][warp] = (uint32_t)v;
  }
  __syncthreads();
  int total = 0;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    int v = (int)wtot[i][lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int s = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += s;
    }
    const int prev = __shfl_sync(0xffffffffu, v, (warp + 31) & 31);
    excl[i] = total + (warp ? prev : 0) + inc[i] - cs[i];
    total += __shfl_sync(0xffffffffu, v, 31);
  }
  if constexpr (WIDE) {             // tie members in lower slices rank first
    __shared__ uint32_t gcnt[MAX_SLICES];
    cg::cluster_group cl = cg::this_cluster();
    if ((int)threadIdx.x < sl.n()) *cl.map_shared_rank(&gcnt[sl.rank()], (int)threadIdx.x) = (uint32_t)total;
    cl.sync();
    int below = 0;
    for (int r = 0; r < sl.rank(); ++r) below += (int)gcnt[r];
#pragma unroll
    for (int i = 0; i < CH; ++i) excl[i] += below;
  }
  const int t_keep = k - (int)before;
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = i * NT + threadIdx.x;
    if (c >= nvec) continue;
    bool any = false;
    int rank = excl[i];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int key = (int)topk_key(x[i].h[e]);
      const bool rm = (key < key_b) || (key == key_b && rank >= t_keep);
      if (key == key_b) ++rank;
      if (rm) x[i].h[e] = __ushort_as_half((unsigned short)0xFC00u);     // -inf
      any |= rm;
    }
    if (any) reinterpret_cast<uint4*>(row)[c] = x[i].u;
  }
}

// ---------------------------------------------------------------------------------------------
// Min-p filter, in place: token i keeps its logit when softmax(x / T)_i >= min_p * max_j softmax(x / T)_j, else becomes
// -inf.  Decided in logit space, exp((x_i - m) / T) >= min_p <=> x_i - m >= T * ln(min_p), so neither side needs an exp or
// a log: with m the NaN-ignoring row max (fmaxf) and thr = fp32(T) * fp32(ln min_p) (one round-to-nearest multiply; the
// host supplies ln min_p), token i stays when it is NaN, equals m, or fp32(x_i - m) >= thr.  NaN stays NaN (the walk's
// NaN flag still ends the sequence), a +inf entry stays and drops every finite one, -inf stays -inf.  Only 16-byte packs
// holding a dropped finite entry are written.  One read of the row, one block max (WIDE: plus one cluster max), no
// histogram, no atomics.  Row r belongs to sequence r / rows_per_seq; a row whose log_min_p is -inf (off) returns after
// griddepcontrol.wait without touching memory (the whole cluster reads the same value).
template <bool WIDE>
__global__ void __launch_bounds__(NT) min_p_filter_kernel(__half* __restrict__ logits, int64_t ld, int V,
                                                           const float* __restrict__ log_min_p,
                                                           const float* __restrict__ T, int rows_per_seq) {
  __shared__ float red[NW];
  pdl_wait();
  Slice sl{};
  if constexpr (WIDE) sl = slice_of(V);
  const int seq = (WIDE ? sl.row : (int)blockIdx.x) / rows_per_seq;
  const float lmp = log_min_p[seq];
  if (lmp == -INFINITY) return;
  const float thr = __fmul_rn(T[seq], lmp);
  __half* row;
  if constexpr (WIDE) {
    row = logits + sl.row * ld + sl.base;
    V = sl.V;
  } else {
    row = logits + blockIdx.x * ld;
  }
  const int nvec = V / 8;
  Pack8 x[CH];
  load_row(row, V, x);
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < CH; ++i)
#pragma unroll
    for (int e = 0; e < 8; ++e) m = fmaxf(m, h2f(x[i].h[e]));      // (padding chunks are -inf)
  m = block_max<NW>(m, red);
  if constexpr (WIDE) {
    __shared__ float xs[MAX_SLICES];
    m = cl_max(m, xs, sl);
  }
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = i * NT + threadIdx.x;
    if (c >= nvec) continue;
    bool any = false;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float v = h2f(x[i].h[e]);
      // (v > -inf is false for NaN and -inf, which stay as they are)
      const bool drop = v > -INFINITY && v != m && !(__fsub_rn(v, m) >= thr);
      if (drop) x[i].h[e] = __ushort_as_half((unsigned short)0xFC00u);     // -inf
      any |= drop;
    }
    if (any) reinterpret_cast<uint4*>(row)[c] = x[i].u;
  }
}

}  // namespace sq

using namespace sq;

#define SQ_CHECK_V(V) \
  SQ_CHECK_ARG((V) % 8 == 0 && (V) > 0 && (V) <= NT * CH * 8, "V=%d must be a multiple of 8, <= 32768", (V))
#define SQ_CHECK_V_WIDE(V)                                                                                         \
  SQ_CHECK_ARG((V) % 8 == 0 && (V) > 0 && (V) <= SLICE * MAX_SLICES, "V=%d must be a multiple of 8, <= %d", (V), \
               SLICE * MAX_SLICES)

// the host's view of a sample_level_batch `mode` argument: 0 / 1, or 0 for a greedy array (some sequence may sample)
static int seq_mode_host(int mode) { return mode; }
static int seq_mode_host(const int32_t*) { return 0; }

// V > SLICE: `rows` clusters of ceil(V / SLICE) CTAs along x (times grid_y)
template <typename... KArgs, typename... Args>
static cudaError_t launch_wide(void (*kern)(KArgs...), int rows, int grid_y, int V, cudaStream_t st, Args&&... args) {
  const unsigned n = (unsigned)((V + SLICE - 1) / SLICE);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(rows * n, grid_y);
  cfg.blockDim = dim3(NT);
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = n;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

#define SQ_CHECK_WIDE_LAUNCH(call, name)                                                   \
  do {                                                                                     \
    cudaError_t e_ = (call);                                                               \
    if (e_ != cudaSuccess) {                                                               \
      sq::set_error("%s: launch failed: %s", name, cudaGetErrorString(e_));                \
      return SQ_ERR_CUDA;                                                                  \
    }                                                                                      \
    SQ_CHECK_LAUNCH(name);                                                                 \
  } while (0)

// (a test and tooling entry point; the decode path has no softmax_T launch, so it keeps the single-CTA bound)
extern "C" int sq_softmax_T(const sq_half* logits, int64_t ld_in, sq_half* out, int64_t ld_out, int n, int V, float T,
                            void* stream) {
  SQ_CHECK_V(V);
  if (n == 0) return SQ_OK;
  softmax_T_kernel<<<n, NT, 0, (cudaStream_t)stream>>>((const __half*)logits, ld_in, (__half*)out, ld_out, V, 1.0f / T);
  SQ_CHECK_LAUNCH("sq_softmax_T");
  return SQ_OK;
}

extern "C" int sq_sample_level(const sq_half* logits, int64_t ld_logits, const sq_half* rand, int64_t ld_rand,
                               const int32_t* parent_rows, const int32_t* child_first, const int32_t* n_branch,
                               int n_parents, int k_max, int V, float T, int mode, int64_t* positions, int64_t* tokens,
                               const int32_t* state, void* stream) {
  SQ_CHECK_V_WIDE(V);
  if (n_parents == 0 || k_max == 0) return SQ_OK;
  SQ_CHECK_ARG(mode == 1 || rand != nullptr, "sq_sample_level: rand required for mode 0");
  SQ_CHECK_ARG(tokens == nullptr || (child_first && n_branch), "sq_sample_level: tokens needs child_first/n_branch");
  SQ_CHECK_ARG(k_max <= V, "sq_sample_level: k_max > V");
  if (V > SLICE) {
    SQ_CHECK_ARG(k_max <= WIDE_KMAX, "sq_sample_level: k_max=%d > %d with V > %d", k_max, WIDE_KMAX, SLICE);
    SQ_CHECK_WIDE_LAUNCH(launch_wide(sample_level_kernel<false, true>, n_parents, 1, V, (cudaStream_t)stream,
                                     (const __half*)logits, ld_logits, (const __half*)rand, ld_rand, parent_rows,
                                     child_first, n_branch, k_max, V, 1.0f / T, mode, positions, tokens, state,
                                     (const int32_t*)nullptr, (const int32_t*)nullptr, (int64_t)0, (int64_t)0),
                         "sq_sample_level");
    return SQ_OK;
  }
  sample_level_kernel<false, false><<<n_parents, NT, 0, (cudaStream_t)stream>>>(
      (const __half*)logits, ld_logits, (const __half*)rand, ld_rand, parent_rows, child_first, n_branch, k_max, V, 1.0f / T,
      mode, positions, tokens, state, nullptr, nullptr, 0, 0);
  SQ_CHECK_LAUNCH("sq_sample_level");
  return SQ_OK;
}

// sq_sample_level_batch and its per-sequence forms: `temp` is 1/T (PER_SEQ = false) or the (B,) T array; `mode` is 0 / 1
// or (MIXED) the (B,) greedy array
template <bool PER_SEQ, bool MIXED = false>
static int sample_level_batch(const char* name, const sq_half* logits, int64_t ld_logits, const int32_t* row_base,
                              const int32_t* row_step, const sq_half* rand, int64_t ld_rand, int64_t ld_rand_seq,
                              const int32_t* parent_rows, const int32_t* child_first, const int32_t* n_branch,
                              int n_parents, int k_max, int V, SeqParam<PER_SEQ> temp, ModeArg<MIXED> mode,
                              int64_t* tokens, int64_t ld_seq, const int32_t* state, int B, void* stream) {
  SQ_CHECK_V_WIDE(V);
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH, "%s: B=%d (1..%d)", name, B, SQ_MAX_BATCH);
  if (n_parents == 0 || k_max == 0) return SQ_OK;
  // (MIXED: any sequence may draw as mode 0, so rand is always required)
  SQ_CHECK_ARG(seq_mode_host(mode) == 1 || rand != nullptr, "%s: rand required for mode 0", name);
  SQ_CHECK_ARG(tokens && child_first && n_branch && parent_rows && state && row_base && row_step,
               "%s: null table or buffer", name);
  SQ_CHECK_ARG(k_max <= V, "%s: k_max > V", name);
  if (V > SLICE) {
    SQ_CHECK_ARG(k_max <= WIDE_KMAX, "%s: k_max=%d > %d with V > %d", name, k_max, WIDE_KMAX, SLICE);
    SQ_CHECK_WIDE_LAUNCH(launch_wide(sample_level_kernel<true, true, PER_SEQ, MIXED>, n_parents, B, V, (cudaStream_t)stream,
                                     (const __half*)logits, ld_logits, (const __half*)rand, ld_rand, parent_rows,
                                     child_first, n_branch, k_max, V, temp, mode, (int64_t*)nullptr, tokens, state,
                                     row_base, row_step, ld_rand_seq, ld_seq),
                         name);
    return SQ_OK;
  }
  sample_level_kernel<true, false, PER_SEQ, MIXED><<<dim3(n_parents, B), NT, 0, (cudaStream_t)stream>>>(
      (const __half*)logits, ld_logits, (const __half*)rand, ld_rand, parent_rows, child_first, n_branch, k_max, V, temp,
      mode, nullptr, tokens, state, row_base, row_step, ld_rand_seq, ld_seq);
  SQ_CHECK_LAUNCH(name);
  return SQ_OK;
}

extern "C" int sq_sample_level_batch(const sq_half* logits, int64_t ld_logits, const int32_t* row_base,
                                     const int32_t* row_step, const sq_half* rand, int64_t ld_rand, int64_t ld_rand_seq,
                                     const int32_t* parent_rows, const int32_t* child_first, const int32_t* n_branch,
                                     int n_parents, int k_max, int V, float T, int mode, int64_t* tokens, int64_t ld_seq,
                                     const int32_t* state, int B, void* stream) {
  return sample_level_batch<false>("sq_sample_level_batch", logits, ld_logits, row_base, row_step, rand, ld_rand,
                                   ld_rand_seq, parent_rows, child_first, n_branch, n_parents, k_max, V, 1.0f / T, mode,
                                   tokens, ld_seq, state, B, stream);
}

extern "C" int sq_sample_level_batch_per_seq(const sq_half* logits, int64_t ld_logits, const int32_t* row_base,
                                             const int32_t* row_step, const sq_half* rand, int64_t ld_rand,
                                             int64_t ld_rand_seq, const int32_t* parent_rows, const int32_t* child_first,
                                             const int32_t* n_branch, int n_parents, int k_max, int V, const float* T,
                                             int mode, int64_t* tokens, int64_t ld_seq, const int32_t* state, int B,
                                             void* stream) {
  SQ_CHECK_ARG(T != nullptr, "sq_sample_level_batch_per_seq: null temperature array");
  return sample_level_batch<true>("sq_sample_level_batch_per_seq", logits, ld_logits, row_base, row_step, rand, ld_rand,
                                  ld_rand_seq, parent_rows, child_first, n_branch, n_parents, k_max, V, T, mode, tokens,
                                  ld_seq, state, B, stream);
}

extern "C" int sq_sample_level_batch_mixed(const sq_half* logits, int64_t ld_logits, const int32_t* row_base,
                                           const int32_t* row_step, const sq_half* rand, int64_t ld_rand,
                                           int64_t ld_rand_seq, const int32_t* parent_rows, const int32_t* child_first,
                                           const int32_t* n_branch, int n_parents, int k_max, int V, const float* T,
                                           const int32_t* greedy, int64_t* tokens, int64_t ld_seq, const int32_t* state,
                                           int B, void* stream) {
  SQ_CHECK_ARG(T != nullptr && greedy != nullptr, "sq_sample_level_batch_mixed: null temperature or greedy array");
  return sample_level_batch<true, true>("sq_sample_level_batch_mixed", logits, ld_logits, row_base, row_step, rand,
                                        ld_rand, ld_rand_seq, parent_rows, child_first, n_branch, n_parents, k_max, V, T,
                                        greedy, tokens, ld_seq, state, B, stream);
}

// Sampling with replacement (the SpecInfer policy) has no large-vocabulary instance: V <= 32768 only.
extern "C" int sq_sample_replace(const sq_half* logits, int64_t ld_logits, const int64_t* words,
                                 const int32_t* parent_rows, const int32_t* child_first, const int32_t* n_branch,
                                 int n_parents, int k_max, int V, float T, int64_t* positions, int64_t* tokens,
                                 const int32_t* state, void* stream) {
  SQ_CHECK_ARG(V % 8 == 0 && V > 0 && V <= SLICE,
               "sq_sample_replace: V=%d must be a multiple of 8, <= 32768 (sampling with replacement has no "
               "large-vocabulary kernel)", V);
  if (n_parents == 0 || k_max == 0) return SQ_OK;
  SQ_CHECK_ARG(words != nullptr, "sq_sample_replace: words required");
  SQ_CHECK_ARG(tokens == nullptr || (child_first && n_branch), "sq_sample_replace: tokens needs child_first/n_branch");
  SQ_CHECK_ARG(positions != nullptr || tokens != nullptr, "sq_sample_replace: no output");
  sample_replace_kernel<<<n_parents, NT, 0, (cudaStream_t)stream>>>((const __half*)logits, ld_logits, words, parent_rows,
                                                                   child_first, n_branch, k_max, V, 1.0f / T, positions,
                                                                   tokens, state);
  SQ_CHECK_LAUNCH("sq_sample_replace");
  return SQ_OK;
}

extern "C" int sq_residual(const sq_half* p, const sq_half* q, sq_half* out, int V, void* stream) {
  SQ_CHECK_V_WIDE(V);
  if (V > SLICE) {
    SQ_CHECK_WIDE_LAUNCH(launch_wide(residual_kernel<true>, 1, 1, V, (cudaStream_t)stream, (const __half*)p,
                                     (const __half*)q, (__half*)out, V), "sq_residual");
    return SQ_OK;
  }
  residual_kernel<false><<<1, NT, 0, (cudaStream_t)stream>>>((const __half*)p, (const __half*)q, (__half*)out, V);
  SQ_CHECK_LAUNCH("sq_residual");
  return SQ_OK;
}

extern "C" int sq_argmax_rows(const sq_half* logits, int64_t ld, int n, int V, int64_t* out, void* stream) {
  SQ_CHECK_V_WIDE(V);
  if (n == 0) return SQ_OK;
  if (V > SLICE) {
    SQ_CHECK_WIDE_LAUNCH(launch_wide(argmax_rows_kernel<true>, n, 1, V, (cudaStream_t)stream, (const __half*)logits, ld, V,
                                     out), "sq_argmax_rows");
    return SQ_OK;
  }
  argmax_rows_kernel<false><<<n, NT, 0, (cudaStream_t)stream>>>((const __half*)logits, ld, V, out);
  SQ_CHECK_LAUNCH("sq_argmax_rows");
  return SQ_OK;
}

extern "C" int sq_top_p_filter(sq_half* logits, int64_t ld, int n, int V, float top_p, float T, void* stream) {
  SQ_CHECK_V_WIDE(V);
  if (n == 0 || top_p >= 1.0f) return SQ_OK;                       // utils.py:68: only when top_p < 1
  const float tp = __half2float(__float2half_rn(top_p));           // torch compares in the tensor's dtype (fp16)
  if (V > SLICE) {
    SQ_CHECK_WIDE_LAUNCH(launch_wide(top_p_filter_kernel<true>, n, 1, V, (cudaStream_t)stream, (__half*)logits, ld, V,
                                     1.0f / T, tp, 0), "sq_top_p_filter");
    return SQ_OK;
  }
  top_p_filter_kernel<false><<<n, NT, 0, (cudaStream_t)stream>>>((__half*)logits, ld, V, 1.0f / T, tp, 0);
  SQ_CHECK_LAUNCH("sq_top_p_filter");
  return SQ_OK;
}

extern "C" int sq_top_p_filter_per_seq(sq_half* logits, int64_t ld, int n, int V, const float* top_p, const float* T,
                                       int rows_per_seq, void* stream) {
  SQ_CHECK_V_WIDE(V);
  SQ_CHECK_ARG(top_p != nullptr && T != nullptr, "sq_top_p_filter_per_seq: null top_p or temperature array");
  SQ_CHECK_ARG(rows_per_seq >= 1 && n >= 0 && n % rows_per_seq == 0,
               "sq_top_p_filter_per_seq: rows_per_seq=%d does not divide n=%d", rows_per_seq, n);
  if (n == 0) return SQ_OK;
  if (V > SLICE) {
    SQ_CHECK_WIDE_LAUNCH(launch_wide(top_p_filter_kernel<true, true>, n, 1, V, (cudaStream_t)stream, (__half*)logits, ld,
                                     V, T, top_p, rows_per_seq), "sq_top_p_filter_per_seq");
    return SQ_OK;
  }
  top_p_filter_kernel<false, true><<<n, NT, 0, (cudaStream_t)stream>>>((__half*)logits, ld, V, T, top_p, rows_per_seq);
  SQ_CHECK_LAUNCH("sq_top_p_filter_per_seq");
  return SQ_OK;
}

extern "C" int sq_top_k_filter(sq_half* logits, int64_t ld, int n, int V, int k, void* stream) {
  SQ_CHECK_V_WIDE(V);
  SQ_CHECK_ARG(k >= 0, "sq_top_k_filter: k=%d must be >= 0 (0 = off)", k);
  if (n == 0 || k == 0 || k >= V) return SQ_OK;                    // off, or every token is among the k best
  if (V > SLICE) {
    SQ_CHECK_WIDE_LAUNCH(launch_wide(top_k_filter_kernel<true>, n, 1, V, (cudaStream_t)stream, (__half*)logits, ld, V, k,
                                     0), "sq_top_k_filter");
    return SQ_OK;
  }
  top_k_filter_kernel<false><<<n, NT, 0, (cudaStream_t)stream>>>((__half*)logits, ld, V, k, 0);
  SQ_CHECK_LAUNCH("sq_top_k_filter");
  return SQ_OK;
}

extern "C" int sq_top_k_filter_per_seq(sq_half* logits, int64_t ld, int n, int V, const int32_t* top_k, int rows_per_seq,
                                       void* stream) {
  SQ_CHECK_V_WIDE(V);
  SQ_CHECK_ARG(top_k != nullptr, "sq_top_k_filter_per_seq: null top_k array");
  SQ_CHECK_ARG(rows_per_seq >= 1 && n >= 0 && n % rows_per_seq == 0,
               "sq_top_k_filter_per_seq: rows_per_seq=%d does not divide n=%d", rows_per_seq, n);
  if (n == 0) return SQ_OK;
  if (V > SLICE) {
    SQ_CHECK_WIDE_LAUNCH(launch_wide(top_k_filter_kernel<true, true>, n, 1, V, (cudaStream_t)stream, (__half*)logits, ld,
                                     V, top_k, rows_per_seq), "sq_top_k_filter_per_seq");
    return SQ_OK;
  }
  top_k_filter_kernel<false, true><<<n, NT, 0, (cudaStream_t)stream>>>((__half*)logits, ld, V, top_k, rows_per_seq);
  SQ_CHECK_LAUNCH("sq_top_k_filter_per_seq");
  return SQ_OK;
}

extern "C" int sq_min_p_filter_per_seq(sq_half* logits, int64_t ld, int n, int V, const float* log_min_p, const float* T,
                                       int rows_per_seq, void* stream) {
  SQ_CHECK_V_WIDE(V);
  SQ_CHECK_ARG(log_min_p != nullptr && T != nullptr, "sq_min_p_filter_per_seq: null log_min_p or temperature array");
  SQ_CHECK_ARG(rows_per_seq >= 1 && n >= 0 && n % rows_per_seq == 0,
               "sq_min_p_filter_per_seq: rows_per_seq=%d does not divide n=%d", rows_per_seq, n);
  if (n == 0) return SQ_OK;
  if (V > SLICE) {
    SQ_CHECK_WIDE_LAUNCH(launch_wide(min_p_filter_kernel<true>, n, 1, V, (cudaStream_t)stream, (__half*)logits, ld, V,
                                     log_min_p, T, rows_per_seq), "sq_min_p_filter_per_seq");
    return SQ_OK;
  }
  min_p_filter_kernel<false><<<n, NT, 0, (cudaStream_t)stream>>>((__half*)logits, ld, V, log_min_p, T, rows_per_seq);
  SQ_CHECK_LAUNCH("sq_min_p_filter_per_seq");
  return SQ_OK;
}
