// Per-sequence counter-based random numbers for BatchTree (include/sequoia_b200.h, "per-sequence counter-based random
// numbers"): Philox4x32-10 keyed by the sequence's 64-bit seed, so every draw is a pure function of (seed, purpose, step,
// element) and a sequence's numbers do not depend on its slot, its neighbours or the order of admissions.
// Each thread makes two Philox blocks = 8 fp16 values and stores them as one 16-byte vector.
#include "sq_common.cuh"

namespace sq {

constexpr int RNG_THREADS = 256;
constexpr int NOISE_CLUSTER = 8;      // CTAs per sequence of the noise kernel: one cluster writes one row

// Random123 philox4x32-10: counter (x, y, z, w), key (k0, k1)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}

// 8 consecutive elements 8t .. 8t+7 of stream (seed, purpose, step): counters i = 2t and 2t + 1, element e = word e % 4
// of counter e / 4
__device__ __forceinline__ void philox8(uint64_t seed, uint32_t purpose, uint32_t step, int64_t t, uint32_t w[8]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint64_t i = 2 * (uint64_t)t + h;
    const uint4 o = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), purpose, step), (uint32_t)seed,
                                  (uint32_t)(seed >> 32));
    w[4 * h + 0] = o.x;
    w[4 * h + 1] = o.y;
    w[4 * h + 2] = o.z;
    w[4 * h + 3] = o.w;
  }
}

// u = k / 2048, k = the word's top 11 bits: exact in fp16, the grid torch's CPU fp16 uniform_ draws from
__device__ __forceinline__ __half uniform_h(uint32_t w) { return __float2half_rn((float)(w >> 21) * 0x1p-11f); }

// Exp(1): u = fp32((k + 0.5) * 2^-24), k = the word's top 24 bits (one rounding, to nearest even; exact below k = 2^23),
// noise = fp16(max(-logf(u), 2^-24)), never zero
__device__ __forceinline__ __half exponential_h(uint32_t w) {
  const float u = ((float)(w >> 8) + 0.5f) * 0x1p-24f;
  return __float2half_rn(fmaxf(-logf(u), 0x1p-24f));
}

struct SlotList {
  int slot[SQ_MAX_BATCH];
};

// grid (chunks, n_seqs): row slot[blockIdx.y] of `out`, `count` uniforms of `purpose` at step 0.  vec: the rows are
// 16-byte aligned, so every full group of 8 is one vector store.
__global__ void __launch_bounds__(RNG_THREADS) rng_uniform_kernel(__half* __restrict__ out, int64_t ld_seq, int64_t count,
                                                                 const uint64_t* __restrict__ seeds,
                                                                 const __grid_constant__ SlotList sl, uint32_t purpose,
                                                                 int vec) {
  pdl_wait();
  pdl_trigger();
  const int b = sl.slot[blockIdx.y];
  const uint64_t seed = seeds[b];
  __half* row = out + (int64_t)b * ld_seq;
  const int64_t groups = (count + 7) / 8;
  for (int64_t t = (int64_t)blockIdx.x * RNG_THREADS + threadIdx.x; t < groups; t += (int64_t)gridDim.x * RNG_THREADS) {
    uint32_t w[8];
    philox8(seed, purpose, 0, t, w);
    Pack8 p;
#pragma unroll
    for (int j = 0; j < 8; ++j) p.h[j] = uniform_h(w[j]);
    const int64_t e0 = 8 * t;
    if (vec && e0 + 8 <= count) {
      *reinterpret_cast<uint4*>(row + e0) = p.u;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (e0 + j < count) row[e0 + j] = p.h[j];
    }
  }
}

// grid (NOISE_CLUSTER, B), one cluster per sequence: row b of the noise at step steps[b], then steps[b] += 1.  The cluster
// barrier orders every CTA's read of steps[b] before the one write.  A frozen sequence's cluster leaves as a whole.
__global__ void __cluster_dims__(NOISE_CLUSTER, 1, 1) __launch_bounds__(RNG_THREADS)
    rng_exponential_kernel(__half* __restrict__ noise, int64_t ld_noise, int V, const uint64_t* __restrict__ seeds,
                           int64_t* __restrict__ steps, const int32_t* __restrict__ state) {
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.y;
  if (state[b * ST_WORDS + ST_FROZEN]) return;
  const uint64_t seed = seeds[b];
  const int64_t step = steps[b];
  uint4* row = reinterpret_cast<uint4*>(noise + (int64_t)b * ld_noise);
  for (int t = blockIdx.x * RNG_THREADS + threadIdx.x; t < V / 8; t += NOISE_CLUSTER * RNG_THREADS) {
    uint32_t w[8];
    philox8(seed, 2, (uint32_t)step, t, w);
    Pack8 p;
#pragma unroll
    for (int j = 0; j < 8; ++j) p.h[j] = exponential_h(w[j]);
    row[t] = p.u;
  }
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  if (blockIdx.x == 0 && threadIdx.x == 0) steps[b] = step + 1;
}

}  // namespace sq

using namespace sq;

extern "C" int sq_rng_uniform_seqs(sq_half* out, int64_t ld_seq, int64_t count, const uint64_t* seeds,
                                   const int32_t* host_seqs, int n_seqs, int B, int purpose, void* stream) {
  SQ_CHECK_ARG(out != nullptr && seeds != nullptr && host_seqs != nullptr,
               "sq_rng_uniform_seqs: null output, seeds or slot list");
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH, "sq_rng_uniform_seqs: B=%d (1..%d)", B, SQ_MAX_BATCH);
  SQ_CHECK_ARG(purpose == 0 || purpose == 1, "sq_rng_uniform_seqs: purpose %d is not 0 (r) or 1 (rand)", purpose);
  SQ_CHECK_ARG(count >= 1 && ld_seq >= count, "sq_rng_uniform_seqs: count=%lld, ld_seq=%lld", (long long)count,
               (long long)ld_seq);
  SQ_CHECK_ARG(n_seqs >= 1 && n_seqs <= B, "sq_rng_uniform_seqs: %d slots for %d sequences", n_seqs, B);
  SlotList sl{};
  unsigned seen = 0;
  for (int j = 0; j < n_seqs; ++j) {
    const int b = host_seqs[j];
    SQ_CHECK_ARG(b >= 0 && b < B, "sq_rng_uniform_seqs: slot %d of %d", b, B);
    SQ_CHECK_ARG(!(seen >> b & 1u), "sq_rng_uniform_seqs: slot %d listed twice", b);
    seen |= 1u << b;
    sl.slot[j] = b;
  }
  const int vec = (ld_seq % 8 == 0) && ((uintptr_t)out % 16 == 0);
  const int64_t groups = (count + 7) / 8;
  const int64_t want = (groups + RNG_THREADS - 1) / RNG_THREADS;
  const int chunks = (int)(want < 1024 ? want : 1024);
  launch_k(rng_uniform_kernel, dim3(chunks, n_seqs), dim3(RNG_THREADS), 0, (cudaStream_t)stream, (__half*)out, ld_seq,
           count, seeds, sl, (uint32_t)purpose, vec);
  SQ_CHECK_LAUNCH("sq_rng_uniform_seqs");
  return SQ_OK;
}

extern "C" int sq_rng_exponential_batch(sq_half* noise, int64_t ld_noise, int V, const uint64_t* seeds, int64_t* steps,
                                        const int32_t* state, int B, void* stream) {
  SQ_CHECK_ARG(noise != nullptr && seeds != nullptr && steps != nullptr && state != nullptr,
               "sq_rng_exponential_batch: null noise, seeds, steps or state");
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH, "sq_rng_exponential_batch: B=%d (1..%d)", B, SQ_MAX_BATCH);
  SQ_CHECK_ARG(V >= 8 && V % 8 == 0 && ld_noise >= V && ld_noise % 8 == 0 && (uintptr_t)noise % 16 == 0,
               "sq_rng_exponential_batch: V=%d and ld_noise=%lld must be multiples of 8 (ld_noise >= V), rows 16-byte "
               "aligned", V, (long long)ld_noise);
  launch_k(rng_exponential_kernel, dim3(NOISE_CLUSTER, B), dim3(RNG_THREADS), 0, (cudaStream_t)stream, (__half*)noise,
           ld_noise, V, seeds, steps, state);
  SQ_CHECK_LAUNCH("sq_rng_exponential_batch");
  return SQ_OK;
}
