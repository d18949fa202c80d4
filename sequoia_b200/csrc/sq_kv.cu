// Accepted-path KV compaction (Engine/Llama_KV.py:50-68).  One CTA per (layer, kv-head, K|V) plane stages every
// source row on chip (registers, 16 B per thread per row-chunk) before writing, which gives the reference's
// gather-to-temp-then-copy semantics for arbitrary (also overlapping) index lists with no extra HBM traffic:
// algorithmic bytes = 2 (K,V) * 2 (read+write) * L * Hkv * n * D * 2.
#include "sq_common.cuh"

namespace sq {

// threads: ROWS_PER_PASS rows x (D/8) 16-byte lanes.  Dynamic shared memory holds all n rows when n > ROWS_PER_PASS.
// BATCH: the cache is (L, B, Hkv, M, D); plane x belongs to sequence (x / Hkv) % B, which reads its own state row and
// index row (idx + b * ld_idx) and is skipped when frozen.
template <bool BATCH>
__global__ void kv_gather_kernel(__half* __restrict__ k_cache, __half* __restrict__ v_cache, int M, int D,
                                 const int32_t* __restrict__ idx, int n_host, int offset_host,
                                 const int32_t* __restrict__ state, int max_n, int Hkv, int B, int ld_idx) {
  extern __shared__ uint4 stage[];
  __half* plane = (blockIdx.y == 0 ? k_cache : v_cache) + (int64_t)blockIdx.x * M * D;
  if (BATCH) {
    const int b = (blockIdx.x / Hkv) % B;
    state += b * ST_WORDS;
    idx += b * ld_idx;
    if (state[ST_FROZEN]) return;
  }
  int n = n_host, offset = offset_host;
  if (state) { n = state[ST_N_NEW]; offset = state[ST_P_OLD]; }
  if (n > max_n) n = max_n;
  const int lanes = D / 8;
  const int total = n * lanes;
  // phase 1: gather every source row chunk into shared memory
  for (int t = threadIdx.x; t < total; t += blockDim.x) {
    const int j = t / lanes, c = t % lanes;
    stage[t] = reinterpret_cast<const uint4*>(plane + (int64_t)idx[j] * D)[c];
  }
  __syncthreads();
  // phase 2: write to the compacted destination rows
  for (int t = threadIdx.x; t < total; t += blockDim.x) {
    const int j = t / lanes, c = t % lanes;
    reinterpret_cast<uint4*>(plane + (int64_t)(offset + j) * D)[c] = stage[t];
  }
}

// zero rows >= offset + n of every plane (Llama_KV.py:65-66).  grid (planes, 2, chunks)
__global__ void kv_zero_tail_kernel(__half* __restrict__ k_cache, __half* __restrict__ v_cache, int M, int D,
                                    int n_host, int offset_host, const int32_t* __restrict__ state) {
  __half* plane = (blockIdx.y == 0 ? k_cache : v_cache) + (int64_t)blockIdx.x * M * D;
  int n = n_host, offset = offset_host;
  if (state) { n = state[ST_N_NEW]; offset = state[ST_P_OLD]; }
  const int64_t first = (int64_t)(offset + n) * D / 8;
  const int64_t last = (int64_t)M * D / 8;
  uint4* p = reinterpret_cast<uint4*>(plane);
  const uint4 z = make_uint4(0, 0, 0, 0);
  for (int64_t i = first + blockIdx.z * (int64_t)blockDim.x + threadIdx.x; i < last;
       i += (int64_t)gridDim.z * blockDim.x)
    p[i] = z;
}

// Index lists too long to stage on chip (reference API: gather_kv with a whole accept list of several hundred rows):
// gather into a global scratch (planes, n, D), then copy back -- literally the reference's temp-then-copy.
// grid (planes, 2, chunks); dir 0: cache[idx[j]] -> scratch[j], dir 1: scratch[j] -> cache[offset + j]
__global__ void kv_gather_scratch_kernel(__half* __restrict__ k_cache, __half* __restrict__ v_cache, int M, int D,
                                         const int32_t* __restrict__ idx, int n, int offset, uint4* __restrict__ scratch,
                                         int dir) {
  __half* plane = (blockIdx.y == 0 ? k_cache : v_cache) + (int64_t)blockIdx.x * M * D;
  const int lanes = D / 8;
  uint4* sp = scratch + ((int64_t)blockIdx.x * 2 + blockIdx.y) * n * lanes;
  for (int t = blockIdx.z * blockDim.x + threadIdx.x; t < n * lanes; t += gridDim.z * blockDim.x) {
    const int j = t / lanes, c = t % lanes;
    if (dir == 0) sp[t] = reinterpret_cast<const uint4*>(plane + (int64_t)idx[j] * D)[c];
    else reinterpret_cast<uint4*>(plane + (int64_t)(offset + j) * D)[c] = sp[t];
  }
}

// Prefix copy between two sequences of a (L, B, Hkv, M, D) cache: rows [0, n) of each (layer, kv-head) plane of sequence
// src to the same rows of sequence dst.  Those rows are one contiguous run of n*D/8 16-byte words per plane, so a plane
// is a flat copy.  grid (L*Hkv, K|V, chunks); a CTA moves COPY_ITEMS words per thread per pass, all loads before the
// stores, and strides over its plane by gridDim.z chunks.
constexpr int COPY_ITEMS = 4;

__global__ void kv_copy_prefix_kernel(__half* __restrict__ k_cache, __half* __restrict__ v_cache, int B, int Hkv, int M,
                                      int D, int src, int dst, int n) {
  const int l = blockIdx.x / Hkv, h = blockIdx.x % Hkv;
  __half* cache = blockIdx.y == 0 ? k_cache : v_cache;
  const int64_t plane = (int64_t)M * D;
  const uint4* s = reinterpret_cast<const uint4*>(cache + ((int64_t)(l * B + src) * Hkv + h) * plane);
  uint4* d = reinterpret_cast<uint4*>(cache + ((int64_t)(l * B + dst) * Hkv + h) * plane);
  const int64_t words = (int64_t)n * D / 8;
  const int64_t chunk = (int64_t)blockDim.x * COPY_ITEMS;
  for (int64_t base = blockIdx.z * chunk + threadIdx.x; base < words; base += gridDim.z * chunk) {
    uint4 v[COPY_ITEMS];
#pragma unroll
    for (int i = 0; i < COPY_ITEMS; ++i) {
      const int64_t j = base + (int64_t)i * blockDim.x;
      if (j < words) v[i] = s[j];
    }
#pragma unroll
    for (int i = 0; i < COPY_ITEMS; ++i) {
      const int64_t j = base + (int64_t)i * blockDim.x;
      if (j < words) d[j] = v[i];
    }
  }
}

}  // namespace sq

using namespace sq;

extern "C" int64_t sq_kv_gather_scratch_bytes(int L, int Hkv, int D, int n) { return (int64_t)L * Hkv * 2 * n * D * 2; }

extern "C" int sq_kv_gather_big(sq_half* k_cache, sq_half* v_cache, int L, int Hkv, int M, int D, const int32_t* idx,
                                int n, int offset, void* scratch, int64_t scratch_bytes, int zero_tail, void* stream) {
  SQ_CHECK_ARG(D % 8 == 0 && n >= 0, "sq_kv_gather_big: bad shape");
  SQ_CHECK_ARG(n == 0 || (scratch && scratch_bytes >= sq_kv_gather_scratch_bytes(L, Hkv, D, n)),
               "sq_kv_gather_big: scratch too small");
  SQ_CHECK_ARG(offset >= 0 && offset + n <= M, "sq_kv_gather_big: offset %d + n %d > M %d", offset, n, M);
  cudaStream_t st = (cudaStream_t)stream;
  const int planes = L * Hkv;
  if (n > 0) {
    const int chunks = (n * (D / 8) + 1023) / 1024;
    for (int dir = 0; dir < 2; ++dir) {
      kv_gather_scratch_kernel<<<dim3(planes, 2, chunks), 256, 0, st>>>((__half*)k_cache, (__half*)v_cache, M, D, idx, n,
                                                                       offset, (uint4*)scratch, dir);
      SQ_CHECK_LAUNCH("sq_kv_gather_big");
    }
  }
  if (zero_tail) {
    kv_zero_tail_kernel<<<dim3(planes, 2, 4), 256, 0, st>>>((__half*)k_cache, (__half*)v_cache, M, D, n, offset, nullptr);
    SQ_CHECK_LAUNCH("sq_kv_zero_tail");
  }
  return SQ_OK;
}

template <bool BATCH>
static int launch_gather(sq_half* k_cache, sq_half* v_cache, int planes, int M, int D, const int32_t* idx, int n, int offset,
                         const int32_t* state, int max_n, int Hkv, int B, int ld_idx, cudaStream_t st) {
  const size_t smem = (size_t)max_n * D * 2;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kv_gather_kernel<BATCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("sq_kv_gather: smem attr: %s", cudaGetErrorString(e)); return SQ_ERR_CUDA; }
  }
  int threads = max_n * (D / 8);
  threads = threads < 64 ? 64 : (threads > 512 ? 512 : ((threads + 31) / 32) * 32);
  kv_gather_kernel<BATCH><<<dim3(planes, 2), threads, smem, st>>>((__half*)k_cache, (__half*)v_cache, M, D, idx, n, offset,
                                                                  state, max_n, Hkv, B, ld_idx);
  return SQ_OK;
}

extern "C" int sq_kv_gather_batch(sq_half* k_cache, sq_half* v_cache, int L, int B, int Hkv, int M, int D,
                                  const int32_t* accept_idx, int ld_idx, const int32_t* state, int max_n, void* stream) {
  SQ_CHECK_ARG(D % 8 == 0, "sq_kv_gather_batch: D %% 8 != 0");
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH && state != nullptr && accept_idx != nullptr,
               "sq_kv_gather_batch: B=%d (1..%d) needs a state array and an index array", B, SQ_MAX_BATCH);
  SQ_CHECK_ARG(max_n >= 0 && max_n <= ld_idx && (int64_t)max_n * D * 2 <= 200 * 1024,
               "sq_kv_gather_batch: max_n=%d rows do not fit on chip or in an index row of %d", max_n, ld_idx);
  if (max_n == 0) return SQ_OK;
  const int rc = launch_gather<true>(k_cache, v_cache, L * B * Hkv, M, D, accept_idx, 0, 0, state, max_n, Hkv, B, ld_idx,
                                     (cudaStream_t)stream);
  if (rc) return rc;
  SQ_CHECK_LAUNCH("sq_kv_gather_batch");
  return SQ_OK;
}

extern "C" int sq_kv_copy_prefix(sq_half* k_cache, sq_half* v_cache, int L, int B, int Hkv, int M, int D, int src,
                                 int dst, int n, void* stream) {
  SQ_CHECK_ARG(k_cache != nullptr && v_cache != nullptr, "sq_kv_copy_prefix: null cache");
  SQ_CHECK_ARG(((uintptr_t)k_cache | (uintptr_t)v_cache) % 16 == 0, "sq_kv_copy_prefix: caches not 16-byte aligned");
  SQ_CHECK_ARG(L >= 1 && Hkv >= 1 && D >= 8 && D % 8 == 0, "sq_kv_copy_prefix: bad shape L=%d Hkv=%d D=%d (D %% 8 == 0)",
               L, Hkv, D);
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH, "sq_kv_copy_prefix: B=%d outside 1..%d", B, SQ_MAX_BATCH);
  SQ_CHECK_ARG(src >= 0 && src < B && dst >= 0 && dst < B && src != dst,
               "sq_kv_copy_prefix: src=%d / dst=%d must be distinct sequences in [0, %d)", src, dst, B);
  SQ_CHECK_ARG(n >= 1 && n <= M, "sq_kv_copy_prefix: n=%d rows outside 1..M=%d", n, M);
  // one 16-byte word per thread and pass: a short copy gets warp-sized CTAs, one per plane; a long one 256 threads and
  // as many chunks of 256 * COPY_ITEMS words as its planes hold
  const int64_t words = (int64_t)n * D / 8;
  const int threads = (int)(words >= 256 ? 256 : (words + 31) / 32 * 32);
  const int64_t chunks = (words + (int64_t)threads * COPY_ITEMS - 1) / ((int64_t)threads * COPY_ITEMS);
  kv_copy_prefix_kernel<<<dim3(L * Hkv, 2, (unsigned)(chunks < 65535 ? chunks : 65535)), threads, 0,
                          (cudaStream_t)stream>>>((__half*)k_cache, (__half*)v_cache, B, Hkv, M, D, src, dst, n);
  SQ_CHECK_LAUNCH("sq_kv_copy_prefix");
  return SQ_OK;
}

extern "C" int sq_kv_gather(sq_half* k_cache, sq_half* v_cache, int L, int Hkv, int M, int D, const int32_t* idx,
                            int n, int offset, const int32_t* state, int max_n, int zero_tail, void* stream) {
  SQ_CHECK_ARG(D % 8 == 0, "sq_kv_gather: D %% 8 != 0");
  if (!state) max_n = n;
  SQ_CHECK_ARG(max_n >= 0 && (int64_t)max_n * D * 2 <= 200 * 1024, "sq_kv_gather: max_n=%d rows do not fit on chip",
               max_n);
  cudaStream_t st = (cudaStream_t)stream;
  const int planes = L * Hkv;
  if (max_n > 0) {
    const int rc = launch_gather<false>(k_cache, v_cache, planes, M, D, idx, n, offset, state, max_n, Hkv, 1, 0, st);
    if (rc) return rc;
    SQ_CHECK_LAUNCH("sq_kv_gather");
  }
  if (zero_tail) {
    kv_zero_tail_kernel<<<dim3(planes, 2, 4), 256, 0, st>>>((__half*)k_cache, (__half*)v_cache, M, D, n, offset, state);
    SQ_CHECK_LAUNCH("sq_kv_zero_tail");
  }
  return SQ_OK;
}
