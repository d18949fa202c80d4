// Shared helpers for the sequoia_b200 kernels (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/sequoia_b200.h"

namespace sq {

void set_error(const char* fmt, ...);
void count_launch(int n);

#define SQ_CHECK_ARG(cond, ...)                     \
  do {                                              \
    if (!(cond)) {                                  \
      sq::set_error(__VA_ARGS__);                   \
      return SQ_ERR_INVALID_ARG;                    \
    }                                               \
  } while (0)

#define SQ_CHECK_LAUNCH(name)                                                   \
  do {                                                                          \
    cudaError_t e__ = cudaGetLastError();                                       \
    if (e__ != cudaSuccess) {                                                   \
      sq::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));    \
      return SQ_ERR_CUDA;                                                       \
    }                                                                           \
    sq::count_launch(1);                                                        \
  } while (0)

// Programmatic dependent launch (SQ_PDL=1): kernel N+1 is scheduled while kernel N drains; every kernel launched this
// way executes pdl_wait() FIRST (before any global access and before any early return), so completion stays transitive
// along the stream (N+1 cannot finish before N has finished and flushed), then pdl_trigger() to let N+2 be scheduled.
bool pdl_enabled();
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// Device-side decode state (int32 words), owned by the Tree object, read by every kernel
// that needs the dynamic prefix length so that whole iterations are CUDA-graph static.
enum StateWord : int {
  ST_P = 0,          // ground_truth_len: committed tokens incl. the root (bonus) token
  ST_ACCEPT_LEN = 1, // a = len(accept_list) of the last verify
  ST_TERMINAL = 2,   // 1 if the last verify hit EOS/pad or a NaN residual
  ST_N_NEW = 3,      // number of tree nodes accepted by the last verify (a - P_old)
  ST_P_OLD = 4,      // ground_truth_len the last verify started from
  ST_BONUS = 5,      // bonus token (-1 when terminal)
  ST_NAN = 6,        // residual had a NaN
  ST_SKIPPED = 7,    // prepare_for_next_iter was skipped (a + 1 > max_target_seq, or the tree would overrun the buffers)
  ST_M = 8,          // length of the tokens / position_ids buffers (max_length), written by the host once per prompt
  ST_FROZEN = 9,     // batched entry points only: nonzero = finished sequence, its tokens / state / KV rows are not written
  ST_FINISH = 10,    // *_batch_stop walks only: 1 = a stop id ended the sequence, 2 = its length limit, 0 = neither
  ST_END = 11,       // *_batch_stop walks only: the sequence's final length when ST_FINISH != 0, else 0
  ST_GUIDED = 12,    // batched entry points only, host-written: nonzero = the sequence follows a token guide
  ST_GUIDE_STATE = 13, // guided sequences: the guide state after the committed tokens (-1 = a token left the guide)
  ST_GUIDE_POS = 14,   // guided sequences: the tokens before this position have been consumed by the guide
  ST_WORDS = 16
};

// Batched entry points: sequence b is the grid's batch index.  BATCH = false compiles the single-sequence kernel unchanged.
template <bool BATCH>
__device__ __forceinline__ int seq_index(unsigned grid_coord) { return BATCH ? (int)grid_coord : 0; }

// Per-sequence sampling parameters (PER_SEQ = true): the kernel argument is a (B,) fp32 device array read at the
// sequence's index; PER_SEQ = false keeps the scalar argument, so those instances compile as before.
template <bool PER_SEQ>
using SeqParam = typename std::conditional<PER_SEQ, const float*, float>::type;
// temperature argument -> 1/T of sequence b: the scalar form already carries the host's fp32 1/T; the per-sequence form
// divides on the device, which rounds the same (IEEE division, no fast-math)
__device__ __forceinline__ float inv_temp(float inv_T, int) { return inv_T; }
__device__ __forceinline__ float inv_temp(const float* T, int b) { return 1.0f / T[b]; }

// Ragged launches (RAGGED = true): a by-value kernel argument holding the part list (sq_ragged_part, in list order) and
// its prefix sums.  row0[j] = sum of n over parts < j (row0[n_parts] = all rows); tile0[j] the same over q tiles of
// rows_per_tile rows (attention).  RAGGED = false instances take a plain int in its place, so they compile as before.
struct RaggedParts {
  int n_parts;
  int seq[SQ_MAX_BATCH], n[SQ_MAX_BATCH], n0[SQ_MAX_BATCH], kv_end[SQ_MAX_BATCH];
  int row0[SQ_MAX_BATCH + 1], tile0[SQ_MAX_BATCH + 1];
};
template <bool RAGGED>
using RaggedArg = typename std::conditional<RAGGED, RaggedParts, int>::type;

// Validates a host part list against B sequences and n_max activation rows, and fills `out` (prefix sums over tiles of
// rows_per_tile rows).  SQ_ERR_INVALID_ARG with a message naming `who` on any bad part.
int make_ragged(const sq_ragged_part* parts, int n_parts, int B, int n_max, int rows_per_tile, const char* who,
                RaggedParts* out);

// the part list of a RAGGED instance; nullptr for the placeholder (never dereferenced: RAGGED = false)
__device__ __forceinline__ const RaggedParts* ragged_ptr(const RaggedParts& rp) { return &rp; }
__device__ __forceinline__ const RaggedParts* ragged_ptr(int) { return nullptr; }

// the part whose [prefix[j], prefix[j+1]) holds x (at most SQ_MAX_BATCH steps)
__device__ __forceinline__ int ragged_part(const int* prefix, int n_parts, int x) {
  int j = 0;
  while (j + 1 < n_parts && x >= prefix[j + 1]) ++j;
  return j;
}

__device__ __forceinline__ int row_base(const int32_t* P_ptr, int n0) {
  return (P_ptr ? (P_ptr[ST_P] - 1) : 0) + n0;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide reductions for blockDim.x = 32 * NW threads; `red` is NW floats of shared memory.
// The result is identical in every thread (fixed combination order => deterministic).
template <int NW>
__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float r = (l < NW) ? red[l] : -INFINITY;
  return warp_max(r);
}
template <int NW>
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float r = (l < NW) ? red[l] : 0.f;
  return warp_sum(r);
}

// fp16 helpers that reproduce torch's "compute in fp32, round to fp16" element-wise semantics.
__device__ __forceinline__ float h2f(__half h) { return __half2float(h); }
__device__ __forceinline__ __half f2h(float f) { return __float2half_rn(f); }
__device__ __forceinline__ float rnd16(float f) { return __half2float(__float2half_rn(f)); }

// fp16 bits -> uint16 whose unsigned order equals the float order (-inf lowest, +inf highest)
__device__ __forceinline__ uint32_t ord16(__half h) {
  const uint32_t b = __half_as_ushort(h);
  return (b & 0x8000u) ? (~b & 0xFFFFu) : (b | 0x8000u);
}

// ord16 with the order torch.sort gives fp16 values: -0 equal to +0, NaN above +inf (the top-k filter's and the logprobs'
// ranking key)
__device__ __forceinline__ uint32_t topk_key(__half h) {
  const uint32_t b = __half_as_ushort(h);
  if ((b & 0x7FFFu) > 0x7C00u) return 0xFFFFu;
  return b == 0x8000u ? 0x8000u : ord16(h);
}

union Pack8 {
  uint4 u;
  __half h[8];
  __half2 h2[4];
};

}  // namespace sq
