// Weight-streaming GEMM for the tree-verify shapes:  C[n <= 128, N] = A[n, K] * W[N, K]^T   (fp16 in, fp32 accumulate
// in registers, fp16 out) -- nn.Linear of the target / draft forward (Engine/Llama_modules.py:108-110,138,270-272,
// Llama_model.py:213) for at most 128 rows.  With 128 rows every weight byte is used once: the kernel is a pure HBM
// stream (roofline = weight bytes / HBM bandwidth), so the design goal is bytes in flight, not FLOPs:
//   * one CTA per 64- to 256-wide slice of N (at most one wave on the device's SMs), warp-specialised: 1 TMA producer
//     lane and 2 consumer warpgroups (64 rows each); a 4-8 stage mbarrier ring of (A 128x64, W BNx64) SWIZZLE_128B tiles
//     keeps 192-200 KB per SM in flight; wgmma m64n64k16 (fp16 in, fp32 accumulators in registers), BN/64 per k-step;
//   * narrow outputs (o_proj / down_proj: N = hidden = 32 slices only) are split along K over a thread-block cluster
//     (1, SPLIT, 1): each CTA streams 1/SPLIT of K, pushes its fp32 partial rows into the shared memory of the row's
//     owner CTA (st.shared::cluster), one cluster barrier, owners add in a fixed order and store fp16;
//     gemm_tn_deep_kernel does the same at split 2 with the full ring, pushing into the owner's ring once it is drained.
#include <cstdio>
#include <cstdlib>

#include "sq_common.cuh"
#include "sq_ptx.cuh"

struct sq_gemm_plan {
  CUtensorMap tm_a, tm_w;
  __half* c;
  int ldc, n_max, N, K, bn, split, stages, mc, pdl, tiled, epi, n_out;
  int deep;   // split-K on gemm_tn_deep_kernel (ring as deep as the split-1 instance of that BN)
  int* err_flag;
#ifdef SQ_GEMM_STAMPS
  unsigned long long* stamps;
  int max_clusters;
#endif
};

namespace sq {

struct GemmArgs {
  __half* c;
  int ldc, n, N, K, kb_per_split;   // kb = 64-wide K blocks handled by one CTA
  int tiled, kb_total;              // weights pre-tiled: tile (n-tile, kb) is one contiguous BN x 64 block
  int m0;                           // first activation / output row of this launch (row tiles of 128 for n > 128)
  int epi, n_out;                   // epi 1: weight rows interleave 16 gate | 16 up rows -> out = silu(gate) * up, n_out columns
  int* err_flag;
#ifdef SQ_GEMM_STAMPS
  unsigned long long* stamps;       // per CTA: SM id, %globaltimer at first TMA issue, first full slot, last full slot, exit
#endif
};

#ifdef SQ_GEMM_STAMPS
// Probe build only (tools/gemm_mc_probe.py compiles this file with -DSQ_GEMM_STAMPS): the library never defines it.
__device__ __forceinline__ unsigned long long globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
#define SQ_STAMP(slot, value) \
  do { if (g.stamps) g.stamps[(blockIdx.y * gridDim.x + blockIdx.x) * 5 + (slot)] = (value); } while (0)
#else
#define SQ_STAMP(slot, value) do { } while (0)
#endif

constexpr int G_BK = 64;
constexpr int G_THREADS = 384;       // warpgroup 0: TMA (one lane), warpgroups 1, 2: wgmma + epilogue for rows 0-63 / 64-127
constexpr int G_CONSUMER_WARPS = 8;  // arrivals per CTA on an empty-slot barrier

// RING_RED: the split-K reduction slots reuse the ring (free once the k-loop is over) instead of their own region, which
// leaves room for a deeper ring at split > 1 (gemm_tn_deep_kernel)
template <int BN, int STAGES, int SPLIT, bool RING_RED = false>
struct GemmSmem {
  static constexpr int A_BYTES = 128 * 128;            // 128 rows x 64 halfs
  static constexpr int W_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + ((W_BYTES + 1023) / 1024) * 1024;   // stages stay 1024 B aligned (SW128)
  static constexpr int OFF_BAR = STAGES * STAGE_BYTES; // full[STAGES], empty[STAGES]
  static constexpr int OFF_RED = RING_RED ? 0 : OFF_BAR + 256;   // split-K: SPLIT slots x (128/SPLIT rows) x (BN+4) floats
  static constexpr int R_STRIDE = BN + 4;
  static constexpr int RED_BYTES = SPLIT > 1 ? 128 * R_STRIDE * 4 : 0;
  static constexpr int TOTAL = RING_RED ? OFF_BAR + 256 : OFF_RED + RED_BYTES;
  static_assert(!RING_RED || RED_BYTES <= OFF_BAR, "reduction slots must fit in the ring");
};

// barrier.cluster without .aligned: the producer warpgroup reaches it divergently (lane 0 after its loop)
__device__ __forceinline__ void cluster_arrive_wait() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}

// Weight tiles are read once per forward: load them with an L2 evict-first policy so that the 405 MB a 7B layer streams
// through the 50 MB L2 does not push out the activation slab every CTA re-reads (evict-last).
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void tma_load_2d_hint(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(dst),
      "l"(tm), "r"(bar), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}

__device__ __forceinline__ void tma_load_2d_mc(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%4, %5}], [%2], %3;" ::"r"(dst),
      "l"(tm), "r"(bar), "h"(mask), "r"(c0), "r"(c1)
      : "memory");
}

// MC = CTAs (along N) that share one activation K-slab: each loads 128/MC of its rows and multicasts them to all.
// RING_RED (split > 1, MC == 1): the partial rows land in the owners' rings, after a cluster barrier that every CTA passes
// once its k-loop has read its last slot.
template <int BN, int STAGES, int SPLIT, int MC, bool RING_RED>
__device__ __forceinline__ void gemm_tn_body(const CUtensorMap& tm_a, const CUtensorMap& tm_w, GemmArgs g) {
  // cluster (MC, SPLIT): rank = mcr + MC * ks.  CTAs with the same ks share the activation slab (multicast group); CTAs
  // with the same mcr hold the K-splits of one output tile (DSMEM reduction group).
  static_assert(!RING_RED || (SPLIT > 1 && MC == 1), "ring reduction: split-K without multicast");
  using SM = GemmSmem<BN, STAGES, SPLIT, RING_RED>;
  constexpr int NCH = BN / 64;                             // 64-column accumulator chunks (one wgmma m64n64k16 each)
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n0 = blockIdx.x * BN;
  const int ks = blockIdx.y;                               // K split index == rank in the (1, SPLIT) cluster
  const int mcr = (MC > 1) ? (int)(blockIdx.x % MC) : 0;   // rank in the (MC, 1) cluster
  const int kb0 = ks * g.kb_per_split;
  const int nkb = g.kb_per_split;
  const uint32_t s_base = ptx::smem_u32(smem);
  const uint32_t bar_full = s_base + SM::OFF_BAR, bar_empty = bar_full + 8 * STAGES;

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(bar_full + 8 * s, 1);
      ptx::mbar_init(bar_empty + 8 * s, G_CONSUMER_WARPS * MC);   // every consumer warp of every CTA that received the slot
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  if (MC > 1)   // the peers' barriers must be initialised before any multicast / remote arrive can target them
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");

  if (warp < 4) {
    // ===== TMA producer =====
    if (tid == 0) {
      asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#ifdef SQ_GEMM_STAMPS
      uint32_t smid;
      asm volatile("mov.u32 %0, %smid;" : "=r"(smid));
      SQ_STAMP(0, smid);
      SQ_STAMP(1, globaltimer());
#endif
      // Weights do not depend on the previous kernel: under programmatic dependent launch the first ring of weight
      // tiles streams in while that kernel is still running; only the activation loads wait for it.
      const uint64_t pol_w = l2_policy_evict_first(), pol_a = l2_policy_evict_last();
      const int pre = nkb < STAGES ? nkb : STAGES;
      for (int kb = 0; kb < pre; ++kb) {
        const uint32_t sa = s_base + kb * SM::STAGE_BYTES, sw = sa + SM::A_BYTES;
        ptx::mbar_expect_tx(bar_full + 8 * kb, SM::A_BYTES + SM::W_BYTES);
        if (g.tiled) tma_load_2d_hint(sw, &tm_w, bar_full + 8 * kb, 0, ((int)blockIdx.x * g.kb_total + kb0 + kb) * BN, pol_w);
        else tma_load_2d_hint(sw, &tm_w, bar_full + 8 * kb, (kb0 + kb) * G_BK, n0, pol_w);
      }
      asm volatile("griddepcontrol.wait;" ::: "memory");
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < nkb; ++kb) {
        const uint32_t sa = s_base + stage * SM::STAGE_BYTES, sw = sa + SM::A_BYTES;
        if (kb >= pre) {
          ptx::mbar_wait_one(bar_empty + 8 * stage, phase ^ 1, g.err_flag, 11);   // slot free in EVERY CTA of the cluster
          ptx::mbar_expect_tx(bar_full + 8 * stage, SM::A_BYTES + SM::W_BYTES);
          if (g.tiled) tma_load_2d_hint(sw, &tm_w, bar_full + 8 * stage, 0, ((int)blockIdx.x * g.kb_total + kb0 + kb) * BN, pol_w);
          else tma_load_2d_hint(sw, &tm_w, bar_full + 8 * stage, (kb0 + kb) * G_BK, n0, pol_w);
        }
        if (MC == 1) tma_load_2d_hint(sa, &tm_a, bar_full + 8 * stage, (kb0 + kb) * G_BK, g.m0, pol_a);
        else tma_load_2d_mc(sa + mcr * (SM::A_BYTES / MC), &tm_a, bar_full + 8 * stage, (kb0 + kb) * G_BK, g.m0 + mcr * (128 / MC),
                            (uint16_t)(((1u << MC) - 1u) << (MC * ks)));
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    if constexpr (RING_RED) cluster_arrive_wait();   // (the consumers' barrier before their pushes: see below)
  } else {
    // ===== consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64), all BN columns, accumulators in registers =====
    const int wg = (warp >> 2) - 1;
    float acc[NCH][32];
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
      for (int e = 0; e < 32; ++e) acc[c][e] = 0.f;
    // frees a slot -- in every CTA whose multicast writes into this CTA's slot
    auto release = [&](int s) {
      if (lane == 0) {
        if (MC == 1) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar_empty + 8 * s) : "memory");
        else
          for (int r = 0; r < MC; ++r) ptx::mbar_arrive_cluster(bar_empty + 8 * s, (uint32_t)(MC * ks + r));
      }
    };
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int kb = 0; kb < nkb; ++kb) {
      ptx::mbar_wait(bar_full + 8 * stage, phase, g.err_flag, 12);               // TMA bytes have landed
#ifdef SQ_GEMM_STAMPS
      if (tid == 128 && kb == 0) SQ_STAMP(2, globaltimer());
      if (tid == 128 && kb == nkb - 1) SQ_STAMP(3, globaltimer());
#endif
      const uint32_t sa = s_base + stage * SM::STAGE_BYTES + wg * 8192, sw = s_base + stage * SM::STAGE_BYTES + SM::A_BYTES;
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < G_BK / 16; ++k)
#pragma unroll
        for (int c = 0; c < NCH; ++c)
          ptx::wgmma_ss<0>(acc[c], gmma_desc(sa + k * 32, 16, 1024), gmma_desc(sw + c * 8192 + k * 32, 16, 1024), 1);
      ptx::wgmma_commit();
      // keep this k-block's group in flight: only the previous one has to be done before its slot is handed back
      asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
      if (prev >= 0) release(prev);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    ptx::wgmma_wait_all();
    if (prev >= 0) release(prev);
    // every CTA of the cluster has read its last ring slot (and no TMA write is pending: each was waited for) before any
    // partial row is pushed into a ring
    if constexpr (RING_RED) cluster_arrive_wait();
    // accumulator fragment: acc[c][4j + 2h + e] = tile row rbase + 8h, column 64c + 8j + 2q + e
    const int rbase = wg * 64 + (warp & 3) * 16 + (lane >> 2), q2 = 2 * (lane & 3);
    if (SPLIT == 1 && g.epi == 1) {
      // fused SwiGLU epilogue (Engine/Llama_modules.py:272: down(act(gate(x)) * up(x))): the weight rows interleave 16 gate
      // rows with their 16 up rows, so 8-column group j (j % 4 < 2) holds gates whose ups are group j + 2 of the same
      // thread.  Rounding points of the unfused path: gate, up -> fp16; silu in fp32 -> fp16; product -> fp16.
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = rbase + 8 * h;
        if (row >= g.n) continue;
        __half* orow = g.c + (int64_t)(g.m0 + row) * g.ldc;
#pragma unroll
        for (int c = 0; c < NCH; ++c)
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if ((j & 3) >= 2) continue;
            const int ob = (n0 + c * 64 + (j >> 2) * 32) / 2;
            if (ob >= g.n_out) continue;
            __half o[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float x = h2f(f2h(acc[c][4 * j + 2 * h + e]));
              const __half act = f2h(x / (1.0f + expf(-x)));
              o[e] = f2h(h2f(act) * h2f(f2h(acc[c][4 * (j + 2) + 2 * h + e])));
            }
            *reinterpret_cast<__half2*>(orow + ob + (j & 3) * 8 + q2) = __halves2half2(o[0], o[1]);
          }
      }
    } else if (SPLIT == 1) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = rbase + 8 * h;
        if (row >= g.n) continue;
        __half* crow = g.c + (int64_t)(g.m0 + row) * g.ldc + n0;
#pragma unroll
        for (int c = 0; c < NCH; ++c)
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (n0 + c * 64 + j * 8 < g.N)                    // (ragged last tile: N is a multiple of 32)
              *reinterpret_cast<__half2*>(crow + c * 64 + j * 8 + q2) =
                  __floats2half2_rn(acc[c][4 * j + 2 * h], acc[c][4 * j + 2 * h + 1]);
      }
    } else {
      // push this K-split's fp32 partial rows to the CTA that owns each row (rows dealt in blocks of 128/SPLIT)
      constexpr int RPC = 128 / SPLIT;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = rbase + 8 * h;
        uint32_t dst;
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(dst) : "r"(s_base + SM::OFF_RED), "r"((uint32_t)mcr + MC * (row / RPC)));
        dst += (uint32_t)((ks * RPC + row % RPC) * SM::R_STRIDE * 4);
#pragma unroll
        for (int c = 0; c < NCH; ++c)
#pragma unroll
          for (int j = 0; j < 8; ++j)
            asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(dst + (c * 64 + j * 8 + q2) * 4),
                         "f"(acc[c][4 * j + 2 * h]), "f"(acc[c][4 * j + 2 * h + 1])
                         : "memory");
      }
    }
  }
  __syncthreads();

  // (MC > 1: no CTA may leave while a peer can still multicast into its slots / arrive on its barriers;
  //  SPLIT > 1: the partial rows of every K-split must have landed in the owners' shared memory)
  if (MC > 1 || SPLIT > 1)
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");

  if (SPLIT > 1) {
    // owner CTA ks reduces rows [ks*RPC, (ks+1)*RPC): sum of the SPLIT slots in split order, fp16 out
    constexpr int RPC = 128 / SPLIT;
    constexpr int CPR = BN / 4;
    const float* red = reinterpret_cast<const float*>(smem + SM::OFF_RED);
    for (int i = tid; i < RPC * CPR; i += G_THREADS) {
      const int lr = i / CPR, cc = i % CPR;
      const int row = ks * RPC + lr;
      if (row >= g.n) continue;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int s = 0; s < SPLIT; ++s) {
        const float4 o = *reinterpret_cast<const float4*>(red + (s * RPC + lr) * SM::R_STRIDE + cc * 4);
        acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w;
      }
      const __half2 lo = __floats2half2_rn(acc.x, acc.y), hi = __floats2half2_rn(acc.z, acc.w);
      uint2 pk;
      pk.x = *reinterpret_cast<const uint32_t*>(&lo);
      pk.y = *reinterpret_cast<const uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(g.c + (int64_t)(g.m0 + row) * g.ldc + n0 + cc * 4) = pk;
    }
  }
#ifdef SQ_GEMM_STAMPS
  __syncthreads();
  if (tid == 0) SQ_STAMP(4, globaltimer());
#endif
}

template <int BN, int STAGES, int SPLIT, int MC>
__global__ void __launch_bounds__(G_THREADS, 1)
    gemm_tn_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w, GemmArgs g) {
  gemm_tn_body<BN, STAGES, SPLIT, MC, false>(tm_a, tm_w, g);
}

// Split-K with the ring of the split-1 instances (8 stages at BN 64, 6 at BN 128): at split 2 the 4-stage ring of
// gemm_tn_kernel keeps too few bytes in flight per SM to stream the narrow o_proj / down_proj shapes at HBM rate.
template <int BN, int STAGES, int SPLIT>
__global__ void __launch_bounds__(G_THREADS, 1)
    gemm_tn_deep_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w, GemmArgs g) {
  gemm_tn_body<BN, STAGES, SPLIT, 1, true>(tm_a, tm_w, g);
}

}  // namespace sq

using namespace sq;

typedef CUresult (*PFN_tmapEncodeTiledG)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                         const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                         CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int encode_2d(CUtensorMap* tm, const void* base, uint64_t inner, uint64_t outer, uint64_t pitch_bytes,
                     uint32_t box_inner, uint32_t box_outer, CUtensorMapL2promotion prom) {
  static PFN_tmapEncodeTiledG fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (PFN_tmapEncodeTiledG)p;
  }
  if (!fn) { set_error("cuTensorMapEncodeTiled unavailable"); return SQ_ERR_CUDA; }
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {pitch_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, prom, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed: %d", (int)r); return SQ_ERR_CUDA; }
  return SQ_OK;
}

// Tile selection: put a CTA on (nearly) every SM with the widest N tile that allows -- per-SM ingest, not HBM, is what
// limits a 128-row weight stream, and the activation tile every CTA re-reads is pure overhead: a wider BN and a 2-CTA
// multicast of the activation slab both raise the weight share of each SM's ingest.  Clusters of more than 2 CTAs are not
// picked: the H100 holds 30 clusters of 4 at this kernel's shared memory (cudaOccupancyMaxActiveClusters), so the 32 of
// an N = 4096 split-4 grid ran in two waves (DESIGN §4).
static int sm_count() {
  static int n_sm = 0;
  if (!n_sm) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        n_sm <= 0) {
      cudaGetLastError();
      n_sm = 132;                                       // H100 SXM: tile choice for a host without a device
    }
  }
  return n_sm;
}

static void choose_tiles(sq_gemm_plan* p, bool allow_split) {
  const int N = p->N, kb = p->K / 64;
  const int n_sm = sm_count();
  const int cands[] = {256, 192, 128, 64};              // whole wgmma n64 chunks
  int best_bn = 128, best_split = 1, best_mc = 1;
  double best_score = -1.0;
  for (int bn : cands) {
    const int tiles = (N + bn - 1) / bn;
    for (int split : {1, 2}) {
      if (kb % split || (split > 1 && !allow_split)) continue;
      if (split > 1 && (bn > 128 || N % bn)) continue;       // split-K instances: BN <= 128, no ragged tile
      const int ctas = tiles * split;
      if (ctas > n_sm) continue;
      for (int mc : {1, 2}) {
        if (mc == 2 && (tiles % 2 || split > 1)) continue;   // a cluster of at most 2 CTAs
        // modelled weight bandwidth ~ CTAs x weight share of the per-SM ingest; split-K pays a reduction tail
        const double a_share = 128.0 / mc, share = bn / (bn + a_share);
        double score = ctas * share;
        if (split > 1) score *= 0.85;
        if (score > best_score) { best_score = score; best_bn = bn; best_split = split; best_mc = mc; }
      }
    }
  }
  p->bn = best_bn; p->split = best_split; p->mc = best_mc;
  p->deep = best_split > 1;                             // split-K on the deep ring (gemm_tn_deep_kernel)
}

static void pick_tiles(sq_gemm_plan* p) {
  const int kb = p->K / 64;
  const bool allow_split = p->epi == 0;                 // a fused epilogue needs the whole K sum in one CTA
  choose_tiles(p, allow_split);
  // tuning / tests: "bn,split,mc" names an instance of run_tile's table; "bn,2,1,1" the deep-ring split-K kernel (an
  // illegal tile is ignored: check sq_gemm_plan_info).  The attention kernel's counterpart is SQ_ATTN_SPLITS (sq_attn.cu).
  const char* force = getenv("SQ_GEMM_FORCE");
  if (force) {
    int fb = 0, fs = 0, fm = 1, fd = 0;
    const int nf = sscanf(force, "%d,%d,%d,%d", &fb, &fs, &fm, &fd);
    const bool bn_ok = fb == 64 || fb == 128 || fb == 192 || fb == 256;
    if (nf >= 2 && bn_ok && (fs == 1 || fs == 2 || fs == 4) && kb % fs == 0 && (fm == 1 || fm == 2) &&
        !(fs > 1 && (fb > 128 || p->N % fb || !allow_split)) && !(fm == 2 && ((p->N + fb - 1) / fb) % 2)) {
      p->bn = fb; p->split = fs; p->mc = fm;
      p->deep = nf == 4 && fd == 1 && fs == 2 && fm == 1;
    }
  }
}

/* The tile shape a plan for (N, K) will use: callers that pre-tile the weights need BN before they build the copy. */
extern "C" int sq_gemm_pick_tiles(int N, int K, int* bn, int* split, int* mc) { return sq_gemm_pick_tiles_ex(N, K, 0, bn, split, mc); }

extern "C" int sq_gemm_pick_tiles_ex(int N, int K, int flags, int* bn, int* split, int* mc) {
  SQ_CHECK_ARG(K % 64 == 0 && N % 32 == 0, "sq_gemm_pick_tiles: K %% 64, N %% 32");
  sq_gemm_plan p{};
  p.N = N; p.K = K; p.epi = (flags & SQ_GEMM_SWIGLU) ? 1 : 0;
  pick_tiles(&p);
  *bn = p.bn; *split = p.split; *mc = p.mc;
  return SQ_OK;
}

static int plan_create(sq_gemm_plan** plan, const sq_half* a, int lda, int n_max, const sq_half* w, int N, int K, sq_half* c,
                       int ldc, int* err_flag, int flags);

extern "C" int sq_gemm_plan_create(sq_gemm_plan** plan, const sq_half* a, int lda, int n_max, const sq_half* w, int N,
                                   int K, sq_half* c, int ldc, int* err_flag) {
  return plan_create(plan, a, lda, n_max, w, N, K, c, ldc, err_flag, 0);
}

/* Same, for weights stored PRE-TILED: (ceil(N/BN), K/64, BN, 64) fp16 contiguous (rows beyond N zero), BN from
 * sq_gemm_pick_tiles -- every TMA weight load is then ONE contiguous BN*128-byte block of HBM instead of BN separate
 * 128-byte segments K*2 bytes apart. */
extern "C" int sq_gemm_plan_create_tiled(sq_gemm_plan** plan, const sq_half* a, int lda, int n_max, const sq_half* w_tiled,
                                         int N, int K, sq_half* c, int ldc, int* err_flag) {
  return plan_create(plan, a, lda, n_max, w_tiled, N, K, c, ldc, err_flag, SQ_GEMM_TILED);
}

/* flags: SQ_GEMM_TILED (weights pre-tiled as above) | SQ_GEMM_SWIGLU (fused epilogue, see sq_gemm_plan_set_epilogue; the
 * tile choice then excludes split-K) */
extern "C" int sq_gemm_plan_create_ex(sq_gemm_plan** plan, const sq_half* a, int lda, int n_max, const sq_half* w, int N,
                                      int K, sq_half* c, int ldc, int* err_flag, int flags) {
  return plan_create(plan, a, lda, n_max, w, N, K, c, ldc, err_flag, flags);
}

static int plan_create(sq_gemm_plan** plan, const sq_half* a, int lda, int n_max, const sq_half* w, int N, int K, sq_half* c,
                       int ldc, int* err_flag, int flags) {
  const int tiled = (flags & SQ_GEMM_TILED) ? 1 : 0;
  SQ_CHECK_ARG(plan && a && w && c, "sq_gemm_plan_create: null pointer");
  SQ_CHECK_ARG(K % 64 == 0 && N % 32 == 0 && lda % 8 == 0 && ldc % 8 == 0, "sq_gemm_plan_create: K %% 64, N %% 32");
  sq_gemm_plan* p = new sq_gemm_plan();
  p->c = (__half*)c; p->ldc = ldc; p->n_max = n_max; p->N = N; p->K = K; p->err_flag = err_flag;
  p->tiled = tiled; p->epi = (flags & SQ_GEMM_SWIGLU) ? 1 : 0; p->n_out = p->epi ? N / 2 : 0;
  if (p->epi) SQ_CHECK_ARG(N % 32 == 0, "sq_gemm_plan_create: SwiGLU needs N %% 32 == 0");
  pick_tiles(p);
  {
    p->pdl = pdl_enabled() ? 1 : 0;
  }
  p->stages = p->split > 1 && !p->deep ? 4 : (p->bn == 256 ? 4 : p->bn == 192 ? 5 : p->bn == 128 ? 6 : 8);   // == run_tile / run_deep_tile
  int rc = encode_2d(&p->tm_a, a, (uint64_t)K, (uint64_t)n_max, (uint64_t)lda * 2, 64, (uint32_t)(128 / p->mc),
                     CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
  if (!rc) {
    if (tiled) rc = encode_2d(&p->tm_w, w, 64, (uint64_t)((N + p->bn - 1) / p->bn) * (uint64_t)(K / 64) * (uint64_t)p->bn, 128, 64,
                              (uint32_t)p->bn, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    else rc = encode_2d(&p->tm_w, w, (uint64_t)K, (uint64_t)N, (uint64_t)K * 2, 64, (uint32_t)p->bn, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  }
  if (rc) { delete p; return rc; }
  *plan = p;
  return SQ_OK;
}

extern "C" int sq_gemm_plan_destroy(sq_gemm_plan* plan) {
  delete plan;
  return SQ_OK;
}

template <int BN, int STAGES, int SPLIT, int MC, bool DEEP = false>
static int launch_gemm(sq_gemm_plan* p, GemmArgs& g, cudaStream_t st) {
  using SM = GemmSmem<BN, STAGES, SPLIT, DEEP>;
  constexpr int smem = SM::TOTAL + 1024;
  static_assert(smem <= 227 * 1024, "shared memory budget");
  static_assert(!DEEP || MC == 1, "gemm_tn_deep_kernel has no multicast");
  void (*kernel)(CUtensorMap, CUtensorMap, GemmArgs);
  if constexpr (DEEP) kernel = gemm_tn_deep_kernel<BN, STAGES, SPLIT>;
  else kernel = gemm_tn_kernel<BN, STAGES, SPLIT, MC>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { set_error("sq_gemm: smem attr: %s", cudaGetErrorString(e)); return SQ_ERR_CUDA; }
    attr = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((p->N + BN - 1) / BN, SPLIT, 1);
  cfg.blockDim = dim3(G_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = MC;
  at[0].val.clusterDim.y = SPLIT;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  if (p->pdl) {
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.numAttrs = 2;
  }
#ifdef SQ_GEMM_STAMPS
  if (p->max_clusters < 0) {   // probe build: how many (MC, SPLIT) clusters of this instance the device holds at once
    cfg.numAttrs = 1;
    if (cudaOccupancyMaxActiveClusters(&p->max_clusters, kernel, &cfg) != cudaSuccess) {
      cudaGetLastError();
      p->max_clusters = -2;
    }
    return SQ_OK;
  }
#endif
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, p->tm_a, p->tm_w, g);
  if (e != cudaSuccess) { set_error("sq_gemm: launch failed: %s", cudaGetErrorString(e)); return SQ_ERR_CUDA; }
  SQ_CHECK_LAUNCH("sq_gemm");
  return SQ_OK;
}

static int run_tile(sq_gemm_plan* plan, GemmArgs& g, cudaStream_t st) {
  const int bn = plan->bn, sp = plan->split, mc = plan->mc;
#define SQ_G(BN_, ST_, SP_, MC_) if (bn == BN_ && sp == SP_ && mc == MC_) return launch_gemm<BN_, ST_, SP_, MC_>(plan, g, st)
  SQ_G(256, 4, 1, 1); SQ_G(256, 4, 1, 2);
  SQ_G(192, 5, 1, 1); SQ_G(192, 5, 1, 2);
  SQ_G(128, 6, 1, 1); SQ_G(128, 6, 1, 2); SQ_G(128, 4, 2, 1); SQ_G(128, 4, 4, 1); SQ_G(128, 4, 2, 2); SQ_G(128, 4, 4, 2);
  SQ_G(64, 8, 1, 1); SQ_G(64, 8, 1, 2); SQ_G(64, 4, 2, 1); SQ_G(64, 4, 4, 1); SQ_G(64, 4, 2, 2); SQ_G(64, 4, 4, 2);
#undef SQ_G
  set_error("sq_gemm_run: no kernel for bn=%d split=%d mc=%d", bn, sp, mc);
  return SQ_ERR_UNSUPPORTED;
}

// Split-K tiles on the deep ring (picked by choose_tiles only; SQ_GEMM_FORCE always names a run_tile instance)
static int run_deep_tile(sq_gemm_plan* plan, GemmArgs& g, cudaStream_t st) {
  if (plan->bn == 64 && plan->split == 2) return launch_gemm<64, 8, 2, 1, true>(plan, g, st);
  if (plan->bn == 128 && plan->split == 2) return launch_gemm<128, 6, 2, 1, true>(plan, g, st);
  set_error("sq_gemm_run: no deep-ring kernel for bn=%d split=%d", plan->bn, plan->split);
  return SQ_ERR_UNSUPPORTED;
}

extern "C" int sq_gemm_run(sq_gemm_plan* plan, int n, void* stream) { return sq_gemm_run_at(plan, n, 0, nullptr, 0, stream); }

/* rows [a_row0, a_row0 + n) of the plan's activation buffer -> rows [0, n) of `c` (pitch ldc halfs; NULL = the plan's own
 * output buffer, rows [a_row0, ...)). */
extern "C" int sq_gemm_run_at(sq_gemm_plan* plan, int n, int a_row0, sq_half* c, int ldc, void* stream) {
  SQ_CHECK_ARG(plan != nullptr, "sq_gemm_run: null plan");
  SQ_CHECK_ARG(n >= 0 && a_row0 >= 0 && a_row0 + n <= plan->n_max, "sq_gemm_run: rows [%d, %d) exceed the plan's n_max=%d", a_row0, a_row0 + n, plan->n_max);
  SQ_CHECK_ARG(c == nullptr || (ldc % 8 == 0 && ((uintptr_t)c % 16) == 0), "sq_gemm_run: output override must be 16 B aligned, pitch %% 8");
  // more than 128 rows (prefill): one launch per 128-row tile, each streaming the weights again (once per prompt)
  for (int m0 = 0; m0 < n; m0 += 128) {
    GemmArgs g;
    g.n = n - m0 < 128 ? n - m0 : 128; g.N = plan->N; g.K = plan->K;
    g.kb_per_split = plan->K / 64 / plan->split;
    g.tiled = plan->tiled; g.kb_total = plan->K / 64;
    g.m0 = a_row0 + m0; g.epi = plan->epi; g.n_out = plan->n_out;
    // the kernel addresses output row (g.m0 + row): bias the base so that activation row a_row0 lands on output row 0
    if (c) { g.ldc = ldc; g.c = (__half*)c - (int64_t)a_row0 * ldc; }
    else { g.ldc = plan->ldc; g.c = plan->c; }
    g.err_flag = plan->err_flag;
#ifdef SQ_GEMM_STAMPS
    g.stamps = plan->stamps;
#endif
    const int rc = plan->deep ? run_deep_tile(plan, g, (cudaStream_t)stream) : run_tile(plan, g, (cudaStream_t)stream);
    if (rc != SQ_OK) return rc;
  }
  return SQ_OK;
}

/* Fused epilogue.  kind 0: C = A W^T (default).  kind 1 (SwiGLU): the weight rows interleave 16 gate rows / 16 up rows
 * (row 32b + t = gate[16b + t], row 32b + 16 + t = up[16b + t]); C (n, n_out = N/2) = silu(gate) * up.  Split-K plans
 * cannot fuse it. */
extern "C" int sq_gemm_plan_set_epilogue(sq_gemm_plan* plan, int kind, int n_out) {
  SQ_CHECK_ARG(plan != nullptr && (kind == 0 || kind == 1), "sq_gemm_plan_set_epilogue: bad arguments");
  SQ_CHECK_ARG(kind == 0 || (plan->split == 1 && n_out % 16 == 0 && 2 * n_out <= plan->N + 31), "sq_gemm_plan_set_epilogue: SwiGLU needs split 1, n_out %% 16 == 0");
  plan->epi = kind; plan->n_out = n_out;
  return SQ_OK;
}

extern "C" int sq_gemm_plan_info(sq_gemm_plan* plan, int* bn, int* split, int* stages) {
  *bn = plan->bn; *split = plan->split; *stages = plan->stages + 100 * plan->mc;
  return SQ_OK;
}

#ifdef SQ_GEMM_STAMPS
/* Probe build only.  Stamps: NULL or 5 u64 per CTA (see GemmArgs::stamps) for the plan's following runs. */
extern "C" int sq_gemm_probe_set_stamps(sq_gemm_plan* plan, unsigned long long* stamps) {
  plan->stamps = stamps;
  return SQ_OK;
}
/* cudaOccupancyMaxActiveClusters for the plan's instance at its grid, cluster shape and shared-memory size (no launch). */
extern "C" int sq_gemm_probe_max_clusters(sq_gemm_plan* plan, int* max_clusters) {
  plan->max_clusters = -1;
  GemmArgs g{};
  const int rc = run_tile(plan, g, nullptr);
  *max_clusters = plan->max_clusters;
  plan->max_clusters = 0;
  return rc;
}
#endif
