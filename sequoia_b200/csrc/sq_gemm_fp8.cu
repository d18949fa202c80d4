// FP8 (E4M3) weight-streaming GEMM for the target's layer projections:  C[n, N] = A[n, K] * W'[N, K]^T, where
// W'[j, k] = fp16(fp16(q[j, k]) * s[j]) is the dequantized weight (q e4m3, one fp16 scale per output channel), fp16
// activations, fp32 accumulation in registers, fp16 out.  It computes what sq_gemm computes on the fp16 matrix W', up to
// the order of the fp32 sum, while streaming half the weight bytes.
//   * swap-AB: a CTA computes C^T tiles of 64 NWG weight rows x R activation rows (R = 64 or 128, chosen per launch from
//     the row count) with wgmma m64nRk16.  The dequantized weights are the A operand, in registers: each consumer thread
//     loads its fragment bytes of a TMA-filled shared-memory ring, converts them with cvt.rn.f16x2.e4m3x2 and multiplies
//     by its rows' scales (one HMUL2 per pair), so every weight element is converted once per launch.  The activations
//     are the B operand: K-major SWIZZLE_128B tiles in the same ring.
//   * the weights are stored pre-tiled (sq_gemm_fp8_tile_weights, the only producer of the layout): one 4 KB block per
//     (64-row tile, 64-wide K block), in which each consumer thread's 32 fragment bytes are two 16-byte pieces 2 KB apart.
//   * warp-specialised: one TMA producer lane and NWG consumer warpgroups; an mbarrier ring whose waits are bounded and
//     report through err_flag.  Weight loads of the first ring are issued before griddepcontrol.wait.
//   * narrow outputs (o_proj / down_proj) split K over a (1, SPLIT, 1) thread-block cluster: each CTA pushes its fp32
//     partial tile into the shared memory of the CTA that owns those activation rows, and the owner adds the SPLIT
//     partials in rank order, so the result does not vary from run to run.
#include <cstdio>
#include <cstdlib>

#include "sq_common.cuh"
#include "sq_ptx.cuh"

struct sq_gemm_fp8_plan {
  CUtensorMap tm_a;
  const uint8_t* w;
  const __half* scale;
  __half* c;
  int ldc, n_max, N, K, nwg, split;
  int* err_flag;
};

namespace sq {
namespace fp8 {

constexpr int BK = 64;
constexpr int W_BLOCK = 4096;          // bytes of one (64-row tile, 64-wide K block) of e4m3 weights
constexpr int RING_BYTES = 200 * 1024;

struct Args {
  const uint8_t* w;                    // pre-tiled e4m3 weights: block (t, kb) at (t * KB + kb) * 4096
  const __half* scale;                 // (N) per-output-channel scales
  __half* c;
  int ldc, n, N, KB, m0;               // m0: first activation / output row of this launch
  int* err_flag;
};

template <int R, int NWG>
struct Smem {
  static constexpr int A_BYTES = R * 128;                    // R activation rows x 64 halfs, SW128
  static constexpr int STAGE_BYTES = A_BYTES + NWG * W_BLOCK;
  static constexpr int STAGES = RING_BYTES / STAGE_BYTES < 8 ? RING_BYTES / STAGE_BYTES : 8;
  static constexpr int OFF_BAR = STAGES * STAGE_BYTES;
  static constexpr int TOTAL = OFF_BAR + 256;
};

// split-K reduction buffer (reuses the ring once every CTA of the cluster has left its main loop): SPLIT slots of RPO
// activation rows x (64 NWG + 4) fp32 partial sums in the CTA that owns those rows
template <int R, int NWG, int SPLIT>
struct Red {
  static constexpr int RPO = ((R + SPLIT - 1) / SPLIT + 7) / 8 * 8;
  static constexpr int STRIDE = 64 * NWG + 4;
  static constexpr int BYTES = SPLIT * RPO * STRIDE * 4;
};

__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

// two e4m3 (low byte = lower column) -> f16x2, exact
__device__ __forceinline__ uint32_t e4m3x2_to_f16x2(uint32_t two) {
  uint32_t out;
  asm("{\n\t.reg .b16 t;\n\tcvt.u16.u32 t, %1;\n\tcvt.rn.f16x2.e4m3x2 %0, t;\n\t}" : "=r"(out) : "r"(two));
  return out;
}

__device__ __forceinline__ uint32_t hmul2_u32(uint32_t x, __half2 s) {
  __half2 h = *reinterpret_cast<__half2*>(&x);
  h = __hmul2(h, s);
  return *reinterpret_cast<uint32_t*>(&h);
}

// D[64 x 64] += A[registers: the m64k16 fragment] * B[smem desc, 16 x 64, K-major]
__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc)
      : "memory");
}
// D[64 x 128] += A[registers: the m64k16 fragment] * B[smem desc, 16 x 128, K-major]
__device__ __forceinline__ void wgmma_rs_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc)
      : "memory");
}

template <int R>
__device__ __forceinline__ void wgmma_rs(float (&d)[R / 2], const uint32_t (&a)[4], uint64_t bdesc) {
  if constexpr (R == 128) wgmma_rs_n128(d, a, bdesc);
  else wgmma_rs_n64(d, a, bdesc);
}

template <int R, int NWG, int SPLIT>
__global__ void __launch_bounds__(128 * (NWG + 1), 1) gemm_fp8_kernel(const __grid_constant__ CUtensorMap tm_a, Args g) {
  using SM = Smem<R, NWG>;
  constexpr int STAGES = SM::STAGES;
  constexpr int CONSUMER_WARPS = 4 * NWG;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int t0 = blockIdx.x * NWG;                                // first 64-row weight tile of this CTA
  const int tiles = g.N / 64;
  const int n_valid = tiles - t0 < NWG ? tiles - t0 : NWG;        // (the last CTA may hold fewer tiles)
  const int ks = blockIdx.y;                                      // K split == rank in the (1, SPLIT, 1) cluster
  const int kb0 = ks * g.KB / SPLIT, nkb = (ks + 1) * g.KB / SPLIT - kb0;
  const uint32_t s_base = ptx::smem_u32(smem);
  const uint32_t bar_full = s_base + SM::OFF_BAR, bar_empty = bar_full + 8 * STAGES;

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(bar_full + 8 * s, 1);
      ptx::mbar_init(bar_empty + 8 * s, CONSUMER_WARPS);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  const uint32_t tx_bytes = SM::A_BYTES + n_valid * W_BLOCK;
  if (warp < 4) {
    // ===== TMA producer =====
    if (tid == 0) {
      asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
      // weights do not depend on the previous kernel: the first ring of them streams in while it still runs
      const int pre = nkb < STAGES ? nkb : STAGES;
      for (int kb = 0; kb < pre; ++kb) {
        const uint32_t sw = s_base + kb * SM::STAGE_BYTES + SM::A_BYTES;
        ptx::mbar_expect_tx(bar_full + 8 * kb, tx_bytes);
        for (int w = 0; w < n_valid; ++w)
          bulk_load(sw + w * W_BLOCK, g.w + ((int64_t)(t0 + w) * g.KB + kb0 + kb) * W_BLOCK, W_BLOCK, bar_full + 8 * kb);
      }
      asm volatile("griddepcontrol.wait;" ::: "memory");
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < nkb; ++kb) {
        const uint32_t sa = s_base + stage * SM::STAGE_BYTES, sw = sa + SM::A_BYTES;
        if (kb >= pre) {
          ptx::mbar_wait_one(bar_empty + 8 * stage, phase ^ 1, g.err_flag, 21);
          ptx::mbar_expect_tx(bar_full + 8 * stage, tx_bytes);
          for (int w = 0; w < n_valid; ++w)
            bulk_load(sw + w * W_BLOCK, g.w + ((int64_t)(t0 + w) * g.KB + kb0 + kb) * W_BLOCK, W_BLOCK, bar_full + 8 * stage);
        }
#pragma unroll
        for (int r = 0; r < R / 64; ++r)
          ptx::tma_load_2d(sa + r * 8192, &tm_a, bar_full + 8 * stage, (kb0 + kb) * BK, g.m0 + 64 * r);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ===== consumers: warpgroup wg owns weight tile t0 + wg (64 weight rows) x all R activation rows =====
    const int wg = (warp >> 2) - 1, tt = tid & 127;
    const bool valid = wg < n_valid;
    const int jrow = (tt >> 5) * 16 + (lane >> 2);                // this thread's weight rows: jrow, jrow + 8
    __half2 s_lo = __float2half2_rn(0.f), s_hi = s_lo;
    if (valid) {
      s_lo = __half2half2(g.scale[(t0 + wg) * 64 + jrow]);
      s_hi = __half2half2(g.scale[(t0 + wg) * 64 + jrow + 8]);
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    float acc[R / 2];
#pragma unroll
    for (int e = 0; e < R / 2; ++e) acc[e] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    for (int kb = 0; kb < nkb; ++kb) {
      ptx::mbar_wait(bar_full + 8 * stage, phase, g.err_flag, 22);
      const uint32_t sa = s_base + stage * SM::STAGE_BYTES;
      if (valid) {
        const uint8_t* wblk = smem + stage * SM::STAGE_BYTES + SM::A_BYTES + wg * W_BLOCK + tt * 16;
        const uint4 lo = *reinterpret_cast<const uint4*>(wblk);          // k16 steps 0, 1
        const uint4 hi = *reinterpret_cast<const uint4*>(wblk + 2048);   // k16 steps 2, 3
        const uint32_t raw[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
        uint32_t a[4][4];
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            // fragment register r of k16 step k: 2 bytes of word raw[2k + r / 2]; registers 0, 2 hold row jrow, 1, 3 row jrow + 8
            const uint32_t two = raw[2 * k + (r >> 1)] >> (16 * (r & 1));
            a[k][r] = hmul2_u32(e4m3x2_to_f16x2(two), (r & 1) ? s_hi : s_lo);
          }
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_rs<R>(acc, a[k], gmma_desc(sa + k * 32, 16, 1024));
        ptx::wgmma_commit();
        ptx::wgmma_wait_all();
      }
      if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar_empty + 8 * stage) : "memory");
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    // accumulator fragment (C^T): acc[4j + 2h + e] = weight row jrow + 8h, activation row 8j + 2q + e
    const int q2 = 2 * (lane & 3);
    if constexpr (SPLIT == 1) {
      if (valid) {
        __half* cbase = g.c + (int64_t)g.m0 * g.ldc + (t0 + wg) * 64 + jrow;
#pragma unroll
        for (int j = 0; j < R / 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int i = 8 * j + q2 + e;
            if (i < g.n) {
              cbase[(int64_t)i * g.ldc] = __float2half_rn(acc[4 * j + e]);
              cbase[(int64_t)i * g.ldc + 8] = __float2half_rn(acc[4 * j + 2 + e]);
            }
          }
      }
    } else {
      using RD = Red<R, NWG, SPLIT>;
      // every CTA of the cluster must be out of its main loop before peers overwrite its ring with partial sums
      asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
#pragma unroll
      for (int j = 0; j < R / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int i = 8 * j + q2 + e;
          if (i >= g.n) continue;
          uint32_t dst;
          asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(dst) : "r"(s_base), "r"((uint32_t)(i / RD::RPO)));
          dst += (uint32_t)(((ks * RD::RPO + i % RD::RPO) * RD::STRIDE + wg * 64 + jrow) * 4);
          asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(dst), "f"(acc[4 * j + e]) : "memory");
          asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(dst + 32), "f"(acc[4 * j + 2 + e]) : "memory");
        }
    }
  }
  if constexpr (SPLIT > 1) {
    using RD = Red<R, NWG, SPLIT>;
    static_assert(RD::BYTES <= SM::OFF_BAR, "split-K partials must fit the ring");
    // the producer warpgroup takes part in the first cluster barrier too (the consumers' one above)
    if (warp < 4) asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
    // the partial rows of every K split have landed in their owner's shared memory
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
    // owner ks adds the SPLIT partials of activation rows [ks RPO, (ks + 1) RPO) in rank order
    const float* red = reinterpret_cast<const float*>(smem);
    constexpr int CP = 32 * NWG;                                  // column pairs of a row
    for (int idx = tid; idx < RD::RPO * CP; idx += 128 * (NWG + 1)) {
      const int lr = idx / CP, cp = idx % CP;
      const int i = ks * RD::RPO + lr, col = 2 * cp;
      if (i >= g.n || col / 64 >= n_valid) continue;
      float x = 0.f, y = 0.f;
#pragma unroll
      for (int s = 0; s < SPLIT; ++s) {
        const float2 v = *reinterpret_cast<const float2*>(red + (s * RD::RPO + lr) * RD::STRIDE + col);
        x += v.x; y += v.y;
      }
      *reinterpret_cast<__half2*>(g.c + (int64_t)(g.m0 + i) * g.ldc + t0 * 64 + col) = __floats2half2_rn(x, y);
    }
  }
}

// pre-tiled layout: block (t, kb) = 4096 bytes; byte h * 2048 + tt * 16 + 8 (k & 1) + 2 r + e (h = k / 2) holds the
// fragment element (register r, half e) of k16 step k of consumer thread tt (warp tt / 32, lane tt % 32) of weight tile t
__global__ void tile_weights_kernel(const uint8_t* __restrict__ q, uint8_t* __restrict__ out, int N, int K) {
  const int KB = K / 64;
  const int64_t blocks = (int64_t)(N / 64) * KB;
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;      // one 16-byte piece of the output
  if (v >= blocks * 256) return;
  const int64_t blk = v / 256;
  const int t = (int)(blk / KB), kb = (int)(blk % KB);
  const int piece = (int)(v % 256), h = piece / 128, tt = piece % 128;
  const int g = (tt & 31) >> 2, tq = tt & 3, wrow = (tt >> 5) * 16;
  uint8_t b[16];
#pragma unroll
  for (int x = 0; x < 16; ++x) {
    const int k = 2 * h + x / 8, r = (x % 8) / 2, e = x % 2;
    const int row = wrow + g + 8 * (r & 1), col = 16 * k + 2 * tq + 8 * (r >> 1) + e;
    b[x] = q[(int64_t)(t * 64 + row) * K + kb * 64 + col];
  }
  *reinterpret_cast<uint4*>(out + v * 16) = *reinterpret_cast<const uint4*>(b);
}

}  // namespace fp8
}  // namespace sq

using namespace sq;
using namespace sq::fp8;

typedef CUresult (*PFN_tmapEncodeTiledF8)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                          const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                          CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// activations (rows, K) fp16 with row pitch lda: boxes of 64 rows x 64 halfs, SWIZZLE_128B; rows past n_max read as zero
static int encode_act(CUtensorMap* tm, const void* base, int K, int rows, int lda) {
  static PFN_tmapEncodeTiledF8 fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (PFN_tmapEncodeTiledF8)p;
  }
  if (!fn) { set_error("cuTensorMapEncodeTiled unavailable"); return SQ_ERR_CUDA; }
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)lda * 2};
  cuuint32_t box[2] = {64, 64};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed: %d", (int)r); return SQ_ERR_CUDA; }
  return SQ_OK;
}

static int fp8_sm_count() {
  static int n_sm = 0;
  if (!n_sm) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        n_sm <= 0) {
      cudaGetLastError();
      n_sm = 132;                                       // H100 SXM: the choice for a host without a device
    }
  }
  return n_sm;
}

// Instance choice: at most one CTA per SM, as many SMs busy as the shape allows.  A CTA's time per K block is modelled as
// its ingest, 64 NWG weight rows (1 byte each) plus 128 activation rows (2 bytes each), so a wider CTA re-reads the
// activations less often; a K split costs a reduction tail.
static void choose(int N, int K, int* nwg_out, int* split_out) {
  const int tiles = N / 64, KB = K / 64, n_sm = fp8_sm_count();
  double best = 1e30;
  int bn = 2, bs = 1;
  for (int nwg : {2, 3})
    for (int split : {1, 2, 3, 4}) {
      if (KB < split) continue;
      const int ctas = (tiles + nwg - 1) / nwg * split;
      const int waves = (ctas + n_sm - 1) / n_sm;
      double cost = waves * ((double)KB / split) * (64.0 * nwg + 256.0);
      if (split > 1) cost *= 1.05;
      if (cost < best) { best = cost; bn = nwg; bs = split; }
    }
  *nwg_out = bn; *split_out = bs;
}

extern "C" int sq_gemm_fp8_tile_weights(const uint8_t* q, uint8_t* q_tiled, int N, int K, void* stream) {
  SQ_CHECK_ARG(q && q_tiled, "sq_gemm_fp8_tile_weights: null pointer");
  SQ_CHECK_ARG(N > 0 && K > 0 && N % 64 == 0 && K % 64 == 0, "sq_gemm_fp8_tile_weights: N %% 64 and K %% 64 must be 0 (N=%d K=%d)", N, K);
  const int64_t pieces = (int64_t)N * K / 16;
  tile_weights_kernel<<<(unsigned)((pieces + 255) / 256), 256, 0, (cudaStream_t)stream>>>(q, q_tiled, N, K);
  SQ_CHECK_LAUNCH("sq_gemm_fp8_tile_weights");
  return SQ_OK;
}

extern "C" int sq_gemm_fp8_plan_create(sq_gemm_fp8_plan** plan, const sq_half* a, int lda, int n_max, const uint8_t* w_q,
                                       const sq_half* w_scale, int N, int K, sq_half* c, int ldc, int* err_flag) {
  SQ_CHECK_ARG(plan && a && w_q && w_scale && c, "sq_gemm_fp8_plan_create: null pointer");
  SQ_CHECK_ARG(N > 0 && K > 0 && N % 64 == 0 && K % 64 == 0, "sq_gemm_fp8_plan_create: N %% 64 and K %% 64 must be 0 (N=%d K=%d)", N, K);
  SQ_CHECK_ARG(n_max > 0, "sq_gemm_fp8_plan_create: n_max must be positive (got %d)", n_max);
  SQ_CHECK_ARG(lda >= K && lda % 8 == 0 && ldc >= N && ldc % 8 == 0,
               "sq_gemm_fp8_plan_create: lda >= K, ldc >= N, both multiples of 8 (lda=%d ldc=%d)", lda, ldc);
  sq_gemm_fp8_plan* p = new sq_gemm_fp8_plan();
  p->w = w_q; p->scale = (const __half*)w_scale; p->c = (__half*)c;
  p->ldc = ldc; p->n_max = n_max; p->N = N; p->K = K; p->err_flag = err_flag;
  choose(N, K, &p->nwg, &p->split);
  // tests / tuning: "nwg,split" (an illegal pair is ignored: check sq_gemm_fp8_plan_info)
  const char* force = getenv("SQ_GEMM_FP8_FORCE");
  if (force) {
    int fw = 0, fs = 0;
    if (sscanf(force, "%d,%d", &fw, &fs) == 2 && (fw == 2 || fw == 3) && fs >= 1 && fs <= 4 && K / 64 >= fs) {
      p->nwg = fw; p->split = fs;
    }
  }
  const int rc = encode_act(&p->tm_a, a, K, n_max, lda);
  if (rc) { delete p; return rc; }
  *plan = p;
  return SQ_OK;
}

extern "C" int sq_gemm_fp8_plan_destroy(sq_gemm_fp8_plan* plan) {
  delete plan;
  return SQ_OK;
}

extern "C" int sq_gemm_fp8_plan_info(sq_gemm_fp8_plan* plan, int* nwg, int* split, int* stages) {
  SQ_CHECK_ARG(plan && nwg && split && stages, "sq_gemm_fp8_plan_info: null pointer");
  *nwg = plan->nwg; *split = plan->split;
  *stages = plan->nwg == 2 ? Smem<128, 2>::STAGES : Smem<128, 3>::STAGES;
  return SQ_OK;
}

template <int R, int NWG, int SPLIT>
static int launch_fp8(sq_gemm_fp8_plan* p, const Args& g, cudaStream_t st) {
  constexpr int smem = Smem<R, NWG>::TOTAL + 1024;
  static_assert(smem <= 227 * 1024, "shared memory budget");
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(gemm_fp8_kernel<R, NWG, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { set_error("sq_gemm_fp8: smem attr: %s", cudaGetErrorString(e)); return SQ_ERR_CUDA; }
    attr = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((p->N / 64 + NWG - 1) / NWG, SPLIT, 1);
  cfg.blockDim = dim3(128 * (NWG + 1));
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = 1;
  at[0].val.clusterDim.y = SPLIT;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  if (pdl_enabled()) {
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.numAttrs = 2;
  }
  cudaError_t e = cudaLaunchKernelEx(&cfg, gemm_fp8_kernel<R, NWG, SPLIT>, p->tm_a, g);
  if (e != cudaSuccess) { set_error("sq_gemm_fp8: launch failed: %s", cudaGetErrorString(e)); return SQ_ERR_CUDA; }
  SQ_CHECK_LAUNCH("sq_gemm_fp8");
  return SQ_OK;
}

template <int R>
static int run_tile(sq_gemm_fp8_plan* p, const Args& g, cudaStream_t st) {
  const int w = p->nwg, s = p->split;
#define SQ_F8(NWG_, SP_) if (w == NWG_ && s == SP_) return launch_fp8<R, NWG_, SP_>(p, g, st)
  SQ_F8(2, 1); SQ_F8(2, 2); SQ_F8(2, 3); SQ_F8(2, 4);
  SQ_F8(3, 1); SQ_F8(3, 2); SQ_F8(3, 3); SQ_F8(3, 4);
#undef SQ_F8
  set_error("sq_gemm_fp8_run: no kernel for nwg=%d split=%d", w, s);
  return SQ_ERR_UNSUPPORTED;
}

/* rows [a_row0, a_row0 + n) of the plan's activation buffer -> rows [0, n) of `c` (pitch ldc halfs; NULL = the plan's own
 * output buffer, rows [a_row0, ...)).  More than 128 rows: one launch per 128-row tile; a tile of at most 64 rows runs
 * the R = 64 instance. */
extern "C" int sq_gemm_fp8_run_at(sq_gemm_fp8_plan* plan, int n, int a_row0, sq_half* c, int ldc, void* stream) {
  SQ_CHECK_ARG(plan != nullptr, "sq_gemm_fp8_run: null plan");
  SQ_CHECK_ARG(n >= 0 && a_row0 >= 0 && a_row0 + n <= plan->n_max, "sq_gemm_fp8_run: rows [%d, %d) exceed the plan's n_max=%d",
               a_row0, a_row0 + n, plan->n_max);
  SQ_CHECK_ARG(c == nullptr || (ldc >= plan->N && ldc % 8 == 0 && ((uintptr_t)c % 16) == 0),
               "sq_gemm_fp8_run: output override must be 16 B aligned, pitch >= N and %% 8");
  for (int m0 = 0; m0 < n; m0 += 128) {
    Args g;
    g.w = plan->w; g.scale = plan->scale;
    g.n = n - m0 < 128 ? n - m0 : 128; g.N = plan->N; g.KB = plan->K / 64;
    g.m0 = a_row0 + m0;
    if (c) { g.ldc = ldc; g.c = (__half*)c - (int64_t)a_row0 * ldc; }
    else { g.ldc = plan->ldc; g.c = plan->c; }
    g.err_flag = plan->err_flag;
    const int rc = g.n <= 64 ? run_tile<64>(plan, g, (cudaStream_t)stream) : run_tile<128>(plan, g, (cudaStream_t)stream);
    if (rc != SQ_OK) return rc;
  }
  return SQ_OK;
}
