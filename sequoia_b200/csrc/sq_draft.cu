// Tree-masked attention for the small draft model's forwards of <= 64 rows (the reference's draft SDPA,
// Engine/Llama_modules.py:127-134, inside the per-level graph replay of Engine/Engine.py:158-164).
//
// A JackFram-68m-class draft (head_dim 64, no GQA) runs each tree level as a forward of a few dozen rows against a prefix
// of at most max_length keys.  At that size the wgmma tree attention's 128-row tiles are mostly padding, so this kernel
// takes one (head, 16-row tile) per CTA: the head's whole K and V are staged into shared memory with cp.async, the 8
// warps take 32-key blocks round-robin (mma.sync m16n8k16, fp16 in, fp32 accumulate, online softmax per warp), and the
// per-warp (max, sum, O) partials are combined through shared memory in warp order (deterministic).  Rounding points:
// P rounds to fp16 as the A operand of PV, the output rounds to fp16 once.  The shared-memory footprint bounds max_length
// (640 for head_dim 64, see sq_draft_supported).
#include "sq_common.cuh"
#include "sq_mask.cuh"

namespace sq {

constexpr int DT = 256;            // threads per CTA (8 warps)
constexpr int DPAD = 8;            // shared-memory row padding (halfs): conflict-free ldmatrix
constexpr int D_ROWS = 64;         // max rows per launch
constexpr int HD = 64;             // head dim

struct DraftAttnArgs {
  int h, H, M, n, n0, kv_end;
  float scale;
  const __half *k_cache, *v_cache;   // this layer's (H, M, 64) planes
  const __half* qkv;                 // (n, 3h): q part read
  __half* attn;                      // (n, h)
  const int32_t* state;
  const uint32_t* tree_bits;
  int tree_words, tree_size;
};

// dynamic shared memory: K_s, V_s [kv_pad][72] | Q_s [16][72] halfs | O partials [8][16][64] | max, sum [8][16] floats
static size_t draft_attn_smem(int max_length) {
  return (size_t)(2 * ((max_length + 31) & ~31) + 16) * (HD + DPAD) * 2 + (8 * 16 * 64 + 2 * 8 * 16) * 4;
}

__device__ __forceinline__ uint32_t s_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp16(void* smem, const void* g) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s_u32(smem)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm4t(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// Item = (head, 16-row tile); CTAs stride over the items.  Row r is tree-relative slot base + n0 + r (base = P - 1); keys
// [0, base + kv_end) are visible under the structured tree mask.
__global__ void __launch_bounds__(DT, 1) draft_attention_kernel(const DraftAttnArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  pdl_trigger();
  pdl_wait();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const int h = a.h, n = a.n;
  const int MT = (n + 15) / 16;
  const int P = a.state[ST_P];
  const int base = P - 1;
  const int kv_len = base + a.kv_end;
  const int nblk = gridDim.x, bid = blockIdx.x;
  const int items = a.H * MT;
  const int ldk = HD + DPAD;                                       // 72 halfs
  __half* Ks = reinterpret_cast<__half*>(smem_raw);
  const int kv_pad = (kv_len + 31) & ~31;
  __half* Vs = Ks + (size_t)kv_pad * ldk;
  __half* Qs = Vs + (size_t)kv_pad * ldk;
  float* sO = reinterpret_cast<float*>(Qs + 16 * ldk);             // [8][16][64]
  float* sM = sO + 8 * 16 * 64;                                    // [8][16]
  float* sL = sM + 8 * 16;
  for (int it = bid; it < items; it += nblk) {
    const int head = it / MT, mt = it % MT;
    const __half* kg = a.k_cache + (int64_t)head * a.M * HD;
    const __half* vg = a.v_cache + (int64_t)head * a.M * HD;
    for (int i = tid; i < kv_pad * 8; i += DT) {
      const int r = i >> 3, c = i & 7;
      if (r < kv_len) {
        cp16(Ks + r * ldk + c * 8, kg + (int64_t)r * HD + c * 8);
        cp16(Vs + r * ldk + c * 8, vg + (int64_t)r * HD + c * 8);
      } else {
        *reinterpret_cast<uint4*>(Ks + r * ldk + c * 8) = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4*>(Vs + r * ldk + c * 8) = make_uint4(0, 0, 0, 0);
      }
    }
    if (tid < 128) {
      const int r = tid >> 3, c = tid & 7;
      const int row = mt * 16 + r;
      uint4 v = make_uint4(0, 0, 0, 0);
      if (row < n) v = *reinterpret_cast<const uint4*>(a.qkv + (int64_t)row * (3 * h) + head * HD + c * 8);
      *reinterpret_cast<uint4*>(Qs + r * ldk + c * 8) = v;
    }
    cp_commit();
    cp_wait<0>();
    __syncthreads();
    // this thread's two rows
    const int row_lo = mt * 16 + g, row_hi = row_lo + 8;
    const RowMask rm_lo = row_mask(base + a.n0 + row_lo, P), rm_hi = row_mask(base + a.n0 + row_hi, P);
    const uint32_t* bits_lo = (rm_lo.node >= 1 && rm_lo.node < a.tree_size) ? a.tree_bits + (int64_t)rm_lo.node * a.tree_words : nullptr;
    const uint32_t* bits_hi = (rm_hi.node >= 1 && rm_hi.node < a.tree_size) ? a.tree_bits + (int64_t)rm_hi.node * a.tree_words : nullptr;
    RowMask rl = rm_lo, rh = rm_hi;
    if (bits_lo == nullptr) rl.node = -1;
    if (bits_hi == nullptr) rh.node = -1;
    uint32_t qa[4][4];
    {
      const uint32_t q_addr = s_u32(Qs) + ((lane & 15) * ldk) * 2 + (lane >> 4) * 16;
#pragma unroll
      for (int s = 0; s < 4; ++s) ldsm4(qa[s], q_addr + s * 32);
    }
    float m[2] = {-INFINITY, -INFINITY}, lsum[2] = {0.f, 0.f};
    float o[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f; }
    const float sc = a.scale * 1.4426950408889634f;
    for (int kb = warp; kb * 32 < kv_len; kb += 8) {
      const int c0 = kb * 32;
      float s[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; }
      const uint32_t k_addr = s_u32(Ks) + ((c0 + (lane & 7) + (lane >> 4) * 8) * ldk) * 2 + ((lane >> 3) & 1) * 16;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int jp = 0; jp < 2; ++jp) {
          uint32_t b[4];
          ldsm4(b, k_addr + (jp * 16 * ldk) * 2 + ks * 32);
          mma16816(s[jp * 2], qa[ks], b[0], b[1]);
          mma16816(s[jp * 2 + 1], qa[ks], b[2], b[3]);
        }
      }
      const uint32_t vl = vis_word(rl, c0, P, kv_len, bits_lo, a.tree_words);
      const uint32_t vh = vis_word(rh, c0, P, kv_len, bits_hi, a.tree_words);
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = j * 8 + t4 * 2 + e;
          s[j][e] = ((vl >> c) & 1u) ? s[j][e] * sc : -INFINITY;
          s[j][2 + e] = ((vh >> c) & 1u) ? s[j][2 + e] * sc : -INFINITY;
          mx[0] = fmaxf(mx[0], s[j][e]);
          mx[1] = fmaxf(mx[1], s[j][2 + e]);
        }
#pragma unroll
      for (int r2 = 0; r2 < 2; ++r2) {
        mx[r2] = fmaxf(mx[r2], __shfl_xor_sync(0xffffffffu, mx[r2], 1));
        mx[r2] = fmaxf(mx[r2], __shfl_xor_sync(0xffffffffu, mx[r2], 2));
      }
      float alpha[2], mref[2];
#pragma unroll
      for (int r2 = 0; r2 < 2; ++r2) {
        const float mn = fmaxf(m[r2], mx[r2]);
        alpha[r2] = (m[r2] == -INFINITY) ? 0.f : exp2f(m[r2] - mn);
        m[r2] = mn;
        mref[r2] = (mn == -INFINITY) ? 0.f : mn;
        lsum[r2] *= alpha[r2];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) { o[j][0] *= alpha[0]; o[j][1] *= alpha[0]; o[j][2] *= alpha[1]; o[j][3] *= alpha[1]; }
      uint32_t pa[2][4];                               // P as the A operand of two 16-key k-steps
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float p0 = exp2f(s[j][0] - mref[0]), p1 = exp2f(s[j][1] - mref[0]);
        const float p2 = exp2f(s[j][2] - mref[1]), p3 = exp2f(s[j][3] - mref[1]);
        lsum[0] += p0 + p1;
        lsum[1] += p2 + p3;
        pa[j >> 1][(j & 1) * 2] = pack_h2(p0, p1);     // a0 / a2: row g
        pa[j >> 1][(j & 1) * 2 + 1] = pack_h2(p2, p3); // a1 / a3: row g+8
      }
      // O += P V : V_s is [key][dim] -> transposed ldmatrix gives the (k = key, n = dim) B fragments
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        const uint32_t v_addr = s_u32(Vs) + ((c0 + ks * 16 + (lane & 15)) * ldk) * 2 + (lane >> 4) * 16;
#pragma unroll
        for (int jp = 0; jp < 4; ++jp) {
          uint32_t b[4];
          ldsm4t(b, v_addr + jp * 32);
          mma16816(o[jp * 2], pa[ks], b[0], b[1]);
          mma16816(o[jp * 2 + 1], pa[ks], b[2], b[3]);
        }
      }
    }
#pragma unroll
    for (int r2 = 0; r2 < 2; ++r2) {
      lsum[r2] += __shfl_xor_sync(0xffffffffu, lsum[r2], 1);
      lsum[r2] += __shfl_xor_sync(0xffffffffu, lsum[r2], 2);
    }
    if (t4 == 0) {
      sM[warp * 16 + g] = m[0]; sM[warp * 16 + g + 8] = m[1];
      sL[warp * 16 + g] = lsum[0]; sL[warp * 16 + g + 8] = lsum[1];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float* d0 = sO + ((warp * 16 + g) * 64) + j * 8 + t4 * 2;
      d0[0] = o[j][0]; d0[1] = o[j][1];
      d0[8 * 64] = o[j][2]; d0[8 * 64 + 1] = o[j][3];
    }
    __syncthreads();
    {
      const int r = tid >> 4, d0 = (tid & 15) * 4;
      float mm = -INFINITY;
#pragma unroll
      for (int w = 0; w < 8; ++w) mm = fmaxf(mm, sM[w * 16 + r]);
      float den = 0.f, acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        const float mw = sM[w * 16 + r];
        if (mw == -INFINITY) continue;
        const float f = exp2f(mw - mm);
        den += f * sL[w * 16 + r];
        const float4 ov = *reinterpret_cast<const float4*>(sO + (w * 16 + r) * 64 + d0);
        acc[0] += f * ov.x; acc[1] += f * ov.y; acc[2] += f * ov.z; acc[3] += f * ov.w;
      }
      const float inv = den > 0.f ? 1.f / den : 0.f;
      const int row = mt * 16 + r;
      if (row < n) {
        uint2 pk;
        pk.x = pack_h2(acc[0] * inv, acc[1] * inv);
        pk.y = pack_h2(acc[2] * inv, acc[3] * inv);
        *reinterpret_cast<uint2*>(a.attn + (int64_t)row * h + head * HD + d0) = pk;
      }
    }
    __syncthreads();
  }
}

}  // namespace sq

using namespace sq;

struct sq_draft_plan {
  int h, L, H, M;
  const __half *k_cache, *v_cache;     // (L, 1, H, M, 64)
  int n_sm, smem;
};

/* 1 if the draft attention supports a model of these shapes (else the draft forward uses sq_tree_attn). */
extern "C" int sq_draft_supported(int hidden, int n_heads, int n_kv_heads, int head_dim, int max_length) {
  return head_dim == HD && n_heads == n_kv_heads && n_heads * HD == hidden && max_length >= 1 &&
         draft_attn_smem(max_length) <= 220 * 1024;
}

extern "C" int sq_draft_plan_create(sq_draft_plan** plan, int hidden, int n_layers, int n_heads, int max_length,
                                    sq_half* k_cache, sq_half* v_cache) {
  SQ_CHECK_ARG(plan && k_cache && v_cache, "sq_draft_plan_create: null pointer");
  SQ_CHECK_ARG(n_layers >= 1 && sq_draft_supported(hidden, n_heads, n_heads, HD, max_length),
               "sq_draft_plan_create: unsupported model shape (hidden %d, layers %d, heads %d, M %d)", hidden, n_layers,
               n_heads, max_length);
  sq_draft_plan* p = new sq_draft_plan();
  p->h = hidden; p->L = n_layers; p->H = n_heads; p->M = max_length;
  p->k_cache = (const __half*)k_cache; p->v_cache = (const __half*)v_cache;
  p->smem = (int)draft_attn_smem(max_length);
  int dev = 0;
  cudaGetDevice(&dev);
  if (cudaDeviceGetAttribute(&p->n_sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || p->n_sm <= 0) p->n_sm = 132;
  cudaError_t e = cudaFuncSetAttribute(draft_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, p->smem);
  if (e != cudaSuccess) { set_error("sq_draft_plan_create: smem attr: %s", cudaGetErrorString(e)); delete p; return SQ_ERR_CUDA; }
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, draft_attention_kernel, DT, p->smem);
  if (e != cudaSuccess || occ < 1) { set_error("sq_draft_plan_create: kernel does not fit an SM"); delete p; return SQ_ERR_CUDA; }
  *plan = p;
  return SQ_OK;
}

extern "C" int sq_draft_plan_destroy(sq_draft_plan* plan) {
  delete plan;
  return SQ_OK;
}

/* Attention of layer `layer` for `n` (<= 64) rows = tree nodes [n0, n0+n) in tree-relative addressing (base = state[P]-1),
 * on caller-owned buffers: q rows in `qkv` (n, 3*hidden; q part read), output to `attn_out` (n, hidden).  K/V come from
 * the plan's caches (the rows of this forward must already be appended); keys [0, base+kv_end) are visible under the
 * packed tree mask.  A small-shape alternative to sq_tree_attn for the draft model's forwards. */
extern "C" int sq_draft_attention(sq_draft_plan* plan, int layer, int n, const sq_half* qkv, sq_half* attn_out,
                                  const int32_t* state, int n0, int kv_end, const uint32_t* tree_bits, int tree_words,
                                  int tree_size, void* stream) {
  SQ_CHECK_ARG(plan != nullptr && state != nullptr && qkv && attn_out, "sq_draft_attention: null argument");
  SQ_CHECK_ARG(n >= 1 && n <= D_ROWS && layer >= 0 && layer < plan->L, "sq_draft_attention: n=%d / layer=%d out of range", n, layer);
  SQ_CHECK_ARG(tree_words <= 32, "sq_draft_attention: tree_size > 1024 unsupported");
  DraftAttnArgs a;
  a.h = plan->h; a.H = plan->H; a.M = plan->M; a.n = n; a.n0 = n0; a.kv_end = kv_end;
  a.scale = 1.0f / sqrtf((float)HD);
  a.k_cache = plan->k_cache + (int64_t)layer * plan->H * plan->M * HD;
  a.v_cache = plan->v_cache + (int64_t)layer * plan->H * plan->M * HD;
  a.qkv = (const __half*)qkv; a.attn = (__half*)attn_out; a.state = state;
  a.tree_bits = tree_bits; a.tree_words = tree_bits ? tree_words : 0; a.tree_size = tree_bits ? tree_size : 0;
  int grid = a.H * ((n + 15) / 16);
  if (grid > plan->n_sm) grid = plan->n_sm;
  cudaError_t e = launch_k(draft_attention_kernel, dim3(grid), dim3(DT), (size_t)plan->smem, (cudaStream_t)stream, a);
  if (e != cudaSuccess) { set_error("sq_draft_attention: launch failed: %s", cudaGetErrorString(e)); return SQ_ERR_CUDA; }
  SQ_CHECK_LAUNCH("sq_draft_attention");
  return SQ_OK;
}
