// Tree-masked attention for the draft (Engine/Llama_modules.py:127-134) and target / verify
// (Engine/Llama_modules.py:220-248) forwards.
//
// Product kernel (impl 0): see the comment above tree_attn_tc_kernel -- TMA-staged Q/K/V tiles (SWIZZLE_128B) straight from
// the fused qkv activation and the static (L,1,Hkv,M,D) caches, S = Q K^T and O = P V on wgmma with accumulators in
// registers (P stays in registers as the A operand of the second MMA), the tree-causal mask as packed ancestor bits +
// the device-resident prefix length (a dense additive fp16 mask, the reference API, is supported too), flash-style loop
// over KV tiles inside a CTA, GQA heads packed into the MMA M dimension, optional split-KV over a thread-block cluster.
// Any max_length (the KV loop has no tile limit); trees up to 1024 nodes (32 mask words per row).
// Roofline: HBM-bound for configs 2/3 (bytes = 2*D*2*(Hkv*kv + H*q) per layer), tensor-pipe-bound for config 4.
//
// impl 1 is a plain SIMT kernel used by the tests as an on-device cross-check of the tensor-core path.
#include <cooperative_groups.h>
#include <cuda.h>

#include <cstdio>
#include <cstdlib>

#include "sq_common.cuh"
#include "sq_ptx.cuh"
#include "sq_mask.cuh"

struct sq_attn_plan {
  const __half* q;
  int ld, n_max, H, Hkv, D, L, M;
  int B;          // sequences in the cache: (L, B, Hkv, M, D)
  const __half* k_cache;
  const __half* v_cache;
  __half* out;
  int splits_max;
  int splits_force;   // SQ_ATTN_SPLITS (tuning / tests): KV splits per cluster instead of the SM-count heuristic; 0 = off
  int last_splits;    // KV splits (Z) of the last tensor-core launch
  int GP;         // query heads packed into one MMA tile (H/Hkv when that divides 128, else 1)
  int pdl;        // launch with programmatic stream serialization (SQ_PDL=1)
  int debug_flags;
  int* err_flag;  // device word set by a watchdog timeout
  long long* dbg; // phase timestamps (SQ_ATTN_TIMING=1)
  CUtensorMap tm_q, tm_k, tm_v;
};

namespace sq {

constexpr int TILE_Q = 128;
constexpr int TILE_KV = 128;
constexpr float LOG2E = 1.4426950408889634f;

struct AttnArgs {
  const __half* q;
  int ld;
  const __half* k_layer;   // (Hkv, M, D) of this layer
  const __half* v_layer;
  __half* out;
  int n, H, Hkv, M, GP;
  int B;                   // sequences of a batched launch (rows of sequence b start at b*n; grid.y = B * q tiles)
  int layer;
  const int32_t* state;
  int n0, kv_end, prefix_len_host;
  const __half* dense_mask;
  int64_t mask_ld;
  const uint32_t* tree_bits;
  int tree_words, tree_size;
  float scale;
  int debug_flags;
  int* err_flag;
  long long* dbg;          // optional phase timestamps (SQ_ATTN_TIMING=1): [split][16] clock64 values of CTA (0,0,split)
};

// ------------------------------------------------------------------------------------------------------------------
// impl 1: SIMT cross-check kernel.  grid (n, H), 128 threads; warp w takes keys w, w+4, ...
template <int D>
__global__ void __launch_bounds__(128) tree_attn_simt_kernel(AttnArgs a) {
  constexpr int DPL = D / 32;
  __shared__ float sh_m[4], sh_l[4];
  __shared__ float sh_acc[4][D];
  const int r = blockIdx.x, h = blockIdx.y;
  const int hkv = h / (a.H / a.Hkv);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int P = a.state ? a.state[ST_P] : a.prefix_len_host;
  const int base = (a.state ? (P - 1) : 0);
  const int slot = base + a.n0 + r;
  const int kv_len = base + a.kv_end;
  const RowMask rm = row_mask(slot, P);
  const uint32_t* bits = (rm.node >= 0 && a.tree_bits) ? a.tree_bits + (int64_t)rm.node * a.tree_words : nullptr;
  float qv[DPL], acc[DPL];
#pragma unroll
  for (int i = 0; i < DPL; ++i) {
    qv[i] = h2f(a.q[(int64_t)r * a.ld + h * D + lane * DPL + i]);
    acc[i] = 0.f;
  }
  float m = -INFINITY, l = 0.f;
  const __half* kbase = a.k_layer + (int64_t)hkv * a.M * D;
  const __half* vbase = a.v_layer + (int64_t)hkv * a.M * D;
  for (int c = warp; c < kv_len; c += 4) {
    float madd = 0.f;
    if (a.dense_mask) {
      madd = h2f(a.dense_mask[(int64_t)r * a.mask_ld + c]);
    } else {
      bool vis = c <= rm.lim;
      if (!vis && bits != nullptr && c >= P - 1) {
        const int j = c - (P - 1);
        vis = (j < a.tree_size) && ((bits[j >> 5] >> (j & 31)) & 1u);
      }
      if (!vis) continue;
    }
    float d = 0.f;
#pragma unroll
    for (int i = 0; i < DPL; ++i) d += qv[i] * h2f(kbase[(int64_t)c * D + lane * DPL + i]);
    d = warp_sum(d) * a.scale + madd;
    const float mn = fmaxf(m, d);
    const float corr = (m == -INFINITY) ? 0.f : expf(m - mn);
    const float p = expf(d - mn);
    l = l * corr + p;
#pragma unroll
    for (int i = 0; i < DPL; ++i) acc[i] = acc[i] * corr + p * h2f(vbase[(int64_t)c * D + lane * DPL + i]);
    m = mn;
  }
  if (lane == 0) { sh_m[warp] = m; sh_l[warp] = l; }
#pragma unroll
  for (int i = 0; i < DPL; ++i) sh_acc[warp][lane * DPL + i] = acc[i];
  __syncthreads();
  if (threadIdx.x < D) {
    float mm = fmaxf(fmaxf(sh_m[0], sh_m[1]), fmaxf(sh_m[2], sh_m[3]));
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      if (sh_m[w] == -INFINITY) continue;
      const float f = expf(sh_m[w] - mm);
      num += f * sh_acc[w][threadIdx.x];
      den += f * sh_l[w];
    }
    a.out[(int64_t)r * (a.H * D) + h * D + threadIdx.x] = f2h(den > 0.f ? num / den : 0.f);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// impl 0: the tensor-core kernel.
//
// Work decomposition.  G = H / Hkv query heads share one KV head (Engine/Llama_modules.py:223-224 repeat_kv).  The 128
// rows of one MMA tile are "packed" (query row, head-in-group) pairs: tile row i = (q row q0 + i / GP, head grp*GP + i % GP)
// with GP = G when G divides 128 (1 for Llama-2-7B/13B, 8 for 70B), so that ONE staged K/V tile serves all GP heads.  The
// Q tile comes in as a 3-D TMA box (64, GP, 128/GP) of the fused qkv activation -- its shared-memory image is exactly
// the packed 128-row K-major tile.  Grid (head groups, packed q tiles, Z) launched as clusters (1,1,Z): the Z CTAs of a
// cluster split the ACTIVE KV tiles of one (group, q tile) into contiguous chunks; each CTA loops over its chunk
// flash-attention style (2-stage TMA ring for K and for V; S = Q K^T by wgmma from shared memory into registers, P
// converted in registers to the fp16 A fragments of O += P V, O accumulated in registers across tiles with LAZY
// rescaling: the running maximum used in the exponent only moves when it grows by more than 2^8, so O is rarely touched).
// Z > 1: partial rows (normalised fp16 O_s / l_s, log2-domain reference max, sum) are pushed into the shared memory of
// the row's owner CTA (st.shared::cluster), one cluster barrier, owners combine and store.  No global workspace.
template <int D>
struct TcSmem {
  static constexpr int HALVES = D / 64;                 // 64-element (128 B) column halves
  static constexpr int TILE_BYTES = HALVES * 128 * 128; // one 128-row tile
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = TILE_BYTES;              // 2 stages
  static constexpr int OFF_V = 3 * TILE_BYTES;          // 2 stages
  static constexpr int OFF_MASK = 5 * TILE_BYTES;       // (128/GP) x tree_words u32 ancestor bits of this q tile
  static constexpr int MASK_BYTES = 128 * 32 * 4;
  static constexpr int OFF_BAR = OFF_MASK + MASK_BYTES;  // bar_q, bar_k[2], bar_v[2]
  // Split-KV reduction buffers, written REMOTELY by the peer CTAs of the cluster (push model), so they may not alias
  // anything live during the KV loop: row r of the tile is owned by CTA (r % Z); slot [src split][r / Z].
  static constexpr int O_STRIDE = D + 8;                // halfs: partial rows travel as NORMALISED fp16 (O_s / l_s)
  static constexpr int R_ROWS = 128 + 8;                // Z * ceil(128 / Z) <= 136 for Z <= 8
  static constexpr int OFF_RML = OFF_BAR + 128;         // [owned row][8 splits] float2 (log2-domain max, sum)
  static constexpr int OFF_R = OFF_RML + 128 * 8 * 8;   // R_ROWS x O_STRIDE halfs
  static constexpr int TOTAL = OFF_R + R_ROWS * O_STRIDE * 2;
};

#define SQ_STAMP(k) do { if (a.dbg && tid == 0 && blockIdx.x == 0 && blockIdx.y == 0) a.dbg[split * 16 + (k)] = clock64(); } while (0)

__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_smem_addr, uint32_t cta_rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(cta_rank));
  return r;
}
__device__ __forceinline__ void st_cluster_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared::cluster.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void st_cluster_v2(uint32_t addr, float a, float b) {
  asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
constexpr float RESCALE_THRESHOLD = 8.0f;   // log2 units: P stays <= 2^8 under a stale reference maximum

// 256 threads = 2 warpgroups; warpgroup g owns tile rows [64 g, 64 g + 64): S, P and O of those rows live in its registers
// in the wgmma accumulator layout -- thread holds rows r0 = 64 g + 16 (warp % 4) + lane / 4 and r0 + 8, and of every
// 64-column chunk the columns 8 j + 2 (lane % 4) + {0, 1}: element [4 j + 2 h + e] is (row r0 + 8 h, column 8 j + 2 q + e).
// BATCH (structured mask only): grid.y = B * q tiles, sequence b = blockIdx.y / q tiles reads its own state row, its Q rows
// and writes its output rows at offset b*n, and reads cache heads (layer*B + b)*Hkv + h.
// RAGGED (structured mask only): grid.y = the q tiles of all parts; the CTA's part j is found from the q-tile prefix
// sums, n / n0 / kv_end are part j's, its Q rows and output rows start at row0_j, and it reads cache heads
// (layer*B + seq)*Hkv + h.
// The Q box of a part's last tile may cover the next part's rows: those rows are never written.
template <int D, bool DENSE, bool BATCH, bool RAGGED = false>
__global__ void __launch_bounds__(256, 1)
    tree_attn_tc_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                        const __grid_constant__ CUtensorMap tm_v, AttnArgs a,
                        const __grid_constant__ RaggedArg<RAGGED> rp) {
  using SM = TcSmem<D>;
  constexpr int DC = D / 64;                     // 64-column chunks of O
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // dynamic smem base is only guaranteed 16 B aligned: re-align to 1024 B for SWIZZLE_128B (same offset in every CTA)
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  constexpr bool SEQ = BATCH || RAGGED;          // per-sequence state row and cache planes
  const RaggedParts* R = ragged_ptr(rp);
  const int pj = RAGGED ? ragged_part(R->tile0, R->n_parts, blockIdx.y) : 0;   // RAGGED: this CTA's part
#define SQ_PART(f) (RAGGED ? R->f[pj] : a.f)
  const int q_tiles = BATCH ? (int)gridDim.y / a.B : (int)gridDim.y;
  const int b = RAGGED ? R->seq[pj] : BATCH ? (int)blockIdx.y / q_tiles : 0;
  const int grp = blockIdx.x, split = blockIdx.z, Z = gridDim.z;
  const int qt = RAGGED ? (int)blockIdx.y - R->tile0[pj] : BATCH ? (int)blockIdx.y % q_tiles : (int)blockIdx.y;
  const int32_t* state = SEQ ? a.state + b * ST_WORDS : a.state;
  __half* out = RAGGED  ? a.out + (int64_t)R->row0[pj] * (a.H * D)
                : BATCH ? a.out + (int64_t)b * a.n * (a.H * D) : a.out;
  const int GP = a.GP, RPT = TILE_Q / GP;        // heads per tile, query rows per tile
  const int hkv = (grp * GP) / (a.H / a.Hkv);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's tile rows: r0, r0 + 8
  const int q2 = 2 * (lane & 3);
  const int q0 = qt * RPT;
  const uint32_t sQ = ptx::smem_u32(smem + SM::OFF_Q), sK = ptx::smem_u32(smem + SM::OFF_K),
                 sV = ptx::smem_u32(smem + SM::OFF_V);
  const uint32_t bar_q = ptx::smem_u32(smem + SM::OFF_BAR), bar_k = bar_q + 8, bar_v = bar_q + 24;
  const uint32_t sR_local = ptx::smem_u32(smem + SM::OFF_R), sRML_local = ptx::smem_u32(smem + SM::OFF_RML);
  const int rpc = (TILE_Q + Z - 1) / Z;          // rows owned per CTA

  // ---- prologue that does not depend on earlier kernels (overlaps their tail under programmatic dependent launch) -----
  if (tid == 0) {
    ptx::mbar_init(bar_q, 1);
    ptx::mbar_init(bar_k, 1);
    ptx::mbar_init(bar_k + 8, 1);
    ptx::mbar_init(bar_v, 1);
    ptx::mbar_init(bar_v + 8, 1);
    ptx::fence_barrier_init();
  }
  __syncwarp();
  asm volatile("griddepcontrol.wait;" ::: "memory");      // q / k / v / state of this launch are now visible
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // Everything that does not need the device-resident prefix length goes first, so that the state load, the Q tile and
  // the ancestor-bit loads are all in flight together: under tree-relative addressing the node id of a row is
  // n0 + q0 + r, independent of P.
  if (tid == 0) {
    ptx::mbar_expect_tx(bar_q, SM::TILE_BYTES);
#pragma unroll
    for (int hh = 0; hh < SM::HALVES; ++hh)
      ptx::tma_load_3d(sQ + hh * 16384, &tm_q, bar_q, hh * 64, grp * GP, RAGGED ? R->row0[pj] + q0 : b * a.n + q0);
  }
  uint32_t* sbits = reinterpret_cast<uint32_t*>(smem + SM::OFF_MASK);
  if (!DENSE && a.tree_words > 0 && tid < RPT) {
    const int node = state ? (SQ_PART(n0) + q0 + tid) : (a.n0 + q0 + tid - (a.prefix_len_host - 1));
    const bool has = node >= 1 && node < a.tree_size;
#pragma unroll 4
    for (int w = 0; w < a.tree_words; ++w)
      sbits[tid * a.tree_words + w] = has ? a.tree_bits[(int64_t)node * a.tree_words + w] : 0u;
  }
  const int P = state ? state[ST_P] : a.prefix_len_host;
  const int base = state ? (P - 1) : 0;
  const int kv_len = base + SQ_PART(kv_end);
  // active KV tiles of this q tile (tiles wholly beyond what its last row may see are never touched), split in chunks
  int T;
  {
    const int last_slot = base + SQ_PART(n0) + min(q0 + RPT, SQ_PART(n)) - 1;
    const int max_vis = DENSE ? (kv_len - 1) : ((last_slot >= P) ? (kv_len - 1) : min(last_slot, P - 1));
    T = min((kv_len + TILE_KV - 1) / TILE_KV, max_vis / TILE_KV + 1);
  }
  const int tps = (T + Z - 1) / Z;               // tiles per split
  const int nsplit = (T + tps - 1) / tps;        // splits that own at least one tile
  const int t_begin = split * tps;
  const int NT = max(0, min(T, t_begin + tps) - t_begin);
  const int kvrow = (SEQ ? a.layer * a.B + b : a.layer) * a.Hkv + hkv;
  SQ_STAMP(0);

  if (NT > 0) {
    if (tid == 0) {
#pragma unroll 1
      for (int t = 0; t < 2 && t < NT; ++t) {
        ptx::mbar_expect_tx(bar_k + 8 * t, SM::TILE_BYTES);
        ptx::mbar_expect_tx(bar_v + 8 * t, SM::TILE_BYTES);
#pragma unroll
        for (int hh = 0; hh < SM::HALVES; ++hh) {
          ptx::tma_load_3d(sK + t * SM::TILE_BYTES + hh * 16384, &tm_k, bar_k + 8 * t, hh * 64, (t_begin + t) * TILE_KV, kvrow);
          ptx::tma_load_3d(sV + t * SM::TILE_BYTES + hh * 16384, &tm_v, bar_v + 8 * t, hh * 64, (t_begin + t) * TILE_KV, kvrow);
        }
      }
    }
    RowMask rm[2];
    const uint32_t* my_bits[2];
    bool row_ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int qr = (r0 + 8 * h) / GP;          // query row inside the tile
      rm[h] = row_mask(base + SQ_PART(n0) + q0 + qr, P);
      my_bits[h] = sbits + qr * a.tree_words;
      row_ok[h] = (q0 + qr) < SQ_PART(n);
    }
    __syncthreads();                             // ancestor bits staged, barriers initialised
    SQ_STAMP(1);
    ptx::mbar_wait(bar_q, 0, a.err_flag, 1);
    const float sc = a.scale * LOG2E;            // work in the log2 domain
    float o[DC][32];
#pragma unroll
    for (int c = 0; c < DC; ++c)
#pragma unroll
      for (int e = 0; e < 32; ++e) o[c][e] = 0.f;
    float m_used[2] = {-INFINITY, -INFINITY};    // reference maximum in the exponent (log2 domain), lazily updated
    float lsum[2] = {0.f, 0.f};                  // this thread's share (its columns) of the row sums

#pragma unroll 1
    for (int j = 0; j < NT; ++j) {
      const int st = j & 1;
      const uint32_t par = (uint32_t)((j >> 1) & 1);
      const int kv0 = (t_begin + j) * TILE_KV;
      // ---- S_j = Q K_j^T: two 64-key chunks ---------------------------------------------------------------------------
      float s[2][32];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 32; ++e) s[hh][e] = 0.f;
      ptx::mbar_wait(bar_k + 8 * st, par, a.err_flag, 2);
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < D / 16; ++k) {
        const uint32_t off = (k / 4) * 16384 + (k % 4) * 32;        // 4 k-steps per 128 B swizzle atom
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
          ptx::wgmma_ss<0>(s[hh], gmma_desc(sQ + wg * 8192 + off, 16, 1024),
                           gmma_desc(sK + st * SM::TILE_BYTES + hh * 8192 + off, 16, 1024), 1);
      }
      ptx::wgmma_commit();
      // visibility words of the 128 keys of this tile for both rows, while the MMAs run
      uint32_t vis[2][4];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          const int c0 = kv0 + 32 * w;
          if (DENSE) {
            const int rem = kv_len - c0;
            vis[h][w] = rem >= 32 ? 0xFFFFFFFFu : (rem <= 0 ? 0u : ((1u << rem) - 1u));
          } else {
            vis[h][w] = vis_word(rm[h], c0, P, kv_len, my_bits[h], a.tree_words);
          }
        }
      ptx::wgmma_wait_all();
      if (j == 0) SQ_STAMP(2);
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = hh * 64 + jj * 8 + q2 + e;             // key column inside the tile
              const bool v = (vis[h][col >> 5] >> (col & 31)) & 1u;
              float t = v ? s[hh][4 * jj + 2 * h + e] * sc : -INFINITY;
              if (DENSE && v && row_ok[h])         // additive fp16 mask (reference API), straight from global memory
                t += h2f(a.dense_mask[(int64_t)(q0 + (r0 + 8 * h) / GP) * a.mask_ld + kv0 + col]) * LOG2E;
              s[hh][4 * jj + 2 * h + e] = t;
              mx[h] = fmaxf(mx[h], t);
            }
      uint32_t pf[TILE_KV / 16][4];              // P_j as the fp16 A fragments of the second MMA (16 keys each)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float m_tile = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));   // the 4 threads of a row agree on it
        m_tile = fmaxf(m_tile, __shfl_xor_sync(0xffffffffu, m_tile, 2));
        // lazy rescale: move the reference maximum only when it would grow by more than 2^8
        if (m_used[h] == -INFINITY) {
          m_used[h] = m_tile;                    // nothing accumulated for this row yet
        } else if (m_tile - m_used[h] > RESCALE_THRESHOLD) {
          const float alpha = exp2f(m_used[h] - m_tile);
          m_used[h] = m_tile;
#pragma unroll
          for (int c = 0; c < DC; ++c)
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) { o[c][4 * jj + 2 * h] *= alpha; o[c][4 * jj + 2 * h + 1] *= alpha; }
          lsum[h] *= alpha;
        }
        const float mref = (m_used[h] == -INFINITY) ? 0.f : m_used[h];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const float p0 = exp2f(s[hh][4 * jj + 2 * h] - mref), p1 = exp2f(s[hh][4 * jj + 2 * h + 1] - mref);
            lsum[h] += p0 + p1;
            const __half2 hp = __floats2half2_rn(p0, p1);           // P is fp16 like the reference's attn_weights
            // keys 16 kk + [0, 8) -> registers 0 (row r0) / 1 (row r0 + 8); keys 16 kk + [8, 16) -> registers 2 / 3
            pf[hh * 4 + jj / 2][(jj & 1) * 2 + h] = *reinterpret_cast<const uint32_t*>(&hp);
          }
      }
      if (j == 0) SQ_STAMP(4);
      // ---- O (+)= P_j V_j (V: MN-major, 16 KB between the 64-wide D chunks, 1 KB per 8 keys) ---------------------------
      ptx::mbar_wait(bar_v + 8 * st, par, a.err_flag, 6);
      ptx::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < TILE_KV / 16; ++kk)
#pragma unroll
        for (int c = 0; c < DC; ++c)
          ptx::wgmma_rs<1>(o[c], pf[kk], gmma_desc(sV + st * SM::TILE_BYTES + c * 16384 + kk * 2048, 16384, 1024), 1);
      ptx::wgmma_commit();
      ptx::wgmma_wait_all();
      __syncthreads();                           // both warpgroups are done with K / V stage st: refill it with tile j + 2
      if (tid == 0 && j + 2 < NT) {
        ptx::mbar_expect_tx(bar_k + 8 * st, SM::TILE_BYTES);
        ptx::mbar_expect_tx(bar_v + 8 * st, SM::TILE_BYTES);
#pragma unroll
        for (int hh = 0; hh < SM::HALVES; ++hh) {
          ptx::tma_load_3d(sK + st * SM::TILE_BYTES + hh * 16384, &tm_k, bar_k + 8 * st, hh * 64, kv0 + 2 * TILE_KV, kvrow);
          ptx::tma_load_3d(sV + st * SM::TILE_BYTES + hh * 16384, &tm_v, bar_v + 8 * st, hh * 64, kv0 + 2 * TILE_KV, kvrow);
        }
      }
    }
    SQ_STAMP(5);

    // stage this CTA's rows, normalised by its own row sum and rounded to fp16 (|O / l| <= max|v|), row-major in the now
    // dead Q/K tiles ...
    __half* sO = reinterpret_cast<__half*>(smem);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float l = lsum[h] + __shfl_xor_sync(0xffffffffu, lsum[h], 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const float linv = l > 0.f ? 1.f / l : 0.f;
      const int trow = r0 + 8 * h;
#pragma unroll
      for (int c = 0; c < DC; ++c)
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
          *reinterpret_cast<__half2*>(sO + trow * SM::O_STRIDE + c * 64 + jj * 8 + q2) =
              __floats2half2_rn(o[c][4 * jj + 2 * h] * linv, o[c][4 * jj + 2 * h + 1] * linv);
      if (Z > 1 && (lane & 3) == 0)
        st_cluster_v2(mapa_u32(sRML_local, (uint32_t)(trow % Z)) + (uint32_t)(((trow / Z) * 8 + split) * 8), m_used[h], l);
    }
    __syncthreads();
    SQ_STAMP(10);
    constexpr int CPR = D / 8, RPW = 32 / CPR;
    const int sub = lane / CPR, cc = lane % CPR;
    if (Z == 1) {
      // single split: the staged rows are final -- coalesced copy-out (D/8 lanes move one packed row = one head's row)
#pragma unroll 4
      for (int rr = warp * RPW + sub; rr < TILE_Q; rr += 8 * RPW) {
        const int qrow = q0 + rr / GP;
        if (qrow < SQ_PART(n))
          *reinterpret_cast<uint4*>(out + (int64_t)qrow * (a.H * D) + (grp * GP + rr % GP) * D + cc * 8) =
              *reinterpret_cast<const uint4*>(sO + rr * SM::O_STRIDE + cc * 8);
      }
      SQ_STAMP(8);
      return;
    }
    // ... and push every row to the CTA that owns it: D/8 lanes move one row (16 B each, contiguous remote store)
#pragma unroll 4
    for (int rr = warp * RPW + sub; rr < TILE_Q; rr += 8 * RPW) {
      const uint4 val = *reinterpret_cast<const uint4*>(sO + rr * SM::O_STRIDE + cc * 8);
      const uint32_t dst = mapa_u32(sR_local, (uint32_t)(rr % Z)) + (uint32_t)(((split * rpc + rr / Z) * SM::O_STRIDE + cc * 8) * 2);
      st_cluster_v4(dst, val.x, val.y, val.z, val.w);
    }
    SQ_STAMP(6);
  } else {
    // no tile for this split (it pushes nothing; the owners ignore splits >= nsplit).  Still a member of the cluster.
    if (tid == 0) ptx::mbar_wait_one(bar_q, 0, a.err_flag, 8);     // the Q tile was requested before NT was known
    __syncthreads();
    if (Z == 1) {                                 // (cannot happen for n > 0: T >= 1)
      return;
    }
  }

  // ---- split-KV reduction: every CTA normalises the rows it owns, from its OWN shared memory -------------------------
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  SQ_STAMP(7);
  {
    constexpr int CPR = D / 8;
    const float2* sRML = reinterpret_cast<const float2*>(smem + SM::OFF_RML);
    const __half* sR = reinterpret_cast<const __half*>(smem + SM::OFF_R);
    float* wts = reinterpret_cast<float*>(smem + SM::OFF_MASK);       // [rpc][8] normalised split weights (mask is dead)
    // phase 1: one thread per owned row -> weight of every split: 2^(m_s - m) l_s / sum_s 2^(m_s - m) l_s
    if (tid < rpc) {
      const float4* mlp = reinterpret_cast<const float4*>(sRML + tid * 8);
      float4 q[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) q[i] = mlp[i];
      float m[8], l[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) { m[2 * i] = q[i].x; l[2 * i] = q[i].y; m[2 * i + 1] = q[i].z; l[2 * i + 1] = q[i].w; }
      float mm = -INFINITY;
#pragma unroll
      for (int sp = 0; sp < 8; ++sp) { if (sp >= nsplit) m[sp] = -INFINITY; mm = fmaxf(mm, m[sp]); }
      float f[8], den = 0.f;
#pragma unroll
      for (int sp = 0; sp < 8; ++sp) {            // partial rows arrive normalised by l_s: weight = 2^(m_s-m) * l_s / den
        f[sp] = (m[sp] == -INFINITY) ? 0.f : exp2f(m[sp] - mm) * l[sp];
        den += f[sp];
      }
      const float inv = den > 0.f ? 1.f / den : 0.f;
      float4* wp = reinterpret_cast<float4*>(wts + tid * 8);
      wp[0] = make_float4(f[0] * inv, f[1] * inv, f[2] * inv, f[3] * inv);
      wp[1] = make_float4(f[4] * inv, f[5] * inv, f[6] * inv, f[7] * inv);
    }
    __syncthreads();
    SQ_STAMP(9);
    // phase 2: flat weighted sum over (row, 8-column chunk); weights and all partial chunks are loaded up front
#pragma unroll 1
    for (int i = tid; i < rpc * CPR; i += 256) {
      const int lr = i / CPR, cc = i % CPR;
      const int rr = lr * Z + split;             // tile row owned by this CTA
      const int qrow = q0 + rr / GP;
      if (rr >= TILE_Q || qrow >= SQ_PART(n)) continue;
      const float4 w0 = *reinterpret_cast<const float4*>(wts + lr * 8), w1 = *reinterpret_cast<const float4*>(wts + lr * 8 + 4);
      const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
      Pack8 o[8];
#pragma unroll
      for (int sp = 0; sp < 8; ++sp)             // a zero weight marks a masked / inactive split whose slot was never written
        o[sp].u = (sp < Z && w[sp] != 0.f) ? *reinterpret_cast<const uint4*>(sR + (sp * rpc + lr) * SM::O_STRIDE + cc * 8)
                                           : make_uint4(0, 0, 0, 0);
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int sp = 0; sp < 8; ++sp)
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] += w[sp] * h2f(o[sp].h[e]);
      Pack8 res;
#pragma unroll
      for (int e = 0; e < 8; ++e) res.h[e] = f2h(acc[e]);
      *reinterpret_cast<uint4*>(out + (int64_t)qrow * (a.H * D) + (grp * GP + rr % GP) * D + cc * 8) = res.u;
    }
  }
  SQ_STAMP(8);
#undef SQ_PART
}

}  // namespace sq

using namespace sq;

// ------------------------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled get_encode_fn() {
  static PFN_tmapEncodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (PFN_tmapEncodeTiled)p;
  }
  return fn;
}

static int encode_map(CUtensorMap* tm, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                      const cuuint32_t* box) {
  PFN_tmapEncodeTiled fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)"); return SQ_ERR_CUDA; }
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed: %d", (int)r); return SQ_ERR_CUDA; }
  return SQ_OK;
}

extern "C" int64_t sq_attn_workspace_bytes(int n_max, int H, int D, int M) {
  (void)n_max; (void)H; (void)D; (void)M;
  return 256 + 8 * 16 * 8;   // watchdog word + optional phase timestamps (the split-KV partials live in shared memory)
}

extern "C" int sq_attn_plan_create(sq_attn_plan** plan, const sq_half* q, int ld, int n_max, int H, int Hkv, int D,
                                   const sq_half* k_cache, const sq_half* v_cache, int L, int M, sq_half* out,
                                   void* workspace, int64_t workspace_bytes) {
  return sq_attn_plan_create_batch(plan, q, ld, n_max, H, Hkv, D, k_cache, v_cache, L, 1, M, out, workspace, workspace_bytes);
}

extern "C" int sq_attn_plan_create_batch(sq_attn_plan** plan, const sq_half* q, int ld, int n_max, int H, int Hkv, int D,
                                         const sq_half* k_cache, const sq_half* v_cache, int L, int B, int M, sq_half* out,
                                         void* workspace, int64_t workspace_bytes) {
  SQ_CHECK_ARG(plan != nullptr, "sq_attn_plan_create: null plan");
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH, "sq_attn_plan_create: B=%d (1..%d)", B, SQ_MAX_BATCH);
  SQ_CHECK_ARG(D == 64 || D == 128, "sq_attn_plan_create: head_dim %d unsupported (64 or 128)", D);
  SQ_CHECK_ARG(H >= 1 && Hkv >= 1 && H % Hkv == 0 && ld % 8 == 0 && n_max >= 1 && M >= 1, "sq_attn_plan_create: bad shape");
  SQ_CHECK_ARG(workspace_bytes >= sq_attn_workspace_bytes(n_max, H, D, M), "sq_attn_plan_create: workspace too small");
  SQ_CHECK_ARG(((uintptr_t)q % 16 == 0) && ((uintptr_t)k_cache % 16 == 0) && ((uintptr_t)v_cache % 16 == 0),
               "sq_attn_plan_create: pointers must be 16 B aligned");
  sq_attn_plan* p = new sq_attn_plan();
  p->q = (const __half*)q; p->ld = ld; p->n_max = n_max; p->H = H; p->Hkv = Hkv; p->D = D; p->L = L; p->M = M; p->B = B;
  p->k_cache = (const __half*)k_cache; p->v_cache = (const __half*)v_cache; p->out = (__half*)out;
  p->splits_max = (M + TILE_KV - 1) / TILE_KV;
  {
    const int G = H / Hkv;
    p->GP = (G <= TILE_Q && TILE_Q % G == 0) ? G : 1;
    p->pdl = pdl_enabled() ? 1 : 0;
  }
  p->err_flag = (int*)workspace;
  {
    const char* tenv = getenv("SQ_ATTN_TIMING");
    p->dbg = (tenv && atoi(tenv)) ? (long long*)((char*)workspace + 256) : nullptr;
  }
  const char* dbg = getenv("SQ_ATTN_DEBUG");
  p->debug_flags = dbg ? atoi(dbg) : 0;
  {
    // "Z": replaces only the SM-count heuristic, the clamps below still apply (the GEMM's counterpart: SQ_GEMM_FORCE)
    const char* zs = getenv("SQ_ATTN_SPLITS");
    p->splits_force = zs ? atoi(zs) : 0;
  }
  cudaMemset(workspace, 0, 256 + 8 * 16 * 8);
  {
    // Q as (D, H, rows): a (64, GP, 128/GP) box lands in shared memory as the packed 128-row tile
    cuuint64_t dims[3] = {(cuuint64_t)D, (cuuint64_t)H, (cuuint64_t)n_max};
    cuuint64_t strides[2] = {(cuuint64_t)D * 2, (cuuint64_t)ld * 2};
    cuuint32_t box[3] = {64, (cuuint32_t)p->GP, (cuuint32_t)(TILE_Q / p->GP)};
    int rc = encode_map(&p->tm_q, q, 3, dims, strides, box);
    if (rc) { delete p; return rc; }
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)D, (cuuint64_t)M, (cuuint64_t)L * B * Hkv};
    cuuint64_t strides[2] = {(cuuint64_t)D * 2, (cuuint64_t)M * D * 2};
    cuuint32_t box[3] = {64, (cuuint32_t)TILE_KV, 1};
    int rc = encode_map(&p->tm_k, k_cache, 3, dims, strides, box);
    if (!rc) rc = encode_map(&p->tm_v, v_cache, 3, dims, strides, box);
    if (rc) { delete p; return rc; }
  }
  *plan = p;
  return SQ_OK;
}

extern "C" int sq_attn_plan_destroy(sq_attn_plan* plan) {
  delete plan;
  return SQ_OK;
}

extern "C" int sq_attn_plan_debug_times(sq_attn_plan* plan, long long* host_out) {
  if (!plan->dbg) return SQ_ERR_UNSUPPORTED;
  cudaMemcpy(host_out, plan->dbg, 8 * 16 * sizeof(long long), cudaMemcpyDeviceToHost);
  return SQ_OK;
}

extern "C" int sq_attn_plan_info(sq_attn_plan* plan, int* gp, int* splits) {
  SQ_CHECK_ARG(plan != nullptr && gp != nullptr && splits != nullptr, "sq_attn_plan_info: null argument");
  *gp = plan->GP;
  *splits = plan->last_splits;
  return SQ_OK;
}

extern "C" int sq_attn_plan_error(sq_attn_plan* plan) {
  int v = 0;
  cudaMemcpy(&v, plan->err_flag, sizeof(int), cudaMemcpyDeviceToHost);
  return v;
}

template <int D, bool BATCH, bool RAGGED = false>
static int launch_attn(sq_attn_plan* p, AttnArgs& a, int impl, cudaStream_t st, const RaggedArg<RAGGED>& rp = {}) {
  if (impl == 1) {
    tree_attn_simt_kernel<D><<<dim3(a.n, a.H), 128, 0, st>>>(a);
    SQ_CHECK_LAUNCH("sq_tree_attn(simt)");
    return SQ_OK;
  }
  constexpr int smem = TcSmem<D>::TOTAL + 1024;
  decltype(&tree_attn_tc_kernel<D, false, false, RAGGED>) kern;
  if constexpr (RAGGED) kern = tree_attn_tc_kernel<D, false, false, true>;
  else kern = BATCH ? tree_attn_tc_kernel<D, false, true>
                    : (a.dense_mask ? tree_attn_tc_kernel<D, true, false> : tree_attn_tc_kernel<D, false, false>);
  static bool attr_set[2] = {false, false};    // (a process drives one device: bench / tests / torchrun ranks)
  if (!attr_set[a.dense_mask ? 1 : 0]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { set_error("sq_tree_attn: smem attr: %s", cudaGetErrorString(e)); return SQ_ERR_CUDA; }
    attr_set[a.dense_mask ? 1 : 0] = true;
  }
  const int RPT = TILE_Q / p->GP;
  // a ragged launch has one y block per q tile of every part; the others q_tiles per sequence, B sequences
  int q_tiles;
  if constexpr (RAGGED) q_tiles = rp.tile0[rp.n_parts];
  else q_tiles = (a.n + RPT - 1) / RPT;
  const int groups = a.H / p->GP;
  // KV splits per cluster: as many as it takes to put a CTA on every SM, never more than the KV tiles the cache can hold
  // (graph-static launches read the length from the device) or that this call touches (host-known kv_end)
  static int n_sm = 0;
  if (!n_sm) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n_sm <= 0) n_sm = 132;
  }
  const int seqs = RAGGED ? 1 : a.B;
  int Z = p->splits_force > 0 ? p->splits_force : n_sm / std::max(1, groups * q_tiles * seqs);
  Z = std::max(1, std::min(8, Z));
  Z = std::min(Z, p->splits_max);
  if (a.state == nullptr) Z = std::max(1, std::min(Z, (a.kv_end + TILE_KV - 1) / TILE_KV));
  p->last_splits = Z;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(groups, q_tiles * seqs, Z);
  cfg.blockDim = dim3(256);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;     // the KV splits of one (head group, q tile) form a cluster
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = Z;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (p->pdl) {                                         // start under the tail of the previous kernel (RoPE + KV append)
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.numAttrs = 2;
  }
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, p->tm_q, p->tm_k, p->tm_v, a, rp);
  if (e != cudaSuccess) { set_error("sq_tree_attn(tc): launch failed: %s", cudaGetErrorString(e)); return SQ_ERR_CUDA; }
  SQ_CHECK_LAUNCH("sq_tree_attn(tc)");
  return SQ_OK;
}

extern "C" int sq_tree_attn(sq_attn_plan* plan, int layer, int n, const int32_t* state, int n0, int kv_end,
                            int prefix_len_host, const sq_half* dense_mask, int64_t mask_ld, const uint32_t* tree_bits,
                            int tree_words, int tree_size, int impl, void* stream) {
  SQ_CHECK_ARG(plan != nullptr, "sq_tree_attn: null plan");
  SQ_CHECK_ARG(plan->B == 1, "sq_tree_attn: the plan holds %d sequences (use sq_tree_attn_batch)", plan->B);
  SQ_CHECK_ARG(n >= 0 && n <= plan->n_max, "sq_tree_attn: n=%d exceeds plan n_max=%d", n, plan->n_max);
  SQ_CHECK_ARG(layer >= 0 && layer < plan->L, "sq_tree_attn: bad layer %d", layer);
  SQ_CHECK_ARG(tree_words <= 32, "sq_tree_attn: tree_size > 1024 unsupported (32 mask words per row)");
  SQ_CHECK_ARG(state != nullptr || kv_end <= plan->M, "sq_tree_attn: kv_end %d > M %d", kv_end, plan->M);
  if (n == 0) return SQ_OK;
  AttnArgs a;
  a.q = plan->q; a.ld = plan->ld;
  a.k_layer = plan->k_cache + (int64_t)layer * plan->Hkv * plan->M * plan->D;
  a.v_layer = plan->v_cache + (int64_t)layer * plan->Hkv * plan->M * plan->D;
  a.out = plan->out;
  a.n = n; a.H = plan->H; a.Hkv = plan->Hkv; a.M = plan->M; a.GP = plan->GP; a.B = 1; a.layer = layer;
  a.state = state; a.n0 = n0; a.kv_end = kv_end; a.prefix_len_host = prefix_len_host;
  a.dense_mask = (const __half*)dense_mask; a.mask_ld = mask_ld;
  a.tree_bits = tree_bits; a.tree_words = tree_bits ? tree_words : 0; a.tree_size = tree_bits ? tree_size : 0;
  a.scale = 1.0f / sqrtf((float)plan->D);
  a.debug_flags = plan->debug_flags; a.err_flag = plan->err_flag; a.dbg = plan->dbg;
  cudaStream_t st = (cudaStream_t)stream;
  if (plan->D == 64) return launch_attn<64, false>(plan, a, impl, st);
  return launch_attn<128, false>(plan, a, impl, st);
}

extern "C" int sq_tree_attn_batch(sq_attn_plan* plan, int layer, int n, int B, const int32_t* state, int n0, int kv_end,
                                  const uint32_t* tree_bits, int tree_words, int tree_size, void* stream) {
  SQ_CHECK_ARG(plan != nullptr, "sq_tree_attn_batch: null plan");
  SQ_CHECK_ARG(B == plan->B, "sq_tree_attn_batch: B=%d but the plan's cache holds %d sequences", B, plan->B);
  SQ_CHECK_ARG(n >= 0 && (int64_t)n * B <= plan->n_max, "sq_tree_attn_batch: %d x %d rows exceed plan n_max=%d", B, n,
               plan->n_max);
  SQ_CHECK_ARG(layer >= 0 && layer < plan->L, "sq_tree_attn_batch: bad layer %d", layer);
  SQ_CHECK_ARG(tree_words <= 32, "sq_tree_attn_batch: tree_size > 1024 unsupported (32 mask words per row)");
  SQ_CHECK_ARG(state != nullptr, "sq_tree_attn_batch: needs the state array");
  if (n == 0) return SQ_OK;
  AttnArgs a{};
  a.q = plan->q; a.ld = plan->ld;
  a.out = plan->out;
  a.n = n; a.H = plan->H; a.Hkv = plan->Hkv; a.M = plan->M; a.GP = plan->GP; a.B = B; a.layer = layer;
  a.state = state; a.n0 = n0; a.kv_end = kv_end; a.prefix_len_host = 0;
  a.tree_bits = tree_bits; a.tree_words = tree_bits ? tree_words : 0; a.tree_size = tree_bits ? tree_size : 0;
  a.scale = 1.0f / sqrtf((float)plan->D);
  a.debug_flags = plan->debug_flags; a.err_flag = plan->err_flag; a.dbg = plan->dbg;
  cudaStream_t st = (cudaStream_t)stream;
  if (plan->D == 64) return launch_attn<64, true>(plan, a, 0, st);
  return launch_attn<128, true>(plan, a, 0, st);
}

extern "C" int sq_tree_attn_ragged(sq_attn_plan* plan, int layer, const sq_ragged_part* parts, int n_parts,
                                   const int32_t* state, const uint32_t* tree_bits, int tree_words, int tree_size,
                                   void* stream) {
  SQ_CHECK_ARG(plan != nullptr, "sq_tree_attn_ragged: null plan");
  SQ_CHECK_ARG(layer >= 0 && layer < plan->L, "sq_tree_attn_ragged: bad layer %d", layer);
  SQ_CHECK_ARG(tree_words <= 32, "sq_tree_attn_ragged: tree_size > 1024 unsupported (32 mask words per row)");
  SQ_CHECK_ARG(state != nullptr, "sq_tree_attn_ragged: needs the state array");
  RaggedParts rp;
  const int rc = make_ragged(parts, n_parts, plan->B, plan->n_max, TILE_Q / plan->GP, "sq_tree_attn_ragged", &rp);
  if (rc != SQ_OK) return rc;
  AttnArgs a{};
  a.q = plan->q; a.ld = plan->ld;
  a.out = plan->out;
  a.n = 0; a.H = plan->H; a.Hkv = plan->Hkv; a.M = plan->M; a.GP = plan->GP; a.B = plan->B; a.layer = layer;
  a.state = state; a.prefix_len_host = 0;
  a.tree_bits = tree_bits; a.tree_words = tree_bits ? tree_words : 0; a.tree_size = tree_bits ? tree_size : 0;
  a.scale = 1.0f / sqrtf((float)plan->D);
  a.debug_flags = plan->debug_flags; a.err_flag = plan->err_flag; a.dbg = plan->dbg;
  cudaStream_t st = (cudaStream_t)stream;
  if (plan->D == 64) return launch_attn<64, false, true>(plan, a, 0, st, rp);
  return launch_attn<128, false, true>(plan, a, 0, st, rp);
}
