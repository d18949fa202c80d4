// Element-wise model ops of the tree-masked Llama forward: embedding gather, RMSNorm (+ fused residual add),
// SiLU*up, RoPE + KV append.  All HBM/latency-bound, 128-bit vectorised, fp16 roundings identical to the
// reference's torch ops (compute in fp32, round to fp16 after every torch-level op).
#include "sq_common.cuh"

namespace sq {

// ---------------------------------------------------------------------------------------------
// grid (n, B): sequence b's rows go to out rows [b*n, b*n + n); a frozen sequence's rows are left as they are.
// RAGGED: grid (sum of n); out row x belongs to the part whose row range holds it and is that part's row x - row0, of
// sequence seq at its own n0 (the frozen word is not read).
template <bool BATCH, bool RAGGED = false>
__global__ void embed_rows_kernel(const __half* __restrict__ table, const int64_t* __restrict__ tokens, int64_t ld_seq,
                                  const int32_t* __restrict__ state, int n0, int hidden, __half* __restrict__ out,
                                  const __grid_constant__ RaggedArg<RAGGED> rp) {
  pdl_wait();
  pdl_trigger();
  const RaggedParts* R = ragged_ptr(rp);
  const int pj = RAGGED ? ragged_part(R->row0, R->n_parts, blockIdx.x) : 0;   // RAGGED: this CTA's part
  const int b = RAGGED ? R->seq[pj] : seq_index<BATCH>(blockIdx.y);
  if (BATCH || RAGGED) {
    state += b * ST_WORDS;
    if (BATCH && state[ST_FROZEN]) return;          // its P may leave no room for n rows in tokens
    tokens += b * ld_seq;
  }
  const int r = RAGGED ? (int)blockIdx.x - R->row0[pj] : blockIdx.x;
  const int base = row_base(state, RAGGED ? R->n0[pj] : n0);
  const int64_t tok = tokens[base + r];
  const uint4* src = reinterpret_cast<const uint4*>(table + tok * (int64_t)hidden);
  uint4* dst = reinterpret_cast<uint4*>(out + (RAGGED ? (int64_t)blockIdx.x : (int64_t)b * gridDim.x + r) * hidden);
  for (int i = threadIdx.x; i < hidden / 8; i += blockDim.x) dst[i] = src[i];
}

// ---------------------------------------------------------------------------------------------
// One CTA (256 threads) per row.  hidden <= 256*8*MAXV.
template <int MAXV, bool ADD>
__global__ void __launch_bounds__(256) rmsnorm_kernel(__half* __restrict__ resid, const __half* __restrict__ delta,
                                                       const __half* __restrict__ x_in, const __half* __restrict__ w,
                                                       __half* __restrict__ out, int hidden, float eps) {
  __shared__ float red[8];
  const int r = blockIdx.x;
  const int nvec = hidden / 8;
  Pack8 v[MAXV];
  Pack8 wv[MAXV];
  if (out != nullptr) {                       // the norm weight does not depend on the previous kernel
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int c = threadIdx.x + i * 256;
      if (c < nvec) wv[i].u = reinterpret_cast<const uint4*>(w)[c];
    }
  }
  pdl_wait();
  pdl_trigger();
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = threadIdx.x + i * 256;
    if (c < nvec) {
      if (ADD) {
        Pack8 a, b;
        a.u = reinterpret_cast<const uint4*>(resid + (int64_t)r * hidden)[c];
        b.u = reinterpret_cast<const uint4*>(delta + (int64_t)r * hidden)[c];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[i].h[j] = f2h(h2f(a.h[j]) + h2f(b.h[j]));   // residual + x  (fp16 add)
        reinterpret_cast<uint4*>(resid + (int64_t)r * hidden)[c] = v[i].u;
      } else {
        v[i].u = reinterpret_cast<const uint4*>(x_in + (int64_t)r * hidden)[c];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float f = h2f(v[i].h[j]); ss += f * f; }
    }
  }
  if (out == nullptr) return;   // uniform across the block
  ss = block_sum<8>(ss, red);
  const float inv = rsqrtf(ss / (float)hidden + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = threadIdx.x + i * 256;
    if (c < nvec) {
      Pack8 o;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const __half xn = f2h(h2f(v[i].h[j]) * inv);        // hidden_states.to(input_dtype)
        o.h[j] = f2h(h2f(wv[i].h[j]) * h2f(xn));            // weight * x  (fp16 mul)
      }
      reinterpret_cast<uint4*>(out + (int64_t)r * hidden)[c] = o.u;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// interleaved = 0: gu row = [gate (inter) | up (inter)]; 1: blocks of 32 = 16 gate | 16 up (the row order of the fused
// SwiGLU GEMM's weights, ops.interleave_gate_up)
__global__ void silu_mul_kernel(const __half* __restrict__ gu, __half* __restrict__ out, int n, int inter, int interleaved) {
  pdl_wait();
  pdl_trigger();
  const int64_t nvec = (int64_t)n * (inter / 8);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / (inter / 8);
    const int c = (int)(i % (inter / 8));
    Pack8 g, u, o;
    if (interleaved) {
      const int off = (c >> 1) * 32 + (c & 1) * 8;
      g.u = *reinterpret_cast<const uint4*>(gu + r * 2 * inter + off);
      u.u = *reinterpret_cast<const uint4*>(gu + r * 2 * inter + off + 16);
    } else {
      g.u = reinterpret_cast<const uint4*>(gu + r * 2 * inter)[c];
      u.u = reinterpret_cast<const uint4*>(gu + r * 2 * inter + inter)[c];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float x = h2f(g.h[j]);
      const __half act = f2h(x / (1.0f + expf(-x)));        // F.silu in fp32 -> fp16
      o.h[j] = f2h(h2f(act) * h2f(u.h[j]));                 // * up (fp16 mul)
    }
    reinterpret_cast<uint4*>(out + r * inter)[c] = o.u;
  }
}

// ---------------------------------------------------------------------------------------------
// One CTA (256 threads) per row.  Work items: for every q/k head and every 16-byte chunk c of the first half of the
// head, rotate the pair (chunk c, chunk c + D/16) -> two 16-byte loads, two stores; then copy the V heads.
// grid (n, B): sequence b's rows are qkv rows [b*n, b*n + n), its cache planes k_layer + b*Hkv*M*D (a (B, Hkv, M, D)
// layer); a frozen sequence writes nothing.  RAGGED: grid (sum of n), qkv row x is row x - row0 of the part holding it,
// addressed in sequence seq's ids, state row and cache planes as the BATCH instance addresses sequence b.
template <bool BATCH, bool RAGGED = false>
__global__ void __launch_bounds__(256) rope_kv_append_kernel(
    __half* __restrict__ qkv, int ld, int H, int Hkv, int D, const __half* __restrict__ cosc,
    const __half* __restrict__ sinc, const int64_t* __restrict__ position_ids, const int64_t* __restrict__ storage_ids,
    int64_t ld_seq, const int32_t* __restrict__ state, int n0, __half* __restrict__ k_layer, __half* __restrict__ v_layer,
    int M, const __grid_constant__ RaggedArg<RAGGED> rp) {
  // under programmatic dependent launch: wait for the qkv GEMM, then let the attention launch start its prologue (it
  // waits for this grid's completion itself)
  pdl_wait();
  pdl_trigger();
  const RaggedParts* R = ragged_ptr(rp);
  const int pj = RAGGED ? ragged_part(R->row0, R->n_parts, blockIdx.x) : 0;   // RAGGED: this CTA's part
  const int b = RAGGED ? R->seq[pj] : seq_index<BATCH>(blockIdx.y);
  if (BATCH || RAGGED) {
    state += b * ST_WORDS;
    if (BATCH && state[ST_FROZEN]) return;
    position_ids += b * ld_seq;
    storage_ids += b * ld_seq;
    k_layer += (int64_t)b * Hkv * M * D;
    v_layer += (int64_t)b * Hkv * M * D;
  }
  const int r = RAGGED ? (int)blockIdx.x - R->row0[pj] : blockIdx.x;
  const int base = row_base(state, RAGGED ? R->n0[pj] : n0);
  const int64_t pos = position_ids[base + r];
  const int64_t slot = storage_ids[base + r];
  __half* row = qkv + (RAGGED ? (int64_t)blockIdx.x : (int64_t)b * gridDim.x + r) * ld;
  const int cph = D / 16;                                   // chunk pairs per head
  const uint4* cs = reinterpret_cast<const uint4*>(cosc + pos * D);
  const uint4* sn = reinterpret_cast<const uint4*>(sinc + pos * D);
  for (int w = threadIdx.x; w < (H + Hkv) * cph; w += blockDim.x) {
    const int head = w / cph, c = w % cph;
    uint4* src = reinterpret_cast<uint4*>(row + (int64_t)head * D);
    Pack8 x1, x2, c1, c2, s1, s2, o1, o2;
    x1.u = src[c]; x2.u = src[c + cph];
    c1.u = cs[c]; c2.u = cs[c + cph];
    s1.u = sn[c]; s2.u = sn[c + cph];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float a = h2f(x1.h[e]), b = h2f(x2.h[e]);
      // q*cos + rotate_half(q)*sin, each op rounded to fp16 (rotate_half = cat(-x2, x1))
      o1.h[e] = f2h(rnd16(a * h2f(c1.h[e])) + rnd16(-b * h2f(s1.h[e])));
      o2.h[e] = f2h(rnd16(b * h2f(c2.h[e])) + rnd16(a * h2f(s2.h[e])));
    }
    uint4* dst = (head < H) ? src : reinterpret_cast<uint4*>(k_layer + ((int64_t)(head - H) * M + slot) * D);
    dst[c] = o1.u;
    dst[c + cph] = o2.u;
  }
  const int cpv = D / 8;
  for (int w = threadIdx.x; w < Hkv * cpv; w += blockDim.x) {
    const int head = w / cpv, c = w % cpv;
    reinterpret_cast<uint4*>(v_layer + ((int64_t)head * M + slot) * D)[c] =
        reinterpret_cast<const uint4*>(row + (int64_t)(H + Hkv + head) * D)[c];
  }
}

}  // namespace sq

using namespace sq;

extern "C" int sq_embed_rows(const sq_half* table, const int64_t* tokens, const int32_t* state, int n0, int n,
                             int hidden, sq_half* out, void* stream) {
  SQ_CHECK_ARG(hidden % 8 == 0 && n >= 0, "sq_embed_rows: hidden %% 8 != 0");
  if (n == 0) return SQ_OK;
  launch_k(embed_rows_kernel<false>, dim3(n), dim3(128), 0, (cudaStream_t)stream, (const __half*)table, tokens, (int64_t)0,
           state, n0, hidden, (__half*)out, 0);
  SQ_CHECK_LAUNCH("sq_embed_rows");
  return SQ_OK;
}

extern "C" int sq_embed_rows_ragged(const sq_half* table, const int64_t* tokens, int64_t ld_seq, const int32_t* state,
                                    const sq_ragged_part* parts, int n_parts, int B, int n_max, int hidden, sq_half* out,
                                    void* stream) {
  SQ_CHECK_ARG(hidden % 8 == 0, "sq_embed_rows_ragged: hidden %% 8 != 0");
  SQ_CHECK_ARG(state != nullptr, "sq_embed_rows_ragged: needs the state array");
  RaggedParts rp;
  const int rc = make_ragged(parts, n_parts, B, n_max, 1, "sq_embed_rows_ragged", &rp);
  if (rc != SQ_OK) return rc;
  launch_k(embed_rows_kernel<false, true>, dim3(rp.row0[n_parts]), dim3(128), 0, (cudaStream_t)stream,
           (const __half*)table, tokens, ld_seq, state, 0, hidden, (__half*)out, rp);
  SQ_CHECK_LAUNCH("sq_embed_rows_ragged");
  return SQ_OK;
}

extern "C" int sq_embed_rows_batch(const sq_half* table, const int64_t* tokens, int64_t ld_seq, const int32_t* state,
                                   int n0, int n, int B, int hidden, sq_half* out, void* stream) {
  SQ_CHECK_ARG(hidden % 8 == 0 && n >= 0, "sq_embed_rows_batch: hidden %% 8 != 0");
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH && state != nullptr, "sq_embed_rows_batch: B=%d (1..%d) needs a state array", B,
               SQ_MAX_BATCH);
  if (n == 0) return SQ_OK;
  launch_k(embed_rows_kernel<true>, dim3(n, B), dim3(128), 0, (cudaStream_t)stream, (const __half*)table, tokens, ld_seq,
           state, n0, hidden, (__half*)out, 0);
  SQ_CHECK_LAUNCH("sq_embed_rows_batch");
  return SQ_OK;
}

template <bool ADD>
static int launch_rmsnorm(__half* resid, const __half* delta, const __half* x, const __half* w, __half* out, int n,
                          int hidden, float eps, cudaStream_t st) {
  SQ_CHECK_ARG(hidden % 8 == 0 && hidden <= 256 * 8 * 8, "sq_rmsnorm: hidden=%d unsupported", hidden);
  if (n == 0) return SQ_OK;
  const int nvec = hidden / 8;
  if (nvec <= 256) launch_k(rmsnorm_kernel<1, ADD>, dim3(n), dim3(256), 0, st, resid, delta, x, w, out, hidden, eps);
  else if (nvec <= 512) launch_k(rmsnorm_kernel<2, ADD>, dim3(n), dim3(256), 0, st, resid, delta, x, w, out, hidden, eps);
  else if (nvec <= 1024) launch_k(rmsnorm_kernel<4, ADD>, dim3(n), dim3(256), 0, st, resid, delta, x, w, out, hidden, eps);
  else launch_k(rmsnorm_kernel<8, ADD>, dim3(n), dim3(256), 0, st, resid, delta, x, w, out, hidden, eps);
  SQ_CHECK_LAUNCH("sq_rmsnorm");
  return SQ_OK;
}

extern "C" int sq_rmsnorm(const sq_half* x, const sq_half* weight, sq_half* out, int n, int hidden, float eps,
                          void* stream) {
  return launch_rmsnorm<false>(nullptr, nullptr, (const __half*)x, (const __half*)weight, (__half*)out, n, hidden, eps,
                               (cudaStream_t)stream);
}

extern "C" int sq_add_rmsnorm(sq_half* resid, const sq_half* delta, const sq_half* weight, sq_half* out, int n,
                              int hidden, float eps, void* stream) {
  return launch_rmsnorm<true>((__half*)resid, (const __half*)delta, nullptr, (const __half*)weight, (__half*)out, n,
                              hidden, eps, (cudaStream_t)stream);
}

extern "C" int sq_silu_mul(const sq_half* gate_up, sq_half* out, int n, int inter, void* stream) {
  return sq_silu_mul_ex(gate_up, out, n, inter, 0, stream);
}

extern "C" int sq_silu_mul_ex(const sq_half* gate_up, sq_half* out, int n, int inter, int interleaved, void* stream) {
  SQ_CHECK_ARG(inter % 8 == 0 && (!interleaved || inter % 16 == 0), "sq_silu_mul: inter %% 8 != 0 (16 when interleaved)");
  if (n == 0) return SQ_OK;
  const int64_t nvec = (int64_t)n * (inter / 8);
  int blocks = (int)((nvec + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  launch_k(silu_mul_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, (const __half*)gate_up, (__half*)out, n, inter,
           interleaved);
  SQ_CHECK_LAUNCH("sq_silu_mul");
  return SQ_OK;
}

extern "C" int sq_rope_kv_append(sq_half* qkv, int ld, int H, int Hkv, int D, const sq_half* cos, const sq_half* sin,
                                 const int64_t* position_ids, const int64_t* storage_ids, const int32_t* state, int n0,
                                 int n, sq_half* k_layer, sq_half* v_layer, int M, void* stream) {
  SQ_CHECK_ARG(D % 16 == 0 && ld % 8 == 0, "sq_rope_kv_append: head dim %d / pitch %d must be multiples of 16 / 8", D, ld);
  if (n == 0) return SQ_OK;
  launch_k(rope_kv_append_kernel<false>, dim3(n), dim3(256), 0, (cudaStream_t)stream, (__half*)qkv, ld, H, Hkv, D,
           (const __half*)cos, (const __half*)sin, position_ids, storage_ids, (int64_t)0, state, n0, (__half*)k_layer,
           (__half*)v_layer, M, 0);
  SQ_CHECK_LAUNCH("sq_rope_kv_append");
  return SQ_OK;
}

extern "C" int sq_rope_kv_append_batch(sq_half* qkv, int ld, int H, int Hkv, int D, const sq_half* cos, const sq_half* sin,
                                       const int64_t* position_ids, const int64_t* storage_ids, int64_t ld_seq,
                                       const int32_t* state, int n0, int n, int B, sq_half* k_layer, sq_half* v_layer, int M,
                                       void* stream) {
  SQ_CHECK_ARG(D % 16 == 0 && ld % 8 == 0, "sq_rope_kv_append_batch: head dim %d / pitch %d must be multiples of 16 / 8", D,
               ld);
  SQ_CHECK_ARG(B >= 1 && B <= SQ_MAX_BATCH && state != nullptr, "sq_rope_kv_append_batch: B=%d (1..%d) needs a state array",
               B, SQ_MAX_BATCH);
  if (n == 0) return SQ_OK;
  launch_k(rope_kv_append_kernel<true>, dim3(n, B), dim3(256), 0, (cudaStream_t)stream, (__half*)qkv, ld, H, Hkv, D,
           (const __half*)cos, (const __half*)sin, position_ids, storage_ids, ld_seq, state, n0, (__half*)k_layer,
           (__half*)v_layer, M, 0);
  SQ_CHECK_LAUNCH("sq_rope_kv_append_batch");
  return SQ_OK;
}

extern "C" int sq_rope_kv_append_ragged(sq_half* qkv, int ld, int H, int Hkv, int D, const sq_half* cos,
                                        const sq_half* sin, const int64_t* position_ids, const int64_t* storage_ids, int64_t ld_seq,
                                        const int32_t* state, const sq_ragged_part* parts, int n_parts, int B, int n_max,
                                        sq_half* k_layer, sq_half* v_layer, int M, void* stream) {
  SQ_CHECK_ARG(D % 16 == 0 && ld % 8 == 0, "sq_rope_kv_append_ragged: head dim %d / pitch %d must be multiples of 16 / 8",
               D, ld);
  SQ_CHECK_ARG(state != nullptr, "sq_rope_kv_append_ragged: needs the state array");
  RaggedParts rp;
  const int rc = make_ragged(parts, n_parts, B, n_max, 1, "sq_rope_kv_append_ragged", &rp);
  if (rc != SQ_OK) return rc;
  launch_k(rope_kv_append_kernel<false, true>, dim3(rp.row0[n_parts]), dim3(256), 0, (cudaStream_t)stream, (__half*)qkv,
           ld, H, Hkv, D, (const __half*)cos, (const __half*)sin, position_ids, storage_ids, ld_seq, state, 0,
           (__half*)k_layer, (__half*)v_layer, M, rp);
  SQ_CHECK_LAUNCH("sq_rope_kv_append_ragged");
  return SQ_OK;
}
