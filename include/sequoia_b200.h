/* sequoia_b200 -- C ABI of the H100-native (sm_90a) Sequoia hot path (libsequoia_b200.so).
 *
 * The reference (Infini-AI-Lab/Sequoia) has no FFI layer: its boundary is the Python class API
 * (Engine.GraphInferenceEngine[TG], Tree.SpecTree / GreedyTree, utils.*).  This header is the
 * boundary a maintainer would bind from those classes (ctypes stub in INTEGRATION.md).  Each
 * entry point cites the reference code it replaces (paths relative to the Sequoia repo).
 *
 * Conventions: every function returns SQ_OK (0) or a negative SQ_ERR_* code and records a message
 * retrievable with sq_last_error(); all pointers are DEVICE pointers unless named host_*; no
 * ownership transfer; `stream` is a cudaStream_t passed as void*; every launch is asynchronous and
 * CUDA-graph capturable (no allocation, no synchronisation).  fp16 = IEEE binary16 (`uint16_t` bits).
 *
 * "Tree-relative" addressing: many calls take (state, n0).  If `state` is non-NULL the first row of
 * the call lives at absolute slot  state[SQ_ST_P] - 1 + n0  (tree node n0 of the current iteration:
 * node k sits at slot P-1+k, SURVEY.md appendix A); if `state` is NULL the first row is slot n0.
 * This lets a captured graph follow the dynamic prefix length P without host involvement.
 */
#ifndef SEQUOIA_B200_H_
#define SEQUOIA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SQ_OK 0
#define SQ_ERR_INVALID_ARG (-1)
#define SQ_ERR_CUDA (-2)
#define SQ_ERR_UNSUPPORTED (-3)

/* words of the int32 device state array (>= SQ_ST_WORDS entries) */
#define SQ_ST_P 0
#define SQ_ST_ACCEPT_LEN 1
#define SQ_ST_TERMINAL 2
#define SQ_ST_N_NEW 3
#define SQ_ST_P_OLD 4
#define SQ_ST_BONUS 5
#define SQ_ST_NAN 6
#define SQ_ST_SKIPPED 7
#define SQ_ST_M 8 /* host-written: length of tokens / position_ids (max_length); bounds the walk's epilogue writes */
#define SQ_ST_FROZEN 9 /* host-written, batched calls only: nonzero = finished sequence, nothing of it is written */
#define SQ_ST_FINISH 10 /* the *_batch_stop walks only: 0 = go on, 1 = a stop id ended the sequence, 2 = its length limit */
#define SQ_ST_END 11    /* the *_batch_stop walks only: the sequence's final length when SQ_ST_FINISH != 0, else 0 */
#define SQ_ST_GUIDED 12 /* host-written, batched calls only: nonzero = the sequence follows a token guide (sq_guide_*) */
#define SQ_ST_GUIDE_STATE 13 /* guided sequences: the guide state after the committed tokens, -1 = dead */
#define SQ_ST_GUIDE_POS 14   /* guided sequences: the position up to which the guide has consumed the tokens */
#define SQ_ST_WORDS 16

typedef uint16_t sq_half;

const char* sq_last_error(void);
int sq_version(void);
/* number of kernels this library has launched so far in this process (bench.py's gpu_launches) */
uint64_t sq_launch_count(void);

/* ---- element-wise model ops (Engine/Llama_modules.py:259-288,327-349; Llama_model.py:53-72) ---- */

/* out[r,:] = table[tokens[base+r],:]   (nn.Embedding, Llama_model.py:53) */
int sq_embed_rows(const sq_half* table, const int64_t* tokens, const int32_t* state, int n0, int n, int hidden,
                  sq_half* out, void* stream);
/* LlamaRMSNorm_FI (Llama_modules.py:274-288): fp32 variance, cast to fp16, then weight * x (fp16). */
int sq_rmsnorm(const sq_half* x, const sq_half* weight, sq_half* out, int n, int hidden, float eps, void* stream);
/* resid += delta (fp16 add, Llama_modules.py:341,347) ; out = rmsnorm(resid).  out may be NULL (add only). */
int sq_add_rmsnorm(sq_half* resid, const sq_half* delta, const sq_half* weight, sq_half* out, int n, int hidden,
                   float eps, void* stream);
/* LlamaMLP_FI (Llama_modules.py:270-272): out = fp16(silu(gate)) * up, gate_up = [gate | up] rows of 2*inter. */
int sq_silu_mul(const sq_half* gate_up, sq_half* out, int n, int inter, void* stream);
/* interleaved = 1: gate_up rows are blocks of 32 = 16 gate | 16 up columns (the fused SwiGLU GEMM's weight row order). */
int sq_silu_mul_ex(const sq_half* gate_up, sq_half* out, int n, int inter, int interleaved, void* stream);

/* RoPE (transformers 4.36 apply_rotary_pos_emb, Llama_modules.py:117-118,213-214) applied in place to the
 * Q columns of the fused qkv rows, and K (rotated) + V appended to the cache at storage slots
 * (KV_Cache.update_kv_cache, Llama_KV.py:72-89).  qkv row layout: [H*D q | Hkv*D k | Hkv*D v], row pitch ld.
 * cos/sin: (max_pos, D) fp16 caches (Llama_modules.py:16-45).  position_ids / storage_ids are indexed at
 * base + r (see tree-relative addressing).  k_layer / v_layer: (Hkv, M, D) of this layer. */
int sq_rope_kv_append(sq_half* qkv, int ld, int H, int Hkv, int D, const sq_half* cos, const sq_half* sin,
                      const int64_t* position_ids, const int64_t* storage_ids, const int32_t* state, int n0, int n,
                      sq_half* k_layer, sq_half* v_layer, int M, void* stream);

/* ---- KV cache (Engine/Llama_KV.py) ---- */

/* gather_kv_incremental (Llama_KV.py:60-68): cache[..., offset+j, :] = cache[..., idx[j], :] for j < n, all
 * layers/heads, in place with gather-then-copy semantics.  n and offset come from the host values, or -- when
 * `state` is non-NULL -- from state[SQ_ST_N_NEW] / state[SQ_ST_P_OLD] (device-driven, graph static);
 * max_n bounds n for the launch.  zero_tail != 0 also zeroes rows >= offset+n like the reference does.
 * k_cache / v_cache: (L, 1, Hkv, M, D). */
int sq_kv_gather(sq_half* k_cache, sq_half* v_cache, int L, int Hkv, int M, int D, const int32_t* idx, int n,
                 int offset, const int32_t* state, int max_n, int zero_tail, void* stream);

/* Same compaction for index lists too long to stage on chip (n * D * 2 B > 200 KB; reference API gather_kv with a whole
 * accept list, Engine/Llama_KV.py:50-58): gather into the caller's scratch, then copy back.  Host-known n / offset only. */
int64_t sq_kv_gather_scratch_bytes(int L, int Hkv, int D, int n);
int sq_kv_gather_big(sq_half* k_cache, sq_half* v_cache, int L, int Hkv, int M, int D, const int32_t* idx, int n,
                     int offset, void* scratch, int64_t scratch_bytes, int zero_tail, void* stream);

/* ---- tree-masked attention (Llama_modules.py:127-134 draft SDPA, :220-248 target explicit attention) ---- */

/* Opaque plan: TMA descriptors (+ a small debug workspace) for one (q buffer, cache) pair.  Host call, not capturable;
 * create once per engine and reuse inside graphs.  (Split-KV partials are reduced through distributed shared memory
 * inside the kernel; no global workspace.) */
typedef struct sq_attn_plan sq_attn_plan;
/* q: (n_max rows, ld) fp16 with head h at columns [h*D,(h+1)*D); k_cache/v_cache: (L,1,Hkv,M,D);
 * out: (n_max, H*D) fp16.  workspace: device buffer of sq_attn_workspace_bytes(...) bytes. */
int64_t sq_attn_workspace_bytes(int n_max, int H, int D, int M);
int sq_attn_plan_create(sq_attn_plan** plan, const sq_half* q, int ld, int n_max, int H, int Hkv, int D,
                        const sq_half* k_cache, const sq_half* v_cache, int L, int M, sq_half* out,
                        void* workspace, int64_t workspace_bytes);
int sq_attn_plan_destroy(sq_attn_plan* plan);
/* Synchronous: returns the watchdog word of the plan (0 = no tensor-core / TMA wait ever timed out). */
int sq_attn_plan_error(sq_attn_plan* plan);
/* Launch shape of the plan: gp = query heads packed into one 128-row tile; splits = KV splits per cluster (Z) of the last
 * tensor-core launch (0 before the first).  Z comes from the SM count, or from the environment variable SQ_ATTN_SPLITS
 * read at plan creation (tuning / tests); either way it is clamped to 8, to the cache's KV tiles and, for calls without
 * a state array, to the tiles of kv_end. */
int sq_attn_plan_info(sq_attn_plan* plan, int* gp, int* splits);
/* Debug: with SQ_ATTN_TIMING=1 the kernel records clock64() phase stamps of CTA (head 0, q tile 0, split s) at
 * host_out[s*16 + k] (128 values); SQ_ERR_UNSUPPORTED otherwise. */
int sq_attn_plan_debug_times(sq_attn_plan* plan, long long* host_out);

/* Attention of n query rows (slots base..base+n-1) of `layer` against cache slots [0, kv_len).
 *   kv_len = (state ? state[P]-1 : 0) + kv_end          (device-driven when state != NULL)
 * Mask, one of:
 *   dense_mask != NULL: additive fp16 mask, row r at dense_mask + r*mask_ld, kv_len columns  (reference semantics);
 *   else structured tree mask (SURVEY.md appendix A): key slot c is visible from row slot s iff
 *        c <= min(s, P-1)  ||  (s >= P && c >= P-1 && bit(tree_bits, s-(P-1), c-(P-1)))
 *   where tree_bits is the growmap's ancestor-or-self matrix packed 32 columns per word, row pitch
 *   tree_words, tree_size S; with state == NULL, P = prefix_len_host.
 * scale = 1/sqrt(D).  impl: 0 = wgmma/TMA kernel (product), 1 = SIMT cross-check kernel (tests only). */
int sq_tree_attn(sq_attn_plan* plan, int layer, int n, const int32_t* state, int n0, int kv_end,
                 int prefix_len_host, const sq_half* dense_mask, int64_t mask_ld, const uint32_t* tree_bits,
                 int tree_words, int tree_size, int impl, void* stream);

/* ---- sampling (utils.py) ---- */

/* out = fp16(softmax(fp16(logits / T)))  (Tree/SpecTree.py:198).  rows of V, pitches in elements. */
int sq_softmax_T(const sq_half* logits, int64_t ld_in, sq_half* out, int64_t ld_out, int n, int V, float T,
                 void* stream);

/* One tree level of drafting (Tree/SpecTree.py:103-104 / GreedyTree.py:102-103 + tests/testbed.py:277-285):
 * for each parent row j < n_parents, top-k (k = k_max) of
 *     mode 0: fp16(log(rand_row)) / softmax(fp16(logits_row / T))     (utils.py:10-18, exponential race, all fp16)
 *     mode 1: logits_row                                              (utils.py:29-32, sampling_argmax)
 * in descending order (ties: lower vocabulary index first), written to positions[j*k_max + i] (may be NULL),
 * and the first n_branch[j] of them to tokens[base + child_first[j] + i]  (tokens may be NULL).
 * logits row = logits + parent_rows[j]*ld (parent_rows NULL => row j); rand likewise.  V <= 32768, V % 8 == 0. */
int sq_sample_level(const sq_half* logits, int64_t ld_logits, const sq_half* rand, int64_t ld_rand,
                    const int32_t* parent_rows, const int32_t* child_first, const int32_t* n_branch, int n_parents,
                    int k_max, int V, float T, int mode, int64_t* positions, int64_t* tokens, const int32_t* state,
                    void* stream);

/* One tree level of SpecInfer-style drafting (Tree/SpecInferTree.py:100-105): children drawn i.i.d. WITH replacement
 * from q = softmax(fp16(logits_row / T)) (fp16).  Exact integer inverse-CDF: w_v = q_v * 2^24 (exact), draw c is the
 * first v whose inclusive prefix sum exceeds (words[wbase + c] * sum_v w_v) >> 32, words = uniform integers in
 * [0, 2^32) stored as int64 (the caller's RNG; the reference uses torch.multinomial's).  wbase = child_first[j]
 * (node id of the first child) or j*k_max when child_first is NULL; n_branch[j] (or k_max) draws per parent, written
 * to positions[j*k_max + c] (may be NULL) and tokens[base + child_first[j] + c] (may be NULL). */
int sq_sample_replace(const sq_half* logits, int64_t ld_logits, const int64_t* words, const int32_t* parent_rows,
                      const int32_t* child_first, const int32_t* n_branch, int n_parents, int k_max, int V, float T,
                      int64_t* positions, int64_t* tokens, const int32_t* state, void* stream);

/* get_residual (utils.py:5-8): out = relu(p-q) / sum(relu(p-q)), fp16 roundings as torch. */
int sq_residual(const sq_half* p, const sq_half* q, sq_half* out, int V, void* stream);

/* get_sampling_logits (utils.py:65-77), in place on n rows: tokens whose predecessor in descending-logit order has
 * cumulative probability fp16(cumsum(softmax(fp16(logits/T)))) > fp16(top_p) are set to -inf; equal logits rank by
 * ascending index.  No-op when top_p >= 1. */
int sq_top_p_filter(sq_half* logits, int64_t ld, int n, int V, float top_p, float T, void* stream);

/* Top-k filter, in place on n rows: exactly k tokens of each row keep their logit, every other one is set to -inf.
 * Ranking is on the raw fp16 logit, value descending, equal values by ascending index (a stable descending sort, the tie
 * rule of sq_top_p_filter; -0 ranks with +0, NaN above +inf), so the kept set does not depend on the temperature.  -inf
 * entries rank last: a row with fewer than k finite logits loses nothing finite.  k == 0 is off and k >= V filters
 * nothing (no launch); k < 0 is refused.  To compose with top-p, run this first: sq_top_p_filter then renormalises over
 * the survivors (a -inf logit has probability 0), the temperature -> top_k -> top_p order of common samplers. */
int sq_top_k_filter(sq_half* logits, int64_t ld, int n, int V, int k, void* stream);

/* argmax over V per row -> int64 (GreedyTree.py:186). */
int sq_argmax_rows(const sq_half* logits, int64_t ld, int n, int V, int64_t* out, void* stream);

/* ---- verification walk (Tree/SpecTree.py:137-157,196-227,261-281; GreedyTree.py:132-146,186-240) ---- */

/* Static tree tables on the device (built once per growmap): succ_off (S+1) / succ (CSR children, node ids),
 * depth (S) int32.  */
/* Stochastic accept/reject walk from the root, entirely on the device (one CTA):
 *   p = softmax(fp16(target_logits[cur] / T)); for child c of cur in Successors order:
 *       q = softmax(fp16(draft_logits[cur] / T)); accept iff p[tok] > fp16(r[slot(c)] * q[tok])  (strict >)
 *       else p = get_residual(p, q); draft_logits[cur][tok] = fp16 min
 *   terminal on accepted token in {0, 2} or NaN residual; bonus = argmax(fp16(residual / noise)) (the n=1 form of
 *   torch.multinomial; `noise` = Exp(1) fp16 row generated by torch).
 * Then (SpecTree.py:224, 261-271): compact tokens / position_ids, write the bonus token, re-lay tree positions,
 * and publish state[] (P, accept_len, terminal, n_new, P_old, bonus, nan, skipped) and accept_idx[0..n_new).
 * target_logits: (S, V) raw logits rows (row k = node k).  draft_logits: (>=S, V) rows, READ ONLY (the masking
 * of rejected tokens is kept on chip; the reference's in-place edit is dead state).
 * policy: 0 = SpecTree.  SQ_ACCEPT_GE: accept on >= ; SQ_ACCEPT_KEEP_Q: q is not edited after a rejection — both set
 * = the SpecInfer walk (Tree/SpecInferTree.py:143-162).  */
#define SQ_ACCEPT_GE 1
#define SQ_ACCEPT_KEEP_Q 2
int sq_accept_stochastic(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits, int64_t ld_d,
                         const sq_half* r, const sq_half* noise, const int32_t* succ_off, const int32_t* succ,
                         const int32_t* depth, int S, int V, float T, int64_t* tokens, int64_t* position_ids,
                         int32_t* accept_idx, int32_t* state, int max_target_seq, int policy, void* stream);
/* Greedy walk (GreedyTree.py): target_token (S) int64 from sq_argmax_rows; accept the first child whose token
 * equals target_token[cur]; bonus = target_token[last accepted]. Same outputs as above. */
int sq_accept_greedy(const int64_t* target_token, const int32_t* succ_off, const int32_t* succ,
                     const int32_t* depth, int S, int64_t* tokens, int64_t* position_ids, int32_t* accept_idx,
                     int32_t* state, int max_target_seq, void* stream);

/* ---- weight-streaming GEMM for <= 128 rows (nn.Linear, Llama_modules.py:108-110,138,270-272; Llama_model.py:213) ---- */

/* C[n, N] = A[n, K] * W[N, K]^T, fp16 in / fp32 accumulate / fp16 out, n <= 128.  A: (n_max, lda), W: (N, K) row-major
 * (the nn.Linear weight as stored), C: (n_max, ldc).  K % 64 == 0, N % 128 == 0.  Plans hold the TMA descriptors; create
 * once per (activation buffer, weight, output buffer), run inside graphs.  err_flag: optional device word set by the
 * pipeline watchdog.  n > 128 (prefill) runs one launch per 128-row tile. */
typedef struct sq_gemm_plan sq_gemm_plan;
int sq_gemm_plan_create(sq_gemm_plan** plan, const sq_half* a, int lda, int n_max, const sq_half* w, int N, int K,
                        sq_half* c, int ldc, int* err_flag);
#define SQ_GEMM_TILED 1
#define SQ_GEMM_SWIGLU 2
/* Tile shape (BN, K splits, multicast width) a plan for (N, K) will use -- needed to pre-tile weights. */
int sq_gemm_pick_tiles(int N, int K, int* bn, int* split, int* mc);
int sq_gemm_pick_tiles_ex(int N, int K, int flags, int* bn, int* split, int* mc);
/* sq_gemm_plan_create with flags: SQ_GEMM_TILED (w = the pre-tiled copy) | SQ_GEMM_SWIGLU (fused SwiGLU epilogue, n_out = N/2;
 * excludes split-K tiles). */
int sq_gemm_plan_create_ex(sq_gemm_plan** plan, const sq_half* a, int lda, int n_max, const sq_half* w, int N, int K,
                           sq_half* c, int ldc, int* err_flag, int flags);
/* As sq_gemm_plan_create, for weights stored pre-tiled as (ceil(N/BN), K/64, BN, 64) fp16 contiguous (rows beyond N
 * zero): every weight TMA load is one contiguous BN*128-byte block of HBM. */
int sq_gemm_plan_create_tiled(sq_gemm_plan** plan, const sq_half* a, int lda, int n_max, const sq_half* w_tiled, int N, int K,
                              sq_half* c, int ldc, int* err_flag);
/* Fused epilogue.  kind 0: plain (default).  kind 1 (SwiGLU, Engine/Llama_modules.py:272): W's rows interleave 16 gate
 * rows / 16 up rows (row 32b+t = gate[16b+t], row 32b+16+t = up[16b+t]); C (n, n_out = N/2) = silu(gate) * up with the
 * reference's fp16 rounding points.  Not for split-K plans. */
int sq_gemm_plan_set_epilogue(sq_gemm_plan* plan, int kind, int n_out);
int sq_gemm_plan_destroy(sq_gemm_plan* plan);
int sq_gemm_plan_info(sq_gemm_plan* plan, int* bn, int* split, int* stages);
int sq_gemm_run(sq_gemm_plan* plan, int n, void* stream);
/* Rows [a_row0, a_row0 + n) of the plan's activation buffer -> rows [0, n) of `c` (pitch ldc halfs); c == NULL: the plan's
 * own output buffer, rows [a_row0, a_row0 + n). */
int sq_gemm_run_at(sq_gemm_plan* plan, int n, int a_row0, sq_half* c, int ldc, void* stream);

/* ---- FP8 (E4M3) weight-streaming GEMM: the target's layer projections on quantized weights (csrc/sq_gemm_fp8.cu) ---- */

/* C[n, N] = A[n, K] * W'[N, K]^T with W'[j, k] = fp16(fp16(q[j, k]) * w_scale[j]): q e4m3 (one byte per weight), one fp16
 * scale per output channel; fp16 activations, fp32 accumulation, fp16 out.  q is stored pre-tiled by
 * sq_gemm_fp8_tile_weights (its only producer).  N % 64 == 0, K % 64 == 0, lda and ldc multiples of 8.  err_flag: optional
 * device word set by the pipeline watchdog.  n > 128 runs one launch per 128-row tile.  SQ_GEMM_FP8_FORCE="nwg,split"
 * (nwg 2 or 3 weight tiles of 64 rows per CTA, split 1-4 K splits over a cluster), read at plan creation, forces the
 * instance; sq_gemm_fp8_plan_info reports the one chosen (stages: ring depth of the 128-row instance). */
typedef struct sq_gemm_fp8_plan sq_gemm_fp8_plan;
/* (N, K) row-major e4m3 q -> the kernel's pre-tiled copy (N * K bytes): block (t, kb) of 4096 bytes per 64-row tile t
 * and 64-wide K block kb, at (t * K/64 + kb) * 4096; byte h * 2048 + u * 16 + 8 (k % 2) + 2 r + e (h = k / 2) of a
 * block holds register r, half e of the wgmma m64k16 A fragment of k16 step k of consumer thread u (0-127). */
int sq_gemm_fp8_tile_weights(const uint8_t* q, uint8_t* q_tiled, int N, int K, void* stream);
int sq_gemm_fp8_plan_create(sq_gemm_fp8_plan** plan, const sq_half* a, int lda, int n_max, const uint8_t* w_q,
                            const sq_half* w_scale, int N, int K, sq_half* c, int ldc, int* err_flag);
int sq_gemm_fp8_plan_info(sq_gemm_fp8_plan* plan, int* nwg, int* split, int* stages);
int sq_gemm_fp8_plan_destroy(sq_gemm_fp8_plan* plan);
/* Rows [a_row0, a_row0 + n) of the plan's activation buffer -> rows [0, n) of `c` (pitch ldc halfs); c == NULL: the plan's
 * own output buffer, rows [a_row0, a_row0 + n). */
int sq_gemm_fp8_run_at(sq_gemm_fp8_plan* plan, int n, int a_row0, sq_half* c, int ldc, void* stream);

/* ---- target tensor parallelism: fused one-shot all-reduce over NVLink peer memory (no reference counterpart) ---- */

/* Peer-mappable device buffers (cudaMalloc + CUDA IPC).  handle64: 64-byte cudaIpcMemHandle_t. */
int sq_tp_alloc(void** ptr, int64_t bytes);
int sq_tp_free(void* ptr);
int sq_tp_ipc_export(void* ptr, uint8_t* handle64);
int sq_tp_ipc_open(const uint8_t* handle64, void** ptr);
int sq_tp_ipc_close(void* ptr);
/* resid += sum_r proj_r ; out = rmsnorm(resid) * weight   for n rows, in ONE kernel on every rank:
 * replaces NCCL all-reduce + sq_add_rmsnorm after the row-parallel o_proj / down_proj (Llama_modules.py:341,347).
 * host_proj_ptrs[N]: device pointers to rank 0..N-1's partial output (n_max, hidden) fp16 (own + peer-mapped);
 * host_flag_ptrs[N]: device pointers to each rank's N-word flag array; epoch: 4 local words (epoch, ticket, error, -).
 * Every rank must launch the matching call; the partial buffers of consecutive reductions must alternate (A, B). */
int sq_tp_allreduce_add_rmsnorm(sq_half* resid, const void* const* host_proj_ptrs, void* const* host_flag_ptrs,
                                uint32_t* epoch, int rank, int N, const sq_half* weight, sq_half* out, int n,
                                int hidden, float eps, void* stream);

/* Two-shot variant (row r owned by rank r % N: the owner pulls the N partial rows, stores the fp16 sum into every rank's
 * `red` buffer and raises a per-row flag; every rank then adds the residual and normalises from its local copy): per
 * rank (N-1)/N of the payload pulled + (N-1)/N pushed instead of (N-1) x pulled.  host_red_ptrs[r] / host_rowflag_ptrs[r]:
 * peer-mapped (n_max, hidden) fp16 buffer / n_max uint32 words on rank r; same epoch / flag words as the one-shot call. */
int sq_tp_allreduce2_add_rmsnorm(sq_half* resid, const void* const* host_proj_ptrs, void* const* host_red_ptrs,
                                 void* const* host_flag_ptrs, void* const* host_rowflag_ptrs, uint32_t* epoch, int rank,
                                 int N, const sq_half* weight, sq_half* out, int n, int hidden, float eps, void* stream);

/* One-shot PUSH variant for small payloads: every rank stores its partial row (proj_local, (n, hidden)) into receive slot
 * [rank][row] of every peer (host_recv_ptrs[r] = (N, rows_max, hidden) fp16 area on rank r for this buffer parity), one system
 * fence, per-(source, row) epoch flags (host_pflag_ptrs[r] = (N, rows_max) uint32 on rank r), then reduces from LOCAL memory in
 * rank order + residual + RMSNorm.  One NVLink one-way trip instead of flag + fetch. */
int sq_tp_allreduce3_add_rmsnorm(sq_half* resid, const sq_half* proj_local, void* const* host_recv_ptrs,
                                 void* const* host_pflag_ptrs, uint32_t* epoch, int rank, int N, int rows_max,
                                 const sq_half* weight, sq_half* out, int n, int hidden, float eps, void* stream);

/* LL two-shot for small payloads: every 8-byte word crossing NVLink carries two halfs + the reduction's epoch (one atomic
 * store), readers poll the words they need -- no flags, no fences, two one-way trips.  host_ll1_ptrs[r]: gather area on rank r,
 * (N, own_max, hidden/4) 16-byte pairs; host_ll2_ptrs[r]: reduced-row area on rank r, (rows_max, hidden/4) pairs; both for this
 * buffer parity, zero-initialised.  Row r is owned by rank r %% N.  own_max == rows_max selects the ONE-shot form (every rank
 * pushes its row to every peer's gather slot and reduces locally: one trip, (N-1) x the bytes; meant for N <= 3). */
int sq_tp_allreduce_ll_add_rmsnorm(sq_half* resid, const sq_half* proj_local, void* const* host_ll1_ptrs,
                                   void* const* host_ll2_ptrs, uint32_t* epoch, int rank, int N, int rows_max, int own_max,
                                   const sq_half* weight, sq_half* out, int n, int hidden, float eps, void* stream);

/* Driver -> follower messages over peer memory as LL words (4 bytes of payload + the message's epoch per 8-byte store; the
 * reader polls): replaces the NCCL broadcasts of tokens / position ids / state / accept list.  host_mbox_ptrs[i]: the channel's
 * mailbox on follower i (2 x cap_words 8-byte words, zero-initialised, double-buffered by epoch parity); `epoch`: this rank's
 * device counter for the channel.  Up to three segments of 4-byte words per message. */
int sq_tp_ll_publish(void* const* host_mbox_ptrs, int n_peers, int cap_words, uint32_t* epoch, const void* src0, int words0,
                     const void* src1, int words1, const void* src2, int words2, void* stream);
int sq_tp_ll_consume(const void* mbox_local, int cap_words, uint32_t* epoch, uint32_t* err, void* dst0, int words0, void* dst1,
                     int words1, void* dst2, int words2, void* stream);

/* ---- draft attention (csrc/sq_draft.cu): tree-masked attention of the small draft model's forwards of <= 64 rows
 * (Engine/Llama_modules.py:127-134 inside the per-level graph of Engine/Engine.py:158-164).  Supported: head_dim 64,
 * n_heads * 64 == hidden, no GQA, max_length <= 640 (a head's K and V live in shared memory; see sq_draft_supported).
 * k_cache / v_cache: (n_layers, 1, n_heads, max_length, 64). ---- */
typedef struct sq_draft_plan sq_draft_plan;
int sq_draft_supported(int hidden, int n_heads, int n_kv_heads, int head_dim, int max_length);
int sq_draft_plan_create(sq_draft_plan** plan, int hidden, int n_layers, int n_heads, int max_length, sq_half* k_cache,
                         sq_half* v_cache);
int sq_draft_plan_destroy(sq_draft_plan* plan);

/* Attention of `layer` for n (<= 64) rows = tree nodes [n0, n0+n) in tree-relative addressing (base = state[P]-1; keys
 * [0, base+kv_end) under the packed tree mask), as one launch on caller-owned buffers: q rows from `qkv` (n, 3*hidden),
 * K/V from the plan's caches (rows already appended), output (n, hidden).  Small-shape alternative to sq_tree_attn. */
int sq_draft_attention(sq_draft_plan* plan, int layer, int n, const sq_half* qkv, sq_half* attn_out, const int32_t* state,
                       int n0, int kv_end, const uint32_t* tree_bits, int tree_words, int tree_size, void* stream);

/* ---- batches: B <= SQ_MAX_BATCH sequences that share one growmap, one launch per op for all of them ----
 * Sequence b is a batch index of the grid.  Per-sequence data:
 *   state:            B rows of SQ_ST_WORDS words (sequence b at state + b*SQ_ST_WORDS); tree-relative addressing uses
 *                     that row's P.  A sequence whose SQ_ST_FROZEN word is nonzero writes nothing except its own
 *                     activation / attention-output rows, and embed and the walks skip it entirely.
 *   tokens, position_ids, storage_ids, r: B rows of ld_seq elements;
 *   activation rows:  sequence-major, sequence b's n rows start at row b*n;
 *   KV cache:         (L, B, Hkv, M, D), sequence b of layer l at planes (l*B + b)*Hkv + h;
 *   target logits:    (B*S, V), node k of sequence b at row b*S + k;
 *   draft logits:     node k of sequence b at row row_base[k] + b*row_step[k] (static int32 tables of S entries), so that
 *                     one GEMM can write a whole tree level of all sequences: level rows n0..n0+tb-1 as one block of B*tb
 *                     rows at row B*n0 gives row_base[k] = B*n0 + (k - n0), row_step[k] = tb;
 *   accept_idx:       B rows of ld_acc (>= S) words; bonus-token noise: B rows of ld_noise (>= V) halfs.
 * With B = 1 every call computes bit for bit what its single-sequence counterpart computes. */
#define SQ_MAX_BATCH 8
int sq_embed_rows_batch(const sq_half* table, const int64_t* tokens, int64_t ld_seq, const int32_t* state, int n0, int n,
                        int B, int hidden, sq_half* out, void* stream);
/* k_layer / v_layer: (B, Hkv, M, D) of this layer */
int sq_rope_kv_append_batch(sq_half* qkv, int ld, int H, int Hkv, int D, const sq_half* cos, const sq_half* sin,
                            const int64_t* position_ids, const int64_t* storage_ids, int64_t ld_seq, const int32_t* state,
                            int n0, int n, int B, sq_half* k_layer, sq_half* v_layer, int M, void* stream);
/* device-driven compaction of every sequence (n = state[N_NEW], offset = state[P_OLD] of its own row, indices from its
 * accept_idx row); tail rows are left stale as in sq_kv_gather with state */
int sq_kv_gather_batch(sq_half* k_cache, sq_half* v_cache, int L, int B, int Hkv, int M, int D, const int32_t* accept_idx,
                       int ld_idx, const int32_t* state, int max_n, void* stream);
/* prefix reuse: copy rows [0, n) of sequence src to the same rows of sequence dst, K and V of every layer and kv head, in
 * one launch (grid (L*Hkv, 2, chunks), 16-byte loads and stores, no shared memory).  Every other byte of both caches,
 * dst's rows >= n included, is left as it was.  Refused with SQ_ERR_INVALID_ARG before any launch: a null or not 16-byte
 * aligned cache, L or Hkv < 1, D % 8 != 0, B outside 1..SQ_MAX_BATCH, src or dst outside [0, B), src == dst, n outside
 * 1..M. */
int sq_kv_copy_prefix(sq_half* k_cache, sq_half* v_cache, int L, int B, int Hkv, int M, int D, int src, int dst, int n,
                      void* stream);
/* attention plan over a (L, B, Hkv, M, D) cache; q / out hold B*n rows (n_max counts all of them) */
int sq_attn_plan_create_batch(sq_attn_plan** plan, const sq_half* q, int ld, int n_max, int H, int Hkv, int D,
                              const sq_half* k_cache, const sq_half* v_cache, int L, int B, int M, sq_half* out,
                              void* workspace, int64_t workspace_bytes);
/* n query rows per sequence under the structured tree mask (state required, B == the plan's B); the KV split count is
 * chosen once for the whole launch */
int sq_tree_attn_batch(sq_attn_plan* plan, int layer, int n, int B, const int32_t* state, int n0, int kv_end,
                       const uint32_t* tree_bits, int tree_words, int tree_size, void* stream);
/* sq_sample_level for every sequence: parent node parent_rows[j]'s logits from the draft-row table, its rand row at
 * rand + b*ld_rand_seq + node*ld_rand (mode 0); children to tokens + b*ld_seq */
int sq_sample_level_batch(const sq_half* logits, int64_t ld_logits, const int32_t* row_base, const int32_t* row_step,
                          const sq_half* rand, int64_t ld_rand, int64_t ld_rand_seq, const int32_t* parent_rows,
                          const int32_t* child_first, const int32_t* n_branch, int n_parents, int k_max, int V, float T,
                          int mode, int64_t* tokens, int64_t ld_seq, const int32_t* state, int B, void* stream);
/* one walk (one 8-CTA cluster) per sequence; target_logits (B*S, V).  Every batched stochastic walk (this one and its
 * _per_seq, _mixed and _stop forms) writes the bonus token at slot a before it gathers the accepted slots, as SpecTree
 * does, except for a sequence whose SQ_ST_GUIDED word is nonzero: that one gathers first and then writes the bonus, as
 * GreedyTree does, so every committed token is the token its own row drew.
 * SQ_ACCEPT_SKIP_DEAD (policy bit of the _per_seq, _mixed and _stop forms only; refused elsewhere): the walk for draft
 * rows processed by sq_draft_rows_batch.  A child whose token's entry in its parent's raw draft row (before the
 * temperature) is -inf (0xFC00) is dead: it is never accepted and leaves p and q exactly as they were, and the walk
 * moves on to the next sibling.  Without it such a child, once q's support is used up, turns q and then the residual
 * into NaN and ends the sequence by the NaN flag. */
#define SQ_ACCEPT_SKIP_DEAD 8
int sq_accept_stochastic_batch(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits, int64_t ld_d,
                               const int32_t* row_base, const int32_t* row_step, const sq_half* r, const sq_half* noise,
                               int64_t ld_noise, const int32_t* succ_off, const int32_t* succ, const int32_t* depth, int S,
                               int V, float T, int64_t* tokens, int64_t* position_ids, int64_t ld_seq, int32_t* accept_idx,
                               int64_t ld_acc, int32_t* state, int B, int max_target_seq, int policy, void* stream);
/* Per-sequence sampling parameters: as sq_sample_level_batch / sq_accept_stochastic_batch / sq_top_p_filter, with the
 * temperature (and top_p) of sequence b read from (B,) fp32 device arrays T[b] / top_p[b] instead of one scalar, so a
 * captured graph serves sequences with any settings.  With all-equal arrays each computes bit for bit what the scalar
 * call computes.  sq_sample_level_batch_per_seq: mode 0 uses T[b], mode 1 ignores it.  sq_top_p_filter_per_seq: row r of
 * the n rows belongs to sequence r / rows_per_seq (rows_per_seq must divide n); a row whose sequence has top_p >= 1 is left
 * untouched.  Null arrays are refused with SQ_ERR_INVALID_ARG. */
int sq_sample_level_batch_per_seq(const sq_half* logits, int64_t ld_logits, const int32_t* row_base,
                                  const int32_t* row_step, const sq_half* rand, int64_t ld_rand, int64_t ld_rand_seq,
                                  const int32_t* parent_rows, const int32_t* child_first, const int32_t* n_branch,
                                  int n_parents, int k_max, int V, const float* T, int mode, int64_t* tokens,
                                  int64_t ld_seq, const int32_t* state, int B, void* stream);
int sq_accept_stochastic_batch_per_seq(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits,
                                       int64_t ld_d, const int32_t* row_base, const int32_t* row_step, const sq_half* r,
                                       const sq_half* noise, int64_t ld_noise, const int32_t* succ_off,
                                       const int32_t* succ, const int32_t* depth, int S, int V, const float* T,
                                       int64_t* tokens, int64_t* position_ids, int64_t ld_seq, int32_t* accept_idx,
                                       int64_t ld_acc, int32_t* state, int B, int max_target_seq, int policy,
                                       void* stream);
int sq_top_p_filter_per_seq(sq_half* logits, int64_t ld, int n, int V, const float* top_p, const float* T,
                            int rows_per_seq, void* stream);
/* sq_top_k_filter with row r of the n rows at the k of sequence r / rows_per_seq, read from the (B,) int32 device array
 * top_k (rows_per_seq must divide n); a row whose k <= 0 or k >= V is left untouched.  With an all-equal array it computes
 * bit for bit what the scalar call computes.  A null array is refused with SQ_ERR_INVALID_ARG. */
int sq_top_k_filter_per_seq(sq_half* logits, int64_t ld, int n, int V, const int32_t* top_k, int rows_per_seq,
                            void* stream);
/* Min-p filter, in place on n rows; row r belongs to sequence b = r / rows_per_seq (rows_per_seq must divide n), whose
 * fp32 ln(min_p) and temperature are log_min_p[b] and T[b], (B,) float32 device arrays; log_min_p[b] = -inf is off and
 * leaves the rows untouched.  vLLM's rule, softmax(x / T)_i >= min_p * max softmax(x / T), decided in logit space: with
 * x_i the fp32 value of the fp16 logit, m the row max over its non-NaN entries and thr = fp32(T[b] * log_min_p[b]) (one
 * round-to-nearest multiply), token i keeps its logit when x_i is NaN, x_i == m or fp32(x_i - m) >= thr, and becomes -inf
 * otherwise.  So NaN stays (the walk's NaN flag still ends the sequence), a +inf entry stays and drops every finite entry
 * of its row, -inf stays, min_p = 1 (ln 1 = 0) keeps only the ties with the max, and a -inf threshold keeps everything.
 * Min-p and top-k both keep an upper set of the value order that contains the max, so on NaN-free rows they commute bit
 * for bit; run before sq_top_p_filter_per_seq, which then renormalises over the survivors.  Deterministic (no atomics).
 * A null array, a rows_per_seq that does not divide n and a bad V are refused with SQ_ERR_INVALID_ARG; n == 0 is a
 * no-op. */
int sq_min_p_filter_per_seq(sq_half* logits, int64_t ld, int n, int V, const float* log_min_p, const float* T,
                            int rows_per_seq, void* stream);
/* target_token (B*S) int64 */
int sq_accept_greedy_batch(const int64_t* target_token, const int32_t* succ_off, const int32_t* succ, const int32_t* depth,
                           int S, int64_t* tokens, int64_t* position_ids, int64_t ld_seq, int32_t* accept_idx,
                           int64_t ld_acc, int32_t* state, int B, int max_target_seq, void* stream);
/* Per-sequence policy: greedy is a (B,) int32 device array, nonzero = the sequence decodes greedily (GreedyTree), zero = it
 * samples (SpecTree).  One decode step of a mixed batch launches all three forms, each of which writes only its own
 * policy's sequences:
 *   sq_sample_level_batch_mixed: sq_sample_level_batch_per_seq with mode 1 (top-k) for a greedy sequence, mode 0 at T[b]
 *     otherwise (T[b] of a greedy sequence is never read); rand is required;
 *   sq_accept_greedy_batch_mixed: sq_accept_greedy_batch for the greedy sequences only;
 *   sq_accept_stochastic_batch_mixed: sq_accept_stochastic_batch_per_seq for the sampling sequences only.
 * A frozen sequence is left alone as in the per-sequence forms.  Refused with SQ_ERR_INVALID_ARG before any launch: a null
 * greedy or T array, and everything the per-sequence forms refuse (B outside 1..SQ_MAX_BATCH included). */
int sq_sample_level_batch_mixed(const sq_half* logits, int64_t ld_logits, const int32_t* row_base, const int32_t* row_step,
                                const sq_half* rand, int64_t ld_rand, int64_t ld_rand_seq, const int32_t* parent_rows,
                                const int32_t* child_first, const int32_t* n_branch, int n_parents, int k_max, int V,
                                const float* T, const int32_t* greedy, int64_t* tokens, int64_t ld_seq,
                                const int32_t* state, int B, void* stream);
int sq_accept_greedy_batch_mixed(const int64_t* target_token, const int32_t* succ_off, const int32_t* succ,
                                 const int32_t* depth, int S, int64_t* tokens, int64_t* position_ids, int64_t ld_seq,
                                 int32_t* accept_idx, int64_t ld_acc, int32_t* state, const int32_t* greedy, int B,
                                 int max_target_seq, void* stream);
int sq_accept_stochastic_batch_mixed(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits,
                                     int64_t ld_d, const int32_t* row_base, const int32_t* row_step, const sq_half* r,
                                     const sq_half* noise, int64_t ld_noise, const int32_t* succ_off, const int32_t* succ,
                                     const int32_t* depth, int S, int V, const float* T, const int32_t* greedy,
                                     int64_t* tokens, int64_t* position_ids, int64_t ld_seq, int32_t* accept_idx,
                                     int64_t ld_acc, int32_t* state, int B, int max_target_seq, int policy, void* stream);
/* Per-sequence stop ids and length limits (stop mode).  stop_ids: (B, SQ_MAX_STOP) int32 device array, sequence b's ids
 * padded with -1 (an id < 0 never matches); end_limit: (B,) int32 device array, sequence b's absolute length limit E_b
 * (prompt length + new-token budget), <= 0 = none.  greedy: as in the mixed forms, or NULL:
 *   sq_accept_stochastic_batch_stop: sq_accept_stochastic_batch_per_seq (greedy NULL: every sequence samples) or
 *     sq_accept_stochastic_batch_mixed (greedy set: only the sampling sequences walk);
 *   sq_accept_greedy_batch_stop: sq_accept_greedy_batch (greedy NULL: every sequence walks) or
 *     sq_accept_greedy_batch_mixed (greedy set: only the greedy sequences walk).
 * Each walk runs without the fixed 0 / 2 end rule and commits exactly what that walk commits (tokens, position_ids,
 * accept_idx, state words 0..9).  Then, with P = state[SQ_ST_P] at the start of the step and n = a + 1 (n = a when the
 * NaN flag ended the walk, or no bonus token fitted the buffer), the committed tokens[P .. n) are scanned for the first
 * stop id, at j: its end is j + 1; E_b counts too when E_b <= n.  SQ_ST_END = the smaller end, SQ_ST_FINISH = 1 when the
 * stop id ends first or on a tie, 2 when E_b does; both 0 when neither applies.  The output of a stop-mode step is thus
 * exactly tokens[:SQ_ST_END] of the step without a stop rule.  Refused with SQ_ERR_INVALID_ARG before any launch: a null
 * stop_ids, end_limit (or T), and everything the per-sequence and mixed forms refuse. */
#define SQ_MAX_STOP 8
int sq_accept_stochastic_batch_stop(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits,
                                    int64_t ld_d, const int32_t* row_base, const int32_t* row_step, const sq_half* r,
                                    const sq_half* noise, int64_t ld_noise, const int32_t* succ_off, const int32_t* succ,
                                    const int32_t* depth, int S, int V, const float* T, const int32_t* greedy,
                                    const int32_t* stop_ids, const int32_t* end_limit, int64_t* tokens,
                                    int64_t* position_ids, int64_t ld_seq, int32_t* accept_idx, int64_t ld_acc,
                                    int32_t* state, int B, int max_target_seq, int policy, void* stream);
int sq_accept_greedy_batch_stop(const int64_t* target_token, const int32_t* succ_off, const int32_t* succ,
                                const int32_t* depth, int S, int64_t* tokens, int64_t* position_ids, int64_t ld_seq,
                                int32_t* accept_idx, int64_t ld_acc, int32_t* state, const int32_t* greedy,
                                const int32_t* stop_ids, const int32_t* end_limit, int B, int max_target_seq,
                                void* stream);
/* Per-sequence repetition, frequency and presence penalties (csrc/sq_penalty.cu), in place on the (B*S, V) target rows
 * (row b*S + k = node k of sequence b, row pitch ld >= V), before any filter or walk reads them.  rep, freq, pres: (B,)
 * fp32 device arrays (rho_b, f_b, p_b); prompt_len: (B,) int32, L_b = the length of sequence b's prompt.
 *   Context of row k: with P = state[b][SQ_ST_P], the committed tokens[b, 0 .. P) (slot P-1 is node 0), then the tokens
 *   at slots P-1+j of the ancestors-or-self j >= 1 of node k (the bits of row k of tree_bits).  These are the tokens the
 *   row's logits were computed from.  c_all(t) counts t in the context, c_out(t) only at slots >= L_b (path slots count
 *   as output).  Ids outside [0, V) are ignored.
 *   Once for each distinct id t of the context, if x = float(logit[row, t]) is finite (inf and NaN are left alone):
 *     c_all > 0: x = x < 0 ? x * rho : x / rho;
 *     c_out > 0: x = x - f * c_out, then x = x - p;
 *   each operation one IEEE fp32 round-to-nearest operation (no FMA), then x is clamped to [-65504, 65504] and rounded
 *   to fp16, so a finite logit stays finite.
 * A sequence with SQ_ST_FROZEN set, or with rho = 1, f = 0 and p = 0, has its rows left untouched; rows from B*S on are
 * never touched.  scratch: caller-owned int32 of at least B * (3 * ld_seq + 1) words, rewritten by every call before it
 * is read.  Two PDL-chained launches.  Refused with SQ_ERR_INVALID_ARG before any launch: a null array, B outside
 * 1..SQ_MAX_BATCH, V not a multiple of 8 in 8..131072, ld < V, S < 1 or tree_words != ceil(S/32) or tree_words > 32,
 * ld_seq outside 1..SQ_PENALTY_MAX_LEN, and a scratch too small. */
#define SQ_PENALTY_MAX_LEN 4096
int sq_penalize_rows_batch(sq_half* logits, int64_t ld, int V, const int64_t* tokens, int64_t ld_seq,
                           const int32_t* state, const int32_t* prompt_len, const uint32_t* tree_bits, int tree_words,
                           int S, const float* rep, const float* freq, const float* pres, int32_t* scratch,
                           int64_t scratch_words, int B, void* stream);
/* Per-sequence allowed-token mask and logit bias (csrc/sq_logit_bias.cu), in place on the (B*S, V) target rows (row b*S + k
 * = node k of sequence b, row pitch ld >= V), before the penalties, the walks and the filters read them.  The rule does not
 * depend on the tree: every row of sequence b is processed alike.
 *   allowed: (B, allowed_words) bitmask, id t allowed for sequence b when bit (t & 31) of word [b][t >> 5] is set
 *   (allowed_words >= ceil(V/32); bits from V on are not read); has_mask: (B,) int32, nonzero = sequence b has an allowed
 *   set.  bias_ids / bias_vals: (B, SQ_MAX_LOGIT_BIAS) int32 / fp32, the first n = min(n_bias[b], SQ_MAX_LOGIT_BIAS)
 *   entries of row b with ids in ascending order; ids outside [0, V) are skipped.
 *   1. Mask: when has_mask[b], every entry of the rows whose id is not allowed becomes -inf (0xFC00), NaN and +inf
 *      included; allowed entries are not touched.
 *   2. Bias: for each entry (t, beta) in order, if t is allowed (or there is no mask) and x = float(logit[row, t]) is
 *      finite, the logit becomes fp16(clamp(x + beta, -65504, 65504)), the add one IEEE fp32 round-to-nearest operation.
 *      Non-finite logits are left alone.
 * A sequence with SQ_ST_FROZEN set, or with no mask and n_bias <= 0, has its rows left byte-identical; rows from B*S on
 * are never touched.  One PDL-chained launch, grid (ceil(V/4096), S, B); no state, no scratch.  Refused with
 * SQ_ERR_INVALID_ARG before any launch: a null array, B outside 1..SQ_MAX_BATCH, V not a multiple of 8 in 8..131072,
 * ld < V, S < 1, allowed_words < ceil(V/32). */
#define SQ_MAX_LOGIT_BIAS 1024
int sq_logit_bias_rows_batch(sq_half* logits, int64_t ld, int V, int S, const int32_t* state, const uint32_t* allowed,
                             int64_t allowed_words, const int32_t* has_mask, const int32_t* bias_ids,
                             const float* bias_vals, const int32_t* n_bias, int B, void* stream);
/* Per-sequence bad words and min_tokens (csrc/sq_ban.cu), in place on the (B*S, V) target rows (row b*S + k = node k of
 * sequence b, row pitch ld >= V), right after sq_logit_bias_rows_batch and before the penalties, the walks and the
 * filters read them.  Each row gets a small set of banned ids that become -inf; the set depends on the tree path.
 *   Context of row k: with P = state[b][SQ_ST_P], the committed tokens[b, 0 .. P) at positions 0 .. P-1, then the path
 *   tokens at slots P-1+j of the ancestors-or-self j >= 1 of node k (the bits of row k of tree_bits), at positions
 *   P .. P+d-1 in slot order, d = depth[k] (node indices increase along every path).  The row's token lands at position
 *   P + d.  The generated context is the part at positions >= L = prompt_len[b].  A context token outside [0, V) matches
 *   no word id.
 *   Bad words (vLLM v1's rule, on output tokens only): words (B, SQ_MAX_BAD_WORDS, SQ_MAX_BAD_WORD_LEN) int32, word w of
 *   sequence b at [b][w][0 .. n), n = word_len[b][w]; the first min(n_words[b], SQ_MAX_BAD_WORDS) words are read.  When
 *   the generated context has at least n - 1 tokens and its last n - 1 equal w[0 .. n-2], id w[n-1] is banned (a
 *   one-token word in every row; a prefix that would reach into the prompt does not match).  A word with n outside
 *   1..SQ_MAX_BAD_WORD_LEN, or whose last id is outside [0, V), bans nothing.
 *   min_tokens: min_end (B,) int32, the absolute limit L + min_tokens (0 = off).  When P + d < min_end[b], every id of
 *   row b of end_ids (B, SQ_MAX_STOP) int32 in [0, V) is banned (-1 pads the row).
 *   A banned entry becomes -inf (0xFC00) unconditionally, NaN and +inf included; nothing else of the row is touched.
 * A sequence with SQ_ST_FROZEN set, or with n_words <= 0 and min_end <= 0, has its rows left byte-identical (its CTAs
 * return right after the PDL wait); rows from B*S on are never touched.  One PDL-chained launch, grid (S, B) of 128
 * threads; no state, no scratch.  Refused with SQ_ERR_INVALID_ARG before any launch: a null array, B outside
 * 1..SQ_MAX_BATCH, V not a multiple of 8 in 8..131072, ld < V, S < 1 or tree_words != ceil(S/32) or tree_words > 32,
 * ld_seq < 1. */
#define SQ_MAX_BAD_WORDS 128
#define SQ_MAX_BAD_WORD_LEN 16
int sq_ban_tokens_rows_batch(sq_half* logits, int64_t ld, int V, const int64_t* tokens, int64_t ld_seq,
                             const int32_t* state, const int32_t* prompt_len, const int32_t* depth,
                             const uint32_t* tree_bits, int tree_words, int S, const int32_t* words,
                             const int32_t* word_len, const int32_t* n_words, const int32_t* min_end,
                             const int32_t* end_ids, int B, void* stream);
/* Guided decoding (csrc/sq_guide.cu): a per-sequence token automaton that constrains every target row along its tree path.
 *   Guide blob: one int32 array per guided sequence, at the address guide_table[b] ((B,) int64 device table, 0 = none):
 *     [0] n = n_states (1..SQ_MAX_GUIDE_STATES), [1] W = ceil(V/32), [2] E = n_edges (<= SQ_MAX_GUIDE_EDGES), [3] V;
 *     default_next[n] at word SQ_GUIDE_HEADER (-1 = none); edge_off[n + 1] (edge_off[0] = 0, edge_off[n] = E); edge_id[E],
 *     ascending within each state's range [edge_off[s], edge_off[s+1]); edge_next[E]; then one allowed bitmask of W words
 *     per state (id t allowed in state s when bit t & 31 of mask word [s][t >> 5] is set; sq_logit_bias_rows_batch's
 *     layout).  The blob is consistent: the mask of s is exactly its edge ids, plus, when default_next[s] >= 0, the ids
 *     with no edge that the guide's default allows; every next state is in [0, n).  Masks dominate the size:
 *     n * W * 4 bytes, 16 KB per state at V = 128256.
 *   step(s, t): -1 when s < 0, t is outside [0, V) or the mask of s does not allow t; else edge_next of t's edge in s
 *   when t has one, else default_next[s].
 *   State words of a guided sequence (SQ_ST_GUIDED nonzero): SQ_ST_GUIDE_STATE = the state after the committed tokens
 *   (the guide's start for a new prompt), SQ_ST_GUIDE_POS = the position of the first token not yet consumed (the
 *   prompt length for a new prompt).
 * A sequence that is frozen, or whose SQ_ST_GUIDED word is 0 or guide_table[b] is 0, is left alone by all three calls.
 * Each is one PDL-chained launch; bad arguments are refused with SQ_ERR_INVALID_ARG before any launch (a null array, B
 * outside 1..SQ_MAX_BATCH, V not a multiple of 8 in 8..131072, and the checks named below).
 *
 * sq_guide_states_batch: node_state[b*S + k] (int32, (B, S)) = the state of node k of sequence b: the walk of step()
 * from state[b][SQ_ST_GUIDE_STATE] (node 0, the root) through the tokens at slots P-1+j of node k's ancestors-or-self
 * j >= 1 (the bits of row k of tree_bits, in slot order), P = state[b][SQ_ST_P]; -1 from the first disallowed id on.
 * depth: (S,) int32, node indices increasing along every path.  Grid (B).  Refused also: S outside 1..1024, tree_words !=
 * ceil(S/32), ld_seq < 1.
 *
 * sq_guide_mask_rows_batch: in place on the (B*S, V) target rows (row b*S + k = node k, pitch ld >= V), right after
 * sq_ban_tokens_rows_batch: with s = node_state[b*S + k], every entry whose id state s does not allow becomes -inf
 * (0xFC00), NaN and +inf included, and every entry of the row when s < 0; allowed entries stay bit-identical.  Rows from
 * B*S on are never touched.  Grid (ceil(V/4096), S, B).  Refused also: ld < V, S < 1.
 *
 * sq_guide_advance_batch: after the walk, moves state[b][SQ_ST_GUIDE_STATE] by step() through tokens[b][pos .. n), pos
 * = state[b][SQ_ST_GUIDE_POS], n = the step's committed length (a + 1 when !SQ_ST_TERMINAL and a < M, else a; a =
 * SQ_ST_ACCEPT_LEN, M = SQ_ST_M or ld_seq when 0; SQ_ST_END when SQ_ST_FINISH is set), then sets SQ_ST_GUIDE_POS = n.  On
 * a disallowed id at position q it sets SQ_ST_GUIDE_STATE = -1 and SQ_ST_GUIDE_POS = q: tokens[b][:q] is the longest
 * prefix the guide accepts.  A dead sequence (SQ_ST_GUIDE_STATE < 0) is left alone.  Grid (B) of one warp.  Refused
 * also: ld_seq < 1. */
#define SQ_MAX_GUIDE_STATES 4096
#define SQ_MAX_GUIDE_EDGES (1 << 20)
#define SQ_GUIDE_HEADER 4
int sq_guide_states_batch(const int64_t* guide_table, const int64_t* tokens, int64_t ld_seq, const int32_t* state,
                          const int32_t* depth, const uint32_t* tree_bits, int tree_words, int S, int V,
                          int32_t* node_state, int B, void* stream);
int sq_guide_mask_rows_batch(sq_half* logits, int64_t ld, int V, int S, const int32_t* state,
                             const int64_t* guide_table, const int32_t* node_state, int B, void* stream);
int sq_guide_advance_batch(const int64_t* guide_table, const int64_t* tokens, int64_t ld_seq, int32_t* state, int V,
                           int B, void* stream);
/* Constrained drafting (csrc/sq_draft_rows.cu): the processing of sq_logit_bias_rows_batch, sq_ban_tokens_rows_batch and
 * sq_guide_mask_rows_batch applied, in that order and bit for bit as they define it, to the draft rows of nodes
 * [k0, k0 + nk) of every sequence, in place (draft row of node k, sequence b: row_base[k] + b * row_step[k], pitch
 * ld >= V).  A draft row of node k is the distribution of the token after node k, the same context as target row k, so
 * it gets the same treatment: row k's context is the committed tokens plus node k's tree path, its token lands at
 * position P + depth[k], and its guide state is node k's.  flags selects the kinds (a nonzero set); the arrays of a kind
 * that is not selected are not read and may be NULL:
 *   SQ_DRAFT_BIAS: allowed, allowed_words, has_mask, bias_ids, bias_vals, n_bias as sq_logit_bias_rows_batch takes them;
 *   SQ_DRAFT_BAN: tokens, ld_seq, tree_bits, tree_words, prompt_len, depth, words, word_len, n_words, min_end, end_ids as
 *     sq_ban_tokens_rows_batch takes them;
 *   SQ_DRAFT_GUIDE: tokens, ld_seq, tree_bits, tree_words and guide_table as sq_guide_states_batch takes them, and
 *     node_state ((B, S) int32): the state of node k is one step() from node_state[b*S + parent(k)] by the token at slot
 *     P-1+k (the root's is state[b][SQ_ST_GUIDE_STATE]); the call writes it to node_state[b*S + k] and masks the row
 *     with it.  So the parent of every node in the range must lie below k0 and have been processed by an earlier call
 *     (a tree level at a time, the root first).
 * A frozen sequence, and one whose selected kinds are all neutral (no mask, n_bias <= 0, n_words <= 0, min_end <= 0, no
 * guide), has its rows left byte-identical, as have all rows outside the range.  One PDL-chained launch, grid
 * (ceil(V/4096), nk, B) of 256 threads.  Refused with SQ_ERR_INVALID_ARG before any launch: flags empty or with unknown
 * bits, a null array of a selected kind (or of draft_logits, row_base, row_step, state), B outside 1..SQ_MAX_BATCH, V not
 * a multiple of 8 in 8..131072, ld < V, S outside 1..1024 or tree_words != ceil(S/32), a node range that is neither the
 * root alone (k0 = 0, nk = 1) nor within [1, S), allowed_words < ceil(V/32), ld_seq < 1. */
#define SQ_DRAFT_BIAS 1
#define SQ_DRAFT_BAN 2
#define SQ_DRAFT_GUIDE 4
int sq_draft_rows_batch(sq_half* draft_logits, int64_t ld, int V, const int32_t* row_base, const int32_t* row_step,
                        int k0, int nk, int S, const int32_t* state, int flags, const uint32_t* allowed,
                        int64_t allowed_words, const int32_t* has_mask, const int32_t* bias_ids, const float* bias_vals,
                        const int32_t* n_bias, const int64_t* tokens, int64_t ld_seq, const uint32_t* tree_bits,
                        int tree_words, const int32_t* prompt_len, const int32_t* depth, const int32_t* words,
                        const int32_t* word_len, const int32_t* n_words, const int32_t* min_end, const int32_t* end_ids,
                        const int64_t* guide_table, int32_t* node_state, int B, void* stream);
/* Per-sequence logprobs of the committed tokens (csrc/sq_logprobs.cu), after the walk, from the (B*S, V) target rows as the
 * walk read them (penalised, top-k and top-p filtered; row pitch ld >= V, a multiple of 8).  With P = state[b][SQ_ST_P_OLD],
 * n_new = state[b][SQ_ST_N_NEW], a = P + n_new and M = state[b][SQ_ST_M] (ld_seq when 0), the step committed position
 * P + j for j < n_new (the accepted tokens) and for j = n_new when !state[b][SQ_ST_TERMINAL] && a < M (the bonus token).
 *   Row of position P + j: node 0 (row b*S) for j = 0, else node k = accept_idx[b][j-1] - (P - 1) (row b*S + k): the row
 *   the committed token was drawn from.  Token: tokens[b][P + j] as the walk left it.  SpecTree writes the bonus at slot a
 *   before it gathers the accepted slots, so an accepted node living at slot a (accept_idx[b][j-1] == a) is committed as
 *   the bonus token; that position still reads its path row.
 *   Value: s_i = fp16(float(x_i) * (1.0f / T_b)), T_b = T[b] for a sampled sequence and 1 for a greedy one (greedy[b] != 0),
 *   the values the walk's softmax reads; the fp32 log-softmax s_t - (m + log sum_i exp(s_i - m)), m = max s.
 *   A filtered token (-inf) has logprob -inf.  A row holding a +inf or NaN scaled value, or only -inf, gives NaN for every
 *   value.  At T = 1 with no filter, penalty, logit bias or allowed set this is the model's log-probability.
 *   Top entries: n = min(n_top[b], SQ_MAX_LOGPROBS, V) ids of the row ranked as sq_top_k_filter ranks them (raw fp16 value
 *   descending, equal values by ascending index, -0 equal to +0, NaN above +inf, -inf last; so the ids do not depend on T)
 *   with their logprobs, which do not increase down the list.
 * Output at absolute positions: lp_token (B, ld_seq) fp32 [b][P + j]; lp_ids (B, ld_seq, SQ_MAX_LOGPROBS) int32 and lp_top
 * (same shape, fp32) entries [b][P + j][0 .. n).  Nothing else is written: not a frozen sequence (SQ_ST_FROZEN), not a
 * sequence with n_top[b] < 0 (off), not a position the step did not commit, not entries from n on.  The token of an id
 * outside [0, V) gets NaN.  One PDL-chained launch, grid (max_depth + 1, B) of one CTA per position; no state between
 * calls.  Refused with SQ_ERR_INVALID_ARG before any launch: a null array, B outside 1..SQ_MAX_BATCH,
 * V not a multiple of 8 in 8..131072, ld < V or not a multiple of 8, logits not 16-byte aligned, S < 1, max_depth outside
 * 0..S-1, ld_seq < 1, ld_acc < max_depth. */
#define SQ_MAX_LOGPROBS 20
int sq_token_logprobs_batch(const sq_half* logits, int64_t ld, int V, int S, int max_depth, const int64_t* tokens,
                            int64_t ld_seq, const int32_t* state, const int32_t* accept_idx, int64_t ld_acc,
                            const float* T, const int32_t* greedy, const int32_t* n_top, float* lp_token,
                            int32_t* lp_ids, float* lp_top, int B, void* stream);
/* Prompt logprobs (csrc/sq_logprobs.cu): the log-probability of each prompt token under the model's raw distribution, from
 * the fp16 logits of the prompt rows of a first verify (row pitch ld >= V, a multiple of 8, n_logit_rows rows).  parts is
 * a HOST array of n_parts entries, copied into the kernel arguments; part j scores sequence seq:
 *   Row r < n_rows of part j is logits row logits_row0 + r, the model's prediction after prompt tokens 0 .. r.  It scores
 *   tokens[seq][r + 1] and writes position r + 1 of the outputs.  Position 0 is never written.
 *   Value: the rule of sq_token_logprobs_batch at T = 1 (s_i = the fp16 logit itself), the fp32 log-softmax
 *   s_t - (m + log sum_i exp(s_i - m)); a row holding +inf or NaN, or only -inf, gives NaN for every value; a token
 *   outside [0, V) gets NaN.  Top entries: n = min(n_top, V) ids ranked as sq_top_k_filter ranks them, with their logprobs.
 *   No temperature, filter, penalty, bias, ban or guide applies: no prompt token was drawn from a processed row.
 * Output at absolute positions: plp_token (B, ld_seq) fp32 [seq][r + 1]; plp_ids (B, ld_seq, SQ_MAX_LOGPROBS) int32 and
 * plp_top (same shape, fp32) entries [seq][r + 1][0 .. n).  Nothing else is written: not an unlisted sequence, not
 * position 0 or positions from n_rows + 1 on, not entries from n on.  One PDL-chained launch, grid (max n_rows, n_parts)
 * of one 1024-thread CTA per row; no state between calls.  Refused with SQ_ERR_INVALID_ARG before any launch: a null
 * array, B outside 1..SQ_MAX_BATCH, V not a multiple of 8 in 8..131072, ld < V or not a multiple of 8, logits not
 * 16-byte aligned, n_parts outside 1..B, a seq outside [0, B) or listed twice, n_rows < 1 or n_rows + 1 > ld_seq, rows
 * outside [0, n_logit_rows), n_top outside 0..SQ_MAX_LOGPROBS. */
typedef struct {
  int32_t seq, logits_row0, n_rows, n_top;
} sq_prompt_lp_part;
int sq_prompt_logprobs_ragged(const sq_half* logits, int64_t ld, int V, int64_t n_logit_rows,
                              const sq_prompt_lp_part* parts, int n_parts, const int64_t* tokens, int64_t ld_seq,
                              float* plp_token, int32_t* plp_ids, float* plp_top, int B, void* stream);

/* ---- ragged batches: a forward over a chosen set of the B sequences, each with its own row count ----
 * A part list names the sequences to run.  Part j is n rows of sequence seq in that sequence's tree-relative addressing:
 * rows base + n0 + r (r < n), base = state[seq][SQ_ST_P] - 1, attending slots [0, base + kv_end) under the structured tree
 * mask.  Activation rows are packed in list order: part j starts at row row0_j = sum of n over the parts before it.
 * parts is a HOST array; each call copies it into its kernel arguments (no device table, no host-to-device copy) and is
 * one launch for all parts.  Refused with SQ_ERR_INVALID_ARG before any launch: n_parts outside 1..B, a seq outside
 * [0, B) or listed twice, n < 1, more rows in all than n_max (the activation buffer's rows, or the plan's), and
 * tree_words > 32.  The list is the selection: SQ_ST_FROZEN is not read, and nothing of an unlisted sequence (tokens,
 * state, KV bytes) is read or written by embed / RoPE + KV append; attention reads only the listed sequences' cache
 * planes.  A single part at B = 1 computes bit for bit what the corresponding _batch call computes. */
typedef struct {
  int32_t seq, n, n0, kv_end;
} sq_ragged_part;
/* the packed layout of a part list: row0[j] / tile0[j] (host arrays of n_parts + 1 entries, either may be NULL) = rows /
 * q tiles of rows_per_tile rows before part j; the same checks as the calls below */
int sq_ragged_layout(const sq_ragged_part* parts, int n_parts, int B, int n_max, int rows_per_tile, int32_t* row0,
                     int32_t* tile0);
/* out: n_max rows of hidden halfs */
int sq_embed_rows_ragged(const sq_half* table, const int64_t* tokens, int64_t ld_seq, const int32_t* state,
                         const sq_ragged_part* parts, int n_parts, int B, int n_max, int hidden, sq_half* out,
                         void* stream);
/* qkv: n_max rows; k_layer / v_layer: (B, Hkv, M, D) of this layer */
int sq_rope_kv_append_ragged(sq_half* qkv, int ld, int H, int Hkv, int D, const sq_half* cos, const sq_half* sin,
                             const int64_t* position_ids, const int64_t* storage_ids, int64_t ld_seq,
                             const int32_t* state, const sq_ragged_part* parts, int n_parts, int B, int n_max,
                             sq_half* k_layer, sq_half* v_layer, int M, void* stream);
/* on a plan made by sq_attn_plan_create_batch (its B and n_max); the KV split count is chosen once for the launch from all
 * parts' q tiles (SQ_ATTN_SPLITS forces it, sq_attn_plan_info reports it) */
int sq_tree_attn_ragged(sq_attn_plan* plan, int layer, const sq_ragged_part* parts, int n_parts, const int32_t* state,
                        const uint32_t* tree_bits, int tree_words, int tree_size, void* stream);

/* ---- per-sequence counter-based random numbers (csrc/sq_rng.cu): seeded BatchTree sequences draw r, rand and the bonus
 * noise on the device, each from a stream of its own ----
 * Generator: Random123 philox4x32-10.  Sequence b's key is its 64-bit seed, (seeds[b] & 0xffffffff, seeds[b] >> 32).
 * Element e of a stream is word e % 4 of the output block for counter (i & 0xffffffff, i >> 32, purpose, step),
 * i = e / 4.  Purposes:
 *   0 = r:           M elements, step 0;
 *   1 = rand:        S*V elements, node-major (node*V + v), step 0;
 *   2 = bonus noise: V elements, step = the sequence's verify count since it was seeded (0-based), mod 2^32.
 * Uniforms (purposes 0, 1): u = fp16((w >> 21) * 2^-11), the 2048 values k/2048 of torch's CPU fp16 uniform_.
 * Noise (purpose 2): u = fp32((w >> 8) + 0.5) * 2^-24 (one round-to-nearest-even), noise = fp16(max(-logf(u), 2^-24)):
 * positive and finite, so the walk's residual / noise never divides by zero.
 * seeds: (B,) uint64 and steps: (B,) int64 device arrays. */
/* `count` uniforms of `purpose` (0 or 1) into row b of `out` (row pitch ld_seq halfs) for every slot b of the host list
 * host_seqs[0 .. n_seqs), one launch.  Refused with SQ_ERR_INVALID_ARG before any launch: B outside 1..SQ_MAX_BATCH,
 * a slot out of range or listed twice, a null pointer, a purpose other than 0 or 1, count < 1 or ld_seq < count. */
int sq_rng_uniform_seqs(sq_half* out, int64_t ld_seq, int64_t count, const uint64_t* seeds, const int32_t* host_seqs,
                        int n_seqs, int B, int purpose, void* stream);
/* Row b of the (B, ld_noise) noise at step steps[b] for every sequence whose SQ_ST_FROZEN word is 0, then steps[b] += 1
 * on the device; a frozen sequence's row and counter are left untouched.  Graph capturable, needs nothing from the host
 * per replay.  V and ld_noise multiples of 8, ld_noise >= V, rows 16-byte aligned. */
int sq_rng_exponential_batch(sq_half* noise, int64_t ld_noise, int V, const uint64_t* seeds, int64_t* steps,
                             const int32_t* state, int B, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SEQUOIA_B200_H_ */
