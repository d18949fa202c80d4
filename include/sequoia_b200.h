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
/* one walk (one 8-CTA cluster) per sequence; target_logits (B*S, V) */
int sq_accept_stochastic_batch(const sq_half* target_logits, int64_t ld_t, const sq_half* draft_logits, int64_t ld_d,
                               const int32_t* row_base, const int32_t* row_step, const sq_half* r, const sq_half* noise,
                               int64_t ld_noise, const int32_t* succ_off, const int32_t* succ, const int32_t* depth, int S,
                               int V, float T, int64_t* tokens, int64_t* position_ids, int64_t ld_seq, int32_t* accept_idx,
                               int64_t ld_acc, int32_t* state, int B, int max_target_seq, int policy, void* stream);
/* target_token (B*S) int64 */
int sq_accept_greedy_batch(const int64_t* target_token, const int32_t* succ_off, const int32_t* succ, const int32_t* depth,
                           int S, int64_t* tokens, int64_t* position_ids, int64_t ld_seq, int32_t* accept_idx,
                           int64_t ld_acc, int32_t* state, int B, int max_target_seq, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SEQUOIA_B200_H_ */
