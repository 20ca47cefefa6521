/* rlaifv_b200.h — C ABI of librlaifv_b200.so: the H100 (sm_90a) kernels of the LLaVA-1.5 DPO
 * training step that replaces the reference's HF/torch hot path.
 *
 * Conventions
 *  - Every function returns 0 on success, <0 on error (-1 bad argument, -2 CUDA error, -3 driver /
 *    tensor-map error); the message is available from rlaifv_last_error() (thread-local).
 *    Nothing throws or aborts.
 *  - All pointers are raw DEVICE pointers owned by the caller (PyTorch storage in this repo);
 *    the library borrows them for the duration of the enqueued work and allocates nothing.
 *    One exception to the first rule: rlaifv_adamw_offload_bucket and rlaifv_adamw8bit_offload_bucket also take
 *    pinned HOST pointers (the optimizer state the caller keeps in page-locked host memory); the caller owns those
 *    buffers too.
 *  - `stream` is a cudaStream_t (the caller's current stream); all work is enqueued asynchronously,
 *    no host synchronisation happens inside.
 *  - "bf16" = __nv_bfloat16 storage. Row-major everywhere; `ld*` = elements between rows.
 *  - The reference has no FFI of its own (pure Python): each entry point names the reference code
 *    whose arithmetic it replaces. "HF:" = transformers/models/ (pinned 4.35.0, pyproject.toml:22).
 */
#ifndef RLAIFV_B200_H_
#define RLAIFV_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* rlaifv_last_error(void);

/* ---- dense contractions (wgmma / TMA) ----------------------------------------------------------
 * C[M,N] (+)= op(A) * op(B)^T (+ bias[N]) -> act -> (+ residual[M,N]).
 *   a_mn_major = 0: A is [M][K] (K contiguous)      1: A is stored [K][M]
 *   b_mn_major = 0: B is [N][K] (K contiguous)      1: B is stored [K][N]
 *   act: 0 none, 1 GELU(erf), 2 quick_gelu.  accumulate: C += result.  tile_n: 0 auto, 128, 256, or 512 = a
 *   256x256 tile per 2-CTA cluster (each CTA 128 rows; the B operand is TMA-multicast to both).
 * Replaces every nn.Linear forward / dgrad / wgrad of HF LlamaDecoderLayer (HF:llama/modeling_llama.py
 * :182-184,:262-264,:289), lm_head (llava/model/language_model/llava_llama.py:91-102), CLIP layers
 * (HF:clip/modeling_clip.py:300-351), the patch-embedding conv as im2col GEMM (:148-154) and the
 * mm_projector (llava/model/multimodal_projector/builder.py:39-46). */
int rlaifv_gemm_bf16(const void* A, long long lda, int a_mn_major, const void* B, long long ldb,
                     int b_mn_major, void* C, long long ldc, int M, int N, int K, const void* bias,
                     const void* residual, long long ldr, int act, int accumulate, int tile_n,
                     void* stream);

/* As rlaifv_gemm_bf16 with the product scaled first: bf16(bf16(A*B)*alpha) then bias/act/residual/accumulate.
 * Used for the LoRA adapters (peft 0.10.0 `result + lora_B(lora_A(x)) * scaling`;
 * muffin/train/train_llava15_lora.py:304-318, alpha/r = 16/64). */
int rlaifv_gemm_bf16_scaled(const void* A, long long lda, int a_mn_major, const void* B, long long ldb,
                            int b_mn_major, void* C, long long ldc, int M, int N, int K, const void* bias,
                            const void* residual, long long ldr, int act, int accumulate, int tile_n, float alpha,
                            void* stream);

/* Two operand pairs, one accumulator: C (+)= A*B^T + A2[:, koff:koff+K2]*B2^T with koff = (n0/n_sub)*r
 * (n_sub > 0: forward over fused sub-linears whose adapters' lora_A outputs sit side by side in A2) or 0.
 * The LoRA rank-r update is computed in the same CTA pass as the frozen base GEMM — no extra pass over C. */
int rlaifv_gemm_bf16_dual(const void* A, long long lda, int a_mn_major, const void* B, long long ldb, int b_mn_major,
                          const void* A2, long long lda2, const void* B2, long long ldb2, int K2, int r, int n_sub,
                          void* C, long long ldc, int M, int N, int K, const void* bias, const void* residual,
                          long long ldr, int act, int accumulate, void* stream);

/* Fused SwiGLU backward (replaces the autograd of `down_proj(act_fn(gate_proj(x)) * up_proj(x))`, HF
 * llama/modeling_llama.py:182-184, between the down-projection dgrad and the gate|up dgrad): with
 * d = bf16(A[M,K] @ op(B)^T) = d(act) [M, F] held in the accumulator,
 *   dgu[:, n] = d * up * silu'(gate),   dgu[:, F + n] = d * silu(gate)      (gu = [gate | up], [M, 2F], bf16)
 * are written by the GEMM epilogue; d(act) never reaches memory. F % 64 == 0. Optional second operand pair
 * (A2 [M, K2], B2, K2 > 0) accumulated into the same tile as in rlaifv_gemm_bf16_dual with n_sub = 0. */
int rlaifv_gemm_bf16_swiglu_bwd(const void* A, long long lda, const void* B, long long ldb, int b_mn_major,
                                const void* A2, long long lda2, const void* B2, long long ldb2, int K2, const void* gu,
                                long long ld_gu, void* dgu, long long ld_dgu, int M, int F, int K, void* stream);

/* raster group size (row-blocks per group, 0 keeps the current one; default 16) and debug switches:
 *   bit 0: skip the epilogue, stores of C included (mainloop only; results are then garbage; for roofline
 *          experiments only);
 *   bit 1: run the plain, residual and SwiGLU-backward forms with the register epilogue (each thread stores C straight
 *          from its accumulators) instead of the staged one (C through shared memory and TMA stores). Results are
 *          bit-identical; for A/B tests and timings. The register epilogue also runs every launch with bias, activation,
 *          alpha or accumulate, and a residual that is not 16-byte aligned or whose row stride is not a multiple of 8.
 * Process-wide. */
int rlaifv_gemm_set_tuning(int group_m, int debug);
/* L2 policy of the GEMM's TMA operand loads: bits 0-1 A loads, 2-3 B loads (0 normal, 1 evict first, 2 evict last;
 * bits 4-5 are accepted and ignored); bit 6: raster walks n-fastest inside groups of group_m column blocks instead of m-fastest
 * inside groups of row blocks. l2 < 0 (default): raster, group size and hints are chosen per launch from the shape
 * (long-K launches keep the smaller operand's panels resident in the L2); l2 >= 0 forces the given bits together
 * with rlaifv_gemm_set_tuning's group size. Process-wide; results are unaffected. */
int rlaifv_gemm_set_l2(int l2);
/* *clusters = the persistent grid's CTA slots for tile_n (128, 256: CTAs; 512: 2-CTA clusters) on the current device:
 * cudaOccupancyMaxActiveClusters of the kernel, at most num_SMs / cluster size. */
int rlaifv_gemm_max_active_clusters(int tile_n, int* clusters);
/* EXPERIMENTAL (default off): run GEMMs with K >= min_k and no bias / activation / residual as n K-slice passes
 * (passes 2.. with C +=) so each pass's operand slabs fit the L2. n <= 1 switches it off. */
int rlaifv_gemm_set_split_k(int n, int min_k);

/* Split attention backward (default for self-attention; replaces HF autograd through the eager attention of
 * llama/modeling_llama.py:199-222): attention_bwd_dkv_kernel (dK, dV per 128-row K/V tile) + attention_bwd_dq_kernel
 * (dQ per 128-row Q tile, written once as bf16 — no fp32 atomics, no zero-fill). dq may be the q column block of a
 * fused dqkv buffer (row stride ld_dq); rlaifv_rope_bwd* accepts dq_f32 == NULL to rotate that block in place.
 * head_dim 128; causal (Sq == Skv) or not; n_kv_heads < n_heads = grouped-query attention. delta_ws fp32
 * [nseq*n_heads*Sq]. */
int rlaifv_attention_bwd_split(const void* q, long long ld_q, const void* k, const void* v, long long ld_kv,
                               const void* out, long long ld_out, const void* d_out, long long ld_dout, const float* lse,
                               void* dq, long long ld_dq, void* dk, void* dv, long long ld_dkv, float* delta_ws, int nseq,
                               int Sq, int Skv, int n_heads, int n_kv_heads, int head_dim, int causal, float scale,
                               void* stream);


/* ---- attention (wgmma, S/O accumulators in registers) -----------------------------------------
 * q/k/v/out: [nseq*S][ld] bf16, head h at columns [h*head_dim, (h+1)*head_dim); lse fp32
 * [nseq][n_heads][S]. head_dim 128 (Llama, causal) or 64 (CLIP, non-causal).
 * Replaces HF:llama/modeling_llama.py:199-222 (eager causal attention; attention_mask=None as set at
 * muffin/train/trainers.py:199) and HF:clip/modeling_clip.py:261-279. */
int rlaifv_attention_fwd(const void* q, const void* k, const void* v, long long ld_qkv, void* out,
                         long long ld_out, float* lse, int nseq, int S, int n_heads, int head_dim,
                         int causal, float scale, void* stream);
/* causal, head_dim 128. dq_f32 [nseq*S][n_heads*128] fp32 must be zeroed by the caller (reduced with
 * atomics); dk/dv bf16 [nseq*S][ld_dkv]; delta_ws fp32 [nseq*n_heads*S] scratch. */
int rlaifv_attention_bwd(const void* q, const void* k, const void* v, long long ld_qkv, const void* out,
                         long long ld_out, const void* d_out, long long ld_dout, const float* lse,
                         float* dq_f32, void* dk, void* dv, long long ld_dkv, float* delta_ws, int nseq,
                         int S, int n_heads, int head_dim, float scale, void* stream);

/* Grouped-query variants (Mistral-7B decoder of OmniLMM-12B, omnilmm/model/omnilmm.py:259-265 -> HF
 * MistralForCausalLM: 32 query / 8 key-value heads): k/v (and dk/dv) hold n_kv_heads heads; query head h uses
 * kv head h / (n_heads / n_kv_heads); the backward sums the group's dK/dV contributions in registers. */
int rlaifv_attention_fwd_gqa(const void* q, const void* k, const void* v, long long ld_qkv, void* out,
                             long long ld_out, float* lse, int nseq, int S, int n_heads, int n_kv_heads,
                             int head_dim, int causal, float scale, void* stream);
int rlaifv_attention_bwd_gqa(const void* q, const void* k, const void* v, long long ld_qkv, const void* out,
                             long long ld_out, const void* d_out, long long ld_dout, const float* lse, float* dq_f32,
                             void* dk, void* dv, long long ld_dkv, float* delta_ws, int nseq, int S, int n_heads,
                             int n_kv_heads, int head_dim, float scale, void* stream);
/* Cross-attention of the perceiver resampler (OmniLMM-12B, omnilmm/model/resampler.py:149-168: the core of
 * nn.MultiheadAttention called at :158-163 — 64 learned queries over the Skv vision tokens, non-causal, no mask).
 * q [(q_shared ? 1 : nseq)*Sq][ld_q], k/v [nseq*Skv][ld_kv], out [nseq*Sq][ld_out], lse fp32 [nseq][n_heads][Sq].
 * q_shared != 0: one query block serves every image (resampler.py:160 `_repeat`), so it is read from sequence 0 and
 * the backward's fp32 dQ reduction also sums over the batch. head_dim 64 or 128 forward, 128 backward. */
int rlaifv_cross_attention_fwd(const void* q, long long ld_q, const void* k, const void* v, long long ld_kv, void* out,
                               long long ld_out, float* lse, int nseq, int Sq, int Skv, int n_heads, int head_dim,
                               int q_shared, float scale, void* stream);
int rlaifv_cross_attention_bwd(const void* q, long long ld_q, const void* k, const void* v, long long ld_kv,
                               const void* out, long long ld_out, const void* d_out, long long ld_dout,
                               const float* lse, float* dq_f32, void* dk, void* dv, long long ld_dkv, float* delta_ws,
                               int nseq, int Sq, int Skv, int n_heads, int head_dim, int q_shared, float scale,
                               void* stream);
/* RoPE on a fused row [q: n_heads*D | k: n_kv_heads*D | v: n_kv_heads*D] */
int rlaifv_rope_fwd_gqa(void* qkv, const void* cos_tab, const void* sin_tab, long long M, int T, int n_heads,
                        int n_kv_heads, int head_dim, long long ld, void* stream);
int rlaifv_rope_bwd_gqa(void* dqkv, const float* dq_f32, const void* cos_tab, const void* sin_tab, long long M,
                        int T, int n_heads, int n_kv_heads, int head_dim, long long ld, void* stream);

/* ---- packed rows: variable-length causal decoder (DESIGN.md §3) ---------------------------------
 * A training batch may drop every row after its sequence's last supervised position: sequence s then occupies rows
 * [cu[s], cu[s+1]) of [n_rows][ld] buffers, row cu[s] + t being position t. cu is int32 [nseq + 1] on the device;
 * max_len >= the longest sequence (sizes the grid). lse and delta_ws are fp32 [n_heads * n_rows], sequence s's
 * [n_heads][len_s] block at offset n_heads * cu[s]. Causal, head_dim 128, n_kv_heads <= n_heads (GQA). Every valid
 * row gets the bits the fixed-length kernels give the same sequence padded. The backward is the split form: dq bf16
 * [n_rows][ld_dq] (may be the q block of a fused dqkv buffer), dk/dv bf16 [n_rows][ld_dkv]. */
int rlaifv_attention_varlen_fwd(const void* q, const void* k, const void* v, long long ld_qkv, void* out,
                                long long ld_out, float* lse, const int* cu, int nseq, int max_len, long long n_rows,
                                int n_heads, int n_kv_heads, int head_dim, float scale, void* stream);
int rlaifv_attention_varlen_bwd(const void* q, const void* k, const void* v, long long ld_qkv, const void* out,
                                long long ld_out, const void* d_out, long long ld_dout, const float* lse, void* dq,
                                long long ld_dq, void* dk, void* dv, long long ld_dkv, float* delta_ws, const int* cu,
                                int nseq, int max_len, long long n_rows, int n_heads, int n_kv_heads, int head_dim,
                                float scale, void* stream);
/* The same with borrowed prefixes: two sequences whose inputs agree below a position keep one copy of those rows.
 * pos0 and partner are int32 [nseq] HOST arrays (nseq <= 64). Sequence s's rows [cu[s], cu[s+1]) hold positions
 * pos0[s] .. pos0[s] + len_s - 1, pos0[s] a multiple of 128; with pos0[s] > 0 its positions t < pos0[s] are the rows
 * cu[partner[s]] + t of its lender (pos0 0, partner s, at least pos0[s] rows). partner -1 = neither lends nor borrows.
 * O, LSE, dQ and the dK/dV of a borrower's rows get the bits the fixed-length kernels give the sequence padded; a
 * lender's rows below its borrower's pos0 get the sum of both sequences' dK/dV. */
int rlaifv_attention_varlen_prefix_fwd(const void* q, const void* k, const void* v, long long ld_qkv, void* out,
                                       long long ld_out, float* lse, const int* cu, const int* pos0,
                                       const int* partner, int nseq, int max_len, long long n_rows, int n_heads,
                                       int n_kv_heads, int head_dim, float scale, void* stream);
int rlaifv_attention_varlen_prefix_bwd(const void* q, const void* k, const void* v, long long ld_qkv, const void* out,
                                       long long ld_out, const void* d_out, long long ld_dout, const float* lse,
                                       void* dq, long long ld_dq, void* dk, void* dv, long long ld_dkv,
                                       float* delta_ws, const int* cu, const int* pos0, const int* partner, int nseq,
                                       int max_len, long long n_rows, int n_heads, int n_kv_heads, int head_dim,
                                       float scale, void* stream);
/* RoPE on the fused [q | k | v] rows with the position of row m taken from pos[m] (int32 [M], device); the backward
 * rotates the q block (split attention backward) and the k block in place. */
int rlaifv_rope_pos_fwd(void* qkv, const void* cos_tab, const void* sin_tab, const int* pos, long long M, int n_heads,
                        int n_kv_heads, int head_dim, long long ld, void* stream);
int rlaifv_rope_pos_bwd(void* dqkv, const void* cos_tab, const void* sin_tab, const int* pos, long long M, int n_heads,
                        int n_kv_heads, int head_dim, long long ld, void* stream);
/* LoRA dropout on packed rows x [n_rows][width]: row r draws the keep bits of row rows[r] of rlaifv_dropout_fwd's
 * element order, so a packed step draws the padded step's masks. */
int rlaifv_dropout_rows_fwd(const void* x, void* out, const int* rows, long long n_rows, int width, float p,
                            unsigned long long seed, void* stream);
int rlaifv_dropout_rows_bwd_add(void* dx, const void* g, const int* rows, long long n_rows, int width, float p,
                                unsigned long long seed, void* stream);

/* ---- norms (HF:llama/modeling_llama.py:62-67; HF:clip LayerNorm) -------------------------------- */
int rlaifv_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd_or_null, int M, int H, float eps,
                       void* stream);
int rlaifv_rmsnorm_bwd_partials(void); /* rows of the fp32 [partials][H] workspace rmsnorm_bwd needs */
/* H % 8 == 0 and H <= 6144 (up to LLaVA-1.5-13B's 5120) */
int rlaifv_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd,
                       const void* dres_or_null, void* dx, void* dw, int dw_accumulate, float* workspace,
                       int M, int H, void* stream);
int rlaifv_layernorm_fwd(const void* x, const void* w, const void* b, void* y, int M, int H, float eps,
                         void* stream);
/* LayerNorm backward for the resampler's trainable ln_q / ln_kv / ln_post (omnilmm/model/resampler.py:137-141;
 * eps 1e-6, :110): statistics recomputed from x; dw/db bf16 [H] overwritten or accumulated; workspace fp32
 * [2 * rlaifv_rmsnorm_bwd_partials() * H]. */
int rlaifv_layernorm_bwd(const void* dy, const void* x, const void* w, void* dx, void* dw, void* db, int accumulate,
                         float* workspace, int M, int H, float eps, void* stream);
/* y[r] = x[r] + table[r % P]: the resampler's position-embedding adds (resampler.py:158-161), table shared by the
 * batch. */
int rlaifv_add_rows_bcast(const void* x, const void* table, void* y, long long M, int P, int H, void* stream);

/* ---- RoPE on the fused qkv buffer (HF:llama/modeling_llama.py:124-168; positions 0..T-1 because
 * position_ids are not forwarded, llava_llama.py:94). cos/sin: bf16 [T][head_dim]. In place. */
int rlaifv_rope_fwd(void* qkv, const void* cos_tab, const void* sin_tab, long long M, int T, int n_heads,
                    int head_dim, long long ld, void* stream);
int rlaifv_rope_bwd(void* dqkv, const float* dq_f32, const void* cos_tab, const void* sin_tab, long long M,
                    int T, int n_heads, int head_dim, long long ld, void* stream);

/* ---- SwiGLU on the fused [gate | up] buffer (HF:llama/modeling_llama.py:182-184), GELU of the projector */
int rlaifv_swiglu_fwd(const void* gu, void* act, long long M, int F, void* stream);
int rlaifv_swiglu_bwd(const void* gu, const void* dact, void* dgu, long long M, int F, void* stream);
int rlaifv_gelu_fwd(const void* pre, void* post, long long n, void* stream);
int rlaifv_gelu_bwd(const void* pre, const void* dpost, void* dpre, long long n, void* stream);
int rlaifv_colsum(const void* x, long long M, int N, void* db, int accumulate, float* workspace_64xN,
                  void* stream);

/* Dropout on the LoRA adapter input (peft lora.Linear, lora_dropout = 0.05, train_llava15_lora.py:115). The keep
 * bit of element i is a stateless hash of (seed, i): dropout_bwd_add regenerates the mask (dx += keep ? g/(1-p) : 0). */
int rlaifv_dropout_fwd(const void* x, void* out, long long n, float p, unsigned long long seed, void* stream);
int rlaifv_dropout_bwd_add(void* dx, const void* g, long long n, float p, unsigned long long seed, void* stream);

/* ---- CLIP embedding helpers (HF:clip/modeling_clip.py:202-219; clip_encoder.py:36-44) ----------- */
int rlaifv_clip_im2col(const void* images, void* out, int n_img, int channels, int size, int patch,
                       int k_pad, void* stream);
int rlaifv_clip_embed(const void* patch, const void* cls, const void* pos, void* x, int n_img, int n_patch,
                      int H, void* stream);
int rlaifv_clip_drop_cls(const void* x, void* out, int n_img, int n_patch, int H, void* stream);

/* ---- image-token splice (llava/model/llava_arch.py:150-330, attention_mask=None path) -----------
 * ids/labels int64 [nseq][L]; IMAGE_TOKEN_INDEX = -200, IGNORE_INDEX = -100. Integer outputs are
 * bit-exact w.r.t. the reference; row gathers are pure copies.
 *   splice_count : n_img[b], len[b] = min(L - n_img + n_img*P, max_len)
 *   splice_map   : src[b][t] (>=0 token position, -1-r feature row r, INT_MIN pad), new_labels[b][t]
 *   splice_gather: out[b][t][:] = embed[ids[b][src]] | feat[r] | 0
 *   splice_scatter: backward (fp32 atomics into d_embed [V][H] / d_feat [rows][H]) */
int rlaifv_splice_count(const long long* ids, int nseq, int L, int P, int max_len, int* n_img, int* len,
                        void* stream);
int rlaifv_splice_map(const long long* ids, const long long* labels, const int* n_img, const int* img_index,
                      int nseq, int L, int P, int T, int max_len, int* src, long long* new_labels,
                      void* stream);
/* OmniLMM in-place splice map (omnilmm/model/omnilmm.py:219-258): src[b][t] = t for text rows, -1-(block*num_query+j)
 * for the j-th row after an <im_start>; blocks consumed in batch order through img_index; length unchanged.
 * status (int32[1], zeroed by the caller): bit0 = unequal <im_start>/<im_end> counts, bit1 = <im_end> not at
 * start+num_query+1 — the two ValueErrors of omnilmm.py:234-247. */
int rlaifv_splice_map_inplace(const long long* ids, const int* img_index, int nseq, int L, int num_query,
                              long long im_patch, long long im_start, long long im_end, int* src, int* status,
                              void* stream);
int rlaifv_splice_gather(const int* src, const long long* ids, const void* embed, const void* feat, void* out,
                         int nseq, int L, int T, int H, void* stream);
int rlaifv_splice_scatter(const int* src, const long long* ids, const void* dx, float* d_embed, float* d_feat,
                          int nseq, int L, int T, int H, void* stream);
int rlaifv_f32_to_bf16(const float* in, void* out, long long n, int accumulate, void* stream);
/* Strided form: fp32 [rows, cols] (row stride ld_in) -> bf16 column block (row stride ld_out); used where an fp32
 * atomic accumulator (attention dQ) lands in the q columns of a fused dqkv buffer without RoPE (EVA tower). */
int rlaifv_f32_to_bf16_2d(const float* in, long long ld_in, void* out, long long ld_out, long long rows, int cols,
                          int accumulate, void* stream);

/* ---- compact lm_head: only positions whose next token is supervised reach the head -----------------
 * get_batch_logps (muffin/eval/muffin_inference_logp.py:93-104) multiplies the per-token log-probs by
 * loss_mask = labels[:, 1:] != -100 before summing, so in TRAINING the final norm, lm_head GEMM (fwd, dgrad, wgrad) and
 * the log-softmax only need those rows (512 of 1135 per config-(b) sequence). row_pos int32 [nseq*cap]:
 * row_pos[s*cap + j] = s*T + t of sequence s's j-th supervised position, -1 in unused slots (cap >= labels per row).
 * rows_gather: out[r] = x[row_pos[r]] (zeros for -1); rows_scatter: dx[row_pos[r]] = dy[r] (dx pre-zeroed).
 * rlaifv_logp_fwd / rlaifv_logp_bwd take this row_pos to run the log-prob head on the gathered rows. */
/* Token weights [nseq][Lw] in TEXT positions (collator: weight i belongs to token i+1) -> [nseq][T-1] in SPLICED
 * positions via the splice map src [nseq][T] (image rows / padding -> 1). Extension beyond the reference, which refuses
 * --dpo_token_weighted for LLaVA-1.5 (muffin/train/trainers.py:246-248). */
int rlaifv_splice_token_weight(const int* src, const float* token_weight, float* out, int nseq, int Lw, int T, void* stream);
int rlaifv_supervised_rows(const long long* labels, int nseq, int T, int cap, int* row_pos, void* stream);
int rlaifv_rows_gather(const int* row_pos, const void* x, void* out, long long n_rows, int H, void* stream);
int rlaifv_rows_scatter(const int* row_pos, const void* dy, void* dx, long long n_rows, int H, void* stream);

/* ---- per-token log-prob gather (muffin/eval/muffin_inference_logp.py:82-115) ---------------------
 * logits bf16, upcast to fp32 inside as pinned transformers 4.35 does; labels = spliced labels [nseq][T].
 * row_pos NULL: the full head, logits [nseq*T][ld], lse [nseq][T]. row_pos given: the compact head above, logits
 * [n_rows][ld] of the gathered rows, lse [n_rows], per_tok pre-zeroed by the caller. per_tok [nseq][T-1],
 * logp_sum/logp_avg/count [nseq].
 * logp_bwd overwrites logits with d loss / d logits given d loss / d logp_sum, in the same layout. token_weight
 * (nullable) scales each row by its weight (the token-weighted loss below); norm != NULL is average mode: the label
 * count, or the weight sum when weighted. */
int rlaifv_logp_fwd(const void* logits, long long ld, const long long* labels, const int* row_pos, long long n_rows,
                    int nseq, int T, int V, float* per_tok, float* lse, float* logp_sum, float* logp_avg, float* count,
                    void* stream);
int rlaifv_logp_bwd(void* logits, long long ld, const long long* labels, const int* row_pos, long long n_rows,
                    const float* lse, const float* d_logp, const float* token_weight, const float* norm, int nseq,
                    int T, int V, void* stream);

/* Token-weighted log-prob reduction: compute_weighted_logp (muffin/train/trainers.py:128-137), used by the
 * `dpo_token_weighted` branch of get_beta_and_logps (:246-261; the reference raises NotImplementedError for LLaVA-1.5
 * there, so this serves the OmniLMM path). token_weight fp32 [nseq][T-1]; weighted_mask = weight * (label != -100);
 * logp_w = sum per_tok * weighted_mask, avg_w = logp_w / sum weighted_mask (wsum). Its backward is rlaifv_logp_bwd
 * with token_weight (and norm = wsum in average mode). */
int rlaifv_logp_weighted_reduce(const float* per_tok, const long long* labels, const float* token_weight, int nseq,
                                int T, float* logp_w, float* avg_w, float* wsum_or_null, void* stream);

/* ---- DPO loss + gradient (muffin/train/trainers.py:91-126, :279-311) ---------------------------
 * out9: [0] loss = DPO_w*mean(losses) - SFT_w*mean(pw); [1..8] local means of chosen_reward,
 * rejected_reward, accuracy, margin, logp_rejected, logp_chosen, ref_rejected, ref_chosen. */
int rlaifv_dpo_loss(const float* policy_win, const float* policy_rej, const float* ref_win,
                    const float* ref_rej, int B, float beta, float dpo_weight, float sft_weight,
                    float grad_scale, float* losses, float* chosen_rewards, float* rejected_rewards,
                    float* d_policy_win, float* d_policy_rej, float* out9, void* stream);

/* ---- fused AdamW on a flat shard (torch.optim.AdamW; optim=adamw_torch, muffin/train/train_llava15.py:75;
 * fp32 master/moments as under DeepSpeed bf16 + ZeRO-2, script/zero2.json). */
int rlaifv_adamw_step(float* master, float* exp_avg, float* exp_avg_sq, const void* grad, int grad_is_f32,
                      void* param_bf16, long long n, float lr, float beta1, float beta2, float eps,
                      float weight_decay, int step, float grad_scale, void* stream);

/* AdamW of one bucket whose fp32 state lives in PINNED HOST memory (the offloaded optimizer, zero2.OffloadAdamW; the
 * DeepSpeed `offload_optimizer: {device: cpu}` of script/zero2_offload.json, with the update kept on the GPU).
 * host_master / host_exp_avg / host_exp_avg_sq: n fp32 each, page-locked (cudaHostRegister / cudaHostAlloc) and owned
 * by the caller; this is the one entry point that takes host pointers. grad / param_bf16: the bucket's bf16 gradient
 * and parameters (n each, device). ring: caller-owned device staging ring of n_slots (2..8) slots, each holding
 * master | m | v of slot_elems (% 4 == 0) floats. The state is streamed through the ring chunk by chunk: H2D on
 * h2d_stream, the update on `stream` (same per-element arithmetic as rlaifv_adamw_step, grad_scale 1, weight decay on
 * elements [0, decay_n)), D2H on d2h_stream, ordered by events only; with 3 slots the H2D of chunk i+1, the update of
 * chunk i and the D2H of chunk i-1 overlap. On return, everything is enqueued: the parameters are final once `stream`
 * reaches its current end, the host state once d2h_stream does. The caller orders h2d_stream after the previous D2H of
 * the same host range. Pageable host or device memory where pinned host memory is expected (and host memory where
 * device memory is expected) returns -1. The library keeps one set of events per (device, ring), created on the ring's
 * first call; it allocates no memory. */
int rlaifv_adamw_offload_bucket(float* host_master, float* host_exp_avg, float* host_exp_avg_sq, const void* grad,
                                void* param_bf16, long long n, long long decay_n, float* ring, int n_slots,
                                long long slot_elems, float lr, float beta1, float beta2, float eps, float weight_decay,
                                int step, void* stream, void* h2d_stream, void* d2h_stream);
/* Destroys the events rlaifv_adamw_offload_bucket / rlaifv_adamw8bit_offload_bucket keep for `ring` on the current
 * device (no-op if there are none). Call it once the ring's work has completed and before the ring is freed; a later
 * call with the same ring starts a fresh set. */
int rlaifv_adamw_offload_release(const void* ring);

/* ---- AdamW with blockwise 8-bit moments (optim=adamw_bnb_8bit / adamw_8bit: bitsandbytes AdamW8bit, Dettmers et
 * al. 2022, percentile clipping off). State per element: fp32 master, one uint8 code each for m and v; per block of
 * 256 consecutive elements (counted from the slice's first element; the last block may be partial) one fp32
 * absmax_m and absmax_v. m = map_m[code_m] * absmax_m, v = map_v[code_v] * absmax_v; map_m / map_v: the signed /
 * unsigned 256-entry dynamic maps (device, strictly increasing fp32, zero2.dynamic_map). Per block: dequantize, the
 * per-element arithmetic of rlaifv_adamw_step (grad_scale 1, weight decay on elements [0, decay_n)), write master and
 * bf16(master), set absmax_m = max|m| and absmax_v = max v over the new fp32 moments, store for each element the code
 * of the map entry nearest to m / absmax_m (v / absmax_v), ties to the lower index, the code of 0 for a zero absmax.
 *
 * One slice of n (% 8 == 0) elements on the device: codes n bytes each (8-byte aligned), absmax ceil(n / 256) floats
 * each; master, grad and param_bf16 16-byte aligned. */
int rlaifv_adamw8bit_step(float* master, uint8_t* code_m, uint8_t* code_v, float* absmax_m, float* absmax_v,
                          const void* grad, void* param_bf16, long long n, long long decay_n, const float* map_m,
                          const float* map_v, float lr, float beta1, float beta2, float eps, float weight_decay,
                          int step, void* stream);
/* The same update of one bucket whose state lives in PINNED HOST memory, through the chunk / slot / event pipeline of
 * rlaifv_adamw_offload_bucket (same streams, same ordering, same release). host_master: n fp32; host_code_m /
 * host_code_v: n bytes; host_absmax_m / host_absmax_v: ceil(n / 256) fp32. ring: caller-owned, 256-byte aligned device
 * memory of n_slots (2..8) slots of slot_bytes = round_up(6 * slot_elems + 8 * slot_elems / 256, 256) bytes, each
 * holding master | code_m | code_v | absmax_m | absmax_v of slot_elems (% 256 == 0) elements, so every chunk starts
 * on a block edge. Bad sizes, misalignment and pageable host memory return -1. */
int rlaifv_adamw8bit_offload_bucket(float* host_master, uint8_t* host_code_m, uint8_t* host_code_v,
                                    float* host_absmax_m, float* host_absmax_v, const void* grad, void* param_bf16,
                                    long long n, long long decay_n, const float* map_m, const float* map_v, void* ring,
                                    int n_slots, long long slot_elems, float lr, float beta1, float beta2, float eps,
                                    float weight_decay, int step, void* stream, void* h2d_stream, void* d2h_stream);

/* ---- FP8 (e4m3) frozen base of LoRA training (DESIGN.md §3 "FP8 frozen base"). Format: a tile (1 x 128 of an
 * operand row, or a 128 x 128 block of a weight) with amax = max|x| has the scale s = 2^e, e the smallest integer with
 * amax <= 448 * 2^e clamped to [-126, 127] (s = 1 for amax = 0), and the codes RNE_e4m3(x / s); x / s is exact and
 * never saturates. oracle/fp8_oracle.py is the reference. K and N must be multiples of 128.
 * rlaifv_quant_fp8_rows: x [M, K] bf16 (row stride ldx) -> codes q [M, K] (ldq bytes, multiple of 16) and the row
 * scales s [K / 128][ld_s] fp32 (ld_s >= M, multiple of 4: the rows of one K-block are contiguous). */
int rlaifv_quant_fp8_rows(const void* x, long long ldx, void* q, long long ldq, float* s, long long ld_s, int M, int K,
                          void* stream);
/* W [N, K] bf16 -> W codes q [N, K] (ldq), W^T codes qt [K, N] (ldt; the byte-for-byte transpose of q) and the block
 * scales s [N / 128][ld_s] (ld_s >= K / 128). Once per weight, when the model loads. */
int rlaifv_quant_fp8_blocks(const void* w, long long ldw, void* q, long long ldq, void* qt, long long ldt, float* s,
                            long long ld_s, int N, int K, void* stream);
/* C[m, n] = sum_kb sa[kb][m] * sb(n / 128, kb) * sum_{k in kb} A[m, k] * B[n, k] over e4m3 codes (A [M, K], lda
 * bytes; B [N, K], ldb bytes), each 128-deep K-block accumulated apart and promoted in fp32, then
 * + A2[:, koff : koff + K2] * B2^T (bf16, as rlaifv_gemm_bf16_dual: koff = (n0 / n_sub) * r, n_sub % 128 == 0),
 * then one of: C = bf16(acc); C = bf16(bf16(acc) + residual) (residual [M, ldr]); glu != NULL: the SwiGLU-backward
 * epilogue of rlaifv_gemm_bf16_swiglu_bwd (N = F, glu = [gate | up] [M, ld_glu], C = d[gate | up] [M, 2F]).
 * sb: the block scales of a weight W [N_w, K_w] ([N_w / 128][K_w / 128]). b_t = 0: B is W (forward), sb(nb, kb) =
 * sb[nb * K / 128 + kb]; b_t = 1: B is W^T (dgrad), sb(nb, kb) = sb[kb * N / 128 + nb], and B2 is MN-major
 * ([K2, N], as rlaifv_gemm_bf16_dual with b_mn_major = 1). C and the residual are 16-byte aligned, ldc and ldr
 * multiples of 8; C may be a column block of a wider buffer. */
int rlaifv_gemm_fp8(const void* A, long long lda, const float* sa, long long ld_sa, const void* B, long long ldb,
                    const float* sb, int b_t, const void* A2, long long lda2, const void* B2, long long ldb2, int K2,
                    int r, int n_sub, void* C, long long ldc, int M, int N, int K, const void* residual, long long ldr,
                    const void* glu, long long ld_glu, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RLAIFV_B200_H_ */
