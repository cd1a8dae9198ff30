/*
 * hpc_b200.h — C ABI of the H100 (sm_90a) build of the HPC-Ops quantized-inference hot path.
 *
 * Every entry point is `extern "C"`, takes raw device/host pointers, plain integer sizes and
 * ELEMENT strides, float scalars and a cudaStream_t last — the same shape as the reference's
 * L1 host launchers (`*_async(void*…, cudaStream_t)`), which is what the reference's torch op
 * entries (src/<op>/entry.cc) bind.  No torch types cross this boundary.
 *
 * Return value: HPC_OK (0) or an HPC_ERR_* code; `hpc_last_error()` returns a thread-local,
 * human-readable message for the last failure (the Python layer raises RuntimeError with it,
 * mirroring the reference's TORCH_CHECK behaviour).
 *
 * Nothing here falls back to the CPU: a launcher either enqueues sm_90a kernels on `stream`
 * or fails loudly.
 *
 * The Python package binds its ctypes argtypes from this file (hpc/_ffi.py `bind`), so a
 * declaration may only use int, int64_t, uint64_t, float, double, pointers and cudaStream_t
 * parameters, (void), and int, int64_t or const char* returns; anything else fails the CPU tests.
 */
#ifndef INCLUDE_HPC_B200_H_
#define INCLUDE_HPC_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef __CUDA_RUNTIME_API_H__
typedef struct CUstream_st* cudaStream_t;
#endif

enum {
  HPC_OK = 0,
  HPC_ERR_UNSUPPORTED = 1, /* shape / dtype / argument rejected (reference: TORCH_CHECK) */
  HPC_ERR_CUDA = 2,        /* a CUDA runtime call failed                                  */
  HPC_ERR_DRIVER = 3       /* a CUDA driver entry point (TMA descriptor encode) failed    */
};

/* ---- library ------------------------------------------------------------------------------- */
const char* hpc_last_error(void);
int hpc_sm_count(void);
/* replaces torch.ops.hpc.version / built_json (reference src/C/version.cc, src/C/built_json.cu) */
const char* hpc_version(void);
const char* hpc_built_json(void);

/* ---- decode attention: dynamic split-k task map ---------------------------------------------
 * replaces reference src/attention/decode/decode.h:39-46
 *   assign_attention_decode_task_sync  (CPU)  / assign_attention_decode_task_async (CUDA)
 * The CPU variant writes the packed host map of reference src/attention/entry.cc:750-776:
 *   row 0 = {num_tile_per_cta+1, num_total_ctas, 0,0,0, max_num_chunks}, then
 *   num_total_ctas*(num_tile_per_cta+1) 48-byte task rows, then num_chunks[h*num_batch+b].
 * The CUDA variant fills a workspace from get_attention_decode_task_workspace (hpc/attention.py).
 */
int64_t hpc_assign_attention_decode_task_host_bytes(const int* num_seq_kvcache,
                                                    int num_total_ctas, int num_batch,
                                                    int num_head_kv, int num_seq_q, int tilen,
                                                    int new_kv_included, int min_process_len);
int hpc_assign_attention_decode_task_sync(const int* num_seq_kvcache, int num_total_ctas,
                                          int num_batch, int num_head_kv, int num_seq_q, int tilen,
                                          int new_kv_included, int min_process_len,
                                          void* task_map_host, int64_t task_map_bytes);
int hpc_assign_attention_decode_task_async(int* task_map, const int* num_seq_kvcache,
                                           int num_total_ctas, int num_batch, int num_head_kv,
                                           int num_seq_q, int tilen, int new_kv_included,
                                           int min_process_len, cudaStream_t stream);

/* ---- decode attention: FP8 paged KV, split-k partials + combine -----------------------------
 * replaces reference src/attention/decode/decode.h:28-37 (attention_decode_fp8_async);
 * argument order and meaning are identical (strides in elements == bytes for fp8).
 *   lse        f32 [num_batch, splitk, num_head_k, num_seq_q, pad8(heads_per_group)]
 *   split_out  f32 [num_batch, splitk, num_seq_q, num_head_q, num_dim_v]
 *   splitk     = num_total_ctas of the task map (max chunks per (batch, kv head))
 */
int hpc_attention_decode_fp8_async(
    void* y_ptr, void* lse_ptr, void* split_out_ptr, const int* task_map_ptr, const void* q_ptr,
    void* kcache_ptr, void* vcache_ptr, const int* block_ids_ptr, const int* num_seq_kvcache_ptr,
    const float* qscale_ptr, const float* kscale_ptr, const float* vscale_ptr, int* split_flag_ptr,
    int new_kv_included, int splitk, int splitk_min_len, int consumers, int quant_type,
    int num_batch, int num_seq_q, int num_head_q, int num_head_k, int num_head_v, int num_dim_qk,
    int num_dim_v, int num_kvcache_blocks, int block_size, int num_seq_max_blocks,
    int qscale_pad_stride, int ldY, int ldQ, int64_t kcache_block_stride,
    int64_t kcache_token_stride, int64_t kcache_head_stride, int64_t vcache_block_stride,
    int64_t vcache_token_stride, int64_t vcache_head_stride, cudaStream_t stream);

/* ---- decode attention: BF16 paged KV (block size 16 / 32 / 64) --------------------------------
 * replaces reference src/attention/decode/decode.h:16-25 (attention_decode_bf16_async); argument
 * order and meaning are identical (strides in bf16 elements). lse / split_out as above. */
int hpc_attention_decode_bf16_async(
    void* y_ptr, void* lse_ptr, void* split_out_ptr, const int* task_map_ptr, const void* q_ptr,
    void* kcache_ptr, void* vcache_ptr, const int* block_ids_ptr, const int* num_seq_kvcache_ptr,
    int* split_flag_ptr, int new_kv_included, int splitk, int num_batch, int num_seq_q,
    int num_head_q, int num_head_k, int num_head_v, int num_dim_qk, int num_dim_v,
    int num_kvcache_blocks, int block_size, int num_seq_max_blocks, int ldY, int ldQ,
    int64_t kcache_block_stride, int64_t kcache_token_stride, int64_t kcache_head_stride,
    int64_t vcache_block_stride, int64_t vcache_token_stride, int64_t vcache_head_stride,
    cudaStream_t stream);

/* ---- decode attention: absorbed MLA over a paged bf16 latent cache -----------------------------
 * y[b * Sq + sq, h, :512] = softmax_k(q[b * Sq + sq, h, :] . kv[k, :] * softmax_scale) . kv[k, :512]
 * over the n = num_seq_kvcache[b] (+ Sq unless new kv is included) cached tokens of request b; MTP
 * row sq sees keys k <= n - Sq + sq. q: [B * Sq, H, 576] bf16, heads contiguous (576 apart), row
 * stride ldQ; kv: [num_kvcache_blocks, 64, 576] bf16 with token / block strides in elements
 * (multiples of 8); y: [B * Sq, H, 512] bf16 with row stride ldY. H in {8, 16, 32, 64, 128}, Sq
 * 1..4, B <= 2048. Cache slots past a request's last token never reach y, whatever they hold.
 *   task_map   : the decode task map built with num_head_kv = T = ceil(H * Sq / 64) (query tiles)
 *                for the same num_total_ctas (the grid)
 *   workspace  : fp32, 2 * C * 64 * 513 + C * (256 * 128 + 512) floats for C = num_total_ctas
 *                (split-chunk partials and LSEs, and the rotated walk's carried state); any contents
 *   chunk_base : int32 [B * T], any contents
 * No allocation and no host synchronisation: capturable in a CUDA graph. */
int hpc_attention_decode_mla_bf16_async(
    void* y_ptr, void* workspace_ptr, int* chunk_base_ptr, const int* task_map_ptr,
    const void* q_ptr, const void* kv_ptr, const int* block_ids_ptr, int num_batch,
    int num_seq_q, int num_head_q, int num_dim_qk, int num_kvcache_blocks, int block_size,
    int num_seq_max_blocks, int ldY, int ldQ, int64_t kv_block_stride, int64_t kv_token_stride,
    float softmax_scale, int num_total_ctas, cudaStream_t stream);

/* The two stages of hpc_attention_decode_fp8_async on their own, same argument list: the split-k
 * attention kernel (writes lse / split_out) and the LSE combine (reads them, writes y). The
 * reference launches them back to back inside one launcher
 * (src/attention/decode/sm90/dynamic/...dynamic.cu:44-195); they are exposed separately so the
 * dominant kernel can be timed alone. */
int hpc_attention_decode_fp8_partial_async(
    void* y_ptr, void* lse_ptr, void* split_out_ptr, const int* task_map_ptr, const void* q_ptr,
    void* kcache_ptr, void* vcache_ptr, const int* block_ids_ptr, const int* num_seq_kvcache_ptr,
    const float* qscale_ptr, const float* kscale_ptr, const float* vscale_ptr, int* split_flag_ptr,
    int new_kv_included, int splitk, int splitk_min_len, int consumers, int quant_type,
    int num_batch, int num_seq_q, int num_head_q, int num_head_k, int num_head_v, int num_dim_qk,
    int num_dim_v, int num_kvcache_blocks, int block_size, int num_seq_max_blocks,
    int qscale_pad_stride, int ldY, int ldQ, int64_t kcache_block_stride,
    int64_t kcache_token_stride, int64_t kcache_head_stride, int64_t vcache_block_stride,
    int64_t vcache_token_stride, int64_t vcache_head_stride, cudaStream_t stream);
int hpc_attention_decode_fp8_combine_async(
    void* y_ptr, void* lse_ptr, void* split_out_ptr, const int* task_map_ptr, const void* q_ptr,
    void* kcache_ptr, void* vcache_ptr, const int* block_ids_ptr, const int* num_seq_kvcache_ptr,
    const float* qscale_ptr, const float* kscale_ptr, const float* vscale_ptr, int* split_flag_ptr,
    int new_kv_included, int splitk, int splitk_min_len, int consumers, int quant_type,
    int num_batch, int num_seq_q, int num_head_q, int num_head_k, int num_head_v, int num_dim_qk,
    int num_dim_v, int num_kvcache_blocks, int block_size, int num_seq_max_blocks,
    int qscale_pad_stride, int ldY, int ldQ, int64_t kcache_block_stride,
    int64_t kcache_token_stride, int64_t kcache_head_stride, int64_t vcache_block_stride,
    int64_t vcache_token_stride, int64_t vcache_head_stride, cudaStream_t stream);

/* ---- grouped FP8 GEMM -------------------------------------------------------------------------
 * replaces reference src/group_gemm/group_gemm.h:12-29. X [m, k] e4m3 with the rows of group g at
 * cu_seqlens[g] .. +seqlens[g]; W [num_group, n, k] e4m3; Y [m, n] bf16.
 *   blockwise : xscale f32 [k/128, m_pad] (column of row i of group g = sum_{g'<g} pad(seqlens[g'],
 *               tile(num_seq_per_group_avg)) + i), wscale f32 [num_group, n/128, num_block_k_pad4]
 *   per-tensor: y_scale f32 [num_group]
 * tmas / tiles / cu_tiles / task_map / num_waves / update_tma / use_pdl are accepted and ignored
 * (the kernel derives its schedule on the device).
 */
int hpc_group_gemm_blockwise_fp8_async(
    void* y_ptr, const void* x_ptr, const void* w_ptr, const void* seqlens_ptr,
    const void* cu_seqlens_ptr, const void* xscale_ptr, const void* wscale_ptr, void* tmas_ptr,
    void* tiles_ptr, void* cu_tiles_ptr, void* task_map_ptr, int num_waves, int num_group, int m,
    int n, int k, int m_pad, int num_block_k_pad4, int num_seq_per_group_avg, int update_tma,
    int use_pdl, cudaStream_t stream);
int hpc_group_gemm_fp8_async(void* y_ptr, const void* x_ptr, const void* w_ptr,
                             const void* seqlens_ptr, const void* cu_seqlens_ptr,
                             const void* y_scale, void* tmas_ptr, void* tiles_ptr,
                             void* cu_tiles_ptr, void* task_map_ptr, int num_waves, int num_group,
                             int m, int n, int k, int num_seq_per_group_avg, int update_tma,
                             int use_pdl, cudaStream_t stream);
/* Column granule of the transposed activation-scale layout for a given average of rows per group:
 * 8 / 16 / 32 / 48 / 64 up to 64 rows, then 48 (<= 96), 32 (<= 128), 48 (<= 144) and 64. The blockwise
 * GEMMs read that layout with this granule; pass it as `tilem` to hpc_reformat_x_scale_async. */
int hpc_scale_tile_from_avg(int num_seq_per_group_avg);
/* replaces reference src/group_gemm/group_gemm.h:31-33 (row-major [m, n] scales -> transposed,
 * tile-padded [n, m] layout the blockwise GEMM reads) */
int hpc_reformat_x_scale_async(void* output_ptr, const void* xscale_ptr, const void* seqlens_ptr,
                               const void* cu_seqlens_ptr, int num_group, int m, int n, int tilem,
                               cudaStream_t stream);

/* replaces reference src/group_gemm/cp_async/group_gemm.h:11-24 (the small-M cp.async grouped GEMMs:
 * y[rows of g] = (x[rows of g] . w[g]^T) * y_scale[g], bf16 out). Served by the same wgmma grouped
 * GEMM; tiles / cu_tiles / task_map are accepted and ignored. The scatter variant reads row i of
 * the compact problem from row row_indices[i] of the pool x [pool_rows, k]; it needs an e4m3
 * scratch of m * k bytes (gather_ptr) because the gather runs as a streaming pre-pass. */
int hpc_group_gemm_fp8_multistage_async(
    void* y_ptr, const void* x_ptr, const void* w_ptr, const void* y_scale_ptr,
    const void* seqlens_ptr, const void* cu_seqlens_ptr, const void* tiles_ptr,
    const void* cu_tiles_ptr, const void* task_map_ptr, int task_map_len, int m, int n, int k,
    int num_group, int num_seq_per_group_avg, int use_pdl, cudaStream_t stream);
int hpc_group_gemm_fp8_scatter_async(
    void* y_ptr, const void* x_ptr, const void* w_ptr, const void* y_scale_ptr,
    const void* row_indices_ptr, const void* seqlens_ptr, const void* cu_seqlens_ptr,
    const void* tiles_ptr, const void* cu_tiles_ptr, const void* task_map_ptr, int task_map_len,
    int m, int n, int k, int num_group, int num_seq_per_group_avg, int use_pdl, void* gather_ptr,
    int pool_rows, cudaStream_t stream);

/* ---- stand-alone activation / quantisation (HBM-bound streaming kernels) --------------------------
 * replace reference src/activation/activation.h:15-17 (act_mul_and_quant_async: gate_up bf16
 * [num_row, num_col = 2C] -> e4m3 [num_row, C] = silu(gate) * up * scale[0], optional bf16-rounded
 * multiply) and :46-53 (scaled_fp8_quant_async: out = e4m3(in / scale[0]); in_dtype 0 = f32,
 * 1 = f16, 2 = bf16). */
int hpc_act_mul_and_quant_async(void* y_ptr, const void* x_ptr, const float* scale_ptr, int num_row,
                                int num_col, int use_bf16_mul, cudaStream_t stream);
int hpc_scaled_fp8_quant_async(void* y_ptr, const void* x_ptr, const float* scale_ptr,
                               int64_t numel, int in_dtype, cudaStream_t stream);
/* Masked (per-expert padded, DeepEP low-latency) layout: input bf16 [N = E * T_max, 2C], rows
 * e * T_max + t with t < clamp(num_per_expert[e], 0, T_max) valid (num_per_expert int32 [E] on the
 * device), N % T_max == 0, 16-byte aligned input. Only valid rows of the outputs are written; the
 * others keep whatever the caller's buffer held. Per-tensor: e4m3(silu(gate) * up * scale[0]) in
 * fp32 (act_mul_and_quant with use_bf16_mul = 0), C % 8 == 0. Blockwise: per (row, 128 columns)
 * sc = amax / 448, out = e4m3(v / (sc + 1e-8)), output_scale f32 row-major [N, C / 128],
 * C % 128 == 0. Stream-ordered, no allocation or host synchronisation: capturable. */
int hpc_masked_act_mul_and_quant_async(void* output_ptr, const void* input_ptr,
                                       const float* scale_ptr, const int* num_per_expert_ptr,
                                       int num_total_tokens, int num_intermediate_size,
                                       int num_tokens_per_expert, cudaStream_t stream);
int hpc_masked_act_mul_and_blockwise_quant_async(void* output_ptr, float* output_scale_ptr,
                                                 const void* input_ptr,
                                                 const int* num_per_expert_ptr,
                                                 int num_total_tokens, int num_intermediate_size,
                                                 int num_tokens_per_expert, cudaStream_t stream);
/* 1x128 blockwise activation quantiser, no reference counterpart: input bf16 [num_row, num_col]
 * (elements of a row contiguous, input_ld elements between rows, a multiple of 8, 16-byte aligned
 * base), num_col % 128 == 0. Per (row, 128 columns), in fp32: sc = amax / 448, output e4m3
 * [num_row, num_col] = e4m3_rn_satfinite(v * (1 / (sc + 1e-8))), output_scale f32 row-major
 * [num_row, num_col / 128] = sc: the x / x_scale pair of hpc_gemm_blockwise_fp8_async and of the
 * blockwise FusedMoE. num_row = 0 launches nothing. PDL launch, no allocation or host
 * synchronisation: capturable. */
int hpc_blockwise_fp8_quant_async(void* output_ptr, float* output_scale_ptr, const void* input_ptr,
                                  int num_row, int num_col, int64_t input_ld, cudaStream_t stream);

/* ---- dense blockwise FP8 GEMM ---------------------------------------------------------------------
 * No reference counterpart: the linear layers of a blockwise-FP8 checkpoint.
 *   y [m, n] bf16 = x [m, k] e4m3 . w [n, k]^T e4m3 with x_scale f32 [m, k / 128] and w_scale f32
 *   [ceil(n / 128), k / 128], all contiguous and 16-byte aligned.
 * Per 128-column K block kb in ascending order: P = e4m3 wgmma products accumulated over the block's
 * four k = 32 steps from zero, acc = fmaf(P, fl32(x_scale[m, kb] * w_scale[n / 128, kb]), acc); with
 * a K split each split does this over its contiguous share of the K blocks and the split partials
 * are added in fp32 in split order; y = bf16_rn(acc). Deterministic. k % 128 == 0, 128 <= k <=
 * 65536, n % 8 == 0 (a ragged last weight-scale block is allowed), any m >= 0 (0 launches nothing),
 * checked before any launch. PDL launch, no allocation or host synchronisation: capturable.
 * hpc_gemm_blockwise_fp8_config returns the K split (1, 2, 4 or 8; the tile is always 128 x 128)
 * the launcher picks for a shape on the current device. */
int hpc_gemm_blockwise_fp8_config(int m, int n, int k);
int hpc_gemm_blockwise_fp8_async(void* y_ptr, const void* x_ptr, const float* x_scale_ptr,
                                 const void* w_ptr, const float* w_scale_ptr, int m, int n, int k,
                                 cudaStream_t stream);

/* ---- fused RMSNorm -> FP8 --------------------------------------------------------------------------
 * replaces reference src/normalization/fused_rmsnorm_with_scale.h. input bf16 [batch_size,
 * hidden_state] (rows contiguous), weight bf16 [hidden_state], scale f32 on the device ([1], or [2]
 * with is_moe). y = (x * w) * rsqrtf(sum(x^2) / H + eps) in fp32; output = e4m3_rn_satfinite(
 * y * (1 / scale[0])); with is_moe also output_fp32 = y and output_fp8_scale2 =
 * e4m3_rn_satfinite(y * (1 / scale[1])). Any hidden_state % 8 == 0 in [8, 16384]. Capturable. */
int hpc_fused_rmsnorm_with_scale_async(const void* input_ptr, const void* weight_ptr,
                                       void* output_ptr, void* output_fp32_ptr,
                                       void* output_fp8_scale2_ptr, const void* scale_ptr,
                                       float eps, int batch_size, int hidden_state, int is_moe,
                                       cudaStream_t stream);

/* ---- MoE top-k gating -----------------------------------------------------------------------------
 * No reference counterpart: turns router logits into the topk_ids / topk_scale that FusedMoE
 * consumes. router_logits [num_tokens, num_experts] float32 (logits_dtype 0) or bfloat16 (1),
 * elements of a row contiguous, row_stride elements between rows (>= num_experts, a multiple of
 * 16 bytes; unused for a single row), 16-byte aligned base. scoring 0 = softmax over all experts,
 * 1 = sigmoid. correction_bias f32 [num_experts] or NULL. Per row, in fp32: key = logit (softmax
 * without bias) or score + bias; with num_expert_group G > 1 only the topk_group best groups
 * (max key, or sum of the top-2 keys with a bias) are eligible; the topk largest keys, ties to the
 * lower id, NaN below -inf, give topk_ids int32 [num_tokens, topk]; topk_weights f32
 * [num_tokens, topk] = the unbiased scores, divided by their sum (rank order) when renormalize,
 * then times routed_scaling_factor. 1 <= num_experts <= 512, 1 <= topk <= min(16, num_experts),
 * num_experts % G == 0, topk_group <= G, topk <= topk_group * num_experts / G, groups of at least
 * 2 experts with a bias. No allocation or host synchronisation: capturable. */
int hpc_moe_topk_gating_async(const void* router_logits_ptr, const float* correction_bias_ptr,
                              int* topk_ids_ptr, float* topk_weights_ptr, int num_tokens,
                              int num_experts, int logits_dtype, int topk, int scoring,
                              int renormalize, int num_expert_group, int topk_group,
                              int64_t row_stride, float routed_scaling_factor, cudaStream_t stream);

/* ---- FusedMoE -----------------------------------------------------------------------------------
 * replace reference src/fuse_moe/fuse_moe.h:15-62, argument for argument (bool -> int).
 * `intermediate_size` is gate_up_weight.size(1) (= 2*I) as in the reference entries.
 * In this build gate_up_output_ptr may be NULL: SiLU*mul + FP8 re-quant is the epilogue of the
 * Gate-Up GEMM and the bf16 Gate-Up matrix is never materialised.
 */
int hpc_count_and_gather_async(
    void* gate_up_input_ptr, void* gate_up_output_ptr, void* down_input_ptr, void* down_output_ptr,
    const void* x_ptr, const void* topk_ids_ptr, void* topk_pos_ptr, void* seqlens_ptr,
    void* cu_seqlens_ptr, void* gate_up_tmas_ptr, void* down_tmas_ptr, void* tiles_ptr,
    void* cu_tiles_ptr, void* gateup_task_map_ptr, void* down_task_map_ptr, int num_seq,
    int hidden_size, int intermediate_size, int num_topk, int num_expert, int eprank,
    int num_seq_per_group_avg, cudaStream_t stream);
int hpc_blockwise_count_and_gather_async(
    const void* input_ptr, const void* input_scale_ptr, void* gate_up_input_ptr,
    void* gate_up_output_ptr, void* gate_up_input_scale_ptr, void* down_input_ptr,
    void* down_output_ptr, const void* topk_ids_ptr, void* topk_pos_ptr,
    void* num_tokens_per_group_ptr, void* cu_num_tokens_per_group_ptr, void* gate_up_tmas_ptr,
    void* down_tmas_ptr, void* tiles_ptr, void* cu_tiles_ptr, void* gateup_task_map_ptr,
    void* down_task_map_ptr, int num_tokens, int num_padded_tokens, int hidden_size,
    int intermediate_size, int num_topk, int num_expert_local, int eprank,
    int num_tokens_per_group_avg, int use_pdl, cudaStream_t stream);
int hpc_reduce_async(void* y_ptr, const void* x_ptr, const void* topk_pos_ptr,
                     const void* topk_scale_ptr, const void* shared_output_ptr, int total_num_seq,
                     int num_seq, int hidden_size, int num_topk, int use_pdl, cudaStream_t stream);
int hpc_fuse_moe_async(
    void* output_ptr, const void* input_ptr, void* gate_up_input_ptr, void* gate_up_output_ptr,
    const void* gate_up_weight_ptr, const void* gate_up_scale_ptr, void* gate_up_tmas_ptr,
    const void* act_and_mul_scale_ptr, void* down_input_ptr, void* down_output_ptr,
    const void* down_weight_ptr, const void* down_scale_ptr, void* down_tmas_ptr,
    const void* topk_ids_ptr, const void* topk_scale_ptr, void* topk_pos_ptr, void* seqlens_ptr,
    void* cu_seqlens_ptr, void* tiles_ptr, void* cu_tiles_ptr, const void* shared_output_ptr,
    void* gateup_task_map_ptr, void* down_task_map_ptr, int num_gateup_waves, int num_down_waves,
    int num_seq, int hidden_size, int intermediate_size, int num_topk, int num_expert_total,
    int num_expert_local, int rank_ep, int use_bf16_mul, cudaStream_t stream);
int hpc_fuse_moe_blockwise_async(
    void* output_ptr, const void* input_ptr, const void* input_scale_ptr, void* gate_up_input_ptr,
    void* gate_up_input_scale_ptr, void* gate_up_output_ptr, const void* gate_up_weight_ptr,
    const void* gate_up_weight_scale_ptr, void* gate_up_tmas_ptr, void* down_input_ptr,
    void* down_input_scale_ptr, void* down_output_ptr, const void* down_weight_ptr,
    const void* down_weight_scale_ptr, void* down_tmas_ptr, const void* topk_ids_ptr,
    const void* topk_scale_ptr, void* topk_pos_ptr, void* num_tokens_per_group_ptr,
    void* cu_num_tokens_per_group_ptr, void* tiles_ptr, void* cu_tiles_ptr,
    const void* shared_output_ptr, void* gateup_task_map_ptr, void* down_task_map_ptr,
    int num_gateup_waves, int num_down_waves, int num_tokens, int num_padded_tokens,
    int hidden_size, int intermediate_size, int num_topk, int num_expert_total,
    int num_expert_local, int gate_up_weight_scale_lastdim_pad4, int down_weight_scale_lastdim_pad4,
    int rank_ep, cudaStream_t stream);

/* ---- bf16 FusedMoE and its grouped bf16 GEMM ----------------------------------------------------
 * No reference counterpart. x [num_tokens, H] bf16, gate_up_weight [E_local, 2I, H] bf16 (gate
 * rows, then up rows), down_weight [E_local, H, I] bf16 (intermediate_size = I), topk_ids int32 /
 * topk_scale f32 [num_tokens, num_topk]; experts [rank_ep E_local, (rank_ep+1) E_local) are local,
 * other ids contribute nothing. Scratch (rows = num_tokens * num_topk): gate_up_input [rows, H],
 * down_input [rows, I] and down_output [rows, H] bf16, topk_pos int32 [num_tokens, num_topk],
 * counts / tiles int32 [E_local], cu_counts / cu_tiles int32 [E_local + 1] (tiles in 128-row
 * m-tiles). Per routed row: g, u = bf16(fp32 GEMM), a = bf16(silu(g) * u) (fp32 product), d =
 * bf16(a . W2^T), output[t] = bf16(sum_k topk_scale * d (+ shared_output[t])) in k order. H and I
 * multiples of 128, E_local <= 512, num_topk <= 128, 16-byte aligned tensors, checked before any
 * launch; num_tokens = 0 launches nothing. Route -> Gate-Up -> Down -> reduce on `stream` as one
 * PDL chain, no allocation or host synchronisation: capturable. */
int hpc_fuse_moe_bf16_async(
    void* output_ptr, const void* input_ptr, void* gate_up_input_ptr, const void* gate_up_weight_ptr,
    void* down_input_ptr, void* down_output_ptr, const void* down_weight_ptr,
    const void* topk_ids_ptr, const void* topk_scale_ptr, void* topk_pos_ptr, void* counts_ptr,
    void* cu_counts_ptr, void* tiles_ptr, void* cu_tiles_ptr, const void* shared_output_ptr,
    int num_tokens, int hidden_size, int intermediate_size, int num_topk, int num_expert_total,
    int num_expert_local, int rank_ep, cudaStream_t stream);
/* y [m, n] bf16 = x [m, k] bf16 . w[g]^T (w [num_group, n, k] bf16) for the rows of group g
 * (seqlens / cu_seqlens int32 as hpc_group_gemm_fp8_async), fp32 accumulation; rows outside every
 * group are not written. k and n multiples of 128, 0 < num_group <= 512, 16-byte aligned x, w, y.
 * Persistent, PDL, capturable. */
int hpc_group_gemm_bf16_async(void* y_ptr, const void* x_ptr, const void* w_ptr,
                              const void* seqlens_ptr, const void* cu_seqlens_ptr, int num_group,
                              int m, int n, int k, cudaStream_t stream);

/* ---- fused AllReduce + residual + RMSNorm -------------------------------------------------------
 * High throughput: replaces reference src/allreduce/fuse_allreduce_rmsnorm_high_throughput.h:12-18
 * (same arguments). `signal_ptr`: device int64[world_size] of signal-pad addresses; `mc_*`: the
 * NVLS multicast addresses of the slices. The _p2p variant additionally takes HOST int64
 * tables of every rank's slice address and is used when the fabric offers no multicast mapping
 * (mc pointers NULL).
 * Low latency: replaces ...low_latency.h:29-49,503-504 (AllReduceFusionParams flattened;
 * num_max_blocks 0 = one block per SM). The _ex variant adds `protocol`: 1 = the reference's
 * Lamport two-shot (what the plain entry uses), 0 = one-shot multicast of every rank's row when the
 * batch is small and the caller's workspace holds [tokens][world][hidden] per buffer.
 * Signal pads and the Lamport workspace must come zeroed / filled with 0x80000000 words as in the
 * reference tests; buffer_flags = {0, 2, bytes_per_buffer, 0, 0, 0, 0, 0, 0}.
 */
int hpc_fuse_allreduce_rmsnorm_high_throughput_async(
    const void* input_ptr, const void* mc_input_ptr, const void* in_res_ptr, const void* weight_ptr,
    void* output_ptr, void* mc_output_ptr, void* out_res_ptr, void* signal_ptr, int64_t rank,
    int64_t world_size, int64_t num_max_blocks, double rms_norm_eps, int num_tokens,
    int hidden_size, cudaStream_t stream);
int hpc_fuse_allreduce_rmsnorm_high_throughput_p2p_async(
    const void* input_ptr, const void* mc_input_ptr, const void* in_res_ptr, const void* weight_ptr,
    void* output_ptr, void* mc_output_ptr, void* out_res_ptr, void* signal_ptr,
    const int64_t* peer_input_ptrs_host, const int64_t* peer_output_ptrs_host, int64_t rank,
    int64_t world_size, int64_t num_max_blocks, double rms_norm_eps, int num_tokens,
    int hidden_size, cudaStream_t stream);
int hpc_fuse_allreduce_rmsnorm_low_latency_async(
    int n_ranks, int rank, int num_tokens, int token_dim, void** buffer_ptrs_dev,
    void* buffer_ptr_local, void* multicast_ptr, uint32_t* buffer_flags, int rmsnorm_fusion,
    int launch_with_pdl, const void* input, const void* residual_in, const void* gamma,
    double epsilon, void* residual_out, void* output, int num_max_blocks, cudaStream_t stream);
int hpc_fuse_allreduce_rmsnorm_low_latency_ex_async(
    int n_ranks, int rank, int num_tokens, int token_dim, void** buffer_ptrs_dev,
    void* buffer_ptr_local, void* multicast_ptr, uint32_t* buffer_flags, int rmsnorm_fusion,
    int launch_with_pdl, const void* input, const void* residual_in, const void* gamma,
    double epsilon, void* residual_out, void* output, int num_max_blocks, int protocol,
    cudaStream_t stream);

/* ---- BF16 x "FP32" route GEMM ---------------------------------------------------------------------
 * replaces reference src/gemm/gemm.h:12-15 (gemm_bf16xfp32_async):
 *   Y[m, n] = X . W_high^T + scale * (X . W_low^T), fp32 accumulate, bf16 or fp32 output.
 * split_k in {1, 2, 4, 8}: the k-splits of an output tile run as one thread-block cluster and
 * reduce through distributed shared memory, so the reference's global workspaces split_y /
 * split_flag / flag_ld (and its sm_90 tile knobs tile_m / k_warpgroup_n) are accepted and ignored;
 * split_flag is never written and therefore stays zeroed. hpc_gemm_bf16xfp32_select_splitk is
 * the host heuristic (role of reference src/gemm/sm90/entry.cc:25-84).
 */
int hpc_gemm_bf16xfp32_select_splitk(int m, int n, int k, int use_splitk);
int hpc_gemm_bf16xfp32_async(void* y_ptr, void* split_y_ptr, void* split_flag_ptr,
                             const void* x_ptr, const void* w_high_ptr, const void* w_low_ptr,
                             int m, int n, int k, float scale, int use_fp32_output, int split_k,
                             int tile_m, int k_warpgroup_n, int flag_ld, cudaStream_t stream);

/* ---- FP8 block-sparse / dense causal prefill over the paged KV cache ------------------------------
 * replace reference src/attention/prefill/prefill.h:46-63. q e4m3 [total_seq_q, Hq, 128] (ldQ =
 * token stride), caches [blocks, 64, Hkv, 128] e4m3 with element strides (blk, tok, head),
 * qscale f32 [B, Hq, qscale_ld], out bf16 (ldY = token stride), block_mask u8
 * [B, Hq, mask_mq, mask_kb] or NULL (dense). kv-per-tensor: kscale/vscale f32[1];
 * k-per-token: kscale f32 [blocks, 2, Hkv, 32] with strides (ks_blk, ks_grp, ks_head) in floats,
 * vscale f32 [Hkv].
 */
int hpc_attention_blocksparse_prefill_qpertoken_perhead_kvpertensor_fp8_async(
    void* y_ptr, const void* q_ptr, const void* kcache_ptr, const void* vcache_ptr,
    const float* qscale_ptr, const float* kscale_ptr, const float* vscale_ptr,
    const int* cu_seqlens_q_ptr, const int* block_ids_ptr, const int* seqlens_kv_ptr,
    const uint8_t* block_mask_ptr, int num_batch, int total_seq_q, int max_seq_q, int num_head_q,
    int num_head_kv, int num_dim, int num_kvcache_blocks, int block_size, int max_blocks,
    int qscale_ld, int mask_mq, int mask_kb, int ldY, int ldQ, int64_t k_blk, int64_t k_tok,
    int64_t k_head, int64_t v_blk, int64_t v_tok, int64_t v_head, cudaStream_t stream);
int hpc_attention_blocksparse_prefill_qkpertoken_perhead_vperhead_fp8_async(
    void* y_ptr, const void* q_ptr, const void* kcache_ptr, const void* vcache_ptr,
    const float* qscale_ptr, const float* kscale_ptr, const float* vscale_ptr,
    const int* cu_seqlens_q_ptr, const int* block_ids_ptr, const int* seqlens_kv_ptr,
    const uint8_t* block_mask_ptr, int num_batch, int total_seq_q, int max_seq_q, int num_head_q,
    int num_head_kv, int num_dim, int num_kvcache_blocks, int block_size, int max_blocks,
    int qscale_ld, int mask_mq, int mask_kb, int ldY, int ldQ, int64_t k_blk, int64_t k_tok,
    int64_t k_head, int64_t v_blk, int64_t v_tok, int64_t v_head, int64_t ks_blk, int64_t ks_grp,
    int64_t ks_head, cudaStream_t stream);

/* ---- BF16 causal prefill --------------------------------------------------------------------------
 * replace reference src/attention/prefill/prefill.h:12-25 without the `tmas` scratch. Head dim 128
 * for qk and v, num_head_q % num_head_kv == 0, softmax scale 1/sqrt(128), causal mask aligned to
 * the bottom right (query i of a request with sq new and skv total tokens sees keys
 * j <= skv - sq + i, and no key j >= skv). Out bf16 [total_seq_q, Hq, 128], ldY = token stride;
 * rows of requests with sq = 0 are not written. Strides in elements, multiples of 8; q, k, v, out
 * are 16-byte aligned with heads 128 elements apart within a token.
 * Dense: q [total_seq_q, Hq, 128], k / v [total_seq_q, Hkv, 128] (token strides ldQ / ldK / ldV);
 *   request b is rows cu_seqlens_q[b] .. cu_seqlens_q[b + 1] - 1 of each, attending to itself;
 *   seqlens_q[b] must equal its length.
 * Paged: caches [blocks, block_size, Hkv, 128], block_size 16 / 32 / 64, strides (blk, tok, head)
 *   = (ldK, ldK1, ldK2) and (ldV, ldV1, ldV2), NHD or HND; block_ids [B, num_seq_max_blocks];
 *   seqlens_kvcache [B] = cached tokens including the new ones.
 */
int hpc_attention_prefill_bf16_async(void* y_ptr, const void* q_ptr, const void* k_ptr,
                                     const void* v_ptr, const int* seqlens_q_ptr,
                                     const int* cu_seqlens_q_ptr, int num_batch, int total_seq_q,
                                     int max_seq_q, int num_dim_qk, int num_dim_v, int num_head_q,
                                     int num_head_kv, int ldY, int ldQ, int ldK, int ldV,
                                     cudaStream_t stream);
int hpc_attention_with_kvcache_prefill_bf16_async(
    void* y_ptr, const void* q_ptr, const void* kcache_ptr, const void* vcache_ptr,
    const int* cu_seqlens_q_ptr, const int* block_ids_ptr, const int* seqlens_kvcache_ptr,
    int num_batch, int total_seq_q, int max_seq_q, int num_dim_qk, int num_dim_v, int num_head_q,
    int num_head_kv, int num_kvcache_blocks, int block_size, int num_seq_max_blocks, int ldY,
    int ldQ, int64_t ldK, int64_t ldK1, int64_t ldK2, int64_t ldV, int64_t ldV1, int64_t ldV2,
    cudaStream_t stream);

/* ---- prefill attention: MLA in the un-absorbed form (DeepSeek-V2/V3-style), bf16 ----------------
 * y[t, h, :] = softmax_j(s_j) . v[kv0 + j, h, :] over the visible keys j of t's request, with
 * s_j = (q[t, h, :128] . k_nope[kv0 + j, h, :] + q[t, h, 128:] . k_pe[kv0 + j, :]) * softmax_scale.
 * Request b has nq = cu_seqlens_q[b+1] - cu_seqlens_q[b] queries (rows cu_seqlens_q[b] .. of q and
 * y) and nk = cu_seqlens_kv[b+1] - cu_seqlens_kv[b] keys (rows kv0 = cu_seqlens_kv[b] .. of k_nope,
 * k_pe and v); query i sees keys j <= nk - nq + i (bottom-right causal). A query that sees no key
 * (nk < nq) gets a row of zeros; rows of requests with nq = 0 are not written.
 *   q      [total_seq_q, H, 192] bf16, [q_nope (128) | q_pe (64)] per head, heads 192 apart,
 *          token stride ldQ;  num_dim_qk must be 192, num_dim_v 128, 1 <= H <= 128
 *   k_nope [total_seq_kv, H, 128], v [total_seq_kv, H, 128]: any token / head strides
 *   k_pe   [total_seq_kv, 64], shared by all heads: any token stride
 *   y      [total_seq_q, H, 128] bf16, heads 128 apart, token stride ldY
 * Strides in elements, positive multiples of 8; every base 16-byte aligned; softmax_scale finite
 * and positive, used as given. max_seq_q >= the longest request's nq. No allocation and no host
 * synchronisation: capturable in a CUDA graph, and graphs may be replayed on several streams. */
int hpc_attention_prefill_mla_bf16_async(
    void* y_ptr, const void* q_ptr, const void* k_nope_ptr, const void* k_pe_ptr,
    const void* v_ptr, const int* cu_seqlens_q_ptr, const int* cu_seqlens_kv_ptr, int num_batch,
    int total_seq_q, int total_seq_kv, int max_seq_q, int num_head, int num_dim_qk, int num_dim_v,
    int ldY, int ldQ, int64_t k_nope_token_stride, int64_t k_nope_head_stride,
    int64_t k_pe_token_stride, int64_t v_token_stride, int64_t v_head_stride, float softmax_scale,
    cudaStream_t stream);

/* ---- RoPE + QK RMSNorm + paged KV-cache store (the producer of the cache layout attention reads) --
 * replaces reference src/rope/rope.h:15-25 (rope_norm_store_kv_async) and :27-38
 * (rope_norm_store_kv_fp8_async), argument for argument (bool -> int). Cache pages are
 * [block_size, num_kv_heads, head_dim] contiguous, `*_block_offset` = elements between pages.
 * fp8: k/v stored as x / scale (static per tensor); q dynamic per token-head (quant_policy 1, scale
 * = amax / upper_max written to q_scale) or static (quant_policy 2, q * q_scale_inv[0]).
 */
int hpc_rope_norm_store_kv_async(
    void* out_q_ptr, void* kcache_ptr, void* vcache_ptr, void* out_k_ptr, void* out_v_ptr,
    const void* in_qkv_ptr, const float* cos_sin_ptr, const int* num_seqlen_per_req_ptr,
    const int* q_index_ptr, const int* kvcache_indices_ptr, const float* q_norm_weight_ptr,
    const float* k_norm_weight_ptr, int kcache_block_offset, int vcache_block_offset, int num_batch,
    int max_num_kv_block_per_batch, int kv_block_size, int num_rows, int num_q_heads,
    int num_kv_heads, int qk_head_dim, int v_head_dim, int is_prefill, int qk_norm_policy,
    cudaStream_t stream);
int hpc_rope_norm_store_kv_fp8_async(
    void* out_q_ptr, void* kcache_ptr, void* vcache_ptr, void* out_k_ptr, void* out_v_ptr,
    int32_t* split_k_flag_ptr, float* q_scale_ptr, const void* in_qkv_ptr, const float* cos_sin_ptr,
    const int* num_seqlen_per_req_ptr, const int* q_index_ptr, const int* kvcache_indices_ptr,
    const float* q_norm_weight_ptr, const float* k_norm_weight_ptr, const float* k_scale_ptr,
    const float* v_scale_ptr, const float* q_scale_inv_ptr, float upper_max, int max_seqlens,
    int kcache_block_offset, int vcache_block_offset, int num_batch, int max_num_kv_block_per_batch,
    int kv_block_size, int num_rows, int num_q_heads, int num_kv_heads, int qk_head_dim,
    int v_head_dim, int is_prefill, int qk_norm_policy, int quant_policy, cudaStream_t stream);

/* ---- fused sampler ---------------------------------------------------------------------------
 * replaces reference src/sampler/entry.cc (fused_sampler, fused_sampler_temperature_sample).
 * logits [batch, vocab] fp32 (dtype 0) or bf16 (dtype 1), `row_stride` elements between rows, rows
 * 16-byte aligned, vocab % 8 == 0 and max_topk <= vocab <= 262144; out: int32 [batch].
 * Per-row parameters are a [batch] array or, when the pointer is null, the scalar `*_val`; topk is
 * int32 or int64 (topk_is_int64). penalty_mask [*, mask_stride] uint8, one bit per token, read
 * at row slot_id[b]; the sampled token's bit is set with an atomicOr on the aligned 4-byte word
 * holding it, so the mask must start 4-byte aligned and span a multiple of 4 bytes. gumbel_noise [batch, vocab]
 * fp32 contiguous, or null: then Philox4x32-10 noise keyed by `seed` (> 0) is drawn in the kernel.
 */
int hpc_fused_sampler_async(
    int* out, const void* logits, int64_t row_stride, int dtype, int batch, int vocab,
    uint8_t* penalty_mask, int64_t mask_stride, const int* slot_id, const float* repetition_penalty,
    float repetition_penalty_val, const float* temperature, float temperature_val,
    int softmax_policy, const void* topk, int topk_is_int64, int topk_val, const float* topp,
    float topp_val, int max_topk, const float* gumbel_noise, uint64_t seed, cudaStream_t stream);
/* temperature-only Gumbel-max; rows with temperature <= 0 (or NaN) take the argmax of the logits.
 * draft_token_ids [batch] int64 or null: that token of row b scores -inf when in [0, vocab). */
int hpc_fused_sampler_temperature_sample_async(
    int* out, const void* logits, int64_t row_stride, int dtype, int batch, int vocab,
    const float* temperature, float temperature_val, const float* gumbel_noise,
    const int64_t* draft_token_ids, uint64_t seed, cudaStream_t stream);
/* The Philox launch offset the next sampler launch on `stream` will use (synchronises `stream`).
 * For tests: the internal noise of that launch is then known to the caller. */
int hpc_sampler_rng_offset(cudaStream_t stream, uint64_t* offset);

/* ---- fused speculative sampling ---------------------------------------------------------------
 * No reference counterpart: verifies K draft tokens per request (multi-token prediction) against
 * the target logits and draws the recovered or bonus token. target_logits [batch * (K + 1), vocab]
 * fp32 (dtype 0) or bf16 (1), row b * (K + 1) + i = position i of request b, `row_stride` elements
 * between rows, rows 16-byte aligned, vocab % 8 == 0, vocab <= 262144, 1 <= K = num_draft <= 8,
 * batch * (K + 1) <= 65535. draft_token_ids [batch, K] int32 or int64 (draft_is_int64);
 * draft_probs [batch, K, vocab] fp32 contiguous, 16-byte aligned, or null for one-hot drafts;
 * temperature [batch] or, when null, temperature_val for every request (t <= 0 or NaN: greedy).
 * uniform [batch, K] and gumbel_noise [batch * (K + 1), vocab] fp32 contiguous come together; when
 * both are null a request with t > 0 draws Philox4x32-10 noise keyed by `seed` (>= 1) from the
 * sampler's per-stream launch word, which the call then advances by one. Writes
 * output_token_ids int32 [batch, K + 1] (accepted drafts, then the recovered or bonus token, then
 * -1) and num_accepted int32 [batch]. row_records is a 16-byte aligned scratch of
 * 32 * batch * (K + 1) bytes. Two launches chained by PDL, no allocation or host
 * synchronisation: capturable. */
int hpc_fused_speculative_sampler_async(
    int* output_token_ids, int* num_accepted, void* row_records, const void* target_logits,
    int64_t row_stride, int dtype, int batch, int num_draft, int vocab, const void* draft_token_ids,
    int draft_is_int64, const float* draft_probs, const float* temperature, float temperature_val,
    const float* uniform, const float* gumbel_noise, uint64_t seed, cudaStream_t stream);

/* ---- Stem block-mask generation (block-sparse FP8 prefill) ----------------------------------
 * replaces reference src/stem/*.h, argument for argument (bool -> int), with cache and scale
 * strides added. Only stem_block_size 128, stem_stride 16 and head dim 128.
 * prep_paged_kv: caches [blocks, page (32 or 64), Hkv, 128] e4m3 read through ldK/ldV (block),
 * ldK1/ldV1 (token) and ldK2/ldV2 (head) strides in elements, so NHD and HND both work;
 * kflat [B, Hkv, max_num_stem_blocks, 2048] bf16, vbias [B, Hkv, max_num_stem_blocks] fp32,
 * v_norm_down [B, Hkv, max_k_down_len = 8 * max_num_stem_blocks] fp32 scratch. Blocks past a
 * request's ceil(kv / 128) are not written. quant "kvpertensor": kscale, vscale [1] fp32;
 * "qkpertoken_perhead_vperhead": kscale [blocks, page / 32, Hkv, 32] fp32 (ldKS, ldKS1, ldKS2 in
 * fp32 elements), vscale [Hkv].
 */
int hpc_stem_oam_prep_paged_kv_qpertoken_perhead_kvpertensor_dim128_async(
    void* kflat_ptr, void* vbias_ptr, const void* kcache_ptr, const void* vcache_ptr,
    const void* kscale_ptr, const void* vscale_ptr, const void* block_ids_ptr,
    const void* kv_seq_lens_ptr, int num_batch, int num_dim_qk, int num_dim_v, int num_head_kv,
    int num_kvcache_blocks, int block_size, int num_seq_max_blocks, int stem_block_size,
    int stem_stride, float lambda_mag, int max_num_stem_blocks, int max_k_down_len, int64_t ldK,
    int64_t ldV, int64_t ldK1, int64_t ldK2, int64_t ldV1, int64_t ldV2, void* v_norm_down_ptr,
    cudaStream_t stream);
int hpc_stem_oam_prep_paged_kv_qkpertoken_perhead_vperhead_dim128_async(
    void* kflat_ptr, void* vbias_ptr, const void* kcache_ptr, const void* vcache_ptr,
    const void* kscale_ptr, const void* vscale_ptr, const void* block_ids_ptr,
    const void* kv_seq_lens_ptr, int num_batch, int num_dim_qk, int num_dim_v, int num_head_kv,
    int num_kvcache_blocks, int block_size, int scale_block_size, int num_seq_max_blocks,
    int stem_block_size, int stem_stride, float lambda_mag, int max_num_stem_blocks,
    int max_k_down_len, int64_t ldK, int64_t ldV, int64_t ldKS, int64_t ldKS1, int64_t ldKS2,
    int64_t ldK1, int64_t ldK2, int64_t ldV1, int64_t ldV2, void* v_norm_down_ptr,
    cudaStream_t stream);
/* q_fp8 [total, Hq, 128] e4m3 (ldQ elements between tokens), qscale [B, Hq, >= max q] fp32 read
 * through its strides ldQS, ldQS1, ldQS2 (elements); qflat [B, Hq, max_num_q_blocks, 2048] bf16. */
int hpc_stem_oam_prep_varlen_q_dim128_async(
    void* qflat_ptr, const void* q_fp8_ptr, const void* qscale_ptr, const void* q_seq_lens_ptr,
    const void* cu_seqlens_q_ptr, int num_batch, int num_head_q, int ldQ, int stem_block_size,
    int stem_stride, int max_num_q_blocks, int64_t ldQS, int64_t ldQS1, int64_t ldQS2,
    cudaStream_t stream);
/* block_logits [B, Hq, max_num_qb, max_num_kb] bf16 contiguous, every element written. No host
 * synchronisation: capturable. */
int hpc_stem_oam_gemm_dim128_async(
    void* block_logits_ptr, const void* qflat_ptr, const void* kflat_ptr, const void* vbias_ptr,
    const void* q_seq_lens_ptr, const void* kv_seq_lens_ptr, int num_batch, int num_head_q,
    int num_head_kv, int max_num_qb, int max_num_kb, int stem_block_size, int stem_stride,
    int causal, cudaStream_t stream);
/* mask [B, Hq, max_Qb, max_Kb] u8, every byte written; max_Kb <= 32768. Capturable. */
int hpc_stem_tpd_async(
    void* mask_ptr, const void* block_logits_ptr, const void* q_seq_lens_ptr,
    const void* kv_seq_lens_ptr, const void* num_prompt_tokens_ptr, int num_batch, int num_heads,
    int max_Qb, int max_Kb, int block_size, float alpha, int initial_blocks, int window_size,
    float k_block_num_rate_medium, int k_block_num_bias_medium, float k_block_num_rate_large,
    int k_block_num_bias_large, cudaStream_t stream);

#ifdef __cplusplus
}
#endif

#endif /* INCLUDE_HPC_B200_H_ */
