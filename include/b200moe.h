/*
 * b200moe.h — C ABI of libb200moe.so: the H100-native (sm_90a) replacement for the expert hot path that
 * Lvllm delegates to the closed `lk_moe` wheel, plus the routing / permutation / decode-attention
 * operators that sit next to it in a decoder layer.
 *
 * Every entry point is `extern "C"`, takes plain pointers and sizes (no torch types) and returns 0 on
 * success or a negative error code; b200moe_last_error() returns a thread-local message.
 * All device work is enqueued on the caller's `stream` (a cudaStream_t passed as void*), is CUDA-graph
 * capturable (no allocation, no synchronisation, pointer-stable workspaces) unless stated otherwise.
 *
 * Reference interfaces replaced (file:line in guqiong96/Lvllm):
 *   lk_moe.MOEConfigV2 fields ............. vllm/model_executor/layers/fused_moe/routed_experts.py:1490-1511
 *   lk_moe.MOE_* constructors ............. routed_experts.py:1514-1533, 1598-1616, 1650-1668, 1724-1742, 1795-1813
 *   lk_moe.cpu_decode ..................... routed_experts.py:1840-1855
 *   lk_moe.cpu_prefill .................... routed_experts.py:1858-1882
 *   lk_moe.gpu_prefill .................... routed_experts.py:1884-1899
 *   _moe_C.topk_softmax / topk_sigmoid .... csrc/libtorch_stable/moe/topk_softmax_kernels.cu:822-897
 *   _moe_C.grouped_topk ................... csrc/libtorch_stable/moe/grouped_topk_kernels.cu:1447-1556
 *   GateLinear.forward (router GEMM) ...... vllm/model_executor/layers/fused_moe/router/gate_linear.py:171-221
 *   _moe_C.moe_permute / moe_unpermute .... csrc/libtorch_stable/moe/moe_permute_unpermute_op.cu:59-207
 *   _C.sm100_cutlass_mla_decode ........... csrc/libtorch_stable/attention/mla/sm100_cutlass_mla_kernel.cu:225-262
 *   paged GQA decode (FlashInfer backend) . vllm/v1/attention/backends/flashinfer.py (cache layout :398-433, K / V views
 *                                           :2276-2290)
 *   fused_qk_norm_rope + reshape_and_cache_flash .. vllm/_custom_ops.py:279, csrc/libtorch_stable/cache_kernels.cu:315-400
 */
#ifndef B200MOE_H_
#define B200MOE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- error codes --------------------------------------------------------------------------- */
#define B200_OK 0
#define B200_ERR_INVALID (-1)   /* bad argument / unsupported shape */
#define B200_ERR_CUDA (-2)      /* a CUDA runtime call failed */
#define B200_ERR_NO_DEVICE (-3) /* no sm_90 device */

const char* b200moe_last_error(void);
/* library build info: "b200moe <version> sm_90a" */
const char* b200moe_version(void);

/* ---- lk_moe.MOEConfigV2 (routed_experts.py:1490-1511) ------------------------------------------ */
typedef struct b200moe_config {
  int32_t num_processes;    /* TP or EP world size the layer is sharded over */
  int32_t process_id;       /* this rank */
  int32_t gpu_id;           /* CUDA device ordinal */
  int32_t has_gate_proj;    /* 1: w13 = [gate;up] rows, 0: single up projection */
  int32_t expert_num;       /* LOCAL experts held by this object */
  int32_t top_k;
  int32_t hidden_size;      /* H */
  int32_t intermediate_size;/* I per partition */
  int32_t max_batch_size;   /* max tokens per prefill call */
  int32_t max_num_seqs;     /* max tokens per decode call */
  int32_t stride;           /* lk_moe CPU tiling knobs: accepted, unused */
  int32_t group_min_len;
  int32_t group_max_len;
  int32_t groupN;           /* weight rows per scale row */
  int32_t groupK;           /* weight cols per scale col */
  int32_t activation_type;  /* 0 silu, 1 swigluoai (layout stated by B200MOE_SWIGLUOAI_LAYOUT), 2 relu^2 (non-gated),
                               3 silu(min(gate, limit)) * clamp(up, -limit, limit) (DeepSeek-V4; swiglu_limit > 0) */
  float swiglu_alpha;
  float swiglu_limit;
  int32_t use_gpu_prefill;
} b200moe_config;

/* weight formats == the lk_moe.MOE_* class families */
#define B200_FMT_16BIT 0 /* MOE_BF16 / MOE_FP16: w13 [E,2I,H], w2 [E,H,I] in the activation dtype */
#define B200_FMT_FP8 1   /* MOE_FP8: e4m3 + f32 block scales [E,2I/gN,H/gK] (or per-tensor [E,2]/[E]) */
#define B200_FMT_WNA16 2 /* MOE_WNA16: uint4b8 packed u8 [E,2I,H/2], group scales act-dtype [E,2I,H/g] */
#define B200_FMT_NVFP4 3 /* MOE_NVFP4: e2m1 u8 [E,2I,H/2], e4m3 scales [E,2I,H/16], f32 global [E,2]/[E] */
#define B200_FMT_MXFP4 4 /* MOE_MXFP4: e2m1 u8 [E,2I,H/2], e8m0 scales [E,2I,H/32] */

#define B200_ACT_BF16 0
#define B200_ACT_FP16 1

typedef struct b200moe_layer* b200moe_handle;

/* Construct one MoE layer object.  Weight pointers are raw checkpoint-layout tensors (see format list);
 * `weights_on_device` = 0: pageable/pinned HOST memory (the lk_moe contract: the caller frees them right
 * after the call, so everything is copied/repacked into HBM before returning);  1: device memory (fast
 * path used by loaders that already staged the checkpoint in HBM).  Absent tensors are NULL.
 * Synchronous; not graph-capturable. */
int b200moe_create(const b200moe_config* cfg, const void* w13, const void* w2, const void* w13_scale,
                   const void* w2_scale, const void* w13_global_scale, const void* w2_global_scale,
                   int format, int act_dtype, int weights_on_device, b200moe_handle* out);
/* Per-expert ingest (SURVEY.md 8f row 4; reference weight_loader routed_experts.py:644-1168 builds stacked [E, ...] CPU
 * parameters first): create the layer without weights, feed expert ranges straight from wherever the checkpoint shards
 * live (host or device memory, raw checkpoint layout of those experts only), then finalize.  Each range is staged
 * through a bounded device buffer and re-tiled into its final place; the caller may free / unmap its tensors as soon as
 * b200moe_load_experts returns.  b200moe_create is this sequence over the whole stacked tensor. */
int b200moe_create_empty(const b200moe_config* cfg, int format, int act_dtype, b200moe_handle* out);
int b200moe_load_experts(b200moe_handle h, int first_expert, int num_experts, const void* w13, const void* w2,
                         const void* w13_scale, const void* w2_scale, const void* w13_global_scale,
                         const void* w2_global_scale, int weights_on_device);
int b200moe_finalize(b200moe_handle h);
int b200moe_destroy(b200moe_handle h);
/* bytes of HBM held by the layer (repacked weights + scales + workspaces) */
int64_t b200moe_device_bytes(b200moe_handle h);

/* layer introspection (tests / bring-up): what = 0: 0 (MXFP4 layers run the W4A16 dequant kernel; a native block-scaled
 * W4A8-MX kernel would report 1); 1: tokens per pass; 2: 1 when w13 arrived with interleaved gate/up rows (SwiGLU-OAI,
 * B200MOE_SWIGLUOAI_LAYOUT=interleaved); 3: 4-bit flavour (0 none, 1 int4, 2 nvfp4, 3 mxfp4); 4: 1 when an FP8 layer
 * runs in ue8m0 mode (B200MOE_FP8_E8M0=1: power-of-two block scales, the reference's DeepGEMM ue8m0 numerics,
 * fp8_utils.py:986-1043).  < 0: unknown. */
int b200moe_query(b200moe_handle h, int what);

/* lk_moe.cpu_decode(stream, M, k, hidden, ids, weights, out_f32): all DEVICE pointers; hidden [M,H] in
 * the activation dtype, ids int32 [M,k] (<0 or >=E: skip), weights f32 [M,k], out f32 [M,H].
 * Graph-capturable. */
int b200moe_cpu_decode(b200moe_handle h, void* stream, int num_tokens, int top_k, const void* hidden,
                       const int32_t* topk_ids, const float* topk_weights, float* out_f32);
/* lk_moe.cpu_prefill(M, k, ids, weights, hidden, out_f32): all HOST pointers; synchronous (copies in,
 * runs the same device path, copies out). */
int b200moe_cpu_prefill(b200moe_handle h, int num_tokens, int top_k, const int32_t* topk_ids_host,
                        const float* topk_weights_host, const void* hidden_host, float* out_f32_host);
/* lk_moe.gpu_prefill(hidden, out, ids, weights, M, k, stream): DEVICE pointers, out in the activation
 * dtype. */
int b200moe_gpu_prefill(b200moe_handle h, const void* hidden, void* out, const int32_t* topk_ids,
                        const float* topk_weights, int num_tokens, int top_k, void* stream);

/* ---- routing operators ---------------------------------------------------------------------------- */
/* softmax (scoring=0) / sigmoid (scoring=1) / sqrt(softplus) (scoring=2, DeepSeek-V4) top-k; logits [M,E] f32/bf16/f16
 * (logits_dtype 0 f32, 1 bf16, 2 f16); bias f32 [E] or NULL (selection only: weights are the unbiased scores);
 * ids int32 [M,k], weights f32 [M,k], token_expert_indices int32 [M,k] = j*M+t or NULL.  Ties -> lower expert index. */
int b200_topk_gating(void* stream, const void* logits, int logits_dtype, const float* bias, int num_tokens,
                     int num_experts, int top_k, int scoring, int renormalize, float routed_scaling_factor,
                     float* topk_weights, int32_t* topk_ids, int32_t* token_expert_indices);
/* DeepSeek-V4 hash routing (topk_softplus_sqrt_kernels.cu:326-403): ids[t] = tid2eid[input_ids[t], :] (int32 table
 * [vocab, top_k], top_k <= 32), weights = sqrt(softplus(logits)) of those experts, renormalised (optional) and scaled
 * by routed_scaling_factor.  No bias.  An input id outside [0, vocab) gives the whole row, a table entry outside
 * [0, E) its slot, id -1 and weight 0. */
int b200_hash_topk(void* stream, const void* logits, int logits_dtype, const int32_t* input_ids, const int32_t* tid2eid,
                   int vocab, int num_tokens, int num_experts, int top_k, int renormalize, float routed_scaling_factor,
                   float* topk_weights, int32_t* topk_ids);
/* DeepSeek group-limited routing (scoring 0 none, 1 sigmoid); bias f32 [E] or NULL. */
int b200_grouped_topk(void* stream, const void* logits, int logits_dtype, const float* bias, int num_tokens,
                      int num_experts, int n_group, int topk_group, int top_k, int scoring, int renormalize,
                      float routed_scaling_factor, float* topk_weights, int32_t* topk_ids);
/* EP id remap: local = expert_map[clamp(id)] ; id<0 -> -1  (routed_experts.py:1332-1342) */
int b200_global_to_local_ids(void* stream, const int32_t* topk_ids, const int32_t* expert_map, int num_global,
                             int64_t numel, int32_t* local_ids);

/* Fused router: logits = hidden . gate_weight^T (fp32 accumulate on wgmma, split-K with a deterministic fixed-order
 * reduction), then top-k routing and the optional EP id remap, in ONE kernel.  Replaces GateLinear.forward
 * (router/gate_linear.py:171-221, csrc/libtorch_stable/moe/dsv3_router_gemm_entry.cu:112) + fused_topk / grouped_topk
 * (fused_topk_router.py:81-124, grouped_topk_kernels.cu:523-678) + global_to_local_expert_ids (routed_experts.py:1332-1342).
 * hidden [M,H] and gate_weight [E,H] in the activation dtype (16-byte aligned, H % 64 == 0, E <= 1024);
 * mode 0 softmax top-k, 1 sigmoid top-k (bias for selection only), 2 grouped top-k (scoring 0 none / 1 sigmoid, bias,
 * n_group, topk_group), 3 sqrt-softplus top-k (DeepSeek-V4, bias for selection only); topk_ids are GLOBAL expert ids; local_ids (optional) = expert_map[id] (-1 stays -1; with
 * expert_map NULL a copy); logits_out (optional) f32 [M,E].
 * Shared experts (reference runner/shared_experts.py; SURVEY.md 8f row 2) are folded into the routed launch as always-on
 * experts: with n_shared > 0 every output row has top_k + n_shared columns, the extra ones carrying weight
 * shared_weight, global id E + s and local id shared_local_base + s (-1 when shared_local_base < 0: another rank holds
 * them); the caller appends the shared expert(s) to the layer's stacked weights and calls cpu_decode with
 * top_k + n_shared — the stream-K schedule then overlaps them with the routed experts by construction.  workspace: b200_router_workspace_bytes() bytes of device
 * memory, zero-filled once by the caller (the kernel hands its counters back clean, so it is CUDA-graph replayable). */
int64_t b200_router_workspace_bytes(int num_tokens, int num_experts, int hidden_size);
int b200_router_topk(void* stream, const void* hidden, int act_dtype, const void* gate_weight, int num_tokens,
                     int num_experts, int hidden_size, const float* bias, int mode, int scoring, int top_k, int renormalize,
                     int n_group, int topk_group, float routed_scaling_factor, const int32_t* expert_map, int n_shared,
                     int shared_local_base, float shared_weight, void* workspace, int64_t workspace_bytes,
                     float* topk_weights, int32_t* topk_ids, int32_t* local_ids, float* logits_out);
/* The fused router with DeepSeek-V4 hash routing (mode must be 3): the same GEMM, then the routing of b200_hash_topk on
 * the token's logits; EP remap, shared columns and logits_out as in b200_router_topk. */
int b200_router_hash_topk(void* stream, const void* hidden, int act_dtype, const void* gate_weight, int num_tokens,
                          int num_experts, int hidden_size, const float* bias, int mode, int scoring, int top_k,
                          int renormalize, int n_group, int topk_group, float routed_scaling_factor,
                          const int32_t* expert_map, int n_shared, int shared_local_base, float shared_weight,
                          void* workspace, int64_t workspace_bytes, float* topk_weights, int32_t* topk_ids,
                          int32_t* local_ids, float* logits_out, const int32_t* input_ids, const int32_t* tid2eid,
                          int vocab);

/* ---- permutation operators (stable sort by expert) ------------------------------------------------- */
/* sorted_slot int32 [M*k] (source slot t*k+j of each permuted row, valid rows first in (expert, slot)
 * order), expert_first_offset int64 [E+1], inv_perm int32 [M*k] (-1 for skipped slots);
 * permuted_hidden [M*k,H] (same dtype as hidden, 2 bytes/elt) or NULL. */
int b200_moe_permute(void* stream, const void* hidden, const int32_t* topk_ids, int num_tokens, int top_k,
                     int num_local_experts, int hidden_size, int32_t* sorted_slot,
                     int64_t* expert_first_offset, int32_t* inv_perm, void* permuted_hidden);
/* out[t,:] = sum_j w[t,j] * permuted[inv_perm[t,j],:] (fp32 accumulate); act dtype in, out_dtype
 * 0 bf16 / 1 fp16 / 2 f32 out. */
int b200_moe_unpermute(void* stream, const void* permuted, int act_dtype, const float* topk_weights,
                       const int32_t* inv_perm, int num_tokens, int top_k, int hidden_size, void* out,
                       int out_dtype);

/* fp32 -> activation dtype cast of the lk_moe output (routed_experts.py:1855) fused with an RMS
 * normalisation: out[t] = cast(in[t] * gain * rsqrt(mean(in[t]^2) + eps)); out_dtype 0 bf16 / 1 fp16. */
int b200_rmsnorm_cast(void* stream, const float* in, void* out, int num_tokens, int hidden_size, float gain,
                      float eps, int out_dtype);

/* ---- decode attention ----------------------------------------------------------------------------- */
/* Paged MLA decode, absorbed form.  q_nope [B,Hq,512], q_pe [B,Hq,64] (bf16), kv cache
 * [num_pages,page_size,576] bf16, seq_lens int32 [B], page_table int32 [B,max_pages];
 * out bf16 [B,Hq,512], lse f32 [B,Hq] (may be NULL); Hq <= 128.  workspace: b200_mla_decode_workspace_bytes(). */
int64_t b200_mla_decode_workspace_bytes(int batch, int num_heads, int num_splits);
int b200_mla_decode(void* stream, const void* q_nope, const void* q_pe, const void* kv_cache,
                    const int32_t* seq_lens, const int32_t* page_table, int batch, int num_heads,
                    int page_size, int max_pages, float sm_scale, int num_splits, void* workspace, void* out,
                    float* lse);
/* Same with an e4m3 latent cache (kv_cache_dtype "fp8": [num_pages,page_size,576] bytes, half the HBM traffic) and,
 * optionally, e4m3 queries — the fp8 mode of the reference's CUTLASS MLA (backends/mla/cutlass_mla.py:44-45,
 * tests/kernels/attention/test_cutlass_mla_decode.py:101-110).  q_dtype / kv_dtype: 0 bf16, 1 e4m3; descale_q /
 * descale_k are the per-tensor dequantisation scales (q_scale * k_scale folds into the softmax scale, k_scale into the
 * output).  The cache is widened to bf16 on its way into shared memory: probabilities are not re-quantised. */
int b200_mla_decode_ex(void* stream, const void* q_nope, const void* q_pe, int q_dtype, const void* kv_cache,
                       int kv_dtype, float descale_q, float descale_k, const int32_t* seq_lens,
                       const int32_t* page_table, int batch, int num_heads, int page_size, int max_pages, float sm_scale,
                       int num_splits, void* workspace, void* out, float* lse);
/* Speculative-decode verification (multi-token prediction): the arguments of b200_mla_decode_ex plus q_len = Q query
 * tokens per request (uniform over the batch, 1 <= Q <= 16; B200_ERR_INVALID otherwise, nothing launched) and the optional
 * up-projection of b200_mla_decode_vup.  q_nope [B*Q, Hq, 512], q_pe [B*Q, Hq, 64] with request b's Q tokens contiguous in
 * draft order; seq_lens[b] = S_b counts all of request b's keys, its Q new tokens included (written to the cache before this
 * call).  Query token i of request b attends to key positions [0, S_b - Q + i]: the end-aligned causal mask of the
 * reference's FlashMLA decode (QueryLenSupport.UNIFORM, v1/attention/backends/mla/flashmla.py:120; the query reshaped to
 * [B, Q, Hq, D] by reshape_query_for_spec_decode, backends/utils.py:745-758, and the kernel called with causal=True,
 * flashmla.py:284-344).  Rows are (b * Q + i, h): out bf16 [B*Q, Hq, 512], lse f32 [B*Q, Hq] (natural log) or NULL; a row
 * with no visible key (S_b - Q + 1 + i <= 0) gives out = 0, lse = -inf.  w_uv == NULL: out is required.  w_uv != NULL
 * ([Hq,512,128] bf16): the split merge is fused with the v up-projection as in b200_mla_decode_vup, out_v bf16
 * [B*Q, Hq, 128] is required, out is the optional latent output and num_splits <= 512.  The workspace is
 * b200_mla_decode_workspace_bytes(batch * q_len, num_heads, num_splits) bytes.  q_len = 1 is b200_mla_decode_ex
 * (w_uv == NULL) or b200_mla_decode_vup. */
int b200_mla_decode_spec(void* stream, const void* q_nope, const void* q_pe, int q_dtype, const void* kv_cache,
                         int kv_dtype, float descale_q, float descale_k, const int32_t* seq_lens,
                         const int32_t* page_table, int batch, int q_len, int num_heads, int page_size, int max_pages,
                         float sm_scale, int num_splits, void* workspace, void* out, float* lse, const void* w_uv,
                         void* out_v);
/* Sparse MLA decode (DeepSeek-V3.2 / GLM-5 layers, config.index_topk): query token t attends only to the keys its lightning
 * indexer selected.  Replaces the reference's triton_convert_req_index_to_global_index (v1/attention/backends/mla/
 * sparse_utils.py:120) followed by the FlashMLA sparse decode (flashmla_sparse.py:587-611, 763-830): the conversion is fused
 * into the kernel's gather.  q_nope [T,Hq,512], q_pe [T,Hq,64] bf16 (T = num_tokens query tokens; the draft tokens of a
 * request are simply tokens with the same req_id); topk_indices int32 [T, topk], request-local key positions, entry j of
 * token t is key row page_table[req_id[t]][idx / page_size] * page_size + idx % page_size; an entry with idx < 0 or
 * idx / page_size >= max_pages is skipped.  req_id int32 [T] (rows of page_table, int32 [*, max_pages]).  kv_dtype 0: bf16
 * cache [pages, page_size, 576]; kv_dtype 2: fp8_ds_mla cache [pages, page_size, 656] bytes (512 e4m3 | 4 fp32 scales, one per
 * 128 dims | 64 bf16 rope dims, flashmla_sparse.py:63-72), widened to bf16(float(e4m3) * scale) on the way into shared
 * memory.  out bf16 [T,Hq,512], lse f32 [T,Hq] (natural log) or NULL; a token with no valid entry gets out = 0, lse = -inf.
 * w_uv / out_v as in b200_mla_decode_spec.  Workspace: b200_mla_decode_workspace_bytes(num_tokens, num_heads, num_splits).
 * B200_ERR_INVALID, nothing launched: kv_dtype other than 0 / 2, num_heads > 128, topk < 1, a NULL required pointer,
 * num_splits <= 0, or num_splits > 512 with w_uv. */
int b200_mla_decode_sparse(void* stream, const void* q_nope, const void* q_pe, const void* kv_cache, int kv_dtype,
                           const int32_t* topk_indices, int topk, const int32_t* req_id, const int32_t* page_table,
                           int max_pages, int num_tokens, int num_heads, int page_size, float sm_scale, int num_splits,
                           void* workspace, void* out, float* lse, const void* w_uv, void* out_v);
/* DeepSeek-V4 sparse attention decode (the reference's FlashMLA call with indices / extra_k_cache / attn_sink,
 * models/deepseek_v4/nvidia/flashmla.py:151-244).  Head dim 512 = 448 NoPE + 64 RoPE dims; one cache row is both K and V.
 * q bf16 [num_tokens, num_heads, 512].  Both caches hold 584-byte tokens per block (flashmla_sparse.py:76-85): block b starts at
 * b * block_stride bytes, token p's data (448 e4m3 | 64 bf16 rope) at + p * 576, its scale record (7 ue8m0 bytes, one per 64
 * NoPE dims, then a pad byte) at + block_size * 576 + p * 8; a NoPE value is bf16(e4m3) * 2^(s - 127).  Keys of token t:
 * swa_indices[t, :swa_lens[t]] (int32 [num_tokens, swa_topk], global slots of swa_cache) followed, when extra_cache is given,
 * by extra_indices[t, :extra_lens[t]] (global slots of extra_cache, its own block size); lengths are clamped to [0, topk].
 * A slot resolves to (slot / block_size, slot % block_size); a slot < 0 or >= num_blocks * block_size is no key.
 * s_j = sm_scale * q . k_j; out bf16 [num_tokens, num_heads, 512] = sum_j p_j k_j with the softmax over the valid keys, and
 * with attn_sink (f32 [num_heads], or NULL) m' = max(m, sink_h), l' = l e^(m - m') + e^(sink_h - m'), out = acc e^(m - m') / l',
 * folded in once after the split merge.  A token with no valid key gets out = 0.  Workspace:
 * b200_mla_decode_workspace_bytes(num_tokens, num_heads, num_splits).  No allocation, no synchronisation (graph-capturable).
 * B200_ERR_INVALID, nothing launched: a NULL required pointer, q / caches / workspace / out not 16-byte aligned, index and
 * length arrays not 4-byte aligned, num_tokens outside [1, 65535], num_heads outside [1, 128], topk < 1, a block stride below
 * block_size * 584 or not a multiple of 16, num_splits outside [1, 512]. */
int b200_dsv4_sparse_decode(void* stream, const void* q, int num_tokens, int num_heads, const void* swa_cache,
                            int swa_block_size, int swa_num_blocks, int64_t swa_block_stride, const int32_t* swa_indices,
                            int swa_topk, const int32_t* swa_lens, const void* extra_cache, int extra_block_size,
                            int extra_num_blocks, int64_t extra_block_stride, const int32_t* extra_indices, int extra_topk,
                            const int32_t* extra_lens, const float* attn_sink, float sm_scale, int num_splits,
                            void* workspace, void* out);
/* DeepSeek-V4 q-norm + RoPE + cache insert, one launch (the reference's fused_deepseek_v4_qnorm_rope_kv_rope_quant_insert,
 * csrc/libtorch_stable/fused_deepseek_v4_qnorm_rope_kv_insert_kernel.cu).  q bf16 [num_tokens, num_heads, 512]: per-head RMSNorm
 * without weight (eps), then GPT-J pair RoPE of dims 448-511, all in fp32, rounded once into q_out bf16
 * [num_tokens, q_head_padded, 512]; heads num_heads .. q_head_padded - 1 are written as zeros.  kv bf16 [num_tokens, 512]
 * (after kv_norm): RoPE of dims 448-511; NoPE dims quantised per 64 with scale 2^ceil(log2(max(amax, 1e-4) / 448)) to e4m3 and
 * a ue8m0 byte, written with the bf16 rope dims to row slot_mapping[t] (int64; < 0 or past the cache: nothing written) of the
 * 584-byte cache laid out as in b200_dsv4_sparse_decode.  positions int64 [num_tokens] (clamped to [0, max_position));
 * cos_sin_cache f32 [max_position, 64] = cos | sin. */
int b200_dsv4_qnorm_rope_kv_insert(void* stream, const void* q, const void* kv, const int64_t* positions,
                                   const float* cos_sin_cache, int max_position, const int64_t* slot_mapping, void* cache,
                                   int block_size, int num_blocks, int64_t block_stride, void* q_out, int num_tokens,
                                   int num_heads, int q_head_padded, float eps);
/* DeepSeek-V4 KV compressor (the reference's DeepseekCompressor.forward, models/deepseek_v4/compressor.py), two launches in
 * stream order.  (head_dim D, compress_ratio R): (512, 4) and (128, 4) with overlapping windows (coff = 2), (512, 128)
 * without (coff = 1).  kv_score f32 [num_tokens, 2 coff D] (rows kv_score_stride floats apart) = kv | score; ape f32
 * [R, coff D]; positions, slot_mapping int64 [num_tokens]; state_cache f32 [blocks, state_block_size, 2 coff D], blocks
 * state_block_stride floats apart.
 *   state write  token t with s = slot_mapping[t] >= 0: row s of the state = kv | score + ape[position % R];
 *   compression  token t with s >= 0 and a position p >= 0 with (p + 1) % R == 0: the state rows of positions
 *                p - (1 + overlap) R + 1 .. p of its request (token_to_req int32 [num_tokens], rows of block_table int32
 *                [*, block_table_stride] holding state block numbers); positions below 0 are no row.  With overlap the
 *                older R rows use columns [0, D) of their kv and score halves, the newer R rows [D, 2D).  Per column
 *                c = sum kv softmax(score) over the rows (fp32); c * rsqrt(mean(c^2) + eps) * w (norm_weight bf16 [D]);
 *                GPT-J pair RoPE of the last 64 dims at position (p / R) R (clamped to [0, max_position)), cos_sin_cache
 *                f32 [max_position, 64] = cos | sin; the row goes to slot kv_slot_mapping[t] (int64; < 0 or past the cache:
 *                nothing written) of kv_cache, blocks block_stride bytes apart:
 *                  D 512: the 584-byte row of b200_dsv4_qnorm_rope_kv_insert (every value rounded to bf16, NoPE dims
 *                         per 64 to e4m3 with a ue8m0 scale byte, rope dims bf16);
 *                  D 128: the 132-byte row of the indexer cache (block_size x 128 e4m3 bytes, then block_size fp32
 *                         scales): every value rounded to bf16, one scale 2^ceil(log2(max(amax, 1e-4) / 448)).
 * A window reads the rows the state write of the same call wrote.  No allocation, no synchronisation (graph-capturable).
 * B200_ERR_INVALID, nothing launched: another (head_dim, compress_ratio), a NULL or misaligned pointer (kv_score, ape,
 * state_cache, norm_weight, kv_cache 16 bytes; int64 arrays 8; int32 arrays and cos_sin_cache 4), kv_score_stride below
 * 2 coff D or not a multiple of 4, a state block stride below state_block_size * 2 coff D or not a multiple of 4, a cache
 * block stride below block_size * 584 (132) bytes or not a multiple of 16 (4), a block size or block count below 1,
 * max_position < 1, eps < 0 or NaN, num_tokens outside [0, 2^20].  num_tokens 0 launches nothing. */
int b200_dsv4_compress(void* stream, const float* kv_score, int64_t kv_score_stride, const float* ape,
                       const int64_t* positions, const int64_t* slot_mapping, const int32_t* token_to_req,
                       const int32_t* block_table, int64_t block_table_stride, float* state_cache, int state_block_size,
                       int64_t state_block_stride, const void* norm_weight, float eps, const float* cos_sin_cache,
                       int max_position, const int64_t* kv_slot_mapping, void* kv_cache, int block_size, int num_blocks,
                       int64_t block_stride, int head_dim, int compress_ratio, int num_tokens);
/* DeepSeek-V4 manifold hyper-connections (mHC) for decode, hc_mult = 4 (the reference's mhc_pre / mhc_post /
 * mhc_fused_post_pre / hc_head, vllm/model_executor/kernels/mhc/torch.py:6-106, tilelang_kernels.py:305-350, 884-977).
 * residual bf16 [T, 4, H], x bf16 [T, H], post_layer_mix f32 [T, 4], comb_res_mix f32 [T, 4, 4] (comb[i][j] maps stream i to
 * stream j), fn f32 [24, 4H] row-major, hc_scale f32 [3], hc_base f32 [24]; norm_weight bf16 [H] or NULL.
 *   post   r'[t, j] = bf16(post[t, j] x[t] + sum_i comb[t, i, j] residual[t, i]), fp32, rounded once;
 *   pre    on r (= r' when x is given, else residual), r_flat the fp32 row [4H]:
 *          mixes = (r_flat . fn^T) * rsqrt(sum r_flat^2 / 4H + rms_eps),
 *          pre_i = sigmoid(mixes_i s0 + base_i) + hc_pre_eps, post_mix_j = sigmoid(mixes_{4+j} s1 + base_{4+j}) * post_mult,
 *          comb_mix = sinkhorn(mixes_{8..23} s2 + base_{8..23}) as [4, 4] (row softmax + eps, column normalise, then
 *          sinkhorn_repeat - 1 times row and column normalisation, each dividing by sum + hc_sinkhorn_eps),
 *          layer_input = bf16(sum_i pre_i r_i); with norm_weight: the fp32 row o is stored as bf16 and
 *          layer_input = bf16(float(bf16(o)) * rsqrt(mean(o^2) + norm_eps) * w), the mean square from the unrounded o.
 * Outputs: residual_out bf16 [T, 4, H] (r'), post_mix f32 [T, 4], comb_mix f32 [T, 4, 4], layer_input bf16 [T, H].
 * x NULL: pre only, and post_layer_mix, comb_res_mix and residual_out must be NULL.  A token's outputs do not depend on the
 * other tokens of the batch (the reduction is split by H only), and the fused call gives the bits of b200_mhc_post followed
 * by the pre-only call.  Workspace: b200_mhc_workspace_bytes(T, H) bytes, 16-byte aligned.  No allocation, no
 * synchronisation (graph-capturable).  B200_ERR_INVALID, nothing launched: a NULL required pointer, a bf16 tensor, fn or the
 * workspace not 16-byte aligned, an f32 array not 4-byte aligned, T outside [1, 2^20], H not a multiple of 64 in
 * [256, 16384], sinkhorn_repeat < 1, a negative (or NaN) eps. */
int64_t b200_mhc_workspace_bytes(int num_tokens, int hidden_size);   /* = T * (H / 64) * 25 * 4 */
int b200_mhc_post_pre(void* stream, const void* x, const void* residual, const float* post_layer_mix,
                      const float* comb_res_mix, const float* fn, const float* hc_scale, const float* hc_base,
                      const void* norm_weight, int num_tokens, int hidden_size, float rms_eps, float hc_pre_eps,
                      float hc_sinkhorn_eps, float hc_post_mult_value, int sinkhorn_repeat, float norm_eps,
                      void* workspace, void* residual_out, float* post_mix, float* comb_mix, void* layer_input);
/* post alone: out bf16 [T, 4, H] = r' as above (the same expression, the same bits). */
int b200_mhc_post(void* stream, const void* x, const void* residual, const float* post_layer_mix, const float* comb_res_mix,
                  int num_tokens, int hidden_size, void* out);
/* hc_head: fn f32 [4, 4H], hc_scale f32 [1], hc_base f32 [4];
 * out bf16 [T, H] = bf16(sum_i (sigmoid(mixes_i s0 + base_i) + hc_eps) residual_i), mixes as in the pre step.
 * Workspace b200_mhc_workspace_bytes(T, H); refusals as b200_mhc_post_pre. */
int b200_hc_head(void* stream, const void* residual, const float* fn, const float* hc_scale, const float* hc_base,
                 int num_tokens, int hidden_size, float rms_eps, float hc_eps, void* workspace, void* out);
/* The MLA decode kernel's neighbours (SURVEY.md 8f row 3), bf16:
 *  b200_mla_rope_cache_write  RoPE of q_pe [T,Hq,64] and k_pe [T,64] in place (rotary_embedding/base.py:161-201; cos_sin_cache
 *      bf16 [max_pos,64] = cos | sin; is_neox 0 = GPT-J pairs (DeepSeek), 1 = NeoX halves) fused with concat_and_cache_mla
 *      (csrc/libtorch_stable/cache_kernels.cu:403-444): row slot_mapping[t] (i64, < 0 = padded token) of the paged latent
 *      cache [blocks*block_size, 576] <- [kv_c[t] (512) | rotated k_pe[t]]; kv_dtype 1 = e4m3 cache storing value / kv_scale;
 *      kv_dtype 2 = fp8_ds_mla cache [blocks*block_size, 656] bytes (concat_and_cache_ds_mla_kernel, cache_kernels.cu:496-590:
 *      per 128-dim tile scale = max(amax / 448, FLT_MIN) as fp32 and e4m3(value / scale); kv_scale unused);
 *  b200_mla_q_absorb          ql_nope [T,Hq,512] = q_nope [T,Hq,128] x W_UK_T [Hq,128,512]  (mla_attention.py:875-893);
 *  b200_mla_decode_vup        b200_mla_decode_ex whose split merge is fused with the v up-projection
 *      out_v [B,Hq,128] = o [B,Hq,512] x W_UV [Hq,512,128] (mla_attention.py:1154-1176); out_latent (optional) = o. */
int b200_mla_rope_cache_write(void* stream, void* q_pe, void* k_pe, const void* kv_c, const int64_t* positions,
                              const void* cos_sin_cache, int is_neox, const int64_t* slot_mapping, void* kv_cache,
                              int kv_dtype, float kv_scale, int num_tokens, int num_heads);
int b200_mla_q_absorb(void* stream, const void* q_nope, const void* w_uk_t, void* out, int num_tokens, int num_heads);
int b200_mla_decode_vup(void* stream, const void* q_nope, const void* q_pe, int q_dtype, const void* kv_cache, int kv_dtype,
                        float descale_q, float descale_k, const int32_t* seq_lens, const int32_t* page_table, int batch,
                        int num_heads, int page_size, int max_pages, float sm_scale, int num_splits, void* workspace,
                        const void* w_uv, void* out_v, void* out_latent, float* lse);
/* The lightning indexer of DeepSeek-V3.2 / GLM-5 layers for decode: it produces the topk_indices that
 * b200_mla_decode_sparse takes.  Index heads H, head dim 128 = [64 rotary | 64 nope].  The indexer cache is uint8
 * [num_blocks, block_size, 132] (indexer_k_quant_and_cache's layout): block b holds block_size x 128 e4m3 bytes, then
 * block_size fp32 scales, one per token.  It shares the latent cache's page table.  All three are CUDA-graph capturable:
 * no allocation, no synchronisation; a bad shape or misaligned pointer returns B200_ERR_INVALID and launches nothing.
 *
 *  b200_indexer_qk_rope_quant_cache_write  replaces the reference's _fused_indexer_q_rope_quant_kernel
 *      (sparse_attn_indexer.py:127-251), the RoPE of the indexer k (RotaryEmbedding.forward_static) and
 *      indexer_k_quant_and_cache (csrc/libtorch_stable/cache_kernels.cu:599-659), in one launch.
 *      q [T,H,128] bf16 contiguous (wq_b output), weights bf16 [T, >= H] with row stride weights_row_stride elements (a
 *      column slice of the fused projection), k [T,128] bf16 (after k_norm), positions i64 [T] (clamped to the table),
 *      cos_sin_cache bf16 [max_position, 64] = cos | sin, is_neox 1 = NeoX halves, 0 = interleaved pairs.
 *      q: RoPE in fp32 (products and sum rounded separately, no FMA), each rotated value rounded to bf16; q_scale = the power of two >= max(amax, 1e-10) / 448 over the
 *      128 dims; q_fp8 [T,H,128] = e4m3(q / q_scale); weights_out f32 [T,H] = weight * q_scale * softmax_scale * head_scale.
 *      k: RoPE in bf16 arithmetic; scale = max(amax, 1e-4) / 448 (its power-of-two ceiling when use_ue8m0); row
 *      slot_mapping[t] (< 0: nothing written) <- e4m3(k / scale) and the fp32 scale.
 *      1 <= num_heads <= 128; q, k, q_fp8, k_cache 16-byte aligned.
 *  b200_indexer_logits  replaces DeepGEMM fp8_fp4_paged_mqa_logits (fp8_paged_mqa_logits_torch,
 *      rocm_aiter_mla_sparse.py:264-363).  q_fp8 [B*Q,H,128] e4m3, weights f32 [B*Q,H] (weights_out above), seq_lens i32 [B]
 *      (<= max_pages * page_size), page_table i32 [B, max_pages], k_cache with num_blocks blocks of page_size rows.
 *      logits f32 [B*Q, logits_stride], logits_stride >= max_pages * page_size: row r = b*Q + i,
 *      logits[r, j] = k_scale[j] * sum_h weights[r, h] * relu(q_fp8[r, h] . k[j]) for j < row_end = S_b - Q + i + 1 (the
 *      end-aligned causal mask); -inf from row_end to the end of request b's last page; nothing else is written.
 *      num_heads 32 or 64, 1 <= q_len <= 16, page_size 16, 32 or 64.
 *  b200_indexer_topk  replaces top_k_per_row_decode (csrc/libtorch_stable/sampler.cu:567-614, 661-720).  Row r of the
 *      logits starts at r * logits_stride and holds row_width <= logits_stride values.  For row r = b*Q + i with
 *      row_end = min(max(0, S_b - Q + i + 1), row_width): out i32 [B*Q, topk] = the positions of the
 *      topk largest logits of [0, row_end) in ascending order, ties at the threshold to the lowest positions; row_end <=
 *      topk gives 0 .. row_end - 1; -1 pads.  The same bits on every call.  1 <= topk <= 2048. */
int b200_indexer_qk_rope_quant_cache_write(void* stream, const void* q, const void* weights, int64_t weights_row_stride,
                                           const void* k, const int64_t* positions, const void* cos_sin_cache,
                                           int max_position, int is_neox, const int64_t* slot_mapping, void* k_cache,
                                           int block_size, int use_ue8m0, float softmax_scale, float head_scale,
                                           void* q_fp8, float* weights_out, int num_tokens, int num_heads);
int b200_indexer_logits(void* stream, const void* q_fp8, const float* weights, const void* k_cache, int num_blocks,
                        int page_size, const int32_t* seq_lens, const int32_t* page_table, int batch, int q_len,
                        int num_heads, int max_pages, float* logits, int64_t logits_stride);
int b200_indexer_topk(void* stream, const float* logits, int64_t logits_stride, int64_t row_width, const int32_t* seq_lens,
                      int batch, int q_len, int topk, int32_t* out);
/* The C4A indexer of DeepSeek-V4 layers for decode: it picks the compressed keys a token attends to, over the indexer's
 * 132-byte cache that b200_dsv4_compress writes (head dim 128 at ratio 4; layout as above).  Graph-capturable, no
 * allocation, no synchronisation; a bad argument returns B200_ERR_INVALID and launches nothing.
 *
 *  b200_dsv4_indexer_q_quant  replaces the fp8 path of the reference's _fused_indexer_q_rope_quant_kernel
 *      (models/deepseek_v4/common/ops/fused_indexer_q.py:70-176).  q bf16 [T,H,128] contiguous = [64 nope | 64 rope],
 *      weights bf16 [T, >= H] with row stride weights_row_stride elements, positions i64 [T] (clamped to the table),
 *      cos_sin_cache f32 [max_position, 64] = cos | sin (b200_dsv4_compress's table).  Per (token, head): GPT-J pair RoPE
 *      of dims 64-127 (pair (64 + 2i, 65 + 2i) with cos[i], sin[i]; fp32 products and sum, no FMA, one bf16 rounding);
 *      scale = 2^ceil(log2(max(amax, 1e-4) / 448)) over the 128 values (nope as loaded, rope after rounding); q_fp8
 *      e4m3 [T,H,128] = x / scale, saturating; weights_out f32 [T,H] = w * scale * softmax_scale * head_scale.  No k row.
 *      1 <= num_heads <= 128, 0 <= num_tokens <= 2^20; q and q_fp8 16-byte aligned.
 *  b200_dsv4_indexer_decode  the indexer's logits and top-k with one row per token (the reference's
 *      SparseAttnIndexer decode over the compressed cache).  Token t has n_t = (positions[t] + 1) / compress_ratio
 *      candidates (0 for positions < 0), at most max_blocks * page_size; its pages are row token_to_req[t] of
 *      block_table i32 [*, max_blocks] (contiguous).  q_fp8 / weights as b200_dsv4_indexer_q_quant wrote them.  logits f32
 *      [T, logits_stride] (logits_stride >= max_blocks * page_size): logits[t, j] for j < n_t as b200_indexer_logits
 *      computes them, -inf to the end of the token's last page.  out i32 [T, topk] = the positions of the topk largest
 *      logits of [0, n_t), ascending, ties to the lowest positions, -1 padding; n_t <= topk gives 0 .. n_t - 1.
 *      max_seq_len > 0 promises every positions[t] < max_seq_len: when max_seq_len / compress_ratio <= topk no logit is
 *      computed (logits untouched) and out is the same.  num_heads 32 or 64, page_size 16, 32 or 64, compress_ratio 4 or
 *      128, 1 <= topk <= 2048, 0 <= num_tokens <= 2^20; q_fp8 and k_cache 16-byte aligned. */
int b200_dsv4_indexer_q_quant(void* stream, const void* q, const void* weights, int64_t weights_row_stride,
                              const int64_t* positions, const float* cos_sin_cache, int max_position, float softmax_scale,
                              float head_scale, void* q_fp8, float* weights_out, int num_tokens, int num_heads);
int b200_dsv4_indexer_decode(void* stream, const void* q_fp8, const float* weights, const void* k_cache, int num_blocks,
                             int page_size, const int64_t* positions, const int32_t* token_to_req,
                             const int32_t* block_table, int max_blocks, int compress_ratio, int num_tokens,
                             int num_heads, int64_t max_seq_len, float* logits, int64_t logits_stride, int topk,
                             int32_t* out);
/* Global key lists of DeepSeek-V4 decode: what b200_dsv4_sparse_decode (swa / extra indices and lengths) and
 * b200_dsv4_compress (kv_slot_mapping) take.  One launch; graph-capturable.  Token t has position p = positions[t] and
 * request row token_to_req[t] of block_table i32 [*, block_table_stride] (the first max_blocks columns used); local index i
 * of the request is global slot block_table[req][i / block_size] * block_size + i % block_size, and -1 (no key) when
 * i / block_size >= max_blocks.  A token with slot_mapping[t] < 0 gets length 0 and a row of -1, and its request row is not
 * read.  out i32 [T, out_stride] (width columns written) and lens i32 [T] for the lists:
 *   kind 0 SWA            (_compute_swa_indices_and_lens_kernel) param = window W, 1 <= W <= width: keys
 *                         [max(p - W + 1, 0), p] of the SWA cache's table, length p + 1 - start (0 for p < 0);
 *   kind 1 C128A          (_build_c128a_topk_metadata_kernel, decode) param = compress_ratio 4 or 128: compressed rows
 *                         [0, min((p + 1) / ratio, width)) (p < 0: none);
 *   kind 2 top-k → global (_compute_global_topk_indices_and_lens_kernel) local_topk i32 [T, local_stride >= width], the
 *                         request-local output of b200_dsv4_indexer_decode: entry j -> its global slot (-1 stays -1),
 *                         length = the count of entries >= 0;
 * entries past a list's length are -1.
 *   kind 3 slot mapping   (_compressed_slot_mapping_kernel) param = compress_ratio 4 or 128: out i64 [T] = the global slot
 *                         of compressed row p / ratio when p >= 0 and (p + 1) % ratio == 0, else -1; lens, width and
 *                         out_stride are not used.
 * B200_ERR_INVALID, nothing launched: another kind, a NULL or misaligned pointer (int64 arrays 8 bytes, int32 4;
 * positions may be NULL for kind 2),
 * max_blocks < 1 or > block_table_stride, block_size < 1, num_tokens outside [0, 2^20], for the lists width outside
 * [1, min(out_stride, 2^20)], and the kind's parameter out of range. */
int b200_dsv4_indices(void* stream, int kind, const int64_t* positions, const int64_t* slot_mapping,
                      const int32_t* token_to_req, const int32_t* block_table, int64_t block_table_stride, int max_blocks,
                      int block_size, int param, const int32_t* local_topk, int64_t local_stride, void* out,
                      int64_t out_stride, int width, int32_t* lens, int num_tokens);
/* The DeepSeek-V4 attention output projection's first two steps (the reference's deep_gemm_fp8_o_proj,
 * models/deepseek_v4/nvidia/ops/o_proj.py:28-73; wo_b stays with the caller).  G = n_groups, heads_per_group hpg = H / G,
 * D = hpg * 512, R = o_lora_rank.  One launch each, no allocation, no synchronisation: graph-capturable.  A bad argument
 * returns B200_ERR_INVALID and launches nothing; num_tokens 0 launches nothing.
 *
 *  b200_dsv4_inv_rope_quant  replaces fused_inv_rope_fp8_quant, fp32-scale path (common/ops/fused_inv_rope_fp8_quant.py).
 *      o bf16 [T, H, 512] = [448 nope | 64 rope], heads and dims contiguous, token stride o_token_stride elements (>= H * 512,
 *      a multiple of 8); positions i64 [T] (clamped to the table); cos_sin_cache f32 [max_position, 64] = cos | sin
 *      (b200_dsv4_qnorm_rope_kv_insert's table).  Per (token, head): the inverse GPT-J pair rotation of dims 448-511, pair
 *      (448 + 2i, 449 + 2i) = (x, y) -> (x cos[i] + y sin[i], y cos[i] - x sin[i]) in fp32, products and sum rounded
 *      separately (no FMA), not rounded to bf16.  Per 128 values of a group (a head's dims [128 b, 128 b + 128)):
 *      scale = 2^ceil(log2(max(absmax, 1e-10) * (1 / 448))), the ceiling taken exactly from the fp32 bits of the product;
 *      codes = e4m3(clamp(x / scale, -448, 448)), round to nearest even.  Outputs in this module's layout:
 *      o_fp8 e4m3 [G][T][D] (element (t, g, d) at (g * T + t) * D + d) and o_scale f32 [G][D / 128][T] (element (t, g, b)
 *      at (g * D / 128 + b) * T + t).  0 <= num_tokens <= 2^20, 1 <= hpg <= 16; o and o_fp8 16-byte aligned.
 *  b200_dsv4_wo_a_workspace_bytes  workspace b200_dsv4_wo_a needs on the current device (0: none).  A workspace sized for
 *      some T serves every smaller T of every shape; its first bytes hold arrival counters that must be zero before the
 *      first call and that every call leaves zero.
 *  b200_dsv4_wo_a  replaces DeepGEMM's fp8_einsum("bhr,hdr->bhd") with recipe (1, 128, 128): z bf16 [T, G * R],
 *      z[t, g * R + r] = sum over k-blocks kb of (sum_k o_fp8[t, g, 128 kb + k] * wo_a[g * R + r, 128 kb + k]) *
 *      wo_a_scale[(g * R + r) / 128, kb] * o_scale[t, g, kb], the inner sum one tensor-core accumulation, the outer in fp32,
 *      rounded to bf16 once.  o_fp8 / o_scale as b200_dsv4_inv_rope_quant wrote them; wo_a e4m3 [G * R, D] row-major (the
 *      checkpoint tensor, read in place); wo_a_scale f32 [G * R / 128, D / 128] (checkpoints that store e8m0 scales convert
 *      them to f32 once: exact).  K is split over CTAs by G, R, D and the SM count, never by T, and the splits are added in
 *      fixed order: z of a token does not depend on the other tokens of the call, and repeated calls give the same bits.
 *      0 <= num_tokens <= 2^20, n_groups >= 1, heads_per_group 1-16, o_lora_rank a multiple of 128, G * R / 64 <= 65535;
 *      o_fp8, wo_a and workspace 16-byte aligned. */
int b200_dsv4_inv_rope_quant(void* stream, const void* o, int64_t o_token_stride, const int64_t* positions,
                             const float* cos_sin_cache, int max_position, int num_tokens, int num_heads, int n_groups,
                             void* o_fp8, float* o_scale);
int64_t b200_dsv4_wo_a_workspace_bytes(int num_tokens, int n_groups, int heads_per_group, int o_lora_rank);
int b200_dsv4_wo_a(void* stream, const void* o_fp8, const float* o_scale, const void* wo_a, const float* wo_a_scale,
                   int num_tokens, int n_groups, int heads_per_group, int o_lora_rank, void* workspace,
                   int64_t workspace_bytes, void* z);
/* Paged GQA decode.  q [B,Hq,D] bf16, k_cache/v_cache [num_pages,page_size,Hkv,D] bf16 (contiguous), D=128;
 * out bf16 [B,Hq,D], lse f32 [B,Hq] or NULL. */
int64_t b200_gqa_decode_workspace_bytes(int batch, int num_q_heads, int head_dim, int num_splits);
int b200_gqa_decode(void* stream, const void* q, const void* k_cache, const void* v_cache,
                    const int32_t* seq_lens, const int32_t* page_table, int batch, int num_q_heads,
                    int num_kv_heads, int head_dim, int page_size, int max_pages, float sm_scale,
                    int num_splits, void* workspace, void* out, float* lse);
/* Same on caches described by base pointer + strides in elements: row (page, slot, kv head) of a cache starts at
 * page * block_stride + slot * page_stride + head * head_stride, its D elements contiguous.  This reads the FlashInfer
 * backend's cache in place: one tensor per layer, logical (blocks, Hkv, page, 2D), NHD (blocks, page, Hkv, 2D) or HND
 * in memory (flashinfer.py:398-433), handed out as kv_cache.transpose(1, 2).split(D, -1) (flashinfer.py:2276-2290),
 * i.e. k_cache = base, v_cache = base + D with the tensor's own strides.  b200_gqa_decode passes the contiguous strides
 * (page_size*Hkv*D, Hkv*D, D).  Strides must be positive multiples of 8 elements and the cache pointers 16-byte aligned
 * (16-byte cp.async rows); B200_ERR_INVALID otherwise. */
int b200_gqa_decode_ex(void* stream, const void* q, const void* k_cache, const void* v_cache, int64_t block_stride,
                       int64_t page_stride, int64_t head_stride, const int32_t* seq_lens, const int32_t* page_table,
                       int batch, int num_q_heads, int num_kv_heads, int head_dim, int page_size, int max_pages,
                       float sm_scale, int num_splits, void* workspace, void* out, float* lse);
/* Speculative-decode verification: the arguments of b200_gqa_decode_ex plus q_len = Q query tokens per request (uniform
 * over the batch, 1 <= Q <= 16; B200_ERR_INVALID otherwise, nothing launched).  q [B*Q, Hq, D] bf16 with request b's Q
 * tokens contiguous in draft order (vLLM's decode_query layout); seq_lens[b] = S_b counts all of request b's keys, its Q
 * new tokens included (written to the cache before this call).  Query token i of request b attends to key positions
 * [0, S_b - Q + i] (the end-aligned causal mask of a multi-token decode, reference tests/kernels/attention/
 * test_flashinfer.py:29-80 with query_lens = [Q] * B).  out bf16 [B*Q, Hq, D], lse f32 [B*Q, Hq] (natural log) or NULL,
 * row (b * Q + i, h); a row with no visible key (S_b - Q + 1 + i <= 0) gives out = 0, lse = -inf.  The workspace is
 * b200_gqa_decode_workspace_bytes(batch * q_len, num_q_heads, head_dim, num_splits) bytes.  q_len = 1 is
 * b200_gqa_decode_ex. */
int b200_gqa_decode_spec(void* stream, const void* q, const void* k_cache, const void* v_cache, int64_t block_stride,
                         int64_t page_stride, int64_t head_stride, const int32_t* seq_lens, const int32_t* page_table,
                         int batch, int q_len, int num_q_heads, int num_kv_heads, int head_dim, int page_size,
                         int max_pages, float sm_scale, int num_splits, void* workspace, void* out, float* lse);
/* The GQA decode kernel's neighbour, bf16: one launch per step for what the reference runs as Qwen3's per-head q/k RMSNorm
 * (models/qwen3_moe.py:333-351) + RoPE (fused_qk_norm_rope, vllm/_custom_ops.py:279; rotary_embedding/base.py:161-201)
 * + reshape_and_cache_flash (csrc/libtorch_stable/cache_kernels.cu:315-400, called at flashinfer.py:2276-2290).
 *   qkv           [T, (Hq + 2 Hkv) * D] bf16, contiguous: the fused QKV projection's output (q heads, k heads, v heads);
 *   q_weight / k_weight  bf16 [D] RMSNorm weights, or NULL to skip that norm (Mixtral); eps its epsilon.  The norm is
 *                 vllm/ir/ops/layernorm.py:10-21 in its order: fp32 statistics, rounded to bf16, times the weight with one
 *                 rounding;
 *   cos_sin_cache bf16 [max_position, rotary_dim] = cos | sin (RotaryEmbedding._match_cos_sin_cache_dtype); rotary_dim
 *                 even, <= D; is_neox 1 = NeoX halves (p, p + rotary_dim/2), 0 = GPT-J pairs (2p, 2p + 1).  positions
 *                 (i64 [T]) are CLAMPED to [0, max_position): the table is never read outside its rows.  RoPE is computed
 *                 in fp32 from the bf16 inputs and rounded once (<= 2 bf16 ulp from forward_static's bf16 arithmetic);
 *   q_out         [T, Hq, D] bf16, contiguous: the rotated q, b200_gqa_decode's q;
 *   k_cache / v_cache  base pointers + block_stride / page_stride / head_stride (elements) as b200_gqa_decode_ex takes them
 *                 (= what reshape_and_cache_flash is given: NHD / HND packed views or separate caches); page_size = block
 *                 size.  Row slot_mapping[t] (i64, slot = block * page_size + offset; < 0 = padded token, nothing
 *                 written) of every kv head <- rotated k / the untouched v.
 * D = head_dim must be 128; strides positive multiples of 8 elements, pointers 16-byte aligned; NULL only for the weights.
 * B200_ERR_INVALID otherwise. */
int b200_gqa_qknorm_rope_cache_write(void* stream, const void* qkv, const int64_t* positions, const void* cos_sin_cache,
                                     int max_position, int rotary_dim, int is_neox, const void* q_weight,
                                     const void* k_weight, float eps, const int64_t* slot_mapping, void* k_cache,
                                     void* v_cache, int64_t block_stride, int64_t page_stride, int64_t head_stride,
                                     int page_size, void* q_out, int num_tokens, int num_heads, int num_kv_heads,
                                     int head_dim);

/* ---- expert-parallel exchange over NVLink peer memory ---------------------------------------------- */
/* Sum-combine of per-rank partial MoE outputs through peer-mapped buffers (the lk_moe EP/TP contract:
 * replicated tokens, local experts, all-reduce; moe_runner.py:488-494).  peer_bufs[r] is rank r's
 * staging buffer mapped into this process (CUDA IPC), peer_flags[r] its flag word array.
 * out = sum over ranks (fixed rank order, bit-identical on every rank) of each rank's local_in[0:numel];
 * fp32 in, out_dtype out (0 bf16, 1 fp16, 2 f32).  CUDA-graph replayable (epochs live in device memory). */
/* buffers: data buffer of 2*slot_elems floats and a flag buffer of b200_ep_flag_bytes() bytes per rank,
 * both created with b200_ep_buffer_create (cudaMalloc + zero + IPC export) and opened by the peers. */
int64_t b200_ep_flag_bytes(void);
int b200_ep_buffer_create(int64_t bytes, void** dev_ptr, void* ipc_handle_64B);
int b200_ep_buffer_open(const void* ipc_handle_64B, void** dev_ptr);
int b200_ep_buffer_close(void* dev_ptr, int is_owner);
int b200_ep_allreduce(void* stream, void* const* peer_bufs, int32_t* const* peer_flags, int world, int rank,
                      const float* local_in, int64_t numel, int64_t slot_elems, void* out, int out_dtype);

/* Push all-reduce fused with residual add + RMSNorm (the op pair that follows the MoE block in a decoder layer;
 * reference moe_runner.py:462-496 + fused_add_rms_norm, flashinfer_all_reduce.py): every rank stores its fp32
 * [num_tokens, hidden] partial straight into every peer's buffer, then reduces from local memory in fixed rank order:
 *   x = sum_r partial_r (+ residual);  residual <- cast(x) (in place, may be NULL);  sum_out <- x (f32, may be NULL);
 *   out = cast(x * rsqrt(mean(x^2) + eps)) * gamma   (gamma act-dtype [hidden]; NULL: out = cast(x * rsqrt(..) * gain)).
 * peer_bufs[r]: data buffers of (2 + 2 * world) * slot_elems floats (b200_ep_buffer_create; the first two slots are the
 * pull all-reduce's), flags as b200_ep_allreduce.
 * hidden <= 8192, num_tokens * hidden <= slot_elems.  CUDA-graph replayable. */
int b200_ep_allreduce_norm(void* stream, void* const* peer_bufs, int32_t* const* peer_flags, int world, int rank,
                           const float* local_in, int num_tokens, int hidden, int64_t slot_elems, void* residual,
                           const void* gamma, float gain, float eps, void* out, float* sum_out, int act_dtype);

/* Dispatch / combine all-to-all for token-sharded callers (DP attention + EP experts): rank r owns tokens
 * [r*m_local, (r+1)*m_local) of the global batch M = world*m_local and experts [r*experts_per_rank, ...).
 * Replaces the dispatch/combine pair around the experts in the reference's EP path
 * (vllm/model_executor/layers/fused_moe/runner/moe_runner.py:462-496, 600; SURVEY.md 8e).
 * Every rank creates one data buffer of b200_ep_a2a_layout(...) bytes with b200_ep_buffer_create and opens the
 * peers'; the flag buffers are the ones of b200_ep_allreduce.  b200_ep_a2a_layout returns the buffer size and the
 * byte offsets of X [M][hidden] 16-bit, IDS [M][top_k] i32 (ids local to the rank, -1 = skip), W [M][top_k] f32,
 * Y [M][hidden] f32 inside it.
 *   b200_ep_dispatch pushes this rank's rows to the ranks owning one of their experts; when it retires, the local
 *     X / IDS / W are complete: run b200moe_cpu_decode(handle, stream, M, top_k, buf+off_x, buf+off_ids, buf+off_w,
 *     buf+off_y) on them.
 *   b200_ep_combine then pulls the partial rows of this rank's tokens from those ranks and writes
 *     out [m_local][hidden] (out_dtype 0 bf16, 1 fp16, 2 f32), summed in ascending rank order.
 * ids_global are global expert ids (< 0 = padding).  All ranks must call both with identical shapes; both are
 * CUDA-graph capturable (epochs live in device memory). */
int64_t b200_ep_a2a_layout(int global_tokens, int hidden, int top_k, int64_t* off_x, int64_t* off_ids, int64_t* off_w,
                           int64_t* off_y);
int b200_ep_dispatch(void* stream, void* const* peer_bufs, int32_t* const* peer_flags, int world, int rank,
                     const void* hidden_local, const int32_t* ids_global, const float* weights, int m_local, int top_k,
                     int hidden, int experts_per_rank);
int b200_ep_combine(void* stream, void* const* peer_bufs, int32_t* const* peer_flags, int world, int rank,
                    const int32_t* ids_global, int m_local, int top_k, int hidden, int experts_per_rank, void* out,
                    int out_dtype);

/* b200_ep_combine fused with residual add + RMSNorm (arithmetic and arguments of b200_ep_allreduce_norm): the fp32
 * combine output never goes to HBM. */
int b200_ep_combine_norm(void* stream, void* const* peer_bufs, int32_t* const* peer_flags, int world, int rank,
                         const int32_t* ids_global, int m_local, int top_k, int hidden, int experts_per_rank,
                         void* residual, const void* gamma, float gain, float eps, void* out, int act_dtype);

/* per-kernel timing of the expert GEMMs with CUDA events on the launching stream (eager calls only;
 * ignored under stream capture).  profile(1) starts a window, profile_read returns the summed GEMM1 /
 * GEMM2 milliseconds and the number of forward calls in the window, then resets it. */
int b200moe_profile(int enable);
int b200moe_profile_read(double* gemm1_ms, double* gemm2_ms, int64_t* calls);

/* bring-up aid: copy `bytes` of an internal workspace buffer of the current device to host memory
 * (what: 0 tiled activations, 1 activation scales, 2 tiled intermediate, 3 intermediate scales,
 * 4 expert outputs y, 5 route state, 6 chunk table, 7 row_of_slot, 8 slot_of_row).  Synchronous. */
int b200moe_debug_read(int what, void* dst_host, int64_t bytes);

/* kernel-launch counter (number of this library's kernels launched by this process so far) */
int64_t b200moe_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200MOE_H_ */
