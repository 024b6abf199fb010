// Internal structures shared by the MoE translation units (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/b200moe.h"

namespace b200 {

constexpr int TILE_BYTES = 16384;   // one [128 rows x 128 B] swizzled operand tile
constexpr int ROW_ALIGN = 16;       // every expert's permuted row range starts on a multiple of 16 rows
constexpr int MAX_EXPERTS = 1024;

// chunk = up to tn_max consecutive permuted rows of one expert
struct Chunk {
  int32_t expert;
  int32_t row0;   // first (padded) permuted row, multiple of 16
  int32_t nrows;  // valid rows (1..tn_max)
  int32_t pad;
};

// Device-side per-call routing state (lives in the workspace; rewritten by every call's prep kernel)
struct RouteState {
  int32_t n_chunks;
  int32_t n_rows_padded;
  int32_t unit_ctr[2];  // dynamic tile schedulers of GEMM1 / GEMM2
  int32_t done_ctr[2];
  int32_t reserved[2];
};

// ---- fused decode kernel (moe_fused.cu) limits and cross-CTA synchronisation block
constexpr int FUSED_MAX_SLOTS = 2048;    // M * top_k
constexpr int FUSED_MAX_TOKENS = 256;
constexpr int FUSED_MAX_ROWS = 6144;     // padded permuted rows
constexpr int FUSED_MAX_EXPERTS = 512;   // local experts
constexpr int FUSED_MAX_CHUNKS = 512;
constexpr int FUSED_MAX_TILES = 65536;   // chunks * tiles-per-expert of either GEMM
constexpr int FUSED_MAX_J2 = 256;

struct FusedSync {     // generation-tagged counters (gen << 16 | count); never zeroed between launches
  int32_t gen;
  int32_t finished;
  int32_t x_ready;
  int32_t pad;
  int32_t g1_done[FUSED_MAX_CHUNKS];
  int32_t comb[FUSED_MAX_J2];
  int32_t tcnt1[FUSED_MAX_TILES];
  int32_t tcnt2[FUSED_MAX_TILES];
};

struct Workspace {  // process-wide, per device; sized for the largest layer / batch seen so far
  int device = -1;
  int64_t cap_slots = 0, cap_rows = 0, cap_hidden = 0, cap_inter = 0;
  int32_t* row_of_slot = nullptr;  // [slots]
  int32_t* slot_of_row = nullptr;  // [rows]
  int32_t* pad_off = nullptr;      // [MAX_EXPERTS+1]
  int32_t* sort_hist = nullptr;    // [128 CTAs][MAX_EXPERTS] per-CTA expert histograms of the multi-CTA routing sort
  Chunk* chunks = nullptr;         // [rows/16 + MAX_EXPERTS]
  RouteState* state = nullptr;
  uint8_t* xt = nullptr;   // tiled activations  [rows/8][KB1][1024]
  float* xs = nullptr;     // act scales          [KB1][rows]
  uint8_t* it = nullptr;   // tiled intermediate  [rows/8][KB2][1024]
  float* is = nullptr;     // inter scales        [KB2][rows]
  float* y = nullptr;      // expert outputs fp32 [rows][H]
  float* partials = nullptr;   // stream-K partial tiles [2 phases][SMs][2][2*64*128] fp32
  FusedSync* fsync = nullptr;
  // host<->device staging of cpu_prefill
  void* d_hidden = nullptr;
  int32_t* d_ids = nullptr;
  float* d_w = nullptr;
  float* d_out = nullptr;
  int64_t cap_stage_tokens = 0, cap_stage_hidden = 0, cap_stage_k = 0;
  // 4-bit layers, prefill-class batches: the layer's experts expanded to fp16 MMA tiles (one layer at a time)
  uint8_t* dq13 = nullptr;
  uint8_t* dq2 = nullptr;
  int64_t cap_dq13 = 0, cap_dq2 = 0;
  int64_t bytes = 0;
  std::vector<void*> retired;      // outgrown buffers: kept alive for CUDA graphs captured against them
  int live_layers = 0;             // layers of this device; the workspace is released with the last one
  // every layer (and stream) of a device shares this workspace and the fused kernel's cross-CTA counters: eager calls
  // from a second stream are ordered behind the previous call with this event (graph-captured calls are ordered
  // by the graph itself)
  cudaEvent_t last_use = nullptr;
  cudaStream_t last_stream = nullptr;
  bool last_valid = false;
};

}  // namespace b200

struct b200moe_layer {
  b200moe_config cfg;
  int fmt, act_dtype, device;
  int E, H, I, N1;     // N1 = rows of w13 (2I gated, I otherwise)
  int gated;
  int esz_bits;        // operand element size fed to the MMA: 8 (fp8) or 16
  int KB1, KB2;        // 128-byte k-blocks of GEMM1 (over H) and GEMM2 (over I)
  int J1, J2;          // 128-row output tiles of GEMM1 (I/128) and GEMM2 (H/128)
  uint8_t* w13t = nullptr;  // tiled: [E][J1][KB1][NA][16 KB]
  uint8_t* w2t = nullptr;   // tiled: [E][J2][KB2][16 KB], or paired [E][J2/2][KB2][2][16 KB] when w2_paired
  int w2_paired = 0;
  // 4-bit weight formats (W4A16): wq 0 none, 1 int4 (uint4b8, fp16 group-32 scales), 2 nvfp4 (e4m3 group-16
  // scales + f32 global), 3 mxfp4 (e8m0 group-32 scales).  Tiles are [128 rows x 64 cols]: 4096 B of nibbles followed
  // by w4_scale_bytes of scales, both in the fused kernel's wgmma fragment order (w4_layout.cuh); MMA operands are fp16.
  int wq = 0;
  int w4_tile_bytes = 0, w4_scale_bytes = 0;
  int w13_interleaved = 0;   // activation_type 1 only: gate/up rows interleaved in the checkpoint (de-interleaved at ingest)
  float* g13 = nullptr;     // nvfp4 global scales [E][2] (gate, up)
  float* g2 = nullptr;      // [E]
  float* ws13 = nullptr;    // fp8 block scales expanded to [E][N1/128][KB1]
  float* ws2 = nullptr;     // [E][H/128][KB2]
  int64_t weight_bytes = 0;
  int max_tokens;      // largest M a single pass handles without growing the workspace
  int counted = 0;     // registered in the device workspace's live-layer count
  int experts_loaded = 0;   // b200moe_create_empty / b200moe_load_experts: experts ingested so far
  int finalized = 0;
  // FP8 block-128 layers, opt-in (B200MOE_FP8_E8M0=1): DeepGEMM ue8m0 numerics of the reference — weights are
  // re-quantised at ingest to power-of-two (ue8m0) block scales (fp8_utils.py:986-1043) and every activation group scale is
  // rounded up to a power of two (fp8_utils.py:112)
  int fp8_e8m0 = 0;
  int cvt_bf16_to_fp16 = 0;   // set on the fp16 shadow of a 4-bit layer (prefill path): gather converts bf16 rows to fp16
};

namespace b200 {
void set_error(const std::string& msg);
int cuda_fail(cudaError_t e, const char* what);
extern long long g_launches;

int tm_encode_2d(CUtensorMap* tm, int dtype, const void* base, uint64_t d0, uint64_t d1, uint64_t stride1_bytes,
                 uint32_t b0, uint32_t b1);   // 2-D tiled tensor map, SWIZZLE_128B (api.cu)
// per-device launch set-up (api.cu), safe to call from several host threads.  kernel_smem raises fn's dynamic
// shared-memory limit on the current device when `bytes` exceeds what was set there before (`what` labels a failure);
// device_sms returns the SM count of `dev`.  Both return a negative B200_ERR_* code on failure.
int kernel_smem(const void* fn, int bytes, const char* what);
int device_sms(int dev);
Workspace* get_workspace(int device);
int ensure_workspace(Workspace* ws, const b200moe_layer* L, int64_t tokens, int top_k, bool may_alloc);
void release_workspace(Workspace* ws);
int ensure_dequant_scratch(Workspace* ws, int64_t bytes13, int64_t bytes2);
int launch_w4_dequant(const b200moe_layer* L, uint8_t* dq13, uint8_t* dq2, cudaStream_t st);   // repack.cu
int grow_staging(Workspace* ws, int64_t hidden_elems, int64_t slots);   // cpu_prefill host<->device staging

// kernels (moe_prep.cu / moe_gemm.cu / repack.cu)
int launch_prep(const b200moe_layer* L, Workspace* ws, cudaStream_t st, const void* hidden, const int32_t* ids,
                int M, int k, int tn_max);
int launch_gemms(const b200moe_layer* L, Workspace* ws, cudaStream_t st, int M, int k, int tn_max,
                 cudaEvent_t* ev = nullptr);
int launch_combine(const b200moe_layer* L, Workspace* ws, cudaStream_t st, const float* topk_w, int M, int k,
                   void* out, int out_dtype);
// expert-range ingest: raw checkpoint tensors of experts [e0, e0 + ne) (device memory) -> tiled layout; the destination
// buffers are allocated for the whole layer on the first call
int repack_weights(b200moe_layer* L, int e0, int ne, const void* w13_dev, const void* w2_dev, const void* s13_dev,
                   const void* s2_dev, const void* g13_dev, const void* g2_dev, cudaStream_t st);
int repack_weights_w4(b200moe_layer* L, int e0, int ne, const void* w13_dev, const void* w2_dev, const void* s13_dev,
                      const void* s2_dev, const void* g13_dev, const void* g2_dev, cudaStream_t st);
int pick_tn_max(int M, int k, int E);
int launch_mla_tc(cudaStream_t st, const void* q_nope, const void* q_pe, const void* kv, const int32_t* seq_lens,
                  const int32_t* page_table, int batch, int q_len, int Hq, int page_size, int max_pages, float sm_scale,
                  int num_splits, float* part_o, float* part_ml, int kv_fp8 = 0, int q_fp8 = 0, float descale_q = 1.f,
                  float descale_k = 1.f);
// sparse MLA decode (attention over each query token's top-k keys); kv_ds_mla: 656-byte fp8_ds_mla rows, else bf16
int launch_mla_sparse_tc(cudaStream_t st, const void* q_nope, const void* q_pe, const void* kv, int kv_ds_mla,
                         const int32_t* topk_idx, int topk, const int32_t* req_id, const int32_t* page_table, int max_pages,
                         int num_tokens, int Hq, int page_size, float sm_scale, int num_splits, float* part_o,
                         float* part_ml);
// DeepSeek-V4 sparse decode over 584-byte caches: main (sliding-window) list || optional extra (compressed) list
int launch_dsv4_sparse_tc(cudaStream_t st, const void* q, const void* swa_kv, int swa_block, int swa_blocks,
                          int64_t swa_stride, const int32_t* swa_idx, int swa_topk, const int32_t* swa_lens,
                          const void* extra_kv, int extra_block, int extra_blocks, int64_t extra_stride,
                          const int32_t* extra_idx, int extra_topk, const int32_t* extra_lens, int num_tokens, int Hq,
                          float sm_scale, int num_splits, float* part_o, float* part_ml);
// split merge of the MLA partials fused with the v up-projection (mla_aux.cu), over rows (b * q_len + i, h)
void launch_mla_merge_vup(cudaStream_t st, const float* part_o, const float* part_ml, int rows, int num_splits, int Hq,
                          const void* w_uv, void* out_v, void* out_latent, float* lse);
int launch_gqa_tc(cudaStream_t st, const void* q, const void* kc, const void* vc, int64_t block_stride, int64_t page_stride,
                  int64_t head_stride, const int32_t* seq_lens, const int32_t* page_table, int batch, int q_len, int Hq,
                  int Hkv, int page_size, int max_pages, float sm_scale, int num_splits, float* part_o, float* part_ml,
                  void* out, float* lse);
bool fused_supported(const b200moe_layer* L, int M, int k);
int launch_fused(const b200moe_layer* L, Workspace* ws, cudaStream_t st, const void* hidden, const int32_t* ids,
                 const float* topk_w, int M, int k, void* out, int out_dtype);
}  // namespace b200
