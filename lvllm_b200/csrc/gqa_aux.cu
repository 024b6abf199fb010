// The GQA decode kernel's neighbour in a Qwen3 / Mixtral decoder layer, hand-written so that the attention block is
// [qk norm + rope + cache write]  ->  paged GQA decode on the same cache:
//   gqa_qknorm_rope_cache_kernel  per-head RMSNorm of q and k (Qwen3, models/qwen3_moe.py:333-351; optional), RoPE of q
//                                 and k (rotary_embedding/base.py:161-201, common.py:146-185) and reshape_and_cache_flash
//                                 (csrc/libtorch_stable/cache_kernels.cu:315-400) of the new k / v rows in one launch;
//                                 the reference runs fused_qk_norm_rope (vllm/_custom_ops.py:279) and the cache write
//                                 separately.  The rotated q goes to a contiguous [T, Hq, 128] buffer, the layout
//                                 b200_gqa_decode takes.
// Warp = one (token, head) of 128 dims: lane l owns dims [4l, 4l + 4) and moves them with 8-byte accesses.  q-head warps
// write q_out; kv-head warps write the k and v rows of the token's slot.  HBM / launch-latency bound
// (2 * T * (Hq + 2 Hkv) * 128 * 2 bytes).
// Numerics: the norm is vllm/ir/ops/layernorm.py:10-21 in its order (fp32 statistics, round to bf16, times the weight with
// one rounding); RoPE is computed in fp32 from the bf16 inputs and rounded once (the policy of mla_rope_cache_kernel,
// <= 2 bf16 ulp of the pair's magnitude from forward_static, which rounds after every bf16 op).
#include "common.cuh"
#include "moe_internal.cuh"

namespace b200 {

constexpr int GQA_AUX_WARPS = 4;

B200_DEVICE float bfr(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

// grid = ceil(T * (Hq + Hkv) / 4), 128 threads.  qkv [T, (Hq + 2 Hkv) * 128]; warp w -> token w / (Hq + Hkv), head
// w % (Hq + Hkv) (q heads first, then kv heads).
__global__ void __launch_bounds__(GQA_AUX_WARPS * 32)
    gqa_qknorm_rope_cache_kernel(const __nv_bfloat16* __restrict__ qkv, const int64_t* __restrict__ positions,
                                 const __nv_bfloat16* __restrict__ cos_sin, int max_position, int rot, int is_neox,
                                 const __nv_bfloat16* __restrict__ q_w, const __nv_bfloat16* __restrict__ k_w, float eps,
                                 const int64_t* __restrict__ slot_mapping, __nv_bfloat16* __restrict__ k_cache,
                                 __nv_bfloat16* __restrict__ v_cache, int64_t block_stride, int64_t page_stride,
                                 int64_t head_stride, int page_size, __nv_bfloat16* __restrict__ q_out, int T, int Hq,
                                 int Hkv) {
  __shared__ float xs[GQA_AUX_WARPS][128];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int w = blockIdx.x * GQA_AUX_WARPS + warp;
  const int nh = Hq + Hkv;
  if (w >= T * nh) return;   // whole warps only: nothing below synchronises more than the warp
  const int t = w / nh, h = w % nh;
  const bool is_k = h >= Hq;
  const int64_t slot = is_k ? slot_mapping[t] : 0;
  if (slot < 0) return;      // padded token: the kv warp writes nothing
  const __nv_bfloat16* src = qkv + (size_t)t * (Hq + 2 * Hkv) * 128 + (size_t)h * 128 + lane * 4;
  const uint2 raw = *reinterpret_cast<const uint2*>(src);
  uint2 vraw;
  if (is_k) vraw = *reinterpret_cast<const uint2*>(src + (size_t)Hkv * 128);   // v row: copied untouched
  int64_t pos = positions[t];
  pos = pos < 0 ? 0 : (pos >= max_position ? max_position - 1 : pos);
  const __nv_bfloat16* hx = reinterpret_cast<const __nv_bfloat16*>(&raw);
  float x[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) x[i] = __bfloat162float(hx[i]);
  const __nv_bfloat16* nw = is_k ? k_w : q_w;
  if (nw) {
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) ss = fmaf(x[i], x[i], ss);
    ss = warp_sum(ss);
    const float inv = 1.f / sqrtf(ss / 128.f + eps);
    const uint2 wraw = *reinterpret_cast<const uint2*>(nw + lane * 4);
    const __nv_bfloat16* hw = reinterpret_cast<const __nv_bfloat16*>(&wraw);
#pragma unroll
    for (int i = 0; i < 4; ++i) x[i] = bfr(bfr(x[i] * inv) * __bfloat162float(hw[i]));
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) xs[warp][lane * 4 + i] = x[i];
  __syncwarp();
  // pair p of the rotated dims = (x1, x2): NeoX (p, p + rot/2), GPT-J (2p, 2p + 1); o1 = x1 c - x2 s, o2 = x2 c + x1 s
  const __nv_bfloat16* cs = cos_sin + pos * rot;
  const int half = rot >> 1;
  float o[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int e = lane * 4 + i;
    o[i] = x[i];
    if (e < rot) {
      const bool second = is_neox ? e >= half : (e & 1);
      const int p = is_neox ? (second ? e - half : e) : e >> 1;
      const int partner = is_neox ? (second ? e - half : e + half) : (e ^ 1);
      const float c = __bfloat162float(cs[p]), s = __bfloat162float(cs[half + p]);
      const float y = xs[warp][partner];
      o[i] = second ? x[i] * c + y * s : x[i] * c - y * s;
    }
  }
  const __nv_bfloat162 lo = __floats2bfloat162_rn(o[0], o[1]), hi = __floats2bfloat162_rn(o[2], o[3]);
  uint2 pk;
  pk.x = *reinterpret_cast<const uint32_t*>(&lo);
  pk.y = *reinterpret_cast<const uint32_t*>(&hi);
  if (!is_k) {
    *reinterpret_cast<uint2*>(q_out + ((size_t)t * Hq + h) * 128 + lane * 4) = pk;
    return;
  }
  const int64_t off = (slot / page_size) * block_stride + (slot % page_size) * page_stride + (int64_t)(h - Hq) * head_stride +
                      lane * 4;
  *reinterpret_cast<uint2*>(k_cache + off) = pk;
  *reinterpret_cast<uint2*>(v_cache + off) = vraw;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_gqa_qknorm_rope_cache_write(void* stream, const void* qkv, const int64_t* positions, const void* cos_sin_cache,
                                     int max_position, int rotary_dim, int is_neox, const void* q_weight,
                                     const void* k_weight, float eps, const int64_t* slot_mapping, void* k_cache,
                                     void* v_cache, int64_t block_stride, int64_t page_stride, int64_t head_stride,
                                     int page_size, void* q_out, int num_tokens, int num_heads, int num_kv_heads,
                                     int head_dim) {
  if (!qkv || !positions || !cos_sin_cache || !slot_mapping || !k_cache || !v_cache || !q_out || num_heads <= 0 ||
      num_kv_heads <= 0 || page_size <= 0 || max_position <= 0 || num_tokens < 0) {
    set_error("b200_gqa_qknorm_rope_cache_write: bad argument");
    return B200_ERR_INVALID;
  }
  if (head_dim != 128) {
    set_error("b200_gqa_qknorm_rope_cache_write: head_dim must be 128");
    return B200_ERR_INVALID;
  }
  if (rotary_dim <= 0 || rotary_dim % 2 || rotary_dim > head_dim) {
    set_error("b200_gqa_qknorm_rope_cache_write: rotary_dim must be even and in (0, head_dim]");
    return B200_ERR_INVALID;
  }
  if (block_stride <= 0 || page_stride <= 0 || head_stride <= 0 || block_stride % 8 || page_stride % 8 || head_stride % 8 ||
      (reinterpret_cast<uintptr_t>(k_cache) | reinterpret_cast<uintptr_t>(v_cache) | reinterpret_cast<uintptr_t>(qkv) |
       reinterpret_cast<uintptr_t>(q_out)) % 16) {
    set_error("b200_gqa_qknorm_rope_cache_write: cache strides must be positive multiples of 8 elements, pointers 16-byte aligned");
    return B200_ERR_INVALID;
  }
  if (num_tokens == 0) return 0;
  const int warps = num_tokens * (num_heads + num_kv_heads);
  gqa_qknorm_rope_cache_kernel<<<(warps + GQA_AUX_WARPS - 1) / GQA_AUX_WARPS, GQA_AUX_WARPS * 32, 0,
                                 reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(qkv), positions, reinterpret_cast<const __nv_bfloat16*>(cos_sin_cache),
      max_position, rotary_dim, is_neox, reinterpret_cast<const __nv_bfloat16*>(q_weight),
      reinterpret_cast<const __nv_bfloat16*>(k_weight), eps, slot_mapping, reinterpret_cast<__nv_bfloat16*>(k_cache),
      reinterpret_cast<__nv_bfloat16*>(v_cache), block_stride, page_stride, head_stride, page_size,
      reinterpret_cast<__nv_bfloat16*>(q_out), num_tokens, num_heads, num_kv_heads);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "gqa_qknorm_rope_cache launch");
  return 0;
}

}  // extern "C"
