// The MLA decode kernel's neighbours in a DeepSeek decoder layer (SURVEY.md 8f row 3), hand-written so that the
// attention block is [rope + cache write | q absorb]  ->  paged latent attention  ->  [split merge + v up-projection]:
//   mla_rope_cache_kernel   RoPE of q_pe / k_pe (reference rotary_embedding/base.py:161-201, common.py:146-185) fused with
//                           concat_and_cache_mla (csrc/libtorch_stable/cache_kernels.cu:403-444): one launch per step
//                           instead of rotary_embedding + concat_and_cache_mla, the rotated k_pe never returns to HBM twice;
//                           With kv_dtype 2 the row is the 656-byte fp8_ds_mla entry of concat_and_cache_ds_mla_kernel
//                           (cache_kernels.cu:496-590): 512 e4m3 | four fp32 scales, one per 128 dims | 64 bf16 rope dims;
//   mla_absorb_kernel       ql_nope = q_nope x W_UK^T per head (mla_attention.py:875-893; torch.bmm in the reference);
//   mla_merge_vup_kernel    the split merge of the decode kernel fused with the v up-projection (mla_attention.py:1154-1176):
//                           the merged [512] latent output of a (request, head) never leaves shared memory;
//   dsv4_qnorm_rope_kv_insert_kernel  DeepSeek-V4: q per-head RMSNorm (no weight) + GPT-J RoPE of the last 64 dims, and kv
//                           RoPE + ue8m0 e4m3 quantisation + insert into the 584-byte cache, in one launch (reference
//                           csrc/libtorch_stable/fused_deepseek_v4_qnorm_rope_kv_insert_kernel.cu:179-379).
// All three are HBM / latency bound (W_UK_T and W_UV are 16.8 MB each for 128 heads): coalesced 16-byte loads, every
// load of a thread's work issued before the first use, fp32 accumulation in a fixed order (deterministic).
#include <math_constants.h>

#include <cfloat>

#include "common.cuh"
#include "kv_pack.cuh"
#include "moe_internal.cuh"

namespace b200 {

B200_DEVICE float bf(const __nv_bfloat16& v) { return __bfloat162float(v); }

// grid = tokens, 128 threads
__global__ void __launch_bounds__(128)
    mla_rope_cache_kernel(__nv_bfloat16* __restrict__ q_pe, __nv_bfloat16* __restrict__ k_pe,
                          const __nv_bfloat16* __restrict__ kv_c, const int64_t* __restrict__ positions,
                          const __nv_bfloat16* __restrict__ cos_sin, int is_neox, const int64_t* __restrict__ slot_mapping,
                          void* __restrict__ kv_cache, int kv_dtype, float inv_scale, int Hq) {
  const int t = blockIdx.x, tid = threadIdx.x;
  __shared__ float cs[64];   // cos[0..32) | sin[0..32) of this token's position
  if (tid < 64) cs[tid] = bf(cos_sin[(size_t)positions[t] * 64 + tid]);
  __syncthreads();
  // rotate the Hq query rope heads in place and the (single) key rope head; pair p of a head = (x1, x2):
  // GPT-J style (DeepSeek): elements (2p, 2p+1); NeoX style: (p, p + 32)
  const int64_t slot = slot_mapping ? slot_mapping[t] : -1;
  const bool kv_fp8 = kv_dtype == 1, ds_mla = kv_dtype == 2;
  uint8_t* crow8 = reinterpret_cast<uint8_t*>(kv_cache) + (size_t)(slot < 0 ? 0 : slot) * (ds_mla ? 656 : 576);
  __nv_bfloat16* crow = reinterpret_cast<__nv_bfloat16*>(kv_cache) + (size_t)(slot < 0 ? 0 : slot) * 576;
  for (int i = tid; i < (Hq + 1) * 32; i += 128) {
    const int hd = i >> 5, p = i & 31;
    const bool is_k = hd == Hq;
    __nv_bfloat16* x = is_k ? k_pe + (size_t)t * 64 : q_pe + ((size_t)t * Hq + hd) * 64;
    const int i1 = is_neox ? p : 2 * p, i2 = is_neox ? p + 32 : 2 * p + 1;
    const float x1 = bf(x[i1]), x2 = bf(x[i2]);
    const float c = cs[p], s = cs[32 + p];
    const __nv_bfloat16 o1 = __float2bfloat16_rn(x1 * c - x2 * s), o2 = __float2bfloat16_rn(x2 * c + x1 * s);
    x[i1] = o1;
    x[i2] = o2;
    if (is_k && slot >= 0) {
      if (ds_mla) {
        reinterpret_cast<__nv_bfloat16*>(crow8 + 528)[i1] = o1;
        reinterpret_cast<__nv_bfloat16*>(crow8 + 528)[i2] = o2;
      } else if (kv_fp8) {
        crow8[512 + i1] = __nv_cvt_float_to_fp8(bf(o1) * inv_scale, __NV_SATFINITE, __NV_E4M3);
        crow8[512 + i2] = __nv_cvt_float_to_fp8(bf(o2) * inv_scale, __NV_SATFINITE, __NV_E4M3);
      } else {
        crow[512 + i1] = o1;
        crow[512 + i2] = o2;
      }
    }
  }
  if (slot >= 0 && ds_mla) {
    // threads 0-63 take 8 values each, a half-warp per 128-dim tile: scale = max(amax / 448, FLT_MIN), e4m3(value / scale)
    if (tid < 64) {
      const uint4 v = *reinterpret_cast<const uint4*>(kv_c + (size_t)t * 512 + tid * 8);
      const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&v);
      float amax = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(bf(h[j])));
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, off, 16));
      const float scale = fmaxf(__fdiv_rn(amax, 448.f), FLT_MIN);
      if ((tid & 15) == 0) reinterpret_cast<float*>(crow8 + 512)[tid >> 4] = scale;
      uint8_t o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = __nv_cvt_float_to_fp8(__fdiv_rn(bf(h[j]), scale), __NV_SATFINITE, __NV_E4M3);
      *reinterpret_cast<uint2*>(crow8 + tid * 8) = *reinterpret_cast<const uint2*>(o);
    }
  } else if (slot >= 0) {
    const __nv_bfloat16* src = kv_c + (size_t)t * 512;
    for (int i = tid; i < 512 / 8; i += 128) {
      const uint4 v = *reinterpret_cast<const uint4*>(src + i * 8);
      if (kv_fp8) {
        const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&v);
        uint8_t o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = __nv_cvt_float_to_fp8(bf(h[j]) * inv_scale, __NV_SATFINITE, __NV_E4M3);
        *reinterpret_cast<uint2*>(crow8 + i * 8) = *reinterpret_cast<const uint2*>(o);
      } else {
        *reinterpret_cast<uint4*>(crow + i * 8) = v;
      }
    }
  }
}

// out[t,h,n] = sum_k q[t,h,k] * W[h,k,n];  q [T,Hq,128], W_UK_T [Hq,128,512], out [T,Hq,512]
// grid (Hq, 4): thread = one output column; tokens in blocks of 8 share every weight load
__global__ void __launch_bounds__(128)
    mla_absorb_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ w,
                      __nv_bfloat16* __restrict__ out, int T, int Hq) {
  const int h = blockIdx.x, n = blockIdx.y * 128 + threadIdx.x;
  __shared__ float qs[8][128];
  const __nv_bfloat16* wh = w + (size_t)h * 128 * 512 + n;
  for (int t0 = 0; t0 < T; t0 += 8) {
    const int nt = min(8, T - t0);
    __syncthreads();
    for (int i = threadIdx.x; i < 8 * 128; i += 128) {
      const int tt = i >> 7, k = i & 127;
      qs[tt][k] = tt < nt ? bf(q[((size_t)(t0 + tt) * Hq + h) * 128 + k]) : 0.f;
    }
    __syncthreads();
    float acc[8];
#pragma unroll
    for (int tt = 0; tt < 8; ++tt) acc[tt] = 0.f;
    for (int k0 = 0; k0 < 128; k0 += 16) {
      float wv[16];
#pragma unroll
      for (int u = 0; u < 16; ++u) wv[u] = bf(wh[(size_t)(k0 + u) * 512]);
#pragma unroll
      for (int u = 0; u < 16; ++u)
#pragma unroll
        for (int tt = 0; tt < 8; ++tt) acc[tt] = fmaf(qs[tt][k0 + u], wv[u], acc[tt]);
    }
    for (int tt = 0; tt < nt; ++tt) out[((size_t)(t0 + tt) * Hq + h) * 512 + n] = __float2bfloat16_rn(acc[tt]);
  }
}

// grid = B*Q*Hq (rows w = (b * Q + i) * Hq + h), 512 threads.  Partials from mla_decode_tc_kernel: part_o [B*Q*Hq][splits][512]
// (un-normalised), part_ml [B*Q*Hq][splits][2] = (m * scale * log2e, l).  out_v [B*Q,Hq,128] = (merged o, rounded to bf16 as
// the unfused path would) x W_UV[h] ([512,128]); out_o (optional) the merged latent output [B*Q,Hq,512]; lse optional.  A row
// whose every split published m = -inf (no visible key) gets out_v = 0, out_o = 0 and lse = -inf.
__global__ void __launch_bounds__(512)
    mla_merge_vup_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml, int num_splits, int Hq,
                         const __nv_bfloat16* __restrict__ w_uv, __nv_bfloat16* __restrict__ out_v,
                         __nv_bfloat16* __restrict__ out_o, float* __restrict__ lse) {
  __shared__ float wgt[512];
  __shared__ float red[16];
  __shared__ float4 osum[4][128];
  __shared__ float o_s[512];
  __shared__ float vred[32][128];
  const int w = blockIdx.x, tid = threadIdx.x, h = w % Hq;
  const float* ml = part_ml + (size_t)w * num_splits * 2;
  float mx = -CUDART_INF_F;
  for (int s = tid; s < num_splits; s += 512) mx = fmaxf(mx, ml[s * 2]);
  mx = warp_max(mx);
  if ((tid & 31) == 0) red[tid >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int i = 1; i < 16; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float ls = 0.f;
  for (int s = tid; s < num_splits; s += 512) {
    const float ms = ml[s * 2];
    const float f = (ms == -CUDART_INF_F) ? 0.f : exp2f(ms - mx);
    wgt[s] = f;
    ls += f * ml[s * 2 + 1];
  }
  ls = warp_sum(ls);
  if ((tid & 31) == 0) red[tid >> 5] = ls;
  __syncthreads();
  float lsum = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) lsum += red[i];
  // merge: thread (sg, d4) sums the splits s = sg (mod 4) of float4 column d4; the four group sums are added in order
  {
    const int sg = tid >> 7, d4 = tid & 127;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const float* po = part_o + (size_t)w * num_splits * 512 + d4 * 4;
    for (int s0 = sg; s0 < num_splits; s0 += 4 * 8) {
      float4 v[8];
      float f[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int s = s0 + 4 * u;
        f[u] = (s < num_splits) ? wgt[s] : 0.f;
        v[u] = (f[u] != 0.f) ? __ldcs(reinterpret_cast<const float4*>(po + (size_t)s * 512)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        acc.x = fmaf(f[u], v[u].x, acc.x);
        acc.y = fmaf(f[u], v[u].y, acc.y);
        acc.z = fmaf(f[u], v[u].z, acc.z);
        acc.w = fmaf(f[u], v[u].w, acc.w);
      }
    }
    osum[sg][d4] = acc;
  }
  __syncthreads();
  const float inv = lsum > 0.f ? 1.f / lsum : 0.f;
  if (tid < 128) {
    float4 a = osum[0][tid];
#pragma unroll
    for (int g = 1; g < 4; ++g) {
      a.x += osum[g][tid].x;
      a.y += osum[g][tid].y;
      a.z += osum[g][tid].z;
      a.w += osum[g][tid].w;
    }
    const __nv_bfloat162 lo = __floats2bfloat162_rn(a.x * inv, a.y * inv), hi = __floats2bfloat162_rn(a.z * inv, a.w * inv);
    o_s[tid * 4 + 0] = __low2float(lo);
    o_s[tid * 4 + 1] = __high2float(lo);
    o_s[tid * 4 + 2] = __low2float(hi);
    o_s[tid * 4 + 3] = __high2float(hi);
    if (out_o) {
      uint2 pk;
      pk.x = *reinterpret_cast<const uint32_t*>(&lo);
      pk.y = *reinterpret_cast<const uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(out_o + (size_t)w * 512 + tid * 4) = pk;
    }
  }
  if (tid == 0 && lse) lse[w] = (lsum > 0.f) ? (mx + log2f(lsum)) * 0.6931471805599453f : -CUDART_INF_F;
  __syncthreads();
  // v up-projection: thread (kg, n8) handles k = kg + 32*kk (kk < 16) for 8 output columns: 16 independent 16-byte loads
  {
    const int kg = tid >> 4, n8 = tid & 15;
    const __nv_bfloat16* wb = w_uv + (size_t)h * 512 * 128 + n8 * 8;
    uint4 wv[16];
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) wv[kk] = __ldg(reinterpret_cast<const uint4*>(wb + (size_t)(kg + 32 * kk) * 128));
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      const float ov = o_s[kg + 32 * kk];
      const __nv_bfloat16* hv = reinterpret_cast<const __nv_bfloat16*>(&wv[kk]);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaf(ov, bf(hv[j]), acc[j]);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) vred[kg][n8 * 8 + j] = acc[j];
  }
  __syncthreads();
  if (tid < 128) {
    float s = 0.f;
#pragma unroll
    for (int kg = 0; kg < 32; ++kg) s += vred[kg][tid];
    out_v[(size_t)w * 128 + tid] = __float2bfloat16_rn(s);
  }
}

// grid = tokens, 256 threads.  Warp w takes the head slots w, w + 8, ... of [0, Hp]: slot h < Hq is query head h, Hq <= h < Hp a
// padded head (written as zeros) and Hp the token's kv row.  Lane l holds dims [16l, 16l + 16); lanes 28-31 the 64 rope dims.
//   q:  x * rsqrt(mean(x^2) + eps), then the rope pairs (2p, 2p+1) rotated by (cos, sin)[pos][p]; fp32 throughout, rounded to
//       bf16 once, into q_out [T, Hp, 512].
//   kv: the rope pairs rotated, every value rounded to bf16; NoPE dims [64g, 64g + 64) (one quad of lanes) quantised with
//       scale = 2^ceil(log2(max(amax, 1e-4) / 448)), byte e4m3(x / scale) (saturating) and ue8m0 byte log2(scale) + 127;
//       row slot_mapping[t] of the cache (block slot / block_size, position slot % block_size, blocks block_stride bytes
//       apart): 448 e4m3 | 64 bf16 rope at pos * 576, the 7 scale bytes and a zero pad byte at block_size * 576 + pos * 8.
//       A slot < 0 or past the cache writes nothing.
__global__ void __launch_bounds__(256)
    dsv4_qnorm_rope_kv_insert_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ kv,
                                     const int64_t* __restrict__ positions, const float* __restrict__ cos_sin, int max_pos,
                                     const int64_t* __restrict__ slot_mapping, uint8_t* __restrict__ cache, int block_size,
                                     int num_blocks, int64_t block_stride, __nv_bfloat16* __restrict__ q_out, int Hq, int Hp,
                                     float eps) {
  const int t = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d0 = lane * 16;
  const bool rope = d0 >= 448;
  int64_t pos = positions[t];
  pos = pos < 0 ? 0 : (pos >= max_pos ? max_pos - 1 : pos);
  float cs[8], sn[8];
  if (rope) {
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      cs[p] = cos_sin[pos * 64 + (d0 - 448) / 2 + p];
      sn[p] = cos_sin[pos * 64 + 32 + (d0 - 448) / 2 + p];
    }
  }
  for (int h = warp; h <= Hp; h += 8) {
    const bool is_kv = h == Hp;
    __nv_bfloat16* qo = q_out + ((size_t)t * Hp + h) * 512 + d0;
    if (!is_kv && h >= Hq) {
      *reinterpret_cast<uint4*>(qo) = make_uint4(0u, 0u, 0u, 0u);
      *reinterpret_cast<uint4*>(qo + 8) = make_uint4(0u, 0u, 0u, 0u);
      continue;
    }
    const int64_t slot = is_kv ? slot_mapping[t] : 0;
    if (is_kv && (slot < 0 || slot >= (int64_t)num_blocks * block_size)) continue;
    const __nv_bfloat16* src = is_kv ? kv + (size_t)t * 512 + d0 : q + ((size_t)t * Hq + h) * 512 + d0;
    uint4 raw[2] = {*reinterpret_cast<const uint4*>(src), *reinterpret_cast<const uint4*>(src + 8)};
    const __nv_bfloat16* hv = reinterpret_cast<const __nv_bfloat16*>(raw);
    float x[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) x[i] = bf(hv[i]);
    if (!is_kv) {
      float ss = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) ss = fmaf(x[i], x[i], ss);
      ss = warp_sum(ss);
      const float r = rsqrtf(ss / 512.f + eps);
#pragma unroll
      for (int i = 0; i < 16; ++i) x[i] *= r;
    }
    if (rope) {
#pragma unroll
      for (int p = 0; p < 8; ++p) {
        const float e = x[2 * p], o = x[2 * p + 1];
        x[2 * p] = fmaf(e, cs[p], -(o * sn[p]));
        x[2 * p + 1] = fmaf(e, sn[p], o * cs[p]);
      }
    }
    if (is_kv) {   // the NoPE values are bf16 already, so the packer's rounding leaves them as they are
      dsv4_pack_row584(x, cache + (size_t)(slot / block_size) * (size_t)block_stride, block_size, (int)(slot % block_size),
                       lane);
      continue;
    }
    uint32_t pk[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const __nv_bfloat162 b2 = __floats2bfloat162_rn(x[2 * i], x[2 * i + 1]);
      pk[i] = *reinterpret_cast<const uint32_t*>(&b2);
    }
    *reinterpret_cast<uint4*>(qo) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    *reinterpret_cast<uint4*>(qo + 8) = make_uint4(pk[4], pk[5], pk[6], pk[7]);
  }
}

void launch_mla_merge_vup(cudaStream_t st, const float* part_o, const float* part_ml, int rows, int num_splits, int Hq,
                          const void* w_uv, void* out_v, void* out_latent, float* lse) {
  mla_merge_vup_kernel<<<rows * Hq, 512, 0, st>>>(part_o, part_ml, num_splits, Hq, reinterpret_cast<const __nv_bfloat16*>(w_uv),
                                                 reinterpret_cast<__nv_bfloat16*>(out_v),
                                                 reinterpret_cast<__nv_bfloat16*>(out_latent), lse);
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_mla_rope_cache_write(void* stream, void* q_pe, void* k_pe, const void* kv_c, const int64_t* positions,
                              const void* cos_sin_cache, int is_neox, const int64_t* slot_mapping, void* kv_cache,
                              int kv_dtype, float kv_scale, int num_tokens, int num_heads) {
  if (!q_pe || !k_pe || !kv_c || !positions || !cos_sin_cache || !kv_cache || num_heads <= 0 || kv_dtype < 0 || kv_dtype > 2 ||
      !(kv_scale > 0.f)) {
    set_error("b200_mla_rope_cache_write: bad argument");
    return B200_ERR_INVALID;
  }
  if (num_tokens <= 0) return 0;
  mla_rope_cache_kernel<<<num_tokens, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<__nv_bfloat16*>(q_pe), reinterpret_cast<__nv_bfloat16*>(k_pe),
      reinterpret_cast<const __nv_bfloat16*>(kv_c), positions, reinterpret_cast<const __nv_bfloat16*>(cos_sin_cache), is_neox,
      slot_mapping, kv_cache, kv_dtype, 1.0f / kv_scale, num_heads);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "mla_rope_cache launch");
  return 0;
}

int b200_mla_q_absorb(void* stream, const void* q_nope, const void* w_uk_t, void* out, int num_tokens, int num_heads) {
  if (!q_nope || !w_uk_t || !out || num_heads <= 0) {
    set_error("b200_mla_q_absorb: bad argument");
    return B200_ERR_INVALID;
  }
  if (num_tokens <= 0) return 0;
  mla_absorb_kernel<<<dim3(num_heads, 4), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(q_nope), reinterpret_cast<const __nv_bfloat16*>(w_uk_t),
      reinterpret_cast<__nv_bfloat16*>(out), num_tokens, num_heads);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "mla_absorb launch");
  return 0;
}

int b200_mla_decode_vup(void* stream, const void* q_nope, const void* q_pe, int q_dtype, const void* kv_cache, int kv_dtype,
                        float descale_q, float descale_k, const int32_t* seq_lens, const int32_t* page_table, int batch,
                        int num_heads, int page_size, int max_pages, float sm_scale, int num_splits, void* workspace,
                        const void* w_uv, void* out_v, void* out_latent, float* lse) {
  if (!w_uv) {   // without W_UV this is b200_mla_decode_ex, which has its own entry point
    set_error("b200_mla_decode_vup: bad argument (w_uv, num_heads <= 128, num_splits <= 512)");
    return B200_ERR_INVALID;
  }
  return b200_mla_decode_spec(stream, q_nope, q_pe, q_dtype, kv_cache, kv_dtype, descale_q, descale_k, seq_lens, page_table,
                              batch, 1, num_heads, page_size, max_pages, sm_scale, num_splits, workspace, out_latent, lse,
                              w_uv, out_v);
}

int b200_dsv4_qnorm_rope_kv_insert(void* stream, const void* q, const void* kv, const int64_t* positions,
                                   const float* cos_sin_cache, int max_position, const int64_t* slot_mapping, void* cache,
                                   int block_size, int num_blocks, int64_t block_stride, void* q_out, int num_tokens,
                                   int num_heads, int q_head_padded, float eps) {
  auto a16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
  if (!q || !a16(q) || !kv || !a16(kv) || !positions || !cos_sin_cache || (reinterpret_cast<uintptr_t>(cos_sin_cache) & 3u) ||
      max_position <= 0 || !slot_mapping || !cache || !a16(cache) || block_size <= 0 || num_blocks <= 0 ||
      block_stride < (int64_t)block_size * 584 || block_stride % 16 != 0 || !q_out || !a16(q_out) || num_tokens < 0 ||
      num_heads <= 0 || q_head_padded < num_heads || !(eps >= 0.f)) {
    set_error("b200_dsv4_qnorm_rope_kv_insert: bad argument (16-byte aligned q, kv, cache and q_out, q_head_padded >= "
              "num_heads, block stride >= block_size * 584 and a multiple of 16)");
    return B200_ERR_INVALID;
  }
  if (num_tokens == 0) return 0;
  dsv4_qnorm_rope_kv_insert_kernel<<<num_tokens, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(kv), positions, cos_sin_cache,
      max_position, slot_mapping, reinterpret_cast<uint8_t*>(cache), block_size, num_blocks, block_stride,
      reinterpret_cast<__nv_bfloat16*>(q_out), num_heads, q_head_padded, eps);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "dsv4_qnorm_rope_kv_insert launch");
  return 0;
}

}  // extern "C"
