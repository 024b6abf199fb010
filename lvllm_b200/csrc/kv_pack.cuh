// Row packers of the two fp8 key caches DeepSeek-V4 layers write, shared by every kernel that stores into them (the V4 kv
// insert, the V3.2 indexer's k side and the V4 compressor), so that each format's bytes are written by one piece of code.
#pragma once
#include "common.cuh"

namespace b200 {

// One 584-byte row of the DeepSeek-V4 attention cache, written by a whole warp (every lane calls it): lane l holds dims
// [16l, 16l + 16) of the 512 as fp32; lanes 28-31 are the 64 rope dims.  Every value is rounded to bf16 first; the NoPE
// dims [64g, 64g + 64) (one quad of lanes) are quantised with scale = 2^ceil(log2(max(amax, 1e-4) / 448)), byte
// e4m3(x / scale) (saturating) and ue8m0 byte log2(scale) + 127; the rope dims are stored as bf16.  blk is the row's cache
// block: 448 e4m3 | 64 bf16 at p_in * 576, the 7 scale bytes and a zero pad byte at block_size * 576 + p_in * 8.
B200_DEVICE void dsv4_pack_row584(const float (&x)[16], uint8_t* blk, int block_size, int p_in, int lane) {
  const int d0 = lane * 16;
  const bool rope = d0 >= 448;
  uint32_t pk[8];
  float xr[16];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const __nv_bfloat162 b2 = __floats2bfloat162_rn(x[2 * i], x[2 * i + 1]);
    pk[i] = *reinterpret_cast<const uint32_t*>(&b2);
    xr[2 * i] = __low2float(b2);
    xr[2 * i + 1] = __high2float(b2);
  }
  uint8_t* row = blk + (size_t)p_in * 576;
  if (rope) {
    *reinterpret_cast<uint4*>(row + 448 + (d0 - 448) * 2) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    *reinterpret_cast<uint4*>(row + 448 + (d0 - 448) * 2 + 16) = make_uint4(pk[4], pk[5], pk[6], pk[7]);
  }
  // the quantised block is a quad of lanes
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) amax = fmaxf(amax, fabsf(xr[i]));
  amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
  amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
  if (!rope) {
    const uint32_t e = __float_as_uint(ue8m0_ceil(__fdiv_rn(fmaxf(amax, 1e-4f), 448.f))) >> 23;   // ue8m0 byte
    const float inv = __uint_as_float((254u - e) << 23);                                            // 1 / scale, exact
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t lo =
          __nv_cvt_float2_to_fp8x2(make_float2(xr[4 * i] * inv, xr[4 * i + 1] * inv), __NV_SATFINITE, __NV_E4M3);
      const uint32_t hi =
          __nv_cvt_float2_to_fp8x2(make_float2(xr[4 * i + 2] * inv, xr[4 * i + 3] * inv), __NV_SATFINITE, __NV_E4M3);
      o[i] = lo | (hi << 16);
    }
    *reinterpret_cast<uint4*>(row + d0) = make_uint4(o[0], o[1], o[2], o[3]);
    uint8_t* srec = blk + (size_t)block_size * 576 + (size_t)p_in * 8;
    if ((lane & 3) == 0) srec[lane >> 2] = (uint8_t)e;
    if (lane == 0) srec[7] = 0;
  }
}

// One 132-byte row of the indexer's key cache (indexer_k_quant_and_cache layout), written by a whole warp: lane l holds
// dims [4l, 4l + 4) of the 128 as fp32.  Every value is rounded to bf16 first; scale = max(amax, 1e-4) / 448 over the
// row, its power-of-two ceiling when ue8m0; byte = e4m3(x / scale), saturating.  blk is the row's cache block:
// block_size x 128 e4m3 bytes, then block_size fp32 scales.
B200_DEVICE void indexer_pack_row132(const float (&x)[4], bool ue8m0, uint8_t* blk, int block_size, int p_in, int lane) {
  float xr[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) xr[i] = __bfloat162float(__float2bfloat16_rn(x[i]));
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) amax = fmaxf(amax, fabsf(xr[i]));
  amax = warp_max(amax);
  float sc = __fdiv_rn(fmaxf(amax, 1e-4f), 448.0f);
  if (ue8m0) sc = ue8m0_ceil(sc);
  const uint32_t lo =
      __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(xr[0], sc), __fdiv_rn(xr[1], sc)), __NV_SATFINITE, __NV_E4M3);
  const uint32_t hi =
      __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(xr[2], sc), __fdiv_rn(xr[3], sc)), __NV_SATFINITE, __NV_E4M3);
  *reinterpret_cast<uint32_t*>(blk + (size_t)p_in * 128 + lane * 4) = (lo & 0xFFFFu) | (hi << 16);
  if (lane == 0) *reinterpret_cast<float*>(blk + (size_t)block_size * 128 + p_in * 4) = sc;
}

}  // namespace b200
