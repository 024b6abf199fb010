// One-time weight ingest: raw checkpoint layout -> kernel-native tiled layout in HBM.
//
// raw  : w13 [E][N1][Kbytes] row-major (N1 = 2I gated: rows [0,I) gate, [I,2I) up; reference
//        vllm/model_executor/layers/fused_moe/routed_experts.py:564-570),  w2 [E][H][Kbytes]
// tiled: [E][J][KB][NA][16 KB]; each 16 KB block is a [128 rows x 128 B] K-major operand tile that already
//        carries the 128-byte swizzle (16-B chunk index XOR row%8), so the GEMM streams it with one
//        contiguous bulk copy and hands it to wgmma untouched.  For gated w13, NA = 2: the gate tile
//        of output features [128j,128j+128) is followed by the matching up tile.
#include "common.cuh"
#include "moe_internal.cuh"
#include "w4_layout.cuh"

namespace b200 {

// one thread per 16-byte chunk of the destination
__global__ void __launch_bounds__(256)
    tile_weights_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int E, int J, int KB, int NA,
                        int rows_per_expert, int up_row_off, int tile_rows, int64_t row_bytes, int row_step) {
  const int64_t n_chunks = (int64_t)E * J * KB * NA * (TILE_BYTES / 16);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_chunks;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t t = i;
    const int pc = t % 8;  t /= 8;    // physical chunk within the 128-B row
    const int r = t % 128;  t /= 128;  // row within the tile
    const int na = t % NA;  t /= NA;
    const int kb = t % KB;  t /= KB;
    const int j = t % J;  t /= J;
    const int e = (int)t;
    const int lc = pc ^ (r & 7);      // logical chunk stored at this physical position
    const int64_t srow = (int64_t)e * rows_per_expert + (na ? up_row_off : 0) + ((int64_t)j * tile_rows + r) * row_step;
    const uint4 v = *reinterpret_cast<const uint4*>(src + srow * row_bytes + (int64_t)kb * 128 + lc * 16);
    *reinterpret_cast<uint4*>(dst + i * 16) = v;
  }
}

// block scales [E][N/gN][K/gK] -> [E][N/128][KB]   (gN, gK multiples of 128, or covering the whole dim)
__global__ void expand_scales_kernel(const float* __restrict__ src, float* __restrict__ dst, int E, int NB, int KB,
                                     int SN, int SK, int gN, int gK) {
  const int64_t n = (int64_t)E * NB * KB;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int kb = i % KB;
    const int nb = (i / KB) % NB;
    const int e = (int)(i / ((int64_t)KB * NB));
    int sn = (nb * 128) / gN;
    int sk = (kb * 128) / gK;
    if (sn >= SN) sn = SN - 1;
    if (sk >= SK) sk = SK - 1;
    dst[i] = src[((int64_t)e * SN + sn) * SK + sk];
  }
}

// FP8 block-128 layers in ue8m0 mode: every [128 x 128] tile (= one scale block) is de-quantised with its fp32 scale and
// re-quantised with the power-of-two scale 2^ceil(log2(max(amax, 1e-4) / 448)) — the reference's
// requant_weight_ue8m0_inplace (fp8_utils.py:986-1043) -> per_block_cast_to_fp8(use_ue8m0=True) (vllm/utils/deep_gemm.py:662-681),
// what vLLM runs when DeepGEMM serves the FP8 experts in ue8m0 mode.  In place on the tiled layout (the swizzle is irrelevant
// to an element-wise pass); one CTA per tile.  `up_off` < 0: NA tiles of a stage are consecutive row blocks (paired w2).
__global__ void __launch_bounds__(256)
    requant_e8m0_tiles_kernel(uint8_t* __restrict__ tiles, float* __restrict__ scales, int64_t n_tiles, int J, int KB, int NA,
                              int NB, int up_off) {
  __shared__ float red[8];
  for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    int64_t q = t;
    const int na = (int)(q % NA);  q /= NA;
    const int kb = (int)(q % KB);  q /= KB;
    const int j = (int)(q % J);
    const int64_t e = q / J;
    const int rb = (NA == 2) ? (up_off >= 0 ? (na ? up_off + j : j) : 2 * j + na) : j;
    float* sp = scales + (e * NB + rb) * KB + kb;
    const float s_old = *sp;
    uint4* p = reinterpret_cast<uint4*>(tiles + t * TILE_BYTES) + threadIdx.x * 4;
    float v[64];
    float am = 0.f;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const uint4 w = p[u];
      const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int b = 0; b < 16; ++b) {
        const __half_raw hr = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)((ww[b >> 2] >> (8 * (b & 3))) & 0xFFu), __NV_E4M3);
        const float f = __half2float(*reinterpret_cast<const __half*>(&hr)) * s_old;
        v[u * 16 + b] = f;
        am = fmaxf(am, fabsf(f));
      }
    }
    am = warp_max(am);
    __syncthreads();   // red[] of the previous tile has been read
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = am;
    __syncthreads();
    am = fmaxf(fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3])), fmaxf(fmaxf(red[4], red[5]), fmaxf(red[6], red[7])));
    const uint32_t sb = __float_as_uint(fmaxf(am, 1e-4f) / 448.0f);
    const float sf = __uint_as_float(((sb >> 23) + ((sb & 0x7FFFFFu) ? 1u : 0u)) << 23);
    const float inv = 1.0f / sf;   // exact: sf is a power of two
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      uint32_t ww[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int b = 0; b < 16; ++b) {
        const __nv_fp8_e4m3 qv(v[u * 16 + b] * inv);
        ww[b >> 2] |= (uint32_t)(*reinterpret_cast<const uint8_t*>(&qv)) << (8 * (b & 3));
      }
      p[u] = make_uint4(ww[0], ww[1], ww[2], ww[3]);
    }
    if (threadIdx.x == 0) *sp = sf;
  }
}

// ---------------------------------------------------------------------------------- 4-bit formats
// raw: packed nibbles u8 [E][N][K/2] (low nibble = even k; reference quant_utils.py:493-512 / nvfp4_utils.py:64-88)
// tiled: [E][J][KB][2][tile]: tile = 4096 B of nibbles in the consumers' wgmma fragment order + scales (w4_layout.cuh).
// One thread per nibble word: it gathers the word's 8 codes, two columns per source byte.
__global__ void __launch_bounds__(256)
    tile_w4_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int E, int J, int KB, int rows_per_expert,
                   int up_row_off, int tile_rows, int64_t row_bytes, int tile_bytes, int e2m1, int row_step) {
  const int64_t n_words = (int64_t)E * J * KB * 2 * (W4_NIBBLE_BYTES / 4);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t t = i;
    const int wd = t % (W4_NIBBLE_BYTES / 4);  t /= W4_NIBBLE_BYTES / 4;
    const int na = t % 2;  t /= 2;
    const int kb = t % KB;  t /= KB;
    const int j = t % J;  t /= J;
    const int e = (int)t;
    uint32_t v = 0;
#pragma unroll
    for (int reg = 0; reg < 4; ++reg) {
      const int r = w4_row(wd, reg), c = w4_col(wd, reg, 0);   // columns c (low nibble) and c + 1 (high nibble)
      const int64_t srow = (int64_t)e * rows_per_expert + (na ? up_row_off : 0) + ((int64_t)j * tile_rows + r) * row_step;
      const uint32_t by = src[srow * row_bytes + (int64_t)kb * 32 + c / 2];
      v |= w4_code_bits(e2m1, reg, 0, by & 0xFu) | w4_code_bits(e2m1, reg, 1, by >> 4);
    }
    const int64_t tile = (((int64_t)(e * J + j) * KB + kb) * 2 + na);
    reinterpret_cast<uint32_t*>(dst + tile * tile_bytes)[wd] = v;
  }
}

// scales of one tile (w4_layout.cuh): fmt 1: fp16, 2 groups of 32 columns, from act-dtype scales [E][N][K/gs]; fmt 2:
// e4m3, 4 groups of 16, from [E][N][K/16]; fmt 3: e8m0, 2 groups of 32, from [E][N][K/32]
__global__ void __launch_bounds__(256)
    tile_w4_scales_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int E, int J, int KB,
                          int rows_per_expert, int up_row_off, int tile_rows, int K, int fmt, int gs, int src_fp16,
                          int tile_bytes, int row_step) {
  const int per_tile = (fmt == 2) ? 512 : 256;
  const int64_t n = (int64_t)E * J * KB * 2 * per_tile;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t t = i;
    const int u = t % per_tile;  t /= per_tile;
    const int na = t % 2;  t /= 2;
    const int kb = t % KB;  t /= KB;
    const int j = t % J;  t /= J;
    const int e = (int)t;
    const int r = u % 128, g = u / 128;
    const int64_t srow = (int64_t)e * rows_per_expert + (na ? up_row_off : 0) + ((int64_t)j * tile_rows + r) * row_step;
    const int64_t tile = (((int64_t)(e * J + j) * KB + kb) * 2 + na);
    uint8_t* d = dst + tile * tile_bytes + W4_NIBBLE_BYTES + w4_scale_off(fmt, r, g);
    if (fmt == 1) {
      const int col = kb * 64 + g * 32;
      const int64_t si = srow * (K / gs) + col / gs;
      float f;
      if (src_fp16)
        f = __half2float(reinterpret_cast<const __half*>(src)[si]);
      else
        f = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(src)[si]);
      *reinterpret_cast<__half*>(d) = __float2half_rn(f);
    } else if (fmt == 2) {
      *d = src[srow * (K / 16) + kb * 4 + g];
    } else {
      *d = src[srow * (K / 32) + kb * 2 + g];
    }
  }
}

// Both repack entry points ingest an expert RANGE [e0, e0 + ne): the source pointers address that range's raw
// checkpoint tensors (device memory), the destination buffers are allocated for the whole layer on the first call.
int repack_weights_w4(b200moe_layer* L, int e0, int ne, const void* w13, const void* w2, const void* s13, const void* s2,
                      const void* g13, const void* g2, cudaStream_t st) {
  const int KB1 = L->H / 64, KB2 = L->I / 64;
  L->KB1 = KB1;
  L->KB2 = KB2;
  const int tb = L->w4_tile_bytes;
  const int64_t pe13 = (int64_t)L->J1 * KB1 * 2 * tb, pe2 = (int64_t)(L->J2 / 2) * KB2 * 2 * tb;   // bytes per expert
  const int64_t w13_bytes = (int64_t)L->E * pe13;
  const int64_t w2_bytes = (int64_t)L->E * pe2;
  cudaError_t e;
  if (!L->w13t) {
    if ((e = cudaMalloc(reinterpret_cast<void**>(&L->w13t), w13_bytes)) != cudaSuccess) return cuda_fail(e, "cudaMalloc(w13 w4 tiled)");
    if ((e = cudaMalloc(reinterpret_cast<void**>(&L->w2t), w2_bytes)) != cudaSuccess) return cuda_fail(e, "cudaMalloc(w2 w4 tiled)");
    L->weight_bytes = w13_bytes + w2_bytes;
    if (L->wq == 2) {
      if ((e = cudaMalloc(reinterpret_cast<void**>(&L->g13), (size_t)L->E * 2 * 4)) != cudaSuccess) return cuda_fail(e, "cudaMalloc(g13)");
      if ((e = cudaMalloc(reinterpret_cast<void**>(&L->g2), (size_t)L->E * 4)) != cudaSuccess) return cuda_fail(e, "cudaMalloc(g2)");
    }
  }
  uint8_t* d13 = L->w13t + e0 * pe13;
  uint8_t* d2 = L->w2t + e0 * pe2;
  const int e2m1 = (L->wq != 1);
  const int il = L->w13_interleaved;   // gate = even rows, up = odd rows of w13 (de-interleaved here)
  tile_w4_kernel<<<2048, 256, 0, st>>>(reinterpret_cast<const uint8_t*>(w13), d13, ne, L->J1, KB1, L->N1,
                                      il ? 1 : L->I, 128, (int64_t)L->H / 2, tb, e2m1, il ? 2 : 1);
  tile_w4_kernel<<<2048, 256, 0, st>>>(reinterpret_cast<const uint8_t*>(w2), d2, ne, L->J2 / 2, KB2, L->H, 128, 256,
                                      (int64_t)L->I / 2, tb, e2m1, 1);
  const int gs = L->cfg.groupK > 0 ? L->cfg.groupK : 32;
  tile_w4_scales_kernel<<<1024, 256, 0, st>>>(reinterpret_cast<const uint8_t*>(s13), d13, ne, L->J1, KB1, L->N1,
                                             il ? 1 : L->I, 128, L->H, L->wq, gs, L->act_dtype == B200_ACT_FP16, tb,
                                             il ? 2 : 1);
  tile_w4_scales_kernel<<<1024, 256, 0, st>>>(reinterpret_cast<const uint8_t*>(s2), d2, ne, L->J2 / 2, KB2, L->H, 128,
                                             256, L->I, L->wq, gs, L->act_dtype == B200_ACT_FP16, tb, 1);
  g_launches += 4;
  if (L->wq == 2) {
    if ((e = cudaMemcpyAsync(L->g13 + (size_t)e0 * 2, g13, (size_t)ne * 2 * 4, cudaMemcpyDefault, st)) != cudaSuccess) return cuda_fail(e, "copy g13");
    if ((e = cudaMemcpyAsync(L->g2 + e0, g2, (size_t)ne * 4, cudaMemcpyDefault, st)) != cudaSuccess) return cuda_fail(e, "copy g2");
  }
  if ((e = cudaGetLastError()) != cudaSuccess) return cuda_fail(e, "w4 repack launch");
  return 0;
}

int repack_weights(b200moe_layer* L, int e0, int ne, const void* w13, const void* w2, const void* s13, const void* s2,
                   const void* g13, const void* g2, cudaStream_t st) {
  (void)g13;
  (void)g2;
  const int NA = L->gated ? 2 : 1;
  const int64_t pe13 = (int64_t)L->J1 * L->KB1 * NA * TILE_BYTES, pe2 = (int64_t)L->J2 * L->KB2 * TILE_BYTES;
  const int64_t w13_bytes = (int64_t)L->E * pe13;
  const int64_t w2_bytes = (int64_t)L->E * pe2;
  const int NB1 = L->N1 / 128, NB2 = L->H / 128;
  const int64_t n1 = (int64_t)L->E * NB1 * L->KB1, n2 = (int64_t)L->E * NB2 * L->KB2;
  cudaError_t e;
  if (!L->w13t) {
    if ((e = cudaMalloc(reinterpret_cast<void**>(&L->w13t), w13_bytes)) != cudaSuccess) return cuda_fail(e, "cudaMalloc(w13 tiled)");
    if ((e = cudaMalloc(reinterpret_cast<void**>(&L->w2t), w2_bytes)) != cudaSuccess) return cuda_fail(e, "cudaMalloc(w2 tiled)");
    L->weight_bytes = w13_bytes + w2_bytes;
    if (L->esz_bits == 8) {
      if ((e = cudaMalloc(reinterpret_cast<void**>(&L->ws13), n1 * 4)) != cudaSuccess) return cuda_fail(e, "cudaMalloc(ws13)");
      if ((e = cudaMalloc(reinterpret_cast<void**>(&L->ws2), n2 * 4)) != cudaSuccess) return cuda_fail(e, "cudaMalloc(ws2)");
      L->weight_bytes += (n1 + n2) * 4;
    }
  }
  uint8_t* d13 = L->w13t + e0 * pe13;
  uint8_t* d2 = L->w2t + e0 * pe2;
  const int64_t rb1 = (int64_t)L->KB1 * 128, rb2 = (int64_t)L->KB2 * 128;
  const int il = L->w13_interleaved;   // gate = even rows, up = odd rows of w13 (de-interleaved here)
  tile_weights_kernel<<<2048, 256, 0, st>>>(reinterpret_cast<const uint8_t*>(w13), d13, ne, L->J1, L->KB1, NA,
                                           L->N1, il ? 1 : L->I, 128, rb1, il ? 2 : 1);
  // w2: when H/128 is even, tiles are stored in PAIRS ([E][J2/2][KB2][2][16 KB]) so that a GEMM2 stage (two
  // 128-row tiles x one k-block) is one contiguous 32 KB copy, like the (gate, up) stage of w13
  if (L->w2_paired)
    tile_weights_kernel<<<2048, 256, 0, st>>>(reinterpret_cast<const uint8_t*>(w2), d2, ne, L->J2 / 2, L->KB2, 2,
                                             L->H, 128, 256, rb2, 1);
  else
    tile_weights_kernel<<<2048, 256, 0, st>>>(reinterpret_cast<const uint8_t*>(w2), d2, ne, L->J2, L->KB2, 1,
                                             L->H, 0, 128, rb2, 1);
  g_launches += 2;
  if (L->esz_bits == 8) {
    const int gN = L->cfg.groupN > 0 ? L->cfg.groupN : 128, gK = L->cfg.groupK > 0 ? L->cfg.groupK : 128;
    const int SN1 = (L->N1 + gN - 1) / gN, SK1 = (L->H + gK - 1) / gK;
    const int SN2 = (L->H + gN - 1) / gN, SK2 = (L->I + gK - 1) / gK;
    expand_scales_kernel<<<256, 256, 0, st>>>(reinterpret_cast<const float*>(s13), L->ws13 + (int64_t)e0 * NB1 * L->KB1, ne, NB1,
                                             L->KB1, SN1, SK1, gN, gK);
    expand_scales_kernel<<<256, 256, 0, st>>>(reinterpret_cast<const float*>(s2), L->ws2 + (int64_t)e0 * NB2 * L->KB2, ne, NB2,
                                             L->KB2, SN2, SK2, gN, gK);
    g_launches += 2;
    if (L->fp8_e8m0) {
      requant_e8m0_tiles_kernel<<<4096, 256, 0, st>>>(d13, L->ws13 + (int64_t)e0 * NB1 * L->KB1, (int64_t)ne * L->J1 * L->KB1 * NA,
                                                      L->J1, L->KB1, NA, NB1, L->gated ? L->I / 128 : 0);
      if (L->w2_paired)
        requant_e8m0_tiles_kernel<<<4096, 256, 0, st>>>(d2, L->ws2 + (int64_t)e0 * NB2 * L->KB2, (int64_t)ne * L->J2 * L->KB2,
                                                        L->J2 / 2, L->KB2, 2, NB2, -1);
      else
        requant_e8m0_tiles_kernel<<<4096, 256, 0, st>>>(d2, L->ws2 + (int64_t)e0 * NB2 * L->KB2, (int64_t)ne * L->J2 * L->KB2,
                                                        L->J2, L->KB2, 1, NB2, 0);
      g_launches += 2;
    }
  }
  if ((e = cudaGetLastError()) != cudaSuccess) return cuda_fail(e, "repack launch");
  return 0;
}

// ---------------------------------------------------------------------------------- 4-bit layers, prefill-class batches
// A prefill batch (hundreds of rows per expert) is compute bound: instead of re-streaming the packed weights through the
// fused decode kernel once per 256-token pass, the layer's experts are expanded ONCE per call into fp16 MMA tiles in a
// device scratch buffer (all scales folded in, fp32 product rounded once to fp16) and the batch runs through the 16-bit
// grouped GEMM (moe_gemm_kernel).  One thread = 32 weights of one tile row.
__constant__ float c_e2m1[16] = {0.f, 0.5f, 1.f, 1.5f, 2.f, 3.f, 4.f, 6.f, -0.f, -0.5f, -1.f, -1.5f, -2.f, -3.f, -4.f, -6.f};

B200_DEVICE void store_fp16x32(uint8_t* dst_tile, int r, int chunk0, const float* v) {
#pragma unroll
  for (int ci = 0; ci < 4; ++ci) {
    uint32_t pk[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float lo = fminf(fmaxf(v[ci * 8 + 2 * q], -65504.f), 65504.f), hi = fminf(fmaxf(v[ci * 8 + 2 * q + 1], -65504.f), 65504.f);
      const __half2 h2 = __floats2half2_rn(lo, hi);
      pk[q] = *reinterpret_cast<const uint32_t*>(&h2);
    }
    *reinterpret_cast<uint4*>(dst_tile + sw128_offset(r, (chunk0 + ci) * 16)) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
  }
}

// 4-bit tiles (w4_layout.cuh) -> fp16 tiles, same tile order.  Thread (g, r) expands columns [32g, 32g + 32) of row r:
// the 8 nibble words of slices 2g and 2g + 1 that hold row r, four codes from each.
__global__ void __launch_bounds__(256)
    dequant_w4_tiles_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int64_t n_tiles, int tiles_per_expert,
                            int tile_bytes, int wq, const float* __restrict__ gscale, int gs_per_expert) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n_tiles * 256; i += (int64_t)gridDim.x * 256) {
    const int64_t t = i >> 8;
    const int u = (int)(i & 255), g = u >> 7, r = u & 127;
    const uint8_t* tile = src + t * tile_bytes;
    const uint8_t* sc = tile + W4_NIBBLE_BYTES;
    float s2[2];   // scales of columns [32g, 32g + 16) and [32g + 16, 32g + 32)
    if (wq == 1) {
      s2[0] = s2[1] = __half2float(*reinterpret_cast<const __half*>(sc + w4_scale_off(1, r, g)));
    } else if (wq == 2) {
      const int na = (int)(t & 1);
      const int e = (int)(t / tiles_per_expert);
      const float gsc = gscale[(size_t)e * gs_per_expert + (gs_per_expert == 2 ? na : 0)];
      const __half_raw h0 = __nv_cvt_fp8_to_halfraw(sc[w4_scale_off(2, r, 2 * g)], __NV_E4M3);
      const __half_raw h1 = __nv_cvt_fp8_to_halfraw(sc[w4_scale_off(2, r, 2 * g + 1)], __NV_E4M3);
      s2[0] = __half2float(*reinterpret_cast<const __half*>(&h0)) * gsc;
      s2[1] = __half2float(*reinterpret_cast<const __half*>(&h1)) * gsc;
    } else {
      s2[0] = s2[1] = __uint_as_float((uint32_t)sc[w4_scale_off(3, r, g)] << 23);   // e8m0 -> 2^(E-127)
    }
    float v[32];
#pragma unroll
    for (int c0 = 0; c0 < 32; c0 += 2) {
      const int c = 32 * g + c0;
      const uint32_t w = reinterpret_cast<const uint32_t*>(tile)[w4_word(r, c)];
      const int reg = w4_reg(r, c);
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const uint32_t q = w4_code(wq != 1, reg, e, w);
        v[c0 + e] = (wq == 1 ? (float)((int)q - 8) : c_e2m1[q]) * s2[c0 >> 4];
      }
    }
    store_fp16x32(dst + t * TILE_BYTES, r, g * 4, v);
  }
}

// expand a 4-bit layer into fp16 tiles (layout of a gated 16-bit layer with paired w2): dq13 [E][J1][H/64][2][16 KB],
// dq2 [E][J2/2][I/64][2][16 KB]
int launch_w4_dequant(const b200moe_layer* L, uint8_t* dq13, uint8_t* dq2, cudaStream_t st) {
  const int p13 = L->J1 * L->KB1 * 2, p2 = (L->J2 / 2) * L->KB2 * 2;
  dequant_w4_tiles_kernel<<<2048, 256, 0, st>>>(L->w13t, dq13, (int64_t)L->E * p13, p13, L->w4_tile_bytes, L->wq, L->g13, 2);
  dequant_w4_tiles_kernel<<<2048, 256, 0, st>>>(L->w2t, dq2, (int64_t)L->E * p2, p2, L->w4_tile_bytes, L->wq, L->g2, 1);
  g_launches += 2;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "w4 dequant launch");
  return 0;
}

}  // namespace b200
