// DeepSeek-V4 attention output projection for decode: the first two of the three steps of the reference's
// deep_gemm_fp8_o_proj (models/deepseek_v4/nvidia/ops/o_proj.py:28-73).  The third, wo_b, is a dense linear and stays with
// the caller.
//   dsv4_inv_rope_quant_kernel  fused_inv_rope_fp8_quant, fp32-scale path (common/ops/fused_inv_rope_fp8_quant.py):
//                               inverse GPT-J RoPE of each head's last 64 dims, then e4m3 with one ue8m0 scale per 128
//                               values of a group's D = heads_per_group * 512 values.
//   dsv4_wo_a_kernel            DeepGEMM fp8_einsum("bhr,hdr->bhd") with recipe (1, 128, 128): the grouped W8A8 block-128
//                               GEMM z[t, g, :] = wo_a[g] . o_fp8[t, g, :].
//
// Intermediate layout (this module's own): o_fp8 e4m3 [G][T][D], o_scale f32 [G][D/128][T] (token-contiguous, as the
// reference's SM90 path stores it).
//
// GEMM shape of the work: G * R x D e4m3 weights (64 heads in 8 groups, R 1024: 33.6 MB) against T <= a few hundred
// tokens, so the weight stream from HBM bounds it.  Swap-AB as in router.cu: 64 weight rows form the MMA M side (tiles of
// every group side by side), a tile of TN tokens the N side.  Both operands come through 2-D tensor maps straight from the
// row-major tensors, one 128-byte k-block (= one scale block) per box.  Each k-block is a fresh tensor-core accumulation,
// promoted into fp32 registers as part * w_scale * x_scale (DESIGN §1).  K is split over CTAs so that about one CTA per SM
// pulls weights; the split count depends on G, R, D and the SM count only, never on T, so a token's z does not depend
// on its batch.  Splits meet in an fp32 workspace, and the last-arriving CTA of a tile adds them in split order
// (self-resetting counters, CUDA-graph replayable).
//
// Roofline: HBM.  Algorithmic bytes = G*R*D + G*(R/128)*(D/128)*4 (weights) + T*G*D*(1 + 4/128) (activations)
// + T*G*R*2 (z).
#include <cuda.h>

#include <mutex>

#include "common.cuh"
#include "moe_internal.cuh"

namespace b200 {

constexpr int OP_HEAD = 512;         // head dim: 448 NoPE | 64 RoPE
constexpr int OP_NOPE = 448;
constexpr int OP_ROT = 64;
constexpr int IR_WARPS = 8;          // inverse RoPE + quant: one warp per (token, head)

constexpr int WA_THREADS = 160;      // warps 0-3 MMA + epilogue warpgroup, warp 4 TMA producer
constexpr int WA_ROWS = 64;          // weight rows per tile (one M = 64 wgmma)
constexpr int WA_A_BYTES = WA_ROWS * 128;
constexpr int WA_PIPE = 96 * 1024;   // pipeline bytes per CTA: two CTAs fit an SM
constexpr int WA_MAX_TOKENS = 1 << 20;
// split-K counters: one per (token tile, weight tile), a fixed area so that one workspace serves every T and shape.
// Splits are only used when the weight tiles are at most half the SMs.
constexpr int WA_CTR_TILES = 128;
constexpr int WA_CTR_TT = WA_MAX_TOKENS / 128;
constexpr int64_t WA_CTR_BYTES = (int64_t)WA_CTR_TILES * WA_CTR_TT * 4;

// ------------------------------------------------------------------------------------------- inverse RoPE + quant
// Lane l holds dims [16l, 16l + 16) of the head: lanes 8b .. 8b + 7 form scale block b, lanes 28-31 the rotary dims.
// The explicit _rn operations keep the compiler from contracting the rotation into FMAs, so the codes are a function of
// the inputs that the oracle restates bit for bit.
__global__ void __launch_bounds__(IR_WARPS * 32)
    dsv4_inv_rope_quant_kernel(const __nv_bfloat16* __restrict__ o, int64_t o_stride,
                               const int64_t* __restrict__ positions, const float* __restrict__ cos_sin,
                               int max_position, uint8_t* __restrict__ o_fp8, float* __restrict__ o_scale, int T, int H,
                               int hpg) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * IR_WARPS + (threadIdx.x >> 5);
  if (w >= (int64_t)T * H) return;   // whole warps only: nothing below synchronises more than the warp
  const int t = (int)(w / H), h = (int)(w % H);
  const int g = h / hpg, hg = h % hpg;
  const uint4* src = reinterpret_cast<const uint4*>(o + t * o_stride + (int64_t)h * OP_HEAD + lane * 16);
  const uint4 raw[2] = {src[0], src[1]};
  const __nv_bfloat16* hx = reinterpret_cast<const __nv_bfloat16*>(raw);
  float x[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) x[i] = __bfloat162float(hx[i]);
  if (lane >= OP_NOPE / 16) {
    int64_t pos = positions[t];
    pos = pos < 0 ? 0 : (pos >= max_position ? max_position - 1 : pos);
    const float* cs = cos_sin + pos * OP_ROT;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int p = (lane - OP_NOPE / 16) * 8 + i;   // pair (448 + 2p, 449 + 2p)
      const float c = cs[p], s = cs[OP_ROT / 2 + p], x0 = x[2 * i], x1 = x[2 * i + 1];
      x[2 * i] = __fadd_rn(__fmul_rn(x0, c), __fmul_rn(x1, s));
      x[2 * i + 1] = __fsub_rn(__fmul_rn(x1, c), __fmul_rn(x0, s));
    }
  }
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) amax = fmaxf(amax, fabsf(x[i]));
#pragma unroll
  for (int m = 1; m < 8; m <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, m));
  // 2^ceil(log2(max(amax, 1e-10) * (1 / 448))) from the exponent bits; dividing by it is exact, as is multiplying by
  // its inverse (2^-119 .. 2^42, all normal)
  const float sc = ue8m0_ceil(__fmul_rn(fmaxf(amax, 1e-10f), 1.0f / 448.0f));
  const float inv = __uint_as_float((254u << 23) - __float_as_uint(sc));
  uint32_t q[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = fminf(fmaxf(__fmul_rn(x[4 * i + j], inv), -448.f), 448.f);
    const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(v[0], v[1]), __NV_SATFINITE, __NV_E4M3);
    const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(v[2], v[3]), __NV_SATFINITE, __NV_E4M3);
    q[i] = (lo & 0xFFFFu) | (hi << 16);
  }
  const int64_t D = (int64_t)hpg * OP_HEAD;
  *reinterpret_cast<uint4*>(o_fp8 + ((int64_t)g * T + t) * D + hg * OP_HEAD + lane * 16) = make_uint4(q[0], q[1], q[2], q[3]);
  if ((lane & 7) == 0) o_scale[((int64_t)g * (D / 128) + hg * (OP_HEAD / 128) + (lane >> 3)) * T + t] = sc;
}

// ------------------------------------------------------------------------------------------------------ wo_a GEMM
struct WoaArgs {
  alignas(64) CUtensorMap tmW;   // wo_a e4m3 [G*R][D], box 128 x 64
  alignas(64) CUtensorMap tmX;   // o_fp8 e4m3 [G*T][D], box 128 x TN
  const float* w_scale;          // [G*R/128][KB]
  const float* x_scale;          // [G][KB][T]
  __nv_bfloat16* z;              // [T][G*R]
  float* partial;                // [KS][T][G*R]
  int32_t* counters;             // [token tiles][weight tiles], zero between launches
  int T, R, GR, KB, KS, tiles;
};

B200_DEVICE void bar_sync_mma() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

template <int TN>
__global__ void __launch_bounds__(WA_THREADS, TN == 128 ? 1 : 2) dsv4_wo_a_kernel(const __grid_constant__ WoaArgs a) {
  constexpr int STAGE = WA_A_BYTES + TN * 128;
  constexpr int STAGES = WA_PIPE / STAGE < 8 ? WA_PIPE / STAGE : 8;
  static_assert(TN * 128 * 4 <= STAGES * STAGE, "the accumulator exchange overlays the pipeline");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ uint64_t full[STAGES], empty[STAGES];
  __shared__ int last_flag;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ks = blockIdx.x, m = blockIdx.y, tt = blockIdx.z;
  const int kb0 = (int)(((long long)ks * a.KB) / a.KS), kb1 = (int)(((long long)(ks + 1) * a.KB) / a.KS);
  const int t0 = tt * TN, nt = min(TN, a.T - t0);
  const int g = (m * WA_ROWS) / a.R;

  if (tid == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (elect_one()) {
      const uint64_t pol_w = policy_evict_first(), pol_x = policy_evict_last();
      for (int kb = kb0, i = 0; kb < kb1; ++kb, ++i) {
        const int s = i % STAGES;
        mbar_wait(&empty[s], ((i / STAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(&full[s], (uint32_t)STAGE);
        uint8_t* sa = smem + s * STAGE;
        tma_load_2d_hint(sa, &a.tmW, kb * 128, m * WA_ROWS, &full[s], pol_w);
        // rows past the group's T tokens belong to the next group (or are zero-filled past the last): their columns are
        // computed and never stored
        tma_load_2d_hint(sa + WA_A_BYTES, &a.tmX, kb * 128, g * a.T + t0, &full[s], pol_x);
      }
    }
  } else {
    // thread holds rows 16 w + l/4 (+8) and token columns 8 j + 2 (l % 4) (+1) of the tile (wgmma.cuh)
    float acc[TN / 2], tot[TN / 2];
#pragma unroll
    for (int j = 0; j < TN / 2; ++j) acc[j] = tot[j] = 0.f;
    const float* wsp = a.w_scale + (size_t)((m * WA_ROWS) >> 7) * a.KB;
    const float* xsp = a.x_scale + (size_t)g * a.KB * a.T + t0;
    const uint32_t sm0 = smem_u32(smem);
    for (int kb = kb0, i = 0; kb < kb1; ++kb, ++i) {
      const int s = i % STAGES;
      const float ws = __ldg(wsp + kb);
      float xs[TN / 4];
#pragma unroll
      for (int j = 0; j < TN / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * j + 2 * (lane & 3) + e;
          xs[2 * j + e] = c < nt ? __ldg(xsp + (size_t)kb * a.T + c) : 0.f;
        }
      mbar_wait(&full[s], (i / STAGES) & 1);
      const uint32_t sa = sm0 + s * STAGE, sb = sa + WA_A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int q = 0; q < 4; ++q)
        WgmmaSS<TN, 2>::mma(acc, wgmma_desc_sw128(sa + q * 32, 1024), wgmma_desc_sw128(sb + q * 32, 1024), q > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      if (tid == 0) mbar_arrive(&empty[s]);
#pragma unroll
      for (int j = 0; j < TN / 8; ++j) {
        tot[4 * j] = fmaf(acc[4 * j] * ws, xs[2 * j], tot[4 * j]);
        tot[4 * j + 1] = fmaf(acc[4 * j + 1] * ws, xs[2 * j + 1], tot[4 * j + 1]);
        tot[4 * j + 2] = fmaf(acc[4 * j + 2] * ws, xs[2 * j], tot[4 * j + 2]);
        tot[4 * j + 3] = fmaf(acc[4 * j + 3] * ws, xs[2 * j + 1], tot[4 * j + 3]);
      }
    }
    // every stage has been consumed: the finished tile crosses to row-per-thread order through the pipeline area
    const uint32_t xch = xch_base(smem);
    xch_store_frag<TN>(xch, 0, tot);
    bar_sync_mma();
    const int row = (warp & 1) * 32 + lane, r = m * WA_ROWS + row;
    const int c_begin = (warp >> 1) * (TN / 2);
#pragma unroll
    for (int c0 = c_begin; c0 < c_begin + TN / 2; c0 += 8) {
      float v[8];
      xch_ld<8>(xch + ((uint32_t)((warp & 1) * 32) << 16) + c0, v);
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        if (c0 + c >= nt) break;
        const size_t tg = (size_t)(t0 + c0 + c);
        if (a.KS == 1)
          a.z[tg * a.GR + r] = __float2bfloat16_rn(v[c]);
        else
          a.partial[((size_t)ks * a.T + tg) * a.GR + r] = v[c];
      }
    }
  }
  if (a.KS == 1) return;
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    int32_t* ctr = a.counters + (size_t)tt * a.tiles + m;
    const int last = atomicAdd(ctr, 1) == a.KS - 1;
    if (last) *ctr = 0;   // hand the counter back clean for the next launch / graph replay
    last_flag = last;
  }
  __syncthreads();
  if (!last_flag) return;
  __threadfence();   // acquire side: every split's partial tile is visible
  // fixed split order 0, 1, .., KS - 1: the sum does not depend on which CTA arrived last
  const size_t split = (size_t)a.T * a.GR;
  for (int it = tid; it < nt * WA_ROWS; it += WA_THREADS) {
    const int t = it / WA_ROWS, row = it % WA_ROWS;
    const float* p = a.partial + (size_t)(t0 + t) * a.GR + m * WA_ROWS + row;
    float s = 0.f;
    for (int k0 = 0; k0 < a.KS; k0 += 8) {   // eight loads in flight, added in split order
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = k0 + u < a.KS ? __ldcg(p + (k0 + u) * split) : 0.f;
#pragma unroll
      for (int u = 0; u < 8; ++u) s += v[u];
    }
    a.z[(size_t)(t0 + t) * a.GR + m * WA_ROWS + row] = __float2bfloat16_rn(s);
  }
}

static int wa_splits(int G, int R, int hpg, int sms) {
  const int tiles = G * R / WA_ROWS, KB = hpg * (OP_HEAD / 128);
  if (tiles > WA_CTR_TILES) return 1;
  int ks = sms / tiles;
  if (ks > KB / 2) ks = KB / 2;   // at least two k-blocks (16 KB of weights) per split
  return ks < 1 ? 1 : ks;
}

static int wa_tn(int T) { return T <= 16 ? 16 : T <= 32 ? 32 : T <= 64 ? 64 : 128; }

static bool wa_shape_ok(int T, int G, int hpg, int R) {
  return T >= 0 && T <= WA_MAX_TOKENS && G >= 1 && hpg >= 1 && hpg <= 16 && R >= 128 && R % 128 == 0 &&
         (int64_t)G * R / WA_ROWS <= 65535 && (int64_t)G * T <= INT32_MAX;
}

static int current_sms() {
  int dev = 0;
  const cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return cuda_fail(e, "cudaGetDevice");
  return device_sms(dev);
}

// cache of weight tensor maps (the checkpoint tensor's pointer is stable for the life of the model)
struct WoaMapKey {
  const void* w;
  int GR, D;
};
static std::mutex g_woa_mu;
static WoaMapKey g_woa_key[64];
static CUtensorMap g_woa_val[64];
static int g_woa_n = 0;

template <int TN>
static int wa_launch(const WoaArgs& a, int TT, cudaStream_t st) {
  const int smem = 1024 + WA_PIPE;
  int rc = kernel_smem(reinterpret_cast<const void*>(dsv4_wo_a_kernel<TN>), smem, "cudaFuncSetAttribute(dsv4_wo_a)");
  if (rc) return rc;
  dsv4_wo_a_kernel<TN><<<dim3(a.KS, a.tiles, TT), WA_THREADS, smem, st>>>(a);
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_dsv4_inv_rope_quant(void* stream, const void* o, int64_t o_token_stride, const int64_t* positions,
                             const float* cos_sin_cache, int max_position, int num_tokens, int num_heads, int n_groups,
                             void* o_fp8, float* o_scale) {
  const int T = num_tokens, H = num_heads, G = n_groups;
  if (!o || !positions || !cos_sin_cache || !o_fp8 || !o_scale || T < 0 || T > WA_MAX_TOKENS || G < 1 || H < G ||
      H % G || H / G > 16 || max_position < 1 || o_token_stride < (int64_t)H * OP_HEAD || o_token_stride % 8) {
    set_error("b200_dsv4_inv_rope_quant: bad argument (0 <= num_tokens <= 2^20, num_heads = n_groups * (1-16), "
              "o_token_stride >= num_heads * 512 and a multiple of 8, max_position >= 1)");
    return B200_ERR_INVALID;
  }
  if (reinterpret_cast<uintptr_t>(o) % 16 || reinterpret_cast<uintptr_t>(o_fp8) % 16 ||
      reinterpret_cast<uintptr_t>(positions) % 8 || reinterpret_cast<uintptr_t>(cos_sin_cache) % 4 ||
      reinterpret_cast<uintptr_t>(o_scale) % 4) {
    set_error("b200_dsv4_inv_rope_quant: o and o_fp8 must be 16-byte aligned, positions 8, cos_sin_cache and o_scale 4");
    return B200_ERR_INVALID;
  }
  if (T == 0) return 0;
  const int64_t warps = (int64_t)T * H;
  dsv4_inv_rope_quant_kernel<<<(unsigned)((warps + IR_WARPS - 1) / IR_WARPS), IR_WARPS * 32, 0,
                               reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(o), o_token_stride, positions, cos_sin_cache, max_position,
      reinterpret_cast<uint8_t*>(o_fp8), o_scale, T, H, H / G);
  ++g_launches;
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "dsv4_inv_rope_quant launch");
  return 0;
}

int64_t b200_dsv4_wo_a_workspace_bytes(int num_tokens, int n_groups, int heads_per_group, int o_lora_rank) {
  if (!wa_shape_ok(num_tokens, n_groups, heads_per_group, o_lora_rank) || num_tokens == 0) return 0;
  const int sms = current_sms();
  if (sms <= 0) return 0;
  const int KS = wa_splits(n_groups, o_lora_rank, heads_per_group, sms);
  if (KS == 1) return 0;
  return WA_CTR_BYTES + (int64_t)KS * num_tokens * n_groups * o_lora_rank * 4;
}

int b200_dsv4_wo_a(void* stream, const void* o_fp8, const float* o_scale, const void* wo_a, const float* wo_a_scale,
                   int num_tokens, int n_groups, int heads_per_group, int o_lora_rank, void* workspace,
                   int64_t workspace_bytes, void* z) {
  const int T = num_tokens, G = n_groups, R = o_lora_rank, hpg = heads_per_group;
  if (!o_fp8 || !o_scale || !wo_a || !wo_a_scale || !z || !wa_shape_ok(T, G, hpg, R)) {
    set_error("b200_dsv4_wo_a: bad argument (0 <= num_tokens <= 2^20, n_groups >= 1, heads_per_group 1-16, "
              "o_lora_rank a multiple of 128, n_groups * o_lora_rank / 64 <= 65535)");
    return B200_ERR_INVALID;
  }
  if (reinterpret_cast<uintptr_t>(o_fp8) % 16 || reinterpret_cast<uintptr_t>(wo_a) % 16 ||
      reinterpret_cast<uintptr_t>(o_scale) % 4 || reinterpret_cast<uintptr_t>(wo_a_scale) % 4 ||
      reinterpret_cast<uintptr_t>(z) % 2) {
    set_error("b200_dsv4_wo_a: o_fp8 and wo_a must be 16-byte aligned, the scales 4, z 2");
    return B200_ERR_INVALID;
  }
  if (T == 0) return 0;
  const int sms = current_sms();
  if (sms < 0) return sms;
  const int D = hpg * OP_HEAD, GR = G * R, KS = wa_splits(G, R, hpg, sms);
  if (KS > 1 && (!workspace || reinterpret_cast<uintptr_t>(workspace) % 16 ||
                 workspace_bytes < b200_dsv4_wo_a_workspace_bytes(T, G, hpg, R))) {
    set_error("b200_dsv4_wo_a: workspace missing, misaligned or too small (b200_dsv4_wo_a_workspace_bytes)");
    return B200_ERR_INVALID;
  }
  const int TN = wa_tn(T), TT = (T + TN - 1) / TN;
  WoaArgs a{};
  {
    std::lock_guard<std::mutex> lk(g_woa_mu);
    int hit = -1;
    for (int i = 0; i < g_woa_n; ++i)
      if (g_woa_key[i].w == wo_a && g_woa_key[i].GR == GR && g_woa_key[i].D == D) hit = i;
    if (hit < 0) {
      CUtensorMap tm;
      const int rc = tm_encode_2d(&tm, (int)CU_TENSOR_MAP_DATA_TYPE_UINT8, wo_a, (uint64_t)D, (uint64_t)GR, (uint64_t)D,
                                  128, WA_ROWS);
      if (rc) return rc;
      hit = g_woa_n < 64 ? g_woa_n++ : 0;
      g_woa_key[hit] = WoaMapKey{wo_a, GR, D};
      g_woa_val[hit] = tm;
    }
    a.tmW = g_woa_val[hit];
  }
  int rc = tm_encode_2d(&a.tmX, (int)CU_TENSOR_MAP_DATA_TYPE_UINT8, o_fp8, (uint64_t)D, (uint64_t)G * T, (uint64_t)D, 128,
                        (uint32_t)TN);
  if (rc) return rc;
  a.w_scale = wo_a_scale;
  a.x_scale = o_scale;
  a.z = reinterpret_cast<__nv_bfloat16*>(z);
  a.counters = KS > 1 ? reinterpret_cast<int32_t*>(workspace) : nullptr;
  a.partial = KS > 1 ? reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + WA_CTR_BYTES) : nullptr;
  a.T = T;
  a.R = R;
  a.GR = GR;
  a.KB = D / 128;
  a.KS = KS;
  a.tiles = GR / WA_ROWS;
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  rc = TN == 16 ? wa_launch<16>(a, TT, st) : TN == 32 ? wa_launch<32>(a, TT, st) : TN == 64 ? wa_launch<64>(a, TT, st)
                                                                                              : wa_launch<128>(a, TT, st);
  if (rc) return rc;
  ++g_launches;
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "dsv4_wo_a launch");
  return 0;
}

}  // extern "C"
