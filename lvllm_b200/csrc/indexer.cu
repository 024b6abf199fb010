// The DeepSeek-V3.2 / GLM-5 lightning indexer for decode: what picks the top-k keys that sparse MLA decode
// (b200_mla_decode_sparse) attends over.  Three kernels:
//   indexer_qk_rope_quant_cache_kernel  q side: RoPE + per-(token, head) ue8m0 e4m3 quantisation + the folded head weights
//                                       (the reference's _fused_indexer_q_rope_quant_kernel, sparse_attn_indexer.py:127-251);
//                                       k side: RoPE (RotaryEmbedding.forward_static) + indexer_k_quant_and_cache
//                                       (csrc/libtorch_stable/cache_kernels.cu:599-659), one launch for both.
//   indexer_logits_kernel               logit[r, j] = k_scale[j] * sum_h w[r, h] * relu(q8[r, h] . k8[j]) over the paged fp8
//                                       cache (DeepGEMM fp8_fp4_paged_mqa_logits; fp8_paged_mqa_logits_torch,
//                                       rocm_aiter_mla_sparse.py:264-363).  wgmma e4m3: a 64-key tile of the cache is the
//                                       M = 64 A operand, the q tile of a q-group (Qg tokens x H heads) the N operand.
//   indexer_topk_kernel                 per-row radix select (top_k_per_row_decode, sampler.cu:567-614, 661-720): indices of
//                                       the topk largest logits of [0, row_end), ascending, ties at the threshold to the
//                                       lowest positions, -1 padding.
// Cache layout (indexer_k_quant_and_cache): uint8 [num_blocks, block_size, 132]: a block holds block_size x 128 e4m3 bytes,
// then block_size fp32 scales (quant_block_size = head_dim = 128: one scale per row).
// DeepSeek-V4's C4A indexer reuses the logits and top-k kernels with per-token rows (ROWS): row t is one decode token with
// (positions[t] + 1) / ratio candidate keys in row token_to_req[t] of the compressed cache's block table; its q side is
// dsv4_indexer_q_quant_kernel (the reference's _fused_indexer_q_rope_quant_kernel, fused_indexer_q.py:70-176, fp8 path).
#include <cooperative_groups.h>
#include <cuda.h>

#include <algorithm>
#include <mutex>

#include "common.cuh"
#include "kv_pack.cuh"
#include "moe_internal.cuh"

namespace cg = cooperative_groups;

namespace b200 {

constexpr int IDX_AUX_WARPS = 4;
constexpr int IDX_DIM = 128;    // index_head_dim
constexpr int IDX_ROT = 64;     // rotary dims, [pe | nope]
constexpr int IDX_ROW = 132;    // cache bytes per token: 128 e4m3 + one fp32 scale

B200_DEVICE float bf16r(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

B200_DEVICE uint32_t e4m3x4(float a, float b, float c, float d) {
  const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
  const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
  return (lo & 0xFFFFu) | (hi << 16);
}

// grid = ceil(T * (H + 1) / 4) warps of 32: warp w < T * H is q head (w / H, w % H), warp T * H + t is token t's k row.
// Lane l owns dims [4l, 4l + 4); lanes 0-15 hold the rotary dims.
__global__ void __launch_bounds__(IDX_AUX_WARPS * 32)
    indexer_qk_rope_quant_cache_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ weights,
                                       int64_t w_stride, const __nv_bfloat16* __restrict__ k,
                                       const int64_t* __restrict__ positions, const __nv_bfloat16* __restrict__ cos_sin,
                                       int max_position, int is_neox, const int64_t* __restrict__ slot_mapping,
                                       uint8_t* __restrict__ k_cache, int block_size, int k_ue8m0, float softmax_scale,
                                       float head_scale, uint8_t* __restrict__ q_fp8, float* __restrict__ weights_out,
                                       int T, int H) {
  __shared__ float xs[IDX_AUX_WARPS][IDX_DIM];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int w = blockIdx.x * IDX_AUX_WARPS + warp;
  if (w >= T * (H + 1)) return;   // whole warps only: nothing below synchronises more than the warp
  const bool is_k = w >= T * H;
  const int t = is_k ? w - T * H : w / H, h = is_k ? 0 : w % H;
  const int64_t slot = is_k ? slot_mapping[t] : 0;
  if (slot < 0) return;   // padded token: nothing written
  const __nv_bfloat16* src = is_k ? k + (size_t)t * IDX_DIM : q + ((size_t)t * H + h) * IDX_DIM;
  const uint2 raw = *reinterpret_cast<const uint2*>(src + lane * 4);
  const __nv_bfloat16* hx = reinterpret_cast<const __nv_bfloat16*>(&raw);
  float x[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) x[i] = __bfloat162float(hx[i]);
#pragma unroll
  for (int i = 0; i < 4; ++i) xs[warp][lane * 4 + i] = x[i];
  __syncwarp();
  int64_t pos = positions[t];
  pos = pos < 0 ? 0 : (pos >= max_position ? max_position - 1 : pos);
  const __nv_bfloat16* cs = cos_sin + pos * IDX_ROT;
  // pair p = (x1, x2): NeoX (p, p + 32), interleaved (2p, 2p + 1); o1 = x1 c - x2 s, o2 = x2 c + x1 s.
  // q: fp32 products, their sum, then one rounding to bf16; k: bf16 after every op (forward_static).  The explicit _rn
  // operations keep the compiler from contracting them into FMAs, so the bytes are the oracle's.  The reference's Triton
  // kernel writes the same expression but compiles with fp fusion on, so it may contract it into an FMA, which can move
  // a rotated value's bf16 rounding by one ulp in rare cases; the unfused form is the stated one here.
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int e = lane * 4 + i;
    if (e < IDX_ROT) {
      const bool second = is_neox ? e >= IDX_ROT / 2 : (e & 1);
      const int p = is_neox ? (second ? e - IDX_ROT / 2 : e) : e >> 1;
      const int partner = is_neox ? (second ? e - IDX_ROT / 2 : e + IDX_ROT / 2) : (e ^ 1);
      const float c = __bfloat162float(cs[p]), s = __bfloat162float(cs[IDX_ROT / 2 + p]);
      const float y = xs[warp][partner];
      if (is_k) {
        const float a = bf16r(__fmul_rn(x[i], c)), b = bf16r(__fmul_rn(y, s));
        x[i] = bf16r(second ? __fadd_rn(a, b) : __fsub_rn(a, b));
      } else {
        const float a = __fmul_rn(x[i], c), b = __fmul_rn(y, s);
        x[i] = bf16r(second ? __fadd_rn(a, b) : __fsub_rn(a, b));
      }
    }
  }
  if (is_k) {   // the values are bf16 already, so the packer's rounding leaves them as they are
    indexer_pack_row132(x, k_ue8m0 != 0, k_cache + (slot / block_size) * (int64_t)block_size * IDX_ROW, block_size,
                        (int)(slot % block_size), lane);
    return;
  }
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) amax = fmaxf(amax, fabsf(x[i]));
  amax = warp_max(amax);
  // q_scale = exp2(ceil(log2(max(amax, 1e-10) * (1 / 448)))), always ue8m0; x / q_scale is exact
  const float sc = ue8m0_ceil(__fmul_rn(fmaxf(amax, 1e-10f), 1.0f / 448.0f));
  const uint32_t v = e4m3x4(__fdiv_rn(x[0], sc), __fdiv_rn(x[1], sc), __fdiv_rn(x[2], sc), __fdiv_rn(x[3], sc));
  *reinterpret_cast<uint32_t*>(q_fp8 + ((size_t)t * H + h) * IDX_DIM + lane * 4) = v;
  if (lane == 0) {
    const float wt = __bfloat162float(weights[(size_t)t * w_stride + h]);
    weights_out[(size_t)t * H + h] = __fmul_rn(__fmul_rn(__fmul_rn(wt, sc), softmax_scale), head_scale);
  }
}

// The V4 q side, a kernel of its own: V4 rotates the last 64 dims GPT-J style (both dims of a pair sit in one lane, so
// nothing goes through shared memory), reads an f32 cos | sin table, takes scale = 2^ceil(log2(max(amax, 1e-4) / 448)) and
// writes no k row; as branches of indexer_qk_rope_quant_cache_kernel those differences would reach every part of it.
// grid = ceil(T * H / 4) warps of 32, warp w is head (w / H, w % H); lane l owns dims [4l, 4l + 4), lanes 16-31 the rotary
// dims.  The rotation is fp32 products, their sum, then one rounding to bf16; as in the V3.2 kernel the explicit _rn
// operations keep the compiler from contracting them into FMAs, which the reference's Triton kernel may do.
__global__ void __launch_bounds__(IDX_AUX_WARPS * 32)
    dsv4_indexer_q_quant_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ weights,
                                int64_t w_stride, const int64_t* __restrict__ positions, const float* __restrict__ cos_sin,
                                int max_position, float softmax_scale, float head_scale, uint8_t* __restrict__ q_fp8,
                                float* __restrict__ weights_out, int T, int H) {
  const int lane = threadIdx.x & 31;
  const int w = blockIdx.x * IDX_AUX_WARPS + (threadIdx.x >> 5);
  if (w >= T * H) return;   // whole warps only
  const int t = w / H, h = w % H;
  const uint2 raw = *reinterpret_cast<const uint2*>(q + (size_t)w * IDX_DIM + lane * 4);
  const __nv_bfloat16* hx = reinterpret_cast<const __nv_bfloat16*>(&raw);
  float x[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) x[i] = __bfloat162float(hx[i]);
  if (lane >= 16) {
    int64_t pos = positions[t];
    pos = pos < 0 ? 0 : (pos >= max_position ? max_position - 1 : pos);
    const float* cs = cos_sin + pos * IDX_ROT;
#pragma unroll
    for (int i = 0; i < 4; i += 2) {
      const int p = (lane - 16) * 2 + i / 2;   // pair (64 + 2p, 64 + 2p + 1)
      const float c = cs[p], s = cs[IDX_ROT / 2 + p], x0 = x[i], x1 = x[i + 1];
      x[i] = bf16r(__fsub_rn(__fmul_rn(x0, c), __fmul_rn(x1, s)));
      x[i + 1] = bf16r(__fadd_rn(__fmul_rn(x1, c), __fmul_rn(x0, s)));
    }
  }
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) amax = fmaxf(amax, fabsf(x[i]));
  amax = warp_max(amax);
  // amax is a bf16 value, so max(amax, 1e-4) / 448 is a power of two or far from one: the exponent ceiling is
  // exp2(ceil(log2(.))) exactly
  const float sc = ue8m0_ceil(__fdiv_rn(fmaxf(amax, 1e-4f), 448.0f));
  const uint32_t v = e4m3x4(__fdiv_rn(x[0], sc), __fdiv_rn(x[1], sc), __fdiv_rn(x[2], sc), __fdiv_rn(x[3], sc));
  *reinterpret_cast<uint32_t*>(q_fp8 + (size_t)w * IDX_DIM + lane * 4) = v;
  if (lane == 0) {
    const float wt = __bfloat162float(weights[(size_t)t * w_stride + h]);
    weights_out[w] = __fmul_rn(__fmul_rn(__fmul_rn(wt, sc), softmax_scale), head_scale);
  }
}

// candidate keys of a V4 decode token at position p: the compressed rows its window closes
B200_DEVICE int64_t v4_keys(int64_t p, int ratio) { return p < 0 ? 0 : (p + 1) / ratio; }

// ----------------------------------------------------------------------------------------------------------- logits
constexpr int LG_STAGES = 6;
constexpr int LG_THREADS = 160;          // warps 0-3: MMA + epilogue warpgroup, warp 4: TMA producer
constexpr int LG_TILE = 64 * IDX_DIM;    // one 64-key tile of e4m3 rows, 128B-swizzled
constexpr int LG_SCALES = 64 * 4;

struct LogitsArgs {
  alignas(64) CUtensorMap tmK;   // the cache's e4m3 rows as [block][slot][128 B], box 128 x page x 1
  const uint8_t* k_cache;
  const uint8_t* q_fp8;          // [B * Q, H, 128]
  const float* weights;          // [B * Q, H]
  const int32_t* seq_lens;       // [B]
  const int32_t* page_table;     // [B, max_pages]
  float* logits;                 // [B * Q, stride]
  int64_t stride;
  int B, Q, H, page, max_pages, qg, n_qg;
  // ROWS (V4, Q = 1, B = tokens): row b has v4_keys(positions[b], ratio) keys in page_table row row_req[b]
  const int64_t* positions;
  const int32_t* row_req;
  int ratio;
};

B200_DEVICE void tma_load_3d(void* smem_dst, const void* tmap, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(smem_u32(smem_dst)),
      "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
      : "memory");
}

template <bool ROWS>
B200_DEVICE int lg_keys(const LogitsArgs& a, int b) {
  if constexpr (ROWS) return (int)min(v4_keys(a.positions[b], a.ratio), (int64_t)a.max_pages * a.page);
  const int S = a.seq_lens[b];
  return S < 0 ? 0 : min(S, a.max_pages * a.page);
}

// work item -> (request, q-group, run of `run` 64-key tiles); the q-groups of one run are neighbours so that they meet
// the run's cache rows in L2.  Returns the tile range [t0, t1) (empty past the request's keys) and the request's key count.
struct LgItem {
  int b, g0, qn, t0, t1, S;
};
template <bool ROWS>
B200_DEVICE LgItem lg_item(const LogitsArgs& a, int item, int run_len) {
  LgItem w;
  const int qgi = item % a.n_qg, rb = item / a.n_qg;
  w.b = rb % a.B;
  const int run = rb / a.B;
  w.g0 = qgi * a.qg;
  w.qn = min(a.qg, a.Q - w.g0);
  w.S = lg_keys<ROWS>(a, w.b);
  w.t0 = run * run_len;
  w.t1 = min(w.t0 + run_len, (w.S + 63) / 64);
  return w;
}

template <int N, int H, bool ROWS>
__global__ void __launch_bounds__(LG_THREADS) indexer_logits_kernel(const __grid_constant__ LogitsArgs a) {
  constexpr int NT = N / H;   // token slots of the q tile (the last ones zero when the q-group is shorter)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* qt = smem;                                   // [N rows x 128 B] swizzled
  uint8_t* kt = smem + N * IDX_DIM;                     // [LG_STAGES][64 rows x 128 B] swizzled
  float* ks = reinterpret_cast<float*>(kt + LG_STAGES * LG_TILE);   // [LG_STAGES][64] fp32 scales
  __shared__ uint64_t full[LG_STAGES], empty[LG_STAGES];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int i = 0; i < LG_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 4);
    }
    fence_barrier_init();
  }
  // the schedule, from the contexts themselves (every CTA derives the same one): runs of at least 4 tiles (the q tile load
  // is amortised), short enough for about 4 items per CTA; every request has as many runs as the longest one needs
  __shared__ long long s_red[LG_THREADS / 32][2];
  __shared__ int s_run, s_items;
  {
    long long sum = 0, mx = 0;
    for (int b = tid; b < a.B; b += LG_THREADS) {
      const long long t = (lg_keys<ROWS>(a, b) + 63) / 64;
      sum += t;
      mx = max(mx, t);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      sum += __shfl_xor_sync(0xffffffffu, sum, off);
      mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    }
    if (lane == 0) {
      s_red[warp][0] = sum;
      s_red[warp][1] = mx;
    }
    __syncthreads();
    if (tid == 0) {
      sum = mx = 0;
      for (int w = 0; w < LG_THREADS / 32; ++w) {
        sum += s_red[w][0];
        mx = max(mx, s_red[w][1]);
      }
      const long long per = 4ll * gridDim.x;
      const long long run = max(4ll, (sum * a.n_qg + per - 1) / per);
      s_run = (int)run;
      s_items = (int)((mx + run - 1) / run * a.B * a.n_qg);   // <= the host's bound for run = 4, which fits an int
    }
  }
  __syncthreads();
  const int run_len = s_run, n_items = s_items;
  const int ppt = 64 / a.page;   // pages per tile

  if (warp == 4) {
    if (!elect_one()) return;
    int it = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const LgItem w = lg_item<ROWS>(a, item, run_len);
      const int npages = (w.S + a.page - 1) / a.page;
      const int32_t* pt = a.page_table + (size_t)(ROWS ? a.row_req[w.b] : w.b) * a.max_pages;
      for (int t = w.t0; t < w.t1; ++t, ++it) {
        const int s = it % LG_STAGES;
        mbar_wait(&empty[s], ((it / LG_STAGES) & 1) ^ 1);
        const int p0 = t * ppt, np = min(ppt, npages - p0);
        mbar_arrive_expect_tx(&full[s], (uint32_t)(np * a.page * IDX_ROW));
        for (int i = 0; i < np; ++i) {
          const int blk = pt[p0 + i];
          tma_load_3d(kt + s * LG_TILE + i * a.page * IDX_DIM, &a.tmK, 0, 0, blk, &full[s]);
          bulk_g2s(reinterpret_cast<uint8_t*>(ks + s * 64 + i * a.page),
                   a.k_cache + (int64_t)blk * a.page * IDX_ROW + a.page * IDX_DIM, a.page * 4, &full[s]);
        }
      }
    }
    return;
  }

  // ---- MMA + epilogue warpgroup: thread (warp w, lane l) holds keys 16w + l/4 and +8 of the tile, columns
  // 8j + 2(l%4) and +1 of the q tile (column = token slot * H + head)
  const uint32_t qa = smem_u32(qt), ka = smem_u32(kt);
  int it = 0;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const LgItem w = lg_item<ROWS>(a, item, run_len);
    if (w.t0 >= w.t1) continue;
    const int row0 = w.b * a.Q + w.g0;   // first logits row of the q-group
    // the previous item's MMAs have retired (wait_group 0 after each tile); every thread is past its reads of the q tile
    asm volatile("bar.sync 1, 128;" ::: "memory");
    for (int c = tid; c < N * 8; c += 128) {
      const int r = c >> 3, ch = c & 7, g = r / H;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (g < w.qn) v = *reinterpret_cast<const uint4*>(a.q_fp8 + ((size_t)(row0 + g) * H + r % H) * IDX_DIM + ch * 16);
      *reinterpret_cast<uint4*>(qt + sw128_offset(r, ch * 16)) = v;
    }
    float wv[N / 4];
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = j * 8 + (lane & 3) * 2 + e, g = col / H;
        wv[2 * j + e] = g < w.qn ? a.weights[(size_t)(row0 + g) * H + col % H] : 0.f;
      }
    fence_proxy_async();   // the generic-proxy q tile stores become visible to wgmma
    asm volatile("bar.sync 1, 128;" ::: "memory");
    const int npages = (w.S + a.page - 1) / a.page;
    const int limit = npages * a.page;   // keys of the request's pages; nothing past them is written
    for (int t = w.t0; t < w.t1; ++t, ++it) {
      const int s = it % LG_STAGES;
      mbar_wait(&full[s], (it / LG_STAGES) & 1);
      float acc[N / 2];
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        WgmmaSS<N, 2>::mma(acc, wgmma_desc_sw128(ka + s * LG_TILE + kk * 32, 1024), wgmma_desc_sw128(qa + kk * 32, 1024),
                           kk > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      const int r_lo = warp * 16 + (lane >> 2);
      const float sc_lo = ks[s * 64 + r_lo], sc_hi = ks[s * 64 + r_lo + 8];
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
      float lo[NT], hi[NT];
#pragma unroll
      for (int g = 0; g < NT; ++g) lo[g] = hi[g] = 0.f;
#pragma unroll
      for (int j = 0; j < N / 8; ++j) {
        const int g = (j * 8) / H;
        lo[g] += wv[2 * j] * fmaxf(acc[4 * j], 0.f) + wv[2 * j + 1] * fmaxf(acc[4 * j + 1], 0.f);
        hi[g] += wv[2 * j] * fmaxf(acc[4 * j + 2], 0.f) + wv[2 * j + 1] * fmaxf(acc[4 * j + 3], 0.f);
      }
      const int key = t * 64 + r_lo;
#pragma unroll
      for (int g = 0; g < NT; ++g) {
        lo[g] += __shfl_xor_sync(0xffffffffu, lo[g], 1);
        lo[g] += __shfl_xor_sync(0xffffffffu, lo[g], 2);
        hi[g] += __shfl_xor_sync(0xffffffffu, hi[g], 1);
        hi[g] += __shfl_xor_sync(0xffffffffu, hi[g], 2);
        if (g < w.qn && (lane & 3) == (g & 3)) {
          const int row_end = w.S - a.Q + w.g0 + g + 1;   // keys [0, S - Q + i] of draft token i
          float* out = a.logits + (size_t)(row0 + g) * a.stride;
          if (key < limit) out[key] = key < row_end ? lo[g] * sc_lo : -INFINITY;
          if (key + 8 < limit) out[key + 8] = key + 8 < row_end ? hi[g] * sc_hi : -INFINITY;
        }
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------------------- top-k
constexpr int TK_THREADS = 512;
constexpr int TK_BINS = 2048;
constexpr int TK_ITEMS = 4;   // consecutive logits per thread per chunk of the ordered compaction

// order-preserving image of a float: a > b  <=>  key(a) > key(b) (unsigned); -0 is mapped to +0, which it equals
B200_DEVICE uint32_t tk_key(float f) {
  const uint32_t b = __float_as_uint(f) == 0x80000000u ? 0u : __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// exclusive scan over the CTA (thread order) of a (gt << 32 | eq) pair; returns the prefix, *total the CTA's sum
B200_DEVICE unsigned long long tk_scan(unsigned long long v, unsigned long long* sh, unsigned long long* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) sh[warp] = x;
  __syncthreads();
  if (warp == 0) {
    unsigned long long s = lane < TK_THREADS / 32 ? sh[lane] : 0ull;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < TK_THREADS / 32) sh[32 + lane] = s;   // inclusive warp-total prefix
  }
  __syncthreads();
  const unsigned long long base = warp ? sh[32 + warp - 1] : 0ull;
  *total = sh[32 + TK_THREADS / 32 - 1];
  __syncthreads();   // sh is reused by the next call
  return base + x - v;
}

// One row per cluster of CS CTAs (CS = 1: one CTA per row).  The CTAs split the row into contiguous segments; radix
// histograms of 11 / 11 / 10 bits are summed over the cluster through distributed shared memory (in rank order: every
// CTA derives the same threshold).  Each CTA's own histograms also give its segment's counts of keys above and equal to
// the threshold, and one ordered compaction writes the selected positions in ascending order, each CTA at the offset the
// lower ranks' counts give it.  Row r starts at r * stride; positions past `width` are never read.
// ROWS (V4, Q = 1): row r has v4_keys(positions[r], ratio) positions; seq_lens is not read.
template <bool ROWS>
__global__ void __launch_bounds__(TK_THREADS)
    indexer_topk_kernel(const float* __restrict__ logits, int64_t stride, int64_t width,
                        const int32_t* __restrict__ seq_lens, int Q, int topk, int32_t* __restrict__ out,
                        const int64_t* __restrict__ positions, int ratio) {
  __shared__ int hist[TK_BINS];
  __shared__ int ghist[TK_BINS];
  __shared__ unsigned long long scan_sh[64];
  __shared__ unsigned long long seg_cnt;   // this CTA's (gt << 32 | eq), read by the higher ranks
  __shared__ uint32_t s_prefix;
  __shared__ int s_krem;
  __shared__ int s_gt, s_eq;   // this CTA's segment: keys above / equal to the threshold
  cg::cluster_group cluster = cg::this_cluster();
  const int CS = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int row = blockIdx.x / CS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = row / Q, i = row % Q;
  const int64_t n = min(ROWS ? v4_keys(positions[row], ratio) : (int64_t)max(0, seq_lens[b] - Q + i + 1), width);
  int32_t* o = out + (size_t)row * topk;
  if (n <= topk) {   // every position, in order, then -1
    if (rank == 0)
      for (int j = tid; j < topk; j += TK_THREADS) o[j] = j < n ? j : -1;
    return;
  }
  const float* x = logits + (size_t)row * stride;
  const int64_t seg = (n + CS - 1) / CS;
  const int64_t s0 = min(n, seg * rank), s1 = min(n, s0 + seg);

  if (tid == 0) {
    s_prefix = 0u;
    s_krem = topk;
    s_gt = 0;
  }
  for (int pass = 0; pass < 3; ++pass) {
    const int shift = pass == 0 ? 21 : pass == 1 ? 10 : 0;
    const int bins = pass == 2 ? 1024 : 2048;
    const uint32_t hi_mask = pass == 0 ? 0u : (0xFFFFFFFFu << (shift + (pass == 2 ? 10 : 11)));
    for (int j = tid; j < TK_BINS; j += TK_THREADS) hist[j] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix;
    for (int64_t j = s0 + tid; j < s1; j += TK_THREADS) {
      const uint32_t kx = tk_key(x[j]);
      if (((kx ^ prefix) & hi_mask) == 0u) atomicAdd(&hist[(kx >> shift) & (bins - 1)], 1);
    }
    cluster.sync();
    for (int j = tid; j < bins; j += TK_THREADS) {
      int c = 0;
      for (int r = 0; r < CS; ++r) c += cluster.map_shared_rank(hist, r)[j];
      ghist[j] = c;
    }
    cluster.sync();   // no CTA zeroes its histogram for the next pass before every CTA has read it
    // the bin d holding the k_rem-th largest remaining key: count(> d) < k_rem <= count(>= d); one warp, bins from the top
    if (warp == 0) {
      const int per = bins / 32;
      const int top = bins - 1 - lane * per;   // lane covers bins (top - per, top]
      int c = 0;
      for (int j = 0; j < per; ++j) c += ghist[top - j];
      int incl = c;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += y;
      }
      const int krem = s_krem;
      const int before = incl - c;
      const unsigned hit = __ballot_sync(0xffffffffu, before < krem && incl >= krem);
      if (lane == __ffs(hit) - 1) {
        int acc = before, d = top;
        for (;; --d) {
          if (acc + ghist[d] >= krem) break;
          acc += ghist[d];
        }
        s_prefix = prefix | ((uint32_t)d << shift);
        s_krem = krem - acc;
      }
    }
    __syncthreads();
    // keys of this segment in the local bins above the chosen digit are above the threshold (they match the prefix of
    // the earlier digits); after the last digit the chosen bin holds the keys equal to it
    const uint32_t d = (s_prefix >> shift) & (uint32_t)(bins - 1);
    int c = 0;
    for (int j = (int)d + 1 + tid; j < bins; j += TK_THREADS) c += hist[j];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) c += __shfl_xor_sync(0xffffffffu, c, off);
    if (lane == 0 && c) atomicAdd(&s_gt, c);
    if (pass == 2 && tid == 0) s_eq = hist[d];
    __syncthreads();   // the local histogram is read before the next pass zeroes it
  }
  const uint32_t thr = s_prefix;
  const int need = s_krem;   // keys equal to the threshold to take, lowest positions first

  // ordered compaction.  Selected before position p: gt(<p) + min(eq(<p), need).
  if (tid == 0) seg_cnt = ((unsigned long long)s_gt << 32) | (unsigned)s_eq;
  cluster.sync();
  unsigned long long run = 0ull;   // (gt << 32 | eq) before the current chunk: the lower ranks' segments first
  for (int r = 0; r < rank; ++r) run += *cluster.map_shared_rank(&seg_cnt, r);
  for (int64_t c0 = s0; c0 < s1; c0 += TK_THREADS * TK_ITEMS) {
    const int64_t p = c0 + (int64_t)tid * TK_ITEMS;
    uint32_t kx[TK_ITEMS];
    unsigned long long v = 0ull;
#pragma unroll
    for (int u = 0; u < TK_ITEMS; ++u) {
      kx[u] = p + u < s1 ? tk_key(x[p + u]) : 0u;
      if (p + u < s1) v += kx[u] > thr ? (1ull << 32) : (kx[u] == thr ? 1ull : 0ull);
    }
    unsigned long long tot;
    const unsigned long long pre = run + tk_scan(v, scan_sh, &tot);
    int gt = (int)(pre >> 32), eq = (int)(pre & 0xFFFFFFFFull);
#pragma unroll
    for (int u = 0; u < TK_ITEMS; ++u) {
      if (p + u >= s1) continue;
      if (kx[u] > thr) {
        o[gt + min(eq, need)] = (int32_t)(p + u);
        ++gt;
      } else if (kx[u] == thr) {
        if (eq < need) o[gt + eq] = (int32_t)(p + u);
        ++eq;
      }
    }
    run += tot;
  }
  cluster.sync();   // the higher ranks have read seg_cnt before this CTA's shared memory goes away
}

// 3-D tiled tensor map over the cache's e4m3 rows, SWIZZLE_128B (cuTensorMapEncodeTiled from the driver at run time)
typedef CUresult (*TmEncodeFn3)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static int tm_encode_cache(CUtensorMap* tm, const void* k_cache, int num_blocks, int page) {
  static std::mutex mu;
  static TmEncodeFn3 fn = nullptr;
  {
    std::lock_guard<std::mutex> lk(mu);
    if (!fn) {
      void* p = nullptr;
      cudaDriverEntryPointQueryResult q;
      cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
      if (e != cudaSuccess || !p || q != cudaDriverEntryPointSuccess) {
        set_error("cuTensorMapEncodeTiled is not available from this driver");
        return B200_ERR_CUDA;
      }
      fn = reinterpret_cast<TmEncodeFn3>(p);
    }
  }
  const cuuint64_t gdim[3] = {(cuuint64_t)IDX_DIM, (cuuint64_t)page, (cuuint64_t)num_blocks};
  const cuuint64_t gstr[2] = {(cuuint64_t)IDX_DIM, (cuuint64_t)page * IDX_ROW};
  const cuuint32_t box[3] = {(cuuint32_t)IDX_DIM, (cuuint32_t)page, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(k_cache), gdim, gstr, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
    return B200_ERR_CUDA;
  }
  return 0;
}

static bool misaligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 != 0; }

template <int N, int H, bool ROWS>
static int run_logits(const LogitsArgs& a, int grid, cudaStream_t st) {
  const int smem = 1024 + N * IDX_DIM + LG_STAGES * (LG_TILE + LG_SCALES);
  const int rc = kernel_smem(reinterpret_cast<const void*>(indexer_logits_kernel<N, H, ROWS>), smem,
                             "cudaFuncSetAttribute(indexer_logits)");
  if (rc) return rc;
  indexer_logits_kernel<N, H, ROWS><<<grid, LG_THREADS, smem, st>>>(a);
  return 0;
}

// Encodes the cache's tensor map, sizes the q-groups and launches indexer_logits_kernel; the caller has checked and
// filled every other field of a (ROWS: Q = 1, so one token per q tile and N = 64).
template <bool ROWS>
static int launch_logits(LogitsArgs& a, int num_blocks, cudaStream_t st, const char* who) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return cuda_fail(e, "cudaGetDevice");
  const int sms = device_sms(dev);
  if (sms < 0) return sms;
  int rc = tm_encode_cache(&a.tmK, a.k_cache, num_blocks, a.page);
  if (rc) return rc;
  a.qg = std::min(a.Q, 128 / a.H);
  a.n_qg = (a.Q + a.qg - 1) / a.qg;
  // the kernel sizes its runs of tiles from the rows' key counts; the most items it can make are those of 4-tile runs
  // over the page table's width
  const int64_t tiles = ((int64_t)a.max_pages * a.page + 63) / 64;
  const int64_t items = (tiles + 3) / 4 * a.B * a.n_qg;
  if (items > 0x7FFFFFFFll) {
    set_error(std::string(who) + ": too much work for one launch");
    return B200_ERR_INVALID;
  }
  const int grid = (int)std::min<int64_t>(items, 2 * sms);
  if constexpr (ROWS) rc = a.H == 32 ? run_logits<64, 32, true>(a, grid, st) : run_logits<64, 64, true>(a, grid, st);
  else if (a.qg * a.H <= 64) rc = a.H == 32 ? run_logits<64, 32, false>(a, grid, st) : run_logits<64, 64, false>(a, grid, st);
  else rc = a.H == 32 ? run_logits<128, 32, false>(a, grid, st) : run_logits<128, 64, false>(a, grid, st);
  if (rc) return rc;
  ++g_launches;
  e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "indexer_logits launch");
  return 0;
}

// rows of the top-k, each on a cluster of CS CTAs while the rows alone would leave most SMs idle
template <bool ROWS>
static int launch_topk(const float* logits, int64_t stride, int64_t width, const int32_t* seq_lens, int Q, int topk,
                       int32_t* out, const int64_t* positions, int ratio, int64_t rows, cudaStream_t st, const char* who) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return cuda_fail(e, "cudaGetDevice");
  const int sms = device_sms(dev);
  if (sms < 0) return sms;
  int cs = 1;
  while (cs < 8 && rows * cs * 2 <= sms) cs *= 2;
  if (rows * cs > 0x7FFFFFFFll) {
    set_error(std::string(who) + ": too many rows");
    return B200_ERR_INVALID;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(rows * cs));
  cfg.blockDim = dim3(TK_THREADS);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  e = cudaLaunchKernelEx(&cfg, indexer_topk_kernel<ROWS>, logits, stride, width, seq_lens, Q, topk, out, positions, ratio);
  ++g_launches;
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "indexer_topk launch");
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_indexer_qk_rope_quant_cache_write(void* stream, const void* q, const void* weights, int64_t weights_row_stride,
                                           const void* k, const int64_t* positions, const void* cos_sin_cache,
                                           int max_position, int is_neox, const int64_t* slot_mapping, void* k_cache,
                                           int block_size, int use_ue8m0, float softmax_scale, float head_scale,
                                           void* q_fp8, float* weights_out, int num_tokens, int num_heads) {
  if (!q || !weights || !k || !positions || !cos_sin_cache || !slot_mapping || !k_cache || !q_fp8 || !weights_out ||
      num_tokens < 0 || num_heads <= 0 || num_heads > 128 || block_size <= 0 || max_position <= 0 ||
      weights_row_stride < num_heads) {
    set_error("b200_indexer_qk_rope_quant_cache_write: bad argument");
    return B200_ERR_INVALID;
  }
  if (misaligned16(q) || misaligned16(k) || misaligned16(q_fp8) || misaligned16(k_cache) ||
      reinterpret_cast<uintptr_t>(weights) % 2 || reinterpret_cast<uintptr_t>(weights_out) % 4 ||
      reinterpret_cast<uintptr_t>(cos_sin_cache) % 2) {
    set_error("b200_indexer_qk_rope_quant_cache_write: q, k, q_fp8 and k_cache must be 16-byte aligned");
    return B200_ERR_INVALID;
  }
  if (num_tokens == 0) return 0;
  const int64_t warps = (int64_t)num_tokens * (num_heads + 1);
  if (warps > 0x7FFFFFFFll) {
    set_error("b200_indexer_qk_rope_quant_cache_write: too many tokens");
    return B200_ERR_INVALID;
  }
  indexer_qk_rope_quant_cache_kernel<<<(unsigned)((warps + IDX_AUX_WARPS - 1) / IDX_AUX_WARPS), IDX_AUX_WARPS * 32, 0,
                                       reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(weights), weights_row_stride,
      reinterpret_cast<const __nv_bfloat16*>(k), positions, reinterpret_cast<const __nv_bfloat16*>(cos_sin_cache),
      max_position, is_neox, slot_mapping, reinterpret_cast<uint8_t*>(k_cache), block_size, use_ue8m0, softmax_scale,
      head_scale, reinterpret_cast<uint8_t*>(q_fp8), weights_out, num_tokens, num_heads);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "indexer_qk_rope_quant_cache launch");
  return 0;
}

int b200_indexer_logits(void* stream, const void* q_fp8, const float* weights, const void* k_cache, int num_blocks,
                        int page_size, const int32_t* seq_lens, const int32_t* page_table, int batch, int q_len,
                        int num_heads, int max_pages, float* logits, int64_t logits_stride) {
  if (!q_fp8 || !weights || !k_cache || !seq_lens || !page_table || !logits || batch < 0 || num_blocks <= 0 ||
      max_pages <= 0) {
    set_error("b200_indexer_logits: bad argument");
    return B200_ERR_INVALID;
  }
  if ((num_heads != 32 && num_heads != 64) || q_len < 1 || q_len > 16 ||
      (page_size != 16 && page_size != 32 && page_size != 64)) {
    set_error("b200_indexer_logits: needs num_heads 32 or 64, 1 <= q_len <= 16, page_size 16, 32 or 64");
    return B200_ERR_INVALID;
  }
  if (logits_stride < (int64_t)max_pages * page_size) {
    set_error("b200_indexer_logits: logits_stride must be >= max_pages * page_size");
    return B200_ERR_INVALID;
  }
  if (misaligned16(q_fp8) || misaligned16(k_cache) || reinterpret_cast<uintptr_t>(weights) % 4 ||
      reinterpret_cast<uintptr_t>(logits) % 4) {
    set_error("b200_indexer_logits: q_fp8 and k_cache must be 16-byte aligned");
    return B200_ERR_INVALID;
  }
  if (batch == 0) return 0;
  LogitsArgs a{};
  a.k_cache = reinterpret_cast<const uint8_t*>(k_cache);
  a.q_fp8 = reinterpret_cast<const uint8_t*>(q_fp8);
  a.weights = weights;
  a.seq_lens = seq_lens;
  a.page_table = page_table;
  a.logits = logits;
  a.stride = logits_stride;
  a.B = batch;
  a.Q = q_len;
  a.H = num_heads;
  a.page = page_size;
  a.max_pages = max_pages;
  return launch_logits<false>(a, num_blocks, reinterpret_cast<cudaStream_t>(stream), "b200_indexer_logits");
}

int b200_indexer_topk(void* stream, const float* logits, int64_t logits_stride, int64_t row_width, const int32_t* seq_lens,
                      int batch, int q_len, int topk, int32_t* out) {
  if (!logits || !seq_lens || !out || batch < 0 || q_len < 1 || row_width <= 0 || logits_stride < row_width || topk < 1 ||
      topk > 2048) {
    set_error("b200_indexer_topk: bad argument (1 <= topk <= 2048, q_len >= 1, 0 < row_width <= logits_stride)");
    return B200_ERR_INVALID;
  }
  if (reinterpret_cast<uintptr_t>(logits) % 4 || reinterpret_cast<uintptr_t>(out) % 4 || logits_stride > 0x7FFFFFFFll) {
    set_error("b200_indexer_topk: logits / out must be 4-byte aligned, logits_stride < 2^31");
    return B200_ERR_INVALID;
  }
  const int64_t rows = (int64_t)batch * q_len;
  if (rows == 0) return 0;
  return launch_topk<false>(logits, logits_stride, row_width, seq_lens, q_len, topk, out, nullptr, 0, rows,
                            reinterpret_cast<cudaStream_t>(stream), "b200_indexer_topk");
}

int b200_dsv4_indexer_q_quant(void* stream, const void* q, const void* weights, int64_t weights_row_stride,
                              const int64_t* positions, const float* cos_sin_cache, int max_position, float softmax_scale,
                              float head_scale, void* q_fp8, float* weights_out, int num_tokens, int num_heads) {
  if (!q || !weights || !positions || !cos_sin_cache || !q_fp8 || !weights_out || num_tokens < 0 ||
      num_tokens > (1 << 20) || num_heads < 1 || num_heads > 128 || max_position < 1 || weights_row_stride < num_heads) {
    set_error("b200_dsv4_indexer_q_quant: bad argument (1 <= num_heads <= 128, 0 <= num_tokens <= 2^20, "
              "weights_row_stride >= num_heads, max_position >= 1)");
    return B200_ERR_INVALID;
  }
  if (misaligned16(q) || misaligned16(q_fp8) || reinterpret_cast<uintptr_t>(weights) % 2 ||
      reinterpret_cast<uintptr_t>(positions) % 8 || reinterpret_cast<uintptr_t>(cos_sin_cache) % 4 ||
      reinterpret_cast<uintptr_t>(weights_out) % 4) {
    set_error("b200_dsv4_indexer_q_quant: q and q_fp8 must be 16-byte aligned, positions 8, cos_sin_cache and "
              "weights_out 4, weights 2");
    return B200_ERR_INVALID;
  }
  if (num_tokens == 0) return 0;
  const int64_t warps = (int64_t)num_tokens * num_heads;
  dsv4_indexer_q_quant_kernel<<<(unsigned)((warps + IDX_AUX_WARPS - 1) / IDX_AUX_WARPS), IDX_AUX_WARPS * 32, 0,
                                reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(weights), weights_row_stride,
      positions, cos_sin_cache, max_position, softmax_scale, head_scale, reinterpret_cast<uint8_t*>(q_fp8), weights_out,
      num_tokens, num_heads);
  ++g_launches;
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "dsv4_indexer_q_quant launch");
  return 0;
}

int b200_dsv4_indexer_decode(void* stream, const void* q_fp8, const float* weights, const void* k_cache, int num_blocks,
                             int page_size, const int64_t* positions, const int32_t* token_to_req,
                             const int32_t* block_table, int max_blocks, int compress_ratio, int num_tokens,
                             int num_heads, int64_t max_seq_len, float* logits, int64_t logits_stride, int topk,
                             int32_t* out) {
  if (!q_fp8 || !weights || !k_cache || !positions || !token_to_req || !block_table || !logits || !out ||
      num_blocks < 1 || max_blocks < 1 || num_tokens < 0 || num_tokens > (1 << 20)) {
    set_error("b200_dsv4_indexer_decode: bad argument (NULL pointer, num_blocks or max_blocks < 1, num_tokens outside "
              "[0, 2^20])");
    return B200_ERR_INVALID;
  }
  if ((num_heads != 32 && num_heads != 64) || (page_size != 16 && page_size != 32 && page_size != 64) ||
      (compress_ratio != 4 && compress_ratio != 128) || topk < 1 || topk > 2048) {
    set_error("b200_dsv4_indexer_decode: needs num_heads 32 or 64, page_size 16, 32 or 64, compress_ratio 4 or 128, "
              "1 <= topk <= 2048");
    return B200_ERR_INVALID;
  }
  const int64_t width = (int64_t)max_blocks * page_size;
  if (logits_stride < width || logits_stride > 0x7FFFFFFFll) {
    set_error("b200_dsv4_indexer_decode: logits_stride must be >= max_blocks * page_size and < 2^31");
    return B200_ERR_INVALID;
  }
  if (misaligned16(q_fp8) || misaligned16(k_cache) || reinterpret_cast<uintptr_t>(weights) % 4 ||
      reinterpret_cast<uintptr_t>(positions) % 8 || reinterpret_cast<uintptr_t>(token_to_req) % 4 ||
      reinterpret_cast<uintptr_t>(block_table) % 4 || reinterpret_cast<uintptr_t>(logits) % 4 ||
      reinterpret_cast<uintptr_t>(out) % 4) {
    set_error("b200_dsv4_indexer_decode: q_fp8 and k_cache must be 16-byte aligned, positions 8, the rest 4");
    return B200_ERR_INVALID;
  }
  if (num_tokens == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // every token of a short context selects all of its candidates: the top-k writes them without reading a logit
  if (max_seq_len <= 0 || max_seq_len / compress_ratio > topk) {
    LogitsArgs a{};
    a.k_cache = reinterpret_cast<const uint8_t*>(k_cache);
    a.q_fp8 = reinterpret_cast<const uint8_t*>(q_fp8);
    a.weights = weights;
    a.page_table = block_table;
    a.logits = logits;
    a.stride = logits_stride;
    a.B = num_tokens;
    a.Q = 1;
    a.H = num_heads;
    a.page = page_size;
    a.max_pages = max_blocks;
    a.positions = positions;
    a.row_req = token_to_req;
    a.ratio = compress_ratio;
    const int rc = launch_logits<true>(a, num_blocks, st, "b200_dsv4_indexer_decode");
    if (rc) return rc;
  }
  return launch_topk<true>(logits, logits_stride, width, nullptr, 1, topk, out, positions, compress_ratio, num_tokens, st,
                           "b200_dsv4_indexer_decode");
}

}  // extern "C"
