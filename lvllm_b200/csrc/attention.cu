// Paged decode attention, split-KV + LSE merge: the entry points, the split merges and the CUDA-core GQA kernel.
// MLA and GQA take Q >= 1 query tokens per request (speculative decode: query token i of request b sees keys
// [0, S_b - Q + i], the end-aligned causal mask).
//   MLA (absorbed): q = [q_nope(512) | q_pe(64)], one shared latent KV head, K = all 576 cols, V = first 512
//                   (op contract of reference csrc/libtorch_stable/attention/mla/sm100_cutlass_mla_kernel.cu:225-262);
//                   up to 128 heads, on the tensor-core kernel (attention_mla.cu)
//   GQA           : q [B,Hq,D], K / V caches [pages,page,Hkv,D] given by base pointer + (page, slot, head) strides:
//                   separate contiguous caches or the halves of the FlashInfer backend's packed NHD / HND cache
//                   (reference tests/kernels/attention/test_flashinfer.py:29-80); the tensor-core kernel
//                   (attention_gqa.cu) where it applies, decode_attn_kernel otherwise
//
// decode_attn_kernel (CUDA cores): a CTA owns (request, kv-head, head-group, split); KV tiles of TOK tokens are staged
// ONCE in shared memory with 16-byte coalesced loads and shared by all heads of the group (one warp per q
// head), so HBM traffic == algorithmic KV bytes; the warp does the dot product over its lane-strided dims,
// online softmax in fp32 (exp2 domain), and accumulates V.  It serves groups of more than 32 query heads per kv head,
// more work items per CTA than the tensor-core kernel's table holds, and split counts that do not cover the page table.
// With Q query tokens per request each query row (b, i) is a CTA row of its own that does exactly the arithmetic of a
// single-token decode over its S_b - Q + 1 + i keys, so this path reads a request's KV Q times (acceptable for a fallback).
// Partial (o, m, l) per split are merged by a second tiny kernel that also emits the natural-log LSE.
// Roofline: HBM (KV bytes).
#include <math_constants.h>

#include "common.cuh"
#include "moe_internal.cuh"

namespace b200 {

constexpr int ATT_TOK = 16;  // tokens per smem tile

template <int DK, int DV, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
    decode_attn_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ kc,
                       const __nv_bfloat16* __restrict__ vc, const int32_t* __restrict__ seq_lens,
                       const int32_t* __restrict__ page_table, int Hq, int Hkv, int page_size, int max_pages,
                       float scale_log2, int num_splits, float* __restrict__ part_o, float* __restrict__ part_ml,
                       int64_t block_stride, int64_t page_stride, int64_t head_stride, int Q) {
  // blockIdx.x = (((b * Q + i) * Hkv + hkv) * groups_per_kv + hg) for draft token i, blockIdx.y = split
  // K / V row of (page, slot in page, kv head) at page * block_stride + slot * page_stride + hkv * head_stride (elements)
  const int G = Hq / Hkv;
  const int groups_per_kv = (G + WARPS - 1) / WARPS;
  int bx = blockIdx.x;
  const int hg = bx % groups_per_kv;
  bx /= groups_per_kv;
  const int hkv = bx % Hkv;
  const int row = bx / Hkv;   // query row b * Q + i
  const int b = row / Q;
  const int split = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int head_in_group = hg * WARPS + warp;
  const bool head_ok = head_in_group < G;
  const int hq = hkv * G + (head_ok ? head_in_group : 0);

  const int S = max(seq_lens[b] - Q + 1 + row % Q, 0);   // keys this query token sees
  const int per = ((S + num_splits - 1) / num_splits + ATT_TOK - 1) / ATT_TOK * ATT_TOK;
  const int s0 = split * per;
  const int s1 = min(S, s0 + per);

  __shared__ __align__(16) __nv_bfloat16 ks[ATT_TOK][DK];
  __shared__ __align__(16) __nv_bfloat16 vs[ATT_TOK][DV];

  constexpr int NK = DK / 32, NV = DV / 32;
  float qr[NK];
#pragma unroll
  for (int i = 0; i < NK; ++i) qr[i] = __bfloat162float(q[((size_t)row * Hq + hq) * DK + lane + 32 * i]) * scale_log2;
  float o[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) o[i] = 0.f;
  float m = -CUDART_INF_F, l = 0.f;

  for (int t0 = s0; t0 < s1; t0 += ATT_TOK) {
    const int nt = min(ATT_TOK, s1 - t0);
    __syncthreads();
    // cooperative 16-byte loads of the K and V rows of this tile
    constexpr int KCH = DK / 8;
    for (int i = threadIdx.x; i < ATT_TOK * KCH; i += WARPS * 32) {
      const int tt = i / KCH, c = i % KCH;
      if (tt < nt) {
        const int tok = t0 + tt;
        const int page = page_table[(size_t)b * max_pages + tok / page_size];
        const __nv_bfloat16* src = kc + page * block_stride + (tok % page_size) * page_stride + hkv * head_stride;
        *reinterpret_cast<uint4*>(&ks[tt][c * 8]) = *reinterpret_cast<const uint4*>(src + c * 8);
      }
    }
    constexpr int VCH = DV / 8;
    for (int i = threadIdx.x; i < ATT_TOK * VCH; i += WARPS * 32) {
      const int tt = i / VCH, c = i % VCH;
      if (tt < nt) {
        const int tok = t0 + tt;
        const int page = page_table[(size_t)b * max_pages + tok / page_size];
        *reinterpret_cast<uint4*>(&vs[tt][c * 8]) = *reinterpret_cast<const uint4*>(
            vc + page * block_stride + (tok % page_size) * page_stride + hkv * head_stride + c * 8);
      }
    }
    __syncthreads();
    if (head_ok) {
      float sc[ATT_TOK];
#pragma unroll
      for (int tt = 0; tt < ATT_TOK; ++tt) {
        float acc = 0.f;
#pragma unroll
        for (int i = 0; i < NK; ++i) acc = fmaf(qr[i], __bfloat162float(ks[tt][lane + 32 * i]), acc);
        sc[tt] = acc;
      }
#pragma unroll
      for (int tt = 0; tt < ATT_TOK; ++tt) {
        sc[tt] = warp_sum(sc[tt]);
        if (tt >= nt) sc[tt] = -CUDART_INF_F;
      }
      float mt = m;
#pragma unroll
      for (int tt = 0; tt < ATT_TOK; ++tt) mt = fmaxf(mt, sc[tt]);
      const float corr = (m == -CUDART_INF_F) ? 0.f : exp2f(m - mt);
      l *= corr;
#pragma unroll
      for (int i = 0; i < NV; ++i) o[i] *= corr;
#pragma unroll
      for (int tt = 0; tt < ATT_TOK; ++tt) {
        if (tt >= nt) break;   // rows past the tile's tokens hold stale shared memory: 0 * NaN would poison o
        const float p = exp2f(sc[tt] - mt);
        l += p;
#pragma unroll
        for (int i = 0; i < NV; ++i) o[i] = fmaf(p, __bfloat162float(vs[tt][lane + 32 * i]), o[i]);
      }
      m = mt;
    }
  }
  if (head_ok) {
    const size_t base = ((size_t)row * Hq + hq) * num_splits + split;
#pragma unroll
    for (int i = 0; i < NV; ++i) part_o[base * DV + lane + 32 * i] = o[i];
    if (lane == 0) {
      part_ml[base * 2] = m;
      part_ml[base * 2 + 1] = l;
    }
  }
}

// merge splits: one warp per (b, head)
template <int DV>
__global__ void __launch_bounds__(128) decode_merge_kernel(const float* __restrict__ part_o,
                                                          const float* __restrict__ part_ml, int BH, int num_splits,
                                                          __nv_bfloat16* __restrict__ out, float* __restrict__ lse) {
  const int w = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= BH) return;
  float mx = -CUDART_INF_F;
  for (int s = 0; s < num_splits; ++s) mx = fmaxf(mx, part_ml[((size_t)w * num_splits + s) * 2]);
  float lsum = 0.f;
  float acc[DV / 32];
#pragma unroll
  for (int i = 0; i < DV / 32; ++i) acc[i] = 0.f;
  for (int s = 0; s < num_splits; ++s) {
    const size_t base = (size_t)w * num_splits + s;
    const float ms = part_ml[base * 2], ls = part_ml[base * 2 + 1];
    if (ms == -CUDART_INF_F) continue;
    const float f = exp2f(ms - mx);
    lsum += ls * f;
#pragma unroll
    for (int i = 0; i < DV / 32; ++i) acc[i] = fmaf(f, part_o[base * DV + lane + 32 * i], acc[i]);
  }
  const float inv = lsum > 0.f ? 1.f / lsum : 0.f;
#pragma unroll
  for (int i = 0; i < DV / 32; ++i) out[(size_t)w * DV + lane + 32 * i] = __float2bfloat16_rn(acc[i] * inv);
  if (lse && lane == 0) lse[w] = (lsum > 0.f) ? (mx * 0.6931471805599453f + logf(lsum)) : -CUDART_INF_F;
}

// merge for many splits (tensor-core MLA): one CTA per (b, head), thread = float4 of the 512 dims; the split
// weights are computed once in shared memory, partial rows are read 8 splits at a time (independent loads)
// SINK (DeepSeek-V4 attn_sink, f32 [Hq], natural-log units, row w is head w % Hq): folded in once, after every split is
// merged: m' = max(m, sink), l' = l e^(m - m') + e^(sink - m'), out = acc e^(m - m') / l'.  A row with no valid key keeps
// l = 0 and gets out = 0; sink = -inf gives the bits of the merge without a sink.
template <bool SINK>
__global__ void __launch_bounds__(128) mla_merge_kernel(const float* __restrict__ part_o,
                                                       const float* __restrict__ part_ml, int num_splits,
                                                       __nv_bfloat16* __restrict__ out, float* __restrict__ lse,
                                                       const float* __restrict__ sink, int Hq) {
  __shared__ float wgt[512];
  __shared__ float red[4];
  const int w = blockIdx.x, tid = threadIdx.x;
  const float* ml = part_ml + (size_t)w * num_splits * 2;
  float mx = -CUDART_INF_F;
  for (int s = tid; s < num_splits; s += 128) mx = fmaxf(mx, ml[s * 2]);
  mx = warp_max(mx);
  if ((tid & 31) == 0) red[tid >> 5] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  __syncthreads();
  float ls = 0.f;
  for (int s = tid; s < num_splits; s += 128) {
    const float ms = ml[s * 2];
    const float f = (ms == -CUDART_INF_F) ? 0.f : exp2f(ms - mx);
    wgt[s] = f;
    ls += f * ml[s * 2 + 1];
  }
  ls = warp_sum(ls);
  if ((tid & 31) == 0) red[tid >> 5] = ls;
  __syncthreads();
  const float lsum = red[0] + red[1] + red[2] + red[3];
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  const float* po = part_o + (size_t)w * num_splits * 512 + tid * 4;
  for (int s0 = 0; s0 < num_splits; s0 += 16) {   // 16 independent 16-byte loads in flight per thread
    float4 v[16];
    float f[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int s = s0 + u;
      f[u] = (s < num_splits) ? wgt[s] : 0.f;
      v[u] = (f[u] != 0.f) ? __ldcs(reinterpret_cast<const float4*>(po + (size_t)s * 512)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      acc.x = fmaf(f[u], v[u].x, acc.x);
      acc.y = fmaf(f[u], v[u].y, acc.y);
      acc.z = fmaf(f[u], v[u].z, acc.z);
      acc.w = fmaf(f[u], v[u].w, acc.w);
    }
  }
  float inv = lsum > 0.f ? 1.f / lsum : 0.f;
  if (SINK && lsum > 0.f) {   // exp2 domain: the partials' m are in log2 units
    const float sk = sink[w % Hq] * 1.4426950408889634f, m2 = fmaxf(mx, sk);
    const float f = exp2f(mx - m2);
    inv = f / fmaf(lsum, f, exp2f(sk - m2));
  }
  __nv_bfloat162 a = __floats2bfloat162_rn(acc.x * inv, acc.y * inv), c = __floats2bfloat162_rn(acc.z * inv, acc.w * inv);
  uint2 pk;
  pk.x = *reinterpret_cast<uint32_t*>(&a);
  pk.y = *reinterpret_cast<uint32_t*>(&c);
  *reinterpret_cast<uint2*>(out + (size_t)w * 512 + tid * 4) = pk;
  if (lse && tid == 0) lse[w] = (lsum > 0.f) ? (mx * 0.6931471805599453f + logf(lsum)) : -CUDART_INF_F;
}

// split partials of the MLA-family decode kernel in the workspace: O [rows * num_heads * num_splits][512], then (m, l)
struct MlaPartials {
  float *o, *ml;
};
static MlaPartials mla_partials(void* workspace, int rows, int num_heads, int num_splits) {
  float* po = reinterpret_cast<float*>(workspace);
  return {po, po + (size_t)rows * num_heads * num_splits * 512};
}

// merge of the MLA decode kernel's partials over query rows x heads: fused with the v up-projection when w_uv is given
// (mla_aux.cu), mla_merge_kernel up to 512 splits (with the DeepSeek-V4 attention sink when sink is given),
// decode_merge_kernel above.  The fused v up-projection has no sink: the two are exclusive.
static int mla_merge(cudaStream_t st, const MlaPartials& p, int rows, int num_heads, int num_splits, void* out, float* lse,
                     const void* w_uv, void* out_v, const float* sink = nullptr) {
  const float *po = p.o, *pml = p.ml;
  auto bo = reinterpret_cast<__nv_bfloat16*>(out);
  if (w_uv)
    launch_mla_merge_vup(st, po, pml, rows, num_splits, num_heads, w_uv, out_v, out, lse);
  else if (sink)
    mla_merge_kernel<true><<<rows * num_heads, 128, 0, st>>>(po, pml, num_splits, bo, lse, sink, num_heads);
  else if (num_splits <= 512)
    mla_merge_kernel<false><<<rows * num_heads, 128, 0, st>>>(po, pml, num_splits, bo, lse, nullptr, num_heads);
  else
    decode_merge_kernel<512><<<(rows * num_heads + 3) / 4, 128, 0, st>>>(po, pml, rows * num_heads, num_splits, bo, lse);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "mla merge launch");
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" {

int64_t b200_mla_decode_workspace_bytes(int batch, int num_heads, int num_splits) {
  return (int64_t)batch * num_heads * num_splits * (512 + 2) * 4;
}
int64_t b200_gqa_decode_workspace_bytes(int batch, int num_q_heads, int head_dim, int num_splits) {
  return (int64_t)batch * num_q_heads * num_splits * (head_dim + 2) * 4;
}

int b200_mla_decode(void* stream, const void* q_nope, const void* q_pe, const void* kv_cache,
                    const int32_t* seq_lens, const int32_t* page_table, int batch, int num_heads, int page_size,
                    int max_pages, float sm_scale, int num_splits, void* workspace, void* out, float* lse) {
  return b200_mla_decode_ex(stream, q_nope, q_pe, 0, kv_cache, 0, 1.f, 1.f, seq_lens, page_table, batch, num_heads,
                            page_size, max_pages, sm_scale, num_splits, workspace, out, lse);
}

int b200_mla_decode_ex(void* stream, const void* q_nope, const void* q_pe, int q_dtype, const void* kv_cache,
                       int kv_dtype, float descale_q, float descale_k, const int32_t* seq_lens,
                       const int32_t* page_table, int batch, int num_heads, int page_size, int max_pages, float sm_scale,
                       int num_splits, void* workspace, void* out, float* lse) {
  return b200_mla_decode_spec(stream, q_nope, q_pe, q_dtype, kv_cache, kv_dtype, descale_q, descale_k, seq_lens, page_table,
                              batch, 1, num_heads, page_size, max_pages, sm_scale, num_splits, workspace, out, lse, nullptr,
                              nullptr);
}

int b200_mla_decode_spec(void* stream, const void* q_nope, const void* q_pe, int q_dtype, const void* kv_cache,
                         int kv_dtype, float descale_q, float descale_k, const int32_t* seq_lens,
                         const int32_t* page_table, int batch, int q_len, int num_heads, int page_size, int max_pages,
                         float sm_scale, int num_splits, void* workspace, void* out, float* lse, const void* w_uv,
                         void* out_v) {
  if (q_len < 1 || q_len > 16) {
    set_error("b200_mla_decode: q_len must be in [1, 16]");
    return B200_ERR_INVALID;
  }
  if (!q_nope || !q_pe || !kv_cache || !seq_lens || !page_table || !workspace || batch <= 0 || num_heads <= 0 ||
      num_heads > 128 || page_size <= 0 || num_splits <= 0 || q_dtype < 0 || q_dtype > 1 || kv_dtype < 0 || kv_dtype > 1 ||
      (w_uv ? (!out_v || num_splits > 512) : !out)) {
    set_error("b200_mla_decode: bad argument (num_heads <= 128; out, or with w_uv out_v and num_splits <= 512)");
    return B200_ERR_INVALID;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int rows = batch * q_len;   // query rows (b, i), b * q_len + i
  const MlaPartials p = mla_partials(workspace, rows, num_heads, num_splits);
  // each CTA walks ceil(tiles / num_splits) 128-token tiles (online softmax)
  int rc = launch_mla_tc(st, q_nope, q_pe, kv_cache, seq_lens, page_table, batch, q_len, num_heads, page_size, max_pages,
                         sm_scale, num_splits, p.o, p.ml, kv_dtype, q_dtype, descale_q, descale_k);
  if (rc) return rc;
  return mla_merge(st, p, rows, num_heads, num_splits, out, lse, w_uv, out_v);
}

int b200_mla_decode_sparse(void* stream, const void* q_nope, const void* q_pe, const void* kv_cache, int kv_dtype,
                           const int32_t* topk_indices, int topk, const int32_t* req_id, const int32_t* page_table,
                           int max_pages, int num_tokens, int num_heads, int page_size, float sm_scale, int num_splits,
                           void* workspace, void* out, float* lse, const void* w_uv, void* out_v) {
  if (!q_nope || !q_pe || !kv_cache || !topk_indices || !req_id || !page_table || !workspace || num_tokens <= 0 ||
      num_heads <= 0 || num_heads > 128 || topk < 1 || page_size <= 0 || max_pages <= 0 || num_splits <= 0 ||
      (kv_dtype != 0 && kv_dtype != 2) || (w_uv ? (!out_v || num_splits > 512) : !out)) {
    set_error("b200_mla_decode_sparse: bad argument (kv_dtype 0 or 2, num_heads <= 128, topk >= 1; out, or with w_uv out_v "
              "and num_splits <= 512)");
    return B200_ERR_INVALID;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const MlaPartials p = mla_partials(workspace, num_tokens, num_heads, num_splits);
  const int rc = launch_mla_sparse_tc(st, q_nope, q_pe, kv_cache, kv_dtype == 2, topk_indices, topk, req_id, page_table,
                                      max_pages, num_tokens, num_heads, page_size, sm_scale, num_splits, p.o, p.ml);
  if (rc) return rc;
  return mla_merge(st, p, num_tokens, num_heads, num_splits, out, lse, w_uv, out_v);
}

int b200_dsv4_sparse_decode(void* stream, const void* q, int num_tokens, int num_heads, const void* swa_cache,
                            int swa_block_size, int swa_num_blocks, int64_t swa_block_stride, const int32_t* swa_indices,
                            int swa_topk, const int32_t* swa_lens, const void* extra_cache, int extra_block_size,
                            int extra_num_blocks, int64_t extra_block_stride, const int32_t* extra_indices, int extra_topk,
                            const int32_t* extra_lens, const float* attn_sink, float sm_scale, int num_splits,
                            void* workspace, void* out) {
  auto a16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
  auto a4 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3u) == 0; };
  // a cache: 16-byte aligned, blocks of block_size x 584 bytes at a 16-byte multiple stride
  auto cache_ok = [&](const void* c, int bs, int nb, int64_t stride) {
    return c && a16(c) && bs > 0 && nb > 0 && stride >= (int64_t)bs * 584 && stride % 16 == 0;
  };
  const bool extra = extra_cache != nullptr;
  if (!q || !a16(q) || num_tokens <= 0 || num_tokens > 65535 || num_heads <= 0 || num_heads > 128 ||
      !cache_ok(swa_cache, swa_block_size, swa_num_blocks, swa_block_stride) || !swa_indices || !a4(swa_indices) ||
      swa_topk < 1 || !swa_lens || !a4(swa_lens) ||
      (extra && (!cache_ok(extra_cache, extra_block_size, extra_num_blocks, extra_block_stride) || !extra_indices ||
                 !a4(extra_indices) || extra_topk < 1 || !extra_lens || !a4(extra_lens))) ||
      (attn_sink && !a4(attn_sink)) || num_splits <= 0 || num_splits > 512 || !workspace || !a16(workspace) || !out ||
      !a16(out)) {
    set_error("b200_dsv4_sparse_decode: bad argument (num_tokens <= 65535, num_heads <= 128, topk >= 1, 16-byte aligned q, "
              "caches, workspace and out, block stride >= block_size * 584 and a multiple of 16, 1 <= num_splits <= 512; "
              "extra_cache given: its indices, lengths and shape too)");
    return B200_ERR_INVALID;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const MlaPartials p = mla_partials(workspace, num_tokens, num_heads, num_splits);
  int rc = launch_dsv4_sparse_tc(st, q, swa_cache, swa_block_size, swa_num_blocks, swa_block_stride, swa_indices, swa_topk,
                                 swa_lens, extra_cache, extra_block_size, extra_num_blocks, extra_block_stride,
                                 extra ? extra_indices : nullptr, extra_topk, extra_lens, num_tokens, num_heads, sm_scale,
                                 num_splits, p.o, p.ml);
  if (rc) return rc;
  return mla_merge(st, p, num_tokens, num_heads, num_splits, out, nullptr, nullptr, nullptr, attn_sink);
}

int b200_gqa_decode(void* stream, const void* q, const void* k_cache, const void* v_cache, const int32_t* seq_lens,
                    const int32_t* page_table, int batch, int num_q_heads, int num_kv_heads, int head_dim,
                    int page_size, int max_pages, float sm_scale, int num_splits, void* workspace, void* out,
                    float* lse) {
  const int64_t hs = head_dim, ps = (int64_t)num_kv_heads * head_dim, bs = (int64_t)page_size * num_kv_heads * head_dim;
  return b200_gqa_decode_ex(stream, q, k_cache, v_cache, bs, ps, hs, seq_lens, page_table, batch, num_q_heads,
                            num_kv_heads, head_dim, page_size, max_pages, sm_scale, num_splits, workspace, out, lse);
}

int b200_gqa_decode_ex(void* stream, const void* q, const void* k_cache, const void* v_cache, int64_t block_stride,
                       int64_t page_stride, int64_t head_stride, const int32_t* seq_lens, const int32_t* page_table,
                       int batch, int num_q_heads, int num_kv_heads, int head_dim, int page_size, int max_pages,
                       float sm_scale, int num_splits, void* workspace, void* out, float* lse) {
  return b200_gqa_decode_spec(stream, q, k_cache, v_cache, block_stride, page_stride, head_stride, seq_lens, page_table,
                              batch, 1, num_q_heads, num_kv_heads, head_dim, page_size, max_pages, sm_scale, num_splits,
                              workspace, out, lse);
}

int b200_gqa_decode_spec(void* stream, const void* q, const void* k_cache, const void* v_cache, int64_t block_stride,
                         int64_t page_stride, int64_t head_stride, const int32_t* seq_lens, const int32_t* page_table,
                         int batch, int q_len, int num_q_heads, int num_kv_heads, int head_dim, int page_size,
                         int max_pages, float sm_scale, int num_splits, void* workspace, void* out, float* lse) {
  if (q_len < 1 || q_len > 16) {
    set_error("b200_gqa_decode: q_len must be in [1, 16]");
    return B200_ERR_INVALID;
  }
  if (!q || !k_cache || !v_cache || !seq_lens || !page_table || !workspace || !out || batch <= 0 ||
      num_q_heads <= 0 || num_kv_heads <= 0 || num_q_heads % num_kv_heads || page_size <= 0 || num_splits <= 0) {
    set_error("b200_gqa_decode: bad argument");
    return B200_ERR_INVALID;
  }
  if (head_dim != 128) {
    set_error("b200_gqa_decode: head_dim must be 128");
    return B200_ERR_INVALID;
  }
  // 16-byte cp.async / vector loads of every K / V row: strides in multiples of 8 elements, 16-byte aligned bases
  if (block_stride <= 0 || page_stride <= 0 || head_stride <= 0 || block_stride % 8 || page_stride % 8 || head_stride % 8 ||
      (reinterpret_cast<uintptr_t>(k_cache) | reinterpret_cast<uintptr_t>(v_cache)) % 16) {
    set_error("b200_gqa_decode: cache strides must be positive multiples of 8 elements, cache pointers 16-byte aligned");
    return B200_ERR_INVALID;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int G = num_q_heads / num_kv_heads;
  float* po = reinterpret_cast<float*>(workspace);
  const int rows = batch * q_len;   // query rows (b, i), b * q_len + i
  float* pml = po + (size_t)rows * num_q_heads * num_splits * 128;
  const float sl2 = sm_scale * 1.4426950408889634f;
  // tensor-core path (persistent CTAs over (request, kv head, q-group, 128-token split) items): needs the split count
  // to cover the longest sequence the page table can describe
  if (G <= 128 && num_splits <= 1024 && (int64_t)num_splits * 128 >= (int64_t)max_pages * page_size) {
    const int rc = launch_gqa_tc(st, q, k_cache, v_cache, block_stride, page_stride, head_stride, seq_lens, page_table, batch,
                                 q_len, num_q_heads, num_kv_heads, page_size, max_pages, sm_scale, num_splits, po, pml, out,
                                 lse);
    if (rc <= 0) return rc;   // rc == 1: more work items per CTA than the kernel's table holds
  }
#define LAUNCH_GQA(W)                                                                                          \
  {                                                                                                            \
    const int groups = (G + W - 1) / W;                                                                        \
    dim3 grid(rows * num_kv_heads * groups, num_splits);                                                       \
    decode_attn_kernel<128, 128, W><<<grid, W * 32, 0, st>>>(                                                  \
        reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(k_cache),            \
        reinterpret_cast<const __nv_bfloat16*>(v_cache), seq_lens, page_table, num_q_heads, num_kv_heads,      \
        page_size, max_pages, sl2, num_splits, po, pml, block_stride, page_stride, head_stride, q_len);        \
  }
  if (G <= 4)
    LAUNCH_GQA(4)
  else if (G <= 8)
    LAUNCH_GQA(8)
  else
    LAUNCH_GQA(16)
#undef LAUNCH_GQA
  decode_merge_kernel<128><<<(rows * num_q_heads + 3) / 4, 128, 0, st>>>(
      po, pml, rows * num_q_heads, num_splits, reinterpret_cast<__nv_bfloat16*>(out), lse);
  g_launches += 2;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "gqa_decode launch");
  return 0;
}

}  // extern "C"
