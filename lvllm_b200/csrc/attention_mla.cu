// Paged MLA decode (absorbed form) on wgmma tensor cores.
//
//   S[128 heads, 128 tokens] = Q[128, 576] * K^T        (9 k-blocks of 64 dims, accumulator in registers)
//   P = exp2(S*scale - m) (bf16, straight from the accumulator registers), l = sum P
//   O[128 heads, 128 dims]   = P[128, 128 tokens] * V[128 tokens, 128]     (V = first 512 latent dims; this
//                                                                          CTA owns one quarter of them)
//
// One CTA = (request, q-group, run of 128-token KV tiles, quarter of the 512 value dims).  A KV tile is loaded ONCE into
// shared memory as nine [128 tokens x 128 B] blocks with the 128-byte swizzle: block kb is the K-major B
// operand of the QK^T MMA for dims [64kb, 64kb+64) and — the same bytes, read through an MN-major
// descriptor — the B operand of the PV MMA for value dims [64kb, 64kb+64).  Two consumer warpgroups take 64 heads
// each: a thread keeps its share of S (64 fp32) and of O (64 fp32) in registers, the softmax runs on the accumulator
// fragment (row statistics over the four threads of a quad) and P feeds the PV MMA as a register operand, so neither S
// nor P touches shared memory.  A quarter of the value dims per CTA is what keeps both accumulators in registers.
// Partial (O, m, l) per split are merged by mla_merge_kernel (attention.cu), by decode_merge_kernel above 512 splits.
//
// Speculative decode (multi-token-prediction verification): a request has Q query tokens (its last Q positions, in draft
// order); query token i sees keys [0, S_b - Q + i] (the end-aligned causal mask, reference FlashMLA with causal=True,
// v1/attention/backends/mla/flashmla.py:284-344).  The 128 MMA rows become (draft token, head) pairs: a q-group holds
// Qg = min(Q, 128 / Hq) draft tokens and row r is draft token qg * Qg + r / Hq, head r % Hq, i.e. q / output row
// (b * Q + qg * Qg) * Hq + r.  Rows past the group's last token load zero q and are never written.  The q-group index
// varies with the value-dim part in blockIdx.y, so the CTAs reading the same KV tile are scheduled together.  Each
// accumulator row masks with its own key count; Q = 1 is the single-token decode (one q-group, rows = heads).
//
// Sparse decode (DeepSeek-V3.2 / GLM-5 layers with a lightning indexer): query token t attends only to the keys its
// indexer picked, topk_indices[t, 0 .. topk), request-local positions of request req_id[t] (-1 = no key).  A CTA is (token,
// split over index tiles, value-dim quarter); a tile is 128 consecutive entries of the token's index row, and the loaders
// take each key row from the index (page_table[req_id[t]][idx / page] * page + idx % page, the reference's
// triton_convert_req_index_to_global_index, v1/attention/backends/mla/sparse_utils.py:120, fused into the gather).  An entry
// with idx < 0 or idx / page >= max_pages is invalid: its row is zero-filled and its column masked for every row of the CTA
// through a per-tile 128-bit mask the loaders publish in shared memory.  The cache is bf16 (576 elements per token) or
// fp8_ds_mla (656 bytes per token: 512 e4m3, four fp32 scales, one per 128 dims, 64 bf16 rope dims; reference
// v1/attention/backends/mla/flashmla_sparse.py:63-72), widened to bf16 by the loaders.
//
// DeepSeek-V4 sparse decode (V4): head dim 512 = 448 NoPE + 64 RoPE dims, and the key row is also the value row (shared-KV
// MQA, no absorb).  The keys of token t are the concatenation main || extra: swa_indices[t, :swa_lens[t]] (global slots of the
// sliding-window cache) followed by extra_indices[t, :extra_lens[t]] (global slots of the compressed cache, its own block
// size); a slot resolves to (block = slot / block_size, pos = slot % block_size), and a slot < 0 or >= num_blocks * block_size
// is no key (zero-filled, masked as above).  Both caches hold 584-byte tokens laid out per block (reference
// flashmla_sparse.py:76-85, _read_fp8_ds_mla_cache in tests/kernels/attention/test_rocm_triton_attn_dsv4.py:125-147): the
// block's block_size x 576 data bytes (448 e4m3 | 64 bf16 rope) come first, then block_size x 8 scale bytes (7 ue8m0, one per
// 64 NoPE dims, and a pad byte); blocks are block_stride bytes apart.  QK^T runs over 8 k-blocks (kb 7 = rope, by cp.async),
// the loaders widen kb 0-6 to bf16(e4m3) * 2^(s - 127) (exact), and value quarter p is k-blocks 2p, 2p + 1 (quarter 3 = NoPE
// 384-447 | rope).  The q row is the 512-dim [T, Hq, 512] row, read through q_nope.  The attention sink is folded in by the
// split merge (attention.cu).
//
// Warp roles (384 threads): warps 0-3 / 4-7 consumer warpgroups (MMA + softmax + epilogue), warps 8-11 loaders
// (16-byte gathers of q rows / paged KV rows -> swizzled smem, generic->async proxy fence).
// The op contract is reference csrc/libtorch_stable/attention/mla/sm100_cutlass_mla_kernel.cu:225-262.
// Roofline: KV bytes (HBM / L2) — at B=1 the kernel is latency bound.  Algorithmic bytes = sum_b S_b * 576 * {2, 1} (bf16,
// e4m3 cache) * n_qg (n_qg = ceil(Q / Qg) q-groups, each reading the request's tiles again).
#include <math_constants.h>

#include "common.cuh"
#include "moe_internal.cuh"

namespace b200 {

constexpr int MLA_TOK = 128;            // tokens per CTA
constexpr int MLA_KB = 9;               // 576 / 64
constexpr int MLA_THREADS = 384;
constexpr int MLA_QSTAGES = 4;
constexpr int MLA_PARTS = 4;            // CTAs sharing the 512 value dims of a split
constexpr int MLA_DV = 512 / MLA_PARTS; // value dims per CTA (two 64-dim blocks)
constexpr int MLA_K_AREA = MLA_KB * TILE_BYTES;          // 144 KB
constexpr int MLA_Q_RING = MLA_QSTAGES * TILE_BYTES;     // 64 KB
constexpr int MLA_SMEM = MLA_K_AREA + MLA_Q_RING + 1024 + 1024;

struct MlaBars {
  uint64_t full[MLA_KB], empty[MLA_QSTAGES];
  uint64_t s_full, o_full;   // QK^T / PV of the tile complete in both warpgroups: its blocks may be refilled
  int8_t row_off[128];       // SPEC: MMA row r sees row_off[r] keys fewer than the q-group's last draft token
  // SPARSE: the valid columns of tile ti in kvalid[ti & 1]; loader warp w publishes word w, bit 4u + r = column
  // 16u + 4w + r, and arrives on v_full once the word is written
  uint64_t v_full;
  uint32_t kvalid[2][4];
};

// V4: the parts of the key lists the kernel's shared arguments do not carry (the main list's cache, index rows, lengths,
// block size and block count go in kv, topk_idx, seq_lens, page_size and max_pages); extra_idx == nullptr: no extra list
struct Dsv4Keys {
  const void* extra_kv;
  const int32_t* extra_idx;
  const int32_t* extra_lens;
  int extra_topk, extra_block, extra_blocks;
  int64_t main_stride, extra_stride;   // block strides in bytes
};

B200_DEVICE void mla_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}

// eight e4m3 bytes -> eight bf16 (exact: e4m3 has 4 exponent / 3 mantissa bits)
B200_DEVICE uint4 fp8x8_to_bf16x8(uint2 v) {
  const uint32_t w[2] = {v.x, v.y};
  uint32_t o[4];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)((w[i] >> (16 * h)) & 0xFFFFu), __NV_E4M3);
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hr));
      const __nv_bfloat162 b = __floats2bfloat162_rn(f.x, f.y);
      o[i * 2 + h] = *reinterpret_cast<const uint32_t*>(&b);
    }
  }
  return make_uint4(o[0], o[1], o[2], o[3]);
}

// V4: scale of NoPE k-block kb of a 584-byte row, 2^(s - 127) for its ue8m0 byte s (s = 0 is the fp32 subnormal 2^-127)
B200_DEVICE float ue8m0_scale(uint2 rec, int kb) {
  const uint32_t s = ((kb < 4 ? rec.x : rec.y) >> (8 * (kb & 3))) & 0xFFu;
  return __uint_as_float(s ? s << 23 : 0x00400000u);
}

// eight e4m3 bytes of an fp8_ds_mla row -> eight bf16 bf16(float(e4m3) * scale): the fp32 product, rounded once to bf16
B200_DEVICE uint4 fp8x8_scaled_to_bf16x8(uint2 v, float scale) {
  const uint32_t w[2] = {v.x, v.y};
  uint32_t o[4];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)((w[i] >> (16 * h)) & 0xFFFFu), __NV_E4M3);
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hr));
      const __nv_bfloat162 b = __floats2bfloat162_rn(__fmul_rn(f.x, scale), __fmul_rn(f.y, scale));
      o[i * 2 + h] = *reinterpret_cast<const uint32_t*>(&b);
    }
  }
  return make_uint4(o[0], o[1], o[2], o[3]);
}

// KV8: the latent cache is e4m3 (kv_cache_dtype "fp8": 576 bytes per token, half the HBM traffic of the bf16 cache;
// reference fp8 dtypes backends/mla/cutlass_mla.py:44-45).  The loaders widen it to bf16 on the way into shared memory
// (exact), so the tensor-core pipeline and its numerics are those of the bf16 kernel — P is NOT re-quantised to fp8.
// q8: the queries are e4m3 too (the reference's fp8 test feeds fp8 q, tests/kernels/attention/test_cutlass_mla_decode.py:101-110).
// SPEC: Q > 1 query tokens per request.  Without it every q-group expression below is a compile-time constant (Q = Qg = 1,
// rows = heads, one limit for every row), which keeps the single-token decode free of the per-row bookkeeping.
// SPARSE: blockIdx.z is a query token, its keys come from topk_idx (see the header); with KV8 the cache is fp8_ds_mla (the
// queries are bf16 then, q8 = 0).  The three trailing arguments are read by the sparse instantiations only.
// V4 (with KV8 && SPARSE): the DeepSeek-V4 cache (see the header).  kv / topk_idx / topk / seq_lens / page_size / max_pages are
// the main list's cache, index rows, row width, lengths, block size and block count; v4 holds the rest.
template <bool KV8, bool SPEC, bool SPARSE, bool V4>
__global__ void __launch_bounds__(MLA_THREADS, 1)
    mla_decode_tc_kernel(const void* __restrict__ q_nope_v, const void* __restrict__ q_pe_v,
                         const void* __restrict__ kv_v, const int32_t* __restrict__ seq_lens,
                         const int32_t* __restrict__ page_table, int Hq, int page_size, int max_pages,
                         float scale_log2, int num_splits, float* __restrict__ part_o, float* __restrict__ part_ml,
                         int q8, float out_scale, int tiles_per_cta, int Q_, int Qg_,
                         const int32_t* __restrict__ topk_idx, const int32_t* __restrict__ req_id, int topk,
                         Dsv4Keys v4) {
  const __nv_bfloat16* q_nope = reinterpret_cast<const __nv_bfloat16*>(q_nope_v);
  const __nv_bfloat16* q_pe = reinterpret_cast<const __nv_bfloat16*>(q_pe_v);
  const __nv_bfloat16* kv = reinterpret_cast<const __nv_bfloat16*>(kv_v);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* k_area = smem;
  uint8_t* q_ring = smem + MLA_K_AREA;
  MlaBars* bars = reinterpret_cast<MlaBars*>(q_ring + MLA_Q_RING);

  const int Q = SPEC ? Q_ : 1, Qg = SPEC ? Qg_ : 1;
  const int split = blockIdx.x, b = blockIdx.z;
  const int part = SPEC ? blockIdx.y % MLA_PARTS : blockIdx.y, qg = SPEC ? blockIdx.y / MLA_PARTS : 0;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int qn = SPEC ? min(Qg, Q - qg * Qg) : 1;   // draft tokens of this q-group
  const int nrows = qn * Hq;                         // MMA rows that carry a query
  const size_t row0 = (size_t)(b * Q + qg * Qg) * Hq;   // q / output row of MMA row 0
  // keys of the group's last draft token: the most any row of this CTA sees (all of them when Q = 1)
  // (SPARSE: the entries of the token's index row; V4: the main entries then the extra ones)
  const int n_main = V4 ? min(max(seq_lens[b], 0), topk) : 0;
  const int S = V4 ? n_main + (v4.extra_idx ? min(max(v4.extra_lens[b], 0), v4.extra_topk) : 0)
                   : SPARSE ? topk : SPEC ? seq_lens[b] - Q + qg * Qg + qn : seq_lens[b];
  const int t_first = split * tiles_per_cta * MLA_TOK;
  // this CTA walks n_tiles consecutive 128-token tiles of the request with an online softmax: O stays in registers,
  // partial (O, m, l) leave the CTA once
  const int n_tiles = min(tiles_per_cta, (S - t_first + MLA_TOK - 1) / MLA_TOK);
  const size_t pbase = row0 * num_splits;

  if (n_tiles <= 0) {
    // empty split: publish (m = -inf, l = 0) for every row of the q-group so that the merge ignores it
    if (part == 0 && tid < nrows) {
      part_ml[(pbase + (size_t)tid * num_splits + split) * 2] = -CUDART_INF_F;
      part_ml[(pbase + (size_t)tid * num_splits + split) * 2 + 1] = 0.f;
    }
    return;
  }

  // V4: no q_pe k-block; kb 7 is the rope block
  constexpr int KB = V4 ? MLA_KB - 1 : MLA_KB, ROPE_KB = KB - 1;
  if (tid == 0) {
    for (int i = 0; i < KB; ++i) mbar_init(&bars->full[i], 128);
    for (int i = 0; i < MLA_QSTAGES; ++i) mbar_init(&bars->empty[i], 2);   // one arrival per consumer warpgroup
    mbar_init(&bars->s_full, 2);
    mbar_init(&bars->o_full, 2);
    if (SPARSE) mbar_init(&bars->v_full, 4);   // one arrival per loader warp
    fence_barrier_init();
  }
  // row r is draft token j = r / Hq of the group (rows past its last token take that token's limit)
  if (SPEC && tid < 128) bars->row_off[tid] = (int8_t)(qn - 1 - min(tid / Hq, qn - 1));
  __syncthreads();
  // k-block order of a tile: the seven (V4: six) blocks the PV MMA of THIS CTA does not read (the other CTAs' value dims and
  // the rope block) come first — they can be refilled as soon as QK^T of the previous tile has completed, the two value
  // blocks only after its PV
  constexpr int MLA_NV = MLA_DV / 64, MLA_NO = KB - MLA_NV;
  auto kb_of = [&](int j) { return j < MLA_NO ? (j < part * MLA_NV ? j : j + MLA_NV) : part * MLA_NV + (j - MLA_NO); };

  if (warp >= 8) {
    // ======================================================================= loaders
    const int lt = tid - 256;                 // 0..127
    const int c = lt & 7;                     // 16-byte chunk within the 128-byte row segment
    const int r0 = lt >> 3;                   // rows r0 + 16u, u = 0..7
    const uint8_t* qn8 = reinterpret_cast<const uint8_t*>(q_nope_v);
    const uint8_t* qp8 = reinterpret_cast<const uint8_t*>(q_pe_v);
    uint32_t qit = 0;                         // q-ring slot counter, continuous over the tiles
    for (int ti = 0; ti < n_tiles; ++ti) {
      const int t0 = t_first + ti * MLA_TOK;
      const int nt = min(MLA_TOK, S - t0);
      // base pointers of this thread's 8 KV rows (paged)
      const __nv_bfloat16* krow[8];
      const uint8_t* krow8[8];
      float kscale[8][4];   // SPARSE && KV8: the row's four fp8_ds_mla scales
      uint2 kue[8];         // V4: the row's scale record, 7 ue8m0 bytes and a pad byte
      uint32_t vword = 0;   // SPARSE: this warp's word of the tile's valid mask
      if (V4) {
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int e = t0 + r0 + 16 * u;   // entry of the concatenated list main || extra
          const bool extra = e >= n_main;
          const int slot = e >= S ? -1 : !extra ? topk_idx[(size_t)b * topk + e]
                                                : v4.extra_idx[(size_t)b * v4.extra_topk + (e - n_main)];
          const int bs = extra ? v4.extra_block : page_size;
          const bool ok = slot >= 0 && (int64_t)slot < (int64_t)(extra ? v4.extra_blocks : max_pages) * bs;
          const uint8_t* blk = reinterpret_cast<const uint8_t*>(extra ? v4.extra_kv : kv_v) +
                               (size_t)(ok ? slot / bs : 0) * (size_t)(extra ? v4.extra_stride : v4.main_stride);
          const int pos = ok ? slot % bs : 0;
          krow8[u] = ok ? blk + (size_t)pos * 576 : nullptr;
          kue[u] = ok ? __ldg(reinterpret_cast<const uint2*>(blk + (size_t)bs * 576 + (size_t)pos * 8)) : make_uint2(0u, 0u);
          const uint32_t bal = __ballot_sync(0xffffffffu, ok);
          vword |= ((bal & 1u) | ((bal >> 7) & 2u) | ((bal >> 14) & 4u) | ((bal >> 21) & 8u)) << (4 * u);
        }
      } else if (SPARSE) {
        const int32_t* pt_row = page_table + (size_t)req_id[b] * max_pages;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int tt = r0 + 16 * u;
          const int idx = tt < nt ? topk_idx[(size_t)b * topk + t0 + tt] : -1;
          const bool ok = idx >= 0 && idx / page_size < max_pages;
          const size_t row = ok ? (size_t)pt_row[idx / page_size] * page_size + idx % page_size : 0;
          krow[u] = ok ? kv + row * 576 : nullptr;
          krow8[u] = ok ? reinterpret_cast<const uint8_t*>(kv_v) + row * 656 : nullptr;
          if (KV8) {
            const float4 sc = ok ? __ldg(reinterpret_cast<const float4*>(krow8[u] + 512)) : make_float4(0.f, 0.f, 0.f, 0.f);
            kscale[u][0] = sc.x;
            kscale[u][1] = sc.y;
            kscale[u][2] = sc.z;
            kscale[u][3] = sc.w;
          }
          // lanes 0, 8, 16, 24 hold rows 4 * (warp - 8) + 0..3 + 16u
          const uint32_t bal = __ballot_sync(0xffffffffu, ok);
          vword |= ((bal & 1u) | ((bal >> 7) & 2u) | ((bal >> 14) & 4u) | ((bal >> 21) & 8u)) << (4 * u);
        }
      } else {
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int tt = r0 + 16 * u;
        if (tt < nt) {
          const int tok = t0 + tt;
          const int page = page_table[(size_t)b * max_pages + tok / page_size];
          krow[u] = kv + ((size_t)page * page_size + tok % page_size) * 576;
          krow8[u] = reinterpret_cast<const uint8_t*>(kv_v) + ((size_t)page * page_size + tok % page_size) * 576;
        } else {
          krow[u] = nullptr;
          krow8[u] = nullptr;
        }
      }
      }
      // KV8: e4m3 cache (and, with q8, e4m3 queries): 8-byte loads, widened to bf16 in registers, 16-byte stores into the
      // swizzled tiles; MLA_PF k-blocks of loads are kept in flight per thread (register ring).  Otherwise every block goes
      // in by cp.async (LDGSTS) straight into the swizzled tiles, with no register staging.
      constexpr int MLA_PF = KV8 ? 3 : 1;
      uint2 kreg[MLA_PF][8], qreg[MLA_PF][8];
      auto issue = [&](int j, int buf) {
        const int kb = kb_of(j);
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int r = r0 + 16 * u;
          // fp8_ds_mla: the rope block (kb 8, V4: kb 7) is bf16 and goes in by cp.async
          kreg[buf][u] = krow8[u] && !(SPARSE && kb == ROPE_KB)
                             ? __ldg(reinterpret_cast<const uint2*>(krow8[u] + kb * 64 + c * 8)) : make_uint2(0u, 0u);
          qreg[buf][u] = make_uint2(0u, 0u);
          if (!SPARSE && q8 && r < nrows)
            qreg[buf][u] = __ldg(reinterpret_cast<const uint2*>(kb < 8 ? qn8 + (row0 + r) * 512 + kb * 64 + c * 8
                                                                         : qp8 + (row0 + r) * 64 + c * 8));
        }
      };
      // one k-block per step, the same sequence for every key source and cache format: wait until the block's previous
      // readers are done, (SPARSE) publish the tile's mask, wait for a q-ring slot, fill q and k, signal full[kb]
      auto step = [&](int j) {
        const int kb = kb_of(j);
        const int s = qit % MLA_QSTAGES, buf = j % MLA_PF;
        if (KV8 && j + MLA_PF - 1 < KB) issue(j + MLA_PF - 1, (j + MLA_PF - 1) % MLA_PF);
        if (ti > 0) mla_wait(j < MLA_NO ? &bars->s_full : &bars->o_full, (ti - 1) & 1);
        if (SPARSE && j == 0 && lane == 0) {   // publish the mask once tile ti - 1's QK^T is done (see v_full)
          bars->kvalid[ti & 1][warp - 8] = vword;
          mbar_arrive(&bars->v_full);
        }
        mla_wait(&bars->empty[s], ((qit / MLA_QSTAGES) & 1) ^ 1);
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int r = r0 + 16 * u;
          if (KV8 && !SPARSE && q8) {
            *reinterpret_cast<uint4*>(q_ring + s * TILE_BYTES + sw128_offset(r, c * 16)) = fp8x8_to_bf16x8(qreg[buf][u]);
          } else {
            const bool qok = r < nrows;
            const __nv_bfloat16* qsrc = !qok ? q_nope
                                             : (kb < 8 ? q_nope + (row0 + r) * 512 + kb * 64 + c * 8
                                                       : q_pe + (row0 + r) * 64 + c * 8);
            cp_async16(q_ring + s * TILE_BYTES + sw128_offset(r, c * 16), qsrc, qok);
          }
          if (!KV8)
            cp_async16(k_area + kb * TILE_BYTES + sw128_offset(r, c * 16), krow[u] ? krow[u] + kb * 64 + c * 8 : kv,
                       krow[u] != nullptr);
          else if (!SPARSE)
            *reinterpret_cast<uint4*>(k_area + kb * TILE_BYTES + sw128_offset(r, c * 16)) = fp8x8_to_bf16x8(kreg[buf][u]);
          else if (kb < ROPE_KB)
            *reinterpret_cast<uint4*>(k_area + kb * TILE_BYTES + sw128_offset(r, c * 16)) =
                fp8x8_scaled_to_bf16x8(kreg[buf][u], V4 ? ue8m0_scale(kue[u], kb) : kscale[u][kb >> 1]);
          else
            cp_async16(k_area + kb * TILE_BYTES + sw128_offset(r, c * 16),
                       krow8[u] ? krow8[u] + (V4 ? 448 : 528) + c * 16 : kv_v, krow8[u] != nullptr);
        }
        if (!KV8) {
          cp_async_mbar_arrive_noinc(&bars->full[kb]);   // arrives when this thread's cp.async writes have landed
        } else {
          if (SPARSE || !q8) asm volatile("cp.async.wait_all;" ::: "memory");
          fence_proxy_async();   // generic-proxy stores -> wgmma (async proxy) reads
          mbar_arrive(&bars->full[kb]);
        }
      };
      // the register ring needs the k-block loop unrolled; the cp.async loop stays rolled
      if (KV8) {
#pragma unroll
        for (int j = 0; j < MLA_PF - 1; ++j) issue(j, j);
#pragma unroll
        for (int j = 0; j < KB; ++j, ++qit) step(j);
      } else {
        for (int j = 0; j < KB; ++j, ++qit) step(j);
      }
    }
  } else {
    // ======================================================================= consumer warpgroups (64 heads each)
    // accumulator fragment (wgmma.cuh): this thread holds rows h0 and h0 + 8, tokens / dims 8j + 2(lane % 4) and + 1
    const int wg = warp >> 2;
    const bool lead = (tid & 127) == 0;
    const int quad = lane & 3;
    const int h0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    float sacc[MLA_TOK / 2], oacc[MLA_DV / 2];
    float m_run[2] = {-CUDART_INF_F, -CUDART_INF_F};   // running row maxima (raw logits)
    float l[2] = {0.f, 0.f};                           // this thread's share of the row sums
    // SPEC: row h0 + 8r sees the keys before S - row_off (its draft token j sees S - (qn - 1 - j) keys); its masked logits
    // are set to -inf right after QK^T, so that no per-row limit stays live through the P loop (the consumers have no
    // registers to spare; for the same reason the offsets are read from shared memory every tile).  The visible keys of a
    // row are a prefix of the sequence, so a row that sees nothing in the CTA's first tile sees nothing in any later one:
    // its m_run stays -inf (the lazy-rescale test compares NaN, which is false), it takes ms = 0 so that every P of it is
    // exp2(-inf) = 0 (exp2f never sees -inf - -inf), and it publishes exactly m = -inf, l = 0, O = 0, which the merges skip.
    // SPARSE: the valid entries of a tile may be anywhere and a fully masked tile may come before a valid one; the masked
    // logits are -inf and the same rules keep a row that has seen no valid key at m_run = -inf, P = 0, l = 0.
    constexpr bool MASKED = SPEC || SPARSE;
    uint32_t qit = 0;
    for (int ti = 0; ti < n_tiles; ++ti) {
      // SPARSE: wait for the tile's mask before the first wgmma of the tile.  The loaders publish the mask of tile ti + 1
      // only after this warpgroup's QK^T of tile ti has completed, which needs every warp of it past this wait, so no
      // warp can see the barrier two phases ahead.
      if (SPARSE) mla_wait(&bars->v_full, ti & 1);
      const int nt = min(MLA_TOK, S - (t_first + ti * MLA_TOK));
      // valid tokens of the tile per row (row h0 + 8r), t < ntr[r]
      const int ntr[2] = {S - (t_first + ti * MLA_TOK) - bars->row_off[h0], S - (t_first + ti * MLA_TOK) - bars->row_off[h0 + 8]};
      // S = Q K^T over the nine (V4: eight) k-blocks, in the order the loaders fill them
      for (int j = 0; j < KB; ++j, ++qit) {
        const int kb = kb_of(j);
        const int s = qit % MLA_QSTAGES;
        mla_wait(&bars->full[kb], ti & 1);
        fence_proxy_async();   // LDGSTS / st.shared (generic proxy) writes -> wgmma (async proxy) reads
        const uint32_t qa = smem_u32(q_ring + s * TILE_BYTES) + wg * 8192;
        const uint32_t ka = smem_u32(k_area + kb * TILE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          WgmmaSS<MLA_TOK, 1>::mma(sacc, wgmma_desc_sw128(qa + ks * 32, 1024), wgmma_desc_sw128(ka + ks * 32, 1024),
                                   (j > 0 || ks > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        if (lead) mbar_arrive(&bars->empty[s]);
      }
      if (lead) mbar_arrive(&bars->s_full);
      if (SPEC) {   // masked logits -> -inf once, so that no per-row limit stays live through the P loop
#pragma unroll
        for (int i = 0; i < MLA_TOK / 2; ++i)
          if ((i >> 2) * 8 + quad * 2 + (i & 1) >= ntr[(i >> 1) & 1]) sacc[i] = -CUDART_INF_F;
      }
      if (SPARSE) {   // column 8k + 2 quad + e is bit 4 (k / 2) + 2 (quad % 2) + e of mask word 2 (k % 2) + quad / 2
        const uint32_t* vm = bars->kvalid[ti & 1];
        const uint32_t v0 = vm[quad >> 1] >> (2 * (quad & 1)), v1 = vm[2 + (quad >> 1)] >> (2 * (quad & 1));
#pragma unroll
        for (int i = 0; i < MLA_TOK / 2; ++i) {
          const int k = i >> 2;
          if (!((((k & 1) ? v1 : v0) >> (4 * (k >> 1) + (i & 1))) & 1u)) sacc[i] = -CUDART_INF_F;
        }
      }
      // row maxima over the valid tokens of the tile: own columns, then the quad
      float m[2] = {-CUDART_INF_F, -CUDART_INF_F};
#pragma unroll
      for (int i = 0; i < MLA_TOK / 2; ++i) {
        const int t = (i >> 2) * 8 + quad * 2 + (i & 1);
        if (MASKED || t < nt) m[(i >> 1) & 1] = fmaxf(m[(i >> 1) & 1], sacc[i]);
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 1));
        m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 2));
      }
      // online softmax with a LAZY rescale: the running maximum moves (and O, l are rescaled) only when the tile's
      // maximum exceeds it by more than 2^8 in the exponent domain; otherwise P = exp2(s - m_run) <= 256 is accumulated as is
      float ms[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        if (ti == 0) {
          m_run[r] = m[r];
        } else if ((m[r] - m_run[r]) * scale_log2 > 8.f) {
          const float factor = exp2f((m_run[r] - m[r]) * scale_log2);
          m_run[r] = m[r];
#pragma unroll
          for (int i = 0; i < MLA_DV / 2; ++i)
            if (((i >> 1) & 1) == r) oacc[i] *= factor;
          l[r] *= factor;
        }
        // SPEC: a row with no visible key so far (m_run = -inf) takes ms = 0, so that its masked logits give
        // exp2(-inf - 0) = 0 and never -inf - -inf
        ms[r] = MASKED && m_run[r] == -CUDART_INF_F ? 0.f : m_run[r] * scale_log2;
      }
      // P = exp2(s*scale - m*scale) -> bf16 pairs: the accumulator fragment of 16 tokens IS the A fragment of a k-step
      uint32_t pa[MLA_TOK / 16][4];
#pragma unroll
      for (int i = 0; i < MLA_TOK / 2; i += 2) {
        const int t = (i >> 2) * 8 + quad * 2, r = (i >> 1) & 1;
        const float p0 = (MASKED || t < nt) ? exp2f(fmaf(sacc[i], scale_log2, -ms[r])) : 0.f;
        const float p1 = (MASKED || t + 1 < nt) ? exp2f(fmaf(sacc[i + 1], scale_log2, -ms[r])) : 0.f;
        const __nv_bfloat162 pb = __floats2bfloat162_rn(p0, p1);
        // accumulate l from the ROUNDED probabilities so that O / l is consistent with the bf16 P used by the MMA
        l[r] += __low2float(pb) + __high2float(pb);
        pa[i >> 3][(i >> 1) & 3] = *reinterpret_cast<const uint32_t*>(&pb);
      }
      // O (+)= P * V: A = P (registers), B = V (MN-major view of this CTA's two value blocks, 16 tokens per k-step)
      const uint32_t va = smem_u32(k_area + (part * MLA_NV) * TILE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k16 = 0; k16 < MLA_TOK / 16; ++k16)
        WgmmaRS<MLA_DV, 1, 1>::mma(oacc, pa[k16], wgmma_desc_sw128_mn(va + k16 * 2048, TILE_BYTES, 1024),
                                   (ti > 0 || k16 > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      if (lead) mbar_arrive(&bars->o_full);
    }
    // epilogue: partial O (un-normalised) + (m, l) in the exp2 domain expected by the merge kernels
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
      const int h = h0 + 8 * r;   // MMA row: q / output row row0 + h
      if (h < nrows) {
        float* po = part_o + (pbase + (size_t)h * num_splits + split) * 512 + part * MLA_DV + quad * 2;
#pragma unroll
        for (int j = 0; j < MLA_DV / 8; ++j)
          *reinterpret_cast<float2*>(po + j * 8) = make_float2(oacc[4 * j + 2 * r] * out_scale, oacc[4 * j + 2 * r + 1] * out_scale);
        if (part == 0 && quad == 0) {
          part_ml[(pbase + (size_t)h * num_splits + split) * 2] = m_run[r] * scale_log2;
          part_ml[(pbase + (size_t)h * num_splits + split) * 2 + 1] = l[r];
        }
      }
    }
  }
}

// each CTA walks ceil(tiles / num_splits) of the ceil(max_keys / 128) key tiles with an online softmax
static int tiles_per_cta(int64_t max_keys, int num_splits) {
  const int tiles = (int)((max_keys + MLA_TOK - 1) / MLA_TOK);
  return (tiles + num_splits - 1) / num_splits;
}
// the tail every MLA-family launch shares: raise the kernel's dynamic shared memory, launch, check
template <class Kern, class... Args>
static int launch_mla(Kern kern, dim3 grid, cudaStream_t st, Args... args) {
  const int rc = kernel_smem(reinterpret_cast<const void*>(kern), MLA_SMEM, "cudaFuncSetAttribute(mla_decode_tc)");
  if (rc) return rc;
  kern<<<grid, MLA_THREADS, MLA_SMEM, st>>>(args...);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "mla_decode_tc launch");
  return 0;
}

int launch_mla_tc(cudaStream_t st, const void* q_nope, const void* q_pe, const void* kv, const int32_t* seq_lens,
                  const int32_t* page_table, int batch, int q_len, int Hq, int page_size, int max_pages, float sm_scale,
                  int num_splits, float* part_o, float* part_ml, int kv_fp8, int q_fp8, float descale_q, float descale_k) {
  if (q_fp8 && !kv_fp8) {
    set_error("b200_mla_decode: e4m3 queries need the e4m3 cache");
    return B200_ERR_INVALID;
  }
  // draft tokens per q-group (as many as fill the 128 MMA rows), q-groups; the q-group varies with the part in grid.y
  const int Qg = min(q_len, 128 / Hq), n_qg = (q_len + Qg - 1) / Qg;
  dim3 grid(num_splits, MLA_PARTS * n_qg, batch);
  // the splits together cover the page table
  const int tpc = tiles_per_cta((int64_t)max_pages * page_size, num_splits);
  // descales (reference cutlass_mla.py: q_scale * k_scale folded into the softmax scale, k_scale into the output)
  const float sl2 = sm_scale * 1.4426950408889634f * (kv_fp8 ? descale_k * (q_fp8 ? descale_q : 1.f) : 1.f);
  const float osc = kv_fp8 ? descale_k : 1.f;
  auto kern = q_len == 1 ? (!kv_fp8 ? mla_decode_tc_kernel<false, false, false, false>
                                    : mla_decode_tc_kernel<true, false, false, false>)
                         : (!kv_fp8 ? mla_decode_tc_kernel<false, true, false, false>
                                    : mla_decode_tc_kernel<true, true, false, false>);
  return launch_mla(kern, grid, st, q_nope, q_pe, kv, seq_lens, page_table, Hq, page_size, max_pages, sl2, num_splits, part_o,
                    part_ml, kv_fp8 ? q_fp8 : 0, kv_fp8 ? osc : 1.f, tpc, q_len, Qg, nullptr, nullptr, 0, Dsv4Keys{});
}

// sparse decode: one CTA row (grid.z) per query token; kv_ds_mla selects the fp8_ds_mla cache
int launch_mla_sparse_tc(cudaStream_t st, const void* q_nope, const void* q_pe, const void* kv, int kv_ds_mla,
                         const int32_t* topk_idx, int topk, const int32_t* req_id, const int32_t* page_table, int max_pages,
                         int num_tokens, int Hq, int page_size, float sm_scale, int num_splits, float* part_o,
                         float* part_ml) {
  dim3 grid(num_splits, MLA_PARTS, num_tokens);
  const float sl2 = sm_scale * 1.4426950408889634f;
  auto kern = kv_ds_mla ? mla_decode_tc_kernel<true, false, true, false> : mla_decode_tc_kernel<false, false, true, false>;
  return launch_mla(kern, grid, st, q_nope, q_pe, kv, nullptr, page_table, Hq, page_size, max_pages, sl2, num_splits, part_o,
                    part_ml, 0, 1.f, tiles_per_cta(topk, num_splits), 1, 1, topk_idx, req_id, topk, Dsv4Keys{});
}

// DeepSeek-V4 sparse decode: one CTA row (grid.z) per query token over the concatenated main || extra list
int launch_dsv4_sparse_tc(cudaStream_t st, const void* q, const void* swa_kv, int swa_block, int swa_blocks,
                          int64_t swa_stride, const int32_t* swa_idx, int swa_topk, const int32_t* swa_lens,
                          const void* extra_kv, int extra_block, int extra_blocks, int64_t extra_stride,
                          const int32_t* extra_idx, int extra_topk, const int32_t* extra_lens, int num_tokens, int Hq,
                          float sm_scale, int num_splits, float* part_o, float* part_ml) {
  dim3 grid(num_splits, MLA_PARTS, num_tokens);
  const int tpc = tiles_per_cta(swa_topk + (extra_idx ? extra_topk : 0), num_splits);
  const float sl2 = sm_scale * 1.4426950408889634f;
  const Dsv4Keys v4{extra_kv, extra_idx, extra_lens, extra_topk, extra_block, extra_blocks, swa_stride, extra_stride};
  return launch_mla(mla_decode_tc_kernel<true, false, true, true>, grid, st, q, q, swa_kv, swa_lens, nullptr, Hq, swa_block,
                    swa_blocks, sl2, num_splits, part_o, part_ml, 0, 1.f, tpc, 1, 1, swa_idx, nullptr, swa_topk, v4);
}

}  // namespace b200
