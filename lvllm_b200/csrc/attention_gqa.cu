// Paged GQA decode on wgmma tensor cores (head_dim 128), persistent CTAs, multi-stage KV pipeline.
//
// Work item = (request b, kv head, q-group, 128-token split).  The kernel is KV-bandwidth bound, so the tiles are laid
// out to make every thread useful: tokens are the M rows of the MMAs and the G = Hq/Hkv query heads sharing the
// kv head are the N columns (N = G rounded up to 16).
// Speculative decode: a request has Q query tokens (its last Q positions, in draft order); query token i sees keys
// [0, S_b - Q + i] (end-aligned causal mask).  A q-group holds Qg = min(Q, 32 / G) of them: column c of the item is
// (draft token qg * Qg + c / G, head c % G), N = G * Qg rounded up to 16, so while G * Q <= 32 K and V are read once per
// request; beyond that every q-group reads them again.  Q = 1 is the single-token decode (one q-group, columns = heads).
// The MMAs below, per item:
//   S^T[128 tokens, N]  = K[128 tokens, 128 dims] . Q^T           (A = K tile, K-major; B = Q rows, K-major)
//   P^T = exp2(S^T * scale - m)                                    (thread = token; m via warp shuffles)
//   O^T[128 dims, N]    = V^T[128 dims, 128 tokens] . P^T          (A = V tile read MN-major; B = P rows, K-major)
//   L[128, N]           = 1[128, 128 tokens] . P^T                 (row sums of P on the tensor core: every
//                                                                   epilogue thread reads l[h] from its own lane)
// K and V tiles are gathered with cp.async straight into 128B-swizzled [64-dim block][128 tokens][128 B] blocks; a row is
// found through (page, slot, head) strides, so the K / V halves of a packed NHD / HND cache are read in place.
// Two rings let the loaders run ahead of the MMAs: NK stages of (Q, K), each freed as soon as QK^T of its item has
// completed, and NV stages of V, each freed after PV of its item (which waits for the item's softmax).  Splitting them
// keeps K from sitting in shared memory through the softmax, so the freed space carries the next item's K early.  The
// accumulators cross from the MMA warpgroup to the softmax / epilogue threads through the exchange area (common.cuh),
// S^T double-buffered so that QK^T of item n+1 overlaps softmax of item n.  Softmax and epilogue stop at the item's
// real columns (ncols <= N, in runs of 4); the P tiles are zeroed once, so the columns they skip feed PV finite values
// that reach only O / L columns nobody reads.  Partial (O, m, l) per split are merged by attn_merge_kernel.
// Reference semantics: tests/kernels/attention/test_flashinfer.py:29-80 (ref_paged_attn, decode case).
// Roofline: HBM — algorithmic bytes = sum_b S_b * Hkv * 128 * 2 (K and V) * 2 B * n_qg (n_qg = ceil(Q / Qg) q-groups).
#include <math_constants.h>
#include <stdio.h>

#include "common.cuh"
#include "moe_internal.cuh"

namespace b200 {

constexpr int GQA_TOK = 128;
constexpr int GQA_THREADS = 512;          // warps 0-3 / 4-7: softmax+epilogue groups, 8-11 loaders, 12-15 MMA warpgroup
constexpr int GQA_MAX_STAGES = 3;         // per ring
constexpr int GQA_MIN_STAGES = 2;         // per ring: the MMA warpgroup issues QK of item n + 1 before PV of item n
constexpr int GQA_V_STAGES = 2;           // V stages: the rest of shared memory goes to (Q, K) stages
constexpr int GQA_SMEM_MAX = 232448;
constexpr int GQA_MAX_ITEMS = 1024;       // items per CTA the token-count table holds
constexpr int GQA_MAX_N = 32;             // query heads per kv head (rounded up to 16) that leave two stages per ring: the exchange area
                                          // (512 B per head and group), the P tiles and the Q rows of a (Q, K) stage grow with it

struct GqaBars {
  uint64_t qk_full[GQA_MAX_STAGES], k_free[GQA_MAX_STAGES], v_full[GQA_MAX_STAGES], v_free[GQA_MAX_STAGES];
  uint64_t s_full[2], p_full[2], o_full[2], o_done[2];
  float lsum[2][GQA_MAX_N];        // row sums of P per head (the rows of L are all the same: one is kept)
  alignas(16) float wmax[2][4][GQA_MAX_N];
  int16_t nt_tab[GQA_MAX_ITEMS];   // valid tokens of this CTA's i-th item (<= 0: empty split): those of its last column
  int16_t vis_tab[GQA_MAX_ITEMS];  // v of the i-th item: local draft token j of the q-group sees split tokens t <= v + j
                                   // (clamped to [-32, 128], which keeps every mask the same)
  int col_row[GQA_MAX_N];          // output row of column c relative to the item's first: (c / G) * Hq + c % G
};

// intra-CTA mbarrier wait (producer / MMA / softmax warps of ONE CTA: no other CTA or GPU is waited for).  A protocol bug
// must not hang the box: back off after a while, trap after seconds.
B200_DEVICE void gqa_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 20)) __nanosleep(128);
    if (spins > (1u << 26)) __trap();
  }
}
B200_DEVICE float ex2_approx(float v) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
  return r;
}
B200_DEVICE void bar_sync_group(int g) { asm volatile("bar.sync %0, 128;" ::"r"(g + 1) : "memory"); }

// SPEC: Q > 1 query tokens per request.  Without it every q-group expression below is a compile-time constant (Q = Qg = 1,
// columns = heads), which keeps the single-token decode free of the per-column bookkeeping.
// smem: [ones 1 KB][P group 0 | P group 1: 2 x N x 128 B each][(Q (2 x N x 128 B) | K 32 KB) x NK][V 32 KB x NV]
//       [exchange: 2 groups x N columns x 512 B][bars]
template <int N, bool SPEC>
__global__ void __launch_bounds__(GQA_THREADS, 1)
    gqa_decode_tc_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ kc,
                         const __nv_bfloat16* __restrict__ vc, const int32_t* __restrict__ seq_lens,
                         int64_t block_stride, int64_t page_stride, int64_t head_stride,
                         const int32_t* __restrict__ page_table, int B, int Hq, int Hkv, int page_size, int max_pages,
                         float scale_log2, int num_splits, int Q_, int Qg_, int NK, int NV, float* __restrict__ part_o,
                         float* __restrict__ part_ml) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int qbytes = N * 128;                       // one 64-dim block of the Q (or P) rows
  const int pbytes = (2 * qbytes + 1023) & ~1023;   // one group's P tile
  const int kstage_bytes = 2 * qbytes + 2 * TILE_BYTES;
  uint8_t* ones = smem;
  uint8_t* p_base = smem + 1024;
  uint8_t* kstages = p_base + 2 * pbytes;
  uint8_t* vstages = kstages + (size_t)NK * kstage_bytes;
  uint8_t* xch_area = vstages + (size_t)NV * 2 * TILE_BYTES;
  GqaBars* bars = reinterpret_cast<GqaBars*>(xch_area + 2 * N * 512);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int G = Hq / Hkv;
  const int Q = SPEC ? Q_ : 1, Qg = SPEC ? Qg_ : 1;
  const int n_qg = SPEC ? (Q + Qg - 1) / Qg : 1;
  const int total = B * Hkv * n_qg * num_splits;
  // item = ((b * Hkv + kvh) * n_qg + qg) * num_splits + split; its rows (b * Q + qg * Qg + c / G, kvh * G + c % G) start at
  // row0 = (b * Q + qg * Qg) * Hq + kvh * G and it has ncols = G * (number of draft tokens of the q-group) columns

  if (tid == 0) {
    for (int i = 0; i < GQA_MAX_STAGES; ++i) {
      mbar_init(&bars->qk_full[i], 128);
      mbar_init(&bars->k_free[i], 1);
      mbar_init(&bars->v_full[i], 128);
      mbar_init(&bars->v_free[i], 1);
    }
    for (int g = 0; g < 2; ++g) {
      mbar_init(&bars->s_full[g], 128);   // every MMA thread, after parking its fragment
      mbar_init(&bars->p_full[g], 128);
      mbar_init(&bars->o_full[g], 128);
      mbar_init(&bars->o_done[g], 128);   // the epilogue threads of the group have read O^T
    }
    fence_barrier_init();
  }
  const int my_items = blockIdx.x < total ? (total - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  for (int i = tid; i < my_items; i += GQA_THREADS) {
    const int item = blockIdx.x + i * gridDim.x;
    const int rest = item / num_splits, qg = rest % n_qg;
    const int qn = min(Qg, Q - qg * Qg);
    const int v = seq_lens[rest / (n_qg * Hkv)] - Q + qg * Qg - (item % num_splits) * GQA_TOK;
    bars->nt_tab[i] = (int16_t)max(0, min(GQA_TOK, v + qn));
    if (SPEC) bars->vis_tab[i] = (int16_t)max(-32, min(GQA_TOK, v));
  }
  if (SPEC && tid < GQA_MAX_N) bars->col_row[tid] = (tid / G) * Hq + tid % G;
  auto col_row = [&](int c) { return SPEC ? bars->col_row[c] : c; };
  if (tid < 64) reinterpret_cast<uint4*>(ones)[tid] = make_uint4(0x3F803F80u, 0x3F803F80u, 0x3F803F80u, 0x3F803F80u);
  for (int i = tid; i < 2 * pbytes / 16; i += GQA_THREADS) reinterpret_cast<uint4*>(p_base)[i] = make_uint4(0u, 0u, 0u, 0u);
  fence_proxy_async();
  __syncthreads();
  // group g owns columns [N*g, N*g + N): S^T of an item until its softmax has written P, then O^T of the same item
  const uint32_t tm = xch_base(xch_area);

  if (warp >= 8 && warp < 12) {
    // ======================================================================= loaders
    const int lt = tid - 256, c = lt & 7, r0 = lt >> 3;
    // page-table entries are looked up one item ahead so that their latency is off the issue path
    int pg[8], pg_next[8];
    auto lookup = [&](int i, int* out) {
      if (i >= my_items) return;
      const int item = blockIdx.x + i * gridDim.x;
      const int split = item % num_splits, b = item / (num_splits * n_qg * Hkv);
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int pi = min((split * GQA_TOK + r0 + 16 * u) / page_size, max_pages - 1);
        out[u] = page_table[(size_t)b * max_pages + pi];
      }
    };
    lookup(0, pg);
    uint32_t n = 0;
    for (int i = 0; i < my_items; ++i) {
      lookup(i + 1, pg_next);
      const int nt = bars->nt_tab[i];
      if (nt > 0) {
        const int item = blockIdx.x + i * gridDim.x;
        const int split = item % num_splits, rest = item / num_splits, qg = rest % n_qg, kvh = (rest / n_qg) % Hkv,
                  b = rest / (n_qg * Hkv);
        const int ncols = SPEC ? G * min(Qg, Q - qg * Qg) : G;
        const __nv_bfloat16* qrow0 = q + ((size_t)(b * Q + qg * Qg) * Hq + kvh * G) * 128 + c * 8;
        const int sk = n % NK, sv = n % NV;
        uint8_t* q_t = kstages + (size_t)sk * kstage_bytes;
        uint8_t* k_t = q_t + 2 * qbytes;
        uint8_t* v_t = vstages + (size_t)sv * 2 * TILE_BYTES;
        gqa_wait(&bars->k_free[sk], ((n / NK) & 1) ^ 1);
        for (int r = r0; r < N; r += 16) {
          const bool qok = r < ncols;
          const __nv_bfloat16* src = qrow0 + (size_t)(qok ? col_row(r) : 0) * 128;
          cp_async16(q_t + sw128_offset(r, c * 16), src, qok);
          cp_async16(q_t + qbytes + sw128_offset(r, c * 16), src + 64, qok);
        }
        int64_t rowoff[8];   // cache element offsets (strides in elements: packed K|V views or separate caches)
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int tok = split * GQA_TOK + r0 + 16 * u;
          rowoff[u] = pg[u] * block_stride + (tok % page_size) * page_stride + kvh * head_stride + c * 8;
        }
#pragma unroll
        for (int kb = 0; kb < 2; ++kb) {
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const bool ok = r0 + 16 * u < nt;
            cp_async16(k_t + kb * TILE_BYTES + sw128_offset(r0 + 16 * u, c * 16), ok ? kc + rowoff[u] + kb * 64 : kc, ok);
          }
        }
        cp_async_mbar_arrive_noinc(&bars->qk_full[sk]);
        gqa_wait(&bars->v_free[sv], ((n / NV) & 1) ^ 1);
#pragma unroll
        for (int kb = 0; kb < 2; ++kb) {
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const bool ok = r0 + 16 * u < nt;
            cp_async16(v_t + kb * TILE_BYTES + sw128_offset(r0 + 16 * u, c * 16), ok ? vc + rowoff[u] + kb * 64 : vc, ok);
          }
        }
        cp_async_mbar_arrive_noinc(&bars->v_full[sv]);
        ++n;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) pg[u] = pg_next[u];
    }
  } else if (warp >= 12) {
    // ======================================================================= MMA warpgroup
    const bool lead = tid == 12 * 32;
    const uint32_t oa = smem_u32(ones);
    auto issue_qk = [&](uint32_t n) {
      const int s = n % NK, g = n & 1;
      gqa_wait(&bars->qk_full[s], (n / NK) & 1);
      fence_proxy_async();   // LDGSTS (generic proxy) writes -> wgmma (async proxy) reads
      const uint32_t qa = smem_u32(kstages + (size_t)s * kstage_bytes), ka = qa + 2 * qbytes;
      float sacc[2][N / 2];                                               // A = K (K-major), B = Q (K-major)
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < 2; ++kb)
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          wgmma_tile128<N, 1>(sacc, ka + kb * TILE_BYTES + ks * 32, qa + kb * qbytes + ks * 32, (kb > 0 || ks > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      if (lead) mbar_arrive(&bars->k_free[s]);
      // the columns still hold O^T of the group's previous item until its epilogue has read them (its PV was issued
      // before this QK, so the wait cannot block the MMAs it depends on)
      if (n >= 2) gqa_wait(&bars->o_done[g], ((n >> 1) - 1) & 1);
      xch_store_frag<N>(tm + g * N, 0, sacc[0]);
      xch_store_frag<N>(tm + g * N, 1, sacc[1]);
      mbar_arrive(&bars->s_full[g]);
    };
    auto issue_pv = [&](uint32_t n) {
      const int s = n % NV, g = n & 1;
      gqa_wait(&bars->p_full[g], (n >> 1) & 1);
      gqa_wait(&bars->v_full[s], (n / NV) & 1);
      fence_proxy_async();
      const uint32_t va = smem_u32(vstages + (size_t)s * 2 * TILE_BYTES);
      const uint32_t pa = smem_u32(p_base + g * pbytes);
      float oacc[2][N / 2], lacc[N / 2];   // the rows of L are all the same: one 64-row half serves both
      wgmma_fence();
#pragma unroll
      for (int k16 = 0; k16 < GQA_TOK / 16; ++k16) {
        const uint64_t pd = wgmma_desc_sw128(pa + (k16 >> 2) * qbytes + (k16 & 3) * 32, 1024);
#pragma unroll
        for (int h = 0; h < 2; ++h)   // A = V read MN-major: 64-dim block h, 16 tokens (2 KB) per k-step
          WgmmaSS<N, 1, 1, 0>::mma(oacc[h], wgmma_desc_sw128_mn(va + h * TILE_BYTES + k16 * 2048, TILE_BYTES, 1024), pd,
                                   k16 > 0 ? 1u : 0u);
        WgmmaSS<N, 1, 0, 0>::mma(lacc, wgmma_desc_sw128(oa + (k16 & 3) * 32, 0), pd, k16 > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (lead) mbar_arrive(&bars->v_free[s]);
      // p_full was waited for above: the group's softmax is done with S^T, O^T takes its place
#pragma unroll
      for (int h = 0; h < 2; ++h) xch_store_frag<N>(tm + g * N, h, oacc[h]);
      if ((tid & 127) < 4) {   // row 0 of the fragment: columns 8j + 2 * lane, + 1
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
          bars->lsum[g][j * 8 + lane * 2] = lacc[4 * j];
          bars->lsum[g][j * 8 + lane * 2 + 1] = lacc[4 * j + 1];
        }
      }
      mbar_arrive(&bars->o_full[g]);
    };
    // order: QK(0), QK(1), PV(0), QK(2), PV(1), ...  — item n belongs to softmax group n & 1
    uint32_t issued = 0;
    for (int i = 0; i < my_items; ++i) {
      if (bars->nt_tab[i] <= 0) continue;
      issue_qk(issued++);
      if (issued > 1) issue_pv(issued - 2);
    }
    if (issued > 0) issue_pv(issued - 1);
  } else if (warp < 8) {
    // ======================================================================= softmax (thread = token) + epilogue (thread = dim)
    const int g = warp >> 2, t = tid & 127;
    const uint32_t lane_off = (uint32_t)((warp & 3) * 32) << 16;
    const uint32_t tm_s = tm + g * N + lane_off, tm_o = tm_s;
    uint8_t* prow = p_base + g * pbytes + (t >> 6) * qbytes;
    const uint32_t boff = (t & 63) * 2, bch = boff >> 4, blo = boff & 15;
    float(*wmax)[GQA_MAX_N] = bars->wmax[g];
    uint32_t n = 0;
    for (int i = 0; i < my_items; ++i) {
      const int nt = bars->nt_tab[i];
      const int item = blockIdx.x + i * gridDim.x;
      const int split = item % num_splits, rest = item / num_splits, qg = rest % n_qg, kvh = (rest / n_qg) % Hkv,
                b = rest / (n_qg * Hkv);
      const int ncols = SPEC ? G * min(Qg, Q - qg * Qg) : G;
      const size_t pbase = ((size_t)(b * Q + qg * Qg) * Hq + kvh * G) * num_splits + split;   // + col_row[c] * num_splits
      if (nt <= 0) {
        if (g == 0 && t < ncols) {
          const size_t r = pbase + (size_t)col_row(t) * num_splits;
          part_ml[r * 2] = -CUDART_INF_F;
          part_ml[r * 2 + 1] = 0.f;
        }
        continue;
      }
      if ((int)(n & 1) != g) {
        ++n;
        continue;
      }
      const uint32_t ph = (n >> 1) & 1;
      // token t is visible to the columns c >= cmin (those of draft tokens j >= t - v); t >= nt: to none of the item's
      const int cmin = SPEC ? max(t - bars->vis_tab[i], 0) * G : 0;
      const bool tv = t < nt;
      gqa_wait(&bars->s_full[g], ph);
      float my_ms = 0.f;                          // thread t == h keeps m[h] * scale for the partial record
      // columns >= ncols (zero Q rows) are skipped in runs of 4, which keeps 4 columns of shuffles and ex2 in flight
      // (the columns of a run past ncols compute finite values nobody reads).  ncols is the same for every thread of the
      // CTA, so the group's barriers stay matched.  The blocks of 16 columns: one at N = 16, a loop of compile-time
      // length; at N = 32 a loop over the blocks that hold real columns (unrolled over both, it ran slower).
      const int cend = N == 16 ? 16 : ncols;
      for (int c0 = 0; c0 < cend; c0 += 16) {
        float v[16];
        __syncwarp();
        xch_ld<16>(tm_s + c0, v);
#pragma unroll
        for (int j4 = 0; j4 < 16; j4 += 4) {
          if (c0 + j4 >= ncols) break;
#pragma unroll
          for (int j = j4; j < j4 + 4; ++j) {
            v[j] = (SPEC ? c0 + j >= cmin : tv) ? v[j] : -CUDART_INF_F;
            const float wm = warp_max(v[j]);
            if (lane == j) wmax[warp & 3][c0 + j] = wm;
          }
        }
        bar_sync_group(g);
        float m[16];
#pragma unroll
        for (int j4 = 0; j4 < 16; j4 += 4) {
          const float4 a = *reinterpret_cast<const float4*>(&wmax[0][c0 + j4]);
          const float4 bq = *reinterpret_cast<const float4*>(&wmax[1][c0 + j4]);
          const float4 cq = *reinterpret_cast<const float4*>(&wmax[2][c0 + j4]);
          const float4 d = *reinterpret_cast<const float4*>(&wmax[3][c0 + j4]);
          m[j4 + 0] = fmaxf(fmaxf(a.x, bq.x), fmaxf(cq.x, d.x));
          m[j4 + 1] = fmaxf(fmaxf(a.y, bq.y), fmaxf(cq.y, d.y));
          m[j4 + 2] = fmaxf(fmaxf(a.z, bq.z), fmaxf(cq.z, d.z));
          m[j4 + 3] = fmaxf(fmaxf(a.w, bq.w), fmaxf(cq.w, d.w));
        }
        uint8_t* pr = prow + (c0 >> 3) * 1024;
#pragma unroll
        for (int j4 = 0; j4 < 16; j4 += 4) {
          if (c0 + j4 >= ncols) break;
#pragma unroll
          for (int j = j4; j < j4 + 4; ++j) {
            const float ms = m[j] * scale_log2;
            my_ms = (t == c0 + j) ? ms : my_ms;
            // masked tokens: ex2(-inf) = 0; a column with no visible token in this split (m = -inf) gets P = 0, l = 0
            // and records m = -inf, which the merge skips
            const float p = SPEC && m[j] == -CUDART_INF_F ? 0.f : ex2_approx(fmaf(v[j], scale_log2, -ms));
            *reinterpret_cast<__nv_bfloat16*>(pr + (j >> 3) * 1024 + (j & 7) * 128 + ((bch ^ (j & 7)) << 4) + blo) =
                __float2bfloat16_rn(p);
          }
        }
        if (c0 + 16 < ncols) bar_sync_group(g);   // wmax is reused by the next 16 heads
      }
      fence_proxy_async();
      mbar_arrive(&bars->p_full[g]);
      gqa_wait(&bars->o_full[g], ph);
      // epilogue: thread = value dim d, columns = heads
      float* po = part_o + pbase * 128 + t;
      const size_t hstride = (size_t)num_splits * 128;
      for (int c0 = 0; c0 < cend; c0 += 16) {
        float o[16];
        __syncwarp();
        xch_ld<16>(tm_o + c0, o);
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (c0 + j < ncols) po[(size_t)col_row(c0 + j) * hstride] = o[j];
      }
      if (t < ncols) {
        const size_t r = pbase + (size_t)col_row(t) * num_splits;
        part_ml[r * 2] = my_ms;
        part_ml[r * 2 + 1] = bars->lsum[g][t];
      }
      mbar_arrive(&bars->o_done[g]);   // the group's columns and row sums may be overwritten
      ++n;
    }
  }
}

// merge of the split partials: one CTA per (b, head), DV/4 threads (thread = float4 of the output row)
template <int DV>
__global__ void __launch_bounds__(DV / 4) attn_merge_kernel(const float* __restrict__ part_o,
                                                           const float* __restrict__ part_ml, int num_splits,
                                                           __nv_bfloat16* __restrict__ out, float* __restrict__ lse) {
  constexpr int NT = DV / 4;
  __shared__ float wgt[1024];
  __shared__ float red[NT / 32 > 0 ? NT / 32 : 1];
  const int w = blockIdx.x, tid = threadIdx.x;
  const float* ml = part_ml + (size_t)w * num_splits * 2;
  float mx = -CUDART_INF_F;
  for (int s = tid; s < num_splits; s += NT) mx = fmaxf(mx, ml[s * 2]);
  mx = warp_max(mx);
  if ((tid & 31) == 0) red[tid >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < NT / 32; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float ls = 0.f;
  for (int s = tid; s < num_splits; s += NT) {
    const float msv = ml[s * 2];
    const float f = (msv == -CUDART_INF_F) ? 0.f : exp2f(msv - mx);
    wgt[s] = f;
    ls += f * ml[s * 2 + 1];
  }
  ls = warp_sum(ls);
  if ((tid & 31) == 0) red[tid >> 5] = ls;
  __syncthreads();
  float lsum = 0.f;
  for (int i = 0; i < NT / 32; ++i) lsum += red[i];
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  const float* po = part_o + (size_t)w * num_splits * DV + tid * 4;
  for (int s0 = 0; s0 < num_splits; s0 += 8) {
    float4 v[8];
    float f[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int s = s0 + u;
      f[u] = (s < num_splits) ? wgt[s] : 0.f;
      v[u] = (f[u] != 0.f) ? *reinterpret_cast<const float4*>(po + (size_t)s * DV) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      acc.x = fmaf(f[u], v[u].x, acc.x);
      acc.y = fmaf(f[u], v[u].y, acc.y);
      acc.z = fmaf(f[u], v[u].z, acc.z);
      acc.w = fmaf(f[u], v[u].w, acc.w);
    }
  }
  const float inv = lsum > 0.f ? 1.f / lsum : 0.f;
  __nv_bfloat162 a = __floats2bfloat162_rn(acc.x * inv, acc.y * inv), c = __floats2bfloat162_rn(acc.z * inv, acc.w * inv);
  uint2 pk;
  pk.x = *reinterpret_cast<uint32_t*>(&a);
  pk.y = *reinterpret_cast<uint32_t*>(&c);
  *reinterpret_cast<uint2*>(out + (size_t)w * DV + tid * 4) = pk;
  if (lse && tid == 0) lse[w] = (lsum > 0.f) ? (mx * 0.6931471805599453f + logf(lsum)) : -CUDART_INF_F;
}

int launch_gqa_tc(cudaStream_t st, const void* q, const void* kc, const void* vc, int64_t block_stride, int64_t page_stride,
                  int64_t head_stride, const int32_t* seq_lens, const int32_t* page_table, int batch, int q_len, int Hq,
                  int Hkv, int page_size, int max_pages, float sm_scale, int num_splits, float* part_o, float* part_ml,
                  void* out, float* lse) {
  const int G = Hq / Hkv;
  if (G > GQA_MAX_N) return 1;   // not handled here
  const int Qg = min(q_len, GQA_MAX_N / G), n_qg = (q_len + Qg - 1) / Qg;   // draft tokens per q-group, q-groups
  const int N = (G * Qg + 15) / 16 * 16;
  const int qbytes = N * 128;
  const int fixed = 1024 /*align*/ + 1024 /*ones*/ + 2 * ((2 * qbytes + 1023) & ~1023) + 2 * N * 512 /*exchange*/ +
                    (int)sizeof(GqaBars) + 64;
  const int kstage_bytes = 2 * qbytes + 2 * TILE_BYTES, vstage_bytes = 2 * TILE_BYTES;
  // GQA_V_STAGES of V (a V stage is held through the softmax of its item), as many (Q, K) stages as the rest holds
  const int nv = GQA_V_STAGES;
  const int nk = min(GQA_MAX_STAGES, (GQA_SMEM_MAX - fixed - nv * vstage_bytes) / kstage_bytes);
  static_assert(GQA_MIN_STAGES <= GQA_V_STAGES && GQA_V_STAGES <= GQA_MAX_STAGES, "gqa_decode_tc: V ring size");
  static_assert((GQA_SMEM_MAX - (2048 + 4 * GQA_MAX_N * 128 + 2 * GQA_MAX_N * 512 + (int)sizeof(GqaBars) + 64) -
                 GQA_V_STAGES * 2 * TILE_BYTES) / (2 * GQA_MAX_N * 128 + 2 * TILE_BYTES) >= GQA_MIN_STAGES,
                "gqa_decode_tc: two (Q, K) stages at the largest group");
  if (nk < GQA_MIN_STAGES) {
    set_error("gqa_decode_tc: group size does not fit shared memory");
    return B200_ERR_INVALID;
  }
  const int smem = fixed + nk * kstage_bytes + nv * vstage_bytes;
  int dev = 0;
  if (const cudaError_t e = cudaGetDevice(&dev); e != cudaSuccess) return cuda_fail(e, "cudaGetDevice");
  const int num_sms = device_sms(dev);
  if (num_sms < 0) return num_sms;
  const int total = batch * Hkv * n_qg * num_splits;
  const int grid = total < num_sms ? total : num_sms;
  if ((total + grid - 1) / grid > GQA_MAX_ITEMS) return 1;   // not handled here: caller uses the split-KV CUDA-core path
  auto kern = q_len == 1 ? (N == 16 ? gqa_decode_tc_kernel<16, false> : gqa_decode_tc_kernel<32, false>)
                         : (N == 16 ? gqa_decode_tc_kernel<16, true> : gqa_decode_tc_kernel<32, true>);
  const int rc = kernel_smem(reinterpret_cast<const void*>(kern), GQA_SMEM_MAX, "cudaFuncSetAttribute(gqa_decode_tc)");
  if (rc) return rc;
  kern<<<grid, GQA_THREADS, smem, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(kc),
      reinterpret_cast<const __nv_bfloat16*>(vc), seq_lens, block_stride, page_stride, head_stride, page_table, batch, Hq, Hkv, page_size, max_pages,
      sm_scale * 1.4426950408889634f, num_splits, q_len, Qg, nk, nv, part_o, part_ml);
  attn_merge_kernel<128><<<batch * q_len * Hq, 32, 0, st>>>(part_o, part_ml, num_splits, reinterpret_cast<__nv_bfloat16*>(out), lse);
  g_launches += 2;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "gqa_decode_tc launch");
  return 0;
}

}  // namespace b200
