// Fused decode MoE layer on sm_90a: ONE persistent kernel per layer.
//
//   phase 0  every CTA rebuilds the (tiny) routing table in shared memory — stable counting sort of the
//            (token,k) slots by expert, padded permuted rows, chunk table — and the CTAs share the row
//            gather (+ per-token-group-128 FP8 quantisation) into the swizzled tile layout;
//   phase 1  GEMM1 (w13, gate+up) + SiLU*mul (+ FP8 requantisation) -> tiled intermediate;
//   phase 2  GEMM2 (w2) -> y, then the LAST finisher of every 128-column output tile reduces
//            out[t] = sum_j w[t,j] * y[row(t,j)] in fixed j order (deterministic, no atomics on data).
//
// Both GEMMs are STREAM-K: the linearised (tile, k-iteration) space of a phase is cut into one equal
// contiguous range per SM (132), so every SM streams the same share of the weight bytes whatever the number of active
// experts (1 expert per GPU under EP8 still uses every SM).  A tile split across CTAs is fixed up by the
// last contributor (partials in a small workspace, summed in fixed CTA order -> bit-reproducible).
// Cross-CTA dependencies (rows ready, GEMM1 of a chunk done, contributors of a tile, finishers of an output
// tile) are generation-tagged counters in global memory: nothing is zeroed between launches, the kernel is
// CUDA-graph replayable, and all CTAs are co-resident (1 CTA/SM) so spinning is deadlock-free.
//
// Inside a CTA the pipeline is the same as moe_gemm.cu: producer warp (bulk async copies, A and B of a stage
// are ONE copy each), MMA warpgroup (wgmma, register accumulators parked in the exchange area of common.cuh), 4 drain
// warps (FP8 block-scale promotion, activation, stores).  The producer runs ahead across phase boundaries: weight tiles are
// requested as soon as a ring slot frees up, the dependent B operand is requested when its flag is up.
// 4-bit layers (W4A16) have two consumer warpgroups instead of the MMA warpgroup: each converts the raw nibbles of its
// 64 weight rows straight from the stage into wgmma A fragments (registers) and multiplies them with the token tile
// (shared memory); a chunk holds up to 64 rows of one expert, so a decode batch streams each active expert once.
//
// Roofline: HBM.  Algorithmic bytes per launch = weight bytes of the distinct active experts.
#include <cstdio>
#include <cstdlib>

#include "common.cuh"
#include "moe_internal.cuh"
#include "w4_layout.cuh"

namespace b200 {

constexpr int F_SCG = 32;           // k-blocks of scales staged in shared memory at a time
constexpr int F_QD = 4;             // drain -> fix-up hand-over queue depth
constexpr int F_EPI_WARPS = 4;
constexpr int F_SMEM_BUDGET = 226 * 1024;

struct FusedArgs {
  // layer
  const uint8_t* w13t;
  const uint8_t* w2t;
  const float* ws13;
  const float* ws2;
  int E, H, I, N1, gated, w2_paired;
  int KB1, KB2, J1, J2;
  int act_type, act_fp16;
  int e8m0;                 // FP8 layers in ue8m0 mode: group scales rounded up to powers of two
  int cmp_fp16;             // compute dtype of the 16-bit MMAs / intermediate: 1 fp16, 0 bf16 (4-bit formats: fp16)
  int w4_tile_bytes, w4_scale_bytes;
  const float* g13;         // nvfp4 per-expert global scales [E][2] / [E]
  const float* g2;
  float alpha, limit, silu_limit;   // silu_limit: type 3's clamp, +inf for plain SiLU (type 0)
  // call
  const uint16_t* hidden;
  const int32_t* ids;
  const float* topk_w;
  void* out;
  int out_dtype;  // 0 bf16, 1 fp16, 2 f32
  int M, top_k;
  // workspace
  uint8_t* xt;
  float* xs;
  uint8_t* it;
  float* is;
  float* y;
  float* partials;
  FusedSync* sync;
  int rows_stride;
  int align_g1;             // cut GEMM1 at tile boundaries too when whole tiles fill this percentage of <= 3 waves (B200MOE_ALIGN_G1, default 60)
};

constexpr int W4_TILE_MAX = 4096 + 512;   // nibbles + scales of one [128 x 64] 4-bit tile

template <bool FP8, int NA, int TNMAX, int WQ>
struct FCfg {
  // WQ: 0 none, 1 int4 / 2 nvfp4 / 3 mxfp4 converted to fp16 wgmma A fragments in registers (W4A16)
  static constexpr int WD = WQ;
  static constexpr int TN = TNMAX;
  // WD == 0: 32 KB of MMA-ready tiles per stage; WD != 0: two k-blocks x two raw 4-bit tiles per stage
  static constexpr int A_STAGE = WD ? 4 * W4_TILE_MAX : 2 * TILE_BYTES;
  static constexpr int B_STAGE = 2 * TNMAX * 128;   // up to two k-blocks of tn rows
  static constexpr int STAGE = A_STAGE + B_STAGE;
  static constexpr int TABLES = 24 * 1024;
  // warps 0-3 drain, 4 A-producer, 6-9 fix-up, 10 B-producer; from warp 12: the MMA warpgroup (WD: two consumer
  // warpgroups, rows [0,64) and [64,128) of the gate and up tiles)
  static constexpr int MMA_WARP0 = 12;
  static constexpr int MMA_THREADS = WD ? 256 : 128;
  static constexpr int NTHREADS = MMA_WARP0 * 32 + MMA_THREADS;
  // WD: registers after setmaxnreg (consumers / everything else); the pool is the launch's 65536 / NTHREADS rounded
  // down to 8 per thread.  At 64 columns a consumer holds 64 fp32 accumulators, two slices of A fragments (16) and two
  // k-blocks of nibble words and scale records (up to 24): below 144 ptxas serialises the wgmmas (C7512).  The narrower
  // instantiations pipeline at 120 and keep 80 for the other warps.
  static constexpr int REG_MMA = (WD && TNMAX == 64) ? 144 : 120;
  static constexpr int REG_REST = (WD && TNMAX == 64) ? 64 : 80;
  static_assert(!WD || REG_MMA * MMA_THREADS + REG_REST * (NTHREADS - MMA_THREADS) <= (65536 / NTHREADS) / 8 * 8 * NTHREADS,
                "register split exceeds the launch allocation");
  static constexpr int BUFCOLS = 2 * TNMAX;       // gate + up accumulators (GEMM2 uses the first TNMAX)
  // WD at 64 columns: one buffer (a tile accumulates over 32 stages, long enough for the drain to empty it)
  static constexpr int NBUF = (WD && TNMAX == 64) ? 1 : 2;
  static constexpr int XCH = NBUF * BUFCOLS * 128 * 4;   // accumulator exchange area
  static constexpr int STAGES_RAW = (F_SMEM_BUDGET - TABLES - XCH - 1024) / STAGE;
  static constexpr int STAGES = STAGES_RAW > 6 ? 6 : STAGES_RAW;
  static constexpr int SMEM = STAGES * STAGE + XCH + TABLES + 1024;
  static_assert(STAGES >= 2, "shared-memory budget");
};

struct FChunk {
  int16_t expert;
  int16_t nrows;
  int32_t row0;
};

// shared-memory bookkeeping (fits FCfg::TABLES)
struct __align__(16) FTables {
  uint64_t full[8], empty[8];
  uint64_t tfull[4], tempty[4];
  uint64_t qfull[F_QD], qempty[F_QD];
  int32_t n_chunks, n_rows, n_valid, flag;
  float red[F_EPI_WARPS][64];
  int16_t row_of_slot[FUSED_MAX_SLOTS];   // permuted row of slot, -1 = skipped
  float sc_w[2][F_SCG];                   // staged FP8 weight scales of the current k-block group
  float sc_x[F_SCG][32];                  // staged activation scales [k-block][token column]
  int16_t cnt[FUSED_MAX_EXPERTS];
  int16_t eid[FUSED_MAX_SLOTS];           // expert of slot (-1 = skipped): the gather never re-reads ids from global
  int32_t off[FUSED_MAX_EXPERTS];
  FChunk chunks[FUSED_MAX_CHUNKS];
  int32_t scan_tmp[64];
};
static_assert(sizeof(FTables) <= 24 * 1024, "FTables too large");

// The 4-bit consumer warpgroups time out through a call (OUTLINED_TRAP): ptxas gives a setmaxnreg.inc region its raised
// register count only when no trap instruction lies inside it; otherwise it allocates the region at about the launch's
// count, and the 64-column consumers serialise their wgmmas for want of registers.
__device__ __noinline__ void f_timeout() { __trap(); }
template <bool OUTLINED_TRAP = false>
B200_DEVICE void f_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  if (OUTLINED_TRAP) {   // the call stays out of the polling loop
    bool done;
    while (!(done = mbar_try_wait(bar, parity)) && ++spins <= (1u << 27)) {
    }
    if (!done) f_timeout();
    return;
  }
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 27)) __trap();
  }
}

// Cross-CTA counters start at zero and are returned to zero before the launch ends (tile counters by their
// last arriver, the polled ones by the last CTA to finish), so one atomic per event is enough.
// Writers: stores -> bar.sync (epilogue warps) -> thread 0: __threadfence + atomicAdd  (grid.sync idiom).
B200_DEVICE int cnt_inc(int32_t* p) {
  __threadfence();
  return atomicAdd(p, 1);
}
B200_DEVICE bool cnt_reached(const int32_t* p, int target) { return ld_acquire(p) >= target; }
B200_DEVICE void cnt_wait(const int32_t* p, int target) {
  uint32_t spins = 0;
  while (!cnt_reached(p, target)) {
    if (++spins > (1u << 26)) __trap();
  }
}

// called by the last CTA of a launch: return the polled counters to zero for the next launch
B200_DEVICE void finish_launch(FusedSync* sy, int n_chunks, int J2) {
  sy->finished = 0;
  sy->x_ready = 0;
  for (int i = 0; i < n_chunks; ++i) sy->g1_done[i] = 0;
  for (int i = 0; i < J2; ++i) sy->comb[i] = 0;
  __threadfence();
}

B200_DEVICE float f_silu(float x) { return x / (1.0f + expf(-x)); }
B200_DEVICE float round_act(float v, int fp16) {
  return fp16 ? __half2float(__float2half_rn(v)) : __bfloat162float(__float2bfloat16_rn(v));
}

constexpr int F_COMBINE_INLINE_M = 4;

struct Seg {      // one (phase, chunk-group) of the per-CTA work list
  int ph, grp, c0, c1, KI, J, N, P, begin, end;
};
struct SegList {
  Seg s[4];
  int n;
};
// contiguous, balanced partition of [0, n) over `parts` CTAs (all non-empty when parts <= n)
B200_DEVICE int part_start(int c, int n, int parts) { return (int)(((long long)c * n) / parts); }
B200_DEVICE int part_owner(int i, int n, int parts) {
  int c = (int)(((long long)i * parts) / n);
  while (c + 1 < parts && part_start(c + 1, n, parts) <= i) ++c;
  while (c > 0 && part_start(c, n, parts) > i) --c;
  return c;
}

// out[t, j*128+col] = sum_jj w[t,jj] * y[row(t,jj), j*128+col] for t in [t0,t1): fixed jj order, k loads in flight
template <int TNMAX>
B200_DEVICE void combine_cols(const FusedArgs& a, const FTables* tb, int j, int t0, int t1, int col_in_tile) {
  const int col = j * 128 + col_in_tile;
  const int k = a.top_k;
  for (int t = t0; t < t1; ++t) {
    float s = 0.f;
    for (int j0 = 0; j0 < k; j0 += 8) {
      float v[8], w[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int jj = j0 + u;
        const int row = (jj < k) ? tb->row_of_slot[t * k + jj] : -1;
        w[u] = (row >= 0) ? a.topk_w[t * k + jj] : 0.f;
        v[u] = (row >= 0) ? __ldcg(a.y + (size_t)row * a.H + col) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) s = fmaf(w[u], v[u], s);
    }
    const size_t o = (size_t)t * a.H + col;
    if (a.out_dtype == 2)
      reinterpret_cast<float*>(a.out)[o] = s;
    else if (a.out_dtype == 0)
      reinterpret_cast<__nv_bfloat16*>(a.out)[o] = __float2bfloat16_rn(s);
    else
      reinterpret_cast<__half*>(a.out)[o] = __float2half_rn(s);
  }
}

// ------------------------------------------------------------------------------- 4-bit consumer warpgroups
// A raw 4-bit tile is stored in the consumers' wgmma fragment order (w4_layout.cuh): per k-block a thread reads its 16
// nibble bytes and its scale record with one load each, and word ks of the 16 bytes converts to its A fragment of k16
// slice ks.  The operation sequence per format is fixed, so the fp16 values are exactly those of the dequantised tile:
// int4 (1024 + q) - 1032, or (1024 + 16q) / 16 - 72, then * scale; e2m1 bits placed at value * 2^-14, * 2^14, then
// * scale.
B200_DEVICE uint4 lds_u4(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
B200_DEVICE uint2 lds_u2(uint32_t addr) {
  uint2 v;
  asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
  return v;
}
B200_DEVICE uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
// (a & B) | C in one LOP3: written out, the compiler may emit an AND and an OR
template <uint32_t B, uint32_t C>
B200_DEVICE uint32_t and_or(uint32_t a) {
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(a), "n"(B), "n"(C));
  return d;
}
B200_DEVICE __half2 u32_h2(uint32_t u) { return *reinterpret_cast<const __half2*>(&u); }
B200_DEVICE uint32_t h2_u32(__half2 h) { return *reinterpret_cast<const uint32_t*>(&h); }

// scales of rows (r0, r0 + 8) for slice ks from the thread's scale record
template <int WQ>
B200_DEVICE __half2 w4_scales(uint2 rec, int ks) {
  if (WQ == 1) return u32_h2(ks < 2 ? rec.x : rec.y);
  if (WQ == 2) {
    const uint32_t w = ks < 2 ? rec.x : rec.y;
    const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w >> (16 * (ks & 1))), __NV_E4M3);
    return *reinterpret_cast<const __half2*>(&h);
  }
  // e8m0 -> fp16 2^(E-127): exponent field E-112 clamped to [0,30] (scales < 2^-14 flush to 0)
  const uint32_t w = rec.x >> (16 * (ks >> 1));
  int f0 = (int)(w & 0xFFu) - 112, f1 = (int)((w >> 8) & 0xFFu) - 112;
  f0 = f0 < 0 ? 0 : (f0 > 30 ? 30 : f0);
  f1 = f1 < 0 ? 0 : (f1 > 30 ? 30 : f1);
  return u32_h2(((uint32_t)f0 << 10) | ((uint32_t)f1 << 26));
}
// one nibble word -> the four A fragment registers of one tile (s: scales of rows r0 and r0 + 8)
template <int WQ>
B200_DEVICE void w4_frag(uint32_t (&f)[4], uint32_t w, __half2 s) {
  const __half2 s0 = __low2half2(s), s1 = __high2half2(s);
  if (WQ == 1) {
    const __half2 lo_off = __float2half2_rn(-1032.0f), hi_mul = __float2half2_rn(0.0625f), hi_off = __float2half2_rn(-72.0f);
    const uint32_t l0 = and_or<0x000F000Fu, 0x64006400u>(w), h0 = and_or<0x00F000F0u, 0x64006400u>(w);
    w >>= 8;
    const uint32_t l1 = and_or<0x000F000Fu, 0x64006400u>(w), h1 = and_or<0x00F000F0u, 0x64006400u>(w);
    f[0] = h2_u32(__hmul2(__hadd2(u32_h2(l0), lo_off), s0));            // q - 8 is exact in both forms
    f[1] = h2_u32(__hmul2(__hfma2(u32_h2(h0), hi_mul, hi_off), s1));
    f[2] = h2_u32(__hmul2(__hadd2(u32_h2(l1), lo_off), s0));
    f[3] = h2_u32(__hmul2(__hfma2(u32_h2(h1), hi_mul, hi_off), s1));
  } else {
    // sign to bit 15, exponent + mantissa to bits [11:9]: value * 2^-14 (the e2m1 subnormal 0.5 lands on an fp16 subnormal)
    const uint32_t e[4] = {w & 0x8E008E00u, (w << 3) & 0x8E008E00u, ((w << 9) & 0x0E000E00u) | ((w << 2) & 0x80008000u),
                           ((w << 6) & 0x0E000E00u) | ((w << 1) & 0x80008000u)};
    const __half2 p14 = __float2half2_rn(16384.0f);
#pragma unroll
    for (int i = 0; i < 4; ++i) f[i] = h2_u32(__hmul2(__hmul2(u32_h2(e[i]), p14), (i & 1) ? s1 : s0));
  }
}

// One thread's shared-memory words of one k-block: the gate (na = 0) and up (na = 1) tiles' 16 nibble bytes and scale
// records (mxfp4: .x only)
struct W4Block {
  uint4 q[2];
  uint2 s[2];
};
template <int WQ>
B200_DEVICE void w4_load(W4Block& b, uint32_t raw, int tile_bytes, int kk, uint32_t u) {
#pragma unroll
  for (int na = 0; na < 2; ++na) {
    const uint32_t tile = raw + (kk * 2 + na) * tile_bytes;
    b.q[na] = lds_u4(tile + u * 16);
    const uint32_t rec = tile + W4_NIBBLE_BYTES + (u >> 2) * w4_scale_record_bytes(WQ);
    if (WQ == 3)
      b.s[na] = make_uint2(lds_u32(rec), 0u);
    else
      b.s[na] = lds_u2(rec);
  }
}
template <int WQ>
B200_DEVICE void w4_convert(uint32_t (&f)[2][4], const W4Block& b, int ks) {
#pragma unroll
  for (int na = 0; na < 2; ++na) {
    const uint32_t w = ks == 0 ? b.q[na].x : ks == 1 ? b.q[na].y : ks == 2 ? b.q[na].z : b.q[na].w;
    w4_frag<WQ>(f[na], w, w4_scales<WQ>(b.s[na], ks));
  }
}

// pins the accumulators in their registers across the asynchronous MMAs: without it the compiler may rematerialise or move
// them, and ptxas then serialises every wgmma
template <int N>
B200_DEVICE void acc_fence(float (&acc)[2][N]) {
#pragma unroll
  for (int na = 0; na < 2; ++na)
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(acc[na][i])::"memory");
}
// a use of one slice's A fragments at the point from which they may be overwritten
B200_DEVICE void frag_hold(uint32_t (&f)[2][4]) {
#pragma unroll
  for (int na = 0; na < 2; ++na)
#pragma unroll
    for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(f[na][i]));
}

// k-iterations [ki0, ki1) of one tile at NN token columns, walked as a flat sequence of k-blocks (two per stage, the
// last stage of a tile may hold one).  Per k16 slice: convert the gate and up fragments of this warpgroup's rows from
// registers, then issue their two MMAs (A registers, B = token tile of the stage).  Two slices are in flight: the
// conversion of slice n runs while the MMAs of slice n - 1 execute (wait_group 1).  The next k-block's words are loaded
// after the MMAs of the last slice are issued, into the registers of the current block's (now dead) words: no
// shared-memory load sits between a wait and the next MMAs, and at 64 columns nothing spills.  A stage is released once
// the MMAs of the next one have been waited for, the last one of the tile after wait_group 0.  Waiting for the next stage
// only after slice 0 keeps the order safe with two stages: by then the previous stage has been released.
template <class C, int NN>
B200_DEVICE void w4_tile(const FusedArgs& a, FTables* tb, const uint8_t* smem, int KB, int ki0, int ki1,
                         float (&acc)[2][C::TN / 2], uint32_t& itc) {
  constexpr int WQ = C::WD;
  const uint32_t u = threadIdx.x - C::MMA_WARP0 * 32;   // consumer thread, 0..255 (w4_layout.cuh)
  const bool lead = (threadIdx.x & 127) == 0;
  const uint32_t smem_u = smem_u32(smem);
  int pend = -1;   // stage whose last MMAs may still be in flight
  // A fragments, double-buffered by slice parity: slice n converts into fa[n & 1] while the MMAs of slice n - 1 still
  // read fa[(n - 1) & 1].  frag_hold below keeps the older buffer live until those MMAs have been waited for, so the
  // register allocator has to give the two buffers distinct registers and ptxas need not serialise the wgmmas.
  uint32_t fa[2][2][4] = {};
  acc_fence(acc);
  uint32_t it = itc;
  int ki = ki0, kk = 0, s = it % C::STAGES;
  f_wait<true>(&tb->full[s], (it / C::STAGES) & 1);
  W4Block cur;
  w4_load<WQ>(cur, smem_u + s * C::STAGE, a.w4_tile_bytes, 0, u);
  while (true) {
    const int nkb = (KB - 2 * ki) < 2 ? (KB - 2 * ki) : 2;
    const bool last_of_stage = kk + 1 == nkb;
    const bool more = !last_of_stage || ki + 1 < ki1;
    const uint32_t bbase = smem_u + s * C::STAGE + C::A_STAGE + kk * (uint32_t)((NN >> 3) * 1024);
    W4Block nxt;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      uint32_t (&f)[2][4] = fa[ks & 1];
      w4_convert<WQ>(f, cur, ks);
      const uint64_t bd = wgmma_desc_sw128(bbase + ks * 32, 1024);
      const uint32_t accum = (ki > ki0 || kk > 0 || ks > 0) ? 1u : 0u;
      wgmma_fence();
      WgmmaRS<NN, 0>::mma(acc[0], f[0], bd, accum);
      WgmmaRS<NN, 0>::mma(acc[1], f[1], bd, accum);
      wgmma_commit();
      if (ks == 3) {   // after the tile's last k-block this reloads the current one, unused: no branch around the load
        uint32_t ns = s;
        int nkk = more ? kk + 1 : kk;
        if (last_of_stage && more) {
          ns = (it + 1) % C::STAGES;
          nkk = 0;
          f_wait<true>(&tb->full[ns], ((it + 1) / C::STAGES) & 1);
        }
        w4_load<WQ>(nxt, smem_u + ns * C::STAGE, a.w4_tile_bytes, nkk, u);
      }
      wgmma_wait<1>();
      frag_hold(fa[(ks + 1) & 1]);   // the previous slice's MMAs are complete: its buffer may be overwritten now
      if (pend >= 0) {
        if (lead) mbar_arrive(&tb->empty[pend]);
        pend = -1;
      }
    }
    if (last_of_stage) {
      pend = s;
      ++it;
      ++ki;
      kk = 0;
      s = it % C::STAGES;
    } else {
      ++kk;
    }
    if (!more) break;
    cur = nxt;
  }
  itc = it;
  wgmma_wait<0>();
  acc_fence(acc);
  if (lead && pend >= 0) mbar_arrive(&tb->empty[pend]);
}

// Consumer warpgroup of the 4-bit variants: walks the same schedule as the producers and the drain; every finished
// accumulator (this warpgroup's 64 rows of gate and up) is parked in the exchange area.  The instruction width follows
// the chunk's padded row count, so a 16-row chunk pays for 16 columns of tensor work.
template <class C>
B200_DEVICE void w4_consumer(const FusedArgs& a, FTables* tb, const uint8_t* smem, uint32_t xch, const SegList& sl) {
  constexpr int TNMAX = C::TN;
  const int half = ((int)threadIdx.x >> 7) - C::MMA_WARP0 / 4;
  float acc[2][TNMAX / 2];
#pragma unroll
  for (int na = 0; na < 2; ++na)
#pragma unroll
    for (int i = 0; i < TNMAX / 2; ++i) acc[na][i] = 0.f;
  uint32_t itc = 0, acc_it = 0;
  for (int si = 0; si < sl.n; ++si) {
    const Seg& sg = sl.s[si];
    const int KI = sg.KI, sg_end = sg.end;
    const int KB = sg.ph == 0 ? a.KB1 : a.KB2;
    int it = sg.begin;
    while (it < sg_end) {
      const int tile = it / KI, k0 = it % KI;
      const int k1 = (KI - k0 < sg_end - it) ? KI : k0 + (sg_end - it);
      const int tn = ((int)tb->chunks[sg.c0 + tile / sg.J].nrows + 15) & ~15;
      const uint32_t buf = acc_it % C::NBUF;
      const uint32_t base = xch + buf * C::BUFCOLS;
      switch (tn) {
        case 16:
          w4_tile<C, 16>(a, tb, smem, KB, k0, k1, acc, itc);
          f_wait<true>(&tb->tempty[buf], ((acc_it / C::NBUF) & 1) ^ 1);
          xch_store_frag<16>(base, half, acc[0]);
          xch_store_frag<16>(base + TNMAX, half, acc[1]);
          break;
        case 32:
          if constexpr (TNMAX >= 32) {
            w4_tile<C, 32>(a, tb, smem, KB, k0, k1, acc, itc);
            f_wait<true>(&tb->tempty[buf], ((acc_it / C::NBUF) & 1) ^ 1);
            xch_store_frag<32>(base, half, acc[0]);
            xch_store_frag<32>(base + TNMAX, half, acc[1]);
          }
          break;
        case 48:
          if constexpr (TNMAX >= 48) {
            w4_tile<C, 48>(a, tb, smem, KB, k0, k1, acc, itc);
            f_wait<true>(&tb->tempty[buf], ((acc_it / C::NBUF) & 1) ^ 1);
            xch_store_frag<48>(base, half, acc[0]);
            xch_store_frag<48>(base + TNMAX, half, acc[1]);
          }
          break;
        default:
          if constexpr (TNMAX >= 64) {
            w4_tile<C, 64>(a, tb, smem, KB, k0, k1, acc, itc);
            f_wait<true>(&tb->tempty[buf], ((acc_it / C::NBUF) & 1) ^ 1);
            xch_store_frag<64>(base, half, acc[0]);
            xch_store_frag<64>(base + TNMAX, half, acc[1]);
          }
          break;
      }
      mbar_arrive(&tb->tfull[buf]);
      ++acc_it;
      it += k1 - k0;
    }
  }
}

template <bool FP8, int NA, int TNMAX, int WQ>
__global__ void __launch_bounds__((FCfg<FP8, NA, TNMAX, WQ>::NTHREADS), 1)
    moe_fused_kernel(const __grid_constant__ FusedArgs a) {
  using C = FCfg<FP8, NA, TNMAX, WQ>;
  constexpr int NT = C::NTHREADS;
  static_assert(WQ == 0 || (!FP8 && NA == 2), "4-bit formats: gated experts");
  constexpr int WD = C::WD;     // dequant flavour
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* xch_area = smem + C::STAGES * C::STAGE;
  const uint32_t xch = xch_base(xch_area);
  FTables* tb = reinterpret_cast<FTables*>(xch_area + C::XCH);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int G = gridDim.x, cta = blockIdx.x;
  FusedSync* sy = a.sync;

  if (tid == 0) {
    for (int i = 0; i < C::STAGES; ++i) {
      mbar_init(&tb->full[i], 1);
      mbar_init(&tb->empty[i], C::MMA_THREADS / 128);   // one arrival per MMA warpgroup
    }
    for (int i = 0; i < C::NBUF; ++i) {
      mbar_init(&tb->tfull[i], C::MMA_THREADS);   // every MMA thread, after parking its fragment
      mbar_init(&tb->tempty[i], F_EPI_WARPS);
    }
    for (int i = 0; i < F_QD; ++i) {
      mbar_init(&tb->qfull[i], F_EPI_WARPS);
      mbar_init(&tb->qempty[i], F_EPI_WARPS);
    }
    fence_barrier_init();
  }

  // ------------------------------------------------------------------------------- phase 0a: routing table
  const int n_slots = a.M * a.top_k;
  const int E = a.E;
  // stable per-expert ranks without block-wide serialisation: warp w ranks a contiguous range of slots with
  // warp-private counters (kept in the still idle pipeline stages), then the counters are prefix-summed over
  // the warps per expert
  constexpr int NW = NT / 32;
  int16_t* wcnt = reinterpret_cast<int16_t*>(smem);   // [NW][E]
  for (int i = tid; i < NW * E; i += NT) wcnt[i] = 0;
  __syncthreads();
  const int spw = ((n_slots + NW - 1) / NW + 31) & ~31;   // slots per warp
  {
    const int s_end = min(n_slots, (warp + 1) * spw);
    for (int s0 = warp * spw; s0 < s_end; s0 += 32) {
      const int s = s0 + lane;
      int e = (s < s_end) ? a.ids[s] : -1;
      if (e < 0 || e >= E) e = -1;
      const unsigned m = __match_any_sync(0xffffffffu, e);
      const int rank = __popc(m & ((1u << lane) - 1u));
      const int base = (e >= 0) ? wcnt[warp * E + e] : 0;
      __syncwarp();
      if (e >= 0 && rank == 0) wcnt[warp * E + e] = (int16_t)(base + __popc(m));
      __syncwarp();
      if (s < s_end) {
        tb->row_of_slot[s] = (e >= 0) ? (int16_t)(base + rank) : (int16_t)-1;
        tb->eid[s] = (int16_t)e;
      }
    }
  }
  __syncthreads();
  for (int e = tid; e < E; e += NT) {
    int acc = 0;
    for (int w = 0; w < NW; ++w) {
      const int c = wcnt[w * E + e];
      wcnt[w * E + e] = (int16_t)acc;
      acc += c;
    }
    tb->cnt[e] = (int16_t)acc;
  }
  __syncthreads();
  {
    // exclusive scan over experts of (padded rows, chunks); thread t owns a contiguous span of experts
    const int per = (E + NT - 1) / NT;
    const int e0 = tid * per;
    int lrows = 0, lch = 0;
    for (int i = 0; i < per; ++i) {
      const int e = e0 + i;
      if (e < E) {
        const int c = tb->cnt[e];
        lrows += (c + ROW_ALIGN - 1) & ~(ROW_ALIGN - 1);
        lch += (c + TNMAX - 1) / TNMAX;
      }
    }
    int irows = lrows, ich = lch;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int x = __shfl_up_sync(0xffffffffu, irows, o);
      const int z = __shfl_up_sync(0xffffffffu, ich, o);
      if (lane >= o) {
        irows += x;
        ich += z;
      }
    }
    if (lane == 31) {
      tb->scan_tmp[warp] = irows;
      tb->scan_tmp[32 + warp] = ich;
    }
    __syncthreads();
    int brows = 0, bch = 0;
    for (int w = 0; w < warp; ++w) {
      brows += tb->scan_tmp[w];
      bch += tb->scan_tmp[32 + w];
    }
    int xrows = brows + irows - lrows, xch = bch + ich - lch;
    for (int i = 0; i < per; ++i) {
      const int e = e0 + i;
      if (e < E) {
        tb->off[e] = xrows;
        const int c = tb->cnt[e];
        const int nch = (c + TNMAX - 1) / TNMAX;
        for (int q = 0; q < nch; ++q) {
          FChunk ch;
          ch.expert = (int16_t)e;
          ch.row0 = xrows + q * TNMAX;
          ch.nrows = (int16_t)min(TNMAX, c - q * TNMAX);
          if (xch + q < FUSED_MAX_CHUNKS) tb->chunks[xch + q] = ch;
        }
        xrows += (c + ROW_ALIGN - 1) & ~(ROW_ALIGN - 1);
        xch += nch;
      }
    }
    if (tid == NT - 1) {
      tb->n_rows = brows + irows;
      tb->n_chunks = bch + ich;
    }
  }
  __syncthreads();
  const int n_chunks = tb->n_chunks;
  int n_valid_local = 0;
  for (int sidx = tid; sidx < n_slots; sidx += NT) {
    const int lr = tb->row_of_slot[sidx];
    if (lr >= 0) {
      const int e = tb->eid[sidx];
      tb->row_of_slot[sidx] = (int16_t)(tb->off[e] + wcnt[(sidx / spw) * E + e] + lr);
    }
  }
  if (tid == 0) {
    int nv = 0;
    for (int e = 0; e < E; ++e) nv += tb->cnt[e];
    tb->n_valid = nv;
  }
  __syncthreads();
  const int n_valid = tb->n_valid;
  (void)n_valid_local;

  // nothing routed here: the output is all zeros
  if (n_chunks == 0) {
    const size_t n = (size_t)a.M * a.H;
    for (size_t i = (size_t)cta * NT + tid; i < n; i += (size_t)G * NT) {
      if (a.out_dtype == 2)
        reinterpret_cast<float*>(a.out)[i] = 0.f;
      else
        reinterpret_cast<uint16_t*>(a.out)[i] = 0;
    }
    __syncthreads();
    if (tid == 0) {
      const int old = atomicAdd(&sy->finished, 1);
      if (old == G - 1) finish_launch(sy, 0, 0);
    }
    return;
  }

  // ------------------------------------------------------------------------------- phase 0b: row gather (+quant)
  // done by the four epilogue warps (the producer / MMA warps start streaming weights meanwhile); valid rows
  // are dealt round-robin to the CTAs; chunk-contiguous tiled layout:
  //   xt[row0_q * KB*128 + kb * (tn_q/8*1024) + ((r-row0_q)/8)*1024 + sw128((r-row0_q)%8, byte)]
  const int SEGS = (a.H + 1023) / 1024;
  // gather groups of 128 threads: the drain warps, the fix-up warps and (4-bit formats) the consumer warpgroups —
  // none of them has anything else to do before the first rows are gathered
  const int ggrp = warp < 4 ? 0 : (warp >= 6 && warp < 10) ? 1 : (WQ && warp >= C::MMA_WARP0) ? 2 + ((warp - C::MMA_WARP0) >> 2) : -1;
  constexpr int NGG = WQ ? 4 : 2;
  if (ggrp >= 0) {
    const int gt = ggrp == 0 ? tid : ggrp == 1 ? tid - 192 : tid - C::MMA_WARP0 * 32 - (ggrp - 2) * 128;   // 0..127
    int mine = 0;
    const int vcta = cta * NGG + ggrp, VG = G * NGG;
    // A round = GSL slots x all of their 1024-element segments (<= 8: H <= 8192): the routing metadata of a slot is
    // looked up once, and every 16-byte row load of the round is in flight before the first conversion starts
    constexpr int GSL = WD ? 1 : 2;   // 4-bit variants: 640 threads, 96 registers
    for (int sb = vcta; sb < n_slots; sb += GSL * VG) {
      uint4 raw[GSL][8];
      int rr_[GSL], row0_[GSL], tn_[GSL], r_[GSL];
      bool ok_[GSL];
#pragma unroll
      for (int u = 0; u < GSL; ++u) {
        const int slot = sb + u * VG;
        ok_[u] = false;
        rr_[u] = row0_[u] = r_[u] = 0;
        tn_[u] = 16;
        const uint16_t* hrow = a.hidden;
        if (slot < n_slots) {
          const int r = tb->row_of_slot[slot];
          if (r >= 0) {
            const int e = tb->eid[slot];
            const int c = (r - tb->off[e]) / TNMAX;
            const int row0 = tb->off[e] + c * TNMAX;
            const int nr = min(TNMAX, (int)tb->cnt[e] - c * TNMAX);
            ok_[u] = true;
            r_[u] = r;
            row0_[u] = row0;
            rr_[u] = r - row0;
            tn_[u] = (nr + 15) & ~15;
            hrow = a.hidden + (size_t)(slot / a.top_k) * a.H;
          }
        }
#pragma unroll
        for (int sg = 0; sg < 8; ++sg) {
          const int el = sg * 1024 + gt * 8;
          raw[u][sg] = (ok_[u] && el < a.H) ? *reinterpret_cast<const uint4*>(hrow + el) : make_uint4(0u, 0u, 0u, 0u);
        }
      }
#pragma unroll
      for (int u = 0; u < GSL; ++u) {
       if (!ok_[u]) continue;   // uniform across the 128 gather threads
#pragma unroll
       for (int sg = 0; sg < 8; ++sg) {
        if (sg >= SEGS) break;
        ++mine;
        const int rr = rr_[u], r = r_[u], el = sg * 1024 + gt * 8;
        const uint4 raw_u = raw[u][sg];
        const bool valid = el < a.H;
        uint8_t* dst = a.xt + (size_t)row0_[u] * a.KB1 * 128 + (size_t)(rr >> 3) * 1024;
        const size_t kb_stride = (size_t)(tn_[u] >> 3) * 1024;
        if (FP8) {
          const uint16_t* h = reinterpret_cast<const uint16_t*>(&raw_u);
          float f[8];
          float am = 0.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            f[i] = a.act_fp16 ? __half2float(*reinterpret_cast<const __half*>(&h[i]))
                              : __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(&h[i]));
            am = fmaxf(am, fabsf(f[i]));
          }
#pragma unroll
          for (int o = 8; o > 0; o >>= 1) am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));
          if (valid) {
            const float sc = fp8_group_scale(am, a.e8m0);
            uint8_t qv[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const __nv_fp8_e4m3 v(f[i] / sc);
              qv[i] = *reinterpret_cast<const uint8_t*>(&v);
            }
            const int kb = el >> 7;
            *reinterpret_cast<uint2*>(dst + kb * kb_stride + sw128_offset(rr & 7, el & 127)) =
                *reinterpret_cast<const uint2*>(qv);
            if ((gt & 15) == 0) a.xs[(size_t)kb * a.rows_stride + r] = sc;
          }
        } else if (valid) {
          const int kb = el >> 6;
          uint4 rv = raw_u;
          if (a.cmp_fp16 && !a.act_fp16) {   // 4-bit formats compute in fp16: bf16 -> fp16 (saturating)
            const __nv_bfloat162* hb = reinterpret_cast<const __nv_bfloat162*>(&rv);
            uint32_t pk[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float lo = fminf(fmaxf(__low2float(hb[i]), -65504.f), 65504.f);
              const float hi = fminf(fmaxf(__high2float(hb[i]), -65504.f), 65504.f);
              const __half2 h2 = __floats2half2_rn(lo, hi);
              pk[i] = *reinterpret_cast<const uint32_t*>(&h2);
            }
            rv = make_uint4(pk[0], pk[1], pk[2], pk[3]);
          }
          *reinterpret_cast<uint4*>(dst + kb * kb_stride + sw128_offset(rr & 7, (el & 63) * 2)) = rv;
        }
      }
       }

    }
    if (mine > 0) {
      asm volatile("fence.proxy.async.global;" ::: "memory");  // rows are read through the async proxy
      asm volatile("bar.sync %0, 128;" ::"r"(8 + ggrp) : "memory");
      if (gt == 0) {
        __threadfence();
        atomicAdd(&sy->x_ready, mine);
      }
    }
  }

  // ------------------------------------------------------------------------------- stream-K schedule
  // Work list of every CTA: (GEMM1, group 0), (GEMM1, group 1), (GEMM2, group 0), (GEMM2, group 1).  A group
  // is a contiguous run of chunks; inside a (phase, group) the linearised (tile, k-iteration) space is cut
  // into equal contiguous ranges over the CTAs.  With two groups, GEMM2 of group 0 can start while the
  // fix-ups / activation of group 1 are still in flight (the GEMM1 -> GEMM2 dependency is per chunk).
  // iterations per tile: one k-block of two tiles (32 KB), or two k-blocks (single tile / 4-bit tile pairs)
  const int KI1e = (NA == 2 && !WD) ? a.KB1 : (a.KB1 + 1) / 2;
  const bool pair2 = a.w2_paired != 0;                   // GEMM2: two 128-row tiles per stage
  const int KI2 = (pair2 && !WD) ? a.KB2 : (a.KB2 + 1) / 2;
  const int J2e = pair2 ? a.J2 / 2 : a.J2;
  const int NG = n_chunks >= 4 ? 2 : 1;
  SegList sl;
  {
    const int split = NG == 2 ? n_chunks / 2 : n_chunks;
    int n = 0;
    for (int ph = 0; ph < 2; ++ph) {
      for (int g = 0; g < NG; ++g) {
        Seg& sg = sl.s[n++];
        sg.ph = ph;
        sg.grp = g;
        sg.c0 = g == 0 ? 0 : split;
        sg.c1 = (g == NG - 1) ? n_chunks : split;
        sg.KI = ph == 0 ? KI1e : KI2;
        sg.J = ph == 0 ? a.J1 : J2e;
        sg.N = (sg.c1 - sg.c0) * sg.J * sg.KI;
        sg.P = sg.N < G ? sg.N : G;
        sg.begin = sg.end = 0;
        const int n_tiles = (sg.c1 - sg.c0) * sg.J;
        const int waves = (n_tiles + G - 1) / G;
        // GEMM1 tiles are long (K = hidden size), so whole tiles cost more imbalance — but with at most three tiles per CTA
        // (EP shards: 96-384 tiles per group) every tile of a stream-K cut is split and its fix-up (partials through L2,
        // cross-CTA flags, activation, re-quantisation) sits between GEMM1 and GEMM2
        if ((ph == 1 && n_tiles * 10 >= waves * G * 7) ||
            (ph == 0 && a.align_g1 > 0 && waves <= 3 && n_tiles * 100 >= waves * G * a.align_g1)) {
          // GEMM2 tiles are short (K = intermediate size): cut at tile boundaries whenever whole tiles fill >= 70 % of the
          // CTA slots of their waves.  No GEMM2 tile needs the cross-CTA reduction then — every accumulator goes straight
          // to y — which removes the split-tile fix-up chain from the end of the kernel, against a little more
          // streaming time for the fullest CTA
          sg.P = G;
          sg.begin = part_start(cta, n_tiles, G) * sg.KI;
          sg.end = part_start(cta + 1, n_tiles, G) * sg.KI;
        } else if (cta < sg.P) {
          sg.begin = part_start(cta, sg.N, sg.P);
          sg.end = part_start(cta + 1, sg.N, sg.P);
        }
      }
    }
    sl.n = n;
  }

  if constexpr (WD != 0) {
    // the consumer warpgroups hold 2 x 32 fp32 accumulators per thread at 64 columns: registers move to them from the
    // producer, drain and fix-up warps (the consumers take them in their own branch)
    if (warp < C::MMA_WARP0) setmaxnreg_dec<C::REG_REST>();
  }

  if (warp == 4 || warp == 10) {
    // ======================================================================= producers
    // warp 4 streams the weight stages (A), warp 10 the activation stages (B): two independent issue
    // threads, no integer divisions in the loops (a single thread's instruction latency was the limiter).
    // elect.sync (not `lane == 0`): ptxas keeps the copy operands in uniform registers, one UBLKCP per copy
    if (elect_one()) {
      const bool is_a = (warp == 4);
      const uint64_t pol = policy_evict_first();
      bool x_ok = false;
      int g1_ok_chunk = -1;
      uint32_t cur = 0;  // flat iteration counter -> stage / parity
      for (int si = 0; si < sl.n; ++si) {
        const Seg& sg = sl.s[si];
        if (sg.begin == sg.end) continue;
        const bool ph1 = sg.ph == 0;
        const bool two = WD ? false : (ph1 ? (NA == 2) : pair2);   // 4-bit dequant: two k-blocks x two tiles per stage
        const int KB = ph1 ? a.KB1 : a.KB2;
        const int KI = sg.KI, J = sg.J;
        int tile = sg.begin / KI, ki = sg.begin % KI;
        int q = sg.c0 + tile / J, j = tile % J;
        FChunk ch = tb->chunks[q];
        int tn = (ch.nrows + 15) & ~15;
        for (int it = sg.begin; it < sg.end; ++it, ++cur) {
          const uint32_t s = cur % C::STAGES;
          const uint32_t par = ((cur / C::STAGES) & 1) ^ 1;
          const int kb0 = two ? ki : ki * 2;
          const int nkb = two ? 1 : ((KB - kb0) < 2 ? (KB - kb0) : 2);
          const uint32_t bbytes = (uint32_t)(tn >> 3) * nkb * 1024;
          uint8_t* sa = smem + s * C::STAGE;
          if (is_a) {
            const uint32_t abytes = WD ? nkb * 2 * a.w4_tile_bytes : (two ? 2 * TILE_BYTES : nkb * TILE_BYTES);
            const uint8_t* wsrc;
            if (WD)
              wsrc = (ph1 ? a.w13t : a.w2t) +
                     (((size_t)(ch.expert * J + j) * KB + kb0) * 2) * (size_t)a.w4_tile_bytes;
            else if (ph1)
              wsrc = a.w13t + ((size_t)(ch.expert * a.J1 + j) * a.KB1 + kb0) * (size_t)(NA * TILE_BYTES);
            else if (pair2)
              wsrc = a.w2t + ((size_t)(ch.expert * (a.J2 / 2) + j) * a.KB2 + kb0) * (size_t)(2 * TILE_BYTES);
            else
              wsrc = a.w2t + ((size_t)(ch.expert * a.J2 + j) * a.KB2 + kb0) * (size_t)TILE_BYTES;
            f_wait(&tb->empty[s], par);
            mbar_arrive_expect_tx(&tb->full[s], abytes + bbytes);
            bulk_g2s_hint(sa, wsrc, abytes, &tb->full[s], pol);
          } else {
            // dependency of the B operand: rows gathered (GEMM1) / intermediate of the chunk complete (GEMM2)
            if (ph1) {
              if (!x_ok) {
                cnt_wait(&sy->x_ready, n_valid * SEGS);
                asm volatile("fence.proxy.async.global;" ::: "memory");
                x_ok = true;
              }
            } else if (g1_ok_chunk != q) {
              cnt_wait(&sy->g1_done[q], a.J1);
              asm volatile("fence.proxy.async.global;" ::: "memory");
              g1_ok_chunk = q;
            }
            const uint8_t* base = ph1 ? a.xt : a.it;
            const uint8_t* bsrc = base + (size_t)ch.row0 * KB * 128 + (size_t)kb0 * ((tn >> 3) * 1024);
            f_wait(&tb->empty[s], par);
            bulk_g2s(sa + C::A_STAGE, bsrc, bbytes, &tb->full[s]);
          }
          // advance (tile, ki) without divisions
          if (++ki == KI) {
            ki = 0;
            if (++j == J) {
              j = 0;
              ++q;
              if (it + 1 < sg.end) {
                ch = tb->chunks[q];
                tn = (ch.nrows + 15) & ~15;
              }
            }
          }
        }
      }
    }
  } else if (WD && warp >= C::MMA_WARP0) {
    // ======================================================================= consumer warpgroups (4-bit formats)
    setmaxnreg_inc<C::REG_MMA>();
    w4_consumer<C>(a, tb, smem, xch, sl);
    setmaxnreg_dec<C::REG_REST>();   // the combine below runs at the same count in every warp
  } else if (!WD && warp >= C::MMA_WARP0) {
    // ======================================================================= MMA warpgroup
    // Walks the schedule with register accumulators: acc[na][h] = accumulator na (gate | up, or tile of a pair), rows
    // [64h, 64h + 64).  The instruction shape is fixed at N = TNMAX columns; columns beyond the chunk's rows multiply
    // whatever the stage holds there and are never read.  A finished accumulator is parked in the exchange area for
    // the drain warps; the buffer is waited for only then, so its MMAs ran while the drain still read the previous one.
    const bool mma_lead = tid == C::MMA_WARP0 * 32;
    const uint32_t smem_base_u = smem_u32(smem);
    float acc[2][2][TNMAX / 2];
    uint32_t itc = 0, acc_it = 0;
    for (int si = 0; si < sl.n; ++si) {
      const Seg& sg = sl.s[si];
      const int KI = sg.KI, sg_end = sg.end;
      const int KB = sg.ph == 0 ? a.KB1 : a.KB2;
      const bool two = WD ? false : (sg.ph == 0 ? (NA == 2) : pair2);
      const int nacc = (two || WD) ? 2 : 1;
      auto park = [&]() {
        const uint32_t buf = acc_it % C::NBUF;
        f_wait(&tb->tempty[buf], ((acc_it / C::NBUF) & 1) ^ 1);
#pragma unroll
        for (int na = 0; na < 2; ++na)
          if (na < nacc) {
#pragma unroll
            for (int h = 0; h < 2; ++h) xch_store_frag<TNMAX>(xch + buf * C::BUFCOLS + na * TNMAX, h, acc[na][h]);
          }
        mbar_arrive(&tb->tfull[buf]);
        ++acc_it;
      };
      int it = sg.begin;
      while (it < sg_end) {
        const int tile = it / KI, k0 = it % KI;
        const int k1 = (KI - k0 < sg_end - it) ? KI : k0 + (sg_end - it);
        const int nrows = (int)tb->chunks[sg.c0 + tile / sg.J].nrows;
        const int tn = (nrows + 15) & ~15;
        for (int ki = k0; ki < k1; ++ki, ++itc) {
          const int s = itc % C::STAGES;
          f_wait(&tb->full[s], (itc / C::STAGES) & 1);
          const int kb0 = two ? ki : ki * 2;
          const int nkb = two ? 1 : ((KB - kb0) < 2 ? (KB - kb0) : 2);
          const uint32_t sa = smem_base_u + s * C::STAGE;
          const uint32_t sb = sa + C::A_STAGE;
          for (int kk = 0; kk < nkb; ++kk) {
            const uint32_t bbase = sb + kk * (uint32_t)((tn >> 3) * 1024);
            const uint32_t acc0 = (ki > k0 || kk > 0) ? 1u : 0u;
            {
              const uint32_t a0 = sa + (two ? 0 : kk) * TILE_BYTES;
              wgmma_fence();
#pragma unroll
              for (int na = 0; na < 2; ++na) {
                if (na < nacc) {
#pragma unroll
                  for (int ks = 0; ks < 4; ++ks) {
                    const uint32_t aa = a0 + na * TILE_BYTES + ks * 32, bb = bbase + ks * 32;
                    if (FP8)
                      wgmma_tile128<TNMAX, 2>(acc[na], aa, bb, ks > 0 ? 1u : 0u);
                    else if (a.cmp_fp16)
                      wgmma_tile128<TNMAX, 0>(acc[na], aa, bb, ks > 0 ? 1u : acc0);
                    else
                      wgmma_tile128<TNMAX, 1>(acc[na], aa, bb, ks > 0 ? 1u : acc0);
                  }
                }
              }
              wgmma_commit();
              wgmma_wait<0>();
              if (FP8) park();   // every 128-wide k-block is promoted with its own scales by the drain warps
            }
          }
          if (mma_lead) mbar_arrive(&tb->empty[s]);
        }
        if (!FP8) park();
        it += k1 - k0;
      }
    }
  } else if (warp < 4) {
    // ======================================================================= drain warps 0..3
    // exchange area -> registers (FP8: block-scale promotion per k-block), then the tile part is parked in global
    // memory and handed to the fix-up warps so that the drain never waits on cross-CTA latencies.
    uint32_t acc_it = 0, part_no = 0;
    const uint32_t lane_off = (uint32_t)(warp * 32) << 16;
    const int row_in_tile = warp * 32 + lane;
    for (int si = 0; si < sl.n; ++si) {
      const Seg& sg = sl.s[si];
      const int ph = sg.ph;
      const int KI = sg.KI;
      const int J = sg.J;
      const int KB = ph == 0 ? a.KB1 : a.KB2;
      const bool two = ph == 0 ? (NA == 2) : pair2;
      const int nacc = (two || WD) ? 2 : 1;
      int pend_y = 0;   // whole GEMM2 tiles written straight to y in this segment
      int it = sg.begin;
      while (it < sg.end) {
        const int tile = it / KI, k0 = it % KI;
        const int k1 = (KI - k0 < sg.end - it) ? KI : k0 + (sg.end - it);
        const int q = sg.c0 + tile / J, j = tile % J;
        const FChunk ch = tb->chunks[q];
        const int tn = (ch.nrows + 15) & ~15;

        float acc[2][TNMAX];
#pragma unroll
        for (int na = 0; na < 2; ++na)
#pragma unroll
          for (int c = 0; c < TNMAX; ++c) acc[na][c] = 0.f;

        if (FP8) {
          const float* wsc_base = ph == 0 ? a.ws13 : a.ws2;
          const int NB = ph == 0 ? a.N1 / 128 : a.H / 128;
          const float* bsc = ph == 0 ? a.xs : a.is;
          const int rb0 = (ph == 1 && pair2) ? 2 * j : j;
          const int rb1 = ph == 0 ? a.I / 128 + j : 2 * j + 1;
          const float* wrow0 = wsc_base + ((size_t)ch.expert * NB + rb0) * KB;
          const float* wrow1 = two ? wsc_base + ((size_t)ch.expert * NB + rb1) * KB : wrow0;
          const int kbA = two ? k0 : k0 * 2;
          const int kbB = two ? k1 : (k1 * 2 < KB ? k1 * 2 : KB);
          // NOTE: activation scales are produced by OTHER CTAs in this launch (phase 0b / GEMM1 finalisers);
          // they may only be read after the first full accumulator of the segment (which transitively orders them)
          // and are read with ld.cg so that no stale L1 line can be hit.
          for (int kb = kbA; kb < kbB; ++kb, ++acc_it) {
            const uint32_t buf = acc_it % C::NBUF;
            f_wait(&tb->tfull[buf], (acc_it / C::NBUF) & 1);
            const int rel = (kb - kbA) % F_SCG;
            if (rel == 0) {
              // stage the scales of the next F_SCG k-blocks in shared memory: one L2 latency per group
              // instead of one per k-block on the drain's critical path
              asm volatile("bar.sync 1, 128;" ::: "memory");  // every drain warp is done with the old group
              const int n = (kbB - kb < F_SCG) ? kbB - kb : F_SCG;
              const int dt = warp * 32 + lane;
              for (int i = dt; i < 2 * n; i += 128) {
                const int which = i / n, kk = i - which * n;
                tb->sc_w[which][kk] = __ldg((which ? wrow1 : wrow0) + kb + kk);
              }
              for (int i = dt; i < n * 32; i += 128) {
                const int kk = i >> 5, c = i & 31;
                tb->sc_x[kk][c] = (c < tn) ? __ldcg(bsc + (size_t)(kb + kk) * a.rows_stride + ch.row0 + c) : 0.f;
              }
              asm volatile("bar.sync 1, 128;" ::: "memory");
            }
            const float w0 = tb->sc_w[0][rel], w1 = tb->sc_w[1][rel];
            float xs_cur[(TNMAX + 31) / 32];
#pragma unroll
            for (int w = 0; w < (TNMAX + 31) / 32; ++w) xs_cur[w] = tb->sc_x[rel][lane];
#pragma unroll
            for (int na = 0; na < 2; ++na) {
              if (na < nacc) {
#pragma unroll
                for (int c16 = 0; c16 < TNMAX / 16; ++c16) {
                  if (c16 * 16 < tn) {
                    float part[16];
                    xch_ld<16>(xch + lane_off + buf * C::BUFCOLS + na * TNMAX + c16 * 16, part);
                    const float wv = na == 0 ? w0 : w1;
#pragma unroll
                    for (int c = 0; c < 16; ++c) {
                      const int cc = c16 * 16 + c;
                      const float xsc = __shfl_sync(0xffffffffu, xs_cur[cc / 32], cc % 32);
                      acc[na][cc] = fmaf(part[c], wv * xsc, acc[na][cc]);
                    }
                  }
                }
              }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&tb->tempty[buf]);
          }
        }

        const bool split = (k0 != 0 || k1 != KI);
        if (ph == 1 && !split) {
          // a whole GEMM2 tile computed by this CTA needs no reduction and no activation: straight to y from the
          // accumulator (the fix-up warps skip it; its publication is batched per segment below)
          const float gsy = (WQ == 2) ? a.g2[ch.expert] : 1.f;   // NVFP4 per-expert global scale of w2
          if (FP8) {
#pragma unroll
            for (int na = 0; na < 2; ++na) {
              if (na < nacc) {
                float* yb = a.y + (size_t)ch.row0 * a.H + (size_t)(pair2 ? 2 * j + na : j) * 128 + row_in_tile;
#pragma unroll
                for (int c = 0; c < TNMAX; ++c)
                  if (c < ch.nrows) yb[(size_t)c * a.H] = acc[na][c];
              }
            }
          } else {
            const uint32_t buf = acc_it % C::NBUF;
            f_wait(&tb->tfull[buf], (acc_it / C::NBUF) & 1);
#pragma unroll
            for (int na = 0; na < 2; ++na) {
              if (na < nacc) {
                float* yb = a.y + (size_t)ch.row0 * a.H + (size_t)(pair2 ? 2 * j + na : j) * 128 + row_in_tile;
#pragma unroll
                for (int c16 = 0; c16 < TNMAX / 16; ++c16) {
                  if (c16 * 16 < tn) {
                    float part[16];
                    xch_ld<16>(xch + lane_off + buf * C::BUFCOLS + na * TNMAX + c16 * 16, part);
#pragma unroll
                    for (int c = 0; c < 16; ++c)
                      if (c16 * 16 + c < ch.nrows) yb[(size_t)(c16 * 16 + c) * a.H] = (WQ == 2) ? part[c] * gsy : part[c];
                  }
                }
              }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&tb->tempty[buf]);
            ++acc_it;
          }
          ++pend_y;
          it += k1 - k0;
          continue;
        }
        // park the tile part and hand it to the fix-up warps
        const int qe = part_no % F_QD;
        f_wait(&tb->qempty[qe], ((part_no / F_QD) & 1) ^ 1);
        float* slot = split ? a.partials + ((size_t)(si * G + cta) * 2 + (k0 != 0 ? 0 : 1)) * (size_t)(2 * TNMAX * 128)
                            : a.partials + ((size_t)(4 * G * 2) + (size_t)cta * F_QD + qe) * (size_t)(2 * TNMAX * 128);
        if (FP8) {
#pragma unroll
          for (int na = 0; na < 2; ++na)
            if (na < nacc)
#pragma unroll
              for (int c = 0; c < TNMAX; ++c)
                if (c < ch.nrows) slot[(na * TNMAX + c) * 128 + row_in_tile] = acc[na][c];
        } else {
          // 16-bit MMAs accumulate the whole segment in registers: stream it to the slot 16 columns at a time
          const uint32_t buf = acc_it % C::NBUF;
          f_wait(&tb->tfull[buf], (acc_it / C::NBUF) & 1);
#pragma unroll
          for (int na = 0; na < 2; ++na) {
            if (na < nacc) {
#pragma unroll
              for (int c16 = 0; c16 < TNMAX / 16; ++c16) {
                if (c16 * 16 < tn) {
                  float part[16];
                  xch_ld<16>(xch + lane_off + buf * C::BUFCOLS + na * TNMAX + c16 * 16, part);
#pragma unroll
                  for (int c = 0; c < 16; ++c)
                    if (c16 * 16 + c < ch.nrows) slot[(na * TNMAX + c16 * 16 + c) * 128 + row_in_tile] = part[c];
                }
              }
            }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&tb->tempty[buf]);
          ++acc_it;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&tb->qfull[qe]);
        ++part_no;
        it += k1 - k0;
      }
      // publish the y tiles this segment wrote directly (grid.sync idiom: stores -> bar -> fence + one atomic)
      if (ph == 1) {
        asm volatile("bar.sync 3, 128;" ::: "memory");
        if (tid == 0 && pend_y > 0) {
          __threadfence();
          atomicAdd(&sy->comb[0], pend_y);
        }
        pend_y = 0;
      }
    }
  } else if (warp >= 6 && warp < 10) {
    // ======================================================================= fix-up warps 6..9
    // stream-K reduction, activation / requantisation / publication, combine: everything that has a
    // cross-CTA latency chain runs here, off the streaming path.
    const int ftid = tid - 192;            // 0..127
    const int fwarp = warp - 6;
    const int row_in_tile = ftid;
    uint32_t part_no = 0;
    for (int si = 0; si < sl.n; ++si) {
      const Seg& sg = sl.s[si];
      const int ph = sg.ph;
      const int KI = sg.KI;
      const int J = sg.J;
      const bool two = ph == 0 ? (NA == 2) : pair2;
      const int nacc = (two || WD) ? 2 : 1;
      int pend_chunk = -1, pend_n = 0;   // batched publication of finalised tiles
      int it = sg.begin;
      while (it < sg.end) {
        const int tile = it / KI, k0 = it % KI;
        const int k1 = (KI - k0 < sg.end - it) ? KI : k0 + (sg.end - it);
        const int q = sg.c0 + tile / J, j = tile % J;
        const FChunk ch = tb->chunks[q];
        const int tn = (ch.nrows + 15) & ~15;
        const bool split = (k0 != 0 || k1 != KI);
        if (ph == 1 && !split) {   // whole GEMM2 tile: the drain warps wrote y themselves, nothing was queued
          it += k1 - k0;
          continue;
        }
        const int qe = part_no % F_QD;
        f_wait(&tb->qfull[qe], (part_no / F_QD) & 1);
        bool finalize = true;
        int cf = cta, cl = cta;
        if (split) {
          const int t_begin = tile * KI, t_last = tile * KI + KI - 1;
          cf = part_owner(t_begin, sg.N, sg.P);
          cl = part_owner(t_last, sg.N, sg.P);
          int32_t* cnt = (ph == 0 ? sy->tcnt1 : sy->tcnt2) + (q * J + j);
          if (ftid == 0) {
            const int old = cnt_inc(cnt);
            if (old == cl - cf) *cnt = 0;   // last contributor: hand the counter back clean
            tb->flag = old;
          }
          asm volatile("bar.sync 2, 128;" ::: "memory");
          const int arrived = tb->flag;
          asm volatile("bar.sync 2, 128;" ::: "memory");
          finalize = (arrived == cl - cf);
          if (finalize) __threadfence();  // acquire side of the contributor counter
        }
        // Finalisation runs in blocks of FB token columns so that every array stays in registers: the fix-up warps of
        // the 4-bit variants have 80 registers per thread (64 at 64 columns), and whole-tile arrays (acc[2][32] +
        // tmp[4][32]) would live in local memory, serialising the L2 round trips.  The blocking does not change the order
        // in which a column's partials are summed.
        constexpr int FB = WD ? (TNMAX == 64 ? 4 : 8) : 16;
        if (finalize) {
          const float* own = a.partials + ((size_t)(4 * G * 2) + (size_t)cta * F_QD + qe) * (size_t)(2 * TNMAX * 128);
          // NVFP4 per-expert global scales (gate / up of w13, w2): linear, applied once to the reduced sums
          float gs0 = 1.f, gs1 = 1.f;
          if (WQ == 2) {
            gs0 = ph == 0 ? a.g13[ch.expert * 2] : a.g2[ch.expert];
            gs1 = ph == 0 ? a.g13[ch.expert * 2 + 1] : gs0;
          }
          uint8_t* itb = a.it + (size_t)ch.row0 * a.KB2 * 128;
          const size_t kb_stride = (size_t)(tn >> 3) * 1024;
          for (int c0 = 0; c0 < ch.nrows; c0 += FB) {   // padded token columns are never consumed
            float acc[2][FB];
            if (!split) {
              // whole tile computed by this CTA: one batch of loads from its own hand-over slot
#pragma unroll
              for (int na = 0; na < 2; ++na)
#pragma unroll
                for (int c = 0; c < FB; ++c)
                  acc[na][c] = (na < nacc && c0 + c < ch.nrows) ? __ldcg(own + (na * TNMAX + c0 + c) * 128 + row_in_tile) : 0.f;
            } else if (ch.nrows <= 4) {
              // decode-sized tile (batch 1..4 per expert) split over many CTAs: the partials of up to 16 contributors
              // are fetched in ONE round trip (fixed CTA order -> deterministic sum)
#pragma unroll
              for (int na = 0; na < 2; ++na)
#pragma unroll
                for (int c = 0; c < FB; ++c) acc[na][c] = 0.f;
              for (int cb = cf; cb <= cl; cb += 16) {
#pragma unroll
                for (int na = 0; na < 2; ++na) {
                  if (na < nacc) {
                    float tmp[16][4];
#pragma unroll
                    for (int u = 0; u < 16; ++u) {
                      const int cc = cb + u;
                      const float* src = a.partials + ((size_t)(si * G + cc) * 2 + (cc == cf ? 1 : 0)) * (size_t)(2 * TNMAX * 128);
#pragma unroll
                      for (int c = 0; c < 4; ++c)
                        tmp[u][c] = (cc <= cl && c < ch.nrows) ? __ldcg(src + (na * TNMAX + c) * 128 + row_in_tile) : 0.f;
                    }
#pragma unroll
                    for (int u = 0; u < 16; ++u)
#pragma unroll
                      for (int c = 0; c < 4; ++c) acc[na][c] += tmp[u][c];
                  }
                }
              }
            } else {
#pragma unroll
              for (int na = 0; na < 2; ++na)
#pragma unroll
                for (int c = 0; c < FB; ++c) acc[na][c] = 0.f;
              // fixed CTA order -> deterministic sum; loads of up to 4 contributors are issued back to back
              for (int cb = cf; cb <= cl; cb += 4) {
#pragma unroll
                for (int na = 0; na < 2; ++na) {
                  if (na < nacc) {
                    float tmp[4][FB];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                      const int cc = cb + u;
                      const float* src = a.partials + ((size_t)(si * G + cc) * 2 + (cc == cf ? 1 : 0)) * (size_t)(2 * TNMAX * 128);
#pragma unroll
                      for (int c = 0; c < FB; ++c)
                        tmp[u][c] = (cc <= cl && c0 + c < ch.nrows) ? __ldcg(src + (na * TNMAX + c0 + c) * 128 + row_in_tile) : 0.f;
                    }
#pragma unroll
                    for (int u = 0; u < 4; ++u)
#pragma unroll
                      for (int c = 0; c < FB; ++c) acc[na][c] += tmp[u][c];
                  }
                }
              }
            }
            if (WQ == 2) {
#pragma unroll
              for (int c = 0; c < FB; ++c) {
                acc[0][c] *= gs0;
                acc[1][c] *= gs1;
              }
            }
            if (ph == 0) {
              // -------------------------------------------------------- activation (+FP8 requant) -> tiled intermediate
              float v[FB];
#pragma unroll
              for (int c = 0; c < FB; ++c) {
                const float g0 = round_act(acc[0][c], a.cmp_fp16);
                float r;
                if (NA == 2) {
                  const float u0 = round_act(acc[1][c], a.cmp_fp16);
                  if (a.act_type == 1) {
                    const float gg = fminf(g0, a.limit);
                    const float uu = fminf(fmaxf(u0, -a.limit), a.limit);
                    r = (uu + 1.0f) * __fdividef(gg, 1.0f + __expf(-a.alpha * gg));
                  } else {
                    // SiLU(g) * u, fast intrinsics (fp32, ~1e-6 rel), with DeepSeek-V4's clamp for type 3.  Types 0 and 3
                    // share the instructions: for type 0 the limit is +inf, which leaves every non-NaN value unchanged.
                    const float gg = fminf(g0, a.silu_limit), uu = fminf(fmaxf(u0, -a.silu_limit), a.silu_limit);
                    r = __fdividef(gg, 1.0f + __expf(-gg)) * uu;
                  }
                } else {
                  const float t = fmaxf(g0, 0.f);
                  r = t * t;
                }
                v[c] = round_act(fminf(fmaxf(r, -65504.f), 65504.f), a.cmp_fp16);
              }
              if (FP8) {
#pragma unroll
                for (int c = 0; c < FB; ++c) {
                  const float m = warp_max(fabsf(v[c]));
                  if (lane == 0) tb->red[fwarp][c0 + c] = m;
                }
                asm volatile("bar.sync 2, 128;" ::: "memory");
#pragma unroll
                for (int c = 0; c < FB; ++c) {
                  const int cc = c0 + c;
                  if (cc < ch.nrows) {
                    const float m = fmaxf(fmaxf(tb->red[0][cc], tb->red[1][cc]), fmaxf(tb->red[2][cc], tb->red[3][cc]));
                    const float sc = fp8_group_scale(m, a.e8m0);
                    const __nv_fp8_e4m3 qv(v[c] * (a.e8m0 ? __frcp_rn(sc) : __fdividef(448.0f, fmaxf(m, 1e-10f))));
                    *(itb + j * kb_stride + (cc >> 3) * 1024 + sw128_offset(cc & 7, row_in_tile)) =
                        *reinterpret_cast<const uint8_t*>(&qv);
                    if (row_in_tile == 0) a.is[(size_t)j * a.rows_stride + ch.row0 + cc] = sc;
                  }
                }
                asm volatile("bar.sync 2, 128;" ::: "memory");   // red[] is rewritten by the next block / tile part
              } else {
                const int kb2 = j * 2 + (row_in_tile >> 6);
                const int boff = (row_in_tile & 63) * 2;
#pragma unroll
                for (int c = 0; c < FB; ++c) {
                  const int cc = c0 + c;
                  if (cc < ch.nrows) {
                    uint8_t* dst = itb + kb2 * kb_stride + (cc >> 3) * 1024 + sw128_offset(cc & 7, boff);
                    if (a.cmp_fp16)
                      *reinterpret_cast<__half*>(dst) = __float2half_rn(v[c]);
                    else
                      *reinterpret_cast<__nv_bfloat16*>(dst) = __float2bfloat16_rn(v[c]);
                  }
                }
              }
            } else {
              // -------------------------------------------------------- y tile(s)
#pragma unroll
              for (int na = 0; na < 2; ++na) {
                if (na < nacc) {
                  const int jt = pair2 ? 2 * j + na : j;
                  float* yb = a.y + (size_t)ch.row0 * a.H + (size_t)jt * 128 + row_in_tile;
#pragma unroll
                  for (int c = 0; c < FB; ++c)
                    if (c0 + c < ch.nrows) yb[(size_t)(c0 + c) * a.H] = acc[na][c];
                }
              }
            }
          }
        }
        // the queue entry (and its ring slot) can be reused once the data is in registers
        __syncwarp();
        if (lane == 0) mbar_arrive(&tb->qempty[qe]);
        ++part_no;
        if (finalize) {
          if (ph == 0) {
            // the intermediate is consumed through the async proxy (bulk copy) by other CTAs; publication of
            // finalised tiles is batched per chunk
            asm volatile("fence.proxy.async.global;" ::: "memory");
            if (pend_chunk != q && pend_n > 0) {
              asm volatile("bar.sync 2, 128;" ::: "memory");
              if (ftid == 0) {
                __threadfence();
                atomicAdd(&sy->g1_done[pend_chunk], pend_n);
              }
              pend_n = 0;
            }
            pend_chunk = q;
            ++pend_n;
          } else {
            ++pend_n;   // y tile(s): publication is batched per segment
          }
        }
        it += k1 - k0;
      }
      // flush the batched publication of this segment
      asm volatile("bar.sync 2, 128;" ::: "memory");
      if (ftid == 0 && pend_n > 0) {
        __threadfence();
        if (ph == 0)
          atomicAdd(&sy->g1_done[pend_chunk], pend_n);
        else
          atomicAdd(&sy->comb[0], pend_n);
      }
    }
  }

  // ---------------------------------------------------------------- phase 3: distributed combine (whole CTA)
  // out[t] = sum_j w[t,j] * y[row(t,j)] once every GEMM2 tile of the launch is finalised; every thread of every
  // CTA takes (token, 4-column) units: k float4 loads in flight per thread, fixed j order (deterministic)
  {
    if (tid == 0) cnt_wait(&sy->comb[0], n_chunks * J2e);
    __syncthreads();
    __threadfence();
    const int H4 = a.H >> 2, k = a.top_k;
    const int units = a.M * H4;
    for (int u = cta * NT + tid; u < units; u += G * NT) {
      const int t = u / H4, c4 = u - t * H4;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int j0 = 0; j0 < k; j0 += 8) {
        float4 v[8];
        float w[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int jj = j0 + q;
          const int row = (jj < k) ? tb->row_of_slot[t * k + jj] : -1;
          w[q] = (row >= 0) ? a.topk_w[t * k + jj] : 0.f;
          v[q] = (row >= 0) ? __ldcg(reinterpret_cast<const float4*>(a.y + (size_t)row * a.H) + c4)
                            : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          acc.x = fmaf(w[q], v[q].x, acc.x);
          acc.y = fmaf(w[q], v[q].y, acc.y);
          acc.z = fmaf(w[q], v[q].z, acc.z);
          acc.w = fmaf(w[q], v[q].w, acc.w);
        }
      }
      const size_t o = (size_t)t * a.H + (size_t)c4 * 4;
      if (a.out_dtype == 2) {
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(a.out) + o) = acc;
      } else if (a.out_dtype == 0) {
        const __nv_bfloat162 lo = __floats2bfloat162_rn(acc.x, acc.y), hi = __floats2bfloat162_rn(acc.z, acc.w);
        uint2 pk;
        pk.x = *reinterpret_cast<const uint32_t*>(&lo);
        pk.y = *reinterpret_cast<const uint32_t*>(&hi);
        *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(a.out) + o) = pk;
      } else {
        const __half2 lo = __floats2half2_rn(acc.x, acc.y), hi = __floats2half2_rn(acc.z, acc.w);
        uint2 pk;
        pk.x = *reinterpret_cast<const uint32_t*>(&lo);
        pk.y = *reinterpret_cast<const uint32_t*>(&hi);
        *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(a.out) + o) = pk;
      }
    }
  }

  __syncthreads();
  if (tid == 0) {
    __threadfence();
    const int old = atomicAdd(&sy->finished, 1);
    if (old == G - 1) finish_launch(sy, n_chunks, a.J2);
  }
}

template <bool FP8, int NA, int TNMAX, int WQ>
static int launch_fused_t(const FusedArgs& a, cudaStream_t st, int num_sms) {
  using C = FCfg<FP8, NA, TNMAX, WQ>;
  auto kern = moe_fused_kernel<FP8, NA, TNMAX, WQ>;
  const int rc = kernel_smem(reinterpret_cast<const void*>(kern), C::SMEM, "cudaFuncSetAttribute(moe_fused)");
  if (rc) return rc;
  // Cooperative launch: the cross-CTA spin waits need every CTA of the grid resident at once; a plain launch that
  // shares the GPU with another stream's kernels could be scheduled piecemeal and dead-lock.
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(num_sms);
  cfg.blockDim = dim3(C::NTHREADS);
  cfg.dynamicSmemBytes = C::SMEM;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, a);
  ++g_launches;
  if (e != cudaSuccess) return cuda_fail(e, "moe_fused launch");
  e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "moe_fused launch");
  return 0;
}

bool fused_supported(const b200moe_layer* L, int M, int k) {
  if (L->wq && !(L->gated && L->w2_paired)) return false;
  const long slots = (long)M * k;
  if (slots > FUSED_MAX_SLOTS || L->E > FUSED_MAX_EXPERTS || M > FUSED_MAX_TOKENS) return false;
  // rows bound: slots + 15 per active expert
  const long act = slots < L->E ? slots : L->E;
  if (slots + 15 * act > FUSED_MAX_ROWS) return false;
  const long chunks = act + slots / 16;
  if (chunks > FUSED_MAX_CHUNKS) return false;
  if (L->J2 > FUSED_MAX_J2 || chunks * L->J1 > FUSED_MAX_TILES || chunks * L->J2 > FUSED_MAX_TILES) return false;
  return true;
}

int launch_fused(const b200moe_layer* L, Workspace* ws, cudaStream_t st, const void* hidden, const int32_t* ids,
                 const float* topk_w, int M, int k, void* out, int out_dtype) {
  const int num_sms = device_sms(L->device);
  if (num_sms < 0) return num_sms;
  FusedArgs a{};
  a.w13t = L->w13t;
  a.w2t = L->w2t;
  a.ws13 = L->ws13;
  a.ws2 = L->ws2;
  a.E = L->E;
  a.H = L->H;
  a.I = L->I;
  a.N1 = L->N1;
  a.gated = L->gated;
  a.w2_paired = L->w2_paired;
  a.KB1 = L->KB1;
  a.KB2 = L->KB2;
  a.J1 = L->J1;
  a.J2 = L->J2;
  a.act_type = L->cfg.activation_type;
  a.act_fp16 = (L->act_dtype == B200_ACT_FP16);
  a.e8m0 = L->fp8_e8m0;
  a.cmp_fp16 = (a.act_fp16 || L->wq) ? 1 : 0;
  a.w4_tile_bytes = L->w4_tile_bytes;
  a.w4_scale_bytes = L->w4_scale_bytes;
  a.g13 = L->g13;
  a.g2 = L->g2;
  a.alpha = L->cfg.swiglu_alpha;
  a.limit = L->cfg.swiglu_limit;
  a.silu_limit = L->cfg.activation_type == 3 ? L->cfg.swiglu_limit : INFINITY;
  a.hidden = reinterpret_cast<const uint16_t*>(hidden);
  a.ids = ids;
  a.topk_w = topk_w;
  a.out = out;
  a.out_dtype = out_dtype;
  a.M = M;
  a.top_k = k;
  a.xt = ws->xt;
  a.xs = ws->xs;
  a.it = ws->it;
  a.is = ws->is;
  a.y = ws->y;
  a.partials = ws->partials;
  a.sync = ws->fsync;
  a.rows_stride = (int)ws->cap_rows;
  const char* g1 = getenv("B200MOE_ALIGN_G1");
  a.align_g1 = g1 ? atoi(g1) : 60;   // percent of the CTA slots whole GEMM1 tiles must fill (0: always stream-K)
  const bool fp8 = L->esz_bits == 8;
  // experts with more rows are processed in chunks of TNMAX; 4-bit layers take chunks of up to 64 rows, so that at
  // M <= 64 every active expert's weights are streamed once
  const int tn = M <= 16 ? 16 : 32;
  const int tn4 = M <= 16 ? 16 : M <= 32 ? 32 : 64;
#define F_DISPATCH(FP8_, NA_)                                          \
  switch (tn) {                                                        \
    case 16: return launch_fused_t<FP8_, NA_, 16, 0>(a, st, num_sms);  \
    default: return launch_fused_t<FP8_, NA_, 32, 0>(a, st, num_sms);  \
  }
#define F_DISPATCH_W4(WQ_)                                             \
  switch (tn4) {                                                       \
    case 16: return launch_fused_t<false, 2, 16, WQ_>(a, st, num_sms); \
    case 32: return launch_fused_t<false, 2, 32, WQ_>(a, st, num_sms); \
    default: return launch_fused_t<false, 2, 64, WQ_>(a, st, num_sms); \
  }
  if (L->wq == 1) { F_DISPATCH_W4(1) }
  if (L->wq == 2) { F_DISPATCH_W4(2) }
  if (L->wq == 3) { F_DISPATCH_W4(3) }
  if (L->gated) {
    if (fp8) { F_DISPATCH(true, 2) } else { F_DISPATCH(false, 2) }
  } else {
    if (fp8) { F_DISPATCH(true, 1) } else { F_DISPATCH(false, 1) }
  }
#undef F_DISPATCH
#undef F_DISPATCH_W4
}

}  // namespace b200
