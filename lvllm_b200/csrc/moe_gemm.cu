// Grouped expert GEMM on sm_90a: weight-streaming, swap-AB, wgmma.
//
// Y_e^T[n, t] = sum_k W_e[n, k] * X[t, k]       (n = output feature, t = permuted token row)
//
// The 128-row weight tile is the MMA *A* operand (M = 128: two M = 64 wgmma), the tokens of one expert are the *B*
// operand (N = the chunk size TNMAX), so one pass over an expert's weights serves all of its tokens and the tensor
// core never limits the stream.  Weights live in HBM pre-tiled as [128 rows x 128 B] blocks that already
// carry the 128-byte swizzle, so a pipeline stage is ONE contiguous 32 KB bulk async copy (UBLKCP) — no
// tensor maps, perfect DRAM page locality.  Activations are pre-tiled the same way by the prep kernel.
//
// Warp roles (384 threads, 1 CTA / SM, persistent, dynamic unit scheduler):
//   warps 0-3  epilogue: accumulators from the exchange area, block-scale promotion (FP8), activation,
//              re-quantisation and stores
//   warp  4    producer: bulk copies global -> smem ring, full/empty mbarriers; also owns the scheduler
//   warps 8-11 MMA warpgroup: wgmma with register accumulators; a finished accumulator is parked in the exchange
//              area (common.cuh) for the epilogue warps, and the next one is computed while they work on it
//
// Chunks are at most 64 token rows: the gate + up accumulators of a chunk (2 x 128 x 64 fp32) are what the MMA
// warpgroup holds in registers and one exchange buffer holds in shared memory next to the pipeline stages.
//
// FP8 (W8A8, DeepSeek block-128 numerics): each 128-wide k-block is a fresh accumulation; the epilogue warps fold
// part * w_scale[n/128,kb] * x_scale[t,kb]  into fp32 registers.  16-bit formats accumulate the whole K in the MMA
// warpgroup's registers.  FP8 layers in ue8m0 mode (power-of-two block scales, the reference's DeepGEMM numerics:
// vllm/utils/deep_gemm.py:662-681 per_block_cast_to_fp8(use_ue8m0), fp8_utils.py:112, :986-1043) take the same path: their
// scales are fp32 powers of two.
//
// Roofline: HBM.  Algorithmic bytes per unit = weight tile bytes (activations are <1%).
#include "common.cuh"
#include "moe_internal.cuh"

namespace b200 {

constexpr int NUM_EPI_WARPS = 4;   // one warp per 32-row quarter of the tile
constexpr int GEMM_THREADS = 384;
constexpr int MMA_WARP0 = 8;    // first warp of the MMA warpgroup
constexpr int QDEPTH = 4;       // scheduler queue depth
constexpr int KBG = 28;         // k-blocks whose FP8 scales are staged in shared memory at a time
constexpr int SMEM_BUDGET = 225 * 1024;
constexpr int XCH_BUDGET = 64 * 1024;   // exchange area: two accumulator buffers, or one of a 64-row gated chunk

enum { EPI_GATED = 0, EPI_ACT1 = 1, EPI_OUT = 2 };

struct GemmArgs {
  const uint8_t* wt;    // tiled weights
  const float* wscale;  // [E][NB][KB] (fp8) or nullptr
  const uint8_t* bt;    // tiled B operand (activations)   [rows/8][KB][1024]
  const float* bscale;  // [KB][rows_stride] (fp8)
  uint8_t* it;          // tiled intermediate out (EPI_GATED / EPI_ACT1)
  float* iscale;        // [KB2][rows_stride]
  float* y;             // [rows][n_out] fp32 (EPI_OUT)
  const Chunk* chunks;
  RouteState* state;
  int which;            // 0: GEMM1, 1: GEMM2 (selects the scheduler counter)
  int KB;               // k-blocks (128 B) of this GEMM
  int J;                // output tiles per expert
  int NB;               // scale row-blocks per expert (fp8): N_total/128
  int up_block_off;     // scale row-block offset of the "up" half (= I/128) for EPI_GATED
  int KB_out;           // k-blocks of the NEXT GEMM's operand (intermediate width / elems-per-128B)
  int rows_stride;      // stride of the transposed scale arrays
  int n_out;            // leading dim of y
  int act_type;         // 0 silu, 1 swigluoai, 2 relu2, 3 silu with clamp
  float alpha, limit, silu_limit;   // silu_limit: type 3's clamp, +inf for plain SiLU (type 0)
  int act_fp16;         // activation dtype of the 16-bit intermediate: 0 bf16, 1 fp16
  int e8m0;             // FP8 layers in ue8m0 mode: activation / intermediate group scales are rounded up to powers of two
};

enum { MODE_16 = 0, MODE_FP8 = 1 };

template <int MODE, int NA, int TNMAX>
struct Cfg {
  static constexpr int KBS = 2 / NA;                       // k-blocks per stage
  static constexpr int A_STAGE = 2 * TILE_BYTES;           // 32 KB
  static constexpr int B_STAGE = KBS * TNMAX * 128;        // activation bytes per stage
  static constexpr int STAGE = A_STAGE + B_STAGE;
  static constexpr int MISC = 21504;
  static constexpr int BUFCOLS = NA * TNMAX;               // columns of one accumulator buffer
  static constexpr int BUF_BYTES = BUFCOLS * 128 * 4;
  static constexpr int NBUF = XCH_BUDGET / BUF_BYTES > 2 ? 2 : XCH_BUDGET / BUF_BYTES;
  static constexpr int XCH = NBUF * BUF_BYTES;
  static constexpr int STAGES_RAW = (SMEM_BUDGET - MISC - XCH - 1024) / STAGE;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM = STAGES * STAGE + XCH + MISC + 1024;
  static_assert(NBUF >= 1 && STAGES >= 2, "shared-memory budget");
};

struct __align__(16) Misc {
  uint64_t full[8], empty[8];
  uint64_t tfull[2], tempty[2];
  uint64_t qfull[QDEPTH], qempty[QDEPTH];
  int32_t qunit[QDEPTH];
  float red[NUM_EPI_WARPS][128];   // [row quarter][token column]
  alignas(16) float gsx[KBG][128];   // FP8: activation scales of the current group of k-blocks [k-block][token column]
  float gws[2][KBG];                 // FP8: weight block scales of the group [gate|up][k-block]
};

B200_DEVICE void bounded_wait(uint64_t* bar, uint32_t parity) {
  // A protocol bug must not hang the GPU: trap after ~2^27 polls (seconds).
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 27)) __trap();
  }
}

B200_DEVICE float silu_f(float x) { return x / (1.0f + expf(-x)); }

template <int MODE, int NA, int EPI, int TNMAX>
__global__ void __launch_bounds__(GEMM_THREADS, 1) moe_gemm_kernel(const GemmArgs a) {
  using C = Cfg<MODE, NA, TNMAX>;
  constexpr bool FP8 = (MODE != MODE_16);        // 8-bit operands, fp8 intermediate + group scales; fp32 block scales
                                                 // are applied per k-block by the epilogue warps
  constexpr int CW = TNMAX;                      // token columns per epilogue thread
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t xch = xch_base(smem + C::STAGES * C::STAGE);
  Misc* ms = reinterpret_cast<Misc*>(smem + C::STAGES * C::STAGE + C::XCH);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < C::STAGES; ++i) {
      mbar_init(&ms->full[i], 1);
      mbar_init(&ms->empty[i], 1);
    }
    for (int i = 0; i < C::NBUF; ++i) {
      mbar_init(&ms->tfull[i], 128);             // every MMA thread, after parking its fragment
      mbar_init(&ms->tempty[i], NUM_EPI_WARPS);
    }
    for (int i = 0; i < QDEPTH; ++i) {
      mbar_init(&ms->qfull[i], 1);
      mbar_init(&ms->qempty[i], 128 + NUM_EPI_WARPS);   // MMA threads + one lane per epilogue warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int n_units = a.state->n_chunks * a.J;
  const int KB = a.KB;
  const int n_iters = (KB + C::KBS - 1) / C::KBS;  // pipeline iterations per unit

  if (warp == 4) {
    // ======================================================================= producer + scheduler
    if (elect_one()) {
      const uint64_t pol = policy_evict_first();
      uint32_t it = 0, q = 0;
      for (;;) {
        const int u = atomicAdd(&a.state->unit_ctr[a.which], 1);
        const int qs = q % QDEPTH;
        bounded_wait(&ms->qempty[qs], ((q / QDEPTH) & 1) ^ 1);
        ms->qunit[qs] = (u < n_units) ? u : -1;
        mbar_arrive(&ms->qfull[qs]);
        ++q;
        if (u >= n_units) break;
        const int ci = u / a.J, j = u % a.J;
        const Chunk ch = a.chunks[ci];
        const int tn = (ch.nrows + 15) & ~15;
        const uint8_t* wsrc = a.wt + ((size_t)(ch.expert * a.J + j) * KB) * (size_t)(NA * TILE_BYTES);
        for (int i = 0; i < n_iters; ++i, ++it) {
          const int s = it % C::STAGES;
          bounded_wait(&ms->empty[s], ((it / C::STAGES) & 1) ^ 1);
          const int kb0 = i * C::KBS;
          const int nkb = (KB - kb0 < C::KBS) ? (KB - kb0) : C::KBS;
          const uint32_t abytes = nkb * NA * TILE_BYTES;
          const uint32_t bbytes = (tn >> 3) * nkb * 1024;
          uint8_t* sa = smem + s * C::STAGE;
          uint8_t* sb = sa + C::A_STAGE;
          mbar_arrive_expect_tx(&ms->full[s], abytes + bbytes);
          bulk_g2s_hint(sa, wsrc + (size_t)kb0 * (NA * TILE_BYTES), abytes, &ms->full[s], pol);
          // the chunk's activation tiles are chunk-contiguous ([k-block][row group][1 KB]): ONE bulk copy per stage
          bulk_g2s(sb, a.bt + (size_t)ch.row0 * KB * 128 + (size_t)kb0 * (size_t)((tn >> 3) * 1024), bbytes, &ms->full[s]);
        }
      }
    }
  } else if (warp >= MMA_WARP0) {
    // ======================================================================= MMA warpgroup
    // The instruction shape is fixed at N = TNMAX columns: columns beyond the chunk's rows multiply whatever the stage
    // holds there and are never read.  acc[na][h]: accumulator na (gate | up, or tile of a w2 pair), rows [64h, 64h + 64).
    float acc[NA][2][TNMAX / 2];
    uint32_t it = 0, q = 0, acc_it = 0;
    // hand the finished accumulators to the epilogue warps; the buffer is waited for only now, so the MMAs of this
    // accumulation ran while the epilogue was still reading the previous one
    auto park = [&]() {
      const uint32_t buf = acc_it % C::NBUF;
      bounded_wait(&ms->tempty[buf], ((acc_it / C::NBUF) & 1) ^ 1);
#pragma unroll
      for (int na = 0; na < NA; ++na)
#pragma unroll
        for (int h = 0; h < 2; ++h) xch_store_frag<TNMAX>(xch + buf * C::BUFCOLS + na * TNMAX, h, acc[na][h]);
      mbar_arrive(&ms->tfull[buf]);
      ++acc_it;
    };
    for (;;) {
      const int qs = q % QDEPTH;
      bounded_wait(&ms->qfull[qs], (q / QDEPTH) & 1);
      const int u = ms->qunit[qs];
      mbar_arrive(&ms->qempty[qs]);
      ++q;
      if (u < 0) break;
      const int tn = (a.chunks[u / a.J].nrows + 15) & ~15;
      for (int i = 0; i < n_iters; ++i, ++it) {
        const int s = it % C::STAGES;
        bounded_wait(&ms->full[s], (it / C::STAGES) & 1);
        const int kb0 = i * C::KBS;
        const int nkb = (KB - kb0 < C::KBS) ? (KB - kb0) : C::KBS;
        const uint32_t sa = smem_u32(smem + s * C::STAGE);
        const uint32_t sb = sa + C::A_STAGE;
        for (int kk = 0; kk < nkb; ++kk) {
          wgmma_fence();
#pragma unroll
          for (int na = 0; na < NA; ++na) {
            // stage layout: NA==2 -> [gate tile][up tile] of one k-block; NA==1 -> [kb0 tile][kb1 tile]
            const uint32_t abase = sa + (NA == 2 ? na : kk) * TILE_BYTES;
            const uint32_t bbase = sb + kk * (uint32_t)((tn >> 3) * 1024);
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
              const uint32_t accum = FP8 ? (ks > 0) : ((kb0 + kk) > 0 || ks > 0);
              if (FP8)
                wgmma_tile128<TNMAX, 2>(acc[na], abase + ks * 32, bbase + ks * 32, accum);
              else if (a.act_fp16)
                wgmma_tile128<TNMAX, 0>(acc[na], abase + ks * 32, bbase + ks * 32, accum);
              else
                wgmma_tile128<TNMAX, 1>(acc[na], abase + ks * 32, bbase + ks * 32, accum);
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
          if (FP8) park();
        }
        if (threadIdx.x == MMA_WARP0 * 32) mbar_arrive(&ms->empty[s]);
      }
      if (!FP8) park();
    }
  } else if (warp < NUM_EPI_WARPS) {
    // ======================================================================= epilogue warps 0..3
    uint32_t q = 0, acc_it = 0;
    const int q4 = warp;                         // 32-row quarter of the tile this warp reads
    constexpr int c_base = 0;
    const uint32_t lane_off = (uint32_t)(q4 * 32) << 16;
    const int row_in_tile = q4 * 32 + lane;  // output feature within the 128-row tile
    for (;;) {
      const int qs = q % QDEPTH;
      bounded_wait(&ms->qfull[qs], (q / QDEPTH) & 1);
      const int u = ms->qunit[qs];
      __syncwarp();
      if (lane == 0) mbar_arrive(&ms->qempty[qs]);
      ++q;
      if (u < 0) break;
      const int ci = u / a.J, j = u % a.J;
      const Chunk ch = a.chunks[ci];
      const int tn = (ch.nrows + 15) & ~15;

      float acc[NA][CW];
#pragma unroll
      for (int na = 0; na < NA; ++na)
#pragma unroll
        for (int c = 0; c < CW; ++c) acc[na][c] = 0.f;

      const int n_groups = FP8 ? KB : 1;
      // FP8: the scales of KBG k-blocks at a time are staged in shared memory by ALL epilogue threads (one global
      // latency per group instead of one per k-block: a prefetch distance of one k-block cannot cover a global load's
      // latency), pre-multiplied: gsx[kk][c] = x_scale[token c, k-block], gws[na][kk]
      const float* wrow[NA];
      const int etid = threadIdx.x;
      if (FP8) {
#pragma unroll
        for (int na = 0; na < NA; ++na) {
          const int rb = (EPI == EPI_GATED) ? (na == 0 ? j : a.up_block_off + j) : (NA == 2 ? 2 * j + na : j);
          wrow[na] = a.wscale + ((size_t)ch.expert * a.NB + rb) * KB;
        }
      }
      for (int g = 0; g < n_groups; ++g) {
        const uint32_t buf = acc_it % C::NBUF;
        const int rel = g % KBG;
        if (FP8 && rel == 0) {
          asm volatile("bar.sync 2, 128;" ::: "memory");   // every epilogue warp is done with the old group
          const int n = (n_groups - g < KBG) ? n_groups - g : KBG;
          for (int i = etid; i < n * TNMAX; i += 128) {
            const int kk = i / TNMAX, c = i - kk * TNMAX;
            ms->gsx[kk][c] = (c < tn) ? __ldg(a.bscale + (size_t)(g + kk) * a.rows_stride + ch.row0 + c) : 0.f;
          }
          for (int i = etid; i < NA * n; i += 128) {
            const int na = i / n, kk = i - na * n;
            ms->gws[na][kk] = __ldg(wrow[na] + g + kk);
          }
          asm volatile("bar.sync 2, 128;" ::: "memory");
        }
        bounded_wait(&ms->tfull[buf], (acc_it / C::NBUF) & 1);
        if (FP8) {
          // gate and up partial sums of the same token columns are promoted with  part * (w_scale[na] * x_scale[token])
          float ws_cur[NA];
#pragma unroll
          for (int na = 0; na < NA; ++na) ws_cur[na] = ms->gws[na][rel];
          const float* sxw = &ms->gsx[rel][c_base];
#pragma unroll
          for (int c8 = 0; c8 < CW / 8; ++c8) {
            if (c_base + c8 * 8 < tn) {
              float part[NA][8];
#pragma unroll
              for (int na = 0; na < NA; ++na)
                xch_ld<8>(xch + lane_off + buf * C::BUFCOLS + na * TNMAX + c_base + c8 * 8, part[na]);
#pragma unroll
              for (int c4 = 0; c4 < 2; ++c4) {
                const float4 xs4 = *reinterpret_cast<const float4*>(sxw + c8 * 8 + c4 * 4);
                const float xv[4] = {xs4.x, xs4.y, xs4.z, xs4.w};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
#pragma unroll
                  for (int na = 0; na < NA; ++na)
                    acc[na][c8 * 8 + c4 * 4 + q] = fmaf(part[na][c4 * 4 + q], ws_cur[na] * xv[q], acc[na][c8 * 8 + c4 * 4 + q]);
                }
              }
            }
          }
        } else {
#pragma unroll
          for (int na = 0; na < NA; ++na) {
#pragma unroll
            for (int c16 = 0; c16 < CW / 16; ++c16) {
              if (c_base + c16 * 16 < tn) {
                float part[16];
                xch_ld<16>(xch + lane_off + buf * C::BUFCOLS + na * TNMAX + c_base + c16 * 16, part);
#pragma unroll
                for (int c = 0; c < 16; ++c) acc[na][c16 * 16 + c] = part[c];
              }
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&ms->tempty[buf]);
        ++acc_it;
      }

      // ------------------------------------------------------------------ final epilogue of the unit
      if (EPI == EPI_OUT) {
        // NA == 2: paired layout, accumulator na is output tile 2j+na
#pragma unroll
        for (int na = 0; na < NA; ++na) {
          const int jt = (NA == 2) ? 2 * j + na : j;
          float* yb = a.y + (size_t)ch.row0 * a.n_out + (size_t)jt * 128 + row_in_tile;
#pragma unroll
          for (int c = 0; c < CW; ++c)
            if (c_base + c < ch.nrows) yb[(size_t)(c_base + c) * a.n_out] = acc[na][c];
        }
      } else {
        // activation in fp32 on values rounded to the activation dtype (matches the reference chain:
        // GEMM output -> act dtype -> act -> act dtype -> (fp8 group quant))
        float v[CW];
#pragma unroll
        for (int c = 0; c < CW; ++c) {
          float g0, r;
          if (a.act_fp16)
            g0 = __half2float(__float2half_rn(acc[0][c]));
          else
            g0 = __bfloat162float(__float2bfloat16_rn(acc[0][c]));
          if (EPI == EPI_GATED) {
            float u0;
            if (a.act_fp16)
              u0 = __half2float(__float2half_rn(acc[NA - 1][c]));
            else
              u0 = __bfloat162float(__float2bfloat16_rn(acc[NA - 1][c]));
            if (a.act_type == 1) {
              const float gg = fminf(g0, a.limit);
              const float uu = fminf(fmaxf(u0, -a.limit), a.limit);
              r = (uu + 1.0f) * gg * (1.0f / (1.0f + expf(-a.alpha * gg)));
            } else {
              // SiLU, with DeepSeek-V4's clamp for type 3; for type 0 the limit is +inf (every non-NaN value unchanged)
              r = silu_f(fminf(g0, a.silu_limit)) * fminf(fmaxf(u0, -a.silu_limit), a.silu_limit);
            }
          } else {
            const float t = fmaxf(g0, 0.f);
            r = t * t;
          }
          if (a.act_fp16)
            v[c] = __half2float(__float2half_rn(r));
          else
            v[c] = __bfloat162float(__float2bfloat16_rn(r));
        }
        if (FP8) {
          // per-token group-128 quantisation: the 128 features of this tile are exactly one group
#pragma unroll
          for (int c = 0; c < CW; ++c) {
            if (c_base + c < tn) {
              const float m = warp_max(fabsf(v[c]));
              if (lane == 0) ms->red[q4][c_base + c] = m;
            }
          }
          asm volatile("bar.sync 1, 128;" ::: "memory");
          const int kb2 = j;  // 128 features == one 128-B k-block of the next GEMM
#pragma unroll
          for (int c = 0; c < CW; ++c) {
            const int cc = c_base + c;
            if (cc < ch.nrows) {
              float m = fmaxf(fmaxf(ms->red[0][cc], ms->red[1][cc]), fmaxf(ms->red[2][cc], ms->red[3][cc]));
              const float sc = fp8_group_scale(m, a.e8m0);
              const int r = ch.row0 + cc;
              const __nv_fp8_e4m3 qv(v[c] / sc);
              uint8_t* dst = a.it + (size_t)ch.row0 * a.KB_out * 128 + (size_t)kb2 * (size_t)((tn >> 3) * 1024) +
                             (size_t)(cc >> 3) * 1024 + sw128_offset(cc & 7, row_in_tile);
              *dst = *reinterpret_cast<const uint8_t*>(&qv);
              if (row_in_tile == 0) a.iscale[(size_t)kb2 * a.rows_stride + r] = sc;
            }
          }
          asm volatile("bar.sync 1, 128;" ::: "memory");
        } else {
          const int kb2 = j * 2 + (row_in_tile >> 6);  // 64 16-bit features per 128-B k-block
          const int boff = (row_in_tile & 63) * 2;
#pragma unroll
          for (int c = 0; c < CW; ++c) {
            if (c_base + c < ch.nrows) {
              const int r = ch.row0 + c_base + c;
              const int cc = c_base + c;
              uint8_t* dst = a.it + (size_t)ch.row0 * a.KB_out * 128 + (size_t)kb2 * (size_t)((tn >> 3) * 1024) +
                             (size_t)(cc >> 3) * 1024 + sw128_offset(cc & 7, boff);
              if (a.act_fp16)
                *reinterpret_cast<__half*>(dst) = __float2half_rn(v[c]);
              else
                *reinterpret_cast<__nv_bfloat16*>(dst) = __float2bfloat16_rn(v[c]);
            }
          }
        }
      }
    }
  }

}

template <int MODE, int NA, int EPI, int TNMAX>
static int launch_one(const GemmArgs& a, cudaStream_t st, int num_sms) {
  using C = Cfg<MODE, NA, TNMAX>;
  auto kern = moe_gemm_kernel<MODE, NA, EPI, TNMAX>;
  const int rc = kernel_smem(reinterpret_cast<const void*>(kern), C::SMEM, "cudaFuncSetAttribute(moe_gemm)");
  if (rc) return rc;
  kern<<<num_sms, GEMM_THREADS, C::SMEM, st>>>(a);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "moe_gemm launch");
  return 0;
}

template <int MODE, int TNMAX>
static int launch_pair(const b200moe_layer* L, Workspace* ws, cudaStream_t st, int num_sms, cudaEvent_t* ev) {
  GemmArgs g1{};
  g1.wt = L->w13t;
  g1.wscale = L->ws13;
  g1.bt = ws->xt;
  g1.bscale = ws->xs;
  g1.it = ws->it;
  g1.iscale = ws->is;
  g1.y = nullptr;
  g1.chunks = ws->chunks;
  g1.state = ws->state;
  g1.which = 0;
  g1.KB = L->KB1;
  g1.J = L->J1;
  g1.NB = L->N1 / 128;
  g1.up_block_off = L->I / 128;
  g1.KB_out = L->KB2;
  g1.rows_stride = (int)ws->cap_rows;
  g1.n_out = 0;
  g1.act_type = L->cfg.activation_type;
  g1.alpha = L->cfg.swiglu_alpha;
  g1.limit = L->cfg.swiglu_limit;
  g1.silu_limit = L->cfg.activation_type == 3 ? L->cfg.swiglu_limit : INFINITY;
  g1.act_fp16 = (L->act_dtype == B200_ACT_FP16);
  g1.e8m0 = L->fp8_e8m0;
  int rc;
  if (ev) cudaEventRecord(ev[0], st);
  if (L->gated)
    rc = launch_one<MODE, 2, EPI_GATED, TNMAX>(g1, st, num_sms);
  else
    rc = launch_one<MODE, 1, EPI_ACT1, TNMAX>(g1, st, num_sms);
  if (rc) return rc;
  if (ev) cudaEventRecord(ev[1], st);

  GemmArgs g2 = g1;
  g2.wt = L->w2t;
  g2.wscale = L->ws2;
  g2.bt = ws->it;
  g2.bscale = ws->is;
  g2.it = nullptr;
  g2.iscale = nullptr;
  g2.y = ws->y;
  g2.which = 1;
  g2.KB = L->KB2;
  g2.J = L->J2;
  g2.NB = L->H / 128;
  g2.up_block_off = 0;
  g2.KB_out = 0;
  g2.n_out = L->H;
  if (L->w2_paired) {
    g2.J = L->J2 / 2;
    rc = launch_one<MODE, 2, EPI_OUT, TNMAX>(g2, st, num_sms);
  } else {
    rc = launch_one<MODE, 1, EPI_OUT, TNMAX>(g2, st, num_sms);
  }
  if (ev) cudaEventRecord(ev[2], st);
  return rc;
}

// chunk size (token rows of one expert per pass over its weights): 64 at most, see the head of this file
int pick_tn_max(int M, int k, int E) {
  (void)k;
  (void)E;
  if (M <= 16) return 16;
  if (M <= 32) return 32;
  return 64;
}

int launch_gemms(const b200moe_layer* L, Workspace* ws, cudaStream_t st, int M, int k, int tn_max, cudaEvent_t* ev) {
  const int num_sms = device_sms(L->device);
  if (num_sms < 0) return num_sms;
  const bool fp8 = (L->esz_bits == 8);
  switch (tn_max) {
    case 16: return fp8 ? launch_pair<MODE_FP8, 16>(L, ws, st, num_sms, ev) : launch_pair<MODE_16, 16>(L, ws, st, num_sms, ev);
    case 32: return fp8 ? launch_pair<MODE_FP8, 32>(L, ws, st, num_sms, ev) : launch_pair<MODE_16, 32>(L, ws, st, num_sms, ev);
    default: return fp8 ? launch_pair<MODE_FP8, 64>(L, ws, st, num_sms, ev) : launch_pair<MODE_16, 64>(L, ws, st, num_sms, ev);
  }
}

}  // namespace b200
