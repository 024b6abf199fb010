// Routing bookkeeping around the expert GEMMs (HBM/latency-bound integer + byte work):
//   route_sort_kernel   stable counting sort of the (token,k) slots by local expert id -> padded permuted
//                       rows, chunk table, scheduler reset.  Deterministic: order = (expert, slot).
//   gather_rows_kernel  gathers the hidden rows of every permuted row into the 128B-swizzled tiled layout
//                       the MMA B operand wants; FP8 layers also quantise per token per 128 (vLLM
//                       per_token_group_quant_fp8 semantics, reference tests/kernels/quant_utils.py:157-180).
//   combine_kernel      out[t] = sum_j w[t,j] * y[row(t,j)]  in fp32, fixed j order (reference
//                       finalizeMoeRoutingKernel, moe_permute_unpermute_kernel.inl:92-167).
#include "common.cuh"
#include "moe_internal.cuh"

namespace b200 {

constexpr int SORT_THREADS = 512;

// exclusive scan over the experts of (padded rows, chunk count) from the per-expert slot counts in shared memory, chunk
// table, scheduler reset and slot_of_row = -1; one CTA of SORT_THREADS threads (shared by the single-CTA sort and the
// scan step of the multi-CTA sort)
B200_DEVICE void route_scan_tables(const int* cnt, int* off, int* choff, int (*warp_tot)[SORT_THREADS / 32], int* totals, int E,
                                   int tn_max, int32_t* __restrict__ slot_of_row, int32_t* __restrict__ pad_off_out,
                                   Chunk* __restrict__ chunks, RouteState* __restrict__ state) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // exclusive scan over experts of (padded rows, chunk count); each thread owns a contiguous span
  const int per = (E + SORT_THREADS - 1) / SORT_THREADS;
  const int e0 = tid * per;
  int lrows = 0, lch = 0;
  for (int i = 0; i < per; ++i) {
    const int e = e0 + i;
    if (e < E) {
      lrows += (cnt[e] + ROW_ALIGN - 1) & ~(ROW_ALIGN - 1);
      lch += (cnt[e] + tn_max - 1) / tn_max;
    }
  }
  int irows = lrows, ich = lch;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int a = __shfl_up_sync(0xffffffffu, irows, o);
    const int b = __shfl_up_sync(0xffffffffu, ich, o);
    if (lane >= o) {
      irows += a;
      ich += b;
    }
  }
  if (lane == 31) {
    warp_tot[0][warp] = irows;
    warp_tot[1][warp] = ich;
  }
  __syncthreads();
  int brows = 0, bch = 0;
  for (int w = 0; w < warp; ++w) {
    brows += warp_tot[0][w];
    bch += warp_tot[1][w];
  }
  int xrows = brows + irows - lrows, xch = bch + ich - lch;
  for (int i = 0; i < per; ++i) {
    const int e = e0 + i;
    if (e < E) {
      off[e] = xrows;
      choff[e] = xch;
      pad_off_out[e] = xrows;
      const int c = cnt[e];
      const int nch = (c + tn_max - 1) / tn_max;
      for (int q = 0; q < nch; ++q) {
        Chunk ch;
        ch.expert = e;
        ch.row0 = xrows + q * tn_max;
        ch.nrows = min(tn_max, c - q * tn_max);
        ch.pad = 0;
        chunks[xch + q] = ch;
      }
      xrows += (c + ROW_ALIGN - 1) & ~(ROW_ALIGN - 1);
      xch += nch;
    }
  }
  if (tid == SORT_THREADS - 1) {
    totals[0] = brows + irows;
    totals[1] = bch + ich;
  }
  __syncthreads();
  const int total_rows = totals[0];
  if (tid == 0) {
    pad_off_out[E] = total_rows;
    state->n_chunks = totals[1];
    state->n_rows_padded = total_rows;
    state->unit_ctr[0] = 0;
    state->unit_ctr[1] = 0;
    state->done_ctr[0] = 0;
    state->done_ctr[1] = 0;
  }
  for (int r = tid; r < total_rows; r += SORT_THREADS) slot_of_row[r] = -1;
  __syncthreads();

}

__global__ void __launch_bounds__(SORT_THREADS, 1)
    route_sort_kernel(const int32_t* __restrict__ ids, int n_slots, int E, int tn_max,
                      int32_t* __restrict__ row_of_slot, int32_t* __restrict__ slot_of_row,
                      int32_t* __restrict__ pad_off_out, Chunk* __restrict__ chunks, RouteState* __restrict__ state) {
  __shared__ int cnt[MAX_EXPERTS];
  __shared__ int off[MAX_EXPERTS];    // padded row offset of each expert
  __shared__ int choff[MAX_EXPERTS];  // chunk offset of each expert
  __shared__ int run[MAX_EXPERTS];
  __shared__ int warp_tot[2][SORT_THREADS / 32];
  __shared__ int totals[2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  for (int e = tid; e < E; e += SORT_THREADS) {
    cnt[e] = 0;
    run[e] = 0;
  }
  __syncthreads();
#pragma unroll 4
  for (int s = tid; s < n_slots; s += SORT_THREADS) {
    const int e = ids[s];
    if (e >= 0 && e < E) atomicAdd(&cnt[e], 1);
  }
  __syncthreads();

  route_scan_tables(cnt, off, choff, warp_tot, totals, E, tn_max, slot_of_row, pad_off_out, chunks, state);

  // stable rank without block-wide serialisation: warp w ranks a CONTIGUOUS range of slots with warp-private
  // per-expert counters (dynamic shared memory [warps][E]), the counters are prefix-summed over the warps per
  // expert, then every slot's row = off[e] + (slots of e in earlier warps) + (rank inside its warp).  Order =
  // (expert, slot): identical to the serial counting sort.
  extern __shared__ int wcnt[];   // [NW][E]
  constexpr int NW = SORT_THREADS / 32;
  for (int i = tid; i < NW * E; i += SORT_THREADS) wcnt[i] = 0;
  __syncthreads();
  const int spw = ((n_slots + NW - 1) / NW + 31) & ~31;   // slots per warp
  {
    const int s_end = min(n_slots, (warp + 1) * spw);
    for (int s0 = warp * spw; s0 < s_end; s0 += 128) {
      int ev[4];   // four independent id loads in flight per lane (a 65 536-slot prefill batch is 128 rounds per warp)
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int s = s0 + u * 32 + lane;
        ev[u] = (s < s_end) ? ids[s] : -1;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int s = s0 + u * 32 + lane;
        int e = ev[u];
        if (e < 0 || e >= E) e = -1;
        const unsigned m = __match_any_sync(0xffffffffu, e);
        const int rank = __popc(m & ((1u << lane) - 1u));
        const int base = (e >= 0) ? wcnt[warp * E + e] : 0;
        __syncwarp();
        if (e >= 0 && rank == 0) wcnt[warp * E + e] = base + __popc(m);
        __syncwarp();
        if (s < s_end) row_of_slot[s] = (e >= 0) ? base + rank : -1;   // rank inside (warp, expert) for now
      }
    }
  }
  __syncthreads();
  for (int e = tid; e < E; e += SORT_THREADS) {
    int acc = 0;
    for (int w = 0; w < NW; ++w) {
      const int c = wcnt[w * E + e];
      wcnt[w * E + e] = acc;
      acc += c;
    }
  }
  __syncthreads();
#pragma unroll 4
  for (int s = tid; s < n_slots; s += SORT_THREADS) {
    const int lr = row_of_slot[s];
    if (lr >= 0) {
      const int e = ids[s];
      const int row = off[e] + wcnt[(s / spw) * E + e] + lr;
      row_of_slot[s] = row;
      slot_of_row[row] = s;
    }
  }
}

// ---- the same sort over several CTAs for prefill-class batches: per-CTA expert
// histograms over contiguous slot ranges, one scan CTA (prefix over the CTAs per expert + the tables above), then every CTA
// ranks its own range.  Order = (expert, slot) as before: bit-identical row assignment.
constexpr int SORT_MAX_CTAS = 128;

__global__ void __launch_bounds__(SORT_THREADS, 1)
    route_hist_kernel(const int32_t* __restrict__ ids, int n_slots, int E, int slots_per_cta, int32_t* __restrict__ hist) {
  __shared__ int cnt[MAX_EXPERTS];
  for (int e = threadIdx.x; e < E; e += SORT_THREADS) cnt[e] = 0;
  __syncthreads();
  const int s0 = blockIdx.x * slots_per_cta, s1 = min(n_slots, s0 + slots_per_cta);
#pragma unroll 4
  for (int s = s0 + threadIdx.x; s < s1; s += SORT_THREADS) {
    const int e = ids[s];
    if (e >= 0 && e < E) atomicAdd(&cnt[e], 1);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < E; e += SORT_THREADS) hist[(size_t)blockIdx.x * E + e] = cnt[e];
}

__global__ void __launch_bounds__(SORT_THREADS, 1)
    route_scan_kernel(int32_t* __restrict__ hist, int n_ctas, int E, int tn_max, int32_t* __restrict__ slot_of_row,
                      int32_t* __restrict__ pad_off_out, Chunk* __restrict__ chunks, RouteState* __restrict__ state) {
  __shared__ int cnt[MAX_EXPERTS];
  __shared__ int off[MAX_EXPERTS];
  __shared__ int choff[MAX_EXPERTS];
  __shared__ int warp_tot[2][SORT_THREADS / 32];
  __shared__ int totals[2];
  // hist[b][e] becomes the number of slots of e in earlier CTAs: one warp per expert, lane = four consecutive CTAs
  // (not a serial load -> store chain per expert)
  {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int e = warp; e < E; e += SORT_THREADS / 32) {
      int c[4], tot = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int b = lane * 4 + i;
        c[i] = (b < n_ctas) ? hist[(size_t)b * E + e] : 0;
        tot += c[i];
      }
      int inc = tot;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
      }
      int run = inc - tot;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int b = lane * 4 + i;
        if (b < n_ctas) hist[(size_t)b * E + e] = run;
        run += c[i];
      }
      if (lane == 31) cnt[e] = inc;
    }
  }
  __syncthreads();
  route_scan_tables(cnt, off, choff, warp_tot, totals, E, tn_max, slot_of_row, pad_off_out, chunks, state);
}

__global__ void __launch_bounds__(SORT_THREADS, 1)
    route_scatter_kernel(const int32_t* __restrict__ ids, int n_slots, int E, int slots_per_cta,
                         const int32_t* __restrict__ hist, const int32_t* __restrict__ pad_off,
                         int32_t* __restrict__ row_of_slot, int32_t* __restrict__ slot_of_row) {
  extern __shared__ int wcnt[];   // [NW][E]
  constexpr int NW = SORT_THREADS / 32;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < NW * E; i += SORT_THREADS) wcnt[i] = 0;
  __syncthreads();
  const int c0 = blockIdx.x * slots_per_cta, c1 = min(n_slots, c0 + slots_per_cta);
  const int spw = (((c1 - c0) + NW - 1) / NW + 31) & ~31;   // slots per warp
  {
    const int s_begin = c0 + warp * spw, s_end = min(c1, s_begin + spw);
    for (int s0 = s_begin; s0 < s_end; s0 += 128) {
      int ev[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int s = s0 + u * 32 + lane;
        ev[u] = (s < s_end) ? ids[s] : -1;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int s = s0 + u * 32 + lane;
        int e = ev[u];
        if (e < 0 || e >= E) e = -1;
        const unsigned m = __match_any_sync(0xffffffffu, e);
        const int rank = __popc(m & ((1u << lane) - 1u));
        const int base = (e >= 0) ? wcnt[warp * E + e] : 0;
        __syncwarp();
        if (e >= 0 && rank == 0) wcnt[warp * E + e] = base + __popc(m);
        __syncwarp();
        if (s < s_end) row_of_slot[s] = (e >= 0) ? base + rank : -1;   // rank inside (CTA, warp, expert) for now
      }
    }
  }
  __syncthreads();
  for (int e = tid; e < E; e += SORT_THREADS) {
    int acc = pad_off[e] + hist[(size_t)blockIdx.x * E + e];   // first row of this CTA's slots of expert e
    for (int w = 0; w < NW; ++w) {
      const int c = wcnt[w * E + e];
      wcnt[w * E + e] = acc;
      acc += c;
    }
  }
  __syncthreads();
  for (int s = c0 + tid; s < c1; s += SORT_THREADS) {
    const int lr = row_of_slot[s];
    if (lr >= 0) {
      const int e = ids[s];
      const int row = wcnt[((s - c0) / spw) * E + e] + lr;
      row_of_slot[s] = row;
      slot_of_row[row] = s;
    }
  }
}

// One CTA (128 threads) per permuted row.
template <bool FP8>
__global__ void __launch_bounds__(128) gather_rows_kernel(const uint16_t* __restrict__ hidden, int H, int top_k,
                                                         const int32_t* __restrict__ slot_of_row,
                                                         const RouteState* __restrict__ state,
                                                         uint8_t* __restrict__ xt, float* __restrict__ xs,
                                                         int KB, int rows_stride, int act_fp16,
                                                         const int32_t* __restrict__ ids, const int32_t* __restrict__ pad_off,
                                                         int tn_max, int e8m0) {
  // the grid is a few CTAs per SM looping over the padded rows (a launch sized by the worst-case row bound would be
  // 66 016 CTAs for an EP8 shard's 8192-token batch, nine in ten of them empty)
  const int n_rows = state->n_rows_padded;
  for (int r = blockIdx.x; r < n_rows; r += gridDim.x) {
  const int slot = slot_of_row[r];
  if (slot < 0) continue;
  const int t = slot / top_k;
  const uint16_t* src = hidden + (size_t)t * H;
  // chunk-contiguous tiled layout (the one moe_fused.cu uses): chunk = up to tn_max rows of one expert starting at row0;
  //   xt[row0 * KB*128 + kb * (tn/8 * 1024) + ((r - row0) / 8) * 1024 + sw128((r - row0) % 8, byte)]
  // so that a pipeline stage of the GEMM fetches the chunk's k-block with ONE bulk copy
  const int e = ids[slot];
  const int e_off = pad_off[e], e_rows = pad_off[e + 1] - e_off;      // padded rows of the expert (multiple of 16)
  const int cidx = (r - e_off) / tn_max;
  const int row0 = e_off + cidx * tn_max;
  const int tn = min(tn_max, e_rows - cidx * tn_max);
  const int rr = r - row0;
  uint8_t* dst_row = xt + (size_t)row0 * KB * 128 + (size_t)(rr >> 3) * 1024;
  const size_t kb_stride = (size_t)(tn >> 3) * 1024;
  const int tid = threadIdx.x;
  // four 16-byte loads in flight per thread (one row = H / 1024 rounds of the CTA, instead of a serial load ->
  // shuffle-reduce -> store chain per round)
  for (int base0 = 0; base0 < H; base0 += 4 * 128 * 8) {
   uint4 raw4[4];
#pragma unroll
   for (int u = 0; u < 4; ++u) {
     const int el = base0 + u * 128 * 8 + tid * 8;
     raw4[u] = make_uint4(0u, 0u, 0u, 0u);
     if (el < H) raw4[u] = *reinterpret_cast<const uint4*>(src + el);
   }
#pragma unroll
   for (int u = 0; u < 4; ++u) {
    const int el = base0 + u * 128 * 8 + tid * 8;
    if (base0 + u * 128 * 8 >= H) break;   // uniform over the CTA
    const bool valid = el < H;  // H % 128 == 0, so 16-thread groups are valid or invalid as a whole
    uint4 raw = raw4[u];
    if (FP8) {
      const uint16_t* h = reinterpret_cast<const uint16_t*>(&raw);
      float f[8];
      float am = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (act_fp16)
          f[i] = __half2float(*reinterpret_cast<const __half*>(&h[i]));
        else
          f[i] = __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(&h[i]));
        am = fmaxf(am, fabsf(f[i]));
      }
      // a 128-element group = 16 consecutive threads
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));
      if (valid) {
        const float sc = fp8_group_scale(am, e8m0);
        uint8_t q[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const __nv_fp8_e4m3 v(f[i] / sc);
          q[i] = *reinterpret_cast<const uint8_t*>(&v);
        }
        const int kb = el >> 7;
        const int boff = el & 127;
        *reinterpret_cast<uint2*>(dst_row + (size_t)kb * kb_stride + sw128_offset(rr & 7, boff)) =
            *reinterpret_cast<const uint2*>(q);
        if ((tid & 15) == 0) xs[(size_t)kb * rows_stride + r] = sc;
      }
    } else if (valid) {
      if (act_fp16 == 2) {   // 4-bit layers' prefill path: bf16 activations feed an fp16 x fp16 MMA
        uint16_t* h = reinterpret_cast<uint16_t*>(&raw);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float f = __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(&h[i]));
          const __half hv = __float2half_rn(fminf(fmaxf(f, -65504.f), 65504.f));
          h[i] = *reinterpret_cast<const uint16_t*>(&hv);
        }
      }
      const int kb = el >> 6;
      const int boff = (el & 63) * 2;
      *reinterpret_cast<uint4*>(dst_row + (size_t)kb * kb_stride + sw128_offset(rr & 7, boff)) = raw;
    }
   }
  }
  }
}

// one CTA per token: the token's k (row, weight) pairs are fetched once, then the CTA sweeps the H columns with eight row
// loads in flight per thread (a (H/1024, M) grid of single-float4 threads would spend its time on CTA
// scheduling and on re-reading the indices per column block)
__global__ void __launch_bounds__(256) combine_kernel(const float* __restrict__ y, const float* __restrict__ topk_w,
                                                     const int32_t* __restrict__ row_of_slot, int top_k, int H,
                                                     void* __restrict__ out, int out_dtype) {
  __shared__ int s_row[64];
  __shared__ float s_w[64];
  const int t = blockIdx.x;
  for (int j = threadIdx.x; j < top_k; j += 256) {
    const int row = row_of_slot[t * top_k + j];
    s_row[j] = row;
    s_w[j] = (row >= 0) ? topk_w[t * top_k + j] : 0.f;
  }
  __syncthreads();
  for (int h = threadIdx.x * 4; h < H; h += 256 * 4) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j0 = 0; j0 < top_k; j0 += 8) {   // eight row loads in flight, fixed j order in the sum
      float4 v[8];
      float w[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int j = j0 + u;
        const int row = (j < top_k) ? s_row[j] : -1;
        w[u] = (row >= 0) ? s_w[j] : 0.f;
        v[u] = (row >= 0) ? __ldcs(reinterpret_cast<const float4*>(y + (size_t)row * H + h)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        acc.x = fmaf(w[u], v[u].x, acc.x);
        acc.y = fmaf(w[u], v[u].y, acc.y);
        acc.z = fmaf(w[u], v[u].z, acc.z);
        acc.w = fmaf(w[u], v[u].w, acc.w);
      }
    }
    const size_t o = (size_t)t * H + h;
    if (out_dtype == 2) {
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + o) = acc;
    } else if (out_dtype == 0) {
      __nv_bfloat162 a = __floats2bfloat162_rn(acc.x, acc.y), b = __floats2bfloat162_rn(acc.z, acc.w);
      uint2 pk;
      pk.x = *reinterpret_cast<uint32_t*>(&a);
      pk.y = *reinterpret_cast<uint32_t*>(&b);
      *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + o) = pk;
    } else {
      __half2 a = __floats2half2_rn(acc.x, acc.y), b = __floats2half2_rn(acc.z, acc.w);
      uint2 pk;
      pk.x = *reinterpret_cast<uint32_t*>(&a);
      pk.y = *reinterpret_cast<uint32_t*>(&b);
      *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(out) + o) = pk;
    }
  }
}

static int64_t rows_bound(int64_t slots, int E) {
  const int64_t act = slots < E ? slots : E;
  return ((slots + (ROW_ALIGN - 1) * act) + ROW_ALIGN - 1) / ROW_ALIGN * ROW_ALIGN;
}

int launch_prep(const b200moe_layer* L, Workspace* ws, cudaStream_t st, const void* hidden, const int32_t* ids,
                int M, int k, int tn_max) {
  const int n_slots = M * k;
  // dynamic shared memory: warp-private rank counters [warps][E] (E <= 1024: 64 KB)
  const int wc_max = (SORT_THREADS / 32) * MAX_EXPERTS * 4;
  int rc = kernel_smem(reinterpret_cast<const void*>(route_sort_kernel), wc_max, "cudaFuncSetAttribute(route_sort)");
  if (rc) return rc;
  const size_t wc_bytes = (size_t)(SORT_THREADS / 32) * L->E * 4;
  if (n_slots >= 8192 && ws->sort_hist) {
    // prefill-class batch: histogram / scan / scatter over up to 128 CTAs (same (expert, slot) order)
    rc = kernel_smem(reinterpret_cast<const void*>(route_scatter_kernel), wc_max, "cudaFuncSetAttribute(route_scatter)");
    if (rc) return rc;
    int n_ctas = (n_slots + 1023) / 1024;
    if (n_ctas > SORT_MAX_CTAS) n_ctas = SORT_MAX_CTAS;
    const int spc = (((n_slots + n_ctas - 1) / n_ctas) + 31) & ~31;
    n_ctas = (n_slots + spc - 1) / spc;
    route_hist_kernel<<<n_ctas, SORT_THREADS, 0, st>>>(ids, n_slots, L->E, spc, ws->sort_hist);
    route_scan_kernel<<<1, SORT_THREADS, 0, st>>>(ws->sort_hist, n_ctas, L->E, tn_max, ws->slot_of_row, ws->pad_off,
                                                  ws->chunks, ws->state);
    route_scatter_kernel<<<n_ctas, SORT_THREADS, wc_bytes, st>>>(ids, n_slots, L->E, spc, ws->sort_hist, ws->pad_off,
                                                                 ws->row_of_slot, ws->slot_of_row);
    g_launches += 3;
  } else {
    route_sort_kernel<<<1, SORT_THREADS, wc_bytes, st>>>(ids, n_slots, L->E, tn_max, ws->row_of_slot, ws->slot_of_row,
                                                         ws->pad_off, ws->chunks, ws->state);
    ++g_launches;
  }
  int rb = (int)rows_bound(n_slots, L->E);
  if (rb > 132 * 12) rb = 132 * 12;   // row loop inside the kernel
  if (L->esz_bits == 8)
    gather_rows_kernel<true><<<rb, 128, 0, st>>>(reinterpret_cast<const uint16_t*>(hidden), L->H, k,
                                                 ws->slot_of_row, ws->state, ws->xt, ws->xs, L->KB1,
                                                 (int)ws->cap_rows, L->act_dtype == B200_ACT_FP16, ids, ws->pad_off, tn_max,
                                                 L->fp8_e8m0);
  else
    gather_rows_kernel<false><<<rb, 128, 0, st>>>(reinterpret_cast<const uint16_t*>(hidden), L->H, k,
                                                  ws->slot_of_row, ws->state, ws->xt, ws->xs, L->KB1,
                                                  (int)ws->cap_rows, L->cvt_bf16_to_fp16 ? 2 : (L->act_dtype == B200_ACT_FP16), ids,
                                                  ws->pad_off, tn_max, 0);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "prep launch");
  return 0;
}

int launch_combine(const b200moe_layer* L, Workspace* ws, cudaStream_t st, const float* topk_w, int M, int k,
                   void* out, int out_dtype) {
  combine_kernel<<<M, 256, 0, st>>>(ws->y, topk_w, ws->row_of_slot, k, L->H, out, out_dtype);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "combine launch");
  return 0;
}

// ------------------------------------------------------------------------------------------- workspace
static Workspace g_ws[16];

Workspace* get_workspace(int device) {
  if (device < 0 || device >= 16) return nullptr;
  g_ws[device].device = device;
  return &g_ws[device];
}

// Growth never frees: CUDA graphs captured earlier (cpu_decode) keep replaying against the old buffers, which
// are parked in `retired` until the last layer of the device is destroyed (include/b200moe.h promises pointer-stable
// workspaces).  A failed allocation resets the capacities so that the next call grows again instead of using a hole.
static int ws_alloc(Workspace* ws, void** ptr, int64_t nbytes) {
  if (*ptr) {
    ws->retired.push_back(*ptr);
    *ptr = nullptr;
  }
  cudaError_t e = cudaMalloc(ptr, (size_t)nbytes);
  if (e != cudaSuccess) {
    *ptr = nullptr;
    ws->cap_slots = ws->cap_rows = ws->cap_hidden = ws->cap_inter = ws->cap_stage_hidden = 0;
    return cuda_fail(e, "cudaMalloc(workspace)");
  }
  ws->bytes += nbytes;
  return 0;
}
#define WS_ALLOC(PTR_, NBYTES_)                                                        \
  do {                                                                                 \
    int rc_ = ws_alloc(ws, reinterpret_cast<void**>(&(PTR_)), (int64_t)(NBYTES_));     \
    if (rc_) return rc_;                                                               \
  } while (0)

int ensure_workspace(Workspace* ws, const b200moe_layer* L, int64_t tokens, int top_k, bool may_alloc) {
  const int64_t slots = tokens * top_k;
  const int64_t rows = rows_bound(slots, L->E);
  const int64_t hid_b = (int64_t)L->KB1 * 128;  // operand bytes per row of GEMM1
  const int64_t int_b = (int64_t)L->KB2 * 128;
  const bool ok = ws->state && slots <= ws->cap_slots && rows <= ws->cap_rows && hid_b <= ws->cap_hidden &&
                  int_b <= ws->cap_inter && L->H <= ws->cap_stage_hidden;
  if (ok) return 0;
  if (!may_alloc) {
    set_error("workspace too small for this call and allocation is not allowed here (stream capture); "
              "raise max_num_seqs / max_batch_size in the layer config");
    return B200_ERR_INVALID;
  }
  const int64_t nslots = slots > ws->cap_slots ? slots : ws->cap_slots;
  const int64_t nrows = rows > ws->cap_rows ? rows : ws->cap_rows;
  const int64_t nh = hid_b > ws->cap_hidden ? hid_b : ws->cap_hidden;
  const int64_t ni = int_b > ws->cap_inter ? int_b : ws->cap_inter;
  const int64_t nH = L->H > ws->cap_stage_hidden ? L->H : ws->cap_stage_hidden;
  WS_ALLOC(ws->row_of_slot, nslots * 4);
  WS_ALLOC(ws->slot_of_row, nrows * 4);
  WS_ALLOC(ws->pad_off, (MAX_EXPERTS + 1) * 4);
  WS_ALLOC(ws->sort_hist, (int64_t)SORT_MAX_CTAS * MAX_EXPERTS * 4);
  WS_ALLOC(ws->chunks, (nrows / ROW_ALIGN + MAX_EXPERTS) * sizeof(Chunk));
  WS_ALLOC(ws->state, sizeof(RouteState));
  WS_ALLOC(ws->xt, nrows * nh);
  WS_ALLOC(ws->xs, (nh / 128) * nrows * 4);
  WS_ALLOC(ws->it, nrows * ni);
  WS_ALLOC(ws->is, (ni / 128) * nrows * 4);
  WS_ALLOC(ws->y, nrows * nH * 4);
  if (!ws->partials) {
    WS_ALLOC(ws->partials, (int64_t)(4 * 160 * 2 + 160 * 4) * (2 * 64 * 128) * 4);
    WS_ALLOC(ws->fsync, (int64_t)sizeof(FusedSync));
    cudaMemset(ws->fsync, 0, sizeof(FusedSync));
  }
  cudaMemset(ws->state, 0, sizeof(RouteState));
  // the fresh buffers are first touched by work enqueued after this point; the legacy-stream memsets above are
  // ordered before any later kernel of a blocking stream, and callers on non-blocking streams synchronise here
  cudaError_t se = cudaDeviceSynchronize();
  if (se != cudaSuccess) return cuda_fail(se, "cudaDeviceSynchronize(workspace grow)");
  ws->cap_slots = nslots;
  ws->cap_rows = nrows;
  ws->cap_hidden = nh;
  ws->cap_inter = ni;
  ws->cap_stage_hidden = nH;
  return 0;
}

// fp16 expansion scratch of the 4-bit prefill path.  Never used under stream capture, so an outgrown buffer is freed
// (cudaFree synchronises the device) instead of retired: it is tens of GB for a DeepSeek-sized layer.
int ensure_dequant_scratch(Workspace* ws, int64_t bytes13, int64_t bytes2) {
  if (bytes13 <= ws->cap_dq13 && bytes2 <= ws->cap_dq2) return 0;
  cudaError_t e;
  if (bytes13 > ws->cap_dq13) {
    if (ws->dq13) cudaFree(ws->dq13);
    ws->bytes -= ws->cap_dq13;
    ws->dq13 = nullptr;
    ws->cap_dq13 = 0;
    if ((e = cudaMalloc(reinterpret_cast<void**>(&ws->dq13), (size_t)bytes13)) != cudaSuccess) {
      ws->dq13 = nullptr;
      return cuda_fail(e, "cudaMalloc(4-bit prefill scratch, w13)");
    }
    ws->cap_dq13 = bytes13;
    ws->bytes += bytes13;
  }
  if (bytes2 > ws->cap_dq2) {
    if (ws->dq2) cudaFree(ws->dq2);
    ws->bytes -= ws->cap_dq2;
    ws->dq2 = nullptr;
    ws->cap_dq2 = 0;
    if ((e = cudaMalloc(reinterpret_cast<void**>(&ws->dq2), (size_t)bytes2)) != cudaSuccess) {
      ws->dq2 = nullptr;
      return cuda_fail(e, "cudaMalloc(4-bit prefill scratch, w2)");
    }
    ws->cap_dq2 = bytes2;
    ws->bytes += bytes2;
  }
  return 0;
}

int grow_staging(Workspace* ws, int64_t hidden_elems, int64_t slots) {
  if (hidden_elems <= ws->cap_stage_tokens && slots <= ws->cap_stage_k && ws->d_hidden) return 0;
  const int64_t ce = hidden_elems > ws->cap_stage_tokens ? hidden_elems : ws->cap_stage_tokens;
  const int64_t cs = slots > ws->cap_stage_k ? slots : ws->cap_stage_k;
  ws->cap_stage_tokens = ws->cap_stage_k = 0;
  WS_ALLOC(ws->d_hidden, ce * 2);
  WS_ALLOC(ws->d_ids, cs * 4);
  WS_ALLOC(ws->d_w, cs * 4);
  WS_ALLOC(ws->d_out, ce * 4);
  ws->cap_stage_tokens = ce;
  ws->cap_stage_k = cs;
  return 0;
}

// called when the last layer of a device is destroyed: nothing can replay against the buffers any more
void release_workspace(Workspace* ws) {
  cudaDeviceSynchronize();
  void** cur[] = {reinterpret_cast<void**>(&ws->row_of_slot), reinterpret_cast<void**>(&ws->slot_of_row),
                  reinterpret_cast<void**>(&ws->pad_off), reinterpret_cast<void**>(&ws->sort_hist),
                  reinterpret_cast<void**>(&ws->chunks),
                  reinterpret_cast<void**>(&ws->state), reinterpret_cast<void**>(&ws->xt), reinterpret_cast<void**>(&ws->xs),
                  reinterpret_cast<void**>(&ws->it), reinterpret_cast<void**>(&ws->is), reinterpret_cast<void**>(&ws->y),
                  reinterpret_cast<void**>(&ws->partials), reinterpret_cast<void**>(&ws->fsync),
                  &ws->d_hidden, reinterpret_cast<void**>(&ws->d_ids),
                  reinterpret_cast<void**>(&ws->d_w), reinterpret_cast<void**>(&ws->d_out),
                  reinterpret_cast<void**>(&ws->dq13), reinterpret_cast<void**>(&ws->dq2)};
  for (void** p : cur) {
    if (*p) cudaFree(*p);
    *p = nullptr;
  }
  for (void* p : ws->retired) cudaFree(p);
  ws->retired.clear();
  ws->cap_slots = ws->cap_rows = ws->cap_hidden = ws->cap_inter = ws->cap_stage_hidden = 0;
  ws->cap_stage_tokens = ws->cap_stage_k = 0;
  ws->cap_dq13 = ws->cap_dq2 = 0;
  ws->bytes = 0;
}

}  // namespace b200
