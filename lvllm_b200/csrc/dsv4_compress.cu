// The DeepSeek-V4 KV compressor for decode (the reference's DeepseekCompressor.forward, models/deepseek_v4/compressor.py):
// every compress_ratio tokens of a request become one row of a compressed key cache.  Two launches, in stream order:
//   dsv4_compress_state_kernel  the state write (common/ops/save_partial_states.py): token t's kv and score + ape go to row
//                               slot_mapping[t] of the fp32 state cache;
//   dsv4_compress_kernel        for each token that closes a window, the softmax-pooled compression of the window's state
//                               rows, RMSNorm, GPT-J RoPE of the last 64 dims and the fp8 store into the 584-byte
//                               attention cache (D 512) or the indexer's 132-byte cache (D 128)
//                               (common/ops/fused_compress_quant_cache.py:113-297, 657-828).
// A window reads the state rows written by the first launch in the same call (its own row, and with several tokens of a
// request in one call its neighbours' rows), so the compression runs as a second launch, without programmatic dependent
// launch.  The rows are written by the shared packers of kv_pack.cuh, so the bytes are those of dsv4_qnorm_rope_kv_insert
// and of the indexer's k-cache write.
#include <cooperative_groups.h>

#include "common.cuh"
#include "kv_pack.cuh"
#include "moe_internal.cuh"

namespace cg = cooperative_groups;

namespace b200 {

struct CompressArgs {
  const float* kv_score;         // [T, 2 * coff * D] rows kv_score_stride floats apart: kv | score
  int64_t kv_score_stride;
  const float* ape;              // [ratio, coff * D]
  const int64_t* positions;      // [T]
  const int64_t* slot_mapping;   // [T] state slots
  const int32_t* token_to_req;   // [T] rows of block_table
  const int32_t* block_table;    // [*, block_table_stride] state blocks of a request
  int64_t block_table_stride;
  float* state;                  // [blocks, state_block_size, 2 * coff * D], blocks state_block_stride floats apart
  int state_block_size;
  int64_t state_block_stride;
  const __nv_bfloat16* norm_weight;   // [D]
  float eps;
  const float* cos_sin;          // [max_pos, 64] = cos | sin
  int max_pos;
  const int64_t* kv_slot_mapping;     // [T] rows of the output cache
  uint8_t* cache;
  int block_size, num_blocks;
  int64_t block_stride;          // bytes
  int T;
};

// grid = T, HALF / 4 float4 columns per token, NT threads.  row = [kv | score + ape[position % ratio]], HALF floats each.
template <int HALF, int RATIO, int NT>
__global__ void __launch_bounds__(NT) dsv4_compress_state_kernel(const CompressArgs a) {
  const int t = blockIdx.x;
  const int64_t s = a.slot_mapping[t];
  if (s < 0) return;
  int64_t r = a.positions[t] % RATIO;
  r = r < 0 ? r + RATIO : r;
  const float4* kv = reinterpret_cast<const float4*>(a.kv_score + (size_t)t * a.kv_score_stride);
  const float4* ape = reinterpret_cast<const float4*>(a.ape + r * HALF);
  float4* dst = reinterpret_cast<float4*>(a.state + (s / a.state_block_size) * a.state_block_stride +
                                          (s % a.state_block_size) * (2 * HALF));
#pragma unroll
  for (int j = threadIdx.x; j < HALF / 4; j += NT) {
    const float4 k = kv[j], sc = kv[HALF / 4 + j], e = ape[j];
    dst[j] = k;
    dst[HALF / 4 + j] = make_float4(sc.x + e.x, sc.y + e.y, sc.z + e.z, sc.w + e.w);
  }
}

// grid = T clusters of CL CTAs; CTA `rank` of token t's cluster owns columns [rank * CW, rank * CW + CW) of the D.
// A token computes when its state slot is >= 0, its position p >= 0 closes a window ((p + 1) % RATIO == 0) and its
// kv_slot_mapping entry names a row of the cache; any other token writes nothing.  The window is the state rows of
// positions p - W + 1 .. p (W = (1 + OVL) * RATIO) of the token's request, found through its block table row; positions
// below 0 are no row.  With OVL the older RATIO rows take columns [0, D) of their kv and score halves, the newer ones
// [D, 2D).  Per column: softmax of the scores over the window rows, then sum kv * weight, fp32.  Thread (g, q) takes the
// float4 column q of rows g, g + RG, ... (all its loads issued before the first use); the RG row groups are merged in
// a fixed order.  The pooled columns go to the leader CTA (rank 0) through distributed shared memory; its first warp
// normalises (c * rsqrt(mean(c^2) + eps) * w), rotates the last 64 dims' pairs (2k, 2k + 1) by (cos, sin) of position
// (p / RATIO) * RATIO (clamped to [0, max_pos)) and packs the row.
template <int D, int RATIO, bool OVL, int CL, int NT>
__global__ void __launch_bounds__(NT) dsv4_compress_kernel(const CompressArgs a) {
  constexpr int COFF = OVL ? 2 : 1, HALF = COFF * D, W = (OVL ? 2 : 1) * RATIO;
  constexpr int CW = D / CL, Q = CW / 4, RG = NT / Q, RPT = W / RG, VPL = D / 32;
  static_assert(NT % Q == 0 && W % RG == 0 && (VPL == 16 || VPL == 4), "unsupported compressor shape");
  __shared__ __align__(16) float pooled[D];
  __shared__ float part[RG > 1 ? 3 : 1][RG > 1 ? RG : 1][RG > 1 ? CW : 1];
  const int t = blockIdx.x / CL, rank = blockIdx.x % CL, tid = threadIdx.x;
  const int64_t p = a.positions[t], ks = a.kv_slot_mapping[t];
  if (a.slot_mapping[t] < 0 || p < 0 || (p + 1) % RATIO != 0 || ks < 0 || ks >= (int64_t)a.num_blocks * a.block_size)
    return;   // the same for every CTA of the cluster
  if constexpr (CL > 1) asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
  const int g = tid / Q, qd = tid % Q, col = rank * CW + qd * 4;
  const int32_t* bt = a.block_table + (int64_t)a.token_to_req[t] * a.block_table_stride;
  float4 kv[RPT], sc[RPT];
#pragma unroll
  for (int i = 0; i < RPT; ++i) {
    const int r = g + i * RG;
    const int64_t pr = p - W + 1 + r;
    if (pr >= 0) {
      const float* row = a.state + (int64_t)bt[pr / a.state_block_size] * a.state_block_stride +
                         (pr % a.state_block_size) * (2 * HALF) + ((OVL && r >= RATIO) ? D : 0) + col;
      kv[i] = *reinterpret_cast<const float4*>(row);
      sc[i] = *reinterpret_cast<const float4*>(row + HALF);
    } else {
      kv[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      sc[i] = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    }
  }
  float m[4], l[4], acc[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    m[k] = -INFINITY;
#pragma unroll
    for (int i = 0; i < RPT; ++i) m[k] = fmaxf(m[k], reinterpret_cast<const float*>(&sc[i])[k]);
    l[k] = 0.f;
    acc[k] = 0.f;
#pragma unroll
    for (int i = 0; i < RPT; ++i) {
      const float s = reinterpret_cast<const float*>(&sc[i])[k];
      const float e = s == -INFINITY ? 0.f : expf(s - m[k]);
      l[k] += e;
      acc[k] = fmaf(e, reinterpret_cast<const float*>(&kv[i])[k], acc[k]);
    }
  }
  float* dst = pooled;
  if constexpr (CL > 1) {
    asm volatile("barrier.cluster.wait.aligned;" ::: "memory");   // every CTA of the cluster runs: its shared memory exists
    dst = cg::this_cluster().map_shared_rank(pooled, 0);
  }
  if constexpr (RG == 1) {
    *reinterpret_cast<float4*>(dst + col) = make_float4(acc[0] / l[0], acc[1] / l[1], acc[2] / l[2], acc[3] / l[3]);
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      part[0][g][qd * 4 + k] = m[k];
      part[1][g][qd * 4 + k] = l[k];
      part[2][g][qd * 4 + k] = acc[k];
    }
    __syncthreads();
    if (tid < CW) {
      float mm = -INFINITY;
#pragma unroll
      for (int j = 0; j < RG; ++j) mm = fmaxf(mm, part[0][j][tid]);
      float ls = 0.f, as = 0.f;
#pragma unroll
      for (int j = 0; j < RG; ++j) {
        const float mj = part[0][j][tid];
        const float f = mj == -INFINITY ? 0.f : expf(mj - mm);
        ls = fmaf(part[1][j][tid], f, ls);
        as = fmaf(part[2][j][tid], f, as);
      }
      dst[rank * CW + tid] = as / ls;
    }
  }
  if constexpr (CL > 1) {
    cg::this_cluster().sync();
    if (rank != 0) return;
  } else {
    __syncthreads();
  }
  if (tid >= 32) return;
  // the leader's first warp: lane l holds dims [VPL * l, VPL * l + VPL)
  const int lane = tid, d0 = lane * VPL;
  float x[VPL], w[VPL];
#pragma unroll
  for (int i = 0; i < VPL; i += 4) {
    const float4 v = *reinterpret_cast<const float4*>(pooled + d0 + i);
    x[i] = v.x, x[i + 1] = v.y, x[i + 2] = v.z, x[i + 3] = v.w;
    const uint2 wb = *reinterpret_cast<const uint2*>(a.norm_weight + d0 + i);
    const __nv_bfloat16* wh = reinterpret_cast<const __nv_bfloat16*>(&wb);
#pragma unroll
    for (int j = 0; j < 4; ++j) w[i + j] = __bfloat162float(wh[j]);
  }
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) ss = fmaf(x[i], x[i], ss);
  const float rr = rsqrtf(warp_sum(ss) / D + a.eps);
#pragma unroll
  for (int i = 0; i < VPL; ++i) x[i] = x[i] * rr * w[i];
  if (d0 >= D - 64) {
    int64_t cp = (p / RATIO) * RATIO;
    cp = cp >= a.max_pos ? a.max_pos - 1 : cp;
    const float* cs = a.cos_sin + cp * 64 + (d0 - (D - 64)) / 2;
#pragma unroll
    for (int k = 0; k < VPL / 2; ++k) {
      const float e = x[2 * k], o = x[2 * k + 1], c = cs[k], s = cs[32 + k];
      x[2 * k] = e * c - o * s;
      x[2 * k + 1] = o * c + e * s;
    }
  }
  uint8_t* blk = a.cache + (ks / a.block_size) * a.block_stride;
  if constexpr (D == 512)
    dsv4_pack_row584(x, blk, a.block_size, (int)(ks % a.block_size), lane);
  else
    indexer_pack_row132(x, true, blk, a.block_size, (int)(ks % a.block_size), lane);
}

template <int D, int RATIO, bool OVL, int CL, int NT>
int launch_compress(cudaStream_t st, const CompressArgs& a) {
  constexpr int HALF = (OVL ? 2 : 1) * D, SNT = HALF / 4 < 128 ? HALF / 4 : 128;
  dsv4_compress_state_kernel<HALF, RATIO, SNT><<<a.T, SNT, 0, st>>>(a);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "dsv4_compress_state launch");
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)a.T * CL);
  cfg.blockDim = dim3(NT);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  e = cudaLaunchKernelEx(&cfg, dsv4_compress_kernel<D, RATIO, OVL, CL, NT>, a);
  ++g_launches;
  if (e == cudaSuccess) e = cudaGetLastError();
  return e == cudaSuccess ? 0 : cuda_fail(e, "dsv4_compress launch");
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_dsv4_compress(void* stream, const float* kv_score, int64_t kv_score_stride, const float* ape,
                       const int64_t* positions, const int64_t* slot_mapping, const int32_t* token_to_req,
                       const int32_t* block_table, int64_t block_table_stride, float* state_cache, int state_block_size,
                       int64_t state_block_stride, const void* norm_weight, float eps, const float* cos_sin_cache,
                       int max_position, const int64_t* kv_slot_mapping, void* kv_cache, int block_size, int num_blocks,
                       int64_t block_stride, int head_dim, int compress_ratio, int num_tokens) {
  auto al = [](const void* p, uintptr_t n) { return p && (reinterpret_cast<uintptr_t>(p) & (n - 1)) == 0; };
  const bool c4a = head_dim == 512 && compress_ratio == 4, c128a = head_dim == 512 && compress_ratio == 128,
             idx = head_dim == 128 && compress_ratio == 4;
  const int64_t half = (int64_t)(compress_ratio == 4 ? 2 : 1) * head_dim;
  const int64_t row_bytes = head_dim == 512 ? 584 : 132;
  if (!(c4a || c128a || idx) || !al(kv_score, 16) || kv_score_stride < 2 * half || kv_score_stride % 4 != 0 ||
      !al(ape, 16) || !al(positions, 8) || !al(slot_mapping, 8) || !al(token_to_req, 4) || !al(block_table, 4) ||
      block_table_stride < 1 || !al(state_cache, 16) || state_block_size < 1 ||
      state_block_stride < (int64_t)state_block_size * 2 * half || state_block_stride % 4 != 0 || !al(norm_weight, 16) ||
      !(eps >= 0.f) || !al(cos_sin_cache, 4) || max_position < 1 || !al(kv_slot_mapping, 8) || !al(kv_cache, 16) ||
      block_size < 1 || num_blocks < 1 || block_stride < (int64_t)block_size * row_bytes ||
      block_stride % (head_dim == 512 ? 16 : 4) != 0 || num_tokens < 0 || num_tokens > (1 << 20)) {
    set_error("b200_dsv4_compress: bad argument ((head_dim, compress_ratio) (512, 4), (512, 128) or (128, 4); 16-byte "
              "aligned kv_score, ape, state_cache, norm_weight and kv_cache; row strides in 16-byte units covering a row; "
              "block strides covering a block (584-byte cache: a multiple of 16); eps >= 0; 0 <= num_tokens <= 2^20)");
    return B200_ERR_INVALID;
  }
  if (num_tokens == 0) return 0;
  CompressArgs a{kv_score, kv_score_stride, ape, positions, slot_mapping, token_to_req, block_table, block_table_stride,
                 state_cache, state_block_size, state_block_stride, reinterpret_cast<const __nv_bfloat16*>(norm_weight), eps,
                 cos_sin_cache, max_position, kv_slot_mapping, reinterpret_cast<uint8_t*>(kv_cache), block_size, num_blocks,
                 block_stride, num_tokens};
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (c4a) return launch_compress<512, 4, true, 1, 128>(st, a);
  if (c128a) return launch_compress<512, 128, false, 8, 256>(st, a);
  return launch_compress<128, 4, true, 1, 32>(st, a);
}

}  // extern "C"
