// Fused router: logits = x . W_g^T  (wgmma, split-K)  ->  top-k / grouped top-k  ->  [EP id remap], ONE kernel.
//
// Replaces, for the MoE hot path, the chain  GateLinear.forward (reference router/gate_linear.py:171-221 ->
// dsv3_router_gemm, csrc/libtorch_stable/moe/dsv3_router_gemm_entry.cu:112)  ->  fused_topk / grouped_topk
// (fused_topk_router.py:81-124, grouped_topk_kernels.cu:523-678)  ->  global_to_local_expert_ids
// (routed_experts.py:1332-1342): four launches (one of them a library GEMM) in round 1.
//
// Shape of the work: E x H weights (DeepSeek-V3: 256 x 7168 bf16 = 3.7 MB) against M <= a few hundred tokens — an HBM /
// latency bound skinny GEMM.  Swap-AB like the expert kernels: the 128 experts of a tile are the MMA M rows, a tile of
// TN tokens the N columns, so M = 1 costs one 16-column MMA.  Both operands are fetched with 2-D tensor maps
// (SWIZZLE_128B boxes of 64 K-elements: the K-major operand layout wgmma reads, straight from the row-major
// tensors; rows beyond E / M are zero-filled by the TMA unit).  K is split over CTAs so that the 132 SMs pull the weights
// together; partial logits go to a small fp32 workspace and the LAST CTA of a token tile (self-resetting arrival
// counter, CUDA-graph replayable) sums them in fixed split order — deterministic logits, hence reproducible ids — and
// routes the tile's tokens, one warp per token, with the same device functions as the stand-alone routing kernels.
//
// Roofline: HBM / latency.  Algorithmic bytes = E*H*2 (weights) + M*H*2 (activations) + M*k*8 (outputs).
#include <cuda.h>

#include <mutex>

#include "moe_internal.cuh"
#include "routing_device.cuh"

namespace b200 {

constexpr int R_THREADS = 384;   // warp 0 TMA producer, 2-5 drain, 8-11 MMA warpgroup, all 12 route
constexpr int R_STAGES = 4;
constexpr int R_A_BYTES = 128 * 128;   // [128 experts x 64 k] 16-bit

struct RouterArgs {
  alignas(64) CUtensorMap tmW;   // gate weights [E][H], box 64 x 128
  alignas(64) CUtensorMap tmX;   // activations  [M][H], box 64 x TN
  int M, E, H, KB, KS, TN, EZ, Epad;
  int cmp_fp16;
  float* partial;        // [KS][M][Epad]
  int32_t* counters;     // [token tiles], zero between launches
  float* logits_out;     // optional [M][E]
  int mode;              // 0 softmax top-k, 1 sigmoid top-k, 2 grouped top-k, 3 sqrt-softplus top-k (or hash)
  int scoring;           // grouped: 0 none, 1 sigmoid
  int k, renorm, n_group, topk_group;
  float rsf;
  const float* bias;
  const int32_t* emap;   // optional global -> local expert ids
  const int32_t* input_ids, *tid2eid;   // hash routing (mode 3): ids = tid2eid[input_ids[t]], tid2eid [vocab][k]
  int vocab;
  // shared experts folded into the routed launch as always-on experts (SURVEY.md 8f row 2): n_shared extra columns per
  // token, weight shared_w; global id E + s, local id shared_local_base + s (or -1 when this rank does not hold them)
  int n_shared, shared_local_base;
  float shared_w;
  float* out_w;
  int32_t* out_ids;
  int32_t* out_local;
};

// MMA warpgroup (warps 8-11): logits^T[128 experts, TN tokens] accumulate in registers over the CTA's k-blocks, then cross
// to the drain warps through the exchange area
template <int TN>
B200_DEVICE void router_mma(uint32_t smem0, int stage_bytes, int n_kb, int fp16, uint64_t* full, uint64_t* empty,
                            uint64_t* tfull, uint32_t xch) {
  float acc[2][TN / 2];
  for (int i = 0; i < n_kb; ++i) {
    const int s = i % R_STAGES;
    mbar_wait(&full[s], (i / R_STAGES) & 1);
    const uint32_t sa = smem0 + s * stage_bytes, sb = sa + R_A_BYTES;
    wgmma_fence();
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (fp16)
        wgmma_tile128<TN, 0>(acc, sa + q * 32, sb + q * 32, (i > 0 || q > 0) ? 1u : 0u);
      else
        wgmma_tile128<TN, 1>(acc, sa + q * 32, sb + q * 32, (i > 0 || q > 0) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[s]);
  }
  xch_store_frag<TN>(xch, 0, acc[0]);
  xch_store_frag<TN>(xch, 1, acc[1]);
  mbar_arrive(tfull);
}

__global__ void __launch_bounds__(R_THREADS, 1) router_gemm_topk_kernel(const __grid_constant__ RouterArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int stage_bytes = R_A_BYTES + a.TN * 128;
  float* lg = reinterpret_cast<float*>(smem + R_STAGES * stage_bytes);        // [TN][Epad] logits of the tile
  float* scratch = lg + (size_t)a.TN * a.Epad;                               // [warps][2][Epad] (grouped) / reduce
  __shared__ uint64_t full[R_STAGES], empty[R_STAGES], tfull;
  __shared__ int last_flag;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ks = blockIdx.x, tt = blockIdx.y, ez = blockIdx.z;
  const int kb0 = (int)(((long long)ks * a.KB) / a.KS), kb1 = (int)(((long long)(ks + 1) * a.KB) / a.KS);
  const int t0 = tt * a.TN;
  const int nt = min(a.TN, a.M - t0);

  if (tid == 0) {
    for (int i = 0; i < R_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 1);
    }
    mbar_init(&tfull, 128);
    fence_barrier_init();
  }
  __syncthreads();
  // the finished accumulator crosses from the MMA warpgroup to the drain warps through the logits area, which the
  // routing phase only fills after the drain
  const uint32_t xch = xch_base(lg);

  if (warp == 0) {
    if (elect_one()) {
      const uint64_t pol_w = policy_evict_first(), pol_x = policy_evict_last();
      for (int kb = kb0, i = 0; kb < kb1; ++kb, ++i) {
        const int s = i % R_STAGES;
        mbar_wait(&empty[s], ((i / R_STAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(&full[s], (uint32_t)stage_bytes);
        uint8_t* sa = smem + s * stage_bytes;
        tma_load_2d_hint(sa, &a.tmW, kb * 64, ez * 128, &full[s], pol_w);
        tma_load_2d_hint(sa + R_A_BYTES, &a.tmX, kb * 64, t0, &full[s], pol_x);
      }
    }
  } else if (warp >= 8) {
    const uint32_t sm0 = smem_u32(smem);
    if (a.TN == 16)
      router_mma<16>(sm0, stage_bytes, kb1 - kb0, a.cmp_fp16, full, empty, &tfull, xch);
    else if (a.TN == 32)
      router_mma<32>(sm0, stage_bytes, kb1 - kb0, a.cmp_fp16, full, empty, &tfull, xch);
    else
      router_mma<64>(sm0, stage_bytes, kb1 - kb0, a.cmp_fp16, full, empty, &tfull, xch);
  } else if (warp >= 2 && warp < 6) {
    // drain: thread = expert row of the tile, columns = tokens; partial[ks][t][e] (e contiguous over the lanes)
    const int q4 = warp & 3;                    // the 32-row quarter of the tile this warp drains
    const int e = ez * 128 + q4 * 32 + lane;
    mbar_wait(&tfull, 0);
    for (int c0 = 0; c0 < a.TN; c0 += 16) {
      float v[16];
      xch_ld<16>(xch + ((uint32_t)(q4 * 32) << 16) + c0, v);
      if (e < a.Epad) {
#pragma unroll
        for (int c = 0; c < 16; ++c)
          if (c0 + c < nt) a.partial[((size_t)ks * a.M + t0 + c0 + c) * a.Epad + e] = v[c];
      }
    }
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    const int old = atomicAdd(&a.counters[tt], 1);
    const int last = (old == a.KS * a.EZ - 1);
    if (last) a.counters[tt] = 0;   // hand the counter back clean for the next launch / graph replay
    last_flag = last;
  }
  __syncthreads();
  if (!last_flag) return;
  __threadfence();   // acquire side: every split's partial logits are visible

  // ---- reduce the K splits in fixed order (deterministic): work items = (token, 4 experts)
  const int E4 = a.Epad >> 2;
  const int items = nt * E4;
  const int G = (items * 4 <= R_THREADS) ? 4 : (items * 2 <= R_THREADS) ? 2 : 1;   // thread groups over the splits
  if (G == 1) {
    for (int it = tid; it < items; it += R_THREADS) {
      const int t = it / E4, e4 = it - t * E4;
      const float4* src = reinterpret_cast<const float4*>(a.partial + ((size_t)(t0 + t)) * a.Epad) + e4;
      const size_t stride = (size_t)a.M * a.Epad / 4;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int s0 = 0; s0 < a.KS; s0 += 8) {
        float4 v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u)
          v[u] = (s0 + u < a.KS) ? __ldcg(src + (size_t)(s0 + u) * stride) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          acc.x += v[u].x;
          acc.y += v[u].y;
          acc.z += v[u].z;
          acc.w += v[u].w;
        }
      }
      *reinterpret_cast<float4*>(lg + (size_t)t * a.Epad + e4 * 4) = acc;
    }
  } else {
    // few items (decode batches): G thread groups each sum a contiguous range of splits, then the group sums are added
    // in group order — the summation tree is a function of (KS, G) only
    const int g = tid / (R_THREADS / G), it = tid % (R_THREADS / G);
    float4* red = reinterpret_cast<float4*>(scratch);   // [G][items]
    if (it < items) {
      const int t = it / E4, e4 = it - t * E4;
      const float4* src = reinterpret_cast<const float4*>(a.partial + ((size_t)(t0 + t)) * a.Epad) + e4;
      const size_t stride = (size_t)a.M * a.Epad / 4;
      const int sA = (g * a.KS) / G, sB = ((g + 1) * a.KS) / G;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int s0 = sA; s0 < sB; s0 += 8) {
        float4 v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u)
          v[u] = (s0 + u < sB) ? __ldcg(src + (size_t)(s0 + u) * stride) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          acc.x += v[u].x;
          acc.y += v[u].y;
          acc.z += v[u].z;
          acc.w += v[u].w;
        }
      }
      red[g * items + it] = acc;
    }
    __syncthreads();
    if (tid < items) {
      float4 acc = red[tid];
      for (int gg = 1; gg < G; ++gg) {
        const float4 v = red[gg * items + tid];
        acc.x += v.x;
        acc.y += v.y;
        acc.z += v.z;
        acc.w += v.w;
      }
      const int t = tid / E4, e4 = tid - t * E4;
      *reinterpret_cast<float4*>(lg + (size_t)t * a.Epad + e4 * 4) = acc;
    }
  }
  __syncthreads();
  if (a.logits_out) {
    for (int i = tid; i < nt * a.E; i += R_THREADS) {
      const int t = i / a.E, e = i - t * a.E;
      a.logits_out[(size_t)(t0 + t) * a.E + e] = lg[(size_t)t * a.Epad + e];
    }
  }
  // ---- route: one warp per token
  const int ld = a.k + a.n_shared;   // row stride of the outputs
  for (int t = warp; t < nt; t += R_THREADS / 32) {
    float* row = lg + (size_t)t * a.Epad;
    const int tg = t0 + t;
    if (a.mode == 2) {
      float* sc = scratch + (size_t)warp * 2 * a.Epad;
      route_row_grouped(row, sc, sc + a.Epad, a.bias, a.E, a.n_group, a.topk_group, a.k, a.scoring, a.renorm, a.rsf, a.out_w,
                        a.out_ids, tg, lane, ld);
    } else if (a.tid2eid) {
      route_row_hash(row, a.input_ids[tg], a.tid2eid, a.vocab, a.E, a.k, a.renorm, a.rsf, a.out_w, a.out_ids, tg, lane, ld);
    } else {
      route_row_topk(row, a.bias, a.E, a.k, a.mode == 3 ? 2 : a.mode, a.renorm, a.rsf, a.out_w, a.out_ids, nullptr, tg,
                     a.M, lane, ld);
    }
    __syncwarp();
    for (int j = lane; j < a.n_shared; j += 32) {
      a.out_ids[(size_t)tg * ld + a.k + j] = a.E + j;
      a.out_w[(size_t)tg * ld + a.k + j] = a.shared_w;
    }
    if (a.out_local) {
      __syncwarp();
      for (int j = lane; j < ld; j += 32) {
        const int v = a.out_ids[(size_t)tg * ld + j];
        int lv;
        if (j >= a.k) lv = a.shared_local_base >= 0 ? a.shared_local_base + (j - a.k) : -1;
        else lv = (v < 0 || !a.emap) ? v : a.emap[v < a.E ? v : a.E - 1];
        a.out_local[(size_t)tg * ld + j] = lv;
      }
    }
  }
}

// cache of gate-weight tensor maps (the pointer is stable for the life of the model)
struct WMapKey {
  const void* w;
  int E, H, dt;
};
static std::mutex g_wm_mu;
static WMapKey g_wm_key[64];
static CUtensorMap g_wm_val[64];
static int g_wm_n = 0;

static int router_shape(int M, int E, int H, int* TN, int* TT, int* EZ, int* KS) {
  const int ez = (E + 127) / 128, epad = ez * 128;
  int tn = 16;
  if (M > 256) tn = epad <= 256 ? 64 : epad <= 512 ? 32 : 16;
  const int tt = (M + tn - 1) / tn;
  const int kb = H / 64;
  // K splits: enough CTAs to pull the weights with the whole chip, but at least 4 k-blocks (64 KB of weights) per CTA
  // so that the partial-logit reduction of the last arriver stays one round trip
  int ks = 132 / (tt * ez);
  if (ks > kb / 4) ks = kb / 4;
  if (ks < 1) ks = 1;
  if (ks > kb) ks = kb;
  *TN = tn;
  *TT = tt;
  *EZ = ez;
  *KS = ks;
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" {

int64_t b200_router_workspace_bytes(int num_tokens, int num_experts, int hidden_size) {
  if (num_tokens <= 0 || num_experts <= 0 || hidden_size <= 0) return 0;
  int TN, TT, EZ, KS;
  router_shape(num_tokens, num_experts, hidden_size, &TN, &TT, &EZ, &KS);
  const int64_t counters = ((int64_t)TT * 4 + 255) / 256 * 256;
  return counters + (int64_t)KS * num_tokens * EZ * 128 * 4;
}

}  // extern "C"

// b200_router_topk and b200_router_hash_topk: tid2eid NULL routes by top-k
static int router_launch(const char* name, void* stream, const void* hidden, int act_dtype, const void* gate_weight,
                         int num_tokens, int num_experts, int hidden_size, const float* bias, int mode, int scoring,
                         int top_k, int renormalize, int n_group, int topk_group, float routed_scaling_factor,
                         const int32_t* expert_map, int n_shared, int shared_local_base, float shared_weight,
                         void* workspace, int64_t workspace_bytes, float* topk_weights, int32_t* topk_ids,
                         int32_t* local_ids, float* logits_out, const int32_t* input_ids, const int32_t* tid2eid,
                         int vocab) {
  const std::string fn(name);

  const int M = num_tokens, E = num_experts, H = hidden_size;
  if (!hidden || !gate_weight || !workspace || !topk_weights || !topk_ids || E <= 0 || E > MAX_EXPERTS || H <= 0 || H % 64 ||
      top_k <= 0 || top_k > E || mode < 0 || mode > 3 || n_shared < 0 || n_shared > 8 ||
      (act_dtype != B200_ACT_BF16 && act_dtype != B200_ACT_FP16)) {
    set_error(fn + ": bad argument (E <= 1024, H % 64 == 0, mode 0|1|2|3)");
    return B200_ERR_INVALID;
  }
  if (mode == 2 && (n_group <= 0 || n_group > 32 || E % n_group || topk_group <= 0 || topk_group > n_group ||
                    (scoring != 0 && scoring != 1))) {
    set_error(fn + ": bad grouped-routing argument (n_group <= 32, E % n_group == 0)");
    return B200_ERR_INVALID;
  }
  if (tid2eid && (!input_ids || vocab <= 0 || mode != 3 || top_k > 32)) {
    set_error(fn + ": bad hash-routing argument (input_ids non-NULL, vocab > 0, mode 3, top_k <= 32)");
    return B200_ERR_INVALID;
  }
  if (M <= 0) return 0;
  if (((uintptr_t)hidden & 15) || ((uintptr_t)gate_weight & 15)) {
    set_error(fn + ": hidden / gate_weight must be 16-byte aligned");
    return B200_ERR_INVALID;
  }
  int TN, TT, EZ, KS;
  router_shape(M, E, H, &TN, &TT, &EZ, &KS);
  if (workspace_bytes < b200_router_workspace_bytes(M, E, H)) {
    set_error(fn + ": workspace too small (b200_router_workspace_bytes)");
    return B200_ERR_INVALID;
  }
  RouterArgs a{};
  const int dt = act_dtype == B200_ACT_FP16 ? (int)CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : (int)CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  {
    std::lock_guard<std::mutex> lk(g_wm_mu);
    int hit = -1;
    for (int i = 0; i < g_wm_n; ++i)
      if (g_wm_key[i].w == gate_weight && g_wm_key[i].E == E && g_wm_key[i].H == H && g_wm_key[i].dt == dt) hit = i;
    if (hit < 0) {
      CUtensorMap tm;
      int rc = tm_encode_2d(&tm, dt, gate_weight, (uint64_t)H, (uint64_t)E, (uint64_t)H * 2, 64, 128);
      if (rc) return rc;
      hit = g_wm_n < 64 ? g_wm_n++ : 0;
      g_wm_key[hit] = WMapKey{gate_weight, E, H, dt};
      g_wm_val[hit] = tm;
    }
    a.tmW = g_wm_val[hit];
  }
  int rc = tm_encode_2d(&a.tmX, dt, hidden, (uint64_t)H, (uint64_t)M, (uint64_t)H * 2, 64, (uint32_t)TN);
  if (rc) return rc;
  a.M = M;
  a.E = E;
  a.H = H;
  a.KB = H / 64;
  a.KS = KS;
  a.TN = TN;
  a.EZ = EZ;
  a.Epad = EZ * 128;
  a.cmp_fp16 = act_dtype == B200_ACT_FP16;
  a.counters = reinterpret_cast<int32_t*>(workspace);
  a.partial = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + ((int64_t)TT * 4 + 255) / 256 * 256);
  a.logits_out = logits_out;
  a.mode = mode;
  a.scoring = scoring;
  a.k = top_k;
  a.renorm = renormalize;
  a.n_group = n_group;
  a.topk_group = topk_group;
  a.rsf = routed_scaling_factor;
  a.bias = bias;
  a.emap = expert_map;
  a.input_ids = input_ids;
  a.tid2eid = tid2eid;
  a.vocab = vocab;
  a.out_w = topk_weights;
  a.out_ids = topk_ids;
  a.out_local = local_ids;
  a.n_shared = n_shared;
  a.shared_local_base = shared_local_base;
  a.shared_w = shared_weight;
  const size_t route_scratch = (size_t)(R_THREADS / 32) * 2 * a.Epad * 4;
  const size_t smem = 1024 + (size_t)R_STAGES * (R_A_BYTES + TN * 128) + (size_t)TN * a.Epad * 4 + route_scratch;
  if ((rc = kernel_smem(reinterpret_cast<const void*>(router_gemm_topk_kernel), (int)smem, "cudaFuncSetAttribute(router)")))
    return rc;
  router_gemm_topk_kernel<<<dim3(KS, TT, EZ), R_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "router launch");
  return 0;
}

extern "C" {

int b200_router_topk(void* stream, const void* hidden, int act_dtype, const void* gate_weight, int num_tokens,
                     int num_experts, int hidden_size, const float* bias, int mode, int scoring, int top_k, int renormalize,
                     int n_group, int topk_group, float routed_scaling_factor, const int32_t* expert_map, int n_shared,
                     int shared_local_base, float shared_weight, void* workspace, int64_t workspace_bytes,
                     float* topk_weights, int32_t* topk_ids, int32_t* local_ids, float* logits_out) {
  return router_launch("b200_router_topk", stream, hidden, act_dtype, gate_weight, num_tokens, num_experts, hidden_size,
                       bias, mode, scoring, top_k, renormalize, n_group, topk_group, routed_scaling_factor, expert_map,
                       n_shared, shared_local_base, shared_weight, workspace, workspace_bytes, topk_weights, topk_ids,
                       local_ids, logits_out, nullptr, nullptr, 0);
}

int b200_router_hash_topk(void* stream, const void* hidden, int act_dtype, const void* gate_weight, int num_tokens,
                          int num_experts, int hidden_size, const float* bias, int mode, int scoring, int top_k,
                          int renormalize, int n_group, int topk_group, float routed_scaling_factor,
                          const int32_t* expert_map, int n_shared, int shared_local_base, float shared_weight,
                          void* workspace, int64_t workspace_bytes, float* topk_weights, int32_t* topk_ids,
                          int32_t* local_ids, float* logits_out, const int32_t* input_ids, const int32_t* tid2eid,
                          int vocab) {
  if (!tid2eid) {
    set_error("b200_router_hash_topk: tid2eid is NULL");
    return B200_ERR_INVALID;
  }
  return router_launch("b200_router_hash_topk", stream, hidden, act_dtype, gate_weight, num_tokens, num_experts,
                       hidden_size, bias, mode, scoring, top_k, renormalize, n_group, topk_group, routed_scaling_factor,
                       expert_map, n_shared, shared_local_base, shared_weight, workspace, workspace_bytes, topk_weights,
                       topk_ids, local_ids, logits_out, input_ids, tid2eid, vocab);
}

}  // extern "C"
