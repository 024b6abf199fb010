// Routing + permutation operators (latency / HBM bound integer & fp32 work; one warp per token).
//   b200_topk_gating      softmax / sigmoid / sqrt-softplus top-k, lower-index tie-break
//                                                                             (reference topk_softmax_kernels.cu:408-592)
//   b200_hash_topk        DeepSeek-V4 token-id hash routing                  (reference topk_softplus_sqrt_kernels.cu:326-403)
//   b200_grouped_topk     DeepSeek group-limited routing                     (reference grouped_topk_kernels.cu:477-675)
//   b200_global_to_local_ids                                                  (reference routed_experts.py:1332-1342)
//   b200_moe_permute / b200_moe_unpermute   stable sort by expert, gather, fp32 weighted reduce
//                                           (reference moe_permute_unpermute_op.cu:59-207)
#include "moe_internal.cuh"
#include "routing_device.cuh"

namespace b200 {

constexpr int ROUTE_WARPS = 4;
constexpr int MAX_VPT = MAX_EXPERTS / 32;

__global__ void __launch_bounds__(ROUTE_WARPS * 32)
    topk_gating_kernel(const void* __restrict__ logits, int dtype, const float* __restrict__ bias, int M, int E, int k,
                       int scoring, int renorm, float rsf, float* __restrict__ out_w, int32_t* __restrict__ out_ids,
                       int32_t* __restrict__ tok_exp_idx, const int32_t* __restrict__ input_ids,
                       const int32_t* __restrict__ tid2eid, int vocab) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * ROUTE_WARPS + warp;
  if (t >= M) return;
  float* p = sm + (size_t)warp * E;
  for (int e = lane; e < E; e += 32) p[e] = load_logit(logits, dtype, (size_t)t * E + e);
  __syncwarp();
  if (tid2eid)
    route_row_hash(p, input_ids[t], tid2eid, vocab, E, k, renorm, rsf, out_w, out_ids, t, lane, k);
  else
    route_row_topk(p, bias, E, k, scoring, renorm, rsf, out_w, out_ids, tok_exp_idx, t, M, lane, k);
}

__global__ void __launch_bounds__(ROUTE_WARPS * 32)
    grouped_topk_kernel(const void* __restrict__ logits, int dtype, const float* __restrict__ bias, int M, int E,
                        int n_group, int topk_group, int k, int scoring, int renorm, float rsf,
                        float* __restrict__ out_w, int32_t* __restrict__ out_ids) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * ROUTE_WARPS + warp;
  if (t >= M) return;
  float* raw = sm + (size_t)warp * 3 * E;
  for (int e = lane; e < E; e += 32) raw[e] = load_logit(logits, dtype, (size_t)t * E + e);
  __syncwarp();
  route_row_grouped(raw, raw + E, raw + 2 * E, bias, E, n_group, topk_group, k, scoring, renorm, rsf, out_w, out_ids, t, lane, k);
}

__global__ void g2l_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ emap, int n_global,
                           int64_t n, int32_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int v = ids[i];
  int c = v < 0 ? 0 : (v > n_global - 1 ? n_global - 1 : v);
  out[i] = v < 0 ? -1 : emap[c];
}

// ---------------------------------------------------------------------------------------- permute op
constexpr int PS_THREADS = 256;
__global__ void __launch_bounds__(PS_THREADS, 1)
    permute_sort_kernel(const int32_t* __restrict__ ids, int n_slots, int E, int32_t* __restrict__ sorted_slot,
                        int64_t* __restrict__ first_off, int32_t* __restrict__ inv_perm) {
  __shared__ int cnt[MAX_EXPERTS + 1];
  __shared__ int off[MAX_EXPERTS + 1];
  __shared__ int run[MAX_EXPERTS + 1];
  __shared__ int warp_tot[PS_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int NB = E + 1;  // bucket E collects the invalid slots (they sort to the end, stably)
  for (int e = tid; e < NB; e += PS_THREADS) {
    cnt[e] = 0;
    run[e] = 0;
  }
  __syncthreads();
  for (int s = tid; s < n_slots; s += PS_THREADS) {
    int e = ids[s];
    if (e < 0 || e >= E) e = E;
    atomicAdd(&cnt[e], 1);
  }
  __syncthreads();
  const int per = (NB + PS_THREADS - 1) / PS_THREADS;
  const int e0 = tid * per;
  int l = 0;
  for (int i = 0; i < per; ++i)
    if (e0 + i < NB) l += cnt[e0 + i];
  int inc = l;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int a = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += a;
  }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  int base = 0;
  for (int w = 0; w < warp; ++w) base += warp_tot[w];
  int x = base + inc - l;
  for (int i = 0; i < per; ++i) {
    const int e = e0 + i;
    if (e < NB) {
      off[e] = x;
      if (e <= E) first_off[e] = x;  // first_off[E] = number of valid rows
      x += cnt[e];
    }
  }
  __syncthreads();
  for (int b = 0; b < n_slots; b += PS_THREADS) {
    const int s = b + tid;
    int e = -2;
    if (s < n_slots) {
      e = ids[s];
      if (e < 0 || e >= E) e = E;
    }
    for (int w = 0; w < PS_THREADS / 32; ++w) {
      if (warp == w) {
        const unsigned m = __match_any_sync(0xffffffffu, e);
        const int rank = __popc(m & ((1u << lane) - 1u));
        if (e >= 0) {
          const int row = off[e] + run[e] + rank;
          sorted_slot[row] = s;
          inv_perm[s] = (e < E) ? row : -1;
        }
        __syncwarp();
        if (e >= 0 && rank == 0) run[e] += __popc(m);
      }
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(128) permute_gather_kernel(const uint4* __restrict__ hidden, int H8, int top_k,
                                                            const int32_t* __restrict__ sorted_slot,
                                                            const int64_t* __restrict__ first_off, int E,
                                                            uint4* __restrict__ out) {
  const int r = blockIdx.x;
  if (r >= (int)first_off[E]) return;
  const int t = sorted_slot[r] / top_k;
  for (int i = threadIdx.x; i < H8; i += 128) out[(size_t)r * H8 + i] = hidden[(size_t)t * H8 + i];
}

__global__ void __launch_bounds__(256)
    unpermute_kernel(const uint16_t* __restrict__ perm, int act_fp16, const float* __restrict__ w,
                     const int32_t* __restrict__ inv, int top_k, int H, void* __restrict__ out, int out_dtype) {
  const int t = blockIdx.y;
  const int h = (blockIdx.x * 256 + threadIdx.x) * 2;
  if (h >= H) return;
  float a0 = 0.f, a1 = 0.f;
  for (int j = 0; j < top_k; ++j) {
    const int row = inv[t * top_k + j];
    if (row < 0) continue;
    const float ww = w[t * top_k + j];
    const uint32_t raw = *reinterpret_cast<const uint32_t*>(perm + (size_t)row * H + h);
    float x0, x1;
    if (act_fp16) {
      const __half2 v = *reinterpret_cast<const __half2*>(&raw);
      x0 = __low2float(v);
      x1 = __high2float(v);
    } else {
      const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&raw);
      x0 = __low2float(v);
      x1 = __high2float(v);
    }
    a0 = fmaf(ww, x0, a0);
    a1 = fmaf(ww, x1, a1);
  }
  const size_t o = (size_t)t * H + h;
  if (out_dtype == 2) {
    reinterpret_cast<float*>(out)[o] = a0;
    reinterpret_cast<float*>(out)[o + 1] = a1;
  } else if (out_dtype == 0) {
    *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(out) + o) = __floats2bfloat162_rn(a0, a1);
  } else {
    *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(out) + o) = __floats2half2_rn(a0, a1);
  }
}

// out[t,:] = act_dtype( in[t,:] * gain * rsqrt(mean(in[t,:]^2) + eps) ): the fp32 -> activation-dtype cast
// the reference applies to lk_moe's output (routed_experts.py:1855) fused with an RMS normalisation (the op
// that follows in the decoder layer); one CTA per token.
__global__ void __launch_bounds__(256) rmsnorm_cast_kernel(const float* __restrict__ in, void* __restrict__ out,
                                                          int H, float gain, float eps, int out_fp16) {
  const int t = blockIdx.x;
  const float* x = in + (size_t)t * H;
  float ss = 0.f;
  for (int h = threadIdx.x * 4; h < H; h += 256 * 4) {
    const float4 v = *reinterpret_cast<const float4*>(x + h);
    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  __shared__ float red[8];
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  const float r = gain * rsqrtf(tot / (float)H + eps);
  for (int h = threadIdx.x * 4; h < H; h += 256 * 4) {
    const float4 v = *reinterpret_cast<const float4*>(x + h);
    uint2 pk;
    if (out_fp16) {
      __half2 a = __floats2half2_rn(v.x * r, v.y * r), b = __floats2half2_rn(v.z * r, v.w * r);
      pk.x = *reinterpret_cast<uint32_t*>(&a);
      pk.y = *reinterpret_cast<uint32_t*>(&b);
    } else {
      __nv_bfloat162 a = __floats2bfloat162_rn(v.x * r, v.y * r), b = __floats2bfloat162_rn(v.z * r, v.w * r);
      pk.x = *reinterpret_cast<uint32_t*>(&a);
      pk.y = *reinterpret_cast<uint32_t*>(&b);
    }
    *reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(out) + (size_t)t * H + h) = pk;
  }
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_topk_gating(void* stream, const void* logits, int logits_dtype, const float* bias, int num_tokens,
                     int num_experts, int top_k, int scoring, int renormalize, float routed_scaling_factor,
                     float* topk_weights, int32_t* topk_ids, int32_t* token_expert_indices) {
  if (!logits || !topk_weights || !topk_ids || num_experts <= 0 || num_experts > MAX_EXPERTS || top_k <= 0 ||
      top_k > num_experts || logits_dtype < 0 || logits_dtype > 2 || scoring < 0 || scoring > 2) {
    set_error("b200_topk_gating: bad argument (scoring 0 softmax | 1 sigmoid | 2 sqrtsoftplus)");
    return B200_ERR_INVALID;
  }
  if (num_tokens <= 0) return 0;
  const int grid = (num_tokens + ROUTE_WARPS - 1) / ROUTE_WARPS;
  const size_t smem = (size_t)ROUTE_WARPS * num_experts * sizeof(float);
  topk_gating_kernel<<<grid, ROUTE_WARPS * 32, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      logits, logits_dtype, bias, num_tokens, num_experts, top_k, scoring, renormalize, routed_scaling_factor,
      topk_weights, topk_ids, token_expert_indices, nullptr, nullptr, 0);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "topk_gating launch");
  return 0;
}

int b200_hash_topk(void* stream, const void* logits, int logits_dtype, const int32_t* input_ids, const int32_t* tid2eid,
                   int vocab, int num_tokens, int num_experts, int top_k, int renormalize, float routed_scaling_factor,
                   float* topk_weights, int32_t* topk_ids) {
  if (!logits || !input_ids || !tid2eid || !topk_weights || !topk_ids || vocab <= 0 || num_experts <= 0 ||
      num_experts > MAX_EXPERTS || top_k <= 0 || top_k > 32 || top_k > num_experts || logits_dtype < 0 ||
      logits_dtype > 2) {
    set_error("b200_hash_topk: bad argument (table and ids non-NULL, vocab > 0, top_k <= 32)");
    return B200_ERR_INVALID;
  }
  if (num_tokens <= 0) return 0;
  const int grid = (num_tokens + ROUTE_WARPS - 1) / ROUTE_WARPS;
  const size_t smem = (size_t)ROUTE_WARPS * num_experts * sizeof(float);
  topk_gating_kernel<<<grid, ROUTE_WARPS * 32, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      logits, logits_dtype, nullptr, num_tokens, num_experts, top_k, 2, renormalize, routed_scaling_factor,
      topk_weights, topk_ids, nullptr, input_ids, tid2eid, vocab);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "hash_topk launch");
  return 0;
}

int b200_grouped_topk(void* stream, const void* logits, int logits_dtype, const float* bias, int num_tokens,
                      int num_experts, int n_group, int topk_group, int top_k, int scoring, int renormalize,
                      float routed_scaling_factor, float* topk_weights, int32_t* topk_ids) {
  if (!logits || !topk_weights || !topk_ids || num_experts <= 0 || num_experts > MAX_EXPERTS || n_group <= 0 ||
      n_group > 32 || num_experts % n_group || topk_group <= 0 || topk_group > n_group || top_k <= 0 ||
      top_k > num_experts || logits_dtype < 0 || logits_dtype > 2 || (scoring != 0 && scoring != 1)) {
    set_error("b200_grouped_topk: bad argument (n_group <= 32, E % n_group == 0, scoring 0|1)");
    return B200_ERR_INVALID;
  }
  if (num_tokens <= 0) return 0;
  const int grid = (num_tokens + ROUTE_WARPS - 1) / ROUTE_WARPS;
  const size_t smem = (size_t)ROUTE_WARPS * 3 * num_experts * sizeof(float);
  grouped_topk_kernel<<<grid, ROUTE_WARPS * 32, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      logits, logits_dtype, bias, num_tokens, num_experts, n_group, topk_group, top_k, scoring, renormalize,
      routed_scaling_factor, topk_weights, topk_ids);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "grouped_topk launch");
  return 0;
}

int b200_global_to_local_ids(void* stream, const int32_t* topk_ids, const int32_t* expert_map, int num_global,
                             int64_t numel, int32_t* local_ids) {
  if (!topk_ids || !expert_map || !local_ids || num_global <= 0) {
    set_error("b200_global_to_local_ids: bad argument");
    return B200_ERR_INVALID;
  }
  if (numel <= 0) return 0;
  g2l_kernel<<<(unsigned)((numel + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      topk_ids, expert_map, num_global, numel, local_ids);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "g2l launch");
  return 0;
}

int b200_rmsnorm_cast(void* stream, const float* in, void* out, int num_tokens, int hidden_size, float gain,
                      float eps, int out_dtype) {
  if (!in || !out || hidden_size % 4 || (out_dtype != 0 && out_dtype != 1)) {
    set_error("b200_rmsnorm_cast: bad argument");
    return B200_ERR_INVALID;
  }
  if (num_tokens <= 0) return 0;
  rmsnorm_cast_kernel<<<num_tokens, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(in, out, hidden_size, gain,
                                                                                    eps, out_dtype);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "rmsnorm_cast launch");
  return 0;
}

int b200_moe_permute(void* stream, const void* hidden, const int32_t* topk_ids, int num_tokens, int top_k,
                     int num_local_experts, int hidden_size, int32_t* sorted_slot, int64_t* expert_first_offset,
                     int32_t* inv_perm, void* permuted_hidden) {
  if (!topk_ids || !sorted_slot || !expert_first_offset || !inv_perm || num_local_experts <= 0 ||
      num_local_experts > MAX_EXPERTS || top_k <= 0 || (permuted_hidden && (!hidden || hidden_size % 8))) {
    set_error("b200_moe_permute: bad argument");
    return B200_ERR_INVALID;
  }
  if (num_tokens <= 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int n = num_tokens * top_k;
  permute_sort_kernel<<<1, PS_THREADS, 0, st>>>(topk_ids, n, num_local_experts, sorted_slot, expert_first_offset,
                                                inv_perm);
  ++g_launches;
  if (permuted_hidden) {
    permute_gather_kernel<<<n, 128, 0, st>>>(reinterpret_cast<const uint4*>(hidden), hidden_size / 8, top_k,
                                             sorted_slot, expert_first_offset, num_local_experts,
                                             reinterpret_cast<uint4*>(permuted_hidden));
    ++g_launches;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "moe_permute launch");
  return 0;
}

int b200_moe_unpermute(void* stream, const void* permuted, int act_dtype, const float* topk_weights,
                       const int32_t* inv_perm, int num_tokens, int top_k, int hidden_size, void* out,
                       int out_dtype) {
  if (!permuted || !topk_weights || !inv_perm || !out || hidden_size % 2 || out_dtype < 0 || out_dtype > 2) {
    set_error("b200_moe_unpermute: bad argument");
    return B200_ERR_INVALID;
  }
  if (num_tokens <= 0) return 0;
  dim3 grid((hidden_size / 2 + 255) / 256, num_tokens);
  unpermute_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint16_t*>(permuted), act_dtype == B200_ACT_FP16, topk_weights, inv_perm, top_k,
      hidden_size, out, out_dtype);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "moe_unpermute launch");
  return 0;
}

}  // extern "C"
