// Per-token routing arithmetic shared by the stand-alone routing kernels (routing.cu) and the fused router
// (router.cu): one warp per token, scores in shared memory, k rounds of warp arg-max (ties -> lower expert index).
//   route_row_topk     softmax / sigmoid / sqrt-softplus top-k     (reference topk_softmax_kernels.cu:408-592,
//                                                                   topk_softplus_sqrt_kernels.cu:404-537)
//   route_row_hash     DeepSeek-V4 token-id hash routing           (reference topk_softplus_sqrt_kernels.cu:326-403)
//   route_row_grouped  DeepSeek group-limited routing              (reference grouped_topk_kernels.cu:477-675)
#pragma once
#include <math_constants.h>

#include "common.cuh"

namespace b200 {

B200_DEVICE float load_logit(const void* p, int dtype, size_t i) {
  if (dtype == 0) return reinterpret_cast<const float*>(p)[i];
  if (dtype == 1) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
  return __half2float(reinterpret_cast<const __half*>(p)[i]);
}

// (value desc, index asc) arg-max over the warp
B200_DEVICE void warp_argmax(float& v, int& idx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ov > v || (ov == v && oi < idx)) {
      v = ov;
      idx = oi;
    }
  }
}

// DeepSeek-V4 score sqrt(softplus(x)), with F.softplus's threshold of 20.  Accurate expf / log1pf (not the fast
// intrinsics) so that a float32 host oracle agrees to a few ulp.
B200_DEVICE float sqrt_softplus(float x) { return sqrtf(x > 20.f ? x : log1pf(expf(x))); }

// p[E] (shared memory): the token's raw fp32 logits on entry, overwritten by the scores (scoring 0 softmax,
// 1 sigmoid, 2 sqrt-softplus).  Writes row t (row stride ld >= k) of out_w / out_ids (/ tok_exp_idx).  Executed by one
// full warp.  Selection is by score + bias; the weight is the unbiased score.  For sqrt-softplus this follows the
// reference's dsv4_topk and torch paths, not its CUDA kernel, which weights by (s + b) - b.
B200_DEVICE void route_row_topk(float* p, const float* __restrict__ bias, int E, int k, int scoring, int renorm, float rsf,
                                float* __restrict__ out_w, int32_t* __restrict__ out_ids, int32_t* __restrict__ tok_exp_idx,
                                int t, int M, int lane, int ld) {
  float mx = -CUDART_INF_F;
  for (int e = lane; e < E; e += 32) mx = fmaxf(mx, p[e]);
  if (scoring == 0) {
    mx = warp_max(mx);
    float s = 0.f;
    for (int e = lane; e < E; e += 32) {
      const float v = expf(p[e] - mx);
      p[e] = v;
      s += v;
    }
    s = warp_sum(s);
    const float r = 1.f / s;
    for (int e = lane; e < E; e += 32) p[e] *= r;
  } else if (scoring == 1) {
    for (int e = lane; e < E; e += 32) p[e] = 1.0f / (1.0f + expf(-p[e]));
  } else {
    for (int e = lane; e < E; e += 32) p[e] = sqrt_softplus(p[e]);
  }
  for (int e = lane; e < E; e += 32) {
    const float v = p[e];
    if (isnan(v) || isinf(v)) p[e] = 0.f;
  }
  __syncwarp();
  uint32_t taken = 0;  // bit i <-> expert lane + 32*i
  float sel_sum = 0.f;
  for (int j = 0; j < k; ++j) {
    float bv = -CUDART_INF_F;
    int bi = 0x7fffffff;
    for (int e = lane, i = 0; e < E; e += 32, ++i) {
      if (taken >> i & 1u) continue;
      const float c = bias ? p[e] + bias[e] : p[e];
      if (c > bv || bi == 0x7fffffff) {  // strict >: lower index wins within the lane
        bv = c;
        bi = e;
      }
    }
    warp_argmax(bv, bi);
    const float w = p[bi];
    if ((bi & 31) == lane) taken |= 1u << (bi >> 5);
    if (lane == 0) {
      out_ids[(size_t)t * ld + j] = bi;
      if (tok_exp_idx) tok_exp_idx[(size_t)t * ld + j] = j * M + t;
      out_w[(size_t)t * ld + j] = w;
      sel_sum += w;
    }
  }
  if (lane == 0) {
    float scale = rsf;
    if (renorm) scale = scale / (sel_sum > 0.f ? sel_sum : 1.f);
    for (int j = 0; j < k; ++j) out_w[(size_t)t * ld + j] *= scale;
  }
}

// Hash routing of DeepSeek-V4's first layers: the experts of token t are tid2eid[token_id, 0..k) in table order (k <= 32,
// one lane per slot), weighted by their sqrt-softplus scores; no bias.  A token id outside [0, vocab) empties the row, a
// table entry outside [0, E) its slot: id -1, weight 0.  p[E]: the token's raw fp32 logits (read only).  One full warp.
B200_DEVICE void route_row_hash(const float* p, int token_id, const int32_t* __restrict__ tid2eid, int vocab, int E,
                                int k, int renorm, float rsf, float* __restrict__ out_w, int32_t* __restrict__ out_ids,
                                int t, int lane, int ld) {
  int id = -1;
  float w = 0.f;
  if (lane < k && token_id >= 0 && token_id < vocab) {
    const int e = tid2eid[(size_t)token_id * k + lane];
    if (e >= 0 && e < E) {
      const float s = sqrt_softplus(p[e]);
      id = e;
      w = (isnan(s) || isinf(s)) ? 0.f : s;
    }
  }
  float sum = 0.f;  // in slot order, like the top-k path
  for (int j = 0; j < k; ++j) sum += __shfl_sync(0xffffffffu, w, j);
  float scale = rsf;
  if (renorm) scale = scale / (sum > 0.f ? sum : 1.f);
  if (lane < k) {
    out_ids[(size_t)t * ld + lane] = id;
    out_w[(size_t)t * ld + lane] = w * scale;
  }
}

// raw[E]: the token's fp32 logits (shared memory, read only); sc[E], cand[E]: scratch.  One full warp.
B200_DEVICE void route_row_grouped(const float* raw, float* sc, float* cand, const float* __restrict__ bias, int E,
                                   int n_group, int topk_group, int k, int scoring, int renorm, float rsf,
                                   float* __restrict__ out_w, int32_t* __restrict__ out_ids, int t, int lane, int ld) {
  const int epg = E / n_group;
  for (int e = lane; e < E; e += 32) {
    const float x = raw[e];
    float s = x;
    if (scoring == 1) s = 0.5f * tanhf(0.5f * x) + 0.5f;
    sc[e] = s;
    // non-finite *inputs* never become candidates (reference :632-637); keep the biased value for the
    // group score like the reference's first phase does
    cand[e] = s + (bias ? bias[e] : 0.f);
  }
  __syncwarp();
  // group score: sum of the two largest biased scores (bias given) or the max (no bias)
  float gs = -CUDART_INF_F;
  if (lane < n_group) {
    float m1 = -CUDART_INF_F, m2 = -CUDART_INF_F;
    for (int i = 0; i < epg; ++i) {
      const float v = cand[lane * epg + i];
      if (v > m1) {
        m2 = m1;
        m1 = v;
      } else if (v > m2) {
        m2 = v;
      }
    }
    if (bias)
      gs = (epg > 1) ? (m1 + m2) : (m1 * 2.f);
    else
      gs = m1;
    if (isnan(gs)) gs = -CUDART_INF_F;
  }
  // rank of my group under (score desc, id asc)
  int rank = 0, n_finite = 0;
  for (int g = 0; g < 32; ++g) {
    const float og = __shfl_sync(0xffffffffu, gs, g);
    if (g < n_group) {
      if (og > gs || (og == gs && g < lane)) ++rank;
      if (og > -CUDART_INF_F) ++n_finite;
    }
  }
  const bool sel = (lane < n_group) && (rank < topk_group);
  const unsigned sel_mask = __ballot_sync(0xffffffffu, sel);
  if (n_finite < topk_group) {  // k-th selected group is -inf -> degenerate row (reference :603-618)
    for (int j = lane; j < k; j += 32) {
      out_ids[(size_t)t * ld + j] = j;
      out_w[(size_t)t * ld + j] = 1.0f / (float)k;
    }
    return;
  }
  for (int e = lane; e < E; e += 32) {
    const int g = e / epg;
    const float x = raw[e];
    const bool fin = !(isnan(x) || isinf(x));
    if (!((sel_mask >> g) & 1u) || !fin) cand[e] = -CUDART_INF_F;
  }
  __syncwarp();
  uint32_t taken = 0;
  float ssum = 1e-20f;
  for (int j = 0; j < k; ++j) {
    float bv = -CUDART_INF_F;
    int bi = 0x7fffffff;
    for (int e = lane, i = 0; e < E; e += 32, ++i) {
      if (taken >> i & 1u) continue;
      const float c = cand[e];
      if (c > bv || bi == 0x7fffffff) {
        bv = c;
        bi = e;
      }
    }
    warp_argmax(bv, bi);
    if ((bi & 31) == lane) taken |= 1u << (bi >> 5);
    if (lane == 0) {
      const float w = sc[bi];
      out_ids[(size_t)t * ld + j] = bi;
      out_w[(size_t)t * ld + j] = w;
      ssum += w;
    }
  }
  if (lane == 0) {
    float scale = rsf;
    if (renorm) scale = scale / ssum;
    for (int j = 0; j < k; ++j) out_w[(size_t)t * ld + j] *= scale;
  }
}

}  // namespace b200
