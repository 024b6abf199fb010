// DeepSeek-V4 manifold hyper-connections (mHC) for decode.  A token carries hc = 4 residual streams r_i [H]; around every
// sublayer the model (vllm/models/deepseek_v4/nvidia/model.py:899-992, 1204) runs
//   post     r'_j = bf16(post_j * x + sum_i comb_ij * r_i)                         (the previous sublayer's output x folded in)
//   pre      mixes = (r_flat . fn^T) * rsqrt(sum r_flat^2 / 4H + rms_eps), r_flat the fp32 row [4H]; three gate groups:
//            pre_i = sigmoid(mixes_i s0 + base_i) + pre_eps, post_mix_j = sigmoid(mixes_{4+j} s1 + base_{4+j}) * post_mult,
//            comb = sinkhorn(mixes_{8..24} s2 + base_{8..24}); layer_input = bf16(sum_i pre_i r_i), optionally RMS-normed
//   hc_head  the pre step with 4 outputs only: out = bf16(sum_i (sigmoid(mixes_i s0 + base_i) + eps) r_i)
// (reference kernels/mhc/torch.py:6-106, tilelang_kernels.py:305-350, 884-977).  One kernel family covers all of them:
//   mhc_partials_kernel<POST, NOUT>  phase 1, split over the reduction: CTA (split, token tile) owns hidden columns
//       [64 split, +64) of all 4 streams (256 flattened columns, one per thread) and 32 tokens.  A thread keeps its column of
//       fn (NOUT floats) in registers; with POST it computes and writes r' for its column.  Per token it writes the NOUT
//       dot products and the sum of squares of its 256 columns to the workspace, summed in a fixed order.
//   mhc_mix_kernel<NOUT, NORM>       phase 2, one CTA per token: sums the splits' partials in a fixed order, computes the
//       gates and the Sinkhorn normalisation (one warp, fp32, IEEE division), and the weighted sum of the streams, with the
//       RMSNorm fused in (NORM: the bf16 row kept in shared memory, the mean square taken from the unrounded fp32 row).
//   mhc_post_kernel                   post alone, elementwise; the post expression is mhc_post_value, shared with phase 1.
// The split count is H / 64 and a token's arithmetic does not depend on its tile or its batch, so every output of a token is
// the same bits at any batch size or position.  In the fused op the mixes come from the bf16 r' that the call returns, so the
// fused call equals mhc_post followed by mhc_pre bit for bit.
#include "common.cuh"
#include "moe_internal.cuh"

namespace b200 {

constexpr int MHC_COLS = 64;     // hidden columns per split (x 4 streams = the CTA's 256 threads)
constexpr int MHC_TILE = 32;     // tokens per phase-1 CTA
constexpr int MHC_BATCH = 4;     // tokens whose loads a phase-1 thread issues together
constexpr int MHC_NP = 25;       // workspace floats per (token, split): up to 24 dot products + the sum of squares
constexpr int MHC_MAX_H = 16384;

B200_DEVICE float bfv(__nv_bfloat16 v) { return __bfloat162float(v); }

// r'_j for one hidden position: post_j x + sum_i comb_ij r_i in fp32, in this order (rounded to bf16 by the caller)
B200_DEVICE float mhc_post_value(float x, float post_j, const float (&r)[4], const float (&comb_j)[4]) {
  float acc = __fmul_rn(post_j, x);
#pragma unroll
  for (int i = 0; i < 4; ++i) acc = fmaf(comb_j[i], r[i], acc);
  return acc;
}

B200_DEVICE float mhc_sigmoid(float z) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-z))); }

// v[0..P) of every lane -> lane l holds the warp's sum of v[l % P] in v[0] (reduce-scatter: P - 1 shuffles, then
// log2(32 / P) more).  The order of the additions is fixed, so the result is deterministic.
template <int O, int P>
B200_DEVICE void reduce_scatter_level(float (&v)[P], int lane) {
  if constexpr (O >= 1) {
    const bool hi = (lane & O) != 0;
#pragma unroll
    for (int k = 0; k < O; ++k) {
      const float send = hi ? v[k] : v[k + O];
      const float keep = hi ? v[k + O] : v[k];
      v[k] = keep + __shfl_xor_sync(0xffffffffu, send, O);
    }
    reduce_scatter_level<O / 2>(v, lane);
  }
}
template <int P>
B200_DEVICE float warp_reduce_scatter(float (&v)[P]) {
  reduce_scatter_level<P / 2>(v, threadIdx.x & 31);
#pragma unroll
  for (int o = P; o < 32; o *= 2) v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
  return v[0];
}

// grid (H / 64, ceil(T / 32)), 256 threads.  Thread = (stream j = tid / 64, hidden h = 64 split + tid % 64).
// part [T][S][MHC_NP] (S = H / 64): dot products 0..NOUT-1, then the sum of squares at NOUT.
template <bool POST, int NOUT>
__global__ void __launch_bounds__(256)
    mhc_partials_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ residual,
                        const float* __restrict__ post_in, const float* __restrict__ comb_in, const float* __restrict__ fn,
                        int T, int H, __nv_bfloat16* __restrict__ residual_out, float* __restrict__ part) {
  constexpr int NP = NOUT + 1, P = NOUT > 8 ? 32 : 8;
  __shared__ float red[MHC_BATCH][8][NP];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int j = tid >> 6, h = blockIdx.x * MHC_COLS + (tid & 63), S = gridDim.x;
  const size_t col = (size_t)j * H + h;
  float f[NOUT];
#pragma unroll
  for (int n = 0; n < NOUT; ++n) f[n] = fn[(size_t)n * 4 * H + col];
  const int t_end = min(T, (int)blockIdx.y * MHC_TILE + MHC_TILE);
  for (int t0 = blockIdx.y * MHC_TILE; t0 < t_end; t0 += MHC_BATCH) {
    float v[MHC_BATCH];
    if constexpr (POST) {
      float xs[MHC_BATCH], ps[MHC_BATCH], r[MHC_BATCH][4], c[MHC_BATCH][4];
#pragma unroll
      for (int b = 0; b < MHC_BATCH; ++b) {
        const int t = min(t0 + b, t_end - 1);
        xs[b] = bfv(x[(size_t)t * H + h]);
        ps[b] = post_in[t * 4 + j];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          r[b][i] = bfv(residual[(size_t)t * 4 * H + (size_t)i * H + h]);
          c[b][i] = comb_in[t * 16 + i * 4 + j];
        }
      }
#pragma unroll
      for (int b = 0; b < MHC_BATCH; ++b) {
        const __nv_bfloat16 o = __float2bfloat16_rn(mhc_post_value(xs[b], ps[b], r[b], c[b]));
        if (t0 + b < t_end) residual_out[(size_t)(t0 + b) * 4 * H + col] = o;
        v[b] = bfv(o);
      }
    } else {
#pragma unroll
      for (int b = 0; b < MHC_BATCH; ++b) v[b] = bfv(residual[(size_t)min(t0 + b, t_end - 1) * 4 * H + col]);
    }
#pragma unroll
    for (int b = 0; b < MHC_BATCH; ++b) {
      if (t0 + b < t_end) {
        float a[P];
#pragma unroll
        for (int n = 0; n < P; ++n) a[n] = n < NOUT ? __fmul_rn(f[n], v[b]) : (n == NOUT ? __fmul_rn(v[b], v[b]) : 0.f);
        const float s = warp_reduce_scatter<P>(a);
        if (lane < NP) red[b][warp][lane] = s;
      }
    }
    __syncthreads();
    if (tid < MHC_BATCH * NP) {
      const int b = tid / NP, n = tid % NP;
      if (t0 + b < t_end) {
        float s = red[b][0][n];
#pragma unroll
        for (int w = 1; w < 8; ++w) s += red[b][w][n];
        part[((size_t)(t0 + b) * S + blockIdx.x) * MHC_NP + n] = s;
      }
    }
    __syncthreads();
  }
}

// grid T, 256 threads.  r [T, 4, H] bf16 (the call's r' in the fused op).  NOUT 24: pre / post_mix / comb gates and the
// Sinkhorn normalisation; NOUT 4: hc_head (pre gates only, eps = pre_eps).
template <int NOUT, bool NORM>
__global__ void __launch_bounds__(256)
    mhc_mix_kernel(const __nv_bfloat16* __restrict__ r, const float* __restrict__ part, int H,
                   const float* __restrict__ hc_scale, const float* __restrict__ hc_base, float rms_eps, float pre_eps,
                   float sk_eps, float post_mult, int repeat, const __nv_bfloat16* __restrict__ norm_w, float norm_eps,
                   float* __restrict__ post_mix, float* __restrict__ comb_mix, __nv_bfloat16* __restrict__ out) {
  constexpr int NP = NOUT + 1;
  __shared__ float sums[8][NP];
  __shared__ float pre[4];
  __shared__ float ssw[8];
  __shared__ __align__(16) __nv_bfloat16 row[NORM ? MHC_MAX_H : 8];
  const int t = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, S = H / MHC_COLS;
  // splits w, w + 8, ... per warp, then the 8 warps in order
  if (lane < NP) {
    const float* p = part + (size_t)t * S * MHC_NP + lane;
    float a = 0.f;
    for (int s = warp; s < S; s += 8) a += p[(size_t)s * MHC_NP];
    sums[warp][lane] = a;
  }
  __syncthreads();
  if (warp == 0) {
    float m = 0.f;
    if (lane < NP) {
      m = sums[0][lane];
#pragma unroll
      for (int w = 1; w < 8; ++w) m += sums[w][lane];
    }
    const float ss = __shfl_sync(0xffffffffu, m, NOUT);
    const float mix = __fmul_rn(m, rsqrtf(__fadd_rn(__fdiv_rn(ss, (float)(4 * H)), rms_eps)));
    if (lane < 4) pre[lane] = __fadd_rn(mhc_sigmoid(fmaf(mix, hc_scale[0], hc_base[lane])), pre_eps);
    if constexpr (NOUT == 24) {
      if (lane >= 4 && lane < 8)
        post_mix[(size_t)t * 4 + lane - 4] = __fmul_rn(mhc_sigmoid(fmaf(mix, hc_scale[1], hc_base[lane])), post_mult);
      // comb element (i, k) = lane i * 4 + k (lanes 16-31 mirror 0-15): rows are lanes ^ 1, ^ 2, columns lanes ^ 4, ^ 8
      const int e = lane & 15;
      const float z = fmaf(__shfl_sync(0xffffffffu, mix, 8 + e), hc_scale[2], hc_base[8 + e]);
      float mx = fmaxf(z, __shfl_xor_sync(0xffffffffu, z, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float ex = expf(__fsub_rn(z, mx));
      float rs = ex + __shfl_xor_sync(0xffffffffu, ex, 1);
      rs += __shfl_xor_sync(0xffffffffu, rs, 2);
      float c = __fadd_rn(__fdiv_rn(ex, rs), sk_eps);
      float cs = c + __shfl_xor_sync(0xffffffffu, c, 4);
      cs += __shfl_xor_sync(0xffffffffu, cs, 8);
      c = __fdiv_rn(c, __fadd_rn(cs, sk_eps));
      for (int it = 1; it < repeat; ++it) {
        rs = c + __shfl_xor_sync(0xffffffffu, c, 1);
        rs += __shfl_xor_sync(0xffffffffu, rs, 2);
        c = __fdiv_rn(c, __fadd_rn(rs, sk_eps));
        cs = c + __shfl_xor_sync(0xffffffffu, c, 4);
        cs += __shfl_xor_sync(0xffffffffu, cs, 8);
        c = __fdiv_rn(c, __fadd_rn(cs, sk_eps));
      }
      if (lane < 16) comb_mix[(size_t)t * 16 + lane] = c;
    }
  }
  __syncthreads();
  const float p0 = pre[0], p1 = pre[1], p2 = pre[2], p3 = pre[3];
  const __nv_bfloat16* rt = r + (size_t)t * 4 * H;
  __nv_bfloat16* ot = out + (size_t)t * H;
  float ss = 0.f;
  for (int c8 = tid * 8; c8 < H; c8 += 256 * 8) {
    uint4 raw[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) raw[i] = *reinterpret_cast<const uint4*>(rt + (size_t)i * H + c8);
    uint32_t pk[4];
#pragma unroll
    for (int k = 0; k < 8; k += 2) {
      float o[2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int kk = k + u;
        float a = __fmul_rn(p0, bfv(reinterpret_cast<const __nv_bfloat16*>(&raw[0])[kk]));
        a = fmaf(p1, bfv(reinterpret_cast<const __nv_bfloat16*>(&raw[1])[kk]), a);
        a = fmaf(p2, bfv(reinterpret_cast<const __nv_bfloat16*>(&raw[2])[kk]), a);
        a = fmaf(p3, bfv(reinterpret_cast<const __nv_bfloat16*>(&raw[3])[kk]), a);
        if constexpr (NORM) ss = fmaf(a, a, ss);
        o[u] = a;
      }
      const __nv_bfloat162 b2 = __floats2bfloat162_rn(o[0], o[1]);
      pk[k / 2] = *reinterpret_cast<const uint32_t*>(&b2);
    }
    *reinterpret_cast<uint4*>(NORM ? row + c8 : ot + c8) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
  }
  if constexpr (NORM) {
    ss = warp_sum(ss);
    if (lane == 0) ssw[warp] = ss;
    __syncthreads();
    float tot = ssw[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) tot += ssw[w];
    const float rn = rsqrtf(__fadd_rn(__fdiv_rn(tot, (float)H), norm_eps));
    for (int c8 = tid * 8; c8 < H; c8 += 256 * 8) {
      const uint4 rv = *reinterpret_cast<const uint4*>(row + c8);
      const uint4 wv = *reinterpret_cast<const uint4*>(norm_w + c8);
      const __nv_bfloat16* rb = reinterpret_cast<const __nv_bfloat16*>(&rv);
      const __nv_bfloat16* wb = reinterpret_cast<const __nv_bfloat16*>(&wv);
      uint32_t pk[4];
#pragma unroll
      for (int k = 0; k < 8; k += 2) {
        const __nv_bfloat162 b2 = __floats2bfloat162_rn(__fmul_rn(__fmul_rn(bfv(rb[k]), rn), bfv(wb[k])),
                                                        __fmul_rn(__fmul_rn(bfv(rb[k + 1]), rn), bfv(wb[k + 1])));
        pk[k / 2] = *reinterpret_cast<const uint32_t*>(&b2);
      }
      *reinterpret_cast<uint4*>(ot + c8) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    }
  }
}

// grid T, 128 threads; a thread takes 8 consecutive hidden positions of all four output streams
__global__ void __launch_bounds__(128)
    mhc_post_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ residual,
                    const float* __restrict__ post_in, const float* __restrict__ comb_in, int H,
                    __nv_bfloat16* __restrict__ out) {
  const int t = blockIdx.x;
  float post[4], comb[4][4];   // comb[j][i] = comb_in[t, i, j]
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    post[j] = post_in[t * 4 + j];
#pragma unroll
    for (int i = 0; i < 4; ++i) comb[j][i] = comb_in[t * 16 + i * 4 + j];
  }
  const __nv_bfloat16* rt = residual + (size_t)t * 4 * H;
  for (int c8 = threadIdx.x * 8; c8 < H; c8 += 128 * 8) {
    const uint4 xv = *reinterpret_cast<const uint4*>(x + (size_t)t * H + c8);
    uint4 rv[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) rv[i] = *reinterpret_cast<const uint4*>(rt + (size_t)i * H + c8);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint32_t pk[4];
#pragma unroll
      for (int k = 0; k < 8; k += 2) {
        float o[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          float r[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) r[i] = bfv(reinterpret_cast<const __nv_bfloat16*>(&rv[i])[k + u]);
          o[u] = mhc_post_value(bfv(reinterpret_cast<const __nv_bfloat16*>(&xv)[k + u]), post[j], r, comb[j]);
        }
        const __nv_bfloat162 b2 = __floats2bfloat162_rn(o[0], o[1]);
        pk[k / 2] = *reinterpret_cast<const uint32_t*>(&b2);
      }
      *reinterpret_cast<uint4*>(out + (size_t)t * 4 * H + (size_t)j * H + c8) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    }
  }
}

}  // namespace b200

using namespace b200;

namespace {

bool a16(const void* p) { return p && (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
bool a4(const void* p) { return p && (reinterpret_cast<uintptr_t>(p) & 3u) == 0; }
bool shape_ok(int T, int H) { return T >= 1 && T <= (1 << 20) && H >= 256 && H <= MHC_MAX_H && H % MHC_COLS == 0; }

int launched(const char* what) {
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : cuda_fail(e, what);
}

}  // namespace

extern "C" {

int64_t b200_mhc_workspace_bytes(int num_tokens, int hidden_size) {
  if (num_tokens < 0 || hidden_size < MHC_COLS) return 0;
  return (int64_t)num_tokens * (hidden_size / MHC_COLS) * MHC_NP * (int64_t)sizeof(float);
}

int b200_mhc_post_pre(void* stream, const void* x, const void* residual, const float* post_layer_mix,
                      const float* comb_res_mix, const float* fn, const float* hc_scale, const float* hc_base,
                      const void* norm_weight, int num_tokens, int hidden_size, float rms_eps, float hc_pre_eps,
                      float hc_sinkhorn_eps, float hc_post_mult_value, int sinkhorn_repeat, float norm_eps,
                      void* workspace, void* residual_out, float* post_mix, float* comb_mix, void* layer_input) {
  const bool post = x != nullptr;
  const bool post_args = post ? a16(x) && a4(post_layer_mix) && a4(comb_res_mix) && a16(residual_out)
                              : !post_layer_mix && !comb_res_mix && !residual_out;
  if (!post_args || !a16(residual) || !a16(fn) || !a4(hc_scale) || !a4(hc_base) || (norm_weight && !a16(norm_weight)) ||
      !shape_ok(num_tokens, hidden_size) || sinkhorn_repeat < 1 || !(rms_eps >= 0.f) || !(hc_pre_eps >= 0.f) ||
      !(hc_sinkhorn_eps >= 0.f) || !(norm_eps >= 0.f) || !a16(workspace) || !a4(post_mix) || !a4(comb_mix) ||
      !a16(layer_input)) {
    set_error("b200_mhc_post_pre: bad argument (16-byte aligned bf16 tensors, fn and workspace; 1 <= num_tokens <= 2^20; "
              "hidden_size a multiple of 64 in [256, 16384]; sinkhorn_repeat >= 1; eps >= 0; with x NULL, "
              "post_layer_mix, comb_res_mix and residual_out NULL)");
    return B200_ERR_INVALID;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int T = num_tokens, H = hidden_size;
  const dim3 g1(H / MHC_COLS, (T + MHC_TILE - 1) / MHC_TILE);
  const auto* res = reinterpret_cast<const __nv_bfloat16*>(residual);
  auto* rout = reinterpret_cast<__nv_bfloat16*>(residual_out);
  auto* part = reinterpret_cast<float*>(workspace);
  if (post)
    mhc_partials_kernel<true, 24><<<g1, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), res, post_layer_mix,
                                                       comb_res_mix, fn, T, H, rout, part);
  else
    mhc_partials_kernel<false, 24><<<g1, 256, 0, st>>>(nullptr, res, nullptr, nullptr, fn, T, H, nullptr, part);
  if (int rc = launched("mhc_partials launch")) return rc;
  const __nv_bfloat16* r = post ? rout : res;
  const auto* w = reinterpret_cast<const __nv_bfloat16*>(norm_weight);
  auto* out = reinterpret_cast<__nv_bfloat16*>(layer_input);
  if (norm_weight)
    mhc_mix_kernel<24, true><<<T, 256, 0, st>>>(r, part, H, hc_scale, hc_base, rms_eps, hc_pre_eps, hc_sinkhorn_eps,
                                                hc_post_mult_value, sinkhorn_repeat, w, norm_eps, post_mix, comb_mix, out);
  else
    mhc_mix_kernel<24, false><<<T, 256, 0, st>>>(r, part, H, hc_scale, hc_base, rms_eps, hc_pre_eps, hc_sinkhorn_eps,
                                                 hc_post_mult_value, sinkhorn_repeat, nullptr, 0.f, post_mix, comb_mix, out);
  return launched("mhc_mix launch");
}

int b200_mhc_post(void* stream, const void* x, const void* residual, const float* post_layer_mix, const float* comb_res_mix,
                  int num_tokens, int hidden_size, void* out) {
  if (!a16(x) || !a16(residual) || !a4(post_layer_mix) || !a4(comb_res_mix) || !a16(out) ||
      !shape_ok(num_tokens, hidden_size)) {
    set_error("b200_mhc_post: bad argument (16-byte aligned x, residual and out; 1 <= num_tokens <= 2^20; hidden_size a "
              "multiple of 64 in [256, 16384])");
    return B200_ERR_INVALID;
  }
  mhc_post_kernel<<<num_tokens, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<const __nv_bfloat16*>(residual), post_layer_mix,
      comb_res_mix, hidden_size, reinterpret_cast<__nv_bfloat16*>(out));
  return launched("mhc_post launch");
}

int b200_hc_head(void* stream, const void* residual, const float* fn, const float* hc_scale, const float* hc_base,
                 int num_tokens, int hidden_size, float rms_eps, float hc_eps, void* workspace, void* out) {
  if (!a16(residual) || !a16(fn) || !a4(hc_scale) || !a4(hc_base) || !shape_ok(num_tokens, hidden_size) ||
      !(rms_eps >= 0.f) || !(hc_eps >= 0.f) || !a16(workspace) || !a16(out)) {
    set_error("b200_hc_head: bad argument (16-byte aligned residual, fn, workspace and out; 1 <= num_tokens <= 2^20; "
              "hidden_size a multiple of 64 in [256, 16384]; eps >= 0)");
    return B200_ERR_INVALID;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int T = num_tokens, H = hidden_size;
  const auto* res = reinterpret_cast<const __nv_bfloat16*>(residual);
  auto* part = reinterpret_cast<float*>(workspace);
  mhc_partials_kernel<false, 4><<<dim3(H / MHC_COLS, (T + MHC_TILE - 1) / MHC_TILE), 256, 0, st>>>(
      nullptr, res, nullptr, nullptr, fn, T, H, nullptr, part);
  if (int rc = launched("hc_head partials launch")) return rc;
  mhc_mix_kernel<4, false><<<T, 256, 0, st>>>(res, part, H, hc_scale, hc_base, rms_eps, hc_eps, 0.f, 0.f, 1, nullptr, 0.f,
                                              nullptr, nullptr, reinterpret_cast<__nv_bfloat16*>(out));
  return launched("hc_head mix launch");
}

}  // extern "C"
