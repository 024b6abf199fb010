// C ABI of libb200moe.so (see include/b200moe.h).  Host-side glue only: validation, HBM ingest of the
// expert weights, workspace management and kernel sequencing.  No CPU compute path exists: every entry
// point fails loudly when there is no sm_90 device.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "moe_internal.cuh"

namespace b200 {

static thread_local std::string g_err;
long long g_launches = 0;

void set_error(const std::string& msg) { g_err = msg; }
int cuda_fail(cudaError_t e, const char* what) {
  g_err = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
  return B200_ERR_CUDA;
}

static int check_device(int* dev_out) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    cuda_fail(e, "cudaGetDevice");
    return B200_ERR_NO_DEVICE;
  }
  int major = 0;
  e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  if (e != cudaSuccess) {
    cuda_fail(e, "cudaDeviceGetAttribute");
    return B200_ERR_NO_DEVICE;
  }
  if (major != 9) {
    set_error("libb200moe needs an sm_90 (H100) device; found compute capability major " + std::to_string(major));
    return B200_ERR_NO_DEVICE;
  }
  *dev_out = dev;
  return 0;
}

// optional per-kernel timing of the two expert GEMMs (bench.py roofline): CUDA events recorded on the
// launching stream around each GEMM when enabled and not capturing
static bool g_profile = false;
struct EvTriple { cudaEvent_t e[3];   bool fused = false;   // one kernel: only e[0]..e[1] is meaningful
};
static std::vector<EvTriple> g_events;
static size_t g_events_used = 0;
static std::mutex g_prof_mu;   // layers may be driven from several host threads (one per stream / ubatch)

static cudaEvent_t* next_events(bool fused) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (g_events_used == g_events.size()) {
    EvTriple t;
    for (int i = 0; i < 3; ++i) cudaEventCreate(&t.e[i]);
    g_events.push_back(t);
  }
  g_events[g_events_used].fused = fused;
  return g_events[g_events_used++].e;
}

// cuTensorMapEncodeTiled is fetched from the driver at run time (no link-time dependency on libcuda)
typedef CUresult (*TmEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static std::mutex g_tm_mu;
// generic 2-D tiled tensor map (dim 0 contiguous); shared by the MoE layer ctor and the router operator
int tm_encode_2d(CUtensorMap* tm, int dtype, const void* base, uint64_t d0, uint64_t d1, uint64_t stride1_bytes,
                 uint32_t b0, uint32_t b1) {
  static TmEncodeFn fn = nullptr;
  {
    std::lock_guard<std::mutex> lk(g_tm_mu);
    if (!fn) {
      void* p = nullptr;
      cudaDriverEntryPointQueryResult q;
      cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
      if (e != cudaSuccess || !p || q != cudaDriverEntryPointSuccess) {
        set_error("cuTensorMapEncodeTiled is not available from this driver");
        return B200_ERR_CUDA;
      }
      fn = reinterpret_cast<TmEncodeFn>(p);
    }
  }
  if (d0 == 0 || d1 == 0 || d1 > 0xFFFFFFFFull) {
    set_error("tensor map: dimension out of range");
    return B200_ERR_INVALID;
  }
  const cuuint64_t gdim[2] = {d0, d1};
  const cuuint64_t gstr[1] = {stride1_bytes};
  const cuuint32_t box[2] = {b0, b1};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(tm, static_cast<CUtensorMapDataType>(dtype), 2, const_cast<void*>(base), gdim, gstr, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
    return B200_ERR_CUDA;
  }
  return 0;
}

// Per-device launch set-up.  A kernel's dynamic shared-memory limit is an attribute of the device's context, so it is
// raised once per (device, kernel); the SM counts and cpu_prefill's streams are per device too.
static std::mutex g_setup_mu;
static std::map<std::pair<int, const void*>, int> g_smem_set;
static std::map<int, int> g_sms;
static std::map<int, cudaStream_t> g_prefill_stream;

int kernel_smem(const void* fn, int bytes, const char* what) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return cuda_fail(e, "cudaGetDevice");
  std::lock_guard<std::mutex> lk(g_setup_mu);
  int& set = g_smem_set[{dev, fn}];
  if (bytes <= set) return 0;
  e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return cuda_fail(e, what);
  set = bytes;
  return 0;
}

int device_sms(int dev) {
  std::lock_guard<std::mutex> lk(g_setup_mu);
  int& n = g_sms[dev];
  if (!n) {
    cudaError_t e = cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) {
      n = 0;
      return cuda_fail(e, "cudaDeviceGetAttribute(SM count)");
    }
  }
  return n;
}

static bool stream_capturing(cudaStream_t st) {
  cudaStreamCaptureStatus s = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &s) != cudaSuccess) return false;
  return s != cudaStreamCaptureStatusNone;
}

// All layers and streams of a device share one workspace and the fused kernel's cross-CTA counters.  Calls on one
// stream are ordered by the stream; an eager call arriving on ANOTHER stream is ordered behind the previous one with
// an event (graph-captured calls are ordered by the graph's own edges: Lvllm captures one stream).
static void wait_last_use(Workspace* ws, cudaStream_t st) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (ws->last_valid && ws->last_stream != st) cudaStreamWaitEvent(st, ws->last_use, 0);
}

static void record_last_use(Workspace* ws, cudaStream_t st) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (!ws->last_use) cudaEventCreateWithFlags(&ws->last_use, cudaEventDisableTiming);
  cudaEventRecord(ws->last_use, st);
  ws->last_stream = st;
  ws->last_valid = true;
}

// one full forward of the routed experts on device buffers
static int forward_device(b200moe_layer* L, cudaStream_t st, int M, int k, const void* hidden, const int32_t* ids,
                          const float* w, void* out, int out_dtype) {
  if (M <= 0) return 0;
  if (k <= 0 || k > 64) {
    set_error("top_k out of range");
    return B200_ERR_INVALID;
  }
  Workspace* ws = get_workspace(L->device);
  const bool cap = stream_capturing(st);
  if (!cap) wait_last_use(ws, st);
  // 4-bit layers, prefill-class batches (eager calls only): expand the experts once into fp16 tiles and run the batch
  // through the 16-bit grouped GEMM in passes of up to 8192 tokens, instead of re-streaming the packed weights through
  // the fused decode kernel once per 256 tokens.  W4A16 numerics for every 4-bit format on this path (native-MX layers
  // too: prefill keeps the activations in 16 bits).
  const int w4_prefill_min = [] {
    const char* v = getenv("B200MOE_W4_PREFILL_MIN");
    return v ? atoi(v) : 1024;
  }();
  const bool expand = L->wq && !cap && w4_prefill_min > 0 && M >= w4_prefill_min;
  b200moe_layer P;                 // fp16 shadow of a 4-bit layer: same geometry, expanded weights
  const b200moe_layer* V = L;      // the layer the passes run
  int pass;
  if (expand) {
    P = *L;
    P.wq = 0;
    P.esz_bits = 16;
    P.KB1 = L->H / 64;
    P.KB2 = L->I / 64;
    P.ws13 = P.ws2 = nullptr;
    P.cvt_bf16_to_fp16 = (L->act_dtype == B200_ACT_BF16);
    P.act_dtype = B200_ACT_FP16;
    const int64_t b13 = (int64_t)L->E * L->J1 * P.KB1 * 2 * TILE_BYTES, b2 = (int64_t)L->E * L->J2 * P.KB2 * TILE_BYTES;
    int rc = ensure_dequant_scratch(ws, b13, b2);
    if (rc) return rc;
    P.w13t = ws->dq13;
    P.w2t = ws->dq2;
    if ((rc = launch_w4_dequant(L, ws->dq13, ws->dq2, st))) return rc;
    V = &P;
    pass = L->cfg.max_batch_size > 0 ? L->cfg.max_batch_size : 4096;
    if (pass > 8192) pass = 8192;
    if (pass < 256) pass = 256;
  } else {
    // passes bound the workspace for very large prefill batches; below the prefill threshold 4-bit formats run through
    // the fused decode kernel, so their pass is the largest batch that kernel's tables hold (M * top_k <= 2048 slots)
    pass = L->max_tokens;
    if (L->wq) {
      if (pass > FUSED_MAX_TOKENS) pass = FUSED_MAX_TOKENS;
      while (pass > 1 && !fused_supported(L, pass, k)) pass = pass > 16 ? pass - 8 : pass - 1;
      if (!fused_supported(L, pass, k)) {
        set_error("4-bit formats are served by the fused decode kernel only and this layer / top_k is outside its limits "
                  "(experts <= 512, top_k <= 2048 slots per pass)");
        return B200_ERR_INVALID;
      }
    }
  }
  for (int t0 = 0; t0 < M; t0 += pass) {
    const int m = (M - t0 < pass) ? (M - t0) : pass;
    int rc = ensure_workspace(ws, V, m, k, !cap);
    if (rc) return rc;
    const size_t osz = (out_dtype == 2) ? 4 : 2;
    void* optr = reinterpret_cast<uint8_t*>(out) + (size_t)t0 * L->H * osz;
    const uint8_t* hptr = reinterpret_cast<const uint8_t*>(hidden) + (size_t)t0 * L->H * 2;
    // The fp16 shadow never takes the fused kernel: launch_fused ignores cvt_bf16_to_fp16 (it would read bf16 rows as
    // fp16), and with fp16 activations a short last pass would switch kernels and so change bits.
    if (!expand && fused_supported(L, m, k)) {
      cudaEvent_t* fev = nullptr;
      if (g_profile && !cap) {
        fev = next_events(true);
        cudaEventRecord(fev[0], st);
      }
      rc = launch_fused(L, ws, st, hptr, ids + (size_t)t0 * k, w + (size_t)t0 * k, m, k, optr, out_dtype);
      if (fev) cudaEventRecord(fev[1], st);
      if (rc) return rc;
      continue;
    }
    if (V->wq) {
      set_error("4-bit formats are served by the fused decode kernel only (this call is outside its limits)");
      return B200_ERR_INVALID;
    }
    const int tn_max = pick_tn_max(m, k, L->E);
    if ((rc = launch_prep(V, ws, st, hptr, ids + (size_t)t0 * k, m, k, tn_max))) return rc;
    cudaEvent_t* ev = (g_profile && !cap) ? next_events(false) : nullptr;
    if ((rc = launch_gemms(V, ws, st, m, k, tn_max, ev))) return rc;
    if ((rc = launch_combine(V, ws, st, w + (size_t)t0 * k, m, k, optr, out_dtype))) return rc;
  }
  if (!cap) record_last_use(ws, st);
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" {

const char* b200moe_last_error(void) { return g_err.c_str(); }
const char* b200moe_version(void) { return "b200moe 0.1 sm_90a"; }
int64_t b200moe_launch_count(void) { return g_launches; }

// ---- per-expert ingest (SURVEY.md 8f row 4: checkpoint -> HBM without a stacked [E, ...] host tensor).  Validation
// and layer geometry; which scale tensors the format needs is checked by b200moe_load_experts.
int b200moe_create_empty(const b200moe_config* cfg, int format, int act_dtype, b200moe_handle* out) {
  if (!cfg || !out) {
    set_error("b200moe_create: null config / output");
    return B200_ERR_INVALID;
  }
  if (cfg->activation_type < 0 || cfg->activation_type > 3) {
    set_error("b200moe_create: activation_type must be 0 silu, 1 swigluoai, 2 relu^2 or 3 silu with clamp");
    return B200_ERR_INVALID;
  }
  // activation_type 3 (DeepSeek-V4): gate = min(gate, limit), up = clamp(up, -limit, limit), silu(gate) * up.  Type 3
  // has no default limit: 0 would clamp every gate to 0.
  if (cfg->activation_type == 3 && !(cfg->swiglu_limit > 0.f)) {
    set_error("b200moe_create: activation_type 3 needs swiglu_limit > 0");
    return B200_ERR_INVALID;
  }
  int dev = 0;
  int rc = check_device(&dev);
  if (rc) return rc;
  const int E = cfg->expert_num, H = cfg->hidden_size, I = cfg->intermediate_size;
  if (E <= 0 || E > MAX_EXPERTS || H <= 0 || I <= 0 || cfg->top_k <= 0) {
    set_error("b200moe_create: bad expert_num / hidden_size / intermediate_size / top_k");
    return B200_ERR_INVALID;
  }
  if (H % 128 || I % 128) {
    set_error("b200moe_create: hidden_size and intermediate_size (per partition) must be multiples of 128");
    return B200_ERR_INVALID;
  }
  if (act_dtype != B200_ACT_BF16 && act_dtype != B200_ACT_FP16) {
    set_error("b200moe_create: act_dtype must be bf16 or fp16");
    return B200_ERR_INVALID;
  }
  if (format < B200_FMT_16BIT || format > B200_FMT_MXFP4) {
    set_error("b200moe_create: unknown weight format " + std::to_string(format));
    return B200_ERR_INVALID;
  }
  const bool w4 = (format == B200_FMT_WNA16 || format == B200_FMT_NVFP4 || format == B200_FMT_MXFP4);
  if (w4) {
    if (!cfg->has_gate_proj || (H / 128) % 2) {
      set_error("b200moe_create: 4-bit formats need gated experts and hidden_size % 256 == 0");
      return B200_ERR_INVALID;
    }
    const int gk = cfg->groupK;
    const bool okg = (format == B200_FMT_WNA16) ? (gk >= 32 && gk % 32 == 0 && H % gk == 0 && I % gk == 0)
                   : (format == B200_FMT_NVFP4) ? (gk == 16) : (gk == 32);
    if (!okg || cfg->groupN > 1) {
      set_error("b200moe_create: unsupported 4-bit group shape (WNA16: groupK multiple of 32, NVFP4: 16, MXFP4: 32; groupN 1)");
      return B200_ERR_INVALID;
    }
  }
  if (w4 && E > FUSED_MAX_EXPERTS) {
    set_error("b200moe_create: 4-bit formats support at most " + std::to_string(FUSED_MAX_EXPERTS) +
              " local experts per layer object (fused decode kernel tables)");
    return B200_ERR_INVALID;
  }
  // activation_type 1 reaches lk_moe for BOTH SwiGLU-OAI layouts (reference routed_experts.py:160-164 maps SWIGLUOAI,
  // gate/up rows interleaved as in gpt-oss, and SWIGLUOAI_UNINTERLEAVE, packed halves, to 1) and the weights arrive as
  // loaded.  The layout therefore has to be stated: B200MOE_SWIGLUOAI_LAYOUT=interleaved|packed.
  int interleaved = 0;
  if (cfg->activation_type == 1) {
    const char* lay = getenv("B200MOE_SWIGLUOAI_LAYOUT");
    if (lay && !strcmp(lay, "interleaved")) interleaved = 1;
    else if (lay && !strcmp(lay, "packed")) interleaved = 0;
    else {
      set_error("b200moe_create: activation_type 1 (SwiGLU-OAI) is ambiguous at the lk_moe boundary: set "
                "B200MOE_SWIGLUOAI_LAYOUT=interleaved (gpt-oss: gate = even rows, up = odd rows of w13) or =packed "
                "(rows [0,I) gate, [I,2I) up)");
      return B200_ERR_INVALID;
    }
    if (interleaved && format == B200_FMT_FP8) {
      set_error("b200moe_create: interleaved SwiGLU-OAI with block-FP8 weights is not supported (a 128-row scale block "
                "would straddle gate and up rows)");
      return B200_ERR_INVALID;
    }
    if (!cfg->has_gate_proj) {
      set_error("b200moe_create: activation_type 1 needs gated experts");
      return B200_ERR_INVALID;
    }
  }
  if (cfg->has_gate_proj && cfg->activation_type == 2) {
    set_error("b200moe_create: relu^2 (activation_type 2) is for non-gated experts");
    return B200_ERR_INVALID;
  }
  if (!cfg->has_gate_proj && cfg->activation_type != 2) {
    set_error("b200moe_create: non-gated experts need activation_type 2 (relu^2)");
    return B200_ERR_INVALID;
  }
  if (format == B200_FMT_FP8) {
    const int gN = cfg->groupN, gK = cfg->groupK;
    const bool okN = gN > 0 && (gN % 128 == 0);
    const bool okK = gK > 0 && (gK % 128 == 0);
    if (!okN || !okK) {
      set_error("b200moe_create: FP8 groupN/groupK must be multiples of 128 (block-128 or coarser scales)");
      return B200_ERR_INVALID;
    }
  }

  b200moe_layer* L = new b200moe_layer();
  L->cfg = *cfg;
  if (L->cfg.swiglu_alpha == 0.f) L->cfg.swiglu_alpha = 1.702f;
  if (L->cfg.swiglu_limit == 0.f) L->cfg.swiglu_limit = 7.0f;
  L->fmt = format;
  L->act_dtype = act_dtype;
  L->device = dev;
  L->E = E;
  L->H = H;
  L->I = I;
  L->gated = cfg->has_gate_proj ? 1 : 0;
  L->w13_interleaved = interleaved;
  L->N1 = L->gated ? 2 * I : I;
  L->esz_bits = (format == B200_FMT_FP8) ? 8 : 16;
  L->wq = (format == B200_FMT_WNA16) ? 1 : (format == B200_FMT_NVFP4) ? 2 : (format == B200_FMT_MXFP4) ? 3 : 0;
  L->w4_scale_bytes = (L->wq == 3) ? 256 : 512;
  L->w4_tile_bytes = 4096 + L->w4_scale_bytes;
  {
    // FP8 block-128 layers: B200MOE_FP8_E8M0=1 selects the reference's DeepGEMM ue8m0 numerics (power-of-two block
    // scales: weights re-quantised at ingest, activation group scales rounded up; VLLM_USE_DEEP_GEMM_E8M0, reference
    // vllm/envs.py:189).  Default: the checkpoint's fp32 scales, bit-for-bit the reference's CUTLASS / Triton block-FP8
    // semantics.
    const char* v = getenv("B200MOE_FP8_E8M0");
    L->fp8_e8m0 = (format == B200_FMT_FP8 && v && v[0] == '1' && cfg->groupN == 128 && cfg->groupK == 128) ? 1 : 0;
  }
  const int epk = (L->esz_bits == 8) ? 128 : 64;  // elements per 128-byte k-block
  L->KB1 = H / epk;
  L->KB2 = I / epk;
  L->J1 = I / 128;
  L->J2 = H / 128;
  L->w2_paired = (L->J2 % 2 == 0) ? 1 : 0;
  // one pass = the largest batch the workspace holds: decode batches (max_num_seqs) and, for the formats with a
  // large-batch GEMM path, prefill chunks of up to 8192 tokens (max_batch_size = max_num_batched_tokens) so that a
  // long prefill does not re-stream the expert weights once per decode-sized pass
  int mt = cfg->max_num_seqs > 0 ? cfg->max_num_seqs : 1;
  if (!w4 && cfg->max_batch_size > mt) mt = cfg->max_batch_size;
  if (mt < 16) mt = 16;
  if (mt > 8192) mt = 8192;
  if (w4 && mt > 256) mt = 256;   // 4-bit formats run through the fused decode kernel only: larger batches in passes
  L->max_tokens = mt;
  *out = L;
  return 0;
}

// raw (checkpoint-layout) bytes of ONE expert's tensors
struct RawSizes {
  int64_t w13, w2, s13, s2, g13, g2;
};
static RawSizes raw_sizes(const b200moe_layer* L) {
  RawSizes r{};
  const int64_t H = L->H, I = L->I, N1 = L->N1;
  if (L->wq) {
    const int gk = L->cfg.groupK;
    const int64_t sb = (L->fmt == B200_FMT_WNA16) ? 2 : 1;
    r.w13 = N1 * H / 2;
    r.w2 = H * I / 2;
    r.s13 = N1 * (H / gk) * sb;
    r.s2 = H * (I / gk) * sb;
    if (L->fmt == B200_FMT_NVFP4) {
      r.g13 = 2 * 4;
      r.g2 = 4;
    }
  } else {
    const int64_t esz = L->esz_bits / 8;
    r.w13 = N1 * H * esz;
    r.w2 = H * I * esz;
    if (L->fmt == B200_FMT_FP8) {
      const int gN = L->cfg.groupN, gK = L->cfg.groupK;
      r.s13 = ((N1 + gN - 1) / gN) * ((H + gK - 1) / gK) * 4;
      r.s2 = ((H + gN - 1) / gN) * ((I + gK - 1) / gK) * 4;
    }
  }
  return r;
}

// Ingest experts [e0, e0 + ne).  Host sources are staged through a per-layer device buffer in chunks of experts (the
// caller may free its tensors as soon as this returns — the lk_moe contract, routed_experts.py:1420-1432), each chunk
// re-tiled by the repack kernels straight into its final place: no full-size raw copy of the layer is ever held in HBM.
static int ingest_range(b200moe_layer* L, int e0, int ne, const void* w13, const void* w2, const void* s13, const void* s2,
                        const void* g13, const void* g2, int on_device) {
  const RawSizes rs = raw_sizes(L);
  cudaStream_t st = 0;
  cudaError_t e;
  auto repack = [&](int f0, int n, const void* a13, const void* a2, const void* b13, const void* b2, const void* c13,
                    const void* c2) {
    return L->wq ? repack_weights_w4(L, f0, n, a13, a2, b13, b2, c13, c2, st)
                 : repack_weights(L, f0, n, a13, a2, b13, b2, c13, c2, st);
  };
  if (on_device) {
    int rc = repack(e0, ne, w13, w2, s13, s2, g13, g2);
    if (rc) return rc;
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return cuda_fail(e, "repack sync");
    return 0;
  }
  const int64_t per = rs.w13 + rs.w2 + rs.s13 + rs.s2 + 256 * 4;
  int chunk = (int)((int64_t)(512ll << 20) / (per > 0 ? per : 1));   // <= 512 MB of raw tensors in flight
  if (chunk < 1) chunk = 1;
  if (chunk > ne) chunk = ne;
  uint8_t* stage = nullptr;
  if ((e = cudaMalloc(reinterpret_cast<void**>(&stage), (size_t)chunk * per)) != cudaSuccess) return cuda_fail(e, "cudaMalloc(ingest stage)");
  auto up = [](int64_t v) { return (v + 255) & ~int64_t(255); };
  int rc = 0;
  for (int c0 = 0; c0 < ne && !rc; c0 += chunk) {
    const int n = (ne - c0 < chunk) ? ne - c0 : chunk;
    uint8_t* p13 = stage;
    uint8_t* p2 = p13 + up(n * rs.w13);
    uint8_t* ps13 = p2 + up(n * rs.w2);
    uint8_t* ps2 = ps13 + up(n * rs.s13);
    auto h2d = [&](void* dst, const void* src, int64_t per_e, const char* what) {
      if (!per_e || !src || rc) return;
      cudaError_t ee = cudaMemcpyAsync(dst, reinterpret_cast<const uint8_t*>(src) + (int64_t)c0 * per_e, (size_t)n * per_e,
                                       cudaMemcpyHostToDevice, st);
      if (ee != cudaSuccess) rc = cuda_fail(ee, what);
    };
    h2d(p13, w13, rs.w13, "H2D w13");
    h2d(p2, w2, rs.w2, "H2D w2");
    h2d(ps13, s13, rs.s13, "H2D s13");
    h2d(ps2, s2, rs.s2, "H2D s2");
    if (rc) break;
    // NVFP4 global scales are copied by the repack itself (cudaMemcpyDefault handles host pointers)
    rc = repack(e0 + c0, n, p13, p2, rs.s13 ? ps13 : nullptr, rs.s2 ? ps2 : nullptr,
                g13 ? reinterpret_cast<const uint8_t*>(g13) + (int64_t)c0 * rs.g13 : nullptr,
                g2 ? reinterpret_cast<const uint8_t*>(g2) + (int64_t)c0 * rs.g2 : nullptr);
    if (!rc && (e = cudaStreamSynchronize(st)) != cudaSuccess) rc = cuda_fail(e, "ingest sync");   // the stage is reused
  }
  cudaFree(stage);
  return rc;
}

int b200moe_create(const b200moe_config* cfg, const void* w13, const void* w2, const void* w13_scale,
                   const void* w2_scale, const void* w13_global_scale, const void* w2_global_scale, int format,
                   int act_dtype, int weights_on_device, b200moe_handle* out) {
  if (!out) {
    set_error("b200moe_create: null output");
    return B200_ERR_INVALID;
  }
  b200moe_handle L = nullptr;
  int rc = b200moe_create_empty(cfg, format, act_dtype, &L);
  if (rc) return rc;
  rc = b200moe_load_experts(L, 0, L->E, w13, w2, w13_scale, w2_scale, w13_global_scale, w2_global_scale,
                            weights_on_device);
  if (!rc) rc = b200moe_finalize(L);
  if (rc) {
    b200moe_destroy(L);
    return rc;
  }
  *out = L;
  return 0;
}

int b200moe_load_experts(b200moe_handle h, int first_expert, int num_experts, const void* w13, const void* w2,
                         const void* w13_scale, const void* w2_scale, const void* w13_global_scale,
                         const void* w2_global_scale, int weights_on_device) {
  if (!h || h->finalized || !w13 || !w2 || first_expert < 0 || num_experts <= 0 || first_expert + num_experts > h->E) {
    set_error("b200moe_load_experts: bad handle / expert range (or the layer is already finalized)");
    return B200_ERR_INVALID;
  }
  if ((h->fmt != B200_FMT_16BIT && (!w13_scale || !w2_scale)) || (h->fmt == B200_FMT_NVFP4 && (!w13_global_scale || !w2_global_scale))) {
    set_error("b200moe_load_experts: this format needs scale tensors");
    return B200_ERR_INVALID;
  }
  int rc = ingest_range(h, first_expert, num_experts, w13, w2, w13_scale, w2_scale, w13_global_scale, w2_global_scale,
                        weights_on_device);
  if (!rc) h->experts_loaded += num_experts;
  return rc;
}

int b200moe_finalize(b200moe_handle h) {
  if (!h || h->finalized) {
    set_error("b200moe_finalize: bad handle");
    return B200_ERR_INVALID;
  }
  if (h->experts_loaded < h->E) {
    set_error("b200moe_finalize: only " + std::to_string(h->experts_loaded) + " of " + std::to_string(h->E) + " experts were loaded");
    return B200_ERR_INVALID;
  }
  // decode workspaces are allocated up front so that cpu_decode can run under stream capture
  Workspace* ws = get_workspace(h->device);
  int rc = ensure_workspace(ws, h, h->max_tokens, h->cfg.top_k, true);
  if (rc) return rc;
  {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    ++ws->live_layers;
    h->counted = 1;
  }
  h->finalized = 1;
  return 0;
}

int b200moe_destroy(b200moe_handle h) {
  if (!h) return 0;
  if (h->w13t) cudaFree(h->w13t);
  if (h->w2t) cudaFree(h->w2t);
  if (h->ws13) cudaFree(h->ws13);
  if (h->ws2) cudaFree(h->ws2);
  if (h->g13) cudaFree(h->g13);
  if (h->g2) cudaFree(h->g2);
  if (h->counted) {
    // the workspace (and the buffers CUDA graphs were captured against) goes with the device's last layer
    Workspace* ws = get_workspace(h->device);
    bool last = false;
    {
      std::lock_guard<std::mutex> lk(g_prof_mu);
      last = (--ws->live_layers == 0);
    }
    if (last) release_workspace(ws);
  }
  delete h;
  return 0;
}

int b200moe_query(b200moe_handle h, int what) {
  if (!h) return -1;
  switch (what) {
    case 0: return 0;                   // 1: MXFP4 runs a native block-scaled (W4A8-MX) kernel: not on this architecture
    case 1: return h->max_tokens;       // tokens per pass
    case 2: return h->w13_interleaved;
    case 3: return h->wq;
    case 4: return h->fp8_e8m0;         // 1: FP8 layer in ue8m0 (DeepGEMM) numerics
    default: return -1;
  }
}

int64_t b200moe_device_bytes(b200moe_handle h) { return h ? h->weight_bytes : 0; }

int b200moe_cpu_decode(b200moe_handle h, void* stream, int num_tokens, int top_k, const void* hidden,
                       const int32_t* topk_ids, const float* topk_weights, float* out_f32) {
  if (!h || !hidden || !topk_ids || !topk_weights || !out_f32) {
    set_error("b200moe_cpu_decode: null argument");
    return B200_ERR_INVALID;
  }
  return forward_device(h, reinterpret_cast<cudaStream_t>(stream), num_tokens, top_k, hidden, topk_ids,
                        topk_weights, out_f32, 2);
}

int b200moe_gpu_prefill(b200moe_handle h, const void* hidden, void* out, const int32_t* topk_ids,
                        const float* topk_weights, int num_tokens, int top_k, void* stream) {
  if (!h || !hidden || !topk_ids || !topk_weights || !out) {
    set_error("b200moe_gpu_prefill: null argument");
    return B200_ERR_INVALID;
  }
  return forward_device(h, reinterpret_cast<cudaStream_t>(stream), num_tokens, top_k, hidden, topk_ids,
                        topk_weights, out, h->act_dtype == B200_ACT_FP16 ? 1 : 0);
}

int b200moe_cpu_prefill(b200moe_handle h, int num_tokens, int top_k, const int32_t* ids_host,
                        const float* w_host, const void* hidden_host, float* out_host) {
  if (!h || !hidden_host || !ids_host || !w_host || !out_host) {
    set_error("b200moe_cpu_prefill: null argument");
    return B200_ERR_INVALID;
  }
  if (num_tokens <= 0) return 0;
  Workspace* ws = get_workspace(h->device);
  cudaError_t e;
  const int64_t M = num_tokens, H = h->H;
  int rc = grow_staging(ws, M * H, M * top_k);
  if (rc) return rc;
  // the caller has synchronised its stream (reference routed_experts.py:1866); the copies and kernels run on the
  // library's own non-blocking stream, ordered against eager calls of other streams by forward_device
  cudaStream_t st = nullptr;
  {
    std::lock_guard<std::mutex> lk(g_setup_mu);
    cudaStream_t& pst = g_prefill_stream[h->device];
    if (!pst && (e = cudaStreamCreateWithFlags(&pst, cudaStreamNonBlocking)) != cudaSuccess)
      return cuda_fail(e, "cudaStreamCreate(cpu_prefill)");
    st = pst;
  }
  wait_last_use(ws, st);   // staging buffers are shared too
  if ((e = cudaMemcpyAsync(ws->d_hidden, hidden_host, M * H * 2, cudaMemcpyHostToDevice, st)) != cudaSuccess) return cuda_fail(e, "H2D hidden");
  if ((e = cudaMemcpyAsync(ws->d_ids, ids_host, M * top_k * 4, cudaMemcpyHostToDevice, st)) != cudaSuccess) return cuda_fail(e, "H2D ids");
  if ((e = cudaMemcpyAsync(ws->d_w, w_host, M * top_k * 4, cudaMemcpyHostToDevice, st)) != cudaSuccess) return cuda_fail(e, "H2D weights");
  rc = forward_device(h, st, num_tokens, top_k, ws->d_hidden, ws->d_ids, ws->d_w, ws->d_out, 2);
  if (rc) return rc;
  if ((e = cudaMemcpyAsync(out_host, ws->d_out, M * H * 4, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return cuda_fail(e, "D2H out");
  if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return cuda_fail(e, "cpu_prefill sync");
  return 0;
}

int b200moe_profile(int enable) {
  g_profile = enable != 0;
  g_events_used = 0;
  return 0;
}

int b200moe_profile_read(double* gemm1_ms, double* gemm2_ms, int64_t* calls) {
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return cuda_fail(e, "profile_read sync");
  double a = 0, b = 0;
  for (size_t i = 0; i < g_events_used; ++i) {
    float t = 0;
    cudaEventElapsedTime(&t, g_events[i].e[0], g_events[i].e[1]);
    a += t;
    if (g_events[i].fused) continue;
    cudaEventElapsedTime(&t, g_events[i].e[1], g_events[i].e[2]);
    b += t;
  }
  if (gemm1_ms) *gemm1_ms = a;
  if (gemm2_ms) *gemm2_ms = b;
  if (calls) *calls = (int64_t)g_events_used;
  g_events_used = 0;
  return 0;
}

int b200moe_debug_read(int what, void* dst_host, int64_t bytes) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return B200_ERR_NO_DEVICE;
  Workspace* ws = get_workspace(dev);
  const void* src = nullptr;
  switch (what) {
    case 0: src = ws->xt; break;
    case 1: src = ws->xs; break;
    case 2: src = ws->it; break;
    case 3: src = ws->is; break;
    case 4: src = ws->y; break;
    case 5: src = ws->state; break;
    case 6: src = ws->chunks; break;
    case 7: src = ws->row_of_slot; break;
    case 8: src = ws->slot_of_row; break;
    default: break;
  }
  if (!src || !dst_host || bytes <= 0) {
    set_error("b200moe_debug_read: bad argument / workspace not allocated");
    return B200_ERR_INVALID;
  }
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return cuda_fail(e, "debug_read sync");
  if ((e = cudaMemcpy(dst_host, src, bytes, cudaMemcpyDeviceToHost)) != cudaSuccess) return cuda_fail(e, "debug_read copy");
  return 0;
}

}  // extern "C"
