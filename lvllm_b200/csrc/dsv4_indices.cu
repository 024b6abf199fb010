// The global key lists of DeepSeek-V4 decode: the cache slots that b200_dsv4_sparse_decode attends over and the compressed
// slot that b200_dsv4_compress writes, from each token's position and its request's row of a block table.  One kernel,
// one instantiation per list kind:
//   DS_IDX_SWA      sliding window [max(p - W + 1, 0), p] into the SWA cache (_compute_swa_indices_and_lens_kernel,
//                   v1/attention/backends/mla/sparse_swa.py:744-800, with p taken from positions);
//   DS_IDX_C128A    every compressed row [0, min((p + 1) / ratio, width)) (the decode branch of
//                   _build_c128a_topk_metadata_kernel, models/deepseek_v4/sparse_mla.py:353-408);
//   DS_IDX_TOPK     the indexer's request-local top-k -> global slots, length = entries >= 0
//                   (_compute_global_topk_indices_and_lens_kernel, common/ops/cache_utils.py:477-525);
//   DS_IDX_SLOTMAP  the compressor's slot: compressed row p / ratio where (p + 1) % ratio == 0, else -1
//                   (_compressed_slot_mapping_kernel, v1/attention/backends/mla/compressor_utils.py:8-50).
// Local index i of a request lies at block_table[req][i / bs] * bs + i % bs.  A column i / bs at or past the table's width
// (max_blocks) is no key (-1): the reference would read past the row there.  Entries past a list's length are -1; a token
// with slot_mapping < 0 gets length 0 and a row of -1, and its request row is never read.
#include "common.cuh"
#include "moe_internal.cuh"

namespace b200 {

constexpr int DS_IDX_SWA = 0, DS_IDX_C128A = 1, DS_IDX_TOPK = 2, DS_IDX_SLOTMAP = 3;
constexpr int IX_THREADS = 256;

struct IndicesArgs {
  const int64_t* positions;      // [T]; not read by TOPK
  const int64_t* slot_mapping;   // [T]; < 0: padded token
  const int32_t* token_to_req;   // [T] rows of block_table
  const int32_t* block_table;    // [*, bt_stride], the first max_blocks columns used
  int64_t bt_stride;
  int max_blocks, block_size;
  int param;                     // SWA: the window; C128A / SLOTMAP: the compression ratio
  const int32_t* local;          // TOPK: [T, local_stride] request-local indices
  int64_t local_stride;
  void* out;                     // int32 [T, out_stride] lists; SLOTMAP: int64 [T]
  int64_t out_stride;
  int width;                     // list columns written
  int32_t* lens;                 // [T]
  int T;
};

B200_DEVICE int64_t ix_global(const IndicesArgs& a, const int32_t* bt, int64_t i) {
  if (i < 0) return -1;
  const int64_t col = i / a.block_size;
  return col < a.max_blocks ? (int64_t)bt[col] * a.block_size + i % a.block_size : -1;
}

// SLOTMAP: one thread per token.  The lists: one CTA per token, columns strided over the CTA.
template <int KIND>
__global__ void __launch_bounds__(IX_THREADS) dsv4_indices_kernel(const __grid_constant__ IndicesArgs a) {
  if constexpr (KIND == DS_IDX_SLOTMAP) {
    const int t = blockIdx.x * IX_THREADS + threadIdx.x;
    if (t >= a.T) return;
    const int64_t p = a.positions[t];
    int64_t s = -1;
    if (a.slot_mapping[t] >= 0 && p >= 0 && (p + 1) % a.param == 0)
      s = ix_global(a, a.block_table + (int64_t)a.token_to_req[t] * a.bt_stride, p / a.param);
    reinterpret_cast<int64_t*>(a.out)[t] = s;
  } else {
    const int t = blockIdx.x;
    const bool valid = a.slot_mapping[t] >= 0;
    const int32_t* bt = valid ? a.block_table + (int64_t)a.token_to_req[t] * a.bt_stride : nullptr;
    int64_t start = 0, len = 0;
    const int64_t p = KIND == DS_IDX_TOPK ? 0 : a.positions[t];
    if (KIND == DS_IDX_SWA) {
      start = max(p - a.param + 1, (int64_t)0);
      len = max(p + 1 - start, (int64_t)0);
    } else if (KIND == DS_IDX_C128A) {
      len = p < 0 ? 0 : min((p + 1) / a.param, (int64_t)a.width);
    }
    int32_t* o = reinterpret_cast<int32_t*>(a.out) + (int64_t)t * a.out_stride;
    const int32_t* loc = KIND == DS_IDX_TOPK ? a.local + (int64_t)t * a.local_stride : nullptr;
    int count = 0;
    for (int j0 = 0; j0 < a.width; j0 += IX_THREADS) {   // uniform trip count: the top-k count syncs the CTA
      const int j = j0 + threadIdx.x;
      int64_t li = -1;
      if (KIND == DS_IDX_TOPK) {
        if (j < a.width) li = loc[j];
        count += __syncthreads_count(li >= 0);
      } else if (j < len) {
        li = start + j;
      }
      if (j < a.width) o[j] = valid ? (int32_t)ix_global(a, bt, li) : -1;
    }
    if (KIND == DS_IDX_TOPK) len = count;
    if (threadIdx.x == 0) a.lens[t] = valid ? (int32_t)len : 0;
  }
}

static bool al(const void* p, int n) { return p && reinterpret_cast<uintptr_t>(p) % n == 0; }

}  // namespace b200

using namespace b200;

extern "C" {

int b200_dsv4_indices(void* stream, int kind, const int64_t* positions, const int64_t* slot_mapping,
                      const int32_t* token_to_req, const int32_t* block_table, int64_t block_table_stride, int max_blocks,
                      int block_size, int param, const int32_t* local_topk, int64_t local_stride, void* out,
                      int64_t out_stride, int width, int32_t* lens, int num_tokens) {
  const bool list = kind != DS_IDX_SLOTMAP;
  bool ok = kind >= DS_IDX_SWA && kind <= DS_IDX_SLOTMAP && (kind == DS_IDX_TOPK || al(positions, 8)) &&
            al(slot_mapping, 8) && al(token_to_req, 4) && al(block_table, 4) && max_blocks >= 1 &&
            block_table_stride >= max_blocks && block_size >= 1 && num_tokens >= 0 && num_tokens <= (1 << 20) &&
            al(out, list ? 4 : 8);
  if (ok && list) ok = al(lens, 4) && width >= 1 && width <= (1 << 20) && out_stride >= width;
  if (ok && kind == DS_IDX_SWA) ok = param >= 1 && width >= param;
  if (ok && (kind == DS_IDX_C128A || kind == DS_IDX_SLOTMAP)) ok = param == 4 || param == 128;
  if (ok && kind == DS_IDX_TOPK) ok = al(local_topk, 4) && local_stride >= width;
  if (!ok) {
    set_error("b200_dsv4_indices: bad argument (kind 0-3; positions, slot_mapping 8-byte and token_to_req, block_table "
              "4-byte aligned; 1 <= max_blocks <= block_table_stride, block_size >= 1, 0 <= num_tokens <= 2^20; lists: "
              "lens, 1 <= width <= min(out_stride, 2^20), SWA window 1..width, ratio 4 or 128, top-k local_stride >= "
              "width)");
    return B200_ERR_INVALID;
  }
  if (num_tokens == 0) return 0;
  const IndicesArgs a{positions, slot_mapping, token_to_req, block_table, block_table_stride, max_blocks, block_size,
                      param, local_topk, local_stride, out, out_stride, width, lens, num_tokens};
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (kind) {
    case DS_IDX_SWA: dsv4_indices_kernel<DS_IDX_SWA><<<num_tokens, IX_THREADS, 0, st>>>(a); break;
    case DS_IDX_C128A: dsv4_indices_kernel<DS_IDX_C128A><<<num_tokens, IX_THREADS, 0, st>>>(a); break;
    case DS_IDX_TOPK: dsv4_indices_kernel<DS_IDX_TOPK><<<num_tokens, IX_THREADS, 0, st>>>(a); break;
    default:
      dsv4_indices_kernel<DS_IDX_SLOTMAP><<<(num_tokens + IX_THREADS - 1) / IX_THREADS, IX_THREADS, 0, st>>>(a);
  }
  ++g_launches;
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "dsv4_indices launch");
  return 0;
}

}  // extern "C"
