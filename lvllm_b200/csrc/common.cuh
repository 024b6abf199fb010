// Common device helpers for the sm_90a kernels: mbarrier, 1-D bulk async copies (UBLKCP), wgmma operand
// descriptors, the accumulator exchange area and small utilities.  Hand-written inline PTX; no CUTLASS dependency.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "wgmma.cuh"

namespace b200 {

#define B200_DEVICE __device__ __forceinline__

B200_DEVICE uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

B200_DEVICE bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t.reg .b32 R;\n\t"
      "elect.sync R|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------- mbarrier
B200_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
B200_DEVICE void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
B200_DEVICE void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

B200_DEVICE void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
B200_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
B200_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
B200_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------- bulk copy (TMA 1-D)
// global -> shared, completion signalled on an mbarrier as transaction bytes.  size % 16 == 0,
// both addresses 16-B aligned.  SASS: UBLKCP.
B200_DEVICE void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// same with an L2 eviction-priority hint (created with createpolicy)
B200_DEVICE void bulk_g2s_hint(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
          "r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
      : "memory");
}
// 2-D tensor-map copy (TMA tile mode, SASS: UTMALDG): box at element coordinate (c0, c1) -> shared memory, completion
// as transaction bytes on an mbarrier.  `tmap` points at a CUtensorMap in the kernel parameter space (__grid_constant__).
B200_DEVICE void tma_load_2d_hint(void* smem_dst, const void* tmap, int c0, int c1, uint64_t* bar, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%2, %3}], [%4], %5;" ::"r"(smem_u32(smem_dst)),
      "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar)), "l"(pol)
      : "memory");
}
B200_DEVICE uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
B200_DEVICE uint64_t policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// ----------------------------------------------------------------------------- cp.async (LDGSTS)
// 16-byte global -> shared copy without register staging; src_size 0 zero-fills the destination.
B200_DEVICE void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  const uint32_t sz = valid ? 16u : 0u;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(sz)
               : "memory");
}
// 8-byte variant (LDGSTS.64): used to spread packed 4-bit data over 16-byte chunks
B200_DEVICE void cp_async8(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
// the mbarrier receives one (pre-counted) arrival when all prior cp.async of this thread have landed
B200_DEVICE void cp_async_mbar_arrive_noinc(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// ----------------------------------------------------------------------------- wgmma operands
// Shared-memory matrix descriptor, K-major operand with 128-byte swizzle.  Rows are 128 B, groups of
// 8 rows form a 1024-B swizzle atom; SBO = distance between consecutive 8-row groups.
// Bit layout (sm_90): [0,14) addr>>4, [16,30) LBO>>4, [32,46) SBO>>4, [49,52) base offset, [62,64) swizzle (1 = 128 B).
// An M = 64 instruction reads 64 rows from the start address: the lower half of a 128-row tile starts 8 KB in.
B200_DEVICE uint64_t wgmma_desc_sw128(uint32_t smem_addr, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// MN-major, 128B-swizzled operand: atoms of 64 elements (128 B) along MN x 8 rows along K.
// LBO = byte distance between 64-element atoms along MN, SBO = byte distance between 8-row groups along K.
B200_DEVICE uint64_t wgmma_desc_sw128_mn(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return wgmma_desc_sw128(smem_addr, sbo_bytes) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16);
}

// ----------------------------------------------------------------------------- accumulator exchange
// wgmma leaves the accumulators in the registers of the warpgroup that issued it, spread over the threads in the
// fragment layout of wgmma.cuh.  The kernels keep the MMA warpgroup apart from the warps that post-process a tile
// (thread = tile row, a run of consecutive columns), so finished accumulators cross over through a shared-memory
// area of fp32 [column][128 rows].  An address is one word: bits [24,32) area base >> 10 (1 KB aligned), bits [16,24)
// first row of the accessing warp, bits [0,16) column — so `base + (row0 << 16) + column` arithmetic works on it.
// Rows are XOR-swizzled with the column so that both the fragment stores and the row-wise loads are conflict-free.
B200_DEVICE uint32_t xch_base(const void* area) { return (smem_u32(area) >> 10) << 24; }
B200_DEVICE uint32_t xch_addr(uint32_t x, uint32_t row, uint32_t col) {
  col += x & 0xFFFFu;
  row += (x >> 16) & 0xFFu;
  return ((x >> 24) << 10) + ((col << 7) + (row ^ (((col >> 1) & 3u) << 3))) * 4u;
}
// the MMA warpgroup parks one 64-row accumulator fragment (rows [64 * half, +64), columns [col0, col0 + N))
template <int N>
B200_DEVICE void xch_store_frag(uint32_t x, int half, const float* d) {
  const uint32_t w = (threadIdx.x >> 5) & 3u, l = threadIdx.x & 31u;
  const uint32_t row = half * 64 + w * 16 + (l >> 2);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const uint32_t col = j * 8 + (l & 3u) * 2;
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(xch_addr(x, row, col)), "f"(d[4 * j]) : "memory");
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(xch_addr(x, row, col + 1)), "f"(d[4 * j + 1]) : "memory");
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(xch_addr(x, row + 8, col)), "f"(d[4 * j + 2]) : "memory");
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(xch_addr(x, row + 8, col + 1)), "f"(d[4 * j + 3]) : "memory");
  }
}
// row-wise access: the thread's row is the address's first row + its lane; NC consecutive columns
template <int NC>
B200_DEVICE void xch_ld(uint32_t x, float* v) {
  const uint32_t lane = threadIdx.x & 31u;
#pragma unroll
  for (int c = 0; c < NC; ++c) asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v[c]) : "r"(xch_addr(x, lane, c)) : "memory");
}
template <int NC>
B200_DEVICE void xch_st(uint32_t x, const float* v) {
  const uint32_t lane = threadIdx.x & 31u;
#pragma unroll
  for (int c = 0; c < NC; ++c) asm volatile("st.shared.f32 [%0], %1;" ::"r"(xch_addr(x, lane, c)), "f"(v[c]) : "memory");
}

// D[128 x N] (+)= A[128 x K] * B[K x N] for one 128-byte k-slice of K-major, 128B-swizzled tiles: two M = 64 instructions;
// acc[0] holds rows [0,64), acc[1] rows [64,128)
template <int N, int KIND>
B200_DEVICE void wgmma_tile128(float (*acc)[N / 2], uint32_t a_addr, uint32_t b_addr, uint32_t accumulate) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
    WgmmaSS<N, KIND>::mma(acc[h], wgmma_desc_sw128(a_addr + h * 8192, 1024), wgmma_desc_sw128(b_addr, 1024), accumulate);
}

// per-token-group FP8 activation scale (reference fp8_utils.py:100-113): absmax / 448, rounded UP to a power of two in
// ue8m0 mode (exp2(ceil(log2(.))), the DeepGEMM ue8m0 convention)
B200_DEVICE float fp8_group_scale(float absmax, int e8m0) {
  float sc = fmaxf(absmax, 1e-10f) / 448.0f;
  if (e8m0) {
    const uint32_t b = __float_as_uint(sc);
    sc = __uint_as_float(((b >> 23) + ((b & 0x7FFFFFu) ? 1u : 0u)) << 23);
  }
  return sc;
}

// ----------------------------------------------------------------------------- register reallocation
// Every warp of a warpgroup executes the same one.  `inc` blocks until other warpgroups have released enough registers
// with `dec`: the sum over the CTA must stay within what the launch allocated (registers of the kernel x threads).
template <int R>
B200_DEVICE void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
B200_DEVICE void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// ----------------------------------------------------------------------------- misc
B200_DEVICE float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
B200_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

B200_DEVICE int ld_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
B200_DEVICE void red_release_add(int* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Byte offset of logical element (row r, byte b of a 128-B K segment) inside a [rows x 128 B] K-major
// tile stored with the 128-byte swizzle (16-B chunk index XOR row%8), 8-row groups of 1024 B.
__host__ __device__ inline uint32_t sw128_offset(uint32_t r, uint32_t b) {
  return (r >> 3) * 1024u + (r & 7u) * 128u + ((((b >> 4) ^ (r & 7u)) & 7u) << 4) + (b & 15u);
}

// smallest power of two >= x for a positive normal float, from the exponent bits (the reference's exp2(ceil(log2(x))) of
// the ue8m0 scale format, without the rounding of an fp32 log2 just above a power of two)
B200_DEVICE float ue8m0_ceil(float x) {
  const uint32_t b = __float_as_uint(x);
  return __uint_as_float(((b >> 23) + ((b & 0x7FFFFFu) ? 1u : 0u)) << 23);
}

}  // namespace b200
