// Byte order inside one 4-bit weight tile: [128 rows x 64 columns] of one k-block, 4096 B of nibbles followed by the
// scales.  The fused decode kernel's two consumer warpgroups read a tile straight into wgmma A fragments, so the tile is
// stored in their fragment order.  This header is the one place that maps (row, column) to (word, nibble) and (row,
// group) to a scale byte; the ingest (tile_w4_kernel, tile_w4_scales_kernel), the prefill expansion
// (dequant_w4_tiles_kernel) and the consumers (moe_fused.cu) all follow it.
//
// Nibbles: consumer thread u = (warpgroup half h, warp w, lane l) = (h * 4 + w) * 32 + l owns the 16 bytes at u * 16.  Its
// word ks holds the 8 values of its A fragment of k16 slice ks: rows R0 = 64h + 16w + l / 4 and R0 + 8, columns
// 16 ks + {2t, 2t + 1, 2t + 8, 2t + 9} (t = l % 4).  Fragment register `reg` (0: row R0, columns 2t, 2t + 1;
// 1: row R0 + 8, same columns; 2 and 3: the same rows at columns 2t + 8, 2t + 9) takes half e (the column's parity) from
//   int4:  nibble reg + 4e.  (w & 0x000F000F) and (w & 0x00F000F0), then the same after w >> 8, give registers 0-3 as
//          fp16 pairs 1024 + q and 1024 + 16q once 0x6400 is OR-ed in (Marlin-style).
//   e2m1:  exponent-mantissa field at bit 16e + {9, 6, 0, 3}[reg], sign at bit 16e + {15, 12, 13, 14}[reg].  Register 0
//          is w & 0x8E008E00, register 1 (w << 3) & 0x8E008E00: field and sign already sit where an fp16 of value
//          * 2^-14 has them.  Registers 2 and 3 take the field and the sign with one shift each.
// Scales: one record per (h, w, l / 4), i.e. per thread quad, at 4096 + (u / 4) * record bytes.  It holds the scales of
// rows R0 and R0 + 8 for every group of the k-block, group-major, row R0 first: int4 4 x fp16 (8 B), nvfp4 8 x e4m3
// (8 B), mxfp4 4 x e8m0 (4 B).  A (R0, R0 + 8) pair is then one fp16x2 (int4) or one e4m3x2 (nvfp4).
#pragma once
#include <stdint.h>

namespace b200 {

constexpr int W4_NIBBLE_BYTES = 4096;

// nibble word (0..1023) that holds weight (r, c), the fragment register within it, and back
__host__ __device__ inline int w4_word(int r, int c) {
  return ((r >> 4) * 32 + (r & 7) * 4 + ((c >> 1) & 3)) * 4 + (c >> 4);
}
__host__ __device__ inline int w4_reg(int r, int c) { return ((r >> 3) & 1) | ((c >> 2) & 2); }
__host__ __device__ inline int w4_row(int word, int reg) {
  const int u = word >> 2;
  return (u >> 5) * 16 + ((u >> 2) & 7) + (reg & 1) * 8;
}
__host__ __device__ inline int w4_col(int word, int reg, int e) {
  return (word & 3) * 16 + ((word >> 2) & 3) * 2 + (reg >> 1) * 8 + e;
}

// the bits of 4-bit code v (int4: the unsigned code; e2m1: sign in bit 3) at half e of register reg, and back
__host__ __device__ inline uint32_t w4_code_bits(bool e2m1, int reg, int e, uint32_t v) {
  if (!e2m1) return (v & 0xFu) << (4 * (reg + 4 * e));
  const int field = (reg == 0 ? 9 : reg == 1 ? 6 : reg == 2 ? 0 : 3) + 16 * e;
  const int sign = (reg == 0 ? 15 : reg == 1 ? 12 : reg == 2 ? 13 : 14) + 16 * e;
  return ((v & 7u) << field) | (((v >> 3) & 1u) << sign);
}
__host__ __device__ inline uint32_t w4_code(bool e2m1, int reg, int e, uint32_t word) {
  if (!e2m1) return (word >> (4 * (reg + 4 * e))) & 0xFu;
  const int field = (reg == 0 ? 9 : reg == 1 ? 6 : reg == 2 ? 0 : 3) + 16 * e;
  const int sign = (reg == 0 ? 15 : reg == 1 ? 12 : reg == 2 ? 13 : 14) + 16 * e;
  return ((word >> field) & 7u) | (((word >> sign) & 1u) << 3);
}

// byte offset, within the scale area, of the scale of row r and group g (wq 1 int4 / 3 mxfp4: 32 columns, g < 2;
// wq 2 nvfp4: 16 columns, g < 4)
__host__ __device__ inline int w4_scale_record_bytes(int wq) { return wq == 3 ? 4 : 8; }
__host__ __device__ inline int w4_scale_off(int wq, int r, int g) {
  const int rec = (r >> 4) * 8 + (r & 7), pos = g * 2 + ((r >> 3) & 1);
  return rec * w4_scale_record_bytes(wq) + pos * (wq == 1 ? 2 : 1);
}

}  // namespace b200
