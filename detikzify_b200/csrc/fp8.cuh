// e4m3 weight codes of the FP8 decode tiles (launch_retile_f8), shared by the tile builder and the two kernels that read
// them: the batch-1 persistent decode kernel (decode_mega.cu) and the batched-decode swapped-operand GEMM (gemm_tc.cu).
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "launch.h"

namespace dtk {

// two e4m3 codes (low 16 bits of v: low byte = first element) -> their values (exact in fp32)
DTK_DEV float2 e4m3x2_to_float2(uint32_t v) {
  uint32_t h;
  asm("{\n\t.reg .b16 t;\n\tcvt.u16.u32 t, %1;\n\tcvt.rn.f16x2.e4m3x2 %0, t;\n\t}\n" : "=r"(h) : "r"(v));
  return __half22float2(*reinterpret_cast<const __half2*>(&h));
}
// the bf16 pair of an A fragment: two codes times the row scale 2^k_r (exact: the product is a bf16 value)
DTK_DEV uint32_t e4m3x2_to_bf16x2(uint32_t v, float scale) {
  const float2 f = e4m3x2_to_float2(v);
  return pack_bf16x2(f.x * scale, f.y * scale);
}
// (a, b) -> two e4m3 codes (round to nearest even, saturating), a in the low byte
DTK_DEV uint32_t float2_to_e4m3x2(float a, float b) {
  uint16_t d;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;\n" : "=h"(d) : "f"(b), "f"(a));
  return d;
}
DTK_DEV float pow2f(int k) { return __uint_as_float((uint32_t)(k + 127) << 23); }   // k in [-126, 127]

// source row of A-operand row ar (0..15) of tile group gi (the decode tiles' row permutation)
// TILE_ROPE: head blocks of hd rows; group gi holds pair rows (i, i + hd/2) for i in 8 consecutive values
DTK_DEV int tile_row(int mode, int hd, int gi, int ar) {
  if (mode == TILE_SEQ) return gi * 16 + ar;
  if (mode == TILE_ROPE) {
    const int gph = hd / 16;   // groups per head block
    return (gi / gph) * hd + ((gi % gph) << 3) + (ar & 7) + (ar >> 3) * (hd / 2);
  }
  return (ar < 8) ? 2 * (gi * 8 + ar) : 2 * (gi * 8 + ar - 8) + 1;  // source rows are interleaved (gate, up)
}

}  // namespace dtk
