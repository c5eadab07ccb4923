// e4m3 quantisation rule of the fp8 inference path (shared by the LayerNorm, the quantise kernel and the weight preparation).
// One scale per row (activations) or per output channel (weights), amax = max |x| of the row in fp32:
//   q = e4m3_satfinite(x * (448 / amax)),  s = amax / 448,  both divisions IEEE;  amax < 2^-119 (zero rows included) gives
//   q = 0, s = 0.
// x * (448 / amax) never reaches 464 in magnitude, so the CPU oracle (x.float() * (448.0 / amax)).to(torch.float8_e4m3fn)
// (which gives NaN instead of saturating there) is bit-exact against it.
#pragma once
#include <cuda_fp8.h>
#include <stdint.h>

namespace b200 {

// A row whose amax is below 2^-119 counts as zero (q = 0, s = 0): 448 / amax would overflow to +inf below about 1.3e-36 (bf16
// subnormal rows, for instance), and 0 * inf would put NaN into the row.
constexpr float kFp8MinAmax = 0x1p-119f;
__device__ __forceinline__ float fp8_row_rinv(float amax) { return amax >= kFp8MinAmax ? __fdiv_rn(448.0f, amax) : 0.f; }
__device__ __forceinline__ float fp8_row_scale(float amax) { return amax >= kFp8MinAmax ? __fdiv_rn(amax, 448.0f) : 0.f; }

// Two values -> two e4m3 bytes (a in the low byte), zero-extended to 32 bits.  Inline PTX with an explicit 16-bit result: built on
// __nv_cvt_float2_to_fp8x2, the compiler packed two conversions into one register with F2FP.PACK_AB_MERGE_C and left the upper
// half of a row of zeros holding stale register contents.
__device__ __forceinline__ uint32_t fp8x2(float a, float b, float rinv) {
  uint32_t out;
  asm("{\n\t.reg .b16 t;\n\tcvt.rn.satfinite.e4m3x2.f32 t, %1, %2;\n\tcvt.u32.u16 %0, t;\n\t}"
      : "=r"(out)
      : "f"(__fmul_rn(b, rinv)), "f"(__fmul_rn(a, rinv)));
  return out;
}
// four values -> four e4m3 bytes, v[0] in the lowest byte (memory order)
__device__ __forceinline__ uint32_t fp8x4(const float* v, float rinv) {
  return fp8x2(v[0], v[1], rinv) | (fp8x2(v[2], v[3], rinv) << 16);
}

}  // namespace b200
