// Epilogue helpers of the persistent 128 x 256 GEMM kernels: the bf16 ones (gemm.cuh: gemm_ws_kernel, gemm_ws_wgrad_kernel) and
// the e4m3 one (fp8.cu: gemm_fp8_kernel) stage their accumulators through the same swizzled buffer layout.
#pragma once
#include "ptx.cuh"

namespace b200 {

__device__ __forceinline__ void add_bf16x4(float* v, uint2 w) {
  const float2 f0 = unpack_bf16x2(w.x), f1 = unpack_bf16x2(w.y);
  v[0] += f0.x; v[1] += f0.y; v[2] += f1.x; v[3] += f1.y;
}
__device__ __forceinline__ uint2 pack_bf16x4(const float* v) { return make_uint2(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3])); }

// Epilogue staging of the 128 x 256 kernels.  Columns 64 j .. 64 j + 63 of a consumer warpgroup's m64n256 accumulators go into
// its 64 x 64 fp32 buffer, XOR-swizzled (column ^ 8 (row & 3)) so that both the fragment stores and the row-segment loads are
// free of bank conflicts.  Warp w then reads rows 16 w + 2 i + lane / 16 (i = 0..7), 4 columns (ws_lane_col) per lane.
__device__ __forceinline__ void ws_stage_chunk(const float* acc, float* stage, int j, int w, int lane) {
#pragma unroll
  for (int i = 32 * j; i < 32 * j + 32; i += 2) {
    const int r = 16 * w + (lane >> 2) + 8 * ((i >> 1) & 1);
    const int cc = 8 * ((i >> 2) - 8 * j) + 2 * (lane & 3);
    *reinterpret_cast<float2*>(stage + r * 64 + (cc ^ ((r & 3) << 3))) = make_float2(acc[i], acc[i + 1]);
  }
}
__device__ __forceinline__ int ws_lane_col(int lane) { return 4 * (lane & 15); }
__device__ __forceinline__ int ws_chunk_row(int w, int i, int lane) { return 16 * w + 2 * i + (lane >> 4); }
__device__ __forceinline__ float4 ws_load_row(const float* stage, int r, int cq) {
  return *reinterpret_cast<const float4*>(stage + r * 64 + (cq ^ ((r & 3) << 3)));
}

}  // namespace b200
